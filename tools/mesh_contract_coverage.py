#!/usr/bin/env python
"""Coverage of meshes extracted in world and in contracted space (Config.mesh_space) on an unbounded scene.

Writes a procedural unbounded scene in the Blender format: a shaded sphere of radius 0.35 at the origin inside a
checkered room (the box |x|_inf <= 6), rendered in closed form from cameras inside the unit ball that look outward
and across the room.  Trains a small model on it with the scene contraction on both MLPs (reciprocal ray distances,
as 360.gin), then runs extract_mesh.py with Config.mesh_eval in both spaces at the same resolution and level, and
prints one JSON line: each space's mean coverage (the fraction of the test pixels the NeRF sees, acc >= 0.5, that the
mesh hits), depth_abs_rel, face count and extraction summary, with the card's name and power limit.

  python tools/mesh_contract_coverage.py [--steps 2000] [--resolution 256] [--level 10] [--out result.json]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SPHERE_R, ROOM = 0.35, 6.0


def _trace(o, d):
  """Closed-form first hit of rays o + t d (d unit) in the scene -> (t, rgb)."""
  b = (o * d).sum(-1)
  c = (o * o).sum(-1) - SPHERE_R ** 2
  disc = b * b - c
  ts = np.where(disc >= 0, -b - np.sqrt(np.maximum(disc, 0)), np.inf)
  ts = np.where(ts > 0, ts, np.inf)
  with np.errstate(divide='ignore'):
    tw = np.min(np.where(d != 0, (np.sign(d) * ROOM - o) / d, np.inf), -1)       # exit of the room's box
  sphere = ts < tw
  t = np.where(sphere, ts, tw)
  p = o + t[:, None] * d
  n = p / SPHERE_R
  shade = 0.25 + 0.75 * np.clip(n @ np.array([0.3, 0.5, 0.81]), 0, 1)
  rgb_s = np.stack([0.9 * shade, 0.45 * shade, 0.2 * shade], -1)
  check = (np.floor(p[:, 0]) + np.floor(p[:, 1]) + np.floor(p[:, 2])) % 2
  axis = np.abs(p).argmax(-1)
  base = np.array([[0.2, 0.5, 0.9], [0.3, 0.8, 0.3], [0.85, 0.85, 0.8]])[axis]
  rgb_w = base * (0.55 + 0.45 * check[:, None])
  return t, np.where(sphere[:, None], rgb_s, rgb_w)


def write_scene(root, n_train=60, n_test=4, W=96, H=72, seed=0):
  """The scene as Blender-format transforms and PNGs under `root` (train and test splits)."""
  from PIL import Image
  from multinerf_b200 import camera_utils
  rng = np.random.default_rng(seed)
  angle_x = 1.2
  focal = .5 * W / math.tan(.5 * angle_x)
  p2c = camera_utils.get_pixtocam(focal, W, H)
  for split, n in (('train', n_train), ('test', n_test)):
    os.makedirs(os.path.join(root, split), exist_ok=True)
    frames = []
    for i in range(n):
      a = 2 * math.pi * (i + (0.5 if split == 'test' else 0.0)) / n
      eye = np.array([0.8 * math.cos(a), 0.8 * math.sin(a), 0.15 * math.sin(3 * a)])
      # look across the room past the sphere: a target on the far side, off the centre line
      target = -eye * rng.uniform(2, 6) + rng.normal(size=3) * np.array([1.5, 1.5, 0.8])
      z = eye - target
      z /= np.linalg.norm(z)
      x = np.cross([0, 0, 1.0], z)
      x /= np.linalg.norm(x)
      c2w = np.eye(4)
      c2w[:3, :4] = np.concatenate([np.stack([x, np.cross(z, x), z], 1), eye[:, None]], 1)
      # pixel centres through the inverse intrinsics, OpenCV -> OpenGL flip, then the pose (camera_utils' rays)
      xs, ys = np.meshgrid(np.arange(W) + 0.5, np.arange(H) + 0.5)
      dc = np.stack([xs, ys, np.ones_like(xs)], -1).reshape(-1, 3) @ np.asarray(p2c, np.float64).T
      d = (dc * np.array([1.0, -1.0, -1.0])) @ c2w[:3, :3].T
      v = d / np.linalg.norm(d, axis=-1, keepdims=True)
      _, rgb = _trace(np.broadcast_to(eye, v.shape), v)
      rgba = np.concatenate([rgb.reshape(H, W, 3), np.ones((H, W, 1))], -1)
      Image.fromarray((rgba * 255 + 0.5).astype(np.uint8)).save(os.path.join(root, split, f'r_{i}.png'))
      frames.append({'file_path': f'./{split}/r_{i}', 'transform_matrix': c2w.tolist()})
    with open(os.path.join(root, f'transforms_{split}.json'), 'w') as f:
      json.dump({'camera_angle_x': angle_x, 'frames': frames}, f)


def train_bindings(data, ckpt, steps):
  """A small model under the scene contraction (both MLPs), reciprocal ray distances, near 0.05, far 1e6."""
  return [f"Config.data_dir = '{data}'", f"Config.checkpoint_dir = '{ckpt}'", 'Config.batch_size = 2048',
          f'Config.max_steps = {steps}', f'Config.print_every = {max(1, steps // 5)}',
          f'Config.checkpoint_every = {steps}', f'Config.train_render_every = {10 * steps}',
          'Config.render_chunk_size = 1024', 'Config.near = 0.05', 'Config.far = 1e6', 'Config.lr_init = 5e-3',
          'Config.lr_final = 5e-4', "Config.dataset_loader = 'blender'", 'Model.raydist_fn = @jnp.reciprocal',
          'Model.opaque_background = True', 'Model.num_prop_samples = 48', 'Model.num_nerf_samples = 32',
          'PropMLP.warp_fn = @coord.contract', 'NerfMLP.warp_fn = @coord.contract', 'PropMLP.net_depth = 2',
          'PropMLP.net_width = 64', 'NerfMLP.net_depth = 4', 'NerfMLP.net_width = 128',
          'NerfMLP.bottleneck_width = 64', 'NerfMLP.net_width_viewdirs = 64', 'PropMLP.disable_density_normals = True',
          'PropMLP.disable_rgb = True', 'NerfMLP.disable_density_normals = True']


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=2000)
  ap.add_argument('--resolution', type=int, default=256)
  ap.add_argument('--level', type=float, default=10.0)
  ap.add_argument('--workdir', default=None)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  import extract_mesh
  import train
  from multinerf_b200 import lib
  lib.require_device()
  work = args.workdir or tempfile.mkdtemp(prefix='mesh_contract_coverage_')
  data, ckpt = os.path.join(work, 'scene'), os.path.join(work, 'ckpt')
  write_scene(data)
  argv = [f'--gin_bindings={b}' for b in train_bindings(data, ckpt, args.steps)]
  train.main(argv)
  res = {'steps': args.steps, 'resolution': args.resolution, 'level': args.level, 'spaces': {}}
  eval_dir = os.path.join(ckpt, 'mesh', f'eval_step_{args.steps}')
  for space in ('world', 'contracted'):
    extract_mesh.main(argv + [f'--gin_bindings=Config.mesh_resolution = {args.resolution}',
                              f'--gin_bindings=Config.mesh_level = {args.level}',
                              f"--gin_bindings=Config.mesh_space = '{space}'", '--gin_bindings=Config.mesh_eval = True'])
    metric = lambda m: float(np.mean([float(x) for x in open(os.path.join(eval_dir, f'metric_{m}.txt')).read().split()]))
    ply = os.path.join(ckpt, 'mesh', f'mesh_step_{args.steps}.ply')
    head = open(ply, 'rb').read(400).split(b'end_header')[0].decode()
    faces = int(head.split('element face ')[1].split()[0])
    res['spaces'][space] = {'coverage': metric('coverage'), 'depth_abs_rel': metric('depth_abs_rel'),
                            'spurious': metric('spurious'), 'faces': faces}
  q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                     text=True)
  res['device'] = q.stdout.strip().splitlines()[:1]
  line = json.dumps(res)
  print(line, flush=True)
  if args.out:
    with open(args.out, 'w') as fh:
      fh.write(line + '\n')


if __name__ == '__main__':
  main()
