#!/usr/bin/env python
"""TSDF mesh extraction timings on one GPU (Config.mesh_method = 'tsdf', multinerf_b200/mesh.py), one JSON line:

  integrate: mnrf_tsdf_integrate alone (CUDA events over --reps launches) on 512^3 and 1024^3 grids spanning
             [-1, 1]^3, fusing K views (--ks) of 1008 x 756 pixels of an analytic sphere (radius 0.6, cameras on a
             sphere of radius 2.6), with and without colours: grid-point views per second (points x K / kernel time),
             and HBM bytes by count over kernel time -- the state read and written once per point (8 B, 24 B with
             colours, each way) plus every view's depth and acc (+ rgb) read once;
  extract:   mesh.extract_mesh_tsdf's three stages on a random-init 360.gin model and --views synthetic cameras of
             1008 x 756 pixels (rendered with the graph-replayed render chunks), fused at --extract_res^3 with
             colours: render, fuse and marching-cubes time, each ending in a device synchronise;
  device:    the card's name and power limit, read in the same run.

  python tools/tsdf_bench.py [--ks 1,8,32] [--reps 5] [--views 8] [--extract_res 512] [--out result.json]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from multinerf_b200 import camera_utils, configs, lib, mesh, models, ops, utils  # noqa: E402

W, H = 1008, 756


def device_info():
  q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                     capture_output=True, text=True)
  return {'torch_name': torch.cuda.get_device_name(), 'nvidia_smi': q.stdout.strip().splitlines()[:1]}


def cameras(n, radius=2.6, focal=900.0):
  """n cameras on a Fibonacci sphere looking at the origin -> (pixtocams [n, 3, 3], camtoworlds [n, 3, 4])."""
  c2w = []
  for i in range(n):
    zc = 1 - 2 * (i + 0.5) / n
    a = i * math.pi * (3 - math.sqrt(5))
    eye = radius * np.array([math.sqrt(1 - zc * zc) * math.cos(a), math.sqrt(1 - zc * zc) * math.sin(a), zc])
    up = np.array([0.0, 0.0, 1.0]) if abs(zc) < 0.95 else np.array([1.0, 0.0, 0.0])
    c2w.append(camera_utils.viewmatrix(eye, up, eye))
  p2c = camera_utils.get_pixtocam(focal, W, H)
  return np.broadcast_to(p2c, (n, 3, 3)).copy(), np.stack(c2w)


def pixels(k, near, far):
  xs, ys = camera_utils.pixel_coordinates(W, H)
  one = lambda v: np.full((H, W, 1), v, np.float32)
  return utils.Pixels(pix_x_int=xs.astype(np.int32), pix_y_int=ys.astype(np.int32), lossmult=one(1.0),
                      near=one(near), far=one(far), cam_idx=np.full((H, W, 1), k, np.int32))


def sphere_views(cams, K):
  """depth, acc [K, H, W] and rgb [K, H, W, 3] of a sphere of radius 0.6 at the origin, traced exactly."""
  out = []
  for k in range(K):
    r = camera_utils.cast_ray_batch(cams, pixels(k, 0.0, 1e6))
    o, d = r.origins.reshape(-1, 3).double(), r.directions.reshape(-1, 3).double()
    a, b, c = (d * d).sum(-1), (o * d).sum(-1), (o * o).sum(-1) - 0.36
    disc = b * b - a * c
    t = (-b - torch.sqrt(disc.clamp_min(0))) / a
    hit = disc > 0
    out.append((torch.where(hit, t, torch.full_like(t, 1e6)).float().view(H, W), hit.float().view(H, W),
                (0.5 + 0.3 * (o + t[:, None] * d)).clamp(0, 1).float().view(H, W, 3)))
  return [torch.stack(x).contiguous() for x in zip(*out)]


def bench_integrate(res, K, reps, colors):
  bbox = (-1.0, -1.0, -1.0, 1.0, 1.0, 1.0)
  (nx, ny, nz), h = mesh.grid_shape(bbox, res)
  p2c, c2w = cameras(K)
  w2c, c2p = mesh.camera_matrices((p2c, c2w, None, None), 'cuda')
  depth, acc, rgb = sphere_views((p2c, c2w, None, None), K)
  n = nx * ny * nz
  z = lambda *sh: torch.zeros(nz, ny, nx, *sh, device='cuda')
  state = [z(), z()] + ([z(3), z()] if colors else [None, None])
  call = lambda: ops.tsdf_integrate((nx, ny, nz), bbox[:3], h, 0, None, w2c, c2p, depth, acc,
                                    rgb if colors else None, 3 * h, *state)
  call()                                            # warm-up
  torch.cuda.synchronize()
  ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
  ev[0].record()
  for _ in range(reps):
    call()
  ev[1].record()
  torch.cuda.synchronize()
  sec = ev[0].elapsed_time(ev[1]) / 1e3 / reps
  state_b = n * (24 if colors else 8) * 2
  view_b = K * H * W * (20 if colors else 8)
  observed = float((state[1] > 0).double().mean())
  del state, depth, acc, rgb
  torch.cuda.empty_cache()
  return {'res': res, 'K': K, 'colors': colors, 'ms': sec * 1e3, 'point_views_per_s': n * K / sec,
          'hbm_GB_per_s_by_count': (state_b + view_b) / sec / 1e9, 'observed_fraction': observed}


class SyntheticCameras:
  """The part of a dataset extract_mesh_tsdf reads: size, cameras, camtype, generate_ray_batch."""

  def __init__(self, n, near, far):
    self.size, self.near, self.far = n, near, far
    self.cameras = cameras(n) + (None, None)
    self.camtype = camera_utils.ProjectionType.PERSPECTIVE

  def generate_ray_batch(self, k):
    return utils.Batch(rays=camera_utils.cast_ray_batch(self.cameras, pixels(k, self.near, self.far)))


def bench_extract(views, res):
  bundle = configs.bundle_360()
  model = models.Model(bundle)
  model.init(seed=0)
  bbox = mesh.default_bbox(bundle)
  data = SyntheticCameras(views, bundle.config.near, bundle.config.far)
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  rendered = list(mesh.render_views(model, data))
  torch.cuda.synchronize()
  t1 = time.perf_counter()
  state, h = mesh.fuse_tsdf(rendered, data.cameras, data.camtype, bbox, res, 3.0, colors=True)
  torch.cuda.synchronize()
  t2 = time.perf_counter()
  v, f, _, _ = mesh.tsdf_mesh(state, bbox, h, colors=True)
  torch.cuda.synchronize()
  t3 = time.perf_counter()
  return {'views': views, 'pixels': W * H, 'res': res, 'render_s': t1 - t0, 'fuse_s': t2 - t1, 'mesh_s': t3 - t2,
          'vertices': int(v.shape[0]), 'faces': int(f.shape[0]),
          'observed_fraction': float((state[1] > 0).double().mean())}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--ks', default='1,8,32')
  ap.add_argument('--reps', type=int, default=5)
  ap.add_argument('--views', type=int, default=8)
  ap.add_argument('--extract_res', type=int, default=512)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  lib.require_device()
  res = {'device': device_info(), 'integrate': [], 'extract': None}
  for r in (512, 1024):
    for K in (int(k) for k in args.ks.split(',')):
      for colors in (False, True):
        res['integrate'].append(bench_integrate(r, K, args.reps, colors))
        print(json.dumps(res['integrate'][-1]), flush=True)
  res['extract'] = bench_extract(args.views, args.extract_res)
  line = json.dumps(res)
  print(line, flush=True)
  if args.out:
    with open(args.out, 'w') as f:
      f.write(line + '\n')


if __name__ == '__main__':
  main()
