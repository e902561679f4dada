#!/usr/bin/env python
"""Mesh extraction entry point: the surface of the newest checkpoint's final-level density as a PLY file.

  python extract_mesh.py --gin_configs=configs/360.gin --gin_bindings="Config.checkpoint_dir = '...'" \
      --gin_bindings="Config.mesh_level = 10." --gin_bindings="Config.mesh_resolution = 512"
Writes <checkpoint_dir>/mesh/mesh_step_<step>.ply (multinerf_b200/mesh.py; Config.mesh_bbox sets the box, and
forward-facing scenes must set it; Config.mesh_vertex_colors = True adds vertex normals and colours).  One process on
one GPU.
"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from multinerf_b200 import checkpoints, configs, mesh, train_utils  # noqa: E402
from train import parse  # noqa: E402


def main(argv=None):
  args = parse(argv)
  bundle = configs.load_config(args.gin_configs, args.gin_bindings, search_paths=[ROOT, os.getcwd()])
  config = bundle.config
  bbox = mesh.default_bbox(bundle)
  if checkpoints.latest_checkpoint(config.checkpoint_dir) is None:
    raise FileNotFoundError(f'no checkpoint in {config.checkpoint_dir!r}')
  model, state, _, _, _ = train_utils.setup_model(bundle, 20200823)
  state = checkpoints.restore_checkpoint(config.checkpoint_dir, state, model=model)
  step = int(state.step)
  t0 = time.time()
  vertices, faces, *extra = mesh.extract_mesh(model, bbox, config.mesh_resolution, config.mesh_level,
                                              colors=config.mesh_vertex_colors)
  torch.cuda.synchronize()
  elapsed = time.time() - t0
  out_dir = os.path.join(config.checkpoint_dir, 'mesh')
  os.makedirs(out_dir, exist_ok=True)
  path = os.path.join(out_dir, f'mesh_step_{step}.ply')
  mesh.write_ply(path, vertices, faces, *extra)
  print(f'{vertices.shape[0]} vertices, {faces.shape[0]} faces in {elapsed:.2f} s '
        f'(grid {config.mesh_resolution} along the longest side of {bbox}, level {config.mesh_level}) -> {path}',
        flush=True)
  return path


if __name__ == '__main__':
  main()
