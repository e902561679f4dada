#!/usr/bin/env python
"""Mesh extraction entry point: the surface of the newest checkpoint's scene as a PLY file.

  python extract_mesh.py --gin_configs=configs/360.gin --gin_bindings="Config.checkpoint_dir = '...'" \\
      --gin_bindings="Config.mesh_level = 10." --gin_bindings="Config.mesh_resolution = 512"
Writes <checkpoint_dir>/mesh/mesh_step_<step>.ply (multinerf_b200/mesh.py; Config.mesh_bbox sets the box, and
forward-facing scenes must set it; Config.mesh_vertex_colors = True adds vertex normals and colours).
Config.mesh_method = 'density' (default) meshes the final level's density at Config.mesh_level; 'tsdf' renders every
training view, fuses the rendered depth into a truncated signed-distance grid (Config.mesh_tsdf_truncation cells) and
meshes its zero crossing.  Config.mesh_min_views drops what fewer training views see, and
Config.mesh_keep_components keeps only the largest connected components (mesh.clean_mesh).
Config.mesh_target_faces then simplifies the mesh to about that many faces by quadric edge collapse
(mesh.simplify_mesh).  Config.mesh_texture_size = S then bakes the surface colour into an S x S texture atlas
(mesh.bake_texture) and writes mesh_step_<step>.{obj,mtl,png} beside the PLY, which is written first and unchanged.
Config.mesh_eval = True then scores the mesh against the test split (mesh.evaluate_mesh): it renders the NeRF on the
test views for reference, traces every test pixel's ray into the mesh, shaded with the most detailed colour the run
produced (the texture, else the vertex colours, else none), and writes mesh/eval_step_<step>/{color,normals}_NNN.png,
distance_NNN.tiff and metric_<name>.txt (per-image values, space-separated).
Config.mesh_space = 'contracted' puts the grid of either method in the contracted space of an unbounded scene
(360.gin), so the background is meshed too: Config.mesh_bbox is then in contracted coordinates (default [-2, 2]^3),
Config.mesh_level a density per unit of contracted length, and the outputs are still in world coordinates.
One process on one GPU.
"""
import dataclasses
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from multinerf_b200 import checkpoints, configs, datasets, mesh, ops, train_utils, utils  # noqa: E402
from train import parse  # noqa: E402


def main(argv=None):
  args = parse(argv)
  bundle = configs.load_config(args.gin_configs, args.gin_bindings, search_paths=[ROOT, os.getcwd()])
  config = bundle.config
  method = mesh.validate_config(bundle)
  bbox = mesh.default_bbox(bundle)
  if checkpoints.latest_checkpoint(config.checkpoint_dir) is None:
    raise FileNotFoundError(f'no checkpoint in {config.checkpoint_dir!r}')
  model, state, _, _, _ = train_utils.setup_model(bundle, 20200823)
  state = checkpoints.restore_checkpoint(config.checkpoint_dir, state, model=model)
  step = int(state.step)
  dataset = None
  if method == 'tsdf' or config.mesh_min_views > 0:
    # every training camera, all pixels, no render path
    dataset = datasets.load_dataset('train', config.data_dir, dataclasses.replace(config, render_path=False),
                                    device=model.device)
  clean = dict(keep_components=config.mesh_keep_components, min_views=config.mesh_min_views,
               target_faces=config.mesh_target_faces, stats={})
  out_dir = os.path.join(config.checkpoint_dir, 'mesh')
  path = os.path.join(out_dir, f'mesh_step_{step}.ply')
  size = config.mesh_texture_size
  t0 = time.time()
  timing = {}

  def save_ply(vertices, faces, normals=None, rgb=None):
    """The PLY as without a texture: normals and colours only with mesh_vertex_colors."""
    torch.cuda.synchronize()
    elapsed = time.time() - t0
    if config.mesh_keep_components or config.mesh_min_views:
      s = clean['stats']
      print(f"cleaning removed {s['vertices_removed']} vertices, {s['faces_removed']} faces and "
            f"{s['components_removed']} components (mesh_min_views {config.mesh_min_views}, "
            f"mesh_keep_components {config.mesh_keep_components})", flush=True)
    if config.mesh_target_faces:
      s = clean['stats']
      print(f"simplified {s['faces_before']} -> {s['faces_after']} faces in {s['rounds']} rounds "
            f"(mesh_target_faces {config.mesh_target_faces})" +
            ('' if s['target_reached'] else ': stalled before the target, no edge left that may be collapsed'),
            flush=True)
    os.makedirs(out_dir, exist_ok=True)
    mesh.write_ply(path, vertices, faces, *((normals, rgb) if config.mesh_vertex_colors else ()))
    print(f'{vertices.shape[0]} vertices, {faces.shape[0]} faces in {elapsed:.2f} s '
          f'(grid {config.mesh_resolution} along the longest side of {bbox} in {config.mesh_space} space, {what}) -> '
          f'{path}', flush=True)
    timing['t'] = time.time()

  texture = dict(texture_size=size, before_texture=save_ply) if size else {}
  if method == 'tsdf':
    what = f'{dataset.size} views fused, truncation {config.mesh_tsdf_truncation} cells'
    vertices, faces, *extra = mesh.extract_mesh_tsdf(model, dataset, bbox, config.mesh_resolution,
                                                     config.mesh_tsdf_truncation, colors=config.mesh_vertex_colors,
                                                     space=config.mesh_space, **clean, **texture)
  else:
    what = f'level {config.mesh_level}'
    vertices, faces, *extra = mesh.extract_mesh(model, bbox, config.mesh_resolution, config.mesh_level,
                                                colors=config.mesh_vertex_colors, dataset=dataset,
                                                space=config.mesh_space, **clean, **texture)
  if not size:
    save_ply(vertices, faces, *extra)
    if config.mesh_eval:
      normals, rgb = extra if extra else (None, None)
      evaluate(model, config, step, out_dir, vertices, faces, normals=normals, rgb=rgb)
    return path
  normals, rgb, uv, tex = extra
  torch.cuda.synchronize()
  baked = time.time() - timing['t']
  _, c = ops.texture_atlas(faces.shape[0], size)
  obj = mesh.write_obj(os.path.splitext(path)[0] + '.obj', vertices, faces, normals, uv, tex)[0]
  print(f'texture {size} x {size}, {c} x {c} texels per cell, {(faces.shape[0] + 1) // 2 * c * c} texels baked in '
        f'{baked:.2f} s -> {obj}', flush=True)
  if config.mesh_eval:
    evaluate(model, config, step, out_dir, vertices, faces, normals=normals, uv=uv, texture=tex)
  return path


def evaluate(model, config, step, out_dir, vertices, faces, **colour):
  """Config.mesh_eval: the mesh against the test split, the NeRF's renders of it as the reference; writes the renders
  and metric files to <out_dir>/eval_step_<step> and prints each metric's mean and where the time went."""
  dataset = datasets.load_dataset('test', config.data_dir, dataclasses.replace(config, render_path=False),
                                  device=model.device)
  eval_dir = os.path.join(out_dir, f'eval_step_{step}')
  os.makedirs(eval_dir, exist_ok=True)
  nerf_time = [0.0]

  def reference():
    views = mesh.render_views(model, dataset)
    while True:
      t0 = time.time()
      view = next(views, None)
      torch.cuda.synchronize()
      nerf_time[0] += time.time() - t0
      if view is None:
        return
      yield view

  def save(idx, render):
    if render['rgb'] is not None:
      utils.save_img_u8(render['rgb'], os.path.join(eval_dir, f'color_{idx:03d}.png'))
    utils.save_img_u8(render['normals'] / 2. + 0.5, os.path.join(eval_dir, f'normals_{idx:03d}.png'))
    utils.save_img_f32(render['distance'], os.path.join(eval_dir, f'distance_{idx:03d}.tiff'))

  lo, hi = model.mcfg.bg_intensity_range
  timing = {}
  metrics = mesh.evaluate_mesh(vertices, faces, dataset, config, reference=reference(), bg=(lo + hi) / 2,
                               save_fn=save, timing=timing, **colour)
  for name in (metrics[0] if metrics else {}):
    with open(os.path.join(eval_dir, f'metric_{name}.txt'), 'w') as f:
      f.write(' '.join(str(m[name]) for m in metrics))
    print(f'mesh eval {name:14s} = {np.mean([m[name] for m in metrics]):.4f}', flush=True)
  print(f'mesh eval: {len(metrics)} test views, NeRF rendering {nerf_time[0]:.2f} s, BVH build '
        f'{timing.get("build", 0.0):.3f} s, tracing and shading {timing.get("trace", 0.0):.3f} s -> {eval_dir}',
        flush=True)
  return metrics


if __name__ == '__main__':
  main()
