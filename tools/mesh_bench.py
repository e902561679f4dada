#!/usr/bin/env python
"""Mesh extraction timings on one GPU (multinerf_b200/mesh.py), printed as one JSON line:

  query:  Model.query_density rows/s over `--rows` random points (wall time around a synchronised window), and the
          query GEMM launches' TFLOP/s over their CUDA-event kernel time, on the NerfMLPs of 360.gin (8 x 1024,
          per-layer GEMMs) and blender_256.gin (8 x 256, the chained trunk), random init;
  mc:     ops.marching_cubes (count, scans, one read-back of the totals, emit) at 256^3 and 512^3 on a sphere plus
          smooth noise;
  extract: mesh.extract_mesh end to end at --extract_res^3 on the 360.gin model (random init, level = the grid's
          median density over a first, untimed extraction);
  color:  Model.query_radiance rows/s and its GEMM TFLOP/s as for `query`, on the same NerfMLPs and points, with
          unit view directions; mnrf_mc_normals alone (CUDA events over --reps launches) at 256^3 and 512^3 on the
          `mc` grids; mesh.extract_mesh at --extract_res^3 without and with colours, alternated --reps times;
  components: ops.mesh_components and mesh.clean_mesh(keep_components=1) (CUDA events over --reps calls) on the
          512^3 `mc` mesh and on the 512^3 random-init 360.gin extraction, with the bytes the union-find moves by
          count; mesh.extract_mesh at --extract_res^3 with mesh_keep_components 0 and 1, alternated --reps times;
  simplify: mesh.simplify_mesh (CUDA events around whole calls, after one warm-up call) on the 512^3 `mc` mesh to
          10 % and 1 % of its faces and on the 512^3 random-init 360.gin extraction after keep_components = 1 to
          --simplify_faces faces: rounds, peak device memory, the PLY size by count before and after, and from one
          more call with CUDA events around each step, the time in the torch topology rebuilds against the kernels;
          mesh.extract_mesh at --extract_res^3 without and with target_faces = --simplify_faces, alternated --reps
          times (not part of `all`);
  texture: the 512^3 `mc` mesh simplified to --texture_faces faces; mnrf_mesh_texture_raster alone (CUDA events over
          --texture_launches launches) on it at S = 4096 and 8192; the colour query over all of the 4096 atlas's texels
          (mesh.vertex_colors, a synchronised window) on the 360.gin and blender_256.gin NerfMLPs; mesh.write_obj and
          the PNG alone; and mesh.extract_mesh at --extract_res^3 on the random-init 360.gin model with target_faces
          = --simplify_faces, without and with texture_size = --texture_extract_size (large enough for the mesh the
          simplification stalls at), alternated --reps times (not part of `all`);
  trace:  ops.mesh_bvh (CUDA events around whole calls after one warm-up, and the peak device memory above the mesh)
          and ops.mesh_trace rays/s (CUDA events over --trace_views 1560 x 1040 perspective views orbiting the
          origin) on the 512^3 `mc` mesh simplified to --simplify_faces faces and on the 512^3 random-init 360.gin
          extraction after mesh_target_faces = --simplify_faces (where the simplification stalls); and
          mesh.evaluate_mesh on one such view of the 360.gin mesh with the NeRF's render_views as its reference,
          split into NeRF rendering, BVH build and tracing with shading (not part of `all`);
  contracted: Config.mesh_space = 'contracted' against 'world' on the random-init 360.gin NerfMLP: mesh.density_grid
          at --extract_res^3 over [-2, 2]^3 (contracted) and over the world default box, with the points queried and
          skipped, rows/s of the queried points and points/s with the skipped ones counted; mesh.extract_mesh end to
          end in both spaces at the same level, alternated --reps times, with the peak device memory of each; and
          ops.tsdf_integrate against ops.tsdf_integrate(contracted=True) in G point-views/s (CUDA events around one
          launch of 32 views of 1008 x 756, random depth and opacity, cameras inside the unit ball) into 512^3 and
          1024^3 grids (not part of `all`);
  device: the card's name and power limit, read in the same run.

  python tools/mesh_bench.py [--rows 8388608] [--extract_res 512]
                             [--sections all|components|simplify|texture|trace|contracted]
                             [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from multinerf_b200 import configs, lib, mesh, models, ops  # noqa: E402


def device_info():
  q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                     capture_output=True, text=True)
  return {'torch_name': torch.cuda.get_device_name(), 'nvidia_smi': q.stdout.strip().splitlines()[:1]}


def timed(fn, reps):
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for _ in range(reps):
    out = fn()
  torch.cuda.synchronize()
  return (time.perf_counter() - t0) / reps, out


def bench_query(bundle, rows, reps, radiance=False):
  """query_density, or with `radiance` query_radiance (view directions uniform on the sphere)."""
  model = models.Model(bundle)
  model.init(seed=0)
  g = torch.Generator(device='cuda')
  g.manual_seed(0)
  pts = torch.rand(rows, 3, device='cuda', generator=g) * 3 - 1.5
  var = (3.0 / 511) ** 2 / 12
  if radiance:
    vd = torch.nn.functional.normalize(torch.randn(rows, 3, device='cuda', generator=g), dim=-1)
    query = lambda: model.query_radiance(pts, var, vd)
  else:
    query = lambda: model.query_density(pts, var)
  query()                                            # warm-up: every chunk shape, plans, module loads
  wall, _ = timed(query, reps)
  ops.GEMM_EVENTS = []
  query()
  torch.cuda.synchronize()
  ev, ops.GEMM_EVENTS = ops.GEMM_EVENTS, None
  kern_s = sum(a.elapsed_time(b) for a, b, _ in ev) / 1e3
  flops = sum(f for _, _, f in ev)
  plan = model.plans['NerfMLP_0']
  return {'rows': rows, 'chained': model._use_chain(plan, bundle.config.render_chunk_size *
                                                     bundle.model.num_nerf_samples),
          'wall_s': round(wall, 4), 'rows_per_s': round(rows / wall), 'gemm_launches': len(ev),
          'gemm_kernel_s': round(kern_s, 4), 'gemm_tflops': round(flops / kern_s / 1e12, 1),
          'gemm_share_of_wall': round(kern_s / wall, 3), 'gemm_flop_per_row': flops / rows}


def sphere_noise(n, seed=0):
  g = torch.Generator(device='cuda')
  g.manual_seed(seed)
  ax = torch.linspace(-1, 1, n, device='cuda')
  z, y, x = torch.meshgrid(ax, ax, ax, indexing='ij')
  f = 0.7 - torch.sqrt(x * x + y * y + z * z)
  k = torch.randn(8, 3, device='cuda', generator=g) * 6
  ph = torch.rand(8, device='cuda', generator=g) * 6.283
  for i in range(8):
    f += 0.03 * torch.cos(k[i, 0] * x + k[i, 1] * y + k[i, 2] * z + ph[i])
  return f.contiguous()


def bench_mc(n, reps):
  grid = sphere_noise(n)
  ops.marching_cubes(grid, 0.0)
  t, (v, f) = timed(lambda: ops.marching_cubes(grid, 0.0), reps)
  return {'grid': n, 's': round(t, 4), 'vertices': int(v.shape[0]), 'faces': int(f.shape[0])}


def bench_mc_normals(n, reps):
  """mnrf_mc_normals alone on the `bench_mc` grid: the count phase and the edge scan once, then CUDA events around
  `reps` normal launches."""
  L = lib.load()
  grid = sphere_noise(n)
  edge_cut = torch.empty(3 * grid.numel(), device='cuda', dtype=torch.uint8)
  cell_tris = torch.empty(grid.numel(), device='cuda', dtype=torch.uint8)
  lib.check(L.mnrf_marching_cubes(lib.MC_COUNT, n, n, n, lib.ptr(grid), 0.0, lib.ptr(edge_cut), lib.ptr(cell_tris),
                                  None, None, None, None, lib.stream_ptr()))
  edge_scan = torch.cumsum(edge_cut, 0, dtype=torch.int64)
  V = int(edge_scan[-1])
  normals = torch.empty(V, 3, device='cuda')

  def launch():
    lib.check(L.mnrf_mc_normals(n, n, n, lib.ptr(grid), 0.0, lib.ptr(edge_cut), lib.ptr(edge_scan), lib.ptr(normals),
                                lib.stream_ptr()))
  launch()
  ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
  ev[0].record()
  for _ in range(reps):
    launch()
  ev[1].record()
  torch.cuda.synchronize()
  return {'grid': n, 'vertices': V, 'ms': round(ev[0].elapsed_time(ev[1]) / reps, 3)}


def events(fn, reps):
  """Mean ms of fn() over `reps` calls between two CUDA events, after one warm-up call."""
  fn()
  ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
  ev[0].record()
  for _ in range(reps):
    fn()
  ev[1].record()
  torch.cuda.synchronize()
  return ev[0].elapsed_time(ev[1]) / reps


def bench_components(name, v, f, reps):
  """ops.mesh_components and clean_mesh(keep_components=1) on one mesh.  Bytes by count: the faces read once
  (12 B a face), the four first parent loads of a face's two unions (16 B), and the labels written by the
  initialisation and read and written by compression (12 B a vertex)."""
  V, F = int(v.shape[0]), int(f.shape[0])
  labels = ops.mesh_components(f, V)
  ncomp = int((labels == torch.arange(V, device='cuda', dtype=torch.int32)).sum())
  del labels
  ms = events(lambda: ops.mesh_components(f, V), reps)
  clean_ms = events(lambda: mesh.clean_mesh(v, f, keep_components=1), reps)
  kv, kf = mesh.clean_mesh(v, f, keep_components=1)
  nbytes = 28 * F + 12 * V
  return {'mesh': name, 'vertices': V, 'faces': F, 'components_incl_lone_vertices': ncomp,
          'kept_vertices': int(kv.shape[0]), 'kept_faces': int(kf.shape[0]), 'mesh_components_ms': round(ms, 3),
          'bytes_by_count': nbytes, 'tb_per_s_by_count': round(nbytes / (ms * 1e-3) / 1e12, 3),
          'clean_mesh_keep1_ms': round(clean_ms, 3)}


def bench_components_section(model, bbox, level, args):
  out = {'meshes': [], 'extract': {'keep0_s': [], 'keep1_s': []}}
  v, f = ops.marching_cubes(sphere_noise(512), 0.0)
  torch.cuda.empty_cache()
  out['meshes'].append(bench_components('mc 512^3 sphere + noise', v, f, args.reps))
  del v, f
  torch.cuda.empty_cache()
  v, f = mesh.extract_mesh(model, bbox, args.extract_res, level)
  out['meshes'].append(bench_components(f'360.gin random init, {args.extract_res}^3', v, f, args.reps))
  del v, f
  torch.cuda.empty_cache()
  mesh.extract_mesh(model, bbox, args.extract_res, level, keep_components=1)      # warm-up
  torch.cuda.empty_cache()
  for _ in range(args.reps):
    for key, keep in (('keep0_s', 0), ('keep1_s', 1)):
      t, o = timed(lambda: mesh.extract_mesh(model, bbox, args.extract_res, level, keep_components=keep), 1)
      out['extract'][key].append(round(t, 3))
      out['extract'][f'{key[:5]}_vertices'] = int(o[0].shape[0])
      del o
      torch.cuda.empty_cache()
  return out


def ply_bytes(v, f):
  """PLY size by count without normals or colours: 12 B a vertex, 13 B a face (plus a header of under 300 B)."""
  return 12 * int(v.shape[0]) + 13 * int(f.shape[0])


def simplify_breakdown(v, f, target):
  """One simplify_mesh call with CUDA events around each topology rebuild (mesh_topology, boundary_edges) and each
  kernel call -> ms per step name, summed over rounds."""
  names = {'topology': (mesh, 'mesh_topology'), 'boundary': (mesh, 'boundary_edges'),
           'quadrics': (ops, 'mesh_quadrics'), 'edge_cost': (ops, 'mesh_edge_cost'),
           'select': (ops, 'mesh_collapse_select'), 'apply': (ops, 'mesh_collapse_apply')}
  spans = {k: [] for k in names}
  saved = {k: getattr(m, a) for k, (m, a) in names.items()}

  def wrap(key, fn):
    def run(*args, **kw):
      ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
      ev[0].record()
      out = fn(*args, **kw)
      ev[1].record()
      spans[key].append(ev)
      return out
    return run
  for k, (m, a) in names.items():
    setattr(m, a, wrap(k, saved[k]))
  try:
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mesh.simplify_mesh(v, f, target_faces=target)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
  finally:
    for k, (m, a) in names.items():
      setattr(m, a, saved[k])
  ms = {k: round(sum(e[0].elapsed_time(e[1]) for e in evs), 2) for k, evs in spans.items()}
  ms['wall_ms_instrumented'] = round(wall * 1e3, 1)
  ms['other_ms'] = round(wall * 1e3 - sum(v for k, v in ms.items() if k != 'wall_ms_instrumented'), 1)
  return ms


def bench_simplify(name, v, f, target, reps):
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  base = torch.cuda.memory_allocated()
  stats = {}
  sv, sf = mesh.simplify_mesh(v, f, target_faces=target, stats=stats)     # warm-up, and the counts
  torch.cuda.synchronize()
  peak = torch.cuda.max_memory_allocated()
  out = {'mesh': name, 'vertices': int(v.shape[0]), 'faces': int(f.shape[0]), 'target_faces': target, **stats,
         'vertices_after': int(sv.shape[0]), 'ply_bytes_before': ply_bytes(v, f), 'ply_bytes_after': ply_bytes(sv, sf),
         'peak_alloc_gb': round(peak / 1e9, 2), 'peak_over_input_gb': round((peak - base) / 1e9, 2)}
  del sv, sf
  torch.cuda.empty_cache()
  out['ms'] = round(events(lambda: mesh.simplify_mesh(v, f, target_faces=target), reps), 1)
  torch.cuda.empty_cache()
  out['breakdown_ms'] = simplify_breakdown(v, f, target)
  torch.cuda.empty_cache()
  return out


def bench_simplify_section(model, bbox, level, args):
  out = {'meshes': [], 'extract': {'plain_s': [], 'simplified_s': []}}
  v, f = ops.marching_cubes(sphere_noise(512), 0.0)
  torch.cuda.empty_cache()
  for frac in (0.1, 0.01):
    out['meshes'].append(bench_simplify('mc 512^3 sphere + noise', v, f, int(f.shape[0] * frac), args.reps))
  del v, f
  torch.cuda.empty_cache()
  v, f = mesh.extract_mesh(model, bbox, args.extract_res, level, keep_components=1)
  torch.cuda.empty_cache()
  out['meshes'].append(bench_simplify(f'360.gin random init, {args.extract_res}^3, keep_components 1', v, f,
                                      args.simplify_faces, 1))
  del v, f
  torch.cuda.empty_cache()
  mesh.extract_mesh(model, bbox, args.extract_res, level, target_faces=args.simplify_faces)      # warm-up
  torch.cuda.empty_cache()
  for _ in range(args.reps):
    for key, target in (('plain_s', 0), ('simplified_s', args.simplify_faces)):
      t, o = timed(lambda: mesh.extract_mesh(model, bbox, args.extract_res, level, target_faces=target), 1)
      out['extract'][key].append(round(t, 3))
      out['extract'][f'{key[:-2]}_faces'] = int(o[1].shape[0])
      del o
      torch.cuda.empty_cache()
  return out


def bench_texture_section(model, bbox, level, args):
  import tempfile
  from PIL import Image
  out = {'raster': [], 'color_query': {}, 'write': {}, 'extract': {'plain_s': [], 'textured_s': []}}
  v, f, n = ops.marching_cubes(sphere_noise(512), 0.0, normals=True)
  v, f, n = mesh.simplify_mesh(v, f, n, target_faces=args.texture_faces)
  torch.cuda.empty_cache()
  L = lib.load()
  F = int(f.shape[0])
  for size in (4096, 8192):
    _, c = ops.texture_atlas(F, size)
    T = (F + 1) // 2 * c * c
    bufs = [torch.empty(F, 3, 2, device='cuda'), torch.empty(T, dtype=torch.int32, device='cuda'),
            torch.empty(T, 3, device='cuda'), torch.empty(T, 3, device='cuda')]
    launch = lambda: lib.check(L.mnrf_mesh_texture_raster(v.shape[0], F, lib.ptr(v), lib.ptr(f), lib.ptr(n), size,
                                                          *(lib.ptr(b) for b in bufs), lib.stream_ptr()))
    ms = events(launch, args.texture_launches)
    # bytes by count: per texel 4 B index + 24 B point and normal written; per face 24 B of uv
    nbytes = 28 * T + 24 * F
    out['raster'].append({'faces': F, 'size': size, 'cell': c, 'texels': T, 'ms': round(ms, 3),
                          'write_tb_per_s_by_count': round(nbytes / (ms * 1e-3) / 1e12, 3)})
    del bufs
    torch.cuda.empty_cache()
  _, _, points, tnormals = ops.mesh_texture_raster(v, f, n, 4096)
  for name, make in (('360', configs.bundle_360), ('blender_256', configs.bundle_blender_256)):
    m = models.Model(make())
    m.init(seed=0)
    mesh.vertex_colors(m, points[:1 << 20], tnormals[:1 << 20], 1e-6)      # warm-up of the chunk shapes
    t, _ = timed(lambda: mesh.vertex_colors(m, points, tnormals, 1e-6), 1)
    out['color_query'][name] = {'texels': int(points.shape[0]), 's': round(t, 3),
                                'rows_per_s': round(points.shape[0] / t / 1e6, 1)}
    del m
    torch.cuda.empty_cache()
  del points, tnormals
  uv, tex = mesh.bake_texture(v, f, n, 4096, lambda p, nn: ((p.abs() * 40) % 256).to(torch.uint8))
  with tempfile.TemporaryDirectory() as tmp:
    t0 = time.perf_counter()
    mesh.write_obj(os.path.join(tmp, 'm.obj'), v, f, n, uv, tex)
    t_obj = time.perf_counter() - t0
    host = tex.cpu().numpy()
    t0 = time.perf_counter()
    Image.fromarray(host).save(os.path.join(tmp, 'p.png'), 'PNG')
    t_png = time.perf_counter() - t0
    out['write'] = {'faces': F, 'size': 4096, 'write_obj_s': round(t_obj, 3), 'png_alone_s': round(t_png, 3),
                    'obj_bytes': os.path.getsize(os.path.join(tmp, 'm.obj')),
                    'png_bytes': os.path.getsize(os.path.join(tmp, 'm.png'))}
  del v, f, n, uv, tex
  torch.cuda.empty_cache()
  size = args.texture_extract_size
  kw = dict(target_faces=args.simplify_faces)
  mesh.extract_mesh(model, bbox, args.extract_res, level, texture_size=size, **kw)      # warm-up
  torch.cuda.empty_cache()
  for _ in range(args.reps):
    for key, tsize in (('plain_s', 0), ('textured_s', size)):
      t, o = timed(lambda: mesh.extract_mesh(model, bbox, args.extract_res, level, texture_size=tsize, **kw), 1)
      out['extract'][key].append(round(t, 3))
      out['extract']['faces'] = int(o[1].shape[0])
      del o
      torch.cuda.empty_cache()
  out['extract'].update(texture_size=size, cell=ops.texture_atlas(out['extract']['faces'], size)[1])
  return out


def orbit_views(n, W=1560, H=1040, radius=2.5):
  """(pixtocam [3, 3], camtoworlds [n, 3, 4]) of n perspective views on a circle around the origin, looking at it."""
  from multinerf_b200 import camera_utils
  p2c = camera_utils.get_pixtocam(0.5 * W / np.tan(0.5 * 0.9), W, H)
  poses = []
  for i in range(n):
    a = 2 * np.pi * i / n
    eye = np.array([radius * np.cos(a), radius * np.sin(a), 0.3 * radius])
    z = eye / np.linalg.norm(eye)
    x = np.cross([0, 0, 1.0], z)
    x /= np.linalg.norm(x)
    poses.append(np.concatenate([np.stack([x, np.cross(z, x), z], 1), eye[:, None]], 1))
  return p2c, np.stack(poses)


class _OrbitDataset:
  """The little of a test split that mesh.evaluate_mesh and mesh.render_views read, for orbit_views."""

  def __init__(self, n, W=1560, H=1040, near=0.2, far=1e6):
    from multinerf_b200 import camera_utils, utils
    self.p2c, self.poses = orbit_views(n, W, H)
    self.size, self.W, self.H, self.near, self.far = n, W, H, near, far
    self.cameras = (self.p2c, self.poses, None, None)
    self.images = np.zeros((n, H, W, 3), np.float32)
    self._cu, self._utils = camera_utils, utils

  def generate_ray_batch(self, idx):
    xs, ys = self._cu.pixel_coordinates(self.W, self.H)
    meta = lambda v: np.full((self.H, self.W, 1), v, np.float32)
    pixels = self._utils.Pixels(pix_x_int=xs, pix_y_int=ys, lossmult=meta(1.0), near=meta(self.near),
                                far=meta(self.far), cam_idx=np.zeros((self.H, self.W, 1), np.int32))
    return self._utils.Batch(rays=self._cu.cast_ray_batch((self.p2c, self.poses[idx], None, None), pixels))


def bench_trace_mesh(name, v, f, views, reps):
  torch.cuda.empty_cache()
  ops.mesh_bvh(v, f)                                           # warm-up
  torch.cuda.synchronize()
  base = torch.cuda.memory_allocated()
  torch.cuda.reset_peak_memory_stats()
  ms = events(lambda: ops.mesh_bvh(v, f), reps)
  bvh = ops.mesh_bvh(v, f)
  torch.cuda.synchronize()
  peak = torch.cuda.max_memory_allocated() - base
  ds = _OrbitDataset(views)
  rays = [ds.generate_ray_batch(i).rays for i in range(views)]
  dev = lambda x: torch.as_tensor(x, device='cuda', dtype=torch.float32).reshape(-1, x.shape[-1]).contiguous()
  flat = [(dev(r.origins), dev(r.directions), dev(r.near), dev(r.far)) for r in rays]
  ops.mesh_trace(bvh, *flat[0])
  n_rays = sum(x[0].shape[0] for x in flat)
  hits = sum(int((ops.mesh_trace(bvh, *x)[0] >= 0).sum()) for x in flat)
  it = iter(range(1 << 30))
  trace_ms = events(lambda: ops.mesh_trace(bvh, *flat[next(it) % views]), reps * views)
  return {'mesh': name, 'faces': int(f.shape[0]), 'build_ms': round(ms, 2), 'build_peak_mb': round(peak / 2 ** 20, 1),
          'views': f'{views} x 1560 x 1040', 'hit_fraction': round(hits / n_rays, 3),
          'trace_ms_per_view': round(trace_ms, 2), 'mrays_per_s': round(n_rays / views / (trace_ms * 1e-3) / 1e6, 1)}


def bench_trace_section(model, bbox, level, args):
  out = {'meshes': []}
  v, f = ops.marching_cubes(sphere_noise(512), 0.0)
  v, f = mesh.simplify_mesh(v * (2 / 511) - 1, f, target_faces=args.simplify_faces)     # grid units -> [-1, 1]^3
  out['meshes'].append(bench_trace_mesh('mc 512^3 sphere + noise, simplified', v, f, args.trace_views, args.reps))
  del v, f
  torch.cuda.empty_cache()
  v, f = mesh.extract_mesh(model, bbox, args.extract_res, level, target_faces=args.simplify_faces)
  out['meshes'].append(bench_trace_mesh(f'360.gin random init, {args.extract_res}^3, target_faces '
                                        f'{args.simplify_faces}', v, f, args.trace_views, args.reps))
  ds = _OrbitDataset(1)
  timing = {}
  nerf = [0.0]

  def reference():
    for view in mesh.render_views(model, ds):
      torch.cuda.synchronize()
      yield view
  t0 = time.perf_counter()
  gen = reference()
  first = next(gen)
  nerf[0] = time.perf_counter() - t0
  mesh.evaluate_mesh(v, f, ds, model.config, reference=[first], bg=1.0, timing=timing)
  out['evaluate'] = {'views': '1 x 1560 x 1040', 'faces': int(f.shape[0]), 'nerf_render_s': round(nerf[0], 3),
                     'build_s': round(timing['build'], 3), 'trace_and_shade_s': round(timing['trace'], 3)}
  return out


def bench_contracted_section(model, bbox, level, args):
  cbox = (-2.0, -2.0, -2.0, 2.0, 2.0, 2.0)
  out = {'grid': args.extract_res, 'world_bbox': list(bbox), 'contracted_bbox': list(cbox), 'level': level}
  n = args.extract_res ** 3
  for space, box in (('world', bbox), ('contracted', cbox)):
    mesh.density_grid(model, box, args.extract_res, space=space)           # warm-up of every slab shape
    torch.cuda.empty_cache()
    t, (grid, _) = timed(lambda: mesh.density_grid(model, box, args.extract_res, space=space), 1)
    queried = int(torch.isfinite(grid).sum()) if space == 'contracted' else n
    out[f'{space}_grid'] = {'s': round(t, 3), 'points': n, 'queried': queried, 'skipped': n - queried,
                            'queried_rows_per_s': round(queried / t), 'points_per_s': round(n / t)}
    del grid
    torch.cuda.empty_cache()
  runs = {'world': [], 'contracted': []}
  for _ in range(args.reps):
    for space, box in (('world', bbox), ('contracted', cbox)):
      torch.cuda.reset_peak_memory_stats()
      base = torch.cuda.memory_allocated()
      t, (v, f) = timed(lambda: mesh.extract_mesh(model, box, args.extract_res, level, space=space), 1)
      runs[space].append({'s': round(t, 3), 'vertices': int(v.shape[0]), 'faces': int(f.shape[0]),
                          'peak_gb': round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 2)})
      del v, f
      torch.cuda.empty_cache()
  out['extract'] = runs
  # TSDF fusion: one launch of K views into the grid, world against contracted
  rng = np.random.default_rng(0)
  K, W, H = 32, 1008, 756
  w2c = []
  for _ in range(K):
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    eye = rng.normal(size=3)
    eye *= 0.8 * rng.uniform() / np.linalg.norm(eye)
    w2c.append(np.concatenate([q.T, -q.T @ eye[:, None]], 1))
  dev = 'cuda'
  w2c = torch.tensor(np.stack(w2c), dtype=torch.float32, device=dev).contiguous()
  f_ = 0.6 * W
  c2p = torch.tensor([[[f_, 0, W / 2], [0, f_, H / 2], [0, 0, 1]]], dtype=torch.float32, device=dev)
  depth = torch.tensor(rng.uniform(0.5, 50, (K, H, W)), dtype=torch.float32, device=dev)
  acc = torch.tensor(rng.uniform(0, 1, (K, H, W)), dtype=torch.float32, device=dev)
  tsdf_rows = []
  for res in (512, 1024):
    for space, box in (('world', bbox), ('contracted', cbox)):
      (nx, ny, nz), h = mesh.grid_shape(box, res)
      state = [torch.zeros(nz, ny, nx, device=dev) for _ in range(2)]
      launch = lambda: ops.tsdf_integrate((nx, ny, nz), box[:3], h, 0, None, w2c, c2p, depth, acc, None, 3 * h,
                                          *state, contracted=space == 'contracted')
      ms = events(launch, args.reps)
      tsdf_rows.append({'grid': res, 'space': space, 'views': K, 'image': [W, H], 'ms': round(ms, 3),
                        'g_point_views_per_s': round(nx * ny * nz * K / ms / 1e6, 2)})
      del state
      torch.cuda.empty_cache()
  out['tsdf'] = tsdf_rows
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--rows', type=int, default=1 << 23)
  ap.add_argument('--reps', type=int, default=3)
  ap.add_argument('--extract_res', type=int, default=512)
  ap.add_argument('--sections', default='all', choices=('all', 'components', 'simplify', 'texture', 'trace',
                                                             'contracted'))
  ap.add_argument('--trace_views', type=int, default=4)
  ap.add_argument('--simplify_faces', type=int, default=1_000_000)
  ap.add_argument('--texture_faces', type=int, default=1_000_000)
  ap.add_argument('--texture_launches', type=int, default=20)
  ap.add_argument('--texture_extract_size', type=int, default=16384)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  lib.require_device()
  res = {'device': device_info(), 'query': {}, 'mc': [], 'extract': None}
  if args.sections in ('components', 'simplify', 'texture', 'trace', 'contracted'):
    b = configs.bundle_360()
    model = models.Model(b)
    model.init(seed=0)
    bbox = mesh.default_bbox(b)
    grid, _ = mesh.density_grid(model, bbox, args.extract_res)
    level = float(grid.median())
    del grid
    torch.cuda.empty_cache()
    section = {'components': bench_components_section, 'simplify': bench_simplify_section,
               'texture': bench_texture_section, 'trace': bench_trace_section,
               'contracted': bench_contracted_section}[args.sections]
    res = {'device': res['device'], 'level': level, args.sections: section(model, bbox, level, args),
           'device_after': device_info()}
    emit(res, args.out)
    return
  for name, make in (('360', configs.bundle_360), ('blender_256', configs.bundle_blender_256)):
    res['query'][name] = bench_query(make(), args.rows, args.reps)
    torch.cuda.empty_cache()
  for n in (256, 512):
    res['mc'].append(bench_mc(n, args.reps))
    torch.cuda.empty_cache()
  b = configs.bundle_360()
  model = models.Model(b)
  model.init(seed=0)
  bbox = mesh.default_bbox(b)
  grid, _ = mesh.density_grid(model, bbox, args.extract_res)
  level = float(grid.median())
  del grid
  torch.cuda.empty_cache()
  t, (v, f) = timed(lambda: mesh.extract_mesh(model, bbox, args.extract_res, level), 1)
  res['extract'] = {'config': '360.gin NerfMLP, random init', 'grid': args.extract_res, 'level': level,
                    's': round(t, 3), 'vertices': int(v.shape[0]), 'faces': int(f.shape[0])}
  del v, f
  torch.cuda.empty_cache()
  color = {'query': {}, 'mc_normals': [], 'extract': {'plain_s': [], 'colors_s': []}}
  for name, make in (('360', configs.bundle_360), ('blender_256', configs.bundle_blender_256)):
    color['query'][name] = bench_query(make(), args.rows, args.reps, radiance=True)
    torch.cuda.empty_cache()
  for n in (256, 512):
    color['mc_normals'].append(bench_mc_normals(n, 20))
    torch.cuda.empty_cache()
  mesh.extract_mesh(model, bbox, args.extract_res, level, colors=True)      # warm-up of the colour query's shapes
  torch.cuda.empty_cache()
  for _ in range(args.reps):
    for key, colors in (('plain_s', False), ('colors_s', True)):
      t, out = timed(lambda: mesh.extract_mesh(model, bbox, args.extract_res, level, colors=colors), 1)
      color['extract'][key].append(round(t, 3))
      color['extract']['vertices'] = int(out[0].shape[0])
      del out
      torch.cuda.empty_cache()
  res['color'] = color
  torch.cuda.empty_cache()
  res['components'] = bench_components_section(model, bbox, level, args)
  res['device_after'] = device_info()
  emit(res, args.out)


def emit(res, path):
  line = json.dumps(res)
  print(line, flush=True)
  if path:
    with open(path, 'w') as fh:
      fh.write(line + '\n')


if __name__ == '__main__':
  main()
