"""GPU checks of mesh evaluation (csrc/mesh_trace.cu, ops.mesh_bvh / ops.mesh_trace, mesh.render_mesh /
evaluate_mesh, extract_mesh.py with Config.mesh_eval): the BVH bit for bit against tests/mesh_trace_ref.py, the trace
against its fp64 brute force, watertightness, determinism, argument checks, camera models, shading and the script."""
import dataclasses
import math
import os
import sys

import numpy as np
import pytest
import torch

import mesh_trace_ref as ref
from test_mesh_trace_cpu import check_tree, degenerate_cases

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def mods():
  from multinerf_b200 import lib, mesh, ops
  lib.require_device()
  return ops, mesh


def mc_mesh(ops, sdf, lo=-1.0, hi=1.0, n=48):
  """Marching cubes of sdf(x, y, z) > 0 (numpy, world units) on an n^3 grid of [lo, hi]^3 -> (vertices, faces, h)
  on the device, vertices in world units."""
  h = (hi - lo) / (n - 1)
  ax = lo + np.arange(n) * h
  z, y, x = np.meshgrid(ax, ax, ax, indexing='ij')
  grid = torch.tensor(sdf(x, y, z), dtype=torch.float32, device='cuda')
  v, f = ops.marching_cubes(grid, 0.0)
  return (v * h + lo).contiguous(), f, h


def sphere_sdf(r=0.8):
  return lambda x, y, z: r - np.sqrt(x * x + y * y + z * z)


def torus_sdf(R=0.6, r=0.25):
  return lambda x, y, z: r - np.sqrt((np.sqrt(x * x + y * y) - R) ** 2 + z * z)


def _host(t):
  return t.detach().cpu().numpy()


def check_bvh(ops, v, f):
  bvh = ops.mesh_bvh(torch.as_tensor(v, device='cuda'), torch.as_tensor(f, device='cuda'))
  torch.cuda.synchronize()
  want = ref.build(_host(torch.as_tensor(v)), _host(torch.as_tensor(f)))
  F = len(f)
  assert np.array_equal(_host(bvh.leaf_face), want['leaf_face'])
  if F > 1:
    assert np.array_equal(_host(bvh.keys), want['keys'])
    assert np.array_equal(_host(bvh.nodes).view(np.int32), want['nodes'].view(np.int32))
    assert np.array_equal(_host(bvh.parent), want['parent'])
  check_tree(want, F)
  return bvh


@pytest.mark.parametrize('case', degenerate_cases(), ids=lambda c: c[0])
def test_bvh_bit_exact_on_degenerate_inputs(mods, case):
  ops, _ = mods
  _, v, f = case
  check_bvh(ops, v, f)


def test_bvh_bit_exact_on_mc_sphere_and_permuted_soup(mods):
  ops, _ = mods
  v, f, _ = mc_mesh(ops, sphere_sdf(), n=40)
  assert len(f) > 1000
  check_bvh(ops, v, f)
  rng = np.random.default_rng(0)
  vs, fs = degenerate_cases()[0][1:]
  check_bvh(ops, vs, fs[rng.permutation(len(fs))])


def _random_rays(rng, N, inside_frac=0.2):
  o = rng.uniform(-1.5, 1.5, (N, 3))
  inside = rng.uniform(size=N) < inside_frac
  o[inside] = rng.uniform(-0.4, 0.4, (inside.sum(), 3))
  target = rng.uniform(-0.9, 0.9, (N, 3))
  d = (target - o) * rng.uniform(0.2, 5.0, (N, 1))          # directions of any length: t is along them
  near = np.zeros(N)
  far = np.full(N, np.inf)
  cut = rng.uniform(size=N) < 0.3                          # intervals that cut hits off
  near[cut] = rng.uniform(0.0, 1.0, cut.sum())
  far[cut] = near[cut] + rng.uniform(0.0, 1.0, cut.sum())
  return (o.astype(np.float32), d.astype(np.float32), near.astype(np.float32), far.astype(np.float32))


def test_trace_against_brute_force(mods):
  """Several hundred thousand rays: outside the exemptions the face is the brute force's, t within 1e-5 relative
  and bary within 1e-3, and a miss is a miss.  The fp32 edge functions are taken of corners relative to the origin,
  so they lose about log2(distance / edge length) bits to cancellation (5 here) on top of fp32 rounding: the bary
  error reached 1.8e-4 on an H100."""
  ops, _ = mods
  rng = np.random.default_rng(1)
  for sdf, n in ((sphere_sdf(), 24), (torus_sdf(), 28)):
    v, f, _ = mc_mesh(ops, sdf, n=n)
    bvh = ops.mesh_bvh(v, f)
    o, d, ne, fa = _random_rays(rng, 150_000)
    face, t, bary = ops.mesh_trace(bvh, *(torch.as_tensor(x, device='cuda') for x in (o, d, ne, fa)))
    bf, bt, bb, ex = ref.brute_force(_host(v), _host(f), o, d, ne, fa, chunk=512, device='cuda', face_block=4096)
    face, t, bary = _host(face), _host(t), _host(bary)
    keep = ~ex
    assert keep.mean() > 0.9
    assert (face[keep] == bf[keep]).all(), np.nonzero(face[keep] != bf[keep])
    hit = keep & (bf >= 0)
    assert hit.sum() > 10000 and (bf[keep] < 0).sum() > 10000
    assert (np.abs(t[hit] - bt[hit]) <= 1e-5 * np.maximum(np.abs(bt[hit]), 1)).all()
    assert np.abs(bary[hit] - bb[hit]).max() <= 1e-3
    miss = keep & (bf < 0)
    assert np.isinf(t[miss]).all() and (bary[miss] == 0).all()


@pytest.mark.parametrize('shape', ['sphere', 'torus'])
def test_watertight(mods, shape):
  """Origins inside a closed mesh, rays aimed exactly at fp32 vertices, at edge midpoints and in random directions:
  every ray hits (far = inf)."""
  ops, _ = mods
  sdf = sphere_sdf() if shape == 'sphere' else torus_sdf()
  v, f, _ = mc_mesh(ops, sdf, n=36)
  bvh = ops.mesh_bvh(v, f)
  rng = np.random.default_rng(2)
  V = v.shape[0]
  if shape == 'sphere':
    origins = rng.uniform(-0.3, 0.3, (64, 3))
  else:
    a = rng.uniform(0, 2 * np.pi, 64)
    origins = np.stack([0.6 * np.cos(a), 0.6 * np.sin(a), np.zeros(64)], -1) + rng.uniform(-0.05, 0.05, (64, 3))
  origins = torch.tensor(origins, dtype=torch.float32, device='cuda')
  fl = f.long()
  mids = (v[fl[:, 0]] + v[fl[:, 1]]) / 2
  for targets in (v, mids):
    for k in range(0, 64, 16):
      o = origins[k:k + 16, None, :].expand(-1, len(targets), -1).reshape(-1, 3).contiguous()
      d = (targets[None].expand(16, -1, -1).reshape(-1, 3) - o).contiguous()
      N = o.shape[0]
      face, t, _ = ops.mesh_trace(bvh, o, d, torch.zeros(N, device='cuda'), torch.full((N,), math.inf, device='cuda'))
      assert bool((face >= 0).all()), f'{int((face < 0).sum())} of {N} rays aimed at {V} vertices or midpoints missed'
  d = torch.tensor(rng.normal(size=(200_000, 3)), dtype=torch.float32, device='cuda')
  o = origins[torch.arange(200_000, device='cuda') % 64]
  face, _, _ = ops.mesh_trace(bvh, o, d, torch.zeros(200_000, device='cuda'),
                              torch.full((200_000,), math.inf, device='cuda'))
  assert bool((face >= 0).all())


def test_deterministic_and_permutation(mods):
  ops, _ = mods
  v, f, _ = mc_mesh(ops, torus_sdf(), n=28)
  rng = np.random.default_rng(3)
  o, d, ne, fa = (torch.as_tensor(x, device='cuda') for x in _random_rays(rng, 100_000))
  a = ops.mesh_trace(ops.mesh_bvh(v, f), o, d, ne, fa)
  b = ops.mesh_trace(ops.mesh_bvh(v, f), o, d, ne, fa)
  for x, y in zip(a, b):
    assert torch.equal(x, y)
  perm = torch.tensor(rng.permutation(f.shape[0]), device='cuda')
  inv = torch.argsort(perm)
  c = ops.mesh_trace(ops.mesh_bvh(v, f[perm].contiguous()), o, d, ne, fa)
  _, _, _, ex = ref.brute_force(_host(v), _host(f), *(_host(x) for x in (o, d, ne, fa)), chunk=512, device='cuda')
  unique = torch.as_tensor(~ex, device='cuda')
  hit = (a[0] >= 0) & unique
  assert torch.equal(a[1][unique], c[1][unique])
  assert torch.equal(a[0][hit], perm[c[0][hit].long()].int())
  assert torch.equal(inv[a[0][hit].long()].int(), c[0][hit])


def test_argument_checks_and_tiny_meshes(mods):
  ops, _ = mods
  v = torch.tensor([[-1, -1, 0], [1, -1, 0], [0, 1, 0], [0, 0, 1]], dtype=torch.float32, device='cuda')
  f = torch.tensor([[0, 1, 2]], dtype=torch.int32, device='cuda')
  with pytest.raises(ValueError, match='outside'):
    ops.mesh_bvh(v, torch.tensor([[0, 1, 4]], dtype=torch.int32, device='cuda'))
  with pytest.raises(ValueError, match='outside'):
    ops.mesh_bvh(v, torch.tensor([[0, -1, 2]], dtype=torch.int32, device='cuda'))
  bad = v.clone()
  bad[3, 1] = float('nan')
  with pytest.raises(ValueError, match='finite'):
    ops.mesh_bvh(bad, f)
  bad[3, 1] = float('inf')
  with pytest.raises(ValueError, match='finite'):
    ops.mesh_bvh(bad, f)
  o = torch.tensor([[0.0, 0.0, -1.0], [0.0, 0.0, -1.0], [5.0, 5.0, -1.0], [float('nan'), 0, -1], [0, 0, -1.0]],
                   device='cuda')
  d = torch.tensor([[0, 0, 2.0], [0, 0, 1.0], [0, 0, 1.0], [0, 0, 1.0], [0, 0, float('inf')]], device='cuda')
  ne, fa = torch.zeros(5, device='cuda'), torch.full((5,), 10.0, device='cuda')
  face, t, bary = ops.mesh_trace(ops.mesh_bvh(v, f[:0]), o, d, ne, fa)                   # F = 0: all miss
  assert (face == -1).all() and torch.isinf(t).all() and (bary == 0).all()
  face, t, bary = ops.mesh_trace(ops.mesh_bvh(v, f), o, d, ne, fa)                       # F = 1: the root is the leaf
  assert face.tolist() == [0, 0, -1, -1, -1]
  assert t[:2].tolist() == [0.5, 1.0]
  # (0, 0, 0) = 1/4 v0 + 1/4 v1 + 1/2 v2
  assert torch.allclose(bary[:2], torch.tensor([[0.25, 0.5]] * 2, device='cuda'))
  f2 = torch.tensor([[0, 1, 2], [0, 1, 3]], dtype=torch.int32, device='cuda')
  face, t, _ = ops.mesh_trace(ops.mesh_bvh(v, f2), o, d, ne, fa)
  assert face.tolist() == [0, 0, -1, -1, -1]


def _camera_rays(camtype_name, W=120, H=90):
  from multinerf_b200 import camera_utils, utils
  focal = 0.5 * W / math.tan(0.5 * 0.9)
  p2c = camera_utils.get_pixtocam(focal, W, H)
  eye = np.array([0.3, -2.6, 0.9])
  z = eye / np.linalg.norm(eye)
  x = np.cross([0, 0, 1.0], z)
  x /= np.linalg.norm(x)
  y = np.cross(z, x)
  c2w = np.concatenate([np.stack([x, y, z], 1), eye[:, None]], 1)
  dist = {'k1': 0.05, 'k2': -0.02, 'p1': 0.001, 'p2': -0.001} if camtype_name == 'opencv' else None
  camtype = (camera_utils.ProjectionType.FISHEYE if camtype_name == 'fisheye' else
             camera_utils.ProjectionType.PERSPECTIVE)
  xs, ys = camera_utils.pixel_coordinates(W, H)
  meta = lambda val: np.full((H, W, 1), val, np.float32)
  pixels = utils.Pixels(pix_x_int=xs, pix_y_int=ys, lossmult=meta(1), near=meta(0.5), far=meta(10.0),
                        cam_idx=np.zeros((H, W, 1), np.int32))
  rays = camera_utils.cast_ray_batch((p2c, c2w, dist, None), pixels, camtype)
  rays.near = torch.as_tensor(rays.near, device='cuda')
  rays.far = torch.as_tensor(rays.far, device='cuda')
  return rays


@pytest.mark.parametrize('camtype', ['perspective', 'opencv', 'fisheye'])
def test_camera_models_against_analytic_sphere(mods, camtype):
  ops, mesh = mods
  v, f, h = mc_mesh(ops, sphere_sdf(0.8), n=49)
  bvh = ops.mesh_bvh(v, f)
  rays = _camera_rays(camtype)
  r = mesh.render_mesh(v, f, bvh, rays, bg=1.0)
  o, d = rays.origins.double(), rays.directions.double()
  a = (d * d).sum(-1)
  b = (o * d).sum(-1)
  c = (o * o).sum(-1) - 0.64
  disc = b * b - a * c
  t_true = (-b - disc.clamp_min(0).sqrt()) / a
  # the line's closest distance to the centre, against the radius: more than a cell inside or outside the silhouette
  miss_dist = ((o - (b / a)[..., None] * d) ** 2).sum(-1).sqrt() - 0.8
  sure_hit = miss_dist < -h
  sure_miss = miss_dist > h
  assert bool(r['hit'][sure_hit].all()) and not bool(r['hit'][sure_miss].any())
  assert int(sure_hit.sum()) > 1000
  err = (r['distance'].double() - t_true).abs() * a.sqrt()
  assert float(err[sure_hit].max()) <= h
  assert bool(torch.isinf(r['distance'][~r['hit']]).all())


def _sphere_colour(points):
  """SyntheticScene.colour's sphere formula at points on the sphere."""
  n = torch.nn.functional.normalize(points, dim=-1)
  return 0.5 + 0.5 * n * torch.tensor([1.0, 0.8, 0.6], device=points.device)


def test_shading_vertex_colours_and_texture(mods, tmp_path):
  """The radius-0.8 sphere coloured by SyntheticScene's formula, as vertex colours and as a baked texture, over
  _write_scene's test views: the sphere's pixels within 0.08 of the test image, and the texture's mean error below
  the vertex colours'."""
  ops, mesh = mods
  from multinerf_b200 import configs, datasets
  from test_gpu_mesh import _write_scene
  data = str(tmp_path / 'scene')
  _write_scene(data, n_test=3, W=80, H=60)
  config = configs.load_config(gin_bindings=[f"Config.data_dir = '{data}'", "Config.dataset_loader = 'blender'",
                                             'Config.near = 1.5', 'Config.far = 5.0']).config
  ds = datasets.load_dataset('test', data, dataclasses.replace(config, render_path=False), device='cuda')
  # coarse cells, so the vertex colours' linear blend of a nonlinear colour is visibly worse than the texture
  v, f, h = mc_mesh(ops, sphere_sdf(0.8), n=17)
  n = torch.nn.functional.normalize(v, dim=-1)
  rgb = (_sphere_colour(v).clamp(0, 1) * 255).round().to(torch.uint8)
  uv, tex = mesh.bake_texture(v, f, n, 2048, lambda p, nn: (_sphere_colour(p).clamp(0, 1) * 255).round()
                              .to(torch.uint8))
  bvh = ops.mesh_bvh(v, f)
  errs = {}
  for name, kw in (('vertex', dict(rgb=rgb)), ('texture', dict(uv=uv, texture=tex))):
    total, count = 0.0, 0
    for idx in range(ds.size):
      rays = ds.generate_ray_batch(idx).rays
      r = mesh.render_mesh(v, f, bvh, rays, normals=n, bg=1.0, **kw)
      gt = torch.as_tensor(ds.images[idx], device='cuda')
      # pixels whose whole footprint is on the sphere: hit, and the analytic ray hits well inside the silhouette
      o, d = rays.origins, rays.directions
      b = (o * d).sum(-1) / (d * d).sum(-1)
      closest = (o - b[..., None] * d).norm(dim=-1)
      inner = r['hit'] & (closest < 0.8 - 2 * h)
      e = (r['rgb'] - gt).abs().max(-1).values[inner]
      assert float(e.max()) < 0.08, (name, idx, float(e.max()))
      total += float(e.sum())
      count += int(inner.sum())
    errs[name] = total / count
  assert errs['texture'] < errs['vertex'], errs
  # normals: unit length where hit, zero elsewhere
  r = mesh.render_mesh(v, f, bvh, ds.generate_ray_batch(0).rays, bg=1.0)
  nn = r['normals'].norm(dim=-1)
  assert torch.allclose(nn[r['hit']], torch.ones_like(nn[r['hit']]), atol=1e-5) and bool((nn[~r['hit']] == 0).all())
  assert r['rgb'] is None


def _train(tmp_path, steps=100):
  sys.path.insert(0, ROOT)
  import train as train_script
  from test_gpu_mesh import _write_scene
  data, ckpt = str(tmp_path / 'scene'), str(tmp_path / 'ckpt')
  _write_scene(data)
  bindings = [f"Config.data_dir = '{data}'", f"Config.checkpoint_dir = '{ckpt}'", 'Config.batch_size = 1024',
              f'Config.max_steps = {steps}', 'Config.print_every = 20', f'Config.checkpoint_every = {steps}',
              f'Config.train_render_every = {10 * steps}', 'Config.render_chunk_size = 512', 'Config.near = 1.5',
              'Config.lr_init = 5e-3', 'Config.lr_final = 5e-4',
              'Config.far = 5.0', "Config.dataset_loader = 'blender'", 'Model.num_prop_samples = 32',
              'Model.num_nerf_samples = 16', 'PropMLP.net_depth = 2', 'PropMLP.net_width = 64',
              'NerfMLP.net_depth = 4', 'NerfMLP.net_width = 128', 'NerfMLP.bottleneck_width = 64',
              'NerfMLP.net_width_viewdirs = 64', 'PropMLP.disable_density_normals = True',
              'PropMLP.disable_rgb = True', 'NerfMLP.disable_density_normals = True']
  argv = [f'--gin_bindings={b}' for b in bindings]
  train_script.main(argv)
  return argv, ckpt, steps


def test_extract_mesh_script_mesh_eval(tmp_path, capsys):
  """extract_mesh.py with mesh_eval: the renders and metric files for the density and TSDF methods, with and without
  colour and with a texture; the PLY and OBJ bytes as without mesh_eval."""
  from multinerf_b200 import lib
  lib.require_device()
  argv, ckpt, steps = _train(tmp_path)
  import extract_mesh as mesh_script
  from PIL import Image
  capsys.readouterr()
  base = argv + ['--gin_bindings=Config.mesh_resolution = 40', '--gin_bindings=Config.mesh_level = 0.5']
  eval_dir = os.path.join(ckpt, 'mesh', f'eval_step_{steps}')
  variants = [
      ('density_plain', []),
      ('density_vertex', ['--gin_bindings=Config.mesh_vertex_colors = True']),
      ('density_texture', ['--gin_bindings=Config.mesh_target_faces = 2000',
                           '--gin_bindings=Config.mesh_texture_size = 512']),
      ('tsdf_plain', ["--gin_bindings=Config.mesh_method = 'tsdf'"]),
      ('tsdf_vertex', ["--gin_bindings=Config.mesh_method = 'tsdf'", '--gin_bindings=Config.mesh_vertex_colors = True']),
  ]
  mesh_dir = os.path.join(ckpt, 'mesh')
  for name, extra in variants:
    for p in os.listdir(mesh_dir) if os.path.isdir(mesh_dir) else []:       # the previous variant's files
      if os.path.isfile(os.path.join(mesh_dir, p)):
        os.remove(os.path.join(mesh_dir, p))
    path = mesh_script.main(base + extra)
    stem = os.path.splitext(path)[0]
    outputs = [p for p in (path, stem + '.obj', stem + '.png') if os.path.exists(p)]
    plain = {p: open(p, 'rb').read() for p in outputs}
    for p in outputs:
      os.remove(p)
    capsys.readouterr()
    assert mesh_script.main(base + extra + ['--gin_bindings=Config.mesh_eval = True']) == path
    printed = capsys.readouterr().out
    for p in outputs:
      assert open(p, 'rb').read() == plain[p], (name, p)
    coloured = name.endswith(('vertex', 'texture'))
    names = ['nerf_psnr', 'nerf_ssim', 'coverage', 'spurious', 'depth_abs_rel'] + (['psnr', 'ssim'] if coloured else [])
    for m in names:
      vals = np.array([float(x) for x in open(os.path.join(eval_dir, f'metric_{m}.txt')).read().split()])
      assert len(vals) == 2 and np.isfinite(vals).all(), (name, m, vals)
      lo, hi = {'coverage': (0, 1), 'spurious': (0, 1), 'ssim': (-1, 1), 'nerf_ssim': (-1, 1),
                'depth_abs_rel': (0, np.inf), 'psnr': (0, np.inf), 'nerf_psnr': (0, np.inf)}[m]
      assert ((vals >= lo) & (vals <= hi)).all(), (name, m, vals)
      assert f'mesh eval {m}' in printed
    assert os.path.exists(os.path.join(eval_dir, 'metric_psnr.txt')) == coloured
    for idx in range(2):
      assert os.path.exists(os.path.join(eval_dir, f'normals_{idx:03d}.png'))
      dist = np.asarray(Image.open(os.path.join(eval_dir, f'distance_{idx:03d}.tiff')))
      assert dist.shape == (30, 40)
      assert os.path.exists(os.path.join(eval_dir, f'color_{idx:03d}.png')) == coloured
    assert 'BVH build' in printed and 'NeRF rendering' in printed
    for p in os.listdir(eval_dir):
      os.remove(os.path.join(eval_dir, p))
