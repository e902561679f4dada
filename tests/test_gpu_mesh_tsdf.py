"""TSDF mesh extraction on the GPU: mnrf_tsdf_integrate against the fp64 fusion of tests/tsdf_ref.py with a bound on
every element (and bit-identical however the views are split into launches), fused meshes of analytic scenes traced
on the rays of camera_utils.cast_ray_batch (closed, the right topology, on the surface, the right colours), marching
cubes over unobserved (NaN) points, and extract_mesh.py with Config.mesh_method = 'tsdf' after a short train.py run.
Needs an H100."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest
import torch

import tsdf_ref
from test_gpu_mesh import check_closed_and_wound, sphere

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def mods():
  from multinerf_b200 import lib, mesh, ops
  lib.require_device()
  return lib, ops, mesh


def _look_at(eye, target, up=(0.0, 0.0, 1.0)):
  eye = np.asarray(eye, np.float64)
  z = eye - np.asarray(target, np.float64)
  z /= np.linalg.norm(z)
  x = np.cross(up, z)
  x /= np.linalg.norm(x)
  return np.concatenate([np.stack([x, np.cross(z, x), z], 1), eye[:, None]], 1)


# ------------------------------------------------------------------ integration against fp64

CAMS = {
    'perspective': (0, None),
    'opencv': (0, {'k1': -0.06, 'k2': 0.015, 'k3': 0.0, 'p1': 1e-3, 'p2': -8e-4}),
    'fisheye': (1, {'k1': 0.02, 'k2': -0.005, 'k3': 1e-3, 'k4': -2e-4}),
}


def _views(rng, K, H, W, camtype, per_view):
  """K random views around the origin: poses, intrinsics, depth (non-finite in places), acc on both sides of 0.5
  and colours.  Returns fp32 arrays (w2c [K, 3, 4], c2p [K or 1, 3, 3], depth, acc, rgb)."""
  w2c = []
  for _ in range(K):
    c2w = _look_at(rng.normal(size=3) * 2.5, rng.normal(size=3) * 0.3)
    r = c2w[:, :3]
    w2c.append(np.concatenate([r.T, -r.T @ c2w[:, 3:]], 1))
  f = (12.0 if camtype == 1 else 30.0)
  c2p = np.stack([[[f * rng.uniform(0.9, 1.1), 0.2 * rng.normal(), W / 2 + rng.normal()],
                   [0.0, f * rng.uniform(0.9, 1.1), H / 2 + rng.normal()], [0.0, 0.0, 1.0]]
                  for _ in range(K if per_view else 1)])
  depth = rng.uniform(1.0, 4.0, (K, H, W))
  depth[rng.uniform(size=depth.shape) < 0.05] = np.nan
  depth[rng.uniform(size=depth.shape) < 0.03] = np.inf
  acc = rng.uniform(0, 1, (K, H, W))
  rgb = rng.uniform(0, 1, (K, H, W, 3))
  f32 = lambda a: np.ascontiguousarray(a, np.float32)
  return f32(np.stack(w2c)), f32(c2p), f32(depth), f32(acc), f32(rgb)


def _fuse(ops, shape, lo, h, camtype, dist, views, tau, colors, batch):
  """State after fusing `views` (numpy fp32) `batch` views per launch."""
  w2c, c2p, depth, acc, rgb = (torch.tensor(a, device='cuda') for a in views)
  nx, ny, nz = shape
  z = lambda *sh: torch.zeros(nz, ny, nx, *sh, device='cuda')
  state = [z(), z()] + ([z(3), z()] if colors else [None, None])
  K = depth.shape[0]
  for k0 in range(0, K, batch):
    sl = slice(k0, k0 + batch)
    ops.tsdf_integrate(shape, lo, h, camtype, dist, w2c[sl].contiguous(),
                       c2p if c2p.shape[0] == 1 else c2p[sl].contiguous(), depth[sl].contiguous(),
                       acc[sl].contiguous(), rgb[sl].contiguous() if colors else None, tau, *state)
  torch.cuda.synchronize()
  return state


@pytest.mark.parametrize('cam', sorted(CAMS))
@pytest.mark.parametrize('K,per_view,colors', [(1, False, True), (4, True, False), (9, True, True),
                                               (9, False, False)])
def test_tsdf_integrate_vs_fp64(mods, cam, K, per_view, colors):
  _, ops, _ = mods
  camtype, dist = CAMS[cam]
  rng = np.random.default_rng(K * 10 + per_view + 100 * camtype)
  H, W = 30, 40
  shape = (37, 29, 23)
  lo, h = (-3.6, -2.8, -2.2), 0.2              # the box holds the cameras: points behind them and off their images
  tau = 2.5 * h
  views = _views(rng, K, H, W, camtype, per_view)
  tsdf, weight, cs, cw = _fuse(ops, shape, lo, h, camtype, dist, views, tau, colors, K)
  pts = tsdf_ref.grid_points(shape, lo, h)
  rt, rw, rcs, rcw, bound, exempt = tsdf_ref.integrate(pts, views[0], views[1], views[2], views[3],
                                                       views[4] if colors else None, tau,
                                                       'fisheye' if camtype else 'perspective', dist)
  live = ~exempt
  assert live.mean() > 0.8, live.mean()
  # every branch is taken: observed points, unobserved ones, truncated and free-space values
  assert (rw[live] > 0).mean() > 0.2 and (rw[live] == 0).any()
  assert (np.abs(rt[live][rw[live] > 0]) < 1).any() and (rt[live] == 1).any()
  g = lambda t: t.reshape(-1).cpu().double().numpy()
  assert np.array_equal(g(weight)[live], rw[live])
  err = np.abs(g(tsdf) - rt)
  assert (err[live] <= bound[live]).all(), float((err - bound)[live].max())
  if colors:
    assert np.array_equal(g(cw)[live], rcw[live])
    assert (rcw[live] > 0).any()
    cerr = np.abs(cs.reshape(-1, 3).cpu().double().numpy() - rcs)
    assert (cerr[live] <= 4 * K * tsdf_ref.EPS32 * (1 + rcs[live])).all()
  # the same state whatever the launches: one view at a time, three at a time, all at once
  for batch in (1, 3):
    other = _fuse(ops, shape, lo, h, camtype, dist, views, tau, colors, batch)
    for a, b in zip((tsdf, weight, cs, cw), other):
      assert (a is None and b is None) or torch.equal(a, b), batch


def test_tsdf_integrate_rejects_bad_arguments(mods):
  lib, _, _ = mods
  L = lib.load()
  t = torch.zeros(8, device='cuda')
  m = torch.zeros(12, device='cuda')
  dm = torch.ones(1, 2, 2, device='cuda')
  P = lib.ptr

  def call(nx=2, K=1, ncam=1, camtype=0, ndc=0, tau=0.1, h=0.5, rgb=None, cs=None, cw=None, depth=dm):
    d = lib.CameraDesc(0, ncam, camtype, 0, 0, 0, 0, 0, 0, 0, 0.0, 0, ndc, 1.0, 1.0, 1.0)
    return L.mnrf_tsdf_integrate(C.byref(d), nx, 2, 2, 0.0, 0.0, 0.0, h, K, 2, 2, P(m), P(m), P(depth), P(dm),
                                 P(rgb), tau, P(t), P(t), P(cs), P(cw), lib.stream_ptr())
  assert call() == 0
  assert call(rgb=t, cs=t, cw=t) == 0
  for kw in (dict(nx=1), dict(nx=1025), dict(ncam=2), dict(camtype=2), dict(ndc=1), dict(tau=0.0),
             dict(tau=float('nan')), dict(h=-1.0), dict(rgb=t), dict(cs=t, cw=t), dict(K=-1), dict(depth=None)):
    assert call(**kw) != 0, kw
  torch.cuda.synchronize()


# ------------------------------------------------------------------ analytic scenes

def _cameras(n, radius, W, H, focal):
  """n cameras on a Fibonacci sphere looking at the origin -> (pixtocam, camtoworlds [n, 3, 4])."""
  from multinerf_b200 import camera_utils
  c2w = []
  for i in range(n):
    zc = 1 - 2 * (i + 0.5) / n
    a = i * math.pi * (3 - math.sqrt(5))
    eye = radius * np.array([math.sqrt(1 - zc * zc) * math.cos(a), math.sqrt(1 - zc * zc) * math.sin(a), zc])
    up = (0.0, 0.0, 1.0) if abs(zc) < 0.95 else (1.0, 0.0, 0.0)
    c2w.append(_look_at(eye, (0, 0, 0), up))
  return camera_utils.get_pixtocam(focal, W, H), np.stack(c2w)


SPHERE_C, SPHERE_R = np.array([0.05, -0.03, 0.02]), 0.6
TORUS_C, TORUS_R, TORUS_r = np.array([0.02, 0.03, -0.04]), 0.55, 0.22
COLOR_B = np.diag([0.2, -0.15, 0.1])


def _sdf(name, x):
  if name == 'sphere':
    return torch.linalg.norm(x - torch.tensor(SPHERE_C, device=x.device), dim=-1) - SPHERE_R
  q = x - torch.tensor(TORUS_C, device=x.device)
  return torch.hypot(torch.hypot(q[..., 0], q[..., 1]) - TORUS_R, q[..., 2]) - TORUS_r


def _color(x):
  return 0.5 + x @ torch.tensor(COLOR_B.T, device=x.device)


def _trace(name, o, d):
  """fp64 ray parameter t of the first hit of o + t d (d not normalised) and whether there is one."""
  o, d = o.double(), d.double()
  if name == 'sphere':
    oc = o - torch.tensor(SPHERE_C, device=o.device)
    a = (d * d).sum(-1)
    b = (oc * d).sum(-1)
    c = (oc * oc).sum(-1) - SPHERE_R ** 2
    disc = b * b - a * c
    t = (-b - torch.sqrt(disc.clamp_min(0))) / a
    return t, disc > 0
  # the first sign change of the exact distance on a fine march (steps of 1e-3 along unit length), then bisection
  n = torch.linalg.norm(d, dim=-1)
  ts = torch.arange(1.0, 4.2, 1e-3, device=o.device, dtype=torch.float64)
  first = torch.full_like(n, len(ts), dtype=torch.long)
  for j0 in range(0, len(ts), 256):
    tj = ts[j0:j0 + 256]
    inside = _sdf(name, o[:, None] + (tj[None, :, None] / n[:, None, None]) * d[:, None]) < 0
    j = torch.where(inside.any(1), inside.float().argmax(1) + j0, torch.full_like(first, len(ts)))
    first = torch.minimum(first, j)
  hit = (first > 0) & (first < len(ts))
  hi = ts[first.clamp(1, len(ts) - 1)]
  lo = hi - 1e-3
  for _ in range(60):
    mid = 0.5 * (lo + hi)
    inside = _sdf(name, o + (mid / n)[:, None] * d) < 0
    lo, hi = torch.where(inside, lo, mid), torch.where(inside, mid, hi)
  return 0.5 * (lo + hi) / n, hit


def _render_analytic(name, cameras, W, H):
  from multinerf_b200 import camera_utils, utils
  p2c, c2w = cameras
  xs, ys = camera_utils.pixel_coordinates(W, H)
  for k in range(len(c2w)):
    pix = utils.Pixels(pix_x_int=xs, pix_y_int=ys, lossmult=None, near=None, far=None,
                       cam_idx=np.full((H, W, 1), k, np.int32))
    rays = camera_utils.cast_ray_batch((p2c, c2w, None, None), pix)
    o, d = rays.origins.reshape(-1, 3), rays.directions.reshape(-1, 3)
    t, hit = _trace(name, o, d)
    depth = torch.where(hit, t, torch.full_like(t, 6.0)).float().view(H, W)
    acc = hit.float().view(H, W)
    rgb = torch.where(hit[:, None], _color(o.double() + t[:, None] * d.double()), torch.zeros_like(o.double()))
    yield k, depth, acc, rgb.float().view(H, W, 3)


@pytest.mark.parametrize('name,euler', [('sphere', 2), ('torus', 0)])
def test_fused_analytic_scene(mods, name, euler):
  _, ops, mesh = mods
  W, H, focal = 200, 150, 220.0
  cameras = _cameras(40, 2.6, W, H, focal)
  bbox, res, trunc = (-1.0, -1.0, -1.0, 1.0, 1.0, 1.0), 128, 3.0
  state, h = mesh.fuse_tsdf(_render_analytic(name, cameras, W, H), (cameras[0], cameras[1], None, None),
                            'perspective', bbox, res, trunc, colors=True, batch=7)
  v, f, nrm, rgb = mesh.tsdf_mesh(state, bbox, h, colors=True)
  torch.cuda.synchronize()
  V = len(v)
  assert V > 1000 and len(f) > 0
  assert torch.isfinite(v).all() and torch.isfinite(nrm).all()
  fn = f.cpu().numpy()
  assert fn.min() >= 0 and fn.max() < V
  assert len(np.unique(fn)) == V, 'unreferenced vertices'
  E = check_closed_and_wound(fn, V)
  assert V - E + len(fn) == euler
  dist = _sdf(name, v.double()).abs()
  assert float(dist.max()) <= h, (float(dist.max()), h)
  # colours: a linear field, so a fused colour is the field within the band (tau + a pixel's footprint) of the vertex
  err = (rgb.double() - (_color(v.double()).clamp(0, 1) * 255)).abs()
  bound = 255 * np.abs(COLOR_B).max() * (trunc * h + 2 * h) * math.sqrt(3) + 0.5
  assert float(err.max()) <= bound, (float(err.max()), bound)
  # normals point out of the surface
  outward = _sdf(name, v.double() + 0.5 * h * nrm.double()) > _sdf(name, v.double() - 0.5 * h * nrm.double())
  assert float(outward.double().mean()) > 0.99


# ------------------------------------------------------------------ marching cubes over unobserved points

def _mc_with_ids(lib, ops, grid):
  """(vertices, faces, normals, vertex edge ids, face cell ids) of ops.marching_cubes on `grid` at level 0."""
  L = lib.load()
  nz, ny, nx = grid.shape
  n = grid.numel()
  cut = torch.empty(3 * n, device='cuda', dtype=torch.uint8)
  tris = torch.empty(n, device='cuda', dtype=torch.uint8)
  lib.check(L.mnrf_marching_cubes(lib.MC_COUNT, nx, ny, nz, lib.ptr(grid), 0.0, lib.ptr(cut), lib.ptr(tris), None,
                                  None, None, None, lib.stream_ptr()))
  v, f, nrm = ops.marching_cubes(grid, 0.0, normals=True)
  edges = torch.nonzero(cut).view(-1)
  cells = torch.repeat_interleave(torch.arange(n, device='cuda'), tris.long())
  torch.cuda.synchronize()
  return v, f, nrm, edges, cells


def test_marching_cubes_skips_unobserved_points(mods):
  lib, ops, _ = mods
  shape = (40, 36, 38)
  full = sphere(shape, (18.3, 17.6, 19.1), 14.2)
  z0, z1 = 12, 27                           # finite z-planes: z0..z1
  nanned = full.copy()
  nanned[:z0] = np.nan
  nanned[z1 + 1:] = np.nan
  nanned[20, 5:9, 3:30] = np.nan            # and a hole inside the slab
  gf, gn = torch.tensor(full, device='cuda'), torch.tensor(nanned, device='cuda')
  v, f, nrm, edges, cells = _mc_with_ids(lib, ops, gn)
  fv, ff, _, fedges, fcells = _mc_with_ids(lib, ops, gf)
  assert len(f) > 0 and torch.isfinite(v).all() and torch.isfinite(nrm).all()
  assert len(torch.unique(f)) == len(v), 'unreferenced vertices'
  nz, ny, nx = shape
  flat = gn.view(-1)
  # no face has a cell with a NaN corner; no vertex an edge with a NaN end
  corners = torch.tensor([(i & 1) + (i >> 1 & 1) * nx + (i >> 2 & 1) * nx * ny for i in range(8)], device='cuda')
  assert not torch.isnan(flat[cells[:, None] + corners]).any()
  strides = torch.tensor([1, nx, nx * ny], device='cuda')
  p, a = edges // 3, edges % 3
  assert not torch.isnan(flat[p]).any() and not torch.isnan(flat[p + strides[a]]).any()
  # the faces are exactly the finite grid's faces in the cells with eight finite corners, edge for edge
  finite_cell = ~torch.isnan(flat[fcells[:, None] + corners]).any(-1)
  want = fedges[ff.long()][finite_cell]
  assert torch.equal(edges[f.long()], want) and torch.equal(cells, fcells[finite_cell])
  # the vertices on those edges sit where the finite grid puts them
  rank = torch.searchsorted(fedges, edges)
  assert torch.equal(fedges[rank], edges) and torch.equal(v, fv[rank])


# ------------------------------------------------------------------ extract_mesh.py end to end

def test_extract_mesh_script_tsdf(tmp_path, capsys):
  sys.path.insert(0, ROOT)
  from multinerf_b200 import lib
  lib.require_device()
  import extract_mesh as mesh_script
  import train as train_script
  from test_gpu_mesh import _write_scene
  from test_mesh_color_cpu import read_ply_props
  data, ckpt = str(tmp_path / 'scene'), str(tmp_path / 'ckpt')
  _write_scene(data)
  steps = 60
  bindings = [f"Config.data_dir = '{data}'", f"Config.checkpoint_dir = '{ckpt}'", 'Config.batch_size = 1024',
              f'Config.max_steps = {steps}', 'Config.print_every = 20', f'Config.checkpoint_every = {steps}',
              f'Config.train_render_every = {10 * steps}', 'Config.lr_init = 5e-3', 'Config.lr_final = 5e-4',
              'Config.render_chunk_size = 512', 'Config.near = 1.5', 'Config.far = 5.0',
              "Config.dataset_loader = 'blender'", 'Model.num_prop_samples = 32', 'Model.num_nerf_samples = 16',
              'PropMLP.net_depth = 2', 'PropMLP.net_width = 64', 'NerfMLP.net_depth = 4', 'NerfMLP.net_width = 128',
              'NerfMLP.bottleneck_width = 64', 'NerfMLP.net_width_viewdirs = 64',
              'PropMLP.disable_density_normals = True', 'PropMLP.disable_rgb = True',
              'NerfMLP.disable_density_normals = True']
  argv = [f'--gin_bindings={b}' for b in bindings]
  train_script.main(argv)
  capsys.readouterr()
  path = mesh_script.main(argv + ['--gin_bindings=Config.mesh_resolution = 40',
                                  "--gin_bindings=Config.mesh_method = 'tsdf'",
                                  '--gin_bindings=Config.mesh_vertex_colors = True'])
  printed = capsys.readouterr().out
  assert path == os.path.join(ckpt, 'mesh', f'mesh_step_{steps}.ply') and os.path.exists(path)
  line = [l for l in printed.splitlines() if 'vertices,' in l][-1]
  assert '10 views fused' in line
  nv, nf = int(line.split(' vertices,')[0]), int(line.split(' vertices, ')[1].split(' faces')[0])
  props, f = read_ply_props(path)
  assert list(props) == ['x', 'y', 'z', 'nx', 'ny', 'nz', 'red', 'green', 'blue']
  assert len(props['x']) == nv and f.shape == (nf, 3)
  assert all(np.isfinite(props[k]).all() for k in ('x', 'y', 'z', 'nx', 'ny', 'nz'))
  if nf:
    assert f.min() >= 0 and f.max() < nv
    assert bool((np.abs(np.stack([props['x'], props['y'], props['z']], 1)) <= 1.5 + 1e-5).all())
