"""Mesh extraction on the GPU: the point form of the encoder against an fp64 reference with a bound on every
element, Model.query_density against the oracle's MLP, marching cubes on analytic grids (closed, consistently
wound, the right topology and volume, deterministic), their composition in mesh.extract_mesh, and extract_mesh.py
after a short train.py run.  Needs an H100."""
import ctypes as C
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

import encode_ref as E
from model_parity import mini360, plumbing_blender, torch_tree
from oracle import o_models

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def mods():
  from multinerf_b200 import lib, mesh, models, ops
  lib.require_device()
  return lib, ops, models, mesh


# ------------------------------------------------------------------ point encode

def point_reference(points, var, basis, *, min_deg, max_deg, warp_contract, disable_integration):
  """fp64 value and bound of every feature of the Gaussian (point, var I), staged like the kernel: the contraction
  with the covariance through the Jacobian, the lift onto the basis, the IPE."""
  p = torch.as_tensor(points).double()
  v32 = float(np.float32(var))
  mean = [E._V(p[:, i:i + 1]) for i in range(3)]
  cov = [[E._V(torch.full_like(p[:, :1], v32 if i == j else 0.0)) for j in range(3)] for i in range(3)]
  if warp_contract:
    mean, cov = E._contract(mean, cov)
  lm, lv = E._lift(mean, cov, torch.as_tensor(basis).double(), disable_integration)
  feat, bound = E._features(lm.val, lv.val, lm.err, lv.err, min_deg, max_deg)
  return feat[:, 0], bound[:, 0], E.bf16_bound(feat, bound)[:, 0]


@pytest.mark.parametrize('warp_contract,disable_integration,var', [
    (False, False, 1e-4), (True, False, 1e-4), (True, True, 1e-4), (True, False, 0.0), (False, False, 0.0),
    (True, False, 3e-2)])
def test_encode_points_vs_fp64(mods, warp_contract, disable_integration, var):
  lib, ops, _, _ = mods
  from multinerf_b200 import geopoly
  basis = np.ascontiguousarray(geopoly.generate_basis('octahedron', 2), dtype=np.float32)
  rng = np.random.default_rng(3)
  # inside the unit ball, outside it, and far out (the contraction's large-|x| regime); 1001 points: ragged groups
  pts = np.concatenate([rng.uniform(-0.57, 0.57, (400, 3)), rng.uniform(-3, 3, (400, 3)),
                        rng.normal(size=(201, 3)) * 50]).astype(np.float32)
  min_deg, max_deg = 0, 12
  p = torch.tensor(pts, device='cuda')
  feat, f32 = ops.encode_points(p, var, torch.tensor(basis, device='cuda'), min_deg=min_deg, max_deg=max_deg,
                                warp_contract=warp_contract, disable_integration=disable_integration, want_f32=True)
  torch.cuda.synchronize()
  ref, bound, bound_bf = point_reference(pts, var, basis, min_deg=min_deg, max_deg=max_deg,
                                         warp_contract=warp_contract, disable_integration=disable_integration)
  F = ref.shape[1]
  live = bound <= E.VACUOUS
  assert float(live.double().mean()) > 0.5
  err = (f32.cpu().double() - ref).abs()
  assert bool((err[live] <= bound[live]).all()), float((err - bound)[live].max())
  errb = (feat[:, :F].float().cpu().double() - ref).abs()
  assert bool((errb[live] <= bound_bf[live]).all()), float((errb - bound_bf)[live].max())
  assert bool((feat[:, F:] == 0).all())                 # zero-filled pad columns


def test_encode_points_rejects_bad_descriptors(mods):
  lib, ops, _, _ = mods
  L = lib.load()
  pts = torch.zeros(8, 3, device='cuda')
  basis = torch.zeros(21, 3, device='cuda')
  feat = torch.zeros(8, 512, device='cuda', dtype=torch.bfloat16)

  def call(var=1e-3, **kw):
    f = dict(num_rays=8, num_samples=1, raydist_fn=0, ray_shape=0, warp_contract=0, disable_integration=0,
             basis_k=21, min_deg=0, max_deg=12, ld_feat=512, feat_cols=512)
    f.update(kw)
    d = lib.EncodeDesc(**f)
    return L.mnrf_encode_points(C.byref(d), lib.ptr(pts), var, lib.ptr(basis), lib.ptr(feat), None, lib.stream_ptr())
  assert call() == 0
  for kw in (dict(num_samples=2), dict(raydist_fn=1), dict(ray_shape=1), dict(feat_cols=500),
             dict(feat_cols=256), dict(ld_feat=256), dict(num_rays=-1)):
    assert call(**kw) != 0, kw
  assert call(var=-1.0) != 0
  assert call(var=float('nan')) != 0
  d = lib.EncodeDesc(8, 1, 0, 0, 0, 0, 21, 0, 12, 512, 512)
  assert L.mnrf_encode_points(C.byref(d), None, 1e-3, lib.ptr(basis), lib.ptr(feat), None, lib.stream_ptr()) != 0
  torch.cuda.synchronize()


# ------------------------------------------------------------------ query_density

def _bundle(which):
  if which == 'plumbing':
    return plumbing_blender()
  b = mini360()
  if which in ('softplus', 'silu'):
    b.nerf_mlp.net_activation = b.prop_mlp.net_activation = which
  if which == 'viewindep':
    b.model.use_viewdirs = False
  return b


@pytest.mark.parametrize('which,N', [('mini360', 3000), ('plumbing', 4096), ('plumbing', 300), ('softplus', 2000),
                                     ('silu', 2000), ('viewindep', 2000)])
def test_query_density_vs_oracle(mods, which, N):
  """mini360: 360.gin's layout with the contraction; plumbing: blender_256 (bounded), whose 256-wide ReLU trunk
  runs as one chained launch at 4096 rows and layer by layer at 300."""
  lib, ops, models, _ = mods
  bundle = _bundle(which)
  model = models.Model(bundle)
  model.init(seed=7)
  rng = np.random.default_rng(11)
  pts = np.concatenate([rng.uniform(-1, 1, (N // 2, 3)), rng.uniform(-4, 4, (N - N // 2, 3))]).astype(np.float32)
  var = 2e-4
  chained = model._use_chain(model.plans['NerfMLP_0'], N)
  assert chained == (which == 'plumbing' and N >= 512)
  dens = model.query_density(torch.tensor(pts, device='cuda'), var)
  torch.cuda.synchronize()
  assert dens.shape == (N,) and dens.dtype == torch.float32
  tree = torch_tree(model.export_flax())['NerfMLP_0']
  means = torch.tensor(pts)[:, None, :]
  covs = (torch.eye(3) * float(np.float32(var))).expand(N, 1, 3, 3).contiguous()
  vd = None
  if bundle.model.use_viewdirs:
    vd = torch.nn.functional.normalize(torch.tensor(rng.normal(size=(N, 3)).astype(np.float32)), dim=-1)
  with torch.no_grad() if bundle.nerf_mlp.disable_density_normals else torch.enable_grad():
    out = o_models.mlp_apply(tree, bundle.nerf_mlp, model.plans['NerfMLP_0'].basis, (means, covs), viewdirs=vd,
                             bf16=True)
  ref = out['density'][:, 0].detach()
  err = (dens.cpu() - ref).abs() / (1.0 + ref.abs())
  assert float(err.max()) < 0.1 and float(err.mean()) < 5e-3, (float(err.max()), float(err.mean()))


# ------------------------------------------------------------------ marching cubes on analytic grids

def _coords(shape):
  nz, ny, nx = shape
  z, y, x = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing='ij')
  return x.astype(np.float64), y.astype(np.float64), z.astype(np.float64)


def sphere(shape, c, r):
  x, y, z = _coords(shape)
  return (r - np.sqrt((x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2)).astype(np.float32)


def torus(shape, c, R, r):
  x, y, z = _coords(shape)
  q = np.sqrt((x - c[0]) ** 2 + (y - c[1]) ** 2) - R
  return (r - np.sqrt(q ** 2 + (z - c[2]) ** 2)).astype(np.float32)


def smooth_field(shape, seed):
  """A sum of random low-frequency waves, pushed below the level near the grid boundary."""
  rng = np.random.default_rng(seed)
  x, y, z = _coords(shape)
  nz, ny, nx = shape
  f = np.zeros(shape)
  for _ in range(12):
    k = rng.normal(size=3) * 0.35
    f += np.cos(k[0] * x + k[1] * y + k[2] * z + rng.uniform(0, 2 * np.pi))
  edge = np.minimum.reduce([x, nx - 1 - x, y, ny - 1 - y, z, nz - 1 - z])
  return (f - 20.0 * np.exp(-edge / 2.0)).astype(np.float32)


def cut_edges(grid, level):
  """(edge ids in order, fp32 crossing t) computed in numpy: edge id = 3 * point + axis."""
  inside = grid > level
  ids, ts = [], []
  n = grid.size
  flat = grid.reshape(-1)
  for axis, sl in enumerate(((slice(None), slice(None), slice(0, -1)), (slice(None), slice(0, -1), slice(None)),
                             (slice(0, -1), slice(None), slice(None)))):
    hi = tuple(slice(1, None) if s.stop == -1 else s for s in sl)
    cut = np.zeros(grid.shape, bool)
    cut[sl] = inside[sl] != inside[hi]
    p = np.flatnonzero(cut)
    stride = (1, grid.shape[2], grid.shape[1] * grid.shape[2])[axis]
    f0, f1 = flat[p], flat[p + stride]
    t = (np.float32(level) - f0) / (f1 - f0)
    ids.append(3 * p + axis)
    ts.append(t.astype(np.float32))
  ids, ts = np.concatenate(ids), np.concatenate(ts)
  order = np.argsort(ids, kind='stable')
  assert ids.max(initial=0) < 3 * n
  return ids[order], ts[order]


def check_closed_and_wound(faces, V):
  """Every directed edge once, and its reverse once: closed and consistently wound.  Returns the edge count."""
  f = faces.astype(np.int64)
  d = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
  key = d[:, 0] * V + d[:, 1]
  assert len(np.unique(key)) == len(key), 'a directed edge is used twice'
  rev = np.sort(d[:, 1] * V + d[:, 0])
  assert np.array_equal(np.sort(key), rev), 'an edge is used by one triangle only'
  return len(key) // 2


def signed_volume(v, f):
  a, b, c = v[f[:, 0]].astype(np.float64), v[f[:, 1]].astype(np.float64), v[f[:, 2]].astype(np.float64)
  return float(np.einsum('ij,ij->i', a, np.cross(b, c)).sum() / 6.0)


def run_mc(ops, grid, level):
  v, f = ops.marching_cubes(torch.tensor(grid, device='cuda'), level)
  torch.cuda.synchronize()
  return v.cpu().numpy(), f.cpu().numpy()


CASES = {
    'sphere': (lambda: sphere((48, 48, 48), (23.5, 24.2, 23.8), 20.0), 2),
    'torus': (lambda: torus((24, 48, 48), (23.7, 24.1, 11.6), 14.0, 6.0), 0),
    'two_spheres': (lambda: np.maximum(sphere((24, 40, 40), (10.3, 12.1, 11.8), 7.5),
                                       sphere((24, 40, 40), (28.6, 27.2, 12.3), 6.5)), 4),
    'nonsquare_sphere': (lambda: sphere((9, 33, 17), (8.2, 16.3, 4.1), 3.3), 2),
    'random': (lambda: smooth_field((40, 36, 44), 5), None),
}


@pytest.mark.parametrize('name', sorted(CASES))
def test_marching_cubes_analytic(mods, name):
  _, ops, _, _ = mods
  make, euler = CASES[name]
  grid = make()
  level = 0.0
  v, f = run_mc(ops, grid, level)
  ids, ts = cut_edges(grid, level)
  assert v.shape == (len(ids), 3) and f.shape[1] == 3 and len(f) > 0
  assert f.min() >= 0 and f.max() < len(v)
  # each vertex on its edge, at the linear crossing
  p, axis = ids // 3, ids % 3
  nz, ny, nx = grid.shape
  base = np.stack([p % nx, (p // nx) % ny, p // (nx * ny)], 1).astype(np.float32)
  want = base.copy()
  want[np.arange(len(ids)), axis] += ts
  assert np.allclose(v, want, rtol=0, atol=4e-6 * max(grid.shape)), float(np.abs(v - want).max())
  E_ = check_closed_and_wound(f, len(v))
  chi = len(v) - E_ + len(f)
  if euler is not None:
    assert chi == euler, chi
  else:
    assert chi % 2 == 0
  vol = signed_volume(v, f)
  assert vol > 0
  if name == 'sphere':
    exact = 4.0 / 3.0 * math.pi * 20.0 ** 3
    assert abs(vol - exact) / exact < 0.01, (vol, exact)
  v2, f2 = run_mc(ops, grid, level)
  assert np.array_equal(v, v2) and np.array_equal(f, f2), 'not deterministic'


def test_marching_cubes_empty_and_exact_level(mods):
  _, ops, _, _ = mods
  grid = sphere((20, 20, 20), (9.5, 9.5, 9.5), 6.0)
  v, f = run_mc(ops, grid, 100.0)                 # nothing above the level
  assert v.shape == (0, 3) and f.shape == (0, 3)
  v, f = run_mc(ops, np.full((5, 6, 7), 3.0, np.float32), 3.0)
  assert v.shape == (0, 3) and f.shape == (0, 3)
  # values on the level: integer-valued field, level an integer -> vertices on grid points
  q = np.round(grid).astype(np.float32)
  v, f = run_mc(ops, q, 2.0)
  assert len(f) > 0 and f.min() >= 0 and f.max() < len(v)
  assert np.isfinite(v).all()
  check_closed_and_wound(f, len(v))


def test_marching_cubes_rejects_bad_arguments(mods):
  lib, _, _, _ = mods
  L = lib.load()
  g = torch.zeros(8, device='cuda')
  cut = torch.zeros(24, device='cuda', dtype=torch.uint8)
  tri = torch.zeros(8, device='cuda', dtype=torch.uint8)
  P = lib.ptr

  def call(phase, nx, ny, nz, grid=g, c=cut, t=tri):
    return L.mnrf_marching_cubes(phase, nx, ny, nz, P(grid), 0.0, P(c), P(t), None, None, None, None, lib.stream_ptr())
  assert call(lib.MC_COUNT, 2, 2, 2) == 0
  for dims in ((1, 2, 2), (2, 1, 2), (2, 2, 0), (1025, 2, 2), (2, 2, 1025), (-4, 2, 2)):
    assert call(lib.MC_COUNT, *dims) != 0, dims
  assert call(lib.MC_COUNT, 2, 2, 2, grid=None) != 0
  assert call(lib.MC_COUNT, 2, 2, 2, c=None) != 0
  assert call(7, 2, 2, 2) != 0
  assert call(lib.MC_EMIT, 2, 2, 2) != 0                  # emit without scans and outputs
  torch.cuda.synchronize()


# ------------------------------------------------------------------ composition

def test_extract_mesh_composition(mods):
  lib, ops, models, mesh = mods
  model = models.Model(plumbing_blender())
  model.init(seed=3)
  bbox = (-1.5, -1.2, -1.0, 1.5, 1.2, 1.0)
  res = 31
  (nx, ny, nz), h = mesh.grid_shape(bbox, res)
  assert nx * ny >= 512             # every slab of one plane takes the chained trunk, like the whole grid
  whole, h1 = mesh.density_grid(model, bbox, res, slab_planes=nz)
  slabs, _ = mesh.density_grid(model, bbox, res, slab_planes=1)
  three, _ = mesh.density_grid(model, bbox, res, slab_planes=3)
  torch.cuda.synchronize()
  assert h1 == h and whole.shape == (nz, ny, nx)
  assert torch.equal(whole, slabs) and torch.equal(whole, three)
  # the grid is query_density at the grid points with var = h^2 / 12
  lo = torch.tensor(bbox[:3], dtype=torch.float64)
  idx = torch.stack(torch.meshgrid(torch.arange(nz), torch.arange(ny), torch.arange(nx), indexing='ij'), -1)
  pts = (lo + idx.flip(-1).double() * h).float().reshape(-1, 3)
  direct = model.query_density(pts.cuda(), h * h / 12)
  assert torch.equal(direct.view(nz, ny, nx), whole)
  level = float(whole.median())
  v, f = mesh.extract_mesh(model, bbox, res, level)
  gv, gf = ops.marching_cubes(whole, level)
  torch.cuda.synchronize()
  assert len(f) > 0 and torch.equal(f, gf)
  assert torch.equal(v, gv * h + lo.float().cuda())
  lo32, hi32 = torch.tensor(bbox[:3]).cuda(), torch.tensor(bbox[3:]).cuda()
  assert bool((v >= lo32 - 1e-5).all() and (v <= hi32 + 1e-5).all())


# ------------------------------------------------------------------ extract_mesh.py end to end

def _write_scene(root, n_train=10, n_test=2, W=40, H=30):
  """A shaded sphere over a gradient sky (train_loop.SyntheticScene.colour), rendered analytically."""
  from PIL import Image
  from multinerf_b200 import camera_utils, train_loop
  angle_x = 0.9
  focal = .5 * W / math.tan(.5 * angle_x)
  p2c = camera_utils.get_pixtocam(focal, W, H)
  for split, n, phase in (('train', n_train, 0.0), ('test', n_test, 0.3)):
    os.makedirs(os.path.join(root, split), exist_ok=True)
    frames = []
    for i in range(n):
      a = 2 * math.pi * (i + phase) / n
      eye = np.array([3.0 * math.cos(a), 3.0 * math.sin(a), 0.5 * math.sin(2 * a)])
      z = eye / np.linalg.norm(eye)
      x = np.cross([0, 0, 1.0], z)
      x /= np.linalg.norm(x)
      y = np.cross(z, x)
      c2w = np.eye(4)
      c2w[:3, :4] = np.concatenate([np.stack([x, y, z], 1), eye[:, None]], 1)
      xs, ys = camera_utils.pixel_coordinates(W, H)
      o, d, v, _, _ = camera_utils.pixels_to_rays(xs, ys, p2c, c2w[:3, :4])
      rgb = train_loop.SyntheticScene.colour(o.reshape(-1, 3), v.reshape(-1, 3)).reshape(H, W, 3).cpu().numpy()
      rgba = np.concatenate([rgb, np.ones((H, W, 1), np.float32)], -1)
      Image.fromarray((rgba * 255 + 0.5).astype(np.uint8)).save(os.path.join(root, split, f'r_{i}.png'))
      frames.append({'file_path': f'./{split}/r_{i}', 'transform_matrix': c2w.tolist()})
    with open(os.path.join(root, f'transforms_{split}.json'), 'w') as f:
      json.dump({'camera_angle_x': angle_x, 'frames': frames}, f)


def test_extract_mesh_script(tmp_path, capsys):
  sys.path.insert(0, ROOT)
  from multinerf_b200 import lib
  lib.require_device()
  import extract_mesh as mesh_script
  import train as train_script
  from test_mesh_cpu import read_ply
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
  path = mesh_script.main(argv + ['--gin_bindings=Config.mesh_resolution = 40', '--gin_bindings=Config.mesh_level = 1.'])
  printed = capsys.readouterr().out
  assert path == os.path.join(ckpt, 'mesh', f'mesh_step_{steps}.ply') and os.path.exists(path)
  line = [l for l in printed.splitlines() if 'vertices,' in l][-1]
  nv, nf = int(line.split(' vertices,')[0]), int(line.split(' vertices, ')[1].split(' faces')[0])
  v, f = read_ply(path)
  assert v.shape == (nv, 3) and f.shape == (nf, 3)
  if nf:
    assert f.min() >= 0 and f.max() < nv
    assert bool((np.abs(v) <= 1.5 + 1e-5).all())
