"""Mesh cleaning on the GPU: mnrf_mesh_components bit-identical to scipy's connected components (relabelled to
minimum vertex indices, tests/mesh_clean_ref.py) on deep, wide and many-component graphs and a 256^3 noise mesh;
mnrf_points_view_count against the fp64 projection of tests/tsdf_ref.py; mesh.clean_mesh against the reference
rules and on separated spheres; and extract_mesh / extract_mesh_tsdf with the cleaning options on a mini model.
Needs an H100."""
import ctypes as C

import numpy as np
import pytest
import torch

import mesh_clean_ref as R
import tsdf_ref
from test_gpu_mesh import sphere
from test_gpu_mesh_tsdf import CAMS, _views

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def mods():
  from multinerf_b200 import lib, mesh, ops
  lib.require_device()
  return lib, ops, mesh


def _labels(ops, faces, V):
  out = ops.mesh_components(torch.tensor(np.ascontiguousarray(faces, np.int32), device='cuda'), V)
  torch.cuda.synchronize()
  return out.cpu().numpy()


# ------------------------------------------------------------------ labels against scipy

def _path(rng):
  """2^20 vertices along one strip of triangles, vertex ids and face order permuted: hook chains as deep as the
  mesh is long."""
  V = 1 << 20
  ids = rng.permutation(V)
  return np.stack([ids[:-2], ids[1:-1], ids[2:]], 1)[rng.permutation(V - 2)], V


def _star(rng):
  """A fan of triangles around one hub, the largest index: every union meets at one root."""
  V = 200_001
  rim = rng.permutation(V - 1)
  return np.stack([np.full(V - 2, V - 1), rim[:-1], rim[1:]], 1), V


def _grid(rng):
  """A triangulated 700 x 700 grid with randomly permuted ids and two rows of cells removed: two halves and the
  700 vertices between the rows, which no face uses."""
  n = 700
  ids = rng.permutation(n * n).reshape(n, n)
  a, b, c, d = ids[:-1, :-1], ids[:-1, 1:], ids[1:, :-1], ids[1:, 1:]
  keep = np.ones((n - 1, n - 1), bool)
  keep[300:302] = False
  f = np.concatenate([np.stack([a, b, d], -1)[keep], np.stack([a, d, c], -1)[keep]])
  return f[rng.permutation(len(f))], n * n


def _many(rng):
  """10^5 small components: random triangle trees of 3 to 12 vertices, ids shuffled across components."""
  sizes = rng.integers(3, 13, 100_000)
  V = int(sizes.sum())
  g = np.arange(V)
  k = g - np.repeat(np.cumsum(sizes) - sizes, sizes)          # index within the component
  g, k = g[k >= 2], k[k >= 2]
  # vertex k joins vertex k - 1 and a random earlier vertex of its component
  f = np.stack([g, g - 1, g - 1 - rng.integers(1, k)], 1)
  f = rng.permutation(V)[f]
  return f[rng.permutation(len(f))], V


def _degenerate(rng):
  """Degenerate faces (a, a, b) and (a, a, a), duplicate faces and isolated vertices."""
  V = 50_000
  a = rng.integers(0, V, 20_000)
  b = rng.integers(0, V, 20_000)
  c = rng.integers(0, V, 20_000)
  f = np.concatenate([np.stack([a, a, b], 1), np.stack([c, c, c], 1), np.stack([a[:5000], b[:5000], c[:5000]], 1)])
  f = np.concatenate([f, f[:3000]])
  return f[rng.permutation(len(f))], V


GRAPHS = {'path': _path, 'star': _star, 'grid': _grid, 'many': _many, 'degenerate': _degenerate}


@pytest.mark.parametrize('name', sorted(GRAPHS))
def test_components_match_scipy(mods, name):
  _, ops, _ = mods
  faces, V = GRAPHS[name](np.random.default_rng(len(name)))
  want = R.components(faces, V)
  got = _labels(ops, faces, V)
  assert got.dtype == np.int32 and np.array_equal(got, want)
  n = len(np.unique(want))
  expect = {'path': 1, 'star': 1, 'grid': 2 + 700, 'many': 100_000}      # grid: two halves, a row of lone vertices
  if name in expect:
    assert n == expect[name], n
  else:
    assert n > 1000 and (want == np.arange(V)).sum() > 1000          # many isolated vertices
  assert np.array_equal(_labels(ops, faces, V), got), 'not deterministic'


def test_components_of_a_noise_mesh(mods):
  """Marching cubes on 256^3 normal noise: about 25 M vertices in many components of every size."""
  _, ops, _ = mods
  g = torch.Generator(device='cuda')
  g.manual_seed(0)
  grid = torch.randn(256, 256, 256, device='cuda', generator=g)
  v, f = ops.marching_cubes(grid, 0.0)
  del grid
  V = v.shape[0]
  assert V > 20_000_000
  labels = ops.mesh_components(f, V)
  again = ops.mesh_components(f, V)
  torch.cuda.synchronize()
  assert torch.equal(labels, again)
  want = R.components(f.cpu().numpy(), V)
  assert np.array_equal(labels.cpu().numpy(), want)


def test_components_reject_out_of_range_indices(mods):
  _, ops, _ = mods
  f = torch.tensor([[0, 1, 2], [2, 3, 4]], dtype=torch.int32, device='cuda')
  assert _labels(ops, f.cpu().numpy(), 5).tolist() == [0, 0, 0, 0, 0]
  for bad, V in (([[0, 1, 5]], 5), ([[0, -1, 2]], 5), ([[0, 1, 2]], 0)):
    with pytest.raises(ValueError, match='outside'):
      ops.mesh_components(torch.tensor(bad, dtype=torch.int32, device='cuda'), V)
  assert ops.mesh_components(torch.zeros(0, 3, dtype=torch.int32, device='cuda'), 0).shape == (0,)
  assert ops.mesh_components(torch.zeros(0, 3, dtype=torch.int32, device='cuda'), 3).tolist() == [0, 1, 2]


def test_components_abi_rejects_bad_arguments(mods):
  lib, _, _ = mods
  L = lib.load()
  f = torch.zeros(3, dtype=torch.int32, device='cuda')
  lab = torch.zeros(3, dtype=torch.int32, device='cuda')
  P = lib.ptr
  assert L.mnrf_mesh_components(3, 1, P(f), P(lab), lib.stream_ptr()) == 0
  for args in ((-1, 1, P(f), P(lab)), (3, -1, P(f), P(lab)), (0, 1, P(f), P(lab)), (3, 1, None, P(lab)),
               (3, 1, P(f), None), (3, 0, P(f), None)):
    assert L.mnrf_mesh_components(*args, lib.stream_ptr()) != 0, args
  torch.cuda.synchronize()


# ------------------------------------------------------------------ view counts against fp64

@pytest.mark.parametrize('cam', sorted(CAMS))
@pytest.mark.parametrize('K,per_view', [(1, False), (7, True), (7, False)])
def test_view_counts_vs_fp64(mods, cam, K, per_view):
  _, ops, _ = mods
  camtype, dist = CAMS[cam]
  rng = np.random.default_rng(K * 3 + per_view + 50 * camtype)
  H, W = 30, 40
  w2c, c2p, _, _, _ = _views(rng, K, H, W, camtype, per_view)
  # a box around the cameras (radius ~2.5): points behind, beside and inside the frusta
  pts = rng.uniform(-4, 4, (200_000, 3)).astype(np.float32)
  got = ops.points_view_count(torch.tensor(pts, device='cuda'), camtype, dist, torch.tensor(w2c, device='cuda'),
                              torch.tensor(c2p, device='cuda'), H, W).cpu().numpy()
  want = np.zeros(len(pts), np.int64)
  exempt = np.zeros(len(pts), bool)
  for k in range(K):
    u, v, _, valid = tsdf_ref.project(pts.astype(np.float64), w2c[k], c2p[k if per_view else 0],
                                      'fisheye' if camtype else 'perspective', dist)
    with np.errstate(invalid='ignore'):
      want += valid & (u >= 0) & (u < W) & (v >= 0) & (v < H)
      exempt |= valid & ((np.abs(u - np.round(u)) < tsdf_ref.PIXEL_MARGIN) |
                         (np.abs(v - np.round(v)) < tsdf_ref.PIXEL_MARGIN))
  live = ~exempt
  assert live.mean() > 0.9
  assert got.dtype == np.int32 and np.array_equal(got[live], want[live])
  # the counts vary: points on and off the one image, or at least three different counts of seven views (a
  # fisheye's field of view is wide enough that every point of the box lands on some view)
  assert len(np.unique(want[live])) >= min(K + 1, 3)


def test_view_counts_abi_rejects_bad_arguments(mods):
  lib, _, _ = mods
  L = lib.load()
  pts = torch.zeros(4, 3, device='cuda')
  m = torch.zeros(12, device='cuda')
  cnt = torch.zeros(4, dtype=torch.int32, device='cuda')
  P = lib.ptr

  def call(n=4, K=1, ncam=1, camtype=0, ndc=0, H=2, W=2, points=pts, counts=cnt, w2c=m, cam=True):
    d = lib.CameraDesc(0, ncam, camtype, 0, 0, 0, 0, 0, 0, 0, 0.0, 0, ndc, 1.0, 1.0, 1.0)
    return L.mnrf_points_view_count(C.byref(d) if cam else None, n, P(points), K, H, W, P(w2c), P(m), P(counts),
                                    lib.stream_ptr())
  assert call() == 0
  assert call(K=0, w2c=None) == 0
  for kw in (dict(n=-1), dict(K=-1), dict(H=0), dict(W=-3), dict(ncam=2), dict(camtype=2), dict(ndc=1),
             dict(points=None), dict(counts=None), dict(w2c=None), dict(cam=False)):
    assert call(**kw) != 0, kw
  torch.cuda.synchronize()


# ------------------------------------------------------------------ clean_mesh

def _three_spheres():
  shape = (40, 40, 100)
  big, mid, small = (20.3, 19.6, 20.2, 14.1), (55.4, 20.2, 19.7, 9.3), (82.1, 19.8, 20.4, 6.2)
  grid = np.maximum.reduce([sphere(shape, s[:3], s[3]) for s in (big, mid, small)])
  return grid, sphere(shape, big[:3], big[3])


def test_keep_largest_sphere_is_marching_cubes_on_it_alone(mods):
  _, ops, mesh = mods
  grid, only_big = _three_spheres()
  v, f, n = ops.marching_cubes(torch.tensor(grid, device='cuda'), 0.0, normals=True)
  stats = {}
  kv, kf, kn = mesh.clean_mesh(v, f, n, keep_components=1, stats=stats)
  bv, bf, bn = ops.marching_cubes(torch.tensor(only_big, device='cuda'), 0.0, normals=True)
  torch.cuda.synchronize()
  assert torch.equal(kv, bv) and torch.equal(kf, bf) and torch.equal(kn, bn)
  assert kf.dtype == torch.int32 and R.euler(kv.cpu().numpy(), kf.cpu().numpy()) == 2
  assert stats['components_removed'] == 2 and stats['vertices_removed'] == len(v) - len(bv)
  assert stats['faces_removed'] == len(f) - len(bf)
  tv, tf = mesh.clean_mesh(v, f, keep_components=2)
  assert R.euler(tv.cpu().numpy(), tf.cpu().numpy()) == 4 and len(bv) < len(tv) < len(v)
  # three or more keeps everything
  av, af = mesh.clean_mesh(v, f, keep_components=5)
  assert torch.equal(av, v) and torch.equal(af, f)


@pytest.mark.parametrize('keep,min_views', [(0, 2), (3, 0), (4, 3)])
def test_clean_mesh_vs_reference(mods, keep, min_views):
  """A noise-field mesh with per-vertex payloads, culled against 9 cameras and/or ranked: the reference's rules
  on the GPU's view counts, bit for bit."""
  lib, ops, mesh = mods
  from multinerf_b200 import camera_utils
  g = torch.Generator(device='cuda')
  g.manual_seed(1)
  grid = torch.randn(64, 72, 80, device='cuda', generator=g)
  v, f, n = ops.marching_cubes(grid, 0.8, normals=True)
  lo = torch.tensor([-2.0, -1.8, -1.6], device='cuda')
  v = v * 0.05 + lo
  rgb = torch.randint(0, 256, (len(v), 3), device='cuda', dtype=torch.uint8)
  rng = np.random.default_rng(3)
  H, W = 30, 40
  c2w = []
  for _ in range(9):
    eye = rng.normal(size=3)
    eye = 3.0 * eye / np.linalg.norm(eye)
    z = eye / np.linalg.norm(eye)
    x = np.cross([0, 0, 1.0], z)
    x /= np.linalg.norm(x)
    c2w.append(np.concatenate([np.stack([x, np.cross(z, x), z], 1), eye[:, None]], 1))
  cameras = (camera_utils.get_pixtocam(30.0, W, H), np.stack(c2w), None, None)
  args = dict(cameras=cameras, camtype='perspective', image_size=(H, W)) if min_views else {}
  out = mesh.clean_mesh(v, f, n, rgb, keep_components=keep, min_views=min_views, **args)
  torch.cuda.synchronize()
  counts = None
  if min_views:
    w2c, c2p = mesh.camera_matrices(cameras, 'cuda')
    counts = ops.points_view_count(v, 0, None, w2c, c2p, H, W).cpu().numpy()
    assert (counts < min_views).any() and (counts >= min_views).any()
  host = [t.cpu().numpy() for t in (v, f, n, rgb)]
  want = R.clean(*host, keep_components=keep, view_counts=counts, min_views=min_views)
  assert len(want[1]) > 0 and len(want[0]) < len(v)
  for a, b in zip(out, want):
    assert np.array_equal(a.cpu().numpy(), b)


# ------------------------------------------------------------------ extract_mesh and extract_mesh_tsdf

@pytest.fixture(scope='module')
def scene(tmp_path_factory):
  from multinerf_b200 import configs, datasets, models
  from test_gpu_mesh import _write_scene
  data = str(tmp_path_factory.mktemp('clean') / 'scene')
  _write_scene(data)
  bindings = [f"Config.data_dir = '{data}'", 'Config.render_chunk_size = 512', 'Config.near = 1.5',
              'Config.far = 5.0', "Config.dataset_loader = 'blender'", 'Model.num_prop_samples = 32',
              'Model.num_nerf_samples = 16', 'PropMLP.net_depth = 2', 'PropMLP.net_width = 64',
              'NerfMLP.net_depth = 4', 'NerfMLP.net_width = 128', 'NerfMLP.bottleneck_width = 64',
              'NerfMLP.net_width_viewdirs = 64', 'PropMLP.disable_density_normals = True',
              'PropMLP.disable_rgb = True', 'NerfMLP.disable_density_normals = True']
  bundle = configs.load_config(gin_bindings=bindings)
  model = models.Model(bundle)
  model.init(seed=5)
  import dataclasses
  dataset = datasets.load_dataset('train', data, dataclasses.replace(bundle.config, render_path=False),
                                  device=model.device)
  return model, dataset


def _equal(a, b):
  assert len(a) == len(b)
  for x, y in zip(a, b):
    assert x.dtype == y.dtype and torch.equal(x, y)


def test_extract_mesh_cleans_before_colouring(mods, scene):
  _, _, mesh = mods
  model, dataset = scene
  bbox, res = (-1.5, -1.5, -1.5, 1.5, 1.5, 1.5), 48
  grid, _ = mesh.density_grid(model, bbox, res)
  level = float(grid.median())
  raw = mesh.extract_mesh(model, bbox, res, level, colors=True)
  assert len(raw[1]) > 0
  cams = dict(cameras=dataset.cameras, camtype=dataset.camtype, image_size=(dataset.height, dataset.width))
  for keep, views in ((2, 0), (0, 6), (3, 4)):
    stats = {}
    got = mesh.extract_mesh(model, bbox, res, level, colors=True, keep_components=keep, min_views=views,
                            dataset=dataset, stats=stats)
    want = mesh.clean_mesh(*raw, keep_components=keep, min_views=views, **(cams if views else {}))
    _equal(got, want)
    assert 0 < len(got[1]) < len(raw[1]) and stats['faces_removed'] == len(raw[1]) - len(got[1])
  _equal(mesh.extract_mesh(model, bbox, res, level, colors=True, keep_components=0, min_views=0), raw)


def test_extract_mesh_tsdf_cleans(mods, scene):
  _, _, mesh = mods
  model, dataset = scene
  bbox, res = (-1.5, -1.5, -1.5, 1.5, 1.5, 1.5), 40
  raw = mesh.extract_mesh_tsdf(model, dataset, bbox, res, colors=True)
  cams = dict(cameras=dataset.cameras, camtype=dataset.camtype, image_size=(dataset.height, dataset.width))
  for keep, views in ((1, 0), (0, 5), (2, 3)):
    got = mesh.extract_mesh_tsdf(model, dataset, bbox, res, colors=True, keep_components=keep, min_views=views)
    _equal(got, mesh.clean_mesh(*raw, keep_components=keep, min_views=views, **(cams if views else {})))
  _equal(mesh.extract_mesh_tsdf(model, dataset, bbox, res, colors=True), raw)


def test_extract_mesh_script_cleans(tmp_path, capsys):
  """extract_mesh.py with both options after a short train.py run: the cleaning line, and a PLY with what it says."""
  import os
  import sys
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  sys.path.insert(0, root)
  from multinerf_b200 import lib
  lib.require_device()
  import extract_mesh as mesh_script
  import train as train_script
  from test_gpu_mesh import _write_scene
  from test_mesh_cpu import read_ply
  data, ckpt = str(tmp_path / 'scene'), str(tmp_path / 'ckpt')
  _write_scene(data)
  steps = 40
  bindings = [f"Config.data_dir = '{data}'", f"Config.checkpoint_dir = '{ckpt}'", 'Config.batch_size = 1024',
              f'Config.max_steps = {steps}', 'Config.print_every = 20', f'Config.checkpoint_every = {steps}',
              f'Config.train_render_every = {10 * steps}', 'Config.render_chunk_size = 512', 'Config.near = 1.5',
              'Config.far = 5.0', "Config.dataset_loader = 'blender'", 'Model.num_prop_samples = 32',
              'Model.num_nerf_samples = 16', 'PropMLP.net_depth = 2', 'PropMLP.net_width = 64',
              'NerfMLP.net_depth = 4', 'NerfMLP.net_width = 128', 'NerfMLP.bottleneck_width = 64',
              'NerfMLP.net_width_viewdirs = 64', 'PropMLP.disable_density_normals = True',
              'PropMLP.disable_rgb = True', 'NerfMLP.disable_density_normals = True']
  argv = [f'--gin_bindings={b}' for b in bindings]
  train_script.main(argv)
  capsys.readouterr()
  mesh_argv = argv + ['--gin_bindings=Config.mesh_resolution = 40', '--gin_bindings=Config.mesh_level = 0.5']
  mesh_script.main(mesh_argv)
  full = capsys.readouterr().out
  path = mesh_script.main(mesh_argv + ['--gin_bindings=Config.mesh_keep_components = 1',
                                       '--gin_bindings=Config.mesh_min_views = 4'])
  printed = capsys.readouterr().out
  count = lambda line: (int(line.split(' vertices,')[0].split()[-1]), int(line.split(' vertices, ')[1].split(' faces')[0]))
  nv0, nf0 = count([l for l in full.splitlines() if 'vertices,' in l][-1])
  lines = [l for l in printed.splitlines() if 'vertices,' in l]
  assert lines[0].startswith('cleaning removed') and 'mesh_min_views 4' in lines[0]
  dv, df = count(lines[0])
  nv, nf = count(lines[-1])
  assert (nv + dv, nf + df) == (nv0, nf0)
  v, f = read_ply(path)
  assert v.shape == (nv, 3) and f.shape == (nf, 3)
  if nf:
    assert f.min() >= 0 and f.max() < nv and len(np.unique(f)) == nv
