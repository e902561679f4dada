"""Mesh simplification on the GPU: mesh.simplify_mesh and its four kernels bit for bit against the numpy restatement
of tests/mesh_simplify_ref.py, round by round and end to end; topology invariants on a 256^3 noise mesh; quality
against coarser marching cubes on a rounded box; open boundaries; extract_mesh, extract_mesh_tsdf and the script
with a face budget; and the entry points' argument checks.  Needs an H100."""
import numpy as np
import pytest
import torch

import mesh_simplify_ref as R
from test_gpu_mesh import smooth_field, sphere, torus
from test_gpu_mesh_clean import scene  # noqa: F401  (the mini model and its training views)
from test_mesh_simplify_cpu import cube, square

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def mods():
  from multinerf_b200 import lib, mesh, ops
  lib.require_device()
  return lib, ops, mesh


def _mc(ops, grid, level=0.0, normals=True):
  return ops.marching_cubes(torch.tensor(np.ascontiguousarray(grid, np.float32), device='cuda'), level,
                            normals=normals)


def _open_sphere():
  """A sphere whose top is unobserved (NaN), as a TSDF leaves it: an open mesh with one boundary loop."""
  g = sphere((40, 40, 40), (19.6, 20.3, 19.2), 15.3)
  g[30:] = np.nan
  return g


def _meshes(ops):
  """name -> (vertices, faces, normals) device tensors, up to about 50 k faces."""
  out = {}
  for name, grid in (('sphere', sphere((60, 60, 60), (29.6, 30.2, 29.3), 24.4)),
                     ('torus', torus((30, 64, 64), (31.7, 32.1, 14.6), 20.0, 8.0)),
                     ('noise', smooth_field((44, 40, 48), 3)), ('open', _open_sphere())):
    out[name] = _mc(ops, grid)
  for name, (v, f) in (('cube', cube(12)), ('square', square(30, jitter=0.2, seed=1))):
    n = np.zeros_like(v)
    n[:, 2] = 1
    out[name] = tuple(torch.tensor(a, device='cuda') for a in (v, f, n))
  return out


TARGETS = {'sphere': (4000, 400), 'torus': (3000, 300), 'noise': (5000, 1), 'open': (1500, 100), 'cube': (12, 200),
           'square': (2, 100)}


def _bits(a):
  a = np.ascontiguousarray(a)
  return a.view(np.uint32 if a.dtype == np.float32 else np.uint64 if a.dtype == np.float64 else a.dtype)


def _same(got, want):
  got = got.cpu().numpy() if isinstance(got, torch.Tensor) else got
  assert got.shape == want.shape and np.array_equal(_bits(got), _bits(want.astype(got.dtype)))


@pytest.fixture(scope='module')
def meshes(mods):
  return _meshes(mods[1])


@pytest.mark.parametrize('name', sorted(TARGETS))
def test_simplify_matches_reference_bit_for_bit(mods, meshes, name):
  _, _, mesh = mods
  v, f, n = meshes[name]
  host = [t.cpu().numpy() for t in (v, f, n)]
  assert len(host[1]) <= 60_000
  for target in TARGETS[name]:
    stats = {}
    got = mesh.simplify_mesh(v, f, n, target_faces=target, stats=stats)
    want, wstats = R.simplify(*host, target_faces=target)
    assert stats == wstats, (stats, wstats)
    for a, b in zip(got, want):
      _same(a, b)
    assert stats['rounds'] > 0 and len(got[1]) < len(f)
    if name not in ('noise', 'open'):
      assert stats['target_reached'], stats
    # without normals: the same vertices and faces
    got2 = mesh.simplify_mesh(v, f, target_faces=target)
    assert len(got2) == 2 and torch.equal(got2[0], got[0]) and torch.equal(got2[1], got[1])
  # the inputs are untouched
  for a, b in zip((v, f, n), host):
    _same(a, b)


@pytest.mark.parametrize('name', ['sphere', 'open', 'noise'])
def test_each_kernel_matches_reference_over_rounds(mods, meshes, name):
  """Quadrics, keys and positions, the selected set and the applied state, each on the same inputs as the reference,
  for the first three rounds."""
  _, ops, mesh = mods
  v, f, n = (t.clone() for t in meshes[name])
  V = v.shape[0]
  topo = mesh.mesh_topology(f, V)
  rtopo = R.topology(f.cpu().numpy(), V)
  for a, b in zip(topo, rtopo):
    _same(a, b)
  q = ops.mesh_quadrics(v, f, topo.vf_off, topo.vf_face, *mesh.boundary_edges(topo, V))
  rq = R.quadrics(v.cpu().numpy(), f.cpu().numpy(), rtopo)
  _same(q, rq)
  if name == 'open':
    assert int((rtopo[1][1:] - rtopo[1][:-1] == 1).sum()) > 50
  for _ in range(3):
    hv, hf, hn, hq = (t.cpu().numpy() for t in (v, f, n, q))
    keys, pos = ops.mesh_edge_cost(v, f, q, *topo)
    rkeys, rpos = R.edge_cost(hv, hf, hq, rtopo)
    _same(keys, rkeys.view(np.int64))
    _same(pos, rpos)
    assert (rkeys != R.NO_KEY).mean() > 0.5
    sel = ops.mesh_collapse_select(f, topo.edges, keys, V)
    rsel = R.select(hf, rtopo[0], rkeys, V)
    _same(sel, rsel.astype(np.uint8))
    ids, _ = R.budget(rkeys, rsel, rtopo[1], len(hf) // 10)
    collapse = torch.zeros(len(keys), device='cuda', dtype=torch.uint8)
    collapse[torch.tensor(ids, device='cuda', dtype=torch.int64)] = 1
    alive = ops.mesh_collapse_apply(collapse, topo.edges, topo.edge_off, topo.edge_face, topo.vf_off, topo.vf_face,
                                    pos, v, q, n, f)
    f = f[alive.bool()]
    rv, rq, rn, rf = R.apply(ids, hv, hq, hn, hf, rtopo, rpos)
    for a, b in zip((v, q, n, f), (rv, rq, rn, rf)):
      _same(a, b)
    topo = mesh.mesh_topology(f, V)
    rtopo = R.topology(rf, V)


# ------------------------------------------------------------------ large mesh invariants

def _invariants(ops, v, f):
  """(sorted [(euler, boundary loops)] per component, duplicate faces, edges in more than 2 faces): the Euler
  characteristic and number of boundary loops of every component, after asserting indices in range and no repeated
  corner.  Marching cubes on white noise has pairs of faces on the same three vertices (a triangle lying in a face
  of the grid, emitted by both cells), whose edges are in more than 2 faces."""
  V, F = v.shape[0], f.shape[0]
  fl = f.long()
  assert int(fl.min()) >= 0 and int(fl.max()) < V
  assert not bool(((fl[:, 0] == fl[:, 1]) | (fl[:, 1] == fl[:, 2]) | (fl[:, 2] == fl[:, 0])).any())
  s = torch.sort(fl, 1).values
  o = torch.sort(s[:, 2], stable=True).indices
  o = o[torch.sort((s[:, 0] * V + s[:, 1])[o], stable=True).indices]
  ss = s[o]
  duplicates = int((ss[1:] == ss[:-1]).all(1).sum())
  del o, ss
  e = torch.cat([s[:, [0, 1]], s[:, [1, 2]], s[:, [0, 2]]])
  ekey, ecount = torch.unique(e[:, 0] * V + e[:, 1], return_counts=True)
  nonmanifold = int((ecount > 2).sum())
  labels = ops.mesh_components(f, V).long()
  comp_f = torch.bincount(labels[fl[:, 0]], minlength=V)
  used = torch.zeros(V, device='cuda', dtype=torch.bool)
  used[fl.view(-1)] = True
  comp_v = torch.bincount(labels[used], minlength=V)
  comp_e = torch.bincount(labels[ekey // V], minlength=V)
  bnd = ekey[ecount == 1]
  bf = torch.stack([bnd // V, bnd % V, bnd % V], 1).int().contiguous()
  loops = torch.zeros(V, device='cuda', dtype=torch.int64)
  if bf.shape[0]:
    bl = ops.mesh_components(bf, V).long()
    roots = torch.unique(bl[bf[:, 0].long()])
    loops = torch.bincount(labels[roots], minlength=V)
  ids = torch.nonzero(comp_f).view(-1)
  chi = comp_v[ids] - comp_e[ids] + comp_f[ids]
  pairs = torch.stack([chi, loops[ids]], 1).cpu().numpy()
  return sorted(map(tuple, pairs.tolist())), duplicates, nonmanifold


def test_large_noise_mesh_invariants(mods):
  _, ops, mesh = mods
  g = torch.Generator(device='cuda')
  g.manual_seed(0)
  grid = torch.randn(256, 256, 256, device='cuda', generator=g)
  v, f = ops.marching_cubes(grid, 0.0)
  del grid
  assert v.shape[0] > 20_000_000
  pairs, duplicates, nonmanifold = _invariants(ops, v, f)
  F = f.shape[0]
  for frac in (0.1, 0.01):
    target = int(F * frac)
    stats = {}
    sv, sf = mesh.simplify_mesh(v, f, target_faces=target, stats=stats)
    assert stats['faces_after'] == sf.shape[0]
    assert sf.shape[0] in (target, target + 1) or not stats['target_reached'], stats
    got = _invariants(ops, sv, sf)
    print(f'noise 256^3: {F} -> {sf.shape[0]} faces (target {target}) in {stats["rounds"]} rounds; '
          f'{len(pairs)} components; duplicate faces {duplicates} -> {got[1]}, edges of > 2 faces '
          f'{nonmanifold} -> {got[2]}')
    # no component changes its topology, and no duplicate face or edge of more than 2 faces appears
    assert got[0] == pairs and got[1] <= duplicates and got[2] <= nonmanifold
    if frac == 0.1:
      again = mesh.simplify_mesh(v, f, target_faces=target)
      assert torch.equal(again[0], sv) and torch.equal(again[1], sf)
      del again
    del sv, sf
    torch.cuda.empty_cache()


# ------------------------------------------------------------------ quality and boundaries

def _rounded_box_sdf(p, b=0.5, r=0.2):
  q = np.abs(p) - b
  outside = np.linalg.norm(np.maximum(q, 0.0), axis=-1)
  return outside + np.minimum(q.max(-1), 0.0) - r


def _rounded_box_mesh(ops, n):
  ax = np.linspace(-1.0, 1.0, n)
  z, y, x = np.meshgrid(ax, ax, ax, indexing='ij')
  grid = -_rounded_box_sdf(np.stack([x, y, z], -1))
  v, f = ops.marching_cubes(torch.tensor(grid.astype(np.float32), device='cuda'), 0.0)
  return v * (2.0 / (n - 1)) - 1.0, f


def _surface_error(v, f):
  v = v.cpu().numpy().astype(np.float64)
  f = f.cpu().numpy()
  return np.abs(_rounded_box_sdf(v)).max(), np.abs(_rounded_box_sdf(v[f].mean(1))).mean()


def test_simplified_beats_coarser_marching_cubes(mods):
  """A box with flat sides and rounded edges: 256^3 simplified to the face count of a coarser grid is closer to the
  surface than that grid's marching cubes, by the worst vertex and by the mean face centroid."""
  _, ops, mesh = mods
  fine_v, fine_f = _rounded_box_mesh(ops, 256)
  for n in (48, 80):
    cv, cf = _rounded_box_mesh(ops, n)
    stats = {}
    sv, sf = mesh.simplify_mesh(fine_v, fine_f, target_faces=cf.shape[0], stats=stats)
    assert stats['target_reached'] and abs(sf.shape[0] - cf.shape[0]) <= 1
    c_max, c_mean = _surface_error(cv, cf)
    s_max, s_mean = _surface_error(sv, sf)
    print(f'rounded box, {cf.shape[0]} faces: mc {n}^3 max {c_max:.2e} mean {c_mean:.2e}; '
          f'simplified 256^3 max {s_max:.2e} mean {s_mean:.2e}')
    assert s_max < c_max and s_mean < c_mean


def _dist_to_polyline(p, a, b):
  ab = b - a
  t = np.clip(((p[:, None] - a[None]) * ab[None]).sum(-1) / (ab * ab).sum(-1)[None], 0, 1)
  return np.linalg.norm(p[:, None] - (a[None] + t[..., None] * ab[None]), axis=-1).min(1)


def _boundary_segments(v, f):
  e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
  u, c = np.unique(e, axis=0, return_counts=True)
  b = u[c == 1]
  return v[b[:, 0]].astype(np.float64), v[b[:, 1]].astype(np.float64), np.unique(b)


BOUNDARY_TOL = 0.25       # grid cells


def test_boundary_stays_on_the_original_boundary(mods, meshes):
  """The open sphere's boundary vertices stay within BOUNDARY_TOL of its original boundary polyline at budgets that
  leave the boundary loop more than a few edges.  (Forced far lower, the loop itself collapses to a few long edges,
  and their summed boundary planes no longer pin a vertex to the polyline.)"""
  _, _, mesh = mods
  v, f, n = meshes['open']
  hv, hf = v.cpu().numpy(), f.cpu().numpy()
  a, b, _ = _boundary_segments(hv, hf)
  assert len(a) > 50
  for target in (1500, 700):
    sv, sf = mesh.simplify_mesh(v, f, target_faces=target)
    sv, sf = sv.cpu().numpy(), sf.cpu().numpy()
    _, _, ids = _boundary_segments(sv, sf)
    d = _dist_to_polyline(sv[ids].astype(np.float64), a, b)
    print(f'open sphere to {target} faces: boundary vertices within {d.max():.3e} cells of the original boundary')
    assert len(ids) >= 3 and d.max() < BOUNDARY_TOL


# ------------------------------------------------------------------ the pipeline

def _equal(a, b):
  assert len(a) == len(b)
  for x, y in zip(a, b):
    assert x.dtype == y.dtype and torch.equal(x, y)


def test_extract_mesh_simplifies_before_colouring(mods, scene):
  _, _, mesh = mods
  model, _ = scene
  bbox, res = (-1.5, -1.5, -1.5, 1.5, 1.5, 1.5), 48
  grid, h = mesh.density_grid(model, bbox, res)
  level = float(grid.median())
  for colors in (False, True):
    raw = mesh.extract_mesh(model, bbox, res, level, colors=colors, keep_components=2)
    _equal(mesh.extract_mesh(model, bbox, res, level, colors=colors, keep_components=2, target_faces=0), raw)
    target = len(raw[1]) // 5
    stats = {}
    got = mesh.extract_mesh(model, bbox, res, level, colors=colors, keep_components=2, target_faces=target,
                            stats=stats)
    want = mesh.simplify_mesh(*raw[:3], target_faces=target)
    if colors:
      want = (*want, mesh.vertex_colors(model, want[0], want[2], h * h / 12))
    _equal(got, want)
    assert stats['faces_after'] == len(got[1]) < len(raw[1]) and stats['components_removed'] >= 0


def test_extract_mesh_tsdf_simplifies_before_colouring(mods, scene):
  _, _, mesh = mods
  model, dataset = scene
  bbox, res = (-1.5, -1.5, -1.5, 1.5, 1.5, 1.5), 40
  state, h = mesh.fuse_tsdf(mesh.render_views(model, dataset), dataset.cameras, dataset.camtype, bbox, res, 3.0,
                            colors=True, device=model.device)
  for colors in (False, True):
    raw = mesh.extract_mesh_tsdf(model, dataset, bbox, res, colors=colors, keep_components=1)
    _equal(mesh.tsdf_mesh(state, bbox, h, colors=colors, clean_args=dict(keep_components=1)), raw)
    _equal(mesh.extract_mesh_tsdf(model, dataset, bbox, res, colors=colors, keep_components=1, target_faces=0), raw)
    target = len(raw[1]) // 4
    got = mesh.extract_mesh_tsdf(model, dataset, bbox, res, colors=colors, keep_components=1, target_faces=target)
    want = mesh.simplify_mesh(*raw[:3], target_faces=target)
    _equal(got[:len(want)], want)
    if colors:
      # the colour grid sampled trilinearly at the simplified vertices, in fp64
      cs, cw = (t.cpu().numpy().astype(np.float64) for t in state[2:])
      nz, ny, nx = cw.shape
      lo = np.array(bbox[:3])
      g = np.clip((got[0].cpu().numpy().astype(np.float64) - lo) / h, 0, [nx - 1, ny - 1, nz - 1])
      base = np.clip(np.floor(g).astype(np.int64), 0, [nx - 2, ny - 2, nz - 2])
      fr = g - base
      s = np.zeros((len(g), 3))
      w = np.zeros(len(g))
      for c in range(8):
        off = np.array([c & 1, c >> 1 & 1, c >> 2 & 1])
        wt = np.where(off, fr, 1 - fr).prod(-1)
        q = base + off
        s += wt[:, None] * cs[q[:, 2], q[:, 1], q[:, 0]]
        w += wt * cw[q[:, 2], q[:, 1], q[:, 0]]
      rgb = np.where(w[:, None] > 0, s / np.maximum(w, 1e-30)[:, None], 0)
      want_rgb = np.round(np.clip(rgb, 0, 1) * 255)
      diff = np.abs(got[3].cpu().numpy().astype(np.float64) - want_rgb)
      assert got[3].dtype == torch.uint8 and diff.max() <= 1 and (diff == 0).mean() > 0.95


def test_extract_mesh_script_simplifies(tmp_path, capsys):
  """extract_mesh.py with mesh_target_faces after a short train.py run: the simplification line, and a PLY with what
  the final line says."""
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
  full = [l for l in capsys.readouterr().out.splitlines() if 'vertices,' in l][-1]
  nf0 = int(full.split(' vertices, ')[1].split(' faces')[0])
  target = max(nf0 // 3, 1)
  path = mesh_script.main(mesh_argv + [f'--gin_bindings=Config.mesh_target_faces = {target}'])
  lines = capsys.readouterr().out.splitlines()
  simp = [l for l in lines if l.startswith('simplified ')]
  assert len(simp) == 1 and f'{nf0} -> ' in simp[0] and f'(mesh_target_faces {target})' in simp[0], simp
  f1 = int(simp[0].split(' -> ')[1].split(' faces')[0])
  last = lines[-1]
  nv = int(last.split(' vertices,')[0].split()[-1])
  nf = int(last.split(' vertices, ')[1].split(' faces')[0])
  assert nf == f1 and (nf <= target + 1 or 'stalled' in simp[0])
  v, f = read_ply(path)
  assert v.shape == (nv, 3) and f.shape == (nf, 3)
  assert f.min() >= 0 and f.max() < nv and len(np.unique(f)) == nv


# ------------------------------------------------------------------ the entry points

def test_entry_points_reject_bad_arguments(mods):
  lib, _, _ = mods
  L = lib.load()
  P = lib.ptr
  s = lib.stream_ptr()
  i32 = lambda n: torch.zeros(n, dtype=torch.int32, device='cuda')
  i64 = lambda n: torch.zeros(n, dtype=torch.int64, device='cuda')
  v, f, q = torch.zeros(4, 3, device='cuda'), i32(6), torch.zeros(4, 10, dtype=torch.float64, device='cuda')
  off, face, e = i64(5), i32(6), i32(2)
  pos, u8 = torch.zeros(1, 3, device='cuda'), torch.zeros(2, dtype=torch.uint8, device='cuda')
  quad = lambda nv=4, nf=2, nb=0, vert=v, qq=q: L.mnrf_mesh_quadrics(nv, nf, P(vert), P(f), P(off), P(face), nb,
                                                                     None, None, P(off), None, P(qq), s)
  assert quad() == 0
  for kw in (dict(nv=-1), dict(nf=-1), dict(nb=-1), dict(vert=None), dict(qq=None), dict(nb=1)):
    assert quad(**kw) != 0, kw
  keys = i64(1)
  cost = lambda ne=1, nv=4, nf=2, k=keys, fl=i32(4): L.mnrf_mesh_edge_cost(nv, nf, ne, P(v), P(f), P(q), P(e), P(off),
                                                                          P(face), P(off), P(face), P(fl), P(k),
                                                                          P(pos), s)
  assert cost(ne=0) == 0 and cost() == 0
  for kw in (dict(ne=-1), dict(nv=-1), dict(nf=-1), dict(ne=2 ** 32), dict(k=None), dict(fl=None), dict(nv=0)):
    assert cost(**kw) != 0, kw
  sel = lambda ne=1, nv=4, nf=2, vmin=i64(4), out=u8: L.mnrf_mesh_collapse_select(nv, nf, ne, P(f), P(e), P(keys),
                                                                                  P(vmin), P(i64(4)), P(out), s)
  assert sel(ne=0) == 0 and sel() == 0
  for kw in (dict(ne=-1), dict(nv=-1), dict(nf=-1), dict(ne=2 ** 32), dict(vmin=None), dict(out=None), dict(nf=0)):
    assert sel(**kw) != 0, kw
  app = lambda nf=2, nv=4, ne=1, alive=u8, col=u8: L.mnrf_mesh_collapse_apply(nv, nf, ne, P(col), P(e), P(off),
                                                                              P(face), P(off), P(face), P(pos), P(v),
                                                                              P(q), None, P(f), P(alive), s)
  assert app() == 0 and app(ne=0, col=None) == 0
  for kw in (dict(nf=-1), dict(nv=-1), dict(ne=-1), dict(ne=2 ** 32), dict(alive=None), dict(col=None),
             dict(nv=0)):
    assert app(**kw) != 0, kw
  torch.cuda.synchronize()
