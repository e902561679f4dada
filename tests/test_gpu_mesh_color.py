"""Coloured meshes on the GPU: marching-cubes vertex normals against an fp64 restatement of their rule, the point
encoder's tangent rows against autograd of the oracle's encoding, per-point colours against the compositing
kernel's per-sample colours, Model.query_radiance against the oracle's MLP, their composition in
mesh.extract_mesh(colors=True), and extract_mesh.py with Config.mesh_vertex_colors.  Needs an H100."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest
import torch

import encode_ref as E
from model_parity import mini360, mini_refnerf, plumbing_blender, torch_tree
from oracle import o_models
from test_gpu_mesh import CASES, _write_scene, cut_edges, sphere
from test_mesh_color_cpu import read_ply_props
from util import close

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24          # unit roundoff of fp32


@pytest.fixture(scope='module')
def mods():
  from multinerf_b200 import lib, mesh, models, ops
  lib.require_device()
  return lib, ops, models, mesh


# ------------------------------------------------------------------ vertex normals

def normals_reference(grid, level):
  """fp64 restatement of mnrf_mc_normals: (normals [V, 3], bound [V], fallback [V] bool), in vertex order.

  The kernel's gradient components are an fp32 difference (relative error <= u, the halving is exact) of the
  grid's values, interpolated as g0 + t (g1 - g0) with the vertex's own fp32 t (shared with the reference): at most
  6 u (|g0| + |g1|) per component.  Normalising moves the unit vector by at most |error| / |g| in first order, and
  the scaling by the largest component, the norm and the division add at most 8 u per component; the bound doubles
  the first-order term."""
  ids, ts = cut_edges(grid, level)
  g = grid.astype(np.float64)
  G = np.stack(np.gradient(g, axis=(2, 1, 0)), -1).reshape(-1, 3)    # central; one-sided on the boundary
  nz, ny, nx = grid.shape
  p, axis = ids // 3, ids % 3
  q = p + np.array([1, nx, nx * ny])[axis]
  g0, g1 = G[p], G[q]
  t = ts.astype(np.float64)[:, None]
  gi = g0 + t * (g1 - g0)
  length = np.linalg.norm(gi, axis=1)
  fallback = length == 0
  n = -gi / np.where(fallback, 1.0, length)[:, None]
  inside = grid.reshape(-1)[p] > level
  n[fallback] = 0.0
  n[fallback, axis[fallback]] = np.where(inside[fallback], 1.0, -1.0)
  err = 6 * U * np.linalg.norm(np.abs(g0) + np.abs(g1), axis=1)
  bound = 2 * err / np.where(fallback, 1.0, length) + 8 * U
  return n, bound, fallback


def fallback_grid():
  """f depends on x only: [-3, 1, -1, -1].  The edge x = 1 -> 2 is cut at t = 1/2 between the gradients +1 and -1,
  so its interpolated gradient is exactly 0 (in fp32 too)."""
  return np.broadcast_to(np.array([-3.0, 1.0, -1.0, -1.0], np.float32), (3, 3, 4)).copy()


NORMAL_CASES = dict({k: v[0] for k, v in CASES.items()},
                    boundary=lambda: sphere((20, 20, 20), (2.3, 9.6, 10.1), 6.0),
                    fallback=fallback_grid)


@pytest.mark.parametrize('name', sorted(NORMAL_CASES))
def test_mc_normals_vs_fp64(mods, name):
  _, ops, _, _ = mods
  grid = NORMAL_CASES[name]()
  level = 0.0
  v, f, n = ops.marching_cubes(torch.tensor(grid, device='cuda'), level, normals=True)
  v0, f0 = ops.marching_cubes(torch.tensor(grid, device='cuda'), level)
  torch.cuda.synchronize()
  assert torch.equal(v, v0) and torch.equal(f, f0)
  n = n.cpu().numpy().astype(np.float64)
  ref, bound, fallback = normals_reference(grid, level)
  assert n.shape == ref.shape and len(n) > 0
  live = bound < 0.1
  assert float(live.mean()) > 0.99
  err = np.abs(n - ref)
  assert (err[live] <= bound[live, None]).all(), float((err - bound[:, None])[live].max())
  assert np.all(np.abs(np.linalg.norm(n, axis=1) - 1) <= 1e-6)
  assert np.array_equal(n[fallback], ref[fallback])
  if name == 'fallback':
    assert fallback.sum() == 9 and (n[fallback] == [1.0, 0.0, 0.0]).all()    # +x: from the inside end x = 1
  if name == 'boundary':
    ids, _ = cut_edges(grid, level)
    x = (ids // 3) % grid.shape[2]
    assert (x == 0).any()                     # vertices whose gradient takes the one-sided difference
  if name == 'sphere':
    # the sphere r - |x - c| of test_gpu_mesh: every normal within 0.1 degree of the outward radial direction
    radial = v.cpu().numpy().astype(np.float64) - np.array([23.5, 24.2, 23.8])
    radial /= np.linalg.norm(radial, axis=1, keepdims=True)
    assert (np.einsum('ij,ij->i', n, radial) > math.cos(math.radians(0.1))).all()


def test_mc_normals_rejects_bad_arguments(mods):
  lib, _, _, _ = mods
  L = lib.load()
  g = torch.zeros(8, device='cuda')
  cut = torch.zeros(24, device='cuda', dtype=torch.uint8)
  scan = torch.zeros(24, device='cuda', dtype=torch.int64)
  out = torch.zeros(3, device='cuda')
  P = lib.ptr

  def call(nx=2, ny=2, nz=2, grid=g, c=cut, s=scan, o=out):
    return L.mnrf_mc_normals(nx, ny, nz, P(grid), 0.0, P(c), P(s), P(o), lib.stream_ptr())
  assert call() == 0
  for dims in ((1, 2, 2), (2, 1, 2), (2, 2, 0), (1025, 2, 2), (-4, 2, 2)):
    assert call(*dims) != 0, dims
  for kw in (dict(grid=None), dict(c=None), dict(s=None), dict(o=None)):
    assert call(**kw) != 0, kw
  torch.cuda.synchronize()


# ------------------------------------------------------------------ point encoder with tangent rows

def _points(rng):
  """inside the unit ball, outside it, and far out; 1001 points: a ragged last group of 32"""
  return np.concatenate([rng.uniform(-0.57, 0.57, (400, 3)), rng.uniform(-3, 3, (400, 3)),
                         rng.normal(size=(201, 3)) * 50]).astype(np.float32)


@pytest.mark.parametrize('warp_contract,disable_integration,var', [
    (False, False, 1e-4), (True, False, 1e-4), (True, True, 1e-4), (True, False, 0.0), (False, False, 0.0),
    (True, False, 3e-2)])
def test_encode_points_tangent_features_vs_fp64(mods, warp_contract, disable_integration, var):
  """The feature rows of the tangent entry point meet the bounds mnrf_encode_points meets, and its tangent rows
  (d feature / d point, stream dir at rows dir * N + i of a tfeat whose pitch exceeds feat_cols) meet
  encode_ref.tangent_reference's, element by element; the pitch's padding survives."""
  _, ops, _, _ = mods
  from multinerf_b200 import geopoly
  basis = np.ascontiguousarray(geopoly.generate_basis('octahedron', 2), dtype=np.float32)
  pts = _points(np.random.default_rng(3))
  N = len(pts)
  min_deg, max_deg = 0, 12
  feat_cols = (2 * len(basis) * (max_deg - min_deg) + 63) // 64 * 64
  tbuf = torch.full((3 * N, feat_cols + 24), 7.0, device='cuda', dtype=torch.bfloat16)
  tfeat = tbuf[:, :feat_cols + 16]                                           # ld_tfeat > feat_cols
  feat, _ = ops.encode_points(torch.tensor(pts, device='cuda'), var, torch.tensor(basis, device='cuda'),
                              min_deg=min_deg, max_deg=max_deg, warp_contract=warp_contract,
                              disable_integration=disable_integration, tfeat=tfeat)
  torch.cuda.synchronize()
  ref = E.points_reference(pts, var, basis, min_deg=min_deg, max_deg=max_deg, warp_contract=warp_contract,
                           disable_integration=disable_integration)
  F = ref.feat.shape[1]
  live = ~ref.vacuous
  assert float(live.double().mean()) > 0.5
  errb = (feat[:, :F].float().cpu().double() - ref.feat).abs()
  assert bool((errb[live] <= ref.bound_bf16[live]).all()), float((errb - ref.bound_bf16)[live].max())
  assert bool((feat[:, F:] == 0).all()) and bool((tfeat[:, F:feat_cols] == 0).all())
  assert bool((tbuf[:, feat_cols:] == 7).all()), 'tangent rows written past feat_cols'
  got = tfeat[:, :F].float().cpu().double().view(3, N, F)
  tlive = ~ref.tangent_vacuous
  ratio = torch.where(tlive, (got - ref.tangent).abs() / ref.tangent_bound_bf16, torch.zeros_like(got))
  worst = [float(ratio[a].max()) for a in range(3)]
  print(f'\ncontract {warp_contract} no_int {disable_integration} var {var}: tangent worst err/bound per stream '
        + ' '.join(f'{w:.2f}' for w in worst) + f' | checked {float(tlive.double().mean()):.3f}')
  assert float(tlive.double().mean()) > 0.5
  bad = ratio > 1
  if bad.any():
    i = tuple(int(v) for v in np.unravel_index(int(ratio.argmax()), ratio.shape))
    raise AssertionError(f'{int(bad.sum())} tangent elements outside their bound; worst at [stream, point, column] '
                         f'{i}: got {float(got[i])!r}, fp64 {float(ref.tangent[i])!r}, '
                         f'bound {float(ref.tangent_bound_bf16[i]):.3e}')


def test_encode_points_tangent_rejects_bad_arguments(mods):
  lib, _, _, _ = mods
  L = lib.load()
  pts = torch.zeros(8, 3, device='cuda')
  basis = torch.zeros(21, 3, device='cuda')
  feat = torch.zeros(8, 512, device='cuda', dtype=torch.bfloat16)
  tfeat = torch.zeros(24, 520, device='cuda', dtype=torch.bfloat16)
  P = lib.ptr

  def call(var=1e-3, p=pts, t=tfeat, ld_t=512, tptr=None, **kw):
    f = dict(num_rays=8, num_samples=1, raydist_fn=0, ray_shape=0, warp_contract=1, disable_integration=0,
             basis_k=21, min_deg=0, max_deg=12, ld_feat=512, feat_cols=512)
    f.update(kw)
    d = lib.EncodeDesc(**f)
    return L.mnrf_encode_points_tangent(C.byref(d), P(p), var, P(basis), P(feat), tptr if tptr else P(t), ld_t,
                                        lib.stream_ptr())
  assert call() == 0
  for kw in (dict(num_samples=2), dict(raydist_fn=1), dict(ray_shape=1), dict(feat_cols=500), dict(feat_cols=256),
             dict(ld_feat=256), dict(num_rays=-1), dict(max_deg=0)):
    assert call(**kw) != 0, kw
  for var in (-1.0, float('nan'), float('inf')):
    assert call(var=var) != 0, var
  assert call(p=None) != 0
  assert call(t=None) != 0
  assert call(ld_t=500) != 0 and call(ld_t=516) != 0                       # < feat_cols, not a multiple of 8
  assert call(tptr=C.c_void_p(tfeat.data_ptr() + 8)) != 0                  # tangent rows not 16-byte aligned
  d = lib.EncodeDesc(8, 1, 0, 0, 0, 0, 21, 0, 12, 512, 512)
  assert L.mnrf_encode_points_tangent(None, P(pts), 1e-3, P(basis), P(feat), P(tfeat), 512, lib.stream_ptr()) != 0
  assert L.mnrf_encode_points_tangent(C.byref(d), P(pts), 1e-3, None, P(feat), P(tfeat), 512, lib.stream_ptr()) != 0
  torch.cuda.synchronize()


# ------------------------------------------------------------------ per-point colour

@pytest.mark.parametrize('act,mode,tint,stacked', [
    ('sigmoid', 0, False, False), ('safe_exp', 0, False, False), ('sigmoid', 1, True, False),
    ('sigmoid', 1, False, False), ('safe_exp', 1, True, False), ('sigmoid', 0, False, True),
    ('safe_exp', 0, False, True)])
def test_point_rgb_matches_composite_samples(mods, act, mode, tint, stacked):
  """ops.point_rgb is bit-identical to composite_fwd's per-sample colours of the same raws with one sample per
  ray; `stacked` reads the rgb columns of a [density | rgb] head in place (ld_rgb = 4)."""
  _, ops, _, _ = mods
  rng = np.random.default_rng(17)
  M = 3001
  cfg = dict(raydist_fn=None, opaque_background=False, density_bias=-1.0, density_noise=0.0, rgb_activation=act,
             rgb_premultiplier=1.3, rgb_bias=0.2, rgb_padding=0.001, bg_const=0.5, rgb_mode=mode)
  dev = 'cuda'
  head = torch.tensor(rng.normal(size=(M, 4)).astype(np.float32) * 4, device=dev)
  raw_rgb = head[:, 1:] if stacked else head[:, 1:].contiguous()
  diffuse = torch.tensor(rng.normal(size=(M, 3)).astype(np.float32) * 3, device=dev) if mode else None
  tint_t = torch.tensor(rng.normal(size=(M, 3)).astype(np.float32) * 3, device=dev) if tint else None
  got = ops.point_rgb(raw_rgb, cfg=cfg, raw_diffuse=diffuse, raw_tint=tint_t)
  sdist = torch.tensor([[0.0, 1.0]], device=dev).expand(M, 2).contiguous()
  dirs = torch.tensor([[0.0, 0.0, 1.0]], device=dev).expand(M, 3).contiguous()
  near, far = torch.full((M,), 1.0, device=dev), torch.full((M,), 2.0, device=dev)
  comp_rgb = head.view(M, 1, 4)[..., 1:] if stacked else raw_rgb.view(M, 1, 3)
  comp = ops.composite_fwd(head[:, :1].contiguous(), comp_rgb, sdist, dirs, near, far, cfg=cfg,
                           raw_diffuse=diffuse, raw_tint=tint_t, want_samples=True)
  torch.cuda.synchronize()
  assert torch.equal(got, comp['rgb_samples'].view(M, 3))
  assert bool(torch.isfinite(got).all())


def test_point_rgb_rejects_bad_arguments(mods):
  lib, ops, _, _ = mods
  L = lib.load()
  raw = torch.zeros(4, 4, device='cuda')
  out = torch.zeros(4, 3, device='cuda')
  P = lib.ptr

  def call(M=4, ld=4, act=0, mode=0, diffuse=None, r=raw, o=out, desc=True):
    d = ops._cdesc(4, 1, raydist_fn=None, opaque_background=False, density_bias=0.0, density_noise=0.0,
                   rgb_activation='sigmoid', rgb_premultiplier=1.0, rgb_bias=0.0, rgb_padding=0.0, bg_const=0.0,
                   rgb_mode=mode)
    d.rgb_act = act
    return L.mnrf_point_rgb(C.byref(d) if desc else None, M, P(r), ld, P(diffuse), None, P(o), lib.stream_ptr())
  assert call() == 0 and call(M=0, r=None, o=None) == 0
  assert call(ld=2) != 0 and call(M=-1) != 0 and call(act=2) != 0 and call(mode=2) != 0
  assert call(mode=1) != 0 and call(mode=1, diffuse=out) == 0
  assert call(r=None) != 0 and call(o=None) != 0 and call(desc=False) != 0
  torch.cuda.synchronize()


# ------------------------------------------------------------------ query_radiance

def _bundle(which):
  if which == 'plumbing':
    return plumbing_blender()
  if which == 'refnerf':
    return mini_refnerf()
  b = mini360()
  if which in ('softplus', 'silu'):
    b.nerf_mlp.net_activation = b.prop_mlp.net_activation = which
  if which == 'viewindep':
    b.model.use_viewdirs = False
  if which == 'glo':
    b.model.num_glo_features = 4
  return b


# colour bounds: the samples= bound pinned_forward uses for the family (test_gpu_model.py)
@pytest.mark.parametrize('which,N,rgb_tol', [
    ('mini360', 3000, 3e-2), ('plumbing', 4096, 3e-2), ('plumbing', 300, 3e-2), ('softplus', 2000, 3e-2),
    ('silu', 2000, 3e-2), ('viewindep', 2000, 3e-2), ('refnerf', 2000, 4e-2), ('glo', 2000, 3e-2)])
def test_query_radiance_vs_oracle(mods, which, N, rgb_tol):
  """plumbing runs its 256-wide ReLU trunk chained at 4096 rows and layer by layer at 300; refnerf: IDE of the
  reflected direction, predicted and density normals, diffuse colour, tint and n.v; glo: the oracle gets a zero
  GLO vector."""
  _, _, models, _ = mods
  bundle = _bundle(which)
  model = models.Model(bundle)
  model.init(seed=7)
  plan = model.plans['NerfMLP_0']
  rng = np.random.default_rng(11)
  pts = np.concatenate([rng.uniform(-1, 1, (N // 2, 3)), rng.uniform(-4, 4, (N - N // 2, 3))]).astype(np.float32)
  vd = torch.nn.functional.normalize(torch.tensor(rng.normal(size=(N, 3)).astype(np.float32)), dim=-1)
  var = 2e-4
  assert model._use_chain(plan, N) == (which == 'plumbing' and N >= 512)
  p = torch.tensor(pts, device='cuda')
  dens, rgb = model.query_radiance(p, var, vd.cuda() if bundle.model.use_viewdirs else None)
  dens_q = model.query_density(p, var)
  torch.cuda.synchronize()
  assert dens.shape == (N,) and rgb.shape == (N, 3) and dens.dtype == rgb.dtype == torch.float32
  assert torch.equal(dens, dens_q)
  tree = torch_tree(model.export_flax())['NerfMLP_0']
  means = torch.tensor(pts)[:, None, :]
  covs = (torch.eye(3) * float(np.float32(var))).expand(N, 1, 3, 3).contiguous()
  glo = torch.zeros(N, bundle.model.num_glo_features) if bundle.model.num_glo_features else None
  with torch.no_grad() if bundle.nerf_mlp.disable_density_normals else torch.enable_grad():
    out = o_models.mlp_apply(tree, bundle.nerf_mlp, plan.basis, (means, covs),
                             viewdirs=vd if bundle.model.use_viewdirs else None, glo_vec=glo, bf16=True)
  ref = out['density'][:, 0].detach()
  err = (dens.cpu() - ref).abs() / (1.0 + ref.abs())
  assert float(err.max()) < 0.1 and float(err.mean()) < 5e-3, (float(err.max()), float(err.mean()))
  close(rgb, out['rgb'][:, 0].detach(), atol=rgb_tol, rtol=0, msg='rgb')
  if which == 'viewindep':
    _, rgb2 = model.query_radiance(p, var, None)
    assert torch.equal(rgb, rgb2)


def test_query_radiance_needs_view_directions(mods):
  _, _, models, _ = mods
  model = models.Model(mini360())
  model.init(seed=1)
  pts = torch.zeros(10, 3, device='cuda')
  with pytest.raises(ValueError, match='viewdirs'):
    model.query_radiance(pts, 1e-4, None)
  with pytest.raises(ValueError, match='view directions'):
    model.query_radiance(pts, 1e-4, torch.zeros(9, 3, device='cuda'))


# ------------------------------------------------------------------ composition

def test_extract_mesh_colors_composition(mods):
  _, ops, models, mesh = mods
  model = models.Model(plumbing_blender())
  model.init(seed=3)
  bbox = (-1.5, -1.2, -1.0, 1.5, 1.2, 1.0)
  res = 31
  grid, h = mesh.density_grid(model, bbox, res)
  level = float(grid.median())
  v0, f0 = mesh.extract_mesh(model, bbox, res, level)
  v, f, n, c = mesh.extract_mesh(model, bbox, res, level, colors=True)
  torch.cuda.synchronize()
  assert len(f) > 0 and torch.equal(v, v0) and torch.equal(f, f0)
  assert n.shape == v.shape and n.dtype == torch.float32 and c.shape == v.shape and c.dtype == torch.uint8
  assert float((n.norm(dim=1) - 1).abs().max()) <= 1e-6
  _, _, gn = ops.marching_cubes(grid, level, normals=True)
  assert torch.equal(n, gn)
  assert torch.equal(c, mesh.vertex_colors(model, v, gn, h * h / 12))
  _, rgb = model.query_radiance(v, h * h / 12, -gn)
  assert torch.equal(c, (rgb.clamp(0, 1) * 255).round().to(torch.uint8))


# ------------------------------------------------------------------ extract_mesh.py end to end

def test_extract_mesh_script_colors(tmp_path, capsys):
  sys.path.insert(0, ROOT)
  from multinerf_b200 import lib
  lib.require_device()
  import extract_mesh as mesh_script
  import train as train_script
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
  path = mesh_script.main(argv + ['--gin_bindings=Config.mesh_resolution = 40', '--gin_bindings=Config.mesh_level = 1.',
                                  '--gin_bindings=Config.mesh_vertex_colors = True'])
  printed = capsys.readouterr().out
  assert path == os.path.join(ckpt, 'mesh', f'mesh_step_{steps}.ply') and os.path.exists(path)
  line = [l for l in printed.splitlines() if 'vertices,' in l][-1]
  nv, nf = int(line.split(' vertices,')[0]), int(line.split(' vertices, ')[1].split(' faces')[0])
  props, f = read_ply_props(path)
  assert list(props) == ['x', 'y', 'z', 'nx', 'ny', 'nz', 'red', 'green', 'blue']
  assert len(props['x']) == nv and f.shape == (nf, 3) and nv > 0
  n = np.stack([props['nx'], props['ny'], props['nz']], 1)
  assert np.all(np.abs(np.linalg.norm(n, axis=1) - 1) <= 1e-6)
  rgb = np.stack([props['red'], props['green'], props['blue']], 1)
  assert len(np.unique(rgb, axis=0)) > 1
