"""Meshes in contracted space on the GPU (Config.mesh_space = 'contracted'): mnrf_mesh_uncontract against fp64, the
encoder's warp_contract 2, the contracted density grid against the world grid where the two coincide, an analytic
unbounded scene through a stub model (a sphere, an off-centre box and a distant shell), mnrf_tsdf_integrate_contracted
against the fp64 fusion of tests/contract_ref.py, and the full option chain on a random-init 360 model.  Needs an
H100."""
import types

import numpy as np
import pytest
import torch

import contract_ref
import tsdf_ref
from model_parity import mini360
from test_gpu_contract_normals import mini360_normals
from test_gpu_mesh_tsdf import CAMS, _views

pytestmark = pytest.mark.gpu
EPS32 = float(np.finfo(np.float32).eps)


@pytest.fixture(scope='module')
def mods():
  from multinerf_b200 import lib, mesh, models, ops
  lib.require_device()
  return ops, mesh, models


def _dirs(rng, n):
  d = rng.normal(size=(n, 3))
  return d / np.linalg.norm(d, axis=-1, keepdims=True)


# ------------------------------------------------------------------ mnrf_mesh_uncontract

@pytest.mark.parametrize('h', [4 / 1023, 4 / 255, 4 / 63])
def test_uncontract_vs_fp64(mods, h):
  """Every point with |p| <= 2 - h: |x - x64| <= 8 eps32 |x64| / (2 - |p|) (the rounding of 2 - r, relative); normals
  within 16 eps32 / (2 - |p|) of the fp64 unit J n."""
  ops, _, _ = mods
  rng = np.random.default_rng(int(4 / h))
  n = 200000
  r = np.concatenate([rng.uniform(0, 2 - h, n - 4), [0.0, 1.0, 1.0 + 1e-6, 2 - h]])
  p = (_dirs(rng, n) * r[:, None]).astype(np.float32)
  nc = _dirs(rng, n).astype(np.float32)
  world, wn = ops.mesh_uncontract(torch.tensor(p, device='cuda'), torch.tensor(nc, device='cuda'))
  p64 = p.astype(np.float64)
  rp = np.linalg.norm(p64, axis=-1)
  x64 = contract_ref.inv_contract(p64)
  amp = 1 + 1 / np.maximum(2 - rp, 1e-30)
  err = np.abs(world.cpu().double().numpy() - x64)
  assert (err <= 8 * EPS32 * amp[:, None] * np.abs(x64).max(-1, keepdims=True) + 1e-37).all(), err.max()
  want = contract_ref.world_normals(p64, nc.astype(np.float64))
  nerr = np.abs(wn.cpu().double().numpy() - want).max(-1)
  assert (nerr <= 16 * EPS32 * amp).all(), float((nerr / amp).max())
  # fallbacks: a zero normal gives (0, 0, 1); points only
  z = torch.zeros(1, 3, device='cuda')
  assert torch.equal(ops.mesh_uncontract(z, z)[1].cpu(), torch.tensor([[0.0, 0.0, 1.0]]))
  assert torch.equal(ops.mesh_uncontract(world.new_tensor(p[:1000])), world[:1000])
  with pytest.raises(ValueError):
    ops.mesh_uncontract(torch.tensor([[2.0, 0.0, 0.0]], device='cuda'))
  with pytest.raises(ValueError):
    ops.mesh_uncontract(torch.tensor([[float('nan'), 0.0, 0.0]], device='cuda'))


# ------------------------------------------------------------------ encoder warp_contract 2

def test_encoder_mode2_features_and_tangents(mods):
  """Feature rows bit-identical to mode 0 (tangent and plain entry points); tangent rows against the fp64 derivative
  of the feature formula times the fp64 J(inv_contract(p)): for feature e sin(y) (cos: e sin(y + pi/2)), y = (b.p) sc,
  e = exp(-var |b|^2 sc^2 / 2), row dir is e cos(y) sc (J b)_dir (cos: -e sin(y) sc (J b)_dir).  Bound: bf16 rounding
  2^-8 |ref|, plus e sc |J| |b| times 8 eps32 (|y| + sum |b_i p_i| sc + 1) for the fp32 argument, 64 eps32 /
  (2 - |p|) for J from fp32 x and 1e-5 for the exponential."""
  ops, _, _ = mods
  rng = np.random.default_rng(9)
  N, K, L = 3000, 21, 12
  basis = torch.tensor(_dirs(rng, K), device='cuda', dtype=torch.float32)
  p = torch.tensor(_dirs(rng, N) * rng.uniform(0, 2 - 4 / 1023, (N, 1)), device='cuda', dtype=torch.float32)
  var = (4 / 511) ** 2 / 12
  KL = K * L
  cols = (2 * KL + 63) // 64 * 64
  out = {}
  for mode in (0, 2):
    feat = torch.empty(N, cols, device='cuda', dtype=torch.bfloat16)
    tfeat = torch.empty(3 * N, cols, device='cuda', dtype=torch.bfloat16)
    ops.encode_points(p, var, basis, min_deg=0, max_deg=L, warp_contract=mode, feat=feat, feat_cols=cols,
                      tfeat=tfeat)
    out[mode] = (feat, tfeat.view(3, N, cols))
  assert torch.equal(out[0][0], out[2][0])
  plain = torch.empty(N, cols, device='cuda', dtype=torch.bfloat16)
  ops.encode_points(p, var, basis, min_deg=0, max_deg=L, warp_contract=2, feat=plain, feat_cols=cols)
  ref0 = torch.empty_like(plain)
  ops.encode_points(p, var, basis, min_deg=0, max_deg=L, warp_contract=0, feat=ref0, feat_cols=cols)
  assert torch.equal(plain, ref0)
  p64 = p.cpu().double().numpy()
  b64 = basis.cpu().double().numpy()                                                   # [K, 3]
  J = contract_ref.jacobian(contract_ref.inv_contract(p64))                           # [N, 3, 3]
  Jb = np.einsum('nij,kj->nki', J, b64)                                                # [N, K, 3]
  sc = 2.0 ** np.arange(L)                                                             # [L]
  y = (p64 @ b64.T)[:, None, :] * sc[None, :, None]                                    # [N, L, K]
  e = np.exp(-0.5 * var * (b64 * b64).sum(-1)[None, None, :] * sc[None, :, None] ** 2)
  esc = e * sc[None, :, None]
  d_sin = (esc * np.cos(y))[..., None] * Jb[:, None]                                  # [N, L, K, 3]
  d_cos = (-esc * np.sin(y))[..., None] * Jb[:, None]
  want = np.concatenate([d_sin.reshape(N, KL, 3), d_cos.reshape(N, KL, 3)], 1)          # [N, 2KL, 3]
  amp = 1 / (2 - np.linalg.norm(p64, axis=-1))
  # u = J b is formed as s b_t + q (xh.b) xh in fp32: its rounding scales with |J| |b|, not with |J b|
  Jb_abs = np.einsum('nij,kj->nki', np.abs(J), np.abs(b64))
  # y = (b.p) sc in fp32: the dot product's rounding scales with sum |b_i p_i|, which cancellation can leave far
  # above |b.p|
  y_abs = (np.abs(p64) @ np.abs(b64).T)[:, None, :] * sc[None, :, None]
  mag = esc[..., None] * Jb_abs[:, None] * (8 * EPS32 * (np.abs(y) + y_abs + 1)[..., None] + 1e-5 +
                                                 64 * EPS32 * amp[:, None, None, None])
  mag = np.concatenate([mag.reshape(N, KL, 3)] * 2, 1)
  got = out[2][1].cpu().double().numpy()[:, :, :2 * KL].transpose(1, 2, 0)             # [N, 2KL, 3]
  err = np.abs(got - want)
  bound = 2 ** -8 * np.abs(want) + mag + 1e-30
  assert (err <= bound).all(), float((err / bound).max())
  assert (got[:, 2 * KL:] == 0).all() if got.shape[1] > 2 * KL else True


# ------------------------------------------------------------------ density grid

def _model(models, bundle):
  m = models.Model(bundle)
  m.init(seed=7)
  return m


def test_density_grid_matches_world_grid_and_skips_outside(mods):
  """[-2, 2]^3 at 2M - 1 against [-1, 1]^3 at M (M = 33): the same points inside the unit ball are bit-identical;
  outside, the unscaled density times (2 - |p|)^-2; NaN and never queried for |p| >= 2.  The faces of cells wholly
  inside the unit ball match the world extraction's."""
  ops, mesh, models = mods
  model = _model(models, mini360())
  M = 33
  calls = []
  query = model.query_density

  def counting(points, var, **kw):
    calls.append(points.shape[0])
    return query(points, var, **kw)

  model.query_density = counting
  gc, hc = mesh.density_grid(model, (-2, -2, -2, 2, 2, 2), 2 * M - 1, space='contracted')
  gw, hw = mesh.density_grid(model, (-1, -1, -1, 1, 1, 1), M)
  model.query_density = query
  assert hc == hw
  n = 2 * M - 1
  ax = (-2 + torch.arange(n, dtype=torch.float64) * hc).float()
  P = torch.stack(torch.meshgrid(ax, ax, ax, indexing='ij')[::-1], -1)           # [z, y, x, (x, y, z)]
  r2 = P.double().square().sum(-1)
  inside = r2 < 4
  assert int(inside.sum()) + M ** 3 == sum(calls)
  assert torch.isnan(gc.cpu()[~inside]).all() and torch.isfinite(gc.cpu()[inside]).all()
  q = slice((n - M) // 2, (n - M) // 2 + M)
  # where the fp32 coordinates coincide (every point of the inner grid here) and |p| <= 1: bit-identical
  axw = (-1 + torch.arange(M, dtype=torch.float64) * hw).float()
  same = (ax[q] == axw)
  assert same.all()
  ball = r2[q, q, q] <= 1
  assert torch.equal(gc.cpu()[q, q, q][ball], gw.cpu()[ball])
  # outside the unit ball: the density of mode 0 on the contracted point, scaled
  pts = P[inside & (r2 > 1)].reshape(-1, 3)[::97].cuda()
  var = hc * hc / 12
  model._contracted_mode = lambda cfg, contracted: 0
  raw = model.query_density(pts, var)
  del model._contracted_mode
  rp = pts.double().norm(dim=-1)
  want = raw.double() / (2 - rp) ** 2
  got = gc.reshape(-1)[(inside & (r2 > 1)).reshape(-1).nonzero().view(-1)[::97].cuda()]
  # the scale is computed in fp32: 2 - |p| carries the rounding of |p|, relative 2 eps32 / (2 - |p|), squared
  assert ((got.double() - want).abs() <= 8 * EPS32 * (1 + 2 / (2 - rp)) * want).all()
  # marching cubes: cells wholly inside the unit ball give the same faces
  level = float(gw.median())
  vw, fw = ops.marching_cubes(gw, level)
  vc, fc = ops.marching_cubes(gc, level)
  cell = lambda v, f, lo: torch.floor(v[f.long()].mean(1) + 0.0).long() + lo
  cw_ = cell(vw, fw, (n - M) // 2)
  cc_ = cell(vc, fc, 0)
  def inner(cells):
    corner = (cells.double() * hc - 2)
    far = torch.maximum(corner.abs(), (corner + hc).abs())
    return far.square().sum(-1) <= 1
  # the two grids' vertices are x + t with the same t at cell indices 16 apart: triangles are matched by the integer
  # parts of their corners and compared to 1e-5 of a cell, which absorbs the offset's fp32 rounding

  def tri(v, f, lo, sel):
    corners = (v[f[sel].long()].double() + lo).cpu().numpy()                    # [T, 3, 3]
    corners = np.sort(corners.view([('', corners.dtype)] * 3).reshape(len(sel), 3), axis=1).view(np.float64)
    corners = corners.reshape(len(sel), 3, 3)
    keys = [tuple(np.floor(c).astype(int).ravel()) for c in corners]
    order = sorted(range(len(keys)), key=keys.__getitem__)
    return [keys[i] for i in order], corners[order]

  sw = inner(cw_).nonzero().view(-1).cpu()
  sc = inner(cc_).nonzero().view(-1).cpu()
  assert len(sw) == len(sc) > 0
  kw, pw = tri(vw, fw, (n - M) // 2, sw)
  kc, pc = tri(vc, fc, 0, sc)
  assert kw == kc and np.abs(pw - pc).max() <= 1e-5


# ------------------------------------------------------------------ analytic scene

SPHERE_R, BOX_C, BOX_H, SHELL_R = 0.5, (3.0, 0.0, 0.0), 0.5, 20.0


def _world_sdf(x):
  """Signed distance (inside < 0) to the union of a sphere of radius 0.5 at the origin, the box |x - (3, 0, 0)|_inf
  <= 0.5 and the solid beyond |x| = 20; and the index of the nearest solid."""
  r = x.norm(dim=-1)
  q = (x - torch.tensor(BOX_C, dtype=x.dtype, device=x.device)).abs() - BOX_H
  box = q.clamp_min(0).norm(dim=-1) + q.max(-1).values.clamp_max(0)
  sds = torch.stack([r - SPHERE_R, box, SHELL_R - r], -1)
  return sds.min(-1).values, sds.argmin(-1)


class AnalyticModel:
  """query_density only: sigma_c = level * 2^(-sd_c / h) with sd_c the world signed distance over the world length
  per unit of contracted length, so the level set sigma_c = level is the union's surface."""
  def __init__(self, level, h):
    self.level, self.h = level, h
    self.device = torch.device('cuda')
    self.config = types.SimpleNamespace(render_chunk_size=4096)
    self.mcfg = types.SimpleNamespace(num_nerf_samples=64)

  def query_density(self, points, var, contracted=False):
    p = points.double()
    if contracted:
      m = p.square().sum(-1, keepdim=True)
      x = torch.where(m <= 1, p, p / (m.sqrt() * (2 - m.sqrt())))
      scale = torch.where(m[:, 0] <= 1, torch.ones_like(m[:, 0]), x.square().sum(-1))
    else:
      x, scale = p, torch.ones_like(p[:, 0])
    sd, _ = _world_sdf(x)
    return (self.level * torch.exp2((-sd / scale / self.h).clamp(-60, 60))).float()


def test_analytic_unbounded_scene(mods):
  _, mesh, _ = mods
  res = 257
  h = 4 / (res - 1)
  level = 10.0
  model = AnalyticModel(level, h)
  v, f = mesh.extract_mesh(model, (-2, -2, -2, 2, 2, 2), res, level, space='contracted')
  grid, _ = mesh.density_grid(model, (-2, -2, -2, 2, 2, 2), res, space='contracted')
  from multinerf_b200 import ops
  out = ops.marching_cubes(grid, level, normals=True)
  vc = out[0] * h - 2
  vw, nw = ops.mesh_uncontract(vc, out[2])
  assert torch.equal(vw, v)
  x = vw.double()
  sd, which = _world_sdf(x)
  r = x.norm(dim=-1)
  z = vc.double()
  rz = z.norm(dim=-1)
  # every vertex within one contracted cell of its solid's contracted surface
  sphere, box, shell = (which == 0), (which == 1), (which == 2)
  assert sphere.sum() > 100 and box.sum() > 100 and shell.sum() > 1000
  assert ((rz[sphere] - SPHERE_R).abs() <= h).all()
  assert ((rz[shell] - (2 - 1 / SHELL_R)).abs() <= h).all()
  # the box's contracted surface: its world distance over the world length of one contracted cell (|x|^2 radially)
  assert (sd[box].abs() <= h * r[box] ** 2).all()
  # normals point out of the solids
  xh = x / r[:, None]
  nd = nw.double()
  assert ((nd[sphere] * xh[sphere]).sum(-1) > 0.99).all()
  # on the shell only the sign is asked: J there scales tangential parts by 39 against radial ones, so the grid
  # gradient's own tangential error of a fraction of a degree turns into tens of degrees in world space
  assert ((nd[shell] * xh[shell]).sum(-1) < 0).all()
  q = x[box] - torch.tensor(BOX_C, dtype=torch.float64, device=x.device)
  face = q.abs().argmax(-1)
  others = q.abs().sort(-1).values[:, 1]
  centre = others < 0.35                         # away from the box's edges
  axis = torch.nn.functional.one_hot(face, 3).double() * q.sign()
  cosang = (nd[box] * axis).sum(-1)
  assert centre.sum() > 50
  ang = torch.rad2deg(torch.acos(cosang[centre].clamp(-1, 1)))
  assert float(ang.median()) < 3 and float(ang.max()) < 15, (float(ang.median()), float(ang.max()))
  # the world-space default box sees none of the shell or the box
  vw0, _ = mesh.extract_mesh(model, (-1, -1, -1, 1, 1, 1), 129, level)
  assert vw0.shape[0] > 0 and (vw0.norm(dim=-1) < 1.0).all()


# ------------------------------------------------------------------ contracted TSDF

def _fuse(ops, shape, lo, h, camtype, dist, views, tau, colors, batch):
  w2c, c2p, depth, acc, rgb = (torch.tensor(a, device='cuda') for a in views)
  nx, ny, nz = shape
  zz = lambda *sh: torch.zeros(nz, ny, nx, *sh, device='cuda')
  state = [zz(), zz()] + ([zz(3), zz()] if colors else [None, None])
  K = depth.shape[0]
  for k0 in range(0, K, batch):
    sl = slice(k0, k0 + batch)
    ops.tsdf_integrate(shape, lo, h, camtype, dist, w2c[sl].contiguous(),
                       c2p if c2p.shape[0] == 1 else c2p[sl].contiguous(), depth[sl].contiguous(),
                       acc[sl].contiguous(), rgb[sl].contiguous() if colors else None, tau, *state, contracted=True)
  return state


@pytest.mark.parametrize('cam', sorted(CAMS))
@pytest.mark.parametrize('K,per_view,colors', [(1, False, True), (6, True, False), (9, False, True)])
def test_tsdf_contracted_vs_fp64(mods, cam, K, per_view, colors):
  ops, _, _ = mods
  camtype, dist = CAMS[cam]
  rng = np.random.default_rng(K * 10 + per_view + 100 * camtype + 7)
  H, W = 30, 40
  shape = (41, 37, 33)
  lo, h = (-2.0, -1.8, -1.6), 0.1
  tau = 2.5 * h
  views = _views(rng, K, H, W, camtype, per_view)
  views = (views[0], views[1], (views[2] * rng.uniform(0.5, 8, views[2].shape)).astype(np.float32)) + views[3:]
  tsdf, weight, cs, cw = _fuse(ops, shape, lo, h, camtype, dist, views, tau, colors, K)
  pts = tsdf_ref.grid_points(shape, lo, h)
  rt, rw, rcs, rcw, bound, exempt = contract_ref.integrate_contracted(
      pts, views[0], views[1], views[2], views[3], views[4] if colors else None, tau,
      'fisheye' if camtype else 'perspective', dist)
  live = ~exempt
  assert live.mean() > 0.8, live.mean()
  assert (rw[live] > 0).mean() > 0.2 and (rw[live] == 0).any()
  assert (np.abs(rt[live][rw[live] > 0]) < 1).any() and (rt[live] == 1).any()
  g = lambda t: t.reshape(-1).cpu().double().numpy()
  assert (g(weight)[np.linalg.norm(pts, axis=-1) >= 2] == 0).all()
  assert np.array_equal(g(weight)[live], rw[live])
  err = np.abs(g(tsdf) - rt)
  assert (err[live] <= bound[live]).all(), float((err - bound)[live].max())
  if colors:
    assert np.array_equal(g(cw)[live], rcw[live])
    cerr = np.abs(cs.reshape(-1, 3).cpu().double().numpy() - rcs)
    assert (cerr[live] <= 4 * K * EPS32 * (1 + rcs[live])).all()
  for batch in (1, 4):
    other = _fuse(ops, shape, lo, h, camtype, dist, views, tau, colors, batch)
    for a, b in zip((tsdf, weight, cs, cw), other):
      assert (a is None and b is None) or torch.equal(a, b), batch


def test_tsdf_contracted_analytic_depth(mods):
  """Depth maps of the analytic scene (sphere and distant shell, closed form) from cameras inside the unit ball,
  fused and meshed in contracted space: every world vertex within `truncation` contracted cells of a surface."""
  from multinerf_b200 import camera_utils
  ops, mesh, _ = mods
  rng = np.random.default_rng(2)
  H, W, focal = 48, 64, 40.0
  c2ws = []
  pix = camera_utils.get_pixtocam(focal, W, H)
  for k in range(24):
    eye = _dirs(rng, 1)[0] * 0.8
    zax = eye / np.linalg.norm(eye) * (1 if k % 2 else -1)       # odd views look at the sphere, even ones away
    xax = np.cross([0.0, 0.0, 1.0], zax)
    xax /= np.linalg.norm(xax)
    R = np.stack([xax, np.cross(zax, xax), zax], 1)
    c2ws.append(np.concatenate([R, eye[:, None]], 1))
  views = []
  for k, c2w in enumerate(c2ws):
    u, v = np.meshgrid(np.arange(W) + 0.5, np.arange(H) + 0.5)
    d = np.stack([u, v, np.ones_like(u)], -1) @ np.asarray(pix).T
    d = np.stack([d[..., 0], -d[..., 1], -np.ones_like(u)], -1) @ c2w[:, :3].T
    o = c2w[:, 3]
    # closed-form hits (t along d): the sphere |o + t d| = 0.5 from outside, else the shell |o + t d| = 20
    a = (d * d).sum(-1)
    b = 2 * (d @ o)
    c = o @ o
    disc_s = b * b - 4 * a * (c - SPHERE_R ** 2)
    ts = np.where(disc_s >= 0, (-b - np.sqrt(np.maximum(disc_s, 0))) / (2 * a), np.inf)
    ts = np.where(ts > 0, ts, np.inf)
    tshell = (-b + np.sqrt(b * b - 4 * a * (c - SHELL_R ** 2))) / (2 * a)
    views.append((k, torch.tensor(np.minimum(ts, tshell), device='cuda'), torch.ones(H, W, device='cuda'), None))
  cams = (pix, np.stack(c2ws), None, None)
  persp = camera_utils.ProjectionType.PERSPECTIVE
  state, hc = mesh.fuse_tsdf(views, cams, persp, (-2, -2, -2, 2, 2, 2), 129, 3.0, batch=5, space='contracted')
  vw, f = mesh.tsdf_mesh(state, (-2, -2, -2, 2, 2, 2), hc, space='contracted')
  assert f.shape[0] > 1000
  z = torch.tensor(contract_ref.contract(vw.cpu().double().numpy()))
  rz = z.norm(dim=-1)
  dist = torch.minimum((rz - SPHERE_R).abs(), (rz - (2 - 1 / SHELL_R)).abs())
  assert (dist <= 3 * hc).all(), float(dist.max())
  assert (rz > 1.9).sum() > 100 and (rz < 0.6).sum() > 100
  # batching does not change the result
  state1, _ = mesh.fuse_tsdf(views, cams, persp, (-2, -2, -2, 2, 2, 2), 129, 3.0, batch=24, space='contracted')
  assert all(torch.equal(a, b) for a, b in zip(state[:2], state1[:2]))


# ------------------------------------------------------------------ the option chain

@pytest.mark.parametrize('which', ['mini360', 'refnerf_normals'])
def test_option_chain_contracted(mods, which, tmp_path):
  """Clean, simplify, vertex colours and texture in contracted space on a random-init model: finite outputs, unit
  normals, PLY and OBJ round trips, and render_mesh on a camera inside the unit ball."""
  from multinerf_b200 import camera_utils, utils
  ops, mesh, models = mods
  bundle = mini360() if which == 'mini360' else mini360_normals(refnerf=True)
  model = _model(models, bundle)
  bbox = (-2, -2, -2, 2, 2, 2)
  grid, _ = mesh.density_grid(model, bbox, 48, space='contracted')
  level = float(grid[torch.isfinite(grid)].quantile(0.6))
  H, W = 24, 32
  pix = camera_utils.get_pixtocam(30.0, W, H)
  c2w = np.concatenate([np.eye(3), [[0.1], [0.2], [0.3]]], 1)[None]
  persp = camera_utils.ProjectionType.PERSPECTIVE
  dataset = types.SimpleNamespace(cameras=(pix, c2w, None, None), camtype=persp, height=H, width=W)
  stats = {}
  saved = {}
  out = mesh.extract_mesh(model, bbox, 48, level, colors=True, keep_components=3, min_views=1, dataset=dataset,
                          stats=stats, target_faces=2000, texture_size=256, space='contracted',
                          before_texture=lambda *a: saved.update(mesh=a))
  v, f, n, rgb, uv, tex = out
  assert f.shape[0] > 0 and stats['faces_after'] <= max(stats['faces_before'], 2000)
  assert torch.isfinite(v).all() and torch.isfinite(n).all() and torch.isfinite(uv).all()
  assert torch.allclose(n.norm(dim=-1), torch.ones(n.shape[0], device='cuda'), atol=1e-5)
  assert saved['mesh'][0] is v and rgb.dtype == torch.uint8 and tex.shape == (256, 256, 3)
  assert (v.norm(dim=-1) > 0).all()
  mesh.write_ply(tmp_path / 'm.ply', v, f, n, rgb)
  obj = mesh.write_obj(str(tmp_path / 'm.obj'), v, f, n, uv, tex)[0]
  vs = np.array([list(map(float, l.split()[1:])) for l in open(obj) if l.startswith('v ')], np.float32)
  assert np.array_equal(vs, v.cpu().numpy())
  data = open(tmp_path / 'm.ply', 'rb').read()
  head = data[:data.index(b'end_header\n') + 11]
  assert f'element vertex {v.shape[0]}'.encode() in head and f'element face {f.shape[0]}'.encode() in head
  rays = utils.Rays(origins=torch.tensor([[0.1, 0.2, 0.3]] * 64, device='cuda'),
                    directions=torch.tensor(_dirs(np.random.default_rng(1), 64), device='cuda', dtype=torch.float32),
                    near=torch.zeros(64, 1, device='cuda'), far=torch.full((64, 1), 1e6, device='cuda'),
                    viewdirs=None, radii=None, imageplane=None, lossmult=None, cam_idx=None, exposure_idx=None,
                    exposure_values=None)
  r = mesh.render_mesh(v, f, ops.mesh_bvh(v, f), rays, normals=n, uv=uv, texture=tex, bg=1.0)
  assert torch.isfinite(r['rgb']).all()
  # the TSDF method in contracted space through the same chain, from rendered-like views of the same camera
  views = [(0, torch.full((H, W), 3.0, device='cuda'), torch.ones(H, W, device='cuda'),
            torch.rand(H, W, 3, device='cuda'))]
  state, hc = mesh.fuse_tsdf(views, dataset.cameras, persp, bbox, 48, 3.0, colors=True, space='contracted')
  out = mesh.tsdf_mesh(state, bbox, hc, colors=True, target_faces=500, texture_size=128, space='contracted',
                       clean_args=dict(keep_components=1, min_views=1, cameras=dataset.cameras, camtype=persp,
                                       image_size=(H, W)))
  v2, f2, n2, rgb2, uv2, tex2 = out
  assert f2.shape[0] > 0 and torch.isfinite(v2).all()
  assert torch.allclose(n2.norm(dim=-1), torch.ones(n2.shape[0], device='cuda'), atol=1e-5)


# ------------------------------------------------------------------ extract_mesh.py on a model trained under the contraction

def read_ply(path):
  """(positions [V, 3], faces [F, 3]) of a binary PLY as mesh.write_ply writes it, with any vertex properties."""
  data = open(path, 'rb').read()
  head, body = data.split(b'end_header\n', 1)
  lines = head.decode('ascii').splitlines()
  nv = int([l for l in lines if l.startswith('element vertex')][0].split()[-1])
  props = [(l.split()[2], {'float': '<f4', 'uchar': 'u1'}[l.split()[1]]) for l in lines
           if l.startswith('property') and 'list' not in l]
  vrec = np.frombuffer(body, dtype=props, count=nv)
  rec = np.frombuffer(body[vrec.nbytes:], dtype=[('n', 'u1'), ('idx', '<i4', (3,))])
  assert np.all(rec['n'] == 3)
  return np.stack([vrec['x'], vrec['y'], vrec['z']], -1), rec['idx']


def test_extract_mesh_script_contracted(tmp_path, capsys):
  """A small model with both MLPs under the scene contraction, trained on tools/mesh_contract_coverage.py's unbounded
  scene (a sphere inside a distant room, cameras inside the unit ball); extract_mesh.py with Config.mesh_space =
  'contracted' and Config.mesh_eval, by the density method (simplified and textured) and the TSDF method (vertex
  colours): the summary names the space, the PLY is in world coordinates and reaches the room, every metric is
  written and finite."""
  import os
  import sys
  from multinerf_b200 import lib
  lib.require_device()
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  sys.path.insert(0, root)
  sys.path.insert(0, os.path.join(root, 'tools'))
  import extract_mesh as mesh_script
  import mesh_contract_coverage as coverage
  import train as train_script
  data, ckpt, steps = str(tmp_path / 'scene'), str(tmp_path / 'ckpt'), 300
  coverage.write_scene(data, n_train=24, n_test=2, W=48, H=36)
  argv = [f'--gin_bindings={b}' for b in coverage.train_bindings(data, ckpt, steps)]
  train_script.main(argv)
  base = argv + ['--gin_bindings=Config.mesh_resolution = 64', '--gin_bindings=Config.mesh_level = 2.0',
                 "--gin_bindings=Config.mesh_space = 'contracted'", '--gin_bindings=Config.mesh_eval = True']
  eval_dir = os.path.join(ckpt, 'mesh', f'eval_step_{steps}')
  for name, extra in (('density', ['--gin_bindings=Config.mesh_target_faces = 3000',
                                   '--gin_bindings=Config.mesh_texture_size = 512']),
                      ('tsdf', ["--gin_bindings=Config.mesh_method = 'tsdf'",
                                '--gin_bindings=Config.mesh_vertex_colors = True'])):
    capsys.readouterr()
    path = mesh_script.main(base + extra)
    printed = capsys.readouterr().out
    assert 'in contracted space' in printed and '(-2.0, -2.0, -2.0, 2.0, 2.0, 2.0)' in printed, printed
    v, f = read_ply(path)
    assert len(f) > 0 and np.isfinite(v).all(), name
    assert (np.linalg.norm(v, axis=-1) > 2).any(), (name, float(np.linalg.norm(v, axis=-1).max()))
    if name == 'density':
      assert os.path.exists(os.path.splitext(path)[0] + '.obj')
    for m in ('coverage', 'spurious', 'depth_abs_rel', 'nerf_psnr', 'psnr'):
      vals = np.array([float(x) for x in open(os.path.join(eval_dir, f'metric_{m}.txt')).read().split()])
      assert len(vals) == 2 and np.isfinite(vals).all(), (name, m, vals)
    for p in os.listdir(eval_dir):
      os.remove(os.path.join(eval_dir, p))
