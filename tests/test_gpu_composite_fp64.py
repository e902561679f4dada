"""Compositing and loss kernels (mnrf_composite_fwd, mnrf_composite_bwd) against an fp64 reference.

The reference (tests/composite_ref.py) is the oracle evaluated on the kernels' own fp32 inputs promoted to float64
and differentiated by torch.autograd.  Tolerance: per ray, the kernel's largest error against fp64 may be at most 4x
the fp32 oracle's own error (the same reference evaluated in float32) plus a few fp32 ulps of the ray's largest
value.  The cases sweep every sample-count instance of the kernels (CH = 1, 2, 4, 8) and its ragged edge, ray counts
that leave warps idle or give each warp several rays, every loss type, ray-distance function and optional input.
Every batch of five or more rays carries the edge rays of `_edge_rays`.  Needs an H100.
"""
import numpy as np
import pytest
import torch

import composite_ref as R

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -23
# (near, far) valid for each ray-distance function; ray 3 of a reciprocal batch gets far = 1e6
NEAR_FAR = {None: (2.0, 6.0), 'reciprocal': (0.2, 100.0), 'log': (0.5, 10.0), 'exp': (0.0, 2.0), 'sqrt': (0.0, 4.0),
            'square': (0.5, 3.0), 'piecewise': (0.2, 50.0)}
BASE = dict(density_bias=-1.0, density_noise=0.0, rgb_premultiplier=1.0, rgb_padding=0.001, bg_const=0.7)

# (S, B, level, loss type, lossmult channels, raydist, rgb activation, opaque background, options, Sf)
# level 'fine': colour, distortion loss; 'prop': no colour, interlevel loss against a final level of Sf samples.
# options: n density_noise, b bg_rgb, s rgb_scale, e extra_dw, m data_mask, r rgb_mode 1 with a tint,
#          R rgb_mode 1 without one.
CASES = [
    (1, 1, 'fine', 'mse', 1, 'reciprocal', 'sigmoid', True, '', 0),
    (1, 5, 'prop', 'charb', 3, None, 'sigmoid', False, 'nb', 17),
    (2, 5, 'fine', 'rawnerf', 3, 'log', 'safe_exp', False, 'se', 0),
    (17, 5, 'fine', 'charb', 1, 'exp', 'sigmoid', True, 'nbr', 0),
    (17, 1, 'prop', 'mse', 1, 'sqrt', 'sigmoid', False, 'm', 32),
    (32, 5, 'prop', 'rawnerf', 1, 'square', 'sigmoid', True, 'ne', 64),
    (33, 5, 'fine', 'mse', 3, 'piecewise', 'sigmoid', False, 'sRm', 0),
    (48, 5, 'fine', 'charb', 3, 'reciprocal', 'safe_exp', False, 'bse', 0),
    (64, 5, 'prop', 'charb', 1, 'reciprocal', 'sigmoid', True, 'bm', 128),
    (65, 5, 'fine', 'rawnerf', 1, None, 'sigmoid', True, 'nrm', 0),
    (100, 5, 'fine', 'mse', 1, 'log', 'sigmoid', False, 'nbsR', 0),
    (128, 1, 'fine', 'charb', 3, 'square', 'safe_exp', False, 'be', 0),
    (129, 5, 'prop', 'mse', 3, 'exp', 'sigmoid', False, 'nbe', 17),
    (200, 5, 'fine', 'mse', 3, 'sqrt', 'sigmoid', True, 'sre', 0),
    (256, 5, 'fine', 'rawnerf', 3, 'piecewise', 'sigmoid', False, 'nbsm', 0),
    (256, 5, 'prop', 'charb', 1, 'reciprocal', 'sigmoid', False, 'e', 32),
    # more rays than one launch has warps (132 SMs x 16 blocks x 4 warps = 8448): every warp composites two or three
    # rays, reusing its shared-memory buffers and carrying its loss partials from one ray to the next
    (48, 20000, 'prop', 'mse', 1, 'reciprocal', 'sigmoid', True, 'n', 64),
    (100, 20000, 'fine', 'charb', 3, 'reciprocal', 'sigmoid', False, 'bsr', 0),
]


@pytest.fixture(scope='module')
def ops():
  from multinerf_b200 import lib, ops as _ops
  lib.require_device()
  return _ops


def _case_id(c):
  S, B, level, loss, lm, rd, act, opaque, opts, Sf = c
  return f'S{S}-B{B}-{level}{Sf or ""}-{loss}{lm}-{rd}-{act}-{"opaque" if opaque else "translucent"}-{opts or "plain"}'


def _edge_rays(rng, S, B, raydist, sdist, raw_d, dirs, far):
  """Rays 0-4 of a batch: an empty ray, a ray whose first sample is opaque (T underflows to 0 after it), a ray of
  zero-width intervals (duplicate knots, delta = 0), a ray with far = 1e6 (under the reciprocal warp) and a ray with
  a direction of norm 3."""
  raw_d[0] = -50.0
  raw_d[1] = 30.0
  sdist[1, 1:] = 0.5 + 0.5 * sdist[1, 1:]     # first interval: half the ray
  dirs[1] *= 200.0 / np.linalg.norm(dirs[1])
  if S == 1:
    sdist[2, 1] = sdist[2, 0]
  else:
    sdist[2, 1:S:3] = sdist[2, 0:S - 1:3]
  if raydist == 'reciprocal':
    far[3] = 1e6
  dirs[4] *= 3.0 / np.linalg.norm(dirs[4])


def _make(case, seed):
  """fp32 inputs (CPU tensors), the composite cfg and the loss settings of one case."""
  S, B, level, loss_type, lm_ch, raydist, act, opaque, opts, Sf = case
  rng = np.random.default_rng(seed)
  f = np.float32
  sdist = np.sort(rng.uniform(0, 1, (B, S + 1)), -1)
  sdist[:, 0], sdist[:, -1] = 0, 1
  dup = rng.uniform(size=B) < 0.2                                  # some more duplicate knots
  sdist[dup, S // 2] = sdist[dup, max(S // 2 - 1, 0)]
  raw_d = rng.normal(size=(B, S)) * 3
  d = rng.normal(size=(B, 3))
  d = d / np.linalg.norm(d, axis=-1, keepdims=True) * rng.uniform(0.8, 1.2, (B, 1))
  near, far = NEAR_FAR[raydist]
  nearv, farv = np.full(B, near), np.full(B, far)
  if B >= 5:
    _edge_rays(rng, S, B, raydist, sdist, raw_d, d, farv)
  inp = dict(raw_density=raw_d, sdist=sdist, directions=d, near=nearv, far=farv,
             target=rng.uniform(0, 1, (B, 3)),
             lossmult=rng.integers(0, 3, (B, lm_ch)) + (rng.uniform(size=(B, lm_ch)) < 0.5) * 0.5)
  inp['lossmult'][0] = 1.0
  rgb = level == 'fine'
  if rgb:
    inp['raw_rgb'] = rng.normal(size=(B, S, 3)) * 1.5
  if 'n' in opts:
    inp['density_noise'] = rng.normal(size=(B, S))
  if 'b' in opts:
    inp['bg_rgb'] = rng.uniform(0, 1, (B, 3))
  if 's' in opts:
    sc = rng.uniform(0.5, 2.0, (B, 3))
    sc[3, 0] = 0.0                                                # a zero and a negative exposure channel
    sc[4, 1] = -0.7
    inp['rgb_scale'] = sc
  if 'e' in opts:
    inp['extra_dw'] = rng.normal(size=(B, S)) * 1e-2
  if 'm' in opts:
    inp['data_mask'] = (rng.uniform(size=B) < 0.7).astype(np.float64)
  if 'r' in opts or 'R' in opts:
    inp['raw_diffuse'] = rng.normal(size=(B, S, 3))
    if 'r' in opts:
      inp['raw_tint'] = rng.normal(size=(B, S, 3))
  if level == 'prop':
    # the final level's intervals share about half their knots with this level's (the envelope)
    k = min(S - 1, Sf // 2)
    own = np.stack([rng.choice(sdist[i, 1:S], k, replace=False) for i in range(B)]) if k > 0 else np.zeros((B, 0))
    sf = np.sort(np.concatenate([own, rng.uniform(0, 1, (B, Sf - 1 - k))], -1), -1)
    inp['sdist_fine'] = np.concatenate([np.zeros((B, 1)), sf, np.ones((B, 1))], -1)
    wf = rng.uniform(0, 1, (B, Sf)) ** 2
    inp['weights_fine'] = wf / wf.sum(-1, keepdims=True) * 0.9
  inp = {k: torch.tensor(np.asarray(v).astype(f)) for k, v in inp.items()}
  cfg = dict(BASE, raydist_fn=raydist, opaque_background=opaque, rgb_activation=act,
             rgb_bias=-1.0 if act == 'safe_exp' else 0.0, density_noise=0.5 if 'n' in opts else 0.0,
             rgb_mode=1 if ('r' in opts or 'R' in opts) else 0)
  if act == 'safe_exp':
    cfg['rgb_padding'] = 0.0
  inv_denom = np.float32(1.0 / float(inp['lossmult'].expand(B, 3).double().sum()))
  loss = dict(loss_type=loss_type, charb_padding=0.001, data_mult=0.1 if level == 'prop' else (0.5 if seed % 2 else 1.0),
              distortion_mult=0.01 if level == 'fine' else 0.0, interlevel_mult=1.0 if level == 'prop' else 0.0,
              inv_denom=float(inv_denom))
  return inp, cfg, loss


def _kernel(ops, inp, cfg, loss):
  """Forward outputs, gradients and stats of the kernels on fp32 CUDA copies of `inp`."""
  g = {k: v.cuda() for k, v in inp.items()}
  B, S = g['raw_density'].shape
  opt = {k: g.get(k) for k in ('density_noise', 'bg_rgb', 'rgb_scale', 'raw_diffuse', 'raw_tint')}
  fwd = ops.composite_fwd(g['raw_density'], g.get('raw_rgb'), g['sdist'], g['directions'], g['near'], g['far'],
                          cfg=cfg, want_samples=True, want_extras=True, **opt)
  stats = torch.zeros(8, device='cuda')
  out = dict(stats=stats)
  if g.get('rgb_scale') is not None:
    out['d_rgb_scale'] = torch.full((B, 3), float('nan'), device='cuda')
  if cfg['rgb_mode'] == 1:
    out['d_raw_diffuse'] = torch.full((B, S, 3), float('nan'), device='cuda')
    out['d_raw_tint'] = torch.full((B, S, 3), float('nan'), device='cuda')
  d_d, d_rgb = ops.composite_bwd(
      g['raw_density'], g.get('raw_rgb'), g['sdist'], g['directions'], g['near'], g['far'], g['target'],
      g['lossmult'], torch.tensor([loss['inv_denom']], device='cuda'), stats, cfg=cfg, loss_type=loss['loss_type'],
      charb_padding=loss['charb_padding'], data_mult=loss['data_mult'], distortion_mult=loss['distortion_mult'],
      interlevel_mult=loss['interlevel_mult'], sdist_fine=g.get('sdist_fine'), weights_fine=g.get('weights_fine'),
      extra_dw=g.get('extra_dw'), data_mask=g.get('data_mask'), d_rgb_scale=out.get('d_rgb_scale'),
      d_raw_diffuse=out.get('d_raw_diffuse'), d_raw_tint=out.get('d_raw_tint'), **opt)
  out.update(fwd=fwd, raw_density=d_d, raw_rgb=d_rgb)
  return out


def _within(name, got, r64, r32, mag=None, floor=None, ulps=8.0):
  """Per ray: max |kernel - fp64| <= 4 max |fp32 oracle - fp64| + `ulps` fp32 ulps of the ray's magnitude (`mag`
  [B], by default max |fp64| over the ray) + `floor` [B] (an error fp32 cannot avoid, see the test)."""
  got, r64, r32 = (x.detach().to('cpu', torch.float64).reshape(x.shape[0], -1) for x in (got, r64, r32))
  assert torch.isfinite(got).all(), f'{name}: non-finite kernel output'
  e_k = (got - r64).abs().amax(1)
  e_o = (r32 - r64).abs().amax(1)
  mag = r64.abs().amax(1) if mag is None else mag.detach().to('cpu', torch.float64)
  allowed = 4 * e_o + ulps * EPS * mag
  if floor is not None:
    allowed = allowed + floor.detach().to('cpu', torch.float64)
  bad = e_k > allowed
  if bad.any():
    i = int(torch.argmax(e_k / allowed.clamp(min=1e-300)))
    raise AssertionError(f'{name}: {int(bad.sum())}/{bad.numel()} rays off; worst ray {i}: err {float(e_k[i]):.3e} > '
                         f'allowed {float(allowed[i]):.3e} (fp32 oracle err {float(e_o[i]):.3e}, '
                         f'|row| {float(r64[i].abs().max()):.3e})')


def _rows_max(x):
  return x.detach().reshape(x.shape[0], -1).abs().amax(1)


@pytest.mark.parametrize('case', CASES, ids=[_case_id(c) for c in CASES])
def test_composite_vs_fp64(ops, case):
  S, B, level, loss_type, lm_ch, raydist, act, opaque, opts, Sf = case
  inp, cfg, loss = _make(case, seed=CASES.index(case))
  k = _kernel(ops, inp, cfg, loss)
  fwd = k['fwd']
  # The background weight max(0, 1 - acc) has zero gradient in the kernel when its fp32 acc rounds to 1 or more
  # (a tie 1 - acc == 0 included, where JAX would pass half the gradient); the reference takes the same branch.
  bg_on = (1.0 - fwd['acc']) > 0
  # fp64 on the CPU (on the GPU for the large batches); the fp32 oracle on the GPU, so that its exp / log have the
  # kernel's accuracy (alpha = 1 - exp(-density delta) cancels for thin intervals in both)
  dev = 'cuda' if B > 1000 else 'cpu'
  in64 = {k_: v.to(dev, torch.float64) for k_, v in inp.items()}
  in32 = {k_: v.cuda() for k_, v in inp.items()}
  # rgb_mode 1: an sRGB value within rounding of 0 or 1 (or a linear value of the piecewise threshold) is on one
  # side in fp32 and on the other in fp64; both references take the side of the kernel's fp32 arithmetic.
  br = None
  if cfg['rgb_mode'] == 1:
    br = R.srgb_branches(in32['raw_rgb'], cfg, in32['raw_diffuse'], in32.get('raw_tint'))
  br64 = None if br is None else {k_: v.to(dev) for k_, v in br.items()}
  with torch.device(dev):
    r64, g64 = R.grads(in64, cfg, loss, bg_on.to(dev), branches=br64)
  with torch.device('cuda'):
    r32, g32 = R.grads(in32, cfg, loss, bg_on, branches=br)

  for name in ('weights', 'density', 'rgb_samples', 'acc'):
    _within(name, fwd[name], r64[name], r32[name])
  # the pixel's scale is that of its terms: sum_s w_s |c_s| + |bg| (1 - acc cancels on an opaque ray)
  bg = in64['bg_rgb'] if 'bg_rgb' in in64 else torch.full((B, 3), R.f32(cfg['bg_const']), dtype=torch.float64,
                                                          device=dev)
  pixmag = _rows_max((r64['weights'][..., None] * r64['rgb_samples'].abs()).sum(-2) + bg.abs())
  _within('rgb', fwd['rgb'], r64['rgb'], r32['rgb'], mag=pixmag)
  _within('distance_mean', fwd['dist'][:, 0], r64['distance_mean'], r32['distance_mean'])
  # A percentile is piecewise linear in the CDF: where a knot of the CDF lies within rounding of p, fp32 and fp64
  # pick different intervals and the distance jumps.  Compare where each answer sits in the fp64 CDF instead (a CDF
  # runs from 0 to 1).
  p = torch.tensor([0.05, 0.5, 0.95], dtype=torch.float64, device=dev).expand(B, 3)
  with torch.device(dev):
    cdf_k = R.cdf_at(r64['t_aug'], r64['cdf'], fwd['dist'][:, 1:].to(dev, torch.float64))
    cdf_o = R.cdf_at(r64['t_aug'], r64['cdf'], r32['percentiles'].to(dev, torch.float64))
  _within('percentiles (through the CDF)', cdf_k - p, torch.zeros_like(p), cdf_o - p, mag=torch.ones(B), ulps=16.0)

  # The charbonnier and RawNeRF losses amplify the pixel's rounding error in their gradients (1 / sqrt(r^2 + pad^2),
  # 1 / (1e-3 + clip)^2): the gradient of the fp64 reference with its pixel moved by 4 fp32 ulps of the pixel's
  # scale is an error no fp32 evaluation avoids, and it is allowed on top.
  shift = 4 * EPS * pixmag.to(dev)[:, None].expand(B, 3)
  floor = {}
  for sgn in (1, -1):
    with torch.device(dev):
      _, gs = R.grads(in64, cfg, loss, bg_on.to(dev), pixel_shift=sgn * shift, branches=br64)
    for name, v in gs.items():
      floor[name] = torch.maximum(floor.get(name, torch.zeros(B, dtype=torch.float64, device=dev)),
                                  _rows_max(v - g64[name]))
  # d loss / d (density delta)_k = g_k T_{k+1} - sum_{i>k} g_i w_i (g = d loss / d w) cancels, exactly so on an
  # opaque level without colour; its scale is that of its terms, max |g| T_{k+1}.  It sums up to S terms (and g
  # the interlevel loss's prefix sums), so 16 ulps of that.
  dd_mag = _rows_max(_rows_max(g64['weights'])[:, None] * r64['trans_after'] * r64['dtau_draw'])
  _within('d_raw_density', k['raw_density'], g64['raw_density'], g32['raw_density'],
          mag=torch.maximum(dd_mag, _rows_max(g64['raw_density'])), floor=floor['raw_density'], ulps=16.0)
  for name in ('raw_rgb', 'rgb_scale', 'raw_diffuse', 'raw_tint'):
    if name in g64:
      got = k[name] if name == 'raw_rgb' else k['d_' + name]
      _within('d_' + name, got, g64[name], g32[name], floor=floor[name])
  if cfg['rgb_mode'] == 1 and 'raw_tint' not in inp:
    assert (k['d_raw_tint'] == 0).all()                          # constant tint 0.5: zero gradient written

  # loss partials: summed over rays in fp32 (per warp, then one atomic per warp), so the floor grows with the
  # number of terms; a ray that loses its partial moves the sum by far more
  st = k['stats'].cpu().double()
  for i, name in enumerate(('data', 'mse', 'distortion', 'interlevel')):
    n = B * (3 if i < 2 else 1)
    ref, o32 = float(r64[name].detach()), float(r32[name].detach())
    allowed = 4 * abs(o32 - ref) + 4 * np.sqrt(n) * EPS * abs(ref) + 1e-30
    assert abs(float(st[i]) - ref) <= allowed, (name, float(st[i]), ref, o32)
  assert (st[4:] == 0).all()


@pytest.mark.parametrize('S', [48, 200])
def test_strided_rows_bitwise(ops, S):
  """raw_density / raw_rgb and their gradients as column views of [B*S, 8] buffers (the stacked [density | rgb]
  head of view-independent colour): bit-identical to the contiguous run, and no other column is written."""
  case = (S, 37, 'fine', 'charb', 3, 'reciprocal', 'sigmoid', False, 'nbs', 0)
  inp, cfg, loss = _make(case, seed=S)
  B = 37
  ref = _kernel(ops, inp, cfg, loss)
  sentinel = -12345.0
  X = torch.full((B * S, 8), sentinel, device='cuda')
  G = torch.full((B * S, 8), sentinel, device='cuda')
  X[:, 3] = inp['raw_density'].reshape(-1).cuda()
  X[:, 4:7] = inp['raw_rgb'].reshape(-1, 3).cuda()
  X0 = X.clone()
  xd, xr = X[:, 3].view(B, S), X[:, 4:7].view(B, S, 3)
  gd, gr = G[:, 0].view(B, S), G[:, 1:4].view(B, S, 3)
  g = {k: v.cuda() for k, v in inp.items()}
  opt = {k: g.get(k) for k in ('density_noise', 'bg_rgb', 'rgb_scale')}
  fwd = ops.composite_fwd(xd, xr, g['sdist'], g['directions'], g['near'], g['far'], cfg=cfg, want_samples=True,
                          want_extras=True, **opt)
  for name, v in fwd.items():
    assert torch.equal(v, ref['fwd'][name]), name
  stats = torch.zeros(8, device='cuda')
  d_scale = torch.empty(B, 3, device='cuda')
  ops.composite_bwd(xd, xr, g['sdist'], g['directions'], g['near'], g['far'], g['target'], g['lossmult'],
                    torch.tensor([loss['inv_denom']], device='cuda'), stats, cfg=cfg, loss_type=loss['loss_type'],
                    charb_padding=loss['charb_padding'], data_mult=loss['data_mult'],
                    distortion_mult=loss['distortion_mult'], interlevel_mult=0.0, d_raw_density=gd, d_raw_rgb=gr,
                    d_rgb_scale=d_scale, **opt)
  assert torch.equal(gd, ref['raw_density']) and torch.equal(gr, ref['raw_rgb'])
  assert torch.equal(d_scale, ref['d_rgb_scale'])
  assert torch.equal(X, X0), 'an input column was written'
  assert (G[:, 4:] == sentinel).all(), 'a column outside the gradient views was written'
