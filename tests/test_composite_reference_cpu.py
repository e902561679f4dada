"""The reference of the compositing kernels (tests/composite_ref.py) checked on the CPU.

Gradcheck: torch.autograd.gradcheck at tiny shapes with each optional input switched on once, and the pixel and
data loss against the oracle functions the reference reassembles: the GPU test trusts its autograd gradients.

Soundness: `Emul` runs composite_ref.walk -- the kernels' arithmetic -- in numpy fp32 with the kernels' lane layout
(CH samples per lane, lane-local sums, the xor butterfly of warp_sum, the Hillis-Steele shuffle scans and the
reverse scan of `after`), expf / logf / log1pf / powf moved by their documented error in each direction, the
interlevel D atomics and the stats atomics summed in shuffled orders.  Every output lands inside its bound on every
case of tests/test_gpu_composite_fp64.py.

Sensitivity: each plausible kernel bug of composite_ref.MUTANTS, applied to the emulation, breaks a non-vacuous bound
in at least one case.  Agreement: the walk's fp64 values are the autograd reference's to fp64 rounding, and in float32
the reference is the fp32 oracle chain.

Refusals: both entry points, called through ctypes with fake non-null addresses, return an error before any launch.
They run only where no CUDA device is visible, so that a missing check can never launch.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import composite_ref as R
from oracle import o_render, o_train
from test_gpu_composite_fp64 import CASES as GPU_CASES, case_id, make

F = np.float32
SMS = 132

CFG = dict(raydist_fn='reciprocal', opaque_background=False, density_bias=-1.0, density_noise=0.0,
           rgb_activation='sigmoid', rgb_premultiplier=1.0, rgb_bias=0.0, rgb_padding=0.001, bg_const=1.0)
LOSS = dict(loss_type='mse', charb_padding=0.001, data_mult=1.0, distortion_mult=0.0, interlevel_mult=0.0)


def _inputs(seed, B=3, S=5, Sf=4, lm_ch=1):
  rng = np.random.default_rng(seed)
  sd = np.sort(rng.uniform(0, 1, (B, S + 1)), -1)
  sd[:, 0], sd[:, -1] = 0, 1
  sf = np.sort(np.concatenate([sd[:, 1:3], rng.uniform(0, 1, (B, Sf - 3))], -1), -1)   # shares two knots
  sf = np.concatenate([np.zeros((B, 1)), sf, np.ones((B, 1))], -1)
  wf = rng.uniform(0, 1, (B, Sf))
  d = rng.normal(size=(B, 3)) * 1.3
  t = lambda x: torch.tensor(np.asarray(x, np.float64))
  return dict(raw_density=t(rng.normal(size=(B, S)) * 2), raw_rgb=t(rng.normal(size=(B, S, 3))), sdist=t(sd),
              directions=t(d), near=t(np.full(B, 0.5)), far=t(np.full(B, 20.0)), target=t(rng.uniform(0, 1, (B, 3))),
              lossmult=t(rng.uniform(0.5, 2, (B, lm_ch))), sdist_fine=t(sf), weights_fine=t(wf / wf.sum(-1, keepdims=True)),
              _rng=rng)


CASES = {
    'plain': {},
    'opaque': dict(cfg=dict(opaque_background=True)),
    'density_noise': dict(cfg=dict(density_noise=0.7), inp=['density_noise']),
    'bg_rgb': dict(inp=['bg_rgb']),
    'rgb_scale': dict(inp=['rgb_scale']),
    'extra_dw': dict(inp=['extra_dw']),
    'data_mask': dict(inp=['data_mask']),
    'tint': dict(cfg=dict(rgb_mode=1), inp=['raw_diffuse', 'raw_tint']),
    'no_tint': dict(cfg=dict(rgb_mode=1), inp=['raw_diffuse']),
    'safe_exp': dict(cfg=dict(rgb_activation='safe_exp', rgb_bias=-1.0, rgb_padding=0.0, raydist_fn='log')),
    'charb_lm3': dict(loss=dict(loss_type='charb'), lm_ch=3),
    'rawnerf': dict(loss=dict(loss_type='rawnerf', data_mult=0.5)),
    'distortion': dict(loss=dict(distortion_mult=0.01)),
    'interlevel': dict(loss=dict(interlevel_mult=1.0), no_rgb=True),
}


def _case(name):
  spec = CASES[name]
  inp = _inputs(sorted(CASES).index(name), lm_ch=spec.get('lm_ch', 1))
  rng = inp.pop('_rng')
  B, S = inp['raw_density'].shape
  t = lambda x: torch.tensor(np.asarray(x, np.float64))
  extra = dict(density_noise=t(rng.normal(size=(B, S))), bg_rgb=t(rng.uniform(0, 1, (B, 3))),
               # one zero and one negative exposure channel: d pixel / d scale is sum_s w_s c_s there too
               rgb_scale=t([[0.0, 1.5, 0.7], [-0.8, 2.0, 1.0], [1.2, 0.3, 0.9]]),
               extra_dw=t(rng.normal(size=(B, S)) * 0.1), data_mask=t([1.0, 0.0, 1.0]),
               raw_diffuse=t(rng.normal(size=(B, S, 3))), raw_tint=t(rng.normal(size=(B, S, 3))))
  for k in spec.get('inp', []):
    inp[k] = extra[k]
  if spec.get('no_rgb'):
    inp['raw_rgb'] = None
  cfg = dict(CFG, **spec.get('cfg', {}))
  loss = dict(LOSS, **spec.get('loss', {}))
  loss['inv_denom'] = 1.0 / float(inp['lossmult'].expand(B, 3).sum())
  return inp, cfg, loss


@pytest.mark.parametrize('name', sorted(CASES))
def test_reference_gradcheck(name):
  inp, cfg, loss = _case(name)
  names = [k for k in R.LEAVES if inp.get(k) is not None]

  def fn(*leaves):
    out = R.composite(dict(inp, **dict(zip(names, leaves))), cfg, loss)
    if loss['loss_type'] == 'rawnerf':
      # the RawNeRF loss weights each residual by a detached 1 / (1e-3 + clip): its gradient is by design not the
      # derivative of its value, so only the pixel and weights are checked here; the loss and its gradient are
      # compared with the oracle's compute_data_loss below
      return out['rgb'], out['weights']
    return out['loss'], out['rgb'], out['weights']
  leaves = tuple(inp[k].clone().requires_grad_(True) for k in names)
  assert torch.autograd.gradcheck(fn, leaves, eps=1e-6, atol=1e-8, rtol=1e-6)


def test_reference_rgb_scale_gradient_at_zero():
  """At a zero exposure channel the scale's gradient is d loss / d pixel * sum_s w_s c_s, not zero."""
  inp, cfg, loss = _case('rgb_scale')
  out, g = R.grads(inp, cfg, loss)
  c = R.colour(inp['raw_rgb'], cfg)
  wc = (out['weights'][..., None] * c).sum(-2)
  dpix = 2 * (out['rgb'] - inp['target']) * inp['lossmult'] * loss['inv_denom']
  torch.testing.assert_close(g['rgb_scale'], dpix * wc, rtol=1e-12, atol=1e-15)
  assert float(g['rgb_scale'][0, 0].abs()) > 1e-3


@pytest.mark.parametrize('loss_type,lm_ch', [('mse', 1), ('charb', 3), ('rawnerf', 3)])
def test_reference_matches_oracle_loss(loss_type, lm_ch):
  """The pixel, the data loss and its gradient are the oracle's volumetric_rendering and compute_data_loss (no
  mask)."""
  inp, cfg, loss = _case('bg_rgb')
  B = inp['raw_density'].shape[0]
  inp['lossmult'] = torch.rand(B, lm_ch, dtype=torch.float64, generator=torch.Generator().manual_seed(lm_ch)) + 0.5
  loss = dict(loss, loss_type=loss_type, inv_denom=1.0 / float(inp['lossmult'].expand(B, 3).sum()))
  out, g = R.grads(inp, cfg, loss)
  r = o_render.volumetric_rendering(out['rgb_samples'], out['weights'], out['t_aug'][:, :-1], inp['bg_rgb'],
                                    inp['far'][:, None], False)
  torch.testing.assert_close(out['rgb'], r['rgb'], rtol=1e-14, atol=1e-15)
  cfg_o = type('C', (), dict(data_loss_type=loss_type, charb_padding=R.f32(0.001), disable_multiscale_loss=False,
                             data_coarse_loss_mult=0.0, data_loss_mult=1.0))
  data, st = o_train.compute_data_loss(inp['target'], [dict(rgb=out['rgb'])], inp['lossmult'], cfg_o)
  torch.testing.assert_close(out['data'], data, rtol=1e-13, atol=0)
  torch.testing.assert_close(out['mse'], st['mses'][0], rtol=1e-13, atol=0)
  # gradient of the oracle's data loss through the same pixel
  leaves = {k: inp[k].detach().requires_grad_(True) for k in ('raw_density', 'raw_rgb')}
  rgb = R.composite(dict(inp, **leaves), cfg)['rgb']
  data_o, _ = o_train.compute_data_loss(inp['target'], [dict(rgb=rgb)], inp['lossmult'], cfg_o)
  g_o = torch.autograd.grad(data_o, list(leaves.values()))
  for k, go in zip(leaves, g_o):
    torch.testing.assert_close(g[k], go, rtol=1e-12, atol=1e-15)


def test_reference_bg_on_pins_the_branch():
  """`bg_on` chooses the background weight's branch whatever acc is (a saturated translucent ray has acc == 1 in
  fp32 and slightly less in fp64)."""
  inp, cfg, loss = _case('plain')
  B = inp['raw_density'].shape[0]
  _, g_on = R.grads(inp, cfg, loss, bg_on=torch.ones(B, dtype=torch.bool))
  _, g_off = R.grads(inp, cfg, loss, bg_on=torch.zeros(B, dtype=torch.bool))
  # with the background on, each weight's gradient loses dpx . bg: the two differ
  assert float((g_on['raw_density'] - g_off['raw_density']).abs().max()) > 1e-6


# ---- the emulation ---------------------------------------------------------------------------------------------------

class Emul:
  """The walk's backend of the emulation: numpy fp32 in the kernels' lane layout, library calls moved by dirn."""

  def __init__(self, dirn, seed=0, mut=None):
    self.dirn, self.mut = dirn, mut
    self.rng = np.random.default_rng(seed)

  def inp(self, x):
    return np.asarray(x.detach().cpu().numpy() if torch.is_tensor(x) else x, F)

  def c(self, v):
    return F(v)

  def k(self, kv):
    return F(kv[0])

  def val(self, x):
    return torch.from_numpy(np.asarray(x, np.float64).copy())

  def err(self, x):
    return torch.zeros(np.shape(x), dtype=torch.float64)

  def zeros(self, shape):
    return np.zeros(shape, F)

  def _lib(self, name, v64):
    """The library's result moved by almost its documented error; an exact result (expf(0) = 1, logf(1) = 0) stays."""
    with np.errstate(all='ignore'):
      v64 = np.asarray(v64, np.float64)
      moved = (v64 * (1 + self.dirn * (2 * R.LIB_ULP[name] - 1) * R.U)).astype(F)
      return np.where(v64.astype(F).astype(np.float64) == v64, v64.astype(F), moved).astype(F)

  def exp(self, x):
    with np.errstate(all='ignore'):
      return self._lib('exp', np.exp(np.asarray(x, np.float64)))

  def log(self, x):
    with np.errstate(all='ignore'):
      return self._lib('log', np.log(np.asarray(x, np.float64)))

  def log1p(self, x):
    return self._lib('log1p', np.log1p(np.asarray(x, np.float64)))

  def pow(self, x, p):
    with np.errstate(all='ignore'):
      return self._lib('pow', np.asarray(x, np.float64) ** np.float64(F(p[0])))

  def sqrt(self, x):
    return np.sqrt(np.asarray(x, F))

  def sigmoid(self, x):
    with np.errstate(all='ignore'):
      return F(1) / (F(1) + self.exp(-np.asarray(x, F)))

  def maxe(self, x, y):
    return np.maximum(x, y)

  def mine(self, x, y):
    return np.minimum(x, y)

  def fmax(self, x, c):
    return np.maximum(np.asarray(x, F), F(c))

  def fmin(self, x, c):
    return np.minimum(np.asarray(x, F), F(c))

  def where(self, cond, a, b):
    cond = cond.cpu().numpy() if torch.is_tensor(cond) else cond
    return np.where(cond, a, b).astype(F)

  def stack(self, xs, dim=-1):
    return np.stack(np.broadcast_arrays(*[np.asarray(x, F) for x in xs]), dim)

  def col(self, x):
    return np.asarray(x, F)[..., None]

  # ---- the kernels' lane layout
  @staticmethod
  def _lanes(x, CH):
    x = np.asarray(x, F)
    B, S = x.shape
    p = np.zeros((B, 32 * CH), F)
    p[:, :S] = x
    return p.reshape(B, 32, CH)

  @staticmethod
  def _local(xl):
    loc = np.zeros(xl.shape[:2], F)
    for j in range(xl.shape[2]):
      loc = loc + xl[:, :, j]
    return loc

  @staticmethod
  def _butterfly(v):
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
      v = v + v[:, lane ^ o]
    return v[:, 0]

  @staticmethod
  def _scan_incl(v):
    lane = np.arange(32)
    for o in (1, 2, 4, 8, 16):
      n = np.zeros_like(v)
      n[:, o:] = v[:, :-o]
      v = np.where(lane >= o, v + n, v).astype(F)
    return v

  def wsum(self, x, CH):
    return self._butterfly(self._local(self._lanes(x, CH)))

  def scan(self, x, CH):
    B, S = np.shape(x)
    xl = self._lanes(x, CH)
    incl = self._scan_incl(self._local(xl))
    run = np.zeros_like(incl)
    run[:, 1:] = incl[:, :-1]
    ex, inc = np.zeros_like(xl), np.zeros_like(xl)
    for j in range(CH):
      ex[:, :, j] = run
      run = run + xl[:, :, j]
      inc[:, :, j] = run
    return ex.reshape(B, -1)[:, :S], inc.reshape(B, -1)[:, :S], incl[:, 31]

  def after(self, gw, CH, mut=None):
    B, S = np.shape(gw)
    xl = self._lanes(gw, CH)
    lgw = self._local(xl)
    v = lgw.copy()
    lane = np.arange(32)
    last = 31 if mut == 'after_no_lane31' else 32
    for o in (1, 2, 4, 8, 16):
      n = np.zeros_like(v)
      n[:, :-o] = v[:, o:]
      v = np.where(lane + o < last, v + n, v).astype(F)
    aft = v - lgw
    out = np.zeros_like(xl)
    for j in range(CH - 1, -1, -1):
      out[:, :, j] = aft
      if mut != 'after_no_own':
        aft = aft + xl[:, :, j]
    return out.reshape(B, -1)[:, :S]

  def fine_sum(self, x, Sf):
    x = np.asarray(x, F)
    B = x.shape[0]
    lanes = np.zeros((B, 32), F)
    for i in range(Sf):
      lanes[:, i % 32] = lanes[:, i % 32] + x[:, i]
    return self._butterfly(lanes)

  def scatter_D(self, gi, lo, hi, live, S, rng=None):
    gi = np.asarray(gi, F)
    lo, hi, live = lo.cpu().numpy(), hi.cpu().numpy(), live.cpu().numpy()
    B, Sf = gi.shape
    D = np.zeros((B, S + 2), F)
    rows = np.arange(B)
    for i in self.rng.permutation(Sf):
      g = np.where(live[:, i], gi[:, i], F(0))
      D[rows, lo[:, i]] = D[rows, lo[:, i]] + g
      D[rows, hi[:, i]] = D[rows, hi[:, i]] + (-g)
    return D

  def gather(self, x, idx):
    return np.take_along_axis(np.asarray(x, F), idx.cpu().numpy(), 1)


def emul_stats(b, o, B, num_sms=SMS, start=None):
  """stats[0:4] as the kernel accumulates them: each warp's rays in grid-stride order (fp32, per ray the data and mse
  partials channel by channel), then one atomicAdd per warp in a shuffled order."""
  blocks = min(-(-B // 4), num_sms * 16)
  nw = blocks * 4
  out = np.zeros(4, F) if start is None else np.asarray(start, F).copy()
  terms = [np.asarray(o.st_data, F), np.asarray(o.st_mse, F), np.asarray(o.st_dist, F), np.asarray(o.st_inter, F)]
  for k, t in enumerate(terms):
    t = t.reshape(B, -1)
    part = np.zeros(nw, F)
    for it in range(-(-B // nw)):
      r = np.arange(it * nw, min((it + 1) * nw, B))
      for c in range(t.shape[1]):
        part[r - it * nw] = part[r - it * nw] + t[r, c]
    for w in b.rng.permutation(nw):
      if part[w] != 0:
        out[k] = out[k] + part[w]
  return out


def emulate(inp, cfg, loss, dirn, seed, mut=None, batch_rays=None):
  b = Emul(dirn, seed, mut)
  x = dict(inp)
  o = R.walk(b, x, cfg, loss, None, batch_rays, mut)
  o.percentiles = _emul_percentiles(o, x)
  o.stats = emul_stats(b, o, inp['raw_density'].shape[0])
  return o


def _emul_percentiles(o, x):
  """The kernel's binary search over cw = [0, cws, 1] and its interpolation, in fp32."""
  cws, tds = np.asarray(o.cws, F), np.asarray(o.tdist, F)
  far = x['far'].numpy().astype(F)
  B, S = cws.shape
  cw = np.concatenate([np.zeros((B, 1), F), cws, np.ones((B, 1), F)], -1)
  tt = np.concatenate([tds, far[:, None]], -1)
  n = S + 2
  out = np.zeros((B, 3), F)
  for k, p in enumerate((F(0.05), F(0.5), F(0.95))):
    lo = (cw <= p).sum(-1)                    # cw is sorted: the binary search's count
    i1 = np.clip(lo, 1, n - 1)
    i0 = i1 - 1
    r = np.arange(B)
    x0, x1, f0, f1 = cw[r, i0], cw[r, i1], tt[r, i0], tt[r, i1]
    dxp = x1 - x0
    with np.errstate(all='ignore'):
      v = np.where(dxp == 0, f0, f0 + (f1 - f0) / dxp * (p - x0))
    out[:, k] = v
  return out


def _compare(o, res, inp, cfg, mut=None):
  """Worst err / bound of the emulation over every checked output; raises AssertionError where one is off."""
  t = lambda v: torch.from_numpy(np.asarray(v, np.float64).copy())
  worst = 0.0
  pairs = [('weights', o.w), ('density', o.dens), ('rgb_samples', o.c), ('rgb', o.rgb), ('acc', o.acc),
           ('distance_mean', o.distance_mean), ('d_raw_density', o.d_raw_density)]
  for k in ('d_raw_rgb', 'd_rgb_scale', 'd_raw_diffuse', 'd_raw_tint'):
    if k in res:
      pairs.append((k, getattr(o, k)))
  for name, v in pairs:
    if name == 'rgb_samples' and 'raw_rgb' not in inp:
      continue
    _, w = R.check(name, t(v), *res[name])
    worst = max(worst, w)
  R.check_percentiles('percentiles', t(o.percentiles), res)
  sv, sb, _ = res['stats']
  got = t(o.stats)
  bad = ((got - sv).abs() > sb) | ~torch.isfinite(got)
  assert not bad.any(), f'stats {got.tolist()} vs {sv.tolist()} bound {sb.tolist()}'
  return worst


def _dec(o):
  """The decisions the reference follows, from the emulation's own (correct) acc and pixel."""
  acc = torch.from_numpy(np.asarray(o.acc, F).copy())
  return dict(bg_on=(1.0 - acc) > 0, v_lt1=torch.from_numpy(np.asarray(o.rgb, F).copy()) < 1)


_REF = {}


def _case_ref(i):
  if i not in _REF:
    inp, cfg, loss = make(GPU_CASES[i], seed=i, num_sms=SMS)
    o0 = emulate(inp, cfg, loss, 0, i)
    res = R.reference(inp, cfg, loss, _dec(o0))
    _REF.clear()
    _REF[i] = (inp, cfg, loss, o0, res)
  return _REF[i]


@pytest.mark.parametrize('i', range(len(GPU_CASES)), ids=[case_id(c) for c in GPU_CASES])
def test_emulation_inside_every_bound(i):
  inp, cfg, loss, o0, res = _case_ref(i)
  assert res['chain_gap'] < 1e-2, res['chain_gap']
  worst = _compare(o0, res, inp, cfg)
  d0 = _dec(o0)
  for dirn in (1, -1):
    oe = emulate(inp, cfg, loss, dirn, 2 * i + (dirn > 0))
    de = _dec(oe)
    # the reference follows the decisions this run of the kernel exposes (its acc and pixel), as on the GPU
    same = all(torch.equal(de[k], d0[k]) for k in d0)
    worst = max(worst, _compare(oe, res if same else R.reference(inp, cfg, loss, de), inp, cfg))
  print(f'{case_id(GPU_CASES[i])}: worst err/bound {worst:.3f}')


def _caught(mut, idxs):
  for i in idxs:
    inp, cfg, loss, o0, res = _case_ref(i)
    try:
      _compare(emulate(inp, cfg, loss, 0, i, mut=mut), res, inp, cfg, mut)
    except AssertionError:
      return True
  return False


def _cases_where(pred, n=12):
  return [i for i, c in enumerate(GPU_CASES) if pred(*c) and c[1] != -1][:n]


MUTANT_CASES = {
    'inclusive_T': lambda S, B, *r: B >= 5,
    'after_no_lane31': lambda S, B, lvl, *r: S > 33 and B >= 5,
    'after_no_own': lambda S, B, lvl, *r: S > 33 and B >= 5,
    'no_inf_ragged': lambda S, B, lvl, lt, lm, rd, act, opaque, *r: opaque and S % R.ch_of(S) and S > 32,
    'bg_on_tie': lambda S, B, lvl, lt, lm, rd, act, opaque, *r: opaque and B >= 5,
    'dist_tdist': lambda S, B, lvl, *r: lvl == 'fine' and B >= 5,
    'dist_two_thirds': lambda S, B, lvl, *r: lvl == 'fine' and B >= 5,
    'inter_off_by_one': lambda S, B, lvl, *r: lvl == 'prop' and B >= 5,
    'inter_wrong_sf': lambda S, B, lvl, *r: lvl == 'prop' and B >= 5,
    'invB_num_rays': None,
    'mse_masked': lambda S, B, lvl, lt, lm, rd, act, opaque, opts, *r: 'm' in opts and B >= 5,
    'lossmult_ray': lambda S, B, lvl, lt, lm, *r: lm == 3 and B >= 5,
    'zero_scale_divides': lambda S, B, lvl, lt, lm, rd, act, opaque, opts, *r: 's' in opts and B >= 5,
    'clip_passes': lambda S, B, lvl, lt, lm, rd, act, opaque, opts, *r: ('r' in opts or 'R' in opts) and B >= 5,
    'tint_no_tt': lambda S, B, lvl, lt, lm, rd, act, opaque, opts, *r: 'r' in opts and B >= 5,
    'pad_twice': lambda S, B, lvl, lt, lm, rd, act, *r: lvl == 'fine' and act == 'sigmoid' and B >= 5,
}


@pytest.mark.parametrize('mut', R.MUTANTS)
def test_mutant_is_caught(mut):
  if mut == 'invB_num_rays':
    # one pass of a two-pass batch: the distortion and interlevel means divide by the whole batch
    for i in _cases_where(lambda S, B, *r: B >= 5)[:6]:
      inp, cfg, loss = make(GPU_CASES[i], seed=i)
      B = inp['raw_density'].shape[0]
      o0 = emulate(inp, cfg, loss, 0, i, batch_rays=2 * B)
      res = R.reference(inp, cfg, loss, _dec(o0), batch_rays=2 * B)
      _compare(o0, res, inp, cfg)
      try:
        _compare(emulate(inp, cfg, loss, 0, i, mut=mut, batch_rays=2 * B), res, inp, cfg)
      except AssertionError:
        return
    pytest.fail(f'{mut} not caught')
  # a tie of the background weight (acc exactly 1 in fp32) is rare: that one searches every case
  n = 1000 if mut == 'bg_on_tie' else 12
  assert _caught(mut, _cases_where(MUTANT_CASES[mut], n)), f'{mut} not caught'


def _stand_in(i):
  """The fp32 oracle (composite_ref.grads in float32) for the kernel, and the fp64 reference of case i."""
  inp, cfg, loss, o0, res = _case_ref(i)
  in32 = {k: v for k, v in inp.items() if k != 'inv_denom'}
  lref = dict(loss, inv_denom=float(inp['inv_denom'][0]))
  _, g32 = R.grads(in32, cfg, lref, bg_on=_dec(o0)['bg_on'])
  return res, g32


@pytest.mark.parametrize('smin,smax', [(100, 256), (65, 128)])
def test_mutants_of_the_old_check_fail(smin, smax):
  """The two mutants the per-ray check let through now fail the per-element check: d_raw_density zeroed where it is
  below 1e-5 of its ray's largest, and d_raw_rgb tripled where the weight is below 1e-6."""
  i = next(j for j, c in enumerate(GPU_CASES) if smin <= c[0] <= smax and c[2] == 'fine' and c[1] >= 5)
  res, g32 = _stand_in(i)
  ref, bd, ex = res['d_raw_density']
  small = ref.abs() < 1e-5 * ref.abs().amax(1, keepdim=True)
  assert small.any()
  with pytest.raises(AssertionError):
    R.check('d_raw_density', torch.where(small, torch.zeros_like(ref), ref), ref, bd, ex)
  ref, bd, ex = res['d_raw_rgb']
  tiny = (res['weights'][0] < 1e-6)[..., None].expand_as(ref)
  assert tiny.any()
  with pytest.raises(AssertionError):
    R.check('d_raw_rgb', torch.where(tiny, 3 * ref, ref), ref, bd, ex)


def test_walk_agrees_with_autograd():
  """The Running walk's values are the fp64 autograd reference's to fp64 rounding on every kind of case."""
  for i in _cases_where(lambda S, B, *r: B >= 5)[:8]:
    _, _, _, _, res = _case_ref(i)
    assert res['chain_gap'] < 1e-2, (case_id(GPU_CASES[i]), res['chain_gap'])


def test_fp32_reference_is_the_oracle_chain():
  """In float32 `composite` is the oracle's compositing chain."""
  inp, cfg, loss = _case('bg_rgb')
  in32 = {k: v.float() if torch.is_tensor(v) else v for k, v in inp.items()}
  cfg = dict(cfg, bg_const=1.0)
  out = R.composite({k: v for k, v in in32.items() if k != 'bg_rgb'}, cfg)
  w, r, dens, rgb = R.oracle_composite(in32['raw_density'], in32['raw_rgb'], in32['sdist'], in32['directions'],
                                       in32['near'][:, None], in32['far'][:, None], cfg)
  assert torch.equal(out['weights'], w) and torch.equal(out['density'], dens)
  torch.testing.assert_close(out['rgb'], r['rgb'], rtol=0, atol=2e-7)


# ---- refusals ---------------------------------------------------------------------------------------------------------

FAKE = 1 << 20            # a non-null address that is never dereferenced: every call below returns before a launch


def _lib():
  if torch.cuda.is_available():
    pytest.skip('refusals run only where no check can launch a kernel')
  from multinerf_b200 import lib as L
  try:
    return L, L.load()
  except L.MnrfError as e:
    pytest.skip(f'library not built: {e}')


REFUSALS = [
    # (entry, descriptor overrides, argument overrides, message)
    ('both', dict(rgb_mode=2), {}, 'unknown rgb_mode 2'),
    ('both', dict(rgb_mode=-1), {}, 'unknown rgb_mode'),
    ('both', dict(rgb_act=2), {}, 'unknown rgb_act'),
    ('both', dict(raydist_fn=7), {}, 'unknown raydist_fn'),
    ('both', dict(raydist_fn=-1), {}, 'unknown raydist_fn'),
    ('both', dict(num_rays=-1), {}, 'negative num_rays'),
    ('both', dict(ld_density=-4), {}, 'negative ld_density'),
    ('both', dict(ld_rgb=1), {}, 'ld_rgb 1'),
    ('both', dict(ld_rgb=2), {}, 'ld_rgb 2'),
    ('both', dict(ld_rgb=-3), {}, 'ld_rgb -3'),
    ('both', dict(num_samples=257), {}, 'num_samples 257'),
    ('both', dict(num_samples=0), {}, 'num_samples 0'),
    ('both', {}, dict(desc=None), 'null descriptor'),
    ('fwd', dict(rgb_mode=1), dict(raw_diffuse=None), 'rgb_mode 1 needs'),
    ('bwd', dict(rgb_mode=1), dict(d_raw_rgb=None), 'rgb_mode 1 needs'),
    ('bwd', dict(rgb_mode=1), dict(d_raw_diffuse=None), 'rgb_mode 1 needs'),
    ('bwd', dict(rgb_mode=1), dict(d_raw_tint=None), 'rgb_mode 1 needs'),
    ('bwd', {}, dict(interlevel_mult=1.0, num_samples_fine=0), 'interlevel loss needs'),
    ('bwd', {}, dict(interlevel_mult=1.0, weights_fine=None), 'interlevel loss needs'),
    ('bwd', {}, dict(lossmult_channels=2), 'lossmult_channels'),
    ('bwd', {}, dict(loss_type=3), 'unknown data_loss_type'),
    ('bwd', {}, dict(batch_rays=7), 'batch_rays 7 < num_rays 8'),
    ('bwd', {}, dict(stats=None), 'null pointer'),
]


def call(L, lib, entry, dk, ak, real=None):
  """One call of `entry` with a valid descriptor for 8 rays of 33 samples in rgb_mode 0 / 1 (as dk says), with dk and
  ak applied.  real: (an input address, {output name: address}) to pass real buffers instead of FAKE.  Returns
  (return code, last error)."""
  inp = real[0] if real else FAKE
  outs = real[1] if real else {}
  o = lambda k: outs.get(k, FAKE)
  d = dict(num_rays=8, num_samples=33, raydist_fn=1, opaque_background=0, density_bias=-1.0, density_noise=0.0,
           rgb_act=0, rgb_premult=1.0, rgb_bias=0.0, rgb_padding=0.001, bg_const=1.0, rgb_mode=0, ld_density=0,
           ld_rgb=0)
  d.update(dk)
  cd = L.CompositeDesc(*[d[k] for k, _ in L.CompositeDesc._fields_])
  a = dict(desc=True, raw_diffuse=inp, raw_tint=inp, d_raw_rgb=o('drgb'), d_raw_diffuse=o('ddf'), d_raw_tint=o('dti'),
           interlevel_mult=0.0, num_samples_fine=17, weights_fine=inp, lossmult_channels=1, loss_type=0, batch_rays=8,
           stats=o('acc'))
  a.update(ak)
  if entry == 'fwd':
    rc = lib.mnrf_composite_fwd(C.byref(cd) if a['desc'] else None, inp, inp, None, inp, inp, inp, inp, None, None,
                                a['raw_diffuse'], a['raw_tint'], o('w'), o('rgb'), o('dens'), o('rgbs'), o('acc'),
                                o('dist'), None)
  else:
    ld = L.LossDesc(cd, a['loss_type'], 0.001, 1.0, 0.0, a['interlevel_mult'], a['num_samples_fine'],
                    a['lossmult_channels'])
    rc = lib.mnrf_composite_bwd(C.byref(ld) if a['desc'] else None, inp, inp, None, inp, inp, inp, inp, None, None,
                                a['raw_diffuse'], a['raw_tint'], None, inp, inp, inp, inp, a['weights_fine'], None,
                                o('drd'), a['d_raw_rgb'], None, a['d_raw_diffuse'], a['d_raw_tint'], a['stats'],
                                a['batch_rays'], None)
  return rc, lib.mnrf_last_error().decode()


@pytest.mark.parametrize('i', range(len(REFUSALS)))
def test_composite_refusals(i):
  L, lib = _lib()
  entry, dk, ak, msg = REFUSALS[i]
  for e in (('fwd', 'bwd') if entry == 'both' else (entry,)):
    rc, err = call(L, lib, e, dk, ak)
    assert rc != 0 and msg in err, (e, dk, ak, rc, err)


def test_composite_accepts_what_it_should():
  """The checks are no stricter than the kernels: valid descriptors get past every one of them (and then fail only
  for want of a device)."""
  L, lib = _lib()
  for dk in (dict(), dict(rgb_mode=1), dict(ld_density=4, ld_rgb=4), dict(ld_density=8, ld_rgb=8), dict(ld_rgb=3),
             dict(raydist_fn=0, rgb_act=1), dict(raydist_fn=6, num_samples=256), dict(num_samples=1)):
    for e in ('fwd', 'bwd'):
      rc, err = call(L, lib, e, dk, {})
      assert not any(m in err for m in ('unknown', 'negative', 'overlaps', 'needs', 'null', 'num_samples')), \
          (e, dk, err)
  # an empty batch returns before touching anything
  for e in ('fwd', 'bwd'):
    rc, err = call(L, lib, e, dict(num_rays=0), {})
    assert rc == 0, (e, err)
