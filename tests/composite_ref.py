"""Reference of the compositing kernels (csrc/composite.cu) in any float dtype, built from the oracle.

`composite` assembles the oracle's colour activations, o_render.compute_alpha_weights / volumetric_rendering
and the o_train losses the way mnrf_composite_fwd and mnrf_composite_bwd combine them for one level, with every
optional input the kernels take.  Evaluated in float64 on the kernels' fp32 inputs and differentiated by
torch.autograd it gives the values of tests/test_gpu_composite_fp64.py; `walk` (below) gives the bound of every
element.  Pure torch: runs on the CPU or on CUDA tensors, and never loads the CUDA library.
"""
import math
import types

import numpy as np
import torch

from oracle import o_coord, o_math, o_render, o_stepfun, o_train

# leaves the kernels differentiate, in the order of `grads`' result
LEAVES = ('raw_density', 'raw_rgb', 'rgb_scale', 'raw_diffuse', 'raw_tint')


def f32(x):
  """A descriptor scalar as the kernel sees it (the descriptors hold fp32)."""
  return float(np.float32(x))


def _act(raw_rgb, cfg):
  z = f32(cfg['rgb_premultiplier']) * raw_rgb + f32(cfg['rgb_bias'])
  return torch.sigmoid(z) if cfg['rgb_activation'] == 'sigmoid' else o_math.safe_exp(z)


def _linear(raw_rgb, cfg, raw_diffuse, raw_tint):
  """rgb_mode 1: tinted specular + diffuse, in linear space."""
  t = torch.sigmoid(raw_tint) if raw_tint is not None else 0.5
  return t * _act(raw_rgb, cfg) + torch.sigmoid(raw_diffuse - math.log(3.0))


def srgb_branches(raw_rgb, cfg, raw_diffuse, raw_tint):
  """rgb_mode 1: the branches this dtype's arithmetic takes -- the linear piece of linear_to_srgb, and the sRGB
  value strictly inside (0, 1), where the kernel passes the gradient (torch.clamp passes it at the bounds too)."""
  with torch.no_grad():
    lin = _linear(raw_rgb, cfg, raw_diffuse, raw_tint)
    sr = o_math.linear_to_srgb(lin)
  return dict(linear=lin <= 0.0031308, inside=(sr > 0) & (sr < 1))


def colour(raw_rgb, cfg, raw_diffuse=None, raw_tint=None, branches=None):
  """Per-sample colour before the exposure scale (models.py rgb head; rgb_mode 1 = Ref-NeRF diffuse + tinted
  specular, with a constant tint of 0.5 when the model has no tint head).  `branches` (of srgb_branches): take
  these branches of linear_to_srgb and of the clip to [0, 1] instead of this dtype's own."""
  if cfg.get('rgb_mode', 0) == 1:
    lin = _linear(raw_rgb, cfg, raw_diffuse, raw_tint)
    if branches is None:
      a = torch.clamp(o_math.linear_to_srgb(lin), 0.0, 1.0)
    else:
      sr = torch.where(branches['linear'], 323.0 / 25.0 * lin,
                       (211.0 * torch.clamp(lin, min=o_math.EPS) ** (5.0 / 12.0) - 11.0) / 200.0)
      a = torch.where(branches['inside'], sr, torch.clamp(sr, 0.0, 1.0).detach())
  else:
    a = _act(raw_rgb, cfg)
  pad = f32(cfg['rgb_padding'])
  return a * (1 + 2 * pad) - pad


def composite(inp, cfg, loss=None, bg_on=None, pixel_shift=None, branches=None):
  """One level's forward outputs and, with `loss`, its loss terms.

  inp: dict of tensors of one dtype -- raw_density [B,S], sdist [B,S+1], directions [B,3], near [B], far [B], and
    optionally raw_rgb [B,S,3], density_noise [B,S], bg_rgb [B,3], rgb_scale [B,3], raw_diffuse / raw_tint [B,S,3],
    extra_dw [B,S]; with `loss` also target [B,3], lossmult [B,1|3], data_mask [B] (optional), sdist_fine
    [B,Sf+1] and weights_fine [B,Sf] (interlevel).
  cfg: the kwargs of ops._cdesc.
  loss: dict(loss_type, charb_padding, data_mult, distortion_mult, interlevel_mult, inv_denom).
  bg_on: optional bool [B]: whether the background weight max(0, 1 - acc) is on its linear branch.  The kernel
    decides this from its fp32 acc and gives the weight zero gradient on a tie (1 - acc == 0, where
    torch.clamp would pass the gradient); passing the kernel's decision makes this reference follow it.
  pixel_shift: optional constant [B,3] added to the pixel before the losses (how far an fp32 rounding of the pixel
    alone moves the gradients).
  branches: rgb_mode 1: the sRGB branches to take (see `colour`).
  """
  raw = inp['raw_density']
  B, S = raw.shape
  dt = raw.dtype
  near, far = inp['near'][:, None], inp['far'][:, None]
  _, s_to_t = o_coord.construct_ray_warps(cfg['raydist_fn'], near, far)
  tdist = s_to_t(inp['sdist'])
  if inp.get('density_noise') is not None:
    raw = raw + f32(cfg['density_noise']) * inp['density_noise']
  density = torch.nn.functional.softplus(raw + f32(cfg['density_bias']))
  w, alpha, trans = o_render.compute_alpha_weights(density, tdist, inp['directions'],
                                                   opaque_background=cfg['opaque_background'])
  if inp.get('raw_rgb') is None:
    c = torch.zeros(B, S, 3, dtype=dt, device=raw.device)
  else:
    c = colour(inp['raw_rgb'], cfg, inp.get('raw_diffuse'), inp.get('raw_tint'), branches)
    if inp.get('rgb_scale') is not None:
      c = c * inp['rgb_scale'][:, None, :]
  bg = inp['bg_rgb'] if inp.get('bg_rgb') is not None else f32(cfg['bg_const'])
  # volumetric_rendering supplies acc, distance_mean and the percentiles; the pixel is its expression with the
  # background weight written out so that `bg_on` can pin its branch.
  r = o_render.volumetric_rendering(c, w, tdist, bg, far, True)
  acc = w.sum(dim=-1)
  bg_w = torch.clamp(1 - acc, min=0.0) if bg_on is None else torch.where(bg_on, 1 - acc, torch.zeros_like(acc))
  rgb = (w[..., None] * c).sum(dim=-2) + bg_w[:, None] * bg
  t_aug = torch.cat([tdist, far], dim=-1)
  out = dict(weights=w, density=density, rgb_samples=c, rgb=rgb, acc=r['acc'], distance_mean=r['distance_mean'],
             percentiles=torch.stack([r['distance_percentile_5'], r['distance_median'],
                                      r['distance_percentile_95']], -1),
             t_aug=t_aug, cdf=o_stepfun.integrate_weights(torch.cat([w, bg_w[:, None]], dim=-1)),
             # transmittance after each sample, and d (density * delta) / d raw_density
             trans_after=(trans * (1 - alpha)).detach(),
             dtau_draw=(torch.sigmoid(raw + f32(cfg['density_bias'])) * (tdist[:, 1:] - tdist[:, :-1]) *
                        torch.linalg.norm(inp['directions'], dim=-1, keepdim=True)).detach())
  if loss is None:
    return out

  # data loss and mse of o_train.compute_data_loss for one level, with the kernels' precomputed
  # 1 / sum(lossmult) and the RobustNeRF mask (a constant weight on each ray's data loss, not on the mse)
  tgt = inp['target']
  lm = inp['lossmult'].expand(B, 3)
  if pixel_shift is not None:
    rgb = rgb + pixel_shift
  resid = rgb - tgt
  if loss['loss_type'] == 'mse':
    lv = resid ** 2
  elif loss['loss_type'] == 'charb':
    lv = torch.sqrt(resid ** 2 + f32(loss['charb_padding']) ** 2)
  else:
    # rawnerf: min(rgb, 1) written as a where so that a pixel at exactly 1 takes the clipped branch, as in the
    # kernel (torch.clamp would pass the gradient there)
    clip = torch.where(rgb < 1, rgb, torch.ones_like(rgb))
    lv = (clip - tgt) ** 2 * (1.0 / (1e-3 + clip.detach())) ** 2
  if inp.get('data_mask') is not None:
    lv = lv * inp['data_mask'][:, None]
  inv_denom = loss['inv_denom']
  out['data'] = f32(loss['data_mult']) * (lm * lv).sum() * inv_denom
  out['mse'] = (lm * resid ** 2).sum() * inv_denom
  zero = torch.zeros((), dtype=dt, device=raw.device)
  out['distortion'] = zero
  if loss['distortion_mult'] > 0:
    out['distortion'] = o_train.distortion_loss(
        [dict(sdist=inp['sdist'], weights=w)], types.SimpleNamespace(distortion_loss_mult=f32(loss['distortion_mult'])))
  out['interlevel'] = zero
  if loss['interlevel_mult'] > 0:
    out['interlevel'] = o_train.interlevel_loss(
        [dict(sdist=inp['sdist'], weights=w), dict(sdist=inp['sdist_fine'], weights=inp['weights_fine'])],
        types.SimpleNamespace(interlevel_loss_mult=f32(loss['interlevel_mult'])))
  # the orientation / predicted-normal losses reach the kernel as dL/dw (extra_dw)
  extra = (w * inp['extra_dw']).sum() if inp.get('extra_dw') is not None else zero
  out['loss'] = out['data'] + out['distortion'] + out['interlevel'] + extra
  return out


def grads(inp, cfg, loss, bg_on=None, pixel_shift=None, branches=None):
  """(outputs of `composite`, {leaf: d loss / d leaf}) for the leaves of LEAVES present in `inp`, and 'weights':
  d loss / d weights."""
  inp = dict(inp)
  names = [k for k in LEAVES if inp.get(k) is not None]
  for k in names:
    inp[k] = inp[k].detach().requires_grad_(True)
  out = composite(inp, cfg, loss, bg_on, pixel_shift, branches)
  g = torch.autograd.grad(out['loss'], [inp[k] for k in names] + [out['weights']])
  return out, dict(zip(names + ['weights'], g))


def cdf_at(t_aug, cdf, t):
  """Piecewise-linear CDF of each row (knots t_aug, values cdf) at t [B, k]: where a percentile sits in it."""
  out = torch.empty_like(t)
  for i in range(t.shape[1]):
    out[:, i] = o_math.interp(t[:, i:i + 1].contiguous(), t_aug, cdf)[:, 0]
  return out


# the plain compositing descriptor of the kernel-parity tests (a reciprocal-distance level with an opaque background)
CFG = dict(raydist_fn='reciprocal', opaque_background=True, density_bias=-1.0, density_noise=0.0,
           rgb_activation='sigmoid', rgb_premultiplier=1.0, rgb_bias=0.0, rgb_padding=0.001, bg_const=1.0)


def oracle_composite(raw_d, raw_rgb, sdist, d, near, far, cfg, extras=False):
  """The oracle's compositing of one level without the optional inputs: (weights, renderings, density, rgb)."""
  _, s_to_t = o_coord.construct_ray_warps(cfg['raydist_fn'], near, far)
  tdist = s_to_t(sdist)
  density = torch.nn.functional.softplus(raw_d + cfg['density_bias'])
  if raw_rgb is None:
    rgb = torch.zeros(raw_d.shape + (3,))
  else:
    z = cfg['rgb_premultiplier'] * raw_rgb + cfg['rgb_bias']
    act = torch.sigmoid(z) if cfg['rgb_activation'] == 'sigmoid' else o_math.safe_exp(z)
    rgb = act * (1 + 2 * cfg['rgb_padding']) - cfg['rgb_padding']
  w = o_render.compute_alpha_weights(density, tdist, d, opaque_background=cfg['opaque_background'])[0]
  r = o_render.volumetric_rendering(rgb, w, tdist, cfg['bg_const'], far, extras)
  return w, r, density, rgb


# ---------------------------------------------------------------------------------------------------------------------
# Running-error walk of csrc/composite.cu
#
# `walk` restates the kernels' order of operations once, against a backend: `Running` (refdir_ref.E: an fp64 value
# and a bound on the absolute error of the kernel's fp32 value) or the CPU tests' numpy fp32 emulation.  composite.cu
# is built with -fmad=false, so every product and sum rounds once, in source order (u = 2^-24 each, refdir_ref.E);
# only the library calls move: expf 2 ulp, logf and log1pf 1 ulp, powf heads_ref.POW_ULPS ulp, each after the
# inherited error through the function's own slope; sqrtf and division are correctly rounded.
#   sums     A warp's sum or scan passes each term through at most D additions whatever their association: lane-local
#            (CH - 1), five shuffle levels, and up to CH more in the per-sample run of a scan.  So a sum carries
#            D u sum (|term| + its bound) on top of its terms' errors (the kernel's term may be larger than the fp64
#            one: a term that cancels to 0 in fp64 can still absorb its neighbours in fp32), with D = CH + 5 for warp_sum and 2 CH + 5 for a prefix or
#            the reverse scan of `after` (whose subtraction of the lane's own partial charges that lane's terms too).
#   D        The interlevel loss scatters +-gi into D with shared-memory atomics in any order: a cell of n terms
#            carries n u sum |terms|.
#   stats    Each warp sums its rays, then one atomic per warp, in any order: n u sum |terms| for n terms.
#   branches The kernel's own decisions are followed where it exposes them (`dec`: bg_on from its acc, the RawNeRF
#            `v < 1` from its pixel).  Otherwise an element whose fp64 value lies within its bound of a branch point
#            is exempt: the sRGB linear piece (the whole ray, since the pixel moves) and the clip to [0, 1] (that
#            sample's colour gradients).
# Constants the kernel folds in fp32 (kLog3, 5/12, 1e-3, ...) carry their rounding as an error.
from encode_ref import SLACK, TINY, U  # noqa: E402
from heads_ref import POW_ULPS  # noqa: E402
from refdir_ref import ULP, E  # noqa: E402

K_EPS = float(np.finfo(np.float32).eps)
F32_MAX = float(np.finfo(np.float32).max)
LIB_ULP = dict(ULP, log=1, pow=POW_ULPS)
RAYDIST = (None, 'reciprocal', 'log', 'exp', 'sqrt', 'square', 'piecewise')
VACUOUS = 0.25
MUTANTS = ('inclusive_T', 'after_no_lane31', 'after_no_own', 'no_inf_ragged', 'bg_on_tie', 'dist_tdist',
           'dist_two_thirds', 'inter_off_by_one', 'inter_wrong_sf', 'invB_num_rays', 'mse_masked', 'lossmult_ray',
           'zero_scale_divides', 'clip_passes', 'tint_no_tt', 'pad_twice')
# Not listed: the percentile CDF without its clamp to 1.  Its knots above 1 lie past every p (at most 0.95) and past
# the final knot 1, so the binary search picks the same interval either way: no output can tell it apart.


def ch_of(S):
  """Samples per lane of the kernel instance for S samples."""
  return 1 if S <= 32 else 2 if S <= 64 else 4 if S <= 128 else 8


def k32(v):
  """A constant the kernel folds in fp32 arithmetic: (fp32 value, exact value)."""
  return float(np.float32(v)), v


class Running:
  """The walk's backend of the bounds: refdir_ref.E values, on `device`."""

  def __init__(self, device='cpu'):
    self.device = device
    self.dirn = 0

  def inp(self, x):
    return E(x.detach().to(self.device, torch.float64))

  def c(self, v):
    return E(torch.tensor(float(v), dtype=torch.float64, device=self.device))

  def k(self, kv):
    v32, v64 = kv
    return E(torch.tensor(v64, dtype=torch.float64, device=self.device),
             torch.tensor(abs(v32 - v64), dtype=torch.float64, device=self.device))

  def val(self, x):
    return E.of(x).val

  def err(self, x):
    return E.of(x).err

  def zeros(self, shape):
    return E(torch.zeros(shape, dtype=torch.float64, device=self.device))

  def _lib(self, name, v, e):
    return E(v, e + 2 * LIB_ULP[name] * U * (v.abs() + e) + TINY)

  def exp(self, x):
    v = torch.exp(x.val)
    e = torch.where(x.err > 0, v * torch.expm1(x.err.clamp(max=700)), torch.zeros_like(v))
    return self._lib('exp', v, e)

  def log(self, x):
    v = torch.log(x.val)
    low = x.val - x.err
    e = torch.where(low > 0, -torch.log1p(-x.err / x.val), torch.full_like(v, math.inf))
    return self._lib('log', v, torch.where(x.err > 0, e, torch.zeros_like(v)))

  def log1p(self, x):
    v = torch.log1p(x.val)
    low = 1 + x.val - x.err
    e = torch.where(low > 0, x.err / low.clamp(min=1e-300), torch.full_like(v, math.inf))
    return self._lib('log1p', v, e)

  def sqrt(self, x):
    v = torch.sqrt(x.val)
    e = torch.maximum(v - torch.sqrt((x.val - x.err).clamp(min=0)), torch.sqrt(x.val + x.err) - v)
    return E(v, e + U * (v + e))

  def pow(self, x, p):
    """powf(x, p) with p = (fp32 exponent, exact exponent), x > 0."""
    p32, p64 = p
    v = x.val ** p64
    lo = (x.val - x.err).clamp(min=1e-300)
    slope = abs(p64) * torch.maximum(lo ** (p64 - 1), (x.val + x.err) ** (p64 - 1))
    e = slope * x.err + v * torch.log(x.val).abs() * abs(p32 - p64)
    return self._lib('pow', v, e)

  def sigmoid(self, x):
    """1 / (1 + expf(-x)): the exp's relative error moves s by s (1 - s) of it; the add and the division round."""
    s = torch.sigmoid(x.val)
    rel = torch.expm1(x.err.clamp(max=700)) + 2 * ULP['exp'] * U * 1.01
    return E(s, s * (1 - s) * rel + 2.01 * U * s + TINY)

  def maxe(self, x, y):
    return E(torch.maximum(x.val, y.val), torch.maximum(x.err, y.err))

  def mine(self, x, y):
    return E(torch.minimum(x.val, y.val), torch.maximum(x.err, y.err))

  def fmax(self, x, c):
    """max(x, c): 1-Lipschitz, and exactly c where x's bound keeps it below c."""
    x = E.of(x)
    e = torch.where(x.val <= c, torch.minimum(x.err, (x.val + x.err - c).clamp(min=0)), x.err)
    return E(x.val.clamp(min=c), e)

  def fmin(self, x, c):
    x = E.of(x)
    return E(x.val.clamp(max=c), x.err)

  def where(self, cond, a, b):
    a, b = E.of(a), E.of(b)
    return E(torch.where(cond, a.val, b.val), torch.where(cond, a.err, b.err))

  def stack(self, xs, dim=-1):
    xs = [E.of(x) for x in xs]
    return E(torch.stack(torch.broadcast_tensors(*[x.val for x in xs]), dim),
             torch.stack(torch.broadcast_tensors(*[x.err for x in xs]), dim))

  def col(self, x):
    return E(x.val[..., None], x.err[..., None])

  # ---- warp reductions (see the module notes): x [B, S]
  def wsum(self, x, CH):
    x = E.of(x)
    return E(x.val.sum(-1), x.err.sum(-1) + (CH + 5) * U * (x.val.abs() + x.err).sum(-1) + TINY)

  def scan(self, x, CH, xlocal=None):
    """(exclusive, inclusive) prefix of x along the samples, and the scan's total."""
    D = 2 * CH + 5
    z = torch.zeros_like(x.val[:, :1])
    cv, ce, ca = (torch.cumsum(t, -1) for t in (x.val, x.err, x.val.abs() + x.err))
    ex = lambda t: torch.cat([z, t[:, :-1]], -1)
    excl = E(ex(cv), ex(ce) + D * U * ex(ca) + TINY)
    incl = E(cv, ce + D * U * ca + TINY)
    return excl, incl, E(cv[:, -1], ce[:, -1] + D * U * ca[:, -1] + TINY)

  def after(self, gw, CH, mut=None):
    """sum_{i > s} gw_i as the kernel's reverse lane scan forms it."""
    D = 2 * CH + 5
    S = gw.val.shape[-1]
    rv = torch.flip(torch.cumsum(torch.flip(gw.val, [-1]), -1), [-1])
    re = torch.flip(torch.cumsum(torch.flip(gw.err, [-1]), -1), [-1])
    ra = torch.flip(torch.cumsum(torch.flip(gw.val.abs() + gw.err, [-1]), -1), [-1])
    z = torch.zeros_like(rv[:, :1])
    sh = lambda t: torch.cat([t[:, 1:], z], -1)
    lane0 = (torch.arange(S, device=rv.device) // CH) * CH           # first sample of each sample's lane
    return E(sh(rv), sh(re) + D * U * ra[:, lane0] + TINY)

  def fine_sum(self, x, Sf):
    """lane i sums the fine intervals i, i + 32, ..., then warp_sum."""
    return E(x.val.sum(-1), x.err.sum(-1) + ((Sf + 31) // 32 + 5) * U * (x.val.abs() + x.err).sum(-1) + TINY)

  def scatter_D(self, gi, lo, hi, live, S, rng=None):
    B = gi.val.shape[0]
    g = torch.where(live, gi.val, torch.zeros_like(gi.val))
    ge = torch.where(live, gi.err, torch.zeros_like(gi.err))
    v = torch.zeros(B, S + 2, dtype=torch.float64, device=g.device)
    e, a, n = v.clone(), v.clone(), v.clone()
    for idx, sg in ((lo, 1.0), (hi, -1.0)):
      v.scatter_add_(1, idx, sg * g)
      e.scatter_add_(1, idx, ge)
      a.scatter_add_(1, idx, g.abs() + ge)
      n.scatter_add_(1, idx, live.double())
    return E(v, e + n * U * a + TINY)

  def gather(self, x, idx):
    return E(torch.gather(x.val, 1, idx), torch.gather(x.err, 1, idx))

  def stat(self, terms, n0=1):
    """Sum of per-ray terms [B] (or [B, k]) into one stats word, in any order."""
    t = E.of(terms)
    n = t.val.numel() + n0
    return E(t.val.sum(), t.err.sum() + n * U * (t.val.abs() + t.err).sum() + TINY)


def tdist(b, x, fn, S):
  """s_to_t of every knot: fn_inv(fl(fl(s s_far) + fl(fl(1 - s) s_near))) with s_near = fn(near), s_far = fn(far)."""
  def fwd(v):
    if fn == 'reciprocal':
      return 1.0 / v
    if fn == 'log':
      return b.log(v)
    if fn == 'exp':
      return b.exp(v)
    if fn == 'sqrt':
      return b.sqrt(v)
    if fn == 'square':
      return v * v
    if fn == 'piecewise':     # branch on the exact fp32 near / far
      lt = b.val(v) < 1
      return b.where(lt, b.c(0.5) * v, 1.0 - b.c(0.5) / v)
    return v

  def inv(v):
    if fn == 'reciprocal':
      return 1.0 / v
    if fn == 'log':
      return b.exp(v)
    if fn == 'exp':
      return b.log(v)
    if fn == 'sqrt':
      return v * v
    if fn == 'square':
      return b.sqrt(v)
    if fn == 'piecewise':     # C1 across x = 0.5: a sample within rounding of it moves by O(e^2)
      lt = b.val(v) < 0.5
      return b.where(lt, b.c(2.0) * v, b.c(0.5) / (1.0 - v))
    return v
  s_near = b.col(fwd(b.inp(x['near'])))
  s_far = b.col(fwd(b.inp(x['far'])))
  s = b.inp(x['sdist'])
  return inv(s * s_far + (1.0 - s) * s_near)


def _rgb_act(b, kind, z):
  return b.exp(b.fmin(z, 88.0)) if kind == 'safe_exp' else b.sigmoid(z)


def _lin2srgb(b, lin, grad=False):
  thr = float(np.float32(0.0031308))
  lin_piece = b.val(lin) <= thr
  near = (b.val(lin) - thr).abs() <= b.err(lin)
  if not grad:
    hi = (b.c(211.0) * b.pow(b.fmax(lin, K_EPS), k32(5.0 / 12.0)) - 11.0) / b.c(200.0)
    return b.where(lin_piece, b.k(k32(323.0 / 25.0)) * lin, hi), near
  g = b.k((float(np.float32(np.float32(211.0 / 200.0) * np.float32(5.0 / 12.0))), 211.0 / 200.0 * 5.0 / 12.0))
  hi = b.where(b.val(lin) > K_EPS, g * b.pow(b.fmax(lin, K_EPS), k32(-7.0 / 12.0)), b.zeros(b.val(lin).shape))
  return b.where(lin_piece, b.k(k32(323.0 / 25.0)) * b.c(1.0) + b.zeros(b.val(lin).shape), hi)


def colour_walk(b, x, cfg, mut=None):
  """colour_fwd of every sample and channel of x['raw_rgb'] [..., 3] (before the per-ray scale).  Returns a namespace:
  c, the activation a and z, t, dl, lin, sr (rgb_mode 1), and the exemptions `unsure_lin` (the sRGB piece, within
  bound of its threshold) and `unsure_clip` (the sRGB value within bound of 0 or 1)."""
  o = types.SimpleNamespace()
  z = b.c(f32(cfg['rgb_premultiplier'])) * b.inp(x['raw_rgb']) + b.c(f32(cfg['rgb_bias']))
  a = _rgb_act(b, cfg['rgb_activation'], z)
  o.z, o.act = z, a
  shape = b.val(z).shape
  o.unsure_lin = o.unsure_clip = torch.zeros(shape, dtype=torch.bool, device=b.val(z).device)
  if cfg.get('rgb_mode', 0) == 1:
    o.t = b.sigmoid(b.inp(x['raw_tint'])) if x.get('raw_tint') is not None else b.c(0.5)
    o.dl = b.sigmoid(b.inp(x['raw_diffuse']) - b.k(k32(math.log(3.0))))
    o.lin = o.t * a + o.dl
    o.sr, o.unsure_lin = _lin2srgb(b, o.lin)
    sv, se = b.val(o.sr), b.err(o.sr)
    o.unsure_clip = ((sv.abs() <= se) | ((sv - 1).abs() <= se)) & ~o.unsure_lin
    a = b.fmin(b.fmax(o.sr, 0.0), 1.0)
  pad = f32(cfg['rgb_padding'])
  o.pad1 = 1.0 + b.c(2 * pad)
  o.c = a * o.pad1 - b.c(pad)
  if mut == 'pad_twice':
    o.c = o.c * o.pad1 - b.c(pad)
  return o


def walk(b, x, cfg, loss=None, dec=None, batch_rays=None, mut=None, want_dist=True):
  """The arithmetic of composite_fwd_kernel (and, with `loss`, composite_bwd_kernel) on backend `b`.

  x: the fp32 inputs (CPU or CUDA tensors) as for `composite`, plus 'inv_denom' (a tensor of one fp32) with `loss`.
  dec: the kernel's decisions -- dict(bg_on [B] bool, v_lt1 [B, 3] bool) -- or None to take this backend's own.
  mut: a kernel bug for the CPU tests' mutants (MUTANTS); the reference passes None.
  Returns a namespace of backend values and exemption masks."""
  o = types.SimpleNamespace()
  raw = x['raw_density']
  B, S = raw.shape
  CH = ch_of(S)
  dev = raw.device
  o.CH = CH
  tds = tdist(b, x, cfg['raydist_fn'], S)
  o.tdist = tds
  d = b.inp(x['directions'])
  dnorm = b.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
  r = b.inp(raw)
  if x.get('density_noise') is not None:
    r = r + b.c(f32(cfg['density_noise'])) * b.inp(x['density_noise'])
  din = r + b.c(f32(cfg['density_bias']))
  ax = b.where(b.val(din) > 0, din, b.zeros((B, S)) - din)          # fabsf: exact
  dens = b.fmax(din, 0.0) + b.log1p(b.exp(b.zeros((B, S)) - ax))
  delta = (tds[:, 1:] - tds[:, :-1]) * b.col(dnorm)
  a = dens * delta
  last = torch.zeros(B, S, dtype=torch.bool, device=dev)
  if cfg['opaque_background'] and not (mut == 'no_inf_ragged' and CH > 1 and S % CH):
    last[:, -1] = True
  a = b.where(last, b.c(math.inf), a)
  o.dens, o.din, o.delta, o.a = dens, din, delta, a
  # T_s = expf(-(exclusive prefix of a)); the opaque last a never enters a prefix that is used
  a_fin = b.where(last, b.zeros((B, S)), a)
  excl, incl, _ = b.scan(a_fin, CH)
  T = b.exp(b.zeros((B, S)) - (incl if mut == 'inclusive_T' else excl))
  alpha = 1.0 - b.exp(b.zeros((B, S)) - a)
  w = alpha * T
  o.T, o.w = T, w
  o.acc = b.wsum(w, CH)
  # colour
  if x.get('raw_rgb') is not None:
    col = colour_walk(b, x, cfg, mut)
    sc = b.inp(x['rgb_scale'])[:, None, :] if x.get('rgb_scale') is not None else b.c(1.0)
    c = col.c * sc
  else:
    col = None
    c = b.zeros((B, S, 3))
  o.col, o.c = col, c
  unsure_ray = torch.zeros(B, dtype=torch.bool, device=dev)
  if col is not None:
    unsure_ray = col.unsure_lin.reshape(B, -1).any(-1)
  o.unsure_ray = unsure_ray
  wc = [b.wsum(w * c[..., ch], CH) for ch in range(3)]
  bg_w = b.fmax(1.0 - o.acc, 0.0)
  bgc = [b.inp(x['bg_rgb'][:, ch]) if x.get('bg_rgb') is not None else b.c(f32(cfg['bg_const'])) for ch in range(3)]
  pix = [wc[ch] + bg_w * bgc[ch] for ch in range(3)]
  o.rgb = b.stack(pix)
  if want_dist:
    tm = b.c(0.5) * (tds[:, :-1] + tds[:, 1:])
    elog = b.wsum(w * b.log(tm), CH)
    dm = b.exp(elog / b.fmax(o.acc, K_EPS))
    dv = b.val(dm)
    nan = torch.isnan(dv)
    dm = b.where(nan, b.zeros(dv.shape), b.where(torch.isinf(dv), b.c(F32_MAX), dm))
    dm = b.mine(b.maxe(dm, tds[:, 0]), tds[:, S])
    o.distance_mean = dm
    _, cw, _ = b.scan(w, CH)
    o.cws = b.fmin(cw, 1.0)
  if loss is None:
    return o

  # ---- backward
  inv_denom = b.inp(x['inv_denom'])
  dmult = b.c(f32(loss['data_mult']))
  nb = B if (mut == 'invB_num_rays' or batch_rays is None) else batch_rays
  invB = 1.0 / b.c(float(nb))
  lm_ch = x['lossmult'].shape[-1]
  if dec is None:
    acc_v = b.val(o.acc)
    bg_on = (1.0 - acc_v) >= 0 if mut == 'bg_on_tie' else (1.0 - acc_v) > 0
  else:
    bg_on = dec['bg_on'].to(dev)
  bg_on_f = bg_on.double()
  dpx, st_data, st_mse, lmv = [], [], [], []
  for ch in range(3):
    tgt = b.inp(x['target'][:, ch])
    li = ch if (lm_ch == 3 and mut != 'lossmult_ray') else 0
    if mut == 'lossmult_ray' and lm_ch == 3:
      lm = b.inp(x['lossmult'].reshape(-1)[torch.arange(B, device=dev)])
    else:
      lm = b.inp(x['lossmult'][:, li])
    v = pix[ch]
    resid = v - tgt
    lt = loss['loss_type']
    if lt == 'mse':
      lv, g = resid * resid, b.c(2.0) * resid
    elif lt == 'charb':
      cp = b.c(f32(loss['charb_padding']))
      lv = b.sqrt(resid * resid + cp * cp)
      g = resid / lv
    else:
      clip = b.fmin(v, 1.0)
      rc = clip - tgt
      scl = 1.0 / (b.k(k32(1e-3)) + clip)
      lv = ((rc * rc) * scl) * scl
      lt1 = (b.val(v) < 1) if dec is None else dec['v_lt1'][:, ch].to(dev)
      g = b.where(lt1, ((b.c(2.0) * rc) * scl) * scl, b.zeros((B,)))
    mse_term = ((lm * resid) * resid) * inv_denom
    if x.get('data_mask') is not None:
      m = b.inp(x['data_mask'])
      lv, g = lv * m, g * m
      if mut == 'mse_masked':
        mse_term = mse_term * m
    dp = ((dmult * lm) * g) * inv_denom
    dpx.append(dp)
    st_data.append(((dmult * lm) * lv) * inv_denom)
    st_mse.append(mse_term)
  o.dpx = dpx
  o.st_data, o.st_mse = b.stack(st_data), b.stack(st_mse)
  if x.get('rgb_scale') is not None:
    scv = b.inp(x['rgb_scale'])
    ds = []
    for ch in range(3):
      zero = b.val(scv[:, ch]) == 0
      wcu = b.wsum(w * col.c[..., ch], CH) if col is not None else b.zeros((B,))
      if mut == 'zero_scale_divides':
        zero = torch.zeros_like(zero)
      ds.append(b.where(zero, dpx[ch] * wcu, (dpx[ch] * wc[ch]) / scv[:, ch]))
    o.d_rgb_scale = b.stack(ds)
  # dL/dw
  g = b.zeros((B, S))
  for ch in range(3):
    g = g + b.col(dpx[ch]) * (c[..., ch] - b.col(bgc[ch] * b.inp(bg_on_f)))
  if x.get('extra_dw') is not None:
    g = g + b.inp(x['extra_dw'])
  o.st_dist = b.zeros((B,))
  if loss['distortion_mult'] > 0:
    src = tds if mut == 'dist_tdist' else b.inp(x['sdist'])
    s0, s1 = src[:, :-1], src[:, 1:]
    m = b.c(0.5) * (s0 + s1)
    dl = s1 - s0
    pw, _, totw = b.scan(w, CH)
    wm = w * m
    pwm, _, totwm = b.scan(wm, CH)
    sw = (b.col(totw) - pw) - w
    swm = (b.col(totwm) - pwm) - wm
    inter = ((m * pw - pwm) + swm) - m * sw
    third = k32(2.0 / 3.0) if mut == 'dist_two_thirds' else k32(1.0 / 3.0)
    lossp = w * inter + ((w * w) * dl) * b.k(third)
    dmi = b.c(f32(loss['distortion_mult'])) * invB
    g = g + dmi * (b.c(2.0) * inter + (b.k(k32(2.0 / 3.0)) * w) * dl)
    o.st_dist = dmi * b.wsum(lossp, CH)
  o.st_inter = b.zeros((B,))
  if loss['interlevel_mult'] > 0:
    senv = x['sdist'].to(dev)
    cf, wf = x['sdist_fine'].to(dev), x['weights_fine'].to(dev)
    Sf = wf.shape[1]
    _, cyi, _ = b.scan(w, CH)
    cy = _cat0(b, cyi)
    lo = (torch.searchsorted(senv.contiguous(), cf[:, :-1].contiguous(), right=True) - 1).clamp(min=0)
    hi = torch.searchsorted(senv.contiguous(), cf[:, 1:].contiguous(), right=(mut != 'inter_off_by_one')).clamp(max=S)
    w_outer = b.gather(cy, hi) - b.gather(cy, lo)
    wfv = b.inp(wf)
    ex = b.fmax(wfv - w_outer, 0.0)
    den = wfv + b.c(K_EPS)
    sf_n = Sf + 1 if mut == 'inter_wrong_sf' else Sf
    scale = b.c(f32(loss['interlevel_mult'])) / (b.c(float(nb)) * b.c(float(sf_n)))
    o.st_inter = scale * b.fine_sum((ex * ex) / den, Sf)
    gi = ((b.c(-2.0) * ex) / den) * scale
    live = hi > lo              # the kernel skips gi == 0: the same as adding zero, but its bound still counts
    D = b.scatter_D(gi, lo, hi, live, S)
    _, rd, _ = b.scan(D[:, :S], CH)
    g = g + rd
    o.lo, o.hi = lo, hi
  o.g = g
  gw = g * w
  after = b.after(gw, CH, mut)
  ea = b.exp(b.zeros((B, S)) - b.where(last, b.zeros((B, S)), a))
  da = b.where(last, b.zeros((B, S)), (g * ea) * T - after)
  o.d_raw_density = (da * delta) * b.sigmoid(din)
  if col is not None:
    scb = b.inp(x['rgb_scale'])[:, None, :] if x.get('rgb_scale') is not None else b.c(1.0)
    gc = ((b.stack(dpx)[:, None, :] * b.col(w)) * scb) * col.pad1
    if cfg['rgb_activation'] == 'safe_exp':
      dact = b.exp(b.fmin(col.z, 88.0))
    else:
      s_ = b.sigmoid(col.z)
      dact = s_ * (1.0 - s_)
    dact = dact * b.c(f32(cfg['rgb_premultiplier']))
    if cfg.get('rgb_mode', 0) == 1:
      sv = b.val(col.sr)
      inside = ((sv > 0) & (sv < 1)) | (mut == 'clip_passes')
      glin = b.where(inside, gc * _lin2srgb(b, col.lin, grad=True), b.zeros(sv.shape))
      o.d_raw_rgb = (glin * col.t) * dact
      o.d_raw_diffuse = (glin * col.dl) * (1.0 - col.dl)
      if x.get('raw_tint') is not None:
        o.d_raw_tint = glin * col.act if mut == 'tint_no_tt' else ((glin * col.act) * col.t) * (1.0 - col.t)
      else:
        o.d_raw_tint = b.zeros(sv.shape)
    else:
      o.d_raw_rgb = gc * dact
  return o


def _cat0(b, x):
  """[0, x] along the samples."""
  if isinstance(x, E):
    z = torch.zeros_like(x.val[:, :1])
    return E(torch.cat([z, x.val], -1), torch.cat([z, x.err], -1))
  return np.concatenate([np.zeros_like(x[:, :1]), x], -1)


def reference(inp, cfg, loss=None, dec=None, batch_rays=None, device='cpu'):
  """fp64 values of every kernel output (fp64 autograd of `composite`) with a bound on each element (the walk's
  error plus its distance from the autograd value, scaled by SLACK) and its exemption mask.  inp: fp32 tensors as
  for `composite` (+ 'inv_denom' with `loss`); dec: the kernel's decisions (see `walk`).

  Returns dict name -> (value, bound, exempt); 'stats' -> (value [4], bound [4], None); 'cws' / 'tdist' -> the walk's
  E values (percentiles), and 'chain_gap': the largest |walk - autograd| / bound seen."""
  x = {k: v.to(device) for k, v in inp.items()}
  b = Running(device)
  o = walk(b, x, cfg, loss, dec, batch_rays)
  in64 = {k: v.to(device, torch.float64) for k, v in inp.items() if k != 'inv_denom'}
  if loss is not None:
    lref = dict(loss, inv_denom=float(inp['inv_denom'].reshape(-1)[0]))
    bg_on = dec['bg_on'].to(device) if dec is not None else None
    with torch.device(device):
      r, g = grads(in64, cfg, lref, bg_on=bg_on, branches=None if cfg.get('rgb_mode', 0) != 1 else _branches(o))
      if batch_rays is not None and batch_rays != inp['raw_density'].shape[0]:
        r, g = _rescaled(in64, cfg, lref, bg_on, o, batch_rays)
  else:
    with torch.device(device):
      r = composite(in64, cfg)
    g = {}
  B, S = inp['raw_density'].shape
  res = dict(chain_gap=0.0, cws=o.cws, tdist=o.tdist, t_aug=r['t_aug'].detach(), cdf=r['cdf'].detach())
  ray_x = o.unsure_ray

  def put(name, e, ref, extra=None):
    ref = ref.detach()
    gap = (e.val - ref).abs()
    bd = torch.nan_to_num(SLACK * (e.err + gap) + TINY, nan=math.inf)   # inf * 0 of a vacuous bound: vacuous
    fin = torch.isfinite(ref) & torch.isfinite(bd)
    res['chain_gap'] = max(res['chain_gap'], float((gap / (e.err + 1e-30))[fin].max()) if fin.any() else 0.0)
    ex = ray_x.reshape((B,) + (1,) * (ref.dim() - 1)).expand_as(ref).clone()
    if extra is not None:
      ex |= extra
    res[name] = (ref, bd, ex)
  put('weights', o.w, r['weights'])
  put('density', o.dens, r['density'])
  put('rgb_samples', o.c, r['rgb_samples'])
  put('rgb', o.rgb, r['rgb'])
  put('acc', o.acc, r['acc'])
  put('distance_mean', o.distance_mean, r['distance_mean'])
  if loss is None:
    return res
  clip_x = o.col.unsure_clip if o.col is not None else None
  put('d_raw_density', o.d_raw_density, g['raw_density'])
  for k in ('raw_rgb', 'raw_diffuse', 'raw_tint'):
    if k in g:
      put('d_' + k, getattr(o, 'd_' + k), g[k], clip_x)
  if cfg.get('rgb_mode', 0) == 1 and 'raw_tint' not in g:
    put('d_raw_tint', o.d_raw_tint, torch.zeros(B, S, 3, dtype=torch.float64, device=device))
  if 'rgb_scale' in g:
    put('d_rgb_scale', o.d_rgb_scale, g['rgb_scale'])
  sv, sb = [], []
  for name, t in (('data', o.st_data), ('mse', o.st_mse), ('distortion', o.st_dist), ('interlevel', o.st_inter)):
    tot = b.stat(t)
    ref = r[name].detach().reshape(())
    gap = (tot.val - ref).abs()
    res['chain_gap'] = max(res['chain_gap'], float(gap / (tot.err + 1e-30)))
    sv.append(ref)
    sb.append(torch.nan_to_num(SLACK * (tot.err + gap) + TINY, nan=math.inf))
  res['stats'] = (torch.stack(sv), torch.stack(sb), torch.zeros(4, dtype=torch.bool, device=device))
  res['stat_terms'] = [o.st_data, o.st_mse, o.st_dist, o.st_inter]
  return res


def _branches(o):
  """The sRGB branches of the walk's fp64 values (an element where they are not decided is exempt anyway)."""
  return dict(linear=o.col.lin.val <= float(np.float32(0.0031308)), inside=(o.col.sr.val > 0) & (o.col.sr.val < 1))


def _rescaled(in64, cfg, lref, bg_on, o, batch_rays):
  """The gradients of one pass of a batch of `batch_rays` rays: the distortion and interlevel means divide by
  batch_rays, so their multipliers scale by B / batch_rays."""
  B = in64['raw_density'].shape[0]
  f = B / batch_rays
  l2 = dict(lref, distortion_mult=lref['distortion_mult'] * f, interlevel_mult=lref['interlevel_mult'] * f)
  return grads(in64, cfg, l2, bg_on=bg_on, branches=None if cfg.get('rgb_mode', 0) != 1 else _branches(o))


def check(name, got, ref, bound, exempt, min_live=0.0):
  """Every non-exempt element of `got` within its bound.  Returns (live fraction, worst err / bound)."""
  got = got.detach().to(ref.device, torch.float64).reshape(ref.shape)
  err = (got - ref).abs()
  ok = (err <= bound) | exempt
  both_inf = torch.isinf(got) & torch.isinf(ref) & (torch.sign(got) == torch.sign(ref))
  ok |= both_inf
  vac = bound > VACUOUS * ref.abs() + 2 * TINY + 1e-30
  live = ~exempt & ~vac & ~both_inf
  ratio = torch.where(exempt | both_inf, torch.zeros_like(err), err / bound)
  ratio = torch.nan_to_num(ratio, nan=math.inf)
  worst = float(ratio.max()) if ratio.numel() else 0.0
  frac = float(live.double().mean()) if live.numel() else 1.0
  if not bool(ok.all()) or not math.isfinite(worst):
    i = tuple(int(v) for v in np.unravel_index(int(torch.argmax(ratio)), ratio.shape))
    raise AssertionError(f'{name}: {int((~ok).sum())} of {ok.numel()} elements outside their bound; worst at {i}: '
                         f'got {float(got[i])!r}, reference {float(ref[i])!r}, bound {float(bound[i]):.3e}')
  assert frac >= min_live, f'{name}: live fraction {frac:.2f} < {min_live}'
  return frac, worst


def check_percentiles(name, got, res, min_live=0.0):
  """Percentiles in CDF space: the fp64 CDF F (knots t_aug, values cdf) over [v - et, v + et] must reach p within
  3 max knot error + 8u, et the row's largest tdist bound plus the interpolation's rounding (see the module notes)."""
  got = got.detach().to(res['cdf'].device, torch.float64)
  B = got.shape[0]
  cw = res['cws']
  kerr = cw.err.amax(-1)
  t = res['tdist']
  terr = t.err.amax(-1)
  tmax = res['t_aug'].abs().amax(-1)
  bc = 3 * kerr + 8 * U
  et = terr[:, None] + 4 * U * (got.abs() + tmax[:, None])
  p = torch.tensor([0.05, 0.5, 0.95], dtype=torch.float64, device=got.device).expand(B, 3)
  lo = cdf_at(res['t_aug'], res['cdf'], got - et) - p
  hi = cdf_at(res['t_aug'], res['cdf'], got + et) - p
  bad = (lo > bc[:, None]) | (hi < -bc[:, None])
  if bad.any():
    i = tuple(int(v) for v in (bad.nonzero()[0]))
    raise AssertionError(f'{name}: {int(bad.sum())} percentiles off; worst at {i}: got {float(got[i])!r}, CDF there '
                         f'[{float(lo[i] + p[i]):.6g}, {float(hi[i] + p[i]):.6g}] vs p {float(p[i])}, bound '
                         f'{float(bc[i[0]]):.3e}')
