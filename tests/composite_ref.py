"""Reference of the compositing kernels (csrc/composite.cu) in any float dtype, built from the oracle.

`composite` assembles the oracle's colour activations, o_render.compute_alpha_weights / volumetric_rendering
and the o_train losses the way mnrf_composite_fwd and mnrf_composite_bwd combine them for one level, with every
optional input the kernels take.  Evaluated in float64 on the kernels' fp32 inputs and differentiated by
torch.autograd it is the yardstick of tests/test_gpu_composite_fp64.py; evaluated in float32 it is the fp32
oracle whose own error sets that test's tolerance.  Pure torch: runs on the CPU or on CUDA tensors, and never
loads the CUDA library.
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
