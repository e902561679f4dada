"""Generate tests/golden/robustnerf.npz by EXECUTING the reference's own internal/robustnerf.py and
`compute_data_loss(..., 'robustnerf')` (internal/train_utils.py:72-136) under the jax stand-ins.

Run in the build container only (needs /root/reference):
    python tests/golden/make_golden_robustnerf.py
robustnerf.py needs three things the shared stand-ins (tests/golden/standin/) do not provide; this script adds
them to the stand-in modules for its own run: `lax.conv` accumulated in fp64 and rounded once, `jnp.quantile`
restating JAX's 'linear' formula in fp32 (numpy's own lerp rounds differently), and `jnp.mean` over a list of
axes.  XLA's own rounding of the first two is not pinned by this fixture.  Every case stores its inputs
(rendered rgb, target, threshold, config) next to the reference's outputs.
"""
import math
import os
import sys
import types
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'standin'))
sys.path.insert(0, '/root/reference')
np.math = math
for missing in ['dm_pix', 'cv2', 'rawpy', 'mediapy', 'optax', 'pycolmap', 'matplotlib', 'tensorflow']:
  try:
    __import__(missing)
  except Exception:  # pylint: disable=broad-except
    sys.modules[missing] = mock.MagicMock()

import jax  # noqa: E402  (the stand-in)
import jax.numpy as jnp  # noqa: E402


def _conv(lhs, rhs, window_strides, padding):
  """lax.conv (NCHW input, OIHW kernel, no dilation) for the box filter of robustnerf.py:45-47: accumulated in
  fp64 and rounded once to fp32 (XLA's accumulation order is not reproduced)."""
  x = np.asarray(lhs, np.float64)
  w = np.asarray(rhs, np.float64)
  n, c, h, wd = x.shape
  o, ci, kh, kw = w.shape
  assert ci == c and tuple(window_strides) == (1, 1) and padding == 'SAME'
  ph, pw = kh - 1, kw - 1
  xp = np.pad(x, ((0, 0), (0, 0), (ph // 2, ph - ph // 2), (pw // 2, pw - pw // 2)))
  out = np.zeros((n, o, h, wd))
  for i in range(kh):
    for j in range(kw):
      out += np.einsum('nchw,oc->nohw', xp[:, :, i:i + h, j:j + wd], w[:, :, i, j])
  return out.astype(np.float32)


def _quantile(a, q, axis=None, method='linear', keepdims=False):
  """jnp.quantile, method 'linear', restated from JAX: the sorted input in fp32, n and q in fp32,
  qn = q * (n - 1), lo = floor(qn), hi = ceil(qn), w = qn - lo, x[lo] * (1 - w) + x[hi] * w.  NaN if any NaN."""
  assert axis is None and method == 'linear' and not keepdims
  x = np.sort(np.asarray(a, np.float32).reshape(-1))
  if np.isnan(x).any():
    return np.float32('nan')
  n = np.float32(x.size)
  qn = np.float32(q) * (n - np.float32(1))
  lo, hi = np.floor(qn), np.ceil(qn)
  w = qn - lo
  lo_i = int(min(max(lo, 0), x.size - 1))
  hi_i = int(min(max(hi, 0), x.size - 1))
  return np.float32(x[lo_i] * (np.float32(1) - w) + x[hi_i] * w)


_stand_in_mean = jnp.mean


def _mean(a, axis=None, **kw):
  return _stand_in_mean(a, axis=tuple(axis) if isinstance(axis, list) else axis, **kw)


jax.lax.conv = _conv
jnp.quantile = _quantile
jnp.mean = _mean

from internal import robustnerf, train_utils, utils  # noqa: E402

F = np.float32
CFG_KEYS = ('patch_size', 'robustnerf_inner_patch_size', 'robustnerf_smoothed_filter_size',
            'robustnerf_inlier_quantile', 'robustnerf_smoothed_inlier_quantile',
            'robustnerf_inner_patch_inlier_quantile', 'enable_robustnerf_loss')


def config(**kw):
  c = dict(patch_size=16, robustnerf_inner_patch_size=8, robustnerf_smoothed_filter_size=3,
           robustnerf_inlier_quantile=0.5, robustnerf_smoothed_inlier_quantile=0.5,
           robustnerf_inner_patch_inlier_quantile=0.5, enable_robustnerf_loss=True,
           data_loss_type='robustnerf', disable_multiscale_loss=False, compute_disp_metrics=False,
           compute_normal_metrics=False, data_coarse_loss_mult=0.1, data_loss_mult=1.0)
  c.update(kw)
  return types.SimpleNamespace(**c)


def patches(rng, n, p, outlier_frac=0.3):
  """Rendered / target colours of n p x p patches: small residuals, plus blobs of large ones in some patches."""
  target = rng.uniform(0, 1, (n, p, p, 3)).astype(F)
  noise = rng.normal(0, 0.05, (n, p, p, 3))
  for i in range(n):
    if rng.uniform() < 0.7:
      cy, cx = rng.integers(0, p, 2)
      r = rng.uniform(0.15, 0.6) * p
      yy, xx = np.mgrid[:p, :p]
      blob = (yy - cy) ** 2 + (xx - cx) ** 2 < r * r
      noise[i][blob] += rng.normal(0, 0.5, (blob.sum(), 3))
    sprinkle = rng.uniform(size=(p, p)) < outlier_frac * rng.uniform()
    noise[i][sprinkle] += rng.normal(0, 0.4, (sprinkle.sum(), 3))
  rgb = (target + noise).astype(F)
  return rgb, target


def run(out, name, rgb, target, thr, cfg):
  resid_sq = (rgb - target) ** 2
  mask, stats = robustnerf.robustnerf_mask(resid_sq, F(thr), cfg)
  out[f'{name}/rgb'], out[f'{name}/target'], out[f'{name}/threshold'] = rgb, target, F(thr)
  for k in CFG_KEYS:
    out[f'{name}/cfg/{k}'] = np.asarray(getattr(cfg, k))
  out[f'{name}/mask'] = np.asarray(mask, F)
  out[f'{name}/error_per_pixel'] = np.mean(resid_sq, axis=-1, keepdims=True).astype(F)
  for k, v in stats.items():
    out[f'{name}/stat/{k}'] = np.asarray(v, F)
  # the data loss of two levels through compute_data_loss (the last level's robust stats survive)
  rgb0 = (rgb + F(0.01)).astype(F)
  lossmult = np.ones(rgb.shape[:-1] + (1,), F)
  batch = utils.Batch(rays=types.SimpleNamespace(lossmult=lossmult), rgb=target)
  loss, dstats = train_utils.compute_data_loss(batch, [{'rgb': rgb0}, {'rgb': rgb}], batch.rays, F(thr), cfg)
  out[f'{name}/loss_data'] = np.asarray(loss, F)
  out[f'{name}/mses'] = np.asarray(dstats['mses'], F)
  for k in stats:
    out[f'{name}/dstat/{k}'] = np.asarray(dstats[k], F)
  m = float(np.asarray(mask).mean())
  print(f'{name}: patches {rgb.shape[0]}x{rgb.shape[1]}, threshold {float(thr):.5g}, mask mean {m:.3f}, '
        f'next threshold {float(stats["loss_threshold"]):.5g}')


def main():
  rng = np.random.default_rng(20240607)
  out = {}
  names = []

  def case(name, n, p, thr_q=0.6, **kw):
    cfg = config(patch_size=p, **kw)
    rgb, target = patches(rng, n, p)
    err = np.mean((rgb - target) ** 2, -1)
    thr = np.quantile(err, thr_q).astype(F)
    run(out, name, rgb, target, thr, cfg)
    names.append(name)

  case('defaults', 6, 16)
  case('asym_inner', 8, 8, robustnerf_inner_patch_size=3)
  case('filter5', 6, 16, robustnerf_smoothed_filter_size=5)
  case('q08', 6, 16, robustnerf_inlier_quantile=0.8)
  case('disabled', 4, 16, enable_robustnerf_loss=False)

  # errors exactly equal to the threshold: the threshold is one pixel's error, copied to a quarter of the pixels
  cfg = config(patch_size=8, robustnerf_inner_patch_size=4)
  rgb, target = patches(rng, 4, 8)
  sel = rng.uniform(size=rgb.shape[:-1]) < 0.25
  rgb[sel], target[sel] = rgb[0, 3, 3], target[0, 3, 3]
  thr = np.mean(((rgb - target) ** 2)[0, 3, 3], -1).astype(F)
  run(out, 'ties', rgb, target, thr, cfg)
  names.append('ties')

  # patch means at the boundary: a 1x1 filter keeps the inlier bits, and patches hold 127, 128, 129 inliers of 256
  # (0.5 is not > 0.5); the inner patch mask decides the rest
  cfg = config(patch_size=16, robustnerf_smoothed_filter_size=1, robustnerf_inner_patch_size=6)
  n = 5
  target = rng.uniform(0, 1, (n, 16, 16, 3)).astype(F)
  rgb = target.copy()
  for i, k in enumerate((127, 128, 129, 0, 256)):
    bad = np.ones(256, bool)
    bad[rng.permutation(256)[:k]] = False
    rgb[i].reshape(256, 3)[bad] += F(0.5)
  run(out, 'patch_boundary', rgb, target, F(0.01), cfg)
  names.append('patch_boundary')
  out['cases'] = np.array(names)

  path = os.path.join(HERE, 'robustnerf.npz')
  np.savez_compressed(path, **out)
  print('robustnerf.npz', len(out), 'arrays')


if __name__ == '__main__':
  main()
