"""Oracle (test infrastructure): the RobustNeRF loss, data_loss_type 'robustnerf'.

Follows /root/reference/internal/robustnerf.py:8-115 (robustnerf_mask, _robustnerf_inner_patch_mask) and the
'robustnerf' branch of train_utils.compute_data_loss :104-108.  Other loss types are o_train's.
jnp.quantile (robustnerf.py:26) is restated from JAX's 'linear' method: n and q in fp32,
qn = q * (n - 1), lo = floor(qn), hi = ceil(qn), w = qn - lo, x_(lo) * (1 - w) + x_(hi) * w.
"""
import torch

from . import o_train


def quantile_linear(x, q):
  """jnp.quantile(x, q) with method='linear' over all elements, in fp32 (NaN if any element is NaN)."""
  x = x.detach().reshape(-1).to(torch.float32)
  if bool(torch.isnan(x).any()):
    return torch.tensor(float('nan'), dtype=torch.float32, device=x.device)
  xs = torch.sort(x).values
  n = xs.numel()
  f32 = lambda v: torch.tensor(v, dtype=torch.float32, device=x.device)
  qn = f32(q) * (f32(float(n)) - f32(1.0))
  lo, hi = torch.floor(qn), torch.ceil(qn)
  w = qn - lo
  lo_i = min(max(int(lo), 0), n - 1)
  hi_i = min(max(int(hi), 0), n - 1)
  return xs[lo_i] * (f32(1.0) - w) + xs[hi_i] * w


def robustnerf_mask(errors, loss_threshold, config):
  """robustnerf.py:8-86.  errors: [n, p, p, c] fp32 per-subpixel errors; loss_threshold: scalar (the previous
  step's threshold).  Returns (mask [n, p, p, 1], stats).  Means of 0/1 values are fl32(count / size), the
  box filter is a count of inlier neighbours (zero padding) divided by f^2."""
  f32 = lambda v: torch.tensor(v, dtype=torch.float32, device=errors.device)
  errors = errors.detach().to(torch.float32)
  error_per_pixel = (errors[..., 0:1] + errors[..., 1:2] + errors[..., 2:3]) / f32(3.0)
  stats = {'loss_threshold': quantile_linear(error_per_pixel, config.robustnerf_inlier_quantile)}
  mean = lambda t: t.sum() / f32(float(t.numel()))
  mask = torch.ones_like(error_per_pixel)
  if config.enable_robustnerf_loss:
    assert config.robustnerf_inner_patch_size <= config.patch_size, \
        'patch_size must be larger than robustnerf_inner_patch_size.'
    thr = torch.as_tensor(loss_threshold, dtype=torch.float32, device=errors.device)
    is_inlier_pixel = (error_per_pixel < thr).to(torch.float32)
    stats['is_inlier_loss'] = mean(is_inlier_pixel)
    f = config.robustnerf_smoothed_filter_size
    counts = torch.nn.functional.conv2d(is_inlier_pixel.permute(0, 3, 1, 2),
                                        torch.ones(1, 1, f, f, device=errors.device), padding=f // 2)
    has_inlier_neighbors = ((counts / f32(float(f * f))) >
                            f32(1 - config.robustnerf_smoothed_inlier_quantile)).to(torch.float32)
    has_inlier_neighbors = has_inlier_neighbors.permute(0, 2, 3, 1)
    stats['has_inlier_neighbors'] = mean(has_inlier_neighbors)
    is_inlier_pixel = ((has_inlier_neighbors + is_inlier_pixel) > 1e-3).to(torch.float32)
    p, inner = config.patch_size, config.robustnerf_inner_patch_size
    lower = (p - inner) // 2
    inner_mask = torch.zeros(1, p, p, 1, device=errors.device)
    inner_mask[:, lower:lower + inner, lower:lower + inner] = 1.0
    patch_frac = is_inlier_pixel.sum(dim=(1, 2), keepdim=True) / f32(float(p * p))
    is_inlier_patch = (patch_frac > f32(1 - config.robustnerf_inner_patch_inlier_quantile)).to(torch.float32)
    is_inlier_patch = is_inlier_patch * inner_mask
    stats['is_inlier_patch'] = mean(is_inlier_patch)
    mask = ((is_inlier_patch + is_inlier_pixel) > 1e-3).to(torch.float32)
  stats['mask'] = mean(mask)
  return mask, stats


def compute_data_loss(batch_rgb, renderings, lossmult, config, loss_threshold=1.0):
  """train_utils.py:72-136 for data_loss_type 'robustnerf' (any other type: o_train.compute_data_loss).
  Rays are patch-major [n * p * p]; the last level's mask statistics are the ones returned (stats.update)."""
  if config.data_loss_type != 'robustnerf':
    return o_train.compute_data_loss(batch_rgb, renderings, lossmult, config)
  data_losses, mses, robust_stats = [], [], {}
  lossmult = lossmult.expand_as(batch_rgb[..., :3])
  if config.disable_multiscale_loss:
    lossmult = torch.ones_like(lossmult)
  p = config.patch_size
  for rendering in renderings:
    resid_sq = (rendering['rgb'] - batch_rgb[..., :3]) ** 2
    denom = lossmult.sum()
    mses.append((lossmult * resid_sq).sum() / denom)
    mask, robust_stats = robustnerf_mask(resid_sq.reshape(-1, p, p, 3), loss_threshold, config)
    data_loss = resid_sq * mask.reshape(resid_sq.shape[:-1] + (1,))      # the mask is a constant for autodiff
    data_losses.append((lossmult * data_loss).sum() / denom)
  data_losses = torch.stack(data_losses)
  loss = (config.data_coarse_loss_mult * data_losses[:-1].sum() +
          config.data_loss_mult * data_losses[-1])
  return loss, dict({'mses': torch.stack(mses)}, **robust_stats)


def train_step(params, opt_state, bundle, bases, rays, batch_rgb, train_frac, rand=None, bf16=False,
               loss_threshold=1.0):
  """o_train.train_step (train_utils.py:239-339) with the robustnerf data loss at `loss_threshold`
  (the loss_threshold argument of train_pstep).  o_train's closure reads its module-level
  compute_data_loss, which is pointed at this one for the duration of the call."""
  plain = o_train.compute_data_loss
  o_train.compute_data_loss = lambda b, r, lm, cfg: compute_data_loss(b, r, lm, cfg, loss_threshold)
  try:
    return o_train.train_step(params, opt_state, bundle, bases, rays, batch_rgb, train_frac, rand=rand, bf16=bf16)
  finally:
    o_train.compute_data_loss = plain
