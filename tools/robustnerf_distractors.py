"""RobustNeRF against transient distractors on the procedural scene: a third of the training cameras see an
opaque disc of a saturated colour (about 10 % of the image, a random place per camera) that the test views do
not have.  The mini model is trained twice from the same seed on the same patch batches, once with
data_loss_type 'mse' and once with 'robustnerf' (360_robustnerf.gin's loss settings), and the PSNR on clean
test views is reported for both.  For the robust run, the fraction of distractor pixels and of clean pixels
that the final mask drops is measured on fresh training batches with the final model and threshold.

    python tools/robustnerf_distractors.py [--steps 1500] [--batch 4096]
"""
import argparse
import json
import math
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from multinerf_b200 import camera_utils, configs, models, ops, train_loop, train_utils, utils  # noqa: E402

COLOURS = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 0, 1], [1, 1, 0], [0, 1, 1]], np.float32)


class DistractorScene(train_loop.SyntheticScene):
  """SyntheticScene whose cameras i % 3 == 0 see one opaque saturated disc covering ~10 % of the image."""

  def __init__(self, config, seed=0, disc_seed=0, **kw):
    super().__init__(config, seed=seed, **kw)
    drng = np.random.default_rng(1000 + disc_seed)
    r = math.sqrt(0.1 * self.width * self.height / math.pi)
    self.discs = {}
    for i in range(0, self.size, 3):
      cx, cy = drng.uniform(r, self.width - r), drng.uniform(r, self.height - r)
      self.discs[i] = (cx, cy, r, COLOURS[drng.integers(0, len(COLOURS))])
    self.last_distractor = None

  def __next__(self):
    px = self.pixels()
    rays = camera_utils.cast_ray_batch(self._dev_cameras, px, self.camtype, device=self.device)
    rgb = self.colour(rays.origins, rays.viewdirs)
    cam = px.cam_idx[:, 0]
    hit = np.zeros(cam.shape, bool)
    for i, (cx, cy, r, col) in self.discs.items():
      h = (cam == i) & ((px.pix_x_int + 0.5 - cx) ** 2 + (px.pix_y_int + 0.5 - cy) ** 2 < r * r)
      hit |= h
      if h.any():
        idx = torch.as_tensor(np.nonzero(h)[0], device=rgb.device)
        rgb[idx] = torch.as_tensor(col, device=rgb.device)
    self.last_distractor = hit
    return utils.Batch(rays=px if self.config.cast_rays_in_train_step else rays, rgb=rgb)


def bundle(loss, steps, batch):
  b = configs.bundle_360()
  b.model.num_prop_samples, b.model.num_nerf_samples = 32, 16
  b.prop_mlp.net_depth, b.prop_mlp.net_width = 2, 64
  b.nerf_mlp.net_depth, b.nerf_mlp.net_width = 6, 128
  b.nerf_mlp.bottleneck_width, b.nerf_mlp.net_width_viewdirs = 64, 64
  c = b.config
  c.batch_size, c.max_steps, c.print_every = batch, steps, max(1, steps // 5)
  c.lr_init, c.lr_final, c.lr_delay_steps = 5e-3, 5e-4, min(100, steps // 10)
  c.checkpoint_dir = None
  c.patch_size, c.data_loss_type = 16, loss
  c.robustnerf_inlier_quantile, c.enable_robustnerf_loss = 0.8, True      # 360_robustnerf.gin
  return b


def clean_view_psnr(model, state, b, scene, n_views=6):
  render = train_utils.create_render_fn(model)
  views = train_loop.SyntheticTestViews(scene)
  out = []
  for _ in range(n_views):
    case = next(views)
    rend = models.render_image(lambda rng_, r: render(state.params, 1.0, None, r), case.rays, None, b,
                               verbose=False)
    mse = float(((rend['rgb'].detach().cpu() - torch.as_tensor(case.rgb)) ** 2).mean())
    out.append(-10 * math.log10(mse))
  return float(np.mean(out))


def masked_fractions(model, state, b, scene, threshold, n_batches=8):
  c = b.config
  model.bind(state.params)
  drop_d = drop_c = n_d = n_c = 0
  for _ in range(n_batches):
    batch = next(scene)
    dist = torch.as_tensor(scene.last_distractor, device='cuda')
    with torch.no_grad():
      rend, _ = model(None, batch.rays, 1.0, False)
    rgb = rend[-1]['rgb'].reshape(-1, 3).contiguous()
    tgt = batch.rgb.reshape(-1, 3).contiguous().float()
    B = rgb.shape[0]
    desc = ops.robust_desc(B, patch_size=c.patch_size, inner_patch_size=c.robustnerf_inner_patch_size,
                           filter_size=c.robustnerf_smoothed_filter_size,
                           smoothed_inlier_quantile=c.robustnerf_smoothed_inlier_quantile,
                           inner_patch_inlier_quantile=c.robustnerf_inner_patch_inlier_quantile, enable=True)
    mask, _ = ops.robust_mask(rgb, tgt, torch.tensor([threshold], device='cuda'), desc)
    dropped = mask == 0
    drop_d += int((dropped & dist).sum())
    drop_c += int((dropped & ~dist).sum())
    n_d += int(dist.sum())
    n_c += int((~dist).sum())
  return drop_d / max(n_d, 1), drop_c / max(n_c, 1), n_d / max(n_d + n_c, 1)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=1500)
  ap.add_argument('--batch', type=int, default=4096)
  ap.add_argument('--seed', type=int, default=0)
  args = ap.parse_args()
  res = {'steps': args.steps, 'batch': args.batch, 'card': torch.cuda.get_device_name()}
  for loss in ('mse', 'robustnerf'):
    b = bundle(loss, args.steps, args.batch)
    scene = DistractorScene(b.config, seed=args.seed, disc_seed=args.seed)
    model, state, hist = train_loop.train(b, scene, seed=args.seed, log=lambda s: None, use_graph=True)
    res[f'{loss}_test_psnr'] = clean_view_psnr(model, state, b, scene)
    res[f'{loss}_train_psnr'] = hist[-1]['psnr']
    if loss == 'robustnerf':
      thr = hist[-1]['loss_threshold']
      res['final_loss_threshold'] = thr
      res['final_mask_mean'] = hist[-1]['mask']
      fresh = DistractorScene(b.config, seed=args.seed + 1, disc_seed=args.seed)
      fd, fc, share = masked_fractions(model, state, b, fresh, thr)
      res.update(masked_distractor_fraction=fd, masked_clean_fraction=fc, distractor_pixel_share=share)
    print(json.dumps({k: v for k, v in res.items()}), flush=True)


if __name__ == '__main__':
  main()
