"""Evaluation and offline rendering around `render_image` (reference: eval.py, render.py).

`evaluate` renders every test image of a dataset from the newest checkpoint, writes the reference's file
set into `<checkpoint_dir>/test_preds` (`color_XXX.png`, `color_cc_XXX.png`, `distance_{mean,median}_XXX.tiff`,
`normals_XXX.png`, `acc_XXX.tiff`, `render_times_<step>.txt`, `metric_<name>_<step>.txt`,
`metric_cc_<name>_<step>.txt`) and returns the per-image metrics.  `render` writes
`<render_dir>/{test_preds,path_renders}_step_<step>/{color,normals,distance_mean,distance_median,acc}_XXX.*`.
One process per GPU: every rank renders its share of each chunk (packed all-gather), rank 0 writes.
"""
import concurrent.futures
import glob
import os
import time

import numpy as np
import torch

from . import checkpoints
from . import image as lib_image
from . import models
from . import raw_utils
from . import ref_utils
from . import train_utils
from . import utils


def _np(x):
  return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _l2_normalize(x, eps=np.finfo(np.float32).eps):
  return x / np.sqrt(np.maximum(np.sum(x ** 2, axis=-1, keepdims=True), eps))


def compute_weighted_mae(weights, normals, normals_gt):
  """Weighted mean angular error in degrees (ref_utils.py:45-50)."""
  one_eps = 1 - np.finfo(np.float32).eps
  cos = np.clip((normals * normals_gt).sum(-1), -one_eps, one_eps)
  return float((weights * np.arccos(cos)).sum() / weights.sum() * 180.0 / np.pi)


def image_metrics(config, postprocess_fn, metric_harness, rgb_gt, *rgbs):
  """One metric dict (psnr, ssim) per image of `rgbs` against `rgb_gt`, all [H, W, 3]: each through
  `postprocess_fn` (RawNeRF's, or the identity), the predictions rounded to 8 bits with Config.eval_quantize_metrics
  (what the saved PNGs hold) and every image cropped by Config.eval_crop_borders."""
  rgbs, rgb_gt = [postprocess_fn(x) for x in rgbs], postprocess_fn(rgb_gt)
  if config.eval_quantize_metrics:
    rgbs = [np.round(x * 255) / 255 for x in rgbs]
  if config.eval_crop_borders > 0:
    c = config.eval_crop_borders
    rgbs, rgb_gt = [x[c:-c, c:-c] for x in rgbs], rgb_gt[c:-c, c:-c]
  return [metric_harness(x, rgb_gt) for x in rgbs]


def evaluate(bundle, dataset, log=print, use_graph=True, summaries=None):
  """eval.py:44-257 for one checkpoint (`eval_only_once` semantics).  Returns (metrics, metrics_cc, step)."""
  config = bundle.config
  world, rank = train_utils._world()
  model, state, _, _, _ = train_utils.setup_model(bundle, 20200823)
  render_eval_pfn = train_utils.create_render_fn(model, use_graph=use_graph)
  metadata = getattr(dataset, 'metadata', None)
  postprocess_fn = metadata['postprocess_fn'] if (config.rawnerf_mode and metadata) else (lambda z: z)
  cc_fun = raw_utils.match_images_affine if config.eval_raw_affine_cc else lib_image.color_correct
  metric_harness = lib_image.MetricHarness()
  out_dir = os.path.join(config.checkpoint_dir, 'path_renders' if config.render_path else 'test_preds')
  path_fn = lambda x: os.path.join(out_dir, x)
  state = checkpoints.restore_checkpoint(config.checkpoint_dir, state, model=model)
  step = int(state.step)
  log(f'Evaluating checkpoint at step {step}.')
  if config.eval_save_output and rank == 0:
    os.makedirs(out_dir, exist_ok=True)
  num_eval = min(dataset.size, config.eval_dataset_limit)
  metrics, metrics_cc, render_times = [], [], []
  for idx in range(dataset.size):
    t0 = time.time()
    batch = next(dataset)
    if idx >= num_eval:
      log(f'Skipping image {idx+1}/{dataset.size}')
      continue
    log(f'Evaluating image {idx+1}/{dataset.size}')
    train_frac = state.step / config.max_steps
    rendering = models.render_image(lambda rng_, r: render_eval_pfn(state.params, train_frac, None, r), batch.rays,
                                    None, bundle, verbose=False, world_size=world, rank=rank)
    torch.cuda.synchronize()
    if rank != 0:
      continue
    render_times.append(time.time() - t0)
    log(f'Rendered in {render_times[-1]:0.3f}s')
    rendering = {k: (_np(v) if not isinstance(v, (list, tuple)) else v) for k, v in rendering.items()}
    gt_rgb = np.array(batch.rgb, dtype=np.float64) if batch.rgb is not None else None
    rendering['rgb'] = np.array(rendering['rgb'], dtype=np.float64)
    if not config.render_path:
      t1 = time.time()
      rendering['rgb_cc'] = cc_fun(rendering['rgb'], gt_rgb)
      log(f'Color corrected in {(time.time() - t1):0.3f}s')
      metric, metric_cc = image_metrics(config, postprocess_fn, metric_harness, gt_rgb, rendering['rgb'],
                                        rendering['rgb_cc'])
      if config.compute_disp_metrics and batch.disps is not None:
        for tag in ['mean', 'median']:
          key = f'distance_{tag}'
          if key in rendering:
            metric[f'disparity_{tag}_mse'] = float(((1 / (1 + rendering[key]) - _np(batch.disps)) ** 2).mean())
      if config.compute_normal_metrics and batch.normals is not None:
        weights = rendering['acc'] * _np(batch.alphas)
        gt_n = _l2_normalize(_np(batch.normals))
        for key, val in rendering.items():
          if key.startswith('normals') and val is not None and not isinstance(val, (list, tuple)):
            metric[key + '_mae'] = compute_weighted_mae(weights, _l2_normalize(val), gt_n)
      for m, v in metric.items():
        log(f'{m:30s} = {v:.4f}')
      metrics.append(metric)
      metrics_cc.append(metric_cc)
    if config.eval_save_output and config.eval_render_interval > 0 and idx % config.eval_render_interval == 0:
      utils.save_img_u8(postprocess_fn(rendering['rgb']), path_fn(f'color_{idx:03d}.png'))
      if 'rgb_cc' in rendering:
        utils.save_img_u8(postprocess_fn(rendering['rgb_cc']), path_fn(f'color_cc_{idx:03d}.png'))
      for key in ['distance_mean', 'distance_median']:
        if key in rendering:
          utils.save_img_f32(rendering[key], path_fn(f'{key}_{idx:03d}.tiff'))
      if 'normals' in rendering:
        utils.save_img_u8(rendering['normals'] / 2. + 0.5, path_fn(f'normals_{idx:03d}.png'))
      utils.save_img_f32(rendering['acc'], path_fn(f'acc_{idx:03d}.tiff'))
  if rank == 0 and summaries is not None and metrics:
    summaries.scalar('eval_median_render_time', np.median(render_times), step)
    for tag, ms in (('eval_metrics/', metrics), ('eval_metrics_cc/', metrics_cc)):
      for name in ms[0]:
        scores = [m[name] for m in ms]
        summaries.scalar(tag + name, np.mean(scores), step)
        summaries.histogram(tag + 'perimage_' + name, scores, step)
  if config.eval_save_output and not config.render_path and rank == 0 and metrics:
    with open(path_fn(f'render_times_{step}.txt'), 'w') as f:
      f.write(' '.join(str(r) for r in render_times))
    for name in metrics[0]:
      with open(path_fn(f'metric_{name}_{step}.txt'), 'w') as f:
        f.write(' '.join(str(m[name]) for m in metrics))
    for name in metrics_cc[0]:
      with open(path_fn(f'metric_cc_{name}_{step}.txt'), 'w') as f:
        f.write(' '.join(str(m[name]) for m in metrics_cc))
  return metrics, metrics_cc, step


def render(bundle, dataset, log=print, use_graph=True):
  """render.py:99-198 without the video muxing (mediapy / ffmpeg are not in this image): per test (or path)
  camera, `color`, `normals`, `distance_mean`, `distance_median` and `acc` files.  Returns the output directory."""
  config = bundle.config
  world, rank = train_utils._world()
  model, state, _, _, _ = train_utils.setup_model(bundle, 20200823)
  render_eval_pfn = train_utils.create_render_fn(model, use_graph=use_graph)
  metadata = getattr(dataset, 'metadata', None)
  postprocess_fn = metadata['postprocess_fn'] if (config.rawnerf_mode and metadata) else (lambda z: z)
  state = checkpoints.restore_checkpoint(config.checkpoint_dir, state, model=model)
  step = int(state.step)
  log(f'Rendering checkpoint at step {step}.')
  out_name = ('path_renders' if config.render_path else 'test_preds') + f'_step_{step}'
  base_dir = config.render_dir if config.render_dir is not None else os.path.join(config.checkpoint_dir, 'render')
  out_dir = os.path.join(base_dir, out_name)
  if rank == 0:
    os.makedirs(out_dir, exist_ok=True)
  path_fn = lambda x: os.path.join(out_dir, x)
  zpad = max(3, len(str(dataset.size - 1)))
  idx_to_str = lambda i: str(i).zfill(zpad)
  pool = concurrent.futures.ThreadPoolExecutor(max_workers=4) if config.render_save_async else None
  futures = []

  def save_fn(fn, *args):
    if pool is not None:
      futures.append(pool.submit(fn, *args))
    else:
      fn(*args)
  for idx in range(dataset.size):
    if idx % config.render_num_jobs != config.render_job_id:
      continue
    s = idx_to_str(idx)
    if os.path.exists(path_fn(f'color_{s}.png')) and \
       os.path.exists(path_fn(f'color_{idx_to_str(idx + config.render_num_jobs)}.png')):
      log(f'Image {idx}/{dataset.size} already exists, skipping')
      continue
    log(f'Evaluating image {idx+1}/{dataset.size}')
    t0 = time.time()
    rays = dataset.generate_ray_batch(idx).rays
    rendering = models.render_image(lambda rng_, r: render_eval_pfn(state.params, 1., None, r), rays, None, bundle,
                                    verbose=False, world_size=world, rank=rank)
    torch.cuda.synchronize()
    log(f'Rendered in {(time.time() - t0):0.3f}s')
    if rank != 0:
      continue
    rendering = {k: _np(v) for k, v in rendering.items() if not isinstance(v, (list, tuple))}
    save_fn(utils.save_img_u8, postprocess_fn(rendering['rgb']), path_fn(f'color_{s}.png'))
    if 'normals' in rendering:
      save_fn(utils.save_img_u8, rendering['normals'] / 2. + 0.5, path_fn(f'normals_{s}.png'))
    save_fn(utils.save_img_f32, rendering['distance_mean'], path_fn(f'distance_mean_{s}.tiff'))
    save_fn(utils.save_img_f32, rendering['distance_median'], path_fn(f'distance_median_{s}.tiff'))
    save_fn(utils.save_img_f32, rendering['acc'], path_fn(f'acc_{s}.tiff'))
  if pool is not None:
    pool.shutdown(wait=True)
    for fu in futures:
      fu.result()                       # surface exceptions of the writer threads
  if rank == 0:
    n = len(glob.glob(path_fn('acc_*.tiff')))
    log(f'{n}/{dataset.size} frames written to {out_dir}')
  return out_dir
