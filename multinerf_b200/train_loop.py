"""The reference's training loop around `train_pstep` (train.py:66-223), for any iterable of
utils.Batch: same step/`train_frac` bookkeeping, the same summary line every `print_every` steps
(`loss`, `psnr`, `lr`, each `losses/*` term, `r/s` = batch_size * steps/s), checkpoints at step 1,
every `checkpoint_every` and on exit, resume from the newest checkpoint.

`SyntheticScene` is a procedural dataset (a shaded sphere over a gradient background seen from
cameras on a ring) used by the tests and `tools/train_synthetic.py`: the reference's loaders need
scene files that are not in this container (SURVEY.md section 8f row 4).
"""
import gc
import math
import os
import time

import numpy as np
import torch

from . import camera_utils
from . import checkpoints
from . import train_utils
from . import utils


class SyntheticScene:
  """Infinite iterator of utils.Batch for a procedurally defined scene.

  rays: utils.Pixels when `cast_rays_in_train_step` (the cameras are in `.cameras`), else utils.Rays
  generated on the device by camera_utils.cast_ray_batch; rgb: [B, 3] analytic colours.  With
  `config.patch_size` p > 1 a batch is B // p^2 whole p x p patches, rays in [patch, y, x] order, each patch
  from one camera (as Dataset._next_train draws them)."""

  def __init__(self, config, n_cameras=24, width=96, height=72, focal=90.0, radius=3.0, seed=0,
               device='cuda', rank=0, world=1):
    self.config = config
    self.width, self.height = width, height
    self.rng = np.random.default_rng(seed + 7919 * rank)
    self.batch = config.batch_size // world
    self.device = device
    self.camtype = camera_utils.ProjectionType.PERSPECTIVE
    self.size = n_cameras
    self.metadata = None
    p2c = camera_utils.get_pixtocam(focal, width, height)
    poses = []
    for i in range(n_cameras):
      a = 2 * math.pi * i / n_cameras
      eye = np.array([radius * math.cos(a), radius * math.sin(a), 0.6 * math.sin(2 * a)])
      z = eye / np.linalg.norm(eye)                      # camera looks down -z at the origin
      x = np.cross(np.array([0.0, 0.0, 1.0]), z)
      x /= np.linalg.norm(x)
      y = np.cross(z, x)
      poses.append(np.concatenate([np.stack([x, y, z], 1), eye[:, None]], 1))
    self.cameras = (np.broadcast_to(p2c, (n_cameras, 3, 3)).copy(), np.stack(poses), None, None)
    self._dev_cameras = (torch.tensor(self.cameras[0], dtype=torch.float32, device=device),
                         torch.tensor(self.cameras[1], dtype=torch.float32, device=device), None, None)

  @staticmethod
  def colour(origins, viewdirs):
    """Analytic radiance: unit-free shaded sphere of radius 0.8 at the origin, else a gradient sky."""
    o, d = origins, viewdirs
    b = (o * d).sum(-1)
    c = (o * o).sum(-1) - 0.64
    disc = b * b - c
    hit = disc > 0
    t = -b - torch.sqrt(disc.clamp(min=0))
    n = torch.nn.functional.normalize(o + t[:, None] * d, dim=-1)
    sphere = 0.5 + 0.5 * n * torch.tensor([1.0, 0.8, 0.6], device=o.device)
    sky = torch.stack([0.15 + 0.1 * d[:, 2], 0.2 + 0.15 * d[:, 2], 0.45 + 0.3 * d[:, 2]], -1)
    return torch.where((hit & (t > 0))[:, None], sphere, sky).clamp(0, 1)

  def pixels(self):
    B = self.batch
    p = max(self.config.patch_size, 1)
    if p > 1:
      return self._patch_pixels(p)
    meta = lambda v: np.full((B, 1), v, np.float32)
    return utils.Pixels(pix_x_int=self.rng.integers(0, self.width, B).astype(np.int32),
                        pix_y_int=self.rng.integers(0, self.height, B).astype(np.int32),
                        lossmult=meta(1.0), near=meta(self.config.near), far=meta(self.config.far),
                        cam_idx=self.rng.integers(0, self.size, (B, 1)).astype(np.int32))

  def _patch_pixels(self, p):
    n = self.batch // (p * p)
    if n < 1:
      raise ValueError(f'Patch size {p}^2 too large for per-process batch size {self.batch}')
    x0 = self.rng.integers(0, self.width - p + 1, (n, 1, 1))
    y0 = self.rng.integers(0, self.height - p + 1, (n, 1, 1))
    cam = self.rng.integers(0, self.size, (n, 1, 1))
    dx, dy = camera_utils.pixel_coordinates(p, p)          # [y, x]
    flat = lambda a: np.ascontiguousarray(np.broadcast_to(a, (n, p, p)).reshape(-1)).astype(np.int32)
    B = n * p * p
    meta = lambda v: np.full((B, 1), v, np.float32)
    return utils.Pixels(pix_x_int=flat(x0 + dx), pix_y_int=flat(y0 + dy), lossmult=meta(1.0),
                        near=meta(self.config.near), far=meta(self.config.far), cam_idx=flat(cam)[:, None])

  def __iter__(self):
    return self

  def __next__(self):
    px = self.pixels()
    rays = camera_utils.cast_ray_batch(self._dev_cameras, px, self.camtype, device=self.device)
    rgb = self.colour(rays.origins, rays.viewdirs)
    return utils.Batch(rays=px if self.config.cast_rays_in_train_step else rays, rgb=rgb)


class SyntheticTestViews:
  """Test split of `SyntheticScene`: one full image (rays [H, W, n] on the device, colours [H, W, 3]) per
  `next()`, cycling over the cameras like Dataset._next_test (datasets.py:519-525)."""

  def __init__(self, scene):
    self.scene, self._idx, self.size, self.metadata = scene, 0, scene.size, None

  def __iter__(self):
    return self

  def __next__(self):
    sc = self.scene
    i, self._idx = self._idx, (self._idx + 1) % sc.size
    xs, ys = camera_utils.pixel_coordinates(sc.width, sc.height)
    one = lambda v: np.full(xs.shape + (1,), v, np.float32)
    px = utils.Pixels(pix_x_int=xs.astype(np.int32), pix_y_int=ys.astype(np.int32), lossmult=one(1.0),
                      near=one(sc.config.near), far=one(sc.config.far), cam_idx=np.full(xs.shape + (1,), i, np.int32))
    rays = camera_utils.cast_ray_batch(sc._dev_cameras, px, sc.camtype, device=sc.device)
    rgb = sc.colour(rays.origins.reshape(-1, 3), rays.viewdirs.reshape(-1, 3)).reshape(sc.height, sc.width, 3)
    return utils.Batch(rays=rays, rgb=rgb.detach().cpu().numpy())


class _Summaries:
  """TensorBoard scalars / histograms / images (train.py:88-96,152-200,226-281) through
  torch.utils.tensorboard when it is importable; otherwise the calls are recorded in memory (`.log`) so
  the loop and the tests do not depend on it."""

  def __init__(self, logdir):
    self.log = []
    self.writer = None
    if logdir:
      try:
        from torch.utils.tensorboard import SummaryWriter
        self.writer = SummaryWriter(logdir)
      except Exception:  # pylint: disable=broad-except
        self.writer = None

  def scalar(self, name, value, step):
    self.log.append(('scalar', name, float(value), int(step)))
    if self.writer:
      self.writer.add_scalar(name, float(value), int(step))

  def histogram(self, name, values, step):
    self.log.append(('histogram', name, len(values), int(step)))
    if self.writer:
      self.writer.add_histogram(name, np.asarray(values, np.float64), int(step))

  def image(self, name, img, step):
    img = np.asarray(img.detach().cpu() if isinstance(img, torch.Tensor) else img, np.float32)
    self.log.append(('image', name, tuple(img.shape), int(step)))
    if self.writer:
      if img.ndim == 2:
        img = img[..., None]
      self.writer.add_image(name, np.clip(np.nan_to_num(img), 0, 1), int(step), dataformats='HWC')

  def text(self, name, text, step):
    self.log.append(('text', name, text, int(step)))
    if self.writer:
      self.writer.add_text(name, text, int(step))

  def flush(self):
    if self.writer:
      self.writer.flush()


TIME_PRECISION = 1000      # integer milliseconds (train.py:40)


def train(bundle, dataset, seed=20200823, log=print, use_graph=False, test_dataset=None, summaries=None):
  """The optimisation loop of train.py:43-290: step / train_frac bookkeeping, the console line and the
  TensorBoard summaries every `print_every` steps (mean, max and histogram of every statistic over the window,
  learning rate, steps/s, rays/s, timed PSNR), checkpoints at step 1 / every `checkpoint_every` / at the end,
  resume from the newest checkpoint, and -- when a `test_dataset` is given -- a test-view render through
  `render_image` every `train_render_every` steps with its metrics and visualisations.
  Returns (model, state, history); history = the summary dicts of the print windows (test metrics are
  appended as dicts with a 'test_step' key)."""
  from . import image as lib_image
  from . import models
  from . import vis
  config = bundle.config
  model, state, render_eval_pfn, _, lr_fn = train_utils.setup_model(bundle, seed, dataset=dataset)
  train_pstep = train_utils.create_train_step(model, config, use_graph=use_graph, dataset=dataset)
  world, rank = train_utils._world()
  if config.batch_size % world != 0:
    raise ValueError('Batch size must be divisible by the number of devices.')                    # train.py:51-52
  num_params = model.num_params()
  if rank == 0:
    log(f'Number of parameters being optimized: {num_params}')
  if getattr(dataset, 'size', 0) > model.num_glo_embeddings and model.num_glo_features > 0:
    raise ValueError(f'Number of glo embeddings {model.num_glo_embeddings} must be at least equal to '
                     f'number of train images {dataset.size}')                      # train.py:74-78
  metadata = getattr(test_dataset, 'metadata', None)
  postprocess_fn = metadata['postprocess_fn'] if (config.rawnerf_mode and metadata) else (lambda z, _=None: z)
  metric_harness = lib_image.MetricHarness()
  if config.checkpoint_dir:
    os.makedirs(config.checkpoint_dir, exist_ok=True)
    state = checkpoints.restore_checkpoint(config.checkpoint_dir, state, model=model)
  init_step = state.step + 1
  if summaries is None:
    summaries = _Summaries(config.checkpoint_dir if rank == 0 else None)
  if rank == 0 and config.rawnerf_mode:
    for name, data in (('train', dataset), ('test', test_dataset)):
      md = getattr(data, 'metadata', None)
      if md:
        for key in ('exposure_idx', 'exposure_values', 'unique_shutters'):
          summaries.text(f'{name}_{key}', str(md[key]), 0)
  cameras = getattr(dataset, 'cameras', None)
  gen = torch.Generator(device=model.device)
  gen.manual_seed(seed + rank)                       # separate random streams per process (train.py:103)
  num_steps = config.early_exit_steps if config.early_exit_steps is not None else config.max_steps
  history, stats_buffer = [], []
  reset_stats, train_start = True, time.time()
  total_time = total_steps = 0
  train_frac = 0.0
  robust = config.data_loss_type == 'robustnerf'
  loss_threshold = 1.0                               # train.py:109; not checkpointed, a resumed run restarts here
  gc.disable()
  try:
    for step, batch in zip(range(init_step, num_steps + 1), dataset):
      if reset_stats:
        stats_buffer, train_start, reset_stats = [], time.time(), False
      learning_rate = lr_fn(step)
      train_frac = float(np.clip((step - 1) / max(1, config.max_steps - 1), 0, 1))
      state, stats, gen = train_pstep(gen, state, batch, cameras, train_frac, loss_threshold)
      if robust and config.enable_robustnerf_loss:
        loss_threshold = stats.device_loss_threshold()   # train.py:128-129, stays on the device
      stats_buffer.append(stats)
      if step % config.gc_every == 0:
        gc.collect()
      if step == init_step or step % config.print_every == 0:
        torch.cuda.synchronize()
        elapsed = time.time() - train_start
        steps_per_sec = len(stats_buffer) / elapsed
        rays_per_sec = config.batch_size * steps_per_sec
        total_time += int(round(TIME_PRECISION * elapsed))
        total_steps += len(stats_buffer)
        approx_total_time = int(round(step * total_time / total_steps))
        mats = [s.materialize() for s in stats_buffer]
        enabled = {'interlevel': config.interlevel_loss_mult > 0, 'distortion': config.distortion_loss_mult > 0,
                   'orientation': config.orientation_coarse_loss_mult > 0 or config.orientation_loss_mult > 0,
                   'predicted_normals': (config.predicted_normal_coarse_loss_mult > 0 or
                                         config.predicted_normal_loss_mult > 0)}      # train_utils.py:283-303
        series = {'loss': [m['loss'] for m in mats], 'psnr': [m['psnr'] for m in mats]}
        for k in mats[0]['losses']:
          if enabled.get(k, True):
            series['losses/' + k] = [m['losses'][k] for m in mats]
        for k in train_utils.ROBUST_STAT_NAMES:
          if k in mats[0]:
            series[k] = [m[k] for m in mats]
        for i in range(len(mats[0]['psnrs'])):           # vector statistics split per level (train.py:160-166)
          series[f'psnrs/{i}'] = [float(m['psnrs'][i]) for m in mats]
          series[f'mses/{i}'] = [float(m['mses'][i]) for m in mats]
        avg = {k: float(np.mean(v)) for k, v in series.items()}
        mx = {k: float(np.max(v)) for k, v in series.items()}
        summary = dict(step=step, lr=learning_rate, steps_per_sec=steps_per_sec, rays_per_sec=rays_per_sec, **avg)
        history.append(summary)
        if rank == 0:
          for k, v in series.items():
            summaries.histogram('train_' + k, v, step)
          for k, v in avg.items():
            summaries.scalar(f'train_avg_{k}', v, step)
          for k, v in mx.items():
            summaries.scalar(f'train_max_{k}', v, step)
          summaries.scalar('train_num_params', num_params, step)
          summaries.scalar('train_learning_rate', learning_rate, step)
          summaries.scalar('train_steps_per_sec', steps_per_sec, step)
          summaries.scalar('train_rays_per_sec', rays_per_sec, step)
          summaries.scalar('train_avg_psnr_timed', avg['psnr'], total_time // TIME_PRECISION)
          summaries.scalar('train_avg_psnr_timed_approx', avg['psnr'], approx_total_time // TIME_PRECISION)
          md = getattr(dataset, 'metadata', None)
          if md is not None and model.learned_exposure_scaling:
            scalings = state.params.seg('exposure_scaling_offsets').view(-1, 3).detach().cpu().numpy()
            for i_s in range(md['unique_shutters'].shape[0]):
              for j_s, value in enumerate(scalings[i_s]):
                summaries.scalar(f'exposure/scaling_{i_s}_{j_s}', value, step)
          precision = int(np.ceil(np.log10(config.max_steps))) + 1
          str_losses = {k[7:11]: (f'{v:0.5f}' if 1e-4 <= v < 10 else f'{v:0.1e}')
                        for k, v in avg.items() if k.startswith('losses/')}
          log(f'{step:{precision}d}/{config.max_steps:d}: loss={avg["loss"]:0.5f}, psnr={avg["psnr"]:6.3f}, '
              f'lr={learning_rate:0.2e} | ' + ', '.join(f'{k}={s}' for k, s in str_losses.items()) +
              f', {rays_per_sec:0.0f} r/s')
        reset_stats = True
      if config.checkpoint_dir and rank == 0 and (step == 1 or step % config.checkpoint_every == 0):
        checkpoints.save_checkpoint(config.checkpoint_dir, state, int(step), keep=100, model=model)
      # test-set evaluation (train.py:225-281): every rank renders its share of each chunk
      if test_dataset is not None and config.train_render_every > 0 and step % config.train_render_every == 0:
        eval_start = time.time()
        test_case = next(test_dataset)
        rendering = models.render_image(
            lambda rng_, r: render_eval_pfn(state.params, train_frac, None, r), test_case.rays, None, bundle,
            verbose=False, world_size=world, rank=rank)
        torch.cuda.synchronize()
        if rank == 0:
          eval_time = time.time() - eval_start
          num_rays = int(np.prod(test_case.rays.directions.shape[:-1]))
          summaries.scalar('test_rays_per_sec', num_rays / eval_time, step)
          log(f'Eval {step}: {eval_time:0.3f}s., {num_rays / eval_time:0.0f} rays/sec')
          rgb = rendering['rgb'].detach().cpu().numpy()
          metric = metric_harness(postprocess_fn(rgb), postprocess_fn(np.asarray(test_case.rgb)))
          for name, val in metric.items():
            if not np.isnan(val):
              log(f'{name} = {val:.4f}')
              summaries.scalar('train_metrics/' + name, val, step)
          history.append(dict(test_step=step, **metric))
          d = config.vis_decimate if config.vis_decimate > 1 else 1
          dec = lambda x: x if (x is None or isinstance(x, (list, tuple))) else x[::d, ::d]
          rend_d = {k: dec(v) for k, v in rendering.items()}
          rays_d = test_case.rays.map(dec)
          vis_suite = vis.visualize_suite(rend_d, rays_d)
          if config.rawnerf_mode and metadata:
            vis_suite['color_raw'] = rend_d['rgb'].detach().cpu().numpy()
            vis_suite['color_auto'] = postprocess_fn(vis_suite['color_raw'], None)
            summaries.image('test_true_auto', postprocess_fn(dec(np.asarray(test_case.rgb)), None), step)
            for p_, x_ in list(metadata['exposure_levels'].items()):
              vis_suite[f'color/{p_}'] = postprocess_fn(vis_suite['color_raw'], x_)
              summaries.image(f'test_true_color/{p_}', postprocess_fn(dec(np.asarray(test_case.rgb)), x_), step)
          summaries.image('test_true_color', dec(np.asarray(test_case.rgb)), step)
          if config.compute_normal_metrics and test_case.normals is not None:
            summaries.image('test_true_normals', dec(np.asarray(test_case.normals)) / 2. + 0.5, step)
          for k, v in vis_suite.items():
            summaries.image('test_output_' + k, v, step)
          summaries.flush()
    if config.checkpoint_dir and rank == 0 and config.max_steps % config.checkpoint_every != 0:
      checkpoints.save_checkpoint(config.checkpoint_dir, state, int(config.max_steps), keep=100, model=model)   # train.py:284-287
  finally:
    gc.enable()
  train.summaries = summaries
  return model, state, history
