"""Cost of the RobustNeRF loss on the train step: configs/360_robustnerf.gin at 16384 rays (64 patches of
16 x 16) against the same config with data_loss_type='mse', both captured as CUDA graphs and timed in
alternation in one process (median of 3 runs of --steps steps each).  Also reports the kernel launches of
each step and the times of the mask and quantile kernels alone (CUDA events over many launches), with the
card name, its power limit and the median SM clock sampled during the timed runs.

    python tools/robustnerf_bench.py [--steps 20] [--rays 16384]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from multinerf_b200 import configs, lib, models, ops, train_utils, utils  # noqa: E402


def smi(query):
  try:
    out = subprocess.run(['nvidia-smi', f'--query-gpu={query}', '--format=csv,noheader,nounits', '-i',
                          str(torch.cuda.current_device())], capture_output=True, text=True, timeout=10)
    return out.stdout.strip()
  except Exception:  # pylint: disable=broad-except
    return ''


def batch(seed, B):
  rng = np.random.default_rng(seed)
  f = np.float32
  o = rng.uniform(-1, 1, (B, 3)).astype(f)
  d = rng.normal(size=(B, 3))
  d /= np.linalg.norm(d, axis=-1, keepdims=True)
  v = d.astype(f)
  d = (d * rng.uniform(0.8, 1.2, (B, 1))).astype(f)
  rays = utils.Rays(origins=o, directions=d, viewdirs=v, radii=rng.uniform(5e-4, 1e-3, (B, 1)).astype(f),
                    imageplane=np.zeros((B, 2), f), lossmult=np.ones((B, 1), f), near=np.full((B, 1), 0.2, f),
                    far=np.full((B, 1), 1e6, f), cam_idx=np.zeros((B, 1), np.int32))
  return rays, rng.uniform(0, 1, (B, 3)).astype(f)


def make(loss, B, rays):
  here = os.path.join(ROOT, 'tests', 'golden', 'configs')
  bundle = configs.load_config([os.path.join(here, '360_robustnerf.gin')], search_paths=[here])
  bundle.config.data_loss_type = loss
  bundle.config.batch_size = B
  model, variables = models.construct_model(0, rays, bundle)
  step = train_utils.create_train_step(model, bundle.config, use_graph=True)
  return dict(loss=loss, step=step, state=train_utils.TrainState(variables), thr=1.0,
              robust=loss == 'robustnerf', gen=torch.Generator(device='cuda').manual_seed(1), n=0)


def run(arm, batches, steps, max_steps=100000):
  for i in range(steps):
    rays, rgb = batches[(arm['n'] + i) % len(batches)]
    arm['state'], stats, arm['gen'] = arm['step'](arm['gen'], arm['state'], utils.Batch(rays=rays, rgb=rgb), None,
                                                  min(1.0, arm['n'] / max_steps), arm['thr'])
    if arm['robust']:
      arm['thr'] = stats.device_loss_threshold()
  arm['n'] += steps
  return stats


def kernel_times(B, p, launches=200):
  rng = np.random.default_rng(3)
  rgb = torch.tensor(rng.uniform(0, 1, (B, 3)).astype(np.float32), device='cuda')
  tgt = torch.tensor(rng.uniform(0, 1, (B, 3)).astype(np.float32), device='cuda')
  thr = torch.tensor([0.05], device='cuda')
  row = torch.zeros(8, device='cuda')
  counts = torch.zeros(5, dtype=torch.int32, device='cuda')
  desc = ops.robust_desc(B, patch_size=p, inner_patch_size=8, filter_size=3, smoothed_inlier_quantile=0.5,
                         inner_patch_inlier_quantile=0.5, enable=True)
  mask, err = ops.robust_mask(rgb, tgt, thr, desc, counts=counts, stats=row)
  out = {}
  for name, fn in (('mask_us', lambda: ops.robust_mask(rgb, tgt, thr, desc, mask=mask, error=err, counts=counts,
                                                       stats=row)),
                   ('quantile_us', lambda: ops.quantile(err, 0.8, out=row[0:1]))):
    for _ in range(10):
      fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
      fn()
    b.record()
    torch.cuda.synchronize()
    out[name] = a.elapsed_time(b) * 1e3 / launches
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--warmup', type=int, default=3)
  ap.add_argument('--rays', type=int, default=16384)
  ap.add_argument('--reps', type=int, default=3)
  args = ap.parse_args()
  lib.require_device()
  B = args.rays
  batches = [batch(10 + i, B) for i in range(4)]
  arms = [make('mse', B, batches[0][0]), make('robustnerf', B, batches[0][0])]
  for arm in arms:
    run(arm, batches, args.warmup)
  torch.cuda.synchronize()
  times = {arm['loss']: [] for arm in arms}
  clocks = []
  for _ in range(args.reps):
    for arm in arms:
      t0 = time.perf_counter()
      run(arm, batches, args.steps)
      c = smi('clocks.sm')
      torch.cuda.synchronize()
      times[arm['loss']].append((time.perf_counter() - t0) * 1e3 / args.steps)
      if c:
        clocks.append(float(c))
  stats = run(arms[1], batches, 1).materialize()
  med = {k: float(np.median(v)) for k, v in times.items()}
  res = dict(card=torch.cuda.get_device_name(), power_limit_w=smi('power.limit'),
             median_sm_clock_mhz=float(np.median(clocks)) if clocks else None, rays=B, steps=args.steps,
             mse_ms=med['mse'], robustnerf_ms=med['robustnerf'],
             overhead_pct=100.0 * (med['robustnerf'] / med['mse'] - 1.0),
             runs_ms={k: [round(x, 3) for x in v] for k, v in times.items()},
             launches={arm['loss']: arm['step'].graph_info['launches'] for arm in arms},
             graphs={arm['loss']: arm['step'].graph_info['state'] == 2 for arm in arms},
             mask_mean=stats['mask'], loss_threshold=stats['loss_threshold'],
             **kernel_times(B, 16))
  print(json.dumps(res))


if __name__ == '__main__':
  main()
