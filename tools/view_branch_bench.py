"""Cost of the colour branch on blender_256.gin: the train step at 16384 rays as shipped against the same config
under `Model.use_viewdirs = False` (view-independent colour: no bottleneck, no view MLP, the rgb head stacked with
the density head), both captured as CUDA graphs and timed in alternation in one process (median of 3 runs of
--steps steps each, with the spread).  Also reports the kernel launches of each step, the peak device memory of
each arm, the multiply-adds per NerfMLP sample computed from the layer table, the card name and its power limit.
Then the chained NerfMLP trunk forward of the view-independent arm alone (one mnrf_mlp_chain launch over the
level's rays x 32 samples), CUDA events over 50 launches, median of 3 alternated runs: with the stacked 4-output
head in its last epilogue, with the density-only head, and with no head, so the cost of each head is visible.

    python tools/view_branch_bench.py [--steps 20] [--rays 16384]
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

GIB = float(1 << 30)


def smi(query):
  try:
    out = subprocess.run(['nvidia-smi', f'--query-gpu={query}', '--format=csv,noheader,nounits', '-i',
                          str(torch.cuda.current_device())], capture_output=True, text=True, timeout=10)
    return out.stdout.strip()
  except Exception:  # pylint: disable=broad-except
    return ''


def batch(seed, B):
  """Cameras on a sphere of radius 4 looking at the origin, as in the Blender scenes (near 2, far 6)."""
  rng = np.random.default_rng(seed)
  f = np.float32
  o = rng.normal(size=(B, 3))
  o = o / np.linalg.norm(o, axis=-1, keepdims=True) * 4.0
  d = -o / 4.0 + rng.normal(size=(B, 3)) * 0.1
  d /= np.linalg.norm(d, axis=-1, keepdims=True)
  v = d.astype(f)
  d = (d * rng.uniform(0.8, 1.2, (B, 1))).astype(f)
  rays = utils.Rays(origins=o.astype(f), directions=d, viewdirs=v, radii=rng.uniform(5e-4, 1e-3, (B, 1)).astype(f),
                    imageplane=np.zeros((B, 2), f), lossmult=np.ones((B, 1), f), near=np.full((B, 1), 2.0, f),
                    far=np.full((B, 1), 6.0, f), cam_idx=np.zeros((B, 1), np.int32))
  return rays, rng.uniform(0, 1, (B, 3)).astype(f)


def bundle_of(view_independent, B):
  here = os.path.join(ROOT, 'tests', 'golden', 'configs')
  bundle = configs.load_config([os.path.join(here, 'blender_256.gin')], search_paths=[here],
                               gin_bindings=['Model.use_viewdirs = False'] if view_independent else [])
  bundle.config.batch_size = B
  return bundle


def macs_per_sample(plan):
  return sum(s.in_dim * s.out_dim for s in plan.specs)


class Arm:
  def __init__(self, name, view_independent, B):
    self.name = name
    self.bundle = bundle_of(view_independent, B)
    assert self.bundle.model.use_viewdirs == (not view_independent)
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    rays, tgt = batch(0, B)
    self.model, variables = models.construct_model(0, rays, self.bundle)
    self.state = train_utils.TrainState(variables)
    self.batches = [utils.Batch(rays=r, rgb=t) for r, t in (batch(s, B) for s in range(4))]
    self.gen = torch.Generator(device='cuda')
    self.gen.manual_seed(0)
    # launches of one eager step (graph replays issue the same kernels in one launch)
    eager = train_utils.create_train_step(self.model, self.bundle.config, use_graph=False)
    n0 = ops.LAUNCHES
    self.state, _, _ = eager(self.gen, self.state, self.batches[0], None, 0.5)
    torch.cuda.synchronize()
    self.launches = ops.LAUNCHES - n0
    self.step = train_utils.create_train_step(self.model, self.bundle.config, use_graph=True)
    for i in range(3):          # capture + warm-up
      self.state, _, _ = self.step(self.gen, self.state, self.batches[i % 4], None, 0.5)
    torch.cuda.synchronize()
    assert self.step.graph_info['state'] == 2, self.step.graph_info
    self.peak_gib = (torch.cuda.max_memory_allocated() - base) / GIB
    self.times = []

  def run(self, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
      self.state, stats, _ = self.step(self.gen, self.state, self.batches[i % 4], None, 0.5)
    torch.cuda.synchronize()
    self.times.append((time.perf_counter() - t0) / steps * 1e3)
    self.loss = float(stats.materialize()['loss'])


def chain_head_times(arm, reps=50):
  """Forward chain of the arm's NerfMLP level with head_n = 4 (as run), 1 and none: ms per launch."""
  model = arm.model
  st = next(s for s in model._levels.values() if s.mname == 'NerfMLP_0')
  mlp = model.mlps['NerfMLP_0']
  d4, _ = model._chain_fwd_desc(st, mlp)
  assert d4.head_n == 4
  d1 = lib.ChainDesc.from_buffer_copy(d4)
  out1 = torch.empty(st.B * st.S, device='cuda')
  d1.head_n, d1.head_w, d1.head_out = 1, mlp.colv_density.data_ptr(), out1.data_ptr()
  d0 = lib.ChainDesc.from_buffer_copy(d4)
  d0.head_n, d0.head_w, d0.head_b, d0.head_out = 0, None, None, None
  descs = {'head_n=4': d4, 'head_n=1': d1, 'no head': d0}
  times = {k: [] for k in descs}
  for _ in range(3):
    for k, d in descs.items():
      ops.mlp_chain((d, 0.0))
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for _ in range(reps):
        ops.mlp_chain((d, 0.0))
      e1.record()
      torch.cuda.synchronize()
      times[k].append(e0.elapsed_time(e1) / reps)
  return {k: dict(ms=round(float(np.median(v)), 4), runs_ms=[round(t, 4) for t in v]) for k, v in times.items()}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--rays', type=int, default=16384)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  lib.require_device()
  torch.cuda.set_device(0)
  arms = [Arm('shipped', False, args.rays), Arm('use_viewdirs=False', True, args.rays)]
  for _ in range(3):
    for arm in arms:
      arm.run(args.steps)
  res = dict(gpu=smi('name'), power_limit_w=smi('power.limit'), rays=args.rays, steps=args.steps, arms={})
  for arm in arms:
    med = float(np.median(arm.times))
    res['arms'][arm.name] = dict(ms_per_step=round(med, 3), runs_ms=[round(t, 3) for t in arm.times],
                                 rays_per_s=round(args.rays / med * 1e3), launches_per_step=arm.launches,
                                 peak_gib=round(arm.peak_gib, 3), loss=round(arm.loss, 5),
                                 nerf_macs_per_sample=macs_per_sample(arm.model.plans['NerfMLP_0']))
  a, b = (res['arms'][k]['ms_per_step'] for k in ('shipped', 'use_viewdirs=False'))
  res['saving_pct'] = round(100 * (a - b) / a, 2)
  res['nerf_chain_forward'] = chain_head_times(arms[1])
  line = json.dumps(res)
  print(line)
  if args.out:
    with open(args.out, 'w') as f:
      f.write(line + '\n')


if __name__ == '__main__':
  main()
