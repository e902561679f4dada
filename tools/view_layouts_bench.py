"""Cost of the view-branch layouts: the train step of a shipped config against the same config in one of the
reference's view-branch ablations, both captured as CUDA graphs and timed in alternation in one process (median of 3
runs of --steps steps each, with the spread):

  blender_refnerf.gin as shipped   against   NerfMLP.bottleneck_width = 0   (the view MLP reads [IDE | n.v])
  blender_256.gin as shipped       against   NerfMLP.net_depth_viewdirs = 0 (the rgb head reads [bottleneck | dir enc])

Each pair is built, timed and freed before the next.  Also reports the kernel launches of each step, the peak device
memory of each arm, the multiply-adds per NerfMLP sample computed from the layer table, the card name and its power
limit.

    python tools/view_layouts_bench.py [--steps 20] [--rays 16384] [--refnerf-rays 4096]
"""
import argparse
import gc
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from multinerf_b200 import configs, lib, models, ops, train_utils, utils  # noqa: E402
import view_branch_bench as vbb  # noqa: E402

PAIRS = [('blender_refnerf.gin', 'NerfMLP.bottleneck_width = 0'), ('blender_256.gin', 'NerfMLP.net_depth_viewdirs = 0')]


class Arm:
  """One config captured as a CUDA graph train step (as view_branch_bench.Arm, on a config file plus gin bindings)."""

  def __init__(self, name, gin_file, bindings, B):
    self.name = name
    here = os.path.join(ROOT, 'tests', 'golden', 'configs')
    self.bundle = configs.load_config([os.path.join(here, gin_file)], search_paths=[here], gin_bindings=bindings)
    self.bundle.config.batch_size = B
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    rays, _ = vbb.batch(0, B)
    self.model, variables = models.construct_model(0, rays, self.bundle)
    self.state = train_utils.TrainState(variables)
    self.batches = [utils.Batch(rays=r, rgb=t) for r, t in (vbb.batch(s, B) for s in range(4))]
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
    self.peak_gib = (torch.cuda.max_memory_allocated() - base) / vbb.GIB
    self.times = []

  run = vbb.Arm.run


def run_pair(gin_file, binding, B, steps):
  arms = [Arm('shipped', gin_file, [], B), Arm(binding, gin_file, [binding], B)]
  for _ in range(3):
    for arm in arms:
      arm.run(steps)
  out = dict(rays=B, arms={})
  for arm in arms:
    med = float(np.median(arm.times))
    out['arms'][arm.name] = dict(ms_per_step=round(med, 3), runs_ms=[round(t, 3) for t in arm.times],
                                 rays_per_s=round(B / med * 1e3), launches_per_step=arm.launches,
                                 peak_gib=round(arm.peak_gib, 3), loss=round(arm.loss, 5),
                                 nerf_macs_per_sample=vbb.macs_per_sample(arm.model.plans['NerfMLP_0']))
  a, b = (out['arms'][k]['ms_per_step'] for k in ('shipped', binding))
  out['saving_pct'] = round(100 * (a - b) / a, 2)
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--rays', type=int, default=16384, help='rays per step of the blender_256.gin pair')
  ap.add_argument('--refnerf-rays', type=int, default=4096, help='rays per step of the blender_refnerf.gin pair')
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  lib.require_device()
  torch.cuda.set_device(0)
  res = dict(gpu=vbb.smi('name'), power_limit_w=vbb.smi('power.limit'), steps=args.steps, pairs={})
  for gin_file, binding in PAIRS:
    B = args.refnerf_rays if 'refnerf' in gin_file else args.rays
    res['pairs'][gin_file] = run_pair(gin_file, binding, B, args.steps)
    gc.collect()
    torch.cuda.empty_cache()
  line = json.dumps(res)
  print(line)
  if args.out:
    with open(args.out, 'w') as f:
      f.write(line + '\n')


if __name__ == '__main__':
  main()
