"""Cost of the smooth activations (MLP.net_activation = softplus | silu) against ReLU: for each config, the train step
with each activation on both MLPs, captured as CUDA graphs and timed in alternation in one process (median of 3 runs
of --steps steps each, with the spread; each run builds and frees its own model), its kernel launches and the peak
device memory of each arm:

  360.gin              at --rays (16384)           per-layer trunks; the smooth arms store every layer's z
  blender_256.gin      at --rays (16384)           ReLU runs the chained 256-wide trunk, the smooth arms cannot
  blender_refnerf.gin  at --refnerf-rays (4096)    density normals: the smooth arms add the second-order pass

Then, in a separate eager run of blender_refnerf.gin with SiLU, the share of the step spent in the second-order pass
(the recomputed tangent u = t_in W and the act_tangent_bwd kernel), timed by CUDA events around each layer's pass.
Also reports the card name and its power limit.

    python tools/activations_bench.py [--steps 20] [--rays 16384] [--refnerf-rays 4096]
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

from multinerf_b200 import lib, models, train_utils  # noqa: E402
import view_branch_bench as vbb  # noqa: E402
import view_layouts_bench as vlb  # noqa: E402

CONFIGS = ['360.gin', 'blender_256.gin', 'blender_refnerf.gin']
ACTS = ['relu', 'softplus', 'silu']


def bindings(act):
  return [f'NerfMLP.net_activation = @jax.nn.{act}', f'PropMLP.net_activation = @jax.nn.{act}']


def run_config(gin_file, B, steps):
  """Three rounds over the activations; each run builds, captures and frees its arm (three 360.gin arms at 16384
  rays do not fit in 80 GB together)."""
  runs = {act: [] for act in ACTS}
  for _ in range(3):
    for act in ACTS:
      arm = vlb.Arm(act, gin_file, bindings(act), B)
      arm.run(steps)
      runs[act].append(dict(ms=arm.times[0], launches=arm.launches, peak_gib=arm.peak_gib, loss=arm.loss,
                            chained=arm.model._use_chain(arm.model.plans['NerfMLP_0'], B * 64)))
      del arm
      gc.collect()
      torch.cuda.empty_cache()
  out = dict(rays=B, arms={})
  for act, rs in runs.items():
    times = [r['ms'] for r in rs]
    out['arms'][act] = dict(ms_per_step=round(float(np.median(times)), 3), runs_ms=[round(t, 3) for t in times],
                            spread_ms=round(max(times) - min(times), 3), launches_per_step=rs[0]['launches'],
                            peak_gib=round(max(r['peak_gib'] for r in rs), 3), loss=round(rs[0]['loss'], 5),
                            chained=rs[0]['chained'])
  return out


def second_order_share(B, steps):
  """Eager steps of blender_refnerf.gin with SiLU: CUDA-event time of the second-order passes over the step time."""
  arm = vlb.Arm('silu', 'blender_refnerf.gin', bindings('silu'), B)
  eager = train_utils.create_train_step(arm.model, arm.bundle.config, use_graph=False)
  events = []
  orig = models.Model._tangent_second_order

  def timed(self, *a, **kw):
    ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
    ev[0].record()
    orig(self, *a, **kw)
    ev[1].record()
    events.append(ev)
  models.Model._tangent_second_order = timed
  try:
    arm.state, _, _ = eager(arm.gen, arm.state, arm.batches[0], None, 0.5)      # warm-up
    torch.cuda.synchronize()
    events.clear()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(steps):
      arm.state, _, _ = eager(arm.gen, arm.state, arm.batches[i % 4], None, 0.5)
    t1.record()
    torch.cuda.synchronize()
  finally:
    models.Model._tangent_second_order = orig
  step_ms = t0.elapsed_time(t1) / steps
  pass_ms = sum(a.elapsed_time(b) for a, b in events) / steps
  return dict(rays=B, eager_ms_per_step=round(step_ms, 3), second_order_ms_per_step=round(pass_ms, 3),
              passes_per_step=len(events) // steps, share_pct=round(100 * pass_ms / step_ms, 2))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--rays', type=int, default=16384, help='rays per step of 360.gin and blender_256.gin')
  ap.add_argument('--refnerf-rays', type=int, default=4096, help='rays per step of blender_refnerf.gin')
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  lib.require_device()
  torch.cuda.set_device(0)
  res = dict(gpu=vbb.smi('name'), power_limit_w=vbb.smi('power.limit'), steps=args.steps, configs={})
  for gin_file in CONFIGS:
    B = args.refnerf_rays if 'refnerf' in gin_file else args.rays
    res['configs'][gin_file] = run_config(gin_file, B, args.steps)
    gc.collect()
    torch.cuda.empty_cache()
  res['second_order'] = second_order_share(args.refnerf_rays, args.steps)
  line = json.dumps(res)
  print(line)
  if args.out:
    with open(args.out, 'w') as f:
      f.write(line + '\n')


if __name__ == '__main__':
  main()
