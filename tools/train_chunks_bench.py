"""Train steps in several forward/backward passes (Config.train_chunk_size): step time and peak memory.

Three cases, each a pair of arms captured as CUDA graphs and timed in alternation in one process (median of --reps
runs of --steps steps each, CUDA events), with the peak of torch.cuda.max_memory_allocated over each arm's
own allocations (model, optimizer state, buffers, inputs):
  refnerf      blender_refnerf.gin at 16384 rays in 4096-ray passes, against the one-pass 4096-ray step (x 4 is
               the time the 16384-ray batch would take as four separate steps);
  360_normals  360.gin with density normals through the contraction and the orientation loss (0.1 / 0.01 on
               'normals') at 16384 rays in 8192-ray passes (alone: its one-pass step does not fit in 80 GB);
  360          360.gin as shipped at 16384 rays, one pass against 8192-ray passes: the cost of the passes.
The card name, its power limit and the median SM clock sampled during the timed runs go with the numbers.

    python tools/train_chunks_bench.py [--cases refnerf,360_normals,360] [--steps 10] [--reps 3]
"""
import argparse
import gc
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from multinerf_b200 import configs, lib, models, train_utils, utils  # noqa: E402

CONFIGS = os.path.join(ROOT, 'tests', 'golden', 'configs')


def smi(query):
  try:
    out = subprocess.run(['nvidia-smi', f'--query-gpu={query}', '--format=csv,noheader,nounits', '-i',
                          str(torch.cuda.current_device())], capture_output=True, text=True, timeout=10)
    return out.stdout.strip()
  except Exception:  # pylint: disable=broad-except
    return ''


def batch(seed, B, near, far, sphere):
  """Origins in the unit cube with random directions, or cameras on a sphere of radius 4 looking at the origin."""
  rng = np.random.default_rng(seed)
  f = np.float32
  if sphere:
    o = rng.normal(size=(B, 3))
    o = o / np.linalg.norm(o, axis=-1, keepdims=True) * 4.0
    d = -o / 4.0 + rng.normal(size=(B, 3)) * 0.1
  else:
    o = rng.uniform(-1, 1, (B, 3))
    d = rng.normal(size=(B, 3))
  d /= np.linalg.norm(d, axis=-1, keepdims=True)
  v = d.astype(f)
  d = (d * rng.uniform(0.8, 1.2, (B, 1))).astype(f)
  rays = utils.Rays(origins=o.astype(f), directions=d, viewdirs=v, radii=rng.uniform(5e-4, 1e-3, (B, 1)).astype(f),
                    imageplane=np.zeros((B, 2), f), lossmult=np.ones((B, 1), f), near=np.full((B, 1), near, f),
                    far=np.full((B, 1), far, f), cam_idx=np.zeros((B, 1), np.int32))
  return rays, rng.uniform(0, 1, (B, 3)).astype(f)


def bundle_of(case):
  name = 'blender_refnerf.gin' if case == 'refnerf' else '360.gin'
  b = configs.load_config([os.path.join(CONFIGS, name)], search_paths=[CONFIGS])
  if case == '360_normals':
    b.prop_mlp.disable_density_normals = b.nerf_mlp.disable_density_normals = False
    b.config.orientation_loss_mult, b.config.orientation_coarse_loss_mult = 0.1, 0.01
    b.config.orientation_loss_target = 'normals'
  return b


class Arm:
  def __init__(self, case, label, B, chunk):
    self.label, self.B = label, B
    b = bundle_of(case)
    b.config.batch_size, b.config.train_chunk_size = B, chunk
    near, far, sphere = (2.0, 6.0, True) if case == 'refnerf' else (0.2, 1e6, False)
    self.batches = [batch(10 + i, B, near, far, sphere) for i in range(2)]
    torch.cuda.synchronize()
    gc.collect()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()            # the other arm of the case stays resident
    torch.cuda.reset_peak_memory_stats()
    self.model, variables = models.construct_model(0, self.batches[0][0], b)
    self.step = train_utils.create_train_step(self.model, b.config, use_graph=True)
    self.state = train_utils.TrainState(variables)
    self.gen = torch.Generator(device='cuda').manual_seed(1)
    self.n, self.times, self.stats = 0, [], None
    self.run(3)                                        # eager warm-up, capture, first replay
    torch.cuda.synchronize()
    self.peak_gib = (torch.cuda.max_memory_allocated() - base) / 2**30

  def run(self, steps, timed=False):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(steps):
      rays, rgb = self.batches[(self.n + i) % len(self.batches)]
      self.state, self.stats, self.gen = self.step(self.gen, self.state, utils.Batch(rays=rays, rgb=rgb), None, 0.5)
    b.record()
    self.n += steps
    if timed:
      torch.cuda.synchronize()
      self.times.append(a.elapsed_time(b) / steps)
    else:
      torch.cuda.synchronize()

  def result(self):
    s = self.stats.materialize()
    return dict(rays=self.B, step_ms=float(np.median(self.times)), runs_ms=[round(t, 3) for t in self.times],
                peak_gib=round(self.peak_gib, 2), launches=self.step.graph_info['launches'],
                graph=self.step.graph_info['state'] == 2, loss=s['loss'], finite=bool(np.isfinite(s['loss'])))


ARMS = {
    'refnerf': [('16384_in_4096', 16384, 4096), ('4096_one_pass', 4096, 0)],
    '360_normals': [('16384_in_8192', 16384, 8192)],
    '360': [('16384_one_pass', 16384, 0), ('16384_in_8192', 16384, 8192)],
}


def run_case(case, steps, reps, clocks):
  arms = [Arm(case, label, B, chunk) for label, B, chunk in ARMS[case]]
  for _ in range(reps):
    for arm in arms:                                   # timed runs alternate between the arms
      arm.run(steps, timed=True)
      c = smi('clocks.sm')
      if c:
        clocks.append(float(c))
  out = {arm.label: arm.result() for arm in arms}
  for arm, (_, _, chunk) in zip(arms, ARMS[case]):
    out[arm.label]['chunk'] = chunk
  if case == 'refnerf':
    out['16384_in_4096']['vs_4x_4096_one_pass'] = round(
        out['16384_in_4096']['step_ms'] / (4 * out['4096_one_pass']['step_ms']), 4)
  if case == '360':
    out['16384_in_8192']['vs_one_pass'] = round(out['16384_in_8192']['step_ms'] / out['16384_one_pass']['step_ms'], 4)
  del arms
  gc.collect()
  torch.cuda.empty_cache()
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--cases', default='refnerf,360_normals,360')
  ap.add_argument('--steps', type=int, default=10)
  ap.add_argument('--reps', type=int, default=3)
  args = ap.parse_args()
  lib.require_device()
  clocks = []
  res = dict(card=torch.cuda.get_device_name(), power_limit_w=smi('power.limit'),
             memory_gib=round(torch.cuda.get_device_properties(0).total_memory / 2**30, 1), steps=args.steps,
             reps=args.reps)
  for case in args.cases.split(','):
    res[case] = run_case(case, args.steps, args.reps, clocks)
    print(json.dumps({case: res[case]}), flush=True)
  res['median_sm_clock_mhz'] = float(np.median(clocks)) if clocks else None
  print(json.dumps(res))


if __name__ == '__main__':
  main()
