"""Cost of density normals through the scene contraction on 360.gin.

1. Encode kernel: the tangent form of csrc/encode.cu (feature row + three tangent rows per sample) with and
   without `warp_contract`, on the 360 PropMLP (64 samples) and NerfMLP (32 samples) shapes; CUDA events over
   --launches launches, achieved bytes/s from the rows each launch stores.
2. Train step: 360.gin as shipped against the same config with `{Prop,Nerf}MLP.disable_density_normals = False`
   and the orientation loss on those normals (0.1 / 0.01, target 'normals'), both on CUDA graphs, timed in
   alternation in one process (median of --reps runs of --steps steps, with the spread), with launches per step
   and the peak device memory of each arm.  The tangent buffers grow with the rays; the batch of both arms is the
   largest multiple of 1024 rays (at most --rays) at which both arms, resident side by side during the
   alternation, fit in 90 % of the free device memory: the shipped step's measured peak per ray for each arm plus
   the normals' tangent buffers counted from the layer shapes.  The same count gives the footprint of a normals
   step alone at --rays.
Also reads the card name and power limit.

    python tools/contract_normals_bench.py [--steps 20] [--rays 16384]
"""
import argparse
import gc
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from multinerf_b200 import configs, geopoly, lib, models, ops, train_utils, utils  # noqa: E402
from prop_normals_bench import GIB, extra_work, run, smi  # noqa: E402


def batch(seed, B):
  """Origins in the unit cube, random directions, near 0.2, far 1e6 (an unbounded capture)."""
  rng = np.random.default_rng(seed)
  f = np.float32
  o = rng.uniform(-1, 1, (B, 3))
  d = rng.normal(size=(B, 3))
  d /= np.linalg.norm(d, axis=-1, keepdims=True)
  v = d.astype(f)
  d = (d * rng.uniform(0.8, 1.2, (B, 1))).astype(f)
  rays = utils.Rays(origins=o.astype(f), directions=d, viewdirs=v, radii=rng.uniform(5e-4, 1e-3, (B, 1)).astype(f),
                    imageplane=np.zeros((B, 2), f), lossmult=np.ones((B, 1), f), near=np.full((B, 1), 0.2, f),
                    far=np.full((B, 1), 1e6, f), cam_idx=np.zeros((B, 1), np.int32))
  return rays, rng.uniform(0, 1, (B, 3)).astype(f)


def bundle_of(normals, B):
  here = os.path.join(ROOT, 'tests', 'golden', 'configs')
  bundle = configs.load_config([os.path.join(here, '360.gin')], search_paths=[here])
  bundle.config.batch_size = B
  if normals:
    bundle.prop_mlp.disable_density_normals = bundle.nerf_mlp.disable_density_normals = False
    bundle.config.orientation_loss_mult, bundle.config.orientation_coarse_loss_mult = 0.1, 0.01
    bundle.config.orientation_loss_target = 'normals'
  return bundle


def make(name, normals, B, batches, warmup):
  torch.cuda.synchronize()
  before = torch.cuda.memory_allocated()
  torch.cuda.reset_peak_memory_stats()
  bundle = bundle_of(normals, B)
  model, variables = models.construct_model(0, batches[0][0], bundle)
  step = train_utils.create_train_step(model, bundle.config, use_graph=True)
  arm = dict(name=name, step=step, state=train_utils.TrainState(variables),
             gen=torch.Generator(device='cuda').manual_seed(1), n=0, model=model)
  run(arm, batches, warmup)
  torch.cuda.synchronize()
  arm['peak_gib'] = (torch.cuda.max_memory_allocated() - before) / GIB
  return arm


def encode_times(B, launches):
  """Tangent-form encode with / without the contraction on the 360 MLP shapes (icosahedron 2, degrees 0-12)."""
  basis = torch.tensor(geopoly.generate_basis('icosahedron', 2), dtype=torch.float32, device='cuda')
  K, L = basis.shape[0], 12
  F = 2 * K * L
  Fpad = (F + 63) // 64 * 64
  rays, _ = batch(3, B)
  t = {k: torch.tensor(np.asarray(getattr(rays, k))).cuda() for k in ('origins', 'directions', 'radii', 'near', 'far')}
  out = {}
  for mlp, S in (('prop', 64), ('nerf', 32)):
    M = B * S
    sdist = torch.sort(torch.rand(B, S + 1, device='cuda', generator=torch.Generator('cuda').manual_seed(2)), -1)[0]
    feat = torch.empty(M, Fpad, dtype=torch.bfloat16, device='cuda')
    tfeat = torch.empty(3 * M, Fpad, dtype=torch.bfloat16, device='cuda')
    for contract in (False, True):
      def fn():
        ops.encode(sdist, t['origins'], t['directions'], t['radii'][:, 0].contiguous(), t['near'][:, 0].contiguous(),
                   t['far'][:, 0].contiguous(), basis, min_deg=0, max_deg=L, raydist_fn='reciprocal',
                   warp_contract=contract, feat=feat, feat_cols=Fpad, tfeat=tfeat)
      for _ in range(10):
        fn()
      a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      a.record()
      for _ in range(launches):
        fn()
      b.record()
      torch.cuda.synchronize()
      us = a.elapsed_time(b) * 1e3 / launches
      # bytes each launch must move: four bf16 rows of Fpad per sample out, S+1 distances per ray in
      nbytes = 4 * M * Fpad * 2 + B * (S + 1) * 4
      key = f'{mlp}_{"contract" if contract else "plain"}'
      out[key + '_us'] = round(us, 1)
      out[key + '_gbps'] = round(nbytes / (us * 1e3), 1)
    out[f'{mlp}_rows'] = M
    del feat, tfeat
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--warmup', type=int, default=3)
  ap.add_argument('--rays', type=int, default=16384)
  ap.add_argument('--reps', type=int, default=3)
  ap.add_argument('--launches', type=int, default=200)
  ap.add_argument('--encode-rays', type=int, default=8192)
  args = ap.parse_args()
  lib.require_device()
  res = dict(card=torch.cuda.get_device_name(), power_limit_w=smi('power.limit'))
  res['encode'] = dict(rays=args.encode_rays, launches=args.launches, **encode_times(args.encode_rays, args.launches))
  torch.cuda.empty_cache()

  # batch of the normals arm, from the shipped step's measured footprint and the counted tangent buffers
  probe_B = 1024
  probe_batches = [batch(10 + i, probe_B) for i in range(2)]
  probe = make('probe', False, probe_B, probe_batches, 2)
  shipped_per_ray = probe['peak_gib'] * GIB / probe_B
  extra_per_ray = sum(e['tacts_gib'] + e['h_gib'] + e['tfeat_gib']
                      for e in extra_work(probe['model'], probe_B).values()) * GIB / probe_B
  del probe
  gc.collect()
  torch.cuda.synchronize()
  torch.cuda.empty_cache()
  free, total = torch.cuda.mem_get_info()
  fit = int(0.9 * free / (2 * shipped_per_ray + extra_per_ray)) // 1024 * 1024
  B = max(1024, min(args.rays, fit))
  res.update(rays=B, requested_rays=args.rays, free_gib=round(free / GIB, 1), total_gib=round(total / GIB, 1),
             counted_gib_per_1k_rays=dict(shipped=round(shipped_per_ray * 1024 / GIB, 3),
                                          normals_extra=round(extra_per_ray * 1024 / GIB, 3)),
             counted_normals_step_gib_at_requested_rays=round((shipped_per_ray + extra_per_ray) * args.rays / GIB, 1))

  batches = [batch(10 + i, B) for i in range(4)]
  arms = [make('shipped', False, B, batches, args.warmup), make('normals', True, B, batches, args.warmup)]
  times = {arm['name']: [] for arm in arms}
  for _ in range(args.reps):
    for arm in arms:
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      run(arm, batches, args.steps)
      torch.cuda.synchronize()
      times[arm['name']].append((time.perf_counter() - t0) * 1e3 / args.steps)
  stats = run(arms[1], batches, 1).materialize()
  med = {k: float(np.median(v)) for k, v in times.items()}
  res.update(steps=args.steps, shipped_ms=round(med['shipped'], 3), normals_ms=round(med['normals'], 3),
             overhead_pct=round(100.0 * (med['normals'] / med['shipped'] - 1.0), 1),
             runs_ms={k: [round(x, 3) for x in v] for k, v in times.items()},
             spread_ms={k: round(max(v) - min(v), 3) for k, v in times.items()},
             launches={arm['name']: arm['step'].graph_info['launches'] for arm in arms},
             graphs={arm['name']: arm['step'].graph_info['state'] == 2 for arm in arms},
             peak_gib={arm['name']: round(arm['peak_gib'], 2) for arm in arms},
             orientation_loss=stats['losses']['orientation'], extra_work=extra_work(arms[1]['model'], B),
             power_limit_w_after=smi('power.limit'))
  print(json.dumps(res))


if __name__ == '__main__':
  main()
