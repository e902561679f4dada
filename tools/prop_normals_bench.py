"""Cost of density normals on every level of blender_256.gin: the train step at 16384 rays as shipped against
the same config with `{Prop,Nerf}MLP.disable_density_normals = False` and the orientation loss on those normals
(orientation_loss_mult 0.1, orientation_coarse_loss_mult 0.01, target 'normals'), both captured as CUDA graphs
and timed in alternation in one process (median of 3 runs of --steps steps each, with the spread).  Also
reports the kernel launches of each step, the peak device memory each arm adds, the times of the colourless
normals stage alone (mnrf_normals_fwd/bwd, CUDA events over many launches on one proposal level), the extra
tensor-core work and buffers of the normals arm computed from the layer shapes, the card name and its power
limit.

    python tools/prop_normals_bench.py [--steps 20] [--rays 16384]
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


def bundle_of(normals, B):
  here = os.path.join(ROOT, 'tests', 'golden', 'configs')
  bundle = configs.load_config([os.path.join(here, 'blender_256.gin')], search_paths=[here])
  bundle.config.batch_size = B
  if normals:
    bundle.prop_mlp.disable_density_normals = bundle.nerf_mlp.disable_density_normals = False
    bundle.config.orientation_loss_mult, bundle.config.orientation_coarse_loss_mult = 0.1, 0.01
    bundle.config.orientation_loss_target = 'normals'
  return bundle


def make(name, normals, B, rays, batches, warmup):
  torch.cuda.synchronize()
  before = torch.cuda.memory_allocated()
  torch.cuda.reset_peak_memory_stats()
  bundle = bundle_of(normals, B)
  model, variables = models.construct_model(0, rays, bundle)
  step = train_utils.create_train_step(model, bundle.config, use_graph=True)
  arm = dict(name=name, step=step, state=train_utils.TrainState(variables),
             gen=torch.Generator(device='cuda').manual_seed(1), n=0, model=model)
  run(arm, batches, warmup)
  torch.cuda.synchronize()
  arm['peak_gib'] = (torch.cuda.max_memory_allocated() - before) / GIB
  return arm


def run(arm, batches, steps):
  for i in range(steps):
    rays, rgb = batches[(arm['n'] + i) % len(batches)]
    arm['state'], stats, arm['gen'] = arm['step'](arm['gen'], arm['state'], utils.Batch(rays=rays, rgb=rgb), None,
                                                  min(1.0, arm['n'] / 100000))
  arm['n'] += steps
  return stats


def extra_work(model, B):
  """Tensor-core FLOP and buffer bytes the density normals add per step, from the layer shapes: the tangent
  forward (3 streams of the level's rows through every trunk layer), its weight gradient and its input gradient
  (every layer but the first), and the tangent activations / input features / adjoint scratch of each level."""
  m = model.mcfg
  out = {}
  for i in range(m.num_levels):
    is_prop = i < m.num_levels - 1
    mname = 'PropMLP_0' if (is_prop and not m.single_mlp) else 'NerfMLP_0'
    plan = model.plans[mname]
    W = plan.cfg.net_width
    R = 3 * B * (m.num_prop_samples if is_prop else m.num_nerf_samples)
    trunk = plan.by_role('trunk')
    fwd = sum(2.0 * R * sp.in_pad * W for sp in trunk)
    dgrad = sum(2.0 * R * W * W for sp in trunk[1:])
    tacts = sum(R * (W + plan.Fpad if j in plan.concat_after else W) * 2 for j in range(len(trunk)))
    e = out.setdefault(mname, dict(tangent_fwd_tflop=0.0, tangent_wgrad_tflop=0.0, tangent_dgrad_tflop=0.0,
                                   tacts_gib=0.0, h_gib=0.0, tfeat_gib=0.0, rows=0))
    e['tangent_fwd_tflop'] += fwd / 1e12
    e['tangent_wgrad_tflop'] += fwd / 1e12
    e['tangent_dgrad_tflop'] += dgrad / 1e12
    e['tacts_gib'] += tacts / GIB
    e['h_gib'] += 2 * R * W * 2 / GIB
    e['tfeat_gib'] += (0 if plan.concat_after else R * plan.Fpad * 2) / GIB
    e['rows'] += R
  for e in out.values():
    e['total_tflop'] = e['tangent_fwd_tflop'] + e['tangent_wgrad_tflop'] + e['tangent_dgrad_tflop']
    for k in list(e):
      if isinstance(e[k], float):
        e[k] = round(e[k], 3)
  return out


def mlp_tflop(model, B):
  """Tensor-core FLOP of the PropMLP's own trunk per step (forward, weight gradient, input gradient)."""
  m = model.mcfg
  plan = model.plans['PropMLP_0']
  W = plan.cfg.net_width
  R = B * m.num_prop_samples * (m.num_levels - 1)
  trunk = plan.by_role('trunk')
  fwd = sum(2.0 * R * sp.in_pad * W for sp in trunk)
  return round((2 * fwd + sum(2.0 * R * W * W for sp in trunk[1:])) / 1e12, 3)


def stage_times(B, S, launches=100):
  """Colourless normals stage on one proposal level (density normals, orientation loss on them), alone."""
  M = B * S
  rng = torch.Generator(device='cuda').manual_seed(5)
  rgd = torch.randn(3, M, device='cuda', generator=rng)
  v = torch.nn.functional.normalize(torch.randn(B, 3, device='cuda', generator=rng), dim=-1).contiguous()
  w = torch.rand(B, S, device='cuda', generator=rng)
  d_raw = torch.randn(B, S, device='cuda', generator=rng)
  normals, edw, d_rgd = torch.empty(M, 3, device='cuda'), torch.empty(B, S, device='cuda'), torch.empty_like(rgd)
  row = torch.zeros(8, device='cuda')
  om = 0.01 / B
  fns = {'normals_fwd_us': lambda: ops.normals_fwd(M, S, None, rgd, v, None, normals, om, 0.0, False, edw),
         'normals_bwd_us': lambda: ops.normals_bwd(M, S, None, rgd, v, w, om, 0.0, False, d_raw, None, d_rgd,
                                                   stats=row)}
  out = {}
  for name, fn in fns.items():
    for _ in range(10):
      fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
      fn()
    b.record()
    torch.cuda.synchronize()
    out[name] = round(a.elapsed_time(b) * 1e3 / launches, 2)
  # bytes each launch must move: fwd reads rgd, writes normals and extra_dw; bwd reads rgd, weights, writes d_rgd
  out['normals_fwd_gbps'] = round((12 + 12 + 4) * M / (out['normals_fwd_us'] * 1e3), 1)
  out['normals_bwd_gbps'] = round((12 + 4 + 12) * M / (out['normals_bwd_us'] * 1e3), 1)
  out['stage_rows'] = M
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
  arms = [make('shipped', False, B, batches[0][0], batches, args.warmup),
          make('normals', True, B, batches[0][0], batches, args.warmup)]
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
  model = arms[1]['model']
  res = dict(card=torch.cuda.get_device_name(), power_limit_w=smi('power.limit'), rays=B, steps=args.steps,
             shipped_ms=round(med['shipped'], 3), normals_ms=round(med['normals'], 3),
             overhead_pct=round(100.0 * (med['normals'] / med['shipped'] - 1.0), 1),
             runs_ms={k: [round(x, 3) for x in v] for k, v in times.items()},
             spread_ms={k: round(max(v) - min(v), 3) for k, v in times.items()},
             launches={arm['name']: arm['step'].graph_info['launches'] for arm in arms},
             graphs={arm['name']: arm['step'].graph_info['state'] == 2 for arm in arms},
             peak_gib={arm['name']: round(arm['peak_gib'], 2) for arm in arms},
             orientation_loss=stats['losses']['orientation'],
             prop_mlp_tflop=mlp_tflop(model, B), extra_work=extra_work(model, B),
             **stage_times(B, model.mcfg.num_prop_samples))
  print(json.dumps(res))


if __name__ == '__main__':
  main()
