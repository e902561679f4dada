"""Per-level PSNR of one train step, CUDA path vs the CPU oracle, on identical rays, weights and random draws
(BASELINE.json: "PSNR parity"; SURVEY.md 8d asks for the agreement of train.py's printed PSNRs).  Runs the three
BASELINE model families at their stated widths (tests/model_parity.py `fullwidth_case`) and prints what is measured.

  python tools/psnr_parity.py            # needs an H100
"""
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from model_parity import fullwidth_case, train_step              # noqa: E402  (test infrastructure: the checker)


def main():
  from multinerf_b200 import lib, models
  lib.require_device()
  print('# per-level PSNR = -10 log10(mse) of one train step (image.py:28-30, train_utils.py:337-338): CUDA path vs oracle')
  print('# (oracle = torch-CPU restatement with bf16-rounded weights and layer inputs, fp32 accumulate), identical rays,')
  print('# weights, jitter and noise draws; 360.gin on 256 rays, blender_refnerf.gin and llff_raw.gin on 128 rays')
  for which in ('360', 'refnerf', 'raw'):
    bundle, rays, target, rand, B, S = fullwidth_case(which)
    model, variables = models.construct_model(41, rays, bundle)
    if which == 'raw':
      tree = model.export_flax()
      tree['exposure_scaling_offsets']['embedding'] = \
          np.random.default_rng(6).normal(size=(1000, 3)).astype(np.float32) * 0.1
      variables = model.init(flax_params=tree)
    t = train_step(model, variables, bundle, rays, target, rand, 0.5)
    stats, stats_o = t.stats, t.stats_o
    mo = stats_o['mses'].detach().double()
    mk = stats['mses'].double()
    po = -10.0 / math.log(10.0) * torch.log(mo)
    pk = -10.0 / math.log(10.0) * torch.log(mk)
    print(f'{which:8s} loss: cuda {stats["loss"]:.6f}  oracle {float(stats_o["loss"]):.6f}')
    for i in range(len(mo)):
      print(f'{which:8s} level {i}: psnr cuda {float(pk[i]):8.4f}  oracle {float(po[i]):8.4f}  '
            f'|d| = {abs(float(pk[i] - po[i])):.4f} dB   (mse rel. diff {abs(float(mk[i] / mo[i] - 1)):.2e})')


if __name__ == '__main__':
  main()
