"""Micro-benchmark of the layer-chained trunk kernel (csrc/chain.cu) against the per-layer GEMMs on the
PropMLP shape of 360.gin (4 x 256, 512 feature columns, M = 16384 rays x 64 samples).

  python tools/chain_bench.py [--m ROWS] [--depth D] [--skip S] [--fpad F] [--iters N] [--only fwd|bwd|layers]
                              [--lib PATH [--lib PATH ...] [--rounds R]]
Prints time per launch, TFLOP/s and the HBM bytes the launch must move (algorithmic), then the card's name, power
limit and SM clock.  `--depth 8` is the NerfMLP trunk of the 256-wide configs: layer 5 takes the features again
(skip connection after layer 4) as streamed k-blocks behind its resident ones.  With `--lib`, each named build of
the library is timed in a process of its own (the library is chosen at import), the builds alternating R times.
A library built with -DMNRF_CHAIN_CLOCKS also gets its clock64() split printed.
"""
import argparse
import ctypes
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from multinerf_b200 import lib as L, ops  # noqa: E402


def timeit(fn, iters):
  for _ in range(3):
    fn()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(iters):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / iters


def card():
  """Name, power limit and SM clock of the card, read right after the timed launches."""
  try:
    q = 'name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active'
    return subprocess.run(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader', '-i', '0'], capture_output=True,
                          text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    return torch.cuda.get_device_name(0)


CLOCK_CLASSES = ('turn wait', 'full-barrier wait', 'wgmma issue + wait', 'epilogue barriers + store wait',
                 'epilogue element loop', 'epilogue stores + head')


def clocks(label):
  """The clock64() split of a measurement build (first thread of consumer warpgroup 1, CTA 0), since the last call."""
  lib = ctypes.CDLL(L.LIB_PATH)
  if not hasattr(lib, 'mnrf_chain_clocks'):
    return
  out = (ctypes.c_ulonglong * len(CLOCK_CLASSES))()
  assert lib.mnrf_chain_clocks(out) == 0
  tot = float(sum(out)) or 1.0
  print(f'  clock64 split, {label}: ' + ', '.join(f'{n} {100 * v / tot:.1f} %' for n, v in zip(CLOCK_CLASSES, out)))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--lib', action='append', default=[])
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--skip', type=int, default=None)
  ap.add_argument('--m', type=int, default=16384 * 64)
  ap.add_argument('--depth', type=int, default=4)
  ap.add_argument('--fpad', type=int, default=512)
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--only', default='all')
  a = ap.parse_args()
  if a.lib:
    args = [sys.executable, os.path.abspath(__file__), '--m', str(a.m), '--depth', str(a.depth), '--fpad', str(a.fpad),
            '--iters', str(a.iters), '--only', a.only] + ([] if a.skip is None else ['--skip', str(a.skip)])
    for r in range(a.rounds):
      for path in a.lib:
        print(f'## round {r}: {path}', flush=True)
        subprocess.run(args, env=dict(os.environ, MNRF_LIB=os.path.abspath(path)), check=True)
    return
  L.require_device()
  M, D, F, W = a.m, a.depth, a.fpad, 256
  skip = (4 if D == 8 else 0) if a.skip is None else a.skip     # layer skip + 1 reads [hidden | features]
  wide = lambda i: skip and i - 1 == skip
  dev = 'cuda'
  g = torch.Generator(device=dev).manual_seed(0)
  bf = torch.bfloat16
  feat = torch.randn(M, F, device=dev, generator=g).to(bf)
  kin = [F if i == 0 else W + F if wide(i) else W for i in range(D)]
  ws = [(torch.randn(W, k, device=dev, generator=g) * math.sqrt(2.0 / k)).to(bf) for k in kin]
  wkn = [(torch.randn(W, W, device=dev, generator=g) / 16).to(bf) for _ in range(D)]
  bs = [torch.zeros(W, device=dev) for _ in range(D)]
  acts = [torch.empty(M, W, device=dev, dtype=bf) for _ in range(D)]
  bits = [torch.empty(M, W // 32, device=dev, dtype=torch.int32) for _ in range(D)]
  head = torch.empty(M, device=dev)
  hw = torch.randn(W, device=dev, generator=g)
  hb = torch.zeros(1, device=dev)
  flops_f = 2.0 * M * W * sum(kin)
  flops_b = 2.0 * M * W * W * (D - 1)

  def layers(train):
    out = []
    for i in range(D):
      ly = dict(w=ws[i], bias=bs[i])
      ly.update(dict(n_stream=F // 64) if i == 0 else dict(n_res=4))
      if wide(i):
        ly.update(n_stream=F // 64, stream_kb0=4)
      if train or i == D - 1:
        ly['out'] = acts[i]
      if train:
        ly['maskbits'] = bits[i]
      out.append(ly)
    return out
  res = {}
  if a.only in ('all', 'fwd'):
    d_train = ops.chain_desc(L.CHAIN_FWD, M, layers(True), stream=feat, stream_cols=F, head_w=hw, head_b=hb, head_out=head)
    d_inf = ops.chain_desc(L.CHAIN_FWD, M, layers(False), stream=feat, stream_cols=F, head_w=hw, head_b=hb, head_out=head)
    t = timeit(lambda: ops.mlp_chain(d_train), a.iters)
    res['chain fwd (train: all stores + masks)'] = (t, flops_f, M * (F * 2 + D * (W * 2 + 32) + 4))
    clocks('fwd train')
    t = timeit(lambda: ops.mlp_chain(d_inf), a.iters)
    res['chain fwd (inference: last store only)'] = (t, flops_f, M * (F * 2 + W * 2 + 4))
    clocks('fwd inference')
  if a.only in ('all', 'layers') and not skip:
    def per_layer():
      x = feat
      for i in range(D):
        ops.gemm(L.GEMM_FWD, x, ws[i], acts[i], m=M, n=W, k=F if i == 0 else W, act=L.ACT_RELU, bias=bs[i], maskbits=bits[i])
        x = acts[i]
      ops.head_fwd(x, hw.to(bf).view(1, W), hb, 1, W, raw=head.view(M, 1))
    t = timeit(per_layer, a.iters)
    res['per-layer fwd (4 GEMMs + head)'] = (t, flops_f, M * (F * 2 + W * 2 + (D - 1) * (W * 4) + D * 32 + W * 2 + 4))
  if a.only in ('all', 'bwd') and D > 1:
    dy = [torch.empty(M, W, device=dev, dtype=bf) for _ in range(D)]
    dy[-1].normal_(generator=g)
    cs = [torch.zeros(W, device=dev) for _ in range(D)]
    lys = []
    for j, i in enumerate(range(D - 1, 0, -1)):
      ly = dict(w=wkn[i], maskbits=bits[i - 1], colsum=cs[i - 1], out=dy[i - 1])
      ly.update(dict(n_stream=4) if j == 0 else dict(n_res=4))
      lys.append(ly)
    d_b = ops.chain_desc(L.CHAIN_BWD, M, lys, stream=dy[-1], stream_cols=W)
    t = timeit(lambda: ops.mlp_chain(d_b), a.iters)
    res['chain bwd (dgrad chain)'] = (t, flops_b, M * (W * 2 + (D - 1) * (W * 2 + 32)))
    clocks('bwd')

    def per_layer_b():
      for i in range(D - 1, 0, -1):
        ops.gemm(L.GEMM_DGRAD, dy[i], wkn[i], dy[i - 1], m=M, n=W, k=W, maskbits=bits[i - 1], colsum=cs[i - 1])
    t = timeit(per_layer_b, a.iters)
    res['per-layer bwd (dgrad GEMMs)'] = (t, flops_b, M * (D - 1) * (W * 4 + 32))
  print(f'# M = {M} rows, depth {D}, Fpad {F}' + (f', skip after layer {skip}' if skip else '') + f'; {card()}')
  for k, (t, fl, by) in res.items():
    print(f'{k:45s} {t * 1e3:8.1f} us  {fl / t / 1e9:7.1f} TFLOP/s  {by / t / 1e6:7.1f} GB/s algorithmic')


if __name__ == '__main__':
  main()
