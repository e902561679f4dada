"""Where the time of the ping-pong Dense-layer GEMM (gemm_tc_pingpong_kernel) goes, on the NerfMLP shapes of 360.gin.

  python tools/gemm_clocks.py [--rows 524288] [--width 1024] [--iters 20] [--hash]
                              [--lib PATH [--lib PATH ...] [--rounds R]]

Times FWD (bias + ReLU + mask bits) of the 1024-wide trunk at K = 512, 1024 and 1536, its DGRAD with mask bits at
K = 1024, the bottleneck FWD (N = 256, K = 1024, bias only) and DGRAD (N = 1024, K = 256, mask bits + rank-1 term),
then prints the card's name, power limit and SM clock, and for each launch the epilogue operand set it ran
(mnrf_gemm_instance.epilogue).  `--width` sets the trunk width.  `--hash` also prints the SHA-256 of each FWD's
output and mask words, to compare two builds on the same data.  A library built with -DMNRF_GEMM_CLOCKS (csrc/gemm_tc.cu) also gets, per consumer warpgroup,
the clock64() split of the first thread of CTA 0 as shares of that thread's time.  `--build DIR` builds such a
library into DIR first (from this tree's sources) and runs with it.  With `--lib`, each named build is run in a
process of its own (the library is chosen at import), the builds alternating R times.
"""
import argparse
import ctypes
import hashlib
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from multinerf_b200 import lib as L, ops  # noqa: E402

CLASSES = ('turn wait', 'full-barrier wait', 'wgmma issue + wait', 'epilogue element loop',
           'store-read waits + named barriers', 'mask-word wait')


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


def build_clocks(out_dir):
  """This tree's library with -DMNRF_GEMM_CLOCKS on gemm_tc.cu, built in out_dir; returns its path."""
  from multinerf_b200 import build as B
  os.makedirs(out_dir, exist_ok=True)
  objs = []
  for name, flags in B.SOURCES.items():
    obj = os.path.join(out_dir, name.replace('.cu', '.o'))
    extra = ['-DMNRF_GEMM_CLOCKS'] if name == 'gemm_tc.cu' else []
    subprocess.run([B._nvcc()] + B.ARCH + B.COMMON + flags + extra + ['-c', os.path.join(B.CSRC, name), '-o', obj],
                   check=True)
    objs.append(obj)
  path = os.path.join(out_dir, 'libmnrf_b200_clocks.so')
  subprocess.run([B._nvcc()] + B.ARCH + ['-shared', '-o', path] + objs, check=True)
  return path


def clocks(lib):
  """Per warpgroup, the shares of each class in the clock64() time since the last call (None without the split)."""
  if not hasattr(lib, 'mnrf_gemm_clocks'):
    return None
  out = (ctypes.c_ulonglong * (2 * len(CLASSES)))()
  assert lib.mnrf_gemm_clocks(out) == 0
  n = len(CLASSES)
  return [[v / (float(sum(out[w * n:(w + 1) * n])) or 1.0) for v in out[w * n:(w + 1) * n]] for w in range(2)]


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--rows', type=int, default=524288)
  ap.add_argument('--width', type=int, default=1024)
  ap.add_argument('--hash', action='store_true')
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--lib', action='append', default=[])
  ap.add_argument('--rounds', type=int, default=2)
  ap.add_argument('--build', default=None, help='build a -DMNRF_GEMM_CLOCKS library into this directory and use it')
  a = ap.parse_args()
  if a.build:
    a.lib = [build_clocks(a.build)]
    a.rounds = 1
  if a.lib:
    args = [sys.executable, os.path.abspath(__file__), '--rows', str(a.rows), '--width', str(a.width), '--iters',
            str(a.iters)] + (['--hash'] if a.hash else [])
    for r in range(a.rounds):
      for path in a.lib:
        print(f'## round {r}: {path}', flush=True)
        subprocess.run(args, env=dict(os.environ, MNRF_LIB=os.path.abspath(path)), check=True)
    return
  L.require_device()
  lib = ctypes.CDLL(L.LIB_PATH)
  dev, bf = 'cuda', torch.bfloat16
  g = torch.Generator(device=dev).manual_seed(0)
  M, W = a.rows, a.width
  rnd = lambda *s, scale=1.0: (torch.randn(*s, device=dev, generator=g) * scale)
  bits = torch.randint(-2**31, 2**31 - 1, (M, W // 32), device=dev, dtype=torch.int32, generator=g)
  out = torch.empty(M, W, device=dev, dtype=bf)
  obits = torch.empty(M, W // 32, device=dev, dtype=torch.int32)
  bias = rnd(W, scale=0.1)
  runs = []
  for k in (512, 1024, 1536):
    x = rnd(M, k, scale=0.5).to(bf)
    w = rnd(W, k, scale=0.05).to(bf)
    runs.append((f'fwd K={k} bias+relu+bits', 2.0 * M * W * k,
                 (L.GEMM_FWD, x, w, out, dict(m=M, n=W, k=k, act=L.ACT_RELU, bias=bias, maskbits=obits))))
  dy = rnd(M, W, scale=0.1).to(bf)
  w_kn = rnd(W, W, scale=0.05).to(bf)
  runs.append(('dgrad K=1024 bits', 2.0 * M * W * W,
               (L.GEMM_DGRAD, dy, w_kn, out, dict(m=M, n=W, k=W, maskbits=bits))))
  # the bottleneck: FWD from the trunk output to 256 columns, bias only, and its DGRAD back
  xb = rnd(M, W, scale=0.5).to(bf)
  wbf = rnd(256, W, scale=0.05).to(bf)
  bout = torch.empty(M, 256, device=dev, dtype=bf)
  bbias = rnd(256, scale=0.1)
  runs.append((f'fwd K={W} bias (bottleneck)', 2.0 * M * 256 * W,
               (L.GEMM_FWD, xb, wbf, bout, dict(m=M, n=256, k=W, bias=bbias))))
  dbott = rnd(M, 256, scale=0.1).to(bf)
  wb = rnd(W, 256, scale=0.05).to(bf)
  rowv, colv = rnd(M), rnd(W)
  runs.append(('dgrad K=256 bits+rank-1 (bottleneck)', 2.0 * M * W * 256,
               (L.GEMM_DGRAD, dbott, wb, out, dict(m=M, n=W, k=256, maskbits=bits, rowv=rowv, colv=colv))))
  has_plan = hasattr(lib, 'mnrf_gemm_plan')
  res = []
  for name, fl, (mode, x, w, o, kw) in runs:
    fn = lambda: ops.gemm(mode, x, w, o, **kw)
    fn()
    torch.cuda.synchronize()
    digest = ''
    if a.hash and mode == L.GEMM_FWD:
      h = hashlib.sha256(o.view(torch.int16).cpu().numpy().tobytes())
      if 'maskbits' in kw:
        h.update(kw['maskbits'].cpu().numpy().tobytes())
      digest = h.hexdigest()[:16]
    epi = ops.gemm_plan(mode, x, w, o, **kw)['epilogue'] if has_plan else '-'
    clocks(lib)                                    # clear: the split below is of the timed launches
    ms = timeit(fn, a.iters)
    res.append((name, ms, fl, clocks(lib), epi, digest))
  print(f'# M = {M}, N = {W}; {card()}; {L.LIB_PATH}')
  for name, ms, fl, split, epi, digest in res:
    print(f'{name:40s} {ms * 1e3:8.1f} us  {fl / ms / 1e9:7.1f} TFLOP/s  set {epi}  {digest}', flush=True)
    for wgi, shares in enumerate(split or []):
      print(f'    warpgroup {wgi}: ' + ', '.join(f'{n} {100 * s:.1f} %' for n, s in zip(CLASSES, shares)))


if __name__ == '__main__':
  main()
