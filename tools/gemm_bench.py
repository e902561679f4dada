"""Micro-benchmark of mnrf_gemm on the shapes of the 360 config (run on an H100).

  python tools/gemm_bench.py [--rows 1048576] [--bottleneck | --side_sums]

Prints ms / TFLOP/s / GB/s per (mode, N, K, features) so epilogue features can be costed in
isolation (each timing: 20 launches after 3 warm-ups, inputs larger than L2), and beside each GEMM the rate of
torch.matmul (cuBLAS, bf16 output) on the same operands as a yardstick of what the card attains at that shape.
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from multinerf_b200 import lib as L      # noqa: E402
from multinerf_b200 import ops           # noqa: E402


def timeit(fn, iters=20):
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


def bottleneck(dev, M):
  """The two launches between the view branch and the trunk of the 360.gin NerfMLP backward (models.py:527):
  d x_last = (d bottleneck @ Wb^T + d_raw_density (x) w_density) * relu'(x_last)   [M, 1024] <- [M, 256]
  dWb = x_last^T d bottleneck (+ bias gradient, + the density head's dW as side sums)  [1024, 256]"""
  W, bw = 1024, 256
  x_last = (torch.randn(M, W, device=dev) * 0.5).bfloat16()
  dbott = (torch.randn(M, bw, device=dev) * 0.1).bfloat16()
  w_kn = (torch.randn(W, bw, device=dev) * 0.05).bfloat16()          # B[N = 1024, K = 256], K-major
  dy = torch.empty(M, W, device=dev, dtype=torch.bfloat16)
  bits = torch.randint(-2**31, 2**31 - 1, (M, W // 32), device=dev, dtype=torch.int32)
  rowv = torch.randn(M, device=dev)
  colv = torch.randn(W, device=dev)
  dw = torch.zeros(W, bw, device=dev)
  db = torch.zeros(bw, device=dev)
  aw = torch.zeros(W, device=dev)

  def report(name, ms, nbytes, flops):
    print(f'M={M} {name:44s} {ms * 1e3:8.1f} us  {flops / ms / 1e9:7.1f} TFLOP/s  {nbytes / ms / 1e6:7.1f} GB/s', flush=True)
  fl = 2.0 * M * W * bw
  ms = timeit(lambda: ops.gemm(L.GEMM_DGRAD, dbott, w_kn, dy, m=M, n=W, k=bw))
  report('dgrad N=1024 K=256 plain', ms, 2.0 * M * (W + bw), fl)
  ms = timeit(lambda: ops.gemm(L.GEMM_DGRAD, dbott, w_kn, dy, m=M, n=W, k=bw, maskbits=bits))
  report('dgrad N=1024 K=256 bits', ms, 2.0 * M * (W + bw) + M * W / 8, fl)
  ms = timeit(lambda: ops.gemm(L.GEMM_DGRAD, dbott, w_kn, dy, m=M, n=W, k=bw, maskbits=bits, rowv=rowv, colv=colv))
  report('dgrad N=1024 K=256 bits+rank-1 (the step)', ms, 2.0 * M * (W + bw) + M * W / 8, fl)
  ms = timeit(lambda: ops.gemm(L.GEMM_WGRAD, x_last, dbott, dw, m=W, n=bw, k=M))
  report('wgrad [1024,256] plain', ms, 2.0 * M * (W + bw), fl)
  ms = timeit(lambda: ops.gemm_wgrad(x_last, dbott, dw, m=W, n=bw, k=M, bsum=db))
  report('wgrad [1024,256] + bias sums', ms, 2.0 * M * (W + bw), fl)
  ms = timeit(lambda: ops.gemm_wgrad(x_last, dbott, dw, m=W, n=bw, k=M, bsum=db, side_w=rowv, side_aw=aw))
  report('wgrad [1024,256] + bias + head dW (the step)', ms, 2.0 * M * (W + bw), fl)
  # the narrow heads of the view branch ([M, 128] activations) and of the PropMLP ([2M, 256])
  for (Mh, K, n_out, with_dx) in [(M, 128, 3, True), (2 * M, 256, 1, True), (M, 1024, 1, False)]:
    xh = (torch.randn(Mh, K, device=dev) * 0.5).bfloat16()
    wh = (torch.randn(n_out, K, device=dev) * 0.05).bfloat16()
    bh = torch.zeros(n_out, device=dev)
    raw = torch.empty(Mh, n_out, device=dev)
    draw = torch.randn(Mh, n_out, device=dev)
    dxh = torch.empty(Mh, K, device=dev, dtype=torch.bfloat16) if with_dx else None
    dwh = torch.zeros(K, n_out, device=dev)
    dxs = torch.zeros(K, device=dev) if with_dx else None
    ms = timeit(lambda: ops.head_fwd(xh, wh, bh, n_out, K, raw=raw))
    print(f'head_fwd  M={Mh} K={K} n_out={n_out}: {ms * 1e3:7.1f} us  {2.0 * Mh * K / ms / 1e6:7.1f} GB/s', flush=True)
    ms = timeit(lambda: ops.head_bwd(xh, wh, draw, n_out, K, dx=dxh, relu_mask=with_dx, dw=dwh, db=bh, dxsum=dxs))
    print(f'head_bwd  M={Mh} K={K} n_out={n_out} dx={with_dx}: {ms * 1e3:7.1f} us  '
          f'{2.0 * Mh * K * (2 if with_dx else 1) / ms / 1e6:7.1f} GB/s', flush=True)


def side_sums(dev, rows):
  """The weight-gradient GEMM with and without the side sums it takes from its staged operand tiles (bias gradient
  `bsum`, Dense(1) head gradient `side_aw`), at the 360.gin shapes: the NerfMLP trunk [1024, 1024] at rows / 2, the
  PropMLP trunk [512 | 256, 256] at `rows`, the bottleneck [1024, 256] with both sums; and the 1024-wide DGRAD with
  mask bits only against mask bits plus column sums."""
  def line(name, ms, flops, base_ms=None):
    rel = f'  {100.0 * (ms / base_ms - 1):+5.1f} % vs plain' if base_ms else ''
    print(f'{name:52s} {ms * 1e3:8.1f} us  {flops / ms / 1e9:7.1f} TFLOP/s{rel}', flush=True)
  for (M, K, N, head) in [(rows // 2, 1024, 1024, False), (rows, 512, 256, False), (rows, 256, 256, False),
                          (rows // 2, 1024, 256, True)]:
    x = (torch.randn(M, K, device=dev) * 0.5).bfloat16()
    dy = (torch.randn(M, N, device=dev) * 0.1).bfloat16()
    dw = torch.zeros(K, N, device=dev)
    db = torch.zeros(N, device=dev)
    w = torch.randn(M, device=dev)
    aw = torch.zeros(K, device=dev)
    fl = 2.0 * M * N * K
    tag = f'R={M} wgrad [{K},{N}]'
    base = timeit(lambda: ops.gemm(L.GEMM_WGRAD, x, dy, dw, m=K, n=N, k=M))
    line(f'{tag} plain', base, fl)
    ms = timeit(lambda: ops.gemm_wgrad(x, dy, dw, m=K, n=N, k=M, bsum=db))
    line(f'{tag} + bsum', ms, fl, base)
    if head:
      ms = timeit(lambda: ops.gemm_wgrad(x, dy, dw, m=K, n=N, k=M, bsum=db, side_w=w, side_aw=aw))
      line(f'{tag} + bsum + side_aw', ms, fl, base)
    del x, dy
  M, W = rows // 2, 1024
  dy = (torch.randn(M, W, device=dev) * 0.1).bfloat16()
  w_kn = (torch.randn(W, W, device=dev) * 0.05).bfloat16()
  dx = torch.empty(M, W, device=dev, dtype=torch.bfloat16)
  bits = torch.randint(-2**31, 2**31 - 1, (M, W // 32), device=dev, dtype=torch.int32)
  cs = torch.zeros(W, device=dev)
  fl = 2.0 * M * W * W
  base = timeit(lambda: ops.gemm(L.GEMM_DGRAD, dy, w_kn, dx, m=M, n=W, k=W, maskbits=bits))
  line(f'R={M} dgrad [{W},{W}] bits', base, fl)
  ms = timeit(lambda: ops.gemm(L.GEMM_DGRAD, dy, w_kn, dx, m=M, n=W, k=W, maskbits=bits, colsum=cs))
  line(f'R={M} dgrad [{W},{W}] bits + colsum', ms, fl, base)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--rows', type=int, default=1 << 20)
  ap.add_argument('--bottleneck', action='store_true',
                  help='only the NerfMLP bottleneck shapes of 360.gin (1024 <-> 256 at 524288 rows)')
  ap.add_argument('--side_sums', action='store_true',
                  help='only the weight-gradient side sums (with / without) and the DGRAD column sums')
  args = ap.parse_args()
  dev = torch.device('cuda:0')
  torch.manual_seed(0)
  if args.bottleneck:
    return bottleneck(dev, args.rows // 2)
  if args.side_sums:
    return side_sums(dev, args.rows)
  # the PropMLP trunk, the NerfMLP trunk and its skip layer (K = 1536: FWD and the [1536, 1024] WGRAD; its DGRAD
  # output is 1536 wide, past the fused column sums' limit, and runs split at the concat in the model)
  for (M, N, K) in [(args.rows, 256, 256), (args.rows, 256, 512), (args.rows // 2, 1024, 1024),
                    (args.rows // 2, 1024, 1536)]:
    x = (torch.randn(M, K, device=dev) * 0.5).bfloat16()
    w_nk = (torch.randn(N, K, device=dev) * 0.05).bfloat16()
    w_kn = w_nk.t().contiguous()
    bias = torch.randn(N, device=dev) * 0.1
    y = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    bits = torch.empty(M, max(N // 32, 4), device=dev, dtype=torch.int32)
    dy = (torch.randn(M, N, device=dev) * 0.1).bfloat16()
    dx = torch.empty(M, K, device=dev, dtype=torch.bfloat16)
    xbits = torch.randint(-2**31, 2**31 - 1, (M, max(K // 32, 4)), device=dev, dtype=torch.int32)
    dw = torch.zeros(K, N, device=dev)
    cs = torch.zeros(K, device=dev)
    flops = 2.0 * M * N * K

    def report(name, ms, nbytes, torch_ms=None):
      ref = f'  torch.matmul {flops / torch_ms / 1e9:7.1f} TFLOP/s' if torch_ms else ''
      print(f'M={M} N={N} K={K} {name:28s} {ms:7.3f} ms  {flops / ms / 1e9:7.1f} TFLOP/s  '
            f'{nbytes / ms / 1e6:7.1f} GB/s{ref}', flush=True)

    t_fwd = timeit(lambda: torch.matmul(x, w_nk.t(), out=y))
    ms = timeit(lambda: ops.gemm(L.GEMM_FWD, x, w_nk, y, m=M, n=N, k=K, act=L.ACT_RELU, bias=bias,
                                 maskbits=bits))
    report('fwd bias+relu+bits', ms, 2.0 * M * (N + K), t_fwd)
    if K <= 1024:
      t_dgrad = timeit(lambda: torch.matmul(dy, w_kn.t(), out=dx))
      ms = timeit(lambda: ops.gemm(L.GEMM_DGRAD, dy, w_kn, dx, m=M, n=K, k=N))
      report('dgrad plain', ms, 2.0 * M * (N + K), t_dgrad)
      ms = timeit(lambda: ops.gemm(L.GEMM_DGRAD, dy, w_kn, dx, m=M, n=K, k=N, maskbits=xbits))
      report('dgrad bits', ms, 2.0 * M * (N + K), t_dgrad)
      ms = timeit(lambda: ops.gemm(L.GEMM_DGRAD, dy, w_kn, dx, m=M, n=K, k=N, maskbits=xbits, colsum=cs))
      report('dgrad bits+colsum', ms, 2.0 * M * (N + K), t_dgrad)
    t_wgrad = timeit(lambda: torch.matmul(x.t(), dy))     # the [K, N] output is too small for its dtype to matter
    ms = timeit(lambda: ops.gemm(L.GEMM_WGRAD, x, dy, dw, m=K, n=N, k=M))
    report('wgrad', ms, 2.0 * M * (N + K), t_wgrad)
    ms = timeit(lambda: ops.colsum(dy, N, cs[:N] if N <= K else torch.zeros(N, device=dev)))
    report('colsum kernel', ms, 2.0 * M * N)
    del x, y, dy, dx, bits, xbits


if __name__ == '__main__':
  main()
