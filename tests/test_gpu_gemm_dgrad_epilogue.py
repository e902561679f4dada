"""DGRAD epilogue of the tensor-core Dense-layer GEMM: column sums when a persistent CTA moves between column
blocks, and the mask words taken either by TMA or by the epilogue's own loads.  Needs an H100."""
import math

import numpy as np
import pytest
import torch

from gemm_ref import pack_bits as _pack
from util import close

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ops():
  from multinerf_b200 import lib, ops as _ops
  lib.require_device()
  return _ops


def _bf(x):
  return torch.tensor(x).to(torch.bfloat16)


# N = 640 and N = 320 run 5 column blocks (of 128 and 64) on 132 SMs, so a CTA's consecutive tiles change column
# block and the column sums are flushed more than once per CTA.  128-column tiles with a mask-word pitch of 20
# (16-byte rows) take their mask words by TMA; a pitch of 22, and 64-column tiles, load them in the epilogue.
@pytest.mark.parametrize('M,N,K,pitch', [(20000, 640, 256, 20), (20000, 640, 256, 22), (20000, 320, 256, 10),
                                         (10000, 768, 128, 24)])
def test_gemm_dgrad_colsum_column_blocks(ops, M, N, K, pitch):
  from multinerf_b200 import lib as L
  rng = np.random.default_rng(M + N + K + pitch)
  dy = _bf(rng.normal(size=(M, K)).astype(np.float32))
  w_kn = _bf(rng.normal(size=(N, K)).astype(np.float32) / math.sqrt(K))
  maskb = torch.tensor(rng.uniform(size=(M, N)) > 0.4)
  rowv = torch.tensor(rng.normal(size=(M,)).astype(np.float32))
  colv = torch.tensor(rng.normal(size=(N,)).astype(np.float32))
  ref = (dy.float() @ w_kn.float().T + rowv[:, None] * colv[None, :]) * maskb
  out = torch.empty(M, N, dtype=torch.bfloat16, device='cuda')
  cs = torch.full((N,), -1.0, device='cuda')
  ops.gemm(L.GEMM_DGRAD, dy.cuda(), w_kn.cuda(), out, m=M, n=N, k=K, rowv=rowv.cuda(), colv=colv.cuda(),
           maskbits=_pack(maskb, pitch).cuda(), colsum=cs)
  torch.cuda.synchronize()
  close(out.float(), ref.to(torch.bfloat16).float(), atol=3e-2, rtol=1.6e-2, msg='dgrad bits')
  close(cs, ref.sum(0) - 1.0, atol=2e-2 * math.sqrt(M), rtol=2e-3, msg='dgrad colsum')


# Three stacked streams share one set of masks (mask row = output row mod M): M a multiple of the 128-row tile lets
# TMA load a tile's mask rows in one box; otherwise a tile's rows wrap and the epilogue loads the words itself.
@pytest.mark.parametrize('M', [384, 200])
def test_gemm_dgrad_mask_mod(ops, M):
  from multinerf_b200 import lib as L
  rng = np.random.default_rng(M)
  N, K = 256, 128
  maskb = torch.tensor(rng.uniform(size=(M, N)) > 0.5)
  a = _bf(rng.normal(size=(3 * M, K)).astype(np.float32))
  w = _bf(rng.normal(size=(N, K)).astype(np.float32) / math.sqrt(K))
  out = torch.empty(3 * M, N, dtype=torch.bfloat16, device='cuda')
  cs = torch.zeros(N, device='cuda')
  ops.gemm(L.GEMM_DGRAD, a.cuda(), w.cuda(), out, m=3 * M, n=N, k=K, maskbits=_pack(maskb, N // 32).cuda(),
           mask_mod=M, colsum=cs)
  torch.cuda.synchronize()
  ref = (a.float() @ w.float().T) * maskb.repeat(3, 1)
  close(out.float(), ref.to(torch.bfloat16).float(), atol=3e-2, rtol=1.6e-2, msg=f'mask_mod={M}')
  close(cs, ref.sum(0), atol=2e-2 * math.sqrt(3 * M), rtol=2e-3, msg=f'mask_mod={M} colsum')
