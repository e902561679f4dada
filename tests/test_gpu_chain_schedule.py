"""The segment-alternating schedule of the layer-chained trunk (csrc/chain.cu): the two consumer warpgroups take
turns segment by segment, the streamed operand has a ring of its own, and the mask words leave (forward) or
arrive (backward) as whole 32-byte rows.  Checked at the sizes the models run (2^20 rows, ragged), with layers of
one, two and three segments, in the train and render forms, with a mask pitch that takes the narrow store, and
with guard bands around every output.  Needs an H100.

Exact where the arithmetic is the same: mask bits against the stored activation, the render form against the
train form, and the narrow mask store against the wide one.  Against the per-layer GEMMs, each fed the chain's
own input of that layer, the bound is test_gpu_chain.py's."""
import math

import numpy as np
import pytest
import torch

from util import close

pytestmark = pytest.mark.gpu

W = 256
GUARD = 64          # rows of guard band after every output


@pytest.fixture(scope='module')
def ops():
  from multinerf_b200 import lib, ops as _ops
  lib.require_device()
  return _ops


def _randn(gen, *shape, scale=1.0):
  return (torch.randn(*shape, device='cuda', generator=gen) * scale).to(torch.bfloat16)


def _unpack(bits):
  sh = torch.arange(32, device=bits.device)
  return ((bits[:, :, None] >> sh) & 1).reshape(bits.shape[0], -1).bool()


def _guarded(M, cols, dtype, fill):
  """[M + GUARD, cols] filled with a sentinel; the chain is given the first M rows."""
  return torch.full((M + GUARD, cols), fill, dtype=dtype, device='cuda')


def _forward(ops, M, depth, Fpad, skip, mask_pitch=W // 32, mask_off=0, render=False, seed=0):
  from multinerf_b200 import lib as L
  gen = torch.Generator(device='cuda').manual_seed(seed)
  feat = _randn(gen, M, Fpad)
  kin = [Fpad] + [W + Fpad if (skip and i - 1 == skip) else W for i in range(1, depth)]
  ws = [_randn(gen, W, k, scale=math.sqrt(2.0 / k)) for k in kin]
  bs = [torch.randn(W, device='cuda', generator=gen) * 0.1 for _ in range(depth)]
  hw = _randn(gen, 1, W, scale=1 / 16)
  hb = torch.tensor([0.37], device='cuda')
  acts = [_guarded(M, W, torch.bfloat16, -7.0) for _ in range(depth)]
  bits = [_guarded(M, mask_pitch, torch.int32, -1) for _ in range(depth)]
  head = torch.full((M + GUARD,), -3.0, device='cuda')
  layers = []
  for i in range(depth):
    ly = dict(w=ws[i], bias=bs[i])
    if not render or i == depth - 1:
      ly['out'] = acts[i][:M]
    if not render:
      ly['maskbits'] = bits[i][:M, mask_off:mask_off + W // 32]
    if i == 0:
      ly.update(n_stream=Fpad // 64, stream_col0=0, stream_kb0=0)
    else:
      ly.update(n_res=4, res_kb0=0)
      if kin[i] == W + Fpad:
        ly.update(n_stream=Fpad // 64, stream_col0=0, stream_kb0=4)
    layers.append(ly)
  ops.mlp_chain(ops.chain_desc(L.CHAIN_FWD, M, layers, stream=feat, stream_cols=Fpad,
                               head_w=hw[0].float().contiguous(), head_b=hb, head_out=head[:M]))
  torch.cuda.synchronize()
  return dict(feat=feat, kin=kin, ws=ws, bs=bs, hw=hw, hb=hb, acts=acts, bits=bits, head=head, mask_off=mask_off)


def _check_forward_guards(r, M, render):
  depth = len(r['acts'])
  for i in range(depth):
    assert (r['acts'][i][M:] == -7).all(), f'layer {i}: rows past M written'
    written = not render or i == depth - 1
    assert bool((r['acts'][i][:M] != -7).any()) == written, f'layer {i}: store'
    b, o = r['bits'][i], r['mask_off']
    assert (b[M:] == -1).all() and (b[:, :o] == -1).all() and (b[:, o + W // 32:] == -1).all(), f'layer {i}: mask guard'
    if render:
      assert (b == -1).all(), f'layer {i}: the render form writes no mask words'
  assert (r['head'][M:] == -3).all()


@pytest.mark.parametrize('M,depth,Fpad,skip', [
    (1 << 20, 4, 512, 0),            # a proposal level of 360.gin: layer 0 is two segments of streamed k-blocks
    ((1 << 20) - 37, 4, 512, 0),     # ragged last unit; warpgroup 1's rows of it lie partly past M
    (20032, 8, 128, 4),              # skip layer of 4 resident + 2 streamed k-blocks; the last unit is warpgroup 0's alone
    (12345, 8, 320, 4),              # skip layer of 4 + 5: three segments, the streamed ring wraps inside a segment
    (4096 + 1, 2, 64, 0),
])
def test_forward_schedule(ops, M, depth, Fpad, skip):
  from multinerf_b200 import lib as L
  r = _forward(ops, M, depth, Fpad, skip)
  _check_forward_guards(r, M, render=False)
  x = r['feat']
  for i in range(depth):
    a = r['acts'][i][:M]
    # the mask words are the sign of what was stored, bit for bit
    assert torch.equal(_unpack(r['bits'][i][:M]), a > 0), f'layer {i} mask bits'
    # per-layer GEMM on the chain's own input of this layer: the same operands and the same fp32 sums
    xin = x if not (skip and i - 1 == skip) else torch.cat([x, r['feat']], 1)
    ref = torch.empty(M, W, dtype=torch.bfloat16, device='cuda')
    rb = torch.empty(M, W // 32, dtype=torch.int32, device='cuda')
    ops.gemm(L.GEMM_FWD, xin, r['ws'][i], ref, m=M, n=W, k=r['kin'][i], act=L.ACT_RELU, bias=r['bs'][i], maskbits=rb)
    close(a.float(), ref.float(), atol=2e-2, rtol=1.6e-2, msg=f'layer {i} activation')
    assert float((a == ref).float().mean()) > 0.999, i
    x = a
  head_ref = ops.head_fwd(r['acts'][-1][:M], r['hw'], r['hb'], 1, W)
  close(r['head'][:M], head_ref[:, 0], atol=2e-3, rtol=2e-3, msg='density head')
  # the render form (`out` on the last layer only, no mask words) computes the same last layer and head
  rr = _forward(ops, M, depth, Fpad, skip, render=True)
  _check_forward_guards(rr, M, render=True)
  assert torch.equal(rr['acts'][-1], r['acts'][-1]) and torch.equal(rr['head'], r['head'])


def test_forward_narrow_mask_store(ops):
  """A mask buffer whose rows start 4 bytes off an 8-byte boundary takes the 4-byte stores: same words, and the
  words on either side of the row's eight stay untouched."""
  M = 5000
  wide = _forward(ops, M, 4, 128, 0)
  for pitch, off in ((9, 0), (10, 1), (11, 2)):
    nar = _forward(ops, M, 4, 128, 0, mask_pitch=pitch, mask_off=off)
    _check_forward_guards(nar, M, render=False)
    for i in range(4):
      assert torch.equal(nar['bits'][i][:M, off:off + 8], wide['bits'][i][:M]), (pitch, off, i)
      assert torch.equal(nar['acts'][i], wide['acts'][i])


@pytest.mark.parametrize('M,depth,pitch,off', [(1 << 20, 4, 8, 0), ((1 << 20) - 37, 4, 8, 0), (20032, 8, 8, 0),
                                               (4097, 2, 8, 0), (5000, 4, 9, 1)])
def test_backward_schedule(ops, M, depth, pitch, off):
  from multinerf_b200 import lib as L
  gen = torch.Generator(device='cuda').manual_seed(M + depth)
  dy_last = _randn(gen, M, W)
  w_kn = [_randn(gen, W, W, scale=1 / 16) for _ in range(depth)]
  masks = [torch.randint(-2 ** 31, 2 ** 31, (M, pitch), device='cuda', generator=gen).to(torch.int32)
           for _ in range(depth)]
  outs = [_guarded(M, W, torch.bfloat16, -7.0) for _ in range(depth - 1)]
  css = [torch.full((W + GUARD,), 1.5, device='cuda') for _ in range(depth - 1)]
  layers = []
  for j, i in enumerate(range(depth - 1, 0, -1)):
    ly = dict(w=w_kn[i], maskbits=masks[i - 1][:, off:off + 8], colsum=css[j][:W], out=outs[j][:M])
    ly.update(dict(n_stream=4, stream_col0=0, stream_kb0=0) if j == 0 else dict(n_res=4, res_kb0=0))
    layers.append(ly)
  ops.mlp_chain(ops.chain_desc(L.CHAIN_BWD, M, layers, stream=dy_last, stream_cols=W))
  torch.cuda.synchronize()
  cur = dy_last
  for j, i in enumerate(range(depth - 1, 0, -1)):
    assert (outs[j][M:] == -7).all() and (css[j][W:] == 1.5).all(), f'dgrad {j}: guard'
    # the per-layer DGRAD of the chain's own input gradient: the same products, the same masks
    mk = masks[i - 1][:, off:off + 8].contiguous()
    ref = torch.empty(M, W, dtype=torch.bfloat16, device='cuda')
    cs = torch.full((W,), 1.5, device='cuda')
    ops.gemm(L.GEMM_DGRAD, cur, w_kn[i], ref, m=M, n=W, k=W, maskbits=mk, colsum=cs)
    a = outs[j][:M]
    close(a.float(), ref.float(), atol=3e-2, rtol=1.6e-2, msg=f'dgrad {j}')
    assert float((a == ref).float().mean()) > 0.999, j
    assert torch.equal(a != 0, _unpack(mk) & (a != 0)), f'dgrad {j}: a masked element is not zero'
    close(css[j][:W], cs, atol=2e-2 * math.sqrt(M), rtol=2e-3, msg=f'bias gradient {j}')
    cur = a
