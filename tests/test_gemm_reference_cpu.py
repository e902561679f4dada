"""The fp64 GEMM checker of tests/gemm_ref.py is sound and sensitive.  CPU only.

Soundness: the Dense-layer GEMM's arithmetic emulated in fp32 -- the K products accumulated in several orders,
including fused blocks of 16 that truncate, the fp32 epilogue with the error of its fast exp / log / divide, round to
nearest even into bf16 -- lands inside the bound for every output, column sum and mask bit.
Sensitivity: each small mutation of a correct output that an epilogue or scheduling bug would make is flagged.
"""
import numpy as np
import pytest
import torch

import gemm_ref as G

ORDERS = ('sequential', 'reversed', 'pairwise', 'truncate16', 'truncate16_blocks')


def _trunc32(x):
  """fp64 -> fp32 rounded toward zero."""
  f = x.float()
  over = f.double().abs() > x.abs()
  return torch.where(over, torch.nextafter(f, torch.zeros_like(f)), f)


def _accumulate(a, b, order):
  """fp32 A B^T of bf16 operands, the K products (exact in fp32) added in `order`."""
  p = (a.float()[:, None, :] * b.float()[None, :, :])          # [M, N, K], exact
  k = p.shape[-1]
  if order in ('sequential', 'reversed'):
    acc = torch.zeros(p.shape[:2])
    for j in (range(k) if order == 'sequential' else reversed(range(k))):
      acc = acc + p[..., j]
    return acc
  if order == 'pairwise':
    while p.shape[-1] > 1:
      if p.shape[-1] % 2:
        p = torch.cat([p, torch.zeros_like(p[..., :1])], -1)
      p = p[..., 0::2] + p[..., 1::2]
    return p[..., 0]
  # blocks of 16 products summed exactly and added to the accumulator with one truncation (truncate16), or
  # truncated on their own first and then added with a second truncation (truncate16_blocks)
  acc = torch.zeros(p.shape[:2], dtype=torch.float64)
  for j in range(0, k, 16):
    blk = p[..., j:j + 16].double().sum(-1)
    if order == 'truncate16_blocks':
      blk = _trunc32(blk).double()
    acc = _trunc32(acc + blk).double()
  return acc.float()


def _fast(x, z, gen):
  """x times a random relative error of the fast exp / divide (2 + 1.173|z| ulp each)."""
  d = (torch.rand(x.shape, generator=gen, dtype=torch.float64) * 2 - 1) * (2 + 1.2 * z.double().abs()) * 2.0 ** -23
  return (x.double() * (1 + d)).float()


def _act32(code, z, gen):
  if code == G.RELU:
    return z.clamp_min(0)
  if code == G.SOFTPLUS:
    return _fast(z.clamp_min(0) + torch.log1p(torch.exp(-z.abs())), z, gen)
  if code == G.SILU:
    return _fast(z * torch.sigmoid(z), z, gen)
  return z


def _d1_32(code, z, gen):
  s = _fast(torch.sigmoid(z), z, gen)
  return s * (1 + z * (1 - s)) if code == G.SILU else s


def _bf16(x):
  return x.to(torch.bfloat16)


def _operands(seed, m, n, k, spread=True):
  """bf16 operands with magnitudes over a few binades, and rows of A that cancel exactly against B."""
  gen = torch.Generator().manual_seed(seed)
  a = torch.randn(m, k, generator=gen)
  if spread:
    a = a * torch.exp2(torch.randint(-6, 7, (m, k), generator=gen).float())
  b = torch.randn(n, k, generator=gen) / k ** 0.5
  a, b = _bf16(a), _bf16(b)
  # rows 0-3: the second half of each row is the negated first half against B rows whose halves are equal, so
  # those outputs are exactly zero and their bound is all accumulation error
  h = k // 2
  a[:4, h:] = -a[:4, :h]
  b[:, h:] = b[:, :h]
  return a, b, gen


def _emulate_fwd(a, b, bias, code, order, gen):
  acc = _accumulate(a, b, order)
  z = acc + bias if bias is not None else acc
  y = _act32(code, z, gen)
  return _bf16(y), _bf16(z), y


def _emulate_dgrad(a, b, order, gen, *, rowv=None, colv=None, maskb=None, z=None, code=G.NONE, addend=None,
                   mask_mod=0):
  acc = _accumulate(a, b, order)
  m = a.shape[0]
  rows = torch.arange(m) % mask_mod if mask_mod else torch.arange(m)
  v = acc
  if rowv is not None:   # one fused multiply-add
    v = (rowv.double()[:, None] * colv.double()[None, :] + acc.double()).float()
  if z is not None:
    v = v * _d1_32(code, z.float()[rows], gen)
  elif maskb is not None:
    v = torch.where(maskb[rows], v, torch.zeros_like(v))
  if addend is not None:
    v = v + addend.float()
  return _bf16(v), v


SHAPES = [(37, 48, 64), (130, 64, 192), (20, 32, 320)]


@pytest.mark.parametrize('order', ORDERS)
@pytest.mark.parametrize('code', [G.NONE, G.RELU, G.SOFTPLUS, G.SILU])
@pytest.mark.parametrize('m,n,k', SHAPES)
def test_fwd_emulation_inside_bound(order, code, m, n, k):
  a, b, gen = _operands(m * n + k + code, m, n, k)
  bias = torch.randn(n, generator=gen) * 4
  out, zq, pre = _emulate_fwd(a, b, bias, code, order, gen)
  r = G.ref_fwd(a, b, bias=bias, act_code=code)
  G.check(out, r['out'], r['out_bound'], f'fwd {order}')
  G.check(zq, r['z'], r['z_bound'], f'fwd z {order}')
  G.check(pre, r['out'], r['pre_bound'], f'fwd fp32 {order}')
  if code == G.RELU and n % 32 == 0:
    G.check_bits(G.pack_bits(out.float() > 0), out, r['z'], r['pre_bound'], 'bits')
  # without a bias, the zero-by-cancellation outputs get a bound of the accumulation error alone, far below the
  # bf16 resolution of the products summed
  r0 = G.ref_fwd(a, b)
  absum = G.products(a, b)[1]
  assert float(r0['out'][:4].abs().max()) == 0
  assert (r0['out_bound'][:4] < 1e-4 * absum[:4]).all()


@pytest.mark.parametrize('order', ORDERS)
@pytest.mark.parametrize('variant', ['plain', 'rowv_mask', 'bits_mod_addend', 'softplus_mod', 'silu_rowv_addend'])
@pytest.mark.parametrize('m,n,k', SHAPES)
def test_dgrad_emulation_inside_bound(order, variant, m, n, k):
  if 'bits' in variant and n % 32:
    pytest.skip('mask bits need N % 32 == 0')
  a, b, gen = _operands(7 * m + n + k, m, n, k)
  kw, emu = {}, {}
  mod = 0
  if 'mod' in variant:
    mod = m // 3 + 1
    kw['mask_mod'] = emu['mask_mod'] = mod
  mrows = mod or m
  if 'rowv' in variant:
    kw['rowv'] = emu['rowv'] = torch.randn(m, generator=gen)
    kw['colv'] = emu['colv'] = torch.randn(n, generator=gen)
  if variant == 'rowv_mask':
    mask = _bf16(torch.randn(mrows, n, generator=gen))
    kw['mask'], emu['maskb'] = mask, mask.float() > 0
  if 'bits' in variant:
    maskb = torch.rand(mrows, n, generator=gen) > 0.5
    kw['maskbits'], emu['maskb'] = G.pack_bits(maskb, n // 32 + 1), maskb
  code = G.SOFTPLUS if 'softplus' in variant else G.SILU if 'silu' in variant else G.NONE
  if code:
    z = _bf16(torch.randn(mrows, n, generator=gen) * 3)
    kw['z'] = emu['z'] = z
    kw['act_code'] = emu['code'] = code
  if 'addend' in variant:
    kw['addend'] = emu['addend'] = _bf16(torch.randn(m, n, generator=gen))
  out, pre = _emulate_dgrad(a, b, order, gen, **emu)
  r = G.ref_dgrad(a, b, **kw)
  G.check(out, r['out'], r['out_bound'], f'dgrad {variant} {order}')
  G.check(pre, r['out'], r['pre_bound'], f'dgrad fp32 {variant} {order}')
  init = torch.randn(n, generator=gen)
  s, sb = G.colsum_ref(r['out'], r['pre_bound'], init)
  G.check(pre.sum(0) + init, s, sb, 'colsum of the fp32 values')
  s1, sb1 = G.colsum_ref(r['out'], r['pre_bound'], init, rounded=True)
  G.check(out.float().sum(0) + init, s1, sb1, 'colsum of the bf16 output')


@pytest.mark.parametrize('order', ORDERS)
def test_wgrad_emulation_inside_bound(order):
  gen = torch.Generator().manual_seed(5)
  r_, mo, n = 37, 40, 64
  x = _bf16(torch.randn(r_, mo, generator=gen))
  dy = _bf16(torch.randn(r_, n, generator=gen))
  w = torch.randn(r_, generator=gen)
  init = torch.randn(mo, n, generator=gen)
  binit, ainit = torch.randn(n, generator=gen), torch.randn(mo, generator=gen)
  ref = G.ref_wgrad(x, dy, init=init, bsum_init=binit, side_w=w, side_aw_init=ainit)
  got = _accumulate(x.T.contiguous(), dy.T.contiguous(), order) + init
  G.check(got, *ref['out'], f'wgrad {order}')
  G.check(dy.float().sum(0) + binit, *ref['bsum'], 'bsum')
  G.check((x.float() * w[:, None]).sum(0) + ainit, *ref['side_aw'], 'side_aw')


# ---------------------------------------------------------------------------------------------- sensitivity
def _flagged(got, value, bound):
  try:
    G.check(got, value, bound, 'mutation')
  except AssertionError:
    return True
  return False


M, N, K = 200, 128, 256   # two row tiles, the second ragged (rows 128-199)


@pytest.fixture(scope='module')
def fwd_case():
  a, b, gen = _operands(11, M, N, K, spread=False)
  bias = torch.randn(N, generator=gen)
  r = G.ref_fwd(a, b, bias=bias, act_code=G.NONE)
  out, _, _ = _emulate_fwd(a, b, bias, G.NONE, 'sequential', gen)
  G.check(out, r['out'], r['out_bound'], 'unmutated')
  return a, b, bias, r, out, gen


def test_flags_dropped_k_block(fwd_case):
  a, b, bias, r, out, _ = fwd_case
  bad = out.clone()
  a2 = a[64:128].clone()
  a2[:, 128:192] = 0            # k-block 2 of the 64 x 64 block at rows 64-127, columns 64-127
  bad[64:128, 64:128] = _bf16(a2.float() @ b[64:128].float().T + bias[64:128])
  assert _flagged(bad, r['out'], r['out_bound'])


def test_flags_missing_bias_column(fwd_case):
  a, b, bias, r, out, _ = fwd_case
  bad = out.clone()
  col = int(bias.abs().argmax())
  bad[:, col] = _bf16(out[:, col].float() - bias[col])
  assert _flagged(bad, r['out'], r['out_bound'])


def test_flags_shifted_ragged_tile(fwd_case):
  _, _, _, r, out, _ = fwd_case
  bad = out.clone()
  bad[129:M] = out[128:M - 1]
  assert _flagged(bad, r['out'], r['out_bound'])


def test_flags_flipped_mask_bit():
  a, b, gen = _operands(12, M, N, K, spread=False)
  bias = torch.randn(N, generator=gen)
  r = G.ref_fwd(a, b, bias=bias, act_code=G.RELU)
  out, _, _ = _emulate_fwd(a, b, bias, G.RELU, 'sequential', gen)
  words = G.pack_bits(out.float() > 0)
  G.check_bits(words, out, r['z'], r['pre_bound'], 'unmutated')
  bad = words.clone()
  bad[150, 3] ^= 1 << 7
  with pytest.raises(AssertionError):
    G.check_bits(bad, out, r['z'], r['pre_bound'], 'mutated')
  # DGRAD reading the flipped bit: the output at that element is masked wrongly
  maskb = torch.rand(M, N, generator=gen) > 0.5
  dy = _bf16(torch.randn(M, K, generator=gen))
  rd = G.ref_dgrad(dy, b, maskbits=G.pack_bits(maskb))
  i, j = 150, 3 * 32 + 7
  flipped = maskb.clone()
  flipped[i, j] = ~flipped[i, j]
  got, _ = _emulate_dgrad(dy, b, 'sequential', gen, maskb=flipped)
  assert abs(float(rd['out'][i, j])) > 0 or abs(float(got[i, j])) > 0
  assert _flagged(got, rd['out'], rd['out_bound'])


def test_flags_missing_rank1_row():
  a, b, gen = _operands(13, M, N, K, spread=False)
  rowv, colv = torch.randn(M, generator=gen), torch.randn(N, generator=gen)
  r = G.ref_dgrad(a, b, rowv=rowv, colv=colv)
  out, _ = _emulate_dgrad(a, b, 'sequential', gen, rowv=rowv, colv=colv)
  G.check(out, r['out'], r['out_bound'], 'unmutated')
  bad = out.clone()
  i = int(rowv.abs().argmax())
  bad[i] = _bf16(out[i].float() - rowv[i] * colv)
  assert _flagged(bad, r['out'], r['out_bound'])


@pytest.mark.parametrize('shift', [1, -1])
@pytest.mark.parametrize('code', [G.SOFTPLUS, G.SILU])
def test_flags_z_row_off_by_one(code, shift):
  mod = 67
  a, b, gen = _operands(14, 3 * mod, N, K, spread=False)
  z = _bf16(torch.randn(mod, N, generator=gen) * 2)
  r = G.ref_dgrad(a, b, z=z, act_code=code, mask_mod=mod)
  out, _ = _emulate_dgrad(a, b, 'sequential', gen, z=z, code=code, mask_mod=mod)
  G.check(out, r['out'], r['out_bound'], 'unmutated')
  bad, _ = _emulate_dgrad(a, b, 'sequential', gen, z=torch.roll(z, shift, 0), code=code, mask_mod=mod)
  assert _flagged(bad, r['out'], r['out_bound'])


def test_flags_addend_twice():
  a, b, gen = _operands(15, M, N, K, spread=False)
  add = _bf16(torch.randn(M, N, generator=gen))
  r = G.ref_dgrad(a, b, addend=add)
  out, _ = _emulate_dgrad(a, b, 'sequential', gen, addend=add)
  G.check(out, r['out'], r['out_bound'], 'unmutated')
  bad = out.clone()
  i, j = divmod(int(add.float().abs().argmax()), N)
  bad[i, j] = _bf16(out[i, j].float() + add[i, j].float())
  assert _flagged(bad, r['out'], r['out_bound'])


def test_flags_colsum_tile_twice():
  a, b, gen = _operands(16, M, N, K, spread=False)
  r = G.ref_dgrad(a, b)
  _, pre = _emulate_dgrad(a, b, 'sequential', gen)
  init = torch.zeros(N)
  s, sb = G.colsum_ref(r['out'], r['pre_bound'], init)
  got = pre.sum(0)
  G.check(got, s, sb, 'unmutated')
  bad = got.clone()
  bad[64:128] += pre[0:128, 64:128].sum(0)     # the tile of rows 0-127, columns 64-127, summed twice
  assert _flagged(bad, s, sb)


def test_embed_padding():
  v, buf = G.embed((5, 16), torch.bfloat16, 'cpu', extra_rows=1, extra_cols=6, col0=2, fill='sentinel')
  assert v.shape == (5, 16) and v.stride(0) == 22 and G.padding_intact(v, buf)
  v.fill_(1)
  assert G.padding_intact(v, buf)
  buf[0, 0] = 0
  assert not G.padding_intact(v, buf)
  x, xb = G.embed((7,), torch.float32, 'cpu', extra_cols=4, col0=2)
  assert torch.isnan(xb).all() and x.shape == (7,)
  w = torch.tensor(np.random.default_rng(0).uniform(size=(3, 64)) > 0.5)
  assert torch.equal(G.unpack_bits(G.pack_bits(w, 3), 64), w)
