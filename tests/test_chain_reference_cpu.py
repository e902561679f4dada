"""The fp64 checker of tests/chain_ref.py is sound and sensitive, and the GPU case matrix reaches every schedule class.
CPU only.

Soundness: the arithmetic of csrc/chain.cu emulated in fp32 -- rows padded to 128-row units, the resident k-blocks
then the streamed ones summed k16 step by k16 step, bias, ReLU and the mask bit from the fp32 pre-activation, bf16
round to nearest even, the head from each quad lane's columns and a two-step butterfly, and the column sums of
the backward chain by per-warp butterflies over 16 rows, shared-memory atomics per CTA and global atomics -- passes
check_launch on random data, and on exact data equals fp64 bit for bit.
Sensitivity: each of the seeded bugs below, applied to the emulation, is flagged.
"""
import pytest
import torch

import chain_ref as R
import gemm_ref as G
import test_gpu_chain_fp64 as GPU

W = R.W
BF = torch.bfloat16


# ---------------------------------------------------------------------------------------------- emulation
def _acc32(a, b):
  """fp32 accumulation of A B^T k16 step by k16 step (each step's 16 exact products summed once, then added)."""
  acc = torch.zeros(a.shape[0], b.shape[0], dtype=torch.float32)
  ad, bd = a.double(), b.double()
  for k0 in range(0, a.shape[1], 16):
    acc = (acc.double() + (ad[:, k0:k0 + 16] @ bd[:, k0:k0 + 16].T).float().double()).float()
  return acc


def _units(m):
  return -(-m // R.CH_ROWS)


def _pad(x, rows):
  out = torch.zeros(rows, x.shape[1], dtype=x.dtype)
  out[:x.shape[0]] = x
  return out


def _swizzle_bug(x):
  """The epilogue's swizzle without the row term: within every 64-column block of row r, 16-byte chunk c holds the
  chunk c ^ (r & 7) the next layer reads."""
  rows = x.shape[0]
  chunks = x.reshape(rows, W // 64, 8, 8)
  idx = torch.arange(8)[None, :] ^ (torch.arange(rows) % 8)[:, None]
  return torch.gather(chunks, 2, idx[:, None, :, None].expand(rows, W // 64, 8, 8)).reshape(rows, W)


def _colsum32(v, init, sms, bug=None):
  """Column sums as the kernel adds them: a warp's 16 rows (rows r and r + 8 per lane, then lanes xor 4, 8, 16),
  the warps' sums into the CTA's shared sums, the CTAs' into init."""
  units = v.shape[0] // R.CH_ROWS
  grid = min(units, sms)
  t = v.reshape(units, 2, 4, 2, 8, W)                       # unit, warpgroup, warp, h, lane >> 2, column
  s = t[:, :, :, 0] + t[:, :, :, 1]
  for sh in (1, 2, 4):
    s = s + s[:, :, :, torch.arange(8) ^ sh]
  warp = s[:, :, :, 0]                                      # [units, 2, 4, W]
  if bug == 'colsum_warp_missing':
    warp[:, 1, 3] = 0
  total = init.float().clone()
  for cta in range(grid):
    sh_sum = torch.zeros(W)
    for u in range(cta, units, grid):
      for c in range(2):
        for w in range(4):
          sh_sum = sh_sum + warp[u, c, w]
    total = total + sh_sum
  return total


def emulate(mode, m, layers, stream, *, head_w=None, head_b=None, colsum_init=None, sms=132, bug=None, render=False):
  """fp32 emulation of one launch (see the module docstring) with an optional seeded bug.  Returns the got dict of
  chain_ref.check_launch: every layer's output, mask words (FWD), head and column sums (BWD)."""
  rows = _units(m) * R.CH_ROWS
  outs, bits, colsums = [], [], []
  head = None
  prev = None
  n = len(layers)
  for j, ly in enumerate(layers):
    ly = dict(ly)
    if bug == 'stream_kb0' and ly.get('n_stream') and ly.get('n_res'):
      ly['stream_kb0'] = ly['stream_kb0'] + 1 if ly['stream_kb0'] == 0 else ly['stream_kb0'] - 1
    if bug == 'stream_col0_ignored':
      ly['stream_col0'] = 0
    if bug == 'res_kb0_ignored':
      ly['res_kb0'] = 0
    st = _pad(stream[:m], rows) if stream is not None else None
    a, b = R.operands(ly, st, prev)
    if bug == 'ring_slot_at_wrap' and ly.get('n_stream', 0) > R.CH_SRING:
      # the first streamed block past the ring's end is read from the slot before the right one
      k0 = ly.get('n_res', 0) * 64 + R.CH_SRING * 64
      a = a.clone()
      a[:, k0:k0 + 64] = a[:, k0 - 64:k0]
    acc = _acc32(a, b)
    if mode == R.FWD:
      v = acc if (bug == 'no_bias_last_render' and render and j == n - 1) else (acc + ly['bias'].float())
      bit = v > 0
      if bug == 'mask_bit_shift':
        bit = torch.roll(bit, 1, 1)
      o = torch.relu(v).to(BF)
    else:
      v = acc
      if ly.get('maskbits') is not None and bug != 'mask_not_zeroed':
        keep = _pad(G.unpack_bits(ly['maskbits'][:m], W), rows)
        v = torch.where(keep, v, torch.zeros_like(v))
      o = v.to(BF)
      if colsum_init is not None and colsum_init[j] is not None:
        colsums.append(_colsum32(v, colsum_init[j], sms, bug))
      else:
        colsums.append(None)
    if bug == 'swizzle_row_term':
      o = _swizzle_bug(o)
    stored = o.clone()
    u_last = rows - R.CH_ROWS
    if bug == 'ragged_rows_dropped' and m - u_last > 64:
      stored[u_last + 64:] = 0
    if bug == 'warpgroups_swapped':
      stored = stored.reshape(-1, 2, 64, W).flip(1).reshape(rows, W)
    outs.append(stored[:m])
    if mode == R.FWD:
      bits.append(G.pack_bits(bit[:m]))
      if j == n - 1 and head_w is not None:
        x = (torch.relu(v) if bug == 'head_unrounded' else o.float())[:m]
        hw = head_w.float()
        part = torch.zeros(m, hw.shape[0], 4)
        for i in range(W // 8):
          for q in range(4):
            c = 8 * i + 2 * q
            part[:, :, q] = part[:, :, q] + (x[:, c:c + 1] * hw[:, c] + x[:, c + 1:c + 2] * hw[:, c + 1])
        part = part + part[:, :, [1, 0, 3, 2]]
        part = part + part[:, :, [2, 3, 0, 1]]
        head = part[:, :, 0] + (head_b.float() if head_b is not None else 0)
    prev = stored
  return dict(outs=outs, bits=bits if mode == R.FWD else None, head=head, colsums=colsums if mode == R.BWD else None)


# ---------------------------------------------------------------------------------------------- cases
def _case(mode, m, lspecs, stream_cols, *, exact, head_n=1, head_b=True, seed=0, amp=8):
  d = R.make_data(mode, m, lspecs, stream_cols, head_n=head_n if mode == R.FWD else 0, head_b=head_b, exact=exact,
                  seed=seed, amp=amp)
  layers = R.layer_dicts(mode, lspecs, d)
  init = d['colsum_init'] if mode == R.BWD and any(ls['colsum'] for ls in lspecs) else None
  if init is not None:
    init = [c if ls['colsum'] else None for c, ls in zip(init, lspecs)]
  return d, layers, init


SL = R.spec_layer
CPU_CASES = {
    # PropMLP layout: 8 streamed k-blocks (two segments, the ring wraps), ragged: the last unit's rows in both
    # warpgroups
    'prop': (R.FWD, 200, [SL(n_stream=8)] + [SL(n_res=4)] * 3, 512),
    # a skip layer (resident + streamed) at weight k-block 4, features at column 128 of a wider tensor, 8 layers
    'skip': (R.FWD, 130, [SL(n_stream=2, stream_col0=128)] + [SL(n_res=4)] * 4 +
             [SL(n_res=4, n_stream=2, stream_col0=128, stream_kb0=4)] + [SL(n_res=4)] * 2, 320),
    # resident operand at weight k-block 2 after the streamed k-blocks 0-1
    'res_kb0': (R.FWD, 100, [SL(n_stream=4)] + [SL(n_res=4, res_kb0=2, n_stream=2, stream_col0=64)], 256),
    # backward with column sums; a later layer that streams
    'bwd': (R.BWD, 200, [SL(n_stream=4, colsum=True), SL(n_res=4, colsum=True),
                         SL(n_res=4, n_stream=4, stream_col0=256, stream_kb0=4, colsum=True)], 512),
}


@pytest.mark.parametrize('exact', [False, True])
@pytest.mark.parametrize('name', sorted(CPU_CASES))
def test_emulation_passes(name, exact):
  mode, m, lspecs, cols = CPU_CASES[name]
  for head_n in ((1, 4) if mode == R.FWD else (0,)):
    d, layers, init = _case(mode, m, lspecs, cols, exact=exact, head_n=head_n, seed=m)
    got = emulate(mode, m, layers, d['stream'], head_w=d.get('head_w'), head_b=d.get('head_b'), colsum_init=init)
    worst = R.check_launch(mode, m, layers, d['stream'], got, exact=exact, head_w=d.get('head_w'),
                           head_b=d.get('head_b'), colsum_init=init)
    if exact:
      assert all(v == 0 for v in worst.values()), worst


# seeded bug -> the case that exposes it
BUGS = {
    'stream_kb0': 'skip', 'stream_col0_ignored': 'skip', 'res_kb0_ignored': 'res_kb0', 'ragged_rows_dropped': 'prop',
    'warpgroups_swapped': 'prop', 'mask_bit_shift': 'prop', 'colsum_warp_missing': 'bwd',
    'no_bias_last_render': 'prop', 'head_unrounded': 'prop', 'ring_slot_at_wrap': 'prop',
    'mask_not_zeroed': 'bwd', 'swizzle_row_term': 'skip',
}


@pytest.mark.parametrize('bug', sorted(BUGS))
def test_seeded_bug_is_caught(bug):
  """Each bug is flagged on exact data, bit for bit.  Where the bug changes the data path it also fails the fp64
  bound on random data; the rounding-only bugs (the head on the unrounded activation) need the exact check."""
  mode, m, lspecs, cols = CPU_CASES[BUGS[bug]]
  # amp 64: activations past 256, where the bf16 rounding of the stored activation drops bits
  d, layers, init = _case(mode, m, lspecs, cols, exact=True, seed=m, amp=64 if bug == 'head_unrounded' else 8)
  render = bug == 'no_bias_last_render'
  got = emulate(mode, m, layers, d['stream'], head_w=d.get('head_w'), head_b=d.get('head_b'), colsum_init=init,
                bug=bug, render=render)
  if render:      # the render form stores the last layer only
    got['outs'] = [None] * (len(layers) - 1) + got['outs'][-1:]
    got['bits'] = None
  with pytest.raises(AssertionError):
    R.check_launch(mode, m, layers, d['stream'], got, exact=True, head_w=d.get('head_w'), head_b=d.get('head_b'),
                   colsum_init=init)
  print(f'\n[chain seeded bug] {bug}: caught')


def test_check_bits_subnormal_rule():
  """A set bit over a stored 0 only where the fp32 pre-activation is in (0, 2^-134]; stored > 0 needs the bit."""
  z = torch.tensor([[0.0, -0.0, 2.0 ** -140, -2.0 ** -140, 2.0 ** -134, 2.0 ** -126] + [1.0] * 26], dtype=torch.float64)
  stored = G.act(G.RELU, z).to(BF)
  assert float(stored[0, 4]) == 0 and float(stored[0, 5]) > 0
  bound = torch.zeros_like(z)
  G.check_bits(G.pack_bits(z > 0), stored, z, bound, 'sign of the fp32 pre-activation')
  for col in (0, 1, 3):            # a bit where the pre-activation is not positive
    bad = (z > 0).clone()
    bad[0, col] = True
    with pytest.raises(AssertionError):
      G.check_bits(G.pack_bits(bad), stored, z, bound, 'mutated')
  bad = (z > 0).clone()
  bad[0, 5] = False                # a positive stored output without its bit
  with pytest.raises(AssertionError):
    G.check_bits(G.pack_bits(bad), stored, z, bound, 'mutated')


# ---------------------------------------------------------------------------------------------- coverage
CLASSES = ({'segs1', 'segs2', 'segs3+', 'ring_wrap', 'one_unit', 'several_per_cta', 'ragged_grid', 'last_both',
            'last_wg0', 'last_m<=64'} |
           {('fwd', 'nh1'), ('fwd', 'nh4'), ('fwd', 'nohead')} |
           {('bwd', cs, mb) for cs in ('colsum', 'nocolsum') for mb in ('maskbits', 'nomask')})


def _classes(sch):
  got = {sch['instance'], f"last_{sch['last']}"}
  for s in sch['segs']:
    got.add('segs1' if s == 1 else 'segs2' if s == 2 else 'segs3+')
  if sch['ring_wrap']:
    got.add('ring_wrap')
  if sch['units'] == 1:
    got.add('one_unit')
  if sch['max_per_cta'] > 1:
    got.add('several_per_cta')
  if sch['units'] % sch['grid']:
    got.add('ragged_grid')
  return got


@pytest.mark.parametrize('sms', [132, 114])
def test_every_schedule_class_has_cases(sms):
  """Every class is reached by a case of the GPU matrix, with the case list built for that SM count."""
  seen = set()
  for c in GPU.cases(sms):
    for mode, lspecs, head_n in GPU.launches(c):
      sch = R.schedule(mode, lspecs, c['M'], sms, head_n=head_n,
                       colsum=any(ls['colsum'] for ls in lspecs), maskbits=any(ls['maskbits'] for ls in lspecs))
      seen |= _classes(sch)
  assert not CLASSES - seen, f'schedule classes without a case: {sorted(CLASSES - seen, key=str)}'
