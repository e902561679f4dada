"""fp64 reference of the layer-chained 256-wide trunk (csrc/chain.cu, mnrf_mlp_chain) with a per-element bound, the
kernel's schedule arithmetic, and an exact-arithmetic data generator.

ref_chain takes the layer dicts ops.chain_desc takes.  Each chained layer is one Dense layer of tests/gemm_ref.py on
the chain's own stored bf16 input of that layer, so every bound is gemm_ref's:
  - FWD: A = [resident | streamed columns], B = weight columns [res_kb0 64, + 256) ++ [stream_kb0 64, + n_stream 64),
    gemm_ref.ref_fwd with the bias and ReLU; the fused head is heads_ref.head_fwd on the last layer's stored output;
  - BWD: the same A and B, gemm_ref.ref_dgrad with the layer's mask bits, gemm_ref.colsum_ref for the column sums
    (taken of the masked fp32 values before their bf16 rounding).
The resident operand is the previous layer's output as the kernel stored it.  A layer the launch did not store has
no such input: there the reference rounds its own fp64 value to bf16, which is exact on exact data only.

schedule mirrors the kernel's arithmetic: segments of at most CH_SEG k-blocks, the streamed blocks of each segment
(both warpgroups' blocks pass through a ring of CH_SRING), units of 128 rows, the persistent grid and the shape of
the last unit.

make_data (exact=True) draws operands on which every fp32 sum the kernel forms is exact: features, weights, biases, dy, head
weights and initial column sums are small integers; a weight row has a few signed +-1 entries at permutation-like
columns, so each output column depends on its own few inputs.  A pre-activation is then an integer below 2^24, exact
in fp32 whatever the summation order; the stored activation is its bf16 rounding (round to nearest even, exact
below 257), so activations, mask bits, head outputs and column sums equal the fp64 reference bit for bit, and a
misrouted row, column, k-block, ring slot or swizzle chunk shows whatever its magnitude.  check_exact asserts that
the data kept that promise.

Pure torch in float64: runs on the CPU or on CUDA tensors, and never loads the CUDA library.
"""
import torch

import gemm_ref as G
import heads_ref as H

W = 256                 # layer width (include/mnrf.h: width must be 256)
CH_ROWS = 128           # rows of a unit
CH_SEG = 4              # k-blocks of a segment (at most)
CH_SRING = 3            # streamed-operand ring
MAX_LAYERS = 8          # MNRF_CHAIN_MAX_LAYERS
FWD, BWD = 0, 1         # MNRF_CHAIN_FWD / _BWD
EXACT_LIMIT = 2.0 ** 24


def kblocks(ly):
  """Weight k-blocks the layer's descriptor spans (the kernel's K of the weight tensor map)."""
  ns, nr = ly.get('n_stream', 0), ly.get('n_res', 0)
  return max(ly.get('stream_kb0', 0) + ns if ns else 0, ly.get('res_kb0', 0) + nr if nr else 0)


def operands(ly, stream, resident):
  """(A [M, K], B [256, K]) of one chained layer: the resident operand then the streamed k-blocks, against the weight
  columns in the same order (the kernel's k-block order)."""
  a, b = [], []
  w = ly['w'][:W]
  if ly.get('n_res', 0):
    a.append(resident)
    c0 = ly.get('res_kb0', 0) * 64
    b.append(w[:, c0:c0 + 64 * ly['n_res']])
  ns = ly.get('n_stream', 0)
  if ns:
    s0 = ly.get('stream_col0', 0)
    a.append(stream[:, s0:s0 + 64 * ns])
    c0 = ly.get('stream_kb0', 0) * 64
    b.append(w[:, c0:c0 + 64 * ns])
  return torch.cat(a, 1), torch.cat(b, 1)


def ref_chain(mode, m, layers, stream, *, stored=None, head_w=None, head_b=None, colsum_init=None):
  """fp64 outputs of one chained launch, layer by layer (a generator, so that only one layer's fp64 tensors live at
  a time).  stored[j]: the kernel's stored output of layer j (bf16 [m, 256]) or None; colsum_init[j]: the initial
  value of layer j's column sums.  Yields (j, dict): FWD out, out_bound, z, z_bound (gemm_ref.ref_fwd), and on the
  last layer with head_w, head (value, bound); BWD out, out_bound, pre_bound (gemm_ref.ref_dgrad) and, with
  colsum_init[j], colsum (value, bound)."""
  stored = stored or [None] * len(layers)
  prev = None
  for j, ly in enumerate(layers):
    a, b = operands(ly, stream[:m] if stream is not None else None, prev)
    if mode == FWD:
      r = G.ref_fwd(a, b, bias=ly['bias'], act_code=G.RELU)
    else:
      r = G.ref_dgrad(a, b, maskbits=ly['maskbits'][:m] if ly.get('maskbits') is not None else None)
      if colsum_init is not None and colsum_init[j] is not None:
        r['colsum'] = G.colsum_ref(r['out'], r['pre_bound'], colsum_init[j].to(a.device))
    cur = stored[j] if stored[j] is not None else r['out'].to(torch.bfloat16)
    if mode == FWD and j == len(layers) - 1 and head_w is not None:
      r['head'] = H.head_fwd(cur, head_w, head_b)
    yield j, r
    prev = cur


# ---------------------------------------------------------------------------------------------- schedule
def segments(ly):
  """Streamed k-blocks of each segment of a layer (the kernel's `ns`, 0 for a resident segment)."""
  nr, ns = ly.get('n_res', 0), ly.get('n_stream', 0)
  nk = nr + ns
  return [max(0, min(s0 + CH_SEG, nk) - max(s0, nr)) for s0 in range(0, nk, CH_SEG)]


def schedule(mode, layers, m, sms, head_n=0, colsum=None, maskbits=None):
  """The kernel's schedule arithmetic for one launch: dict of segs (segments per layer), streamed (streamed blocks
  of each segment, per layer), ring_wrap (a warpgroup's streamed blocks of one segment outnumber the ring), units,
  grid, min / max units per CTA, last (shape of the last unit: 'both' warpgroups have rows, 'wg0' only, or 'm<=64')
  and instance (the kernel instance and the epilogue options it runs)."""
  units = -(-m // CH_ROWS)
  grid = min(units, sms)
  last_rows = m - (units - 1) * CH_ROWS
  if m <= 64:
    last = 'm<=64'
  else:
    last = 'wg0' if last_rows <= 64 else 'both'
  streamed = [segments(ly) for ly in layers]
  if mode == FWD:
    inst = ('fwd', f'nh{head_n}' if head_n else 'nohead')
  else:
    has_cs = any(ly.get('colsum') is not None for ly in layers) if colsum is None else colsum
    has_mb = any(ly.get('maskbits') is not None for ly in layers) if maskbits is None else maskbits
    inst = ('bwd', 'colsum' if has_cs else 'nocolsum', 'maskbits' if has_mb else 'nomask')
  return dict(segs=[len(s) for s in streamed], streamed=streamed,
              ring_wrap=any(ns > CH_SRING for s in streamed for ns in s), units=units, grid=grid,
              min_per_cta=units // grid, max_per_cta=-(-units // grid), last=last, instance=inst)


# ---------------------------------------------------------------------------------------------- exact data
def sparse_weights(n_in_cols, nnz, gen, *, scale=1):
  """[256, n_in_cols] with nnz signed entries of magnitude `scale` per row, at columns that follow a permutation
  (row n uses columns perm[(7 n + 97 t) % n_in_cols], t < nnz), so each output has its own few inputs."""
  perm = torch.randperm(n_in_cols, generator=gen)
  w = torch.zeros(W, n_in_cols, dtype=torch.float64)
  rows = torch.arange(W)
  for t in range(nnz):
    cols = perm[(rows * 7 + t * 97) % n_in_cols]
    sign = torch.randint(0, 2, (W,), generator=gen) * 2 - 1
    w[rows, cols] += sign * scale
  return w


def ints(shape, lo, hi, gen):
  return torch.randint(lo, hi + 1, shape, generator=gen).double()


def check_exact(value, what, abs_sum=None):
  """Assert that exact data stayed exact: every fp64 value an integer, and it (or abs_sum, the sum of the magnitudes
  of its terms, which bounds every partial sum in any order) below 2^24."""
  v = value.double()
  assert bool(torch.isfinite(v).all()), f'{what}: exact data produced non-finite values'
  big = v.abs() if abs_sum is None else abs_sum
  assert float(big.max()) < EXACT_LIMIT if big.numel() else True, f'{what}: exact data outgrew the fp32 integers'
  assert bool((v == torch.round(v)).all()), f'{what}: exact data left the integers'


def spec_layer(n_res=0, res_kb0=0, n_stream=0, stream_col0=0, stream_kb0=0, *, out=True, maskbits=True,
               colsum=False, extra_k=0):
  """One layer of a case: operand layout (as mnrf_chain_layer), which outputs it has, and extra_k weight columns
  past the descriptor's K (a pitch ldw > K)."""
  return dict(n_res=n_res, res_kb0=res_kb0, n_stream=n_stream, stream_col0=stream_col0, stream_kb0=stream_kb0,
              out=out, maskbits=maskbits, colsum=colsum, extra_k=extra_k)


def make_data(mode, m, lspecs, stream_cols, *, head_n=0, head_b=True, exact=True, seed=0, amp=8, nnz=2):
  """The operands of a case as plain CPU tensors: stream [m, stream_cols] bf16 (features, or dy for BWD), w[j]
  [256, K_j + extra_k] bf16 (the weight columns outside the layer's k-blocks are NaN: never read), bias[j] fp32
  (FWD), masks[j] int32 [m, 8] (BWD), colsum_init[j] fp32 [256] (BWD), head_w [head_n, 256] fp32 (bf16 values) and
  head_b [head_n] fp32.  exact: the integer data of the module docstring; otherwise normal draws of the magnitudes
  the models see."""
  gen = torch.Generator().manual_seed(seed)
  bf = torch.bfloat16
  d = dict(w=[], bias=[], masks=[], colsum_init=[])
  if exact:
    d['stream'] = ints((m, stream_cols), -amp if mode == FWD else -2, amp if mode == FWD else 2, gen).to(bf)
  else:
    d['stream'] = torch.randn(m, stream_cols, generator=gen).to(bf)
  for ls in lspecs:
    kb = kblocks(ls)
    w = torch.full((W, kb * 64 + ls['extra_k']), float('nan'), dtype=torch.float64)
    used = []
    if ls['n_res']:
      used += list(range(ls['res_kb0'] * 64, (ls['res_kb0'] + ls['n_res']) * 64))
    if ls['n_stream']:
      used += list(range(ls['stream_kb0'] * 64, (ls['stream_kb0'] + ls['n_stream']) * 64))
    used = torch.tensor(used)
    if exact:
      w[:, used] = sparse_weights(len(used), nnz, gen)
    else:
      scale = (2.0 / len(used)) ** 0.5 if mode == FWD else 1 / 16
      w[:, used] = torch.randn(W, len(used), generator=gen, dtype=torch.float64) * scale
    d['w'].append(w.to(bf))
    if mode == FWD:
      d['bias'].append(ints((W,), -2, 2, gen).float() if exact else torch.randn(W, generator=gen) * 0.1)
    else:
      bits = torch.rand(m, W, generator=gen) > 0.5
      d['masks'].append(G.pack_bits(bits))
      d['colsum_init'].append(ints((W,), -3, 3, gen).float() if exact else torch.randn(W, generator=gen))
  if head_n:
    hw = ints((head_n, W), -2, 2, gen) if exact else torch.randn(head_n, W, generator=gen, dtype=torch.float64) / 16
    d['head_w'] = hw.to(bf).float()
    d['head_b'] = (ints((head_n,), -4, 4, gen).float() if exact else torch.randn(head_n, generator=gen)) \
        if head_b else None
  return d


def layer_dicts(mode, lspecs, data, outs=None, bits=None, colsums=None):
  """The layer dicts of ops.chain_desc for a case's data and output views (outs[j] / bits[j] / colsums[j], None
  where the layer has none)."""
  layers = []
  for j, ls in enumerate(lspecs):
    ly = {k: ls[k] for k in ('n_res', 'res_kb0', 'n_stream', 'stream_col0', 'stream_kb0')}
    ly['w'] = data['w'][j]
    if mode == FWD:
      ly['bias'] = data['bias'][j]
      if bits is not None and bits[j] is not None:
        ly['maskbits'] = bits[j]
    else:
      if ls['maskbits']:
        ly['maskbits'] = data['masks'][j]
      if colsums is not None and colsums[j] is not None:
        ly['colsum'] = colsums[j]
    if outs is not None and outs[j] is not None:
      ly['out'] = outs[j]
    layers.append(ly)
  return layers


# ---------------------------------------------------------------------------------------------- checking a launch
def _exact_equal(got, want, what):
  g, w = got.double(), want.double()
  bad = g != w
  if bool(bad.any()):
    idx = tuple(int(i) for i in torch.nonzero(bad)[0])
    raise AssertionError(f'{what}: {int(bad.sum())} / {bad.numel()} differ from fp64 on exact data, first at {idx}: '
                         f'got {float(g[idx]):.9g}, fp64 {float(w[idx]):.9g}')
  return 0.0


def check_launch(mode, m, layers, stream, got, *, exact, head_w=None, head_b=None, colsum_init=None):
  """Check one chained launch against fp64, layer by layer.  got: dict of the kernel's outputs, outs[j] (bf16
  [m, 256] or None), bits[j] (int32 mask words or None), head ([m, head_n] fp32) and colsums[j] (fp32 [256] or
  None).  exact: bit for bit (the data of make_data(exact=True), whose exactness is asserted on the way); otherwise
  every element within its bound, which needs every layer's input stored.  Returns the worst err / bound ratio of
  each output."""
  outs, bits = got['outs'], got.get('bits') or [None] * len(layers)
  colsums = got.get('colsums') or [None] * len(layers)
  worst = {}
  for j, r in ref_chain(mode, m, layers, stream, stored=outs, head_w=head_w, head_b=head_b,
                        colsum_init=colsum_init if colsum_init is not None else [None] * len(layers)):
    name = f'layer {j}'
    if exact:
      check_exact(r['z'] if mode == FWD else r['out'], name)
    if outs[j] is not None:
      if exact:
        worst[name] = _exact_equal(outs[j], r['out'].to(torch.bfloat16), name)
      else:
        worst[name] = G.check(outs[j], r['out'], r['out_bound'], name)
    if mode == FWD and bits[j] is not None:
      if exact:
        assert torch.equal(G.unpack_bits(bits[j], W), r['z'] > 0), f'{name}: mask bits differ from the fp64 sign'
      else:
        stored = outs[j] if outs[j] is not None else r['out'].to(torch.bfloat16)
        G.check_bits(bits[j], stored, r['z'], r['pre_bound'], f'{name} mask bits')
    if 'head' in r and got.get('head') is not None:
      val, bound = r['head']
      if exact:
        check_exact(val, 'head')
        worst['head'] = _exact_equal(got['head'], val, 'head')
      else:
        worst['head'] = G.check(got['head'], val, bound, 'head')
    if 'colsum' in r and colsums[j] is not None:
      val, bound = r['colsum']
      if exact:
        check_exact(val, f'{name} colsum', abs_sum=r['out'].abs().sum(0) + colsum_init[j].to(val.device).double().abs())
        worst[f'{name} colsum'] = _exact_equal(colsums[j], val, f'{name} colsum')
      else:
        worst[f'{name} colsum'] = G.check(colsums[j], val, bound, f'{name} colsum')
  return worst
