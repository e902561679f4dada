"""fp64 reference of the Dense-layer GEMM (mnrf_gemm / mnrf_gemm_wgrad) with a per-element bound.

`ref_fwd / ref_dgrad / ref_wgrad` take exactly the operands the kernel gets (bf16 A / B, fp32 bias, rowv, colv, bf16
mask or packed mask bits, addend, z) and return the fp64 value of every output together with a bound on how far a
correct kernel may land from it.  The bound is built from the roundings the kernel performs, so it is tight where an
output is small through cancellation and wide where the operands are large:
  - fp32 accumulation of K products in any order, sequential or in truncating fused blocks:
    C_ACC * K * 2^-23 * sum_k |a_mk b_nk|  (a second fp64 GEMM on |A|, |B|);
  - one fp32 rounding per epilogue operation (bias add, rowv * colv product and add, addend add);
  - a smooth activation: sup |a'| (or the value of a'(z) where z is an exact input) times the error carried in, plus
    the error of the epilogue's fast __expf / __logf / __fdividef (csrc/common.cuh act_fwd / act_d1);
  - half a bf16 ulp of the stored result, taken at |x| + delta.
Column sums get the sum of the per-element bounds before rounding plus M * 2^-23 * sum |x|.

Pure torch in float64: runs on the CPU or on CUDA tensors (cuBLAS DGEMM), and never loads the CUDA library.
"""
import torch

NONE, RELU, SOFTPLUS, SILU = 0, 1, 2, 3   # include/mnrf.h MNRF_ACT_*
U = 2.0 ** -24                            # fp32 unit roundoff (round to nearest)
# Accumulation constant: c * K * 2^-23 holds for K products added in fp32 sequentially or in fused blocks that
# truncate, in any order.  How the H100 tensor cores round the fp32 accumulation has not been measured, so the GPU
# tests print the worst err / bound ratio of every instance.
C_ACC = 2.0
SUP_D1 = {NONE: 1.0, RELU: 1.0, SOFTPLUS: 1.0, SILU: 1.1}   # sup |a'| over the reals (SiLU: 1.0998)
CHUNK = 8192                               # rows per fp64 GEMM


def products(a, b, chunk=CHUNK):
  """fp64 A B^T and |A| |B|^T of A [M, K], B [N, K] (any float dtype, converted exactly)."""
  bd = b.double()
  bad = bd.abs()
  prod, absum = [], []
  for r0 in range(0, a.shape[0], chunk):
    ad = a[r0:r0 + chunk].double()
    prod.append(ad @ bd.T)
    absum.append(ad.abs() @ bad.T)
  return torch.cat(prod), torch.cat(absum)


def half_ulp_bf16(x):
  """Half a bf16 ulp at |x| (fp64 tensor): the error of rounding x to bf16 (round to nearest even)."""
  e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
  return torch.exp2(e - 8)


def act(code, z):
  if code == RELU:
    return z.clamp_min(0)
  if code == SOFTPLUS:
    return torch.logaddexp(z, torch.zeros_like(z))
  if code == SILU:
    return z * torch.sigmoid(z)
  return z


def act_d1(code, z):
  s = torch.sigmoid(z)
  return s * (1 + z * (1 - s)) if code == SILU else s


def _fast_act_err(code, z, y):
  """Error of the epilogue's a(z) with __expf (2 + 1.173|x| ulp), __fdividef (2 ulp) and __logf (2^-21.4 absolute
  on [0.5, 2]), doubled for the fp32 roundings between them."""
  rel = (4 + 1.2 * z.abs()) * 2.0 ** -23
  if code == SILU:
    return 2 * y.abs() * rel
  if code == SOFTPLUS:
    return 2 * (2.0 ** -21 + rel + U * y.abs())
  return torch.zeros_like(z)


def _fast_d1_err(code, z):
  """Error of the epilogue's a'(z): the sigmoid's (as above), through d a' / d s = 1 + z (1 - 2s) for SiLU.
  A closed form that grows with |z|: it says little where |z| is large.  tests/tangent_ref.py (act_derivs) bounds
  the same a'(z), and a''(z), by a running error that stays tight for any z; the GEMM tests keep this one."""
  s = torch.sigmoid(z)
  return 2 * s * (1 + 2 * z.abs()) * (6 + 1.2 * z.abs()) * 2.0 ** -23


def _round_add(v, e):
  """Error after one more fp32 rounding of a value v (fp64) known to within e."""
  return e + U * (v.abs() + e)


def unpack_bits(words, n):
  """[rows, >= n/32] int32 mask words -> [rows, n] bool (bit j of word w <-> column 32w + j)."""
  w = words[:, :n // 32].long() & 0xffffffff
  shifts = torch.arange(32, device=words.device)
  return ((w[:, :, None] >> shifts) & 1).reshape(words.shape[0], n).bool()


def pack_bits(maskb, words_pitch=None):
  """[rows, N] bool -> [rows, words_pitch] int32 mask words (bit j of word w <-> column 32w + j), zero padded."""
  rows, n = maskb.shape
  words_pitch = words_pitch or n // 32
  shifts = torch.arange(32, device=maskb.device)
  words = (maskb.reshape(rows, n // 32, 32).long() << shifts).sum(-1)
  words = torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)
  out = torch.zeros(rows, words_pitch, dtype=torch.int32, device=maskb.device)
  out[:, :n // 32] = words
  return out


def ref_fwd(a, b, *, bias=None, act_code=NONE):
  """FWD: out = a(A B^T + bias); z = A B^T + bias.  Returns fp64 dict(out, out_bound, z, z_bound, pre_bound):
  pre_bound bounds the fp32 value before its bf16 rounding."""
  k = a.shape[1]
  acc, absum = products(a, b)
  e = C_ACC * k * 2.0 ** -23 * absum
  z = acc
  if bias is not None:
    z = acc + bias.double()
    e = _round_add(z, e)
  z_bound = e + half_ulp_bf16(z.abs() + e)
  y = act(act_code, z)
  e_y = SUP_D1[act_code] * e + _fast_act_err(act_code, z, y)
  return dict(out=y, out_bound=e_y + half_ulp_bf16(y.abs() + e_y), z=z, z_bound=z_bound, pre_bound=e_y)


def ref_dgrad(a, b, *, rowv=None, colv=None, mask=None, maskbits=None, mask_mod=0, addend=None, z=None,
              act_code=NONE):
  """DGRAD: out = f * (A B^T + rowv colv) + addend, f = [mask > 0] (bf16 mask), the mask bit (maskbits) or a'(z)
  (smooth act_code), mask / z row = output row mod mask_mod (when > 0).  Returns fp64 dict(out, out_bound,
  pre_bound)."""
  m, k = a.shape
  n = b.shape[0]
  acc, absum = products(a, b)
  e = C_ACC * k * 2.0 ** -23 * absum
  t = acc
  if rowv is not None:
    rc = rowv.double()[:, None] * colv.double()[None, :]
    t = acc + rc
    e = _round_add(t, e + U * rc.abs())
  rows = torch.arange(m, device=a.device)
  if mask_mod:
    rows = rows % mask_mod
  if z is not None:
    zz = z.double()[rows]
    f = act_d1(act_code, zz)
    v = t * f
    e = f.abs() * e + t.abs() * _fast_d1_err(act_code, zz)
    e = _round_add(v, e)
  elif maskbits is not None or mask is not None:
    # a select, not a product: a masked-out element is 0 even where the sum is NaN or infinite (jax.nn.relu's JVP,
    # torch's threshold_backward)
    keep = unpack_bits(maskbits, n)[rows] if maskbits is not None else mask.double()[rows] > 0
    v, e = torch.where(keep, t, 0.0), torch.where(keep, e, 0.0)
  else:
    v = t
  if addend is not None:
    v = v + addend.double()
    e = _round_add(v, e)
  return dict(out=v, out_bound=e + half_ulp_bf16(v.abs() + e), pre_bound=e)


def ref_wgrad(x, dy, *, init=None, bsum_init=None, side_w=None, side_aw_init=None):
  """WGRAD: out[Mo, N] = init + X^T dY; bsum = bsum_init + column sums of dY; side_aw = side_aw_init + X^T side_w.
  Every sum is taken in fp32 in some order (split over R with fp32 atomics); the initial value counts as one more
  term.  Returns fp64 dict of (value, bound) pairs."""
  r = x.shape[0]
  xt = x.T
  out, absum = products(xt, dy.T)
  res = {}
  n_terms = r + 2
  if init is not None:
    out = out + init.double()
    absum = absum + init.double().abs()
  res['out'] = (out, C_ACC * n_terms * 2.0 ** -23 * absum)
  if bsum_init is not None:
    s = dy.double().sum(0) + bsum_init.double()
    sa = dy.double().abs().sum(0) + bsum_init.double().abs()
    res['bsum'] = (s, C_ACC * n_terms * 2.0 ** -23 * sa)
  if side_w is not None:
    w = side_w.double()
    s = xt.double() @ w + side_aw_init.double()
    sa = xt.double().abs() @ w.abs() + side_aw_init.double().abs()
    res['side_aw'] = (s, C_ACC * n_terms * 2.0 ** -23 * sa)
  return res


def colsum_ref(value, pre_bound, init, rounded=False):
  """Column sums of an fp64 output (value [M, N], its pre-rounding bound) added to init [N].  rounded: the sums are
  taken of the stored bf16 output (the SIMT reference path), which adds its rounding."""
  m = value.shape[0]
  s = value.sum(0) + init.double()
  e = pre_bound
  if rounded:
    e = e + half_ulp_bf16(value.abs() + e)
  bound = e.sum(0) + (m + 2) * 2.0 ** -23 * ((value.abs() + e).sum(0) + init.double().abs())
  return s, bound


def check(got, value, bound, what):
  """Worst err / bound ratio of got against (value, bound); asserts every element is finite and within its bound."""
  g = got.double()
  assert torch.isfinite(g).all(), f'{what}: {int((~torch.isfinite(g)).sum())} non-finite results'
  err = (g - value).abs()
  ratio = err / bound.clamp_min(1e-300)
  worst = float(ratio.max()) if ratio.numel() else 0.0
  if worst > 1.0:
    idx = tuple(int(i) for i in torch.nonzero(ratio == ratio.max())[0])
    bad = int((ratio > 1).sum())
    raise AssertionError(f'{what}: {bad} / {ratio.numel()} outside the fp64 bound, worst err/bound {worst:.3g} '
                         f'at {idx}: got {float(g[idx]):.6g}, fp64 {float(value[idx]):.6g}, '
                         f'bound {float(bound[idx]):.3g}')
  return worst


def check_bits(words, stored, z, bound, what):
  """FWD ReLU mask bits, the sign of the fp32 pre-activation, against the stored output and the fp64 pre-activation z
  (known to within bound before its bf16 rounding).  stored > 0 implies the bit; a set bit over a stored 0 only where
  the fp32 pre-activation may lie in (0, 2^-134], which rounds to a bf16 zero; against fp64 the bits may differ only
  where |z| <= bound.  A NaN pre-activation has bit 0."""
  n = stored.shape[1]
  bits = unpack_bits(words, n).to(stored.device)
  pos = stored.float() > 0
  assert not (pos & ~bits).any(), f'{what}: a positive stored output without its mask bit'
  tiny = (z - bound <= 2.0 ** -134) & (z + bound > 0)
  assert not (bits & ~pos & ~tiny).any(), f'{what}: a mask bit over a stored 0 whose pre-activation is not tiny'
  disagree = bits != (z > 0)
  assert not (disagree & ~(z.abs() <= bound)).any(), f'{what}: mask bits wrong where fp64 is clearly signed'


# ---------------------------------------------------------------------------------------------- buffers
NAN_BITS = {torch.bfloat16: 0x7fc1, torch.float32: 0x7fc00001}
SENTINEL = {torch.bfloat16: 0x7fa5, torch.float32: 0x7fa5a5a5, torch.int32: 0x5a5a5a5a}
_INT_VIEW = {torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.int32: torch.int32}


def _bit_fill(buf, pattern):
  v = buf.view(_INT_VIEW[buf.dtype])
  if pattern >= 2 ** (8 * v.element_size() - 1):
    pattern -= 2 ** (8 * v.element_size())
  v.fill_(pattern)


def embed(shape, dtype, device, *, extra_rows=1, extra_cols=0, col0=0, fill='nan'):
  """A [rows, cols] (or [n]) view inside a larger buffer: extra_rows padding rows above and below, col0 padding
  columns before and extra_cols - col0 after (row pitch cols + extra_cols).  fill: 'nan' (inputs: a read outside
  the view makes a NaN result; integer inputs get the sentinel), 'sentinel' (outputs: a fixed bit pattern, checked
  by padding_intact) or None (left uninitialised).  Returns (view, buffer)."""
  if len(shape) == 1:
    buf = torch.empty(shape[0] + extra_cols, dtype=dtype, device=device)
    view = buf[col0:col0 + shape[0]]
  else:
    rows, cols = shape
    buf = torch.empty(rows + 2 * extra_rows, cols + extra_cols, dtype=dtype, device=device)
    view = buf[extra_rows:extra_rows + rows, col0:col0 + cols]
  if fill is not None:
    _bit_fill(buf, NAN_BITS[dtype] if fill == 'nan' and dtype in NAN_BITS else SENTINEL[dtype])
  return view, buf


def padding_intact(view, buf):
  """True if every element of buf outside view still holds the sentinel, bitwise."""
  inside = torch.zeros(buf.shape, dtype=torch.bool, device=buf.device)
  off = (view.data_ptr() - buf.data_ptr()) // buf.element_size()
  if buf.dim() == 1:
    inside[off:off + view.shape[0]] = True
  else:
    r0, c0 = divmod(off, buf.stride(0))
    inside[r0:r0 + view.shape[0], c0:c0 + view.shape[1]] = True
  v = buf.view(_INT_VIEW[buf.dtype])
  pat = SENTINEL[buf.dtype]
  if pat >= 2 ** (8 * v.element_size() - 1):
    pat -= 2 ** (8 * v.element_size())
  return bool((v[~inside] == pat).all())
