"""fp64 reference of the trunk's tangent kernels (csrc/refnerf.cu mnrf_outer_mask, mnrf_act_tangent_bwd) with a
bound on every element.

`outer_mask_ref` is exact: out[r, n] = bf16_rn(fl32(rowv[r] colv[n])) where the mask bit of row r mod mask_mod is
set (or there are no mask bits) and +0 otherwise.  The kernel selects, it does not multiply by the bit, so a NaN rowv
under a cleared bit still gives +0.  The tests compare bit for bit.

`act_tangent_ref` takes exactly the bf16 operands of mnrf_act_tangent_bwd -- z [M, N], the three stacked streams T
and u [3M, N], and g's previous contents when accumulating -- and returns the fp64 values
  du_s = a'(z) T_s,     g = [prev +] a''(z) sum_s T_s u_s
with a bound on how far the kernel's bf16 results may lie from them.  The bound is a running error (encode_ref._V:
fp64 value, absolute error) along the kernel's own formula order (common.cuh sigmoid_fast, act_d1, act_d2):

  sigmoid   s = __fdividef(1, fl(1 + __expf(-z))).  __expf is documented at 2 + floor(1.173 |z|) ulp and
            __fdividef at 2 ulp; fl(1 + E) rounds once.  Through ds/dE = -s (1 - s) / E the exponential's relative
            error reaches s as (1 - s) times it, so |s' - s| <= s ((1 - s) (2 + 1.2 |z|) + 3) 2^-23.  Two flushes
            add an absolute 2^-125: __expf(-z) is flushed to 0 below 2^-126, and __fdividef returns 0 once
            1 + e^-z > 2^126 (z < -87.3; the exact s is below 2^-126 there).  Where e^-z (1 + its error) < 2^-25,
            fl(1 + E) is exactly 1 and s' = 1: the error is 1 - s itself.  (That 1 / 1 is exact is the one
            assumption about the approximate reciprocal; without it SiLU's a' = s (1 + z (1 - s)) would carry
            |z| 2^-22 at z = 1e30.)
  a', a''   softplus a' = s, a'' = s (1 - s); SiLU a' = s (1 + z (1 - s)), a'' = s (1 - s) (2 + z (1 - 2 s)), each
            operation rounded once in fp32 (2 s is exact).  gemm_ref._fast_d1_err bounds the same a' for the GEMM
            epilogues in closed form; it grows with |z| (2 s (1 + 2|z|)(6 + 1.2|z|) 2^-23, 5e53 at z = 1e30), so
            this file keeps its own model, which is also the only one for a''.
  du        fl(a' T): one rounding, then bf16.
  gs        T_s u_s is exact in fp32 (two 8-bit significands) unless it underflows; the three-term sum may be
            contracted into FMAs or not, which changes nothing then: two roundings, 2 u sum |T_s u_s|, plus 2^-125
            for underflow.
  g         fl(prev + fl(a'' gs)) or one FMA: the rounding of the product is counted whether or not it happens.
            With accumulate = 0 the kernel must not read g: prev is 0.
  bf16      half a bf16 ulp at |value| + bound (gemm_ref.half_ulp_bf16).

Pure torch in float64: runs on the CPU or on CUDA tensors, and never loads the CUDA library.
"""
import torch

from encode_ref import _V
from gemm_ref import SILU, SOFTPLUS, half_ulp_bf16, unpack_bits

U = 2.0 ** -24
ULP = 2.0 ** -23
FLUSH = 2.0 ** -125         # flushed exponentials, __fdividef's zero, underflowing products


def outer_mask_ref(rowv, colv, maskbits, *, rows, n, mask_mod=0):
  """[rows, n] bf16: the kernel's output bit for bit (fp32 product, round to nearest even, select on the bit)."""
  prod = rowv[:rows].float()[:, None] * colv[:n].float()[None, :]
  if maskbits is None:
    return prod.to(torch.bfloat16)
  r = torch.arange(rows, device=rowv.device)
  keep = unpack_bits(maskbits, n)[r % mask_mod if mask_mod else r]
  return torch.where(keep, prod, torch.zeros_like(prod)).to(torch.bfloat16)


def fast_sigmoid(z):
  """sigmoid_fast(z) as a _V: fp64 value and the bound of the kernel's fp32 value (module docstring)."""
  s = torch.sigmoid(z)
  one_minus = torch.sigmoid(-z)
  general = s * (one_minus * (2 + 1.2 * z.abs()) + 3) * ULP + FLUSH
  e_big = torch.exp((-z).clamp(max=700.0)) * (1 + (2 + 1.2 * z.abs()) * ULP)
  exactly_one = e_big < 2.0 ** -25
  return _V(s, torch.where(exactly_one, one_minus, general))


def act_derivs(code, z):
  """(a'(z), a''(z)) as _V on fp64 z, in the kernel's formula order."""
  if code not in (SOFTPLUS, SILU):
    raise ValueError(f'act {code} is not a smooth activation')
  s = fast_sigmoid(z)
  q = s * (1.0 - s)
  if code == SOFTPLUS:
    return s, q
  zv = _V(z)
  d1 = s * (zv * (1.0 - s) + 1.0)
  d2 = q * (zv * (1.0 - s.scale(2.0)) + 2.0)
  return d1, d2


def act_tangent_ref(code, z, t_adj, u, prev=None):
  """fp64 (du [3M, N], du_bound, g [M, N], g_bound) of mnrf_act_tangent_bwd on bf16 z [M, N], T and u [3M, N] and,
  when accumulating, prev [M, N] (g's contents before the call).  Bounds are of the stored bf16 values."""
  M = z.shape[0]
  zd = z.double()
  d1, d2 = act_derivs(code, zd)
  T = t_adj.double().view(3, M, -1)
  uu = u.double().view(3, M, -1)
  du_val = d1.val * T
  du_err = d1.err * T.abs()
  du_err = du_err + U * (du_val.abs() + du_err)
  prods = T * uu
  gs = prods.sum(0)
  gs_err = 2 * U * prods.abs().sum(0) + 3 * FLUSH
  g_val = d2.val * gs
  g_err = d2.err * gs.abs() + d2.val.abs() * gs_err + d2.err * gs_err
  g_err = g_err + U * (g_val.abs() + g_err)
  if prev is not None:
    g_val = g_val + prev.double()
  g_err = g_err + U * (g_val.abs() + g_err)
  du_val, du_err = du_val.reshape(3 * M, -1), du_err.reshape(3 * M, -1)
  return (du_val, du_err + half_ulp_bf16(du_val.abs() + du_err),
          g_val, g_err + half_ulp_bf16(g_val.abs() + g_err))


# SiLU's a' = 0 at z = -1.27846, a'' = 0 at z = +-2.39936
SILU_D1_ZERO = -1.2784645427610738
SILU_D2_ZEROS = (-2.399357280515467, 2.399357280515467)


def special_z():
  """fp64 values of z where the activations' fast forms go wrong first: signed zeros, bf16 subnormals, the edges of
  __expf's range and __fdividef's flush (|z| ~ 87-89), far beyond them up to 1e30, and SiLU's zeros of a', a''."""
  vals = [0.0, -0.0, 9.2e-41, -9.2e-41, 1e-39, -1e-39, 1.2e-38, -1.2e-38, 1e-3, -1e-3]
  for m in (16.0, 17.0, 17.5, 18.0, 86.0, 87.0, 87.5, 88.0, 88.5, 89.0, 90.0, 104.0, 1e3, 1e6, 1e10, 1e20, 1e30):
    vals += [m, -m]
  for c in (SILU_D1_ZERO,) + SILU_D2_ZEROS:       # the nearest bf16 and its two neighbours
    bits = torch.tensor([c], dtype=torch.bfloat16).view(torch.int16)
    vals += torch.cat([bits - 1, bits, bits + 1]).view(torch.bfloat16).double().tolist()
  return torch.tensor(vals, dtype=torch.float64)
