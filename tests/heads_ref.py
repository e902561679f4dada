"""fp64 reference of the narrow heads, column sums, weight packing and clip+Adam (csrc/heads.cu) with a per-element
bound.

Each function takes exactly the operands the kernel takes and returns the fp64 value of every output together with a
bound on how far a correct kernel may land from it, built from the roundings the kernel performs (tests/gemm_ref.py
for the accumulation constant and the helpers):
  - head_fwd: raw = x w^T + b.  The bf16 x bf16 products are exact in fp32, so raw is K exact products summed in fp32
    in any order plus one bias add (gemm_ref.ref_fwd's pre_bound); the output is fp32, with no bf16 rounding.
  - head_bwd: dx[m, k] = f * sum_o draw[m, o] w[o, k] (f: 1, the ReLU mask x > 0, or a'(z)), rounded to bf16; dx2 the
    same sum without f; dxsum the column sums of the fp32 dx before its rounding; dw[k, o] = init + sum_m draw[m, o]
    x[m, k]; db = init + sum_m draw.  draw is fp32, so the products of dx and dw round.  The accumulation bound
    C_ACC * (terms) * 2^-23 * sum |.| has room for one product rounding per term (a sum of n terms in fp32 is off by
    at most (n - 1) 2^-24 sum |.|, the products by 2^-24 sum |.|), so no separate charge is made for them.
  - colsum: init + sum_m x, bounded like the bias sums of gemm_ref.ref_wgrad.
  - pack_weights: no bound: a shadow must equal master.to(torch.bfloat16) bit for bit (round to nearest even; overflow
    to inf), except that a NaN master only has to give a NaN.
  - clip_adam: train_utils.py:200-218 (value clip, then the global-norm clip with eps), nan_to_num (:328), optax.adam,
    in fp64 from the fp32 descriptor values, with a running error bound: the fp32 norm (n squares summed in any
    order, then sqrtf), a few ulp of beta^t for powf in the bias corrections (relative to 1 - beta^t, which is small
    at steps 1-3), and one rounding per other operation (1 - beta is exact in fp32, Sterbenz).  The NaN and inf rules
    are exact: a NaN anywhere makes the module's mult NaN (every g becomes 0), an infinite norm gives mult = 0,
    without the norm clip nan_to_num maps +-inf to +-FLT_MAX (and the fp32 square of FLT_MAX overflows nu to inf, so
    the element's parameter stays put), and under a value clip a NaN element becomes 0, not -grad_max_val.  An
    infinite gradient with neither clip at step 1 puts m / bc1 on the fp32 overflow threshold; clip_adam refuses it.

Pure torch in float64: runs on the CPU or on CUDA tensors, and never loads the CUDA library.
"""
import math

import torch

import gemm_ref as G

U = G.U
FLT_MAX = 3.4028234663852886e38
POW_ULPS = 8                        # powf: CUDA Math API bound, with room
EPS32 = 1.1920928955078125e-07      # jnp.finfo(float32).eps, the eps of the norm clip (csrc/common.cuh kEps)


def _acc_bound(terms, abs_sum):
  return G.C_ACC * terms * 2.0 ** -23 * abs_sum


# ---------------------------------------------------------------------------------------------- heads
def head_fwd(x, w, b=None):
  """raw [M, n_out] = x [M, K] w [n_out, K]^T + b.  Returns (value, bound), fp64."""
  r = G.ref_fwd(x, w, bias=b)
  return r['out'], r['pre_bound']


def head_bwd(x, w, draw, *, act=G.NONE, z=None, dx_cols=0, dw_split=0, dw_init=None, db_init=None,
             dxsum_init=None, want_dx=True):
  """The outputs of mnrf_head_bwd for x [M, K] (bf16), w [n_out, K] (bf16), draw [M, n_out] (fp32).  act: G.NONE,
  G.RELU (mask x > 0) or a smooth code with z [M, dx_cols] (bf16) the pre-activation.  dx_cols (0: K) and dw_split
  (0: n_out) as the kernel takes them.  Returns a dict of (value, bound) pairs, fp64: dx [M, dx_cols], dx2
  [M, K - dx_cols] (when dx_cols < K), dxsum [dx_cols] (with dxsum_init), dw [K, split] and dw2 [K, n_out - split]
  (with dw_init [K, n_out], the two initial matrices side by side), db [n_out] (with db_init).  want_dx=False leaves
  out dx, dx2 and dxsum (the parameter-gradient-only form, at sizes where [M, K] in fp64 is large)."""
  m, k = x.shape
  n_out = w.shape[0]
  dx_cols = dx_cols or k
  split = dw_split if 0 < dw_split < n_out else n_out
  res = {}
  if want_dx:
    _head_dx(res, x, w, draw, act, z, dx_cols, dxsum_init)
  if dw_init is not None or db_init is not None:
    zero_w = torch.zeros(k, n_out, dtype=torch.float64, device=x.device)
    wg = G.ref_wgrad(x, draw, init=dw_init if dw_init is not None else zero_w,
                     bsum_init=db_init if db_init is not None else torch.zeros(n_out, dtype=torch.float64,
                                                                              device=x.device))
    if dw_init is not None:
      val, bnd = wg['out']
      res['dw'] = (val[:, :split], bnd[:, :split])
      if split < n_out:
        res['dw2'] = (val[:, split:], bnd[:, split:])
    if db_init is not None:
      res['db'] = wg['bsum']
  return res


def _head_dx(res, x, w, draw, act, z, dx_cols, dxsum_init):
  k, n_out = x.shape[1], w.shape[0]
  t, absum = G.products(draw, w.T)
  e_t = _acc_bound(n_out, absum)
  tc, ec = t[:, :dx_cols], e_t[:, :dx_cols]
  if act == G.RELU:
    f = (x[:, :dx_cols].double() > 0).double()
    v, e = tc * f, ec * f
  elif act in (G.SOFTPLUS, G.SILU):
    zz = z[:, :dx_cols].double()
    f = G.act_d1(act, zz)
    v = tc * f
    e = G._round_add(v, f.abs() * ec + tc.abs() * G._fast_d1_err(act, zz))
  else:
    v, e = tc, ec
  res['dx'] = (v, e + G.half_ulp_bf16(v.abs() + e))
  if dx_cols < k:
    t2, e2 = t[:, dx_cols:], e_t[:, dx_cols:]
    res['dx2'] = (t2, e2 + G.half_ulp_bf16(t2.abs() + e2))
  if dxsum_init is not None:
    res['dxsum'] = G.colsum_ref(v, e, dxsum_init, rounded=False)


def colsum(x, init):
  """out [N] = init + sum_m x[m, :] (x bf16 [M, N]).  Returns (value, bound), fp64."""
  s, sa = init.double().clone(), init.double().abs()
  for r0 in range(0, x.shape[0], G.CHUNK):
    xd = x[r0:r0 + G.CHUNK].double()
    s += xd.sum(0)
    sa += xd.abs().sum(0)
  return s, _acc_bound(x.shape[0] + 2, sa)


# ---------------------------------------------------------------------------------------------- weight packing
def pack_matches(got, master):
  """True if a bf16 shadow equals master.to(torch.bfloat16) bit for bit, NaN-ness alone compared where master is
  NaN (got and master of the same shape and layout)."""
  want = master.to(torch.bfloat16)
  nan = torch.isnan(master)
  same = got.view(torch.int16) == want.view(torch.int16)
  return bool(torch.where(nan, torch.isnan(got), same).all())


# ---------------------------------------------------------------------------------------------- clip + Adam
def _mul(a, ea, b, eb):
  """fp32 product of two values known to within ea, eb: value and bound after its rounding."""
  v = a * b
  return v, G._round_add(v, a.abs() * eb + b.abs() * ea + ea * eb)


def _div(a, ea, b, eb):
  """fp32 quotient (b - eb > 0)."""
  v = a / b
  return v, G._round_add(v, (ea + v.abs() * eb) / (b.abs() - eb))


def _add(a, ea, b, eb):
  v = a + b
  return v, G._round_add(v, ea + eb)


def _sqrt(a, ea):
  v = torch.sqrt(a)
  return v, G._round_add(v, v - torch.sqrt((a - ea).clamp_min(0)))


def _pow_bc(beta, step, dev):
  """1 - beta^step and its bound: powf within POW_ULPS ulp of beta^step (or flushed below the normal range), then one
  rounding of the subtraction."""
  pw = torch.tensor(float(beta) ** int(step), dtype=torch.float64, device=dev)
  e_pw = POW_ULPS * 2.0 ** -23 * pw + 2.0 ** -126
  bc = 1 - pw
  return bc, G._round_add(bc, e_pw)


def clip_adam(p, g, mu, nu, *, step, lr, beta1, beta2, eps, grad_max_val, grad_max_norm, grad_scale=1.0, dyn=None):
  """One mnrf_clip_adam call over one module's flat fp32 buffers.  Scalars are taken as the fp32 values the kernel
  gets (dyn: the [lr, bc1, bc2] fp32 buffer that replaces lr and the bias corrections).  Returns a dict of
  (value, bound) pairs for p, mu and nu, fp64.  Where a value is infinite (nu of an element nan_to_num set to
  +-FLT_MAX), its bound is 0: the kernel must give the same infinity."""
  f32 = lambda s: float(torch.tensor(float(s), dtype=torch.float32))
  lr, beta1, beta2, eps = f32(lr), f32(beta1), f32(beta2), f32(eps)
  gmv, gmn, scale = f32(grad_max_val), f32(grad_max_norm), f32(grad_scale)
  dev = g.device
  n = g.numel()
  gd = g.double()
  v = gd * scale
  e = U * v.abs()
  e = torch.where(torch.isfinite(v), e, torch.zeros_like(e))
  if gmv > 0:                                    # clamping is 1-Lipschitz: the bound carries over
    v = torch.where(torch.isnan(v), v, v.clamp(-gmv, gmv))
  mult = torch.tensor(1.0, dtype=torch.float64, device=dev)
  e_mult = torch.tensor(0.0, dtype=torch.float64, device=dev)
  if gmn > 0:
    if torch.isnan(v).any():
      mult = torch.tensor(float('nan'), dtype=torch.float64, device=dev)
    elif torch.isinf(v).any():
      mult = torch.tensor(0.0, dtype=torch.float64, device=dev)
    else:
      sq = v * v
      e_sq = 2 * v.abs() * e + e * e
      nsq = sq.sum()
      e_nsq = e_sq.sum() + _acc_bound(n + 2, sq.sum() + e_sq.sum())
      nrm, e_nrm = _sqrt(nsq, e_nsq)
      den, e_den = _add(torch.tensor(EPS32, dtype=torch.float64, device=dev), 0.0, nrm, e_nrm)
      q, e_q = _div(torch.tensor(gmn, dtype=torch.float64, device=dev), 0.0, den, e_den)
      mult, e_mult = torch.clamp(q, max=1.0), e_q
    v, e = _mul(v, e, mult, e_mult)
  # nan_to_num
  nan = torch.isnan(v)
  v = torch.where(nan, torch.zeros_like(v), v)
  e = torch.where(nan, torch.zeros_like(e), e)
  inf = torch.isinf(v)
  v = torch.where(inf, torch.sign(v) * FLT_MAX, v)
  e = torch.where(inf, torch.zeros_like(e), e)
  zero = torch.zeros_like(v)
  b1, b2 = torch.full_like(v, beta1), torch.full_like(v, beta2)
  a1, ea1 = _mul(b1, zero, mu.double(), zero)
  c1, ec1 = _mul(1 - b1, zero, v, e)
  m, e_m = _add(a1, ea1, c1, ec1)
  a2, ea2 = _mul(b2, zero, nu.double(), zero)
  c2, ec2 = _mul(1 - b2, zero, v, e)
  c2, ec2 = _mul(c2, ec2, v, e)
  over = c2.abs() > FLT_MAX                       # (1 - beta2) v v of v = +-FLT_MAX: inf in fp32
  c2 = torch.where(over, torch.full_like(c2, math.inf), c2)
  ec2 = torch.where(over, zero, ec2)
  s, e_s = _add(a2, ea2, c2, ec2)
  e_s = torch.where(torch.isinf(s), zero, e_s)
  if dyn is not None:
    lr_, bc1, bc2 = (float(t) for t in dyn.double().cpu())
    bc1, e_bc1 = torch.tensor(bc1, dtype=torch.float64, device=dev), 0.0
    bc2, e_bc2 = torch.tensor(bc2, dtype=torch.float64, device=dev), 0.0
    lr = lr_
  else:
    bc1, e_bc1 = _pow_bc(beta1, step, dev)
    bc2, e_bc2 = _pow_bc(beta2, step, dev)
  mh, e_mh = _div(m, e_m, bc1, e_bc1)
  # m of an element set to FLT_MAX is (1 - beta1) FLT_MAX; at step 1 (bc1 = 1 - beta1) m / bc1 lands on the fp32
  # overflow threshold, where whether the update is 0 or NaN depends on the last bit: not a case with one answer
  assert not (mh.abs() > FLT_MAX * (1 - 2.0 ** -20)).any(), 'm / bc1 at the fp32 overflow threshold'
  sh, e_sh = _div(s, e_s, bc2, e_bc2)
  rt, e_rt = _sqrt(sh, torch.where(torch.isinf(sh), zero, e_sh))
  den, e_den = _add(rt, e_rt, torch.full_like(v, eps), zero)
  num, e_num = _mul(torch.full_like(v, lr), zero, mh, e_mh)
  upd, e_upd = _div(num, e_num, den, torch.where(torch.isinf(den), zero, e_den))
  e_upd = torch.where(torch.isinf(den), zero, e_upd)
  pn, e_p = _add(p.double(), zero, -upd, e_upd)
  return dict(p=(pn, e_p), mu=(m, e_m), nu=(s, e_s))


def check_adam(got, value, bound, what):
  """gemm_ref.check on the finite values; infinite values must be matched exactly."""
  inf = torch.isinf(value)
  if inf.any():
    assert torch.equal(got.double()[inf], value[inf]), f'{what}: an infinite result differs'
  keep = ~inf
  return G.check(got[keep], value[keep], bound[keep], what)
