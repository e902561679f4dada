"""Reference of ray casting + integrated positional encoding (csrc/encode.cu) with a bound on every element.

`reference` takes exactly the inputs of mnrf_encode -- fp32 sdist, origins, directions, radii, near, far, basis and
the descriptor fields -- and evaluates the oracle's own chain (o_coord.construct_ray_warps, o_render.cast_rays,
o_coord.track_linearize_contract, lift_and_diagonalize, and integrated_pos_enc's layout with safe_sin reducing by
fl32(100 pi), Python-style, only where |x| >= fl32(100 pi)) in float64.  Beside the values it returns how far the
kernels' fp32 arithmetic may stray from them, element by element.

Staging.  t_var and r_var of a frustum depend on t1 - t0, which cancels: a reference that recomputed t in fp64 from
sdist would need a bound so wide in the far field that it says nothing.  So `tdist` is checked against its own
bound first, and everything downstream is evaluated on the kernel's own fp32 tdist (`tdist=`), which is then exact
input.  The tangent kernels write no tdist; they call the same s_to_t device function, whose roundings are explicit
_rn intrinsics, so the tdist of a fast-path call on the same inputs stands for theirs.

Bounds are running errors, not estimates.  A second evaluation (`_V`: fp64 value, absolute error bound) walks the
kernel's own formula order -- cast_one, contract_gauss as J cov J^T with J = s I + c x x^T, the lift -- and every
operation adds its rounding to the errors it inherits.  With u = 2**-24:

  a + b, a - b   e_a + e_b + u |result|.  Where terms cancel (J cov J^T far out, 1 - d_i d_j / |d|^2, s + c x_i^2)
                 the inherited errors are u times the magnitudes of the TERMS, so the bound does not shrink with
                 the result.
  a * b          |a| e_b + |b| e_a + e_a e_b + u |result|.  Products by a power of two (the halvings of cast_one,
                 2^l and 4^l of the degrees, reached in the kernel by exact doubling) add nothing.
  a / b, sqrt    (e_a + |a / b| e_b) / (|b| - e_b) + u |result|;  the larger of sqrt(a) - sqrt(max(a - e_a, 0))
                 and sqrt(a + e_a) - sqrt(a), + u |result|: both are correctly rounded (the library is built without
                 fast-math).
  constants      4/15 and 5/12 are fp32 constants in the kernel and exact in the reference: relative error u.
  logf, expf     documented at 1 and 2 ulp: 2u and 4u of the result, after the inherited error through the
                 function's own slope.  1/x under `reciprocal` is a division: as s -> 1 the inverse's conditioning
                 enters through e_b / (|b| - e_b).
  sinf, cosf     documented at 2 ulp without fast math: 4u of the result, after the inherited error through the
                 slope (used by camera_ref.py).
  max(c, x)      1-Lipschitz: the error is inherited unchanged; so is min(c, x).
  branches       |x|^2 <= 1 of the contraction and the two halves of `piecewise` are taken on the fp64 value.  Both
                 functions are C^1 across the branch, so a sample within rounding of it moves by O(e^2).
The second evaluation's values agree with the oracle's to fp64 rounding; their difference is added to the bound, and
test_encode_reference_cpu.py asserts it stays negligible, so a slip in the formula order here cannot hide.

tdist    s_near = fwd(near), s_far = fwd(far), x = fl(fl(s s_far) + fl(fl(1 - s) s_near)), t = inv(x): the products
         and the sum are rounded separately, as the rules above do.
feature  With y = lm 2^l and v = lv 4^l the lifted mean and variance at degree l, dy and dv their bounds (the lift's
         bound times 2^l and 4^l), e = exp(-v / 2), sn = safe_sin(y) and f = e sn:
           |f' - f| <= e ds + (|f| + e ds) re + u |f|,      ds = dy + jumps * jump + c_sin,
           re = expm1(dv / 2) + c_exp,
         first-order terms scaled by 1.05 like the other reference files.
  jump   The kernels reduce their own fp32 y exactly as Python's y mod fl32(100 pi) (k = floor or rint of
         y / t may be off by one, the remainder y - k t is exact in one FMA, and the +-t fix-up is exact), so where
         y' and y take the same multiple k the reduced arguments differ by dy.  fl32(100 pi) is not a period:
         each step of k moves the argument by jump = |fl32(100 pi) - 100 pi| = 5.9e-6.  `jumps` is the number of
         steps of k inside the bracket [y - dy, y + dy], with k = 0 for |y| < fl32(100 pi) (the reference does
         not reduce there, so crossing -fl32(100 pi) counts two).
  cos    The cosine half is the sine of fl(y + fl32(pi/2)): dy grows by u |y + pi/2| + |fl32(pi/2) - pi/2|.
  c_sin  sin_below_100pi on |r| < fl32(100 pi): q = rint(r / 2 pi) has |q| <= 50; r - q C_hi is exact (a
         multiple of 2^-21 below 3.2); adding q C_lo rounds once, u pi = 1.9e-7; C_hi - C_lo misses 2 pi by 1e-14 per
         turn; MUFU.SIN on |arg| <= pi is documented at 2^-21.41 = 3.6e-7.  Sum 5.5e-7.
  c_exp  The fast kernel forms ex2.approx.ftz(v c) with c = fl32(-log2(e) / 2): the product's rounding and the
         constant's move the exponent by 2u |v c|, a relative u |v| of the result, and ex2.approx is documented at
         2^-22.  The tangent kernels call __expf(-v / 2), documented at 2 + floor(1.173 |v| / 2) ulp.  One bound covers
         both: (3 + 0.6 (|v| + dv)) 2^-23.
  bf16   round-to-nearest of the fp32 feature: half a bf16 ulp, 2^-8 (|f| + bound), on top.
  vacuous  An element whose bound exceeds 0.25 (far contracted samples at high degrees, where dy or dv is of order
         one) says nothing about the kernel.  It is not dropped silently: `vacuous` marks it, and the tests print the
         share per degree and hold each case to a floor on the checked share.

`plan` restates the host's launch plan of the fast kernel and `tiers` the two warp-uniform tests that pick a sine
form per 32-lane pass; they are a second statement of that logic, which is what makes them a check.
`pos_enc_reference` is coord.pos_enc for the view directions.

Evaluated in float32 (`dtype=torch.float32`) the same chain is the fp32 oracle, with no bounds.  Pure torch: runs on
the CPU (CUDA inputs are copied there) and never loads the CUDA library.
"""
import math
import types

import numpy as np
import torch

from oracle import o_coord, o_render

U = 2.0 ** -24          # fp32 unit roundoff
SLACK = 1.05
EPS = float(np.finfo(np.float32).eps)
T32 = float(np.float32(100 * math.pi))
JUMP = abs(T32 - 100 * math.pi)
HALF_PI32 = float(np.float32(math.pi / 2))
C_SIN = 2.0 ** -21.41 + math.pi * U + 50 * 1e-14
VACUOUS = 0.25
TINY = 2.0 ** -120      # subnormal products and flushed results


class _V:
  """fp64 value with a bound on the absolute error of the kernel's fp32 value; see the module docstring."""

  def __init__(self, val, err=None):
    self.val = torch.as_tensor(val, dtype=torch.float64)
    self.err = torch.zeros_like(self.val) if err is None else err

  @staticmethod
  def of(x):
    return x if isinstance(x, _V) else _V(float(x))

  @staticmethod
  def const32(x):
    return _V(torch.tensor(x, dtype=torch.float64), torch.tensor(U * abs(x), dtype=torch.float64))

  def _rounded(self, v, e):
    return _V(v, e + U * (v.abs() + e))

  def __add__(self, o):
    o = _V.of(o)
    return self._rounded(self.val + o.val, self.err + o.err)

  def __sub__(self, o):
    o = _V.of(o)
    return self._rounded(self.val - o.val, self.err + o.err)

  def __rsub__(self, o):
    return _V.of(o) - self

  def __mul__(self, o):
    o = _V.of(o)
    return self._rounded(self.val * o.val, self.val.abs() * o.err + o.val.abs() * self.err + self.err * o.err)

  def __truediv__(self, o):
    o = _V.of(o)
    v = self.val / o.val
    low = o.val.abs() - o.err
    e = torch.where(low > 0, (self.err + v.abs() * o.err) / low.clamp(min=1e-300), torch.tensor(math.inf, dtype=torch.float64))
    return self._rounded(v, e)

  def __rtruediv__(self, o):
    return _V.of(o) / self

  def sqrt(self):              # sqrt is concave: the step down bounds the step up unless a - e_a < 0
    v = torch.sqrt(self.val)
    return self._rounded(v, torch.maximum(v - torch.sqrt((self.val - self.err).clamp(min=0)),
                                          torch.sqrt(self.val + self.err) - v))

  def log(self):
    v = torch.log(self.val)
    low = self.val - self.err
    e = torch.where(low > 0, -torch.log1p(-(self.err / self.val).clamp(max=1 - 1e-16)), torch.tensor(math.inf, dtype=torch.float64))
    return _V(v, e + 2 * U * (v.abs() + e))

  def exp(self):
    v = torch.exp(self.val)
    e = v * torch.expm1(self.err)
    return _V(v, e + 4 * U * (v + e))

  def sin(self):               # sinf: 2 ulp (4u of the result); the slope over [v - e, v + e] is <= |cos v| + e
    v = torch.sin(self.val)
    e = (torch.cos(self.val).abs() + self.err).clamp(max=1) * self.err
    return _V(v, e + 4 * U * (v.abs() + e))

  def cos(self):               # cosf: 2 ulp, as sinf
    v = torch.cos(self.val)
    e = (torch.sin(self.val).abs() + self.err).clamp(max=1) * self.err
    return _V(v, e + 4 * U * (v.abs() + e))

  def scale(self, p):          # by a power of two (or its negative): exact
    return _V(self.val * p, self.err * abs(p))

  def maxc(self, c):
    return _V(self.val.clamp(min=c), self.err)

  def minc(self, c):
    return _V(self.val.clamp(max=c), self.err)

  def u(self):                 # a trailing axis to broadcast over
    return _V(self.val[..., None], self.err[..., None])

  @staticmethod
  def where(c, a, b):
    a, b = _V.of(a), _V.of(b)
    return _V(torch.where(c, a.val, b.val), torch.where(c, a.err, b.err))


def _fwd(fn, x):
  if fn == 'reciprocal':
    return 1.0 / x
  if fn == 'log':
    return x.log()
  if fn == 'exp':
    return x.exp()
  if fn == 'sqrt':
    return x.sqrt()
  if fn == 'square':
    return x * x
  if fn == 'piecewise':
    return _V.where(x.val < 1, x.scale(0.5), 1.0 - 0.5 / x)
  return x


def _inv(fn, x):
  if fn == 'piecewise':
    return _V.where(x.val < 0.5, x.scale(2.0), 0.5 / (1.0 - x))
  return _fwd({'log': 'exp', 'exp': 'log', 'sqrt': 'square', 'square': 'sqrt'}.get(fn, fn), x)


def _tdist(fn, sdist, near, far):
  s = _V(sdist)
  s_near, s_far = _fwd(fn, _V(near[:, None])), _fwd(fn, _V(far[:, None]))
  return _inv(fn, s * s_far + (1.0 - s) * s_near)


def _cast(ray_shape, t0, t1, o, d, radius):
  """cast_one: mean [3] and cov [3][3] of _V, each [rays, samples]."""
  if ray_shape == 'cone':
    mu, hw = (t0 + t1).scale(0.5), (t1 - t0).scale(0.5)
    hw2, mu2 = hw * hw, mu * mu
    hw4 = hw2 * hw2
    c415, c512 = _V.const32(4 / 15), _V.const32(5 / 12)
    denom = (mu2 * 3.0 + hw2).maxc(EPS)
    t_mean = mu + (mu.scale(2.0) * hw2) / denom
    t_var = hw2 / 3.0 - c415 * hw4 * (mu2 * 12.0 - hw2) / (denom * denom)
    r_var = mu2.scale(0.25) + c512 * hw2 - c415 * hw4 / denom
    r_var = r_var * (radius * radius)
  else:
    t_mean = (t0 + t1).scale(0.5)
    r_var = (radius * radius).scale(0.25)
    dt = t1 - t0
    t_var = (dt * dt) / 12.0
  dmag = (d[0] * d[0] + d[1] * d[1] + d[2] * d[2]).maxc(1e-10)
  mean = [d[i] * t_mean + o[i] for i in range(3)]
  cov = [[t_var * (d[i] * d[j]) + r_var * ((1.0 if i == j else 0.0) - d[i] * (d[j] / dmag)) for j in range(3)]
         for i in range(3)]
  return mean, cov


def _contract(x, cov):
  m = (x[0] * x[0] + x[1] * x[1] + x[2] * x[2]).maxc(EPS)
  inside = m.val <= 1
  m = _V.where(inside, 2.0, m)          # the branch not taken: keep its arithmetic finite
  r = m.sqrt()
  scale = (r.scale(2.0) - 1.0) / m
  s = 2.0 / r - 1.0 / m
  c = 2.0 / (m * m) - 2.0 / (m * r)
  J = [[(s + c * x[i] * x[j]) if i == j else (c * x[i] * x[j]) for j in range(3)] for i in range(3)]
  T = [[J[i][0] * cov[0][j] + J[i][1] * cov[1][j] + J[i][2] * cov[2][j] for j in range(3)] for i in range(3)]
  out = [[T[i][0] * J[j][0] + T[i][1] * J[j][1] + T[i][2] * J[j][2] for j in range(3)] for i in range(3)]
  mean = [_V.where(inside, x[i], scale * x[i]) for i in range(3)]
  return mean, [[_V.where(inside, cov[i][j], out[i][j]) for j in range(3)] for i in range(3)]


def _lift(mean, cov, basis, disable_integration):
  b = [_V(basis[:, i]) for i in range(3)]
  lm = mean[0].u() * b[0] + mean[1].u() * b[1] + mean[2].u() * b[2]
  if disable_integration:
    return lm, _V(torch.zeros_like(lm.val))
  c = [cov[i][0].u() * b[0] + cov[i][1].u() * b[1] + cov[i][2].u() * b[2] for i in range(3)]
  return lm, b[0] * c[0] + b[1] * c[1] + b[2] * c[2]


def _k_eff(y):
  """The multiple of fl32(100 pi) that safe_sin takes out of y: none below it."""
  return torch.where(y.abs() < T32, torch.zeros_like(y), torch.floor(y / T32))


def safe_sin64(y):
  """math.safe_sin on fp64 arguments with the fp32 program's constant: reduce by fl32(100 pi), not by 100 pi."""
  return torch.sin(torch.where(y.abs() < T32, y, torch.remainder(y, T32)))


def _features(lm, lv, lm_err, lv_err, min_deg, max_deg):
  """[.., 2KL] features in integrated_pos_enc's layout (sin half then cos half, degree-major) with their bounds."""
  sc = 2.0 ** torch.arange(min_deg, max_deg, dtype=torch.float64)[:, None]
  y, dy = lm[..., None, :] * sc, lm_err[..., None, :] * sc
  v, dv = lv[..., None, :] * sc ** 2, lv_err[..., None, :] * sc ** 2
  e = torch.exp(-0.5 * v)
  re = torch.expm1((0.5 * dv).clamp(max=40.0)) + (3 + 0.6 * (v.abs() + dv)) * 2 * U
  feats, bounds = [], []
  for half in range(2):
    if half:
      y = y + 0.5 * math.pi
      dy = dy + U * (y.abs() + dy) + abs(HALF_PI32 - 0.5 * math.pi)
    sn = safe_sin64(y)
    jumps = (_k_eff(y + dy) - _k_eff(y - dy)).abs()
    ds = (dy + jumps * JUMP + C_SIN).clamp(max=2.0)
    f = e * sn
    feats.append(f)
    bounds.append(SLACK * (e * ds + (f.abs() + e * ds) * re + U * f.abs()) + TINY)
  shape = lm.shape[:-1] + (-1,)
  return torch.cat([f.reshape(shape) for f in feats], -1), torch.cat([b.reshape(shape) for b in bounds], -1)


def bf16_bound(value, bound):
  """Bound of the bf16-rounded kernel value: the fp32 bound plus half a bf16 ulp of anything within it."""
  return bound + 2.0 ** -8 * (value.abs() + bound) + 2.0 ** -134


def _contract_terms(x):
  """contract_terms on the pre-warp mean: xh, s, q, s_r, q_r (the identity's 0, 1, 1, 0, 0 inside the ball) and
  `unsure`, the samples whose |x|^2 lies within its rounding of 1, where the kernel may take either branch."""
  m = (x[0] * x[0] + x[1] * x[1] + x[2] * x[2]).maxc(EPS)
  inside = m.val <= 1
  unsure = (m.val - 1).abs() <= m.err
  mo = _V.where(inside, 2.0, m)          # the branch not taken: keep its arithmetic finite
  r = mo.sqrt()
  ir = 1.0 / r
  q_r = -2.0 / (mo * r)
  pick = lambda v, ident: _V.where(inside, ident, v)
  return ([pick(x[i] * ir, 0.0) for i in range(3)], pick(2.0 / r - 1.0 / mo, 1.0), pick(1.0 / mo, 1.0),
          pick((r - 1.0) * q_r, 0.0), pick(q_r, 0.0), unsure)


def _lift_tangent(x, cov, basis, disable_integration):
  """d lift_mean / d x_a and d lift_var / d x_a [3] of [.., K] _V, in gauss_tangent_rows' order, and `unsure`."""
  xh, s, q, s_r, q_r, unsure = _contract_terms(x)
  xh = [t.u() for t in xh]
  s, q, s_r, q_r = s.u(), q.u(), s_r.u(), q_r.u()
  b = [_V(basis[:, i]) for i in range(3)]
  cv = [cov[0][0].u(), cov[0][1].u(), cov[0][2].u(), cov[1][1].u(), cov[1][2].u(), cov[2][2].u()]
  beta = xh[0] * b[0] + xh[1] * b[1] + xh[2] * b[2]
  bt = [b[i] - beta * xh[i] for i in range(3)]
  u = [s * bt[i] + (q * beta) * xh[i] for i in range(3)]
  v = [cv[0] * u[0] + cv[1] * u[1] + cv[2] * u[2], cv[1] * u[0] + cv[3] * u[1] + cv[4] * u[2],
       cv[2] * u[0] + cv[4] * u[1] + cv[5] * u[2]]
  gamma = xh[0] * v[0] + xh[1] * v[1] + xh[2] * v[2]
  vt = [v[i] - gamma * xh[i] for i in range(3)]
  btv = bt[0] * v[0] + bt[1] * v[1] + bt[2] * v[2]
  radial = s_r * btv + q_r * (beta * gamma)
  if disable_integration:
    dlv = [_V(torch.zeros_like(beta.val)) for _ in range(3)]
  else:
    dlv = [(xh[a] * radial + s_r * (beta * vt[a] + gamma * bt[a])).scale(2.0) for a in range(3)]
  return u, dlv, unsure


def _reduced(y):
  return torch.where(y.abs() < T32, y, torch.remainder(y, T32))


def _tangent_features(lm, lv, lm_err, lv_err, dl, basis, min_deg, max_deg):
  """[3, .., 2KL] d feature / d x_dir in integrated_pos_enc's layout with its fp32 bound.  dl: (dlm, dlv) of
  _lift_tangent with the contraction, None without it (d lift_mean / d x_dir = basis[k][dir])."""
  sc_all = 2.0 ** torch.arange(min_deg, max_deg, dtype=torch.float64)
  out = [[[], []] for _ in range(3)]
  for sc in sc_all.tolist():
    y, dy = lm * sc, lm_err * sc
    v, dv = lv * sc * sc, lv_err * sc * sc
    e = torch.exp(-0.5 * v)
    re = torch.expm1((0.5 * dv).clamp(max=40.0)) + (3 + 0.6 * (v.abs() + dv)) * 2 * U
    E = _V(e, e * re + 2.0 ** -126)        # __expf flushes results below 2^-126 to 0
    for half in range(2):
      if half:                   # the kernel reduces y + pi/2 on its own, as the feature rows do
        y = y + 0.5 * math.pi
        dy = dy + U * (y.abs() + dy) + abs(HALF_PI32 - 0.5 * math.pi)
      jumps = (_k_eff(y + dy) - _k_eff(y - dy)).abs()
      ds = (dy + jumps * JUMP + C_SIN).clamp(max=2.0)
      arg = _reduced(y)
      f = E * _V(torch.sin(arg), ds)
      cs = _V(torch.cos(arg), ds)
      for a in range(3):
        if dl is None:
          t = cs * (_V(basis[:, a] * sc) * E)
        else:
          dlm, dlv = dl
          t = cs * (dlm[a] * E.scale(sc)) - f * dlv[a].scale(0.5 * sc * sc)
        out[a][half].append(t)
  shape = lm.shape[:-1] + (-1,)
  val = torch.stack([torch.cat([torch.stack([t.val for t in out[a][h]], -2).reshape(shape) for h in range(2)], -1)
                     for a in range(3)])
  err = torch.stack([torch.cat([torch.stack([t.err for t in out[a][h]], -2).reshape(shape) for h in range(2)], -1)
                     for a in range(3)])
  return val, SLACK * err + TINY


def tangent_reference(x, cov, lm, lv, lm_err, lv_err, feat_vacuous, basis, *, min_deg, max_deg, warp_contract,
                      disable_integration):
  """Tangent rows of gauss_tangent_rows on the pre-warp Gaussian (x [3], cov [3][3] of _V): (value, bound,
  bound_bf16, vacuous), each [3, .., 2KL], and `unsure` [..], the samples within rounding of |x| = 1.  Vacuous: the feature's own bound says nothing, or (contraction) the
  sample lies within rounding of |x| = 1, where the q_r term of d lift_var jumps from -2 / r^3 to 0."""
  b = basis.double()
  dl = None
  unsure = torch.zeros(lm.shape[:-1], dtype=torch.bool)
  if warp_contract:
    dlm, dlv, unsure = _lift_tangent(x, cov, b, disable_integration)
    dl = (dlm, dlv)
  val, bound = _tangent_features(lm, lv, lm_err, lv_err, dl, b, min_deg, max_deg)
  vac = feat_vacuous[None] | unsure[None, ..., None] | ~torch.isfinite(bound)
  return val, bound, bf16_bound(val, bound), vac, unsure


def points_reference(points, var, basis, *, min_deg, max_deg, warp_contract=False, disable_integration=False):
  """mnrf_encode_points_tangent: features and tangent rows of the Gaussians (points[i], var I), var and points fp32.
  Returns feat / bound / bound_bf16 / vacuous [N, 2KL], tangent / tangent_bound / tangent_bound_bf16 /
  tangent_vacuous [3, N, 2KL] and chain_gap (the running evaluation against the oracle's lift)."""
  p = torch.as_tensor(points).detach().cpu().double()
  bd = torch.as_tensor(basis).detach().cpu().double()
  v32 = 0.0 if disable_integration else float(np.float32(var))
  x = [_V(p[:, i]) for i in range(3)]
  cov = [[_V(torch.full_like(p[:, 0], float(np.float32(var)) if i == j else 0.0)) for j in range(3)] for i in range(3)]
  mean, covw = _contract(x, cov) if warp_contract else (x, cov)
  lmv, lvv = _lift(mean, covw, bd, disable_integration)
  covs = (torch.eye(3, dtype=torch.float64) * v32).expand(p.shape[0], 3, 3)
  om, oc = o_coord.track_linearize_contract(p, covs) if warp_contract else (p, covs)
  lm, lv = o_coord.lift_and_diagonalize(om, oc, bd.T.contiguous())
  out = types.SimpleNamespace(lm=lm, lv=lv)
  out.chain_gap = max(float(((lmv.val - lm).abs() / (lmv.err + 1e-300)).max()),
                      float(((lvv.val - lv).abs() / (lvv.err + 1e-300)).max()))
  lm_err, lv_err = lmv.err + (lmv.val - lm).abs(), lvv.err + (lvv.val - lv).abs()
  out.feat, out.bound = _features(lm, lv, lm_err, lv_err, min_deg, max_deg)
  out.bound_bf16 = bf16_bound(out.feat, out.bound)
  out.vacuous = ~(out.bound <= VACUOUS)
  out.tangent, out.tangent_bound, out.tangent_bound_bf16, out.tangent_vacuous, out.unsure = tangent_reference(
      x, cov, lm, lv, lm_err, lv_err, out.vacuous, bd, min_deg=min_deg, max_deg=max_deg, warp_contract=warp_contract,
      disable_integration=disable_integration)
  return out


def reference(sdist, origins, directions, radii, near, far, basis, *, min_deg, max_deg, raydist_fn=None,
              ray_shape='cone', warp_contract=False, disable_integration=False, tdist=None, dtype=torch.float64,
              tangent=False):
  """fp64 reference of mnrf_encode with per-element bounds.  `tdist`: the kernel's own fp32 tdist to stage the
  Gaussians on (default: the reference's, rounded to fp32).  Returns tdist / tdist_bound [B, S+1], feat / bound /
  bound_bf16 / vacuous [B, S, 2KL], and the lifted lm, lv [B, S, K] the features were formed from; with `tangent`
  also the tangent rows tangent / tangent_bound / tangent_bound_bf16 / tangent_vacuous [3, B, S, 2KL], `unsure`
  [B, S] (samples within rounding of |x| = 1) and `xnorm` [B, S], the fp64 |x| of the pre-warp means."""
  if ray_shape not in ('cone', 'cylinder'):
    raise ValueError("ray_shape must be 'cone' or 'cylinder'")
  c = lambda t: t.detach().cpu().to(dtype)
  sd, o, d, b = c(sdist), c(origins), c(directions), c(basis)
  rad, nr, fr = c(radii).reshape(-1, 1), c(near).reshape(-1, 1), c(far).reshape(-1, 1)
  _, s_to_t = o_coord.construct_ray_warps(raydist_fn, nr, fr)
  out = types.SimpleNamespace(tdist=s_to_t(sd))
  staged = out.tdist.float() if tdist is None else tdist.detach().cpu().float()
  means, covs = o_render.cast_rays(staged.to(dtype), o, d, rad, ray_shape, diag=False)
  if warp_contract:
    means, covs = o_coord.track_linearize_contract(means, covs)
  lm, lv = o_coord.lift_and_diagonalize(means, covs, b.T.contiguous())
  if disable_integration:
    lv = torch.zeros_like(lv)
  out.lm, out.lv = lm, lv
  if dtype != torch.float64:
    out.feat = o_coord.integrated_pos_enc(lm, lv, min_deg, max_deg)
    return out
  tv = _tdist(raydist_fn, sd, nr[:, 0], fr[:, 0])
  out.tdist_bound = SLACK * (tv.err + (tv.val - out.tdist).abs()) + TINY
  t = _V(staged.double())
  ov, dv = [_V(o[:, i:i + 1]) for i in range(3)], [_V(d[:, i:i + 1]) for i in range(3)]
  x, xcov = _cast(ray_shape, _V(t.val[:, :-1]), _V(t.val[:, 1:]), ov, dv, _V(rad))
  mean, cov = _contract(x, xcov) if warp_contract else (x, xcov)
  lmv, lvv = _lift(mean, cov, b, disable_integration)
  # how far the running evaluation's values are from the oracle's: fp64 rounding (asserted in the CPU tests)
  out.chain_gap = max(float(((lmv.val - lm).abs() / (lmv.err + 1e-300)).max()),
                      float(((lvv.val - lv).abs() / (lvv.err + 1e-300)).max()))
  out.lm_err, out.lv_err = lmv.err + (lmv.val - lm).abs(), lvv.err + (lvv.val - lv).abs()
  out.feat, out.bound = _features(lm, lv, out.lm_err, out.lv_err, min_deg, max_deg)
  out.bound_bf16 = bf16_bound(out.feat, out.bound)
  out.vacuous = ~(out.bound <= VACUOUS)
  if tangent:
    out.xnorm = torch.sqrt(x[0].val ** 2 + x[1].val ** 2 + x[2].val ** 2)
    out.tangent, out.tangent_bound, out.tangent_bound_bf16, out.tangent_vacuous, out.unsure = tangent_reference(
        x, xcov, lm, lv, out.lm_err, out.lv_err, out.vacuous, b, min_deg=min_deg, max_deg=max_deg,
        warp_contract=warp_contract, disable_integration=disable_integration)
  return out


def degree_of(K, L):
  """Degree index of each of the 2KL feature columns."""
  return torch.arange(L).repeat_interleave(K).repeat(2)


def plan(num_rays, S, K, num_sms):
  """The fast kernel's launch plan: G samples per group (the g <= min(16, S) whose g*K items fill their 32-lane
  passes best, the smallest on ties), nseg segments per ray (enough warps for 32 per SM, never shorter than 2G
  samples), seg_len a multiple of G, nseg recounted."""
  G, best = 1, 0.0
  for g in range(1, min(16, S) + 1):
    eff = g * K / (32.0 * -(-g * K // 32))
    if eff > best + 1e-9:
      best, G = eff, g
  want = num_sms * 32
  nseg = max(1, min(-(-want // num_rays), max(1, S // (2 * G))))
  seg_len = -(-(-(-S // nseg)) // G) * G
  nseg = -(-S // seg_len)
  return types.SimpleNamespace(G=G, nseg=nseg, seg_len=seg_len)


def passes(S, K, p):
  """[(sample index [32], basis index [32])] of every 32-lane pass of one ray, in the fast kernel's order: segments,
  groups of G samples, passes over the group's g*K items with the tail lanes repeating the last item."""
  out = []
  lane = np.arange(32)
  for seg in range(p.nseg):
    s_begin, s_end = seg * p.seg_len, min(S, (seg + 1) * p.seg_len)
    for s0 in range(s_begin, s_end, p.G):
      g = min(p.G, s_end - s0)
      for j0 in range(0, g * K, 32):
        j = np.minimum(j0 + lane, g * K - 1)
        out.append((s0 + j // K, j % K))
  return out


def tiers(ref, p, min_deg, max_deg):
  """Which sine form each pass of the fast kernel takes, from the fp64 lifted means: with ymax the largest
  |lm 2^min_deg| over the pass's lanes, the first n_fast = clamp(floor(log2(311 / ymax)) + 1, 0, L) degrees use
  sin_below_100pi (ymax == 0: all of them); the rest use safe_sin_nobranch where ymax 2^(L+1) < 1e9 and
  safe_sin_fast otherwise.  Returns n_fast [rays, passes], the tier of the remaining degrees (2 or 3), `unsure`
  where ymax is within 1e-5 of a threshold, and for the tests' reachability assertions: `padded` (passes with
  repeated tail lanes), `mixed` (lanes' |y| spread over more than 1e3) and `zero` (ymax == 0)."""
  L = max_deg - min_deg
  S, K = ref.lm.shape[1], ref.lm.shape[2]
  ps = passes(S, K, p)
  y = ref.lm.abs() * 2.0 ** min_deg
  lanes = torch.stack([y[:, torch.as_tensor(s), torch.as_tensor(k)] for s, k in ps], 1)      # [rays, passes, 32]
  ymax, ymin = lanes.amax(-1), lanes.amin(-1)
  q = 311.0 / ymax
  n_fast = torch.where(ymax > 0, torch.floor(torch.log2(q)) + 1, torch.tensor(float(L), dtype=torch.float64)).clamp(0, L)
  frac = torch.log2(q) - torch.floor(torch.log2(q))
  top = ymax * 2.0 ** (L + 1)
  unsure = ((ymax > 0) & (torch.minimum(frac, 1 - frac) < 2e-5)) | ((top / 1e9 - 1).abs() < 1e-5)
  rest = torch.where(top < 1e9, 2, 3)
  padded = torch.tensor([len(set(zip(s.tolist(), k.tolist()))) < 32 for s, k in ps])
  return types.SimpleNamespace(n_fast=n_fast.long(), rest=rest, unsure=unsure, padded=padded,
                               mixed=(ymax > 1e3 * ymin) & (ymin > 0), zero=ymax == 0,
                               count=lambda t: int(((n_fast > 0) if t == 1 else (n_fast < L) & (rest == t)).sum()))


def pos_enc_reference(viewdirs, deg):
  """coord.pos_enc(viewdirs, 0, deg) in fp64 with the bound of the kernel's bf16 value: x 2^l is exact, the cosine
  half adds fl32(pi/2) in fp32 (u |x + pi/2| and the constant's own error), sinf is documented at 1 ulp (2u), and
  the store rounds to bf16.  The identity columns only round to bf16."""
  v = viewdirs.detach().cpu().double()
  enc = o_coord.pos_enc(v, 0, deg)
  sc = 2.0 ** torch.arange(deg, dtype=torch.float64)
  x = (v[..., None, :] * sc[:, None]).reshape(v.shape[0], -1)
  darg = torch.cat([torch.zeros_like(x), U * (x + 0.5 * math.pi).abs() + abs(HALF_PI32 - 0.5 * math.pi)], -1)
  b = torch.cat([torch.zeros_like(v), SLACK * (darg + 2 * U)], -1)
  return enc, bf16_bound(enc, b)
