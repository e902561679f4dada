"""Reference of the Ref-NeRF stage and the colourless normals stage (csrc/refnerf.cu) with a bound on every element.

`reference` takes exactly the inputs of mnrf_refdir_fwd / mnrf_refdir_bwd -- fp32 grad_pred [M, 3], raw_rough [M],
raw_grad_density [3, M], viewdirs [M / S, 3], weights [M], the bf16 direction-encoding gradient d_slab, the fp32 IDE
table and the descriptor fields, the two loss multipliers and the optional head gradients -- and evaluates the
oracle's own chain in float64 (complex128 for the IDE): o_coord.l2_normalize, o_coord.reflect, generate_ide_fn or
pos_enc, softplus roughness (logaddexp(x, 0), jax.nn.softplus), n.v, the orientation and predicted-normal losses of
o_train, and torch.autograd for the adjoint and extra_dw.  Beside the values it returns how far the kernels' fp32
arithmetic may stray from them, element by element.

Bounds are running errors, not estimates.  `walk` is the kernels' arithmetic written once against a backend; with
`Running` (fp64 value, absolute error bound) every operation adds its rounding to the errors it inherits, with
u = 2**-24:
  a + b, a * b   e_a + e_b + u |result|;  |a| e_b + |b| e_a + e_a e_b + u |result|.  Every a * b + c is written as a
                 fused multiply-add: the unfused pair rounds twice, the fused one once, and the rule charges both
                 roundings, so it holds whichever the compiler chose (refnerf.cu is built with contraction).  A sum
                 carries u |partial sum| of every addition and the errors of its terms, so cancellation -- the
                 IDE's P_l^m from monomials z^k with coefficients up to 9e4 at l = 16 -- is bounded by the terms and
                 not by the result.
  coefficients   the fp32 ide_mat is the fp64 table rounded: u |c| each.
  a / b, sqrt    correctly rounded (no fast-math): (e_a + |a / b| e_b) / (|b| - e_b) + u |result|.
  library        the CUDA Math API's documented maximum errors: expf, exp2f, sinf, cosf 2 ulp, log1pf 1 ulp, an ulp
                 taken as 2u of the result; each after the inherited error through the function's own slope.
  min, max       1-Lipschitz: the error is inherited unchanged.  So fminf(0, p) of the orientation loss, and the
                 kernel's `p < 0` test, need no staging: the adjoint it guards, 2 w om p v, is continuous at 0.
  clamp          neg_normalize's clamp !(|g|^2 > eps) switches the adjoint between two forms that differ at the
                 boundary, so it is staged on the kernel's own fp32 |g|^2 (with and without contraction; `unsure`
                 marks a row where the two disagree, none in practice).  g = (2^-12, 2^-12, 0) gives |g|^2 = eps
                 exactly in every order: clamped.
  bf16           the slab is rounded to nearest: half a bf16 ulp of (|value| + bound) on top.
  stats          each thread sums its samples over the grid-stride iterations, a 5-level butterfly sums a warp, one
                 atomicAdd per warp in any order: each term passes through at most iterations + 5 + warps additions,
                 u |term| each.
The walk's values agree with the oracle's to fp64 rounding; their difference is added to the bound and
test_refdir_reference_cpu.py asserts it stays negligible.  First-order terms are scaled by 1.05 like the other
reference files.  An element whose bound says nothing -- above VACUOUS for the slab (values are at most ~1.6), above
VACUOUS |value| for a gradient that is not exactly zero -- is marked `vacuous`; the tests count it per degree and hold each case to a floor.

`plan` restates the host's block count of all four entry points.  Pure torch; runs wherever its inputs are (the
large-M cases run in fp64 on the GPU) and never loads the CUDA library.
"""
import math
import types

import numpy as np
import torch

from encode_ref import SLACK, TINY, U
from oracle import o_coord

EPS = float(np.finfo(np.float32).eps)        # kEps
HALF_PI = 0.5 * math.pi
HALF_PI32 = 1.57079637050628662109375       # the kernels' fl32(pi / 2)
VACUOUS = 0.25
ULP = {'exp': 2, 'exp2': 2, 'sin': 2, 'cos': 2, 'log1p': 1}


class E:
  """fp64 value with a bound on the absolute error of the kernel's fp32 value; see the module docstring."""

  def __init__(self, val, err=None):
    self.val = val
    self.err = torch.zeros_like(val) if err is None else err

  @staticmethod
  def of(x):
    return x if isinstance(x, E) else E(torch.as_tensor(x, dtype=torch.float64))

  @staticmethod
  def _r(v, e):
    return E(v, e + U * (v.abs() + e))

  def __add__(self, o):
    o = E.of(o)
    return E._r(self.val + o.val, self.err + o.err)

  __radd__ = __add__

  def __sub__(self, o):
    o = E.of(o)
    return E._r(self.val - o.val, self.err + o.err)

  def __rsub__(self, o):
    return E.of(o) - self

  def __mul__(self, o):
    o = E.of(o)
    return E._r(self.val * o.val, self.val.abs() * o.err + o.val.abs() * self.err + self.err * o.err)

  __rmul__ = __mul__

  def __truediv__(self, o):
    o = E.of(o)
    v = self.val / o.val
    low = o.val.abs() - o.err
    e = torch.where(low > 0, (self.err + v.abs() * o.err) / low.clamp(min=1e-300), torch.full_like(v, math.inf))
    return E._r(v, e)

  def __rtruediv__(self, o):
    return E.of(o) / self

  def __neg__(self):
    return E(-self.val, self.err)

  def __getitem__(self, i):
    return E(self.val[i], self.err[i])

  def col(self):
    return E(self.val[..., None], self.err[..., None])


class Running:
  """The `walk` backend of the bounds: E values."""
  fused = None

  def __init__(self, device='cpu'):
    self.device = device

  def inp(self, x):
    return E(x.detach().to(self.device, torch.float64))

  def coef(self, c32, c64):
    c = torch.as_tensor(c64).to(self.device, torch.float64)
    return E(c, U * c.abs())

  def imul(self, k, x):
    """(float)k * x: k an integer or an integer vector over the trailing axis"""
    return E(torch.as_tensor(k, dtype=torch.float64, device=self.device)) * x

  def mask(self, m):
    return m.to(self.device)

  def cst(self, v64, v32):
    return E(torch.tensor(v64, dtype=torch.float64, device=self.device),
             torch.tensor(abs(v32 - v64), dtype=torch.float64, device=self.device))

  def zeros(self, shape):
    return E(torch.zeros(shape, dtype=torch.float64, device=self.device))

  def fma(self, a, b, c):
    return a * b + c

  def scale(self, x, p):
    return E(x.val * p, x.err * abs(p))

  def sqrt(self, x):
    v = torch.sqrt(x.val)
    return E._r(v, v - torch.sqrt((x.val - x.err).clamp(min=0)))

  def _lib(self, name, v, e):
    return E(v, e + 2 * ULP[name] * U * (v.abs() + e) + TINY)

  def exp(self, x):
    v = torch.exp(x.val)
    return self._lib('exp', v, v * torch.expm1(x.err.clamp(max=700)))

  def exp2(self, l):
    v = torch.tensor(2.0 ** l, dtype=torch.float64, device=self.device)
    return self._lib('exp2', v, torch.zeros_like(v))

  def log1p(self, x):
    v = torch.log1p(x.val)
    low = 1 + x.val - x.err
    e = torch.where(low > 0, x.err / low.clamp(min=1e-300), torch.full_like(v, math.inf))
    return self._lib('log1p', v, e)

  def sin(self, x):
    v = torch.sin(x.val)
    return self._lib('sin', v, x.err.clamp(max=2.0))

  def cos(self, x):
    v = torch.cos(x.val)
    return self._lib('cos', v, x.err.clamp(max=2.0))

  def fmax0(self, x):
    return E(x.val.clamp(min=0), x.err)

  def fmin0(self, x):
    return E(x.val.clamp(max=0), x.err)

  def maxc(self, x, c):
    return E(x.val.clamp(min=c), x.err)

  def abs(self, x):
    return E(x.val.abs(), x.err)

  def where(self, c, a, b):
    a, b = E.of(a), E.of(b)
    return E(torch.where(c, a.val, b.val), torch.where(c, a.err, b.err))

  def col(self, x):
    return x.col()

  def cat(self, xs):
    return E(torch.cat([x.val for x in xs], -1), torch.cat([x.err for x in xs], -1))

  def clamped(self, g):
    """neg_normalize's branch on the kernel's fp32 |g|^2: (clamped, unsure)."""
    g32 = [x.val.float() for x in g]
    unfused = (g32[0] * g32[0] + g32[1] * g32[1]) + g32[2] * g32[2]
    g64 = [x.double() for x in g32]
    fused = ((g64[2] * g64[2] + ((g64[1] * g64[1] + (g64[0] * g64[0]).float().double())).float().double())
             ).float()
    cu, cf = ~(unfused > EPS), ~(fused > EPS)
    return cf, cu != cf

  def orient_add(self, p, t_scale, v, a):
    """if (p < 0) a = fma(t_scale p, -v, a): continuous in p, so taken through fminf(0, p); where p's bound keeps it
    positive the kernel's p is positive too and a is untouched."""
    return self.where(p.val - p.err > 0, a, a + (t_scale * self.fmin0(p)) * (-v))


def _dot(b, x, y):
  return b.fma(x[2], y[2], b.fma(x[1], y[1], x[0] * y[0]))


def _neg_normalize(b, g):
  sq = _dot(b, g, g)
  cl = b.clamped(g)
  s = b.sqrt(b.maxc(sq, EPS))
  return [-(gi / s) for gi in g], s, cl


def _neg_normalize_bwd(b, out, s, cl, a, mut=None):
  dot = _dot(b, out, a)
  c = cl[0] & False if mut == 'project_clamped' else cl[0]
  return [b.where(c, -(a[i] / s), -(b.fma(-out[i], dot, a[i]) / s)) for i in range(3)]


def _softplus(b, x):
  return b.fmax0(x) + b.log1p(b.exp(-b.abs(x)))


def walk(b, x, f, bwd=False, mut=None):
  """The arithmetic of refdir_fwd_kernel (bwd=False) or refdir_bwd_kernel (bwd=True) on backend `b`.

  x: fp32 inputs per sample (gp [M, 3] or None, rgd [3, M] or None, rr [M] or None, v [M, 3] gathered by ray, w [M],
  gin [M, W] the d_slab columns from col0 as fp32, mat [zdeg, n] fp32 and mat64, m / l [n], the optional heads);
  f: descriptor flags and loss scalars.  `mut` names a kernel bug for the CPU tests' mutants; the reference passes
  None.  Returns a namespace of backend values."""
  o = types.SimpleNamespace()
  use_p, use_d = f['use_pred_normals'], f['use_density_normals']
  v = [b.inp(x.v[:, i]) for i in range(3)]
  zero = b.zeros(x.v.shape[:1])
  p = d = [zero, zero, zero]
  cl_p = cl_d = None
  if use_p:
    p, s_p, cl_p = _neg_normalize(b, [b.inp(x.gp[:, i]) for i in range(3)])
  if use_d:
    d, s_d, cl_d = _neg_normalize(b, [b.inp(x.rgd[i]) for i in range(3)])
  o.p, o.d, o.cl_p, o.cl_d = p, d, cl_p, cl_d
  up = use_p if mut != 'ndv_other' else not use_p
  n = p if use_p else d
  nv = p if up else d
  kappa = rin = None
  if f['use_roughness']:
    rin = b.inp(x.rr) + f['bias']
    kappa = _softplus(b, rin)
  o.roughness = kappa
  om, pm = f['orient_mult'], f['prednorm_mult']
  oop = f['orient_on_pred'] if mut != 'orient_flag' else True
  tgt = p if oop else d

  def orient_p():
    return -_dot(b, tgt, v)
  if not bwd:
    dw = zero
    if om > 0:
      pmv = b.fmin0(orient_p())
      dw = (om * pmv) * pmv
    if pm > 0:
      dw = b.fma(pm, 1.0 - _dot(b, d, p), dw)
    o.extra_dw = dw
  ndv = _dot(b, nv, v)
  dir_ = list(v)
  if f['use_reflections']:
    s2 = b.scale(ndv, 2.0 if mut != 'reflect_plus' else -2.0)
    dir_ = [b.fma(-s2, n[i], v[i]) for i in range(3)]
  o.dir = dir_
  W = f['col_end'] - f['col0']
  cols = []
  deg = f['deg_view']
  dk, u = zero, None
  if f['use_ide']:
    n_ = len(x.m)
    mi = torch.as_tensor(x.m, dtype=torch.int64)
    sigma = torch.as_tensor(x.l, dtype=torch.float32)
    sigma = sigma * (sigma + 1) * (1.0 if mut == 'sigma_full' else 0.5)
    zdeg = (1 << (deg - 1)) + 1
    zp = [b.inp(torch.ones(x.v.shape[0]))]
    for k in range(1, zdeg):
      zp.append(zp[-1] * dir_[2])
    P = dP = b.zeros(x.v.shape[:1] + (n_,))
    for k in range(zdeg - 1 if mut == 'drop_last_z' else zdeg):
      co = b.coef(x.mat[k], x.mat64[k])
      P = b.fma(b.col(zp[k]), co, P)
      if bwd and k > 0:
        dP = b.fma(b.imul(k if mut != 'dP_no_k' else 1, b.col(zp[k - 1])), co, dP)
    # (x + iy)^m by repeated multiplication; e = m (x + iy)^(m - 1) captured on the last step
    cr, ci = b.inp(torch.ones(x.v.shape[0], n_)), b.zeros(x.v.shape[:1] + (n_,))
    er = ei = b.zeros(x.v.shape[:1] + (n_,))
    dx, dy = b.col(dir_[0]), b.col(dir_[1])
    late = 1 if mut == 'e_late' else 0
    for q in range(int(mi.max()) + late):
      act, cap = b.mask((q < mi)[None, :]), b.mask((q == mi - 1 + late)[None, :])
      if bwd:
        er = b.where(cap, b.imul(x.m, cr), er)
        ei = b.where(cap, b.imul(x.m, ci), ei)
      t = b.fma(cr, dx, -(ci * dy))
      ci2 = b.fma(cr, dy, ci * dx)
      cr = b.where(act, t, cr)
      ci = b.where(act, ci2, ci)
    if mut == 'conjugate':
      ci, ei = -ci, -ei
    sg = b.inp(-sigma)
    A = b.exp(sg * b.col(kappa))
    if not bwd:
      cols += [(cr * P) * A, (ci * P) * A]
    else:
      gr, gi = b.inp(x.gin[:, :n_]), b.inp(x.gin[:, n_:2 * n_])
      s = b.fma(gi, ci, gr * cr)
      se = b.fma(gi, ei, gr * er)
      so = b.fma(gi, er, (-gr) * ei)
      tk, t2, tp = (sg * A) * P, A * dP, A * P
      u = [zero, zero, zero]
      for i in range(n_):
        dk = b.fma(tk[:, i], s[:, i], dk)
        u[2] = b.fma(t2[:, i], s[:, i], u[2])
        u[0] = b.fma(tp[:, i], se[:, i], u[0])
        u[1] = b.fma(tp[:, i], so[:, i], u[1])
    c = 2 * len(x.m)
  else:
    if not bwd:
      cols.append(b.cat([b.col(dir_[i]) for i in range(3)]))
    else:
      u = [b.inp(x.gin[:, i]) for i in range(3)]
    pe = []
    for half in range(2):
      for l in range(deg):
        for ch in range(3):
          sc = b.exp2(l)
          xa = dir_[ch] * sc
          if half:
            xa = xa + b.cst(-HALF_PI, -HALF_PI32) if mut == 'cos_minus' else xa + b.cst(HALF_PI, HALF_PI32)
          if not bwd:
            pe.append(b.col(b.sin(xa)))
          else:
            g = b.inp(x.gin[:, 3 + half * 3 * deg + l * 3 + ch])
            u[ch] = b.fma(g * b.cos(xa), sc, u[ch])
    if not bwd and pe:
      cols.append(b.cat(pe))
    c = 3 + 6 * deg
  if f['use_n_dot_v']:
    if not bwd:
      cols.append(b.col(ndv))
    c += 1
  o.enc_width = c
  if not bwd:
    o.enc = b.cat(cols)
    o.width = W
    return o
  # ---- backward
  a_n = [zero, zero, zero]
  if f['use_n_dot_v']:
    gq = b.inp(x.gin[:, c - 1])
    a_n = [b.fma(gq, v[i], zero) for i in range(3)]
  if f['use_reflections']:
    un = _dot(b, u, n)
    m2u, p2 = b.scale(un, -2.0), b.scale(ndv, 2.0)
    a_n = [a_n[i] + b.fma(-p2, u[i], m2u * v[i]) for i in range(3)]
  a_p, a_d = ([a_n, [zero] * 3] if use_p else [[zero] * 3, a_n])
  w = b.inp(x.w if mut != 'next_weight' else torch.cat([x.w[1:], x.w[:1]]))
  o.st_or = o.st_pn = zero
  if om > 0:
    pr = orient_p()
    pmv = b.fmin0(pr)
    omw = om * w
    o.st_or = (omw * pmv) * pmv
    ts = b.scale(omw, 2.0)
    if oop:
      a_p = [b.orient_add(pr, ts, v[i], a_p[i]) for i in range(3)]
    else:
      a_d = [b.orient_add(pr, ts, v[i], a_d[i]) for i in range(3)]
  if pm > 0:
    pmw = pm * w
    o.st_pn = pmw * (1.0 - _dot(b, d, p))
    a_p = [b.fma(-pmw, d[i], a_p[i]) for i in range(3)]
    a_d = [b.fma(-pmw, p[i], a_d[i]) for i in range(3)]
  o.d_grad_pred = _neg_normalize_bwd(b, p, s_p, cl_p, a_p, mut) if use_p else None
  o.d_raw_grad_density = _neg_normalize_bwd(b, d, s_d, cl_d, a_d, mut) if use_d else None
  o.d_raw_rough = None
  if f['use_roughness']:
    sig = 1.0 / (1.0 + b.exp(-rin))
    o.d_raw_rough = dk if mut == 'no_sigmoid' else dk * sig
  return o


def plan(M, num_sms):
  """Blocks and grid-stride iterations of all four entry points: min(ceil(M / 128), 16 SMs) blocks of 128."""
  blocks = min((M + 127) // 128, 16 * num_sms)
  return types.SimpleNamespace(blocks=blocks, threads=blocks * 128, iters=-(-M // (blocks * 128)) if M else 0,
                               warps=blocks * 4)


def ide_degree_of(deg_view, n_dot_v=False):
  """l of each IDE slab column (real parts then imaginary parts); -1 for n.v."""
  ls = [2 ** i for i in range(deg_view) for _ in range(2 ** i + 1)]
  return torch.tensor(ls + ls + ([-1] if n_dot_v else []))


def pe_degree_of(deg_view, n_dot_v=False):
  """Frequency index of each PE slab column; -1 for the identity columns and n.v."""
  d = torch.arange(deg_view).repeat_interleave(3)
  return torch.cat([torch.full((3,), -1), d, d] + ([torch.tensor([-1])] if n_dot_v else []))


def _stage(g, cl):
  """-l2_normalize(g) with neg_normalize's branch taken where the kernel took it."""
  s_cl = math.sqrt(EPS)
  return -torch.where(cl[..., None], g / s_cl, o_coord.l2_normalize(g))


def oracle(x, f, dtype=torch.float64, cl_p=None, cl_d=None, device='cpu', graph=False):
  """The oracle chain: dict of forward values and, with x.gin, autograd of the slab gradient and the two losses.
  graph: x's tensors are the leaves (gradcheck); `loss_terms` is the two losses per sample and nothing is
  differentiated here."""
  c = lambda t: None if t is None else (t if graph else t.detach().to(device, dtype).requires_grad_(True))
  gp, rgd, rr = c(x.gp), c(x.rgd), c(x.rr)
  w = x.w.detach().to(device, dtype).requires_grad_(True) if x.w is not None else None
  v = x.v.to(device, dtype)
  M = v.shape[0]
  out = {}
  z = torch.zeros(M, 3, dtype=dtype, device=device)
  if gp is not None and f['use_pred_normals']:
    cp = cl_p if cl_p is not None else torch.zeros(M, dtype=torch.bool, device=device)
    npd = _stage(gp, cp.to(device)) if dtype == torch.float64 else -o_coord.l2_normalize(gp)
  else:
    npd = z
  if rgd is not None and f['use_density_normals']:
    cd = cl_d if cl_d is not None else torch.zeros(M, dtype=torch.bool, device=device)
    nd = _stage(rgd.T, cd.to(device)) if dtype == torch.float64 else -o_coord.l2_normalize(rgd.T)
  else:
    nd = z
  out['normals_pred'], out['normals'] = npd, nd
  n = npd if f['use_pred_normals'] else nd
  rough = None
  if f['use_roughness']:
    rin = rr + f['bias']
    rough = torch.logaddexp(rin, torch.zeros_like(rin))
    out['roughness'] = rough
  om, pm = f['orient_mult'], f['prednorm_mult']
  tgt = npd if f['orient_on_pred'] else nd
  l_or = om * torch.clamp((tgt * -v).sum(-1), max=0.0) ** 2 * w if (om > 0 and w is not None) else None
  l_pn = pm * w * (1.0 - (nd * npd).sum(-1)) if (pm > 0 and w is not None) else None
  dirs = o_coord.reflect(-v, n) if f['use_reflections'] else v
  if f['use_ide']:
    # the oracle builds its table on the CPU
    enc = o_coord.generate_ide_fn(f['deg_view'])(dirs.cpu(), rough.cpu()[:, None]).to(device)
  else:
    enc = o_coord.pos_enc(dirs, 0, f['deg_view'])
  if f['use_n_dot_v']:
    enc = torch.cat([enc, (n * v).sum(-1, keepdim=True)], -1)
  out['enc'] = enc
  if graph:
    out['loss_terms'] = sum(t for t in (l_or, l_pn) if t is not None) if (l_or is not None or l_pn is not None) \
        else torch.zeros(M, dtype=dtype)
    return out
  terms = [t.sum() for t in (l_or, l_pn) if t is not None]
  if terms:
    out['extra_dw'] = torch.autograd.grad(sum(terms), w, retain_graph=True)[0]
  else:
    out['extra_dw'] = torch.zeros(M, dtype=dtype, device=device)
  out['st_or'] = l_or.sum() if l_or is not None else torch.zeros((), dtype=dtype, device=device)
  out['st_pn'] = l_pn.sum() if l_pn is not None else torch.zeros((), dtype=dtype, device=device)
  if getattr(x, 'gin', None) is not None:
    gin = x.gin[:, :enc.shape[1]].to(device, dtype)
    loss = (enc * gin).sum() + sum(terms)
    leaves = [t for t in (gp, rr, rgd) if t is not None and loss.requires_grad]
    grads = torch.autograd.grad(loss, leaves, allow_unused=True) if leaves else []
    gmap = {id(t): g_ for t, g_ in zip(leaves, grads)}
    get = lambda t: None if t is None else (torch.zeros_like(t) if gmap.get(id(t)) is None else gmap[id(t)])
    out['d_grad_pred'], out['d_raw_rough'], out['d_raw_grad_density'] = get(gp), get(rr), get(rgd)
  return out


def head_slab(W, d_raw_density=None, d_grad_pred=None, d_raw_diffuse=None, d_raw_tint=None, d_raw_rough=None):
  """What refdir_bwd writes over d_slab[:, col0:col_end]: bf16 of [d raw_density | d grad_pred | d raw_diffuse |
  d raw_tint | d raw_rough] (zeros where absent) from the kernel's own fp32 outputs and the passed-through heads, then
  zeros to col_end.  [M, W] float32 holding bf16 values."""
  M = next(t for t in (d_raw_density, d_grad_pred, d_raw_diffuse, d_raw_tint, d_raw_rough) if t is not None).shape[0]
  h = torch.zeros(M, W)
  for c, t in ((0, d_raw_density), (1, d_grad_pred), (4, d_raw_diffuse), (7, d_raw_tint), (10, d_raw_rough)):
    if t is not None:
      t = t.detach().float().cpu().reshape(M, -1)
      h[:, c:c + t.shape[1]] = t
  return h.to(torch.bfloat16).float()


def bf16_bound(value, bound):
  return bound + 2.0 ** -8 * (value.abs() + bound) + 2.0 ** -134


def _bound(e, ref):
  gap = (e.val - ref).abs()
  return SLACK * (e.err + gap) + TINY, float((gap / (e.err + 1e-300)).max()) if gap.numel() else 0.0


def reference(x, f, *, num_sms=132, bwd=True, device='cpu'):
  """fp64 reference of mnrf_refdir_fwd (and, with bwd and x.gin, mnrf_refdir_bwd) with per-element bounds.

  Returns a namespace: for each output its value (the oracle's), `<name>_bound` and `<name>_vacuous`; slab values /
  bounds [M, col_end - col0] (bf16 rounding included, zeros past the encoding); `stats_or` / `stats_pn` with their
  bounds; `unsure` rows where the clamp is not decided; `chain_gap`, how far the walk's values are from the oracle's
  in units of their own bound (asserted small on the CPU)."""
  b = Running(device)
  r = types.SimpleNamespace(chain_gap=0.0)
  fw = walk(b, x, f)
  cl_p, cl_d = fw.cl_p, fw.cl_d
  r.unsure = torch.zeros(x.v.shape[0], dtype=torch.bool, device=device)
  for c in (cl_p, cl_d):
    if c is not None:
      r.unsure |= c[1]
  orc = oracle(x, f, cl_p=None if cl_p is None else cl_p[0], cl_d=None if cl_d is None else cl_d[0], device=device)

  def put(name, e, ref, rel=False):
    ref = ref.detach()
    bd, gap = _bound(e, ref)
    r.chain_gap = max(r.chain_gap, gap)
    setattr(r, name, ref)
    setattr(r, name + '_bound', bd)
    setattr(r, name + '_vacuous', bd > (VACUOUS * ref.abs() + 2 * TINY if rel else VACUOUS))
  if f['use_pred_normals']:
    put('normals_pred', b.cat([t.col() for t in fw.p]), orc['normals_pred'])
  if f['use_density_normals']:
    put('normals', b.cat([t.col() for t in fw.d]), orc['normals'])
  if f['use_roughness']:
    put('roughness', fw.roughness, orc['roughness'], rel=True)
  put('extra_dw', fw.extra_dw, orc['extra_dw'], rel=True)
  enc_b, gap = _bound(fw.enc, orc['enc'])
  r.chain_gap = max(r.chain_gap, gap)
  W = f['col_end'] - f['col0']
  M = x.v.shape[0]
  r.slab = torch.zeros(M, W, dtype=torch.float64, device=device)
  r.slab_bound = torch.full_like(r.slab, TINY)
  ne = orc['enc'].shape[1]
  r.slab[:, :ne] = orc['enc'].detach()
  r.slab_bound[:, :ne] = bf16_bound(orc['enc'].detach(), enc_b)
  r.slab_vacuous = r.slab_bound > VACUOUS
  r.enc_width = ne
  if not bwd or getattr(x, 'gin', None) is None:
    return r
  bw = walk(b, x, f, bwd=True)
  if f['use_pred_normals']:
    put('d_grad_pred', b.cat([t.col() for t in bw.d_grad_pred]), orc['d_grad_pred'], rel=True)
    r.d_grad_pred_vacuous |= r.unsure[:, None]
  if f['use_density_normals']:
    g = b.cat([t.col() for t in bw.d_raw_grad_density])
    put('d_raw_grad_density', E(g.val.T.contiguous(), g.err.T.contiguous()), orc['d_raw_grad_density'], rel=True)
    r.d_raw_grad_density_vacuous |= r.unsure[None, :]
  if f['use_roughness']:
    put('d_raw_rough', bw.d_raw_rough, orc['d_raw_rough'], rel=True)
  p = plan(M, num_sms)
  depth = p.iters + 5 + p.warps
  for name, t in (('stats_or', bw.st_or), ('stats_pn', bw.st_pn)):
    tot = E(t.val.sum(), t.err.sum())
    ref = orc['st_or' if name == 'stats_or' else 'st_pn'].detach()
    bd, gap = _bound(tot, ref)
    r.chain_gap = max(r.chain_gap, gap)
    setattr(r, name, ref)
    setattr(r, name + '_bound', bd + SLACK * depth * U * t.val.abs().sum())
  return r
