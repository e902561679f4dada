"""Reference of the proposal resampler (csrc/sampling.cu) with a per-element error bound, built from the oracle.

`reference` takes exactly the inputs of mnrf_sample_level -- fp32 fenceposts and weights, the descriptor's fp32
scalars, the u grid, max_jitter and the jitter -- and evaluates the oracle's own step-function algebra
(o_stepfun.weight_to_pdf / max_dilate / pdf_to_weight, softmax, integrate_weights, o_math.sorted_interp) in
float64.  For every stage the kernel exposes it returns the fp64 value and how far the kernel's fp32 arithmetic may
stray from it.  With u = 2**-24 the fp32 unit roundoff, kw = ceil(3P/32) and kc = ceil(nb/32) the terms each lane
adds in the kernel's lane-strided sums, and every first-order bound scaled by 1.05 for the higher-order terms:

  tdil    exact.  t -/+ dilation is fp32 in the reference too, so the fenceposts are formed in fp32 and sorted,
          clamped to the domain and trimmed as max_dilate does; the kernel's 3-way merge must match bit for bit.
  wdil    |w - w64| <= (kw + 16) u w64 + 2**-120: dt and the pdf division (2u), the width and the product of
          pdf_to_weight (2u), the lane-strided plus butterfly sum of 3P positive terms ((kw + 5) u, all of it
          relative to the sum), the renormalising division (u), with slack; 2**-120 covers subnormal products.
          Without dilation wdil is the input itself.
  cw      |cw_k - cw64_k| <= b_k = sum_{i<k} q_i (r_i + u) + (R + (2 kc + 6) u) cw64_k.  q is the fp64 softmax and
          r_i the relative error of the kernel's softmax numerator exp(l_i - max l):
            r_i = anneal (e_i + 3u |log x_i|) + u |l_i - max l| + 4u,
          x_i = wdil_i + padding with relative error e_i (the wdil bound and the add; without padding only the
          per-weight 6u of it, since the renormalising sum shifts every logit alike), logf (1 ulp = 2u) and the
          anneal product (u) on |anneal log x_i|, the max subtraction, expf (2 ulp = 4u).  R = sum_i q_i r_i +
          (kc + 5) u is the relative error of the lane-strided sum of the numerators, u the division, and
          (2 kc + 6) u the prefix: kc - 1 sequential adds per lane chunk, 5 shuffle-scan adds and up to kc adds into
          the running value, each relative to at most cw_k.  cw_0 = 0 and cw_nb = 1 are exact.  At nb = 3070 this
          is about 1.2e-5 cw plus the softmax terms, far below one bin's mass.
  idx     The kernel's count #{cw' <= u} lies in [n_lo, n_hi], n_lo = #{k : cw64_k + b_k <= u} and
          n_hi = #{k : cw64_k - b_k <= u}; the index is count - 1.  Where u is farther than b from every knot
          n_lo == n_hi and the index equals the fp64 index.
  centre  F^-1 (sorted_interp on the fp64 CDF) is monotone, and the kernel's centre x solves G(x) = u on a CDF G
          within d of F on its segment, so x lies in [F^-1(u - d), F^-1(u + d)], d = max b_k over the knots the
          kernel's segment can end on ([n_lo - 1, n_hi]).  The bracket is widened by 12u max |td| over those knots
          for the division, the product and the sum of the interpolation.
  sdist   interval arithmetic on the centre brackets: midpoints [(lo_s + lo_{s-1})/2, (hi_s + hi_{s-1})/2]; the
          reflected first end 2 c0 - (c1 + c0)/2 = 1.5 c0 - 0.5 c1, increasing in c0 and decreasing in c1, so
          [2 lo_0 - (hi_1 + lo_0)/2, 2 hi_0 - (lo_1 + hi_0)/2] (the last end likewise); widened by the midpoint and
          reflection roundings (2u of the operands), then clamped to the domain.

A row whose fp64 CDF is NaN (every logit -inf, or anneal 0 times log 0) follows the oracle exactly: the inner knots
of the CDF are NaN, every sample collapses onto the first fencepost, and every index is 0.

Evaluated in float32 (`dtype=torch.float32`) the same chain is the fp32 oracle, with no bounds.  Pure torch: runs
on the CPU (CUDA inputs are copied there) and never loads the CUDA library.  Rays are evaluated in chunks, because
max_dilate and sorted_interp build [rays, n, n] masks.
"""
import math
import types

import numpy as np
import torch

from oracle import o_math, o_stepfun

U = 2.0 ** -24          # fp32 unit roundoff
EPS2 = o_stepfun.EPS ** 2
SLACK = 1.05


def f32(x):
  """A descriptor scalar as the kernel sees it (the descriptor holds fp32)."""
  return float(np.float32(x))


def kernel_u(u_base, jitter, jitter_mode, max_jitter, num_rays):
  """[rays, S] fp32 u as the kernel forms it: u_base, or fl(u_base + fl(jitter * max_jitter)) with one jitter per
  ray (mode 1) or per sample (mode 2)."""
  ub = u_base.detach().cpu().float()
  if jitter_mode == 0:
    return ub.expand(num_rays, -1)
  j = jitter.detach().cpu().float().reshape(num_rays, -1)
  assert j.shape[1] == (1 if jitter_mode == 1 else ub.shape[0])
  return ub + j * torch.tensor(f32(max_jitter))


def intervals(c_lo, c_hi, domain, widen=None):
  """stepfun.sample_intervals' interval endpoints from centre brackets [c_lo, c_hi] (c_lo is c_hi: the values):
  midpoints, and the ends reflected about the outer centres and clamped to the domain.  `widen`: per-row factor
  of the operands' magnitude added for the kernel's roundings."""
  mid_lo = (c_lo[..., 1:] + c_lo[..., :-1]) / 2
  mid_hi = (c_hi[..., 1:] + c_hi[..., :-1]) / 2
  first_lo = 2 * c_lo[..., :1] - (c_hi[..., 1:2] + c_lo[..., :1]) / 2
  first_hi = 2 * c_hi[..., :1] - (c_lo[..., 1:2] + c_hi[..., :1]) / 2
  last_lo = 2 * c_lo[..., -1:] - (c_lo[..., -1:] + c_hi[..., -2:-1]) / 2
  last_hi = 2 * c_hi[..., -1:] - (c_hi[..., -1:] + c_lo[..., -2:-1]) / 2
  lo = torch.cat([first_lo, mid_lo, last_lo], -1)
  hi = torch.cat([first_hi, mid_hi, last_hi], -1)
  if widen is not None:
    mag = torch.maximum(lo.abs(), hi.abs())
    ends = torch.zeros_like(mag)
    ends[..., 0] = 2 * torch.maximum(c_lo[..., 0].abs(), c_hi[..., 0].abs())
    ends[..., -1] = 2 * torch.maximum(c_lo[..., -1].abs(), c_hi[..., -1].abs())
    w = widen * (mag + ends)
    lo, hi = lo - w, hi + w
  lo = torch.cat([lo[..., :1].clamp(min=domain[0]), lo[..., 1:-1], lo[..., -1:].clamp(max=domain[1])], -1)
  hi = torch.cat([hi[..., :1].clamp(min=domain[0]), hi[..., 1:-1], hi[..., -1:].clamp(max=domain[1])], -1)
  return lo, hi


def _rows(t, w, u, cw_in, use_dilation, dil, domain, anneal, pad, dtype):
  P = w.shape[-1]
  bound = dtype == torch.float64
  if use_dilation:
    p = o_stepfun.weight_to_pdf(t.to(dtype), w.to(dtype))
    # fp32 fenceposts (t -/+ dilation in fp32, as in the reference), the max of the pdf in `dtype`
    td, pd = o_stepfun.max_dilate(t, p, torch.tensor(dil), domain=domain)
    wd = o_stepfun.pdf_to_weight(td.to(dtype), pd)
    wd = wd / torch.clamp(wd.sum(dim=-1, keepdim=True), min=EPS2)
    td, wd = td[..., 1:-1], wd[..., 1:-1]
    ew = (math.ceil(3 * P / 32) + 16) * U * SLACK
  else:
    td, wd = t, w.to(dtype)
    ew = 0.0
  nb = wd.shape[-1]
  tdd = td.to(dtype)
  out = types.SimpleNamespace(tdil=td, wdil=wd)
  if cw_in is None:
    x = wd + pad
    lgx = torch.log(x)
    logits = torch.where(td[..., 1:] > td[..., :-1], anneal * lgx, torch.tensor(-math.inf, dtype=dtype))
    q = torch.softmax(logits, dim=-1)
    cw = o_stepfun.integrate_weights(q)
  else:
    cw = cw_in.to(dtype)
  out.cw = cw
  uu = u.to(dtype)
  c, idx = o_math.sorted_interp(uu, cw, tdd, return_index=True)
  out.idx = idx
  out.sdist = intervals(c, c, domain)[0]
  if not bound:
    return out

  nan_row = torch.isnan(cw).any(dim=-1, keepdim=True)
  out.nan_row = nan_row[..., 0]
  out.wdil_bound = ew * wd + (2.0 ** -120 if use_dilation else 0.0)
  zero = torch.zeros((), dtype=dtype)
  if cw_in is None:
    kc = math.ceil(nb / 32)
    # the renormalising sum scales every weight alike, which the softmax cancels unless a padding is added
    ew_own = 6 * U * SLACK if use_dilation else 0.0
    ex = torch.where(x > 0, ((ew if pad > 0 else ew_own) * wd + U * x) / x, zero)
    r = anneal * (ex + 3 * U * lgx.abs()) + U * (logits - logits.amax(dim=-1, keepdim=True)).abs() + 4 * U
    r = torch.where(q > 0, r, zero)
    R = (q * r).sum(dim=-1, keepdim=True) + (kc + 5) * U
    b = torch.cumsum(q * (r + U), dim=-1)[..., :-1] + (R + (2 * kc + 6) * U) * cw[..., 1:-1]
    end = torch.zeros_like(cw[..., :1])
    b = torch.cat([end, SLACK * b + 2.0 ** -100, end], -1)
    b = torch.where(nan_row, zero, b)
  else:
    b = torch.zeros_like(cw)
  out.cw_bound = b

  n_lo = ((cw + b)[..., None, :] <= uu[..., None]).sum(dim=-1)
  n_hi = ((cw - b)[..., None, :] <= uu[..., None]).sum(dim=-1)
  out.idx_lo, out.idx_hi = n_lo - 1, n_hi - 1
  k = torch.arange(nb + 1)
  reach = (k >= (n_lo - 1).clamp(min=0)[..., None]) & (k <= n_hi.clamp(max=nb)[..., None])
  d = torch.where(reach, b[..., None, :], zero).amax(dim=-1)
  fmax = torch.where(reach, tdd.abs()[..., None, :], zero).amax(dim=-1)
  wid = torch.where(nan_row, zero, 12 * U * fmax)
  c_lo = o_math.sorted_interp(uu - d, cw, tdd) - wid
  c_hi = o_math.sorted_interp(uu + d, cw, tdd) + wid
  out.sdist_lo, out.sdist_hi = intervals(c_lo, c_hi, domain, widen=torch.where(nan_row, zero, 2 * U + zero))
  return out


def reference(sdist_prev, w_prev, num_samples, *, u_base, use_dilation=False, dilation=0.0, domain=(0.0, 1.0),
              anneal=1.0, resample_padding=0.0, jitter=None, jitter_mode=0, max_jitter=0.0, cw_in=None,
              dtype=torch.float64, max_elems=1 << 23):
  """Every stage of mnrf_sample_level on these inputs, evaluated in `dtype`; with float64 also the bounds of the
  module docstring.  `cw_in` (fp32): use this CDF instead of the softmax, as the kernel does (bounds of the
  interpolation alone).  Returns a namespace of CPU tensors: tdil (fp32), wdil, cw, sdist, idx (int64), u (fp32),
  and for float64 wdil_bound, cw_bound, sdist_lo / sdist_hi, idx_lo / idx_hi, nan_row."""
  t = sdist_prev.detach().cpu().float()
  w = w_prev.detach().cpu().float()
  B, P = w.shape
  assert t.shape == (B, P + 1)
  u = kernel_u(u_base, jitter, jitter_mode, max_jitter, B)
  assert u.shape == (B, num_samples)
  cw_in = None if cw_in is None else cw_in.detach().cpu().float()
  dom = (f32(domain[0]), f32(domain[1]))
  nb = 3 * P - 2 if use_dilation else P
  step = max(1, max_elems // max((3 * P + 1) * P if use_dilation else 1, (nb + 1) * num_samples))
  parts = [_rows(t[i:i + step], w[i:i + step], u[i:i + step], None if cw_in is None else cw_in[i:i + step],
                 use_dilation, f32(dilation), dom, f32(anneal), f32(resample_padding), dtype)
           for i in range(0, B, step)]
  out = types.SimpleNamespace(**{k: torch.cat([getattr(p, k) for p in parts]) for k in vars(parts[0])})
  out.u = u
  return out


def _ratio(x, ref, lo, hi):
  """|x - ref| over the room [lo, hi] leaves on that side of ref: <= 1 inside the bracket, inf outside an exact
  value; NaN counts as equal to NaN only."""
  x = x.detach().cpu().double()
  err = (x - ref).abs()
  room = torch.where(x >= ref, hi - ref, ref - lo)
  r = err / room
  r = torch.where((x == ref) | (torch.isnan(x) & torch.isnan(ref)), torch.zeros_like(r), r)
  return torch.where(torch.isnan(r), torch.full_like(r, math.inf), r)


def ratios(ref, sdist, idx=None, cw=None, tdil=None, wdil=None):
  """Worst err / bound of each kernel output against `reference(...)` (float64); exact checks give 0 or inf."""
  out = {'sdist': float(_ratio(sdist, ref.sdist, ref.sdist_lo, ref.sdist_hi).max())}
  if idx is not None:
    idx = idx.detach().cpu().long()
    ok = (idx >= ref.idx_lo) & (idx <= ref.idx_hi)
    out['idx'] = 0.0 if bool(ok.all()) else math.inf
  if cw is not None:
    out['cw'] = float(_ratio(cw, ref.cw, ref.cw - ref.cw_bound, ref.cw + ref.cw_bound).max())
  if wdil is not None:
    out['wdil'] = float(_ratio(wdil, ref.wdil, ref.wdil - ref.wdil_bound, ref.wdil + ref.wdil_bound).max())
  if tdil is not None:
    same = torch.equal(tdil.detach().cpu().float().view(torch.int32), ref.tdil.view(torch.int32))
    out['tdil'] = 0.0 if same else math.inf
  return out


def step_functions(rng, profile, B, P, domain=(0.0, 1.0), edges=True):
  """B fp32 step functions (fenceposts [B, P+1] inside `domain`, weights [B, P]) of one weight profile:
    random      cubed uniforms, normalised
    positive    uniforms in [0.05, 1), normalised: no zero weight
    peaked      one bin holds the weight, every other bin 1e-30
    zeros       random with runs of exact zeros (leading, trailing or inner, some longer than P/3)
    duplicates  random with runs of zero-width bins: the first bins, the last bins or inner ones
    uniform     equal weights on equally spaced fenceposts
  Even rows touch both domain ends.  With `edges` and B >= 8 the first four rows are the edge rows: all weights
  zero; a single nonzero bin; every fencepost but two equal; fenceposts on both domain ends."""
  lo, hi = domain if math.isfinite(domain[0]) and math.isfinite(domain[1]) else (3.0, 4.0)
  f = np.float32
  if profile == 'uniform':
    t = np.tile(np.linspace(lo, hi, P + 1, dtype=f), (B, 1))
    w = np.full((B, P), 1.0 / P, f)
    return torch.tensor(t), torch.tensor(w)
  t = np.sort(rng.uniform(lo, hi, (B, P + 1)).astype(f), -1)
  t[::2, 0], t[::2, -1] = lo, hi
  if profile == 'positive':
    w = rng.uniform(0.05, 1, (B, P))
  elif profile == 'peaked':
    w = np.full((B, P), 1e-30)
    w[np.arange(B), rng.integers(0, P, B)] = 1.0
  else:
    w = rng.uniform(0, 1, (B, P)) ** 3
  for r in range(B):
    n = int(rng.integers(1, max(2, P // 2)))
    a = (0, P - n, int(rng.integers(0, P - n + 1)))[r % 3]
    if profile == 'zeros':
      w[r, a:a + n] = 0
      if w[r].sum() == 0:
        w[r, 0 if a else -1] = 1.0
    elif profile == 'duplicates' and P > 1:
      t[r, a:a + n + 1] = t[r, (a + n) if r % 3 == 0 else a]
  w = (w / w.sum(-1, keepdims=True)).astype(f)
  if edges and B >= 8:
    w[0] = 0
    k = int(rng.integers(0, P))
    w[1] = 0
    w[1, k] = 1
    t[1, k + 1] = max(t[1, k + 1], np.nextafter(t[1, k], f(np.inf)))
    t[1] = np.maximum.accumulate(t[1])
    k = int(rng.integers(1, P + 1))
    t[2, :k], t[2, k:] = f(lo + 0.3 * (hi - lo)), f(lo + 0.6 * (hi - lo))
    t[3, 0], t[3, -1] = lo, hi
  return torch.tensor(t), torch.tensor(w)


def warp_plan(P, S):
  """Warps per block sample_level_impl picks: 4, halved while the block's shared memory exceeds 200 KiB."""
  per_warp = (13 * P + S + 4) * 4
  warps = 4
  while warps > 1 and per_warp * warps > 200 * 1024:
    warps >>= 1
  return warps
