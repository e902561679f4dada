"""The resampler's fp64 reference (tests/sampling_ref.py) is sound and sensitive.  CPU only.

Soundness: an fp32 emulation of sample_level_kernel -- the 3-way merge by rank, the windowed max by counts, the
lane-strided and butterfly sums, the 32-lane chunked scan, logf / expf moved by their documented error (1 and 2
ulp) in either direction, the index-form inverse CDF -- lands inside every bound.  Sensitivity: each plausible
kernel bug, applied to the emulation, breaks a bound.  Agreement: evaluated in fp32 the reference is the fp32
oracle chain of o_stepfun.
"""
import math

import numpy as np
import pytest
import torch

import sampling_ref as SR
from multinerf_b200 import ops
from oracle import o_stepfun

F = np.float32
EPS2 = F(SR.EPS2)


def _lanes(v):
  """[R, n] -> per-lane sequential sums of the lane-strided terms, then the butterfly of warp_sum (fp32)."""
  R, n = v.shape
  k = -(-n // 32)
  v = np.concatenate([v, np.zeros((R, 32 * k - n), F)], -1).reshape(R, k, 32)
  part = np.zeros((R, 32), F)
  for j in range(k):
    part = part + v[:, j]
  for o in (16, 8, 4, 2, 1):
    part = part + part[:, np.arange(32) ^ o]
  return part[:, 0]


def _move(x, ulps, rng):
  """x moved by `ulps` ulps (a random direction per element when ulps is 'rand:n'); inf / NaN kept."""
  if isinstance(ulps, str):
    n = int(ulps.split(':')[1])
    steps = rng.integers(-n, n + 1, x.shape)
  else:
    steps = np.full(x.shape, ulps)
  y = x.copy()
  for s in range(1, int(np.abs(steps).max(initial=0)) + 1):
    up, dn = steps >= s, steps <= -s
    y = np.where(up, np.nextafter(y, F(np.inf)), np.where(dn, np.nextafter(y, F(-np.inf)), y)).astype(F)
  return np.where(np.isfinite(x), y, x)


def emulate(t, w, S, cfg, mut=(), log_ulps=0, exp_ulps=0, seed=0):
  """sample_level_kernel's arithmetic in numpy fp32 on [R, P+1] / [R, P] inputs; `mut` names deliberate bugs."""
  rng = np.random.default_rng(seed)
  t, w = t.numpy(), w.numpy()
  R, P = w.shape
  rows = np.arange(R)[:, None]
  lo, hi = F(cfg['domain'][0]), F(cfg['domain'][1])
  clip = lambda x: np.minimum(np.maximum(x, lo), hi)
  lt = lambda a, x: (a[:, None, :] < x[:, :, None]).sum(-1)
  le = lambda a, x: (a[:, None, :] <= x[:, :, None]).sum(-1)
  if cfg['use_dilation']:
    d = F(cfg['dilation'])
    p = w / np.maximum(EPS2, t[:, 1:] - t[:, :-1])
    t0, t1 = t[:, :-1] - d, t[:, 1:] + d
    td = np.full((R, 3 * P + 1), np.nan, F)
    td[rows, np.arange(P + 1) + lt(t0, t) + lt(t1, t)] = clip(t)
    td[rows, np.arange(P) + le(t, t0) + lt(t1, t0)] = clip(t0)
    td[rows, np.arange(P) + le(t, t1) + le(t0, t1)] = clip(t1)
    assert not np.isnan(td).any()
    x = td[:, :-1]
    if 'window' in mut:
      ilo, ihi = lt(t1, x), lt(t0, x) - 1
    else:
      ilo, ihi = le(t1, x), le(t0, x) - 1
    i = np.arange(P)
    inwin = (i >= ilo[..., None]) & (i <= ihi[..., None])
    m = np.where(inwin, p[:, None, :], F(0)).max(-1)
    wd = m * (td[:, 1:] - x)
    tot = _lanes(wd[:, 1:-1] if 'renorm_trim' in mut else wd)
    td, wd = td[:, 1:-1], wd[:, 1:-1] / np.maximum(EPS2, tot)[:, None]
  else:
    td, wd = t, w
  nb = wd.shape[1]
  res = dict(tdil=td, wdil=wd)
  anneal = F(1 if 'anneal1' in mut else cfg['anneal'])
  pad = F(0 if 'nopad' in mut else cfg['resample_padding'])
  with np.errstate(divide='ignore', invalid='ignore'):
    lgx = _move(np.log((wd + pad).astype(np.float64)).astype(F), log_ulps, rng)
    lg = np.where(td[:, 1:] > td[:, :-1], anneal * lgx, F(-np.inf))
    mx = np.fmax.reduce(lg, axis=-1, initial=-np.inf).astype(F)
    e = _move(np.exp((lg - mx[:, None]).astype(np.float64)).astype(F), exp_ulps, rng)
    se = _lanes(e)
    q = e / se[:, None]
    ch = -(-nb // 32)
    qc = np.concatenate([q, np.zeros((R, 32 * ch - nb), F)], -1).reshape(R, 32, ch)
    local = np.zeros((R, 32), F)
    for j in range(ch):
      local = local + qc[:, :, j]
    for o in (1, 2, 4, 8, 16):
      n = np.concatenate([np.zeros((R, o), F), local[:, :-o]], -1)
      local = np.where(np.arange(32) >= o, local + n, local)
    run = np.concatenate([np.zeros((R, 1), F), local[:, :-1]], -1)
    cw = np.zeros((R, nb + 1), F)
    for j in range(ch):
      i = np.arange(32) * ch + j
      ok = i < nb - 1
      before = run
      run = np.where(ok, run + qc[:, :, j], run)
      v = before if 'cdf_shift' in mut else run
      v = np.fmin(F(1), v) if 'fminf' in mut else np.where(v > 1, F(1), v)
      cw[:, np.minimum(i, nb - 1)[ok] + 1] = v[:, ok]
    cw[:, 0], cw[:, nb] = 0, 1
  res['cw'] = cw
  u = np.broadcast_to(cfg['u_base'].numpy(), (R, S))
  if cfg['jitter_mode'] and 'nojitter' not in mut:
    j = cfg['jitter'].numpy().reshape(R, -1)
    mj = F(1 if 'nomaxjitter' in mut else cfg['max_jitter'])
    u = u + j * mj
  cnt = lt(cw, u) if 'count_lt' in mut else le(cw, u)
  i0, i1 = np.maximum(cnt - 1, 0), np.minimum(cnt, nb)
  x0, x1 = np.take_along_axis(cw, i0, -1), np.take_along_axis(cw, i1, -1)
  f0, f1 = np.take_along_axis(td, i0, -1), np.take_along_axis(td, i1, -1)
  with np.errstate(divide='ignore', invalid='ignore'):
    off = (u - x0) / (x1 - x0)
  off = np.minimum(np.maximum(np.where(np.isnan(off), F(0), off), F(0)), F(1))
  cen = f0 + off * (f1 - f0)
  mid = (cen[:, 1:] + cen[:, :-1]) * F(0.5)
  first, last = F(2) * cen[:, :1] - mid[:, :1], F(2) * cen[:, -1:] - mid[:, -1:]
  if 'noclamp' not in mut:
    first, last = np.maximum(lo, first), np.minimum(hi, last)
  res['sdist'] = np.concatenate([first, mid, last], -1)
  res['idx'] = cnt - 1
  return {k: torch.tensor(np.ascontiguousarray(v)) for k, v in res.items()}


# P, S, rays, profile, dilation, domain, anneal, padding, jitter mode
PROFILES = {
    'random-dil': (37, 17, 300, 'random', 0.02, (0.0, 1.0), 0.9091, 0.0, 2),
    'positive-anneal0': (16, 24, 200, 'positive', 0.0103, (0.0, 1.0), 0.0, 0.0, 1),
    'zeros-anneal0': (16, 24, 200, 'zeros', 0.0103, (0.0, 1.0), 0.0, 0.0, 1),
    'peaked-pad': (48, 40, 200, 'peaked', 0.0, (0.0, 1.0), 1.0, 0.01, 2),
    'zeros-nodil': (33, 33, 300, 'zeros', 0.0, (0.35, 1.0), 0.5, 0.0, 1),
    'duplicates-eval': (40, 41, 300, 'duplicates', 1e-4, (0.0, 1.0), 1.0, 0.0, 0),
    'chunks-near': (33, 64, 300, 'random', 0.0103, (0.35, 1.0), 0.5, 0.0, 1),
    'uniform-inf': (4, 10, 8, 'uniform', 0.0, (-math.inf, math.inf), 1.0, 0.0, 0),
    'nb3070': (1024, 32, 4, 'random', 0.001, (0.0, 1.0), 1.0, 0.0, 1),
}


def _case(name):
  P, S, B, prof, dil, dom, anneal, pad, jm = PROFILES[name]
  rng = np.random.default_rng(sum(map(ord, name)))
  t, w = SR.step_functions(rng, prof, B, P, domain=dom)
  ub, mj = ops.u_grid(S, jm != 0)
  jit = None
  if jm:
    jit = torch.tensor(rng.uniform(0, 1, (B,) if jm == 1 else (B, S)).astype(F))
    jit[1] = 0        # u = 0 on a ray with a single nonzero bin: the inverse CDF's count of equal knots matters
  cfg = dict(use_dilation=dil > 0, dilation=dil, domain=dom, anneal=anneal, resample_padding=pad, u_base=ub,
             max_jitter=mj, jitter=jit, jitter_mode=jm)
  ref = SR.reference(t, w, S, **cfg)
  return t, w, S, cfg, ref


_CASES = {}


def case(name):
  if name not in _CASES:
    _CASES[name] = _case(name)
  return _CASES[name]


def _worst(ref, em):
  return SR.ratios(ref, em['sdist'], em['idx'], em['cw'], em['tdil'], em['wdil'])


@pytest.mark.parametrize('name', list(PROFILES))
@pytest.mark.parametrize('ulps', [(0, 0), (1, 2), (-1, -2), (1, -2), ('rand:1', 'rand:2')])
def test_emulation_inside_bounds(name, ulps):
  t, w, S, cfg, ref = case(name)
  em = emulate(t, w, S, cfg, log_ulps=ulps[0], exp_ulps=ulps[1])
  worst = _worst(ref, em)
  print(name, ulps, {k: f'{v:.3g}' for k, v in worst.items()})
  assert all(v <= 1 for v in worst.values()), worst


def test_bounds_not_vacuous():
  """At nb = 3070 the CDF bound is below a typical bin's mass, so a one-bin shift breaks it there, and the
  emulation uses a real share of the bounds."""
  t, w, S, cfg, ref = case('nb3070')
  mass = ref.cw[:, 1:] - ref.cw[:, :-1]
  assert float(ref.cw_bound.max()) < float(mass[mass > 0].median())
  assert _worst(ref, emulate(t, w, S, cfg, mut=('cdf_shift',)))['cw'] > 1
  worst = _worst(ref, emulate(t, w, S, cfg, log_ulps=1, exp_ulps=2))
  assert worst['cw'] > 0.01 and worst['wdil'] > 0.01, worst


MUTATIONS = ['cdf_shift', 'count_lt', 'nojitter', 'nomaxjitter', 'anneal1', 'nopad', 'noclamp', 'window',
             'renorm_trim', 'fminf']


@pytest.mark.parametrize('mut', MUTATIONS)
def test_mutation_flagged(mut):
  flagged = []
  for name in PROFILES:
    t, w, S, cfg, ref = case(name)
    worst = _worst(ref, emulate(t, w, S, cfg, mut=(mut,)))
    flagged += [f'{name}:{k}' for k, v in worst.items() if not v <= 1]
  print(mut, 'flagged by', flagged)
  assert flagged, f'mutation {mut} passes every bound'


@pytest.mark.parametrize('P,S,dil,single', [(64, 64, 0.0103125, True), (64, 32, 0.0026220703125, True),
                                            (1, 64, 0.0, True), (128, 128, 0.0, False), (37, 17, 0.02, False)])
def test_fp32_reference_is_oracle_chain(P, S, dil, single):
  """In fp32 the reference is bit for bit the oracle chain: max_dilate_weights, the trim, annealed logits,
  sample_intervals with the oracle's own u."""
  rng = np.random.default_rng(P * 1000 + S)
  B = 257
  t, w = SR.step_functions(rng, 'random', B, P, edges=False)
  use_dil = dil > 0
  anneal, pad = 0.9091, 0.0 if use_dil else 0.01
  jit = torch.tensor(rng.uniform(0, 1, (B, 1 if single else S)).astype(F))
  if use_dil:
    td, wd = o_stepfun.max_dilate_weights(t, w, dil, domain=(0.0, 1.0), renormalize=True)
    td, wd = td[..., 1:-1], wd[..., 1:-1]
  else:
    td, wd = t, w
  logits = torch.where(td[..., 1:] > td[..., :-1], anneal * torch.log(wd + pad), torch.tensor(-math.inf))
  sd_o, idx_o, cw_o = o_stepfun.sample_intervals(jit, td, logits, S, single_jitter=single, domain=(0.0, 1.0),
                                                 return_index=True)
  ub, mj = ops.u_grid(S, True)
  r = SR.reference(t, w, S, u_base=ub, use_dilation=use_dil, dilation=dil, anneal=anneal, resample_padding=pad,
                   jitter=jit, jitter_mode=1 if single else 2, max_jitter=mj, dtype=torch.float32)
  bits = lambda x: x.view(torch.int32)
  for a, b in ((r.tdil, td), (r.wdil, wd), (r.cw, cw_o), (r.sdist, sd_o)):
    assert torch.equal(bits(a), bits(b))
  assert torch.equal(r.idx, idx_o)


def test_nan_cdf_rows_follow_the_oracle():
  """All logits -inf: the oracle's CDF keeps the NaN and every sample collapses onto the first fencepost."""
  t = torch.tensor([[0.1, 0.3, 0.5, 0.9, 1.0]])
  w = torch.zeros(1, 4)
  ub, _ = ops.u_grid(6, False)
  r = SR.reference(t, w, 6, u_base=ub, domain=(0.0, 1.0))
  assert bool(r.nan_row.all()) and torch.isnan(r.cw[0, 1:-1]).all()
  assert torch.equal(r.sdist, torch.full((1, 7), 0.1, dtype=torch.float32).double())
  assert torch.equal(r.idx, torch.zeros(1, 6, dtype=torch.int64))
  assert torch.equal(r.sdist_lo, r.sdist) and torch.equal(r.sdist_hi, r.sdist)


def test_warp_plans():
  assert SR.warp_plan(64, 64) == 4 and SR.warp_plan(1000, 64) == 2 and SR.warp_plan(1024, 12500) == 1
