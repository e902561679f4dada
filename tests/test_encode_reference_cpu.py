"""tests/encode_ref.py is sound and sensitive.  CPU only.

Soundness: `emulate` is a numpy fp32 transcription of the fast kernel's arithmetic -- s_to_t, cast_one in both
shapes, contract_gauss, the lift, exact doubling over the degrees, the three sine forms with rint_small, n_fast read
off the exponent field, and the segmented / grouped traversal that decides which form a lane gets.  The approximate
units (ex2.approx, MUFU.SIN, __fdividef) are the exact function moved by their documented error, once in each
direction.  It lands inside every bound, on every case of tests/test_gpu_encode_fp64.py at a reduced ray count, and
that is also where the floors on the checked share of the GPU cases come from.

Sensitivity: each plausible kernel bug, applied to the emulation, breaks the bound of an element that is not vacuous.
One reduction bug cannot be seen by any honest bound and is asserted to be that small instead: a missing +-t fix-up
after floor / rint moves the reduced argument by one step of fl32(100 pi) - 100 pi (5.9e-6) at |y| >= 100 pi, where
one rounding of y is already 1.9e-5.  (pi/2 added after the reduction instead of before is no bug to find: it only
spares the cosine half the rounding of y + pi/2, which the bound has to allow.)

Agreement: in fp32 the reference is the fp32 oracle chain bit for bit, the running-error evaluation reproduces the
oracle's fp64 values, and plan() equals a transcription of mnrf_encode's host code.
"""
import math

import numpy as np
import pytest
import torch

import encode_ref as ER
from oracle import o_coord, o_render
from test_gpu_encode_fp64 import CASES, case, make_inputs, reach

F = np.float32
I32 = np.int32
SMS = 132
RAYS = 24                   # per case here; the GPU file runs the case's own count
T = F(314.159271240234375)
INV_T = F(1) / T
PI2 = F(1.57079637050628662109375)


def fma(a, b, c):
  return (np.float64(a) * np.float64(b) + np.float64(c)).astype(F)


def rint_small(v):
  return (v + F(12582912.0)) - F(12582912.0)


def host_plan(num_rays, S, K, num_sms):
  """mnrf_encode's host code, statement by statement."""
  G, best = 1, 0.0
  g = 1
  while g <= 16 and g <= S:
    items = g * K
    eff = items / (32.0 * ((items + 31) // 32))
    if eff > best + 1e-9:
      best, G = eff, g
    g += 1
  want_warps = num_sms * 8 * 4
  nseg = min((want_warps + num_rays - 1) // num_rays, max(1, S // (2 * G)))
  nseg = max(1, nseg)
  seg_len = (S + nseg - 1) // nseg
  seg_len = (seg_len + G - 1) // G * G
  nseg = (S + seg_len - 1) // seg_len
  return G, nseg, seg_len


def _fwd(fn, x):
  return {None: lambda: x, 'reciprocal': lambda: F(1) / x, 'log': lambda: np.log(x), 'exp': lambda: np.exp(x),
          'sqrt': lambda: np.sqrt(x), 'square': lambda: x * x,
          'piecewise': lambda: np.where(x < 1, F(0.5) * x, F(1) - F(0.5) / x)}[fn]()


def _inv(fn, x):
  if fn == 'piecewise':
    with np.errstate(divide='ignore'):
      return np.where(x < F(0.5), F(2) * x, F(0.5) / (F(1) - x))
  return _fwd({'log': 'exp', 'exp': 'log', 'sqrt': 'square', 'square': 'sqrt'}.get(fn, fn), x)


def _cast(shape, t0, t1, o, d, radius, mut):
  if shape == 'cone':
    mu, hw = (t0 + t1) / F(2), (t1 - t0) / F(2)
    hw2, mu2 = hw * hw, mu * mu
    hw4 = hw2 * hw2
    c415 = F(4) / F(14 if mut == 'c415' else 15)
    denom = np.maximum(F(ER.EPS), F(3) * mu2 + hw2)
    t_mean = mu + (F(2) * mu * hw2) / denom
    t_var = hw2 / F(3) - c415 * hw4 * (F(12) * mu2 - hw2) / (denom * denom)
    r_var = mu2 / F(4) + (F(5) / F(12)) * hw2
    if mut != 'no_hw4':
      r_var = r_var - c415 * hw4 / denom
    r_var = r_var * (radius * radius)
  else:
    t_mean = (t0 + t1) / F(2)
    r_var = np.broadcast_to((radius * radius) / F(4), t0.shape)
    dt = t1 - t0
    t_var = (dt * dt) / F(12)
  dmag = np.maximum(F(1e-10), d[0] * d[0] + d[1] * d[1] + d[2] * d[2])
  mean = [d[i] * t_mean + o[i] for i in range(3)]
  cov = [[t_var * (d[i] * d[j]) + r_var * (F(i == j) - d[i] * (d[j] if mut == 'null_no_dmag' else d[j] / dmag))
          for j in range(3)] for i in range(3)]
  return mean, cov


def _contract(x, cov, mut):
  m = np.maximum(F(ER.EPS), x[0] * x[0] + x[1] * x[1] + x[2] * x[2])
  inside = m <= 1
  m = np.where(inside, F(2), m)
  r = np.sqrt(m)
  scale = (F(2) * r - F(1)) / m
  s = F(2) / r - F(1) / m
  c = F(2) / (m * m) - F(2) / (m * r)
  J = [[(s if i == j else F(0)) + c * x[i] * x[j] for j in range(3)] for i in range(3)]
  T_ = [[J[i][0] * cov[0][j] + J[i][1] * cov[1][j] + J[i][2] * cov[2][j] for j in range(3)] for i in range(3)]
  out = T_ if mut == 'J_one_side' else [[T_[i][0] * J[j][0] + T_[i][1] * J[j][1] + T_[i][2] * J[j][2]
                                         for j in range(3)] for i in range(3)]
  return ([np.where(inside, x[i], scale * x[i]) for i in range(3)],
          [[np.where(inside, cov[i][j], out[i][j]) for j in range(3)] for i in range(3)])


def _reduce(x, form, mut):
  """The argument sin_below_100pi receives: x itself (form 1), safe_sin_nobranch's (2), safe_sin_fast's (3)."""
  if form == 1:
    return x
  small = np.zeros(x.shape, bool) if mut == 'reduce_small' else np.abs(x) < T
  if form == 2:
    r = fma(-rint_small(x * INV_T), T, x)
    if mut != 'no_fixup':
      r = np.where(r < 0, r + T, r)
  else:
    r = fma(-np.floor(x * INV_T), T, x)
    if mut != 'no_fixup':
      r = np.where(r < 0, r + T, np.where(r >= T, r - T, r))
  return np.where(small, x, r)


def _sin_below(x, dirn):
  q = rint_small(x * F(0.15915494309189535))
  r = fma(-q, F(6.2831854820251465), x)
  r = fma(q, F(1.7484555e-7), r)
  return (np.sin(np.float64(r)) + dirn * 2.0 ** -21.41).astype(F)


def emulate(pos, kw, num_sms=SMS, dirn=1, mut=None):
  """(tdist [B, S+1], feat_f32 [B, S, 2KL], passes per tier) as encode_fast_kernel computes them."""
  sdist, o, d, radii, near, far, basis = [t.numpy() for t in pos]
  B, S = sdist.shape[0], sdist.shape[1] - 1
  K, L = basis.shape[0], kw['max_deg'] - kw['min_deg']
  KL = K * L
  fn = kw['raydist_fn']
  with np.errstate(all='ignore'):
    s_near, s_far = _fwd(fn, near)[:, None], _fwd(fn, far)[:, None]
    tdist = _inv(fn, sdist * s_far + (F(1) - sdist) * s_near).astype(F)
    mean, cov = _cast(kw['ray_shape'], tdist[:, :-1], tdist[:, 1:], [o[:, i:i + 1] for i in range(3)],
                      [d[:, i:i + 1] for i in range(3)], radii[:, None], mut)
    if kw['warp_contract']:
      mean, cov = _contract(mean, cov, mut)
    b = [basis[:, i] for i in range(3)]
    lm = mean[0][..., None] * b[0] + mean[1][..., None] * b[1] + mean[2][..., None] * b[2]
    cc = [cov[i][0][..., None] * b[0] + cov[i][1][..., None] * b[1] + cov[i][2][..., None] * b[2] for i in range(3)]
    lv = np.zeros_like(lm) if kw['disable_integration'] else b[0] * cc[0] + b[1] * cc[1] + b[2] * cc[2]
    G, nseg, seg_len = host_plan(B, S, K, num_sms)
    sc0 = F(2.0 ** kw['min_deg'])
    sc_top = F(2.0 ** (L + 1))
    feat = np.zeros((B, S + 1, 2 * KL), F)          # one spare row for the misplaced-row mutation
    lane = np.arange(32)
    count = {1: 0, 2: 0, 3: 0}
    rows = np.arange(B)[:, None]
    for seg in range(nseg):
      s_begin, s_end = seg * seg_len, min(S, (seg + 1) * seg_len)
      if mut == 'seg_late' and seg > 0:
        s_begin += 1
      for s0 in range(s_begin, s_end, G):
        g = min(G, s_end - s0)
        for j0 in range(0, g * K, 32):
          j = np.minimum(j0 + lane, g * K - 1)
          si, k = s0 + j // K, j % K
          y = lm[:, si, k] * sc0
          v = lv[:, si, k] * (sc0 if mut == 'sc_var' else sc0 * sc0)
          ymax = np.abs(y).max(-1)
          q = (F(311) / np.float64(ymax) * (1 + dirn * 2.0 ** -22)).astype(F)          # __fdividef: 2 ulp
          n_fast = np.clip(((q.view(I32) >> 23) & 0xff) - 126, 0, L)
          rest = np.where(ymax * sc_top < F(1e9), 2, 3)
          count[1] += int((n_fast > 0).sum())
          for t in (2, 3):
            count[t] += int(((n_fast < L) & (rest == t)).sum())
          so = si + (mut == 'row_plus1')
          for l in range(L):
            form = np.where(l < n_fast, 1, rest)[:, None]
            e = (np.exp2(np.float64(v * F(-0.72134751081466674805))) * (1 + dirn * 2.0 ** -22)).astype(F)
            e = np.where(e < F(2.0 ** -126), F(0), e)                                      # .ftz
            yc = y + PI2
            sn = [_sin_below(_reduce(y, f, mut), dirn) for f in (1, 2, 3)]
            cs = [_sin_below(_reduce(yc, f, mut), dirn) for f in (1, 2, 3)]
            fs = e * np.where(form == 1, sn[0], np.where(form == 2, sn[1], sn[2]))
            fc = e * np.where(form == 1, cs[0], np.where(form == 2, cs[1], cs[2]))
            if mut == 'swap_rows':
              fs, fc = fc, fs
            feat[rows, so, l * K + k] = fs
            feat[rows, so, KL + l * K + k] = fc
            y = y * F(2)
            v = v * F(2 if mut == 'v2' else 4)
  return torch.tensor(tdist), torch.tensor(feat[:, :S]), count


def check(name, dirn=1, mut=None):
  """Reference of a case on the emulation's tdist; (reference, got, [B, S, 2KL] mask of broken bounds)."""
  pos, kw = make_inputs(name, SMS, rays=RAYS)
  tdist, got, count = emulate(pos, kw, dirn=dirn, mut=mut)
  ref = ER.reference(*pos, **kw, tdist=tdist)
  broken = ((got.double() - ref.feat).abs() > ref.bound) & ~ref.vacuous
  return ref, tdist, got, broken, count


@pytest.mark.parametrize('name', list(CASES))
def test_emulation_within_bounds(name):
  c = case(name)
  K, L = c['K'], c['max_deg'] - c['min_deg']
  deg = ER.degree_of(K, L)
  for dirn in (1, -1):
    ref, tdist, got, broken, count = check(name, dirn)
    rt = (tdist.double() - ref.tdist).abs() / ref.tdist_bound
    assert float(rt.max()) <= 1, (name, 'tdist', float(rt.max()))
    ratio = torch.where(ref.vacuous, torch.zeros_like(ref.bound), (got.double() - ref.feat).abs() / ref.bound)
    assert not broken.any(), (name, dirn, float(ratio.max()), np.unravel_index(int(ratio.argmax()), ratio.shape))
    assert ref.chain_gap < 1e-3, (name, 'the running-error evaluation left the oracle', ref.chain_gap)
  checked = 1 - float(ref.vacuous.double().mean())
  print(f'\n{name}: tdist {float(rt.max()):.2f} | worst err/bound per degree ' +
        ' '.join(f'{float(ratio[..., deg == l].max()):.2f}' for l in range(L)) + ' | vacuous per degree ' +
        ' '.join(f'{float(ref.vacuous[..., deg == l].double().mean()):.2f}' for l in range(L)) +
        f' | checked {checked:.3f} (floor {c["floor"]}) | passes per tier {count}')
  assert checked >= min(1.0, c['floor'] + 0.02), (name, checked)
  # the tiers read off the fp64 means are the ones the emulation took, and the case reaches what it names
  B = ref.lm.shape[0]
  p = ER.plan(B, c['S'], K, SMS)
  tr = ER.tiers(ref, p, c['min_deg'], c['max_deg'])
  slack = int(tr.unsure.sum())
  for t in (1, 2, 3):
    assert abs(tr.count(t) - count[t]) <= slack, (name, t, tr.count(t), count[t])
  if c['rays'] is not None and not {'nseg>1', 'nseg1', 'short-last'} & set(c['reach']):
    reach(name, p, tr, c['S'])
  else:
    reach(name, ER.plan(c['rays'] or 32 * SMS + 37, c['S'], K, SMS), tr, c['S'])


# mutation: the cases tried, in order
MUTATIONS = {
    'c415': ('S1', 'far-contracted'), 'no_hw4': ('S1', 'far-contracted'), 'null_no_dmag': ('K9', '360'),
    'J_one_side': ('360', 'piecewise'), 'sc_var': ('min-deg-2',), 'v2': ('K9', '360'),
    'reduce_small': ('blender', 'K9'), 'swap_rows': ('S1', 'K9'), 'row_plus1': ('S5-K9', 'K9'),
    'seg_late': ('S33-K21', 'S50-K9'),
}


@pytest.mark.parametrize('mut', list(MUTATIONS))
def test_mutation_is_caught(mut):
  for name in MUTATIONS[mut]:
    ref, _, got, broken, _ = check(name, mut=mut)
    if broken.any():
      r = torch.where(broken, (got.double() - ref.feat).abs() / ref.bound, torch.zeros_like(ref.bound))
      i = tuple(int(v) for v in np.unravel_index(int(r.argmax()), r.shape))
      print(f'\n{mut}: caught by {name} on {int(broken.sum())} elements, worst at [ray, sample, column] {i}: '
            f'{float(r[i]):.1f} bounds')
      return
  raise AssertionError(f'{mut}: no case notices')


def test_missing_fixup_is_jump_level():
  """What no bound can see: it moves the reduced argument by steps of fl32(100 pi) - 100 pi only."""
  pos, kw = make_inputs('huge-uncontracted', SMS, rays=RAYS)
  _, a, _ = emulate(pos, kw)
  _, b, _ = emulate(pos, kw, mut='no_fixup')
  assert float((a - b).abs().max()) <= 2.2 * ER.JUMP + 4 * ER.C_SIN


def test_fp32_is_the_oracle_chain():
  for name in ('360', 'K9', 'llff', 'piecewise'):
    pos, kw = make_inputs(name, SMS, rays=8)
    sd, o, d, rad, near, far, basis = pos
    _, s_to_t = o_coord.construct_ray_warps(kw['raydist_fn'], near[:, None], far[:, None])
    td = s_to_t(sd)
    ref = ER.reference(*pos, **kw, tdist=td, dtype=torch.float32)
    assert torch.equal(ref.tdist, td)
    means, covs = o_render.cast_rays(td, o, d, rad[:, None], kw['ray_shape'], diag=False)
    if kw['warp_contract']:
      means, covs = o_coord.track_linearize_contract(means, covs)
    lm, lv = o_coord.lift_and_diagonalize(means, covs, basis.T.contiguous())
    assert torch.equal(ref.feat, o_coord.integrated_pos_enc(lm, lv, kw['min_deg'], kw['max_deg']))
    # and the fp64 features are the fp32 oracle's to fp32 accuracy where the bound is small
    r64 = ER.reference(*pos, **kw, tdist=td)
    ok = r64.bound < 1e-4
    assert ok.any() and float((ref.feat.double() - r64.feat).abs()[ok].max()) < 3e-4


def test_safe_sin_reduces_by_the_fp32_constant():
  y = torch.tensor([-1.0, 1.0, 314.0, -314.0, 314.2, -314.2, 1e4, -1e4], dtype=torch.float64)
  want = [math.sin(v) if abs(v) < ER.T32 else math.sin(v - math.floor(v / ER.T32) * ER.T32) for v in y.tolist()]
  assert torch.allclose(ER.safe_sin64(y), torch.tensor(want, dtype=torch.float64), atol=1e-12, rtol=0)
  assert abs(ER.JUMP - 5.88e-6) < 1e-8 and 5e-7 < ER.C_SIN < 6e-7


@pytest.mark.parametrize('rays,S,K,sms', [
    (96, 32, 21, 132), (4261, 32, 21, 132), (4224, 64, 21, 132), (4223, 64, 21, 132), (2048, 64, 21, 132),
    (96, 32, 9, 132), (96, 5, 9, 132), (96, 1, 9, 132), (96, 33, 21, 132), (96, 50, 9, 132), (40, 128, 9, 132),
    (24, 256, 21, 132), (96, 16, 3, 132), (96, 16, 32, 132), (96, 16, 33, 132), (1, 1, 1, 1), (7, 13, 5, 108),
    (100000, 48, 21, 132), (96, 2, 21, 132), (96, 6, 21, 132), (96, 31, 16, 114)])
def test_plan_is_the_hosts(rays, S, K, sms):
  p = ER.plan(rays, S, K, sms)
  assert (p.G, p.nseg, p.seg_len) == host_plan(rays, S, K, sms)
  ps = ER.passes(S, K, p)
  seen = {(int(s), int(k)) for si, ki in ps for s, k in zip(si, ki)}
  assert seen == {(s, k) for s in range(S) for k in range(K)}, 'the passes do not cover every (sample, direction) once'


def test_pos_enc_reference():
  v = torch.tensor(np.random.default_rng(0).normal(size=(5, 3)), dtype=torch.float32)
  enc, bound = ER.pos_enc_reference(v, 4)
  got = o_coord.pos_enc(v, 0, 4).to(torch.bfloat16).double()
  assert enc.shape == (5, 27) and float(((got - enc).abs() / bound).max()) <= 1
  assert float(bound[:, 3:].max()) < 2.0 ** -8 + 1e-4
