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


def _sincos(x, dirn):
  """safe_sincos_fast: the floor reduction by fl32(100 pi), Cody-Waite by 2 pi, MUFU.SIN / MUFU.COS moved by 2^-21.41."""
  r = _reduce(x, 3, None)
  q = rint_small(r * F(0.15915494309189535))
  r = fma(q, F(1.7484555e-7), fma(-q, F(6.2831854820251465), r))
  r64 = np.float64(r)
  return (np.sin(r64) + dirn * 2.0 ** -21.41).astype(F), (np.cos(r64) + dirn * 2.0 ** -21.41).astype(F)


def emulate_tangent_rows(x, cov, basis, kw, dirn=1, mut=None):
  """gauss_tangent_rows' tangent rows of the pre-warp fp32 Gaussians x [3] / cov [3][3] (arrays [..]): contract_terms,
  store_gauss, the lift and d lift, __expf moved by its documented error, safe_sincos_fast, the bf16 store.
  Returns [3, .., 2KL] float32 (bf16 values)."""
  K, L = basis.shape[0], kw['max_deg'] - kw['min_deg']
  contract, no_int = kw['warp_contract'], kw['disable_integration']
  with np.errstate(all='ignore'):
    mean, covw = _contract(x, cov, None) if contract else (x, cov)
    b = [basis[:, i] for i in range(3)]
    lm = mean[0][..., None] * b[0] + mean[1][..., None] * b[1] + mean[2][..., None] * b[2]
    cc = [covw[i][0][..., None] * b[0] + covw[i][1][..., None] * b[1] + covw[i][2][..., None] * b[2] for i in range(3)]
    lv = np.zeros_like(lm) if no_int else b[0] * cc[0] + b[1] * cc[1] + b[2] * cc[2]
    if contract:
      m = np.maximum(F(ER.EPS), x[0] * x[0] + x[1] * x[1] + x[2] * x[2])
      inside = m <= 1
      mo = np.where(inside, F(2), m)
      r = np.sqrt(mo)
      ir = F(1) / r
      xh = [np.where(inside, F(0), x[i] * ir)[..., None] for i in range(3)]
      sj = np.where(inside, F(1), F(2) / r - F(1) / mo)[..., None]
      qj = np.where(inside, F(1), F(1) / mo)[..., None]
      q_r = F(-2) / (mo * r)
      s_r = np.where(inside, F(0), ((r + F(1)) if mut == 's_r_r_plus_1' else (r - F(1))) * q_r)[..., None]
      q_r = np.where(inside, F(0), q_r)[..., None]
      cv = [cov[0][0], cov[0][1], cov[0][2], cov[1][1], cov[1][2], cov[2][2]]
      cv = [c[..., None] for c in cv]
      beta = xh[0] * b[0] + xh[1] * b[1] + xh[2] * b[2]
      bt = [b[i] - beta * xh[i] for i in range(3)]
      u = [(qj if mut == 'u_q_for_s' else sj) * bt[i] + (qj * beta) * xh[i] for i in range(3)]
      v = [cv[0] * u[0] + cv[1] * u[1] + cv[2] * u[2], cv[1] * u[0] + cv[3] * u[1] + cv[4] * u[2],
           cv[2] * u[0] + cv[4] * u[1] + cv[5] * u[2]]
      gamma = xh[0] * v[0] + xh[1] * v[1] + xh[2] * v[2]
      vt = [v[i] - gamma * xh[i] for i in range(3)]
      btv = bt[0] * v[0] + bt[1] * v[1] + bt[2] * v[2]
      radial = s_r * btv + (-q_r if mut == 'q_r_sign' else q_r) * (beta * gamma)
      two = F(1) if mut == 'dlv_no2' else F(2)
      dlv = [np.zeros_like(lm) if (no_int or mut == 'no_dlv') else
             two * (xh[a] * radial + s_r * (beta * vt[a] + gamma * bt[a])) for a in range(3)]
    out = np.zeros((3,) + lm.shape[:-1] + (2 * K * L,), F)
    for l in range(L):
      sc = F(2.0 ** (kw['min_deg'] + l))
      y, vv = lm * sc, lv * (sc * sc)
      ex = np.float64(F(-0.5) * vv)
      e = (np.exp(ex) * (1 + dirn * (1.5 + 1.173 * np.abs(ex)) * 2.0 ** -23)).astype(F)
      e = np.where(e < F(2.0 ** -126), F(0), e)
      s0, c0 = _sincos(y, dirn)
      s1, c1 = _sincos(y + PI2, dirn)
      fs, fc = e * s0, e * s1
      for a in range(3):
        if contract:
          esc = sc if mut == 'esc_no_e' else e * sc
          hsc2 = F(0.5) * (sc if mut == 'hsc2_sc' else sc * sc)
          dm, dvar = u[a] * esc, dlv[a] * hsc2
          ts, tc = c0 * dm - fs * dvar, c1 * dm - fc * dvar
        else:
          bk = (basis.reshape(-1)[a * K:(a + 1) * K] if mut == 'basis_dir_k' else basis[:, a]) * sc * e
          ts, tc = c0 * bk, c1 * bk
        out[a, ..., l * K:(l + 1) * K] = ts
        out[a, ..., K * L + l * K:K * L + (l + 1) * K] = tc
  return torch.tensor(out).to(torch.bfloat16).float()


def _pre_warp(pos, kw):
  """tdist and the pre-warp Gaussians [B, S] of the general (tangent) encoder, in fp32."""
  sdist, o, d, radii, near, far, basis = [t.numpy() for t in pos]
  fn = kw['raydist_fn']
  with np.errstate(all='ignore'):
    s_near, s_far = _fwd(fn, near)[:, None], _fwd(fn, far)[:, None]
    tdist = _inv(fn, sdist * s_far + (F(1) - sdist) * s_near).astype(F)
    x, cov = _cast(kw['ray_shape'], tdist[:, :-1], tdist[:, 1:], [o[:, i:i + 1] for i in range(3)],
                   [d[:, i:i + 1] for i in range(3)], radii[:, None], None)
  return tdist, x, cov


def check_tangent(name, dirn=1, mut=None):
  """(reference, emulated tangent rows [3, B, S, 2KL], mask of broken bounds) of a case."""
  pos, kw = make_inputs(name, SMS, rays=RAYS)
  tdist, x, cov = _pre_warp(pos, kw)
  got = emulate_tangent_rows(x, cov, pos[6].numpy(), kw, dirn, mut)
  if mut == 'row_dir_seg':              # stream dir at row dir * S + m of the [3 B S] rows instead of dir * B S + m
    B, S = got.shape[1], got.shape[2]
    rows = torch.zeros_like(got).view(3 * B * S, -1)
    for a in range(3):
      rows[a * S:a * S + B * S] = got[a].reshape(B * S, -1)
    got = rows.view(got.shape)
  ref = ER.reference(*pos, **kw, tdist=torch.tensor(tdist), tangent=True)
  broken = ((got.double() - ref.tangent).abs() > ref.tangent_bound_bf16) & ~ref.tangent_vacuous
  return ref, got, broken


TANGENT_CASES = [n for n in CASES if case(n)['tangent']]


@pytest.mark.parametrize('name', TANGENT_CASES)
def test_tangent_emulation_within_bounds(name):
  c = case(name)
  K, L = c['K'], c['max_deg'] - c['min_deg']
  deg = ER.degree_of(K, L)
  for dirn in (1, -1):
    ref, got, broken = check_tangent(name, dirn)
    ratio = torch.where(ref.tangent_vacuous, torch.zeros_like(ref.tangent),
                        (got.double() - ref.tangent).abs() / ref.tangent_bound_bf16)
    assert not broken.any(), (name, dirn, float(ratio.max()), np.unravel_index(int(ratio.argmax()), ratio.shape))
  checked = 1 - float(ref.tangent_vacuous.double().mean())
  print(f'\n{name} tangent: worst err/bound per stream ' +
        ' '.join(f'{float(ratio[a].max()):.2f}' for a in range(3)) + ' | per degree ' +
        ' '.join(f'{float(ratio[..., deg == l].max()):.2f}' for l in range(L)) +
        f' | checked {checked:.3f} (floor {c.get("tfloor", c["floor"])})')
  assert checked >= min(1.0, c.get('tfloor', c['floor']) + 0.02), (name, checked)


@pytest.mark.parametrize('warp_contract,disable_integration,var', [
    (False, False, 1e-4), (True, False, 1e-4), (True, True, 1e-4), (True, False, 0.0), (False, False, 0.0),
    (True, False, 3e-2)])
def test_points_tangent_emulation_within_bounds(warp_contract, disable_integration, var):
  """The point form (mnrf_encode_points_tangent: mean = point, cov = var I) on the point set of
  test_gpu_mesh_color.test_encode_points_tangent_features_vs_fp64."""
  from multinerf_b200 import geopoly
  basis = np.ascontiguousarray(geopoly.generate_basis('octahedron', 2), dtype=F)
  rng = np.random.default_rng(3)
  pts = np.concatenate([rng.uniform(-0.57, 0.57, (400, 3)), rng.uniform(-3, 3, (400, 3)),
                        rng.normal(size=(201, 3)) * 50]).astype(F)
  kw = dict(min_deg=0, max_deg=12, warp_contract=warp_contract, disable_integration=disable_integration)
  ref = ER.points_reference(pts, var, basis, **kw)
  assert ref.chain_gap < 1e-3
  x = [pts[:, i] for i in range(3)]
  cov = [[np.full(len(pts), F(var) if i == j else F(0), F) for j in range(3)] for i in range(3)]
  for dirn in (1, -1):
    got = emulate_tangent_rows(x, cov, basis, kw, dirn)
    ratio = torch.where(ref.tangent_vacuous, torch.zeros_like(ref.tangent),
                        (got.double() - ref.tangent).abs() / ref.tangent_bound_bf16)
    assert float(ratio.max()) <= 1, (dirn, float(ratio.max()), np.unravel_index(int(ratio.argmax()), ratio.shape))
  assert float(ref.tangent_vacuous.double().mean()) < 0.4
  print(f'\npoints contract {warp_contract} no_int {disable_integration} var {var}: worst err/bound '
        f'{float(ratio.max()):.2f} | checked {1 - float(ref.tangent_vacuous.double().mean()):.3f}')


def _autograd_tangent(pos, kw, tdist):
  """d integrated_pos_enc / d mean of the oracle chain, by forward-mode autograd in fp64: [3, B, S, 2KL]."""
  from torch.func import jvp
  sd, o, d, rad, near, far, basis = [t.double() for t in pos]
  means, covs = o_render.cast_rays(tdist.double(), o, d, rad[:, None], kw['ray_shape'], diag=False)

  def enc(m):
    mm, cc = o_coord.track_linearize_contract(m, covs) if kw['warp_contract'] else (m, covs)
    lm, lv = o_coord.lift_and_diagonalize(mm, cc, basis.T.contiguous())
    return o_coord.integrated_pos_enc(lm, torch.zeros_like(lv) if kw['disable_integration'] else lv,
                                      kw['min_deg'], kw['max_deg'])
  return torch.stack([jvp(enc, (means,), (torch.eye(3, dtype=torch.float64)[a].expand_as(means),))[1]
                      for a in range(3)])


@pytest.mark.parametrize('name', TANGENT_CASES)
def test_tangent_value_is_the_oracle_derivative(name, monkeypatch):
  """The reference's fp64 tangent rows are autograd's derivative of the oracle chain (safe_sin reducing by the fp32
  constant, as the reference does), to fp64 rounding, away from |x| = 1."""
  from oracle import o_math
  monkeypatch.setattr(o_math, '_T_SAFE', ER.T32)
  pos, kw = make_inputs(name, SMS, rays=8)
  tdist, _, _ = _pre_warp(pos, kw)
  ref = ER.reference(*pos, **kw, tdist=torch.tensor(tdist), tangent=True)
  ag = _autograd_tangent(pos, kw, torch.tensor(tdist))
  scale = ag.abs().amax(-1, keepdim=True).clamp_min(1e-300)
  far = ~ref.tangent_vacuous.all(-1, keepdim=True).expand_as(ag)       # samples off the |x| = 1 shell
  rel = float(((ref.tangent - ag).abs() / scale)[far].max())
  assert rel < 1e-12, (name, rel)


def check(name, dirn=1, mut=None, tangent=False):
  """Reference of a case on the emulation's tdist; (reference, got, [B, S, 2KL] mask of broken bounds)."""
  pos, kw = make_inputs(name, SMS, rays=RAYS)
  tdist, got, count = emulate(pos, kw, dirn=dirn, mut=mut)
  ref = ER.reference(*pos, **kw, tdist=tdist, tangent=tangent)
  broken = ((got.double() - ref.feat).abs() > ref.bound) & ~ref.vacuous
  return ref, tdist, got, broken, count


@pytest.mark.parametrize('name', list(CASES))
def test_emulation_within_bounds(name):
  c = case(name)
  K, L = c['K'], c['max_deg'] - c['min_deg']
  deg = ER.degree_of(K, L)
  for dirn in (1, -1):
    ref, tdist, got, broken, count = check(name, dirn, tangent=c['tangent'])
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
    reach(name, p, tr, c['S'], ref)
  else:
    reach(name, ER.plan(c['rays'] or 32 * SMS + 37, c['S'], K, SMS), tr, c['S'])


# mutation: the cases tried, in order
MUTATIONS = {
    'c415': ('S1', 'far-contracted'), 'no_hw4': ('S1', 'far-contracted'), 'null_no_dmag': ('K9', '360'),
    'J_one_side': ('360', 'piecewise'), 'sc_var': ('min-deg-2',), 'v2': ('K9', '360'),
    'reduce_small': ('blender', 'K9'), 'swap_rows': ('S1', 'K9'), 'row_plus1': ('S5-K9', 'K9'),
    'seg_late': ('S33-K21', 'S50-K9'),
}


# tangent-row mutation: the cases tried, in order
TANGENT_MUTATIONS = {
    'no_dlv': ('360', 'far-contracted'), 'dlv_no2': ('360', 'far-contracted'), 'q_r_sign': ('far-contracted', '360'),
    's_r_r_plus_1': ('far-contracted', '360'), 'u_q_for_s': ('far-contracted', '360'),
    'hsc2_sc': ('360', 'piecewise'), 'esc_no_e': ('360', 'piecewise'), 'basis_dir_k': ('K9', 'K32'),
    'row_dir_seg': ('S5-K9', 'K9'),
}


@pytest.mark.parametrize('mut', list(TANGENT_MUTATIONS))
def test_tangent_mutation_is_caught(mut):
  for name in TANGENT_MUTATIONS[mut]:
    ref, got, broken = check_tangent(name, mut=mut)
    if broken.any():
      r = torch.where(broken, (got.double() - ref.tangent).abs() / ref.tangent_bound_bf16, torch.zeros_like(got.double()))
      i = tuple(int(v) for v in np.unravel_index(int(r.argmax()), r.shape))
      print(f'\n{mut}: caught by {name} on {int(broken.sum())} elements, worst at [stream, ray, sample, column] {i}: '
            f'{float(r[i]):.1f} bounds')
      return
  raise AssertionError(f'{mut}: no case notices')


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
