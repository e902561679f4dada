"""tests/camera_ref.py is sound, sensitive and agrees with the oracle and the reference's own outputs.  CPU only.

Soundness: `emulate` is a numpy fp32 transcription of camera.cuh's camera_dir and undistort and camera.cu's to_ndc,
dist3 and kernel body, in their operation order and without FMA.  sinf and cosf are the exact function moved by
their documented 2 ulp, once in each direction.  It lands inside every bound on every case of
tests/test_gpu_camera_fp64.py at a reduced ray count.

Sensitivity: each plausible kernel bug, applied to the emulation, breaks the bound of a ray that is not vacuous, on
the case named beside it.

Agreement: in float64 and with the exact constants (pi, sqrt(12)) the reference's values are oracle/o_camera.py's on
every case, and, fed the reference's own fp64 golden inputs, the golden `*_f64_*` outputs of tests/golden/camera.npz.
"""
import math
import os
import types

import numpy as np
import pytest
import torch

import camera_ref as CR
from oracle import o_camera
from test_gpu_camera_fp64 import CASES, case, centre, make_inputs, monotone

F = np.float32
RAYS = 600                  # per case here; the GPU file runs the case's full count
PI32 = F(CR.PI32)
SQRT12 = F(3.4641016151377544)
HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, 'golden', 'camera.npz'))


def _moved(fn, x, dirn):
  """fn(x) in fp32, pushed by up to 2 ulp in direction dirn and rounded toward the exact value: within sinf's and
  cosf's documented error."""
  exact = fn(x.astype(np.float64))
  r = exact.astype(F)
  if dirn:
    t = exact + dirn * 2 * np.spacing(np.abs(r)).astype(np.float64)
    r = t.astype(F)
    over = np.abs(r.astype(np.float64) - exact) > np.abs(t - exact)
    r = np.where(over, np.nextafter(r, exact.astype(F)), r)
  return r


def _mat3(m, ld, v):
  return [m(r * ld) * v[0] + m(r * ld + 1) * v[1] + m(r * ld + 2) * v[2] for r in range(3)]


def _undistort(d, xd, yd, mut):
  k1, k2, k3, k4, p1, p2 = (F(d[k]) for k in CR.KEYS)
  x, y = xd, yd
  for _ in range(d['undistort_iters']):
    r = x * x + y * y
    dd = F(1.0) + r * (k1 + r * (k2 + r * (k3 + r * k4)))
    fx = dd * x + F(2) * p1 * x * y + p2 * (r + F(2) * x * x) - xd
    fy = dd * y + F(2) * p2 * x * y + p1 * (r + F(2) * y * y) - yd
    d_r = k1 + r * (F(2.0) * k2 + r * (F(3.0) * k3 + r * F(4.0) * k4))
    d_x = F(2.0) * x * d_r
    d_y = F(2.0) * y * d_r
    fx_x = dd + d_x * x + F(2.0) * p1 * y + F(6.0) * p2 * x
    if mut == 'jacobian_p2':
      fx_y = d_y * x + F(2.0) * p2 * x + F(2.0) * p2 * y
    else:
      fx_y = d_y * x + F(2.0) * p1 * x + F(2.0) * p2 * y
    fy_x = d_x * y + F(2.0) * p2 * y + F(2.0) * p1 * x
    fy_y = dd + d_y * y + F(2.0) * p2 * x + F(6.0) * p1 * y
    den = fy_x * fx_y - fx_x * fy_y
    xn = fx * fy_y - fy * fx_y
    yn = fy * fx_x - fx * fy_x
    ok = np.abs(den) > F(d['undistort_eps'])
    sx, sy = np.where(ok, xn / den, F(0)), np.where(ok, yn / den, F(0))
    if mut == 'newton_sign':
      sx, sy = -sx, -sy
    x, y = x + sx, y + sy
  return x, y


def _camera_dir(d, p, px, py, half, dirn, mut):
  v = _mat3(p, 3, [px + half, py + half, np.ones_like(px)])
  if d['has_distortion']:
    x, y = _undistort(d, v[0], v[1], mut)
    v = [x, y, np.ones_like(px)]
  if d['camtype'] == 1:
    theta = np.sqrt(v[0] * v[0] + v[1] * v[1])
    if mut != 'no_pi_clamp':
      theta = np.minimum(PI32, theta)
    sn = _moved(np.sin, theta, dirn)
    q = sn / np.where(theta > 0, theta, F(1))
    s = sn / theta if mut == 'sinc_0_over_0' else np.where(theta > 0, q, F(1))
    v = [v[0] * s, v[1] * s, _moved(np.cos, theta, dirn)]
  return [v[0], v[1] if mut == 'no_flip_y' else -v[1], -v[2]]


def _to_ndc(d, o, dr, mut):
  t = -(F(d['ndc_near']) + o[2]) / dr[2]
  o = [o[i] + t * dr[i] for i in range(3)]
  xm = F(1.0) / F(d['ndc_p02'])
  ym = F(1.0) / F(d['ndc_p02' if mut == 'ndc_p02_both' else 'ndc_p12'])
  o_ndc = [xm * o[0] / o[2], ym * o[1] / o[2], np.full_like(o[0], -1)]
  inf = [xm * dr[0] / dr[2], ym * dr[1] / dr[2], np.ones_like(o[0])]
  return o_ndc, [inf[i] - o_ndc[i] for i in range(3)]


def _dist3(a, b):
  x, y, z = a[0] - b[0], a[1] - b[1], a[2] - b[2]
  return np.sqrt(x * x + y * y + z * z)


def emulate(px, py, idx, p2c, c2w, d, dirn=0, mut=None):
  """{field: [B, n] fp32} as pixels_to_rays_kernel computes them."""
  N = d['num_cameras']
  p2c, c2w = p2c.reshape(-1).astype(F), c2w.reshape(-1).astype(F)
  cam = np.zeros(px.shape[0], np.int64) if N == 1 or idx is None else idx.astype(np.int64)
  if mut != 'no_cam_clamp':
    cam = np.clip(cam, 0, N - 1)
  stride = 16 if mut == 'pose_stride_16' else 12
  P = lambda j: np.take(p2c, cam * 9 + j, mode='wrap')
  R = lambda j: np.take(c2w, cam * stride + j, mode='wrap')
  xf, yf = px.astype(F), py.astype(F)
  nb = F(0) if mut == 'no_half_neighbours' else F(0.5)
  with np.errstate(all='ignore'):
    c0 = _camera_dir(d, P, xf, yf, F(0.5), dirn, mut)
    cx = _camera_dir(d, P, (px + 1).astype(F), yf, nb, dirn, mut)
    cy = _camera_dir(d, P, xf, (py + 1).astype(F), nb, dirn, mut)
    dr, dx, dy = _mat3(R, 4, c0), _mat3(R, 4, cx), _mat3(R, 4, cy)
    o = [R(3), R(7), R(11)]
    n = np.sqrt(dr[0] * dr[0] + dr[1] * dr[1] + dr[2] * dr[2])
    vd = [dr[i] / n for i in range(3)]
    if not d['has_ndc']:
      dxn = _dist3(dx, dr)
      dyn = dxn if mut == 'radii_dx_twice' else _dist3(dy, dr)
    else:
      o_dx, d_dx = _to_ndc(d, o, dx, mut)
      o_dy, d_dy = _to_ndc(d, o, dy, mut)
      o, dr = _to_ndc(d, o, dr, mut)
      if mut == 'viewdirs_from_ndc':
        n = np.sqrt(dr[0] * dr[0] + dr[1] * dr[1] + dr[2] * dr[2])
        vd = [dr[i] / n for i in range(3)]
      if mut == 'ndc_radii_from_dirs':
        dxn, dyn = _dist3(d_dx, dr), _dist3(d_dy, dr)
      else:
        dxn, dyn = _dist3(o_dx, o), _dist3(o_dy, o)
    rad = F(0.5) * (dxn + dyn) * F(2) / SQRT12
  st = lambda vs: np.stack(vs, -1).astype(F)
  return dict(origins=st(o), directions=st(dr), viewdirs=st(vd), radii=st([rad]), imageplane=st(c0[:2]))


def check(name, dirn=0, mut=None):
  px, py, idx, p2c, c2w, d = make_inputs(name, limit=RAYS)
  ref = CR.reference(px, py, idx, p2c, c2w, d)
  got = emulate(px, py, idx, p2c, c2w, d, dirn, mut)
  return ref, got, CR.ratios(ref, got)


@pytest.mark.parametrize('name', list(CASES))
def test_emulation_within_bounds(name):
  c = case(name)
  px, py, idx, p2c, c2w, d = make_inputs(name, limit=RAYS)
  ref = CR.reference(px, py, idx, p2c, c2w, d)
  for dirn in ((1, -1) if c['camtype'] == 1 else (0,)):
    r = CR.ratios(ref, emulate(px, py, idx, p2c, c2w, d, dirn))
    for f in CR.FIELDS:
      assert float(r[f].max()) <= 1, (name, dirn, f, float(r[f].max()), int(r[f].max(-1).values.argmax()))
  checked = 1 - float(ref.vacuous.double().mean())
  print(f'\n{name}: rays {ref.vacuous.shape[0]} | checked {checked:.4f} (floor {c["floor"]}) | worst err/bound ' +
        ' '.join(f'{f} {float(r[f].max()):.3f}' for f in CR.FIELDS))
  assert checked >= c['floor'], (name, checked)


def test_case_matrix_reaches_its_edges():
  """What the cases are for: a grid beyond one grid-stride sweep of a 132-SM H100, exact-zero fisheye centres,
  monotone distortion, fisheye corners past theta = pi, pixel aspects in [0.5, 2], out-of-range indices."""
  px, _, _, _, _, _ = make_inputs('pinhole-grid')
  assert px.shape[0] > 132 * 8 * 256
  for name in CASES:
    c = case(name)
    px, py, idx, p2c, c2w, d = make_inputs(name, limit=RAYS)
    if d['has_distortion']:
      assert monotone(p2c, d, c['W'], c['H']), name
    if c['camtype'] == 1:
      cx, cy = centre(c)
      i = int(np.nonzero((px == cx) & (py == cy))[0][0])
      ip = emulate(px, py, idx, p2c, c2w, d)['imageplane'][i]
      assert (ip == 0).all(), (name, 'the centre pixel must map to exactly (0, 0)', ip)
  px, py, idx, p2c, c2w, d = make_inputs('fisheye-wide')
  x = p2c[0, 0, 0] * (px + 1.5) + p2c[0, 0, 2]
  y = p2c[0, 1, 1] * (py + 1.5) + p2c[0, 1, 2]
  assert (np.sqrt(x * x + y * y) > math.pi).sum() > 50
  px, py, idx, p2c, c2w, d = make_inputs('multi-camera')
  aspect = p2c[:, 0, 0] / p2c[:, 1, 1]
  assert aspect.min() < 0.8 and aspect.max() > 1.25 and (aspect >= 0.5).all() and (aspect <= 2).all()
  assert (idx == -3).any() and (idx == d['num_cameras'] + 5).any()
  _, _, idx, _, _, d = make_inputs('single-garbage-idx')
  assert d['num_cameras'] == 1 and ((idx < 0) | (idx > 0)).mean() > 0.99


# mutation: the cases tried, in order; the first is the one meant to catch it
MUTATIONS = {
    'no_half_neighbours': ('dist-golden-it10', 'fisheye-narrow'),
    'no_flip_y': ('pinhole-general',),
    'jacobian_p2': ('dist-tangential-it1', 'dist-golden-it1'),
    'newton_sign': ('dist-golden-it1', 'dist-barrel-it10'),
    'no_pi_clamp': ('fisheye-wide',),
    'radii_dx_twice': ('multi-camera', 'dist-barrel-it10'),
    'ndc_p02_both': ('ndc',),
    'viewdirs_from_ndc': ('ndc',),
    'ndc_radii_from_dirs': ('ndc',),
    'pose_stride_16': ('multi-camera',),
    'no_cam_clamp': ('multi-camera',),
    'sinc_0_over_0': ('fisheye-narrow', 'fisheye-wide'),
}


@pytest.mark.parametrize('mut', list(MUTATIONS))
def test_mutation_is_caught(mut):
  for name in MUTATIONS[mut]:
    ref, got, r = check(name, mut=mut)
    worst = max(float(r[f].max()) for f in CR.FIELDS)
    if worst > 1:
      f = max(CR.FIELDS, key=lambda f: float(r[f].max()))
      print(f'\n{mut}: caught by {name} on {sum(int((r[f] > 1).any(-1).sum()) for f in CR.FIELDS)} ray fields, '
            f'worst {f}: {worst:.3g} bounds')
      return
  raise AssertionError(f'{mut}: no case notices')


def test_fisheye_centre_was_nan():
  """0 / 0 at the optical axis: with sin(theta) / theta taken as it stands, the centre's direction, viewdir and
  radii are NaN, and so are the radii of its left and upper neighbours (their dx / dy neighbour is the centre).
  o_camera keeps that form only where theta > 0."""
  name = 'fisheye-narrow'
  px, py, idx, p2c, c2w, d = make_inputs(name, limit=RAYS)
  cx, cy = centre(case(name))
  at = lambda x, y: int(np.nonzero((px == x) & (py == y))[0][0])
  i, il, iu = at(cx, cy), at(cx - 1, cy), at(cx, cy - 1)
  bad = emulate(px, py, idx, p2c, c2w, d, mut='sinc_0_over_0')
  assert np.isnan(bad['directions'][i]).all() and np.isnan(bad['viewdirs'][i]).all()
  assert np.isnan(bad['radii'][[i, il, iu], 0]).all()
  good = emulate(px, py, idx, p2c, c2w, d)
  assert all(np.isfinite(good[f]).all() for f in CR.FIELDS)
  assert np.array_equal(good['directions'][i], -c2w[0, :, 2])
  t = lambda a: torch.tensor(a)
  o = o_camera.pixels_to_rays(t(px), t(py), t(p2c[0]), t(c2w[0]), camtype=o_camera.FISHEYE)
  assert all(torch.isfinite(v).all() for v in o)
  assert torch.equal(o[1][i], t(-c2w[0, :, 2]))


def _oracle64(px, py, idx, p2c, c2w, d):
  """o_camera.pixels_to_rays in float64 on the kernel's inputs, with the kernel's gather and descriptor."""
  N = d['num_cameras']
  cam = np.zeros(px.shape[0], int) if N == 1 or idx is None else np.clip(idx, 0, N - 1)
  dist = {k: d[k] for k in CR.KEYS}
  dist.update(eps=d['undistort_eps'], max_iterations=d['undistort_iters'])
  ndc = None
  if d['has_ndc']:
    ndc = torch.tensor([[1.0, 0, d['ndc_p02']], [0, 1.0, d['ndc_p12']], [0, 0, 1.0]], dtype=torch.float64)
  t = lambda a: torch.tensor(np.asarray(a, np.float64))
  conv = o_camera.convert_to_ndc
  try:
    o_camera.convert_to_ndc = lambda o, dr, p: conv(o, dr, p, d['ndc_near'])
    return o_camera.pixels_to_rays(torch.tensor(px), torch.tensor(py), t(p2c[cam]), t(c2w[cam]),
                                   dist if d['has_distortion'] else None, ndc,
                                   o_camera.FISHEYE if d['camtype'] == 1 else o_camera.PERSPECTIVE)
  finally:
    o_camera.convert_to_ndc = conv


def _agree(ref, vals, tag, rel=1e-12):
  for f, v in zip(CR.FIELDS, vals):
    a, b = getattr(ref, f), v.reshape(getattr(ref, f).shape).double()
    scale = b.abs().amax(-1, keepdim=True).clamp(min=1e-300) if f != 'radii' else b.abs().clamp(min=1e-6)
    err = ((a - b).abs() / scale).nan_to_num(nan=math.inf)
    assert float(err.max()) <= rel, (tag, f, float(err.max()))


@pytest.mark.parametrize('name', list(CASES))
def test_reference_is_the_oracle_in_fp64(name):
  px, py, idx, p2c, c2w, d = make_inputs(name, limit=RAYS)
  ref = CR.reference(px, py, idx, p2c, c2w, d, pi=math.pi, sqrt12=math.sqrt(12))
  _agree(ref, _oracle64(px, py, idx, p2c, c2w, d), name)


GOLDEN_CASES = ['persp', 'dist', 'fisheye', 'ndc', 'single', 'corners', 'aniso', 'widefish', 'ndcwide', 'fishcentre']


def _golden_inputs(name):
  pre = '' if name in ('persp', 'dist', 'fisheye', 'ndc', 'single') else f'{name}_'
  px, py = G[f'{pre}pix_x'], G[f'{pre}pix_y']
  idx = G[f'{pre}cam_idx'].reshape(-1)
  p2c = G[f'{pre}pixtocams']
  poses = G['ndc_poses'] if name == 'ndc' else G[f'{pre}camtoworlds']
  if name == 'single':
    p2c, poses = p2c[:1], poses[:1]
  dist = None
  if name in ('dist', 'fisheye'):
    dist = {str(k): float(v) for k, v in zip(G['dist_keys'], G['dist_vals'])}
  elif pre and f'{pre}dist_vals' in G:
    dist = {str(k): float(v) for k, v in zip(G[f'{pre}dist_keys'], G[f'{pre}dist_vals'])}
  ndc = None
  if name == 'ndc':
    ndc = G['pixtocam_ndc']
  elif pre and f'{pre}pixtocam_ndc' in G:
    ndc = G[f'{pre}pixtocam_ndc']
  fish = name in ('fisheye', 'widefish', 'fishcentre')
  d = dict(num_rays=px.size, num_cameras=p2c.shape[0], camtype=int(fish), has_distortion=int(dist is not None),
           **{k: float((dist or {}).get(k, 0.0)) for k in CR.KEYS}, undistort_eps=1e-9, undistort_iters=10,
           has_ndc=int(ndc is not None), ndc_p02=float(ndc[0, 2]) if ndc is not None else 1.0,
           ndc_p12=float(ndc[1, 2]) if ndc is not None else 1.0, ndc_near=1.0)
  return px.reshape(-1), py.reshape(-1), idx, p2c, poses, d


@pytest.mark.parametrize('name', GOLDEN_CASES)
def test_reference_reproduces_the_golden_fp64(name):
  """The reference's own float64 camera_utils, through cast_ray_batch on its seeded inputs."""
  px, py, idx, p2c, poses, d = _golden_inputs(name)
  ref = CR.reference(px, py, idx, p2c, poses, d, pi=math.pi, sqrt12=math.sqrt(12))
  vals = [torch.tensor(np.asarray(G[f'{name}_f64_{f}'], np.float64)).reshape(getattr(ref, f).shape)
          for f in CR.FIELDS]
  if name != 'fishcentre':
    _agree(ref, vals, name)
    return
  # the reference divides 0 by 0 on the optical axis: NaN at the centre and in the radii of its left and upper
  # neighbours, the reference's values everywhere else
  W, H = int(G['fishcentre_size'][0]), int(G['fishcentre_size'][1])
  i = ((H - 1) // 2) * W + (W - 1) // 2
  nan_rays = {f: np.nonzero(np.isnan(v.numpy()).any(-1))[0].tolist() for f, v in zip(CR.FIELDS, vals)}
  assert nan_rays['directions'] == [i] and nan_rays['viewdirs'] == [i], nan_rays
  assert nan_rays['radii'] == sorted([i - W, i - 1, i]), nan_rays
  keep = torch.ones(px.size, dtype=torch.bool)
  keep[[i - W, i - 1, i]] = False
  sub = types.SimpleNamespace(**{f: getattr(ref, f)[keep] for f in CR.FIELDS})
  _agree(sub, [v[keep] for v in vals], name)
  assert torch.equal(ref.directions[i], -torch.tensor(poses[0][:, 2], dtype=torch.float64))
  assert torch.isfinite(ref.radii).all()


def test_golden_inputs_reach_the_edges():
  """Strong distortion at the corners, non-square intrinsics, a fisheye past theta = pi, non-square NDC."""
  px, py, idx, p2c, poses, d = _golden_inputs('widefish')
  x = p2c[0, 0, 0] * (px + 0.5) + p2c[0, 0, 2]
  y = p2c[0, 1, 1] * (py + 0.5) + p2c[0, 1, 2]
  assert (np.hypot(x, y) > math.pi).any()
  _, _, _, p2c, _, d = _golden_inputs('aniso')
  assert (np.abs(p2c[:, 0, 0] / p2c[:, 1, 1] - 1) > 0.2).any()
  _, _, _, _, _, d = _golden_inputs('ndcwide')
  assert abs(d['ndc_p02'] / d['ndc_p12']) > 1.3
  _, _, _, _, _, d = _golden_inputs('corners')
  assert abs(d['k1']) >= 0.2
