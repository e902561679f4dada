"""Ray generation (mnrf_pixels_to_rays through the C ABI) against the fp64 reference of tests/camera_ref.py, on every
camera model, distortion, Newton iteration count, NDC setting and camera gather.  Needs an H100.

Every case fills the five output buffers with NaN before the call, so an element the kernel never writes fails, and
checks element by element: every output within its bound; origins bit-identical to fl32 of the pose translation
(non-NDC cases); on cases without sinf / cosf (every perspective camera) the outputs bit-identical to the numpy-fp32
transcription of tests/test_camera_reference_cpu.py, since camera.cu is built with -fmad=false and IEEE division and
sqrt.  Rays whose bound says nothing (camera_ref.VACUOUS_REL) are counted and printed; each case holds them to a floor
on the checked share.  Fisheye grids are odd-sized and include the exact centre pixel, where the undistorted point is
(0, 0) and sin(theta) / theta must be taken as 1: direction and viewdir there are R (0, 0, -1), and the radii of the
centre and of its left and upper neighbours are finite.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import camera_ref as CR

pytestmark = pytest.mark.gpu

F = np.float32
GOLDEN_DIST = dict(k1=0.05, k2=-0.02, k3=0.004, k4=0.0, p1=0.001, p2=-0.0015)
DISTS = {
    'golden': GOLDEN_DIST,
    'barrel': dict(k1=-0.25, k2=0.03),
    'pincushion': dict(k1=0.3, k2=0.05),
    'tangential': dict(p1=0.02, p2=-0.015),
    'k4': dict(k1=0.05, k2=-0.02, k3=0.01, k4=-0.004, p1=0.002, p2=0.001),
}
# name: overrides of DEFAULT.  intr: 'get' (get_pixtocam(f, W, H) per camera, f from `f`), 'general' (skew,
# fx != fy, last row not (0, 0, 1)), 'aspect' (own intrinsics per camera, pixel aspect in [0.5, 2]).  pixels: 'grid'
# (every pixel of W x H) or 'border' (border rows and columns, the corners, and `rays` random pixels).  idx: 'valid',
# 'out-of-range' (-3 and N + 5 among them), 'garbage' (N = 1 with an index array the kernel must ignore).
DEFAULT = dict(W=160, H=120, N=3, intr='get', f=(100.0, 130.0, 160.0), camtype=0, dist=None, iters=10, eps=1e-9,
               ndc=None, near=1.0, pixels='border', rays=2000, idx='valid', poses='random', floor=0.99)
CASES = {
    'pinhole-general': dict(W=200, H=150, N=1, intr='general'),
    'pinhole-grid': dict(W=1009, H=781, N=1, f=(800.0,), pixels='grid'),
    'multi-camera': dict(W=120, H=90, N=7, intr='aspect', idx='out-of-range', rays=3000),
    'single-garbage-idx': dict(W=64, H=48, N=1, f=(50.0,), idx='garbage'),
    **{f'dist-{k}-it{i}': dict(dist=k, iters=i, f=(140.0, 170.0, 200.0) if k == 'barrel' else DEFAULT['f'])
       for k in DISTS for i in (0, 1, 2, 10)},
    'dist-no-step': dict(dist='golden', eps=1e3),
    'fisheye-narrow': dict(W=101, H=81, N=1, f=(150.0,), camtype=1, pixels='grid'),
    'fisheye-narrow-dist': dict(W=101, H=81, N=1, f=(150.0,), camtype=1, pixels='grid', dist='golden'),
    'fisheye-wide': dict(W=61, H=45, N=1, f=(8.0,), camtype=1, pixels='grid'),
    'fisheye-wide-dist': dict(W=61, H=45, N=1, f=(10.0,), camtype=1, pixels='grid',
                              dist=dict(k1=0.01, k2=0.001)),
    'ndc': dict(W=120, H=80, N=4, f=(100.0, 110.0, 90.0, 120.0), ndc=100.0, poses='forward'),
    'ndc-dist': dict(W=120, H=80, N=4, f=(100.0, 110.0, 90.0, 120.0), ndc=100.0, poses='forward', dist='golden'),
    'ndc-near': dict(W=120, H=80, N=4, f=(100.0, 110.0, 90.0, 120.0), ndc=100.0, poses='forward', near=0.5),
}


def case(name):
  return dict(DEFAULT, **CASES[name])


def get_pixtocam(f, W, H):
  return np.linalg.inv(np.array([[f, 0, W * 0.5], [0, f, H * 0.5], [0, 0, 1.0]]))


def random_pose(rng):
  q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
  if np.linalg.det(q) < 0:
    q[:, 0] *= -1
  return np.concatenate([q, rng.uniform(-1.5, 1.5, (3, 1))], axis=1)


def forward_pose(rng):
  """A small rotation about the identity, looking down -z, as a forward-facing (NDC) capture."""
  w = rng.normal(size=3) * 0.08
  K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
  q, _ = np.linalg.qr(np.eye(3) + K + 0.5 * K @ K)
  q = q * np.sign(np.diag(q))[None, :]
  return np.concatenate([q, rng.uniform(-0.3, 0.3, (3, 1))], axis=1)


def centre(c):
  return (c['W'] - 1) // 2, (c['H'] - 1) // 2


def make_inputs(name, limit=None):
  """(pix_x, pix_y, cam_idx or None, pixtocams [N, 3, 3], camtoworlds [N, 3, 4] (fp32 numpy), desc dict).  limit:
  keep at most about that many rays, always with the corners and the centre pixel and its left and upper
  neighbours (the CPU tests run reduced counts)."""
  c = case(name)
  rng = np.random.default_rng(sum(map(ord, name)))
  W, H, N = c['W'], c['H'], c['N']
  if c['intr'] == 'get':
    p2c = np.stack([get_pixtocam(c['f'][i % len(c['f'])], W, H) for i in range(N)])
  elif c['intr'] == 'general':
    K = np.array([[170.0, 4.5, 97.0], [0.0, 135.0, 80.0], [3e-4, -2e-4, 0.97]])
    p2c = np.linalg.inv(K)[None]
  else:
    p2c = []
    for _ in range(N):
      fx = rng.uniform(60, 140)
      fy = fx * np.exp(rng.uniform(math.log(0.5), math.log(2.0)))
      p2c.append(np.linalg.inv(np.array([[fx, 0, W * rng.uniform(0.4, 0.6)], [0, fy, H * rng.uniform(0.4, 0.6)],
                                         [0, 0, 1.0]])))
    p2c = np.stack(p2c)
  c2w = np.stack([(forward_pose if c['poses'] == 'forward' else random_pose)(rng) for _ in range(N)])
  if c['pixels'] == 'grid':
    px, py = np.meshgrid(np.arange(W), np.arange(H), indexing='xy')
    px, py = px.reshape(-1), py.reshape(-1)
  else:
    xs, ys = np.arange(W), np.arange(H)
    bx = np.concatenate([xs, xs, np.zeros(H, int), np.full(H, W - 1)])
    by = np.concatenate([np.zeros(W, int), np.full(W, H - 1), ys, ys])
    px = np.concatenate([bx, rng.integers(0, W, c['rays'])])
    py = np.concatenate([by, rng.integers(0, H, c['rays'])])
  if limit is not None and px.shape[0] > limit:
    cx, cy = centre(c)
    keep = ((px == cx) | (px == cx - 1)) & ((py == cy) | (py == cy - 1))
    keep |= ((px == 0) | (px == W - 1)) & ((py == 0) | (py == H - 1))
    keep[np.linspace(0, px.shape[0] - 1, limit).astype(int)] = True
    px, py = px[keep], py[keep]
  B = px.shape[0]
  idx = None
  if c['idx'] == 'garbage':
    idx = rng.integers(-2 ** 31, 2 ** 31 - 1, B)
  elif N > 1:
    idx = rng.integers(0, N, B)
    if c['idx'] == 'out-of-range':
      idx[::5], idx[1::5] = -3, N + 5
  dist = DISTS[c['dist']] if isinstance(c['dist'], str) else c['dist']
  ndc = None
  if c['ndc'] is not None:
    pn = get_pixtocam(c['ndc'], W, H)
    ndc = (pn[0, 2], pn[1, 2])
  d = CR.desc(B, N, c['camtype'], dist, c['eps'], c['iters'], ndc, c['near'])
  i32 = lambda a: None if a is None else np.ascontiguousarray(a, np.int32)
  return i32(px), i32(py), i32(idx), p2c.astype(F), c2w.astype(F), d


def monotone(p2c, d, W, H):
  """The forward distortion map has det J > 0 on a disk 10% wider than the undistorted image (every camera)."""
  k = {n: d[n] for n in CR.KEYS}
  xs = np.concatenate([np.arange(W + 1), np.arange(W + 1), np.zeros(H + 1), np.full(H + 1, W)]) + 0.5
  ys = np.concatenate([np.zeros(W + 1), np.full(W + 1, H), np.arange(H + 1), np.arange(H + 1)]) + 0.5
  rmax = 0.0
  from oracle import o_camera
  for P in p2c.astype(np.float64):
    xd = torch.tensor(P[0, 0] * xs + P[0, 1] * ys + P[0, 2])
    yd = torch.tensor(P[1, 0] * xs + P[1, 1] * ys + P[1, 2])
    x, y = o_camera.radial_and_tangential_undistort(xd, yd, **k, max_iterations=50)
    fx, fy = o_camera._residual_and_jacobian(x, y, xd, yd, **k)[:2]
    if float(torch.maximum(fx.abs(), fy.abs()).max()) > 1e-12:
      return False
    rmax = max(rmax, float(torch.sqrt(x * x + y * y).max()))
  r = torch.linspace(0, 1.1 * rmax, 400, dtype=torch.float64)[:, None]
  a = torch.linspace(0, 2 * math.pi, 721, dtype=torch.float64)[None]
  _, _, fx_x, fx_y, fy_x, fy_y = o_camera._residual_and_jacobian(r * torch.cos(a), r * torch.sin(a), 0, 0, **k)
  return bool((fx_x * fy_y - fx_y * fy_x > 0).all())


# ----------------------------------------------------------------------------------------------------------- GPU

def _desc(d):
  from multinerf_b200 import lib as L
  return L.CameraDesc(*[d[n] for n, _ in L.CameraDesc._fields_])


def run(px, py, idx, p2c, c2w, d):
  """One mnrf_pixels_to_rays call into NaN-filled buffers; ({field: [B, n] fp32 numpy}, return code)."""
  from multinerf_b200 import lib as L
  lib = L.load()
  B = px.shape[0]
  dev = lambda a: None if a is None else torch.tensor(a).cuda().contiguous()
  ins = [dev(px), dev(py), dev(idx), dev(p2c.reshape(-1, 9)), dev(c2w.reshape(-1, 12))]
  out = {f: torch.full((B, n), math.nan, device='cuda') for f, n in zip(CR.FIELDS, (3, 3, 3, 1, 2))}
  rc = lib.mnrf_pixels_to_rays(C.byref(_desc(d)), *[L.ptr(t) for t in ins], *[L.ptr(out[f]) for f in CR.FIELDS],
                               L.stream_ptr())
  torch.cuda.synchronize()
  return {f: t.cpu().numpy() for f, t in out.items()}, rc


@pytest.fixture(scope='module')
def lib():
  from multinerf_b200 import lib as L
  L.require_device()
  return L.load()


def report(name, ref, r):
  checked = 1 - float(ref.vacuous.double().mean())
  worst = ' '.join(f'{f} {float(r[f].max()):.3f}' for f in CR.FIELDS)
  return checked, f'{name}: rays {ref.vacuous.shape[0]} | checked {checked:.4f} | worst err/bound {worst}'


@pytest.mark.parametrize('name', list(CASES))
def test_rays_case(lib, name):
  from test_camera_reference_cpu import emulate
  c = case(name)
  px, py, idx, p2c, c2w, d = make_inputs(name)
  if name == 'pinhole-grid':
    assert px.shape[0] > lib.mnrf_num_sms() * 8 * 256, 'the grid must exceed one sweep of the grid-stride loop'
  if d['has_distortion']:
    assert monotone(p2c, d, c['W'], c['H']), name
  got, rc = run(px, py, idx, p2c, c2w, d)
  assert rc == 0, lib.mnrf_last_error().decode()
  ref = CR.reference(px, py, idx, p2c, c2w, d)
  r = CR.ratios(ref, got)
  checked, line = report(name, ref, r)
  print('\n' + line + f' (floor {c["floor"]})')
  assert checked >= c['floor'], (name, checked)
  for f in CR.FIELDS:
    assert not np.isnan(got[f]).any(), (name, f, 'unwritten or NaN element')
    bad = r[f] > 1
    assert not bad.any(), (name, f, float(r[f].max()), int(bad.any(-1).nonzero()[0, 0]))
  if not d['has_ndc']:
    cam = np.zeros(px.shape[0], int) if idx is None or d['num_cameras'] == 1 else np.clip(idx, 0, d['num_cameras'] - 1)
    assert np.array_equal(got['origins'], c2w[cam][:, :, 3]), (name, 'origins are not the pose translation')
  if d['camtype'] == 0:
    em = emulate(px, py, idx, p2c, c2w, d)
    for f in CR.FIELDS:
      same = got[f].view(np.int32) == em[f].view(np.int32)
      assert same.all(), (name, f, 'differs from the fp32 transcription in', int((~same).sum()), 'elements')
    print(f'{name}: bit-identical to the fp32 transcription')
  if d['camtype'] == 1:
    check_centre(name, px, py, c2w, got)


def check_centre(name, px, py, c2w, got):
  cx, cy = centre(case(name))
  at = lambda x, y: int(np.nonzero((px == x) & (py == y))[0][0])
  i = at(cx, cy)
  R = c2w[0, :, :3]
  assert np.array_equal(got['directions'][i], -R[:, 2]), (name, got['directions'][i], -R[:, 2])
  assert np.abs(got['viewdirs'][i] + R[:, 2] / np.linalg.norm(R[:, 2].astype(np.float64))).max() < 1e-6
  for j in (i, at(cx - 1, cy), at(cx, cy - 1)):
    assert np.isfinite(got['radii'][j]).all() and got['radii'][j][0] > 0, (name, j, got['radii'][j])


def test_no_rays_writes_nothing(lib):
  px, py, idx, p2c, c2w, d = make_inputs('multi-camera', limit=16)
  got, rc = run(px, py, idx, p2c, c2w, dict(d, num_rays=0))
  assert rc == 0
  for f in CR.FIELDS:
    assert np.isnan(got[f]).all(), f
  assert lib.mnrf_pixels_to_rays(C.byref(_desc(dict(d, num_rays=0))), *[None] * 10, None) == 0


def test_error_paths(lib):
  from multinerf_b200 import lib as L
  px, py, idx, p2c, c2w, d = make_inputs('multi-camera', limit=16)
  B = px.shape[0]
  ins = [torch.tensor(a).cuda() for a in (px, py, idx, p2c.reshape(-1, 9), c2w.reshape(-1, 12))]
  outs = [torch.full((B, n), math.nan, device='cuda') for n in (3, 3, 3, 1, 2)]
  ptrs = [L.ptr(t) for t in ins + outs]

  def call(dd, p=ptrs):
    rc = lib.mnrf_pixels_to_rays(C.byref(_desc(dd)), *p, L.stream_ptr())
    return rc, lib.mnrf_last_error().decode()

  for dd, p, msg in [(d, ptrs[:5] + [None] + ptrs[6:], 'null pointer'),
                     (dict(d, num_cameras=0), ptrs, 'num_cameras must be >= 1'),
                     (d, ptrs[:2] + [None] + ptrs[3:], 'cam_idx is required'),
                     (dict(d, camtype=2), ptrs, 'camtype must be'),
                     (dict(d, has_distortion=1, undistort_iters=-1), ptrs, 'undistort_iters < 0')]:
    rc, err = call(dd, p)
    assert rc != 0 and msg in err, (msg, rc, err)
  assert lib.mnrf_pixels_to_rays(None, *ptrs, L.stream_ptr()) != 0
  torch.cuda.synchronize()
  assert all(torch.isnan(t).all() for t in outs), 'a refused call wrote its outputs'
