"""Reference of pixel -> ray generation (csrc/camera.cu, camera model in csrc/camera.cuh) with a bound on every element.

`reference` takes exactly the inputs of mnrf_pixels_to_rays -- fp32 pix_x, pix_y, cam_idx, pixtocams [N, 3, 3],
camtoworlds [N, 3, 4] and the mnrf_camera_desc fields as a dict (`desc`) -- and returns origins, directions, viewdirs,
radii and imageplane in float64, each with a bound on how far the kernel's fp32 value may stray from it, element by
element.  It follows the kernel's semantics: the camera gather clamped to [0, N - 1] (cam_idx ignored when N = 1),
the pixel centre at +0.5, mat3_vec's summation order, exactly `undistort_iters` Newton steps with the
|den| > eps branch, the fisheye clamp at fl32(pi) (`pi=`), sin(theta) / theta = 1 at theta = 0, the OpenCV -> OpenGL
flip, viewdirs from the world direction taken before NDC, NDC radii from the differences of the NDC origins, and
cone_radius dividing by fl32(sqrt(12)) (`sqrt12=`).  With pi=math.pi and sqrt12=math.sqrt(12) the values are those of
oracle/o_camera.py and of the reference's camera_utils in float64.

Bounds are running errors (encode_ref._V: fp64 value, absolute error bound of the fp32 value).  camera.cu is built
with -fmad=false and without fast math (multinerf_b200/build.py), so every product and sum rounds on its own, and
division and sqrt are correctly rounded (u = 2^-24 of the result); sinf and cosf are documented at 2 ulp.  Pixel
coordinates + 0.5 and the flip are exact, origins are copies.

Newton.  Carried operation by operation through undistort_iters steps the running error roughly doubles every step,
so at 10 steps it would say nothing.  The Newton map N(x) = x - J(x)^-1 F(x) is what removes input error, so the
error is carried through N instead.  With x_k the fp64 iterate and e_k the bound of the kernel's iterate (per
component):
    e_{k+1} <= |DN(x_k)| e_k + |J(x_k)^-1| e_xd + |D^2N(x_k)| e_k e_k + delta_k
DN and D^2N are derivatives of the fp64 Newton map, carried through o_camera's residual and Jacobian by second-order
forward-mode arithmetic (_D2: exact derivatives of the formula, evaluated in fp64); DN is near 0 at the root.  N is
linear in the distorted point xd, with slope J^-1, which brings in e_xd, the bound of the kernel's xd.  The quadratic term is half of |D^2N| at the iterate, doubled to stand for its
supremum over the error box (e_k < 1e-5, where D^2N hardly changes).  delta_k is the running-error bound of one step
evaluated with exact inputs.  Where the step is not taken (|den| <= eps) N is the identity.
    vacuous  A ray is marked where the kernel may take the other branch (the fp64 |den| within its own bound of
             eps), where the Jacobian of the distortion is singular or folded (det J <= 0: the undistortion has no
             unique root), and where any bound exceeds VACUOUS_REL of its output's scale (1 for the vectors, the
             radius, or 0.01 where it is smaller, for radii: past theta = pi a fisheye's neighbours share one
             direction and the radius is ~0).  It is not dropped silently: the tests print the checked share per case and
             hold it to a floor.

Fisheye.  s = sin(theta) / theta is taken as one function: |sinc'| <= min(theta / 3, 0.44), so the inherited error
is that slope times e_theta, plus sinf's 4u and the division's u of s.  This also covers a kernel theta of 0 (s = 1)
beside a tiny fp64 theta.

Pure torch on the CPU; never loads the CUDA library.
"""
import math
import types

import numpy as np
import torch

from encode_ref import SLACK, TINY, U, _V
from oracle import o_camera

PI32 = float(np.float32(math.pi))
SQRT12_32 = float(np.float32(3.4641016151377544))
VACUOUS_REL = 1e-3
FIELDS = ('origins', 'directions', 'viewdirs', 'radii', 'imageplane')
KEYS = ('k1', 'k2', 'k3', 'k4', 'p1', 'p2')


def desc(num_rays=0, num_cameras=1, camtype=0, dist=None, eps=1e-9, iters=10, ndc=None, near=1.0):
  """The mnrf_camera_desc fields as the kernel sees them (fp32-rounded); dist: {k1..p2}, ndc: (p02, p12)."""
  f = lambda v: float(np.float32(v))
  dist = dist or {}
  return dict(num_rays=num_rays, num_cameras=num_cameras, camtype=camtype, has_distortion=int(bool(dist)),
              **{k: f(dist.get(k, 0.0)) for k in KEYS}, undistort_eps=f(eps), undistort_iters=iters,
              has_ndc=int(ndc is not None), ndc_p02=f(ndc[0]) if ndc is not None else 1.0,
              ndc_p12=f(ndc[1]) if ndc is not None else 1.0, ndc_near=f(near))


def _mat3_vec(m, ld, v):
  """m: [B, 3 * ld] flat rows of _V-able values; mat3_vec's order: ((m0 v0 + m1 v1) + m2 v2)."""
  return [_V(m[:, r * ld]) * v[0] + _V(m[:, r * ld + 1]) * v[1] + _V(m[:, r * ld + 2]) * v[2] for r in range(3)]


def _step(x, y, xd, yd, k, eps):
  """One Newton step of `undistort` on _V operands, in the kernel's order; (x', y', den, ok)."""
  k1, k2, k3, k4, p1, p2 = (_V(k[n]) for n in KEYS)
  r = x * x + y * y
  dd = r * (k1 + r * (k2 + r * (k3 + r * k4))) + 1.0
  fx = dd * x + p1 * 2.0 * x * y + p2 * (r + x * 2.0 * x) - xd
  fy = dd * y + p2 * 2.0 * x * y + p1 * (r + y * 2.0 * y) - yd
  d_r = k1 + r * (k2 * 2.0 + r * (k3 * 3.0 + r * 4.0 * k4))
  d_x = x * 2.0 * d_r
  d_y = y * 2.0 * d_r
  fx_x = dd + d_x * x + p1 * 2.0 * y + p2 * 6.0 * x
  fx_y = d_y * x + p1 * 2.0 * x + p2 * 2.0 * y
  fy_x = d_x * y + p2 * 2.0 * y + p1 * 2.0 * x
  fy_y = dd + d_y * y + p2 * 2.0 * x + p1 * 6.0 * y
  den = fy_x * fx_y - fx_x * fy_y
  xn = fx * fy_y - fy * fx_y
  yn = fy * fx_x - fx * fy_x
  ok = den.val.abs() > eps
  return x + _V.where(ok, xn / den, 0.0), y + _V.where(ok, yn / den, 0.0), den, ok


class _D2:
  """Second-order forward-mode value in two variables: value, gradient [2], Hessian [2][2] (tensors)."""

  def __init__(self, v, g=None, h=None):
    self.v = torch.as_tensor(v, dtype=torch.float64)
    z = torch.zeros_like(self.v)
    self.g = g or [z, z]
    self.h = h or [[z, z], [z, z]]

  @staticmethod
  def of(a):
    return a if isinstance(a, _D2) else _D2(a)

  def __add__(self, o):
    o = _D2.of(o)
    return _D2(self.v + o.v, [a + b for a, b in zip(self.g, o.g)],
               [[self.h[i][j] + o.h[i][j] for j in range(2)] for i in range(2)])

  __radd__ = __add__

  def __neg__(self):
    return _D2(-self.v, [-a for a in self.g], [[-a for a in r] for r in self.h])

  def __sub__(self, o):
    return self + (-_D2.of(o))

  def __rsub__(self, o):
    return _D2.of(o) - self

  def __mul__(self, o):
    o = _D2.of(o)
    return _D2(self.v * o.v, [self.v * o.g[i] + o.v * self.g[i] for i in range(2)],
               [[self.v * o.h[i][j] + o.v * self.h[i][j] + self.g[i] * o.g[j] + o.g[i] * self.g[j]
                 for j in range(2)] for i in range(2)])

  __rmul__ = __mul__

  def inv(self):
    r = 1.0 / self.v
    return _D2(r, [-r * r * a for a in self.g],
               [[2 * r ** 3 * self.g[i] * self.g[j] - r * r * self.h[i][j] for j in range(2)] for i in range(2)])

  def __truediv__(self, o):
    return self * _D2.of(o).inv()


def _derivs(xd, yd, k, x, y):
  """DN (d1[j][i] = dN_i / dx_j) and D^2N (d2[j][l][i]) of the Newton step taken where ok, at (x, y)."""
  one, zero = torch.ones_like(x), torch.zeros_like(x)
  X, Y = _D2(x, [one, zero]), _D2(y, [zero, one])
  fx, fy, fx_x, fx_y, fy_x, fy_y = o_camera._residual_and_jacobian(X, Y, xd, yd, **k)
  den = fy_x * fx_y - fx_x * fy_y
  n = [X + (fx * fy_y - fy * fx_y) / den, Y + (fy * fx_x - fx * fy_x) / den]
  return [[n[i].g[j] for i in range(2)] for j in range(2)], [[[n[i].h[j][l] for i in range(2)] for l in range(2)]
                                                             for j in range(2)]


def _undistort(xd, yd, k, eps, iters):
  """(x, y as _V with the Newton-rule bound, vacuous [B])."""
  x, y = _V(xd.val.clone()), _V(yd.val.clone())
  ex, ey = xd.err.clone(), yd.err.clone()         # the kernel's iterate starts at its own xd
  vac = torch.zeros_like(xd.val, dtype=torch.bool)
  eye = [[torch.ones_like(ex), torch.zeros_like(ex)], [torch.zeros_like(ex), torch.ones_like(ex)]]
  flat = [[[torch.zeros_like(ex)] * 2] * 2] * 2
  for _ in range(iters):
    xs, ys, den, ok = _step(x, y, _V(xd.val), _V(yd.val), k, eps)
    vac |= (den.val.abs() - eps).abs() <= den.err
    _, _, fx_x, fx_y, fy_x, fy_y = o_camera._residual_and_jacobian(x.val, y.val, xd.val, yd.val, **k)
    det = fx_x * fy_y - fx_y * fy_x
    vac |= ok & ~(det > 0)
    d1, d2 = _derivs(xd.val, yd.val, k, x.val, y.val)
    # where the step is not taken N is the identity
    d1 = [[torch.where(ok, d1[j][i], eye[j][i]) for i in range(2)] for j in range(2)]
    d2 = [[[torch.where(ok, d2[j][l][i], flat[j][l][i]) for i in range(2)] for l in range(2)] for j in range(2)]
    e = (ex, ey)
    lin = [d1[0][i].abs() * ex + d1[1][i].abs() * ey for i in range(2)]
    quad = [sum(d2[j][l][i].abs() * e[j] * e[l] for j in range(2) for l in range(2)) for i in range(2)]
    inv = [[fy_y / det, -fx_y / det], [-fy_x / det, fx_x / det]]
    dxd = [torch.where(ok, inv[i][0].abs() * xd.err + inv[i][1].abs() * yd.err, torch.zeros_like(det))
           for i in range(2)]
    ex = SLACK * (lin[0] + quad[0] + dxd[0] + xs.err)
    ey = SLACK * (lin[1] + quad[1] + dxd[1] + ys.err)
    x, y = _V(xs.val), _V(ys.val)
  return _V(x.val, ex), _V(y.val, ey), vac


def _sinc(theta):
  t, e = theta.val, theta.err
  pos = t > 0
  s = torch.where(pos, torch.sin(t) / torch.where(pos, t, torch.ones_like(t)), torch.ones_like(t))
  slope = torch.minimum((t + e) / 3, torch.full_like(t, 0.44))
  inherited = slope * e
  return _V(s, inherited + 5 * U * (s.abs() + inherited))


def camera_dir(d, p2c, px, py, pi=PI32):
  """camera_dir of camera.cuh on [B] pixel columns: (v [3] of _V, vacuous [B])."""
  v = _mat3_vec(p2c, 3, [_V(px + 0.5), _V(py + 0.5), _V(torch.ones_like(px))])
  vac = torch.zeros_like(px, dtype=torch.bool)
  if d['has_distortion']:
    x, y, vac = _undistort(v[0], v[1], {k: d[k] for k in KEYS}, d['undistort_eps'], d['undistort_iters'])
    v = [x, y, _V(torch.ones_like(px))]
  if d['camtype'] == 1:
    theta = (v[0] * v[0] + v[1] * v[1]).sqrt().minc(pi)
    s = _sinc(theta)
    v = [v[0] * s, v[1] * s, theta.cos()]
  return [v[0], v[1].scale(-1.0), v[2].scale(-1.0)], vac


def _to_ndc(d, o, dr):
  t = (_V(d['ndc_near']) + o[2]).scale(-1.0) / dr[2]
  o = [o[i] + t * dr[i] for i in range(3)]
  xm, ym = 1.0 / _V(d['ndc_p02']), 1.0 / _V(d['ndc_p12'])
  o_ndc = [xm * o[0] / o[2], ym * o[1] / o[2], _V(torch.full_like(o[0].val, -1.0))]
  inf = [xm * dr[0] / dr[2], ym * dr[1] / dr[2], _V(torch.ones_like(o[0].val))]
  return o_ndc, [inf[i] - o_ndc[i] for i in range(3)]


def _dist3(a, b):
  x, y, z = a[0] - b[0], a[1] - b[1], a[2] - b[2]
  return (x * x + y * y + z * z).sqrt()


def _np64(a):
  return torch.as_tensor(np.asarray(a.detach().cpu() if isinstance(a, torch.Tensor) else a), dtype=torch.float64)


def reference(pix_x, pix_y, cam_idx, pixtocams, camtoworlds, d, pi=PI32, sqrt12=SQRT12_32):
  """fp64 reference of mnrf_pixels_to_rays with per-element bounds.  Inputs are taken at their values (fp32 inputs
  are exact in fp64); `d`: desc().  Returns a namespace with the five outputs [B, 3|3|3|1|2], `bound` (a dict of the
  same shapes) and `vacuous` [B]."""
  px, py = _np64(pix_x).reshape(-1), _np64(pix_y).reshape(-1)
  B = px.shape[0]
  p2c, c2w = _np64(pixtocams).reshape(-1, 9), _np64(camtoworlds).reshape(-1, 12)
  N = p2c.shape[0]
  cam = torch.zeros(B, dtype=torch.long) if N == 1 or cam_idx is None else _np64(cam_idx).reshape(-1).long()
  cam = cam.clamp(0, N - 1)
  P, R = p2c[cam], c2w[cam]
  c0, v0 = camera_dir(d, P, px, py, pi)
  cx, v1 = camera_dir(d, P, px + 1, py, pi)
  cy, v2 = camera_dir(d, P, px, py + 1, pi)
  dr, dx, dy = _mat3_vec(R, 4, c0), _mat3_vec(R, 4, cx), _mat3_vec(R, 4, cy)
  o = [_V(R[:, 3]), _V(R[:, 7]), _V(R[:, 11])]
  n = (dr[0] * dr[0] + dr[1] * dr[1] + dr[2] * dr[2]).sqrt()
  vd = [dr[i] / n for i in range(3)]
  if not d['has_ndc']:
    dxn, dyn = _dist3(dx, dr), _dist3(dy, dr)
  else:
    o_dx, _ = _to_ndc(d, o, dx)
    o_dy, _ = _to_ndc(d, o, dy)
    o, dr = _to_ndc(d, o, dr)
    dxn, dyn = _dist3(o_dx, o), _dist3(o_dy, o)
  rad = ((dxn + dyn).scale(0.5)).scale(2.0) / sqrt12
  stack = lambda vs: (torch.stack([v.val for v in vs], -1), torch.stack([SLACK * v.err + TINY for v in vs], -1))
  out = types.SimpleNamespace(bound={})
  for name, vs in zip(FIELDS, (o, dr, vd, [rad], [c0[0], c0[1]])):
    val, b = stack(vs)
    setattr(out, name, val)
    out.bound[name] = b
  vac = v0 | v1 | v2
  for name in FIELDS:
    val, b = getattr(out, name), out.bound[name]
    scale = val.abs().clamp(min=0.01) if name == 'radii' else val.norm(dim=-1, keepdim=True).clamp(min=1.0)
    vac |= ~(b <= VACUOUS_REL * scale).all(-1)
  out.vacuous = vac
  return out


def ratios(ref, got):
  """{field: [B, n] |got - ref| / bound}, with vacuous rays at 0; got: {field: array}."""
  out = {}
  for f in FIELDS:
    g = _np64(got[f]).reshape(ref.bound[f].shape)
    r = (g - getattr(ref, f)).abs() / ref.bound[f]
    r = torch.where(torch.isnan(r), torch.full_like(r, math.inf), r)
    out[f] = torch.where(ref.vacuous[:, None], torch.zeros_like(r), r)
  return out
