"""fp64 restatement of the TSDF fusion of csrc/mesh.cu (mnrf_tsdf_integrate) and of its forward camera projection
(project_point, csrc/camera.cuh), for the CPU and GPU tests.  numpy only."""
import numpy as np

EPS32 = float(np.finfo(np.float32).eps)
PIXEL_MARGIN = 1e-3      # pixels: a point this close to a pixel edge may land in either pixel in fp32
DIST_MARGIN = 1e-4       # relative to 1 + |depth| + |t|: d this close to +-tau may fall on either side in fp32


def project(points, w2c, c2p, camtype='perspective', distortion=None):
  """points [N, 3], w2c [3, 4] world-to-camera (OpenGL axes), c2p [3, 3] camera-to-pixel -> (u, v, t, valid) in
  fp64: the continuous pixel (centres at +0.5) and the parameter along that pixel's ray; valid is False for a point
  behind a perspective camera or on the optical axis behind a fisheye."""
  p = np.asarray(points, np.float64)
  w2c, c2p = np.asarray(w2c, np.float64), np.asarray(c2p, np.float64)
  q = p @ w2c[:, :3].T + w2c[:, 3]
  qx, qy, qz = q[:, 0], -q[:, 1], -q[:, 2]          # OpenGL -> OpenCV
  if camtype == 'fisheye':
    r = np.hypot(qx, qy)
    t = np.sqrt(r * r + qz * qz)
    valid = (r > 0) | (qz > 0)
    s = np.where(r > 0, np.arctan2(r, qz) / np.where(r > 0, r, 1.0), 0.0)
    x, y = qx * s, qy * s
  else:
    valid = qz > 0
    t = qz
    z = np.where(valid, qz, 1.0)
    x, y = qx / z, qy / z
  if distortion is not None:
    k = {n: float(distortion.get(n, 0.0)) for n in ('k1', 'k2', 'k3', 'k4', 'p1', 'p2')}
    r2 = x * x + y * y
    dd = 1.0 + r2 * (k['k1'] + r2 * (k['k2'] + r2 * (k['k3'] + r2 * k['k4'])))
    x, y = (dd * x + 2 * k['p1'] * x * y + k['p2'] * (r2 + 2 * x * x),
            dd * y + 2 * k['p2'] * x * y + k['p1'] * (r2 + 2 * y * y))
  h = np.stack([x, y, np.ones_like(x)], -1) @ c2p.T
  return h[:, 0] / h[:, 2], h[:, 1] / h[:, 2], t, valid


def grid_points(shape, lo, h):
  """The fp32 grid points lo + h (x, y, z) of an (nx, ny, nz) grid, x fastest, rounded from fp64 -> [N, 3] fp64."""
  nx, ny, nz = shape
  z, y, x = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing='ij')
  pts = np.stack([lo[0] + x * h, lo[1] + y * h, lo[2] + z * h], -1).reshape(-1, 3)
  return pts.astype(np.float32).astype(np.float64)


def integrate(points, w2c, c2p, depth, acc, rgb, tau, camtype='perspective', distortion=None):
  """fp64 TSDF fusion of K views into fresh state at `points` [N, 3] (fp32 values).  w2c [K, 3, 4], c2p [K or 1, 3,
  3], depth / acc [K, H, W], rgb [K, H, W, 3] or None: the kernel's fp32 inputs.  Returns (tsdf, weight, color_sum,
  color_weight, bound, exempt): `bound` bounds |tsdf - fp32 tsdf| per point; `exempt` flags points whose fate in
  some view turns on a comparison within rounding of its edge (a pixel edge, -tau or +tau)."""
  K, H, W = depth.shape
  N = points.shape[0]
  tau = float(np.float32(tau))
  tsdf, weight = np.zeros(N), np.zeros(N)
  color_sum, color_weight = np.zeros((N, 3)), np.zeros(N)
  exempt = np.zeros(N, bool)
  bound = np.zeros(N)
  scale = np.abs(points).sum(-1)
  for k in range(K):
    u, v, t, valid = project(points, w2c[k], c2p[k if c2p.shape[0] > 1 else 0], camtype, distortion)
    with np.errstate(invalid='ignore'):
      near_edge = valid & ((np.abs(u - np.round(u)) < PIXEL_MARGIN) | (np.abs(v - np.round(v)) < PIXEL_MARGIN))
      inside = valid & (u >= 0) & (u < W) & (v >= 0) & (v < H)
    px = np.where(inside, np.floor(np.where(inside, u, 0)), 0).astype(np.int64)
    py = np.where(inside, np.floor(np.where(inside, v, 0)), 0).astype(np.int64)
    dep = depth[k, py, px].astype(np.float64)
    a = acc[k, py, px]
    use = inside & np.isfinite(dep)
    with np.errstate(invalid='ignore'):
      d = np.where(a >= 0.5, dep - np.where(use, t, 0), np.inf)
      margin = DIST_MARGIN * (1 + np.abs(np.where(use, dep, 0)) + np.abs(np.where(use, t, 0)))
      near_tau = use & np.isfinite(d) & ((np.abs(d + tau) < margin) | (np.abs(d - tau) < margin))
      use &= ~(d < -tau)
    exempt |= near_edge | near_tau
    s = np.minimum(np.where(use, d, 0), tau) / tau
    tsdf = np.where(use, (weight * tsdf + s) / (weight + 1), tsdf)
    weight = weight + use
    # fp32 error of one view's term: t and depth - t to a few ulps of the point's and the pose's scale
    pose = np.abs(w2c[k]).sum()
    err = 16 * EPS32 * (np.abs(np.where(use, dep, 0)) + np.abs(np.where(use, t, 0)) + 3 * pose * (1 + scale)) / tau
    bound = np.maximum(bound, np.where(use & np.isfinite(d), err, 0))
    if rgb is not None:
      col = use & (np.abs(d) <= tau)
      color_sum += np.where(col[:, None], rgb[k, py, px].astype(np.float64), 0)
      color_weight += col
  bound = bound + 8 * (K + 1) * EPS32          # the running mean's own roundings
  return tsdf, weight, color_sum, color_weight, bound, exempt
