"""fp64 restatement of the scene contraction as point maps (coord.contract and coord.inv_contract, csrc/contract.cuh),
its Jacobian and the world normals of contracted level sets (mnrf_mesh_uncontract), and of the contracted-space TSDF
fusion (mnrf_tsdf_integrate_contracted, csrc/mesh.cu), for the CPU and GPU tests.  numpy only."""
import numpy as np

import tsdf_ref

EPS32 = float(np.finfo(np.float32).eps)


def contract(x):
  """contract(x) [N, 3] fp64: x inside the unit ball, (2 - 1 / r) x / r outside (|x|^2 clamped to eps32)."""
  x = np.asarray(x, np.float64)
  m = np.maximum(EPS32, (x * x).sum(-1, keepdims=True))
  r = np.sqrt(m)
  return np.where(m <= 1, x, (2 * r - 1) / m * x)


def inv_contract(z):
  """inv_contract(z) [N, 3] fp64 for |z| < 2: z inside the unit ball, z / (r (2 - r)) outside."""
  z = np.asarray(z, np.float64)
  m = np.maximum(EPS32, (z * z).sum(-1, keepdims=True))
  r = np.sqrt(m)
  with np.errstate(divide='ignore', invalid='ignore'):
    return np.where(m <= 1, z, z / (r * (2 - r)))


def jacobian(x):
  """d contract / dx [N, 3, 3] at world points x: s (I - P) + q P with P = xh xh^T, s = 2/r - 1/r^2, q = 1/r^2
  outside the unit ball, I inside."""
  x = np.asarray(x, np.float64)
  m = np.maximum(EPS32, (x * x).sum(-1))
  r = np.sqrt(m)
  out = m > 1
  xh = np.where(out[:, None], x / r[:, None], 0.0)
  s = np.where(out, 2 / r - 1 / m, 1.0)
  q = np.where(out, 1 / m, 1.0)
  P = xh[:, :, None] * xh[:, None, :]
  eye = np.eye(3)[None]
  return s[:, None, None] * (eye - P) + q[:, None, None] * P


def world_normals(z, n):
  """Unit world normals J(inv_contract(z)) n of contracted level-set normals n [N, 3]."""
  v = np.einsum('nij,nj->ni', jacobian(inv_contract(z)), np.asarray(n, np.float64))
  return v / np.linalg.norm(v, axis=-1, keepdims=True)


def integrate_contracted(points, w2c, c2p, depth, acc, rgb, tau, camtype='perspective', distortion=None):
  """fp64 contracted TSDF fusion of K views into fresh state at contracted grid points `points` [N, 3] (fp32 values),
  as tsdf_ref.integrate returns it: (tsdf, weight, color_sum, color_weight, bound, exempt).  Points with |p| >= 2
  are never observed.  Each point is projected at x = inv_contract(p); where acc >= 0.5, d = sign(depth - t)
  |contract(s) - p| with s = o + (x - o) depth / t, else +inf.  The bound adds to tsdf_ref's the fp32 error of x,
  s and contract(s) -- relative errors of a few eps32 in world points that the contraction shrinks by |dy/dx| <= 1 --
  and `exempt` marks what sits within rounding of a pixel edge or of +-tau, and points with |p| within 1e-5 of 2."""
  p = np.asarray(points, np.float64)
  K, H, W = depth.shape
  N = p.shape[0]
  tau = float(np.float32(tau))
  r = np.linalg.norm(p, axis=-1)
  live = r < 2
  x = np.where(live[:, None], inv_contract(np.where(live[:, None], p, 0.0)), 0.0)
  tsdf, weight = np.zeros(N), np.zeros(N)
  color_sum, color_weight = np.zeros((N, 3)), np.zeros(N)
  exempt = np.abs(r - 2) < 1e-5
  bound = np.zeros(N)
  xs = np.abs(x).sum(-1)
  for k in range(K):
    u, v, t, valid = tsdf_ref.project(x, w2c[k], c2p[k if c2p.shape[0] > 1 else 0], camtype, distortion)
    valid &= live
    with np.errstate(invalid='ignore'):
      near_edge = valid & ((np.abs(u - np.round(u)) < tsdf_ref.PIXEL_MARGIN) |
                           (np.abs(v - np.round(v)) < tsdf_ref.PIXEL_MARGIN))
      inside = valid & (u >= 0) & (u < W) & (v >= 0) & (v < H)
    px = np.where(inside, np.floor(np.where(inside, u, 0)), 0).astype(np.int64)
    py = np.where(inside, np.floor(np.where(inside, v, 0)), 0).astype(np.int64)
    dep = depth[k, py, px].astype(np.float64)
    a = acc[k, py, px]
    use = inside & np.isfinite(dep)
    w = np.asarray(w2c[k], np.float64)
    o = -w[:, :3].T @ w[:, 3]
    tt = np.where(use, t, 1.0)
    s = o + (x - o) * (np.where(use, dep, 0) / tt)[:, None]
    dist = np.linalg.norm(contract(s) - p, axis=-1)
    with np.errstate(invalid='ignore'):
      d = np.where(a >= 0.5, np.where(np.where(use, dep, 0) >= tt, dist, -dist), np.inf)
      scale = 1 + np.abs(np.where(use, dep, 0)) + np.abs(tt) + xs + np.abs(o).sum()
      margin = tsdf_ref.DIST_MARGIN * scale
      near_tau = use & np.isfinite(d) & ((np.abs(d + tau) < margin) | (np.abs(d - tau) < margin) |
                                         (np.abs(np.where(use, dep, 0) - tt) < margin))
      use &= ~(d < -tau)
    exempt |= near_edge | near_tau
    sd = np.minimum(np.where(use, d, 0), tau) / tau
    tsdf = np.where(use, (weight * tsdf + sd) / (weight + 1), tsdf)
    weight = weight + use
    pose = np.abs(w).sum()
    err = 64 * EPS32 * (1 + np.abs(p).sum(-1) + (np.abs(s).sum(-1) + xs + np.abs(o).sum()) *
                        (1 + np.abs(np.where(use, dep, 0)) / np.abs(tt)) * (1 + pose)) / tau
    bound = np.maximum(bound, np.where(use & np.isfinite(d), err, 0))
    if rgb is not None:
      col = use & (np.abs(d) <= tau)
      color_sum += np.where(col[:, None], rgb[k, py, px].astype(np.float64), 0)
      color_weight += col
  bound = bound + 8 * (K + 1) * EPS32
  return tsdf, weight, color_sum, color_weight, bound, exempt
