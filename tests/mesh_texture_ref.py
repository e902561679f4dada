"""fp64 numpy restatement of the texture atlas of csrc/mesh.cu (mnrf_mesh_texture_raster, include/mnrf.h): the cell
grid, each face's chart, texel ownership, the clamped barycentrics of each texel centre, and each texel's surface
point and normal (the unit interpolated vertex normal, else the face's normal, else (0, 0, 1))."""
import math

import numpy as np

EPS32 = 2.0 ** -24


def atlas(num_faces, size):
  """(n, c): cells per row, texels per cell side.  ValueError when a cell would be narrower than 4 texels."""
  cells = (num_faces + 1) // 2
  n = math.isqrt(cells - 1) + 1 if cells else 0
  c = size // n if n else size
  if c < 4:
    raise ValueError(f'{num_faces} faces do not fit a {size} x {size} atlas')
  return n, c


def capacity(size):
  return 2 * (size // 4) ** 2


def chart(f, n, c):
  """(x0, y0, o, d) of faces f [...]: the cell's first texel in the atlas, and corners o, o + (d, 0), o + (0, d) in
  the cell's texel units."""
  f = np.asarray(f, np.int64)
  k, b = f >> 1, f & 1
  return (k % n) * c, (k // n) * c, np.where(b, c - 0.5, 0.5), np.where(b, 2.0 - c, c - 3.0)


def uv(num_faces, size):
  """[F, 3, 2] corner positions in atlas texel units."""
  n, c = atlas(num_faces, size)
  x0, y0, o, d = chart(np.arange(num_faces), n, c)
  u0, v0 = x0 + o, y0 + o
  return np.stack([np.stack([u0, v0], -1), np.stack([u0 + d, v0], -1), np.stack([u0, v0 + d], -1)], 1)


def texels(num_faces, size):
  """For each texel of the used cells, cell-major and row-major within a cell: (owner face [T], i [T], j [T],
  texel_index [T])."""
  n, c = atlas(num_faces, size)
  cells = (num_faces + 1) // 2
  t = np.arange(cells * c * c, dtype=np.int64)
  k, r = t // (c * c), t % (c * c)
  j, i = r // c, r % c
  owner = 2 * k + ((i + j + 2 > c) & (2 * k + 1 < num_faces))
  x0, y0, _, _ = chart(owner, n, c)
  return owner, i, j, (y0 + j) * size + x0 + i


def barycentrics(num_faces, size):
  """[T, 3] fp64 barycentrics of each texel centre in its owner's chart, clamped to the triangle."""
  n, c = atlas(num_faces, size)
  owner, i, j, _ = texels(num_faces, size)
  _, _, o, d = chart(owner, n, c)
  a = np.maximum((i + 0.5 - o) / d, 0.0)
  b = np.maximum((j + 0.5 - o) / d, 0.0)
  over = a + b > 1
  t = np.clip((a - b + 1) * 0.5, 0.0, 1.0)
  a, b = np.where(over, t, a), np.where(over, 1 - t, b)
  return np.stack([1 - a - b, a, b], -1)


def _unit(v):
  n = np.linalg.norm(v, axis=-1, keepdims=True)
  ok = n[..., 0] > 0
  return np.where(ok[..., None], v / np.where(n > 0, n, 1), 0.0), ok


def raster(vertices, faces, normals, size):
  """(uv [F, 3, 2], texel_index [T], points [T, 3], normals [T, 3], weights [T, 3], owner [T]) in fp64."""
  v, f, nv = (np.asarray(a, np.float64) for a in (vertices, faces, normals))
  f = f.astype(np.int64)
  F = len(f)
  owner, _, _, index = texels(F, size)
  w = barycentrics(F, size)
  corners = f[owner]
  p = v[corners]                                   # [T, 3 corners, 3]
  points = (w[:, :, None] * p).sum(1)
  n, ok = _unit((w[:, :, None] * nv[corners]).sum(1))
  g, gok = _unit(np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]))
  n = np.where(ok[:, None], n, np.where(gok[:, None], g, np.array([0.0, 0.0, 1.0])))
  return uv(F, size), index, points, n, w, owner


def point_bound(vertices, faces, owner):
  """Per-element bound on |kernel point - reference point|: 16 eps32 sum_i |p_i| (weights to a few ulps of 1, three
  products and two sums in fp32)."""
  p = np.abs(np.asarray(vertices, np.float64)[np.asarray(faces, np.int64)[owner]])
  return 16 * EPS32 * p.sum(1)


def normal_bound(normals, faces, owner, w):
  """Per-element bound on |kernel normal - reference normal| where the reference takes the interpolated normal: the
  error of the unnormalised sum (as point_bound) over its length, twice, plus the normalisation's roundings.  inf
  where the interpolated sum is zero or too short to fix a direction."""
  nv = np.asarray(normals, np.float64)[np.asarray(faces, np.int64)[owner]]
  s = (w[:, :, None] * nv).sum(1)
  length = np.linalg.norm(s, axis=-1)
  err = 16 * EPS32 * np.abs(nv).sum(1).max(-1)
  with np.errstate(divide='ignore', invalid='ignore'):
    b = 4 * err / length + 8 * EPS32
  return np.where(length > 8 * err, b, np.inf)[:, None]


def bilinear_texels(u, v):
  """The texels (x [N, 4], y [N, 4]) a bilinear sample at (u, v) in texel units reads with a nonzero weight (-1 where
  fewer than four)."""
  fx, fy = u - 0.5, v - 0.5
  x0, y0 = np.floor(fx).astype(np.int64), np.floor(fy).astype(np.int64)
  tx, ty = fx - x0, fy - y0
  xs = np.stack([x0, x0 + 1, x0, x0 + 1], -1)
  ys = np.stack([y0, y0, y0 + 1, y0 + 1], -1)
  wt = np.stack([(1 - tx) * (1 - ty), tx * (1 - ty), (1 - tx) * ty, tx * ty], -1)
  return np.where(wt > 0, xs, -1), np.where(wt > 0, ys, -1)


def bilinear_sample(texture, u, v):
  """texture [S, S, C] sampled bilinearly at (u, v) in texel units (texel (x, y) centred at (x + 0.5, y + 0.5)),
  clamped to the edge -> [N, C] fp64."""
  S = texture.shape[0]
  t = np.asarray(texture, np.float64)
  fx, fy = u - 0.5, v - 0.5
  x0, y0 = np.floor(fx).astype(np.int64), np.floor(fy).astype(np.int64)
  tx, ty = (fx - x0)[:, None], (fy - y0)[:, None]
  at = lambda x, y: t[np.clip(y, 0, S - 1), np.clip(x, 0, S - 1)]
  return ((1 - tx) * (1 - ty) * at(x0, y0) + tx * (1 - ty) * at(x0 + 1, y0) + (1 - tx) * ty * at(x0, y0 + 1) +
          tx * ty * at(x0 + 1, y0 + 1))
