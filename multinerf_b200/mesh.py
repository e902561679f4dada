"""Triangle meshes from a trained model: the final level's density on a grid, then marching cubes on the GPU.

`extract_mesh(model, bbox, resolution, level)` evaluates `Model.query_density` at the points of a grid of cubic
cells spanning `bbox`, z-slab by z-slab, and extracts the level set `density = level` with
`ops.marching_cubes` (csrc/mesh.cu).  Each grid point is queried as the Gaussian (point, h^2/12 I), the moments of
a uniform cell of side h, so the grid samples the anti-aliased field at the footprint of one cell, as the rays'
IPE does at the footprint of a ray interval.  `write_ply` stores the result as binary little-endian PLY.
"""
import math

import numpy as np
import torch

from . import ops


def default_bbox(bundle):
  """Config.mesh_bbox, or the default box of the scene family: [-1, 1]^3 under the scene contraction (the cube
  around the unit ball, inside which the contraction is the identity), [-1.5, 1.5]^3 for a bounded scene.
  Forward-facing scenes live in NDC space, where no default box means anything: they need Config.mesh_bbox."""
  config = bundle.config
  if config.mesh_bbox is not None:
    bbox = tuple(float(v) for v in config.mesh_bbox)
    if len(bbox) != 6:
      raise ValueError(f'Config.mesh_bbox = {config.mesh_bbox!r}: want (x0, y0, z0, x1, y1, z1)')
    return bbox
  if config.forward_facing:
    raise ValueError('forward-facing (NDC) scenes have no default mesh box: set Config.mesh_bbox')
  r = 1.0 if bundle.nerf_mlp.warp_fn == 'contract' else 1.5
  return (-r, -r, -r, r, r, r)


def grid_shape(bbox, resolution):
  """((nx, ny, nz), h): `resolution` points along the longest side of `bbox`, cubic cells of side h, and as many
  points along the other sides as fit in the box."""
  lo, hi = np.asarray(bbox[:3], np.float64), np.asarray(bbox[3:], np.float64)
  ext = hi - lo
  if resolution < 2 or not np.all(ext > 0):
    raise ValueError(f'mesh grid: resolution {resolution} < 2 or empty box {tuple(bbox)}')
  h = float(ext.max()) / (resolution - 1)
  n = [int(math.floor(e / h + 1e-6)) + 1 for e in ext]
  if min(n) < 2:
    raise ValueError(f'mesh grid: box {tuple(bbox)} is thinner than one cell ({h:g}) along an axis')
  return tuple(n), h


def density_grid(model, bbox, resolution, slab_planes=None):
  """The density of `model`'s final level at the grid points of `bbox` -> (grid [nz, ny, nx] fp32 on the device,
  h).  Evaluated `slab_planes` z-planes at a time (default: about one query chunk of rows per slab)."""
  (nx, ny, nz), h = grid_shape(bbox, resolution)
  dev = model.device
  lo = [float(v) for v in bbox[:3]]
  xs, ys, zs = ((lo[a] + torch.arange(n, device=dev, dtype=torch.float64) * h).float()
                for a, n in enumerate((nx, ny, nz)))
  if slab_planes is None:
    chunk = model.config.render_chunk_size * model.mcfg.num_nerf_samples
    slab_planes = max(1, chunk // (nx * ny))
  var = h * h / 12
  grid = torch.empty(nz, ny, nx, device=dev)
  for z0 in range(0, nz, slab_planes):
    z = zs[z0:z0 + slab_planes]
    pts = torch.stack(torch.broadcast_tensors(xs[None, None, :], ys[None, :, None], z[:, None, None]), -1)
    grid[z0:z0 + z.shape[0]] = model.query_density(pts.reshape(-1, 3), var).view(z.shape[0], ny, nx)
  return grid, h


def extract_mesh(model, bbox, resolution, level, slab_planes=None):
  """(vertices [V, 3] fp32, faces [F, 3] int32) on the device: the surface density = `level` of `model`'s final
  level inside `bbox` (x0, y0, z0, x1, y1, z1), on a grid of `resolution` points along the longest side.
  Vertices are in world coordinates; face normals point from dense to empty space."""
  grid, h = density_grid(model, bbox, resolution, slab_planes)
  vertices, faces = ops.marching_cubes(grid, level)
  lo = torch.tensor([float(v) for v in bbox[:3]], device=vertices.device)
  return vertices * h + lo, faces


def write_ply(path, vertices, faces):
  """Binary little-endian PLY: `float x, y, z` per vertex, `list uchar int vertex_indices` per face."""
  v = np.ascontiguousarray(torch.as_tensor(vertices).detach().cpu().numpy(), dtype='<f4').reshape(-1, 3)
  f = np.ascontiguousarray(torch.as_tensor(faces).detach().cpu().numpy(), dtype='<i4').reshape(-1, 3)
  header = ('ply\nformat binary_little_endian 1.0\n'
            f'element vertex {len(v)}\nproperty float x\nproperty float y\nproperty float z\n'
            f'element face {len(f)}\nproperty list uchar int vertex_indices\nend_header\n')
  rec = np.empty(len(f), dtype=[('n', 'u1'), ('idx', '<i4', (3,))])
  rec['n'] = 3
  rec['idx'] = f
  with open(path, 'wb') as fh:
    fh.write(header.encode('ascii'))
    fh.write(v.tobytes())
    fh.write(rec.tobytes())
