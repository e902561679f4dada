"""Triangle meshes from a trained model: the final level's density on a grid, then marching cubes on the GPU.

`extract_mesh(model, bbox, resolution, level)` evaluates `Model.query_density` at the points of a grid of cubic
cells spanning `bbox`, z-slab by z-slab, and extracts the level set `density = level` with
`ops.marching_cubes` (csrc/mesh.cu).  Each grid point is queried as the Gaussian (point, h^2/12 I), the moments of
a uniform cell of side h, so the grid samples the anti-aliased field at the footprint of one cell, as the rays'
IPE does at the footprint of a ray interval.  With `colors=True` each vertex also gets a unit normal from the
density grid's gradient and a colour from `Model.query_radiance`, seen along the inward normal.  `write_ply` stores
the result as binary little-endian PLY.
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


def extract_mesh(model, bbox, resolution, level, slab_planes=None, colors=False):
  """(vertices [V, 3] fp32, faces [F, 3] int32) on the device: the surface density = `level` of `model`'s final
  level inside `bbox` (x0, y0, z0, x1, y1, z1), on a grid of `resolution` points along the longest side.
  Vertices are in world coordinates; face normals point from dense to empty space.  With `colors`, returns
  (vertices, faces, normals [V, 3] fp32, rgb [V, 3] uint8): unit vertex normals from the density grid's gradient,
  and each vertex's colour from `vertex_colors`."""
  grid, h = density_grid(model, bbox, resolution, slab_planes)
  out = ops.marching_cubes(grid, level, normals=colors)
  del grid
  lo = torch.tensor([float(v) for v in bbox[:3]], device=out[0].device)
  vertices = out[0] * h + lo
  if not colors:
    return vertices, out[1]
  # cubic cells: the grid's normals are the world's
  return vertices, out[1], out[2], vertex_colors(model, vertices, out[2], h * h / 12)


def vertex_colors(model, vertices, normals, var):
  """rgb [V, 3] uint8 of each vertex: `model.query_radiance` at the Gaussian (vertex, var * I) seen along -normal,
  the surface viewed head-on from outside, as round(clip(rgb, 0, 1) * 255).  A RawNeRF model's colours are its
  linear raw values, clipped as they are.  var: the footprint the density was sampled at (h^2 / 12 for grid cells
  of side h)."""
  _, rgb = model.query_radiance(vertices, var, -normals)
  return (rgb.clamp(0, 1) * 255).round().to(torch.uint8)


def write_ply(path, vertices, faces, normals=None, colors=None):
  """Binary little-endian PLY: `float x, y, z` per vertex, then `float nx, ny, nz` when `normals` and
  `uchar red, green, blue` when `colors` (uint8) are given, and `list uchar int vertex_indices` per face."""
  def host(t, dtype):
    return np.ascontiguousarray(torch.as_tensor(t).detach().cpu().numpy(), dtype=dtype).reshape(-1, 3)
  v = host(vertices, '<f4')
  f = host(faces, '<i4')
  props = [('x', '<f4'), ('y', '<f4'), ('z', '<f4')]
  cols = [v]
  if normals is not None:
    props += [('nx', '<f4'), ('ny', '<f4'), ('nz', '<f4')]
    cols.append(host(normals, '<f4'))
  if colors is not None:
    props += [('red', 'u1'), ('green', 'u1'), ('blue', 'u1')]
    cols.append(host(colors, 'u1'))
  ply_type = {'<f4': 'float', 'u1': 'uchar'}
  header = ('ply\nformat binary_little_endian 1.0\n'
            f'element vertex {len(v)}\n' + ''.join(f'property {ply_type[t]} {n}\n' for n, t in props) +
            f'element face {len(f)}\nproperty list uchar int vertex_indices\nend_header\n')
  vrec = np.empty(len(v), dtype=props)
  for c, block in enumerate(cols):
    for j in range(3):
      vrec[props[3 * c + j][0]] = block[:, j]
  rec = np.empty(len(f), dtype=[('n', 'u1'), ('idx', '<i4', (3,))])
  rec['n'] = 3
  rec['idx'] = f
  with open(path, 'wb') as fh:
    fh.write(header.encode('ascii'))
    fh.write(vrec.tobytes())
    fh.write(rec.tobytes())
