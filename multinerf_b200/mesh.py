"""Triangle meshes from a trained model: the final level's density on a grid, then marching cubes on the GPU.

`extract_mesh(model, bbox, resolution, level)` evaluates `Model.query_density` at the points of a grid of cubic
cells spanning `bbox`, z-slab by z-slab, and extracts the level set `density = level` with
`ops.marching_cubes` (csrc/mesh.cu).  Each grid point is queried as the Gaussian (point, h^2/12 I), the moments of
a uniform cell of side h, so the grid samples the anti-aliased field at the footprint of one cell, as the rays'
IPE does at the footprint of a ray interval.  With `colors=True` each vertex also gets a unit normal from the
density grid's gradient and a colour from `Model.query_radiance`, seen along the inward normal.  `write_ply` stores
the result as binary little-endian PLY.

`extract_mesh_tsdf(model, dataset, bbox, resolution, truncation)` (Config.mesh_method = 'tsdf') meshes what the
renders show instead: it renders every camera of `dataset`, fuses each pixel's median distance into a truncated
signed-distance grid on the same points (`fuse_tsdf`, `ops.tsdf_integrate`, csrc/mesh.cu), and extracts the zero
crossing where the grid was observed.  No density level is chosen; space a camera saw through is carved away; space
no camera saw gives no faces (marching cubes skips cells with an unobserved, NaN, corner); and a vertex's colour is
the mean of the colours rendered for it across the views whose surface lies within the truncation band.
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


MESH_METHODS = ('density', 'tsdf')


def validate_config(bundle):
  """The mesh method of `bundle`'s Config, checked: 'density' or 'tsdf'; the TSDF method needs perspective or fisheye
  views (not NDC) and a truncation of at least one cell, so no cut edge of the fused grid has an unobserved end."""
  config = bundle.config
  if config.mesh_method not in MESH_METHODS:
    raise ValueError(f'Config.mesh_method = {config.mesh_method!r}: want one of {MESH_METHODS}')
  if config.mesh_method == 'tsdf':
    if config.forward_facing:
      raise ValueError("Config.mesh_method = 'tsdf' does not support forward-facing (NDC) scenes")
    if not config.mesh_tsdf_truncation >= 1:
      raise ValueError(f'Config.mesh_tsdf_truncation = {config.mesh_tsdf_truncation!r}: want at least 1 cell')
  return config.mesh_method


def camera_matrices(cameras, device):
  """(worldtocams [N, 3, 4], camtopixs [N or 1, 3, 3]) fp32 on `device` from a dataset's (pixtocams, camtoworlds,
  ...): the inverses, computed in fp64 and rounded once."""
  pixtocams, camtoworlds = (np.asarray(c.detach().cpu() if isinstance(c, torch.Tensor) else c, np.float64)
                            for c in cameras[:2])
  c2w = camtoworlds.reshape(-1, *camtoworlds.shape[-2:])[:, :3, :4]
  rot_t = np.transpose(c2w[:, :, :3], (0, 2, 1))
  w2c = np.concatenate([rot_t, -rot_t @ c2w[:, :, 3:]], -1)
  c2p = np.linalg.inv(pixtocams.reshape(-1, 3, 3))
  to = lambda a: torch.tensor(a, dtype=torch.float32, device=device).contiguous()
  return to(w2c), to(c2p)


def fuse_tsdf(views, cameras, camtype, bbox, resolution, truncation, colors=False, batch=8, device='cuda'):
  """Fuse rendered views into a TSDF on the grid of `bbox` at `resolution` (grid_shape; the points density_grid
  uses).  views: iterable of (cam_idx, depth [H, W], acc [H, W], rgb [H, W, 3] or None) device tensors -- each
  view's median distance (in the units of its rays' directions), opacity and colour; cameras: (pixtocams,
  camtoworlds, distortion_params, pixtocam_ndc) as a dataset holds them; camtype: camera_utils.ProjectionType or its
  value; truncation: the band in cells.  Views are fused `batch` at a time, in order; the result does not depend on
  `batch`.  Returns ((tsdf, weight, color_sum, color_weight), h): [nz, ny, nx] fp32 grids ([nz, ny, nx, 3] for
  color_sum; the colour pair is None without `colors`) and the cell size."""
  from . import camera_utils
  if cameras[3] is not None:
    raise ValueError('TSDF fusion does not support NDC cameras')
  camtype = camera_utils.ProjectionType(camtype.value if hasattr(camtype, 'value') else camtype)
  (nx, ny, nz), h = grid_shape(bbox, resolution)
  w2c, c2p = camera_matrices(cameras, device)
  tau = float(truncation) * h
  z = lambda *sh: torch.zeros(nz, ny, nx, *sh, device=device)
  tsdf, weight = z(), z()
  color_sum, color_weight = (z(3), z()) if colors else (None, None)

  def flush(items):
    idx = torch.tensor([v[0] for v in items], device=device)
    H, W = items[0][1].shape[:2]
    depth = torch.stack([v[1].reshape(H, W) for v in items]).float()
    acc = torch.stack([v[2].reshape(H, W) for v in items]).float()
    rgb = torch.stack([v[3].reshape(H, W, 3) for v in items]).float() if colors else None
    ops.tsdf_integrate((nx, ny, nz), bbox[:3], h, 0 if camtype == camera_utils.ProjectionType.PERSPECTIVE else 1,
                       cameras[2], w2c[idx].contiguous(), c2p if c2p.shape[0] == 1 else c2p[idx].contiguous(),
                       depth, acc, rgb, tau, tsdf, weight, color_sum, color_weight)

  items = []
  for view in views:
    items.append(tuple(view))
    if len(items) == batch:
      flush(items)
      items = []
  if items:
    flush(items)
  return (tsdf, weight, color_sum, color_weight), h


def tsdf_mesh(state, bbox, h, colors=False):
  """Marching cubes on the fused TSDF `state` (fuse_tsdf): the zero crossing of -tsdf (inside > 0, so faces and
  normals point out of the surface), with every point no view observed (weight 0) NaN, so it gives no faces.
  Returns (vertices, faces) in world coordinates, and with `colors` also (normals [V, 3], rgb [V, 3] uint8): each
  vertex's colour is color_sum / color_weight interpolated linearly along its grid edge, rounded as vertex_colors
  rounds."""
  tsdf, weight, color_sum, color_weight = state
  grid = torch.where(weight > 0, -tsdf, torch.full_like(tsdf, float('nan')))
  out = ops.marching_cubes(grid, 0.0, normals=colors)
  del grid
  lo = torch.tensor([float(v) for v in bbox[:3]], device=out[0].device)
  vertices = out[0] * h + lo
  if not colors:
    return vertices, out[1]
  # a vertex lies on a grid edge: its two other coordinates are integers, so the trilinear weights reduce to the
  # linear interpolation between the edge's two ends
  nz, ny, nx = tsdf.shape
  dims = torch.tensor([nx, ny, nz], device=out[0].device)
  base = torch.minimum(out[0].floor().long(), dims - 2).clamp_min(0)
  frac = out[0] - base
  cs = torch.zeros(len(vertices), 3, device=vertices.device)
  cw = torch.zeros(len(vertices), device=vertices.device)
  for corner in range(8):
    off = torch.tensor([corner & 1, corner >> 1 & 1, corner >> 2 & 1], device=vertices.device)
    wgt = torch.where(off.bool(), frac, 1 - frac).prod(-1)
    q = base + off
    p = (q[:, 2] * ny + q[:, 1]) * nx + q[:, 0]
    cs += wgt[:, None] * color_sum.view(-1, 3)[p]
    cw += wgt * color_weight.view(-1)[p]
  rgb = torch.where(cw[:, None] > 0, cs / cw.clamp_min(1e-30)[:, None], torch.zeros_like(cs))
  return vertices, out[1], out[2], (rgb.clamp(0, 1) * 255).round().to(torch.uint8)


def render_views(model, dataset):
  """Yields (cam_idx, distance_median, acc, rgb) of every camera of `dataset`, rendered by `model` with the
  graph-replayed render chunks of train_utils.create_render_fn, GLO zeroed, at train_frac 1 (as eval_lib.render)."""
  from . import models, train_utils
  render_fn = train_utils.create_render_fn(model, use_graph=True)
  for idx in range(dataset.size):
    rays = dataset.generate_ray_batch(idx).rays
    r = models.render_image(lambda rng_, c: render_fn(model.params, 1., None, c), rays, None, model.config,
                            verbose=False)
    yield idx, r['distance_median'], r['acc'], r['rgb']


def extract_mesh_tsdf(model, dataset, bbox, resolution, truncation=3.0, colors=False, batch=8):
  """Config.mesh_method = 'tsdf': render every camera of `dataset` (render_views), fuse the renders (fuse_tsdf, a
  band of `truncation` cells) and mesh the result (tsdf_mesh).  Returns what extract_mesh returns."""
  state, h = fuse_tsdf(render_views(model, dataset), dataset.cameras, dataset.camtype, bbox, resolution, truncation,
                       colors=colors, batch=batch, device=model.device)
  return tsdf_mesh(state, bbox, h, colors=colors)


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
