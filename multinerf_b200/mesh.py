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

Either method can clean the mesh (`clean_mesh`) and then simplify it to a face budget by quadric edge collapse
(`simplify_mesh`) before any colour is computed, and then bake the colour into a texture atlas (`bake_texture`,
`texture_size`) that `write_obj` stores as a textured OBJ with its MTL and PNG.

Both methods can also work in the contracted space of an unbounded scene (`space='contracted'`,
Config.mesh_space): the grid then spans the model's contracted coordinates (coord.contract; the open ball of radius
2 holds the whole world), so the background becomes faces at the resolution the model itself has there.  Grid points
with |p| >= 2 have no world preimage: they are NaN and never queried.  The density grid holds the density per unit
of contracted length (Model.query_density(contracted=True)), the TSDF measures distances in contracted space
(ops.tsdf_integrate(contracted=True)), cleaning projects world positions, simplification runs on the contracted
mesh, and the result is mapped to world space (ops.mesh_uncontract: vertices, and normals through the contraction's
Jacobian) before colours are queried.  Outputs are always in world coordinates.

`evaluate_mesh` (Config.mesh_eval) scores the result against the test views: it traces every test pixel's ray into
the mesh on the GPU (`ops.mesh_bvh`, `ops.mesh_trace`, csrc/mesh_trace.cu), shades the hits (`render_mesh`) and
compares them with the test images and with the NeRF's own depth and opacity on the same rays (`mesh_metrics`).
"""
import math
import os
from typing import NamedTuple

import numpy as np
import torch

from . import ops


MESH_SPACES = ('world', 'contracted')


def default_bbox(bundle):
  """Config.mesh_bbox, or the default box of the scene family: [-1, 1]^3 under the scene contraction (the cube
  around the unit ball, inside which the contraction is the identity), [-1.5, 1.5]^3 for a bounded scene.
  Forward-facing scenes live in NDC space, where no default box means anything: they need Config.mesh_bbox.
  With Config.mesh_space = 'contracted' the box is in contracted coordinates, and the default [-2, 2]^3 holds all of
  contracted space."""
  config = bundle.config
  _check_space(bundle)
  if config.mesh_bbox is not None:
    bbox = tuple(float(v) for v in config.mesh_bbox)
    if len(bbox) != 6:
      raise ValueError(f'Config.mesh_bbox = {config.mesh_bbox!r}: want (x0, y0, z0, x1, y1, z1)')
    return bbox
  if config.forward_facing:
    raise ValueError('forward-facing (NDC) scenes have no default mesh box: set Config.mesh_bbox')
  r = 2.0 if config.mesh_space == 'contracted' else 1.0 if bundle.nerf_mlp.warp_fn == 'contract' else 1.5
  return (-r, -r, -r, r, r, r)


def _check_space(bundle):
  """Config.mesh_space, checked: 'world' or 'contracted'; 'contracted' needs the final MLP under the scene
  contraction and a scene that is not forward-facing (NDC)."""
  config = bundle.config
  if config.mesh_space not in MESH_SPACES:
    raise ValueError(f'Config.mesh_space = {config.mesh_space!r}: want one of {MESH_SPACES}')
  if config.mesh_space == 'contracted':
    if bundle.nerf_mlp.warp_fn != 'contract':
      raise ValueError("Config.mesh_space = 'contracted' needs the scene contraction (NerfMLP.warp_fn = "
                       "@coord.contract)")
    if config.forward_facing:
      raise ValueError("Config.mesh_space = 'contracted' does not support forward-facing (NDC) scenes")
  return config.mesh_space


def _contracted(space):
  if space not in MESH_SPACES:
    raise ValueError(f'mesh space {space!r}: want one of {MESH_SPACES}')
  return space == 'contracted'


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


def density_grid(model, bbox, resolution, slab_planes=None, space='world'):
  """The density of `model`'s final level at the grid points of `bbox` -> (grid [nz, ny, nx] fp32 on the device,
  h).  Evaluated `slab_planes` z-planes at a time (default: about one query chunk of rows per slab).
  space 'contracted': the grid lies in contracted coordinates and holds Model.query_density(contracted=True), the
  density per unit of contracted length; points with |p| >= 2 are NaN and are not queried."""
  contracted = _contracted(space)
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
    if not contracted:
      grid[z0:z0 + z.shape[0]] = model.query_density(pts.reshape(-1, 3), var).view(z.shape[0], ny, nx)
      continue
    pts = pts.reshape(-1, 3)
    inside = pts.double().square().sum(-1) < 4
    slab = torch.full((pts.shape[0],), float('nan'), device=dev)
    slab[inside] = model.query_density(pts[inside], var, contracted=True)
    grid[z0:z0 + z.shape[0]] = slab.view(z.shape[0], ny, nx)
  return grid, h


def extract_mesh(model, bbox, resolution, level, slab_planes=None, colors=False, keep_components=0, min_views=0,
                 dataset=None, stats=None, target_faces=0, texture_size=0, before_texture=None, space='world'):
  """(vertices [V, 3] fp32, faces [F, 3] int32) on the device: the surface density = `level` of `model`'s final
  level inside `bbox` (x0, y0, z0, x1, y1, z1), on a grid of `resolution` points along the longest side.
  Vertices are in world coordinates; face normals point from dense to empty space.  With `colors`, returns
  (vertices, faces, normals [V, 3] fp32, rgb [V, 3] uint8): unit vertex normals from the density grid's gradient,
  and each vertex's colour from `vertex_colors`.  `keep_components`, `min_views` (with the training cameras of
  `dataset`) and `stats`: clean_mesh, applied before the colours are queried.  target_faces: then simplify_mesh
  (its counts go to `stats` too), the normals carried along.  texture_size > 0: the normals are computed with or
  without `colors`, and the colour is baked into a texture_size x texture_size atlas (bake_texture, each texel's
  colour by `vertex_colors` at its surface point and normal); returns (vertices, faces, normals, rgb or None, uv,
  texture).  before_texture: called with (vertices, faces, normals, rgb or None) before the texture is baked, so a
  caller can save the mesh first (bake_texture raises ValueError when the atlas cannot hold the faces).
  space 'contracted': `bbox` is in contracted coordinates and `level` is a density per unit of contracted length
  (density_grid); the mesh is cleaned (min_views on its world positions) and simplified in contracted space, then
  mapped to world space (ops.mesh_uncontract), where every output lies.  Colours are queried at the contracted
  points, the world normals giving the view directions; the atlas is laid out on the contracted mesh."""
  contracted = _contracted(space)
  grid, h = density_grid(model, bbox, resolution, slab_planes, space=space)
  out = ops.marching_cubes(grid, level, normals=colors or texture_size > 0)
  del grid
  lo = torch.tensor([float(v) for v in bbox[:3]], device=out[0].device)
  vertices, faces, *normals = _clean_in_space(out[0] * h + lo, *out[1:], contracted=contracted,
                                              **_clean_args(keep_components, min_views, dataset, stats))
  vertices, faces, *normals = simplify_mesh(vertices, faces, *normals, target_faces=target_faces, stats=stats)
  if contracted and target_faces:
    vertices = clamp_to_ball(vertices)
  var = h * h / 12
  query = lambda p, n: vertex_colors(model, p, n, var, contracted=contracted)
  # cubic cells: the grid's normals are the world's (in contracted space, after _to_world)
  world, *wnormals = _to_world(vertices, *normals) if contracted else (vertices, *normals)
  if not texture_size:
    if not colors:
      return world, faces
    return world, faces, wnormals[0], query(vertices, wnormals[0])
  rgb = query(vertices, wnormals[0]) if colors else None
  if contracted:
    return _with_texture(world, faces, wnormals[0], rgb, texture_size, before_texture,
                         lambda p, n: query(p, ops.mesh_uncontract(p, n)[1]), chart=(vertices, normals[0]))
  return _with_texture(vertices, faces, normals[0], rgb, texture_size, before_texture, query)


CONTRACTED_MAX_RADIUS = 2 - 2 ** -12


def clamp_to_ball(vertices):
  """Contracted vertices [V, 3] with every radius above CONTRACTED_MAX_RADIUS (2 - 2^-12, a world radius of about
  2048) scaled back to it; the others unchanged.  A quadric collapse position may lie off the surface it
  simplifies, and on a convex surface near |p| = 2 that can be outside the ball, where no world point exists.
  Marching cubes never puts a vertex there, since its vertices lie on grid edges between points with |p| < 2."""
  r = vertices.double().norm(dim=-1, keepdim=True)
  far = r > CONTRACTED_MAX_RADIUS
  return torch.where(far, (vertices.double() * (CONTRACTED_MAX_RADIUS / r.clamp_min(1))).float(), vertices)


def _to_world(vertices, normals=None):
  """A contracted mesh's vertices (and normals) in world space, as a tuple: ops.mesh_uncontract."""
  if normals is None:
    return (ops.mesh_uncontract(vertices),)
  return ops.mesh_uncontract(vertices, normals)


def _clean_in_space(vertices, faces, *per_vertex, contracted=False, **clean_args):
  """clean_mesh of a mesh in grid coordinates.  min_views projects world positions into the views, so a contracted
  mesh is cleaned on its world vertices with its contracted ones riding along; components are topological."""
  if not contracted or not clean_args.get('min_views'):
    return clean_mesh(vertices, faces, *per_vertex, **clean_args)
  _, faces, vertices, *per_vertex = clean_mesh(ops.mesh_uncontract(vertices), faces, vertices, *per_vertex,
                                               **clean_args)
  return (vertices, faces, *per_vertex)


def _with_texture(vertices, faces, normals, rgb, texture_size, before_texture, color_fn, chart=None):
  """(vertices, faces, normals, rgb, uv, texture): the mesh, and bake_texture's atlas of it by `color_fn`, after
  before_texture(vertices, faces, normals, rgb) when given.  chart: (vertices, normals) of the same faces to lay the
  atlas out on and to give color_fn its texel points and normals (the contracted mesh), instead of the mesh's own."""
  if before_texture is not None:
    before_texture(vertices, faces, normals, rgb)
  cv, cn = chart if chart is not None else (vertices, normals)
  return (vertices, faces, normals, rgb) + bake_texture(cv, faces, cn, texture_size, color_fn)


def bake_texture(vertices, faces, normals, size, color_fn):
  """The colour of a mesh baked into a size x size texture atlas on the device -> (uv [F, 3, 2] fp32, each face
  corner's position in texel units, u along a row and v down the rows; texture [size, size, 3] uint8, row 0 on top).
  vertices [V, 3], faces [F, 3] int32, normals [V, 3]: the mesh and its unit vertex normals.  Each face gets its own
  right-triangle chart, two per square cell of c x c texels, c >= 4 (ops.mesh_texture_raster, csrc/mesh.cu); every
  texel of a used cell is given the colour of its face at the texel centre's nearest point of the chart:
  color_fn(points [T, 3], normals [T, 3]) -> uint8 [T, 3] at those surface points and unit interpolated normals.
  Texels of unused cells stay 0.  Raises ValueError when the atlas cannot hold the faces."""
  uv, index, points, tnormals = ops.mesh_texture_raster(vertices, faces.int().contiguous(), normals.contiguous(),
                                                        size)
  texture = torch.zeros(size * size, 3, device=vertices.device, dtype=torch.uint8)
  if index.shape[0]:
    texture[index.long()] = color_fn(points, tnormals)
  return uv, texture.view(size, size, 3)


def vertex_colors(model, vertices, normals, var, contracted=False):
  """rgb [V, 3] uint8 of each vertex: `model.query_radiance` at the Gaussian (vertex, var * I) seen along -normal,
  the surface viewed head-on from outside, as round(clip(rgb, 0, 1) * 255).  A RawNeRF model's colours are its
  linear raw values, clipped as they are.  var: the footprint the density was sampled at (h^2 / 12 for grid cells
  of side h).  contracted: vertices and var in contracted space, normals in world space
  (Model.query_radiance(contracted=True))."""
  _, rgb = model.query_radiance(vertices, var, -normals, **({'contracted': True} if contracted else {}))
  return (rgb.clamp(0, 1) * 255).round().to(torch.uint8)


MESH_METHODS = ('density', 'tsdf')


def validate_config(bundle):
  """The mesh method of `bundle`'s Config, checked: 'density' or 'tsdf'; the TSDF method needs perspective or fisheye
  views (not NDC) and a truncation of at least one cell, so no cut edge of the fused grid has an unobserved end.
  The cleaning and simplification options must not be negative, and mesh_min_views projects into the views, so it
  needs them not NDC either.  mesh_texture_size is 0 (off) or in [4, 16384].  mesh_eval traces world-space
  meshes along the test rays, so it needs them not NDC either.  mesh_space is 'world' or 'contracted', the latter
  only under the scene contraction and not for NDC scenes."""
  config = bundle.config
  _check_space(bundle)
  if config.mesh_method not in MESH_METHODS:
    raise ValueError(f'Config.mesh_method = {config.mesh_method!r}: want one of {MESH_METHODS}')
  for name in ('mesh_keep_components', 'mesh_min_views', 'mesh_target_faces'):
    if getattr(config, name) < 0:
      raise ValueError(f'Config.{name} = {getattr(config, name)!r}: want 0 (off) or more')
  lo, hi = ops.TEXTURE_SIZES
  if config.mesh_texture_size != 0 and not lo <= config.mesh_texture_size <= hi:
    raise ValueError(f'Config.mesh_texture_size = {config.mesh_texture_size!r}: want 0 (off) or [{lo}, {hi}]')
  if config.mesh_min_views > 0 and config.forward_facing:
    raise ValueError('Config.mesh_min_views does not support forward-facing (NDC) scenes')
  if config.mesh_eval and config.forward_facing:
    raise ValueError('Config.mesh_eval does not support forward-facing (NDC) scenes: the mesh is in world space and '
                     'NDC rays are not')
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


def fuse_tsdf(views, cameras, camtype, bbox, resolution, truncation, colors=False, batch=8, device='cuda',
              space='world'):
  """Fuse rendered views into a TSDF on the grid of `bbox` at `resolution` (grid_shape; the points density_grid
  uses).  views: iterable of (cam_idx, depth [H, W], acc [H, W], rgb [H, W, 3] or None) device tensors -- each
  view's median distance (in the units of its rays' directions), opacity and colour; cameras: (pixtocams,
  camtoworlds, distortion_params, pixtocam_ndc) as a dataset holds them; camtype: camera_utils.ProjectionType or its
  value; truncation: the band in cells.  Views are fused `batch` at a time, in order; the result does not depend on
  `batch`.  Returns ((tsdf, weight, color_sum, color_weight), h): [nz, ny, nx] fp32 grids ([nz, ny, nx, 3] for
  color_sum; the colour pair is None without `colors`) and the cell size.  space 'contracted': the grid, and so
  the cell size and the band, are in contracted coordinates (ops.tsdf_integrate(contracted=True)); points with
  |p| >= 2 stay unobserved."""
  from . import camera_utils
  contracted = _contracted(space)
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
                       depth, acc, rgb, tau, tsdf, weight, color_sum, color_weight, contracted=contracted)

  items = []
  for view in views:
    items.append(tuple(view))
    if len(items) == batch:
      flush(items)
      items = []
  if items:
    flush(items)
  return (tsdf, weight, color_sum, color_weight), h


def tsdf_mesh(state, bbox, h, colors=False, clean_args=None, target_faces=0, stats=None, texture_size=0,
              before_texture=None, space='world'):
  """Marching cubes on the fused TSDF `state` (fuse_tsdf): the zero crossing of -tsdf (inside > 0, so faces and
  normals point out of the surface), with every point no view observed (weight 0) NaN, so it gives no faces.
  Returns (vertices, faces) in world coordinates, and with `colors` also (normals [V, 3], rgb [V, 3] uint8): each
  vertex's colour is color_sum / color_weight interpolated linearly along its grid edge, rounded as vertex_colors
  rounds.  clean_args: keyword arguments of clean_mesh, applied before the colours are interpolated.
  target_faces: then simplify_mesh (counts to `stats`); a simplified vertex no longer lies on a grid edge, so its
  colour is interpolated trilinearly at (vertex - lo) / h, clamped to the grid (tsdf_colors).  texture_size > 0
  (the state must hold the colour grid): the normals are computed with or without `colors` and the colour is baked
  into a texture atlas, each texel's by tsdf_colors at its surface point; returns and calls `before_texture` as
  extract_mesh does.  space 'contracted': the state was fused in contracted space (fuse_tsdf); the mesh is cleaned
  and simplified there, its colours interpolated there, and it is returned in world space as extract_mesh returns
  it."""
  contracted = _contracted(space)
  tsdf, weight, color_sum, color_weight = state
  if texture_size and color_sum is None:
    raise ValueError('tsdf_mesh: texture_size needs the fused colour grid (fuse_tsdf with colors=True)')
  grid = torch.where(weight > 0, -tsdf, torch.full_like(tsdf, float('nan')))
  out = ops.marching_cubes(grid, 0.0, normals=colors or texture_size > 0)
  del grid
  lo = torch.tensor([float(v) for v in bbox[:3]], device=out[0].device)
  simplify = target_faces > 0
  # without simplification the grid-unit vertices ride along as a per-vertex array: the colours are interpolated
  # from them
  ride = (out[0],) if colors and not simplify else ()
  vertices, faces, *per = _clean_in_space(out[0] * h + lo, out[1], *out[2:], *ride, contracted=contracted,
                                          **(clean_args or {}))
  if simplify:
    vertices, faces, *per = simplify_mesh(vertices, faces, *per, target_faces=target_faces, stats=stats)
    if contracted:
      vertices = clamp_to_ball(vertices)
  elif stats is not None:
    simplify_mesh(vertices, faces, target_faces=0, stats=stats)
  if not colors and not texture_size:
    return (_to_world(vertices)[0] if contracted else vertices), faces
  rgb = None
  if colors:
    # unsimplified, a vertex lies on a grid edge: its two other coordinates are integers, so the trilinear weights
    # reduce to the linear interpolation between the edge's two ends
    rgb = (tsdf_colors(color_sum, color_weight, (vertices - lo) / h) if simplify else
           tsdf_colors(color_sum, color_weight, per[1], clamp=False))
  color_fn = lambda p, n: tsdf_colors(color_sum, color_weight, (p - lo) / h)
  if contracted:
    world, wnormals = _to_world(vertices, per[0])
    if not texture_size:
      return world, faces, wnormals, rgb
    return _with_texture(world, faces, wnormals, rgb, texture_size, before_texture, color_fn,
                         chart=(vertices, per[0]))
  if not texture_size:
    return vertices, faces, per[0], rgb
  return _with_texture(vertices, faces, per[0], rgb, texture_size, before_texture, color_fn)


def tsdf_colors(color_sum, color_weight, gv, clamp=True):
  """rgb [N, 3] uint8 at points gv [N, 3] in grid units (x, y, z) of the fused colour grids color_sum [nz, ny, nx, 3]
  and color_weight [nz, ny, nx] (fuse_tsdf): both interpolated trilinearly, their quotient (0 where no colour was
  fused nearby) rounded as vertex_colors rounds.  clamp: first clamp gv to the grid, [0, n - 1] along each axis;
  without it gv must lie there already."""
  nz, ny, nx = color_weight.shape
  dims = torch.tensor([nx, ny, nz], device=gv.device)
  if clamp:
    gv = torch.minimum(gv.clamp_min(0), dims - 1)
  base = torch.minimum(gv.floor().long(), dims - 2).clamp_min(0)
  frac = gv - base
  cs = torch.zeros(len(gv), 3, device=gv.device)
  cw = torch.zeros(len(gv), device=gv.device)
  for corner in range(8):
    off = torch.tensor([corner & 1, corner >> 1 & 1, corner >> 2 & 1], device=gv.device)
    wgt = torch.where(off.bool(), frac, 1 - frac).prod(-1)
    q = base + off
    p = (q[:, 2] * ny + q[:, 1]) * nx + q[:, 0]
    cs += wgt[:, None] * color_sum.view(-1, 3)[p]
    cw += wgt * color_weight.view(-1)[p]
  rgb = torch.where(cw[:, None] > 0, cs / cw.clamp_min(1e-30)[:, None], torch.zeros_like(cs))
  return (rgb.clamp(0, 1) * 255).round().to(torch.uint8)


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


def extract_mesh_tsdf(model, dataset, bbox, resolution, truncation=3.0, colors=False, batch=8, keep_components=0,
                      min_views=0, stats=None, target_faces=0, texture_size=0, before_texture=None, space='world'):
  """Config.mesh_method = 'tsdf': render every camera of `dataset` (render_views), fuse the renders (fuse_tsdf, a
  band of `truncation` cells) and mesh the result (tsdf_mesh).  Returns what extract_mesh returns.
  `keep_components`, `min_views` (against the cameras of `dataset`) and `stats`: clean_mesh, applied before the
  colours are interpolated; `target_faces`: then simplify_mesh; `texture_size`, `before_texture`: then the texture
  (tsdf_mesh), the fusion keeping its colour grid for it.  space: the grid's space (fuse_tsdf, tsdf_mesh)."""
  state, h = fuse_tsdf(render_views(model, dataset), dataset.cameras, dataset.camtype, bbox, resolution, truncation,
                       colors=colors or texture_size > 0, batch=batch, device=model.device, space=space)
  return tsdf_mesh(state, bbox, h, colors=colors, clean_args=_clean_args(keep_components, min_views, dataset, stats),
                   target_faces=target_faces, stats=stats, texture_size=texture_size, before_texture=before_texture,
                   space=space)


def clean_mesh(vertices, faces, *per_vertex, keep_components=0, min_views=0, cameras=None, camtype=None,
               image_size=None, stats=None):
  """Drops what a user would cut from a raw marching-cubes mesh first, on the device.  Returns (vertices, faces,
  *per_vertex) in the shape it was given.

  min_views > 0: a vertex counts a view when it lands on that view's image (ops.points_view_count: the pixel rule of
  the TSDF fusion; frustum only, no occlusion); vertices with fewer than `min_views` views and every face using one
  are dropped.  cameras: (pixtocams, camtoworlds, distortion_params, pixtocam_ndc) as a dataset holds them;
  camtype: camera_utils.ProjectionType or its value; image_size: (height, width).
  keep_components > 0: of the connected components of the remaining faces (ops.mesh_components), ranked by face
  count, largest first, ties to the smaller minimum vertex index, only the first `keep_components` are kept.
  A vertex is kept if and only if a kept face uses it; vertices and faces keep their relative order, face indices
  are renumbered, and each per-vertex array [V, ...] (normals, colours) follows its vertices.  With both options
  at 0 the inputs come back untouched and nothing is launched.  stats: a dict, given the counts of vertices,
  faces and components removed (components: those the ranking dropped)."""
  if keep_components < 0 or min_views < 0:
    raise ValueError(f'clean_mesh: keep_components = {keep_components}, min_views = {min_views}: want >= 0')
  if stats is not None:
    stats.update(vertices_removed=0, faces_removed=0, components_removed=0)
  if not keep_components and not min_views:
    return (vertices, faces, *per_vertex)
  V = vertices.shape[0]
  keep_face = torch.ones(faces.shape[0], device=faces.device, dtype=torch.bool)
  if min_views:
    if cameras is None or camtype is None or image_size is None:
      raise ValueError('clean_mesh: min_views needs the cameras, camtype and image_size')
    from . import camera_utils
    if cameras[3] is not None:
      raise ValueError('clean_mesh: min_views does not support NDC cameras')
    camtype = camera_utils.ProjectionType(camtype.value if hasattr(camtype, 'value') else camtype)
    w2c, c2p = camera_matrices(cameras, vertices.device)
    counts = ops.points_view_count(vertices, 0 if camtype == camera_utils.ProjectionType.PERSPECTIVE else 1,
                                   cameras[2], w2c, c2p, *image_size)
    keep_face = (counts >= min_views)[faces.long()].all(-1)
  if keep_components:
    culled = faces[keep_face]
    labels = ops.mesh_components(culled, V)
    comp = labels[culled[:, 0].long()].long()                  # a face's component: its first corner's label
    size = torch.bincount(comp, minlength=V)
    ids = torch.nonzero(size).view(-1)                         # components with faces, by minimum vertex index
    order = torch.sort(size[ids], descending=True, stable=True).indices
    keep_label = torch.zeros(V, device=faces.device, dtype=torch.bool)
    keep_label[ids[order[:keep_components]]] = True
    keep_face[keep_face.clone()] = keep_label[comp]
    if stats is not None:
      stats['components_removed'] = max(0, len(ids) - keep_components)
  kept = faces[keep_face]
  out = _drop_unused(vertices, kept, *per_vertex)
  if stats is not None:
    stats.update(vertices_removed=V - out[0].shape[0], faces_removed=faces.shape[0] - kept.shape[0])
  return out


def _drop_unused(vertices, faces, *per_vertex):
  """(vertices, faces, *per_vertex) without the vertices no face uses: the rest keep their order, face indices are
  renumbered and each per-vertex array follows its vertices."""
  used = torch.zeros(vertices.shape[0], device=faces.device, dtype=torch.bool)
  used[faces.view(-1).long()] = True
  new_index = (torch.cumsum(used, 0, dtype=torch.int32) - 1)
  return (vertices[used], new_index[faces.long()], *(t[used] for t in per_vertex))


class Topology(NamedTuple):
  """The adjacency of a triangle mesh that one round of simplify_mesh reads (csrc/mesh.cu, include/mnrf.h)."""
  edges: torch.Tensor       # [E, 2] int32: unique undirected edges (a, b), a < b, sorted by (a, b)
  edge_off: torch.Tensor    # [E + 1] int64: faces of edge e at edge_face[edge_off[e]:edge_off[e + 1]]
  edge_face: torch.Tensor   # [3 F] int32, ascending within an edge
  vf_off: torch.Tensor      # [V + 1] int64: faces at vertex v at vf_face[vf_off[v]:vf_off[v + 1]]
  vf_face: torch.Tensor     # [3 F] int32, ascending within a vertex


def mesh_topology(faces, num_vertices):
  """Topology of faces [F, 3] int32 on `num_vertices` vertices: stable torch sorts of the corners' edge keys
  min * V + max and of their vertices, so faces come out in face order within an edge and within a vertex."""
  # temporaries are freed as soon as they are used: at 155 M faces each int64 corner array takes 3.7 GB
  corner = faces.view(-1)
  other = faces[:, [1, 2, 0]].reshape(-1)                 # corner k's edge runs to corner k + 1
  key = torch.minimum(corner, other).long() * num_vertices + torch.maximum(corner, other)
  del other
  skey, perm = torch.sort(key, stable=True)
  del key
  edge_face = (perm // 3).int()
  del perm
  uniq, counts = torch.unique_consecutive(skey, return_counts=True)
  del skey
  zero = torch.zeros(1, device=faces.device, dtype=torch.int64)
  edges = torch.stack([uniq // num_vertices, uniq % num_vertices], 1).int()
  del uniq
  edge_off = torch.cat([zero, torch.cumsum(counts, 0)])
  del counts
  vf_face = (torch.sort(corner, stable=True).indices // 3).int()
  vf_off = torch.cat([zero, torch.cumsum(torch.bincount(corner, minlength=num_vertices), 0)])
  return Topology(edges, edge_off, edge_face, vf_off, vf_face)


def boundary_edges(topo, num_vertices):
  """(edges [B, 2] int32, face [B] int32, vb_off [V + 1] int64, vb_edge [2 B] int32): the edges of `topo` in exactly
  one face, in edge order, with their faces, and the boundary edges at each vertex in ascending order."""
  counts = topo.edge_off[1:] - topo.edge_off[:-1]
  idx = torch.nonzero(counts == 1).view(-1)
  edges = topo.edges[idx].contiguous()
  face = topo.edge_face[topo.edge_off[idx]].contiguous()
  B = idx.shape[0]
  ends = edges.t().reshape(-1).long()
  own = torch.arange(B, device=idx.device).repeat(2)
  order = torch.sort(ends * max(B, 1) + own).indices
  zero = torch.zeros(1, device=idx.device, dtype=torch.int64)
  vb_off = torch.cat([zero, torch.cumsum(torch.bincount(ends, minlength=num_vertices), 0)])
  return edges, face, vb_off, own[order].int()


def simplify_mesh(vertices, faces, normals=None, *, target_faces, stats=None):
  """Simplifies a mesh on the device to about `target_faces` faces by parallel greedy quadric edge collapse
  (Garland and Heckbert 1997; csrc/mesh.cu).  vertices [V, 3] fp32, faces [F, 3] int32, normals [V, 3] fp32 or None
  (carried along and blended).  Returns (vertices, faces) or, with normals, (vertices, faces, normals); vertices
  and faces that survive keep their relative order, faces are renumbered and unused vertices dropped.

  Quadrics are built once (mnrf_mesh_quadrics).  Each round rebuilds the topology (mesh_topology), prices every
  edge and checks that it may be collapsed (mnrf_mesh_edge_cost), selects the edges whose key is the least within
  two faces of both ends (mnrf_mesh_collapse_select), keeps the longest prefix in key order that removes no more than
  F - target_faces faces, collapses them (mnrf_mesh_collapse_apply) and compacts the faces.  It stops at
  target_faces or fewer, or after a round with no collapse (a stall: no edge may be collapsed, or the next one would
  overshoot by a face).  The result is bit-deterministic.

  target_faces 0 (off), or a mesh with at most target_faces faces: the inputs come back untouched and nothing is
  launched.  stats: a dict, given faces_before, faces_after, rounds (rounds that collapsed) and target_reached
  (faces_after <= target_faces + 1; True when off)."""
  if target_faces < 0:
    raise ValueError(f'simplify_mesh: target_faces = {target_faces}: want 0 (off) or more')
  out = (vertices, faces) + (() if normals is None else (normals,))
  F = faces.shape[0]
  if stats is not None:
    stats.update(faces_before=F, faces_after=F, rounds=0, target_reached=True)
  if not target_faces or F <= target_faces:
    return out
  V = vertices.shape[0]
  if not 0 < V < 2 ** 31 or F >= 2 ** 31:
    raise ValueError(f'simplify_mesh: {V} vertices, {F} faces')
  assert faces.dtype == torch.int32 and faces.dim() == 2 and faces.shape[1] == 3
  f = faces.contiguous().clone()
  fl = f.long()
  bad = ((fl < 0) | (fl >= V)).any() | (fl[:, 0] == fl[:, 1]).any() | (fl[:, 1] == fl[:, 2]).any() | \
      (fl[:, 2] == fl[:, 0]).any()
  if bool(bad):
    raise ValueError(f'simplify_mesh: a face index lies outside [0, {V}) or a face repeats a vertex')
  del fl
  v = vertices.contiguous().clone()
  n = None if normals is None else normals.contiguous().clone()
  topo = mesh_topology(f, V)
  if topo.edges.shape[0] >= 2 ** 32:
    raise ValueError(f'simplify_mesh: {topo.edges.shape[0]} edges do not fit 32-bit edge indices')
  q = ops.mesh_quadrics(v, f, topo.vf_off, topo.vf_face, *boundary_edges(topo, V))
  rounds = 0
  while True:
    keys, pos = ops.mesh_edge_cost(v, f, q, *topo)
    sel = torch.nonzero(ops.mesh_collapse_select(f, topo.edges, keys, V)).view(-1)
    if sel.shape[0] == 0:
      break
    sel = sel[torch.sort(keys[sel]).indices]                         # key order (keys are unique)
    removed = torch.cumsum(topo.edge_off[sel + 1] - topo.edge_off[sel], 0)
    keep = removed <= F - target_faces                               # a prefix: removed grows
    applied, gone = (int(x) for x in torch.stack([keep.sum(), torch.where(keep, removed, 0).max()]).cpu())
    if applied == 0:
      break
    collapse = torch.zeros(topo.edges.shape[0], device=f.device, dtype=torch.uint8)
    collapse[sel] = keep.to(torch.uint8)
    alive = ops.mesh_collapse_apply(collapse, topo.edges, topo.edge_off, topo.edge_face, topo.vf_off, topo.vf_face,
                                    pos, v, q, n, f)
    f = f[alive.bool()]
    F -= gone
    rounds += 1
    if F <= target_faces:
      break
    del keys, pos, sel, removed, keep, collapse, alive, topo
    topo = mesh_topology(f, V)
  if stats is not None:
    stats.update(faces_after=F, rounds=rounds, target_reached=F <= target_faces + 1)
  return _drop_unused(v, f, *(() if n is None else (n,)))


def render_mesh(vertices, faces, bvh, rays, *, normals=None, rgb=None, uv=None, texture=None, bg):
  """The mesh seen along `rays` (a utils.Rays on the device, any leading shape): each ray's closest hit in
  near <= t <= far (ops.mesh_trace on `bvh`, ops.mesh_bvh of vertices [V, 3] and faces [F, 3] int32).  Returns a dict
  of tensors with the rays' leading shape: hit (bool), distance (t along the rays' directions, inf on a miss),
  normals [..., 3] (the normalised barycentric blend of the vertex `normals` [V, 3]; where there are none or the blend
  is zero, the face normal by its winding; 0 on a miss) and rgb [..., 3] fp32 or None.  rgb: with `texture` (uint8
  [S, S, 3]) and `uv` ([F, 3, 2] texel units, bake_texture's), the atlas sampled bilinearly at the blend of the face's
  corner UVs (texel centres at +0.5); else with `rgb` (uint8 [V, 3] vertex colours) their blend over 255; else None.
  A miss gets the background `bg`.  A mesh without faces is all misses, and nothing is traced or gathered."""
  shape = rays.origins.shape[:-1]
  dev = rays.origins.device
  coloured = texture is not None or rgb is not None
  if faces.shape[0] == 0:
    n = math.prod(shape)
    out = dict(hit=torch.zeros(n, device=dev, dtype=torch.bool), distance=torch.full((n,), math.inf, device=dev),
               normals=torch.zeros(n, 3, device=dev),
               rgb=torch.full((n, 3), float(bg), device=dev) if coloured else None)
    return {k: None if v is None else v.reshape(*shape, *v.shape[1:]) for k, v in out.items()}
  flat = lambda x: torch.as_tensor(x, device=dev, dtype=torch.float32).reshape(-1, x.shape[-1]).contiguous()
  face, t, bary = ops.mesh_trace(bvh, flat(rays.origins), flat(rays.directions), flat(rays.near), flat(rays.far))
  hit = face >= 0
  fi = face.clamp_min(0).long()                  # a miss reads face 0, which exists; its values are masked below
  corners = faces.long()[fi]
  w = torch.cat([1 - bary.sum(-1, keepdim=True), bary], -1)                        # [N, 3]
  blend = lambda per_vertex: (w[..., None] * per_vertex[corners].float()).sum(1)
  p = vertices[corners]
  fn = torch.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0], dim=-1)
  n = blend(normals) if normals is not None else torch.zeros_like(fn)
  n = torch.where((n.norm(dim=-1, keepdim=True) > 0), n, fn)
  n = torch.where(hit[:, None], n / n.norm(dim=-1, keepdim=True).clamp_min(1e-30), torch.zeros_like(n))
  color = None
  if texture is not None:
    S = texture.shape[0]
    st = (w[..., None] * uv[fi]).sum(1) - 0.5                                       # texel index space
    x0 = st.floor()
    frac = st - x0
    x0 = x0.long()
    tex = texture.reshape(-1, 3).float() / 255
    color = torch.zeros(len(fi), 3, device=face.device)
    for dy in (0, 1):
      for dx in (0, 1):
        cx = (x0[:, 0] + dx).clamp(0, S - 1)
        cy = (x0[:, 1] + dy).clamp(0, S - 1)
        wt = (frac[:, 0] if dx else 1 - frac[:, 0]) * (frac[:, 1] if dy else 1 - frac[:, 1])
        color += wt[:, None] * tex[cy * S + cx]
  elif rgb is not None:
    color = blend(rgb) / 255
  if color is not None:
    color = torch.where(hit[:, None], color, torch.full_like(color, float(bg)))
  out = dict(hit=hit, distance=t, normals=n, rgb=color)
  return {k: None if v is None else v.reshape(*shape, *v.shape[1:]) for k, v in out.items()}


def mesh_metrics(render, rgb_gt, config, postprocess_fn=lambda z: z, reference=None):
  """Per-image metrics of a mesh render (render_mesh, [H, W] leading shape) against the test image rgb_gt [H, W, 3]:
  psnr and ssim when the render has colour (eval_lib.image_metrics: RawNeRF postprocessing, 8-bit quantisation and
  border crop as eval_lib.evaluate applies them).  reference (distance_median, acc, rgb) of the NeRF on the same rays
  adds nerf_psnr and nerf_ssim, coverage (the fraction of pixels with acc >= 0.5 the mesh hits), spurious (the
  fraction of mesh hits where acc < 0.5) and depth_abs_rel (the mean |t - distance_median| / distance_median over
  pixels with both); a fraction with no pixel to count over is NaN."""
  from . import eval_lib, image
  host = lambda x: x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)
  harness = image.MetricHarness()
  gt = np.asarray(rgb_gt, np.float64)
  metric = {}
  if render['rgb'] is not None:
    metric.update(eval_lib.image_metrics(config, postprocess_fn, harness, gt, host(render['rgb']).astype(np.float64))[0])
  if reference is not None:
    dm, acc, nerf_rgb = (host(x).astype(np.float64) for x in reference)
    dm, acc = dm.reshape(gt.shape[:2]), acc.reshape(gt.shape[:2])
    m = eval_lib.image_metrics(config, postprocess_fn, harness, gt, nerf_rgb.reshape(gt.shape))[0]
    metric.update(nerf_psnr=m['psnr'], nerf_ssim=m['ssim'])
    hit = host(render['hit']).reshape(gt.shape[:2])
    seen = acc >= 0.5
    frac = lambda num, den: float(num) / float(den) if den else float('nan')
    metric['coverage'] = frac((hit & seen).sum(), seen.sum())
    metric['spurious'] = frac((hit & ~seen).sum(), hit.sum())
    both = hit & seen
    t = host(render['distance']).astype(np.float64).reshape(gt.shape[:2])
    metric['depth_abs_rel'] = float((np.abs(t - dm) / dm)[both].mean()) if both.any() else float('nan')
  return metric


def evaluate_mesh(vertices, faces, dataset, config, *, normals=None, rgb=None, uv=None, texture=None,
                  reference=None, bg=1.0, save_fn=None, timing=None):
  """Scores a mesh against the test views of `dataset` (the test split, not NDC): builds the BVH once, renders every
  view up to Config.eval_dataset_limit with render_mesh (normals, rgb, uv, texture and bg as it takes them) and
  returns the per-image metrics of mesh_metrics, a list of dicts.  reference: an iterable of (idx, distance_median,
  acc, rgb) of the NeRF on the same views, as render_views yields it.  save_fn(idx, render): called per view.
  timing: a dict, given 'build' and 'trace' seconds (device-synchronised; tracing includes the shading)."""
  import time
  if dataset.cameras[3] is not None:
    raise ValueError('evaluate_mesh does not support forward-facing (NDC) scenes: the mesh is in world space')
  metadata = getattr(dataset, 'metadata', None)
  postprocess_fn = metadata['postprocess_fn'] if (config.rawnerf_mode and metadata) else (lambda z: z)
  num_eval = min(dataset.size, config.eval_dataset_limit)
  torch.cuda.synchronize()
  t0 = time.time()
  bvh = ops.mesh_bvh(vertices, faces)
  torch.cuda.synchronize()
  times = dict(build=time.time() - t0, trace=0.0)
  ref_iter = iter(reference) if reference is not None else None
  metrics = []
  for idx in range(num_eval):
    ref = None
    if ref_iter is not None:
      ridx, dm, acc, nerf_rgb = next(ref_iter)
      if ridx != idx:
        raise ValueError(f'evaluate_mesh: reference view {ridx} where view {idx} was expected')
      ref = (dm, acc, nerf_rgb)
    t1 = time.time()
    rays = dataset.generate_ray_batch(idx).rays
    render = render_mesh(vertices, faces, bvh, rays, normals=normals, rgb=rgb, uv=uv, texture=texture, bg=bg)
    torch.cuda.synchronize()
    times['trace'] += time.time() - t1
    metrics.append(mesh_metrics(render, dataset.images[idx], config, postprocess_fn, ref))
    if save_fn is not None:
      save_fn(idx, render)
  if timing is not None:
    timing.update(times)
  return metrics


def _clean_args(keep_components, min_views, dataset, stats):
  """clean_mesh's keyword arguments, the cameras taken from `dataset` when `min_views` needs them."""
  args = dict(keep_components=keep_components, min_views=min_views, stats=stats)
  if min_views:
    if dataset is None:
      raise ValueError('min_views needs the training cameras: pass the dataset')
    args.update(cameras=dataset.cameras, camtype=dataset.camtype, image_size=(dataset.height, dataset.width))
  return args


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


def write_obj(path, vertices, faces, normals, uv, texture):
  """A textured mesh as three files beside each other: <stem>.obj (positions `v`, one texture coordinate `vt` per face
  corner, normals `vn`, faces `f v/vt/vn`), <stem>.mtl (one material whose diffuse map is the PNG) and <stem>.png
  (texture, uint8 [S, S, 3], written as it is).  uv [F, 3, 2]: bake_texture's corner positions in texel units; a
  corner's `vt` is (u / S, 1 - v / S), OBJ's origin being the image's bottom-left corner.  Floats are printed with
  %.9g, so every fp32 value reads back exactly.  Returns the paths (obj, mtl, png)."""
  from PIL import Image
  stem = os.path.splitext(path)[0]
  name = os.path.basename(stem)
  host = lambda t, dtype: np.ascontiguousarray(torch.as_tensor(t).detach().cpu().numpy(), dtype=dtype)
  v, n = host(vertices, np.float32).reshape(-1, 3), host(normals, np.float32).reshape(-1, 3)
  f = host(faces, np.int64).reshape(-1, 3)
  tex = host(texture, np.uint8)
  size = tex.shape[0]
  assert tex.shape == (size, size, 3), 'texture must be [S, S, 3]'
  uvh = host(uv, np.float32).reshape(-1, 2)
  vt = np.stack([uvh[:, 0] / np.float32(size), np.float32(1) - uvh[:, 1] / np.float32(size)], -1)
  # f a/ta/na: 1-based; face k's corners are vt 3k + 1 .. 3k + 3
  corners = np.stack([f + 1, np.arange(1, 3 * len(f) + 1).reshape(-1, 3), f + 1], -1)
  obj, mtl, png = stem + '.obj', stem + '.mtl', stem + '.png'
  with open(obj, 'w') as fh:
    fh.write(f'mtllib {name}.mtl\n')
    fh.write(('v %.9g %.9g %.9g\n' * len(v)) % tuple(v.ravel().tolist()))
    fh.write(('vt %.9g %.9g\n' * len(vt)) % tuple(vt.ravel().tolist()))
    fh.write(('vn %.9g %.9g %.9g\n' * len(n)) % tuple(n.ravel().tolist()))
    fh.write('usemtl texture\n')
    fh.write(('f %d/%d/%d %d/%d/%d %d/%d/%d\n' * len(f)) % tuple(corners.ravel().tolist()))
  with open(mtl, 'w') as fh:
    fh.write(f'newmtl texture\nKa 1 1 1\nKd 1 1 1\nKs 0 0 0\nillum 1\nmap_Kd {name}.png\n')
  Image.fromarray(tex).save(png, 'PNG')
  return obj, mtl, png
