"""Thin tensor-level wrappers over the C ABI (one Python function per entry point).

These mirror the reference's free functions where one exists (stepfun.sample_intervals,
render.cast_rays + coord.integrated_pos_enc, render.compute_alpha_weights +
volumetric_rendering, ...) but operate on flat [B, ...] CUDA tensors.
"""
import ctypes as C
import math
from typing import NamedTuple

import torch

from . import lib as L

EPS = float(torch.finfo(torch.float32).eps)

# Instrumentation used by bench.py: number of kernels launched (counted per ABI call), and --
# when set to a list -- CUDA event pairs around every tensor-core GEMM launch.
LAUNCHES = 0
GEMM_EVENTS = None


def _count(n=1):
  global LAUNCHES
  LAUNCHES += n


def _gemm_call(flops, fn, *args):
  """One counted GEMM launch fn(*args); with GEMM_EVENTS a list, it runs between two CUDA events appended there
  with its `flops`."""
  _count()
  if GEMM_EVENTS is None:
    L.check(fn(*args))
    return
  ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
  ev[0].record()
  L.check(fn(*args))
  ev[1].record()
  GEMM_EVENTS.append((ev[0], ev[1], flops))


def _f32(t):
  assert t is None or (t.dtype == torch.float32 and t.is_contiguous()), 'need contiguous fp32'
  return t


def _sample_ld(t, channels):
  """Floats between consecutive samples of an fp32 per-sample tensor: [B, S] (channels 0) or [B, S, channels] with a
  unit channel stride, whose samples are evenly spaced -- a contiguous tensor, or a column view of a stacked head's
  [B*S, 4] output."""
  if t is None:
    return 0
  assert t.dtype == torch.float32
  ld = t.stride(-1) if channels == 0 else t.stride(-2)
  assert channels == 0 or t.stride(-1) == 1
  assert all(t.stride(i) == ld * math.prod(t.shape[i + 1:len(t.shape) - (1 if channels else 0)])
             for i in range(t.dim() - (2 if channels else 1))), 'samples must be evenly spaced'
  return ld


def u_grid(num_samples, randomized):
  """Host-side u grid of stepfun.sample (stepfun.py:190-209): (u_base[S] fp32, max_jitter)."""
  eps = EPS
  if not randomized:
    pad = 1 / (2 * num_samples)
    return torch.linspace(pad, 1.0 - pad - eps, num_samples, dtype=torch.float32), 0.0
  u_max = eps + (1 - eps) / num_samples
  max_jitter = (1 - u_max) / (num_samples - 1) - eps
  return torch.linspace(0, 1 - u_max, num_samples, dtype=torch.float32), max_jitter


def sample_level(sdist_prev, w_prev, num_samples, *, dilation=0.0, use_dilation=False,
                 domain=(0.0, 1.0), anneal=1.0, resample_padding=0.0, jitter=None,
                 single_jitter=True, u_base=None, max_jitter=None, cw_in=None, want_index=False,
                 want_debug=False, out=None, anneal_dev=None):
  """One level of hierarchical resampling -> sdist [B, S+1] (+ int32 idx, debug arrays)."""
  lib = L.load()
  if num_samples <= 1:
    raise ValueError(f'num_samples must be > 1, is {num_samples}.')
  B, P = w_prev.shape
  assert sdist_prev.shape == (B, P + 1)
  dev = sdist_prev.device
  if u_base is None:
    ub, mj = u_grid(num_samples, jitter is not None)
    u_base = ub.to(dev)
    max_jitter = mj if max_jitter is None else max_jitter
  d = L.SampleDesc(B, P, num_samples, int(use_dilation), float(dilation), float(domain[0]),
                   float(domain[1]), float(anneal), float(resample_padding),
                   0 if jitter is None else (1 if single_jitter else 2), float(max_jitter or 0.0))
  nb = 3 * P - 2 if use_dilation else P
  sdist = out if out is not None else torch.empty(B, num_samples + 1, device=dev)
  idx = torch.empty(B, num_samples, device=dev, dtype=torch.int32) if want_index else None
  cw = torch.empty(B, nb + 1, device=dev) if want_debug else None
  tdil = torch.empty(B, nb + 1, device=dev) if want_debug else None
  wdil = torch.empty(B, nb, device=dev) if want_debug else None
  _count()
  L.check(lib.mnrf_sample_level(C.byref(d), L.ptr(_f32(sdist_prev)), L.ptr(_f32(w_prev)),
                                L.ptr(_f32(u_base)), L.ptr(_f32(jitter)), L.ptr(anneal_dev), L.ptr(_f32(cw_in)),
                                L.ptr(sdist), L.ptr(idx), L.ptr(cw), L.ptr(tdil), L.ptr(wdil),
                                L.stream_ptr()))
  if want_index or want_debug:
    return sdist, dict(idx=idx, cw=cw, tdil=tdil, wdil=wdil)
  return sdist


def encode(sdist, origins, directions, radii, near, far, basis, *, min_deg, max_deg,
           raydist_fn=None, ray_shape='cone', warp_contract=False, disable_integration=False,
           feat=None, feat_cols=None, want_f32=False, want_tdist=False, tfeat=None):
  """cast_rays + (contract) + lift + IPE -> bf16 features [B*S, ld] (row stride from `feat`)."""
  lib = L.load()
  if ray_shape not in L.RAY_SHAPE:
    raise ValueError("ray_shape must be 'cone' or 'cylinder'")
  B, S1 = sdist.shape
  S = S1 - 1
  K = basis.shape[0]
  F = 2 * K * (max_deg - min_deg)
  if feat_cols is None:
    feat_cols = (F + 63) // 64 * 64
  if feat is None:
    feat = torch.empty(B * S, feat_cols, device=sdist.device, dtype=torch.bfloat16)
  assert feat.dtype == torch.bfloat16 and feat.stride(1) == 1
  ld = feat.stride(0)
  d = L.EncodeDesc(B, S, L.RAYDIST[raydist_fn], L.RAY_SHAPE[ray_shape], int(warp_contract),
                   int(disable_integration), K, min_deg, max_deg, ld, feat_cols)
  f32 = torch.empty(B * S, F, device=sdist.device) if want_f32 else None
  tdist = torch.empty(B, S + 1, device=sdist.device) if want_tdist else None
  if tfeat is not None:
    assert tfeat.dtype == torch.bfloat16 and tfeat.stride(1) == 1
  _count()
  L.check(lib.mnrf_encode(C.byref(d), L.ptr(_f32(sdist)), L.ptr(_f32(origins)),
                          L.ptr(_f32(directions)), L.ptr(_f32(radii)), L.ptr(_f32(near)),
                          L.ptr(_f32(far)), L.ptr(_f32(basis)), L.ptr(feat), L.ptr(f32),
                          L.ptr(tdist), L.ptr(tfeat), tfeat.stride(0) if tfeat is not None else 0, L.stream_ptr()))
  return feat, f32, tdist


def encode_points(points, var, basis, *, min_deg, max_deg, warp_contract=False, disable_integration=False,
                  feat=None, feat_cols=None, want_f32=False, tfeat=None):
  """Point form of `encode`: features of the Gaussians (points[i], var * I) -> bf16 [N, ld] (+ fp32 [N, 2KL]).
  With `tfeat` [3N, ld_t] bf16, also the tangent rows d feature / d point (no fp32 copy then).  warp_contract: False
  / True, or 2 for points already contracted: encoded as they are, tangent rows with respect to the world point
  inv_contract(point) (include/mnrf.h)."""
  lib = L.load()
  N = points.shape[0]
  K = basis.shape[0]
  F = 2 * K * (max_deg - min_deg)
  if feat_cols is None:
    feat_cols = (F + 63) // 64 * 64
  if feat is None:
    feat = torch.empty(N, feat_cols, device=points.device, dtype=torch.bfloat16)
  assert feat.dtype == torch.bfloat16 and feat.stride(1) == 1
  d = L.EncodeDesc(N, 1, 0, 0, int(warp_contract), int(disable_integration), K, min_deg, max_deg, feat.stride(0),
                   feat_cols)
  _count()
  if tfeat is not None:
    assert not want_f32 and tfeat.dtype == torch.bfloat16 and tfeat.stride(1) == 1
    L.check(lib.mnrf_encode_points_tangent(C.byref(d), L.ptr(_f32(points)), float(var), L.ptr(_f32(basis)),
                                           L.ptr(feat), L.ptr(tfeat), tfeat.stride(0), L.stream_ptr()))
    return feat, None
  f32 = torch.empty(N, F, device=points.device) if want_f32 else None
  L.check(lib.mnrf_encode_points(C.byref(d), L.ptr(_f32(points)), float(var), L.ptr(_f32(basis)), L.ptr(feat),
                                 L.ptr(f32), L.stream_ptr()))
  return feat, f32


def marching_cubes(grid, level, normals=False):
  """Marching cubes on an fp32 grid [nz, ny, nx] (inside: value > level) -> (vertices [V, 3] fp32 in grid units
  (x, y, z), faces [F, 3] int32), and with `normals` the unit vertex normals [V, 3] (from dense to empty space, the
  grid's gradient interpolated along each vertex's edge).  Reads the two totals back once, between the count and
  emit phases."""
  lib = L.load()
  grid = _f32(grid)
  assert grid.dim() == 3, 'grid must be [nz, ny, nx]'
  nz, ny, nx = grid.shape
  n = grid.numel()
  dev = grid.device
  edge_cut = torch.empty(3 * n, device=dev, dtype=torch.uint8)
  cell_tris = torch.empty(n, device=dev, dtype=torch.uint8)
  args = (nx, ny, nz, L.ptr(grid), float(level), L.ptr(edge_cut), L.ptr(cell_tris))
  _count()
  L.check(lib.mnrf_marching_cubes(L.MC_COUNT, *args, None, None, None, None, L.stream_ptr()))
  edge_scan = torch.cumsum(edge_cut, 0, dtype=torch.int64)
  tri_scan = torch.cumsum(cell_tris, 0, dtype=torch.int64)
  V, F = (int(v) for v in torch.stack([edge_scan[-1], tri_scan[-1]]).cpu())
  if V >= 2 ** 31:
    raise ValueError(f'marching_cubes: {V} vertices do not fit the int32 face indices')
  vertices = torch.empty(V, 3, device=dev)
  faces = torch.empty(F, 3, device=dev, dtype=torch.int32)
  if V:
    _count()
    L.check(lib.mnrf_marching_cubes(L.MC_EMIT, *args, L.ptr(edge_scan), L.ptr(tri_scan), L.ptr(vertices),
                                    L.ptr(faces), L.stream_ptr()))
  if not normals:
    return vertices, faces
  vnormals = torch.empty(V, 3, device=dev)
  if V:
    _count()
    L.check(lib.mnrf_mc_normals(nx, ny, nz, L.ptr(grid), float(level), L.ptr(edge_cut), L.ptr(edge_scan),
                                L.ptr(vnormals), L.stream_ptr()))
  return vertices, faces, vnormals


def _projection_desc(camtype, distortion_params, num_cameras):
  """The camera descriptor the forward projection reads (mnrf_tsdf_integrate, mnrf_points_view_count)."""
  dp = dict(distortion_params or {})
  return L.CameraDesc(0, num_cameras, int(camtype), int(distortion_params is not None),
                      *(float(dp.get(k, 0.0)) for k in ('k1', 'k2', 'k3', 'k4', 'p1', 'p2')), 0.0, 0, 0, 1.0, 1.0,
                      1.0)


def mesh_components(faces, num_vertices):
  """Connected components of the mesh with `num_vertices` vertices and faces [F, 3] int32 on the device
  (mnrf_mesh_components, csrc/mesh.cu) -> labels [V] int32: each vertex's label is the smallest vertex index of its
  component.  Checks on the device that every face index lies in [0, V) and reads that one flag back; an index out
  of range raises ValueError and never reaches the kernel."""
  lib = L.load()
  assert faces.dtype == torch.int32 and faces.is_contiguous() and faces.dim() == 2 and faces.shape[1] == 3
  V, F = int(num_vertices), faces.shape[0]
  if not 0 <= V < 2 ** 31:
    raise ValueError(f'mesh_components: {V} vertices')
  if F and bool(((faces < 0) | (faces >= V)).any()):
    raise ValueError(f'mesh_components: a face index lies outside [0, {V})')
  labels = torch.empty(V, device=faces.device, dtype=torch.int32)
  if V:
    _count(3 if F else 2)
    L.check(lib.mnrf_mesh_components(V, F, L.ptr(faces), L.ptr(labels), L.stream_ptr()))
  return labels


def _i32(t):
  assert t.dtype == torch.int32 and t.is_contiguous(), 'need contiguous int32'
  return t


def _i64(t):
  assert t.dtype == torch.int64 and t.is_contiguous(), 'need contiguous int64'
  return t


def mesh_quadrics(vertices, faces, vf_off, vf_face, boundary_edges, boundary_face, vb_off, vb_edge):
  """Per-vertex error quadrics [V, 10] fp64 of a mesh (mnrf_mesh_quadrics, csrc/mesh.cu): area-weighted face planes,
  then boundary-edge planes.  The topology tensors as mesh.mesh_topology and mesh.boundary_edges build them."""
  lib = L.load()
  V, F, B = vertices.shape[0], faces.shape[0], boundary_edges.shape[0]
  q = torch.empty(V, 10, device=vertices.device, dtype=torch.float64)
  if V:
    _count()
    L.check(lib.mnrf_mesh_quadrics(V, F, L.ptr(_f32(vertices)), L.ptr(_i32(faces)), L.ptr(_i64(vf_off)),
                                   L.ptr(_i32(vf_face)), B, L.ptr(_i32(boundary_edges)), L.ptr(_i32(boundary_face)),
                                   L.ptr(_i64(vb_off)), L.ptr(_i32(vb_edge)), L.ptr(q), L.stream_ptr()))
  return q


def mesh_edge_cost(vertices, faces, quadrics, edges, edge_off, edge_face, vf_off, vf_face):
  """Per edge, the collapse position [E, 3] fp32 and key [E] (uint64 bits in an int64 tensor; -1 where the edge may
  not be collapsed) (mnrf_mesh_edge_cost, csrc/mesh.cu) -> (keys, positions)."""
  lib = L.load()
  V, F, E = vertices.shape[0], faces.shape[0], edges.shape[0]
  dev = vertices.device
  keys = torch.empty(E, device=dev, dtype=torch.int64)
  pos = torch.empty(E, 3, device=dev)
  if E:
    flags = torch.empty(V, device=dev, dtype=torch.int32)
    _count(2)
    L.check(lib.mnrf_mesh_edge_cost(V, F, E, L.ptr(_f32(vertices)), L.ptr(_i32(faces)), L.ptr(quadrics),
                                    L.ptr(_i32(edges)), L.ptr(_i64(edge_off)), L.ptr(_i32(edge_face)),
                                    L.ptr(_i64(vf_off)), L.ptr(_i32(vf_face)), L.ptr(flags), L.ptr(keys), L.ptr(pos),
                                    L.stream_ptr()))
  return keys, pos


def mesh_collapse_select(faces, edges, keys, num_vertices):
  """The edges a round collapses, selected [E] uint8 (mnrf_mesh_collapse_select, csrc/mesh.cu): an edge whose key is
  the least within two faces of each of its ends."""
  lib = L.load()
  E = edges.shape[0]
  dev = edges.device
  sel = torch.empty(E, device=dev, dtype=torch.uint8)
  if E:
    vmin = torch.empty(num_vertices, device=dev, dtype=torch.int64)
    rmin = torch.empty_like(vmin)
    _count(3)
    L.check(lib.mnrf_mesh_collapse_select(num_vertices, faces.shape[0], E, L.ptr(_i32(faces)), L.ptr(_i32(edges)),
                                          L.ptr(_i64(keys)), L.ptr(vmin), L.ptr(rmin), L.ptr(sel), L.stream_ptr()))
  return sel


def mesh_collapse_apply(collapse, edges, edge_off, edge_face, vf_off, vf_face, positions, vertices, quadrics,
                        normals, faces):
  """Collapses the edges with collapse [E] uint8 set, updating vertices, quadrics, normals (or None) and faces in
  place (mnrf_mesh_collapse_apply, csrc/mesh.cu) -> face_alive [F] uint8."""
  lib = L.load()
  V, F, E = vertices.shape[0], faces.shape[0], edges.shape[0]
  alive = torch.empty(F, device=faces.device, dtype=torch.uint8)
  if F:
    _count()
    L.check(lib.mnrf_mesh_collapse_apply(V, F, E, L.ptr(collapse), L.ptr(_i32(edges)), L.ptr(_i64(edge_off)),
                                         L.ptr(_i32(edge_face)), L.ptr(_i64(vf_off)), L.ptr(_i32(vf_face)),
                                         L.ptr(_f32(positions)), L.ptr(_f32(vertices)), L.ptr(quadrics),
                                         L.ptr(_f32(normals)), L.ptr(_i32(faces)), L.ptr(alive), L.stream_ptr()))
  return alive


TEXTURE_SIZES = (4, 16384)


def texture_atlas(num_faces, size):
  """(n, c): cells per row and texels per cell side of the size x size atlas of `num_faces` per-face charts, two per
  cell (mnrf_mesh_texture_raster, include/mnrf.h).  Raises ValueError when `size` lies outside [4, 16384] or a cell
  would be narrower than 4 texels."""
  if not TEXTURE_SIZES[0] <= size <= TEXTURE_SIZES[1]:
    raise ValueError(f'texture size {size}: want [{TEXTURE_SIZES[0]}, {TEXTURE_SIZES[1]}]')
  cells = (num_faces + 1) // 2
  n = math.isqrt(cells - 1) + 1 if cells else 0
  c = size // n if n else size
  if c < 4:
    raise ValueError(f'{num_faces} faces do not fit a {size} x {size} texture atlas, which holds at most '
                     f'{2 * (size // 4) ** 2} faces (cells of at least 4 x 4 texels): raise the texture size or '
                     f'simplify the mesh first (Config.mesh_target_faces)')
  return n, c


def mesh_texture_raster(vertices, faces, normals, size):
  """The texture atlas of a mesh (mnrf_mesh_texture_raster, csrc/mesh.cu): vertices [V, 3], faces [F, 3] int32 and
  vertex normals [V, 3] on the device, a size x size atlas -> (uv [F, 3, 2] fp32 corner positions in texel units,
  texel_index [T] int32 row-major in the atlas, points [T, 3], normals [T, 3]) for the T = ceil(F / 2) c^2 texels of
  the used cells (texture_atlas).  Checks on the device that every face index lies in [0, V) and reads that one flag
  back; an index out of range raises ValueError and never reaches the kernel."""
  lib = L.load()
  assert faces.dtype == torch.int32 and faces.is_contiguous() and faces.dim() == 2 and faces.shape[1] == 3
  V, F = vertices.shape[0], faces.shape[0]
  n, c = texture_atlas(F, size)
  if not 0 <= V < 2 ** 31:
    raise ValueError(f'mesh_texture_raster: {V} vertices')
  if normals.shape != vertices.shape or vertices.dim() != 2 or vertices.shape[1] != 3:
    raise ValueError(f'mesh_texture_raster: vertices {tuple(vertices.shape)} and normals {tuple(normals.shape)}: '
                     'want [V, 3] both')
  if F and bool(((faces < 0) | (faces >= V)).any()):
    raise ValueError(f'mesh_texture_raster: a face index lies outside [0, {V})')
  dev = faces.device
  T = (F + 1) // 2 * c * c
  uv = torch.empty(F, 3, 2, device=dev)
  index = torch.empty(T, device=dev, dtype=torch.int32)
  points = torch.empty(T, 3, device=dev)
  tnormals = torch.empty(T, 3, device=dev)
  if F:
    _count(2)
    L.check(lib.mnrf_mesh_texture_raster(V, F, L.ptr(_f32(vertices)), L.ptr(faces), L.ptr(_f32(normals)), int(size),
                                         L.ptr(uv), L.ptr(index), L.ptr(points), L.ptr(tnormals), L.stream_ptr()))
  return uv, index, points, tnormals


class MeshBVH(NamedTuple):
  """A linear BVH over the faces of a mesh (mnrf_mesh_bvh, include/mnrf.h), with the mesh it was built on."""
  vertices: torch.Tensor    # [V, 3] fp32
  faces: torch.Tensor       # [F, 3] int32
  nodes: torch.Tensor       # [max(F - 1, 0), 16] fp32: both children's boxes, then the children as int32 bits
  parent: torch.Tensor      # [max(2 F - 1, 0)] int32, -1 at the root
  leaf_face: torch.Tensor   # [F] int32: the face of each leaf, in key order
  keys: torch.Tensor        # [F] int64, ascending: morton << 32 | face


def mesh_bvh(vertices, faces):
  """The linear BVH of a mesh on the device (mnrf_mesh_bvh, csrc/mesh_trace.cu) -> MeshBVH.  vertices [V, 3] fp32,
  faces [F, 3] int32.  Checks on the device that every face index lies in [0, V) and every vertex is finite, and
  reads that one flag back: either failure raises ValueError and never reaches a kernel; so does F >= 2^30.  No other
  host synchronisation: the centroid bounds go to the key kernel by device pointer.  F = 0 gives an empty tree and
  F = 1 a tree that is its leaf, with no launch."""
  lib = L.load()
  if vertices.dim() != 2 or vertices.shape[1] != 3 or faces.dim() != 2 or faces.shape[1] != 3:
    raise ValueError(f'mesh_bvh: vertices {tuple(vertices.shape)}, faces {tuple(faces.shape)}: want [V, 3] and [F, 3]')
  vertices, faces = _f32(vertices.contiguous()), _i32(faces.contiguous())
  V, F = vertices.shape[0], faces.shape[0]
  if not 0 <= V < 2 ** 31 or F >= 2 ** 30:
    raise ValueError(f'mesh_bvh: {V} vertices, {F} faces: want V < 2^31 and F < 2^30')
  dev = vertices.device
  bad = ~torch.isfinite(vertices).all()
  if F:
    bad |= ((faces < 0) | (faces >= V)).any()
  if bool(bad):
    raise ValueError(f'mesh_bvh: a vertex is not finite or a face index lies outside [0, {V})')
  i32 = lambda n: torch.empty(n, device=dev, dtype=torch.int32)
  if F <= 1:
    keys = torch.zeros(F, device=dev, dtype=torch.int64)
    return MeshBVH(vertices, faces, torch.empty(0, 16, device=dev), torch.full((F,), -1, device=dev,
                                                                               dtype=torch.int32),
                   torch.zeros(F, device=dev, dtype=torch.int32), keys)
  boxes = torch.empty(F, 6, device=dev)
  centroids = torch.empty(F, 3, device=dev)
  keys = torch.empty(F, device=dev, dtype=torch.int64)
  args = [V, F, L.ptr(vertices), L.ptr(faces), L.ptr(boxes), L.ptr(centroids)]
  _count(4)                                    # boxes, keys, then topology and box fit
  L.check(lib.mnrf_mesh_bvh(L.BVH_BOXES, *args, None, None, None, None, None, None, None, L.stream_ptr()))
  bounds = torch.cat([centroids.amin(0), centroids.amax(0)]).contiguous()
  L.check(lib.mnrf_mesh_bvh(L.BVH_KEYS, *args, L.ptr(bounds), L.ptr(keys), None, None, None, None, None,
                            L.stream_ptr()))
  keys = torch.sort(keys).values
  nodes = torch.empty(F - 1, 16, device=dev)
  parent, leaf_face, counters = i32(2 * F - 1), i32(F), i32(F - 1)
  L.check(lib.mnrf_mesh_bvh(L.BVH_TREE, *args, None, None, L.ptr(keys), L.ptr(nodes), L.ptr(parent),
                            L.ptr(leaf_face), L.ptr(counters), L.stream_ptr()))
  return MeshBVH(vertices, faces, nodes, parent, leaf_face, keys)


def mesh_trace(bvh, origins, directions, near, far):
  """The closest hit of each ray in the mesh of `bvh` (mnrf_mesh_trace, csrc/mesh_trace.cu): origins, directions
  [N, 3], near, far [N] or [N, 1] fp32 on the device; only hits with near <= t <= far count.  Returns (face [N] int32,
  -1 for a miss; t [N] fp32, inf for a miss; bary [N, 2] fp32, the barycentrics of corners faces[f, 1] and
  faces[f, 2]).  Reads the traversal's error flag back once and raises RuntimeError if it is set."""
  lib = L.load()
  origins, directions = _f32(origins.contiguous()), _f32(directions.contiguous())
  N = origins.shape[0]
  near, far = (_f32(x.reshape(-1).contiguous()) for x in (near, far))
  if origins.shape != (N, 3) or directions.shape != (N, 3) or near.shape[0] != N or far.shape[0] != N:
    raise ValueError(f'mesh_trace: origins {tuple(origins.shape)}, directions {tuple(directions.shape)}, near '
                     f'{tuple(near.shape)}, far {tuple(far.shape)}: want [N, 3], [N, 3], [N], [N]')
  dev = origins.device
  face = torch.full((N,), -1, device=dev, dtype=torch.int32)
  t = torch.full((N,), float('inf'), device=dev)
  bary = torch.zeros(N, 2, device=dev)
  F = bvh.faces.shape[0]
  if N == 0 or F == 0:
    return face, t, bary
  flag = torch.zeros(1, device=dev, dtype=torch.int32)
  _count()
  L.check(lib.mnrf_mesh_trace(N, L.ptr(origins), L.ptr(directions), L.ptr(near), L.ptr(far), F,
                              L.ptr(bvh.nodes) if F > 1 else None, L.ptr(bvh.leaf_face), L.ptr(bvh.vertices),
                              L.ptr(bvh.faces), L.ptr(face), L.ptr(t), L.ptr(bary), L.ptr(flag), L.stream_ptr()))
  if int(flag.item()):
    raise RuntimeError('mesh_trace: a ray overflowed the traversal stack (a BVH deeper than 63 levels)')
  return face, t, bary


def mesh_uncontract(points, normals=None):
  """Contracted points [N, 3] (and their level-set normals [N, 3]) fp32 on the device -> world points [N, 3] (and unit
  world normals [N, 3]) by mnrf_mesh_uncontract (csrc/mesh.cu): inv_contract of each point, J n of each normal.
  Checks on the device that every point is finite and lies inside the open ball of radius 2, the contracted
  space's extent, and reads that one flag back: a point outside raises ValueError and never reaches the kernel."""
  lib = L.load()
  points = _f32(points.contiguous())
  if points.dim() != 2 or points.shape[1] != 3 or (normals is not None and normals.shape != points.shape):
    raise ValueError(f'mesh_uncontract: points {tuple(points.shape)}, normals '
                     f'{None if normals is None else tuple(normals.shape)}: want [N, 3] both')
  N = points.shape[0]
  world = torch.empty_like(points)
  wnormals = None if normals is None else torch.empty_like(points)
  if N == 0:
    return world if normals is None else (world, wnormals)
  if bool(~(points.double().square().sum(-1) < 4).all()):
    raise ValueError('mesh_uncontract: a point is not finite or lies outside the open ball of radius 2')
  if normals is not None:
    normals = _f32(normals.contiguous())
  _count()
  L.check(lib.mnrf_mesh_uncontract(N, L.ptr(points), L.ptr(normals), L.ptr(world), L.ptr(wnormals),
                                   L.stream_ptr()))
  return world if normals is None else (world, wnormals)


def points_view_count(points, camtype, distortion_params, worldtocams, camtopixs, height, width):
  """For each point [N, 3] fp32 on the device, the number of views whose height x width image it lands on
  (mnrf_points_view_count, csrc/mesh.cu: the pixel rule of tsdf_integrate) -> counts [N] int32.  camtype 0
  perspective / 1 fisheye; distortion_params: dict of k1..k4, p1, p2 or None; worldtocams [K, 3, 4], camtopixs
  [K or 1, 3, 3] fp32 on the device."""
  lib = L.load()
  N, K = points.shape[0], worldtocams.shape[0]
  d = _projection_desc(camtype, distortion_params, camtopixs.shape[0])
  counts = torch.empty(N, device=points.device, dtype=torch.int32)
  if N:
    _count()
    L.check(lib.mnrf_points_view_count(C.byref(d), N, L.ptr(_f32(points)), K, int(height), int(width),
                                       L.ptr(_f32(worldtocams)), L.ptr(_f32(camtopixs)), L.ptr(counts),
                                       L.stream_ptr()))
  return counts


def tsdf_integrate(shape, lo, h, camtype, distortion_params, worldtocams, camtopixs, depth, acc, rgb, tau, tsdf,
                   weight, color_sum=None, color_weight=None, contracted=False):
  """Fuse K views into the TSDF state in place (mnrf_tsdf_integrate, csrc/mesh.cu).  shape (nx, ny, nz) and lo, h:
  the grid points lo + h (x, y, z); camtype 0 perspective / 1 fisheye; distortion_params: dict of k1..k4, p1, p2
  or None; worldtocams [K, 3, 4], camtopixs [K or 1, 3, 3], depth, acc [K, H, W], rgb [K, H, W, 3] or None, fp32 on
  the device; tsdf, weight [nz, ny, nx] and, with rgb, color_sum [nz, ny, nx, 3], color_weight [nz, ny, nx].
  contracted: the grid, lo, h and tau are in the scene contraction's space (mnrf_tsdf_integrate_contracted)."""
  lib = L.load()
  nx, ny, nz = shape
  K, H, W = depth.shape
  d = _projection_desc(camtype, distortion_params, camtopixs.shape[0])
  _count()
  fn = lib.mnrf_tsdf_integrate_contracted if contracted else lib.mnrf_tsdf_integrate
  L.check(fn(C.byref(d), nx, ny, nz, *(float(v) for v in lo), float(h), K, H, W,
                                  L.ptr(_f32(worldtocams)), L.ptr(_f32(camtopixs)), L.ptr(_f32(depth)),
                                  L.ptr(_f32(acc)), L.ptr(_f32(rgb)), float(tau), L.ptr(_f32(tsdf)),
                                  L.ptr(_f32(weight)), L.ptr(_f32(color_sum)), L.ptr(_f32(color_weight)),
                                  L.stream_ptr()))


def viewdir_enc(viewdirs, num_samples, deg, out, col0, col_end):
  lib = L.load()
  B = viewdirs.shape[0]
  _count()
  L.check(lib.mnrf_viewdir_enc(B, num_samples, deg, L.ptr(_f32(viewdirs)), L.ptr(out),
                               out.stride(0), col0, col_end, L.stream_ptr()))


def gemm(mode, a, b, out, *, m, n, k, act=L.ACT_NONE, bias=None, rowv=None, colv=None, mask=None,
         maskbits=None, colsum=None, mask_mod=0, addend=None, z=None, impl=0):
  """Dense-layer GEMM (see include/mnrf.h).  a/b/out/mask/z are 2-D views with unit inner stride.  With a smooth
  `act` (L.SMOOTH_ACTS), FWD writes the pre-activation to z (optional) and DGRAD multiplies by a'(z)."""
  lib = L.load()
  for t in (a, b, out) + tuple(t for t in (mask, z) if t is not None):
    assert t.stride(-1) == 1
  if maskbits is not None:
    assert maskbits.dtype == torch.int32 and maskbits.stride(-1) == 1
  assert z is None or z.dtype == torch.bfloat16
  d = L.GemmDesc(mode, act, m, n, k, a.stride(0), b.stride(0), out.stride(0),
                 mask.stride(0) if mask is not None else 0,
                 maskbits.stride(0) if maskbits is not None else 0,
                 addend.stride(0) if addend is not None else 0, mask_mod, impl)
  _gemm_call(2.0 * m * n * k, lib.mnrf_gemm, C.byref(d), L.ptr(a), L.ptr(b), L.ptr(bias), L.ptr(rowv), L.ptr(colv),
             L.ptr(mask), L.ptr(maskbits), L.ptr(colsum), L.ptr(addend), L.ptr(z), z.stride(0) if z is not None else 0,
             L.ptr(out), L.stream_ptr())
  return out


def gemm_wgrad(x, dy, out, *, m, n, k, bsum=None, side_w=None, side_aw=None, impl=0):
  """dW[m, n] += x[k, m]^T dy[k, n], plus (optional) bsum[n] += column sums of dy (the layer's bias gradient) and
  side_aw[m] += sum_r side_w[r] x[r, m] (weight gradient of a Dense(1) head on x) -- include/mnrf.h.

  One launch on the tensor-core path: the side sums come from the operand tiles the GEMM stages (the SIMT reference,
  impl=1, adds them in separate passes)."""
  lib = L.load()
  assert x.stride(-1) == 1 and dy.stride(-1) == 1 and out.stride(-1) == 1
  assert (side_w is None) == (side_aw is None)
  d = L.GemmDesc(L.GEMM_WGRAD, L.ACT_NONE, m, n, k, x.stride(0), dy.stride(0), out.stride(0), 0, 0, 0, 0, impl)
  _gemm_call(2.0 * m * n * k, lib.mnrf_gemm_wgrad, C.byref(d), L.ptr(x), L.ptr(dy), L.ptr(bsum),
             L.ptr(_f32(side_w)), L.ptr(side_aw), L.ptr(out), L.stream_ptr())
  return out


def gemm_plan(mode, a, b, out, *, m, n, k, act=L.ACT_NONE, bias=None, rowv=None, colv=None, mask=None,
              maskbits=None, colsum=None, mask_mod=0, addend=None, z=None, bsum=None, side_w=None, side_aw=None):
  """The tensor-core instance that gemm (or gemm_wgrad, with bsum / side_w / side_aw) launches for these arguments:
  a dict of the fields of mnrf_gemm_instance (include/mnrf.h).  Reads only shapes, strides and addresses, so the
  tensors may live on any device."""
  lib = L.load()
  def p(t):
    return None if t is None else C.c_void_p(t.data_ptr())
  def ld(t):
    return t.stride(0) if t is not None else 0
  d = L.GemmDesc(mode, act, m, n, k, a.stride(0), b.stride(0), out.stride(0), ld(mask), ld(maskbits), ld(addend),
                 mask_mod, 0)
  plan = L.GemmInstance()
  L.check(lib.mnrf_gemm_plan(C.byref(d), p(a), p(b), p(bias), p(rowv), p(colv), p(mask), p(maskbits), p(colsum),
                             p(addend), p(z), ld(z), p(out), p(bsum), p(side_w), p(side_aw), C.byref(plan)))
  return {name: int(getattr(plan, name)) for name, _ in L.GemmInstance._fields_}


def chain_desc(mode, m, layers, *, stream=None, stream_cols=0, head_w=None, head_b=None, head_out=None, head_n=1):
  """Descriptor of one layer-chained launch (include/mnrf.h mnrf_chain_desc).  head_w [head_n, 256] fp32, head_out
  [m, head_n]: the narrow head of the last layer's epilogue (head_n 1 or 4).  layers: list of dicts with
  w [256, ldw] bf16, optional bias / maskbits / colsum / out, n_stream, stream_col0, stream_kb0, n_res, res_kb0.
  The tensors must outlive the descriptor (the caller keeps them: level-state / weight buffers)."""
  d = L.ChainDesc()
  d.mode, d.num_layers, d.width, d.stream_cols, d.m = mode, len(layers), 256, stream_cols, m
  if stream is not None:
    assert stream.dtype == torch.bfloat16 and stream.stride(1) == 1
    d.stream, d.ldstream = stream.data_ptr(), stream.stride(0)
  if head_w is not None:
    assert head_w.is_contiguous() and head_w.numel() == head_n * 256 and head_out.is_contiguous()
    d.head_w, d.head_out, d.head_n = head_w.data_ptr(), head_out.data_ptr(), head_n
    d.head_b = head_b.data_ptr() if head_b is not None else None
  flops = 0.0
  for j, ly in enumerate(layers):
    c = d.layer[j]
    w = ly['w']
    assert w.dtype == torch.bfloat16 and w.stride(1) == 1
    c.w, c.ldw = w.data_ptr(), w.stride(0)
    for name in ('bias', 'colsum'):
      t = ly.get(name)
      setattr(c, name, t.data_ptr() if t is not None else None)
    mb = ly.get('maskbits')
    if mb is not None:
      assert mb.dtype == torch.int32 and mb.stride(1) == 1
      c.maskbits, c.ldmaskbits = mb.data_ptr(), mb.stride(0)
    out = ly.get('out')
    if out is not None:
      assert out.dtype == torch.bfloat16 and out.stride(1) == 1
      c.out, c.ldo = out.data_ptr(), out.stride(0)
    c.n_stream, c.stream_col0, c.stream_kb0 = ly.get('n_stream', 0), ly.get('stream_col0', 0), ly.get('stream_kb0', 0)
    c.n_res, c.res_kb0 = ly.get('n_res', 0), ly.get('res_kb0', 0)
    flops += 2.0 * m * 256 * 64 * (c.n_stream + c.n_res)
  return d, flops


def mlp_chain(desc):
  """One launch for a whole 256-wide trunk (forward) or its input-gradient chain (backward)."""
  lib = L.load()
  d, flops = desc
  _gemm_call(flops, lib.mnrf_mlp_chain, C.byref(d), L.stream_ptr())


def head_fwd(x, w_nk, bias, n_out, k, raw=None):
  lib = L.load()
  M = x.shape[0]
  if raw is None:
    raw = torch.empty(M, n_out, device=x.device)
  _count()
  L.check(lib.mnrf_head_fwd(M, k, n_out, L.ptr(x), x.stride(0), L.ptr(w_nk), L.ptr(bias),
                            L.ptr(raw), L.stream_ptr()))
  return raw


def head_bwd(x, w_nk, draw, n_out, k, dx=None, relu_mask=False, dw=None, db=None, dxsum=None, dw2=None, dw_split=0,
             dx_cols=0, dx2=None, act=L.ACT_NONE, z=None):
  """dw2 / dw_split: outputs [dw_split, n_out) put their weight gradient in dw2; dx_cols: dx and dxsum cover the
  first dx_cols columns only; dx2 [M, k - dx_cols]: the input gradient of the columns past dx_cols, unmasked
  (include/mnrf.h).  relu_mask: dx is masked by x > 0; z (with a smooth `act`, instead of relu_mask): dx *= a'(z), z
  the pre-activation of x."""
  lib = L.load()
  M = x.shape[0]
  if z is not None:
    assert not relu_mask and z.dtype == torch.bfloat16 and z.stride(-1) == 1
  else:
    act = L.ACT_RELU if relu_mask else L.ACT_NONE
  _count()
  L.check(lib.mnrf_head_bwd(M, k, n_out, L.ptr(x), x.stride(0), L.ptr(w_nk), L.ptr(_f32(draw)),
                            L.ptr(dx), dx.stride(0) if dx is not None else 0, act,
                            L.ptr(z), z.stride(0) if z is not None else 0, L.ptr(dw), L.ptr(dw2), int(dw_split),
                            L.ptr(db), L.ptr(dxsum), int(dx_cols), L.ptr(dx2), dx2.stride(0) if dx2 is not None else 0,
                            L.stream_ptr()))


def head_plan(x, w_nk, n_out, k, *, act=L.ACT_NONE, z=None, dx=None):
  """The kernel instances and launch shapes head_fwd and head_bwd run for these arguments (M = x.shape[0]): a dict
  of the fields of mnrf_head_instance (include/mnrf.h).  Reads only shapes and addresses, so the tensors may live
  on any device; raises MnrfError where head_bwd refuses the arguments."""
  lib = L.load()
  def p(t):
    return None if t is None else C.c_void_p(t.data_ptr())
  plan = L.HeadInstance()
  L.check(lib.mnrf_head_plan(x.shape[0], k, n_out, p(x), p(w_nk), act, p(z), p(dx), C.byref(plan)))
  return {name: int(getattr(plan, name)) for name, _ in L.HeadInstance._fields_}


def colsum(x, n, out):
  lib = L.load()
  _count()
  L.check(lib.mnrf_colsum(x.shape[0], n, L.ptr(x), x.stride(0), L.ptr(out), L.stream_ptr()))


def _cdesc(B, S, *, raydist_fn, opaque_background, density_bias, density_noise, rgb_activation,
           rgb_premultiplier, rgb_bias, rgb_padding, bg_const, rgb_mode=0):
  if rgb_activation not in L.RGB_ACT:
    raise ValueError(f'rgb_activation {rgb_activation!r} not supported by the CUDA path')
  return L.CompositeDesc(B, S, L.RAYDIST[raydist_fn], int(opaque_background), float(density_bias),
                         float(density_noise), L.RGB_ACT[rgb_activation], float(rgb_premultiplier),
                         float(rgb_bias), float(rgb_padding), float(bg_const), int(rgb_mode))


def composite_fwd(raw_density, raw_rgb, sdist, directions, near, far, *, cfg, density_noise=None,
                  bg_rgb=None, rgb_scale=None, raw_diffuse=None, raw_tint=None, want_samples=False,
                  want_extras=False):
  """compute_alpha_weights + volumetric_rendering.  cfg: kwargs of _cdesc."""
  lib = L.load()
  B, S = raw_density.shape
  dev = raw_density.device
  d = _cdesc(B, S, **cfg)
  d.ld_density, d.ld_rgb = _sample_ld(raw_density, 0), _sample_ld(raw_rgb, 3)
  weights = torch.empty(B, S, device=dev)
  rgb = torch.empty(B, 3, device=dev)
  dens = torch.empty(B, S, device=dev) if want_samples else None
  rgbs = torch.empty(B, S, 3, device=dev) if want_samples else None
  acc = torch.empty(B, device=dev) if want_extras else None
  dist = torch.empty(B, 4, device=dev) if want_extras else None
  _count()
  L.check(lib.mnrf_composite_fwd(C.byref(d), L.ptr(raw_density), L.ptr(raw_rgb),
                                 L.ptr(_f32(density_noise)), L.ptr(_f32(sdist)),
                                 L.ptr(_f32(directions)), L.ptr(_f32(near)), L.ptr(_f32(far)),
                                 L.ptr(_f32(bg_rgb)), L.ptr(_f32(rgb_scale)), L.ptr(_f32(raw_diffuse)),
                                 L.ptr(_f32(raw_tint)), L.ptr(weights), L.ptr(rgb),
                                 L.ptr(dens), L.ptr(rgbs), L.ptr(acc), L.ptr(dist), L.stream_ptr()))
  return dict(weights=weights, rgb=rgb, density=dens, rgb_samples=rgbs, acc=acc, dist=dist)


def point_rgb(raw_rgb, *, cfg, raw_diffuse=None, raw_tint=None, out=None):
  """The activated, padded colour of each row of raw_rgb [M, 3] (row stride from the tensor: a stacked head's
  [M, 4] output is read in place through its column view), without compositing -> fp32 [M, 3].  cfg: kwargs of
  _cdesc."""
  lib = L.load()
  M = raw_rgb.shape[0]
  assert raw_rgb.dtype == torch.float32 and raw_rgb.dim() == 2 and raw_rgb.shape[1] == 3 and raw_rgb.stride(1) == 1
  d = _cdesc(M, 1, **cfg)
  if out is None:
    out = torch.empty(M, 3, device=raw_rgb.device)
  _count()
  L.check(lib.mnrf_point_rgb(C.byref(d), M, L.ptr(raw_rgb), raw_rgb.stride(0), L.ptr(_f32(raw_diffuse)),
                             L.ptr(_f32(raw_tint)), L.ptr(_f32(out)), L.stream_ptr()))
  return out


def composite_bwd(raw_density, raw_rgb, sdist, directions, near, far, target_rgb, lossmult,
                  inv_denom, stats, *, cfg, loss_type, charb_padding, data_mult, distortion_mult,
                  interlevel_mult, sdist_fine=None, weights_fine=None, density_noise=None,
                  bg_rgb=None, rgb_scale=None, d_raw_density=None, d_raw_rgb=None, d_rgb_scale=None,
                  raw_diffuse=None, raw_tint=None, extra_dw=None, d_raw_diffuse=None, d_raw_tint=None,
                  data_mask=None, batch_rays=None):
  """Losses + compositing backward of one level; `data_mask` [B] (optional) weights each ray's data loss
  (robustnerf).  `batch_rays`: these B rays are one pass of a step over that many rays, which the distortion and
  interlevel means divide by (default B)."""
  lib = L.load()
  B, S = raw_density.shape
  dev = raw_density.device
  Sf = sdist_fine.shape[1] - 1 if sdist_fine is not None else 0
  d = L.LossDesc(_cdesc(B, S, **cfg), L.LOSS_TYPE[loss_type], float(charb_padding), float(data_mult),
                 float(distortion_mult), float(interlevel_mult), Sf,
                 lossmult.shape[-1] if lossmult.dim() > 1 else 1)
  if d_raw_density is None:
    d_raw_density = torch.empty(B, S, device=dev)
  if raw_rgb is not None and d_raw_rgb is None:
    d_raw_rgb = torch.empty(B, S, 3, device=dev)
  # the gradients share the raw values' sample spacing (one pair of strides in the descriptor)
  d.c.ld_density, d.c.ld_rgb = _sample_ld(raw_density, 0), _sample_ld(raw_rgb, 3)
  assert _sample_ld(d_raw_density, 0) == d.c.ld_density and (raw_rgb is None or _sample_ld(d_raw_rgb, 3) == d.c.ld_rgb)
  if data_mask is not None:
    assert data_mask.numel() == B
  _count()
  L.check(lib.mnrf_composite_bwd(
      C.byref(d), L.ptr(raw_density), L.ptr(raw_rgb), L.ptr(_f32(density_noise)), L.ptr(_f32(sdist)),
      L.ptr(_f32(directions)), L.ptr(_f32(near)), L.ptr(_f32(far)), L.ptr(_f32(bg_rgb)), L.ptr(_f32(rgb_scale)),
      L.ptr(_f32(raw_diffuse)), L.ptr(_f32(raw_tint)), L.ptr(_f32(extra_dw)), L.ptr(_f32(target_rgb)),
      L.ptr(_f32(lossmult)), L.ptr(_f32(inv_denom)), L.ptr(_f32(sdist_fine)), L.ptr(_f32(weights_fine)),
      L.ptr(_f32(data_mask)), L.ptr(d_raw_density), L.ptr(d_raw_rgb), L.ptr(d_rgb_scale), L.ptr(d_raw_diffuse),
      L.ptr(d_raw_tint), L.ptr(stats), int(B if batch_rays is None else batch_rays), L.stream_ptr()))
  return d_raw_density, d_raw_rgb


def robust_desc(num_rays, *, patch_size, inner_patch_size, filter_size, smoothed_inlier_quantile,
                inner_patch_inlier_quantile, enable):
  """mnrf_robust_desc of robustnerf.py's hyperparameters (the two thresholds are fl32(1 - quantile))."""
  return L.RobustDesc(int(num_rays), int(patch_size), int(inner_patch_size), int(filter_size), int(bool(enable)),
                      1.0 - float(smoothed_inlier_quantile), 1.0 - float(inner_patch_inlier_quantile))


def robust_mask(rgb, target, threshold, desc, *, mask=None, error=None, counts=None, stats=None, batch_rays=None):
  """robustnerf.robustnerf_mask for patch-major rays: returns (mask [B], error_per_pixel [B]).
  `threshold` is a device scalar; with `stats` (a row of >= 5 floats), stats[1:5] += the per-rank means of
  is_inlier_loss, has_inlier_neighbors, is_inlier_patch and mask, using `counts` (int32[5], zero, left zero).
  `batch_rays`: these B rays are one pass of a step over that many rays, and the means divide by it (default B)."""
  lib = L.load()
  B = rgb.shape[0]
  assert desc.num_rays == B and rgb.shape == (B, 3) and target.shape == (B, 3) and threshold.numel() == 1
  if mask is None:
    mask = torch.empty(B, device=rgb.device)
  if error is None:
    error = torch.empty(B, device=rgb.device)
  if stats is not None:
    assert counts is not None and counts.dtype == torch.int32 and counts.numel() >= 5
    assert stats.is_contiguous() and stats.numel() >= 5
  _count()
  L.check(lib.mnrf_robust_mask(C.byref(desc), L.ptr(_f32(rgb)), L.ptr(_f32(target)), L.ptr(_f32(threshold)),
                               L.ptr(mask), L.ptr(error), L.ptr(counts), L.ptr(stats),
                               int(B if batch_rays is None else batch_rays), L.stream_ptr()))
  return mask, error


def quantile(x, q, out=None):
  """out[0] = jnp.quantile(x, q) (method 'linear') of a flat fp32 tensor, on the device (one CTA)."""
  lib = L.load()
  x = _f32(x.reshape(-1))
  if out is None:
    out = torch.empty(1, device=x.device)
  _count()
  L.check(lib.mnrf_quantile(x.numel(), float(q), L.ptr(x), L.ptr(out), L.stream_ptr()))
  return out


def clip_adam(params, grads, mu, nu, scratch, *, step, lr, beta1, beta2, eps, grad_max_val,
              grad_max_norm, grad_scale=1.0, dyn=None):
  lib = L.load()
  d = L.AdamDesc(params.numel(), float(grad_max_val), float(grad_max_norm), float(lr), float(beta1),
                 float(beta2), float(eps), int(step), float(grad_scale))
  _count(2 if grad_max_norm > 0 else 1)
  L.check(lib.mnrf_clip_adam(C.byref(d), L.ptr(params), L.ptr(grads), L.ptr(mu), L.ptr(nu),
                             L.ptr(scratch), L.ptr(dyn), L.stream_ptr()))


def pack_table(layers, device):
  """Device table for pack_weights_batched: layers = [(master[in_pad,out], w_nk or None, w_kn or None)]."""
  import ctypes
  import numpy as np
  items = (L.PackItem * len(layers))()
  tile = 0
  for i, (master, w_nk, w_kn) in enumerate(layers):
    in_pad, out = master.shape
    items[i] = L.PackItem(master.data_ptr(), w_nk.data_ptr() if w_nk is not None else None,
                          w_kn.data_ptr() if w_kn is not None else None, in_pad, out, tile, 0)
    tile += ((out + 31) // 32) * ((in_pad + 31) // 32)
  raw = np.frombuffer(ctypes.string_at(ctypes.addressof(items), ctypes.sizeof(items)), dtype=np.uint8).copy()
  return torch.from_numpy(raw).to(device), len(layers), tile


def pack_weights_batched(table):
  lib = L.load()
  dev_items, count, tiles = table
  _count()
  L.check(lib.mnrf_pack_weights_batched(count, L.ptr(dev_items), tiles, L.stream_ptr()))


def refdir_desc(M, S, *, use_pred_normals, use_density_normals, use_reflections, use_ide, use_n_dot_v,
                use_roughness, deg_view, ide_n, roughness_bias, ld, col0, col_end):
  return L.RefdirDesc(M, S, int(use_pred_normals), int(use_density_normals), int(use_reflections),
                      int(use_ide), int(use_n_dot_v), int(use_roughness), deg_view, ide_n,
                      float(roughness_bias), ld, col0, col_end)


def refdir_fwd(desc, ide_mat, ide_ml, grad_pred, raw_rough, raw_grad_density, viewdirs, normals_pred,
               normals, roughness, slab, orient_mult=0.0, prednorm_mult=0.0, orient_on_pred=True,
               extra_dw=None):
  lib = L.load()
  _count()
  L.check(lib.mnrf_refdir_fwd(C.byref(desc), L.ptr(ide_mat), L.ptr(ide_ml), L.ptr(_f32(grad_pred)),
                              L.ptr(_f32(raw_rough)), L.ptr(_f32(raw_grad_density)), L.ptr(_f32(viewdirs)),
                              L.ptr(normals_pred), L.ptr(normals), L.ptr(roughness), L.ptr(slab),
                              float(orient_mult), float(prednorm_mult), int(orient_on_pred),
                              L.ptr(extra_dw), L.stream_ptr()))


def refdir_bwd(desc, ide_mat, ide_ml, grad_pred, raw_rough, raw_grad_density, viewdirs, weights, d_slab,
               orient_mult, prednorm_mult, orient_on_pred, d_raw_density, d_raw_diffuse, d_raw_tint,
               d_grad_pred, d_raw_rough, d_raw_grad_density, stats):
  lib = L.load()
  _count()
  L.check(lib.mnrf_refdir_bwd(C.byref(desc), L.ptr(ide_mat), L.ptr(ide_ml), L.ptr(_f32(grad_pred)),
                              L.ptr(_f32(raw_rough)), L.ptr(_f32(raw_grad_density)), L.ptr(_f32(viewdirs)),
                              L.ptr(_f32(weights)), L.ptr(d_slab), d_slab.stride(0), float(orient_mult),
                              float(prednorm_mult), int(orient_on_pred), L.ptr(_f32(d_raw_density)),
                              L.ptr(_f32(d_raw_diffuse)), L.ptr(_f32(d_raw_tint)), L.ptr(d_grad_pred),
                              L.ptr(d_raw_rough), L.ptr(d_raw_grad_density), L.ptr(stats), L.stream_ptr()))


def normals_fwd(M, S, grad_pred, raw_grad_density, viewdirs, normals_pred, normals, orient_mult=0.0,
                prednorm_mult=0.0, orient_on_pred=True, extra_dw=None):
  """Colourless normals stage (include/mnrf.h mnrf_normals_fwd): normals of an MLP without a colour branch."""
  lib = L.load()
  _count()
  L.check(lib.mnrf_normals_fwd(M, S, L.ptr(_f32(grad_pred)), L.ptr(_f32(raw_grad_density)), L.ptr(_f32(viewdirs)),
                               L.ptr(_f32(normals_pred)), L.ptr(_f32(normals)), float(orient_mult),
                               float(prednorm_mult), int(orient_on_pred), L.ptr(_f32(extra_dw)), L.stream_ptr()))


def normals_bwd(M, S, grad_pred, raw_grad_density, viewdirs, weights, orient_mult, prednorm_mult, orient_on_pred,
                d_raw_density, d_grad_pred, d_raw_grad_density, head_grads=None, stats=None, d_raw_rgb=None):
  """d_raw_rgb (with head_grads): the gradient of an rgb head on the same trunk, written to head_grads[:, 4:7]."""
  lib = L.load()
  ld_raw = _sample_ld(d_raw_density, 0)
  assert d_raw_rgb is None or _sample_ld(d_raw_rgb, 3) == ld_raw
  if head_grads is not None:
    assert head_grads.dtype == torch.bfloat16 and head_grads.stride(1) == 1
  _count()
  L.check(lib.mnrf_normals_bwd(M, S, L.ptr(_f32(grad_pred)), L.ptr(_f32(raw_grad_density)), L.ptr(_f32(viewdirs)),
                               L.ptr(_f32(weights)), float(orient_mult), float(prednorm_mult), int(orient_on_pred),
                               L.ptr(d_raw_density), L.ptr(d_raw_rgb), ld_raw, L.ptr(_f32(d_grad_pred)),
                               L.ptr(_f32(d_raw_grad_density)),
                               L.ptr(head_grads), head_grads.stride(0) if head_grads is not None else 0,
                               L.ptr(stats), L.stream_ptr()))


def outer_mask(rowv, colv, maskbits, out, *, rows, n, mask_mod=0):
  lib = L.load()
  _count()
  L.check(lib.mnrf_outer_mask(rows, n, mask_mod, L.ptr(_f32(rowv)), L.ptr(_f32(colv)), L.ptr(maskbits),
                              maskbits.stride(0) if maskbits is not None else 0, L.ptr(out), out.stride(0),
                              L.stream_ptr()))


def act_tangent_bwd(act, z, t_adj, u, du, g, *, accumulate=False):
  """One trunk layer of the density-normal backward through a smooth activation (include/mnrf.h): du = a'(z) T per
  tangent stream, g (+)= a''(z) sum_s T_s u_s.  z, g [M, n]; t_adj, u, du [3M, n] (du may be t_adj); bf16."""
  lib = L.load()
  M, n = z.shape
  for t in (z, t_adj, u, du, g):
    assert t.dtype == torch.bfloat16 and t.stride(-1) == 1
  assert t_adj.shape[0] == u.shape[0] == du.shape[0] == 3 * M
  _count()
  L.check(lib.mnrf_act_tangent_bwd(M, n, act, L.ptr(z), z.stride(0), L.ptr(t_adj), t_adj.stride(0), L.ptr(u),
                                   u.stride(0), L.ptr(du), du.stride(0), L.ptr(g), g.stride(0), int(accumulate),
                                   L.stream_ptr()))
