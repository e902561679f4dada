"""Restatement of csrc/mesh_trace.cu (mnrf_mesh_bvh, mnrf_mesh_trace) for the tests.

The BVH: face boxes, centroids, Morton keys, Karras topology and fitted boxes in numpy fp32 / integer arithmetic,
bit for bit what the kernels compute (no rounding happens in the tree; the centroid and the cell of each axis are
single IEEE operations).  The trace: a brute-force closest hit over every face in fp64 (Moeller-Trumbore) with the
(t, face) tie rule, and for each ray whether it is exempt from an exact comparison: within EPS_BARY of a face's edge
(in barycentric units), within EPS_T (relative) of a second candidate t or of near / far, or nearly parallel to a
face it (nearly) hits.
"""
import numpy as np
import torch

EPS_BARY = 1e-4
EPS_T = 1e-4
EPS_COS = 1e-3


def face_boxes(vertices, faces):
  """(boxes [F, 6] fp32 = (min xyz, max xyz), centroids [F, 3] fp32 = ((v0 + v1) + v2) / 3)."""
  v = np.asarray(vertices, np.float32)
  p = v[np.asarray(faces, np.int64)]                                   # [F, 3, 3]
  boxes = np.concatenate([p.min(1), p.max(1)], 1).astype(np.float32)
  c = ((p[:, 0] + p[:, 1]) + p[:, 2]) / np.float32(3)
  return boxes, c.astype(np.float32)


def _expand_bits10(x):
  x = x.astype(np.uint64)
  x = (x | (x << np.uint64(16))) & np.uint64(0x030000FF)
  x = (x | (x << np.uint64(8))) & np.uint64(0x0300F00F)
  x = (x | (x << np.uint64(4))) & np.uint64(0x030C30C3)
  x = (x | (x << np.uint64(2))) & np.uint64(0x09249249)
  return x


def morton_keys(centroids):
  """Unsorted keys [F] int64: morton << 32 | face, cells floor(clamp((c - lo) / (hi - lo), 0, 1) * 1024) <= 1023."""
  c = np.asarray(centroids, np.float32)
  lo, hi = c.min(0), c.max(0)
  ext = (hi - lo).astype(np.float32)
  with np.errstate(divide='ignore', invalid='ignore'):
    t = np.where(ext > 0, (c - lo) / np.where(ext > 0, ext, np.float32(1)), np.float32(0)).astype(np.float32)
  t = np.where(t >= 0, np.where(t <= 1, t, np.float32(1)), np.float32(0)).astype(np.float32)
  cell = np.minimum((t * np.float32(1024)).astype(np.uint32), 1023)
  m = (_expand_bits10(cell[:, 0]) << np.uint64(2)) | (_expand_bits10(cell[:, 1]) << np.uint64(1)) | \
      _expand_bits10(cell[:, 2])
  return ((m << np.uint64(32)) | np.arange(len(c), dtype=np.uint64)).astype(np.int64)


def _clz64(x):
  x = int(x)
  return 64 - x.bit_length()


def karras_topology(sorted_keys):
  """(children [n - 1, 2] int32, parent [2 n - 1] int32) of Karras's tree over sorted unique keys; internal nodes
  0 .. n - 2 (0 the root), leaf k at n - 1 + k."""
  k = [int(x) for x in sorted_keys]
  n = len(k)

  def delta(i, j):
    return -1 if j < 0 or j >= n else _clz64(k[i] ^ k[j])
  children = np.zeros((max(n - 1, 0), 2), np.int32)
  parent = np.full(2 * n - 1, -1, np.int32)
  for i in range(n - 1):
    d = 1 if delta(i, i + 1) > delta(i, i - 1) else -1
    dmin = delta(i, i - d)
    lmax = 2
    while delta(i, i + lmax * d) > dmin:
      lmax *= 2
    l, t = 0, lmax // 2
    while t >= 1:
      if delta(i, i + (l + t) * d) > dmin:
        l += t
      t //= 2
    j = i + l * d
    dnode = delta(i, j)
    s, t = 0, l
    while True:
      t = (t + 1) // 2
      if delta(i, i + (s + t) * d) > dnode:
        s += t
      if t <= 1:
        break
    gamma = i + s * d + min(d, 0)
    left = n - 1 + gamma if min(i, j) == gamma else gamma
    right = n - 1 + gamma + 1 if max(i, j) == gamma + 1 else gamma + 1
    children[i] = left, right
    parent[left] = parent[right] = i
  return children, parent


def build(vertices, faces):
  """Everything mnrf_mesh_bvh writes, as numpy: dict(keys (sorted), leaf_face, children, parent, child_boxes
  [F - 1, 2, 6] fp32, nodes [F - 1, 16] fp32 bits as the kernel lays them out)."""
  boxes, cent = face_boxes(vertices, faces)
  F = len(boxes)
  keys = np.sort(morton_keys(cent)) if F > 1 else np.zeros(F, np.int64)
  leaf_face = (keys & 0xffffffff).astype(np.int32) if F > 1 else np.zeros(F, np.int32)
  children, parent = karras_topology(keys) if F > 1 else (np.zeros((0, 2), np.int32), np.full(F, -1, np.int32))
  node_box = np.zeros((2 * F - 1, 6), np.float32)
  node_box[F - 1:] = boxes[leaf_face]
  # internal nodes in decreasing depth: a child is fitted before its parent
  depth = node_depths(parent)
  for i in sorted(range(F - 1), key=lambda i: -depth[i]):
    l, r = children[i]
    node_box[i, :3] = np.minimum(node_box[l, :3], node_box[r, :3])
    node_box[i, 3:] = np.maximum(node_box[l, 3:], node_box[r, 3:])
  child_boxes = node_box[children] if F > 1 else np.zeros((0, 2, 6), np.float32)
  nodes = np.zeros((max(F - 1, 0), 16), np.float32)
  nodes[:, :12] = child_boxes.reshape(-1, 12)
  nodes.view(np.int32)[:, 12:14] = children
  return dict(keys=keys, leaf_face=leaf_face, children=children, parent=parent, child_boxes=child_boxes,
              nodes=nodes, node_box=node_box, depth=depth)


def node_depths(parent):
  """Depth of every node (root 0) from the parent array."""
  parent = np.asarray(parent)
  depth = np.full(len(parent), -1, np.int64)
  for v in range(len(parent)):
    path = []
    u = v
    while depth[u] < 0 and parent[u] >= 0:
      path.append(u)
      u = parent[u]
    if depth[u] < 0:
      depth[u] = 0
    for w in reversed(path):
      depth[w] = depth[parent[w]] + 1
  return depth


def brute_force(vertices, faces, origins, directions, near, far, chunk=4096, device='cpu', face_block=8192):
  """fp64 closest hit of every ray over every face (Moeller-Trumbore), the least (t, face) with near <= t <= far.
  Returns numpy (face [N] int64, -1 for a miss; t [N] fp64, inf for a miss; bary [N, 2]; exempt [N] bool)."""
  dd = dict(device=device, dtype=torch.float64)
  v = torch.as_tensor(np.asarray(vertices, np.float64), **dd)
  f = torch.as_tensor(np.asarray(faces, np.int64), device=device)
  p0, p1, p2 = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
  e1, e2 = p1 - p0, p2 - p0
  scale = torch.linalg.norm(e1, dim=-1) * torch.linalg.norm(e2, dim=-1)
  O = torch.as_tensor(np.asarray(origins, np.float64), **dd)
  D = torch.as_tensor(np.asarray(directions, np.float64), **dd)
  NE = torch.as_tensor(np.asarray(near, np.float64).reshape(-1), **dd)
  FA = torch.as_tensor(np.asarray(far, np.float64).reshape(-1), **dd)
  N, F = O.shape[0], f.shape[0]
  out_face = torch.full((N,), -1, device=device, dtype=torch.int64)
  out_t = torch.full((N,), float('inf'), **dd)
  out_b = torch.zeros(N, 2, **dd)
  exempt = torch.zeros(N, device=device, dtype=torch.bool)
  inf = torch.tensor(float('inf'), **dd)
  for r0 in range(0, N, chunk):
    o, d, ne, fa = O[r0:r0 + chunk], D[r0:r0 + chunk], NE[r0:r0 + chunk], FA[r0:r0 + chunk]
    n = o.shape[0]
    best_t = torch.full((n,), float('inf'), **dd)
    best_f = torch.full((n,), -1, device=device, dtype=torch.int64)
    best_b = torch.zeros(n, 2, **dd)
    second_t = torch.full((n,), float('inf'), **dd)
    ex = torch.zeros(n, device=device, dtype=torch.bool)
    dn = torch.linalg.norm(d, dim=-1)
    for f0 in range(0, F, face_block):
      sl = slice(f0, f0 + face_block)
      pvec = torch.cross(d[:, None, :].expand(-1, e2[sl].shape[0], -1), e2[sl][None].expand(n, -1, -1), dim=-1)
      det = (e1[sl][None] * pvec).sum(-1)
      tvec = o[:, None, :] - p0[sl][None]
      with np.errstate(all='ignore'):
        inv = 1.0 / det
        u = (tvec * pvec).sum(-1) * inv
        q = torch.cross(tvec, e1[sl][None].expand(n, -1, -1), dim=-1)
        w = (d[:, None, :] * q).sum(-1) * inv
        t = (e2[sl][None] * q).sum(-1) * inv
      b0 = 1 - u - w
      mb = torch.minimum(torch.minimum(u, w), b0)
      cosang = det.abs() / (dn[:, None] * scale[sl][None]).clamp_min(1e-300)
      inside = (mb >= 0) & (det != 0) & torch.isfinite(t)
      tl = torch.where(inside & (t >= ne[:, None]) & (t <= fa[:, None]), t, inf)
      # exemptions: near an edge with t in (or near) the interval; nearly parallel and nearly inside
      tol_t = EPS_T * torch.maximum(t.abs(), torch.ones_like(t))
      in_range = (t >= ne[:, None] - tol_t) & (t <= fa[:, None] + tol_t) & torch.isfinite(t)
      ex |= ((mb.abs() < EPS_BARY) & in_range).any(1)
      ex |= ((cosang < EPS_COS) & (mb > -0.01) & in_range).any(1)
      ex |= ((det == 0) & (mb > -0.01)).any(1)
      # near / far cut-offs
      ex |= (inside & (((t - ne[:, None]).abs() < tol_t) | ((t - fa[:, None]).abs() < tol_t))).any(1)
      # candidate t values of this block against the running best
      vals, idx = torch.topk(tl, k=min(2, tl.shape[1]), dim=1, largest=False)
      cand_t = torch.cat([best_t[:, None], second_t[:, None], vals], 1)
      cand_f = torch.cat([best_f[:, None], best_f[:, None] * 0 - 1, idx + f0], 1)
      cand_b = torch.cat([best_b[:, None], best_b[:, None],
                          torch.stack([u.gather(1, idx), w.gather(1, idx)], -1)], 1)
      # keep the two least t; ties by face index (stable sort on t after sorting by face)
      big = torch.where(cand_f < 0, torch.full_like(cand_f, 1 << 40), cand_f)
      order = torch.argsort(big, dim=1, stable=True)
      ct, cf, cb = cand_t.gather(1, order), cand_f.gather(1, order), cand_b.gather(1, order[..., None].expand(-1, -1, 2))
      order = torch.argsort(ct, dim=1, stable=True)
      ct, cf = ct.gather(1, order), cf.gather(1, order)
      cb = cb.gather(1, order[..., None].expand(-1, -1, 2))
      best_t, best_f, best_b = ct[:, 0], torch.where(torch.isfinite(ct[:, 0]), cf[:, 0], -1), cb[:, 0]
      second_t = ct[:, 1]
    tie = torch.isfinite(second_t) & ((second_t - best_t).abs() < EPS_T * torch.maximum(best_t.abs(),
                                                                                         torch.ones_like(best_t)))
    out_face[r0:r0 + n], out_t[r0:r0 + n], out_b[r0:r0 + n] = best_f, best_t, best_b
    exempt[r0:r0 + n] = ex | tie
  return out_face.cpu().numpy(), out_t.cpu().numpy(), out_b.cpu().numpy(), exempt.cpu().numpy()
