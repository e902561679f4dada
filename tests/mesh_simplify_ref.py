"""numpy restatement of mesh simplification by quadric edge collapse (mesh.simplify_mesh and the kernels of
csrc/mesh.cu it launches) for the CPU and GPU tests.  Every floating-point expression is the kernel's, operation
for operation, in fp64 (the kernels are compiled without FMA contraction), and every per-vertex sum runs
sequentially over the CSR position, so the GPU's results can be compared bit for bit.  Loops are vectorised over
vertices, edges or faces; none of their results depends on the order of those."""
import numpy as np

BOUNDARY_WEIGHT = 1000.0
DET_REL = 1e-10
MAX_VALENCE = 24
NO_KEY = np.uint64(0xFFFFFFFFFFFFFFFF)


def _cross(a, b):
  return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                   a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _dot(a, b):
  return a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1] + a[..., 2] * b[..., 2]


def _f32(x):
  return x.astype(np.float32).astype(np.float64)


def topology(faces, V):
  """(edges [E, 2] int32, edge_off [E + 1], edge_face [3F] int32, vf_off [V + 1], vf_face [3F] int32), as
  mesh.mesh_topology builds them."""
  f = np.asarray(faces, np.int64).reshape(-1, 3)
  corner = f.reshape(-1)
  other = f[:, [1, 2, 0]].reshape(-1)
  key = np.minimum(corner, other) * V + np.maximum(corner, other)
  perm = np.argsort(key, kind='stable')
  uniq, counts = np.unique(key[perm], return_counts=True)
  edges = np.stack([uniq // V, uniq % V], 1).astype(np.int32)
  edge_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
  vperm = np.argsort(corner, kind='stable')
  vf_off = np.concatenate([[0], np.cumsum(np.bincount(corner, minlength=V))]).astype(np.int64)
  return edges, edge_off, (perm // 3).astype(np.int32), vf_off, (vperm // 3).astype(np.int32)


def _padded(off, items, width=None):
  """CSR -> [rows, width] table of its items, -1 where a row is shorter."""
  deg = np.diff(off)
  width = int(deg.max(initial=0)) if width is None else width
  table = np.full((len(deg), max(width, 1)), -1, np.int64)
  row = np.repeat(np.arange(len(deg)), deg)
  col = np.arange(len(items)) - np.repeat(off[:-1], deg)
  m = col < width
  table[row[m], col[m]] = items[m]
  return table


def _plane_terms(u, d, w):
  a, b, c = u[..., 0], u[..., 1], u[..., 2]
  return np.stack([w * (a * a), w * (a * b), w * (a * c), w * (a * d), w * (b * b), w * (b * c), w * (b * d),
                   w * (c * c), w * (c * d), w * (d * d)], -1)


def _face_planes(P, f):
  """Unit normals, twice the areas and nonzero-area flags of faces f [F, 3]."""
  p0, p1, p2 = P[f[:, 0]], P[f[:, 1]], P[f[:, 2]]
  n = _cross(p1 - p0, p2 - p0)
  ln = np.sqrt(_dot(n, n))
  ok = ln > 0
  with np.errstate(invalid='ignore', divide='ignore'):
    u = n / ln[:, None]
  return u, ln, ok


def _accumulate(q, table, terms, valid):
  """q[v] += terms[table[v, k]] for k in order, where valid."""
  for k in range(table.shape[1]):
    t = table[:, k]
    m = (t >= 0) & valid[np.maximum(t, 0)]
    q = np.where(m[:, None], q + terms[np.maximum(t, 0)], q)
  return q


def boundary(topo, V):
  edges, edge_off, edge_face, _, _ = topo
  idx = np.flatnonzero(np.diff(edge_off) == 1)
  be = edges[idx].astype(np.int64)
  bf = edge_face[edge_off[idx]].astype(np.int64)
  B = len(idx)
  ends = be.T.reshape(-1)
  own = np.tile(np.arange(B), 2)
  order = np.argsort(ends * max(B, 1) + own)
  vb_off = np.concatenate([[0], np.cumsum(np.bincount(ends, minlength=V))]).astype(np.int64)
  return be, bf, vb_off, own[order]


def quadrics(vertices, faces, topo):
  """[V, 10] fp64: mnrf_mesh_quadrics."""
  P = np.asarray(vertices, np.float32).astype(np.float64)
  f = np.asarray(faces, np.int64).reshape(-1, 3)
  V = len(P)
  _, _, _, vf_off, vf_face = topo
  u, ln, ok = _face_planes(P, f)
  d = -_dot(u, P[f[:, 0]])
  terms = _plane_terms(u, d, 0.5 * ln)
  q = _accumulate(np.zeros((V, 10)), _padded(vf_off, vf_face.astype(np.int64)), terms, ok)
  be, bf, vb_off, vb_edge = boundary(topo, V)
  if len(be):
    x = P[be[:, 0]]
    ev = P[be[:, 1]] - x
    m = _cross(ev, u[bf])
    ml = np.sqrt(_dot(m, m))
    bok = ok[bf] & (ml > 0)
    with np.errstate(invalid='ignore', divide='ignore'):
      mu = m / ml[:, None]
    bterms = _plane_terms(mu, -_dot(mu, x), BOUNDARY_WEIGHT * _dot(ev, ev))
    q = _accumulate(q, _padded(vb_off, vb_edge), bterms, bok)
  return q


def quadric_eval(q, v):
  x, y, z = v[..., 0], v[..., 1], v[..., 2]
  return x * (q[..., 0] * x + 2.0 * (q[..., 1] * y + q[..., 2] * z + q[..., 3])) + \
      y * (q[..., 4] * y + 2.0 * (q[..., 5] * z + q[..., 6])) + z * (q[..., 7] * z + 2.0 * q[..., 8]) + q[..., 9]


def _positions(P, Q, a, b):
  """(position fp64 of fp32 values [E, 3], cost [E]) of collapsing each edge (a, b)."""
  q = Q[a] + Q[b]
  pa, pb = P[a], P[b]
  c00 = q[:, 4] * q[:, 7] - q[:, 5] * q[:, 5]
  c01 = q[:, 5] * q[:, 2] - q[:, 1] * q[:, 7]
  c02 = q[:, 1] * q[:, 5] - q[:, 4] * q[:, 2]
  c11 = q[:, 0] * q[:, 7] - q[:, 2] * q[:, 2]
  c12 = q[:, 1] * q[:, 2] - q[:, 0] * q[:, 5]
  c22 = q[:, 0] * q[:, 4] - q[:, 1] * q[:, 1]
  det = q[:, 0] * c00 + q[:, 1] * c01 + q[:, 2] * c02
  A = np.abs(q)
  s = np.fmax(np.fmax(np.fmax(A[:, 0], A[:, 1]), np.fmax(A[:, 2], A[:, 4])), np.fmax(A[:, 5], A[:, 7]))
  mid = (pa + pb) * 0.5
  ev = pb - pa
  solved = np.abs(det) > DET_REL * (s * s * s)
  with np.errstate(invalid='ignore', divide='ignore', over='ignore'):
    x = np.stack([-(c00 * q[:, 3] + c01 * q[:, 6] + c02 * q[:, 8]) / det,
                  -(c01 * q[:, 3] + c11 * q[:, 6] + c12 * q[:, 8]) / det,
                  -(c02 * q[:, 3] + c12 * q[:, 6] + c22 * q[:, 8]) / det], -1)
    dm = x - mid
    solved &= _dot(dm, dm) <= _dot(ev, ev)
    ps = _f32(np.where(solved[:, None], x, 0.0))
  cs = quadric_eval(q, ps)
  p, c = pa, quadric_eval(q, pa)
  cb = quadric_eval(q, pb)
  p, c = np.where((cb < c)[:, None], pb, p), np.where(cb < c, cb, c)
  pm = _f32(mid)
  cm = quadric_eval(q, pm)
  p, c = np.where((cm < c)[:, None], pm, p), np.where(cm < c, cm, c)
  p, c = np.where(solved[:, None], ps, p), np.where(solved, cs, c)
  return p, np.where(c > 0.0, c, 0.0)


def _keeps_orientation(P, N, fid, corners, frm, p):
  """Faces fid [...] with corners [..., 3] and normals N[fid]; frm [...] the corner that moves to p [..., 3]."""
  D = np.where((corners == frm[..., None])[..., None], p[..., None, :], P[corners])
  n = N[fid]
  m = _cross(D[..., 1, :] - D[..., 0, :], D[..., 2, :] - D[..., 0, :])
  mzero = (m == 0).all(-1)
  nzero = (n == 0).all(-1)
  return ~mzero & (nzero | (_dot(m, n) > 0))


def edge_cost(vertices, faces, Q, topo):
  """(keys [E] uint64, positions [E, 3] fp32): mnrf_mesh_edge_cost."""
  P = np.asarray(vertices, np.float32).astype(np.float64)
  f = np.asarray(faces, np.int64).reshape(-1, 3)
  V = len(P)
  edges, edge_off, edge_face, vf_off, vf_face = topo
  E = len(edges)
  a, b = edges[:, 0].astype(np.int64), edges[:, 1].astype(np.int64)
  p, cost = _positions(P, Q, a, b)
  cnt = np.diff(edge_off)
  bnd = np.zeros(V, bool)
  nm = np.zeros(V, bool)
  bnd[edges[cnt == 1].reshape(-1)] = True
  nm[edges[cnt > 2].reshape(-1)] = True
  deg = np.diff(vf_off)
  ok = ((cnt == 1) | (cnt == 2)) & ~nm[a] & ~nm[b] & ~((cnt == 2) & bnd[a] & bnd[b]) & (deg[a] <= MAX_VALENCE) & \
      (deg[b] <= MAX_VALENCE) & (deg[a] + deg[b] - cnt > cnt)
  idx = np.flatnonzero(ok)
  if len(idx):
    ea, eb, ep = a[idx], b[idx], p[idx]
    s0 = edge_off[idx]

    def third(fc):
      c = f[fc]
      m = (c != ea[:, None]) & (c != eb[:, None])
      return np.where(m.any(-1), c[np.arange(len(c)), np.argmax(m, -1)], -1)
    apex0 = third(edge_face[s0])
    apex1 = np.where(cnt[idx] == 2, third(edge_face[np.minimum(s0 + 1, len(edge_face) - 1)]), -1)
    VF = _padded(vf_off, vf_face.astype(np.int64), int(max(deg[ea].max(), deg[eb].max())))
    FA, FB = VF[ea], VF[eb]                                     # [n, K]
    CA = np.where((FA >= 0)[..., None], f[np.maximum(FA, 0)], -2)  # [n, K, 3]
    CB = np.where((FB >= 0)[..., None], f[np.maximum(FB, 0)], -2)
    va, vb = ea[:, None, None], eb[:, None, None]
    m = (CA != va) & (CA != vb)
    first = np.argmax(m, -1)
    x = np.where(m.any(-1), np.take_along_axis(CA, first[..., None], -1)[..., 0], -1)
    m2 = m.copy()
    np.put_along_axis(m2, first[..., None], False, -1)
    y = np.where(m2.any(-1), np.take_along_axis(CA, np.argmax(m2, -1)[..., None], -1)[..., 0], -1)
    with_b = (CA == vb).any(-1)
    valid_a = FA >= 0
    nb_b = CB.reshape(len(idx), 1, -1)

    def neighbour_of_b(z):
      return (z[..., None] == nb_b).any(-1)
    ap0, ap1 = apex0[:, None], apex1[:, None]
    bad = valid_a & (x >= 0) & (x != ap0) & (x != ap1) & neighbour_of_b(x)
    bad |= valid_a & (y >= 0) & (y != ap0) & (y != ap1) & neighbour_of_b(y)
    # a face (b, x, y) for a face (a, x, y): the pairs of other corners, as keys min * V + max
    mb = (CB != vb) & (CB >= 0)
    bx = np.where(mb, CB, V).min(-1)
    by = np.where(mb, CB, -1).max(-1)
    pb_key = np.where((FB >= 0) & (mb.sum(-1) == 2), bx * V + by, -1)
    pa_key = np.where(valid_a & ~with_b & (y >= 0), np.minimum(x, y) * V + np.maximum(x, y), -2)
    bad |= (pa_key[:, :, None] == pb_key[:, None, :]).any(-1)
    N = _cross(P[f[:, 1]] - P[f[:, 0]], P[f[:, 2]] - P[f[:, 0]])
    fold = bad.any(-1)
    with_a = (CB == ea[:, None, None]).any(-1)
    for moved, Fm, Cm, need in ((ea, FA, CA, valid_a & ~with_b & (y >= 0)), (eb, FB, CB, (FB >= 0) & ~with_a)):
      r, k = np.nonzero(need)
      flips = ~_keeps_orientation(P, N, Fm[r, k], Cm[r, k], moved[r], ep[r])
      fold |= np.bincount(r[flips], minlength=len(idx)) > 0
    ok[idx] = ~fold
  keys = np.full(E, NO_KEY, np.uint64)
  bits = cost.astype(np.float32).view(np.uint32).astype(np.uint64)
  keys[ok] = (bits[ok] << np.uint64(32)) | np.arange(E, dtype=np.uint64)[ok]
  return keys, p.astype(np.float32)


def select(faces, edges, keys, V):
  """selected [E] bool: mnrf_mesh_collapse_select."""
  f = np.asarray(faces, np.int64).reshape(-1, 3)
  valid = keys != NO_KEY
  vmin = np.full(V, NO_KEY, np.uint64)
  for c in range(2):
    np.minimum.at(vmin, edges[valid, c], keys[valid])
  fmin = np.minimum(vmin[f[:, 0]], np.minimum(vmin[f[:, 1]], vmin[f[:, 2]]))
  rmin = np.full(V, NO_KEY, np.uint64)
  for c in range(3):
    np.minimum.at(rmin, f[:, c], fmin)
  return valid & (rmin[edges[:, 0]] == keys) & (rmin[edges[:, 1]] == keys)


def budget(keys, sel, edge_off, room):
  """The edges a round collapses: the longest prefix in key order of the selected ones removing at most `room`
  faces -> (edge ids, faces removed)."""
  ids = np.flatnonzero(sel)
  ids = ids[np.argsort(keys[ids])]
  removed = np.cumsum(edge_off[ids + 1] - edge_off[ids])
  keep = removed <= room
  return ids[keep], int(removed[keep][-1]) if keep.any() else 0


def apply(collapse_ids, vertices, Q, normals, faces, topo, positions):
  """mnrf_mesh_collapse_apply, then the compaction of the dead faces -> (vertices, Q, normals, faces) new arrays."""
  edges, edge_off, edge_face, vf_off, vf_face = topo
  v, Q, f = vertices.copy(), Q.copy(), np.asarray(faces, np.int64).reshape(-1, 3).copy()
  n = None if normals is None else normals.copy()
  a, b = edges[collapse_ids, 0].astype(np.int64), edges[collapse_ids, 1].astype(np.int64)
  p = positions[collapse_ids].astype(np.float64)
  P = vertices.astype(np.float64)
  if n is not None:
    pa = P[a]
    ev = P[b] - pa
    el2 = _dot(ev, ev)
    with np.errstate(invalid='ignore', divide='ignore'):
      t = np.where(el2 > 0.0, _dot(p - pa, ev) / el2, 0.0)
    t = np.minimum(np.maximum(t, 0.0), 1.0)[:, None]
    na, nb = normals[a].astype(np.float64), normals[b].astype(np.float64)
    nn = (1.0 - t) * na + t * nb
    ln = np.sqrt(_dot(nn, nn))
    with np.errstate(invalid='ignore', divide='ignore'):
      out = (nn / ln[:, None]).astype(np.float32)
    n[a] = np.where((ln > 0.0)[:, None], out, normals[a])
  v[a] = positions[collapse_ids]
  Q[a] = Q[a] + Q[b]
  alive = np.ones(len(f), bool)
  for k in range(2):
    s = edge_off[collapse_ids] + k
    m = s < edge_off[collapse_ids + 1]
    alive[edge_face[s[m]]] = False
  deg = np.diff(vf_off)
  rows = np.repeat(np.arange(len(b)), deg[b])
  fb = vf_face[np.repeat(vf_off[b], deg[b]) + np.arange(len(rows)) - np.repeat(np.cumsum(deg[b]) - deg[b], deg[b])]
  fb = fb.astype(np.int64)
  keepf = ~(f[fb] == a[rows, None]).any(-1)
  fb, rows = fb[keepf], rows[keepf]
  block = f[fb]
  f[fb] = np.where(block == b[rows, None], a[rows, None], block)
  return v, Q, n, f[alive].astype(np.int32)


def drop_unused(vertices, faces, *per_vertex):
  f = np.asarray(faces, np.int64).reshape(-1, 3)
  used = np.zeros(len(vertices), bool)
  used[f.reshape(-1)] = True
  new_index = np.cumsum(used) - 1
  return (vertices[used], new_index[f].astype(np.int32), *(a[used] for a in per_vertex))


def simplify(vertices, faces, normals=None, *, target_faces):
  """mesh.simplify_mesh -> ((vertices, faces) or (vertices, faces, normals), stats dict)."""
  v = np.asarray(vertices, np.float32).copy()
  f = np.asarray(faces, np.int32).reshape(-1, 3).copy()
  n = None if normals is None else np.asarray(normals, np.float32).copy()
  F = len(f)
  stats = dict(faces_before=F, faces_after=F, rounds=0, target_reached=True)
  if not target_faces or F <= target_faces:
    return ((v, f) if n is None else (v, f, n)), stats
  V = len(v)
  topo = topology(f, V)
  Q = quadrics(v, f, topo)
  rounds = 0
  while True:
    keys, pos = edge_cost(v, f, Q, topo)
    sel = select(f, topo[0], keys, V)
    if not sel.any():
      break
    ids, gone = budget(keys, sel, topo[1], F - target_faces)
    if len(ids) == 0:
      break
    v, Q, n, f = apply(ids, v, Q, n, f, topo, pos)
    F -= gone
    assert len(f) == F
    rounds += 1
    if F <= target_faces:
      break
    topo = topology(f, V)
  stats.update(faces_after=F, rounds=rounds, target_reached=F <= target_faces + 1)
  return drop_unused(v, f, *(() if n is None else (n,))), stats


def euler_characteristic(faces):
  """V - E + F over the vertices the faces use."""
  f = np.asarray(faces, np.int64).reshape(-1, 3)
  e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
  return len(np.unique(f)) - len(np.unique(e, axis=0)) + len(f)
