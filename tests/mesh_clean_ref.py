"""numpy + scipy restatement of mesh cleaning (mnrf_mesh_components, mesh.clean_mesh) for the CPU and GPU tests:
connected components labelled by their minimum vertex index, components ranked by face count (ties to the smaller
minimum vertex index), and the stable compaction of the kept faces and the vertices they use."""
import numpy as np
import scipy.sparse
from scipy.sparse import csgraph


def components(faces, num_vertices):
  """labels [V] int32: each vertex's label is the smallest vertex index of its component of the graph whose edges
  are the faces' edges."""
  f = np.asarray(faces, np.int32).reshape(-1, 3)
  V = int(num_vertices)
  if V == 0:
    return np.zeros(0, np.int32)
  # edges (v0, v1) and (v0, v2) join a face's corners as all three would
  rows = np.concatenate([f[:, 0], f[:, 0]])
  cols = np.concatenate([f[:, 1], f[:, 2]])
  g = scipy.sparse.coo_matrix((np.ones(len(rows), np.int8), (rows, cols)), shape=(V, V)).tocsr()
  _, comp = csgraph.connected_components(g, directed=False)
  first = np.full(comp.max() + 1, V, np.int64)
  np.minimum.at(first, comp, np.arange(V))
  return first[comp].astype(np.int32)


def clean(vertices, faces, *per_vertex, keep_components=0, view_counts=None, min_views=0):
  """The rules of mesh.clean_mesh with the per-vertex view counts given -> (vertices, faces, *per_vertex)."""
  v = np.asarray(vertices)
  f = np.asarray(faces, np.int64).reshape(-1, 3)
  V = len(v)
  keep = np.ones(len(f), bool)
  if min_views:
    keep &= (np.asarray(view_counts)[f] >= min_views).all(-1)
  if keep_components:
    culled = f[keep]
    labels = components(culled, V)
    comp = labels[culled[:, 0]]
    ids, size = np.unique(comp, return_counts=True)
    ranked = sorted(zip(ids.tolist(), size.tolist()), key=lambda c: (-c[1], c[0]))[:keep_components]
    keep[np.flatnonzero(keep)] = np.isin(comp, [c for c, _ in ranked])
  kf = f[keep]
  used = np.zeros(V, bool)
  used[kf.reshape(-1)] = True
  new_index = np.cumsum(used) - 1
  return (v[used], new_index[kf].astype(np.int32), *(np.asarray(a)[used] for a in per_vertex))


def euler(vertices, faces):
  """V - E + F of a triangle mesh (E: distinct undirected edges)."""
  f = np.asarray(faces, np.int64).reshape(-1, 3)
  e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
  return len(vertices) - len(np.unique(e, axis=0)) + len(f)
