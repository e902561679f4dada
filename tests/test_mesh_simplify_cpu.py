"""Mesh simplification on the host: the numpy restatement of tests/mesh_simplify_ref.py on hand-built meshes, the
selection's guarantees on random meshes, the torch topology rebuild of mesh.simplify_mesh against the reference, the
Config field and its validation, and the no-op and argument checks of mesh.simplify_mesh.  No GPU needed."""
import numpy as np
import pytest
import torch

import mesh_simplify_ref as R


def square(n, jitter=0.0, seed=0):
  """The unit square in z = 0 as an n x n grid of cells, two triangles each, wound +z; interior points moved by up
  to `jitter` cells in x and y, and by `jitter` cells in z for a non-flat sheet."""
  i, j = np.meshgrid(np.arange(n + 1), np.arange(n + 1), indexing='ij')
  v = np.stack([i.ravel(), j.ravel(), np.zeros(i.size)], 1) / n
  if jitter:
    rng = np.random.default_rng(seed)
    inner = ((i > 0) & (i < n) & (j > 0) & (j < n)).ravel()
    v[inner] += rng.uniform(-jitter, jitter, (inner.sum(), 3)) / n
  idx = np.arange((n + 1) ** 2).reshape(n + 1, n + 1)
  a, b, c, d = idx[:-1, :-1], idx[1:, :-1], idx[1:, 1:], idx[:-1, 1:]
  f = np.concatenate([np.stack([a, b, c], -1).reshape(-1, 3), np.stack([a, c, d], -1).reshape(-1, 3)])
  return v.astype(np.float32), f.astype(np.int32)


def cube(n):
  """The surface of the unit cube, each side an n x n grid of cells, two triangles each, wound outwards."""
  ids, faces = {}, []

  def vid(p):
    return ids.setdefault(tuple(p), len(ids))
  for axis in range(3):
    u, w = [a for a in range(3) if a != axis]
    for side in (0, n):
      for i in range(n):
        for j in range(n):
          q = []
          for di, dj in ((0, 0), (1, 0), (1, 1), (0, 1)):
            p = [0, 0, 0]
            p[axis], p[u], p[w] = side, i + di, j + dj
            q.append(vid(p))
          if (side == 0) != (axis == 1):
            q = q[::-1]
          faces += [[q[0], q[1], q[2]], [q[0], q[2], q[3]]]
  v = np.zeros((len(ids), 3), np.float32)
  for k, i in ids.items():
    v[i] = np.array(k, np.float32) / n
  return v, np.array(faces, np.int32)


def tetrahedron():
  v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
  return v, np.array([[0, 2, 1], [0, 1, 3], [1, 2, 3], [0, 3, 2]], np.int32)


def fan(ring):
  """Vertex 1 at the origin surrounded by vertex 0 = (2, 0, 0) and `ring` (counter-clockwise), one triangle per
  sector: edge (0, 1) is interior, and vertex 0 on the boundary keeps its position under the quadrics."""
  pts = [(2.0, 0.0)] + [None] + list(ring)
  pts[1] = (0.0, 0.0)
  v = np.array([(x, y, 0.0) for x, y in pts], np.float32)
  order = [0] + list(range(2, len(pts)))
  f = [[1, order[k], order[(k + 1) % len(order)]] for k in range(len(order))]
  return v, np.array(f, np.int32)


def _keys(v, f):
  topo = R.topology(f, len(v))
  return R.edge_cost(v, f, R.quadrics(v, f, topo), topo)[0], topo


def _edge(topo, a, b):
  return int(np.flatnonzero((topo[0][:, 0] == a) & (topo[0][:, 1] == b))[0])


def test_flat_square_to_two_faces_on_its_corners():
  v, f = square(8)
  topo = R.topology(f, len(v))
  q = R.quadrics(v, f, topo)
  (ov, of), stats = R.simplify(v, f, target_faces=2)
  assert stats['faces_after'] == 2 and stats['target_reached'] and len(of) == 2
  corners = {(0.0, 0.0), (0.0, 1.0), (1.0, 0.0), (1.0, 1.0)}
  assert {tuple(p[:2]) for p in ov.tolist()} == corners and np.all(ov[:, 2] == 0)
  # zero cost: each corner is where its original quadric vanishes
  src = [int(np.flatnonzero((v == p).all(1))[0]) for p in ov]
  assert np.all(R.quadric_eval(q[src], ov.astype(np.float64)) == 0)
  # both faces keep the +z winding
  p = ov[of].astype(np.float64)
  assert np.all(np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])[:, 2] > 0)


def test_closed_cube_to_twelve_faces_on_its_corners():
  v, f = cube(5)
  (ov, of), stats = R.simplify(v, f, target_faces=12)
  assert stats['faces_after'] == 12 and len(of) == 12 and len(ov) == 8
  corners = np.array([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], np.float64)
  d = np.abs(ov[:, None, :] - corners[None]).max(-1).min(-1)
  assert d.max() < 1e-6
  assert R.euler_characteristic(of) == 2


def test_tetrahedron_and_lone_triangle_are_never_collapsed():
  for v, f in (tetrahedron(), (np.eye(3, dtype=np.float32), np.array([[0, 1, 2]], np.int32))):
    keys, _ = _keys(v, f)
    assert np.all(keys == R.NO_KEY)
    (ov, of), stats = R.simplify(v, f, target_faces=1)
    assert np.array_equal(ov, v) and np.array_equal(of, f)
    assert stats['rounds'] == 0 and stats['target_reached'] == (len(f) <= 2)


def test_faces_axy_and_bxy_block_ab():
  # a tetrahedron: the common neighbours of 0 and 1 are exactly the apexes 2 and 3 (the link rule alone would pass),
  # but faces (0, 3, 2) and (1, 2, 3) exist, so 01 would fold the tetrahedron into a doubled face
  v, f = tetrahedron()
  assert set(f[2]) - {1} == set(f[3]) - {0} == {2, 3}
  keys, topo = _keys(v, f)
  assert keys[_edge(topo, 0, 1)] == R.NO_KEY
  # an octahedron has no such pair: its edges may be collapsed
  ov = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float32)
  of = np.array([[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]], np.int32)
  keys, _ = _keys(ov, of)
  assert np.all(keys != R.NO_KEY)


def test_fold_over_is_rejected():
  # moving the centre 1 onto vertex 0 turns sector (1, r1, r2) over when r1 is pulled in towards the centre
  convex = [(0.5, 1.0), (-1.0, 0.5), (-1.0, -1.0), (1.0, -1.5)]
  folded = [(0.2, 0.2)] + convex[1:]
  for ring, ok in ((convex, True), (folded, False)):
    v, f = fan(ring)
    keys, topo = _keys(v, f)
    e = _edge(topo, 0, 1)
    _, pos = R.edge_cost(v, f, R.quadrics(v, f, topo), topo)
    assert np.abs(pos[e] - v[0]).max() < 1e-5        # the collapse goes to vertex 0
    assert (keys[e] != R.NO_KEY) == ok


def _random_sheet(seed):
  v, f = square(24, jitter=0.3, seed=seed)
  rng = np.random.default_rng(seed)
  return v, f[rng.random(len(f)) > 0.08]       # holes: boundaries and pinched vertices


@pytest.mark.parametrize('seed', range(4))
def test_selection_is_independent_and_takes_the_least_key(seed):
  v, f = _random_sheet(seed)
  keys, topo = _keys(v, f)
  edges = topo[0]
  sel = R.select(f, edges, keys, len(v))
  valid = keys != R.NO_KEY
  assert valid.sum() > 100 and sel.sum() > 5
  assert sel[np.argmin(np.where(valid, keys, R.NO_KEY))]
  # no face touches two selected edges
  touch = np.zeros(len(v), np.int64) - 1
  for e in np.flatnonzero(sel):
    touch[edges[e]] = e
  owner = touch[f]                               # per face corner: the selected edge it is an end of
  for row in owner:
    assert len(set(row[row >= 0].tolist())) <= 1
  # selected edges share no vertex either
  assert len(np.unique(edges[sel].reshape(-1))) == 2 * sel.sum()


def test_rounds_keep_a_manifold_sheet_manifold():
  v, f = square(16, jitter=0.3, seed=7)
  (ov, of), stats = R.simplify(v, f, target_faces=60)
  assert stats['faces_after'] in (60, 61) and stats['target_reached']
  assert R.euler_characteristic(of) == 1
  e = np.sort(np.concatenate([of[:, [0, 1]], of[:, [1, 2]], of[:, [2, 0]]]), 1)
  _, cnt = np.unique(e, axis=0, return_counts=True)
  assert cnt.max() <= 2 and len(np.unique(np.sort(of, 1), axis=0)) == len(of)


def test_torch_topology_matches_the_reference():
  from multinerf_b200 import mesh
  v, f = _random_sheet(11)
  V = len(v)
  t = mesh.mesh_topology(torch.tensor(f), V)
  r = R.topology(f, V)
  for a, b in zip(t, r):
    assert np.array_equal(a.numpy(), b)
  assert t.edges.dtype == torch.int32 and t.edge_face.dtype == torch.int32 and t.vf_face.dtype == torch.int32
  for a, b in zip(mesh.boundary_edges(t, V), R.boundary(r, V)):
    assert np.array_equal(a.numpy(), b)


def test_config_field_and_validation():
  from multinerf_b200 import configs, mesh
  assert configs.Config().mesh_target_faces == 0
  b = configs.load_config(gin_bindings=['Config.mesh_target_faces = 100000'])
  assert b.config.mesh_target_faces == 100000 and mesh.validate_config(b) == 'density'
  with pytest.raises(ValueError, match='mesh_target_faces'):
    mesh.validate_config(configs.load_config(gin_bindings=['Config.mesh_target_faces = -1']))


def test_simplify_mesh_off_returns_its_inputs():
  from multinerf_b200 import mesh
  v, f, n = torch.zeros(4, 3), torch.tensor([[0, 1, 2], [0, 2, 3]], dtype=torch.int32), torch.ones(4, 3)
  for target in (0, 2, 5):
    stats = {}
    out = mesh.simplify_mesh(v, f, n, target_faces=target, stats=stats)
    assert len(out) == 3 and all(a is b for a, b in zip(out, (v, f, n)))
    assert stats == {'faces_before': 2, 'faces_after': 2, 'rounds': 0, 'target_reached': True}
  out = mesh.simplify_mesh(v, f, target_faces=0)
  assert len(out) == 2 and out[0] is v and out[1] is f
  with pytest.raises(ValueError, match='target_faces'):
    mesh.simplify_mesh(v, f, target_faces=-1)
  for bad in ([[0, 1, 4], [0, 2, 3]], [[0, -1, 2], [0, 2, 3]], [[0, 1, 1], [0, 2, 3]]):
    with pytest.raises(ValueError, match='outside'):
      mesh.simplify_mesh(v, torch.tensor(bad, dtype=torch.int32), target_faces=1)
