"""Mesh extraction on the host: the generated marching-cubes case table (closed, consistently wound meshes by
construction), PLY output and the mesh fields of Config.  No GPU needed."""
import importlib.util
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gen():
  spec = importlib.util.spec_from_file_location('gen_mc_tables', os.path.join(ROOT, 'tools', 'gen_mc_tables.py'))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


G = _gen()


def _cut_edges(case):
  return {e for e in range(12) if (case >> G.edge_corners(e)[0] & 1) != (case >> G.edge_corners(e)[1] & 1)}


def _committed_table():
  """kMcNumTris and kMcTris as written in csrc/mc_tables.cuh -> per case, the list of triangles."""
  text = open(os.path.join(ROOT, 'multinerf_b200', 'csrc', 'mc_tables.cuh')).read()
  width = int(text.split('kMcMaxTris = ')[1].split(';')[0])
  counts_txt = text.split('kMcNumTris[256] = {')[1].split('};')[0]
  counts = [int(v) for v in counts_txt.replace('\n', ' ').split(',') if v.strip()]
  rows_txt = text.split('kMcTris[256]')[1].split('= {', 1)[1].split('\n};')[0]
  rows = [[int(v) for v in line.split('{')[1].split('}')[0].split(',')] for line in rows_txt.strip().splitlines()]
  assert len(counts) == 256 and len(rows) == 256 and all(len(r) == 3 * width for r in rows)
  return [[tuple(rows[c][3 * t:3 * t + 3]) for t in range(counts[c])] for c in range(256)]


TABLE = _committed_table()


def test_generator_reproduces_committed_header():
  with open(os.path.join(ROOT, 'multinerf_b200', 'csrc', 'mc_tables.cuh')) as f:
    assert f.read() == G.render()


def test_loops_cover_each_cut_edge_once():
  for case in range(256):
    loops = G.case_loops(case)
    edges = [e for loop in loops for e in loop]
    assert len(edges) == len(set(edges)) and set(edges) == _cut_edges(case), case
    # the committed triangles use exactly the cut edges, and fan each loop: len - 2 triangles per loop
    assert {e for t in TABLE[case] for e in t} == _cut_edges(case), case
    assert len(TABLE[case]) == sum(len(loop) - 2 for loop in loops), case


def _boundary(tris):
  """Directed edges of a cell's triangles not cancelled by their reverse: the loops' segments."""
  directed = [(t[i], t[(i + 1) % 3]) for t in tris for i in range(3)]
  out = [d for d in directed if (d[1], d[0]) not in directed]
  assert len(out) == len(set(out))
  return out


def _face_edges(f):
  n, ring = G.FACES[f]
  return [G.edge_between(ring[k], ring[(k + 1) % 4]) for k in range(4)]


def _rule_segments(inside):
  """The face rule restated: a face with two cut sides joins them; with four (inside corners on a diagonal), each
  inside corner is cut off by a segment joining its two sides, so the two inside corners stay apart."""
  cut = [k for k in range(4) if inside[k] != inside[(k + 1) % 4]]
  if len(cut) == 2:
    return {frozenset(cut)}
  if len(cut) == 4:
    return {frozenset({(k - 1) % 4, k}) for k in range(4) if inside[k]}
  return set()


def test_face_segments_follow_the_face_rule():
  """Every boundary segment of a cell's triangles lies on one face, and on every face the segments are what the
  face rule gives for that face's four corners -- which the neighbouring cell sees too, so the two agree."""
  for case in range(256):
    segs = _boundary(TABLE[case])
    on_face = {f: set() for f in range(6)}
    for a, b in segs:
      faces = [f for f in range(6) if a in _face_edges(f) and b in _face_edges(f)]
      assert len(faces) == 1, (case, a, b)
      on_face[faces[0]].add(frozenset({a, b}))
    for f in range(6):
      _, ring = G.FACES[f]
      sides = _face_edges(f)
      want = {frozenset(sides[k] for k in pair) for pair in _rule_segments([case >> c & 1 for c in ring])}
      assert on_face[f] == want, (case, f)


def test_shared_face_segments_run_opposite_ways():
  """A face seen from the cells on either side: the same segments, in opposite directions."""
  for axis in range(3):
    lo_face = [f for f in range(6) if G.FACES[f][0][axis] == -1][0]
    hi_face = [f for f in range(6) if G.FACES[f][0][axis] == 1][0]
    for case in range(256):
      # the cell above along `axis` has, as its lower face, this cell's upper face: shift the upper corners down
      upper = 0
      for c in range(8):
        if c >> axis & 1 and case >> c & 1:
          upper |= 1 << (c & ~(1 << axis))
      shift = {e: e for e in range(12)}
      for e in range(12):
        a, b = G.edge_corners(e)
        if a >> axis & 1 and b >> axis & 1:
          shift[e] = G.edge_between(a & ~(1 << axis), b & ~(1 << axis))
      mine = {(shift[a], shift[b]) for a, b in G.face_segments(case, hi_face)}
      theirs = set(G.face_segments(upper, lo_face))
      assert mine == {(b, a) for a, b in theirs}, (axis, case)


def test_winding_puts_inside_corners_on_the_negative_side():
  """With the vertices at the edge midpoints, no triangle's normal points into the inside: summed over the
  triangle's three cut edges, (inside corner - outside corner) . normal <= 0 (0 only for a fan triangle that is
  parallel to its edges), and < 0 for every loop's total (vector-area) normal."""
  for case in range(256):
    for loop in G.case_loops(case):
      total = np.zeros(3)
      s_loop = 0.0
      for k in range(1, len(loop) - 1):
        tri = (loop[0], loop[k + 1], loop[k])
        assert tri in TABLE[case]
        a, b, c = (G.edge_mid(e) for e in tri)
        n = np.cross(b - a, c - a)
        total += n
        s = 0.0
        for e in tri:
          lo, hi = G.edge_corners(e)
          i, o = (lo, hi) if case >> lo & 1 else (hi, lo)
          s += np.dot(G.corner_pos(i) - G.corner_pos(o), n)
        assert s <= 0, (case, tri)
      for e in loop:
        lo, hi = G.edge_corners(e)
        i, o = (lo, hi) if case >> lo & 1 else (hi, lo)
        s_loop += np.dot(G.corner_pos(i) - G.corner_pos(o), total)
      assert s_loop < 0, (case, loop)
  # a single inside corner: one triangle whose normal points away from it
  for c in range(8):
    (tri,) = TABLE[1 << c]
    a, b, d = (G.edge_mid(e) for e in tri)
    assert np.dot(G.corner_pos(c) - a, np.cross(b - a, d - a)) < 0


def read_ply(path):
  with open(path, 'rb') as f:
    data = f.read()
  head, body = data.split(b'end_header\n', 1)
  lines = head.decode('ascii').splitlines()
  assert lines[:2] == ['ply', 'format binary_little_endian 1.0']
  nv = int([l for l in lines if l.startswith('element vertex')][0].split()[-1])
  nf = int([l for l in lines if l.startswith('element face')][0].split()[-1])
  assert 'property list uchar int vertex_indices' in lines
  v = np.frombuffer(body[:12 * nv], '<f4').reshape(nv, 3)
  rec = np.frombuffer(body[12 * nv:], dtype=[('n', 'u1'), ('idx', '<i4', (3,))])
  assert len(rec) == nf and np.all(rec['n'] == 3)
  return v, rec['idx']


def test_write_ply_round_trips(tmp_path):
  from multinerf_b200 import mesh
  rng = np.random.default_rng(0)
  v = rng.normal(size=(50, 3)).astype(np.float32)
  f = rng.integers(0, 50, (80, 3)).astype(np.int32)
  path = str(tmp_path / 'm.ply')
  mesh.write_ply(path, v, f)
  v2, f2 = read_ply(path)
  assert np.array_equal(v, v2) and np.array_equal(f, f2)
  mesh.write_ply(path, np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32))
  v3, f3 = read_ply(path)
  assert v3.shape == (0, 3) and f3.shape == (0, 3)


def test_default_boxes_and_gin_fields():
  from multinerf_b200 import configs, mesh
  assert mesh.default_bbox(configs.bundle_360()) == (-1.0, -1.0, -1.0, 1.0, 1.0, 1.0)
  assert mesh.default_bbox(configs.bundle_blender_256()) == (-1.5, -1.5, -1.5, 1.5, 1.5, 1.5)
  ff = configs.bundle_llff_raw()
  assert ff.config.forward_facing
  with pytest.raises(ValueError, match='mesh_bbox'):
    mesh.default_bbox(ff)
  c = configs.Config()
  assert (c.mesh_resolution, c.mesh_level, c.mesh_bbox) == (512, 10.0, None)
  b = configs.load_config(gin_bindings=['Config.mesh_bbox = (-2, -1, -0.5, 2, 1, 0.5)', 'Config.mesh_resolution = 64',
                                        'Config.mesh_level = 25.', 'Config.forward_facing = True'])
  assert (b.config.mesh_resolution, b.config.mesh_level) == (64, 25.0)
  assert mesh.default_bbox(b) == (-2.0, -1.0, -0.5, 2.0, 1.0, 0.5)
  with pytest.raises(ValueError):
    mesh.default_bbox(configs.load_config(gin_bindings=['Config.mesh_bbox = (0, 0, 1, 1)']))


def test_grid_shape():
  from multinerf_b200 import mesh
  (nx, ny, nz), h = mesh.grid_shape((-2, -1, -0.5, 2, 1, 0.5), 65)
  assert (nx, ny, nz) == (65, 33, 17) and h == 4 / 64
  with pytest.raises(ValueError):
    mesh.grid_shape((0, 0, 0, 1, 1, 1e-3), 16)
  with pytest.raises(ValueError):
    mesh.grid_shape((0, 0, 0, 1, 1, 1), 1)
