"""Coloured mesh export without a GPU: the PLY with vertex normals and colours read back through its header, the
plain PLY's bytes, and Config.mesh_vertex_colors."""
import numpy as np

_PLY_TYPES = {'float': '<f4', 'uchar': 'u1', 'int': '<i4'}


def read_ply_props(path):
  """A binary little-endian PLY read by following its header: ({vertex property: array [V]}, faces [F, 3])."""
  with open(path, 'rb') as f:
    data = f.read()
  head, body = data.split(b'end_header\n', 1)
  lines = head.decode('ascii').splitlines()
  assert lines[:2] == ['ply', 'format binary_little_endian 1.0']
  elements, cur = [], None
  for line in lines[2:]:
    w = line.split()
    if w[0] == 'element':
      cur = (w[1], int(w[2]), [])
      elements.append(cur)
    elif w[0] == 'property':
      cur[2].append(tuple(w[1:]))
  assert [e[0] for e in elements] == ['vertex', 'face']
  (_, nv, vprops), (_, nf, fprops) = elements
  assert fprops == [('list', 'uchar', 'int', 'vertex_indices')]
  vdt = np.dtype([(p[1], _PLY_TYPES[p[0]]) for p in vprops])
  verts = np.frombuffer(body[:nv * vdt.itemsize], vdt)
  rec = np.frombuffer(body[nv * vdt.itemsize:], dtype=[('n', 'u1'), ('idx', '<i4', (3,))])
  assert len(rec) == nf and np.all(rec['n'] == 3)
  return {name: verts[name] for name in vdt.names}, rec['idx']


def _mesh(rng, V=50, F=80):
  v = rng.normal(size=(V, 3)).astype(np.float32)
  f = rng.integers(0, V, (F, 3)).astype(np.int32)
  n = rng.normal(size=(V, 3))
  n = (n / np.linalg.norm(n, axis=1, keepdims=True)).astype(np.float32)
  c = rng.integers(0, 256, (V, 3)).astype(np.uint8)
  return v, f, n, c


def test_ply_with_normals_and_colors_round_trips(tmp_path):
  from multinerf_b200 import mesh
  v, f, n, c = _mesh(np.random.default_rng(0))
  for normals, colors, names in ((n, c, 'x y z nx ny nz red green blue'), (n, None, 'x y z nx ny nz'),
                                 (None, c, 'x y z red green blue')):
    path = str(tmp_path / 'm.ply')
    mesh.write_ply(path, v, f, normals=normals, colors=colors)
    props, f2 = read_ply_props(path)
    assert list(props) == names.split()
    assert np.array_equal(np.stack([props[k] for k in 'xyz'], 1), v) and np.array_equal(f2, f)
    if normals is not None:
      assert props['nx'].dtype == np.float32
      assert np.array_equal(np.stack([props[k] for k in ('nx', 'ny', 'nz')], 1), n)
    if colors is not None:
      assert props['red'].dtype == np.uint8
      assert np.array_equal(np.stack([props[k] for k in ('red', 'green', 'blue')], 1), c)
  mesh.write_ply(path, np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32), normals=np.zeros((0, 3), np.float32),
                 colors=np.zeros((0, 3), np.uint8))
  props, f3 = read_ply_props(path)
  assert len(props['red']) == 0 and f3.shape == (0, 3)


def test_plain_ply_bytes_unchanged(tmp_path):
  """Without normals and colours: the header and records of a positions-only PLY, byte for byte."""
  from multinerf_b200 import mesh
  v, f, _, _ = _mesh(np.random.default_rng(1), V=7, F=5)
  path = str(tmp_path / 'm.ply')
  mesh.write_ply(path, v, f)
  header = ('ply\nformat binary_little_endian 1.0\nelement vertex 7\nproperty float x\nproperty float y\n'
            'property float z\nelement face 5\nproperty list uchar int vertex_indices\nend_header\n').encode('ascii')
  faces = b''.join(b'\x03' + row.astype('<i4').tobytes() for row in f)
  with open(path, 'rb') as fh:
    assert fh.read() == header + v.astype('<f4').tobytes() + faces


def test_mesh_vertex_colors_flag():
  from multinerf_b200 import configs
  assert configs.Config().mesh_vertex_colors is False
  assert configs.load_config(gin_bindings=[]).config.mesh_vertex_colors is False
  b = configs.load_config(gin_bindings=['Config.mesh_vertex_colors = True'])
  assert b.config.mesh_vertex_colors is True
