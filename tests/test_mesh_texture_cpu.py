"""The texture atlas without a GPU: the layout of tests/mesh_texture_ref.py (the restatement of csrc/mesh.cu's) keeps
every bilinear sample of a face on that face's own texels, for every cell size and atlas the tests use; the atlas
size check; the Config field; and write_obj's three files read back."""
import numpy as np
import pytest
import torch

import mesh_texture_ref as R

SIZES = (4, 16, 64, 4096)


def _face_counts(size):
  return sorted({f for f in (1, 2, 3, 7, 1000, R.capacity(size)) if f <= R.capacity(size)})


CASES = [(f, s) for s in SIZES for f in _face_counts(s)]


def _owner_map(num_faces, size):
  """[S * S] int64: the face owning each atlas texel, -1 outside the used cells."""
  owner, _, _, index = R.texels(num_faces, size)
  m = np.full(size * size, -1, np.int64)
  m[index] = owner
  return m


def _check_samples(uv, owner_map, size, faces, bary):
  """Bilinear samples at barycentrics bary [N, 3] of faces [N]: every texel read with a nonzero weight is owned by
  the sampled face."""
  p = (bary[:, :, None] * uv[faces]).sum(1)
  xs, ys = R.bilinear_texels(p[:, 0], p[:, 1])
  read = xs >= 0
  assert (xs[read] < size).all() and (ys[read] >= 0).all() and (ys[read] < size).all()
  got = owner_map[np.where(read, ys * size + xs, 0)]
  assert (np.where(read, got, faces[:, None]) == faces[:, None]).all()


@pytest.mark.parametrize('c', range(4, 12))
def test_ownership_invariant_exhaustive_per_cell_size(c):
  """Both faces of one cell of side c, sampled on a 1/64-texel lattice over each triangle (edges and corners
  included), and a cell with face A alone."""
  size = c
  for num_faces in (2, 1):
    assert R.atlas(num_faces, size) == (1, c)
    uv = R.uv(num_faces, size)
    m = _owner_map(num_faces, size)
    assert (m >= 0).all() and set(np.unique(m)) == set(range(num_faces))
    q = 64
    a, b = np.meshgrid(np.arange(q + 1), np.arange(q + 1))
    keep = a + b <= q
    bary1, bary2 = a[keep] / q, b[keep] / q
    bary = np.stack([1 - bary1 - bary2, bary1, bary2], -1)
    for f in range(num_faces):
      _check_samples(uv, m, size, np.full(len(bary), f), bary)


@pytest.mark.parametrize('num_faces,size', CASES)
def test_layout(num_faces, size):
  n, c = R.atlas(num_faces, size)
  from multinerf_b200 import ops
  assert ops.texture_atlas(num_faces, size) == (n, c) and c >= 4
  uv = R.uv(num_faces, size)
  # corners on texel centres, inside the face's own cell
  assert np.array_equal(uv - 0.5, np.floor(uv))
  k = np.arange(num_faces) // 2
  x0, y0 = (k % n) * c, (k // n) * c
  assert (uv[..., 0] > x0[:, None]).all() and (uv[..., 0] < (x0 + c)[:, None]).all()
  assert (uv[..., 1] > y0[:, None]).all() and (uv[..., 1] < (y0 + c)[:, None]).all()
  owner, i, j, index = R.texels(num_faces, size)
  # each used cell's texels once, owned by its own faces; every other texel unowned
  assert len(np.unique(index)) == len(index) == (num_faces + 1) // 2 * c * c
  assert (owner // 2 == np.arange(len(owner)) // (c * c)).all() and (owner < num_faces).all()
  m = _owner_map(num_faces, size)
  used = np.zeros((size, size), bool)
  for kk in range((num_faces + 1) // 2):
    used[(kk // n) * c:(kk // n + 1) * c, (kk % n) * c:(kk % n + 1) * c] = True
  assert np.array_equal(m.reshape(size, size) >= 0, used)
  # the corner texels belong to their faces
  cx, cy = np.floor(uv[..., 0]).astype(np.int64), np.floor(uv[..., 1]).astype(np.int64)
  assert (m[cy * size + cx] == np.arange(num_faces)[:, None]).all()
  # dense random bilinear samples inside random faces
  rng = np.random.default_rng(num_faces * 7 + size)
  N = 200000
  faces = rng.integers(0, num_faces, N)
  bary = rng.dirichlet((1, 1, 1), N)
  _check_samples(uv, m, size, faces, bary)


def test_barycentrics_are_the_nearest_point_of_the_chart():
  """Texels outside their face's triangle take the nearest point of the triangle: checked against a dense
  lattice search in texel units."""
  for c in (4, 5, 11):
    uv = R.uv(2, c)
    owner, i, j, _ = R.texels(2, c)
    w = R.barycentrics(2, c)
    assert (w >= 0).all() and np.allclose(w.sum(1), 1)
    p = (w[:, :, None] * uv[owner]).sum(1)
    q = 400
    a, b = np.meshgrid(np.arange(q + 1), np.arange(q + 1))
    keep = a + b <= q
    lat = np.stack([1 - a[keep] / q - b[keep] / q, a[keep] / q, b[keep] / q], -1)
    for t in range(len(owner)):
      pts = lat @ uv[owner[t]]
      centre = np.array([i[t] + 0.5, j[t] + 0.5])
      best = np.sqrt(((pts - centre) ** 2).sum(1)).min()
      assert np.linalg.norm(p[t] - centre) <= best + 1e-9


def test_corner_texels_have_their_vertices_as_points():
  rng = np.random.default_rng(3)
  v = rng.normal(size=(40, 3))
  f = rng.integers(0, 40, (31, 3))
  n = rng.normal(size=(40, 3))
  uv, index, points, _, w, owner = R.raster(v, f, n, 64)
  pos = {int(x): t for t, x in enumerate(index)}
  for face in range(len(f)):
    for k in range(3):
      t = pos[int(np.floor(uv[face, k, 1])) * 64 + int(np.floor(uv[face, k, 0]))]
      assert owner[t] == face and w[t, k] == 1 and np.array_equal(points[t], v[f[face, k]])


def test_normal_fallbacks():
  """Opposite vertex normals cancel at a texel with weights (1/2, 1/2, 0): the face's normal there; a zero-area face
  whose vertex normals are zero: (0, 0, 1) everywhere."""
  v = np.array([[0, 0, 0], [2, 0, 0], [0, 3, 0], [1, 1, 1], [1, 1, 1], [1, 1, 1]], np.float64)
  f = np.array([[0, 1, 2], [3, 4, 5]])
  nv = np.array([[0.6, 0, 0.8], [-0.6, 0, -0.8], [0, 1, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0]], np.float64)
  _, _, _, n, w, owner = R.raster(v, f, nv, 5)      # c = 5: A's legs are 2 texels
  half = (w[:, 0] == 0.5) & (w[:, 1] == 0.5) & (owner == 0)
  assert half.sum() == 1
  assert np.array_equal(n[half], [[0, 0, 1]])
  assert (owner == 1).sum() > 0 and np.array_equal(n[owner == 1], np.tile([0.0, 0, 1], ((owner == 1).sum(), 1)))
  v[2] = [0, -3, 0]                                 # face 0 now points down
  _, _, _, n, _, _ = R.raster(v, f, nv, 5)
  assert np.array_equal(n[half], [[0, 0, -1]])


@pytest.mark.parametrize('size', (4, 16, 64, 4096, 1000))
def test_atlas_rejects_one_face_too_many(size):
  from multinerf_b200 import ops
  cap = R.capacity(size)
  assert ops.texture_atlas(cap, size)[1] >= 4
  with pytest.raises(ValueError, match=f'{cap + 1} faces .*at most {cap} faces.*mesh_target_faces'):
    ops.texture_atlas(cap + 1, size)
  with pytest.raises(ValueError):
    R.atlas(cap + 1, size)


def test_atlas_rejects_bad_sizes():
  from multinerf_b200 import ops
  for size in (0, 3, 16385, -4):
    with pytest.raises(ValueError, match='texture size'):
      ops.texture_atlas(2, size)
  assert ops.texture_atlas(0, 4) == (0, 4)


def test_config_field_and_validation():
  from multinerf_b200 import configs, mesh
  assert configs.Config().mesh_texture_size == 0
  for size in (4, 4096, 16384):
    b = configs.load_config(gin_bindings=[f'Config.mesh_texture_size = {size}'])
    assert b.config.mesh_texture_size == size and mesh.validate_config(b) == 'density'
  b = configs.load_config(gin_bindings=['Config.mesh_texture_size = 2048', "Config.mesh_method = 'tsdf'",
                                        'Config.mesh_target_faces = 1000', 'Config.mesh_keep_components = 1'])
  assert mesh.validate_config(b) == 'tsdf'
  for size in (-1, 1, 3, 16385):
    with pytest.raises(ValueError, match='mesh_texture_size'):
      mesh.validate_config(configs.load_config(gin_bindings=[f'Config.mesh_texture_size = {size}']))


def read_obj(path):
  """(v [V, 3], vt [K, 2], vn [V, 3], faces [F, 3, 3] 1-based (v, vt, vn), mtllib, usemtl) of write_obj's files."""
  v, vt, vn, f = [], [], [], []
  mtllib = usemtl = None
  with open(path) as fh:
    for line in fh:
      tok = line.split()
      if tok[0] == 'v':
        v.append([float(x) for x in tok[1:]])
      elif tok[0] == 'vt':
        vt.append([float(x) for x in tok[1:]])
      elif tok[0] == 'vn':
        vn.append([float(x) for x in tok[1:]])
      elif tok[0] == 'f':
        f.append([[int(x) for x in c.split('/')] for c in tok[1:]])
      elif tok[0] == 'mtllib':
        mtllib = tok[1]
      elif tok[0] == 'usemtl':
        usemtl = tok[1]
  return (np.array(v, np.float32), np.array(vt, np.float32), np.array(vn, np.float32), np.array(f, np.int64),
          mtllib, usemtl)


@pytest.mark.parametrize('size', (16, 1000))
def test_write_obj_round_trip(tmp_path, size):
  from PIL import Image
  from multinerf_b200 import mesh
  rng = np.random.default_rng(size)
  V, F = 50, 2 * (size // 4) ** 2 if size < 100 else 3001
  v = (rng.normal(size=(V, 3)) * 10 ** rng.uniform(-3, 3, (V, 1))).astype(np.float32)
  n = rng.normal(size=(V, 3)).astype(np.float32)
  f = rng.integers(0, V, (F, 3)).astype(np.int32)
  uv = R.uv(F, size).astype(np.float32)
  tex = rng.integers(0, 256, (size, size, 3)).astype(np.uint8)
  obj, mtl, png = mesh.write_obj(str(tmp_path / 'm.obj'), torch.tensor(v), torch.tensor(f), torch.tensor(n),
                                 torch.tensor(uv), torch.tensor(tex))
  assert (obj, mtl, png) == tuple(str(tmp_path / f'm.{e}') for e in ('obj', 'mtl', 'png'))
  rv, rvt, rvn, rf, mtllib, usemtl = read_obj(obj)
  assert mtllib == 'm.mtl'
  assert np.array_equal(rv, v) and np.array_equal(rvn, n)
  assert np.array_equal(rf[:, :, 0] - 1, f) and np.array_equal(rf[:, :, 2] - 1, f)
  assert np.array_equal(rf[:, :, 1] - 1, np.arange(3 * F).reshape(F, 3))
  vt = rvt[rf[:, :, 1] - 1]
  want = np.stack([uv[..., 0] / np.float32(size), np.float32(1) - uv[..., 1] / np.float32(size)], -1)
  assert np.array_equal(vt, want)
  with open(mtl) as fh:
    text = fh.read().split()
  assert text[text.index('newmtl') + 1] == usemtl and text[text.index('map_Kd') + 1] == 'm.png'
  img = np.asarray(Image.open(png))
  assert img.dtype == np.uint8 and np.array_equal(img, tex)
  # the PNG sampled at each face's first vt, OBJ's origin at the bottom left: the texel of that corner
  x = np.floor(vt[:, 0, 0].astype(np.float64) * size).astype(np.int64)
  y = np.floor((1 - vt[:, 0, 1].astype(np.float64)) * size).astype(np.int64)
  cx, cy = np.floor(uv[:, 0, 0]).astype(np.int64), np.floor(uv[:, 0, 1]).astype(np.int64)
  assert np.array_equal(x, cx) and np.array_equal(y, cy)
  assert np.array_equal(img[y, x], tex[cy, cx])
