"""Mesh cleaning on the host: the numpy/scipy reference of tests/mesh_clean_ref.py on hand-built meshes, the
Config fields and their validation, and the no-op and argument checks of mesh.clean_mesh.  No GPU needed."""
import numpy as np
import pytest
import torch

import mesh_clean_ref as R


def test_components_ties_isolated_degenerate_duplicate():
  # 0..2 one triangle; 3..6 two triangles sharing an edge; 7 isolated; 8, 9 a degenerate face (8, 8, 9);
  # 10..12 one triangle given twice
  faces = np.array([[0, 1, 2], [3, 4, 5], [5, 4, 6], [8, 8, 9], [10, 11, 12], [10, 11, 12]])
  labels = R.components(faces, 13)
  assert labels.dtype == np.int32
  assert labels.tolist() == [0, 0, 0, 3, 3, 3, 3, 7, 8, 8, 10, 10, 10]
  # labels are the minimum index whatever the face order and winding
  perm = np.random.default_rng(0).permutation(len(faces))
  assert np.array_equal(R.components(faces[perm][:, ::-1], 13), labels)


def test_components_of_a_permuted_path():
  V = 1000
  ids = np.random.default_rng(1).permutation(V)
  faces = np.stack([ids[:-1], ids[1:], ids[1:]], 1)
  assert (R.components(faces, V) == 0).all()


def test_clean_ranks_by_face_count_then_minimum_index():
  v = np.arange(13 * 3, dtype=np.float32).reshape(13, 3)
  nrm = -v
  # components: {0,1,2} 1 face, {3..6} 2 faces, {8,9} 1 degenerate face, {10..12} 2 faces (duplicate), 7 isolated
  faces = np.array([[0, 1, 2], [3, 4, 5], [5, 4, 6], [8, 8, 9], [10, 11, 12], [10, 11, 12]])
  ov, of, on = R.clean(v, faces, nrm, keep_components=1)
  # a tie at 2 faces between {3..6} and {10..12}: the smaller minimum index wins
  assert np.array_equal(ov, v[3:7]) and np.array_equal(on, nrm[3:7])
  assert of.tolist() == [[0, 1, 2], [2, 1, 3]] and of.dtype == np.int32
  ov, of = R.clean(v, faces, keep_components=2)
  assert np.array_equal(ov, v[[3, 4, 5, 6, 10, 11, 12]])
  assert of.tolist() == [[0, 1, 2], [2, 1, 3], [4, 5, 6], [4, 5, 6]]
  # then the one-face components, {0,1,2} before {8,9}; the isolated vertex never comes back
  ov, _ = R.clean(v, faces, keep_components=3)
  assert np.array_equal(ov, v[[0, 1, 2, 3, 4, 5, 6, 10, 11, 12]])
  ov, of = R.clean(v, faces, keep_components=100)
  assert np.array_equal(ov, np.delete(v, 7, 0)) and np.array_equal(of, np.where(faces > 7, faces - 1, faces))


def test_clean_by_views_then_components():
  v = np.zeros((7, 3), np.float32)
  faces = np.array([[0, 1, 2], [1, 2, 3], [4, 5, 6]])
  counts = np.array([3, 3, 3, 1, 2, 2, 2])
  ov, of = R.clean(v, faces, view_counts=counts, min_views=2)
  assert len(ov) == 6 and of.tolist() == [[0, 1, 2], [3, 4, 5]]
  # culling first splits nothing here, but it shrinks {0..3} to one face: a tie the smaller index wins
  ov, of = R.clean(v, faces, view_counts=counts, min_views=2, keep_components=1)
  assert len(ov) == 3 and of.tolist() == [[0, 1, 2]]
  ov, of = R.clean(v, faces, view_counts=counts, min_views=4)
  assert ov.shape == (0, 3) and of.shape == (0, 3)


def test_clean_empty_mesh():
  ov, of = R.clean(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32), keep_components=1)
  assert ov.shape == (0, 3) and of.shape == (0, 3)
  assert R.components(np.zeros((0, 3)), 0).shape == (0,)
  assert R.components(np.zeros((0, 3)), 4).tolist() == [0, 1, 2, 3]


def test_euler_of_a_tetrahedron():
  f = np.array([[0, 1, 2], [0, 3, 1], [1, 3, 2], [2, 3, 0]])
  assert R.euler(np.zeros((4, 3)), f) == 2


def test_config_fields_and_validation():
  from multinerf_b200 import configs, mesh
  c = configs.Config()
  assert (c.mesh_min_views, c.mesh_keep_components) == (0, 0)
  b = configs.load_config(gin_bindings=['Config.mesh_min_views = 3', 'Config.mesh_keep_components = 2'])
  assert (b.config.mesh_min_views, b.config.mesh_keep_components) == (3, 2)
  assert mesh.validate_config(b) == 'density'
  b = configs.load_config(gin_bindings=["Config.mesh_method = 'tsdf'", 'Config.mesh_keep_components = 1'])
  assert mesh.validate_config(b) == 'tsdf'
  for name in ('mesh_min_views', 'mesh_keep_components'):
    with pytest.raises(ValueError, match=name):
      mesh.validate_config(configs.load_config(gin_bindings=[f'Config.{name} = -1']))
  with pytest.raises(ValueError, match='mesh_min_views.*forward-facing'):
    mesh.validate_config(configs.load_config(gin_bindings=['Config.mesh_min_views = 1',
                                                           'Config.forward_facing = True',
                                                           'Config.mesh_bbox = (-1, -1, -1, 1, 1, 1)']))
  # keeping components needs no cameras, so forward-facing scenes may use it
  b = configs.load_config(gin_bindings=['Config.mesh_keep_components = 1', 'Config.forward_facing = True'])
  assert mesh.validate_config(b) == 'density'


def test_clean_mesh_off_returns_its_inputs():
  from multinerf_b200 import mesh
  v, f, n = torch.zeros(4, 3), torch.tensor([[0, 1, 2]], dtype=torch.int32), torch.ones(4, 3)
  stats = {}
  out = mesh.clean_mesh(v, f, n, stats=stats)
  assert len(out) == 3 and all(a is b for a, b in zip(out, (v, f, n)))
  assert stats == {'vertices_removed': 0, 'faces_removed': 0, 'components_removed': 0}
  for kw in (dict(keep_components=-1), dict(min_views=-2)):
    with pytest.raises(ValueError):
      mesh.clean_mesh(v, f, **kw)
  with pytest.raises(ValueError, match='cameras'):
    mesh.clean_mesh(v, f, min_views=1)
  with pytest.raises(ValueError, match='NDC'):
    mesh.clean_mesh(v, f, min_views=1, cameras=(np.eye(3), np.zeros((1, 3, 4)), None, np.eye(3)),
                    camtype='perspective', image_size=(4, 4))
  with pytest.raises(ValueError, match='dataset'):
    mesh._clean_args(0, 1, None, None)
