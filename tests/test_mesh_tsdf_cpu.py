"""TSDF mesh extraction on the host: the fp64 forward projection of tests/tsdf_ref.py against the oracle's ray
caster, the camera matrices mesh.fuse_tsdf hands the kernel, and the validation of Config.mesh_method.  No GPU
needed."""
import math

import numpy as np
import pytest
import torch

import tsdf_ref
from oracle import o_camera


def _look_at(eye, target, up=(0.0, 0.0, 1.0)):
  """camtoworld [3, 4] (OpenGL axes: the camera looks along -z)."""
  eye = np.asarray(eye, np.float64)
  z = eye - np.asarray(target, np.float64)
  z /= np.linalg.norm(z)
  x = np.cross(up, z)
  x /= np.linalg.norm(x)
  return np.concatenate([np.stack([x, np.cross(z, x), z], 1), eye[:, None]], 1)


def _w2c(c2w):
  r = c2w[:, :3]
  return np.concatenate([r.T, -r.T @ c2w[:, 3:]], 1)


CAMERAS = {
    'perspective': ('perspective', None),
    'opencv': ('perspective', {'k1': -0.08, 'k2': 0.02, 'k3': 0.0, 'p1': 1.5e-3, 'p2': -1e-3}),
    'fisheye': ('fisheye', None),
    'fisheye_distorted': ('fisheye', {'k1': 0.03, 'k2': -0.01, 'k3': 2e-3, 'k4': -4e-4}),
}


@pytest.mark.parametrize('name', sorted(CAMERAS))
def test_projection_inverts_the_oracle_ray_caster(name):
  """project(o + t d) of each pixel's fp64 ray returns the pixel's centre and t."""
  camtype, dist = CAMERAS[name]
  rng = np.random.default_rng(1)
  W, H = 64, 48
  K = np.array([[55.0, 0.3, 31.2], [0.0, 57.0, 24.9], [0.0, 0.0, 1.0]])
  if camtype == 'fisheye':
    # up to ~150 degrees off the axis at the corners; ~90 with distortion, where the polynomial stays monotonic
    K[:2, :2] = [[14.0, 0.0], [0.0, 14.5]] if dist is None else [[25.0, 0.0], [0.0, 25.5]]
  c2w = _look_at(rng.normal(size=3) * 2, rng.normal(size=3) * 0.2)
  xs, ys = np.meshgrid(np.arange(W), np.arange(H), indexing='xy')
  p2c = np.linalg.inv(K)
  o, d, _, _, _ = o_camera.pixels_to_rays(torch.tensor(xs.reshape(-1)), torch.tensor(ys.reshape(-1)),
                                          torch.tensor(p2c), torch.tensor(c2w), distortion_params=dist,
                                          camtype=o_camera.FISHEYE if camtype == 'fisheye' else o_camera.PERSPECTIVE)
  o, d = o.numpy(), d.numpy()
  t = rng.uniform(0.2, 6.0, len(o))
  u, v, tt, valid = tsdf_ref.project(o + t[:, None] * d, _w2c(c2w), K, camtype, dist)
  assert valid.all()
  tol = 1e-6 if dist is None else 1e-5               # the ray caster's 10 Newton steps of undistortion
  assert np.abs(u - (xs.reshape(-1) + 0.5)).max() < tol
  assert np.abs(v - (ys.reshape(-1) + 0.5)).max() < tol
  assert np.abs(tt - t).max() < 1e-9 * 6 + tol * 1e-2


def test_projection_rejects_points_without_a_pixel():
  c2w = _look_at((0.0, -3.0, 0.0), (0.0, 0.0, 0.0))
  behind = np.array([[0.0, -4.0, 0.0], [0.3, -5.0, 0.2], [0.0, -3.0, 0.0]])
  _, _, _, valid = tsdf_ref.project(behind, _w2c(c2w), np.eye(3), 'perspective')
  assert not valid.any()
  # a fisheye sees behind itself, except straight back along its axis (theta = pi) and at its own centre
  _, _, t, valid = tsdf_ref.project(behind, _w2c(c2w), np.eye(3), 'fisheye')
  assert list(valid) == [False, True, False]
  assert math.isclose(t[1], math.sqrt(0.3 ** 2 + 2.0 ** 2 + 0.2 ** 2))


def test_camera_matrices_are_the_fp64_inverses():
  from multinerf_b200 import mesh
  rng = np.random.default_rng(2)
  c2w = np.stack([_look_at(rng.normal(size=3) * 3, (0, 0, 0)) for _ in range(3)])
  p2c = np.linalg.inv(np.array([[50.0, 0, 20], [0, 52, 15], [0, 0, 1]]))
  w2c, c2p = mesh.camera_matrices((p2c, c2w, None, None), 'cpu')
  assert w2c.shape == (3, 3, 4) and c2p.shape == (1, 3, 3) and w2c.dtype == torch.float32
  for k in range(3):
    assert np.allclose(w2c[k].double().numpy(), _w2c(c2w[k]), atol=1e-6)
    full = np.concatenate([c2w[k], [[0, 0, 0, 1]]]) @ np.concatenate([w2c[k].double().numpy(), [[0, 0, 0, 1]]])
    assert np.allclose(full, np.eye(4), atol=1e-6)
  assert np.allclose(c2p[0].double().numpy() @ p2c, np.eye(3), atol=1e-6)
  _, c2p3 = mesh.camera_matrices((np.stack([p2c] * 3), c2w, None, None), 'cpu')
  assert c2p3.shape == (3, 3, 3)


def test_mesh_method_validation():
  from multinerf_b200 import configs, mesh
  c = configs.Config()
  assert (c.mesh_method, c.mesh_tsdf_truncation) == ('density', 3.0)
  assert mesh.validate_config(configs.bundle_360()) == 'density'
  b = configs.load_config(gin_bindings=["Config.mesh_method = 'tsdf'", 'Config.mesh_tsdf_truncation = 1.5'])
  assert mesh.validate_config(b) == 'tsdf' and b.config.mesh_tsdf_truncation == 1.5
  with pytest.raises(ValueError, match='mesh_method'):
    mesh.validate_config(configs.load_config(gin_bindings=["Config.mesh_method = 'poisson'"]))
  with pytest.raises(ValueError, match='forward-facing'):
    mesh.validate_config(configs.load_config(gin_bindings=["Config.mesh_method = 'tsdf'",
                                                           'Config.forward_facing = True']))
  for bad in ('0.5', '0.', '-2.'):
    with pytest.raises(ValueError, match='truncation'):
      mesh.validate_config(configs.load_config(gin_bindings=["Config.mesh_method = 'tsdf'",
                                                             f'Config.mesh_tsdf_truncation = {bad}']))
  # the density method does not look at the TSDF fields
  assert mesh.validate_config(configs.load_config(gin_bindings=['Config.mesh_tsdf_truncation = 0.5',
                                                                'Config.forward_facing = True'])) == 'density'


def test_fuse_tsdf_rejects_ndc_cameras():
  from multinerf_b200 import mesh
  with pytest.raises(ValueError, match='NDC'):
    mesh.fuse_tsdf([], (np.eye(3), np.zeros((1, 3, 4)), None, np.eye(3)), 'perspective', (-1, -1, -1, 1, 1, 1),
                   8, 3.0, device='cpu')
