"""Meshes in contracted space on the host: the fp64 contraction of tests/contract_ref.py against the reference's own
coord.contract / coord.inv_contract (tests/golden/inv_contract.npz) and round trips, its Jacobian against finite
differences, Config.mesh_space parsing, default box and rejections, and the fp64 contracted TSDF fusion against
the world fusion where the contraction is the identity.  No GPU needed."""
import os

import numpy as np
import pytest

import contract_ref
import tsdf_ref

HERE = os.path.dirname(os.path.abspath(__file__))
EPS32 = float(np.finfo(np.float32).eps)


def test_restatement_matches_the_reference_fixture():
  g = np.load(os.path.join(HERE, 'golden', 'inv_contract.npz'))
  z, x = g['z'], g['x']
  r = np.linalg.norm(z, axis=-1)
  # the reference runs in fp32 and divides by 2 r - r^2, whose rounding grows as r / (2 - r) near r = 2
  want = contract_ref.inv_contract(z)
  tol = 16 * EPS32 * (1 + r / (2 - r))[:, None] * np.abs(want) + 1e-30
  assert np.all(np.abs(g['inv_contract_z'] - want) <= tol)
  want = contract_ref.contract(x)
  assert np.all(np.abs(g['contract_x'] - want) <= 16 * EPS32 * np.abs(want) + 1e-30)


def test_round_trips():
  rng = np.random.default_rng(3)
  d = rng.normal(size=(20000, 3))
  d /= np.linalg.norm(d, axis=-1, keepdims=True)
  z = d * rng.uniform(0, 2 - 4 / 1023, (20000, 1))
  assert np.allclose(contract_ref.contract(contract_ref.inv_contract(z)), z, rtol=1e-12, atol=1e-12)
  x = d * 10 ** rng.uniform(-3, 6, (20000, 1))
  assert np.allclose(contract_ref.inv_contract(contract_ref.contract(x)), x, rtol=1e-9, atol=1e-12)
  assert np.all(np.linalg.norm(contract_ref.contract(x), axis=-1) < 2)


def test_jacobian_against_finite_differences_and_symmetric():
  rng = np.random.default_rng(4)
  d = rng.normal(size=(500, 3))
  d /= np.linalg.norm(d, axis=-1, keepdims=True)
  x = d * 10 ** rng.uniform(-1, 3, (500, 1))
  x = x[np.abs(np.linalg.norm(x, axis=-1) - 1) > 1e-3]
  J = contract_ref.jacobian(x)
  assert np.allclose(J, np.transpose(J, (0, 2, 1)))
  fd = np.zeros_like(J)
  for a in range(3):
    step = 1e-6 * np.maximum(1, np.linalg.norm(x, axis=-1))[:, None] * np.eye(3)[a]
    fd[:, :, a] = (contract_ref.contract(x + step) - contract_ref.contract(x - step)) / (2 * step[:, a:a + 1])
  assert np.allclose(J, fd, rtol=1e-5, atol=1e-9)


def test_world_normals_are_level_set_normals():
  """A world sphere |x| = R is the contracted sphere |z| = 2 - 1/R: both have radial normals."""
  rng = np.random.default_rng(5)
  d = rng.normal(size=(100, 3))
  d /= np.linalg.norm(d, axis=-1, keepdims=True)
  z = d * 1.9
  n = contract_ref.world_normals(z, d)
  assert np.allclose(n, d)
  # a world plane x_0 = 3 is curved in contracted space; its contracted normal is the gradient of x_0(inv_contract(z))
  z = contract_ref.contract(np.stack([np.full(50, 3.0), rng.uniform(-2, 2, 50), rng.uniform(-2, 2, 50)], -1))
  h = 1e-7
  grad = np.stack([(contract_ref.inv_contract(z + h * e)[:, 0] - contract_ref.inv_contract(z - h * e)[:, 0]) / (2 * h)
                   for e in np.eye(3)], -1)
  assert np.allclose(contract_ref.world_normals(z, grad), [1, 0, 0], atol=1e-6)


def test_config_parsing_default_box_and_rejections():
  from multinerf_b200 import configs, mesh
  assert configs.Config().mesh_space == 'world'
  b = configs.load_config(gin_bindings=configs.GIN_360.strip().split('\n') + ["Config.mesh_space = 'contracted'"])
  assert b.config.mesh_space == 'contracted'
  assert mesh.default_bbox(b) == (-2.0, -2.0, -2.0, 2.0, 2.0, 2.0)
  assert mesh.validate_config(b) == 'density'
  assert mesh.default_bbox(configs.bundle_360()) == (-1.0, -1.0, -1.0, 1.0, 1.0, 1.0)
  b2 = configs.load_config(gin_bindings=configs.GIN_360.strip().split('\n') +
                           ["Config.mesh_space = 'contracted'", 'Config.mesh_bbox = (-2, -2, -1, 2, 2, 1)'])
  assert mesh.default_bbox(b2) == (-2.0, -2.0, -1.0, 2.0, 2.0, 1.0)
  with pytest.raises(ValueError, match='mesh_space'):
    mesh.validate_config(configs.load_config(gin_bindings=["Config.mesh_space = 'ndc'"]))
  bounded = configs.load_config(gin_bindings=["Config.mesh_space = 'contracted'"])
  with pytest.raises(ValueError, match='contraction'):
    mesh.validate_config(bounded)
  with pytest.raises(ValueError, match='contraction'):
    mesh.default_bbox(bounded)
  ff = configs.load_config(gin_bindings=configs.GIN_360.strip().split('\n') +
                           ["Config.mesh_space = 'contracted'", 'Config.forward_facing = True'])
  with pytest.raises(ValueError, match='forward-facing'):
    mesh.validate_config(ff)
  with pytest.raises(ValueError, match='mesh space'):
    mesh.density_grid(None, (-1, -1, -1, 1, 1, 1), 8, space='ndc')


def test_contracted_fusion_is_the_world_fusion_inside_the_unit_ball():
  """Inside the unit ball contract is the identity, so for a perspective camera d = sign(depth - t) |s - x| =
  (depth - t) |dir| with dir the direction (z = -1) of the ray through x: the world fusion's value times |dir|.
  Points with |p| >= 2 are never observed."""
  rng = np.random.default_rng(6)
  c2w = np.concatenate([np.eye(3), [[0.0], [0.0], [0.5]]], 1)        # looks along -z from (0, 0, 0.5)
  w2c = np.concatenate([c2w[:, :3].T, -c2w[:, :3].T @ c2w[:, 3:]], 1)[None]
  H = W = 16
  c2p = np.array([[[20.0, 0, W / 2], [0, 20.0, H / 2], [0, 0, 1]]])
  depth = rng.uniform(0.3, 0.8, (1, H, W))            # every surface point s inside the unit ball too
  acc = np.ones((1, H, W))
  pts = tsdf_ref.grid_points((9, 9, 9), (-0.4, -0.4, -0.6), 0.1)
  pts = pts[np.linalg.norm(pts, axis=-1) < 0.95]
  tau = 5.0
  tw, ww, *_ = tsdf_ref.integrate(pts, w2c, c2p, depth, acc, None, tau)
  tc, wc, *_ = contract_ref.integrate_contracted(pts, w2c, c2p, depth, acc, None, tau)
  assert np.array_equal(ww, wc) and ww.sum() > 100
  u, v, _, _ = tsdf_ref.project(pts, w2c[0], c2p[0])
  ok = ww > 0
  # s lies on the ray through x itself (direction at the continuous pixel (u, v), z = -1), not the pixel centre's
  dirn = np.sqrt(((u[ok] - W / 2) / 20.0) ** 2 + ((v[ok] - H / 2) / 20.0) ** 2 + 1)
  assert np.allclose(tc[ok], tw[ok] * dirn, rtol=1e-9, atol=1e-12)
  far = np.array([[0.0, 0.0, -1.99], [0.0, 0.0, 2.0], [2.0, 0.0, 0.0]])
  _, wf, *_ = contract_ref.integrate_contracted(far, w2c, c2p, depth, acc, None, tau)
  assert wf[1] == 0 and wf[2] == 0


def test_clamp_to_ball():
  """Simplified contracted vertices beyond 2 - 2^-12 are scaled back to that radius along their direction; the rest
  are returned bit for bit."""
  import torch
  from multinerf_b200 import mesh
  v = torch.tensor([[0.5, 0.0, 0.0], [1.9, 0.1, 0.0], [2.1, 0.0, 0.0], [0.0, -1.5, 1.5], [0.0, 0.0, 1.9999]])
  out = mesh.clamp_to_ball(v)
  r = out.double().norm(dim=-1)
  assert torch.equal(out[[0, 1]], v[[0, 1]])
  assert (r <= mesh.CONTRACTED_MAX_RADIUS + 1e-6).all() and (r[2:] > mesh.CONTRACTED_MAX_RADIUS - 1e-6).all()
  assert torch.allclose(torch.nn.functional.normalize(out[2:], dim=-1), torch.nn.functional.normalize(v[2:], dim=-1))
  assert (out.double().square().sum(-1) < 4).all()
