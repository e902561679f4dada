"""Shared helpers for the tests."""
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def golden(name):
  return np.load(os.path.join(GOLDEN, name + '.npz'))


# the panorama poses and image sizes of tests/golden/spherical.npz
POSES = ['rot', 'rot_f32', 'skew']
SIZES = [tuple(int(v) for v in s) for s in golden('spherical')['sizes']]


def T(x):
  return torch.as_tensor(np.asarray(x))


def close(a, b, atol=1e-5, rtol=1e-5, msg=''):
  a = np.asarray(a.detach().cpu() if isinstance(a, torch.Tensor) else a, dtype=np.float64)
  b = np.asarray(b.detach().cpu() if isinstance(b, torch.Tensor) else b, dtype=np.float64)
  assert a.shape == b.shape, (msg, a.shape, b.shape)
  a, b = np.atleast_1d(a), np.atleast_1d(b)
  both_inf = np.isinf(a) & np.isinf(b) & (np.sign(a) == np.sign(b))
  both_nan = np.isnan(a) & np.isnan(b)
  err = np.abs(a - b)
  err[both_inf | both_nan] = 0
  tol = atol + rtol * np.abs(b)
  tol[both_inf | both_nan] = 1
  bad = ~(err <= tol)
  assert not bad.any(), (f'{msg}: {bad.sum()} / {bad.size} mismatches, max err '
                         f'{np.nanmax(err):.3e} at {np.unravel_index(np.nanargmax(err), err.shape)}')


def kernel_rays(rng, b):
  """(origins, directions, radii) of b rays for the kernel tests: origins in the unit cube, directions of length
  0.8-1.2."""
  o = rng.uniform(-1, 1, (b, 3)).astype(np.float32)
  d = rng.normal(size=(b, 3)).astype(np.float32)
  d = (d / np.linalg.norm(d, axis=-1, keepdims=True) * rng.uniform(0.8, 1.2, (b, 1))).astype(np.float32)
  radii = rng.uniform(5e-4, 1e-3, (b, 1)).astype(np.float32)
  return torch.tensor(o), torch.tensor(d), torch.tensor(radii)


def write_nerfpp_scene(root, rng, n_train=3, n_test=2, n_path=4, height=6, width=10):
  """A scene in NeRF++'s layout (datasets.py:720-764): <split>/{pose,intrinsics}/*.txt and, outside
  camera_path/, <split>/rgb/*.png.  Poses are random rotations and positions."""
  from PIL import Image
  for split, n in (('train', n_train), ('test', n_test), ('camera_path', n_path)):
    for i in range(n):
      m = np.eye(4)
      m[:3, :3] = np.linalg.qr(rng.normal(size=(3, 3)))[0]
      m[:3, 3] = rng.normal(size=3)
      K = np.eye(4)
      K[0, 0] = K[1, 1] = 37.5
      K[0, 2], K[1, 2] = width / 2, height / 2
      for d, mat in (('pose', m), ('intrinsics', K)):
        os.makedirs(os.path.join(root, split, d), exist_ok=True)
        np.savetxt(os.path.join(root, split, d, f'{i:03d}.txt'), mat.reshape(1, 16))
      if split != 'camera_path':
        os.makedirs(os.path.join(root, split, 'rgb'), exist_ok=True)
        img = rng.integers(0, 256, (height, width, 3), dtype=np.uint8)
        Image.fromarray(img).save(os.path.join(root, split, 'rgb', f'{i:03d}.png'))
