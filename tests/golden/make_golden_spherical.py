"""Generate tests/golden/spherical.npz by EXECUTING the reference's own internal/camera_utils.py.

Run in the build container only (needs /root/reference):
    python tests/golden/make_golden_spherical.py
`cast_spherical_rays(camtoworld, height, width, near, far, xnp=np)` is what the reference's Dataset runs for
`render_camtype = 'pano'` (datasets.py:486-492), in float64.  Three poses (a random rotation plus translation,
the same pose rounded to float32, and a non-orthonormal pose: the rotation scaled by 2.5 and sheared) at six
panorama sizes, from 1 x 1 up.  Inputs and outputs are stored in float64.  `viewdirs` is the same array as
`directions` in the reference, which the generator asserts, so only `directions` is stored.
"""
import math
import os
import sys
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'standin'))
sys.path.insert(0, '/root/reference')
np.math = math
for missing in ['dm_pix', 'cv2', 'rawpy', 'mediapy', 'optax', 'pycolmap', 'matplotlib', 'tensorflow',
                'scipy.interpolate', 'PIL', 'PIL.Image', 'PIL.ExifTags']:
  try:
    __import__(missing)
  except Exception:  # pylint: disable=broad-except
    sys.modules[missing] = mock.MagicMock()

from internal import camera_utils  # noqa: E402

SIZES = [(1, 1), (1, 5), (4, 1), (2, 3), (17, 32), (32, 64)]       # (height, width)
NEAR, FAR = 0.2, 1e6


def main():
  rng = np.random.default_rng(23)
  q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
  if np.linalg.det(q) < 0:
    q[:, 0] *= -1
  pose = np.concatenate([q, rng.uniform(-1.5, 1.5, (3, 1))], axis=1)
  shear = np.array([[1.0, 0.3, 0.0], [0.0, 1.0, -0.2], [0.1, 0.0, 1.0]])
  poses = {'rot': pose,
           'rot_f32': pose.astype(np.float32).astype(np.float64),
           'skew': np.concatenate([2.5 * q @ shear, pose[:, 3:]], axis=1)}
  out = {'sizes': np.array(SIZES), 'near': np.float64(NEAR), 'far': np.float64(FAR)}
  for pname, p in poses.items():
    out[f'pose_{pname}'] = p
    for h, w in SIZES:
      rays = camera_utils.cast_spherical_rays(p, h, w, NEAR, FAR, xnp=np)
      assert rays.viewdirs is rays.directions
      for f in ['origins', 'directions', 'radii', 'imageplane']:
        a = np.asarray(getattr(rays, f))
        assert a.dtype == np.float64 and a.shape[:2] == (h, w), (f, a.dtype, a.shape)
        out[f'{pname}_{h}x{w}_{f}'] = a
      for f, v in (('lossmult', 1.), ('near', NEAR), ('far', FAR), ('cam_idx', 0)):
        assert np.array_equal(np.asarray(getattr(rays, f)), np.full((h, w, 1), v)), f
  path = os.path.join(HERE, 'spherical.npz')
  np.savez_compressed(path, **out)
  print('spherical.npz', len(out), 'arrays,', os.path.getsize(path), 'bytes')


if __name__ == '__main__':
  main()
