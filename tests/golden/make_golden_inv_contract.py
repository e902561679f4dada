"""Generate tests/golden/inv_contract.npz by EXECUTING the reference's own internal/coord.py.

Run in the build container only (needs /root/reference):
    python tests/golden/make_golden_inv_contract.py
`coord.contract` and `coord.inv_contract` (coord.py:21-36) with the jax stand-in of tests/golden/standin (numpy),
on contracted points z whose norms cover [0, 2) -- the origin, the unit sphere from both sides and norms up to
2 - 2^-12 -- and on world points x whose norms run from 0 to 1e6.  Inputs and outputs are stored as the reference
returns them, with their dtype.
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
for missing in ['dm_pix', 'cv2', 'rawpy', 'mediapy', 'optax', 'pycolmap', 'matplotlib', 'tensorflow']:
  try:
    __import__(missing)
  except Exception:  # pylint: disable=broad-except
    sys.modules[missing] = mock.MagicMock()

from internal import coord  # noqa: E402


def main():
  rng = np.random.default_rng(31)
  dirs = rng.normal(size=(4096, 3))
  dirs /= np.linalg.norm(dirs, axis=-1, keepdims=True)
  norms = np.concatenate([[0.0, 1e-4, 0.5, 1.0 - 1e-6, 1.0, 1.0 + 1e-6, 1.5, 2 - 4 / 1023, 2 - 2 ** -12],
                          rng.uniform(0, 2 - 2 ** -12, 4096 - 9)])
  z = dirs * norms[:, None]
  wnorms = np.concatenate([[0.0, 0.5, 1.0, 1.0 + 1e-6, 2.0, 1e3, 1e6], 10 ** rng.uniform(-2, 6, 4096 - 7)])
  x = dirs * wnorms[:, None]
  out = {'z': z, 'inv_contract_z': np.asarray(coord.inv_contract(z)),
         'x': x, 'contract_x': np.asarray(coord.contract(x))}
  path = os.path.join(HERE, 'inv_contract.npz')
  np.savez_compressed(path, **out)
  print('inv_contract.npz', {k: (v.shape, v.dtype) for k, v in out.items()}, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
  main()
