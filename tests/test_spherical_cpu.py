"""Panorama (`render_camtype = 'pano'`) rays on the CPU: the float64 oracle against the reference's own
cast_spherical_rays (tests/golden/spherical.npz), the `mnrf_spherical_rays` ABI symbol and descriptor, and a
render-path dataset that now constructs with a panorama camera."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from oracle import o_spherical
from util import POSES, SIZES, golden, write_nerfpp_scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = golden('spherical')


@pytest.mark.parametrize('pose', POSES)
@pytest.mark.parametrize('hw', SIZES, ids=lambda hw: f'{hw[0]}x{hw[1]}')
def test_oracle_matches_reference(pose, hw):
  h, w = hw
  near, far = float(G['near']), float(G['far'])
  out = o_spherical.cast_spherical_rays(torch.tensor(G[f'pose_{pose}']), h, w, near, far)
  for f, key in (('origins', 'origins'), ('directions', 'directions'), ('viewdirs', 'directions'),
                 ('radii', 'radii'), ('imageplane', 'imageplane')):
    ref = G[f'{pose}_{h}x{w}_{key}']
    got = out[f].numpy()
    assert got.dtype == np.float64 and got.shape == ref.shape, (f, got.dtype, got.shape, ref.shape)
    err = float(np.abs(got - ref).max())
    assert err <= 1e-12 * max(1.0, float(np.abs(ref).max())), (pose, hw, f, err)
  for f, v in (('lossmult', 1.0), ('near', near), ('far', far), ('cam_idx', 0)):
    assert out[f].shape == (h, w, 1) and bool((out[f] == v).all()), f


def test_fixture_cases_are_not_degenerate():
  """The skewed pose really is not a rotation, the float32-rounded pose differs from the float64 one, and the
  grid reaches the poles, where the x neighbour coincides and the radius is half the equator's."""
  r = G['pose_skew'][:, :3]
  assert abs(np.linalg.det(r)) > 2.0 and np.abs(r @ r.T - np.diag(np.diag(r @ r.T))).max() > 0.1
  assert 0 < np.abs(G['pose_rot'] - G['pose_rot_f32']).max() < 1e-6
  rad = G['rot_32x64_radii']
  assert rad.min() > 0 and rad.max() / rad.min() > 1.9


def test_spherical_abi_v2_symbol_exported():
  from multinerf_b200 import lib
  if not os.path.exists(lib.LIB_PATH):
    from multinerf_b200 import build
    build.build()
  l = lib.load()
  assert l.mnrf_abi_version() == 2
  assert 'mnrf_spherical_rays' in lib.EXPORTED and hasattr(l, 'mnrf_spherical_rays')
  src = ('#include <stdio.h>\n#include "mnrf.h"\n'
         'int main(){printf("%zu\\n", sizeof(mnrf_spherical_desc)); return 0;}')
  with tempfile.TemporaryDirectory() as td:
    open(os.path.join(td, 'a.c'), 'w').write(src)
    subprocess.run(['gcc', '-I', os.path.join(ROOT, 'include'), os.path.join(td, 'a.c'), '-o',
                    os.path.join(td, 'a')], check=True)
    size = int(subprocess.run([os.path.join(td, 'a')], capture_output=True, text=True).stdout)
  assert size == ctypes.sizeof(lib.SphericalDesc) == 104


def test_cast_spherical_rays_rejects_bad_sizes_before_any_launch():
  from multinerf_b200 import camera_utils
  pose = G['pose_rot']
  for h, w in ((0, 4), (4, 0), (-1, 3)):
    with pytest.raises(ValueError, match='at least 1 x 1'):
      camera_utils.cast_spherical_rays(pose, h, w, 0.2, 1e6)
  with pytest.raises(ValueError, match=r'\[3, 4\] or \[4, 4\]'):
    camera_utils.cast_spherical_rays(pose[:, :3], 4, 8, 0.2, 1e6)


def test_pano_render_path_dataset_constructs(tmp_path):
  from multinerf_b200 import configs, datasets
  root = str(tmp_path)
  write_nerfpp_scene(root, np.random.default_rng(11))
  cfg = configs.Config(dataset_loader='tat_nerfpp', render_path=True, render_camtype='pano',
                       render_resolution=(16, 8))
  ds = datasets.load_dataset('test', root, cfg, device='cpu')
  assert ds.size == 4 and ds.images is None and (ds.height, ds.width) == (8, 16)
  assert ds.camtoworlds.shape == (4, 4, 4)
