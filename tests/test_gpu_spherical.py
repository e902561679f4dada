"""Panorama rays on the device (mnrf_spherical_rays through multinerf_b200.camera_utils.cast_spherical_rays)
against the reference's own float64 outputs (tests/golden/spherical.npz) and the float64 oracle, and
render.py with `render_camtype = 'pano'` end to end.  Needs an H100.

Bounds: origins are fl32 of the reference bit for bit and imageplane is exactly 0; directions / viewdirs within
2.4e-7 * max(1, |ref|_max) (two fp32 ulps at 1: the output rounding plus the fp64 sin / cos and FMA differences
it can expose); radii within 2.4e-7 relative, element by element, which holds because the kernel takes the
neighbour differences in fp64 before rounding."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

from oracle import o_spherical
from util import POSES, SIZES, golden, write_nerfpp_scene

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = golden('spherical')
TOL = 2.4e-7


def _check(rays, ref, tag):
  """`ref`: dict of float64 arrays (origins, directions, viewdirs, radii, imageplane)."""
  got = {f: getattr(rays, f).cpu().numpy() for f in ref}
  for f in ref:
    assert got[f].dtype == np.float32 and got[f].shape == ref[f].shape, (tag, f, got[f].dtype, got[f].shape)
  np.testing.assert_array_equal(got['origins'], ref['origins'].astype(np.float32), err_msg=tag)
  assert not got['imageplane'].any(), tag
  for f in ('directions', 'viewdirs'):
    err = float(np.abs(got[f].astype(np.float64) - ref[f]).max())
    assert err <= TOL * max(1.0, float(np.abs(ref[f]).max())), (tag, f, err)
  rel = np.abs(got['radii'].astype(np.float64) - ref['radii']) / np.abs(ref['radii'])
  assert float(rel.max()) <= TOL, (tag, 'radii', float(rel.max()))


@pytest.mark.parametrize('pose', POSES)
@pytest.mark.parametrize('hw', SIZES, ids=lambda hw: f'{hw[0]}x{hw[1]}')
def test_kernel_matches_reference(pose, hw):
  from multinerf_b200 import camera_utils
  h, w = hw
  rays = camera_utils.cast_spherical_rays(G[f'pose_{pose}'], h, w, float(G['near']), float(G['far']))
  key = lambda f: G[f'{pose}_{h}x{w}_{f}']
  _check(rays, {'origins': key('origins'), 'directions': key('directions'), 'viewdirs': key('directions'),
                'radii': key('radii'), 'imageplane': key('imageplane')}, f'{pose} {h}x{w}')


def test_kernel_matches_oracle_at_panorama_size():
  from multinerf_b200 import camera_utils
  pose = G['pose_skew']
  for h, w in ((1024, 2048), (1, 1)):
    rays = camera_utils.cast_spherical_rays(torch.tensor(pose), h, w, 0.2, 1e6)
    ref = o_spherical.cast_spherical_rays(torch.tensor(pose), h, w, 0.2, 1e6)
    _check(rays, {f: ref[f].numpy() for f in ('origins', 'directions', 'viewdirs', 'radii', 'imageplane')},
           f'oracle {h}x{w}')
  assert rays.origins.shape == (1, 1, 3) and rays.radii.shape == (1, 1, 1) and rays.imageplane.shape == (1, 1, 2)


def test_metadata_and_errors():
  from multinerf_b200 import camera_utils, lib
  pose4 = np.eye(4)
  pose4[:3, :4] = G['pose_rot']
  rays = camera_utils.cast_spherical_rays(pose4, 3, 7, 0.25, 40.0)
  ref = camera_utils.cast_spherical_rays(G['pose_rot'], 3, 7, 0.25, 40.0)
  assert torch.equal(rays.directions, ref.directions) and torch.equal(rays.radii, ref.radii)
  for f, v, dt in (('lossmult', 1.0, torch.float32), ('near', 0.25, torch.float32), ('far', 40.0, torch.float32),
                   ('cam_idx', 0, torch.int32)):
    t = getattr(rays, f)
    assert t.is_cuda and t.dtype == dt and t.shape == (3, 7, 1) and bool((t == v).all()), f
  assert rays.exposure_idx is None and rays.exposure_values is None
  with pytest.raises(ValueError):
    camera_utils.cast_spherical_rays(pose4, 0, 7, 0.25, 40.0)
  # the C entry rejects what the Python surface would not pass, before any launch
  l = lib.load()
  d = lib.SphericalDesc(0, 4, (ctypes.c_double * 12)(*np.asarray(G['pose_rot']).reshape(-1)))
  buf = torch.empty(64, device='cuda')
  p = lib.ptr(buf)
  assert l.mnrf_spherical_rays(ctypes.byref(d), p, p, p, p, p, lib.stream_ptr()) != 0
  assert 'height and width' in l.mnrf_last_error().decode()
  d.height = 4
  assert l.mnrf_spherical_rays(ctypes.byref(d), p, None, p, p, p, lib.stream_ptr()) != 0
  assert 'null pointer' in l.mnrf_last_error().decode()


def _gin(tmp_path, data, ckpt):
  path = os.path.join(str(tmp_path), 'pano.gin')
  with open(path, 'w') as f:
    f.write(f"""Config.dataset_loader = 'tat_nerfpp'
Config.data_dir = '{data}'
Config.checkpoint_dir = '{ckpt}'
Config.near = 0.2
Config.far = 1e6
Config.render_path = True
Config.render_camtype = 'pano'
Config.render_resolution = (48, 24)
Config.render_chunk_size = 512
Config.render_save_async = False
Model.raydist_fn = @jnp.reciprocal
Model.opaque_background = True
Model.num_prop_samples = 32
Model.num_nerf_samples = 16
PropMLP.warp_fn = @coord.contract
PropMLP.net_depth = 2
PropMLP.net_width = 64
PropMLP.disable_density_normals = True
PropMLP.disable_rgb = True
NerfMLP.warp_fn = @coord.contract
NerfMLP.net_depth = 4
NerfMLP.net_width = 128
NerfMLP.bottleneck_width = 64
NerfMLP.net_width_viewdirs = 64
NerfMLP.disable_density_normals = True
""")
  return path


def test_render_script_writes_panoramas(tmp_path):
  """render.py on a NeRF++ scene's camera path with panorama cameras and no checkpoint (the seeded init):
  one 24 x 48 colour PNG plus distance and acc TIFFs per path pose, and frame k is render_image on
  cast_spherical_rays of path pose k from the same seeded model."""
  sys.path.insert(0, ROOT)
  import render as render_script
  from multinerf_b200 import camera_utils, configs, datasets, models, train_utils, utils
  data, ckpt = str(tmp_path / 'scene'), str(tmp_path / 'ckpt')
  write_nerfpp_scene(data, np.random.default_rng(5))
  gin = _gin(tmp_path, data, ckpt)
  render_script.main([f'--gin_configs={gin}'])
  out = os.path.join(ckpt, 'render', 'path_renders_step_0')
  files = set(os.listdir(out))
  for i in range(4):
    for name in (f'color_{i:03d}.png', f'distance_mean_{i:03d}.tiff', f'distance_median_{i:03d}.tiff',
                 f'acc_{i:03d}.tiff'):
      assert name in files, (name, sorted(files))
  assert utils.load_img(os.path.join(out, 'acc_000.tiff')).shape == (24, 48)

  bundle = configs.load_config([gin])
  ds = datasets.load_dataset('test', data, bundle.config)
  assert (ds.height, ds.width) == (24, 48)
  for b in (ds.peek(), next(ds), ds.generate_ray_batch(2)):
    assert b.rgb is None and b.rays.origins.shape == (24, 48, 3) and b.rays.origins.is_cuda
  k = 2
  rays = camera_utils.cast_spherical_rays(ds.camtoworlds[k], 24, 48, bundle.config.near, bundle.config.far)
  assert torch.equal(ds.generate_ray_batch(k).rays.directions, rays.directions)
  model, state, _, _, _ = train_utils.setup_model(bundle, 20200823)
  pfn = train_utils.create_render_fn(model)
  rendering = models.render_image(lambda rng, r: pfn(state.params, 1., None, r), rays, None, bundle, verbose=False)
  want = (np.clip(np.nan_to_num(rendering['rgb'].cpu().numpy()), 0., 1.) * 255.).astype(np.int32)
  got = utils.load_img(os.path.join(out, f'color_{k:03d}.png')).astype(np.int32)
  assert got.shape == (24, 48, 3)
  assert int(np.abs(got - want).max()) <= 1
