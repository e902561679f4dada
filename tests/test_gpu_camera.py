"""Device ray generation (mnrf_pixels_to_rays through multinerf_b200.camera_utils) vs the CPU oracle
and the reference's own outputs (tests/golden/camera.npz).  Needs an H100.

Tolerance (fp32 path): 1e-5 * max(1, |x|_max) on origins / directions / viewdirs / imageplane;
radii are differences of nearly equal fp32 directions, so 2e-3 relative to the largest radius
(the reference's own fp32 and fp64 paths differ by that much)."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import o_camera

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, 'golden', 'camera.npz'))
FIELDS = ['origins', 'directions', 'viewdirs', 'radii', 'imageplane']


def _cameras(name):
  dist = None
  if name in ('dist', 'fisheye'):
    dist = {str(k): float(v) for k, v in zip(G['dist_keys'], G['dist_vals'])}
  poses = G['ndc_poses'] if name == 'ndc' else G['camtoworlds']
  p2c = G['pixtocams']
  if name == 'single':
    poses, p2c = poses[0], p2c[0]
  ndc = G['pixtocam_ndc'] if name == 'ndc' else None
  return p2c, poses, dist, ndc


def _check(got, ref, f, tag):
  got = got.detach().cpu().numpy().astype(np.float64)
  ref = np.asarray(ref, np.float64)
  assert got.shape == ref.shape, (tag, f, got.shape, ref.shape)
  scale = max(1.0, float(np.abs(ref).max()))
  lim = 1e-5 * scale if f != 'radii' else 2e-3 * float(np.abs(ref).max())
  err = float(np.abs(got - ref).max())
  assert err <= lim, (tag, f, err, lim)


@pytest.mark.parametrize('name', ['persp', 'dist', 'fisheye', 'ndc', 'single'])
def test_cast_ray_batch_vs_oracle_and_reference(name):
  from multinerf_b200 import camera_utils, utils
  p2c, poses, dist, ndc = _cameras(name)
  B = G['pix_x'].shape[0]
  meta = lambda v: np.full((B, 1), v, np.float32)
  pixels = utils.Pixels(pix_x_int=G['pix_x'], pix_y_int=G['pix_y'], lossmult=meta(1), near=meta(0.2),
                        far=meta(1e6), cam_idx=G['cam_idx'])
  camtype = camera_utils.ProjectionType.FISHEYE if name == 'fisheye' else camera_utils.ProjectionType.PERSPECTIVE
  rays = camera_utils.cast_ray_batch((p2c, poses, dist, ndc), pixels, camtype)
  torch.cuda.synchronize()
  # oracle on the same inputs, fp32
  t32 = lambda a: None if a is None else torch.tensor(np.asarray(a), dtype=torch.float32)
  opix = types.SimpleNamespace(pix_x_int=torch.tensor(G['pix_x']), pix_y_int=torch.tensor(G['pix_y']),
                               cam_idx=torch.tensor(G['cam_idx']))
  o = o_camera.cast_ray_batch((t32(p2c), t32(poses), dist, t32(ndc)), opix,
                              o_camera.FISHEYE if name == 'fisheye' else o_camera.PERSPECTIVE)
  for f in FIELDS:
    _check(getattr(rays, f), o[f].numpy(), f, name + ':oracle')
    _check(getattr(rays, f), G[f'{name}_f32_{f}'], f, name + ':reference fp32')
    _check(getattr(rays, f), G[f'{name}_f64_{f}'], f, name + ':reference fp64')
  # metadata passes through untouched (camera_utils.py:676-688)
  assert rays.near is pixels.near and rays.cam_idx is pixels.cam_idx


def test_pixels_to_rays_image_grid_and_errors():
  from multinerf_b200 import camera_utils
  W, H = 37, 23
  p2c = camera_utils.get_pixtocam(55.0, W, H)
  pose = G['camtoworlds'][1]
  px, py = camera_utils.pixel_coordinates(W, H)
  o, d, v, r, ip = camera_utils.pixels_to_rays(px, py, p2c, pose)
  assert o.shape == (H, W, 3) and r.shape == (H, W, 1) and ip.shape == (H, W, 2)
  oo, od, ov, orr, oip = o_camera.pixels_to_rays(torch.tensor(px), torch.tensor(py),
                                                 torch.tensor(p2c, dtype=torch.float32),
                                                 torch.tensor(pose, dtype=torch.float32))
  for f, got, ref in zip(FIELDS, (o, d, v, r, ip), (oo, od, ov, orr, oip)):
    _check(got, ref.numpy(), f, 'grid')
  # per-pixel matrices (SH + [3,3]) give the same rays as the single camera
  o2, d2, v2, r2, ip2 = camera_utils.pixels_to_rays(px, py, np.broadcast_to(p2c, (H, W, 3, 3)),
                                                    np.broadcast_to(pose, (H, W, 3, 4)))
  assert torch.equal(o, o2) and torch.equal(d, d2) and torch.equal(r, r2) and torch.equal(ip, ip2)
  assert float((v.norm(dim=-1) - 1).abs().max()) < 1e-6
  with pytest.raises(ValueError):
    camera_utils.pixels_to_rays(px, py, p2c, pose, camtype='orthographic')
  with pytest.raises(TypeError):
    camera_utils.pixels_to_rays(px, py, p2c, pose, distortion_params={'k9': 1.0})


def test_train_step_with_device_ray_generation():
  """Config.cast_rays_in_train_step (train_utils.py:266-268): a step fed with utils.Pixels + cameras
  equals the step fed with the rays those pixels generate."""
  from multinerf_b200 import camera_utils, models, train_utils, utils
  from model_parity import mini360
  p2c, poses, dist, ndc = _cameras('dist')
  B = 256
  rng = np.random.default_rng(5)
  px, py = rng.integers(0, 160, B).astype(np.int32), rng.integers(0, 120, B).astype(np.int32)
  cam = rng.integers(0, poses.shape[0], (B, 1)).astype(np.int32)
  meta = lambda v: np.full((B, 1), v, np.float32)
  pixels = utils.Pixels(pix_x_int=px, pix_y_int=py, lossmult=meta(1), near=meta(0.2), far=meta(1e6), cam_idx=cam)
  cameras = (p2c, poses, dist, ndc)
  target = rng.uniform(0, 1, (B, 3)).astype(np.float32)
  rand = {'jitter': [torch.tensor(rng.uniform(0, 1, (B, 1)).astype(np.float32)) for _ in range(3)]}
  grads = []
  for cast in (True, False):
    bundle = mini360()
    bundle.config.cast_rays_in_train_step = cast
    rays = pixels if cast else camera_utils.cast_ray_batch(cameras, pixels)
    model, variables = models.construct_model(4, utils.dummy_rays(), bundle)
    step_fn = train_utils.create_train_step(model, bundle.config)
    state = train_utils.TrainState(variables)
    state, stats, _ = step_fn(rand, state, utils.Batch(rays=rays, rgb=target), cameras if cast else None, 0.5)
    torch.cuda.synchronize()
    grads.append((model.params.grads.clone(), stats.materialize()['loss']))
  # same rays -> same step; the split-K weight-gradient reduction uses fp32 atomics, so two runs
  # agree to rounding, not bit for bit
  rel = float((grads[0][0] - grads[1][0]).norm() / grads[1][0].norm())
  assert rel < 1e-3, rel
  assert abs(grads[0][1] - grads[1][1]) <= 1e-5 * abs(grads[1][1])
  bundle = mini360()
  bundle.config.cast_rays_in_train_step = True
  model, variables = models.construct_model(4, utils.dummy_rays(), bundle)
  step_fn = train_utils.create_train_step(model, bundle.config)
  with pytest.raises(ValueError):
    step_fn(rand, train_utils.TrainState(variables), utils.Batch(rays=pixels, rgb=target), None, 0.5)
