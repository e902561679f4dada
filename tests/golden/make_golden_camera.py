"""Generate tests/golden/camera.npz by EXECUTING the reference's own internal/camera_utils.py.

Run in the build container only (needs /root/reference):
    python tests/golden/make_golden_camera.py
`pixels_to_rays` / `cast_ray_batch` / `convert_to_ndc` take an `xnp` module: the fixture holds the
outputs of both the float64 numpy path (`xnp=np`, what the reference's Dataset thread runs) and
the float32 path (`xnp=jnp` under the numpy stand-in for jax.numpy, what the reference runs inside
the train step when `cast_rays_in_train_step=True`).  Inputs are seeded and stored next to the
outputs, so the tests need nothing but the .npz.
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

import jax.numpy as jnp  # noqa: E402  (the stand-in)
from internal import camera_utils, utils  # noqa: E402

F = np.float32


def random_pose(rng):
  a = rng.normal(size=(3, 3))
  q, _ = np.linalg.qr(a)
  if np.linalg.det(q) < 0:
    q[:, 0] *= -1
  t = rng.uniform(-1.5, 1.5, (3, 1))
  return np.concatenate([q, t], axis=1)


def forward_pose(rng):
  w = rng.normal(size=3) * 0.08
  K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
  q, _ = np.linalg.qr(np.eye(3) + K + 0.5 * K @ K)
  q = q * np.sign(np.diag(q))[None, :]
  return np.concatenate([q, rng.uniform(-0.3, 0.3, (3, 1))], axis=1)


def extra_cases(rng, out):
  """The edges of the camera model, each stored under its own prefix with its inputs: `corners` (the border and
  corners of the image under strong barrel distortion), `aniso` (fx != fy and off-centre principal points),
  `widefish` (every pixel of a fisheye whose corners pass theta = pi; even-sized, so no pixel sits on the axis),
  `ndcwide` (NDC on a non-square image) and `fishcentre` (every pixel of a 5 x 5 fisheye: its centre maps to
  (0, 0), where sin(theta) / theta is 0 / 0 and the reference returns NaN)."""
  P, FISH = camera_utils.ProjectionType.PERSPECTIVE, camera_utils.ProjectionType.FISHEYE
  W, H = 160, 120
  xs, ys = np.arange(W), np.arange(H)
  bx = np.concatenate([xs, xs, np.zeros(H, int), np.full(H, W - 1)]).astype(np.int32)
  by = np.concatenate([np.zeros(W, int), np.full(W, H - 1), ys, ys]).astype(np.int32)
  grid = lambda w, h: [a.reshape(-1).astype(np.int32) for a in np.meshgrid(np.arange(w), np.arange(h), indexing='xy')]
  cases = {}
  cases['corners'] = dict(
      p2c=np.stack([camera_utils.get_pixtocam(f, W, H) for f in (140.0, 170.0, 200.0)]),
      poses=np.stack([random_pose(rng) for _ in range(3)]), pix=(bx, by),
      dist=dict(k1=-0.25, k2=0.03, k3=0.0, k4=0.0, p1=0.0, p2=0.0), camtype=P)
  aniso = []
  for _ in range(3):
    fx = rng.uniform(60, 140)
    fy = fx * np.exp(rng.uniform(np.log(0.5), np.log(2.0)))
    aniso.append(np.linalg.inv(camera_utils.intrinsic_matrix(fx, fy, W * rng.uniform(0.4, 0.6),
                                                             H * rng.uniform(0.4, 0.6))))
  cases['aniso'] = dict(p2c=np.stack(aniso), poses=np.stack([random_pose(rng) for _ in range(3)]),
                        pix=(rng.integers(0, W, 300).astype(np.int32), rng.integers(0, H, 300).astype(np.int32)),
                        camtype=P)
  cases['widefish'] = dict(p2c=camera_utils.get_pixtocam(8.0, 60, 44)[None], poses=random_pose(rng)[None],
                           pix=grid(60, 44), camtype=FISH)
  cases['ndcwide'] = dict(p2c=np.stack([camera_utils.get_pixtocam(f, W, 80) for f in (100.0, 110.0, 90.0)]),
                          poses=np.stack([forward_pose(rng) for _ in range(3)]),
                          pix=(rng.integers(0, W, 300).astype(np.int32), rng.integers(0, 80, 300).astype(np.int32)),
                          ndc=camera_utils.get_pixtocam(100.0, W, 80), camtype=P)
  cases['fishcentre'] = dict(p2c=camera_utils.get_pixtocam(7.0, 5, 5)[None], poses=random_pose(rng)[None],
                             pix=grid(5, 5), camtype=FISH)
  out['fishcentre_size'] = np.array([5, 5], np.int32)
  for name, c in cases.items():
    px, py = c['pix']
    B = px.shape[0]
    n = c['p2c'].shape[0]
    cam_idx = (rng.integers(0, n, (B, 1)) if n > 1 else np.zeros((B, 1))).astype(np.int32)
    out.update({f'{name}_pix_x': px, f'{name}_pix_y': py, f'{name}_cam_idx': cam_idx,
                f'{name}_pixtocams': c['p2c'], f'{name}_camtoworlds': c['poses']})
    if c.get('dist'):
      out[f'{name}_dist_keys'] = np.array(list(c['dist'].keys()))
      out[f'{name}_dist_vals'] = np.array(list(c['dist'].values()))
    if c.get('ndc') is not None:
      out[f'{name}_pixtocam_ndc'] = c['ndc']
    meta = lambda v: np.full((B, 1), v, F)
    for tag, xnp, dt in [('f64', np, np.float64), ('f32', jnp, np.float32)]:
      cams = (c['p2c'].astype(dt), c['poses'].astype(dt), c.get('dist'),
              None if c.get('ndc') is None else c['ndc'].astype(dt))
      pixels = utils.Pixels(pix_x_int=px, pix_y_int=py, lossmult=meta(1), near=meta(0.2), far=meta(1e6),
                            cam_idx=cam_idx)
      with np.errstate(all='ignore'):
        rays = camera_utils.cast_ray_batch(cams, pixels, c['camtype'], xnp=xnp)
      for f in ['origins', 'directions', 'viewdirs', 'radii', 'imageplane']:
        out[f'{name}_{tag}_{f}'] = np.asarray(getattr(rays, f))


def main():
  rng = np.random.default_rng(11)
  out = {}
  n_cam, B = 5, 257
  W, H = 160, 120
  focals = rng.uniform(100.0, 200.0, n_cam)
  pixtocams = np.stack([camera_utils.get_pixtocam(f, W, H) for f in focals])
  camtoworlds = np.stack([random_pose(rng) for _ in range(n_cam)])
  # forward-facing poses for the NDC case: small rotations about identity, looking down -z
  ndc_poses = []
  for _ in range(n_cam):
    w = rng.normal(size=3) * 0.08
    K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    R = np.eye(3) + K + 0.5 * K @ K
    q, _ = np.linalg.qr(R)
    q = q * np.sign(np.diag(q))[None, :]
    ndc_poses.append(np.concatenate([q, rng.uniform(-0.3, 0.3, (3, 1))], axis=1))
  ndc_poses = np.stack(ndc_poses)
  pix_x = rng.integers(0, W, B).astype(np.int32)
  pix_y = rng.integers(0, H, B).astype(np.int32)
  cam_idx = rng.integers(0, n_cam, (B, 1)).astype(np.int32)
  dist = dict(k1=0.05, k2=-0.02, k3=0.004, k4=0.0, p1=0.001, p2=-0.0015)
  pixtocam_ndc = camera_utils.get_pixtocam(150.0, W, H)
  out.update(pixtocams=pixtocams, camtoworlds=camtoworlds, ndc_poses=ndc_poses, pix_x=pix_x, pix_y=pix_y,
             cam_idx=cam_idx, pixtocam_ndc=pixtocam_ndc,
             dist_keys=np.array(list(dist.keys())), dist_vals=np.array(list(dist.values())))
  cases = {
      'persp': dict(poses=camtoworlds, dist=None, ndc=None, camtype=camera_utils.ProjectionType.PERSPECTIVE),
      'dist': dict(poses=camtoworlds, dist=dist, ndc=None, camtype=camera_utils.ProjectionType.PERSPECTIVE),
      'fisheye': dict(poses=camtoworlds, dist=dist, ndc=None, camtype=camera_utils.ProjectionType.FISHEYE),
      'ndc': dict(poses=ndc_poses, dist=None, ndc=pixtocam_ndc, camtype=camera_utils.ProjectionType.PERSPECTIVE),
      'single': dict(poses=camtoworlds[0], dist=None, ndc=None, camtype=camera_utils.ProjectionType.PERSPECTIVE,
                     p2c=pixtocams[0]),
  }
  meta = lambda v: np.full((B, 1), v, F)
  for name, c in cases.items():
    p2c = c.get('p2c', pixtocams)
    for tag, xnp, dt in [('f64', np, np.float64), ('f32', jnp, np.float32)]:
      cams = (p2c.astype(dt), c['poses'].astype(dt), c['dist'],
              None if c['ndc'] is None else c['ndc'].astype(dt))
      pixels = utils.Pixels(pix_x_int=pix_x, pix_y_int=pix_y, lossmult=meta(1), near=meta(0.2), far=meta(1e6),
                            cam_idx=cam_idx)
      rays = camera_utils.cast_ray_batch(cams, pixels, c['camtype'], xnp=xnp)
      for f in ['origins', 'directions', 'viewdirs', 'radii', 'imageplane']:
        out[f'{name}_{tag}_{f}'] = np.asarray(getattr(rays, f))
  # convert_to_ndc on its own (tests/camera_utils_test.py:27-69 inputs, numpy instead of jax.random)
  o = np.array([0., 0., 1.]) + rng.uniform(-1, 1, (100, 3))
  d = np.array([0., 0., -1.]) + rng.uniform(-.5, .5, (100, 3))
  on, dn = camera_utils.convert_to_ndc(o, d, pixtocam_ndc, 1.0)
  out.update(ndc_in_o=o, ndc_in_d=d, ndc_out_o=on, ndc_out_d=dn)
  extra_cases(rng, out)
  path = os.path.join(HERE, 'camera.npz')
  np.savez_compressed(path, **out)
  print('camera.npz', len(out), 'arrays')


if __name__ == '__main__':
  main()
