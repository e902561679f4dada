"""Pixel -> ray generation on the device (reference surface: internal/camera_utils.py).

`cast_ray_batch(cameras, pixels, camtype)` and `pixels_to_rays(...)` keep the reference's names,
argument meaning and return order (camera_utils.py:522-688); the work is one launch of
`mnrf_pixels_to_rays` (csrc/camera.cu).  `cast_spherical_rays(...)` (camera_utils.py:716-763) is one
launch of `mnrf_spherical_rays`.  The small host helpers (`intrinsic_matrix`,
`get_pixtocam`, `pixel_coordinates`) are the reference's one-liners in numpy.
"""
import enum

import numpy as np
import torch

from . import lib as L
from . import utils


class ProjectionType(enum.Enum):
  """camera_utils.py:516-519."""
  PERSPECTIVE = 'perspective'
  FISHEYE = 'fisheye'


def intrinsic_matrix(fx, fy, cx, cy):
  """camera_utils.py:398-408."""
  return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.]])


def get_pixtocam(focal, width, height):
  """camera_utils.py:411-417."""
  return np.linalg.inv(intrinsic_matrix(focal, focal, width * .5, height * .5))


def pixel_coordinates(width, height):
  """camera_utils.py:420-424."""
  return np.meshgrid(np.arange(width), np.arange(height), indexing='xy')


def _dev(x, dtype, device):
  t = x if isinstance(x, torch.Tensor) else torch.tensor(np.asarray(x))
  return t.to(device=device, dtype=dtype, non_blocking=True).contiguous()


_checked = False


def _load():
  global _checked
  if not _checked:
    L.require_device()          # queries device properties: once, not per launch
    _checked = True
  return L.load()


def _launch(pix_x, pix_y, cam_idx, pixtocams, camtoworlds, distortion_params, pixtocam_ndc, camtype):
  """All inputs flat on the device; returns the five [B, n] fp32 outputs."""
  lib = _load()
  B = pix_x.shape[0]
  dev = pix_x.device
  if isinstance(camtype, str):
    camtype = ProjectionType(camtype)
  if camtype not in (ProjectionType.PERSPECTIVE, ProjectionType.FISHEYE):
    raise ValueError(f'unknown camtype {camtype!r}')
  dp = dict(distortion_params or {})
  unknown = set(dp) - {'k1', 'k2', 'k3', 'k4', 'p1', 'p2'}
  if unknown:
    raise TypeError(f'unexpected distortion parameters {sorted(unknown)}')   # as **distortion_params would
  ndc = None if pixtocam_ndc is None else np.asarray(
      pixtocam_ndc.detach().cpu() if isinstance(pixtocam_ndc, torch.Tensor) else pixtocam_ndc, np.float64)
  d = L.CameraDesc(B, pixtocams.shape[0], 0 if camtype == ProjectionType.PERSPECTIVE else 1,
                   int(distortion_params is not None),
                   float(dp.get('k1', 0.0)), float(dp.get('k2', 0.0)), float(dp.get('k3', 0.0)),
                   float(dp.get('k4', 0.0)), float(dp.get('p1', 0.0)), float(dp.get('p2', 0.0)),
                   1e-9, 10, int(ndc is not None),
                   float(ndc[0, 2]) if ndc is not None else 1.0, float(ndc[1, 2]) if ndc is not None else 1.0,
                   1.0)
  out = [torch.empty(B, n, device=dev, dtype=torch.float32) for n in (3, 3, 3, 1, 2)]
  from . import ops
  ops._count()
  L.check(lib.mnrf_pixels_to_rays(L.C.byref(d), L.ptr(pix_x), L.ptr(pix_y), L.ptr(cam_idx), L.ptr(pixtocams),
                                  L.ptr(camtoworlds), *[L.ptr(t) for t in out], L.stream_ptr()))
  return out


def pixels_to_rays(pix_x_int, pix_y_int, pixtocams, camtoworlds, distortion_params=None,
                   pixtocam_ndc=None, camtype=ProjectionType.PERSPECTIVE, device='cuda'):
  """camera_utils.py:522-636.  `pixtocams` / `camtoworlds` are one matrix ([3,3] / [3,4]) or one per
  pixel (SH + [3,3] / SH + [3,4]); returns (origins, directions, viewdirs, radii, imageplane) with
  shapes SH + [3|3|3|1|2] as CUDA fp32 tensors."""
  px = _dev(pix_x_int, torch.int32, device)
  sh = tuple(px.shape)
  px = px.reshape(-1)
  py = _dev(pix_y_int, torch.int32, device).reshape(-1)
  p2c = _dev(pixtocams, torch.float32, device)
  c2w = _dev(camtoworlds, torch.float32, device)
  B = px.shape[0]
  if p2c.ndim == 2 and c2w.ndim == 2:
    p2c, c2w, idx = p2c[None], c2w[None, :3, :4].contiguous(), None
  else:
    p2c = p2c.expand(sh + (3, 3)).reshape(B, 3, 3).contiguous()
    c2w = c2w[..., :3, :4].expand(sh + (3, 4)).reshape(B, 3, 4).contiguous()
    idx = torch.arange(B, device=px.device, dtype=torch.int32)
  outs = _launch(px, py, idx, p2c, c2w, distortion_params, pixtocam_ndc, camtype)
  return tuple(o.reshape(sh + (o.shape[-1],)) for o in outs)


def cast_ray_batch(cameras, pixels, camtype=ProjectionType.PERSPECTIVE, device='cuda'):
  """camera_utils.py:639-688: cameras = (pixtocams, camtoworlds, distortion_params, pixtocam_ndc) with
  1 or N stacked matrices; pixels = utils.Pixels.  The per-ray camera gather happens in the kernel."""
  pixtocams, camtoworlds, distortion_params, pixtocam_ndc = cameras
  px = _dev(pixels.pix_x_int, torch.int32, device)
  sh = tuple(px.shape)
  px = px.reshape(-1)
  py = _dev(pixels.pix_y_int, torch.int32, device).reshape(-1)
  idx = _dev(pixels.cam_idx, torch.int32, device).reshape(-1)
  p2c = _dev(pixtocams, torch.float32, device)
  c2w = _dev(camtoworlds, torch.float32, device)
  p2c = p2c[None] if p2c.ndim == 2 else p2c.reshape(-1, 3, 3)
  c2w = (c2w[None] if c2w.ndim == 2 else c2w.reshape((-1,) + tuple(c2w.shape[-2:])))[:, :3, :4].contiguous()
  n_cam = max(p2c.shape[0], c2w.shape[0])
  if p2c.shape[0] != n_cam:
    p2c = p2c.expand(n_cam, 3, 3).contiguous()
  if c2w.shape[0] != n_cam:
    c2w = c2w.expand(n_cam, 3, 4).contiguous()
  o, d, v, r, ip = _launch(px, py, idx if n_cam > 1 else None, p2c, c2w, distortion_params, pixtocam_ndc, camtype)
  rs = lambda t: t.reshape(sh + (t.shape[-1],))
  return utils.Rays(origins=rs(o), directions=rs(d), viewdirs=rs(v), radii=rs(r), imageplane=rs(ip),
                    lossmult=pixels.lossmult, near=pixels.near, far=pixels.far, cam_idx=pixels.cam_idx,
                    exposure_idx=pixels.exposure_idx, exposure_values=pixels.exposure_values)


def cast_spherical_rays(camtoworld, height, width, near, far, device='cuda'):
  """camera_utils.py:716-763: an equirectangular 360-degree panorama from the pose `camtoworld` ([3, 4] or
  [4, 4], numpy or torch).  Returns utils.Rays of [height, width, n] CUDA tensors: fp32 fields and int32
  `cam_idx` (0); `imageplane` is 0, `lossmult` 1, no exposure fields.  The rays are computed in float64 from
  the pose as given, like the reference's `xnp=np` path, and rounded to fp32 once."""
  height, width = int(height), int(width)
  if height < 1 or width < 1:
    raise ValueError(f'panorama size must be at least 1 x 1, got {height} x {width}')
  c2w = np.asarray(camtoworld.detach().cpu() if isinstance(camtoworld, torch.Tensor) else camtoworld, np.float64)
  if c2w.shape not in ((3, 4), (4, 4)):
    raise ValueError(f'camtoworld must be [3, 4] or [4, 4], got {list(c2w.shape)}')
  lib = _load()
  d = L.SphericalDesc(height, width, (L.C.c_double * 12)(*c2w[:3, :4].reshape(-1)))
  out = [torch.empty(height, width, n, device=device, dtype=torch.float32) for n in (3, 3, 3, 1, 2)]
  from . import ops
  ops._count()
  L.check(lib.mnrf_spherical_rays(L.C.byref(d), *[L.ptr(t) for t in out], L.stream_ptr()))
  full = lambda v, dtype: torch.full((height, width, 1), v, device=device, dtype=dtype)
  return utils.Rays(*out, lossmult=full(1., torch.float32), near=full(near, torch.float32),
                    far=full(far, torch.float32), cam_idx=full(0, torch.int32))


# ------------------------------------------------------------------------------------------------
# Host-side pose algebra around the path (camera_utils.py:101-395): dataset normalisation and render
# paths.  Plain numpy on [N, 3, 4] camera-to-world matrices; nothing here touches the device.
# ------------------------------------------------------------------------------------------------
NEAR_STRETCH = .9     # camera_utils.py:148-150
FAR_STRETCH = 5.
FOCUS_DISTANCE = .75


def pad_poses(p):
  """[..., 3, 4] -> [..., 4, 4] with the homogeneous row (camera_utils.py:101-104)."""
  p = np.asarray(p)
  row = np.zeros(p.shape[:-2] + (1, 4), p.dtype)
  row[..., 0, 3] = 1
  return np.concatenate([p[..., :3, :4], row], axis=-2)


def unpad_poses(p):
  return p[..., :3, :4]


def normalize(x):
  return x / np.linalg.norm(x)


def viewmatrix(lookdir, up, position):
  """Look-at frame: columns (right, up', back, position) (camera_utils.py:126-133)."""
  z = normalize(lookdir)
  x = normalize(np.cross(up, z))
  y = normalize(np.cross(z, x))
  return np.stack([x, y, z, position], axis=1)


def average_pose(poses):
  """camera_utils.py:117-123."""
  return viewmatrix(poses[:, :3, 2].mean(0), poses[:, :3, 1].mean(0), poses[:, :3, 3].mean(0))


def recenter_poses(poses):
  """Express the poses in the frame of their average pose; returns (poses, 4x4 transform)."""
  transform = np.linalg.inv(pad_poses(average_pose(poses)))
  return unpad_poses(transform @ pad_poses(poses)), transform


def focus_point_fn(poses):
  """Least-squares point closest to all optical axes (camera_utils.py:141-147)."""
  d, o = poses[:, :3, 2:3], poses[:, :3, 3:4]
  m = np.eye(3) - d * np.transpose(d, [0, 2, 1])
  mtm = np.transpose(m, [0, 2, 1]) @ m
  return np.linalg.inv(mtm.mean(0)) @ (mtm @ o).mean(0)[:, 0]


def generate_spiral_path(poses, bounds, n_frames=120, n_rots=2, zrate=.5):
  """Forward-facing spiral (camera_utils.py:153-184)."""
  near = bounds.min() * NEAR_STRETCH
  far = bounds.max() * FAR_STRETCH
  focal = 1 / ((1 - FOCUS_DISTANCE) / near + FOCUS_DISTANCE / far)
  radii = np.concatenate([np.percentile(np.abs(poses[:, :3, 3]), 90, 0), [1.]])
  c2w = average_pose(poses)
  up = poses[:, :3, 1].mean(0)
  out = []
  for theta in np.linspace(0., 2. * np.pi * n_rots, n_frames, endpoint=False):
    position = c2w @ (radii * [np.cos(theta), -np.sin(theta), -np.sin(theta * zrate), 1.])
    lookat = c2w @ [0, 0, -focal, 1.]
    out.append(viewmatrix(position - lookat, up, position))
  return np.stack(out, axis=0)


def transform_poses_pca(poses):
  """Principal axes of the camera positions onto XYZ, positions scaled into [-1, 1]^3
  (camera_utils.py:187-225).  Returns (poses, 4x4 transform)."""
  t = poses[:, :3, 3]
  mean = t.mean(axis=0)
  t = t - mean
  eigval, eigvec = np.linalg.eig(t.T @ t)
  rot = eigvec[:, np.argsort(eigval)[::-1]].T
  if np.linalg.det(rot) < 0:
    rot = np.diag([1., 1., -1.]) @ rot
  transform = np.concatenate([rot, rot @ -mean[:, None]], -1)
  out = unpad_poses(transform @ pad_poses(poses))
  transform = np.concatenate([transform, np.eye(4)[3:]], axis=0)
  if out.mean(axis=0)[2, 1] < 0:          # keep the average up vector pointing along +z
    out = np.diag([1., -1., -1.]) @ out
    transform = np.diag([1., -1., -1., 1.]) @ transform
  scale = 1. / np.max(np.abs(out[:, :3, 3]))
  out[:, :3, 3] *= scale
  transform = np.diag([scale] * 3 + [1.]) @ transform
  return out, transform


def _resample_deterministic(t, w_logits, num_samples):
  """stepfun.sample(None, t, w_logits, n) on the host (stepfun.py:170-211, rng=None and the default
  deterministic_center=False): inverse CDF of the step function softmax(w_logits) on t at
  u = linspace(0, 1 - eps, n)."""
  eps = np.finfo(np.float32).eps
  w = np.exp(w_logits - np.max(w_logits))
  w = w / w.sum()
  cw = np.concatenate([[0.], np.minimum(1., np.cumsum(w[:-1])), [1.]])
  u = np.linspace(0, 1. - eps, num_samples)
  return np.interp(u, cw, t)


def generate_ellipse_path(poses, n_frames=120, const_speed=True, z_variation=0., z_phase=0.):
  """Inward-facing elliptical path (camera_utils.py:228-281)."""
  center = focus_point_fn(poses)
  offset = np.array([center[0], center[1], 0])
  sc = np.percentile(np.abs(poses[:, :3, 3] - offset), 90, axis=0)
  low, high = -sc + offset, sc + offset
  z_low = np.percentile(poses[:, :3, 3], 10, axis=0)
  z_high = np.percentile(poses[:, :3, 3], 90, axis=0)

  def positions_at(theta):
    return np.stack([low[0] + (high - low)[0] * (np.cos(theta) * .5 + .5),
                     low[1] + (high - low)[1] * (np.sin(theta) * .5 + .5),
                     z_variation * (z_low[2] + (z_high - z_low)[2] *
                                    (np.cos(theta + 2 * np.pi * z_phase) * .5 + .5))], -1)
  theta = np.linspace(0, 2. * np.pi, n_frames + 1, endpoint=True)
  positions = positions_at(theta)
  if const_speed:
    lengths = np.linalg.norm(positions[1:] - positions[:-1], axis=-1)
    theta = _resample_deterministic(theta, np.log(lengths), n_frames + 1)
    positions = positions_at(theta)
  positions = positions[:-1]
  avg_up = normalize(poses[:, :3, 1].mean(0))
  k = int(np.argmax(np.abs(avg_up)))
  up = np.eye(3)[k] * np.sign(avg_up[k])
  return np.stack([viewmatrix(p - center, up, p) for p in positions])


def generate_interpolated_path(poses, n_interp, spline_degree=5, smoothness=.03, rot_weight=.1):
  """B-spline through keyframe poses in (position, look-at point, up point) form
  (camera_utils.py:284-332)."""
  import scipy.interpolate
  pos = poses[:, :3, -1]
  pts = np.stack([pos, pos - rot_weight * poses[:, :3, 2], pos + rot_weight * poses[:, :3, 1]], 1)
  n = n_interp * (pts.shape[0] - 1)
  sh = pts.shape
  k = min(spline_degree, sh[0] - 1)
  tck, _ = scipy.interpolate.splprep(pts.reshape(sh[0], -1).T, k=k, s=smoothness)
  new = np.array(scipy.interpolate.splev(np.linspace(0, 1, n, endpoint=False), tck)).T.reshape(n, sh[1], sh[2])
  return np.array([viewmatrix(p - l, u - p, p) for p, l, u in new])


def interpolate_1d(x, n_interp, spline_degree, smoothness):
  """camera_utils.py:335-345."""
  import scipy.interpolate
  t = np.linspace(0, 1, len(x), endpoint=True)
  tck = scipy.interpolate.splrep(t, x, s=smoothness, k=spline_degree)
  return scipy.interpolate.splev(np.linspace(0, 1, n_interp * (len(x) - 1), endpoint=False), tck)


def create_render_spline_path(config, image_names, poses, exposures):
  """Spline render path through the keyframes named in `config.render_spline_keyframes` (a directory of
  images or a text file of names) (camera_utils.py:348-395)."""
  import os
  if os.path.isdir(config.render_spline_keyframes):
    keyframe_names = sorted(os.listdir(config.render_spline_keyframes))
  else:
    with open(config.render_spline_keyframes, 'r') as fp:
      keyframe_names = fp.read().splitlines()
  spline_indices = np.array([i for i, n in enumerate(image_names) if n in keyframe_names])
  render_poses = generate_interpolated_path(poses[spline_indices], n_interp=config.render_spline_n_interp,
                                            spline_degree=config.render_spline_degree,
                                            smoothness=config.render_spline_smoothness, rot_weight=.1)
  render_exposures = None
  if config.render_spline_interpolate_exposure:
    if exposures is None:
      raise ValueError('config.render_spline_interpolate_exposure is True but '
                       'create_render_spline_path() was passed exposures=None.')
    render_exposures = np.exp(interpolate_1d(np.log(exposures[spline_indices]), config.render_spline_n_interp,
                                             spline_degree=5, smoothness=20))
  return spline_indices, render_poses, render_exposures
