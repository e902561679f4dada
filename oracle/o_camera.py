"""Oracle (test infrastructure): pixel -> ray generation, torch-CPU.

Follows /root/reference/internal/camera_utils.py:
  convert_to_ndc :32-97   intrinsic_matrix :398-408   get_pixtocam :411-417
  pixel_coordinates :420-424   _compute_residual_and_jacobian :427-475
  _radial_and_tangential_undistort :478-513   pixels_to_rays :522-636
  cast_ray_batch :639-688
Computation dtype follows the inputs (float32 = the `xnp=jnp` path the reference runs inside
the train step, camera_utils.py:266-268 of train_utils; float64 = the `xnp=np` dataset path).
Pinned by tests/golden/camera.npz (tests/golden/make_golden_camera.py runs the reference's own
camera_utils.py) and by the reference's tests/camera_utils_test.py known-answer check.
"""
import math

import torch

PERSPECTIVE = 'perspective'
FISHEYE = 'fisheye'


def convert_to_ndc(origins, directions, pixtocam, near=1.0):
  t = -(near + origins[..., 2]) / directions[..., 2]
  origins = origins + t[..., None] * directions
  dx, dy, dz = directions.unbind(-1)
  ox, oy, oz = origins.unbind(-1)
  xmult = 1.0 / pixtocam[0, 2]
  ymult = 1.0 / pixtocam[1, 2]
  origins_ndc = torch.stack([xmult * ox / oz, ymult * oy / oz, -torch.ones_like(oz)], dim=-1)
  infinity_ndc = torch.stack([xmult * dx / dz, ymult * dy / dz, torch.ones_like(oz)], dim=-1)
  return origins_ndc, infinity_ndc - origins_ndc


def intrinsic_matrix(fx, fy, cx, cy, dtype=torch.float64):
  return torch.tensor([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]], dtype=dtype)


def get_pixtocam(focal, width, height, dtype=torch.float64):
  return torch.linalg.inv(intrinsic_matrix(focal, focal, width * 0.5, height * 0.5, dtype))


def pixel_coordinates(width, height):
  return torch.meshgrid(torch.arange(width), torch.arange(height), indexing='xy')


def _residual_and_jacobian(x, y, xd, yd, k1=0.0, k2=0.0, k3=0.0, k4=0.0, p1=0.0, p2=0.0):
  r = x * x + y * y
  d = 1.0 + r * (k1 + r * (k2 + r * (k3 + r * k4)))
  fx = d * x + 2 * p1 * x * y + p2 * (r + 2 * x * x) - xd
  fy = d * y + 2 * p2 * x * y + p1 * (r + 2 * y * y) - yd
  d_r = k1 + r * (2.0 * k2 + r * (3.0 * k3 + r * 4.0 * k4))
  d_x = 2.0 * x * d_r
  d_y = 2.0 * y * d_r
  fx_x = d + d_x * x + 2.0 * p1 * y + 6.0 * p2 * x
  fx_y = d_y * x + 2.0 * p1 * x + 2.0 * p2 * y
  fy_x = d_x * y + 2.0 * p2 * y + 2.0 * p1 * x
  fy_y = d + d_y * y + 2.0 * p2 * x + 6.0 * p1 * y
  return fx, fy, fx_x, fx_y, fy_x, fy_y


def radial_and_tangential_undistort(xd, yd, k1=0.0, k2=0.0, k3=0.0, k4=0.0, p1=0.0, p2=0.0,
                                    eps=1e-9, max_iterations=10):
  x, y = xd.clone(), yd.clone()
  for _ in range(max_iterations):
    fx, fy, fx_x, fx_y, fy_x, fy_y = _residual_and_jacobian(x, y, xd, yd, k1, k2, k3, k4, p1, p2)
    denominator = fy_x * fx_y - fx_x * fy_y
    x_numerator = fx * fy_y - fy * fx_y
    y_numerator = fy * fx_x - fx * fy_x
    ok = denominator.abs() > eps
    zero = torch.zeros_like(denominator)
    x = x + torch.where(ok, x_numerator / denominator, zero)
    y = y + torch.where(ok, y_numerator / denominator, zero)
  return x, y


def pixels_to_rays(pix_x_int, pix_y_int, pixtocams, camtoworlds, distortion_params=None,
                   pixtocam_ndc=None, camtype=PERSPECTIVE):
  """Returns (origins, directions, viewdirs, radii, imageplane); dtype of `pixtocams`."""
  dtype = pixtocams.dtype
  x0, y0 = pix_x_int.to(dtype), pix_y_int.to(dtype)

  def pix_to_dir(x, y):
    return torch.stack([x + 0.5, y + 0.5, torch.ones_like(x)], dim=-1)

  pixel_dirs = torch.stack([pix_to_dir(x0, y0), pix_to_dir(x0 + 1, y0), pix_to_dir(x0, y0 + 1)], dim=0)
  mat_vec = lambda a, b: (a @ b[..., None])[..., 0]
  cam_dirs = mat_vec(pixtocams, pixel_dirs)
  if distortion_params is not None:
    x, y = radial_and_tangential_undistort(cam_dirs[..., 0], cam_dirs[..., 1], **distortion_params)
    cam_dirs = torch.stack([x, y, torch.ones_like(x)], dim=-1)
  if camtype == FISHEYE:
    theta = torch.sqrt((cam_dirs[..., :2] ** 2).sum(dim=-1))
    theta = torch.clamp(theta, max=math.pi)
    # the reference divides 0 by 0 on the optical axis (NaN rays); take sin(theta) / theta at its limit 1 there
    s = torch.where(theta > 0, torch.sin(theta) / theta, torch.ones_like(theta))
    cam_dirs = torch.stack([cam_dirs[..., 0] * s, cam_dirs[..., 1] * s, torch.cos(theta)], dim=-1)
  cam_dirs = cam_dirs * torch.tensor([1.0, -1.0, -1.0], dtype=dtype)     # OpenCV -> OpenGL
  imageplane = cam_dirs[0, ..., :2]
  dirs_stacked = mat_vec(camtoworlds[..., :3, :3], cam_dirs)
  directions, dx, dy = dirs_stacked[0], dirs_stacked[1], dirs_stacked[2]
  origins = camtoworlds[..., :3, -1].expand(directions.shape)
  viewdirs = directions / torch.linalg.norm(directions, dim=-1, keepdim=True)
  if pixtocam_ndc is None:
    dx_norm = torch.linalg.norm(dx - directions, dim=-1)
    dy_norm = torch.linalg.norm(dy - directions, dim=-1)
  else:
    origins_dx, _ = convert_to_ndc(origins, dx, pixtocam_ndc)
    origins_dy, _ = convert_to_ndc(origins, dy, pixtocam_ndc)
    origins, directions = convert_to_ndc(origins, directions, pixtocam_ndc)
    dx_norm = torch.linalg.norm(origins_dx - origins, dim=-1)
    dy_norm = torch.linalg.norm(origins_dy - origins, dim=-1)
  radii = (0.5 * (dx_norm + dy_norm))[..., None] * 2 / math.sqrt(12)
  return origins, directions, viewdirs, radii, imageplane


def cast_ray_batch(cameras, pixels, camtype=PERSPECTIVE):
  """`pixels`: object with pix_x_int, pix_y_int [SH], cam_idx [SH, 1] (+ metadata); returns a dict
  of the ray fields computed here (metadata passes through unchanged in the reference)."""
  pixtocams, camtoworlds, distortion_params, pixtocam_ndc = cameras
  cam_idx = pixels.cam_idx[..., 0].long()
  batch_index = lambda arr: arr if arr.ndim == 2 else arr[cam_idx]
  # pix_x_int / pix_y_int have shape SH; cam_idx (and the other metadata) SH + [1]
  # (internal/datasets.py:410-431)
  o, d, v, r, ip = pixels_to_rays(pixels.pix_x_int, pixels.pix_y_int,
                                  batch_index(pixtocams), batch_index(camtoworlds),
                                  distortion_params=distortion_params, pixtocam_ndc=pixtocam_ndc,
                                  camtype=camtype)
  return dict(origins=o, directions=d, viewdirs=v, radii=r, imageplane=ip)
