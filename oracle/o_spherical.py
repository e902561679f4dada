"""Oracle (test infrastructure): equirectangular panorama rays, torch-CPU float64.

Follows /root/reference/internal/camera_utils.py cast_spherical_rays :716-763, which the reference's
Dataset runs with `xnp=np` (float64) for `render_camtype = 'pano'` (internal/datasets.py:486-492).
Pinned by tests/golden/spherical.npz (tests/golden/make_golden_spherical.py runs the reference's own
camera_utils.py).
"""
import math

import torch


def _np_linspace(stop, num):
  """numpy's linspace(0, stop, num) rounding: node k = k * (stop / (num - 1)), the last node exactly `stop`
  (torch.linspace rounds its upper half differently)."""
  t = torch.arange(num, dtype=torch.float64) * (stop / (num - 1))
  t[-1] = stop
  return t


def cast_spherical_rays(camtoworld, height, width, near, far):
  """`camtoworld` [3|4, 4]; returns a dict of the ray fields with shapes [height, width, n]."""
  c2w = torch.as_tensor(camtoworld).to(torch.float64)
  theta, phi = torch.meshgrid(_np_linspace(2 * math.pi, width + 1), _np_linspace(math.pi, height + 1),
                              indexing='xy')
  directions = torch.stack([-torch.sin(phi) * torch.sin(theta), torch.cos(phi),
                            torch.sin(phi) * torch.cos(theta)], dim=-1)
  directions = (c2w[:3, :3] @ directions[..., None])[..., 0]
  dy = torch.diff(directions[:, :-1], dim=0)
  dx = torch.diff(directions[:-1, :], dim=1)
  directions = directions[:-1, :-1]
  radii = (0.5 * (torch.linalg.norm(dx, dim=-1) + torch.linalg.norm(dy, dim=-1)))[..., None] * 2 / math.sqrt(12)
  one = torch.ones(radii.shape, dtype=torch.float64)
  return dict(origins=c2w[:3, -1].expand(directions.shape), directions=directions, viewdirs=directions,
              radii=radii, imageplane=torch.zeros(directions.shape[:-1] + (2,), dtype=torch.float64),
              lossmult=one, near=one * near, far=one * far, cam_idx=torch.zeros(radii.shape, dtype=torch.int64))
