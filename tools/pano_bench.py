"""Panorama rendering (`render_camtype = 'pano'`) on one GPU: the card name and power limit; the time of the
`mnrf_spherical_rays` kernel at 2048 x 4096 (CUDA events over --launches launches after a warm-up); and, with
the full-width 360.gin model (seeded init), one 1024 x 2048 panorama frame (ray casting plus `render_image`)
against one 1560 x 1040 perspective frame of the same model, for rays/s.  Frame times are the median of
--frames frames after one warm-up frame of each, timed with a device synchronise.  Prints one JSON line.

    python tools/pano_bench.py [--launches 200] [--frames 3]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from multinerf_b200 import camera_utils, configs, lib, models, train_utils, utils  # noqa: E402


def smi(query):
  try:
    out = subprocess.run(['nvidia-smi', f'--query-gpu={query}', '--format=csv,noheader,nounits', '-i',
                          str(torch.cuda.current_device())], capture_output=True, text=True, timeout=10)
    return out.stdout.strip()
  except Exception:  # pylint: disable=broad-except
    return ''


def kernel_us(pose, h, w, launches):
  l = lib.require_device()
  d = lib.SphericalDesc(h, w, (ctypes.c_double * 12)(*pose.reshape(-1)))
  out = [torch.empty(h * w, n, device='cuda') for n in (3, 3, 3, 1, 2)]
  call = lambda: lib.check(l.mnrf_spherical_rays(ctypes.byref(d), *[lib.ptr(t) for t in out], lib.stream_ptr()))
  for _ in range(10):
    call()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(launches):
    call()
  b.record()
  torch.cuda.synchronize()
  return a.elapsed_time(b) * 1e3 / launches


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--launches', type=int, default=200)
  ap.add_argument('--frames', type=int, default=3)
  args = ap.parse_args()
  lib.require_device()
  pose = np.eye(4)[:3]
  pose[:, 3] = [0.05, -0.02, 0.01]
  kh, kw = 2048, 4096
  k_us = kernel_us(pose, kh, kw, args.launches)

  bundle = configs.bundle_360()
  model, state, _, _, _ = train_utils.setup_model(bundle, 20200823)
  pfn = train_utils.create_render_fn(model, use_graph=True)          # as render.py renders
  render_fn = lambda rng, r: pfn(state.params, 1.0, None, r)
  near, far = bundle.config.near, bundle.config.far
  W, H = 1560, 1040
  pixtocam = camera_utils.get_pixtocam(1200.0, W, H)
  xs, ys = camera_utils.pixel_coordinates(W, H)

  def pano():
    return models.render_image(render_fn, camera_utils.cast_spherical_rays(pose, 1024, 2048, near, far), None,
                               bundle, verbose=False)

  def persp():
    o, d, v, r, ip = camera_utils.pixels_to_rays(xs, ys, pixtocam, pose)
    full = lambda x, dt=torch.float32: torch.full((H, W, 1), x, device='cuda', dtype=dt)
    rays = utils.Rays(o, d, v, r, ip, lossmult=full(1.), near=full(near), far=full(far),
                      cam_idx=full(0, torch.int32))
    return models.render_image(render_fn, rays, None, bundle, verbose=False)

  times = {'pano': [], 'persp': []}
  for name, fn in (('pano', pano), ('persp', persp)):
    fn()                                   # warm-up: allocations, graph capture per chunk shape
    torch.cuda.synchronize()
  for _ in range(args.frames):
    for name, fn in (('pano', pano), ('persp', persp)):
      t0 = time.perf_counter()
      out = fn()
      torch.cuda.synchronize()
      times[name].append(time.perf_counter() - t0)
      assert bool(torch.isfinite(out['rgb']).all()), name
  med = {k: float(np.median(v)) for k, v in times.items()}
  print(json.dumps({
      'card': torch.cuda.get_device_name(), 'power_limit_w': smi('power.limit'),
      'kernel_2048x4096_us': k_us, 'kernel_launches': args.launches,
      'kernel_write_GBps': kh * kw * 48 / (k_us * 1e-6) / 1e9,
      'pano_1024x2048_s': med['pano'], 'pano_rays_per_s': 1024 * 2048 / med['pano'],
      'persp_1560x1040_s': med['persp'], 'persp_rays_per_s': W * H / med['persp'],
      'frames_s': {k: [round(x, 4) for x in v] for k, v in times.items()}}))


if __name__ == '__main__':
  main()
