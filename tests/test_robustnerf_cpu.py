"""RobustNeRF on the CPU: the oracle's mask, stats and next threshold against the reference's own
robustnerf.py (tests/golden/robustnerf.npz), the config checks of the CUDA path, and its ABI symbols."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import o_robust
from util import golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = golden('robustnerf')
CASES = [str(c) for c in G['cases']]


def case_config(name):
  kw = {k.split('/')[-1]: G[k].item() for k in G.files if k.startswith(f'{name}/cfg/')}
  kw.update(data_loss_type='robustnerf', disable_multiscale_loss=False, data_coarse_loss_mult=0.1,
            data_loss_mult=1.0)
  return types.SimpleNamespace(**kw)


def bits(x):
  return np.asarray(x, np.float32).view(np.uint32)


@pytest.mark.parametrize('name', CASES)
def test_oracle_mask_matches_reference_exactly(name):
  cfg = case_config(name)
  rgb, target = torch.as_tensor(G[f'{name}/rgb']), torch.as_tensor(G[f'{name}/target'])
  mask, stats = o_robust.robustnerf_mask((rgb - target) ** 2, torch.as_tensor(G[f'{name}/threshold']), cfg)
  np.testing.assert_array_equal(mask.numpy(), G[f'{name}/mask'])
  ref_stats = {k.split('/')[-1] for k in G.files if k.startswith(f'{name}/stat/')}
  assert set(stats) == ref_stats
  for k in ref_stats:      # bit for bit, the threshold (quantile) included
    np.testing.assert_array_equal(bits(stats[k]), bits(G[f'{name}/stat/{k}']), err_msg=k)


@pytest.mark.parametrize('name', CASES)
def test_oracle_data_loss_matches_reference(name):
  cfg = case_config(name)
  rgb, target = torch.as_tensor(G[f'{name}/rgb']), torch.as_tensor(G[f'{name}/target'])
  p = cfg.patch_size
  rends = [{'rgb': (rgb + 0.01).reshape(-1, 3)}, {'rgb': rgb.reshape(-1, 3)}]
  loss, stats = o_robust.compute_data_loss(target.reshape(-1, 3), rends, torch.ones(rgb.numel() // 3, 1), cfg,
                                           loss_threshold=torch.as_tensor(G[f'{name}/threshold']))
  np.testing.assert_allclose(float(loss), float(G[f'{name}/loss_data']), rtol=2e-6)
  np.testing.assert_allclose(stats['mses'].numpy(), G[f'{name}/mses'], rtol=2e-6)
  for k in (k.split('/')[-1] for k in G.files if k.startswith(f'{name}/dstat/')):
    np.testing.assert_array_equal(bits(stats[k]), bits(G[f'{name}/dstat/{k}']), err_msg=k)
  assert rgb.shape[1] == p


def test_golden_cases_are_not_degenerate():
  for name in CASES:
    m = float(G[f'{name}/mask'].mean())
    assert (0.1 < m < 0.95) or name == 'disabled', (name, m)
  # the tie case really has errors equal to the threshold, the boundary case patches at exactly half inliers
  e = G['ties/error_per_pixel']
  assert (e == G['ties/threshold']).sum() >= 4
  assert float(G['patch_boundary/stat/is_inlier_loss']) > 0


def test_oracle_quantile_restates_jax_linear():
  rng = np.random.default_rng(3)
  for n in (1, 2, 255, 1000):
    x = rng.normal(size=n).astype(np.float32)
    for q in (0.0, 0.5, 0.8, 1.0):
      got = float(o_robust.quantile_linear(torch.as_tensor(x), q))
      xs = np.sort(x)
      qn = np.float32(q) * np.float32(n - 1)
      lo, hi = int(np.floor(qn)), int(np.ceil(qn))
      w = qn - np.float32(lo)
      want = xs[lo] * (np.float32(1) - w) + xs[hi] * w
      assert bits(got) == bits(want), (n, q)
  x = torch.tensor([1.0, float('nan'), 2.0])
  assert np.isnan(float(o_robust.quantile_linear(x, 0.5)))


def test_config_validation_errors():
  from multinerf_b200 import configs, train_utils
  ok = configs.Config(data_loss_type='robustnerf', patch_size=16, enable_robustnerf_loss=True)
  train_utils.check_robust_config(ok, 16384)
  with pytest.raises(ValueError, match='robustnerf_inner_patch_size'):
    train_utils.check_robust_config(configs.Config(data_loss_type='robustnerf', patch_size=4,
                                                   enable_robustnerf_loss=True, robustnerf_inner_patch_size=8,
                                                   robustnerf_smoothed_filter_size=3), 64)
  with pytest.raises(ValueError, match='multiple of patch_size'):
    train_utils.check_robust_config(ok, 16384 + 16)
  with pytest.raises(ValueError, match='1024'):
    train_utils.check_robust_config(configs.Config(data_loss_type='robustnerf', patch_size=33,
                                                   enable_robustnerf_loss=False), 33 * 33)
  with pytest.raises(ValueError, match='odd'):
    train_utils.check_robust_config(configs.Config(data_loss_type='robustnerf', patch_size=16,
                                                   enable_robustnerf_loss=True,
                                                   robustnerf_smoothed_filter_size=4), 256)
  # the flag off: only the patch-size limit applies (the mask is all ones)
  train_utils.check_robust_config(configs.Config(data_loss_type='robustnerf', patch_size=4,
                                                 enable_robustnerf_loss=False, robustnerf_inner_patch_size=8), 17)


def test_robust_abi_v2_symbols_exported():
  from multinerf_b200 import lib
  if not os.path.exists(lib.LIB_PATH):
    from multinerf_b200 import build
    build.build()
  l = lib.load()
  assert l.mnrf_abi_version() == 2
  for name in ('mnrf_robust_mask', 'mnrf_quantile', 'mnrf_composite_bwd'):
    assert name in lib.EXPORTED and hasattr(l, name)
  import ctypes
  import subprocess
  import tempfile
  src = ('#include <stdio.h>\n#include "mnrf.h"\n'
         'int main(){printf("%zu\\n", sizeof(mnrf_robust_desc)); return 0;}')
  with tempfile.TemporaryDirectory() as td:
    open(os.path.join(td, 'a.c'), 'w').write(src)
    subprocess.run(['gcc', '-I', os.path.join(ROOT, 'include'), os.path.join(td, 'a.c'), '-o',
                    os.path.join(td, 'a')], check=True)
    size = int(subprocess.run([os.path.join(td, 'a')], capture_output=True, text=True).stdout)
  assert size == ctypes.sizeof(lib.RobustDesc)


def test_synthetic_scene_patches_are_whole_and_patch_major():
  from multinerf_b200 import configs, train_loop
  sc = train_loop.SyntheticScene.__new__(train_loop.SyntheticScene)
  sc.config = configs.Config(patch_size=16, batch_size=1024)
  sc.width, sc.height, sc.size, sc.batch = 96, 72, 24, 1024
  sc.rng = np.random.default_rng(0)
  px = sc.pixels()
  x = px.pix_x_int.reshape(4, 16, 16)
  y = px.pix_y_int.reshape(4, 16, 16)
  cam = px.cam_idx.reshape(4, 16, 16)
  assert (x - x[:, :1, :1] == np.arange(16)[None, None, :]).all()
  assert (y - y[:, :1, :1] == np.arange(16)[None, :, None]).all()
  assert (cam == cam[:, :1, :1]).all()
  assert x.max() < 96 and y.max() < 72 and x.min() >= 0 and y.min() >= 0


def test_synthetic_scene_single_pixel_draws_unchanged():
  """patch_size 1 keeps the per-pixel draws of the scene (x, y, camera from one generator, in that order)."""
  from multinerf_b200 import configs, train_loop
  sc = train_loop.SyntheticScene.__new__(train_loop.SyntheticScene)
  sc.config = configs.Config(batch_size=512)
  sc.width, sc.height, sc.size, sc.batch = 96, 72, 24, 512
  sc.rng = np.random.default_rng(7)
  px = sc.pixels()
  rng = np.random.default_rng(7)
  np.testing.assert_array_equal(px.pix_x_int, rng.integers(0, 96, 512).astype(np.int32))
  np.testing.assert_array_equal(px.pix_y_int, rng.integers(0, 72, 512).astype(np.int32))
  np.testing.assert_array_equal(px.cam_idx, rng.integers(0, 24, (512, 1)).astype(np.int32))
