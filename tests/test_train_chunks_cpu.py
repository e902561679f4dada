"""Train steps in several forward/backward passes (Config.train_chunk_size) on the CPU: the gin binding and its
default, the configuration errors, and the two ABI entry points that take the batch's ray count."""
import ctypes
import os
import re
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_default_and_gin_binding():
  from multinerf_b200 import configs
  assert configs.Config().train_chunk_size == 0
  assert configs.bundle_blender_refnerf().config.train_chunk_size == 0
  b = configs.parse_gin(configs.GIN_BLENDER_REFNERF + '\nConfig.train_chunk_size = 4096\n')
  assert b.config.train_chunk_size == 4096 and b.config.batch_size == 16384


def _cfg(**kw):
  from multinerf_b200 import configs
  return configs.Config(**kw)


def test_accepted_chunk_sizes():
  from multinerf_b200 import train_utils
  for c in (0, 16384, 8192, 4096, 1):
    train_utils.check_chunk_config(_cfg(train_chunk_size=c), 16384)
  # a robustnerf step whose mask is off groups nothing into patches
  train_utils.check_chunk_config(_cfg(train_chunk_size=8, data_loss_type='robustnerf', patch_size=16,
                                      enable_robustnerf_loss=False), 1024)
  train_utils.check_chunk_config(_cfg(train_chunk_size=512, data_loss_type='robustnerf', patch_size=16,
                                      enable_robustnerf_loss=True), 1024)


@pytest.mark.parametrize('chunk,rays,kw,match', [
    (3000, 16384, {}, 'does not divide'),
    (32768, 16384, {}, 'does not divide'),
    (-1, 16384, {}, '>= 0'),
    (128, 1024, dict(data_loss_type='robustnerf', patch_size=16, enable_robustnerf_loss=True), 'patch_size'),
])
def test_errors_name_the_field(chunk, rays, kw, match):
  from multinerf_b200 import train_utils
  with pytest.raises(ValueError, match='train_chunk_size') as e:
    train_utils.check_chunk_config(_cfg(train_chunk_size=chunk, **kw), rays)
  assert re.search(match, str(e.value)), str(e.value)


def _sizeof(types):
  src = '#include <stdio.h>\n#include "mnrf.h"\nint main(){' + ''.join(
      f'printf("%zu\\n", sizeof({t}));' for t in types) + 'return 0;}'
  with tempfile.TemporaryDirectory() as td:
    open(os.path.join(td, 'a.c'), 'w').write(src)
    subprocess.run(['gcc', '-I', os.path.join(ROOT, 'include'), os.path.join(td, 'a.c'), '-o',
                    os.path.join(td, 'a')], check=True)
    out = subprocess.run([os.path.join(td, 'a')], capture_output=True, text=True, check=True).stdout
  return [int(x) for x in out.split()]


def test_batch_rays_declared_on_the_base_entry_points():
  from multinerf_b200 import lib
  header = open(os.path.join(ROOT, 'include', 'mnrf.h')).read()
  for name in ('mnrf_composite_bwd', 'mnrf_robust_mask'):
    decl = re.search(r'\b' + name + r'\(([^;]*)\);', header)
    assert decl and 'int32_t batch_rays' in decl.group(1), name
    assert name in lib.EXPORTED
  assert 'const float* data_mask' in re.search(r'\bmnrf_composite_bwd\(([^;]*)\);', header).group(1)
  if not os.path.exists(lib.LIB_PATH):
    from multinerf_b200 import build
    build.build()
  l = lib.load()
  for name in ('mnrf_composite_bwd_chunk', 'mnrf_composite_bwd_masked', 'mnrf_robust_mask_chunk'):
    assert name not in header and name not in lib.EXPORTED and not hasattr(l, name)


def test_existing_descriptors_unchanged():
  from multinerf_b200 import lib
  sizes = _sizeof(['mnrf_composite_desc', 'mnrf_loss_desc', 'mnrf_robust_desc'])
  assert sizes == [ctypes.sizeof(lib.CompositeDesc), ctypes.sizeof(lib.LossDesc), ctypes.sizeof(lib.RobustDesc)]
  assert sizes == [56, 84, 28]
