"""The training loop around train_pstep (train.py:66-223) on the procedural scene: the loss goes
down (an end-to-end check that forward, losses, backward and Adam fit together), the summary carries
the reference's fields, and a run resumed from a checkpoint continues like the uninterrupted one.
Needs an H100."""
import copy

import numpy as np
import pytest
import torch

from model_parity import plumbing_blender, train_loop_bundle

pytestmark = pytest.mark.gpu


def test_training_reduces_loss_and_logs_reference_fields():
  from multinerf_b200 import train_loop
  lines = []
  b = train_loop_bundle(160, cast=True)
  model, state, hist = train_loop.train(b, train_loop.SyntheticScene(b.config), log=lines.append)
  assert state.step == 160 and hist[-1]['step'] == 160
  first, last = hist[0], hist[-1]
  assert last['psnr'] > first['psnr'] + 4.0, (first['psnr'], last['psnr'])
  assert last['loss'] < 0.6 * first['loss'], (first['loss'], last['loss'])
  assert all(np.isfinite(h['loss']) for h in hist)
  # 'step/max: loss=..., psnr=..., lr=... | data=..., dist=..., inte=..., N r/s'  (train.py:198-204)
  assert lines[0].startswith('Number of parameters being optimized: ')
  assert 'loss=' in lines[-1] and 'psnr=' in lines[-1] and 'lr=' in lines[-1] and lines[-1].endswith(' r/s')
  for key in ('data=', 'dist=', 'inte='):
    assert key in lines[-1], lines[-1]


def test_checkpoint_resume(tmp_path):
  from multinerf_b200 import checkpoints, train_loop
  ck = str(tmp_path / 'ckpt')
  # uninterrupted: 120 steps
  b = train_loop_bundle(120)
  model_a, state_a, _ = train_loop.train(b, train_loop.SyntheticScene(b.config, seed=3), log=lambda s: None)
  # interrupted at 60 (checkpoint_every), then resumed to 120 with a dataset continuing the same stream
  b1 = train_loop_bundle(120, ckpt=ck)
  b1.config.early_exit_steps = 60
  ds = train_loop.SyntheticScene(b1.config, seed=3)
  train_loop.train(b1, ds, log=lambda s: None)
  assert checkpoints.latest_checkpoint(ck).endswith('checkpoint_60')
  b2 = train_loop_bundle(120, ckpt=ck)
  model_b, state_b, hist_b = train_loop.train(b2, ds, log=lambda s: None)
  assert state_b.step == 120 and hist_b[0]['step'] == 61
  pa, pb = state_a.params.flat, state_b.params.flat
  # same data and the same Adam state; only the jitter draws after the restart differ
  rel = float((pa - pb).norm() / pa.norm())
  assert rel < 0.05, rel
  blob = torch.load(checkpoints.latest_checkpoint(ck), map_location='cpu', weights_only=True)
  assert blob['step'] == 120 and set(blob['params_tree']) == {'NerfMLP_0', 'PropMLP_0'}
  assert blob['params_tree']['NerfMLP_0']['Dense_0']['kernel'].shape[1] == 128
  with pytest.raises(ValueError):
    from multinerf_b200 import train_utils
    other = plumbing_blender()
    m2, st2, *_ = train_utils.setup_model(other, 0)
    checkpoints.restore_checkpoint(ck, st2)
