"""Parity of the BASELINE configurations AT THEIR STATED WIDTHS (BASELINE.json configs 2/3/4): the
shipped 360.gin (PropMLP 4x256, NerfMLP 8x1024, 64+64+32 samples), blender_refnerf.gin (8x256 + 8-layer
view MLP, 128+128 samples) and llff_raw.gin (8x256, 128+128 samples) against the CPU oracle on a few
hundred rays.  256 rays x 64 samples = 16384 sample rows, so every Dense layer runs the 256-wide
GEMM tiles that carry the benchmark -- the mini models of test_gpu_model.py only reach the narrow
tiles.  Needs an H100.

Reference: internal/models.py:75-312 (Model.__call__), :402-612 (MLP), internal/train_utils.py:72-218,
239-339; configs/{360,blender_refnerf,llff_raw}.gin.
"""
import numpy as np
import pytest
import torch

from model_parity import beyond, fullwidth_case, grad_report, mlp_leaves, pinned_forward, train_step, worst
from util import close

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def mods():
  from multinerf_b200 import lib, models, train_utils
  lib.require_device()
  return models, train_utils


@pytest.mark.parametrize('which', ['360', 'refnerf', 'raw'])
def test_fullwidth_forward_vs_oracle(mods, which):
  models, _ = mods
  bundle, rays, target, rand, B, S = fullwidth_case(which)
  model, variables = models.construct_model(40, rays, bundle)
  if which == 'raw':
    tree = model.export_flax()
    tree['exposure_scaling_offsets']['embedding'] = \
        np.random.default_rng(5).normal(size=(1000, 3)).astype(np.float32) * 0.1
    variables = model.init(flax_params=tree)

  def normals(i, st, h):
    if which == 'refnerf':
      # unit vectors from a bf16 head: a handful of samples with a tiny raw gradient are ill-conditioned
      ne = (st.normals_pred.cpu().view(B, st.S, 3) - h['normals_pred']).abs()
      assert float((ne < 3e-2).float().mean()) > 0.999 and float(ne.max()) < 0.15, (float(ne.max()),)
      cosn = (st.normals.cpu().view(B, st.S, 3) * h['normals']).sum(-1)
      assert float((cosn > 0.98).float().mean()) > 0.97, float((cosn > 0.98).float().mean())
      close(st.roughness.cpu().view(B, st.S, 1), h['roughness'], atol=2e-2, rtol=0, msg='roughness')
  # the sample positions of each level pinned to the oracle's: compares one level's chain in isolation; bf16
  # tensor-core MLP (8 x 1024-wide layers) vs the bf16-emulating oracle
  rend_o, _ = pinned_forward(model, bundle, rays, rand, dens=(0.1, 5e-3), pixel=1.5e-2, acc=1e-2, samples=4e-2,
                             level=normals)
  # end to end through Model.__call__ (sample positions drift with the bf16-level differences upstream)
  rend, hist = model(rand, rays, 0.5, True)
  close(rend[-1]['rgb'], rend_o[-1]['rgb'], atol=3e-2, rtol=0, msg=f'{which} final pixel end-to-end')
  assert hist[-1]['weights'].shape == (B, S[-1])


@pytest.mark.parametrize('which', ['360', 'refnerf', 'raw'])
def test_fullwidth_train_step_vs_oracle(mods, which):
  models, _ = mods
  bundle, rays, target, rand, B, S = fullwidth_case(which)
  bundle.config.grad_max_norm = 0.0        # raw Adam update; clipping has its own tests
  bundle.config.grad_max_val = 0.0
  model, variables = models.construct_model(41, rays, bundle)
  if which == 'raw':
    tree = model.export_flax()
    tree['exposure_scaling_offsets']['embedding'] = \
        np.random.default_rng(6).normal(size=(1000, 3)).astype(np.float32) * 0.1
    variables = model.init(flax_params=tree)
  t = train_step(model, variables, bundle, rays, target, rand, 0.5)
  stats, stats_o = t.stats, t.stats_o
  # per-level mse, PSNR and loss of the train step against the oracle's (tools/psnr_parity.py prints the same
  # comparison), asserted with an order of magnitude of head-room over bf16 rounding
  close(stats['mses'], stats_o['mses'].detach(), atol=1e-6, rtol=2e-3, msg=f'{which} mses')
  psnr_o = -10.0 / np.log(10.0) * np.log(stats_o['mses'].detach().double().numpy())
  close(stats['psnrs'], psnr_o, atol=5e-3, rtol=0, msg=f'{which} per-level PSNR (dB)')
  lo = float(stats_o['loss'].detach())
  assert abs(stats['loss'] - lo) < 3e-3 * max(1.0, abs(lo)), (stats['loss'], lo)
  for k in ('interlevel', 'distortion', 'orientation', 'predicted_normals'):
    if k in stats_o['losses'] and float(stats_o['losses'][k].detach()) != 0.0:
      v = float(stats_o['losses'][k].detach())
      assert abs(stats['losses'][k] - v) < 0.05 * abs(v) + 1e-7, (k, stats['losses'][k], v)
  heads = [(m, sp.name) for m in model.plans for sp in model.plans[m].specs if sp.out_dim <= 4]
  keys = mlp_leaves(model, ('kernel', 'bias'))
  report, zero = grad_report(model, t.grads_o, [k for k in keys if k[2] == 'kernel' or k[:2] not in heads])
  assert not any(zero.values()), zero
  g = model.export_grads_flax()
  for mname, lname in heads:
    if (mname, lname, 'kernel') in zero:
      continue
    # a head's bias gradient is a plain sum of the per-sample gradients: it cancels to (nearly) nothing,
    # so its error is measured against the size of the same head's kernel-gradient entries
    ba = torch.tensor(g[mname][lname]['bias']).double()
    bb, kb = t.grads_o[(mname, lname, 'bias')].double(), t.grads_o[(mname, lname, 'kernel')].double()
    scale = max(float(bb.abs().max()), float(kb.abs().max()))
    report[(mname, lname, 'bias')] = (round(float((ba - bb).abs().max()) / scale, 3), 1.0)
  report = {k: report[k] for k in keys if k in report}
  # dY travels between layers in bf16 on both sides with different rounding points, and every ReLU whose
  # pre-activation sits within bf16 noise of zero may flip: the error grows with depth and is largest at
  # Dense_0 (the worst leaves are printed below).
  # Ref-NeRF adds the bf16 tangent chain and an 8-layer view MLP.
  lim = {'360': (0.2, 0.98), 'refnerf': (0.3, 0.95), 'raw': (0.1, 0.995)}[which]
  print(f'[fullwidth {which}] worst leaves (rel, cos): {worst(report)}')
  bad = beyond(report, *lim)
  assert not bad, (bad, worst(report))
  if which == 'raw':
    r, z = grad_report(model, t.grads_o, [('exposure_scaling_offsets', 'embedding')])
    assert not z and r[('exposure_scaling_offsets', 'embedding')][0] < 0.05, (r, z)


def test_fullwidth_cta_pair_kernels_ran(mods):
  """The 360.gin layers at 256 rays take the 256-wide GEMM tiles (N % 256 == 0): guard the
  dispatch rule so a silent downgrade to a narrower tile is caught here, not in a profile."""
  from multinerf_b200 import configs
  from multinerf_b200.models import MLPPlan
  b = configs.bundle_360()
  for plan, S in ((MLPPlan(b.prop_mlp), 64), (MLPPlan(b.nerf_mlp), 32)):
    for sp in plan.by_role('trunk'):
      assert (256 * S) % 256 == 0 and sp.out_dim % 256 == 0 and sp.in_pad % 64 == 0
