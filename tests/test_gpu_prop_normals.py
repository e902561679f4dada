"""Normals on a colourless proposal MLP (disable_rgb with density and/or predicted normals): the normals stage
of csrc/refnerf.cu (mnrf_normals_fwd/bwd), the trunk-top dgrad against [w_density | W_grad_pred], and the
orientation / predicted-normal losses on every level, against the CPU oracle.  Needs an H100.

Reference: internal/models.py:468-501 (normals of any MLP), internal/train_utils.py:162-197 (the losses loop
over every level of ray_history).
"""
import numpy as np
import pytest
import torch

from model_parity import (bases, check_train_step, graph_matches_eager, image_rays, oracle_rays, pinned_forward,
                          synth_case, synth_rays, torch_tree)
from oracle import o_models
from util import close

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def mods():
  from multinerf_b200 import lib, models, train_utils
  lib.require_device()
  return models, train_utils


def mini_prop_normals(target='normals_pred', pred=True):
  """A reduced blender_256.gin (bounded, PropMLP without colour) with normals on both MLPs and both losses."""
  from multinerf_b200 import configs
  b = configs.bundle_blender_256()
  c, m, p, n = b.config, b.model, b.prop_mlp, b.nerf_mlp
  m.num_prop_samples, m.num_nerf_samples = 32, 16
  p.net_depth, p.net_width = 2, 64
  n.net_depth, n.net_width, n.bottleneck_width, n.net_width_viewdirs = 4, 128, 64, 64
  for mlp in (p, n):
    mlp.disable_density_normals, mlp.enable_pred_normals = False, pred
  c.orientation_loss_mult, c.orientation_coarse_loss_mult, c.orientation_loss_target = 0.1, 0.01, target
  if pred:
    c.predicted_normal_loss_mult, c.predicted_normal_coarse_loss_mult = 3e-4, 3e-5
  c.grad_max_norm = 0.0
  return b


def fullwidth_normals(pred=False):
  """blender_256.gin as shipped, with density normals on both MLPs and the orientation loss on them (pred: also
  predicted normals on both MLPs, the orientation loss on those, and the predicted-normal loss)."""
  from multinerf_b200 import configs
  b = configs.bundle_blender_256()
  b.prop_mlp.disable_density_normals = b.nerf_mlp.disable_density_normals = False
  b.config.orientation_loss_mult, b.config.orientation_coarse_loss_mult = 0.1, 0.01
  b.config.orientation_loss_target = 'normals'
  if pred:
    b.prop_mlp.enable_pred_normals = b.nerf_mlp.enable_pred_normals = True
    b.config.orientation_loss_target = 'normals_pred'
    b.config.predicted_normal_loss_mult, b.config.predicted_normal_coarse_loss_mult = 3e-4, 3e-5
  b.config.grad_max_norm = b.config.grad_max_val = 0.0
  return b


def _forward_vs_oracle(models, bundle, B, seed, dens_lim, pix_atol):
  rays, rand, _ = synth_case(bundle, B, seed, 2.0, 6.0, unit_cube=False)
  S = [bundle.model.num_prop_samples] * (bundle.model.num_levels - 1) + [bundle.model.num_nerf_samples]
  model, _ = models.construct_model(seed + 1, rays, bundle)
  pred = bundle.prop_mlp.enable_pred_normals

  def normals(i, st, h):
    # density normals: bf16 tangent chain vs fp32 autograd of the bf16-emulated forward (Ref-NeRF test's bound)
    cosn = (st.normals.cpu().view(B, st.S, 3) * h['normals']).sum(-1)
    assert float((cosn > 0.98).float().mean()) > 0.97, (i, float((cosn > 0.98).float().mean()))
    if pred:
      cosp = (st.normals_pred.cpu().view(B, st.S, 3) * h['normals_pred']).sum(-1)
      assert float((cosp > 0.98).float().mean()) > 0.97, (i, float((cosp > 0.98).float().mean()))
  # sample positions of each level pinned to the oracle's: one level's MLP and normals stage in isolation
  rend_o, _ = pinned_forward(model, bundle, rays, rand, dens=dens_lim, pixel=pix_atol, level=normals)
  rend, hist = model(rand, rays, 0.5, True)
  torch.cuda.synchronize()
  keys = ('normals', 'normals_pred') if pred else ('normals',)
  for i in range(len(S)):
    for k in keys:
      assert k in rend[i] and rend[i][k].shape == (B, 3), (i, k)
      assert hist[i][k] is not None and hist[i][k].shape == (B, S[i], 3), (i, k)
    assert hist[i]['raw_grad_density'].shape == (B, S[i], 3)
    assert (hist[i]['grad_pred'] is not None) == pred
  close(rend[-1]['rgb'], rend_o[-1]['rgb'], atol=3e-2, rtol=0, msg='final pixel end-to-end')


def test_construction_and_flax_tree(mods):
  from multinerf_b200 import configs
  models, _ = mods
  for bundle in (mini_prop_normals(), mini_prop_normals('normals', pred=False), fullwidth_normals(),
                 fullwidth_normals(pred=True)):
    model = models.Model(bundle)
    model.init(0)
    prop = model.plans['PropMLP_0']
    assert prop.normals_stage and not prop.has_rgb
    tree = model.export_flax()
    assert model.num_params() == sum(v['kernel'].size + v['bias'].size for t in tree.values() for v in t.values())
    names = sorted(tree['PropMLP_0'], key=lambda s: int(s.split('_')[1]))
    depth = bundle.prop_mlp.net_depth
    if bundle.prop_mlp.enable_pred_normals:
      assert names[-1] == f'Dense_{depth + 1}' and tree['PropMLP_0'][names[-1]]['kernel'].shape[1] == 3
    else:
      assert names[-1] == f'Dense_{depth}'
    # the oracle's flax-style MLP consumes exactly this tree (a missing or extra Dense raises there)
    rays, _ = synth_rays(0, 4, 2.0, 6.0, unit_cube=False)
    o_models.model_apply(torch_tree(tree), bundle, bases(model), oracle_rays(rays), 0.5, False)
  # PropMLP: grad_pred adds one Dense(3) on the 256-wide trunk output
  shipped = models.Model(configs.bundle_blender_256()).num_params()
  b = configs.bundle_blender_256()
  b.prop_mlp.disable_density_normals, b.prop_mlp.enable_pred_normals = False, True
  assert models.Model(b).num_params() == shipped + 256 * 3 + 3


def test_forward_vs_oracle(mods):
  models, _ = mods
  _forward_vs_oracle(models, mini_prop_normals(), 96, 50, (0.08, 4e-3), 1.5e-2)


@pytest.mark.parametrize('target', ['normals_pred', 'normals'])
def test_train_step_vs_oracle(mods, target):
  models, train_utils = mods
  bundle = mini_prop_normals(target, pred=target == 'normals_pred')
  # the PropMLP's gradient then comes from the normal losses alone: the new stage, its adjoint and the tangent
  # adjoint are not hidden behind the interlevel loss
  bundle.config.interlevel_loss_mult = 0.0
  check_train_step(models, train_utils, bundle, 96, 60, (0.2, 0.98))


def test_fullwidth_forward_vs_oracle(mods):
  models, _ = mods
  _forward_vs_oracle(models, fullwidth_normals(), 128, 70, (0.1, 5e-3), 1.5e-2)


@pytest.mark.parametrize('pred', [False, True])
def test_fullwidth_train_step_vs_oracle(mods, pred):
  # pred: the 256-wide PropMLP's trunk-top dgrad against [w_density | W_grad_pred] feeds the chained dgrad launch
  models, train_utils = mods
  check_train_step(models, train_utils, fullwidth_normals(pred), 128, 80, (0.3, 0.95))


def test_cuda_graph_matches_eager(mods):
  models, train_utils = mods
  B, steps = 192, 5
  rng = np.random.default_rng(91)
  batches = []
  for _ in range(steps):
    rays, _ = synth_rays(int(rng.integers(1 << 30)), B, 2.0, 6.0, unit_cube=False)
    rand = {'jitter': [torch.tensor(rng.uniform(0, 1, (B,)).astype(np.float32)) for _ in range(2)]}
    batches.append((rays, rng.uniform(0, 1, (B, 3)).astype(np.float32), rand))
  graph_matches_eager(models, train_utils, mini_prop_normals(), batches, 6,
                      extra=lambda stats: stats['losses']['orientation'])


def test_render_image_normals_chunked_equals_direct_call(mods):
  """render_image with compute_extras: normals on every level of a direct call, and a chunked render equal to it
  bit for bit.  The PropMLP is 256 wide with predicted normals only, so its trunk runs as one chained launch
  that must still store the last layer's output for the grad_pred head."""
  models, train_utils = mods
  bundle = mini_prop_normals()
  bundle.prop_mlp.net_width, bundle.prop_mlp.disable_density_normals = 256, True
  H, W = 29, 41
  bundle.config.render_chunk_size = 256
  bundle.config.vis_num_rays = 8
  rays = image_rays(H, W, focal=40.0)
  rays.origins[...] = np.array([0.0, 0.0, 4.0], np.float32)
  rays.near[...], rays.far[...] = 2.0, 6.0
  model, state, render_eval_pfn, _, _ = train_utils.setup_model(bundle, 3)
  out = models.render_image(lambda rng, r: render_eval_pfn(state.params, 1.0, None, r), rays, None, bundle,
                            verbose=False)
  flat = rays.map(lambda a: a.reshape(H * W, -1))
  rend, hist = model(None, flat, 1.0, True)
  torch.cuda.synchronize()
  for i, r in enumerate(rend):
    assert 'normals_pred' in r and hist[i]['normals_pred'] is not None, i
    assert ('normals' in r) == (i == len(rend) - 1), i
    assert torch.isfinite(r['normals_pred']).all()
  for k in ('rgb', 'acc', 'normals', 'normals_pred'):
    assert torch.equal(out[k].reshape(rend[-1][k].shape), rend[-1][k]), k
  # the proposal level's normals against the oracle's (deterministic call)
  params = torch_tree(model.export_flax())
  rend_o, hist_o = o_models.model_apply(params, bundle, bases(model), oracle_rays(flat), 1.0, True, rand=None,
                                        bf16=True)
  cosp = (hist[0]['normals_pred'].cpu() * hist_o[0]['normals_pred']).sum(-1)
  assert float((cosp > 0.98).float().mean()) > 0.97, float((cosp > 0.98).float().mean())


def test_missing_normals_value_errors(mods):
  models, _ = mods
  rays, _ = synth_rays(1, 8, 2.0, 6.0, unit_cube=False)
  # orientation on the predicted normals, which the PropMLP does not compute
  b = mini_prop_normals()
  b.prop_mlp.enable_pred_normals = False
  b.config.predicted_normal_loss_mult = b.config.predicted_normal_coarse_loss_mult = 0.0
  model, _ = models.construct_model(0, rays, b)
  with pytest.raises(ValueError, match='Normals cannot be None'):
    model.forward_levels(None, model._prep_rays(rays), 0.5, False, False, loss_config=b.config)
  # the predicted-normal loss needs both normals on the PropMLP too
  b = mini_prop_normals('normals')
  b.prop_mlp.enable_pred_normals = False
  model, _ = models.construct_model(0, rays, b)
  with pytest.raises(ValueError, match='Predicted normals and gradient normals'):
    model.forward_levels(None, model._prep_rays(rays), 0.5, False, False, loss_config=b.config)
