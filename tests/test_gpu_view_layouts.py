"""The view-branch layouts of the reference MLP on the GPU, against the CPU oracle: no bottleneck (the Ref-NeRF
ablation, internal/models.py:526-537), no view MLP (net_depth_viewdirs = 0, the rgb head on [bottleneck | dir enc | n.v | GLO],
:575-585) with and without a bottleneck, and a view MLP with several skips that ends on one (the rgb head reads
[hidden | view input], :576-580).  Also the split input gradient of mnrf_head_bwd (dx2) those layouts use.  Needs an
H100.
"""
import numpy as np
import pytest
import torch

from model_parity import (beyond, check_train_step, fullwidth_case, grad_report, graph_matches_eager, level_jitter,
                          mlp_leaves, pinned_forward, synth_case, synth_rays, train_step, worst)
from util import close

pytestmark = pytest.mark.gpu

LAYOUTS = ['no_bottleneck', 'depth0_glo', 'depth0_no_bottleneck', 'skips']


@pytest.fixture(scope='module')
def mods():
  from multinerf_b200 import lib, models, train_utils
  lib.require_device()
  return models, train_utils


def mini_layout(name):
  """A reduced blender_256.gin (two MLPs; a chained 4 x 256 NerfMLP trunk, 64-wide bottleneck and view MLP) in one of
  the view-branch layouts.  The Ref-NeRF ones (IDE, roughness, diffuse, tint, n.v; density and predicted normals on
  both MLPs, with both normal losses) have no bottleneck."""
  from multinerf_b200 import configs
  b = configs.bundle_blender_256()
  c, m, p, n = b.config, b.model, b.prop_mlp, b.nerf_mlp
  m.num_prop_samples, m.num_nerf_samples = 32, 16
  p.net_depth, p.net_width = 2, 64
  n.net_depth, n.net_width = 4, 256
  n.bottleneck_width, n.net_width_viewdirs = 64, 64
  c.grad_max_norm = c.grad_max_val = 0.0
  if name in ('no_bottleneck', 'depth0_no_bottleneck'):
    for mlp in (p, n):
      mlp.disable_density_normals, mlp.enable_pred_normals = False, True
    n.use_directional_enc = n.use_reflections = n.enable_pred_roughness = True
    n.use_diffuse_color = n.use_specular_tint = n.use_n_dot_v = True
    n.deg_view, n.bottleneck_width = 5, 0
    c.orientation_loss_mult, c.orientation_coarse_loss_mult, c.orientation_loss_target = 0.1, 0.01, 'normals_pred'
    c.predicted_normal_loss_mult, c.predicted_normal_coarse_loss_mult = 3e-4, 3e-5
    n.net_depth_viewdirs = 6 if name == 'no_bottleneck' else 0
  else:
    m.num_glo_features, m.num_glo_embeddings = 4, 3
    if name == 'depth0_glo':
      n.net_depth_viewdirs = 0
    else:
      n.net_depth_viewdirs, n.skip_layer_dir = 5, 2      # skips after layers 2 and 4, the last
  return b


def _check_plan(models, bundle, name):
  plan = models.MLPPlan(bundle.nerf_mlp, glo_features=bundle.model.num_glo_features)
  assert plan.has_bottleneck == (name in ('depth0_glo', 'skips'))
  assert plan.rgb_vin == {'skips': 'tail', 'no_bottleneck': None}.get(name, 'all')


@pytest.mark.parametrize('name', LAYOUTS)
def test_forward_vs_oracle(mods, name):
  models, _ = mods
  bundle = mini_layout(name)
  _check_plan(models, bundle, name)
  rays, rand, _ = synth_case(bundle, 96, 60, 2.0, 6.0, unit_cube=False)
  model, _ = models.construct_model(61, rays, bundle)
  rend_o, _ = pinned_forward(model, bundle, rays, rand, dens=(0.08, 4e-3), pixel=1.5e-2, samples=1.5e-2)
  rend, _ = model(rand, rays, 0.5, True)
  torch.cuda.synchronize()
  close(rend[-1]['rgb'], rend_o[-1]['rgb'], atol=3e-2, rtol=0, msg='final pixel end-to-end')


@pytest.mark.parametrize('name', LAYOUTS)
def test_train_step_vs_oracle(mods, name):
  models, train_utils = mods
  check_train_step(models, train_utils, mini_layout(name), 96, 62, (0.2, 0.98))


@pytest.mark.parametrize('name', LAYOUTS)
def test_cuda_graph_matches_eager(mods, name):
  models, train_utils = mods
  bundle = mini_layout(name)
  B, steps = 192, 5
  rng = np.random.default_rng(63)
  batches = []
  for _ in range(steps):
    rays, _ = synth_rays(int(rng.integers(1 << 30)), B, 2.0, 6.0, unit_cube=False)
    rays.cam_idx = rng.integers(0, 3, (B, 1)).astype(np.int32)
    batches.append((rays, rng.uniform(0, 1, (B, 3)).astype(np.float32), level_jitter(rng, bundle, B)))
  graph_matches_eager(models, train_utils, bundle, batches, 64)


@pytest.mark.parametrize('name', LAYOUTS)
def test_chained_trunk_matches_per_layer(mods, monkeypatch, name):
  """The chained 256-wide trunk against one GEMM per layer (MNRF_CHAIN=0): forward pixels, the loss and the gradients
  of the trunk top and of every view-branch layer after one step."""
  models, train_utils = mods
  from multinerf_b200 import utils
  bundle = mini_layout(name)
  B = 256
  rays, rng = synth_rays(65, B, 2.0, 6.0, unit_cube=False)
  target = rng.uniform(0, 1, (B, 3)).astype(np.float32)
  out = []
  for chain in ('1', '0'):
    monkeypatch.setenv('MNRF_CHAIN', chain)
    model, variables = models.construct_model(66, rays, bundle)
    assert model._use_chain(model.plans['NerfMLP_0'], B * bundle.model.num_nerf_samples) == (chain == '1')
    rend, _ = model(None, rays, 0.5, False)
    step = train_utils.create_train_step(model, bundle.config, use_graph=False)
    variables.grads.zero_()
    _, stats, _ = step(None, train_utils.TrainState(variables), utils.Batch(rays=rays, rgb=target), None, 0.5)
    torch.cuda.synchronize()
    stats.materialize()
    out.append((rend[-1]['rgb'].clone(), stats['loss'], model.export_grads_flax()))
  (r1, l1, g1), (r0, l0, g0) = out
  close(r1, r0, atol=2e-3, rtol=0, msg='pixels chained vs per-layer')
  assert abs(l1 - l0) < 1e-3 * max(1.0, abs(l0)), (l1, l0)
  plan = model.plans['NerfMLP_0']
  for sp in plan.specs:
    if sp.role == 'trunk':
      continue
    a, b = torch.tensor(g1['NerfMLP_0'][sp.name]['kernel']), torch.tensor(g0['NerfMLP_0'][sp.name]['kernel'])
    assert float((a - b).norm() / b.norm()) < 3e-2, (sp.name, sp.role)


def fullwidth(name):
  """(bundle, rays, target, rand): blender_refnerf.gin without a bottleneck (chained 256-wide trunk, 128-wide view
  input), 360.gin without a view MLP (per-layer 1024-wide trunk, rgb head over K = 320), blender_256.gin with a 9-layer
  view MLP (skips after layers 4 and 8, rgb head over K = 448)."""
  from multinerf_b200 import configs
  if name == 'refnerf_no_bottleneck':
    bundle, rays, target, rand, _, _ = fullwidth_case('refnerf')
    bundle.nerf_mlp.bottleneck_width = 0
  elif name == '360_depth0':
    bundle, rays, target, rand, _, _ = fullwidth_case('360')
    bundle.nerf_mlp.net_depth_viewdirs = 0
  else:
    bundle = configs.bundle_blender_256()
    bundle.nerf_mlp.net_depth_viewdirs, bundle.nerf_mlp.skip_layer_dir = 9, 4
    rays, rand, target = synth_case(bundle, 128, 70, 2.0, 6.0, unit_cube=False)
  bundle.config.grad_max_norm = bundle.config.grad_max_val = 0.0
  return bundle, rays, target, rand


FULL = ['refnerf_no_bottleneck', '360_depth0', 'blender_256_skips']


@pytest.mark.parametrize('name', FULL)
def test_fullwidth_forward_vs_oracle(mods, name):
  models, _ = mods
  bundle, rays, target, rand = fullwidth(name)
  model, _ = models.construct_model(71, rays, bundle)
  rend_o, _ = pinned_forward(model, bundle, rays, rand, dens=(0.1, 5e-3), pixel=1.5e-2, acc=1e-2, samples=4e-2)
  rend, _ = model(rand, rays, 0.5, True)
  torch.cuda.synchronize()
  close(rend[-1]['rgb'], rend_o[-1]['rgb'], atol=3e-2, rtol=0, msg=f'{name} final pixel end-to-end')


@pytest.mark.parametrize('name', FULL)
def test_fullwidth_train_step_vs_oracle(mods, name):
  """Bounds of the shipped full-width train-step tests: (0.3, 0.95) with the Ref-NeRF stage or a deep view MLP,
  (0.2, 0.98) otherwise."""
  models, _ = mods
  bundle, rays, target, rand = fullwidth(name)
  model, variables = models.construct_model(72, rays, bundle)
  t = train_step(model, variables, bundle, rays, target, rand, 0.5)
  close(t.stats['mses'], t.stats_o['mses'].detach(), atol=1e-6, rtol=2e-3, msg=f'{name} mses')
  for k in ('orientation', 'predicted_normals'):
    if k in t.stats_o['losses'] and float(t.stats_o['losses'][k].detach()) != 0.0:
      v = float(t.stats_o['losses'][k].detach())
      assert abs(t.stats['losses'][k] - v) < 0.05 * abs(v) + 1e-7, (k, t.stats['losses'][k], v)
  report, zero = grad_report(model, t.grads_o, mlp_leaves(model))
  assert not any(zero.values()), zero
  print(f'[{name}] worst leaves (rel, cos): {worst(report)}')
  lim = (0.2, 0.98) if name == '360_depth0' else (0.3, 0.95)
  bad = beyond(report, *lim)
  assert not bad, (bad, worst(report))


@pytest.mark.parametrize('K,dx_cols', [(448, 128), (320, 256), (256, 128)])
@pytest.mark.parametrize('M', [1000, 4099])
@pytest.mark.parametrize('with_dxsum', [False, True])
def test_head_bwd_split_input_gradient(mods, K, dx_cols, M, with_dxsum):
  """mnrf_head_bwd with a second input-gradient output: columns [0, dx_cols) relu-masked into dx (and summed into
  dxsum), columns [dx_cols, K) unmasked into dx2 with its own pitch, against an fp32 product of the bf16 operands.
  K = 448: the rgb head of blender_256.gin's view MLP ending on a skip; 320 and 256 the general and narrow kernels."""
  from multinerf_b200 import ops
  g = torch.Generator(device='cuda')
  g.manual_seed(M * 7 + K)
  x = (torch.randn(M, K, device='cuda', generator=g)).to(torch.bfloat16)
  w = (torch.randn(3, K, device='cuda', generator=g) * 0.05).to(torch.bfloat16)
  draw = torch.randn(M, 3, device='cuda', generator=g)
  sentinel = -7.0
  dx = torch.full((M, dx_cols + 8), sentinel, device='cuda', dtype=torch.bfloat16)[:, :dx_cols]
  tail = K - dx_cols
  dx2_buf = torch.full((M, tail + 64), sentinel, device='cuda', dtype=torch.bfloat16)
  dx2 = dx2_buf[:, :tail]
  dw, db = torch.zeros(K, 3, device='cuda'), torch.zeros(3, device='cuda')
  dxs = torch.zeros(K, device='cuda') if with_dxsum else None
  ops.head_bwd(x, w, draw, 3, K, dx=dx, relu_mask=True, dw=dw, db=db, dxsum=dxs, dx_cols=dx_cols, dx2=dx2)
  # the same call without the second output: the first part is bit-identical
  dx_ref = torch.empty(M, dx_cols, device='cuda', dtype=torch.bfloat16)
  ops.head_bwd(x, w, draw, 3, K, dx=dx_ref, relu_mask=True, dx_cols=dx_cols)
  torch.cuda.synchronize()
  full = draw @ w.float()
  xf = x.float()
  close(dx.float(), full[:, :dx_cols] * (xf[:, :dx_cols] > 0), atol=1e-2, rtol=1e-2, msg='dx (masked part)')
  close(dx2.float(), full[:, dx_cols:], atol=1e-2, rtol=1e-2, msg='dx2 (unmasked tail)')
  assert torch.equal(dx, dx_ref)
  # nothing past either output's columns is written
  assert bool((dx2_buf[:, tail:] == sentinel).all())
  close(dw, xf.t() @ draw, atol=2e-2 * M ** 0.5, rtol=1e-3, msg='dW')
  close(db, draw.sum(0), atol=1e-2, rtol=1e-4, msg='db')
  if with_dxsum:
    close(dxs[:dx_cols], dx.float().sum(0), atol=0.5, rtol=1e-2, msg='dxsum')
    assert not dxs[dx_cols:].any()
