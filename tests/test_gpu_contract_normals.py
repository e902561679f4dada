"""Density normals through the scene contraction (`warp_fn = contract` with `disable_density_normals = False`):
the normals, normal losses and Ref-NeRF stage of 360-style models built on the tangent rows of csrc/encode.cu with
warp_contract, against the CPU oracle.  Needs an H100.  The tangent rows themselves are checked element by element in
test_gpu_encode_fp64.py.

Reference: internal/models.py:441-492 (vmap(value_and_grad(predict_density)) with respect to the world-space
mean, through coord.track_linearize(contract, ...), coord.py:39-60).
"""
import numpy as np
import pytest
import torch

from model_parity import (fullwidth_case, graph_matches_eager, grad_report, image_rays, mini360, mlp_leaves,
                          oracle_rays, oracle_step, pinned_forward, synth_case, synth_rays, torch_tree, train_step,
                          worst)
from oracle import o_coord, o_models, o_render
from util import close

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def mods():
  from multinerf_b200 import lib, models, train_utils
  lib.require_device()
  return models, train_utils


# ------------------------------------------------------------------ model

def mini360_normals(refnerf=False):
  """mini360 (reciprocal ray distances, contraction on both MLPs) with density and predicted normals on both
  MLPs and both normal losses; refnerf: the NerfMLP also reflects the view direction, with the integrated
  directional encoding and a predicted roughness."""
  b = mini360()
  for mlp in (b.prop_mlp, b.nerf_mlp):
    mlp.disable_density_normals, mlp.enable_pred_normals = False, True
  if refnerf:
    n = b.nerf_mlp
    n.use_reflections = n.use_directional_enc = n.enable_pred_roughness = True
  c = b.config
  c.orientation_loss_mult, c.orientation_coarse_loss_mult, c.orientation_loss_target = 0.1, 0.01, 'normals_pred'
  c.predicted_normal_loss_mult, c.predicted_normal_coarse_loss_mult = 3e-4, 3e-5
  c.grad_max_norm = c.grad_max_val = 0.0
  return b


# Where the bf16 arithmetic itself moves a quantity by more than the fixed bounds, the bound is derived from how
# far the oracle's own bf16 evaluation lies from its fp32 one on the same inputs: the tensor-core path rounds at
# other points than the oracle's bf16 emulation, so each may sit on either side of the fp32 value.
SENSITIVITY = 2.5


def _normals_errors(got, ref):
  """(fraction of unit-length reference normals with cosine > 0.98, per-sample max abs error of the normals whose
  raw gradient is under the eps clamp of l2_normalize)."""
  unit = ref.norm(dim=-1) > 0.999
  cos = (got * ref).sum(-1)[unit]
  return float((cos > 0.98).float().mean()), (got - ref).abs().amax(-1)[~unit]


def _check_normals(got, ref, what, inherent=None):
  """Unit-length reference normals by cosine; those whose raw gradient is under the eps clamp (shorter than 1,
  common far out where |J| ~ 1/|x|^2) by absolute error: there the normal is the raw gradient times
  1/sqrt(eps) ~ 2900, so a bf16 chain's absolute error in a tiny gradient shows at that scale.  `inherent`: the
  same errors of the oracle's fp32 normals against its bf16 ones, which widen the bounds."""
  miss, atol = 0.03, 0.05
  if inherent is not None:
    frac_i, err_i = inherent
    miss = max(miss, SENSITIVITY * (1.0 - frac_i))
    if err_i.numel():
      atol = max(atol, SENSITIVITY * float(torch.quantile(err_i, 0.97)))
  frac, err = _normals_errors(got, ref)
  assert frac > 1.0 - miss, (what, frac, miss)
  if err.numel():
    assert float((err < atol).float().mean()) > 0.97, (what, err.numel(), float(err.max()), atol)


def _fp32_normals(params, bundle, model, orays, mname, sdist):
  """The oracle's fp32 density normals at the samples `sdist` of one level."""
  cfg = bundle.prop_mlp if mname == 'PropMLP_0' else bundle.nerf_mlp
  _, s_to_t = o_coord.construct_ray_warps(bundle.model.raydist_fn, orays.near, orays.far)
  gauss = o_render.cast_rays(s_to_t(sdist), orays.origins, orays.directions, orays.radii, bundle.model.ray_shape,
                             diag=False)
  out = o_models.mlp_apply(params[mname], cfg, model.plans[mname].basis, gauss, viewdirs=orays.viewdirs, bf16=False)
  return out['normals'].detach()


def _forward_vs_oracle(models, bundle, rays, rand, seed, dens_lim, pix_atol, derived=False):
  B = rays.origins.shape[0]
  model, _ = models.construct_model(seed, rays, bundle)
  params = torch_tree(model.export_flax())
  pred = bundle.nerf_mlp.enable_pred_normals
  n_clamped = 0

  def normals(i, st, h):
    nonlocal n_clamped
    inherent = None
    if derived:
      inherent = _normals_errors(_fp32_normals(params, bundle, model, oracle_rays(rays), st.mname, h['sdist']),
                                 h['normals'])
      print(f'level {i}: oracle fp32 vs bf16 normals {inherent[0]:.4f}, clamped '
            f'{float(inherent[1].max()) if inherent[1].numel() else 0.0:.3f}; GPU vs oracle bf16 normals '
            f'{_normals_errors(st.normals.cpu().view(B, st.S, 3), h["normals"])[0]:.4f}')
    _check_normals(st.normals.cpu().view(B, st.S, 3), h['normals'], f'normals level {i}', inherent)
    n_clamped += int((h['normals'].norm(dim=-1) < 0.999).sum())
    if pred:
      _check_normals(st.normals_pred.cpu().view(B, st.S, 3), h['normals_pred'], f'normals_pred level {i}')
  # sample positions of each level pinned to the oracle's: one level's MLP and normals stage in isolation
  rend_o, _ = pinned_forward(model, bundle, rays, rand, dens=dens_lim, pixel=pix_atol, level=normals)
  print(f'samples under the eps clamp: {n_clamped}')
  rend, hist = model(rand, rays, 0.5, True)
  torch.cuda.synchronize()
  for i in range(len(hist)):
    assert 'normals' in rend[i] and hist[i]['normals'] is not None and hist[i]['raw_grad_density'] is not None, i
  close(rend[-1]['rgb'], rend_o[-1]['rgb'], atol=3e-2, rtol=0, msg='final pixel end-to-end')


def _oracle_sensitivity(grads_a, grads_b):
  """Per leaf (rel, cos) of two oracle gradient sets."""
  out = {}
  for k, b in grads_b.items():
    a, b = grads_a[k].double().flatten(), b.double().flatten()
    if float(b.norm()) > 0.0:
      out[k] = (float((a - b).norm() / b.norm()), float((a @ b) / (a.norm() * b.norm()).clamp(min=1e-30)))
  return out


def _train_step_vs_oracle(models, train_utils, bundle, rays, rand, target, seed, lim, derived=False):
  model, variables = models.construct_model(seed, rays, bundle)
  t = train_step(model, variables, bundle, rays, target, rand, 0.5)
  stats, stats_o = t.stats, t.stats_o
  close(stats['mses'], stats_o['mses'].detach(), atol=2e-3, rtol=3e-2, msg='mses')
  sens, stats_32 = {}, None
  if derived:
    _, _, stats_32, grads_32 = oracle_step(t.params0, model, bundle, rays, target, rand, 0.5, bf16=False)
    sens = _oracle_sensitivity(t.grads_o, grads_32)
  seen = 0
  for k in ('orientation', 'predicted_normals'):
    if k in stats_o['losses'] and float(stats_o['losses'][k].detach()) != 0.0:
      lo = float(stats_o['losses'][k].detach())
      rel = 0.05
      if stats_32 is not None:
        rel = max(rel, SENSITIVITY * abs(float(stats_32['losses'][k].detach()) - lo) / abs(lo))
      assert abs(stats['losses'][k] - lo) < rel * abs(lo) + 1e-7, (k, stats['losses'][k], lo, rel)
      seen += 1
  assert seen > 0
  report, zero = grad_report(model, t.grads_o, mlp_leaves(model, ('kernel', 'bias')))
  assert not any(zero.values()), zero
  print(f'worst leaves (rel, cos): {worst(report)}')
  if sens:
    print('oracle bf16 vs fp32 at those leaves:', {k[:2] + (k[2],): tuple(round(x, 4) for x in sens.get(k, (0, 1)))
                                                   for k, _ in worst(report)})

  def bound(k):
    rel_i, cos_i = sens.get(k, (0.0, 1.0))
    return max(lim[0], SENSITIVITY * rel_i), min(lim[1], 1.0 - SENSITIVITY * (1.0 - cos_i))
  bad = {k: (v, bound(k)) for k, v in report.items() if not (v[0] < bound(k)[0] and v[1] > bound(k)[1])}
  assert not bad, (bad, worst(report))


@pytest.mark.parametrize('refnerf', [False, True])
def test_forward_vs_oracle(mods, refnerf):
  models, _ = mods
  bundle = mini360_normals(refnerf)
  rays, rand, _ = synth_case(bundle, 128, 150, 0.2, 1e6)
  _forward_vs_oracle(models, bundle, rays, rand, 151, (0.08, 4e-3), 1.5e-2)


@pytest.mark.parametrize('target', ['normals_pred', 'normals'])
def test_train_step_vs_oracle(mods, target):
  models, train_utils = mods
  bundle = mini360_normals()
  bundle.config.orientation_loss_target = target
  # the PropMLP's gradient then comes from the normal losses alone: the tangent rows through the contraction
  # and their adjoint are not hidden behind the interlevel loss
  bundle.config.interlevel_loss_mult = 0.0
  rays, rand, target_rgb = synth_case(bundle, 128, 160, 0.2, 1e6)
  # orientation on the density normals: the loss's gradient runs through the samples under the eps clamp, where
  # it is scaled by 1/sqrt(eps); there the oracle's bf16 and fp32 evaluations already differ at the density head
  _train_step_vs_oracle(models, train_utils, bundle, rays, rand, target_rgb, 161, (0.2, 0.98),
                        derived=target == 'normals')


def fullwidth360_normals():
  """360.gin as shipped with density normals on both MLPs and the orientation loss on them."""
  from multinerf_b200 import configs
  b = configs.bundle_360()
  b.prop_mlp.disable_density_normals = b.nerf_mlp.disable_density_normals = False
  b.config.orientation_loss_mult, b.config.orientation_coarse_loss_mult = 0.1, 0.01
  b.config.orientation_loss_target = 'normals'
  b.config.grad_max_norm = b.config.grad_max_val = 0.0
  return b


def test_fullwidth_forward_vs_oracle(mods):
  models, _ = mods
  _, rays, _, rand, _, _ = fullwidth_case('360')
  _forward_vs_oracle(models, fullwidth360_normals(), rays, rand, 40, (0.1, 5e-3), 1.5e-2, derived=True)


def test_fullwidth_train_step_vs_oracle(mods):
  models, train_utils = mods
  _, rays, target, rand, _, _ = fullwidth_case('360')
  _train_step_vs_oracle(models, train_utils, fullwidth360_normals(), rays, rand, target, 41, (0.3, 0.95),
                        derived=True)


def test_cuda_graph_matches_eager(mods):
  models, train_utils = mods
  B, steps = 192, 5
  rng = np.random.default_rng(93)
  batches = []
  for _ in range(steps):
    rays, _ = synth_rays(int(rng.integers(1 << 30)), B, 0.2, 1e6)
    rand = {'jitter': [torch.tensor(rng.uniform(0, 1, (B,)).astype(np.float32)) for _ in range(3)]}
    batches.append((rays, rng.uniform(0, 1, (B, 3)).astype(np.float32), rand))
  graph_matches_eager(models, train_utils, mini360_normals(), batches, 8,
                      extra=lambda stats: stats['losses']['orientation'])


def test_render_image_normals_chunked_equals_direct_call(mods):
  models, train_utils = mods
  bundle = mini360_normals()
  H, W = 29, 41
  bundle.config.render_chunk_size = 256
  bundle.config.vis_num_rays = 8
  rays = image_rays(H, W, focal=40.0)          # origin inside the unit ball, near 0.2, far 1e6
  model, state, render_eval_pfn, _, _ = train_utils.setup_model(bundle, 3)
  out = models.render_image(lambda rng, r: render_eval_pfn(state.params, 1.0, None, r), rays, None, bundle,
                            verbose=False)
  flat = rays.map(lambda a: a.reshape(H * W, -1))
  rend, hist = model(None, flat, 1.0, True)
  torch.cuda.synchronize()
  for i, r in enumerate(rend):
    assert 'normals' in r and 'normals_pred' in r and hist[i]['normals'] is not None, i
    assert torch.isfinite(r['normals']).all() and torch.isfinite(r['normals_pred']).all()
  for k in ('rgb', 'acc', 'normals', 'normals_pred'):
    assert torch.equal(out[k].reshape(rend[-1][k].shape), rend[-1][k]), k
