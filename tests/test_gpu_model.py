"""Model-level parity on the GPU: Model.__call__ and the train step vs the CPU oracle on
identical synthetic rays and weights (SURVEY.md section 8d).  Needs an H100.

The Dense layers run in bf16 on tensor cores, so the oracle is evaluated with the same
bf16-rounded weights and bf16-rounded layer inputs (fp32 accumulation) -- see
oracle/o_models.py `bf16=True`.  Achieved errors are asserted with explicit tolerances.
"""
import copy

import numpy as np
import pytest
import torch

from model_parity import (bases, beyond, graph_matches_eager, grad_report, level_jitter, mini360, mini_refnerf,
                          mlp_leaves, oracle_rays, pinned_forward, plumbing_blender, raw_rays, synth_rays, torch_tree,
                          train_step)
from oracle import o_models, o_train
from util import close

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def mods():
  from multinerf_b200 import lib, models, train_utils
  lib.require_device()
  return models, train_utils


def test_param_counts_known_answers(mods):
  # scripts/generate_tables.ipynb:145 and sibling rows (SURVEY.md fact 3)
  from multinerf_b200 import configs
  models, _ = mods
  assert models.Model(configs.bundle_360()).num_params() == 9007493
  assert models.Model(configs.bundle_blender_256()).num_params() == 835205
  raw = models.Model(configs.bundle_llff_raw())
  assert raw.num_params() + sum(raw.extra_params.values()) == 615740      # generate_tables.ipynb (llff_raw)


@pytest.mark.parametrize('which', ['plumbing', 'mini360'])
def test_model_forward_vs_oracle(mods, which):
  models, _ = mods
  bundle = plumbing_blender() if which == 'plumbing' else mini360()
  B = 64 if which == 'plumbing' else 160
  near, far = (2.0, 6.0) if which == 'plumbing' else (0.2, 1e6)
  rays, rng = synth_rays(0 if which == 'plumbing' else 1, B, near, far, unit_cube=which != 'plumbing')
  model, variables = models.construct_model(2, rays, bundle)
  for randomized in [False, True]:
    rand = level_jitter(rng, bundle, B) if randomized else None
    rend, hist = model(rand, rays, 0.5, True)
    torch.cuda.synchronize()
    # bf16 tensor-core MLP vs bf16-emulating oracle: state the achieved error
    rend_o, _ = pinned_forward(model, bundle, rays, rand, dens=(0.08, 4e-3), pixel=1e-2, acc=1e-2, samples=3e-2)
    # end to end (sample positions drift with the bf16-level differences of earlier levels)
    close(rend[-1]['rgb'], rend_o[-1]['rgb'], atol=2e-2, rtol=0, msg='final pixel end-to-end')
    assert rend[-1]['rgb'].shape == (B, 3) and hist[-1]['weights'].shape == (B, bundle.model.num_nerf_samples)
    for k in ['acc', 'distance_mean', 'distance_median', 'distance_percentile_5', 'distance_percentile_95',
              'ray_sdist', 'ray_weights', 'ray_rgbs']:
      assert k in rend[-1]


@pytest.mark.parametrize('which,impl', [('mini360', 1), ('mini360', 0), ('plumbing', 0)])
def test_train_step_vs_oracle(mods, which, impl):
  models, _ = mods
  bundle = plumbing_blender() if which == 'plumbing' else mini360()
  bundle.config.grad_max_norm = 0.0      # compare raw Adam first; clipping is covered below
  B = 64 if which == 'plumbing' else 160
  near, far = (2.0, 6.0) if which == 'plumbing' else (0.2, 1e6)
  rays, rng = synth_rays(3, B, near, far, unit_cube=which != 'plumbing')
  target = rng.uniform(0, 1, (B, 3)).astype(np.float32)
  model, variables = models.construct_model(4, rays, bundle)
  t = train_step(model, variables, bundle, rays, target, level_jitter(rng, bundle, B), 0.5, impl=impl)
  close(t.stats['mses'], t.stats_o['mses'].detach(), atol=2e-3, rtol=2e-2, msg='mses')
  lo = float(t.stats_o['loss'].detach())
  assert abs(t.stats['loss'] - lo) < 2e-2 * max(1.0, abs(lo)), (t.stats['loss'], lo)
  report, zero = grad_report(model, t.grads_o, mlp_leaves(model, ('kernel', 'bias')))
  # a module unused by the config (e.g. PropMLP at 1 level) gets no gradient on either side
  assert not any(zero.values()), zero
  # dY travels between layers in bf16 on both sides (different rounding points): the deepest
  # backward path (Dense_0) accumulates the most
  assert not beyond(report, 0.12, 0.993), beyond(report, 0.12, 0.993)
  # parameters after one Adam step (first step moves every weight by ~lr regardless of scale)
  newp = model.export_flax()
  lr = o_train.lr_at(0, bundle.config)
  for mname in newp:
    for lname in newp[mname]:
      a = torch.tensor(newp[mname][lname]['kernel'])
      b = t.new_o[mname][lname]['kernel']
      p0 = t.params0[mname][lname]['kernel']
      assert float((a - b).abs().max()) <= 2.1 * lr, (mname, lname)
      agree = ((a - p0).sign() == (b - p0).sign())
      assert float(agree.float().mean()) > 0.95, (mname, lname, float(agree.float().mean()))


def test_cuda_graph_train_step_matches_eager(mods):
  """The captured two-graph step (forward+backward | clip+Adam+repack) must track the eager step
  while train_frac, the learning rate, the Adam bias corrections and the jitter change per step."""
  models, train_utils = mods
  B, steps = 256, 5
  _, rng = synth_rays(5, B, 0.2, 1e6)
  batches = [(synth_rays(10 + i, B, 0.2, 1e6)[0], rng.uniform(0, 1, (B, 3)).astype(np.float32)) for i in range(steps)]
  rands = [{'jitter': [torch.tensor(rng.uniform(0, 1, (B,)).astype(np.float32)) for _ in range(3)]}
           for _ in range(steps)]
  graph_matches_eager(models, train_utils, mini360(), [b + (r,) for b, r in zip(batches, rands)], 6)


def test_cuda_graph_gradients_track_eager_with_moving_weights(mods):
  """Graph replays must read the CURRENT weights everywhere, including the fp32 density-head row the
  NerfMLP dgrad folds in as a rank-1 term (`colv_density`).  A dozen replays at a large learning rate move
  the weights by tens of percent; then ONE more step is taken twice from the same state -- by graph replay
  and by a fresh eager step function -- and the gradients must agree to fp32-atomics noise.  A pointer
  captured to a stale copy of any weight would show up as a gradient error of the size of the drift."""
  models, train_utils = mods
  from multinerf_b200 import utils
  bundle = mini360()
  bundle.config.lr_init = bundle.config.lr_final = 5e-3
  bundle.config.lr_delay_steps = 0
  B, steps = 256, 12
  rays, rng = synth_rays(55, B, 0.2, 1e6)
  batches = [(synth_rays(60 + i, B, 0.2, 1e6)[0], rng.uniform(0, 1, (B, 3)).astype(np.float32))
             for i in range(steps + 1)]
  rands = [{'jitter': [torch.tensor(rng.uniform(0, 1, (B,)).astype(np.float32)) for _ in range(3)]}
           for _ in range(steps + 1)]
  model, variables = models.construct_model(56, rays, bundle)
  d = model.plans['NerfMLP_0'].one('density')
  w0 = model.mlps['NerfMLP_0'].W(d).clone()
  step_fn = train_utils.create_train_step(model, bundle.config, use_graph=True)
  state = train_utils.TrainState(variables)
  for i in range(steps):
    r, tgt = batches[i]
    state, stats, _ = step_fn(rands[i], state, utils.Batch(rays=r, rgb=tgt), None, i / 20.0)
  torch.cuda.synchronize()
  assert step_fn.graph_info['state'] == 2
  w1 = model.mlps['NerfMLP_0'].W(d)
  assert float((w1 - w0).norm() / w0.norm()) > 0.05            # the head really moved
  # the fp32 row handed to the dgrad epilogue is the bf16 rounding of the current master weights
  assert torch.equal(model.mlps['NerfMLP_0'].colv_density[:w1.shape[0]], w1[:, 0].to(torch.bfloat16).float())
  p = variables
  snap = (p.flat.clone(), p.mu.clone(), p.nu.clone(), p.step)
  r, tgt = batches[steps]
  state, _, _ = step_fn(rands[steps], state, utils.Batch(rays=r, rgb=tgt), None, 0.6)      # replay
  torch.cuda.synchronize()
  g_graph = model.export_grads_flax()
  p.flat.copy_(snap[0]); p.mu.copy_(snap[1]); p.nu.copy_(snap[2]); p.step = snap[3]
  for mlp in model.mlps.values():
    mlp.repack()
  eager_fn = train_utils.create_train_step(model, bundle.config, use_graph=False)
  state, _, _ = eager_fn(rands[steps], state, utils.Batch(rays=r, rgb=tgt), None, 0.6)
  torch.cuda.synchronize()
  g_eager = model.export_grads_flax()
  for mname in g_graph:
    for lname in g_graph[mname]:
      a = torch.tensor(g_graph[mname][lname]['kernel']).double().flatten()
      b = torch.tensor(g_eager[mname][lname]['kernel']).double().flatten()
      rel = float((a - b).norm() / b.norm().clamp(min=1e-30))
      assert rel < 5e-3, (mname, lname, rel)


def test_rawnerf_train_step_vs_oracle(mods):
  """BASELINE config 4 (llff_raw.gin) at reduced size: single MLP for both levels, cylinder rays,
  safe_exp colours, per-sample jitter, density noise, exposure scaling with learned offsets, Bayer
  lossmult, rawnerf loss, coarse data loss, value + norm clipping."""
  models, _ = mods
  from multinerf_b200 import configs
  bundle = configs.bundle_llff_raw()
  bundle.model.num_prop_samples = bundle.model.num_nerf_samples = 32
  bundle.nerf_mlp.net_width, bundle.nerf_mlp.bottleneck_width, bundle.nerf_mlp.net_width_viewdirs = 128, 64, 64
  bundle.config.grad_max_norm = 0.0
  bundle.config.grad_max_val = 0.0
  B, S = 192, 32
  f = np.float32
  rng = np.random.default_rng(21)
  rays = raw_rays(rng, B)
  target = (rng.uniform(0, 1, (B, 3)) ** 2).astype(f)
  model, variables = models.construct_model(8, rays, bundle)
  tree = model.export_flax()
  tree['exposure_scaling_offsets']['embedding'] = rng.normal(size=(1000, 3)).astype(f) * 0.1
  variables = model.init(flax_params=tree)
  rand = {'jitter': [torch.tensor(rng.uniform(0, 1, (B, S)).astype(f)) for _ in range(2)],
          'density_noise': [torch.tensor(rng.normal(size=(B, S)).astype(f)) for _ in range(2)]}
  t = train_step(model, variables, bundle, rays, target, rand, 0.3)
  close(t.stats['mses'], t.stats_o['mses'].detach(), atol=2e-3, rtol=3e-2, msg='mses')
  lo = float(t.stats_o['loss'].detach())
  assert abs(t.stats['loss'] - lo) < 3e-2 * max(1.0, abs(lo)), (t.stats['loss'], lo)
  exposure = ('exposure_scaling_offsets', 'embedding')
  report, zero = grad_report(model, t.grads_o, [exposure] + mlp_leaves(model, modules=['NerfMLP_0']))
  assert not zero, zero
  assert report.pop(exposure)[0] < 0.05
  a = model.export_grads_flax()['exposure_scaling_offsets']['embedding']
  assert float(np.abs(a.reshape(-1, 3)[0]).max()) == 0.0      # index 0 is pinned (mask = idx > 0)
  assert not beyond(report, 0.15, 0.99), beyond(report, 0.15, 0.99)


def test_refnerf_forward_and_train_step_vs_oracle(mods):
  """BASELINE config 3 (blender_refnerf.gin) at reduced size: IDE of reflected directions, predicted
  and density-gradient normals (forward-mode tangent chain), diffuse + tinted specular colour,
  n.v, 6-layer view MLP with a skip connection, orientation + predicted-normal losses."""
  models, _ = mods
  bundle = mini_refnerf()
  bundle.config.grad_max_norm = 0.0
  B, S = 96, 16
  rays, rng = synth_rays(7, B, 2.0, 6.0, unit_cube=False)
  target = rng.uniform(0, 1, (B, 3)).astype(np.float32)
  model, variables = models.construct_model(9, rays, bundle)
  rand = level_jitter(rng, bundle, B)

  def normals(i, st, h):
    close(st.normals_pred.cpu().view(B, S, 3), h['normals_pred'], atol=3e-2, rtol=0, msg='normals_pred')
    # density normals: bf16 tangent chain vs fp32 autograd of the bf16-emulated forward
    cosn = (st.normals.cpu().view(B, S, 3) * h['normals']).sum(-1)
    assert float((cosn > 0.98).float().mean()) > 0.97, float((cosn > 0.98).float().mean())
    close(st.roughness.cpu().view(B, S, 1), h['roughness'], atol=2e-2, rtol=0, msg='roughness')
  rend_o, _ = pinned_forward(model, bundle, rays, rand, dens=(0.08, 4e-3), pixel=1.5e-2, samples=4e-2, level=normals)
  rend, hist = model(rand, rays, 0.5, True)
  for k in ['normals', 'normals_pred', 'roughness']:
    assert k in rend[-1] and hist[-1][k] is not None
  close(rend[-1]['rgb'], rend_o[-1]['rgb'], atol=3e-2, rtol=0, msg='final pixel end-to-end')
  # ---- one train step
  t = train_step(model, variables, bundle, rays, target, rand, 0.5)
  close(t.stats['mses'], t.stats_o['mses'].detach(), atol=2e-3, rtol=3e-2, msg='mses')
  for k in ['orientation', 'predicted_normals']:
    lo = float(t.stats_o['losses'][k].detach())
    assert abs(t.stats['losses'][k] - lo) < 0.05 * abs(lo) + 1e-7, (k, t.stats['losses'][k], lo)
  report, zero = grad_report(model, t.grads_o, mlp_leaves(model, modules=['NerfMLP_0']))
  assert not zero, zero
  bad = beyond(report, 0.2, 0.98)
  assert not bad, (bad, report)


def test_weight_decay_random_background_and_bottleneck_noise(mods):
  """Smaller switches of the path: weight_decay_mults (train_utils.py:304-309), random background
  colours (models.py:240-254) and bottleneck noise (models.py:529-533) against the oracle."""
  models, _ = mods
  bundle = mini360()
  bundle.config.grad_max_norm = 0.0
  bundle.config.weight_decay_mults = {'NerfMLP_0': 1e-3, 'PropMLP_0/Dense_0': 1e-2}
  bundle.model.bg_intensity_range = (0.2, 0.9)
  bundle.nerf_mlp.bottleneck_noise = 0.3
  B = 128
  rays, rng = synth_rays(13, B, 0.2, 1e6)
  target = rng.uniform(0, 1, (B, 3)).astype(np.float32)
  model, variables = models.construct_model(14, rays, bundle)
  S = [32, 32, 16]
  rand = {'jitter': [torch.tensor(rng.uniform(0, 1, (B, 1)).astype(np.float32)) for _ in S],
          'bg': [torch.tensor(rng.uniform(0, 1, (B, 3)).astype(np.float32)) for _ in S],
          'bottleneck_noise': [torch.tensor(rng.normal(size=(B, s, 64)).astype(np.float32)) for s in S]}
  # deterministic render: midpoint background
  rend_o, _ = o_models.model_apply(torch_tree(model.export_flax()), bundle, bases(model), oracle_rays(rays), 0.5,
                                   False, rand=None, bf16=True)
  rend, _ = model(None, rays, 0.5, False)
  close(rend[0]['rgb'], rend_o[0]['rgb'].detach(), atol=1e-2, rtol=0, msg='midpoint background')
  t = train_step(model, variables, bundle, rays, target, rand, 0.5, use_graph=True)   # falls back to eager
  close(t.stats['mses'], t.stats_o['mses'].detach(), atol=3e-3, rtol=3e-2, msg='mses (random bg)')
  keys = [('NerfMLP_0', 'Dense_3', 'kernel'), ('PropMLP_0', 'Dense_0', 'kernel'), ('PropMLP_0', 'Dense_1', 'kernel')]
  report, zero = grad_report(model, t.grads_o, keys)
  assert not zero and all(rel < 0.15 for rel, _ in report.values()), (report, zero)


def test_glo_embeddings_vs_oracle(mods):
  """configs/360_glo4.gin at reduced size: per-camera GLO vectors appended to the view-MLP input
  (models.py:101-110,565-569), their gradient scattered back into the embedding table."""
  models, _ = mods
  bundle = mini360()
  bundle.config.grad_max_norm = 0.0
  bundle.model.num_glo_features = 4
  bundle.model.num_glo_embeddings = 16
  B = 128
  rays, rng = synth_rays(17, B, 0.2, 1e6)
  rays.cam_idx = rng.integers(0, 16, (B, 1)).astype(np.int32)
  target = rng.uniform(0, 1, (B, 3)).astype(np.float32)
  model, variables = models.construct_model(18, rays, bundle)
  params0 = torch_tree(model.export_flax())
  assert params0['Embed_0']['embedding'].shape == (16, 4)
  assert params0['NerfMLP_0']['Dense_8']['kernel'].shape[0] == 64 + 27 + 4
  rand = level_jitter(rng, bundle, B)
  orays = oracle_rays(rays)
  # zero_glo=True (construct/eval default) vs False
  for zero_glo in [True, False]:
    rend_o, _ = o_models.model_apply(params0, bundle, bases(model), orays, 0.5, False, rand=rand, zero_glo=zero_glo,
                                     bf16=True)
    rend, _ = model(rand, rays, 0.5, False, zero_glo=zero_glo)
    close(rend[-1]['rgb'], rend_o[-1]['rgb'].detach(), atol=2e-2, rtol=0, msg=f'pixel zero_glo={zero_glo}')
  t = train_step(model, variables, bundle, rays, target, rand, 0.5)
  report, zero = grad_report(model, t.grads_o, [('Embed_0', 'embedding')])
  assert not zero and report[('Embed_0', 'embedding')][0] < 0.15, (report, zero)


def test_full_size_properties(mods):
  """BASELINE size (360.gin: 16384 rays x (64+64+32) samples, PropMLP 4x256, NerfMLP 8x1024), where the
  oracle is too slow: size-independent properties of the path.
    * every level: sdist sorted inside [0,1], weights >= 0 with sum <= 1, colours inside the padded
      sigmoid range, percentiles ordered, everything finite;
    * rays are independent: rendering the batch == rendering its two halves, bit for bit;
    * the loss is a mean over rays: grad(batch) == (grad(half 1) + grad(half 2)) / 2 up to bf16 noise."""
  models, train_utils = mods
  from multinerf_b200 import configs, utils
  bundle = configs.bundle_360()
  B = 16384
  rays, rng = synth_rays(21, B, 0.2, 1e6)
  model, variables = models.construct_model(3, rays, bundle)
  assert model.num_params() == 9007493
  rend, hist = model(None, rays, 1.0, True)
  torch.cuda.synchronize()
  S = [64, 64, 32]
  pad = bundle.nerf_mlp.rgb_padding
  for lvl, (r, h) in enumerate(zip(rend, hist)):
    sd, w = h['sdist'], h['weights']
    assert sd.shape == (B, S[lvl] + 1) and w.shape == (B, S[lvl])
    assert bool((sd[:, 1:] >= sd[:, :-1]).all()) and float(sd.min()) >= 0.0 and float(sd.max()) <= 1.0
    assert float(w.min()) >= 0.0 and float(w.sum(-1).max()) <= 1.0 + 1e-5
    assert bool(torch.isfinite(r['rgb']).all()) and float(r['rgb'].min()) >= -pad - 1e-6 and float(r['rgb'].max()) <= 1 + pad + 1e-6
    assert float(r['acc'].min()) >= 0.0 and float(r['acc'].max()) <= 1.0 + 1e-5
    assert bool((r['distance_percentile_5'] <= r['distance_median'] + 1e-6).all())
    assert bool((r['distance_median'] <= r['distance_percentile_95'] + 1e-6).all())
    assert bool(torch.isfinite(r['distance_mean']).all()) and bool(torch.isfinite(h['density']).all())
  full_rgb = rend[-1]['rgb'].clone()
  full_w = hist[-1]['weights'].clone()
  import dataclasses
  halves = []
  for sl in (slice(0, B // 2), slice(B // 2, B)):
    sub = utils.Rays(**{f.name: (None if getattr(rays, f.name) is None else getattr(rays, f.name)[sl])
                        for f in dataclasses.fields(rays)})
    r2, h2 = model(None, sub, 1.0, True)
    halves.append((r2[-1]['rgb'].clone(), h2[-1]['weights'].clone(), sub))
  assert torch.equal(torch.cat([halves[0][0], halves[1][0]]), full_rgb)
  assert torch.equal(torch.cat([halves[0][1], halves[1][1]]), full_w)

  # gradient of the mean loss = mean of the halves' gradients (same parameters, no optimizer step applied)
  target = rng.uniform(0, 1, (B, 3)).astype(np.float32)
  cfg = copy.deepcopy(bundle.config)
  cfg.lr_init = cfg.lr_final = 1e-30            # keep the parameters (and their bf16 copies) fixed
  jit = [torch.tensor(rng.uniform(0, 1, (B, 1)).astype(np.float32)) for _ in range(3)]
  step_fn = train_utils.create_train_step(model, cfg)
  state = train_utils.TrainState(variables)

  def grad_of(sl):
    sub = utils.Rays(**{f.name: (None if getattr(rays, f.name) is None else getattr(rays, f.name)[sl])
                        for f in dataclasses.fields(rays)})
    nonlocal state
    state, stats, _ = step_fn({'jitter': [j[sl] for j in jit]}, state, utils.Batch(rays=sub, rgb=target[sl]), None, 0.5)
    torch.cuda.synchronize()
    return model.params.grads.clone().double(), stats.materialize()['loss']

  g_full, l_full = grad_of(slice(0, B))
  g1, l1 = grad_of(slice(0, B // 2))
  g2, l2 = grad_of(slice(B // 2, B))
  g_sum = 0.5 * (g1 + g2)
  rel = float((g_full - g_sum).norm() / g_full.norm())
  assert rel < 2e-2, rel
  assert abs(l_full - 0.5 * (l1 + l2)) < 1e-4 * abs(l_full), (l_full, l1, l2)


@pytest.mark.parametrize('B', [1, 37, 130])
def test_ragged_batches_match_their_rows_in_a_full_batch(mods, B):
  """Ragged ray counts (sample rows not a multiple of any tile: TMA zero-fill / store clipping, the
  single-CTA GEMM variant, partial warps): the first B rays rendered alone == the same rays inside a
  256-ray batch, bit for bit; a train step on them stays finite."""
  models, train_utils = mods
  import dataclasses
  from multinerf_b200 import utils
  bundle = mini360()
  rays, rng = synth_rays(8, 256, 0.2, 1e6)
  model, variables = models.construct_model(2, rays, bundle)
  rend, _ = model(None, rays, 1.0, True)
  want = {k: rend[-1][k][:B].clone() for k in ('rgb', 'acc', 'distance_median')}
  sub = utils.Rays(**{f.name: (None if getattr(rays, f.name) is None else getattr(rays, f.name)[:B])
                      for f in dataclasses.fields(rays)})
  r2, h2 = model(None, sub, 1.0, True)
  for k, v in want.items():
    assert torch.equal(r2[-1][k], v), k
  assert h2[-1]['weights'].shape == (B, bundle.model.num_nerf_samples)
  step_fn = train_utils.create_train_step(model, bundle.config)
  state = train_utils.TrainState(variables)
  state, stats, _ = step_fn(None, state, utils.Batch(rays=sub, rgb=rng.uniform(0, 1, (B, 3)).astype(np.float32)), None, 0.3)
  torch.cuda.synchronize()
  assert np.isfinite(stats.materialize()['loss']) and bool(torch.isfinite(model.params.flat).all())


def test_empty_batch(mods):
  """Zero rays: every entry point returns without launching; outputs are empty with the right shapes."""
  models, _ = mods
  import dataclasses
  from multinerf_b200 import utils
  bundle = mini360()
  rays, _ = synth_rays(8, 4, 0.2, 1e6)
  model, _ = models.construct_model(2, rays, bundle)
  empty = utils.Rays(**{f.name: (None if getattr(rays, f.name) is None else getattr(rays, f.name)[:0])
                        for f in dataclasses.fields(rays)})
  rend, hist = model(None, empty, 1.0, True)
  assert rend[-1]['rgb'].shape == (0, 3) and hist[-1]['sdist'].shape == (0, bundle.model.num_nerf_samples + 1)


def _variant(name):
  b = mini360()
  m = b.model
  if name == 'samples_128_128_64':
    m.num_prop_samples, m.num_nerf_samples = 128, 64
  elif name == 'four_levels':
    m.num_levels = 4
  elif name == 'per_sample_jitter':
    m.single_jitter = False
  elif name == 'cylinder':
    m.ray_shape = 'cylinder'
  elif name == 'no_integration':
    # plain PE: without the Gaussian attenuation a random-init MLP of 2^11-frequency features is not a
    # smooth function of the sample positions, so the end-to-end comparison is only well conditioned at
    # low degrees
    m.disable_integration = True
    b.prop_mlp.max_deg_point = b.nerf_mlp.max_deg_point = 5
  elif name == 'no_dilation_padded':
    m.dilation_multiplier, m.dilation_bias, m.resample_padding = 0.0, 0.0, 0.01
  elif name == 'gpu_resampling_flag':
    m.use_gpu_resampling = True
  elif name == 'piecewise_raydist':
    m.raydist_fn = 'piecewise'
  elif name == 'translucent_white_bg':
    m.opaque_background, m.bg_intensity_range = False, (1.0, 1.0)
  elif name == 'coarse_data_loss_mse':
    b.config.data_coarse_loss_mult, b.config.data_loss_type = 0.1, 'mse'
  # ---- MLP switches
  elif name == 'trunk_skip_every_2':            # several skip concatenations in both trunks
    b.nerf_mlp.skip_layer, b.prop_mlp.skip_layer, b.prop_mlp.net_depth = 2, 2, 4
  elif name == 'deep_view_mlp':                 # view MLP with its own skip (models.py:575-580)
    b.nerf_mlp.net_depth_viewdirs, b.nerf_mlp.skip_layer_dir = 4, 2
  elif name == 'degrees_2_to_9_view_deg_2':
    for c in (b.nerf_mlp, b.prop_mlp):
      c.min_deg_point, c.max_deg_point = 2, 9
    b.nerf_mlp.deg_view = 2
  elif name == 'octahedron_basis':
    for c in (b.nerf_mlp, b.prop_mlp):
      c.basis_shape, c.basis_subdivisions = 'octahedron', 1
  elif name == 'icosahedron_1_basis':
    for c in (b.nerf_mlp, b.prop_mlp):
      c.basis_subdivisions = 1
  elif name == 'rgb_head_settings':
    b.nerf_mlp.rgb_premultiplier, b.nerf_mlp.rgb_bias, b.nerf_mlp.rgb_padding = 2.0, -0.5, 0.0
    b.nerf_mlp.density_bias, b.prop_mlp.density_bias = 0.5, 0.5
  elif name == 'glorot_uniform_init':
    b.nerf_mlp.weight_init = b.prop_mlp.weight_init = 'glorot_uniform'
  elif name == 'single_mlp':
    m.single_mlp = True
  else:
    raise KeyError(name)
  return b


@pytest.mark.parametrize('name', ['samples_128_128_64', 'four_levels', 'per_sample_jitter', 'cylinder',
                                  'no_integration', 'no_dilation_padded', 'gpu_resampling_flag',
                                  'piecewise_raydist', 'translucent_white_bg', 'coarse_data_loss_mse',
                                  'trunk_skip_every_2', 'deep_view_mlp', 'degrees_2_to_9_view_deg_2',
                                  'octahedron_basis', 'icosahedron_1_basis', 'rgb_head_settings',
                                  'glorot_uniform_init', 'single_mlp'])
def test_config_variants_vs_oracle(mods, name):
  """Model / Config switches away from the shipped 360.gin values, each against the oracle: rendered
  pixels and level-0 sample positions of a randomized forward pass, then loss, per-level MSEs and the
  direction of every layer's gradient for one train step."""
  models, _ = mods
  bundle = _variant(name)
  bundle.config.grad_max_norm = 0.0
  B = 96
  near, far = (0.5, 30.0) if name == 'piecewise_raydist' else (0.2, 1e6)
  rays, rng = synth_rays(31, B, near, far)
  target = rng.uniform(0, 1, (B, 3)).astype(np.float32)
  model, variables = models.construct_model(6, rays, bundle)
  rand = level_jitter(rng, bundle, B)
  with torch.no_grad():
    rend_o, hist_o = o_models.model_apply(torch_tree(model.export_flax()), bundle, bases(model), oracle_rays(rays),
                                          0.5, True, rand=rand, bf16=True)
  rend, hist = model(rand, rays, 0.5, True)
  torch.cuda.synchronize()
  assert len(rend) == bundle.model.num_levels
  close(hist[0]['sdist'], hist_o[0]['sdist'], atol=1e-6, rtol=1e-6, msg='level-0 sdist')
  close(rend[-1]['rgb'], rend_o[-1]['rgb'], atol=2e-2, rtol=0, msg='final pixel')
  close(rend[-1]['acc'], rend_o[-1]['acc'], atol=2e-2, rtol=0, msg='final acc')
  t = train_step(model, variables, bundle, rays, target, rand, 0.5)
  close(t.stats['mses'], t.stats_o['mses'].detach(), atol=2e-3, rtol=3e-2, msg='mses')
  lo = float(t.stats_o['loss'].detach())
  assert abs(t.stats['loss'] - lo) < 3e-2 * max(1.0, abs(lo)), (t.stats['loss'], lo)
  report, zero = grad_report(model, t.grads_o, mlp_leaves(model))
  assert not any(zero.values()), zero
  assert not beyond(report, 0.25, 0.98), (name, beyond(report, 0.25, 0.98))


def _refnerf_variant(name):
  b = mini_refnerf()
  c, n = b.config, b.nerf_mlp
  if name == 'pred_normals_only':
    n.disable_density_normals = True
    c.predicted_normal_loss_mult = c.predicted_normal_coarse_loss_mult = 0.0
  elif name == 'density_normals_only':
    n.enable_pred_normals = False
    c.orientation_loss_target = 'normals'
    c.predicted_normal_loss_mult = c.predicted_normal_coarse_loss_mult = 0.0
  elif name == 'reflections_with_plain_pe':
    n.use_directional_enc, n.deg_view = False, 4
  elif name == 'no_diffuse_no_tint_no_ndotv':
    n.use_diffuse_color = n.use_specular_tint = n.use_n_dot_v = False
  else:
    raise KeyError(name)
  return b


@pytest.mark.parametrize('name', ['pred_normals_only', 'density_normals_only', 'reflections_with_plain_pe',
                                  'no_diffuse_no_tint_no_ndotv'])
def test_refnerf_variants_vs_oracle(mods, name):
  """Ref-NeRF switches one at a time (models.py:473-604): which normals feed the reflection and the
  orientation loss, IDE vs plain PE of the (reflected) direction, the colour-composition terms."""
  models, _ = mods
  bundle = _refnerf_variant(name)
  bundle.config.grad_max_norm = 0.0
  B = 96
  rays, rng = synth_rays(17, B, 2.0, 6.0, unit_cube=False)
  target = rng.uniform(0, 1, (B, 3)).astype(np.float32)
  model, variables = models.construct_model(5, rays, bundle)
  rand = level_jitter(rng, bundle, B)
  rend_o, hist_o = o_models.model_apply(torch_tree(model.export_flax()), bundle, bases(model), oracle_rays(rays), 0.5,
                                        True, rand=rand, bf16=True)
  rend, hist = model(rand, rays, 0.5, True)
  torch.cuda.synchronize()
  close(rend[-1]['rgb'], rend_o[-1]['rgb'].detach(), atol=3e-2, rtol=0, msg='final pixel')
  t = train_step(model, variables, bundle, rays, target, rand, 0.5)
  close(t.stats['mses'], t.stats_o['mses'].detach(), atol=2e-3, rtol=3e-2, msg='mses')
  lo = float(t.stats_o['losses']['orientation'].detach())
  assert abs(t.stats['losses']['orientation'] - lo) < 0.05 * abs(lo) + 1e-7, (t.stats['losses']['orientation'], lo)
  report, zero = grad_report(model, t.grads_o, mlp_leaves(model, modules=['NerfMLP_0']))
  assert not any(zero.values()), zero
  # with density-gradient normals alone, every colour gradient reaches the first layers through the
  # bf16 forward-mode tangent streams as well: measured 0.24 / 0.971 on Dense_0
  bad = beyond(report, 0.3, 0.96) if name == 'density_normals_only' else beyond(report, 0.25, 0.98)
  assert not bad, bad
  if name == 'reflections_with_plain_pe':
    broken = _refnerf_variant(name)
    broken.nerf_mlp.use_directional_enc, broken.nerf_mlp.use_reflections = True, False
    with pytest.raises(ValueError):
      models.Model(broken)


def _family(name, rng, B):
  """(bundle, rays) of a reduced-size model family with per-step varying inputs."""
  from multinerf_b200 import configs
  if name == 'rawnerf':
    bundle = configs.bundle_llff_raw()
    bundle.model.num_prop_samples = bundle.model.num_nerf_samples = 32
    bundle.nerf_mlp.net_width, bundle.nerf_mlp.bottleneck_width, bundle.nerf_mlp.net_width_viewdirs = 128, 64, 64
    bundle.nerf_mlp.density_noise = 0.0           # the graph path refreshes jitter only from a generator or dict
    return bundle, raw_rays(rng, B, radii_first=True)
  if name == 'refnerf':
    bundle = mini_refnerf()
    rays, _ = synth_rays(int(rng.integers(1 << 30)), B, 2.0, 6.0, unit_cube=False)
    return bundle, rays
  if name == 'glo':
    bundle = mini360()
    bundle.model.num_glo_features, bundle.model.num_glo_embeddings = 4, 16
    rays, _ = synth_rays(int(rng.integers(1 << 30)), B, 0.2, 1e6)
    rays.cam_idx = rng.integers(0, 16, (B, 1)).astype(np.int32)
    return bundle, rays
  raise KeyError(name)


@pytest.mark.parametrize('family', ['rawnerf', 'refnerf', 'glo'])
def test_cuda_graph_matches_eager_other_families(mods, family):
  """Graph capture of the step for the other model families (exposure-offset and GLO scatter-adds, the
  Ref-NeRF tangent chain and reflection stage): five steps with changing rays, targets, jitter,
  train_frac and learning rate track the eager run."""
  models, train_utils = mods
  B, steps = 192, 5
  rng = np.random.default_rng(77)
  batches = []
  for _ in range(steps):
    bundle, rays = _family(family, rng, B)
    rand = level_jitter(rng, bundle, B)
    batches.append((rays, rng.uniform(0, 1, (B, 3)).astype(np.float32), rand))
  graph_matches_eager(models, train_utils, bundle, batches, 6)
