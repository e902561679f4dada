"""Train steps in several forward/backward passes (Config.train_chunk_size) on the GPU.  Needs an H100.

A step over B rays in B / C passes must compute what the one-pass step computes: every per-ray and per-sample
quantity depends on its own ray only, and the loss normalisers, the random draws and the robustnerf quantile are the
whole batch's.  So the per-sample values of a pass equal the matching rows of the one-pass step bit for bit, and the
gradients and loss statistics, which are sums over rays, agree up to the order of their fp32 reductions.

The mini configurations keep every trunk under 256 wide, so the chained trunk (csrc/chain.cu) is never taken and the
one-pass and the chunked steps both run the per-layer path at every pass size.
"""
import numpy as np
import pytest
import torch

from model_parity import (beyond, grad_report, graph_matches_eager, level_jitter, mini360, mini_refnerf, mlp_leaves,
                          raw_rays, synth_rays, train_loop_bundle, train_step)
from util import close, golden

pytestmark = pytest.mark.gpu
F32 = np.float32


@pytest.fixture(scope='module')
def mods():
  from multinerf_b200 import lib, models, train_utils
  lib.require_device()
  return models, train_utils


# ------------------------------------------------------------------ cases

def _robust(b, p=8, inner=4):
  c = b.config
  c.data_loss_type, c.patch_size, c.enable_robustnerf_loss = 'robustnerf', p, True
  c.robustnerf_inlier_quantile, c.robustnerf_inner_patch_size = 0.8, inner
  return b


def _case(name):
  """(bundle, batch rays, target, rand, B, cameras, flax tree edit) of one configuration."""
  from multinerf_b200 import configs, utils
  edit, cameras = None, None
  if name == 'raw':
    b = configs.bundle_llff_raw()
    b.model.num_prop_samples = b.model.num_nerf_samples = 32
    b.nerf_mlp.net_width, b.nerf_mlp.bottleneck_width, b.nerf_mlp.net_width_viewdirs = 128, 64, 64
    B = 192
    rng = np.random.default_rng(21)
    rays = raw_rays(rng, B)
    target = (rng.uniform(0, 1, (B, 3)) ** 2).astype(F32)
    rand = {'jitter': [torch.tensor(rng.uniform(0, 1, (B, 32)).astype(F32)) for _ in range(2)],
            'density_noise': [torch.tensor(rng.normal(size=(B, 32)).astype(F32)) for _ in range(2)]}
    offsets = rng.normal(size=(1000, 3)).astype(F32) * 0.1

    def edit(tree):
      tree['exposure_scaling_offsets']['embedding'] = offsets
    return b, rays, target, rand, B, None, edit
  if name == 'refnerf':
    b = mini_refnerf()
    B = 192
    rays, rng = synth_rays(7, B, 2.0, 6.0, unit_cube=False)
  else:
    b = _robust(mini360()) if name == 'robust' else mini360()
    B = 256
    rays, rng = synth_rays(13, B, 0.2, 1e6)
    if name == 'glo':
      b.model.num_glo_features, b.model.num_glo_embeddings = 4, 16
      rays.cam_idx = rng.integers(0, 16, (B, 1)).astype(np.int32)
    if name == 'cast':
      G = golden('camera')
      cameras = (G['pixtocams'], G['camtoworlds'], None, None)
      b.config.cast_rays_in_train_step = True
      meta = lambda v: np.full((B, 1), v, F32)
      rays = utils.Pixels(pix_x_int=rng.integers(0, 160, B).astype(np.int32),
                          pix_y_int=rng.integers(0, 120, B).astype(np.int32), lossmult=meta(1), near=meta(0.2),
                          far=meta(1e6), cam_idx=rng.integers(0, G['camtoworlds'].shape[0], (B, 1)).astype(np.int32))
  rand = level_jitter(rng, b, B)
  return b, rays, rng.uniform(0, 1, (B, 3)).astype(F32), rand, B, cameras, edit


CASES = ['mini360', 'refnerf', 'raw', 'glo', 'robust', 'cast']


def _run(mods, name, passes, loss_threshold=1.0, use_graph=False):
  """One step of case `name` in `passes` passes from the case's initial weights: (model, stats, C)."""
  models, train_utils = mods
  from multinerf_b200 import utils
  b, rays, target, rand, B, cameras, edit = _case(name)
  C = B // passes
  b.config.batch_size = B
  b.config.train_chunk_size = 0 if passes == 1 else C
  model, variables = models.construct_model(9, utils.dummy_rays(include_exposure_idx=name == 'raw',
                                                                include_exposure_values=True), b)
  if edit is not None:
    tree = model.export_flax()
    edit(tree)
    variables = model.init(flax_params=tree)
  step_fn = train_utils.create_train_step(model, b.config, use_graph=use_graph)
  extra = (loss_threshold,) if name == 'robust' else ()
  _, stats, _ = step_fn(rand, train_utils.TrainState(variables), utils.Batch(rays=rays, rgb=target), cameras, 0.5,
                        *extra)
  torch.cuda.synchronize()
  return model, stats, C


def _levels(model, C):
  """The level states of pass shape C, level by level."""
  return [st for key, st in sorted(model._levels.items(), key=lambda kv: kv[0][0]) if key[2] == C]


def _leaves(tree, prefix=()):
  for k, v in tree.items():
    if isinstance(v, dict):
      yield from _leaves(v, prefix + (k,))
    else:
      yield prefix + (k,), np.asarray(v, np.float64)


def _grad_rel(a, b):
  """Per gradient leaf, ||a - b|| / ||b|| (0 where both are zero)."""
  lb = dict(_leaves(b))
  out = {}
  for k, va in _leaves(a):
    nb = np.linalg.norm(lb[k])
    d = np.linalg.norm(va - lb[k])
    out[k] = 0.0 if d == 0 else d / max(nb, 1e-30)
  return out


def _stat_values(s):
  v = dict(s['losses'])
  v.update({f'mse{i}': float(m) for i, m in enumerate(s['mses'])})
  return v


def _threshold(mods):
  """A robustnerf threshold inside the case's error range: the next threshold of a first one-pass step."""
  _, stats, _ = _run(mods, 'robust', 1)
  return float(stats.device_loss_threshold())


@pytest.mark.parametrize('name', CASES)
def test_chunked_step_matches_one_pass(mods, name):
  thr = _threshold(mods) if name == 'robust' else 1.0
  m1, s1, B = _run(mods, name, 1, thr)
  m1b, s1b, _ = _run(mods, name, 1, thr)
  g1, g1b = m1.export_grads_flax(), m1b.export_grads_flax()
  noise = _grad_rel(g1b, g1)
  st1 = s1.materialize()
  whole = _levels(m1, B)
  for passes in (2, 4):
    mk, sk, C = _run(mods, name, passes, thr)
    # 1. per-sample values of the last pass == rows [B - C, B) of the one-pass step, bit for bit
    part = _levels(mk, C)
    assert len(part) == len(whole) > 0
    for i, (a, w) in enumerate(zip(part, whole)):
      for key in ('sdist', 'raw_density', 'd_raw_density', 'd_raw_rgb'):
        x, y = getattr(a, key), getattr(w, key)
        if y is None:
          continue
        assert torch.equal(x, y[B - C:]), (name, passes, i, key, float((x - y[B - C:]).abs().max()))
      assert torch.equal(a.comp['weights'], w.comp['weights'][B - C:]), (name, passes, i, 'weights')
    # 2. reductions over rays agree to fp32 order noise
    rel = _grad_rel(mk.export_grads_flax(), g1)
    worst = max(rel.items(), key=lambda kv: kv[1])
    print(f'{name} x{passes}: worst gradient leaf {worst}, one-pass run-to-run {max(noise.values()):.2e}')
    assert worst[1] <= 1e-5, (worst, max(noise.values()))
    if name == 'glo':
      assert ('Embed_0', 'embedding') in rel
    if name == 'raw':
      assert rel[('exposure_scaling_offsets', 'embedding')] <= 1e-5
    stk = sk.materialize()
    for k, v in _stat_values(st1).items():
      got = _stat_values(stk)[k]
      assert abs(got - v) <= 1e-5 * abs(v) + 1e-12, (name, passes, k, got, v)
    if name == 'robust':
      # 3. the next threshold bit for bit, the mask means within 1 ulp
      t1, tk = s1.device_loss_threshold().cpu(), sk.device_loss_threshold().cpu()
      assert t1.view(torch.int32) == tk.view(torch.int32), (float(t1), float(tk))
      for k in ('is_inlier_loss', 'has_inlier_neighbors', 'is_inlier_patch', 'mask'):
        a, b = np.float32(st1[k]), np.float32(stk[k])
        assert abs(int(a.view(np.int32)) - int(b.view(np.int32))) <= 1, (k, a, b)
      assert 0.0 < st1['mask'] < 1.0


def test_chunked_refnerf_step_vs_oracle(mods):
  """4. A Ref-NeRF step in two passes against the oracle's one-pass step, at the bounds of the one-pass Ref-NeRF
  test (test_gpu_model.py): mses, both normal losses, and every NerfMLP kernel gradient (single_mlp)."""
  models, _ = mods
  bundle = mini_refnerf()
  bundle.config.grad_max_norm = 0.0
  B = 96
  bundle.config.batch_size, bundle.config.train_chunk_size = B, B // 2
  rays, rng = synth_rays(7, B, 2.0, 6.0, unit_cube=False)
  target = rng.uniform(0, 1, (B, 3)).astype(F32)
  model, variables = models.construct_model(9, rays, bundle)
  rand = level_jitter(rng, bundle, B)
  t = train_step(model, variables, bundle, rays, target, rand, 0.5)
  close(t.stats['mses'], t.stats_o['mses'].detach(), atol=2e-3, rtol=3e-2, msg='mses')
  for k in ['orientation', 'predicted_normals']:
    lo = float(t.stats_o['losses'][k].detach())
    assert abs(t.stats['losses'][k] - lo) < 0.05 * abs(lo) + 1e-7, (k, t.stats['losses'][k], lo)
  report, zero = grad_report(model, t.grads_o, mlp_leaves(model, modules=['NerfMLP_0']))
  assert not zero, zero
  bad = beyond(report, 0.2, 0.98)
  assert not bad, (bad, report)


def _graph_launches(mods, bundle, rays, target, rand, steps=3):
  models, train_utils = mods
  from multinerf_b200 import utils
  model, variables = models.construct_model(6, rays, bundle)
  step_fn = train_utils.create_train_step(model, bundle.config, use_graph=True)
  state = train_utils.TrainState(variables)
  for i in range(steps):
    state, stats, _ = step_fn(rand, state, utils.Batch(rays=rays, rgb=target), None, 0.5)
  torch.cuda.synchronize()
  assert step_fn.graph_info['state'] == 2
  return step_fn.graph_info['launches'], variables.flat.clone()


def test_graph_replay_and_launch_counts(mods):
  """5. A chunked step replayed from one CUDA graph tracks the eager step, and it launches each pass's kernels once
  per pass plus the optimizer's once.  6. train_chunk_size equal to the batch is the one-pass step."""
  models, train_utils = mods
  B = 256
  batches = []
  for i in range(4):
    rays, rng = synth_rays(50 + i, B, 0.2, 1e6)
    batches.append((rays, rng.uniform(0, 1, (B, 3)).astype(F32), level_jitter(rng, mini360(), B)))
  bundle = mini360()
  bundle.config.batch_size, bundle.config.train_chunk_size = B, B // 2
  graph_matches_eager(models, train_utils, bundle, batches, 6)

  rays, target, rand = batches[0]
  counts, flats = {}, {}
  for chunk in (0, B, B // 2, B // 4):
    b = mini360()
    b.config.batch_size, b.config.train_chunk_size = B, chunk
    counts[chunk], flats[chunk] = _graph_launches(mods, b, rays, target, rand)
  _, flat0b = _graph_launches(mods, mini360(), rays, target, rand)
  per_pass = counts[B // 2] - counts[0]
  optimizer = counts[0] - per_pass
  print(f'launches: {counts}; per pass {per_pass}, optimizer {optimizer}')
  assert per_pass > 20 and optimizer > 0
  assert counts[B // 4] == 4 * per_pass + optimizer, counts
  assert counts[B] == counts[0], counts
  # the same launches: parameters agree as closely as two one-pass runs do (bit for bit unless the weight-gradient
  # split-K atomics reorder)
  d_same = float((flats[B] - flats[0]).abs().max())
  d_noise = float((flat0b - flats[0]).abs().max())
  assert d_same <= d_noise, (d_same, d_noise)


def _bytes(tree):
  if isinstance(tree, (list, tuple)):
    return sum(_bytes(t) for t in tree)
  if isinstance(tree, dict):
    return sum(_bytes(t) for t in tree.values())
  if tree is None:
    return 0
  return int(np.asarray(tree).nbytes) if not torch.is_tensor(tree) else tree.numel() * tree.element_size()


def test_peak_memory_follows_the_chunk(mods):
  """7. blender_256.gin at 16384 rays in 2048-ray passes peaks within 1.1x of a 2048-ray one-pass step, plus the
  whole batch's inputs (rays on the device with their flat near/far/radii, and the targets)."""
  models, train_utils = mods
  from multinerf_b200 import configs, utils
  import dataclasses
  peaks = {}
  inputs = 0
  for B, chunk in ((2048, 0), (16384, 2048)):
    b = configs.bundle_blender_256()
    b.config.batch_size, b.config.train_chunk_size = B, chunk
    rays, rng = synth_rays(3, B, 2.0, 6.0, unit_cube=False)
    target = rng.uniform(0, 1, (B, 3)).astype(F32)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    model, variables = models.construct_model(2, rays, b)
    step_fn = train_utils.create_train_step(model, b.config)
    state = train_utils.TrainState(variables)
    for _ in range(2):
      state, stats, _ = step_fn(None, state, utils.Batch(rays=rays, rgb=target), None, 0.5)
    torch.cuda.synchronize()
    peaks[B] = torch.cuda.max_memory_allocated() - base
    if chunk:
      inputs = sum(_bytes(getattr(rays, f.name)) for f in dataclasses.fields(rays)) + 3 * 4 * B + _bytes(target)
    del model, variables, state, step_fn, stats
  print(f'peak: one pass of 2048 rays {peaks[2048] / 2**20:.1f} MiB, 16384 rays in 8 passes '
        f'{peaks[16384] / 2**20:.1f} MiB, whole-batch inputs {inputs / 2**20:.2f} MiB')
  assert peaks[16384] <= 1.1 * peaks[2048] + inputs, peaks


def test_train_loop_with_gin_bound_chunks(mods, tmp_path):
  """8. A few steps of the training loop on the synthetic scene with train_chunk_size bound by gin."""
  from multinerf_b200 import checkpoints, configs, train_loop
  ck = str(tmp_path / 'ckpt')
  b = train_loop_bundle(8, ckpt=ck)
  b.config.checkpoint_every = 8
  b = configs.parse_gin('Config.train_chunk_size = 512\n', bundle=b)
  assert b.config.train_chunk_size == 512 and b.config.batch_size == 2048
  _, state, hist = train_loop.train(b, train_loop.SyntheticScene(b.config), log=lambda s: None)
  assert state.step == 8
  assert all(np.isfinite(h['loss']) for h in hist)
  assert checkpoints.latest_checkpoint(ck).endswith('checkpoint_8')


def test_generator_step_equals_explicit_draws(mods):
  """9. An eager one-pass step driven by a seeded torch.Generator draws, per level and in this order, the jitter, the
  bottleneck noise, the density noise and the background colours: the same step given those draws explicitly, taken
  from a copy of the generator, computes the same per-sample values bit for bit and consumes no other draw."""
  models, train_utils = mods
  from multinerf_b200 import utils
  B = 256
  b = mini360()
  b.prop_mlp.density_noise = b.nerf_mlp.density_noise = 1.0
  b.nerf_mlp.bottleneck_noise = 1.0
  b.model.bg_intensity_range = (0.0, 1.0)
  b.config.batch_size = B
  m = b.model
  rays, rng = synth_rays(17, B, 0.2, 1e6)
  target = rng.uniform(0, 1, (B, 3)).astype(F32)
  gen = torch.Generator(device='cuda').manual_seed(23)
  copy = torch.Generator(device='cuda')
  copy.set_state(gen.get_state())
  rand = {'jitter': [], 'bottleneck_noise': [], 'density_noise': [], 'bg': []}
  for i in range(m.num_levels):
    fine = i == m.num_levels - 1
    S = m.num_nerf_samples if fine else m.num_prop_samples
    rand['jitter'].append(torch.rand((B,) if m.single_jitter else (B, S), device='cuda', generator=copy))
    rand['bottleneck_noise'].append(
        torch.randn(B * S, b.nerf_mlp.bottleneck_width, device='cuda', generator=copy) if fine else None)
    rand['density_noise'].append(torch.randn(B, S, device='cuda', generator=copy))
    rand['bg'].append(torch.rand(B, 3, device='cuda', generator=copy))
  runs = []
  for draws in (gen, rand):
    model, variables = models.construct_model(9, rays, b)
    step_fn = train_utils.create_train_step(model, b.config)
    step_fn(draws, train_utils.TrainState(variables), utils.Batch(rays=rays, rgb=target), None, 0.5)
    torch.cuda.synchronize()
    runs.append(model)
  assert torch.equal(gen.get_state(), copy.get_state())
  gs, es = _levels(runs[0], B), _levels(runs[1], B)
  assert len(gs) == len(es) == m.num_levels
  for i, (g, e) in enumerate(zip(gs, es)):
    assert g.bneck_noise is not None if i == m.num_levels - 1 else g.bneck_noise is None, i
    assert g.noise is not None and g.bg_rgb is not None, i
    for key in ('sdist', 'raw_density', 'd_raw_density'):
      assert torch.equal(getattr(g, key), getattr(e, key)), (i, key)
    assert torch.equal(g.comp['weights'], e.comp['weights']), (i, 'weights')


def test_validation_before_device_work(mods):
  models, train_utils = mods
  from multinerf_b200 import utils
  b = mini360()
  b.config.batch_size, b.config.train_chunk_size = 256, 96
  model, _ = models.construct_model(1, utils.dummy_rays(), b)
  with pytest.raises(ValueError, match='train_chunk_size'):
    train_utils.create_train_step(model, b.config)
  b.config.batch_size = 192
  step_fn = train_utils.create_train_step(model, b.config)
  rays, rng = synth_rays(2, 256, 0.2, 1e6)
  with pytest.raises(ValueError, match='train_chunk_size'):     # a batch of another size than the config's
    step_fn(None, train_utils.TrainState(model.params), utils.Batch(rays=rays, rgb=np.zeros((256, 3), F32)),
            None, 0.5)
  assert model.params.step == 0
