"""RobustNeRF on the GPU (data_loss_type 'robustnerf', internal/robustnerf.py, train_utils.py:104-108,
train.py:109-129): the mask and quantile kernels bit for bit against the oracle, the masked compositing
backward against oracle autograd, the train step against the oracle at mini and full width, graph replay with
the threshold fed back on the device, and the training loop.  Needs an H100."""
import numpy as np
import pytest
import torch

from composite_ref import CFG, oracle_composite
from model_parity import (bases, beyond, grad_report, mini360, mlp_leaves, oracle_rays, synth_rays, torch_tree,
                          train_loop_bundle, train_step)
from oracle import o_robust, o_train
from util import close, golden, kernel_rays

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def mods():
  from multinerf_b200 import lib, models, ops, train_utils
  lib.require_device()
  return models, ops, train_utils


def _cfg(p, inner, f, q=0.5, qs=0.5, qp=0.5, enable=True):
  from multinerf_b200 import configs
  return configs.Config(data_loss_type='robustnerf', patch_size=p, robustnerf_inner_patch_size=inner,
                        robustnerf_smoothed_filter_size=f, robustnerf_inlier_quantile=q,
                        robustnerf_smoothed_inlier_quantile=qs, robustnerf_inner_patch_inlier_quantile=qp,
                        enable_robustnerf_loss=enable)


def _desc(ops, B, cfg):
  return ops.robust_desc(B, patch_size=cfg.patch_size, inner_patch_size=cfg.robustnerf_inner_patch_size,
                         filter_size=cfg.robustnerf_smoothed_filter_size,
                         smoothed_inlier_quantile=cfg.robustnerf_smoothed_inlier_quantile,
                         inner_patch_inlier_quantile=cfg.robustnerf_inner_patch_inlier_quantile,
                         enable=cfg.enable_robustnerf_loss)


def _bits(x):
  return np.asarray(x.detach().cpu() if torch.is_tensor(x) else x, np.float32).view(np.uint32)


def _run_mask(ops, rgb, target, thr, cfg, counts):
  """GPU mask + stats row for [n, p, p, 3] inputs; returns (mask [n,p,p,1], error [n,p,p,1], stats dict)."""
  from multinerf_b200 import train_utils
  shape = rgb.shape
  B = shape[0] * shape[1] * shape[2]
  row = torch.zeros(8, device='cuda')
  thr_dev = torch.tensor([float(thr)], dtype=torch.float32, device='cuda')
  mask, err = ops.robust_mask(rgb.reshape(B, 3).contiguous().cuda(), target.reshape(B, 3).contiguous().cuda(),
                              thr_dev, _desc(ops, B, cfg), counts=counts, stats=row)
  ops.quantile(err, cfg.robustnerf_inlier_quantile, out=row[0:1])
  torch.cuda.synchronize()
  row = row.cpu()
  names = train_utils.ROBUST_STAT_NAMES if cfg.enable_robustnerf_loss else ('loss_threshold', 'mask')
  stats = {k: row[train_utils.ROBUST_STAT_NAMES.index(k)] for k in names}
  return mask.cpu().reshape(shape[:3] + (1,)), err.cpu().reshape(shape[:3] + (1,)), stats


def _check_against_oracle(ops, rgb, target, thr, cfg, counts):
  mask, err, stats = _run_mask(ops, rgb, target, thr, cfg, counts)
  resid_sq = (rgb - target) ** 2
  mask_o, stats_o = o_robust.robustnerf_mask(resid_sq, torch.tensor(thr, dtype=torch.float32), cfg)
  err_o = (resid_sq[..., 0:1] + resid_sq[..., 1:2] + resid_sq[..., 2:3]) / torch.tensor(3.0)
  np.testing.assert_array_equal(_bits(err), _bits(err_o))
  np.testing.assert_array_equal(mask.numpy(), mask_o.numpy())
  assert set(stats) == set(stats_o)
  for k in stats:
    assert _bits(stats[k]) == _bits(stats_o[k]), (k, float(stats[k]), float(stats_o[k]))
  assert int(counts.abs().sum()) == 0          # the workspace is left zero for the next launch
  return float(mask.mean())


def test_mask_kernel_matches_golden_cases(mods):
  _, ops, _ = mods
  g = golden('robustnerf')
  counts = torch.zeros(5, dtype=torch.int32, device='cuda')
  for name in (str(c) for c in g['cases']):
    kw = {k.split('/')[-1]: g[k].item() for k in g.files if k.startswith(f'{name}/cfg/')}
    cfg = _cfg(kw['patch_size'], kw['robustnerf_inner_patch_size'], kw['robustnerf_smoothed_filter_size'],
               kw['robustnerf_inlier_quantile'], kw['robustnerf_smoothed_inlier_quantile'],
               kw['robustnerf_inner_patch_inlier_quantile'], kw['enable_robustnerf_loss'])
    rgb, target = torch.as_tensor(g[f'{name}/rgb']), torch.as_tensor(g[f'{name}/target'])
    mask, err, stats = _run_mask(ops, rgb, target, g[f'{name}/threshold'], cfg, counts)
    np.testing.assert_array_equal(mask.numpy(), g[f'{name}/mask'], err_msg=name)
    np.testing.assert_array_equal(_bits(err), _bits(g[f'{name}/error_per_pixel']), err_msg=name)
    for k in stats:
      assert _bits(stats[k]) == _bits(g[f'{name}/stat/{k}']), (name, k, float(stats[k]))


@pytest.mark.parametrize('p,inner,f,q,qs,qp', [(8, 4, 3, 0.5, 0.5, 0.5), (8, 3, 5, 0.8, 0.5, 0.5),
                                               (16, 8, 3, 0.8, 0.5, 0.5), (16, 5, 7, 0.5, 0.3, 0.7),
                                               (32, 16, 3, 0.5, 0.5, 0.5), (32, 31, 9, 0.8, 0.6, 0.4),
                                               (13, 6, 1, 0.5, 0.5, 0.5)])
def test_mask_kernel_random_patches_bit_exact(mods, p, inner, f, q, qs, qp):
  _, ops, _ = mods
  rng = np.random.default_rng(p * 100 + inner * 10 + f)
  n = 96
  target = torch.tensor(rng.uniform(0, 1, (n, p, p, 3)).astype(np.float32))
  # smooth error fields with outlier blobs, so that every branch of the mask is taken
  scale = np.exp(rng.normal(-3, 1.5, (n, 1, 1, 1)))
  yy, xx = np.mgrid[:p, :p]
  blobs = np.zeros((n, p, p, 1))
  for i in range(n):
    cy, cx, r = rng.uniform(0, p), rng.uniform(0, p), rng.uniform(0.1, 0.7) * p
    blobs[i, ..., 0] = ((yy - cy) ** 2 + (xx - cx) ** 2 < r * r) * rng.uniform(0, 1)
  rgb = torch.tensor((target.numpy() + rng.normal(0, 1, (n, p, p, 3)) * scale + blobs).astype(np.float32))
  err = ((rgb - target) ** 2).mean(-1)
  counts = torch.zeros(5, dtype=torch.int32, device='cuda')
  means = []
  for thr_q in (0.3, 0.6, 0.9):
    thr = np.float32(np.quantile(err.numpy(), thr_q))
    means.append(_check_against_oracle(ops, rgb, target, thr, _cfg(p, inner, f, q, qs, qp), counts))
  assert min(means) < 0.95 and max(means) > 0.3, means
  # the flag off: all ones, and the error / threshold still come out
  _check_against_oracle(ops, rgb, target, 0.01, _cfg(p, inner, f, q, qs, qp, enable=False), counts)


def test_mask_kernel_rejects_unsupported_shapes(mods):
  from multinerf_b200 import lib
  _, ops, _ = mods
  x = torch.zeros(33 * 33, 3, device='cuda')
  thr = torch.ones(1, device='cuda')
  with pytest.raises(lib.MnrfError, match='p\\*p'):
    ops.robust_mask(x, x, thr, _desc(ops, 33 * 33, _cfg(33, 8, 3)))
  x = torch.zeros(256 + 16, 3, device='cuda')
  with pytest.raises(lib.MnrfError, match='multiple'):
    ops.robust_mask(x, x, thr, _desc(ops, 256 + 16, _cfg(16, 8, 3)))
  x = torch.zeros(256, 3, device='cuda')
  with pytest.raises(lib.MnrfError, match='odd'):
    ops.robust_mask(x, x, thr, _desc(ops, 256, _cfg(16, 8, 4)))


@pytest.mark.parametrize('n', [1, 2, 255, 16384, 16384 * 8 + 37])
def test_quantile_kernel_bit_exact(mods, n):
  _, ops, _ = mods
  rng = np.random.default_rng(n)
  sets = {
      'normal': rng.normal(size=n),
      'exponents': rng.uniform(0.5, 1, n) * np.exp2(rng.integers(-60, 60, n)) * rng.choice([-1, 1], n),
      'duplicates': rng.integers(0, 5, n) * 0.25,
      'errors': rng.uniform(0, 1, n) ** 6,
  }
  out = torch.empty(1, device='cuda')
  for name, x in sets.items():
    xt = torch.tensor(x.astype(np.float32))
    xd = xt.cuda()
    for q in (0.0, 0.5, 0.8, 1.0):
      ops.quantile(xd, q, out=out)
      want = o_robust.quantile_linear(xt, q)
      assert _bits(out.cpu()[0]) == _bits(want), (name, q, float(out.cpu()[0]), float(want))
  if n > 1:
    x = torch.tensor(rng.normal(size=n).astype(np.float32))
    x[n // 2] = float('nan')
    assert np.isnan(float(ops.quantile(x.cuda(), 0.5)[0].cpu()))


@pytest.mark.parametrize('S', [32, 128])
def test_masked_composite_bwd(mods, S):
  _, ops, _ = mods
  rng = np.random.default_rng(5 + S)
  B = 96
  cfg = dict(CFG)
  _, d, _ = kernel_rays(rng, B)
  s = torch.tensor(np.sort(rng.uniform(0, 1, (B, S + 1)).astype(np.float32), -1))
  s[:, 0], s[:, -1] = 0, 1
  raw_d = torch.tensor(rng.normal(size=(B, S)).astype(np.float32) * 2, requires_grad=True)
  raw_rgb = torch.tensor(rng.normal(size=(B, S, 3)).astype(np.float32), requires_grad=True)
  nearv, farv = torch.full((B, 1), 0.2), torch.full((B, 1), 1e6)
  target = torch.tensor(rng.uniform(0, 1, (B, 3)).astype(np.float32))
  mask = torch.tensor((rng.uniform(size=B) < 0.6).astype(np.float32))
  # oracle: resid_sq * mask with the mask a constant (train_utils.py:104-111), distortion on top
  w_o, r_o, _, _ = oracle_composite(raw_d, raw_rgb, s, d, nearv, farv, cfg)
  resid_sq = (r_o['rgb'] - target) ** 2
  data = (resid_sq * mask[:, None]).sum() / (3 * B)
  extra = 0.01 * o_train.o_stepfun.lossfun_distortion(s, w_o).mean()
  grads = torch.autograd.grad(data + extra, [raw_d, raw_rgb])

  def run(m):
    stats = torch.zeros(8, device='cuda')
    g = ops.composite_bwd(
        raw_d.detach().cuda(), raw_rgb.detach().cuda(), s.cuda(), d.cuda(), nearv[:, 0].contiguous().cuda(),
        farv[:, 0].contiguous().cuda(), target.cuda(), torch.ones(B, 1, device='cuda'),
        torch.tensor([1.0 / (3 * B)], device='cuda'), stats, cfg=cfg, loss_type='mse', charb_padding=0.001,
        data_mult=1.0, distortion_mult=0.01, interlevel_mult=0.0, data_mask=m)
    torch.cuda.synchronize()
    return [t.cpu() for t in g], stats.cpu()
  (g_d, g_rgb), st = run(mask.cuda())
  close(g_d, grads[0], atol=2e-5 * float(grads[0].abs().max()), rtol=2e-4, msg='d raw_density')
  close(g_rgb, grads[1], atol=2e-5 * float(grads[1].abs().max()), rtol=2e-4, msg='d raw_rgb')
  close(st[0], data.detach(), rtol=1e-4, atol=1e-7, msg='masked data loss')
  close(st[1], resid_sq.detach().mean(), rtol=1e-4, atol=1e-7, msg='mse stays unmasked')
  # an all-ones mask is the mse path: gradients bit for bit; the loss sums are fp32 atomics across warps,
  # whose order varies from launch to launch
  (a_d, a_rgb), a_st = run(torch.ones(B, device='cuda'))
  (b_d, b_rgb), b_st = run(None)
  assert torch.equal(a_d, b_d) and torch.equal(a_rgb, b_rgb)
  close(a_st, b_st, atol=0, rtol=1e-6, msg='stats')


def _robust_bundle(p=8, inner=4):
  b = mini360()
  c = b.config
  c.data_loss_type, c.patch_size, c.enable_robustnerf_loss = 'robustnerf', p, True
  c.robustnerf_inlier_quantile, c.robustnerf_inner_patch_size = 0.8, inner
  return b


def _oracle_errors(bundle, model, rays, target, rand, train_frac):
  from oracle import o_models
  with torch.no_grad():
    rend, _ = o_models.model_apply(torch_tree(model.export_flax()), bundle, bases(model), oracle_rays(rays),
                                   train_frac, False, rand=rand, zero_glo=False, bf16=True)
  return ((rend[-1]['rgb'] - torch.tensor(target)) ** 2).mean(-1)


def _gap_threshold(err, lo_q, hi_q):
  """A threshold inside the widest gap of the sorted errors between two quantiles: pixels near it would flip
  between the bf16 GPU model and the oracle."""
  e = np.sort(err.numpy().astype(np.float64))
  i0, i1 = int(lo_q * len(e)), int(hi_q * len(e))
  gaps = np.log(e[i0 + 1:i1 + 1]) - np.log(e[i0:i1])
  k = i0 + int(np.argmax(gaps))
  return float(np.float32(np.sqrt(e[k] * e[k + 1])))


def test_mini_train_step_vs_oracle(mods):
  models, _, train_utils = mods
  bundle = _robust_bundle()
  bundle.config.grad_max_norm = 0.0
  B = 4 * 64                                     # 4 patches of 8 x 8
  rays, rng = synth_rays(13, B, 0.2, 1e6)
  target = rng.uniform(0, 1, (B, 3)).astype(np.float32)
  model, variables = models.construct_model(14, rays, bundle)
  rand = {'jitter': [torch.tensor(rng.uniform(0, 1, (B, 1)).astype(np.float32)) for _ in range(3)]}
  thr = _gap_threshold(_oracle_errors(bundle, model, rays, target, rand, 0.5), 0.3, 0.6)
  t = train_step(model, variables, bundle, rays, target, rand, 0.5, oracle=o_robust.train_step, loss_threshold=thr)
  stats, stats_o = t.stats, t.stats_o
  assert 0.1 < float(stats_o['mask']) < 0.9, float(stats_o['mask'])
  for k in train_utils.ROBUST_STAT_NAMES:
    tol = 0.02 if k == 'loss_threshold' else 0.01
    assert abs(stats[k] - float(stats_o[k])) <= tol * max(abs(float(stats_o[k])), 1e-3), \
        (k, stats[k], float(stats_o[k]))
  close(stats['mses'], stats_o['mses'].detach(), atol=2e-3, rtol=2e-2, msg='mses')
  lo = float(stats_o['loss'].detach())
  assert abs(stats['loss'] - lo) < 2e-2 * max(1.0, abs(lo)), (stats['loss'], lo)
  report, zero = grad_report(model, t.grads_o, mlp_leaves(model, ('kernel', 'bias')))
  assert not any(zero.values()), zero
  assert not beyond(report, 0.12, 0.993), beyond(report, 0.12, 0.993)


def test_graph_replay_with_device_threshold_tracks_eager(mods):
  models, _, train_utils = mods
  from multinerf_b200 import ops, utils
  bundle = _robust_bundle()
  B, steps = 4 * 64, 5
  rays, rng = synth_rays(21, B, 0.2, 1e6)
  batches = [(synth_rays(30 + i, B, 0.2, 1e6)[0], rng.uniform(0, 1, (B, 3)).astype(np.float32))
             for i in range(steps)]
  rands = [{'jitter': [torch.tensor(rng.uniform(0, 1, (B,)).astype(np.float32)) for _ in range(3)]}
           for _ in range(steps)]
  results = []
  for use_graph in [False, True]:
    model, variables = models.construct_model(22, rays, bundle)
    step_fn = train_utils.create_train_step(model, bundle.config, use_graph=use_graph)
    state = train_utils.TrainState(variables)
    thr, thrs, mats = 1.0, [], []
    for i in range(steps):
      r, tgt = batches[i]
      state, stats, _ = step_fn(rands[i], state, utils.Batch(rays=r, rgb=tgt), None, i / 10.0, thr)
      thr = stats.device_loss_threshold()
      assert thr.is_cuda and thr.dim() == 0
      thrs.append(thr)
      mats.append(stats)
    torch.cuda.synchronize()
    mats = [m.materialize() for m in mats]
    results.append(([float(t) for t in thrs], mats, variables.flat.clone()))
    if use_graph:
      g = step_fn.graph_info
      assert g['state'] == 2 and g['launches'] > 20
  (t0, m0, p0), (t1, m1, p1) = results
  assert all(t != 1.0 for t in t0)
  for a, b in zip(t0, t1):
    assert abs(a - b) < 2e-3 * abs(a), (t0, t1)
  for a, b in zip(m0, m1):
    assert abs(a['loss'] - b['loss']) < 2e-3 * max(1.0, abs(a['loss'])), (a['loss'], b['loss'])
    for k in train_utils.ROBUST_STAT_NAMES:
      assert abs(a[k] - b[k]) < 0.02 * max(abs(a[k]), 1e-3), (k, a[k], b[k])
  assert 0.0 < m0[-1]['mask'] < 1.0
  rel = float((p0 - p1).norm() / p0.norm())
  assert rel < 2e-3, rel


def test_launches_per_robust_step(mods):
  """One mask launch per masked level and one quantile launch per step on top of the mse step."""
  models, _, train_utils = mods
  from multinerf_b200 import ops, utils
  B = 4 * 64
  rays, rng = synth_rays(41, B, 0.2, 1e6)
  tgt = rng.uniform(0, 1, (B, 3)).astype(np.float32)
  counts = {}
  for loss in ('mse', 'robustnerf'):
    bundle = _robust_bundle()
    bundle.config.data_loss_type = loss
    model, variables = models.construct_model(42, rays, bundle)
    step_fn = train_utils.create_train_step(model, bundle.config, use_graph=True)
    state = train_utils.TrainState(variables)
    for i in range(3):
      state, stats, _ = step_fn(None, state, utils.Batch(rays=rays, rgb=tgt), None, 0.5)
    counts[loss] = step_fn.graph_info['launches']
  masked_levels = 1 + (2 if bundle.config.data_coarse_loss_mult != 0 else 0)
  assert counts['robustnerf'] - counts['mse'] == masked_levels + 1, counts


def test_fullwidth_360_robustnerf_step_vs_oracle(mods):
  """configs/360_robustnerf.gin at its widths, 1024 rays (4 patches of 16 x 16), within the 360.gin bounds of
  test_gpu_fullwidth.py."""
  import os
  models, _, train_utils = mods
  from multinerf_b200 import configs, utils
  here = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'configs')
  bundle = configs.load_config([os.path.join(here, '360_robustnerf.gin')], search_paths=[here])
  c = bundle.config
  assert c.data_loss_type == 'robustnerf' and c.patch_size == 16 and c.enable_robustnerf_loss
  c.grad_max_norm = c.grad_max_val = 0.0
  B = 1024
  rays, rng = synth_rays(51, B, 0.2, 1e6)
  target = rng.uniform(0, 1, (B, 3)).astype(np.float32)
  rand = {'jitter': [torch.tensor(rng.uniform(0, 1, (B, 1)).astype(np.float32)) for _ in range(3)]}
  model, variables = models.construct_model(52, rays, bundle)
  thr = _gap_threshold(_oracle_errors(bundle, model, rays, target, rand, 0.5), 0.3, 0.6)
  t = train_step(model, variables, bundle, rays, target, rand, 0.5, oracle=o_robust.train_step, loss_threshold=thr)
  stats, stats_o = t.stats, t.stats_o
  assert 0.1 < float(stats_o['mask']) < 0.9, float(stats_o['mask'])
  close(stats['mses'], stats_o['mses'].detach(), atol=1e-6, rtol=2e-3, msg='mses')
  lo = float(stats_o['loss'].detach())
  assert abs(stats['loss'] - lo) < 3e-3 * max(1.0, abs(lo)), (stats['loss'], lo)
  assert abs(stats['mask'] - float(stats_o['mask'])) < 0.01, (stats['mask'], float(stats_o['mask']))
  report, zero = grad_report(model, t.grads_o, mlp_leaves(model, ('kernel', 'bias')))
  assert not any(zero.values()), zero
  # a head's bias gradient is a plain sum that cancels to nearly nothing (test_gpu_fullwidth.py measures it
  # against its kernel's scale): trunk leaves and kernels are held to the 360.gin bound
  head = {(m, sp.name) for m in model.plans for sp in model.plans[m].specs if sp.out_dim <= 4}
  bad = {k: v for k, v in beyond(report, 0.2, 0.98).items() if not (k[2] == 'bias' and k[:2] in head)}
  assert not bad, bad


def test_train_loop_feeds_threshold_back_and_logs_robust_stats(mods, monkeypatch):
  _, _, train_utils = mods
  from multinerf_b200 import train_loop
  b = train_loop_bundle(6, cast=True)
  c = b.config
  c.data_loss_type, c.patch_size, c.enable_robustnerf_loss = 'robustnerf', 16, True
  c.robustnerf_inlier_quantile, c.print_every = 0.8, 3
  seen = []
  make = train_utils.create_train_step

  def spy(*a, **k):
    fn = make(*a, **k)

    def step(rng, state, batch, cameras, train_frac, loss_threshold):
      seen.append(loss_threshold)
      return fn(rng, state, batch, cameras, train_frac, loss_threshold)
    step.graph_info = fn.graph_info
    return step
  monkeypatch.setattr(train_utils, 'create_train_step', spy)
  model, state, hist = train_loop.train(b, train_loop.SyntheticScene(c), log=lambda s: None, use_graph=True)
  assert state.step == 6 and len(seen) == 6
  assert seen[0] == 1.0 and not torch.is_tensor(seen[0])
  for t in seen[1:]:
    assert torch.is_tensor(t) and t.is_cuda and float(t) != 1.0
  logged = {name for kind, name, *_ in train_loop.train.summaries.log if kind == 'scalar'}
  for k in train_utils.ROBUST_STAT_NAMES:
    assert f'train_avg_{k}' in logged and f'train_max_{k}' in logged, k
    assert k in hist[-1]
  assert 0.0 < hist[-1]['mask'] <= 1.0 and hist[-1]['loss_threshold'] > 0.0
