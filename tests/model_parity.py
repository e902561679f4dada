"""The model-level parity harness of the GPU tests: synthetic rays and reduced model bundles, and the comparisons of
a GPU model against the CPU oracle on identical rays, weights and random draws (one train step, the per-leaf
gradient report, the per-level forward with the oracle's sample positions pinned) and of graph replay against the
eager step.  A helper module, not a test module: the tests choose the inputs and write the bounds.

The Dense layers run in bf16 on tensor cores, so the oracle is evaluated with the same bf16-rounded weights and
layer inputs (fp32 accumulation, oracle/o_models.py `bf16=True`).
"""
import types

import numpy as np
import torch

from oracle import o_models, o_train
from util import close

F32 = np.float32


# ------------------------------------------------------------------ rays and bundles

def synth_rays(seed, B, near, far, unit_cube=True, radius=4.0):
  """(rays, generator): origins in the unit cube, or cameras on a sphere looking at the origin; the generator
  continues after the rays' draws."""
  from multinerf_b200 import utils
  rng = np.random.default_rng(seed)
  if unit_cube:
    o = rng.uniform(-1, 1, (B, 3))
    d = rng.normal(size=(B, 3))
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
  else:   # cameras on a sphere looking at the origin (tests/render_test.py:137-143 style)
    o = rng.normal(size=(B, 3))
    o = o / np.linalg.norm(o, axis=-1, keepdims=True) * radius
    d = -o / radius + rng.normal(size=(B, 3)) * 0.1
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
  v = d.copy()
  d = d * rng.uniform(0.8, 1.2, (B, 1))
  return utils.Rays(origins=o.astype(F32), directions=d.astype(F32), viewdirs=v.astype(F32),
                    radii=rng.uniform(5e-4, 1e-3, (B, 1)).astype(F32),
                    imageplane=np.zeros((B, 2), F32), lossmult=np.ones((B, 1), F32),
                    near=np.full((B, 1), near, F32), far=np.full((B, 1), far, F32),
                    cam_idx=np.zeros((B, 1), np.int32)), rng


def raw_rays(rng, B, radii_first=False):
  """llff_raw-style rays: forward-facing cylinders on [0, 1], a Bayer lossmult (one channel per ray) and exposure
  indices 0-3 with values 2^-idx.  radii_first: draw the radii before the Bayer channels instead of after."""
  from multinerf_b200 import utils
  o = np.concatenate([rng.uniform(-1, 1, (B, 2)), -np.ones((B, 1))], -1)
  d = np.concatenate([rng.uniform(-.5, .5, (B, 2)), 2 * np.ones((B, 1))], -1)
  eidx = rng.integers(0, 4, (B, 1)).astype(np.int32)
  if radii_first:
    radii = rng.uniform(1e-3, 2e-3, (B, 1)).astype(F32)
  lossmult = np.eye(3, dtype=F32)[rng.integers(0, 3, B)]
  if not radii_first:
    radii = rng.uniform(1e-3, 2e-3, (B, 1)).astype(F32)
  return utils.Rays(origins=o.astype(F32), directions=d.astype(F32),
                    viewdirs=(d / np.linalg.norm(d, axis=-1, keepdims=True)).astype(F32), radii=radii,
                    imageplane=np.zeros((B, 2), F32), lossmult=lossmult, near=np.zeros((B, 1), F32),
                    far=np.ones((B, 1), F32), cam_idx=np.zeros((B, 1), np.int32), exposure_idx=eidx,
                    exposure_values=(2.0 ** -eidx).astype(F32))


def image_rays(H, W, focal=120.0):
  """An H x W pinhole image from (0.5, 0.5, 0.3) looking down -z, near 0.2 and far 1e6."""
  from multinerf_b200 import utils
  ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing='ij')
  d = np.stack([(xs - W / 2) / focal, (ys - H / 2) / focal, -np.ones_like(xs, dtype=np.float64)], -1)
  v = d / np.linalg.norm(d, axis=-1, keepdims=True)
  o = np.broadcast_to(np.array([0.5, 0.5, 0.3]), d.shape)
  return utils.Rays(origins=o.astype(F32), directions=d.astype(F32), viewdirs=v.astype(F32),
                    radii=np.full((H, W, 1), 7e-4, F32), imageplane=np.zeros((H, W, 2), F32),
                    lossmult=np.ones((H, W, 1), F32), near=np.full((H, W, 1), 0.2, F32),
                    far=np.full((H, W, 1), 1e6, F32), cam_idx=np.zeros((H, W, 1), np.int32))


def level_jitter(rng, bundle, B):
  """{'jitter': [...]} with one draw per level: per ray, or per sample without single_jitter."""
  m = bundle.model
  S = [m.num_prop_samples] * (m.num_levels - 1) + [m.num_nerf_samples]
  return {'jitter': [torch.tensor(rng.uniform(0, 1, (B, 1 if m.single_jitter else s)).astype(F32)) for s in S]}


def synth_case(bundle, B, seed, near, far, unit_cube=True):
  """(rays, rand, target): synth_rays, then every level's jitter, then a uniform target colour."""
  rays, rng = synth_rays(seed, B, near, far, unit_cube)
  rand = level_jitter(rng, bundle, B)
  return rays, rand, rng.uniform(0, 1, (B, 3)).astype(F32)


def mini360():
  from multinerf_b200 import configs
  b = configs.bundle_360()
  b.model.num_prop_samples = 32
  b.model.num_nerf_samples = 16
  b.prop_mlp.net_depth, b.prop_mlp.net_width = 2, 64
  b.nerf_mlp.net_depth, b.nerf_mlp.net_width = 6, 128
  b.nerf_mlp.bottleneck_width, b.nerf_mlp.net_width_viewdirs = 64, 64
  return b


def plumbing_blender():
  from multinerf_b200 import configs
  b = configs.bundle_blender_256()
  b.model.num_levels = 1
  b.model.num_nerf_samples = 32
  return b


def mini_refnerf():
  from multinerf_b200 import configs
  b = configs.Bundle()
  c, m, n = b.config, b.model, b.nerf_mlp
  c.data_loss_type, c.distortion_loss_mult, c.interlevel_loss_mult, c.data_coarse_loss_mult = 'mse', 0.0, 0.0, 0.1
  c.orientation_loss_mult, c.orientation_coarse_loss_mult = 0.1, 0.01
  c.predicted_normal_loss_mult, c.predicted_normal_coarse_loss_mult = 3e-4, 3e-5
  c.adam_eps, c.near, c.far = 1e-8, 2.0, 6.0
  m.num_levels, m.single_mlp, m.num_prop_samples, m.num_nerf_samples = 2, True, 16, 16
  m.anneal_slope, m.dilation_multiplier, m.dilation_bias, m.single_jitter, m.resample_padding = 0., 0., 0., False, 0.01
  n.net_depth, n.net_width, n.net_depth_viewdirs, n.net_width_viewdirs = 6, 128, 6, 64
  n.basis_shape, n.basis_subdivisions, n.disable_density_normals, n.enable_pred_normals = 'octahedron', 1, False, True
  n.use_directional_enc = n.use_reflections = n.enable_pred_roughness = True
  n.use_diffuse_color = n.use_specular_tint = n.use_n_dot_v = True
  n.deg_view, n.bottleneck_width, n.density_bias, n.max_deg_point = 5, 64, 0.5, 16
  return b


def train_loop_bundle(steps, ckpt=None, cast=False):
  """mini360 for train_loop.train on the procedural scene: 2048-ray batches, a checkpoint every 60 steps."""
  b = mini360()
  c = b.config
  c.batch_size, c.max_steps, c.print_every = 2048, steps, 20
  c.lr_init, c.lr_final, c.lr_delay_steps = 5e-3, 5e-4, 20
  c.checkpoint_every, c.checkpoint_dir = 60, ckpt
  c.cast_rays_in_train_step = cast
  return b


def fullwidth_case(which):
  """(bundle, rays, target, rand, B, S) of one BASELINE config at its stated widths: '360', 'refnerf' or 'raw'."""
  from multinerf_b200 import configs
  if which == '360':
    bundle = configs.bundle_360()
    B = 256
    rays, rng = synth_rays(31, B, 0.2, 1e6)
    S = [64, 64, 32]
    rand = {'jitter': [torch.tensor(rng.uniform(0, 1, (B, 1)).astype(F32)) for _ in S]}
  elif which == 'refnerf':
    bundle = configs.bundle_blender_refnerf()
    B = 128
    rays, rng = synth_rays(32, B, 2.0, 6.0, unit_cube=False)
    S = [128, 128]
    rand = {'jitter': [torch.tensor(rng.uniform(0, 1, (B, s)).astype(F32)) for s in S]}
  else:
    bundle = configs.bundle_llff_raw()
    B = 128
    rng = np.random.default_rng(33)
    rays = raw_rays(rng, B)
    S = [128, 128]
    rand = {'jitter': [torch.tensor(rng.uniform(0, 1, (B, s)).astype(F32)) for s in S],
            'density_noise': [torch.tensor(rng.normal(size=(B, s)).astype(F32)) for s in S]}
  target = (rng.uniform(0, 1, (B, 3)) ** (2 if which == 'raw' else 1)).astype(F32)
  return bundle, rays, target, rand, B, S


# ------------------------------------------------------------------ oracle inputs

def torch_tree(tree):
  return {k: (torch_tree(v) if isinstance(v, dict) else torch.tensor(v)) for k, v in tree.items()}


def oracle_rays(rays):
  r = types.SimpleNamespace()
  for k, v in rays.__dict__.items():
    setattr(r, k, None if v is None else torch.tensor(np.asarray(v)))
  return r


def bases(model):
  """The oracle's encoding bases of a GPU model; under single_mlp the proposal levels use the NerfMLP's."""
  return {'nerf': model.plans['NerfMLP_0'].basis,
          'prop': model.plans.get('PropMLP_0', model.plans['NerfMLP_0']).basis}


# ------------------------------------------------------------------ comparisons

def oracle_step(params0, model, bundle, rays, target, rand, train_frac, oracle=None, bf16=True, **kw):
  """The oracle's first train step from `params0` with the encoding bases of `model`: (new params, optimizer
  state, stats, grads).  oracle: o_train.train_step by default; bf16: emulate the GPU's bf16 layers, or run in
  fp32."""
  return (oracle or o_train.train_step)(params0, {'count': 0, 'mu': {}, 'nu': {}}, bundle, bases(model),
                                        oracle_rays(rays), torch.tensor(target), train_frac, rand=rand, bf16=bf16, **kw)


def train_step(model, variables, bundle, rays, target, rand, train_frac, oracle=None, loss_threshold=None,
               **step_kw):
  """One train step of the oracle (bf16-emulated forward, fp32 autograd) and of the GPU model from the same
  parameters and draws.  `oracle`: the oracle_step default, or o_robust.train_step with `loss_threshold` (which the
  GPU step also gets); `step_kw` go to create_train_step.  Returns the GPU `stats` (materialized), the oracle's
  `stats_o`, `grads_o` and new parameters `new_o`, and the parameters `params0` both started from."""
  from multinerf_b200 import train_utils, utils
  params0 = torch_tree(model.export_flax())
  kw = {} if loss_threshold is None else {'loss_threshold': loss_threshold}
  new_o, _, stats_o, grads_o = oracle_step(params0, model, bundle, rays, target, rand, train_frac, oracle=oracle, **kw)
  step_fn = train_utils.create_train_step(model, bundle.config, **step_kw)
  state = train_utils.TrainState(variables)
  extra = () if loss_threshold is None else (loss_threshold,)
  state, stats, _ = step_fn(rand, state, utils.Batch(rays=rays, rgb=target), None, train_frac, *extra)
  torch.cuda.synchronize()
  stats.materialize()
  return types.SimpleNamespace(stats=stats, stats_o=stats_o, grads_o=grads_o, new_o=new_o, params0=params0)


def mlp_leaves(model, leaves=('kernel',), modules=None):
  """The gradient keys (module, layer, leaf) of every Dense layer of the named MLPs (all by default)."""
  return [(mname, sp.name, leaf) for mname, plan in model.plans.items() if modules is None or mname in modules
          for sp in plan.specs for leaf in leaves]


def grad_report(model, grads_o, keys):
  """Per gradient key, (rel, cos) of the GPU gradient against the oracle's in float64, rounded to 3 and 4 decimals:
  rel = |a - b| / |b|, cos = a.b / (|a| |b|).  Keys whose oracle gradient is zero are returned apart, with the norm
  of the GPU gradient: (report, zero)."""
  g = model.export_grads_flax()
  report, zero = {}, {}
  for key in keys:
    a = g
    for part in key:
      a = a[part]
    a = torch.tensor(a).double().flatten()
    b = grads_o[key].double().flatten()
    if float(b.norm()) == 0.0:
      zero[key] = float(a.norm())
      continue
    report[key] = (round(float((a - b).norm() / b.norm()), 3),
                   round(float((a @ b) / (a.norm() * b.norm()).clamp(min=1e-30)), 4))
  return report, zero


def beyond(report, rel, cos):
  """The entries of a gradient report with rel >= `rel` or cos <= `cos`."""
  return {k: v for k, v in report.items() if not (v[0] < rel and v[1] > cos)}


def worst(report):
  return sorted(report.items(), key=lambda kv: -kv[1][0])[:6]


def pinned_forward(model, bundle, rays, rand, *, dens, pixel, acc=None, samples=None, level=None):
  """The oracle's randomized forward at train_frac 0.5, then each GPU level with its sample positions pinned to the
  oracle's, so that every level's MLP and compositing are compared in isolation.  Level 0 resamples the trivial
  histogram, so its positions must already agree.  Per level: density (max, mean) relative error under `dens`,
  weights within 2e-2, the pixel within `pixel`, and if given the acc and the per-sample colours; `level(i, st, h)`
  adds a caller's checks on the level's state and oracle history.  Returns the oracle's (renderings, history)."""
  from multinerf_b200 import ops
  rend_o, hist_o = o_models.model_apply(torch_tree(model.export_flax()), bundle, bases(model), oracle_rays(rays),
                                        0.5, True, rand=rand, bf16=True)
  rend_o = [{k: v.detach() for k, v in r.items()} for r in rend_o]
  hist_o = [{k: (v.detach() if v is not None else None) for k, v in h.items()} for h in hist_o]
  r = model._prep_rays(rays)
  states = model.forward_levels(rand, r, 0.5, True, True)
  torch.cuda.synchronize()
  close(states[0].sdist, hist_o[0]['sdist'], atol=1e-6, rtol=1e-6, msg='level-0 sdist')
  for i, st in enumerate(states):
    h = hist_o[i]
    st.sdist.copy_(h['sdist'].cuda())
    model._mlp_forward(st, model.mlps[st.mname], r)
    comp = ops.composite_fwd(st.raw_density, st.raw_rgb, st.sdist, r.directions, r.near_flat, r.far_flat,
                             cfg=st.comp_cfg, density_noise=st.noise, rgb_scale=st.rgb_scale,
                             raw_diffuse=st.heads.get('diffuse'), raw_tint=st.heads.get('tint'),
                             want_samples=True, want_extras=True)
    torch.cuda.synchronize()
    err = (comp['density'].cpu() - h['density']).abs() / (1.0 + h['density'].abs())
    assert float(err.max()) < dens[0] and float(err.mean()) < dens[1], (i, float(err.max()), float(err.mean()))
    close(comp['weights'], h['weights'], atol=2e-2, rtol=0, msg=f'weights level {i}')
    close(comp['rgb'], rend_o[i]['rgb'], atol=pixel, rtol=0, msg=f'pixel level {i}')
    if acc is not None:
      close(comp['acc'], rend_o[i]['acc'], atol=acc, rtol=0, msg=f'acc level {i}')
    if samples is not None and st.raw_rgb is not None:
      close(comp['rgb_samples'], h['rgb'], atol=samples, rtol=0, msg=f'rgb samples level {i}')
    if level is not None:
      level(i, st, h)
  return rend_o, hist_o


def graph_matches_eager(models, train_utils, bundle, batches, seed, extra=None):
  """`batches` ((rays, target, rand) per step, train_frac = step / 10) run eagerly and by graph replay from the
  same initial weights: both take every step, the replay really runs a captured graph, and the losses (and the
  stat `extra(stats)` if given) and the final parameters agree to 2e-3 relative, the noise of fp32 atomics."""
  from multinerf_b200 import utils
  runs = []
  for use_graph in (False, True):
    model, variables = models.construct_model(seed, batches[0][0], bundle)
    step_fn = train_utils.create_train_step(model, bundle.config, use_graph=use_graph)
    state = train_utils.TrainState(variables)
    losses, extras = [], []
    for i, (rays, target, rand) in enumerate(batches):
      state, stats, _ = step_fn(rand, state, utils.Batch(rays=rays, rgb=target), None, i / 10.0)
      s = stats.materialize()
      losses.append(s['loss'])
      if extra is not None:
        extras.append(extra(s))
    torch.cuda.synchronize()
    runs.append((losses + extras, variables.flat.clone()))
    assert variables.step == len(batches), (use_graph, variables.step)
    if use_graph:
      assert step_fn.graph_info['state'] == 2 and step_fn.graph_info['launches'] > 20, step_fn.graph_info
  (v0, p0), (v1, p1) = runs
  for a, b in zip(v0, v1):
    assert abs(a - b) < 2e-3 * max(1.0, abs(a)), (v0, v1)
  rel = float((p0 - p1).norm() / p0.norm())
  assert rel < 2e-3, rel


def check_train_step(models, train_utils, bundle, B, seed, lim):
  """One step on rays from cameras on a sphere (near 2, far 6) against the oracle: the mses, the normal losses the
  config has, and every layer's kernel gradient within `lim` = (rel, cos), on both MLPs."""
  rays, rand, target = synth_case(bundle, B, seed, 2.0, 6.0, unit_cube=False)
  model, variables = models.construct_model(seed + 1, rays, bundle)
  t = train_step(model, variables, bundle, rays, target, rand, 0.5)
  close(t.stats['mses'], t.stats_o['mses'].detach(), atol=2e-3, rtol=3e-2, msg='mses')
  for k in ('orientation', 'predicted_normals'):
    if k in t.stats_o['losses']:
      lo = float(t.stats_o['losses'][k].detach())
      assert abs(t.stats['losses'][k] - lo) < 0.05 * abs(lo) + 1e-7, (k, t.stats['losses'][k], lo)
  report, zero = grad_report(model, t.grads_o, mlp_leaves(model))
  assert not any(zero.values()), zero
  assert any(k[0] == 'PropMLP_0' for k in report) and any(k[0] == 'NerfMLP_0' for k in report)
  print(f'worst leaves (rel, cos): {worst(report)}')
  bad = beyond(report, *lim)
  assert not bad, (bad, worst(report))
