"""One eager train step, every stage of every level's MLP against tests/level_ref.py pinned to the tensors the GPU
stored.  Needs an H100.

The step runs under launch_recorder.Recorder.  The pinned tensors are found by meaning, not by launch order or
ping-pong buffer:
  - forward: the LevelState buffers after the step (features and their tangents, trunk outputs and tangent streams,
    z or mask bits, head outputs, raw_grad_density, view input, view outputs); nothing in the backward writes them;
  - the gradient w.r.t. trunk layer i's output (its tangent adjoint): the dY operand of the WGRAD whose output is that
    layer's slice of mlp.grads and whose X operand is this level's (tangent) input of that layer; the same for view
    layers;
  - a head's output gradient (d_raw_head, d_raw_rgb, each narrow head's, d raw_grad_density): the draw operand of the
    head_bwd that writes that head's weight gradient from this level's input;
  - the trunk-top slab: the A operand of the DGRAD against the slab's weights; d vin: the output of the launch that
    writes it, snapshotted before the Ref-NeRF stage re-uses its columns;
  - a smooth activation's T, u, trunk-top gradient before the second-order term, and second-order term g: the
    operands and output of the act_tangent_bwd launch that reads that layer's z;
  - the parameter gradients: the `grads` each clip_adam launch got, snapshotted there, read through the flax export.
Checks: every pinned stage output and every parameter-gradient leaf (Embed_0 included) with gemm_ref.check; mask
bits with check_bits; feature and view-input copies bit for bit; padding columns of the features, the view input and
d vin, and padding rows of every gradient master, exactly 0.  Teeth on the recorded data: in every stage check at
least 75 % of the nonzero elements have bound <= 2^-5 |value| (d vin, a sum of parts that cancel, is the loosest), and
every contribution (each level's share of a leaf, each term of the trunk-top gradient, each part of d vin) reaches 16
bounds somewhere (4 for a head bias, a head gradient summed over every sample; the level and tangent shares of the
leaves of an MLP with density normals are printed, not asserted: see the test).

The case table is test_level_reference_cpu.CASES, which says which layout reaches which stage.
"""
import numpy as np
import pytest
import torch

import gemm_ref as G
import level_ref as LR
from launch_recorder import Recorder
from test_level_reference_cpu import CASES, _bundle, modules

pytestmark = pytest.mark.gpu

OPS = ('gemm', 'gemm_wgrad', 'head_bwd', 'act_tangent_bwd', 'clip_adam')
BF_INT = torch.int16


def _same_bits(a, b, what):
  assert torch.equal(a.contiguous().view(BF_INT), b.contiguous().view(BF_INT)), f'{what}: not bit for bit equal'


def _one(rec, fn, **ptrs):
  calls = rec.of(fn, **ptrs)
  assert len(calls) == 1, f'{len(calls)} {fn} launches with {sorted(ptrs)} of this level'
  return calls[0]


def pinned(model, st, rec, rays_cam):
  """The stored tensors of one level, named as level_ref reads and checks them; asserts copies and padding.  Forward
  tensors are the level's buffers; every gradient is the operand (or output) a recorded launch saw."""
  mlp = model.mlps[st.mname]
  plan, g = mlp.plan, mlp.grads
  W, M = plan.cfg.net_width, st.M
  trunk = plan.by_role('trunk')
  P = {'feat': st.feat[:, :plan.F]}
  assert not st.feat[:, plan.F:].float().any(), 'feature padding columns are not 0'
  for c in st.feat_copies:
    _same_bits(c, st.feat, 'feature copy')
  if plan.density_normals:
    P['tfeat'] = st.tfeat[:, :plan.F]
    assert not st.tfeat[:, plan.F:].float().any(), 'tangent feature padding columns are not 0'
    for c in st.tfeat_copies:
      _same_bits(c, st.tfeat, 'tangent feature copy')
    P['rgd'] = st.rgd.view(3 * M, 1)
    P['d_rgd'] = _one(rec, 'head_bwd', x=st.t_last, dw=mlp.W(plan.one('density'), g)).before['draw'].view(-1)
  smooth2 = plan.density_normals and not st.bits
  for i in range(len(trunk)):
    P[('out', i)] = st.acts[i][:, :W]
    if st.bits:
      P[('bits', i)] = st.bits[i]
    else:
      P[('z', i)] = st.zs[i]
    xin = st.feat if i == 0 else st.acts[i - 1]
    P[('dy', i)] = _one(rec, 'gemm_wgrad', out=mlp.W(trunk[i], g), x=xin).before['dy']
    if plan.density_normals:
      P[('tout', i)] = st.tacts[i][:, :W]
      tin = st.tfeat if i == 0 else st.tacts[i - 1]
      P[('h', i)] = _one(rec, 'gemm', out=mlp.W(trunk[i], g), a=tin).before['b']
    if smooth2:
      c = _one(rec, 'act_tangent_bwd', z=st.zs[i])
      P[('T', i)], P[('u', i)] = c.before['t_adj'], c.before['u']
      if i == len(trunk) - 1:
        P['dy_top'] = c.before['g']
      else:
        P[('g', i)] = c.after['g']
  P['raw_head'] = st.raw_head
  d = plan.one('density')
  P['d_raw_head'] = _one(rec, 'head_bwd', x=st.x_last, dw=mlp.W(d, g)).before['draw']
  for sp in plan.narrow:
    P[('head', sp.role)] = st.heads[sp.role]
    P[('dhead', sp.role)] = _one(rec, 'head_bwd', x=st.x_last, dw=mlp.W(sp, g)).before['draw']
  if plan.slab_cols:
    slab = _one(rec, 'gemm', b=mlp.wcat_kn, a=st.bwd.d_vin if plan.top == 'view' else st.bwd.dhead).before['a']
    for sp, c0 in plan.slab_heads:
      P[('slab', sp.role)] = slab[:, c0:c0 + sp.out_dim]
    if plan.ref_stage and plan.has_bottleneck:
      P[('slab', 'bottleneck')] = slab[:, :plan.enc_col0]
  if plan.top == 'view':
    bw, V = plan.enc_col0, plan.vin_dim
    vin = st.vin[:, :V]
    assert not st.vin[:, V:].float().any(), 'view input padding columns are not 0'
    for c in st.vin_copies:
      _same_bits(c, st.vin, 'view input copy')
    P.update(vin=vin, dir_enc=vin[:, bw:plan.glo_col0], cam=rays_cam.repeat_interleave(st.S),
             raw_rgb=st.raw_rgb.view(M, 3))
    if bw:
      P['vin_bottleneck'] = vin[:, :bw]
    if plan.glo_features:
      P['vin_glo'] = vin[:, plan.glo_col0:]
    r = plan.one('rgb')
    P['d_raw_rgb'] = _one(rec, 'head_bwd', x=st.v_last, dw=mlp.W(r, g)).before['draw']
    views = plan.by_role('view')
    Wv = plan.cfg.net_width_viewdirs
    for i in range(len(views)):
      P[('vout', i)] = st.vacts[i][:, :Wv]
      if st.vbits:
        P[('vbits', i)] = st.vbits[i]
      else:
        P[('vz', i)] = st.vzs[i]
      xin = st.vin if i == 0 else st.vacts[i - 1]
      P[('dv', i)] = _one(rec, 'gemm', out=mlp.W(views[i], g), a=xin).before['b']
    # d vin as the view MLP's last launch wrote it (the Ref-NeRF stage later re-uses its columns)
    dv = rec.of('gemm', out=st.bwd.d_vin) + rec.of('head_bwd', dx=st.bwd.d_vin)
    assert len(dv) == 1, f'{len(dv)} launches write d vin'
    d_vin = dv[0].after['out' if dv[0].fn == 'gemm' else 'dx']
    cols = V if (plan.glo_features or plan.ref_stage) else bw
    P['d_vin'] = d_vin[:, :cols]
    assert not d_vin[:, V:].float().any(), 'd vin padding columns are not 0'
  return P


@pytest.fixture(scope='module')
def mods():
  from multinerf_b200 import lib, models, ops, train_utils, utils
  lib.require_device()
  return models, ops, train_utils, utils


@pytest.mark.parametrize('name', list(CASES))
def test_train_step_level_stages(mods, monkeypatch, name):
  from model_parity import level_jitter, synth_rays
  models, ops, train_utils, utils = mods
  bundle = _bundle(name)
  bundle.config.grad_max_norm = bundle.config.grad_max_val = 0.0
  B = 96
  rays, rng = synth_rays(91, B, 2.0, 6.0, unit_cube=False)
  m = bundle.model
  if m.num_glo_features:
    rays.cam_idx = rng.integers(0, m.num_glo_embeddings, (B, 1)).astype(np.int32)
  target = rng.uniform(0, 1, (B, 3)).astype(np.float32)
  rand = level_jitter(rng, bundle, B)
  model, variables = models.construct_model(92, rays, bundle)
  tree0 = model.export_flax()
  rec = Recorder(ops, OPS, monkeypatch)
  step_fn = train_utils.create_train_step(model, bundle.config, use_graph=False)
  step_fn(rand, train_utils.TrainState(variables), utils.Batch(rays=rays, rgb=target), None, 0.5)
  torch.cuda.synchronize()
  monkeypatch.undo()

  params = model.params
  grads = torch.zeros_like(params.grads)
  for name_ in params.offsets:
    seg = params.seg(name_, params.grads)
    calls = rec.of('clip_adam', grads=seg)
    assert len(calls) == 1, f'{len(calls)} clip_adam launches for {name_}'
    params.seg(name_, grads).copy_(calls[0].before['grads'])
  got = model._export(grads)
  for mname, plan in model.plans.items():
    seg = params.seg(mname, grads)
    for sp in plan.specs:
      if sp.row_map is not None or sp.in_pad != sp.in_dim:
        rows = np.ones(sp.in_pad, bool)
        rows[sp.row_map if sp.row_map is not None else np.arange(sp.in_dim)] = False
        assert not model.mlps[mname].W(sp, seg)[torch.from_numpy(rows)].any(), f'{mname} {sp.name}: padding rows'

  cam = torch.as_tensor(rays.cam_idx[:, 0]).long().cuda()
  states = sorted(((k[0], st) for k, st in model._levels.items() if isinstance(k[0], int)), key=lambda t: t[0])
  worst, nchecks = {}, 0
  tight, least, leaf_tight = (1.0, ''), (float('inf'), ''), (1.0, '')
  unresolved = (float('inf'), '')
  for mname, cfg, use_viewdirs, glo, nlev in modules(bundle):
    embed = torch.as_tensor(tree0['Embed_0']['embedding']).cuda() if glo else None
    refs = []
    for lv, st in states:
      if st.mname != mname:
        continue
      P = pinned(model, st, rec, cam)
      stored = dict(P)
      R = LR.level(tree0[mname], cfg, P, use_viewdirs=use_viewdirs, embed=embed)
      worst[f'{mname} level {lv}'] = LR.check_level(R, stored, f'{name} {mname} level {lv}')
      for key, (v, b) in R.checks.items():
        frac, ratio = LR.teeth(v, b, R.terms.get(key, []), f'{name} {mname} level {lv} {key}')
        tight = min(tight, (frac, str(key)))
        least = min(least, (ratio, f'{key}'))
        nchecks += 1
      refs.append(R)
    assert len(refs) == nlev, f'{mname}: {len(refs)} levels for {nlev}'
    leaves, eacc, terms = LR.sum_levels(refs)
    flat = {(n, k): v for n, p in got[mname].items() for k, v in p.items()}
    assert set(flat) == set(leaves), f'{mname}: leaves {sorted(set(flat) ^ set(leaves))}'
    worst[f'{mname} leaves'] = LR.check_leaves(leaves, flat, f'{name} {mname}')
    for key, acc in leaves.items():
      # a leaf sums signed terms over every sample of every level and its bound is relative to the sum of their
      # sizes, so how many elements are tight says little (bias gradients cancel to 40 % and less): the leaves keep
      # the per-contribution test alone.  A head bias (one to four elements, each a head gradient summed over every
      # sample) can cancel to a few bounds: each level's share of it must still move it by 4.
      # Under density normals a leaf sums primal shares and tangent shares (tin^T h, 3M rows per level); at the
      # bundles' normal-loss weights a tangent share, or a coarse level's share of a narrow head's bias, is 0.4 to 4
      # bounds of the whole, below what an fp32 sum in any order resolves.  Those modules' shares are printed, not
      # asserted; the tangent stages themselves (h, T, u, g, the trunk-top terms) keep every assertion.
      normals = model.plans[mname].density_normals
      frac, ratio = LR.teeth(acc.value, acc.bound(), terms[key], f'{name} {mname} {key}', tight=0,
                             ratio=0 if normals else 4.0 if acc.value.numel() <= 4 else 16.0)
      if normals:
        unresolved = min(unresolved, (ratio, f'{mname} {key}'))
        continue
      leaf_tight = min(leaf_tight, (frac, f'{mname} {key}'))
      least = min(least, (ratio, f'{mname} {key}'))
    if eacc is not None:
      e = torch.as_tensor(got['Embed_0']['embedding']).cuda()
      worst['Embed_0'] = G.check(e, eacc.value, eacc.bound(), f'{name} Embed_0')
      LR.teeth(eacc.value, eacc.bound(), [('GLO', eacc.value)], f'{name} Embed_0')
  if 'Embed_0' in got and not any(glo for *_, glo, _ in modules(bundle)):
    assert not np.any(got['Embed_0']['embedding']), 'GLO vectors no layer reads got a gradient'
  print(f'\n{name}: {nchecks} stage checks | worst err/bound ' + ', '.join(f'{k} {v:.3f}' for k, v in worst.items()) +
        f' | tightest fraction: stages {tight[0]:.2f} ({tight[1]}), leaves {leaf_tight[0]:.2f} ({leaf_tight[1]})'
        f' | smallest contribution/bound {least[0]:.3g} ({least[1]})' +
        (f' | smallest leaf share under density normals {unresolved[0]:.3g} ({unresolved[1]})'
         if unresolved[1] else ''))
