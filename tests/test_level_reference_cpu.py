"""tests/level_ref.py, the fp64 reference of one level's MLP, checked without a GPU.

Composition: run unpinned (each stage fed the reference's own previous output), the reference is the MLP the flax
model defines: its head outputs, raw_grad_density and every parameter gradient equal torch.autograd (create_graph
for the density normals, so the second-order term included) through oracle/o_models.mlp_apply (bf16=False) in
float64 on the same features, kernels and GLO vectors (all bf16-representable, so the bf16 rounding of the kernels
changes nothing), to 1e-9 of the largest element.  The oracle's encoder is replaced by an affine map of the means, so
the feature tangents are known exactly; the head gradients level_ref takes as given are autograd's totals.  Both sides are float64 sums of a few hundred terms of
size about 1 (error near 1e-13 of the largest term); a dropped or misrouted contribution moves a leaf by far more.

Soundness and teeth: an emulation of what models.py stores passes every check of the pinned reference.  For layouts
without normals or narrow heads it is an fp32 restatement of models.py (fp32 products summed in another order, bf16
wherever a buffer is bf16, d vin's partial sums stored in bf16, each module's leaves summed over its levels); for the
others, the reference's own stage outputs kept in the buffers' precision.  Single mutations of the emulation, each a
wiring mistake the model could make, fail a check.
"""
import dataclasses

import numpy as np
import pytest
import torch

import gemm_ref as G
import level_ref as LR
from model_parity import mini360, mini_refnerf
from oracle import o_coord, o_models
from test_gpu_view_branch import mini_view_independent
from test_gpu_view_layouts import mini_layout

BF = torch.bfloat16


def _bundle(name):
  base, _, act = name.partition('-')
  b = {'mini360': mini360, 'mini_refnerf': mini_refnerf, 'view_independent': mini_view_independent,
       'view_independent_plain': lambda: mini_view_independent(normals=False)}.get(base)
  b = b() if b else mini_layout(base)
  if act:
    b.nerf_mlp.net_activation = b.prop_mlp.net_activation = act
  return b


# which layout reaches which stage (the GPU suite runs the same table)
CASES = {
    'mini360': 'ReLU, per-layer trunk with a skip, PropMLP shared by 2 levels, view MLP of one layer',
    'mini360-softplus': 'stored z, smooth DGRAD',
    'mini360-silu': 'stored z, smooth DGRAD',
    'mini_refnerf-relu': 'Ref-NeRF slab DGRAD, narrow heads, tangents, single_mlp',
    'mini_refnerf-silu': 'the same with the second-order term of a smooth activation',
    'skips': 'chained 256-wide trunk, GLO, view skips, a tail rgb head',
    'depth0_glo': "an 'all' rgb head, GLO",
    'no_bottleneck': 'Ref-NeRF slab without a bottleneck, colourless normals slab on the PropMLP',
    'depth0_no_bottleneck': "the same with an 'all' rgb head",
    'skips-silu': 'per-layer 256-wide trunk, smooth view DGRAD',
    'view_independent': 'stacked head with dw_split, colourless normals slab, heads reading [hidden | features]',
    'view_independent_plain': 'stacked head without normals',
}


def modules(bundle):
  """(name, MLPConfig, use_viewdirs, GLO width, levels that run it) of each MLP of the bundle."""
  m = bundle.model
  nprop = 0 if m.single_mlp else m.num_levels - 1
  glo = m.num_glo_features if m.use_viewdirs else 0       # without a view branch no layer reads GLO
  out = [('NerfMLP_0', bundle.nerf_mlp, m.use_viewdirs, glo, m.num_levels - nprop)]
  if nprop:
    out.append(('PropMLP_0', bundle.prop_mlp, m.use_viewdirs, 0, nprop))
  return out


def _bf(t):
  return t.to(BF).double()


def enc_dim(cfg):
  """Width of the view input's columns between the bottleneck and GLO: the direction encoding (and n.v)."""
  if cfg.use_directional_enc:
    e = o_coord.generate_ide_fn(cfg.deg_view)(torch.tensor([[0.0, 0.0, 1.0]]), torch.ones(1, 1)).shape[-1]
  else:
    e = 3 + 6 * cfg.deg_view
  return e + (1 if cfg.use_n_dot_v else 0)


def make_tree(cfg, lay, F, V, gen):
  """A flax tree with bf16-representable kernels and fp32 biases, widths as the layout reads them."""
  W = cfg.net_width
  shapes = {}
  x = F
  for i, n in enumerate(lay['trunk']):
    shapes[n] = (x, W)
    x = W + F if i in lay['skip'] else W
  shapes[lay['density']] = (x, 1)
  for name, n in lay['narrow'].values():
    shapes[name] = (x, n)
  if lay['top'] == 'stacked':
    shapes[lay['rgb']] = (x, 3)
  elif lay['top'] == 'view':
    if 'bottleneck' in lay:
      shapes[lay['bottleneck']] = (x, cfg.bottleneck_width)
    Wv, v = cfg.net_width_viewdirs, V
    for i, n in enumerate(lay['view']):
      shapes[n] = (v, Wv)
      v = Wv + V if i in lay['vskip'] else Wv
    shapes[lay['rgb']] = (v, 3)
  return {n: {'kernel': _bf(torch.randn(*s, generator=gen, dtype=torch.float64) * (1.5 / s[0]) ** 0.5),
              'bias': (torch.randn(s[1], generator=gen) * 0.1).double()} for n, s in shapes.items()}


def _inputs(cfg, lay, B, S, gen, F=40, glo=0):
  """The tensors level_ref always takes as given (encoder, Ref-NeRF / normals stages, compositing), drawn at random."""
  M = B * S
  r = lambda *shape: torch.randn(*shape, generator=gen, dtype=torch.float64)
  P = {'feat': _bf(r(M, F))}
  P['d_raw_head'] = r(M, 4 if lay['top'] == 'stacked' else 1) / M
  if lay['normals']:
    P['tfeat'], P['d_rgd'] = _bf(r(3 * M, F)), r(3 * M) / M
  for role, (_, n) in lay['narrow'].items():
    P[('dhead', role)] = r(M, n) / M
  V = 0
  if lay['top'] == 'view':
    E = enc_dim(cfg)
    P['dir_enc'] = _bf(torch.rand(M, E, generator=gen, dtype=torch.float64) * 2 - 1)
    P['d_raw_rgb'] = r(M, 3) / M
    P['cam'] = torch.randint(0, 3, (B,), generator=gen).repeat_interleave(S)
    V = max(cfg.bottleneck_width, 0) + E + glo
  return P, V


# ------------------------------------------------------------------ composition against oracle autograd

@pytest.mark.parametrize('name', list(CASES))
def test_composition_matches_oracle_autograd(name, monkeypatch):
  bundle = _bundle(name)
  gen = torch.Generator().manual_seed(sum(name.encode()))
  B, S, F = 3, 8, 40
  M = B * S
  r = lambda *shape: torch.randn(*shape, generator=gen, dtype=torch.float64)
  for mname, cfg0, use_viewdirs, glo, _ in modules(bundle):
    cfg = dataclasses.replace(cfg0, warp_fn=None, density_noise=0.0, bottleneck_noise=0.0)
    lay = LR.layout(cfg, use_viewdirs, glo)
    tree = make_tree(cfg, lay, F, _inputs(cfg, lay, 1, 1, gen, F, glo)[1], gen)
    embed = _bf(r(3, glo)) if glo else None
    cam = torch.randint(0, 3, (B,), generator=gen)
    # the oracle's encoder replaced by an affine map of the means, feat = mean A + C, so the tangents are the rows
    # of A; every Dense layer's input and output recorded
    A, C = r(3, F), r(B, S, F)
    calls, dense = {}, o_models._Dense.__call__

    def record(self, x):
      y = dense(self, x)
      calls[f'Dense_{self.k - 1}'] = (x, y)
      return y
    monkeypatch.setattr(o_coord, 'lift_and_diagonalize', lambda m, c, b: (m @ A + C, c))
    monkeypatch.setattr(o_coord, 'integrated_pos_enc', lambda m, v, a, b: m)
    monkeypatch.setattr(o_models._Dense, '__call__', record)
    ttree = {n: {k: t.clone().requires_grad_(True) for k, t in p.items()} for n, p in tree.items()}
    emb = embed.clone().requires_grad_(True) if glo else None
    viewdirs = torch.nn.functional.normalize(r(B, 3), dim=-1)
    means = r(B, S, 3)
    out = o_models.mlp_apply(ttree, cfg, np.zeros((1, 3)), (means, torch.zeros(B, S, 3, 3, dtype=torch.float64)),
                             viewdirs=viewdirs if use_viewdirs else None, glo_vec=emb[cam] if glo else None)
    monkeypatch.undo()
    # a loss on every head output and on raw_grad_density; its gradients w.r.t. them are the totals (through the
    # Ref-NeRF stage and the view MLP too) that the model's normals and Ref-NeRF backward hand the MLP
    heads = {'density': lay['density']}
    heads.update({role: nm for role, (nm, _) in lay['narrow'].items()})
    if 'rgb' in lay:
      heads['rgb'] = lay['rgb']
    outs = {role: calls[nm][1] for role, nm in heads.items()}
    if lay['normals']:
      outs['rgd'] = out['raw_grad_density']
    loss = sum((o * r(*o.shape)).sum() for o in outs.values())
    leaves = [t for p in ttree.values() for t in p.values()] + ([emb] if glo else [])
    grads = torch.autograd.grad(loss, leaves, retain_graph=True)
    tot = dict(zip(outs, torch.autograd.grad(loss, list(outs.values()))))
    flat = lambda t: t.detach().reshape(M, -1)
    P = {'feat': flat(means @ A + C), 'cam': cam.repeat_interleave(S)}
    if lay['normals']:
      P['tfeat'] = A.repeat_interleave(M, 0)
      P['d_rgd'] = tot['rgd'].detach().reshape(M, 3).T.reshape(-1)
    P['d_raw_head'] = flat(tot['density'])
    if lay['top'] == 'stacked':
      P['d_raw_head'] = torch.cat([P['d_raw_head'], flat(tot['rgb'])], 1)
    elif lay['top'] == 'view':
      P['d_raw_rgb'] = flat(tot['rgb'])
      first = lay['view'][0] if lay['view'] else lay['rgb']
      bw = max(cfg.bottleneck_width, 0)
      P['dir_enc'] = flat(calls[first][0])[:, bw:bw + enc_dim(cfg)]
    for role in lay['narrow']:
      P[('dhead', role)] = flat(tot[role])
    R = LR.level(tree, cfg, P, use_viewdirs=use_viewdirs, embed=embed)

    def close(a, b, what):
      a, b = a.double().reshape(b.shape), b.double()
      tol = 1e-9 * max(1.0, float(b.abs().max()))
      assert float((a - b).abs().max()) <= tol, f'{name} {mname} {what}: {float((a - b).abs().max()):.3g} > {tol:.3g}'
    close(R.checks['raw_head'][0], torch.cat([flat(calls[n][1]) for n in
                                              [lay['density']] + ([lay['rgb']] if lay['top'] == 'stacked' else [])], 1),
          'density (stacked) head')
    for role, (nm, _) in lay['narrow'].items():
      close(R.checks[('head', role)][0], flat(calls[nm][1]), role)
    if lay['top'] == 'view':
      close(R.checks['raw_rgb'][0], flat(calls[lay['rgb']][1]), 'rgb head')
    if lay['normals']:
      close(R.checks['rgd'][0].reshape(3, M).T, flat(out['raw_grad_density']), 'raw_grad_density')
    k = 0
    for n, p in ttree.items():
      for kind in p:
        close(R.leaves[(n, kind)].value, grads[k], f'{n} {kind}')
        k += 1
    assert len(R.leaves) == k, sorted(set(R.leaves) - {(n, kd) for n, p in ttree.items() for kd in p})
    if glo:
      close(R.embed.value, grads[-1], 'Embed_0')


# ------------------------------------------------------------------ the stored tensors, emulated

MUTATIONS = {
    'view_skip_part': 'skips',          # the d vin part of a view layer after a skip is dropped
    'level_share': 'mini360',           # one of the two PropMLP levels adds no weight gradient
    'swap_slots': 'view_independent_plain',  # the stacked head's rgb slots 0 and 1 swap in its weight gradient
    'bias_buffer': 'mini360',           # a trunk bias gradient sums the dy of the layer below
    'density_term': 'mini360',          # the density head's term of the trunk-top gradient is dropped
    'narrow_term': 'mini_refnerf-relu',  # the diffuse head's term of the trunk-top gradient is dropped
    'second_order': 'mini_refnerf-silu',  # the second-order term is not added into the trunk-top gradient
    'tangent_wgrad': 'mini_refnerf-relu',  # one trunk layer's tangent weight gradient is not added
}


def _f32mm(a, b):
  """fp32 product summed in another order than the reference's: K reversed."""
  return a.float().flip(1) @ b.float().flip(0)


def _act32(code, z):
  return G.act(code, z.double()).float()


def emulate(tree, cfg, lay, P, mut=None):
  """What models.py stores for one level, in fp32 with bf16 stores: fills P (the keys level_ref reads and checks),
  returns the level's leaf gradients {(layer, kind): fp32} and its GLO gradient."""
  act = lay['act']
  W = cfg.net_width
  k = {n: torch.as_tensor(p['kernel']).float().to(BF).float() for n, p in tree.items()}
  b = {n: torch.as_tensor(p['bias']).float() for n, p in tree.items()}
  leaves = {}

  def add(key, v):
    leaves[key] = leaves.get(key, 0) + v

  def d1(z):
    return (z > 0).float() if act == G.RELU else G.act_d1(act, z.double()).float()
  feat = P['feat'].float()
  x, xin, zs = feat, [], []
  for i, n in enumerate(lay['trunk']):
    xin.append(x)
    z = _f32mm(x, k[n]) + b[n]
    zs.append(z.to(BF).float() if act != G.RELU else z)
    P[('out', i)] = _act32(act, z).to(BF).float()
    if act == G.RELU:
      P[('bits', i)] = G.pack_bits(z > 0)
    else:
      P[('z', i)] = z.to(BF).float()
    x = torch.cat([P[('out', i)], feat], 1) if i in lay['skip'] else P[('out', i)]
  x_last, last = x, len(xin) - 1
  heads = [lay['density']] + ([lay['rgb']] if lay['top'] == 'stacked' else [])
  wh = torch.cat([k[n] for n in heads], 1)
  P['raw_head'] = _f32mm(x_last, wh) + torch.cat([b[n] for n in heads])
  fz = d1(zs[last])
  if lay['top'] == 'view':
    bn = lay['bottleneck']
    bw = k[bn].shape[1]
    vin = [(_f32mm(x_last, k[bn]) + b[bn]).to(BF).float(), P['dir_enc'].float()]
    if 'embed' in P:
      vin.append(P['embed'].float().to(BF).float()[P['cam']])
    vin = torch.cat(vin, 1)
    P['vin'], P['vin_bottleneck'] = vin, vin[:, :bw]
    if 'embed' in P:
      P['vin_glo'] = vin[:, -P['embed'].shape[1]:]
    v, vxin, vz = vin, [], []
    for i, n in enumerate(lay['view']):
      vxin.append(v)
      z = _f32mm(v, k[n]) + b[n]
      vz.append(z.to(BF).float() if act != G.RELU else z)
      P[('vout', i)] = _act32(act, z).to(BF).float()
      if act == G.RELU:
        P[('vbits', i)] = G.pack_bits(z > 0)
      else:
        P[('vz', i)] = z.to(BF).float()
      v = torch.cat([P[('vout', i)], vin], 1) if i in lay['vskip'] else P[('vout', i)]
    rg = lay['rgb']
    P['raw_rgb'] = _f32mm(v, k[rg]) + b[rg]
    d_rgb = P['d_raw_rgb'].float()
    add((rg, 'kernel'), _f32mm(v.T, d_rgb))
    add((rg, 'bias'), d_rgb.sum(0))
    nv = len(lay['view'])
    if nv == 0:
      d_vin = (_f32mm(d_rgb, k[rg].T)).to(BF).float()
    else:
      Wv = k[lay['view'][0]].shape[1]
      t = _f32mm(d_rgb, k[rg].T)
      dcur = t[:, :Wv] * d1(vz[-1])
      add((lay['view'][-1], 'bias'), dcur.sum(0))
      part = t[:, Wv:].to(BF).float() if (nv - 1) in lay['vskip'] else None
      dcur = dcur.to(BF).float()
      P[('dv', nv - 1)] = dcur
      for i in range(nv - 1, 0, -1):
        n = lay['view'][i]
        add((n, 'kernel'), _f32mm(vxin[i].T, dcur))
        if (i - 1) in lay['vskip'] and mut != 'view_skip_part':
          p = _f32mm(dcur, k[n][Wv:].T)
          part = (p if part is None else p + part).to(BF).float()
        nxt = _f32mm(dcur, k[n][:Wv].T) * d1(vz[i - 1])
        add((lay['view'][i - 1], 'bias'), nxt.sum(0))
        dcur = nxt.to(BF).float()
        P[('dv', i - 1)] = dcur
      add((lay['view'][0], 'kernel'), _f32mm(vxin[0].T, dcur))
      d_vin = _f32mm(dcur, k[lay['view'][0]].T)
      d_vin = (d_vin + part if part is not None else d_vin).to(BF).float()
    cols = vin.shape[1] if 'embed' in P else bw
    P['d_vin'] = d_vin[:, :cols]
    embed_g = None
    if 'embed' in P:
      g = P['embed'].shape[1]
      embed_g = torch.zeros(P['embed'].shape).index_add_(0, P['cam'], d_vin[:, -g:])
    dr = P['d_raw_head'][:, 0].float()
    add((bn, 'kernel'), _f32mm(x_last.T, d_vin[:, :bw]))
    add((bn, 'bias'), d_vin[:, :bw].sum(0))
    add((lay['density'], 'kernel'), _f32mm(x_last.T, dr[:, None]))
    add((lay['density'], 'bias'), dr.sum(0, keepdim=True))
    top = _f32mm(d_vin[:, :bw], k[bn][:W].T)
    if mut != 'density_term':
      top = top + dr[:, None] * k[lay['density']][:W, 0][None, :]
    P[('dy', last)] = (top * fz).to(BF).float()
  else:
    embed_g = None
    dh = P['d_raw_head'].float()
    P[('dy', last)] = (_f32mm(dh, wh[:W].T) * fz).to(BF).float()
    dhw = dh[:, [0, 2, 1, 3]] if mut == 'swap_slots' else dh
    dw = _f32mm(x_last.T, dhw)
    db = dh.sum(0)
    for j, n in enumerate(heads):
      cols = slice(0, 1) if j == 0 else slice(1, dh.shape[1])
      add((n, 'kernel'), dw[:, cols])
      add((n, 'bias'), db[cols])
  for i in range(last, -1, -1):
    n = lay['trunk'][i]
    dy = P[('dy', i)]
    add((n, 'kernel'), _f32mm(xin[i].T, dy))
    add((n, 'bias'), dy.sum(0))
    if i > 0:
      P[('dy', i - 1)] = (_f32mm(dy, k[n][:W].T) * d1(zs[i - 1])).to(BF).float()
  if mut == 'bias_buffer':
    # the last trunk layer's bias gradient summed from the dy of the layer below instead of its own
    leaves[(lay['trunk'][last], 'bias')] = P[('dy', last - 1)].sum(0)
  return leaves, embed_g


def emulate_rounded(tree, cfg, lay, P, use_viewdirs, embed, mut=None):
  """What models.py stores for one level, as the reference's own stage outputs kept in the buffers' precision: each
  bf16 stage output rounded to bf16 before the stages after it read it, fp32 outputs and leaves rounded to fp32.
  Covers the stages the fp32 emulation does not (tangents, narrow heads, the slabs).  Fills P; returns the level's
  leaves and GLO gradient."""
  R = LR.level(tree, cfg, P, use_viewdirs=use_viewdirs, embed=embed, store=lambda k, v: v.to(BF).double())
  for key, (v, _) in R.checks.items():
    if key not in P:
      P[key] = v.float()
  for key, (z, _) in R.bits.items():
    P[('vbits', key[1]) if isinstance(key, tuple) else ('bits', key)] = G.pack_bits(z > 0)
  if 'vin' in P:
    bw = max(cfg.bottleneck_width, 0)
    P['vin_bottleneck'] = P['vin'][:, :bw]
    if embed is not None:
      P['vin_glo'] = P['vin'][:, -embed.shape[1]:]
  leaves = {k: acc.value.float() for k, acc in R.leaves.items()}
  last = len(lay['trunk']) - 1
  if mut == 'narrow_term':
    P[('dy', last)] = (P[('dy', last)] - dict(R.terms[('dy', last)])['diffuse']).to(BF).double()
  elif mut == 'second_order':
    P[('dy', last)] = P['dy_top']
  elif mut == 'tangent_wgrad':
    key = (lay['trunk'][2], 'kernel')
    leaves[key] = leaves[key] - dict(R.terms[key])['tangent'].float()
  return leaves, None if R.embed is None else R.embed.value.float()


def run_emulated(name, mut=None, B=4, S=8):
  """Emulated levels of every module of a case, checked against the pinned reference.  Returns the worst ratio."""
  bundle = _bundle(name)
  gen = torch.Generator().manual_seed(sum(name.encode()) + 7)
  worst = 0.0
  for mname, cfg, use_viewdirs, glo, nlev in modules(bundle):
    lay = LR.layout(cfg, use_viewdirs, glo)
    refs, got, emb_got = [], {}, None
    embed = None
    for lv in range(nlev):
      P, V = _inputs(cfg, lay, B, S, gen, glo=glo)
      if lv == 0:
        tree = make_tree(cfg, lay, P['feat'].shape[1], V, gen)
        embed = _bf(torch.randn(3, glo, generator=gen, dtype=torch.float64)) if glo else None
      if embed is not None:
        P['embed'] = embed
      if lay['normals'] or lay['narrow'] or lay['slab']:
        leaves, emb = emulate_rounded(tree, cfg, lay, P, use_viewdirs, embed, mut)
      else:
        leaves, emb = emulate(tree, cfg, lay, P, mut)
      if not (mut == 'level_share' and lv == 1):
        for key, v in leaves.items():
          got[key] = got.get(key, 0) + v
      if emb is not None:
        emb_got = emb if emb_got is None else emb_got + emb
      R = LR.level(tree, cfg, P, use_viewdirs=use_viewdirs, embed=embed)
      worst = max(worst, LR.check_level(R, P, f'{name} {mname} level {lv}'))
      refs.append(R)
    leaves, eacc, _ = LR.sum_levels(refs)
    worst = max(worst, LR.check_leaves(leaves, got, f'{name} {mname}'))
    if eacc is not None:
      worst = max(worst, G.check(emb_got, eacc.value, eacc.bound(), f'{name} {mname} Embed_0'))
  return worst


@pytest.mark.parametrize('name', list(CASES))
def test_emulated_stored_tensors_pass(name):
  worst = run_emulated(name)
  print(f'\n{name}: worst err/bound {worst:.3f}')


@pytest.mark.parametrize('mut', list(MUTATIONS))
def test_mutation_fails_a_check(mut):
  with pytest.raises(AssertionError):
    run_emulated(MUTATIONS[mut], mut)
