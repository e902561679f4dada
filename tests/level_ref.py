"""fp64 reference of one level's MLP, stage by stage, with a bound on every element of every stage output.

`level(tree, cfg, P, use_viewdirs=..., embed=...)` follows the reference MLP (internal/models.py:402-612,
oracle/o_models.mlp_apply) on the flax tree `tree` of one module (`Model.export_flax()[name]`, taken before the
step) and a dict `P` of the tensors the GPU stored, named by meaning:

  feat             [M, F]   encoder features (bf16; always given: the encoder suite covers them)
  ('out', i)       [M, W]   stored output of trunk layer i (bf16)
  ('z', i)         [M, W]   stored pre-activation of trunk layer i (smooth activations, bf16)
  ('bits', i)      [M, W/32] ReLU mask words of trunk layer i (int32; absent: z > 0 of the reference)
  tfeat            [3M, F]  encoder tangents d feat / d mean, three streams stacked (density normals)
  ('tout', i)      [3M, W]  stored tangent stream of trunk layer i (bf16)
  dir_enc          [M, E]   the view input between the bottleneck and GLO: direction encoding or the Ref-NeRF
                            stage's columns, n.v included (always given: their own suites cover them)
  cam              [M]      camera index of every sample (GLO)
  vin              [M, V]   view input [bottleneck | dir enc | n.v | GLO], logical columns (bf16)
  ('vout', i), ('vz', i), ('vbits', i)   the same for view layer i
  d_raw_head       [M, 1 or 4] gradient of the density (or stacked [density | rgb]) head output, as its weight
                            gradient read it (fp32)
  ('dhead', role)  [M, n]   gradient of a narrow head's output (grad_pred, diffuse, tint, roughness; fp32)
  d_raw_rgb        [M, 3]   gradient of the rgb head output under a view branch (fp32)
  d_rgd            [3M]     gradient of raw_grad_density, stream-major (fp32)
  ('slab', role)   [M, n]   the trunk-top DGRAD's operand columns of one head (or the bottleneck) (bf16)
  dy_top           [M, W]   the trunk-top gradient before a smooth activation's second-order term (bf16)
  ('dy', i)        [M, W]   gradient w.r.t. the output of trunk layer i (bf16, as the layer's WGRAD read it)
  ('h', i)         [3M, W]  tangent adjoint of trunk layer i (bf16, as the layer's tangent WGRAD read it)
  ('T', i), ('u', i), ('g', i)   smooth activations: dL/d t_i, the recomputed u_i = t_{i-1} W_i and the
                            second-order term a''(z_i) sum_s T u (bf16)
  ('dv', i)        [M, Wv]  gradient w.r.t. the output of view layer i (bf16)
  d_vin            [M, V]   gradient w.r.t. the view input as the view MLP left it, logical columns (bf16)

Each stage reads its inputs from P; a stage output missing from P is filled with the reference's own value, so the
same code runs pinned (every stored tensor given: each stage's bound is one launch's rounding) and unpinned (only
feat, dir_enc, cam and the head gradients given: the fp64 MLP, for the composition test against oracle autograd).

Returns a `Level`: `checks[name] = (value, bound)` for every stage output the GPU stores, `bits[i]` = (z, bound) for
gemm_ref.check_bits, `leaves[(layer, 'kernel' | 'bias')]` and `embed` as `Acc` (a sum over launches and levels),
and `terms[name]` = the individual contributions a check or leaf adds, for the test that each one matters.

Bounds come from gemm_ref and heads_ref and hold for any summation order; where models.py stores a partial sum in
bf16 (the running sum of d vin), that rounding is added.  Kernels are rounded to bf16 as the GPU packs them; biases,
fp32 head gradients and GLO vectors are taken as they are.

Layouts: every layout MLPPlan builds: trunks of any depth and skips under ReLU, softplus or SiLU; the density, stacked
and narrow heads; density normals (tangent streams, adjoints, tangent weight gradients and the second-order term);
the Ref-NeRF and colourless normals slabs; view branches with or without a bottleneck, n.v and GLO, view skips and
'tail' or 'all' rgb heads.

Pure torch in float64: runs on the CPU or on CUDA tensors, and never imports multinerf_b200.
"""
import torch

import gemm_ref as G
import heads_ref as H
import tangent_ref as TR

ACTS = {'relu': G.RELU, 'softplus': G.SOFTPLUS, 'silu': G.SILU}


class Acc:
  """A sum of `n` fp32-accumulated terms whose absolute values sum to `absum`, plus `extra` error carried in by its
  terms: value and bound of any order of fp32 additions of all terms of all parts added together (gemm_ref.ref_wgrad's
  C_ACC (n + 2) 2^-23 sum |.| over the union)."""

  def __init__(self, value, n, absum, extra=0.0):
    self.value, self.n, self.absum, self.extra = value, n, absum, extra

  @staticmethod
  def wgrad(x, dy, bias=False):
    """(x^T dy [, colsum dy]) as gemm_wgrad / head_bwd sum them: one Acc each."""
    r = G.ref_wgrad(x, dy, bsum_init=torch.zeros(dy.shape[1], dtype=torch.float64, device=dy.device) if bias else None)
    unit = G.C_ACC * (x.shape[0] + 2) * 2.0 ** -23
    out = [Acc(r['out'][0], x.shape[0], r['out'][1] / unit)]
    if bias:
      out.append(Acc(r['bsum'][0], x.shape[0], r['bsum'][1] / unit))
    return out

  @staticmethod
  def colsum(value, pre_bound):
    """Column sums of an fp32 output known to within pre_bound before its bf16 rounding (DGRAD colsum, dxsum)."""
    return Acc(value.sum(0), value.shape[0], (value.abs() + pre_bound).sum(0), pre_bound.sum(0))

  def __add__(self, o):
    return Acc(self.value + o.value, self.n + o.n, self.absum + o.absum, self.extra + o.extra)

  def bound(self):
    # + 2^-126 per term: fp32 products and sums below the normal range may flush to zero (features of the highest
    # encoding degrees reach the bf16 subnormals)
    return self.extra + G.C_ACC * (self.n + 2) * 2.0 ** -23 * self.absum + self.n * 2.0 ** -126


class Level:
  def __init__(self):
    self.checks, self.bits, self.leaves, self.terms, self.embed = {}, {}, {}, {}, None

  def leaf(self, layer, kind, acc, label):
    key = (layer, kind)
    self.leaves[key] = acc if key not in self.leaves else self.leaves[key] + acc
    self.terms.setdefault(key, []).append((label, acc.value))


NARROW = ('grad_pred', 'diffuse', 'tint', 'roughness')


def layout(cfg, use_viewdirs, glo):
  """Layer names of the reference MLP (flax Dense creation order) and the stages level() runs for it."""
  if cfg.net_activation not in ACTS:
    raise NotImplementedError(f'net_activation {cfg.net_activation!r}')
  top = ('view' if use_viewdirs else 'stacked') if not cfg.disable_rgb else 'density'
  d, nv = cfg.net_depth, cfg.net_depth_viewdirs
  names = iter(f'Dense_{k}' for k in range(d + nv + 8))
  lay = dict(top=top, act=ACTS[cfg.net_activation], trunk=[next(names) for _ in range(d)], density=next(names),
             skip=[i for i in range(d) if i % cfg.skip_layer == 0 and i > 0], glo=glo if top == 'view' else 0,
             normals=not cfg.disable_density_normals, narrow={})
  if cfg.enable_pred_normals:
    lay['narrow']['grad_pred'] = (next(names), 3)
  slab = []
  if top == 'stacked':
    lay['rgb'] = next(names)
  elif top == 'view':
    for role, on, n in (('diffuse', cfg.use_diffuse_color, 3), ('tint', cfg.use_specular_tint, 3),
                        ('roughness', cfg.enable_pred_roughness, 1)):
      if on:
        lay['narrow'][role] = (next(names), n)
    if cfg.bottleneck_width > 0:
      lay['bottleneck'] = next(names)
    lay['view'] = [next(names) for _ in range(nv)]
    lay['rgb'] = next(names)
    lay['vskip'] = [i for i in range(nv) if i % cfg.skip_layer_dir == 0 and i > 0]
    ref = (cfg.enable_pred_normals or lay['normals'] or cfg.use_reflections or cfg.use_directional_enc or
           cfg.use_n_dot_v)
    if ref:      # the Ref-NeRF stage: one DGRAD over [d bottleneck | head gradients] at the trunk top
      slab = (['bottleneck'] if 'bottleneck' in lay else []) + ['density'] + list(lay['narrow'])
    lay['ref'] = ref
  if top != 'view' and cfg.enable_pred_normals:
    # the colourless normals stage: one DGRAD over [d raw_density | d grad_pred (| d raw_rgb)]
    slab = ['density', 'grad_pred'] + (['rgb'] if top == 'stacked' else [])
  lay['slab'] = slab
  return lay


def _dgrad_mask(P, kind, i, z, act, mask_mod=0):
  """ref_dgrad's activation-derivative arguments for the output of layer i (kind 'out' or 'vout')."""
  if act != G.RELU:
    return dict(z=P[('z' if kind == 'out' else 'vz', i)], act_code=act, mask_mod=mask_mod)
  bits = P.get(('bits' if kind == 'out' else 'vbits', i))
  return dict(maskbits=bits, mask_mod=mask_mod) if bits is not None else dict(mask=z, mask_mod=mask_mod)


def _store_id(key, value):
  return value


def level(tree, cfg, P, *, use_viewdirs=True, embed=None, store=_store_id):
  """store(key, value): the form in which an unpinned stage output is kept for the stages after it (identity: the
  fp64 MLP; a rounding to the buffer's dtype: an emulation of what the model stores)."""
  glo = 0 if embed is None else embed.shape[1]
  lay = layout(cfg, use_viewdirs, glo)
  act, top = lay['act'], lay['top']
  dev = P['feat'].device
  kern = {k: torch.as_tensor(v['kernel']).float().to(torch.bfloat16).to(dev) for k, v in tree.items()}
  bias = {k: torch.as_tensor(v['bias']).float().to(dev) for k, v in tree.items()}
  R = Level()

  def take(key, value):                     # a stored tensor, or the reference's value where nothing is pinned
    if key not in P:
      P[key] = store(key, value)
    return P[key]
  feat = P['feat']
  W = cfg.net_width
  M = feat.shape[0]

  # ---- trunk forward
  x, zs = feat, {}
  xin = []
  for i, name in enumerate(lay['trunk']):
    xin.append(x)
    r = G.ref_fwd(x, kern[name].T, bias=bias[name], act_code=act)
    R.checks[('out', i)] = (r['out'], r['out_bound'])
    if act == G.RELU:
      R.bits[i] = (r['z'], r['pre_bound'])
    else:
      R.checks[('z', i)] = (r['z'], r['z_bound'])
      take(('z', i), r['z'])
    zs[i] = r['z']
    h = take(('out', i), r['out'])
    x = torch.cat([h, feat], 1) if i in lay['skip'] else h
  x_last, last = x, len(lay['trunk']) - 1
  heads = [lay['density']] + ([lay['rgb']] if top == 'stacked' else [])
  w_head = torch.cat([kern[n].T for n in heads])
  R.checks['raw_head'] = H.head_fwd(x_last, w_head, torch.cat([bias[n] for n in heads]))
  for role, (name, _) in lay['narrow'].items():
    R.checks[('head', role)] = H.head_fwd(x_last, kern[name].T, bias[name])
  wd = kern[lay['density']][:W, 0]

  # ---- tangent streams t_i = a'(z_i) (t_{i-1} W_i), no bias, and raw_grad_density = t_last w_density
  if lay['normals']:
    tfeat = P['tfeat']
    t, tin = tfeat, []
    for i, name in enumerate(lay['trunk']):
      tin.append(t)
      r = G.ref_dgrad(t, kern[name].T, **_dgrad_mask(P, 'out', i, zs[i], act, M))
      R.checks[('tout', i)] = (r['out'], r['out_bound'])
      h = take(('tout', i), r['out'])
      t = torch.cat([h, tfeat], 1) if i in lay['skip'] else h
    t_last = t
    R.checks['rgd'] = H.head_fwd(t_last, kern[lay['density']].T)

  # ---- view branch forward and backward
  d_vin = None
  if top == 'view':
    bn = lay.get('bottleneck')
    bw = kern[bn].shape[1] if bn else 0
    parts = []
    if bn:
      r = G.ref_fwd(x_last, kern[bn].T, bias=bias[bn])
      parts.append(r['out'])
      R.checks['vin_bottleneck'] = (r['out'], r['out_bound'])
    parts.append(P['dir_enc'].double())
    if glo:
      gv = embed.to(torch.bfloat16).double().to(dev)[P['cam']]
      parts.append(gv)
      R.checks['vin_glo'] = (gv, torch.zeros_like(gv))         # bf16 of Embed_0[cam], exactly
    vin = take('vin', torch.cat(parts, 1))
    v, vxin = vin, []
    for i, name in enumerate(lay['view']):
      vxin.append(v)
      r = G.ref_fwd(v, kern[name].T, bias=bias[name], act_code=act)
      R.checks[('vout', i)] = (r['out'], r['out_bound'])
      if act == G.RELU:
        R.bits[('v', i)] = (r['z'], r['pre_bound'])
      else:
        R.checks[('vz', i)] = (r['z'], r['z_bound'])
        take(('vz', i), r['z'])
      zs[('v', i)] = r['z']
      h = take(('vout', i), r['out'])
      v = torch.cat([h, vin], 1) if i in lay['vskip'] else h
    rg = lay['rgb']
    R.checks['raw_rgb'] = H.head_fwd(v, kern[rg].T, bias[rg])
    _view_bwd(R, P, lay, kern, vin, v, vxin, zs, act, embed, take)
    d_vin = P['d_vin']
    dr = P['d_raw_head'][:, 0]
    if bn:
      for acc, kind in zip(Acc.wgrad(x_last, d_vin[:, :bw], bias=True), ('kernel', 'bias')):
        R.leaf(bn, kind, acc, 'primal')
    R.leaf(lay['density'], 'kernel', Acc.wgrad(x_last, dr[:, None])[0], 'primal')
    R.leaf(lay['density'], 'bias', Acc(dr.double().sum(0, keepdim=True), M, dr.double().abs().sum(0, True)), 'primal')
  else:
    dh = P['d_raw_head']
    dw, db = Acc.wgrad(x_last, dh, bias=True)
    for j, name in enumerate(heads):
      cols = slice(0, 1) if j == 0 else slice(1, dh.shape[1])
      R.leaf(name, 'kernel', Acc(dw.value[:, cols], dw.n, dw.absum[:, cols]), 'primal')
      R.leaf(name, 'bias', Acc(db.value[cols], db.n, db.absum[cols]), 'primal')
  for role, (name, _) in lay['narrow'].items():
    for acc, kind in zip(Acc.wgrad(x_last, P[('dhead', role)], bias=True), ('kernel', 'bias')):
      R.leaf(name, kind, acc, 'primal')

  # ---- trunk top: the gradient w.r.t. the last trunk layer's output, before the second-order term
  mask = _dgrad_mask(P, 'out', last, zs[last], act)
  top_key = 'dy_top' if (lay['normals'] and act != G.RELU) else ('dy', last)
  if lay['slab']:
    # a'(x_last) * sum over the slab's heads of d head @ W_head^T (hidden rows)
    src = {'bottleneck': lambda: d_vin[:, :bw], 'density': lambda: P['d_raw_head'][:, :1],
           'rgb': lambda: P['d_raw_head'][:, 1:4]}
    cols, ws = [], []
    for role in lay['slab']:
      c = take(('slab', role), src[role]() if role in src else P[('dhead', role)])
      name = lay['bottleneck'] if role == 'bottleneck' else (lay['narrow'][role][0] if role in lay['narrow']
                                                            else lay[role])
      cols.append(c)
      ws.append(kern[name][:W])
    r = G.ref_dgrad(torch.cat([c.double() for c in cols], 1), torch.cat(ws, 1), **mask)
    R.terms[top_key] = [(role, G.ref_dgrad(c, w_, **mask)['out']) for role, c, w_ in zip(lay['slab'], cols, ws)]
    topv = (r['out'], r['out_bound'])
  elif top == 'view':
    # a'(x_last) * (d bottleneck @ W_b^T + d_raw_density (x) w_density)
    r = G.ref_dgrad(d_vin[:, :bw], kern[bn][:W], rowv=dr, colv=wd.float(), **mask)
    only_b = G.ref_dgrad(d_vin[:, :bw], kern[bn][:W], **mask)['out']
    R.terms[top_key] = [('bottleneck', only_b), ('density head', r['out'] - only_b)]
    topv = (r['out'], r['out_bound'])
  else:
    # the density or stacked head's input gradient on the hidden columns
    topv = H.head_bwd(x_last, w_head, P['d_raw_head'], act=act, z=P.get(('z', last)), dx_cols=W)['dx']
  R.checks[top_key] = topv
  take(top_key, topv[0])

  # ---- tangent adjoints, their weight gradients, and the second-order term of a smooth activation
  if lay['normals']:
    d_rgd = P['d_rgd']                       # [3M], stream-major
    R.leaf(lay['density'], 'kernel', Acc.wgrad(t_last, d_rgd[:, None])[0], 'tangent')
    # d_rgd (x) w_density on the hidden columns (masked by the last layer's ReLU): one fp32 product, then bf16
    om = d_rgd.double()[:, None] * wd.double()[None, :]
    if act == G.RELU:
      bits = P.get(('bits', last))
      keep = G.unpack_bits(bits, W) if bits is not None else zs[last] > 0
      om = torch.where(keep.repeat(3, 1), om, 0.0)
    e = G.U * om.abs()
    R.checks[('T' if act != G.RELU else 'h', last)] = (om, e + G.half_ulp_bf16(om.abs() + e))
    take(('T' if act != G.RELU else 'h', last), om)
    for i in range(last, -1, -1):
      name = lay['trunk'][i]
      if act != G.RELU:
        r = G.ref_fwd(tin[i], kern[name].T)
        R.checks[('u', i)] = (r['out'], r['out_bound'])
        u = take(('u', i), r['out'])
        du, dub, g, gb = TR.act_tangent_ref(act, P[('z', i)], P[('T', i)], u, P['dy_top'] if i == last else None)
        R.checks[('h', i)] = (du, dub)
        take(('h', i), du)
        if i == last:
          R.checks[('dy', last)] = (g, gb)
          R.terms[('dy', last)] = [('second-order', g - P['dy_top'].double())]
          take(('dy', last), g)
        else:
          R.checks[('g', i)] = (g, gb)
          take(('g', i), g)
      h = P[('h', i)]
      if i > 0:
        if act != G.RELU:
          r = G.ref_dgrad(h, kern[name][:W])
          R.checks[('T', i - 1)] = (r['out'], r['out_bound'])
          take(('T', i - 1), r['out'])
        else:
          r = G.ref_dgrad(h, kern[name][:W], **_dgrad_mask(P, 'out', i - 1, zs[i - 1], act, M))
          R.checks[('h', i - 1)] = (r['out'], r['out_bound'])
          take(('h', i - 1), r['out'])

  # ---- trunk backward
  second = lay['normals'] and act != G.RELU
  for i in range(last, -1, -1):
    name = lay['trunk'][i]
    dy = P[('dy', i)]
    for acc, kind in zip(Acc.wgrad(xin[i], dy, bias=True), ('kernel', 'bias')):
      R.leaf(name, kind, acc, 'primal')
    if lay['normals']:
      R.leaf(name, 'kernel', Acc.wgrad(tin[i], P[('h', i)])[0], 'tangent')
    if i > 0:
      add = dict(addend=P[('g', i - 1)]) if second else {}
      r = G.ref_dgrad(dy, kern[name][:W], **_dgrad_mask(P, 'out', i - 1, zs[i - 1], act), **add)
      R.checks[('dy', i - 1)] = (r['out'], r['out_bound'])
      if second:
        R.terms[('dy', i - 1)] = [('second-order', P[('g', i - 1)].double())]
      take(('dy', i - 1), r['out'])
  return R


def _view_bwd(R, P, lay, kern, vin, v_last, vxin, zs, act, embed, take):
  """rgb head and view MLP backward: the view leaves, every ('dv', i) and d vin as the sum of its consumers' parts."""
  rg, views = lay['rgb'], lay['view']
  nv = len(views)
  d_rgb = P['d_raw_rgb']
  V = vin.shape[1]
  parts, n_stored = [], 0             # (label, value, pre_bound); bf16 partial sums models.py stores
  if nv == 0:                          # 'all': the rgb head reads vin
    hb = H.head_bwd(vin, kern[rg].T, d_rgb)
    parts.append(('rgb head', hb['dx'][0], hb['dx'][1]))
  else:
    Wv = kern[views[-1]].shape[1]
    tail = (nv - 1) in lay['vskip']
    hb = H.head_bwd(v_last, kern[rg].T, d_rgb, act=act, z=P.get(('vz', nv - 1)), dx_cols=Wv,
                    dxsum_init=torch.zeros(Wv, dtype=torch.float64, device=vin.device))
    R.checks[('dv', nv - 1)] = hb['dx']
    s, b = hb['dxsum']            # the last view layer's bias gradient: dxsum, added once into the leaf
    R.leaf(views[-1], 'bias', Acc(s, 1, s.abs() + b, extra=b), 'primal')
    if tail:
      # the head's input gradient past the hidden columns: the vin part of [hidden | vin]
      v2, e2 = hb['dx2']
      parts.append(('rgb head', v2, e2 - G.half_ulp_bf16(v2.abs())))
      n_stored += 1
    dcur = take(('dv', nv - 1), hb['dx'][0])
    for i in range(nv - 1, -1, -1):
      name = views[i]
      R.leaf(name, 'kernel', Acc.wgrad(vxin[i], dcur)[0], 'primal')
      if i == 0:
        r = G.ref_dgrad(dcur, kern[name])
        parts.append(('view 0', r['out'], r['pre_bound']))
        break
      if (i - 1) in lay['vskip']:    # layer i reads [hidden | vin]: its part of d vin
        r = G.ref_dgrad(dcur, kern[name][Wv:])
        parts.append((f'view {i}', r['out'], r['pre_bound']))
        n_stored += 1
      r = G.ref_dgrad(dcur, kern[name][:Wv], **_dgrad_mask(P, 'vout', i - 1, zs[('v', i - 1)], act))
      R.checks[('dv', i - 1)] = (r['out'], r['out_bound'])
      R.leaf(views[i - 1], 'bias', Acc.colsum(r['out'], r['pre_bound']), 'primal')
      dcur = take(('dv', i - 1), r['out'])
  for acc, kind in zip(Acc.wgrad(v_last if nv else vin, d_rgb, bias=True), ('kernel', 'bias')):
    R.leaf(rg, kind, acc, 'primal')
  # d vin: the parts in any order, each fp32 add rounded once, and every stored bf16 partial sum (the last part's
  # output included) rounded once more.  Only the columns a stage upstream reads are computed: the bottleneck's, and
  # with GLO or the Ref-NeRF stage every column.
  cols = V if (embed is not None or lay['ref']) else kern[lay['bottleneck']].shape[1]
  val = sum(p[1] for p in parts)[:, :cols]
  mag = sum(p[1].abs() + p[2] for p in parts)[:, :cols]
  e = sum(p[2] for p in parts)[:, :cols] + (len(parts) - 1) * G.U * mag
  e = e + (n_stored + 1) * G.half_ulp_bf16(mag)
  R.checks['d_vin'] = (val, e)
  R.terms['d_vin'] = [(p[0], p[1][:, :cols]) for p in parts]
  d_vin = take('d_vin', val)
  if embed is not None:
    glo = embed.shape[1]
    d = d_vin[:, V - glo:].double()
    cam = P['cam']
    val = torch.zeros(embed.shape, dtype=torch.float64, device=d.device).index_add_(0, cam, d)
    ab = torch.zeros(embed.shape, dtype=torch.float64, device=d.device).index_add_(0, cam, d.abs())
    R.embed = Acc(val, d.shape[0], ab)


# ---------------------------------------------------------------------------------------------- checks
def check_level(R, stored, what):
  """Every stage output of R against the stored tensors (same keys as R.checks, plus ('bits' | 'vbits', i) and the
  outputs they go with), gemm_ref.check and check_bits.  Returns the worst err / bound."""
  worst = 0.0
  for key, (v, b) in R.checks.items():
    worst = max(worst, G.check(stored[key], v, b, f'{what} {key}'))
  for key, (z, b) in R.bits.items():
    out, bits, i = ('vout', 'vbits', key[1]) if isinstance(key, tuple) else ('out', 'bits', key)
    G.check_bits(stored[(bits, i)], stored[(out, i)], z, b, f'{what} {bits} {i}')
  return worst


def sum_levels(refs):
  """Leaves and GLO gradient of one module summed over the levels that run it: ({key: Acc}, Acc or None, terms)."""
  leaves, terms, embed = {}, {}, None
  for j, R in enumerate(refs):
    for key, acc in R.leaves.items():
      leaves[key] = acc if key not in leaves else leaves[key] + acc
      terms.setdefault(key, []).extend((f'level {j} {lab}', v) for lab, v in R.terms[key])
    if R.embed is not None:
      embed = R.embed if embed is None else embed + R.embed
  return leaves, embed, terms


def check_leaves(leaves, got, what):
  """Every parameter-gradient leaf: got[(layer, kind)] (the flax export of the gradient) against its Acc."""
  worst = 0.0
  for key, acc in leaves.items():
    g = torch.as_tensor(got[key]).to(acc.value.device)
    worst = max(worst, G.check(g.reshape(acc.value.shape), acc.value, acc.bound(), f'{what} {key}'))
  return worst


def teeth(value, bound, terms, what, tight=0.75, ratio=16.0):
  """A check that would catch a dropped contribution: at least `tight` of the elements with a nonzero value (a ReLU
  zero has no relative precision) have bound <= 2^-5 |value|, and every contribution reaches `ratio` times the bound
  somewhere.  Returns (the tight fraction, the smallest contribution / bound)."""
  nz = value != 0
  small = (bound[nz] <= 2.0 ** -5 * value[nz].abs()).double().mean() if nz.any() else torch.tensor(1.0)
  assert float(small) >= tight, f'{what}: only {float(small):.2f} of the elements have bound <= 2^-5 |value|'
  worst = float('inf')
  for label, t in terms:
    r = float((t.abs() / bound.clamp_min(1e-300)).max())
    assert r >= ratio, f'{what}: dropping {label} moves no element more than {r:.3g} bounds'
    worst = min(worst, r)
  return float(small), worst
