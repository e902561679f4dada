"""Host side of the hot path: `Model.__call__` / `render_image` over the sm_90a kernels.

Keeps the reference's surface (internal/models.py):
  Model.__call__(rng, rays, train_frac, compute_extras, zero_glo) -> (renderings, ray_history)
                                                      models.py:75-312
  construct_model(rng, rays, config) -> (model, variables)    models.py:315-338
  render_image(render_fn, rays, rng, config)                  models.py:625-706
Python only orchestrates: per level it launches resample -> cast+IPE -> Dense chain (wgmma)
-> heads -> compositing; the backward chain mirrors it (train_utils.py:239-339 closure lives
in multinerf_b200/train_utils.py).  PyTorch provides device buffers, streams and RNG draws.
There is no CPU path: constructing a Model without an H100 raises.
"""
import dataclasses
import math
import os
from typing import Any, Dict, List, Optional

import numpy as np
import torch

from . import configs
from . import geopoly
from . import lib as L
from . import ops
from . import utils


def _pad64(n):
  return (n + 63) // 64 * 64


@dataclasses.dataclass
class DenseSpec:
  """One nn.Dense of the reference MLP (creation order = flax auto-name Dense_k)."""
  name: str
  role: str            # trunk | density | bottleneck | view | rgb
  in_dim: int          # logical inputs (flax kernel rows)
  in_pad: int          # rows of the padded master / K of the GEMM
  out_dim: int
  head: bool           # True: narrow head kernel, False: wgmma GEMM
  act: int = L.ACT_NONE
  # row map: logical flax row -> padded master row (skip-concat / view-input padding)
  row_map: Optional[np.ndarray] = None
  w_off: int = 0       # offsets (floats) into the module's flat master buffer
  b_off: int = 0


class MLPPlan:
  """Static layout of one MLP: layer table (flax creation order), buffer widths, flat offsets."""

  HEAD_SLOTS = {'density': (0, 1), 'grad_pred': (1, 3), 'diffuse': (4, 3), 'tint': (7, 3),
                'roughness': (10, 1)}     # column slots of the head-gradient slab (csrc/refnerf.cu)
  # net_activation (jax.nn.relu | softplus | silu, internal/configs.py:31) -> the Dense layers' activation code
  ACTIVATIONS = {'relu': L.ACT_RELU, 'softplus': L.ACT_SOFTPLUS, 'silu': L.ACT_SILU}

  def __init__(self, cfg: configs.MLPConfig, use_viewdirs=True, glo_features=0, activations=('relu',)):
    """activations: the net_activation values the caller runs.  A smooth activation changes the per-level buffers
    (pre-activations instead of mask bits) and the backward schedule (no chained trunk, the second-order pass of the
    density normals), so a caller opts into it: Model passes every key of ACTIVATIONS; the bare table is the ReLU
    one."""
    cfg.validate()
    self.glo_features = glo_features
    if cfg.net_activation not in self.ACTIVATIONS:
      raise NotImplementedError(f'net_activation = {cfg.net_activation!r}: the CUDA path runs relu, softplus and silu')
    if cfg.net_activation not in activations:
      raise NotImplementedError(f'net_activation = {cfg.net_activation!r}: this plan is built for {", ".join(activations)}'
                                f' (models.Model runs {", ".join(self.ACTIVATIONS)})')
    if cfg.density_activation != 'softplus':
      raise NotImplementedError(f'density_activation = {cfg.density_activation!r}: the CUDA path runs softplus')
    if cfg.roughness_activation != 'softplus':
      raise NotImplementedError(f'roughness_activation = {cfg.roughness_activation!r}: the CUDA path runs softplus')
    # the activation of every trunk and view layer.  ReLU keeps 1-bit masks for the backward; a smooth one keeps the
    # pre-activation z (bf16), and its density normals add the second-order term a''(z) to the trunk gradient
    self.act = self.ACTIVATIONS[cfg.net_activation]
    if cfg.num_rgb_channels != 3:
      raise NotImplementedError('num_rgb_channels != 3')
    self.cfg = cfg
    self.density_normals = not cfg.disable_density_normals
    self.pred_normals = cfg.enable_pred_normals
    self.basis = np.ascontiguousarray(
        geopoly.generate_basis(cfg.basis_shape, cfg.basis_subdivisions), dtype=np.float32)
    self.K = self.basis.shape[0]
    self.L = cfg.max_deg_point - cfg.min_deg_point
    self.F = 2 * self.K * self.L
    self.Fpad = _pad64(self.F)
    W = cfg.net_width
    # tensor-core tiling constraints are checked by Model (the table itself is layout-agnostic)
    self.device_constraints = [('net_width', W)]
    specs: List[DenseSpec] = []
    k = 0

    def add(role, in_dim, in_pad, out_dim, head, act=L.ACT_NONE, rm=None):
      nonlocal k
      specs.append(DenseSpec(f'Dense_{k}', role, in_dim, in_pad, out_dim, head, act, rm))
      k += 1
    x_dim, x_pad, x_has_feat = self.F, self.Fpad, False
    self.concat_after = []    # trunk layers whose output is concatenated with the features
    for i in range(cfg.net_depth):
      rm = np.concatenate([np.arange(W), W + np.arange(self.F)]) if x_has_feat else None
      add('trunk', x_dim, x_pad, W, False, self.act, rm)
      if i % cfg.skip_layer == 0 and i > 0:
        self.concat_after.append(i)
        x_dim, x_pad, x_has_feat = W + self.F, W + self.Fpad, True
      else:
        x_dim, x_pad, x_has_feat = W, W, False
    self.last_has_feat = x_has_feat       # the heads read [hidden | features] after a skip layer
    self.x_dim, self.x_pad = x_dim, x_pad
    rmx = np.concatenate([np.arange(W), W + np.arange(self.F)]) if x_has_feat else None
    add('density', x_dim, x_pad, 1, True, rm=rmx)
    if self.pred_normals:
      add('grad_pred', x_dim, x_pad, 3, True, rm=rmx)
    self.has_rgb = not cfg.disable_rgb
    self.use_viewdirs = use_viewdirs
    # What sits on top of the trunk, decided here once (every other site reads `top`, `ref_stage`, `slab_cols`):
    #   'view':    bottleneck -> Ref-NeRF stage (`ref_stage`) or direction encoding -> GLO -> view MLP -> rgb head
    #   'density': the Dense(1) density head
    #   'stacked': view-independent colour (models.py:512,584), rgb = act(Dense(3)(x)) on the trunk output.  The rgb
    #              head runs stacked with the density head as one 4-output head: raw [M, 4] = [raw_density | raw_rgb]
    # each with the narrow heads on the trunk output; without a view branch, normals feed only the orientation /
    # predicted-normal losses and the renderings through the colourless normals stage (csrc/refnerf.cu normals_*)
    self.top = ('view' if use_viewdirs else 'stacked') if self.has_rgb else 'density'
    self.head_n = 4 if self.top == 'stacked' else 1
    self.ref_stage = self.has_bottleneck = False
    self.enc_col0, self.view_skips, self.rgb_vin, self.vin_partials = 0, [], None, 0
    if self.top == 'stacked':
      if cfg.use_diffuse_color:
        raise ValueError('use_viewdirs=False with use_diffuse_color: the reference reads raw_rgb_diffuse, which it '
                         'creates only with view directions (internal/models.py:591)')
      # Ref-NeRF heads and encodings are not created without view directions (models.py:512); normals still run
      add('rgb', x_dim, x_pad, cfg.num_rgb_channels, True, rm=rmx)
    elif self.top == 'view':
      if cfg.bottleneck_width <= 0:
        if not cfg.use_reflections:
          raise ValueError('bottleneck_width = 0 needs use_reflections: the reference reads bottleneck.shape to '
                           'broadcast the view encoding (internal/models.py:552-554)')
        if glo_features > 0:
          raise ValueError('bottleneck_width = 0 with num_glo_features > 0: the reference reads bottleneck.shape to '
                           'broadcast the GLO vector (internal/models.py:567-568)')
      if cfg.use_diffuse_color:
        add('diffuse', x_dim, x_pad, 3, True, rm=rmx)
      if cfg.use_specular_tint:
        add('tint', x_dim, x_pad, 3, True, rm=rmx)
      if cfg.enable_pred_roughness:
        add('roughness', x_dim, x_pad, 1, True, rm=rmx)
      if cfg.use_directional_enc and not cfg.enable_pred_roughness:
        raise NotImplementedError('IDE without a predicted roughness (kappa_inv would be None)')
      if cfg.use_directional_enc and not cfg.use_reflections:
        # models.py:548-554: dir_enc_fn(viewdirs [..., 3], roughness [..., S, 1]) does not broadcast in the
        # reference either (ref_utils.py:141-148); every shipped config pairs IDE with reflections
        raise ValueError('use_directional_enc needs use_reflections (per-sample roughness cannot attenuate '
                         'the encoding of a per-ray view direction)')
      # without a bottleneck (the Ref-NeRF ablation, models.py:526-537) the view input starts with the encoding
      bw = max(cfg.bottleneck_width, 0)
      self.has_bottleneck = bw > 0
      if self.has_bottleneck:
        self.device_constraints.append(('bottleneck_width', bw))
        add('bottleneck', x_dim, x_pad, bw, False, L.ACT_NONE, rmx)
      self.enc_col0 = bw        # first column of the direction encoding (and of the head gradients in the slab)
      self.ref_stage = (self.pred_normals or self.density_normals or cfg.use_reflections or
                        cfg.use_directional_enc or cfg.use_n_dot_v)
      if cfg.use_directional_enc:
        from . import ref_utils
        self.dir_dim = ref_utils.ide_dim(cfg.deg_view)
      else:
        self.dir_dim = 3 + 6 * cfg.deg_view
      self.glo_col0 = bw + self.dir_dim + (1 if cfg.use_n_dot_v else 0)
      vin = self.glo_col0 + glo_features            # [bottleneck | dir enc | n.v | GLO] (models.py:556-572)
      vin_pad = _pad64(vin)
      if self.ref_stage and vin_pad - bw < 11:
        vin_pad += 64
      self.vin_dim, self.vin_pad = vin, vin_pad
      Wv = cfg.net_width_viewdirs
      self.device_constraints.append(('net_width_viewdirs', Wv))
      v_dim, v_pad, v_has_in = vin, vin_pad, False
      self.view_concat_after = []     # view layers whose output is concatenated with vin
      for i in range(cfg.net_depth_viewdirs):
        rmv = np.concatenate([np.arange(Wv), Wv + np.arange(vin)]) if v_has_in else None
        add('view', v_dim, v_pad, Wv, False, self.act, rmv)
        if i % cfg.skip_layer_dir == 0 and i > 0:
          self.view_concat_after.append(i)
          v_dim, v_pad, v_has_in = Wv + vin, Wv + vin_pad, True
        else:
          v_dim, v_pad, v_has_in = Wv, Wv, False
      rmv = np.concatenate([np.arange(Wv), Wv + np.arange(vin)]) if v_has_in else None
      add('rgb', v_dim, v_pad, cfg.num_rgb_channels, True, rm=rmv)
      # The consumers of vin besides view layer 0, each one contribution to d vin: the view layers after a skip
      # (`view_skips`, they read [hidden | vin]) and the rgb head, which reads [hidden | vin] when the view MLP ends
      # on a skip ('tail') or vin itself without a view MLP ('all', models.py:575-585).
      nv = cfg.net_depth_viewdirs
      self.view_skips = [i + 1 for i in self.view_concat_after if i + 1 < nv]
      self.rgb_vin = 'all' if nv == 0 else ('tail' if v_has_in else None)
      # d vin summed before view layer 0's dgrad adds the last part: ping-pong buffers of the running sum
      self.vin_partials = len(self.view_skips) + (self.rgb_vin == 'tail')
      # columns of d vin the first view layer's dgrad (or the rgb head over vin) writes: the Ref-NeRF stage and GLO
      # read past the bottleneck
      self.d_vin_cols = vin_pad if (self.ref_stage or glo_features > 0) else bw
    off = 0
    for sp in specs:
      sp.w_off = off
      off += sp.in_pad * sp.out_dim
      off = (off + 3) // 4 * 4
      if self.top == 'stacked' and sp.role == 'rgb':
        # the density head's bias block holds [b_density | b_rgb]: the stacked head's bias and bias gradient
        sp.b_off = self.one('density', specs).b_off + 1
        continue
      sp.b_off = off
      off += self.head_n if sp.role == 'density' else sp.out_dim
      off = (off + 3) // 4 * 4
    self.specs = specs
    self.flat_size = off
    self.num_params = sum(sp.in_dim * sp.out_dim + sp.out_dim for sp in specs)
    self.narrow = [sp for sp in specs if sp.role in ('grad_pred', 'diffuse', 'tint', 'roughness')]
    # the colourless normals stage (normals of an MLP without a view branch); either normals stage takes the losses
    self.normals_stage = self.top != 'view' and (self.pred_normals or self.density_normals)
    self.has_normals_stage = self.ref_stage or self.normals_stage
    # Width of the head-gradient slab that ONE dgrad GEMM runs against `MLPDevice.wcat_kn` at the top of the trunk:
    # [d bottleneck | Ref-NeRF head gradients] with the Ref-NeRF stage, [d raw_density | d grad_pred (| d raw_rgb) |
    # 0] in the colourless normals stage with predicted normals, no slab otherwise.  `slab_heads` are the
    # (head, first slab column) pairs; a view-independent rgb head takes the diffuse slot (it has no diffuse head).
    if self.ref_stage:
      self.slab_cols, c0, slots = self.vin_pad, self.enc_col0, self.HEAD_SLOTS
    else:
      self.slab_cols = 64 if (self.normals_stage and self.pred_normals) else 0
      c0, slots = 0, dict(self.HEAD_SLOTS, rgb=self.HEAD_SLOTS['diffuse'])
    self.slab_heads = [(sp, c0 + slots[sp.role][0]) for sp in specs if self.slab_cols and sp.role in slots]

  # names kept for the layout tests and tools that read them
  rgb_on_trunk = property(lambda self: self.top == 'stacked')
  normals_head_cols = property(lambda self: 0 if self.ref_stage else self.slab_cols)

  def by_role(self, role):
    return [sp for sp in self.specs if sp.role == role]

  def one(self, role, specs=None):
    r = [sp for sp in (self.specs if specs is None else specs) if sp.role == role]
    return r[0] if r else None


class MLPDevice:
  """Device state of one MLP: fp32 master slice, bf16 shadows, gradient views.

  Every buffer is allocated here and only filled afterwards: captured CUDA graphs hold these pointers."""

  def __init__(self, plan: MLPPlan, master, grads, device):
    self.plan = plan
    self.master, self.grads = master, grads           # views into the global flat buffers
    self.device = device
    self.basis = torch.tensor(plan.basis, device=device)
    self.w_nk, self.w_kn = {}, {}
    d = plan.one('density')
    # [head_n, x_pad]: the density head, or [w_density; W_rgb], the density and rgb heads of a view-independent
    # model as one 4-output head
    self.w_head = torch.zeros(plan.head_n, d.in_pad, device=device, dtype=torch.bfloat16)
    self.w_nk[d.name] = self.w_head[:1]
    if plan.top == 'stacked':
      self.w_nk[plan.one('rgb').name] = self.w_head[1:]
    for sp in plan.specs:
      if sp.name in self.w_nk:
        continue
      self.w_nk[sp.name] = torch.zeros(sp.out_dim, sp.in_pad, device=device, dtype=torch.bfloat16)
      if not sp.head:
        self.w_kn[sp.name] = torch.zeros(sp.in_pad, sp.out_dim, device=device, dtype=torch.bfloat16)
    self._pack_table = ops.pack_table([(self.W(sp), self.w_nk[sp.name], self.w_kn.get(sp.name))
                                       for sp in plan.specs], self.device)
    # fp32 rows of the density (or stacked) head, bf16-rounded as the fwd used: the chained trunk's epilogue head,
    # and row 0, colv_density, for DGRAD colv / outer_mask
    self.colv_head = torch.zeros(plan.head_n, d.in_pad, device=device)
    self.colv_density = self.colv_head[0]
    # [x_pad, slab_cols] K-major B operand of the trunk-top dgrad: [ W_bottleneck | head weights ] with the Ref-NeRF
    # stage, [ w_density | W_grad_pred (| W_rgb) | 0 ] in the colourless normals stage
    self.wcat_kn = (torch.zeros(plan.x_pad, plan.slab_cols, device=device, dtype=torch.bfloat16)
                    if plan.slab_cols else None)
    self.ide = None
    if plan.cfg.use_directional_enc:
      from . import ref_utils
      m, l, mat = ref_utils.ide_tables(plan.cfg.deg_view)
      self.ide = (torch.tensor(mat, dtype=torch.float32, device=device).contiguous(),
                  torch.tensor(np.stack([m, l]), dtype=torch.int32, device=device).contiguous(), len(m))
    self.repack()

  def W(self, s, buf=None):
    buf = self.master if buf is None else buf
    return buf[s.w_off:s.w_off + s.in_pad * s.out_dim].view(s.in_pad, s.out_dim)

  def b(self, s, buf=None):
    buf = self.master if buf is None else buf
    return buf[s.b_off:s.b_off + s.out_dim]

  def repack(self):
    """fp32 master -> bf16 operand layouts (after init and after every optimizer step), in place."""
    plan = self.plan
    ops.pack_weights_batched(self._pack_table)
    self.colv_head.copy_(self.w_head)
    if plan.ref_stage and plan.has_bottleneck:
      bt = plan.one('bottleneck')
      self.wcat_kn[:, :bt.out_dim] = self.w_kn[bt.name]
    for sp, c0 in plan.slab_heads:
      self.wcat_kn[:, c0:c0 + sp.out_dim] = self.w_nk[sp.name].t()


class LevelState:
  """Per-level device buffers kept from forward for the backward pass.  Model._level_state allocates them once per
  (level, module, shape): captured CUDA graphs hold their pointers.  Buffers of absent stages stay None."""

  def __init__(self, B, S, mname):
    self.B, self.S, self.M, self.mname = B, S, B * S, mname     # M: rows (samples) of the level
    self.sdist = None
    # trunk activations, features (+ their copies into later skip layers) and ReLU masks (bits) or, for a smooth
    # activation, pre-activations (zs); tangent streams
    self.acts, self.feat, self.feat_copies, self.bits, self.zs = [], None, [], [], []
    self.tacts, self.tfeat, self.tfeat_copies, self.rgd, self.d_rgd = [], None, [], None, None
    # raw_head / d_raw_head [M, head_n]: the density (or stacked [density | rgb]) head's output and gradient, of which
    # raw_density (and a stacked raw_rgb) are views
    self.raw_head = self.d_raw_head = self.raw_density = self.d_raw_density = self.raw_rgb = self.d_raw_rgb = None
    self.heads, self.d_heads = {}, {}          # narrow heads by role
    self.normals = self.normals_pred = self.roughness = self.extra_dw = None
    self.vacts, self.vbits, self.vzs, self.vin, self.vin_copies = [], [], [], None, []   # + vin copies for later skips
    self.x_last = self.t_last = self.v_last = None   # inputs of the last trunk layer / tangent stream / view layer
    self.bwd = None         # BwdScratch, allocated on the first backward
    self.keep_acts = True   # False: render-only pass, the chained trunk skips activation / mask stores
    self.chain = {}         # chain descriptors (Model.bind drops them)
    # set per call by Model.forward_levels
    self.lv, self.is_prop, self.glo_vec, self.bneck_noise, self.loss_mults = None, False, None, None, None
    self.noise = self.comp_cfg = self.bg_rgb = self.comp = self.rgb_scale = None
    self.d_rgb_scale = None   # gradient of rgb_scale, allocated on first use (train_utils)


class BwdScratch:
  """Gradient buffers of one level's backward, allocated on its first backward."""

  def __init__(self, plan, M, chained, dev):
    cfg, bf = plan.cfg, torch.bfloat16
    # trunk: per-layer gradient buffers when the dgrad chain runs as one launch (its wgrads come after), else two
    self.dy = [torch.empty(M, cfg.net_width, device=dev, dtype=bf) for _ in range(cfg.net_depth if chained else 2)]
    self.dv = self.d_vin = self.dhead = self.h = None
    self.d_vin_parts = []
    if plan.top == 'view':
      if cfg.net_depth_viewdirs:
        self.dv = [torch.empty(M, cfg.net_width_viewdirs, device=dev, dtype=bf) for _ in range(2)]
      self.d_vin = torch.empty(M, plan.vin_pad, device=dev, dtype=bf)
      # running sums of the other consumers' contributions to d vin (view layers after a skip, the rgb head after a
      # skip), chained through the dgrad addend: two buffers that take turns as addend and output
      self.d_vin_parts = [torch.empty(M, plan.vin_pad, device=dev, dtype=bf) for _ in range(min(2, plan.vin_partials))]
    elif plan.slab_cols:
      # zero-filled once: the normals backward writes only its first four (seven) columns
      self.dhead = torch.zeros(M, plan.slab_cols, device=dev, dtype=bf)
    self.u = self.g = None
    if plan.density_normals:
      self.h = [torch.empty(3 * M, cfg.net_width, device=dev, dtype=bf) for _ in range(2)]    # tangent adjoints
      if plan.act != L.ACT_RELU:
        # the recomputed tangent before the activation factor, u = t_in W, and the second-order term of dL/dz
        self.u = torch.empty(3 * M, cfg.net_width, device=dev, dtype=bf)
        self.g = torch.empty(M, cfg.net_width, device=dev, dtype=bf)


def _contracted_length_scale(points):
  """|dx/dr_c| at contracted points p [N, 3] (|p| < 2): world length per unit of contracted length along a radial
  ray, 1 inside the unit ball and |x|^2 = (2 - |p|)^-2 outside -> fp32 [N].  |p| is clamped below 2 as
  inv_contract clamps it (csrc/contract.cuh), so a point whose fp32 norm rounds to 2 gets a finite scale."""
  m = points.square().sum(-1)
  return torch.where(m > 1, (2 - m.sqrt().clamp_max(2 - 2 ** -23)).square().reciprocal(), torch.ones_like(m))


def _loss_args(loss_mults):
  """(orient_mult, prednorm_mult, orient_on_pred) of the normals kernels: both losses off without loss_mults."""
  return loss_mults if loss_mults is not None else (0.0, 0.0, True)


class Params:
  """`variables`: flat fp32 parameter/gradient/Adam buffers + per-module views."""

  STATS_TAIL = 64      # floats: [num_levels, 8] loss accumulators (num_levels <= 8)

  def __init__(self, plans: Dict[str, MLPPlan], device, extra: Dict[str, int]):
    self.plans = plans
    self.offsets = {}
    off = 0
    for name, plan in plans.items():
      self.offsets[name] = (off, plan.flat_size)
      off += plan.flat_size
    for name, n in extra.items():
      self.offsets[name] = (off, n)
      off += (n + 3) // 4 * 4
    self.total = off
    self.flat = torch.zeros(off, device=device)
    # gradient buffer + a small tail that carries the step's loss statistics, so the data-parallel
    # exchange of a train step is ONE all-reduce over one flat buffer (pmean of grad and stats,
    # train_utils.py:319-321)
    self.grads_ext = torch.zeros(off + self.STATS_TAIL, device=device)
    self.grads = self.grads_ext[:off]
    self.stats_tail = self.grads_ext[off:]
    self.mu = torch.zeros(off, device=device)
    self.nu = torch.zeros(off, device=device)
    self.step = 0

  def seg(self, name, buf=None):
    o, n = self.offsets[name]
    return (self.flat if buf is None else buf)[o:o + n]


def _init_kernel(rng, name, fan_in, fan_out):
  """flax initialisers (he_uniform / glorot_uniform ...) restated; host numpy.  PARITY UNPINNED:
  threefry streams cannot be reproduced, only the distribution (SURVEY.md section 8c)."""
  if name == 'he_uniform':
    lim = math.sqrt(6.0 / fan_in)
    return rng.uniform(-lim, lim, (fan_in, fan_out)).astype(np.float32)
  if name == 'glorot_uniform':
    lim = math.sqrt(6.0 / (fan_in + fan_out))
    return rng.uniform(-lim, lim, (fan_in, fan_out)).astype(np.float32)
  if name == 'he_normal':
    return (rng.standard_normal((fan_in, fan_out)) * math.sqrt(2.0 / fan_in) / .87962566103423978
            ).clip(-2 * math.sqrt(2.0 / fan_in) / .87962566103423978,
                   2 * math.sqrt(2.0 / fan_in) / .87962566103423978).astype(np.float32)
  if name == 'glorot_normal':
    return (rng.standard_normal((fan_in, fan_out)) * math.sqrt(2.0 / (fan_in + fan_out))
            ).astype(np.float32)
  raise ValueError(f'unknown weight_init {name!r}')


class Model:
  """The mip-NeRF 360 model (reference class `Model`, internal/models.py:47-312)."""

  def __init__(self, bundle: configs.Bundle, device=None):
    L.require_device()
    self.bundle = bundle
    self.config = bundle.config
    self.mcfg = bundle.model
    m = self.mcfg
    self.device = torch.device(device if device is not None else torch.device('cuda', torch.cuda.current_device()))
    for f in dataclasses.fields(m):            # expose Model.<field> like the reference
      setattr(self, f.name, getattr(m, f.name))
    if m.num_glo_features > 0 and m.single_mlp:
      raise ValueError('GLO with single_mlp feeds two input widths to the same view MLP (flax would reject it)')
    if m.ray_shape not in L.RAY_SHAPE:
      raise ValueError("ray_shape must be 'cone' or 'cylinder'")
    if m.raydist_fn not in L.RAYDIST:
      raise ValueError(f'raydist_fn {m.raydist_fn!r} not supported')
    if not m.stop_level_grad:
      raise NotImplementedError('stop_level_grad=False (gradients through resampling)')
    # every activation of the CUDA path: this class runs the smooth ones' buffers and backward schedule
    acts = tuple(MLPPlan.ACTIVATIONS)
    self.plans = {'NerfMLP_0': MLPPlan(bundle.nerf_mlp, m.use_viewdirs, glo_features=m.num_glo_features,
                                       activations=acts)}
    if not m.single_mlp:
      self.plans['PropMLP_0'] = MLPPlan(bundle.prop_mlp, m.use_viewdirs, activations=acts)
    for pname, plan in self.plans.items():
      for field, val in plan.device_constraints:
        if val % 64 != 0:
          raise ValueError(f'{pname}.{field} = {val}: the tensor-core path tiles layer widths in multiples of 64')
    # non-MLP top-level parameter modules (flax names), each clipped/updated on its own
    self.extra_params = {}
    if m.learned_exposure_scaling:
      self.extra_params['exposure_scaling_offsets'] = m.num_glo_embeddings * 3   # Embed [N,3], zeros
    if m.num_glo_features > 0:
      self.extra_params['Embed_0'] = m.num_glo_embeddings * m.num_glo_features    # GLO vectors
    self.params: Optional[Params] = None
    self.mlps: Dict[str, MLPDevice] = {}
    self._levels: Dict[Any, LevelState] = {}
    self._u_cache = {}
    self._init_hist = {}

  # ------------------------------------------------------------------ parameters
  def num_params(self):
    return sum(p.num_params for p in self.plans.values())

  def init(self, seed=0, flax_params=None):
    """Creates `variables` (random init like flax, or from a flax-style tree of arrays)."""
    params = Params(self.plans, self.device, self.extra_params)
    rng = np.random.default_rng(seed)
    host = np.zeros(params.total, np.float32)
    for mname, plan in self.plans.items():
      o, _ = params.offsets[mname]
      for s in plan.specs:
        if flax_params is not None:
          kern = np.asarray(flax_params[mname][s.name]['kernel'], np.float32)
          bias = np.asarray(flax_params[mname][s.name]['bias'], np.float32)
          if kern.shape != (s.in_dim, s.out_dim):
            raise ValueError(f'{mname}/{s.name}: kernel {kern.shape} != {(s.in_dim, s.out_dim)}')
        else:
          kern = _init_kernel(rng, plan.cfg.weight_init, s.in_dim, s.out_dim)
          bias = np.zeros(s.out_dim, np.float32)
        Wp = np.zeros((s.in_pad, s.out_dim), np.float32)
        rows = s.row_map if s.row_map is not None else np.arange(s.in_dim)
        Wp[rows] = kern
        host[o + s.w_off:o + s.w_off + Wp.size] = Wp.reshape(-1)
        host[o + s.b_off:o + s.b_off + s.out_dim] = bias
    if flax_params is not None:
      for name in self.extra_params:
        if name in flax_params:
          o, n = params.offsets[name]
          host[o:o + n] = np.asarray(flax_params[name]['embedding'], np.float32).reshape(-1)
    elif 'Embed_0' in self.extra_params:
      # flax nn.Embed default init: variance_scaling(1.0, 'fan_in', 'normal', out_axis=0)
      o, n = params.offsets['Embed_0']
      host[o:o + n] = rng.standard_normal(n).astype(np.float32) / math.sqrt(self.mcfg.num_glo_features)
    params.flat.copy_(torch.from_numpy(host))
    self.bind(params)
    return params

  def bind(self, params: Params):
    self.params = params
    self.mlps = {n: MLPDevice(p, params.seg(n), params.seg(n, params.grads), self.device)
                 for n, p in self.plans.items()}
    for st in self._levels.values():        # cached chain descriptors point into the previous buffers
      st.chain.clear()

  def _export(self, buf):
    """`buf` (the flat parameters or their gradients) as the reference's flax tree (numpy), without padding rows."""
    out = {}
    for mname, plan in self.plans.items():
      mlp, seg = self.mlps[mname], self.params.seg(mname, buf)
      out[mname] = {}
      for s in plan.specs:
        Wp = mlp.W(s, seg).detach().cpu().numpy()
        rows = s.row_map if s.row_map is not None else np.arange(s.in_dim)
        out[mname][s.name] = {'kernel': Wp[rows].copy(), 'bias': mlp.b(s, seg).detach().cpu().numpy().copy()}
    for name in self.extra_params:
      out[name] = {'embedding': self.params.seg(name, buf).detach().cpu().numpy().reshape(
          self.mcfg.num_glo_embeddings, -1).copy()}
    return out

  def export_flax(self):
    """Parameters as the reference's flax tree (numpy), dropping the padding rows."""
    return self._export(self.params.flat)

  def export_grads_flax(self):
    return self._export(self.params.grads)

  # ------------------------------------------------------------------ schedule
  def level_schedule(self, train_frac):
    m = self.mcfg
    init_s_near = 0.0
    if m.near_anneal_rate is not None:
      init_s_near = min(max(1 - train_frac / m.near_anneal_rate, 0.0), m.near_anneal_init)
    init_s_far = 1.0
    prod = 1
    out = []
    for i in range(m.num_levels):
      is_prop = i < m.num_levels - 1
      ns = m.num_prop_samples if is_prop else m.num_nerf_samples
      dilation = m.dilation_bias + m.dilation_multiplier * (init_s_far - init_s_near) / prod
      prod *= ns
      use_dil = (m.dilation_bias > 0 or m.dilation_multiplier > 0) and i > 0
      if m.anneal_slope > 0:
        s = m.anneal_slope
        anneal = (s * train_frac) / ((s - 1) * train_frac + 1)
      else:
        anneal = 1.0
      out.append(dict(is_prop=is_prop, S=ns, dilation=dilation, use_dilation=use_dil, anneal=anneal))
    return init_s_near, init_s_far, out

  def _u(self, S, randomized):
    key = (S, randomized)
    if key not in self._u_cache:
      ub, mj = ops.u_grid(S, randomized)
      self._u_cache[key] = (ub.to(self.device), mj)
    return self._u_cache[key]

  def _comp_cfg(self, cfg):
    return dict(raydist_fn=self.mcfg.raydist_fn, opaque_background=self.mcfg.opaque_background,
                density_bias=cfg.density_bias, density_noise=cfg.density_noise,
                rgb_activation=cfg.rgb_activation, rgb_premultiplier=cfg.rgb_premultiplier,
                rgb_bias=cfg.rgb_bias, rgb_padding=cfg.rgb_padding,
                bg_const=self.mcfg.bg_intensity_range[0],
                rgb_mode=1 if (cfg.use_diffuse_color and not cfg.disable_rgb) else 0)

  # ------------------------------------------------------------------ buffers
  def _level_state(self, key, mname, B, S, trunk_only=False, keep=True):
    # one buffer set per (level, module, shape), never replaced: captured CUDA graphs (train step, render
    # chunks) hold raw pointers into these buffers, so a differently shaped call (the ragged last chunk of
    # an image) must not free them.  trunk_only: the buffers of encode -> trunk -> density head alone, for a
    # render-only pass no graph captures (query_density).  keep=False, and trunk_only: not kept, so they are freed
    # with the caller's reference (point queries, which no graph captures)
    key = (key, mname, B, S)
    st = self._levels.get(key) if keep else None
    if st is not None:
      return st
    plan = self.plans[mname]
    cfg = plan.cfg
    W = cfg.net_width
    M = B * S
    dev, bf = self.device, torch.bfloat16
    st = LevelState(B, S, mname)
    st.sdist = torch.empty(B, S + 1, device=dev)

    def trunk_buffers(rows):
      # the layer whose output is concatenated with the features owns the feature columns
      # (encode writes there), otherwise features get their own buffer
      acts = [torch.empty(rows, W + plan.Fpad if i in plan.concat_after else W, device=dev, dtype=bf)
              for i in range(cfg.net_depth)]
      if plan.concat_after:
        feat = acts[plan.concat_after[0]][:, W:]
        copies = [acts[i][:, W:] for i in plan.concat_after[1:]]
      else:
        feat, copies = torch.empty(rows, plan.Fpad, device=dev, dtype=bf), []
      return acts, feat, copies
    st.acts, st.feat, st.feat_copies = trunk_buffers(M)
    relu = plan.act == L.ACT_RELU
    if relu:
      st.bits = [torch.empty(M, W // 32, device=dev, dtype=torch.int32) for _ in range(cfg.net_depth)]
    elif not trunk_only:
      st.zs = [torch.empty(M, W, device=dev, dtype=bf) for _ in range(cfg.net_depth)]
    if trunk_only:
      st.keep_acts = False
      st.raw_head = torch.empty(M, plan.head_n, device=dev)
      return st
    if plan.density_normals:
      # forward-mode tangents d(.)/d(mean_x|y|z), three stacked streams of M rows
      st.tacts, st.tfeat, st.tfeat_copies = trunk_buffers(3 * M)
      st.rgd = torch.empty(3, M, device=dev)
      st.d_rgd = torch.empty(3, M, device=dev)
      st.normals = torch.empty(M, 3, device=dev)
    # the head's output and its gradient, [M, head_n] (stacked: [density | rgb]): compositing reads and writes them
    # in place through sample strides
    st.raw_head, st.d_raw_head = torch.empty(M, plan.head_n, device=dev), torch.empty(M, plan.head_n, device=dev)
    st.raw_density = st.raw_head.view(B, S, plan.head_n)[..., 0]
    st.d_raw_density = st.d_raw_head.view(B, S, plan.head_n)[..., 0]
    if plan.top == 'stacked':
      st.raw_rgb, st.d_raw_rgb = st.raw_head.view(B, S, 4)[..., 1:], st.d_raw_head.view(B, S, 4)[..., 1:]
    elif plan.top == 'view':
      Wv = cfg.net_width_viewdirs
      nv = cfg.net_depth_viewdirs
      st.vacts = [torch.empty(M, Wv + plan.vin_pad if i in plan.view_concat_after else Wv, device=dev, dtype=bf)
                  for i in range(nv)]
      if relu:
        st.vbits = [torch.empty(M, Wv // 32, device=dev, dtype=torch.int32) for _ in range(nv)]
      else:
        st.vzs = [torch.empty(M, Wv, device=dev, dtype=bf) for _ in range(nv)]
      # the first layer whose output is concatenated with vin owns the vin columns, later ones get copies
      if plan.view_concat_after:
        st.vin = st.vacts[plan.view_concat_after[0]][:, Wv:]
        st.vin_copies = [st.vacts[i][:, Wv:] for i in plan.view_concat_after[1:]]
      else:
        st.vin = torch.empty(M, plan.vin_pad, device=dev, dtype=bf)
      st.raw_rgb = torch.empty(B, S, 3, device=dev)
      st.d_raw_rgb = torch.empty(B, S, 3, device=dev)
    for sp in plan.narrow:
      st.heads[sp.role] = torch.empty(M, sp.out_dim, device=dev)
      st.d_heads[sp.role] = torch.empty(M, sp.out_dim, device=dev)
    if plan.has_normals_stage:
      if plan.pred_normals:
        st.normals_pred = torch.empty(M, 3, device=dev)
      if plan.ref_stage and cfg.enable_pred_roughness:
        st.roughness = torch.empty(M, device=dev)
      st.extra_dw = torch.empty(B, S, device=dev)
    if keep:
      self._levels[key] = st
    return st

  @staticmethod
  def _act_out(plan, st, i, view=False):
    """What the FWD GEMM of hidden layer i (trunk, or view MLP) keeps for the backward and the tangent GEMMs: ReLU
    mask bits, or the pre-activation z of a smooth activation (neither kept by a render-only pass)."""
    if plan.act == L.ACT_RELU:
      return dict(act=L.ACT_RELU, maskbits=(st.vbits if view else st.bits)[i] if st.keep_acts else None)
    return dict(act=plan.act, z=(st.vzs if view else st.zs)[i] if st.keep_acts else None)

  @staticmethod
  def _act_grad(plan, st, i, view=False, head=False):
    """How a DGRAD (or, head=True, a head_bwd) applies the activation derivative of hidden layer i: ReLU mask bits
    or a'(z)."""
    if plan.act == L.ACT_RELU:
      return dict(relu_mask=True) if head else dict(maskbits=(st.vbits if view else st.bits)[i])
    return dict(act=plan.act, z=(st.vzs if view else st.zs)[i])

  def _refdir_args(self, st, mlp, viewdirs):
    """The leading arguments of ops.refdir_fwd / refdir_bwd: descriptor, IDE tables and the stage's inputs."""
    plan = mlp.plan
    cfg = plan.cfg
    mat, ml, ide_n = mlp.ide or (None, None, 0)
    desc = ops.refdir_desc(
        st.M, st.S, use_pred_normals=plan.pred_normals, use_density_normals=plan.density_normals,
        use_reflections=cfg.use_reflections, use_ide=cfg.use_directional_enc, use_n_dot_v=cfg.use_n_dot_v,
        use_roughness=cfg.enable_pred_roughness, deg_view=cfg.deg_view, ide_n=ide_n,
        roughness_bias=cfg.roughness_bias, ld=st.vin.stride(0), col0=plan.enc_col0, col_end=plan.vin_pad)
    return desc, mat, ml, st.heads.get('grad_pred'), st.heads.get('roughness'), st.rgd, viewdirs

  # ------------------------------------------------------------------ forward
  def _mlp_forward(self, st: LevelState, mlp: MLPDevice, rays, impl=0, loss_mults=None):
    """loss_mults = (orientation, predicted-normal) multipliers of this level divided by the number
    of rays, + orientation target flag: when given, the normals stage (Ref-NeRF or colourless) also emits
    d(loss)/d(weights)."""
    plan = mlp.plan
    cfg = plan.cfg
    m = self.mcfg
    ops.encode(st.sdist, rays.origins, rays.directions, rays.radii_flat, rays.near_flat,
               rays.far_flat, mlp.basis, min_deg=cfg.min_deg_point, max_deg=cfg.max_deg_point,
               raydist_fn=m.raydist_fn, ray_shape=m.ray_shape, warp_contract=cfg.warp_fn == 'contract',
               disable_integration=m.disable_integration, feat=st.feat, feat_cols=plan.Fpad, tfeat=st.tfeat)
    self._mlp_stages(st, mlp, rays.viewdirs, impl, loss_mults)

  def _mlp_stages(self, st, mlp, viewdirs, impl=0, loss_mults=None):
    """The MLP on the encoded st.feat (and st.tfeat), after the ray or the point encoder: trunk, tangents, narrow
    heads, normals or Ref-NeRF stage, view branch.  viewdirs: one unit direction per ray of the level ([B, 3])."""
    plan = mlp.plan
    self._trunk_layers(st, mlp, impl)
    if plan.density_normals:
      self._tangent_fwd(st, mlp, impl)
    for sp in plan.narrow:
      ops.head_fwd(st.x_last, mlp.w_nk[sp.name], mlp.b(sp), sp.out_dim, sp.in_pad, raw=st.heads[sp.role])
    # (orientation, predicted-normal, target flag, d(loss)/d(weights) output) of the normals stage
    normals_args = _loss_args(loss_mults) + (st.extra_dw if loss_mults is not None else None,)
    if plan.normals_stage:
      ops.normals_fwd(st.M, st.S, st.heads.get('grad_pred'), st.rgd, viewdirs, st.normals_pred,
                      st.normals, *normals_args)
    if plan.top == 'view':
      self._view_fwd(st, mlp, viewdirs, impl, normals_args)

  def _trunk_layers(self, st, mlp, impl):
    """The trunk (one chained launch, or one GEMM per layer) and the density (or stacked) head on the encoded
    st.feat."""
    plan = mlp.plan
    W = plan.cfg.net_width
    for c in st.feat_copies:
      c.copy_(st.feat)
    x = st.feat
    chained = self._use_chain(plan, st.M, impl)
    if chained:
      # the whole trunk (+ the density head when it reads the plain 256-wide output) in ONE launch
      ops.mlp_chain(self._chain_fwd_desc(st, mlp))
      x = st.acts[-1]
    else:
      for i, sp in enumerate(plan.by_role('trunk')):
        ops.gemm(L.GEMM_FWD, x, mlp.w_nk[sp.name], st.acts[i][:, :W], m=st.M, n=W, k=sp.in_pad, bias=mlp.b(sp),
                 impl=impl, **self._act_out(plan, st, i))
        x = st.acts[i]          # full width (incl. concatenated features) feeds the next layer
    if not chained or plan.last_has_feat:
      # stacked: density + rgb in one pass over the trunk output (bias block [b_density | b_rgb])
      d = plan.one('density')
      ops.head_fwd(x, mlp.w_head, mlp.b(d), plan.head_n, d.in_pad, raw=st.raw_head)
    st.x_last = x

  def _contracted_mode(self, cfg, contracted):
    """warp_contract of the point encoder: the level's own flag, or 2 (points already contracted) with `contracted`,
    which needs an MLP under the scene contraction."""
    if not contracted:
      return cfg.warp_fn == 'contract'
    if cfg.warp_fn != 'contract':
      raise ValueError('contracted points need an MLP under the scene contraction (warp_fn = contract)')
    return 2

  def query_density(self, points, var, impl=0, contracted=False):
    """Density of the final level's MLP (NerfMLP_0) at world points [N, 3] (tensor or array): the point encoder on
    the Gaussians (point, var * I), the trunk and the density head in their render form, then
    density_activation(raw + density_bias), without density noise -> fp32 [N] on the device.  Runs in chunks of
    render_chunk_size * num_nerf_samples rows, the rows of one render chunk's final level.
    contracted: the points p (|p| < 2) and the footprint var * I are in the scene contraction's space, encoded as
    they are, and the result is the density per unit of contracted length along radial rays, sigma_c = sigma(x)
    |dx/dr_c|: sigma inside the unit ball, sigma / (2 - |p|)^2 outside, so that one level means one opacity per
    contracted cell everywhere."""
    mname = 'NerfMLP_0'
    mlp = self.mlps[mname]
    plan = mlp.plan
    cfg = plan.cfg
    warp = self._contracted_mode(cfg, contracted)
    points = torch.as_tensor(points, dtype=torch.float32, device=self.device).reshape(-1, 3).contiguous()
    N = points.shape[0]
    density = torch.empty(N, device=self.device)
    chunk = self.config.render_chunk_size * self.mcfg.num_nerf_samples
    states = {}
    for i0 in range(0, N, chunk):
      p = points[i0:i0 + chunk]
      n = p.shape[0]
      if n not in states:
        states[n] = self._level_state('query', mname, n, 1, trunk_only=True)
      st = states[n]
      ops.encode_points(p, var, mlp.basis, min_deg=cfg.min_deg_point, max_deg=cfg.max_deg_point,
                        warp_contract=warp, disable_integration=self.mcfg.disable_integration,
                        feat=st.feat, feat_cols=plan.Fpad)
      self._trunk_layers(st, mlp, impl)
      # density_activation: softplus, the only one MLPPlan accepts
      torch.nn.functional.softplus(st.raw_head[:, 0] + cfg.density_bias, out=density[i0:i0 + n])
    if contracted:
      density *= _contracted_length_scale(points)
    return density

  def query_radiance(self, points, var, viewdirs, impl=0, contracted=False):
    """Density and colour of the final level's MLP (NerfMLP_0) at world points [N, 3] seen along unit view
    directions viewdirs [N, 3] (ignored, and may be None, for a view-independent model) -> (density [N], rgb [N, 3])
    fp32 on the device.  Each point is one sample: the point encoder on the Gaussian (point, var * I), then the
    level's MLP as a render runs it (Model._mlp_stages: density normals and the Ref-NeRF stage included), with
    the GLO vector zeroed, no density or bottleneck noise, and no exposure scale; rgb is the activated, padded
    sample colour (ops.point_rgb), zero for an MLP without colour.  Density as query_density.  Runs in chunks of
    render_chunk_size * num_nerf_samples rows.  contracted: points and footprint in contracted space, as
    query_density takes them; viewdirs stay world directions, and density normals are taken with respect to the
    world point (the encoder's warp_contract 2)."""
    mname = 'NerfMLP_0'
    mlp = self.mlps[mname]
    plan = mlp.plan
    cfg = plan.cfg
    warp = self._contracted_mode(cfg, contracted)
    dev = self.device
    points = torch.as_tensor(points, dtype=torch.float32, device=dev).reshape(-1, 3).contiguous()
    N = points.shape[0]
    if plan.top == 'view':
      if viewdirs is None:
        raise ValueError('query_radiance: this model\'s colour depends on the view direction: give viewdirs')
      viewdirs = torch.as_tensor(viewdirs, dtype=torch.float32, device=dev).reshape(-1, 3).contiguous()
      if viewdirs.shape[0] != N:
        raise ValueError(f'query_radiance: {viewdirs.shape[0]} view directions for {N} points')
    density = torch.empty(N, device=dev)
    rgb = torch.zeros(N, 3, device=dev)
    comp_cfg = self._comp_cfg(cfg)
    chunk = self.config.render_chunk_size * self.mcfg.num_nerf_samples
    states = {}
    for i0 in range(0, N, chunk):
      p = points[i0:i0 + chunk]
      n = p.shape[0]
      if n not in states:
        states[n] = self._level_state('radiance', mname, n, 1, keep=False)
        # the tangent GEMMs read the trunk's ReLU masks or pre-activations (as forward_levels sets keep_acts)
        states[n].keep_acts = plan.density_normals
      st = states[n]
      ops.encode_points(p, var, mlp.basis, min_deg=cfg.min_deg_point, max_deg=cfg.max_deg_point,
                        warp_contract=warp, disable_integration=self.mcfg.disable_integration,
                        feat=st.feat, feat_cols=plan.Fpad, tfeat=st.tfeat)
      self._mlp_stages(st, mlp, viewdirs[i0:i0 + n] if plan.top == 'view' else None, impl)
      torch.nn.functional.softplus(st.raw_head[:, 0] + cfg.density_bias, out=density[i0:i0 + n])
      if st.raw_rgb is not None:
        ops.point_rgb(st.raw_rgb.reshape(n, 3), cfg=comp_cfg, raw_diffuse=st.heads.get('diffuse'),
                      raw_tint=st.heads.get('tint'), out=rgb[i0:i0 + n])
    if contracted:
      density *= _contracted_length_scale(points)
    return density, rgb

  def _tangent_fwd(self, st, mlp, impl):
    """raw_grad_density = d raw_density / d mean by forward mode (replaces vmap(value_and_grad),
    models.py:473-492): tangents see the same weights, no bias, and the primal's activation derivative (ReLU masks,
    or a'(z))."""
    plan = mlp.plan
    W = plan.cfg.net_width
    for c in st.tfeat_copies:
      c.copy_(st.tfeat)
    t = st.tfeat
    for i, sp in enumerate(plan.by_role('trunk')):
      ops.gemm(L.GEMM_DGRAD, t, mlp.w_nk[sp.name], st.tacts[i][:, :W], m=3 * st.M, n=W, k=sp.in_pad,
               mask_mod=st.M, impl=impl, **self._act_grad(plan, st, i))
      t = st.tacts[i]
    st.t_last = t
    d = plan.one('density')
    ops.head_fwd(t, mlp.w_nk[d.name], None, 1, d.in_pad, raw=st.rgd.view(3 * st.M, 1))

  def _view_fwd(self, st, mlp, viewdirs, impl, normals_args):
    """Bottleneck, Ref-NeRF stage or direction encoding, GLO, view MLP and rgb head."""
    plan = mlp.plan
    cfg = plan.cfg
    B, S = st.B, st.S
    if plan.has_bottleneck:
      bt = plan.one('bottleneck')
      ops.gemm(L.GEMM_FWD, st.x_last, mlp.w_nk[bt.name], st.vin[:, :bt.out_dim], m=st.M, n=bt.out_dim,
               k=bt.in_pad, act=L.ACT_NONE, bias=mlp.b(bt), impl=impl)
      if st.bneck_noise is not None:
        # models.py:529-533 (regulariser, unused by the shipped configs): plain elementwise add
        st.vin[:, :bt.out_dim].add_((cfg.bottleneck_noise * st.bneck_noise).to(torch.bfloat16))
    if plan.ref_stage:
      ops.refdir_fwd(*self._refdir_args(st, mlp, viewdirs), st.normals_pred, st.normals, st.roughness, st.vin,
                     *normals_args)
    else:
      ops.viewdir_enc(viewdirs, S, cfg.deg_view, st.vin, plan.enc_col0, plan.vin_pad)
    if plan.glo_features > 0:
      # GLO vector of the ray's camera, broadcast over the samples (models.py:565-569).  Written after the Ref-NeRF
      # stage: its slab zero-fill would also clear the GLO columns.
      g0 = plan.glo_col0
      # (unflatten, not view: a vin owned by a skip layer's buffer is a strided slice of it)
      st.vin.unflatten(0, (B, S))[:, :, g0:g0 + plan.glo_features] = \
          (st.glo_vec if st.glo_vec is not None else torch.zeros(B, plan.glo_features, device=st.vin.device)
           )[:, None, :].to(torch.bfloat16)
    # the view layers after the second and later skips read their own copy of the finished vin
    for c in st.vin_copies:
      c.copy_(st.vin)
    v = st.vin
    for i, sp in enumerate(plan.by_role('view')):
      Wv = sp.out_dim
      ops.gemm(L.GEMM_FWD, v, mlp.w_nk[sp.name], st.vacts[i][:, :Wv], m=st.M, n=Wv, k=sp.in_pad,
               bias=mlp.b(sp), impl=impl, **self._act_out(plan, st, i, view=True))
      v = st.vacts[i]
    st.v_last = v
    r = plan.one('rgb')
    ops.head_fwd(v, mlp.w_nk[r.name], mlp.b(r), r.out_dim, r.in_pad, raw=st.raw_rgb.view(st.M, 3))

  # ------------------------------------------------------------------ layer-chained 256-wide trunks
  def _use_chain(self, plan, M, impl=0):
    """One persistent launch per trunk (csrc/chain.cu) when every trunk layer is 256 wide and uses ReLU."""
    if impl != 0 or os.environ.get('MNRF_CHAIN', '1') == '0' or plan.act != L.ACT_RELU:
      return False
    cfg = plan.cfg
    return (cfg.net_width == 256 and cfg.net_depth <= L.CHAIN_MAX_LAYERS and M >= 512 and
            plan.Fpad % 64 == 0)

  def _chain_fwd_desc(self, st, mlp):
    key = ('fwd', st.keep_acts)
    if key in st.chain:
      return st.chain[key]
    plan = mlp.plan
    W = plan.cfg.net_width
    nf = plan.Fpad // 64
    trunk = plan.by_role('trunk')
    # the trunk output is read outside the chain: by the view branch, by heads after a skip, by the narrow heads
    out_read = plan.top == 'view' or plan.last_has_feat or bool(plan.narrow)
    layers = []
    for i, sp in enumerate(trunk):
      ly = dict(w=mlp.w_nk[sp.name], bias=mlp.b(sp))
      if i == 0:
        ly.update(n_stream=nf, stream_col0=0, stream_kb0=0)
      else:
        ly.update(n_res=W // 64, res_kb0=0)
        if sp.in_pad == W + plan.Fpad:          # skip layer: [hidden | features] against [W | Fpad] weight columns
          ly.update(n_stream=nf, stream_col0=0, stream_kb0=W // 64)
      if st.keep_acts or (i == len(trunk) - 1 and out_read):
        ly['out'] = st.acts[i][:, :W]
      if st.keep_acts:
        ly['maskbits'] = st.bits[i]
      layers.append(ly)
    head = {}
    if not plan.last_has_feat:
      head = dict(head_w=mlp.colv_head, head_b=mlp.b(plan.one('density')), head_out=st.raw_head, head_n=plan.head_n)
    st.chain[key] = ops.chain_desc(L.CHAIN_FWD, st.M, layers, stream=st.feat, stream_cols=plan.Fpad, **head)
    return st.chain[key]

  def _chain_bwd_desc(self, st, mlp, dyl):
    """dyl[i] = gradient w.r.t. the (pre-activation-masked) output of trunk layer i; dyl[-1] is the input."""
    if 'bwd' in st.chain:
      return st.chain['bwd']
    W = mlp.plan.cfg.net_width
    trunk = mlp.plan.by_role('trunk')
    layers = []
    for j, i in enumerate(range(len(trunk) - 1, 0, -1)):
      ly = dict(w=mlp.w_kn[trunk[i].name], maskbits=st.bits[i - 1], out=dyl[i - 1])
      if j == 0:
        ly.update(n_stream=W // 64, stream_col0=0, stream_kb0=0)
      else:
        ly.update(n_res=W // 64, res_kb0=0)
      layers.append(ly)
    st.chain['bwd'] = ops.chain_desc(L.CHAIN_BWD, st.M, layers, stream=dyl[-1], stream_cols=W)
    return st.chain['bwd']

  def _prep_rays(self, rays):
    r = utils.to_device_flat(rays, self.device)
    r.radii_flat = r.radii[:, 0].contiguous()
    r.near_flat = r.near[:, 0].contiguous()
    r.far_flat = r.far[:, 0].contiguous()
    return r

  def level_loss_mults(self, config, i_level, B):
    """(orientation, predicted-normal) multipliers of level i divided by the ray count, target flag
    (train_utils.py:162-197)."""
    fine = i_level == self.mcfg.num_levels - 1
    om = config.orientation_loss_mult if fine else config.orientation_coarse_loss_mult
    pm = config.predicted_normal_loss_mult if fine else config.predicted_normal_coarse_loss_mult
    if config.orientation_loss_target not in ('normals', 'normals_pred'):
      raise ValueError(f'orientation_loss_target {config.orientation_loss_target!r}')
    return om / B, pm / B, config.orientation_loss_target == 'normals_pred'

  def forward_levels(self, rng, rays, train_frac, compute_extras, want_samples, impl=0, anneal_dev=None,
                     loss_config=None, zero_glo=True, batch_rays=None):
    """Runs all levels; returns the list of LevelState (buffers stay valid until the next call).  `batch_rays`: the
    rays are one pass of a train step over that many rays, whose count the per-ray loss multipliers divide by."""
    if self.params is None:
      raise RuntimeError('Model has no parameters: call construct_model()/init() first')
    m = self.mcfg
    B = rays.origins.shape[0]
    s_near, s_far, sched = self.level_schedule(train_frac)
    dev = self.device
    # RawNeRF exposure logic (models.py:257-267): one per-ray colour scale for every level
    rgb_scale = None
    if getattr(rays, 'exposure_idx', None) is not None:
      rgb_scale = rays.exposure_values.expand(B, 3)
      if m.learned_exposure_scaling:
        eidx = rays.exposure_idx[:, 0].long()
        mask = (eidx > 0).to(torch.float32)[:, None]
        off = self.params.seg('exposure_scaling_offsets').view(-1, 3)[eidx]
        rgb_scale = rgb_scale * (1 + mask * off)
      rgb_scale = rgb_scale.contiguous()
    # the initial one-interval histogram [s_near, s_far] with weight 1 is a constant of (B, s_near, s_far): built
    # once, so a captured step does not replay three fill kernels for it
    ck = (B, float(s_near), float(s_far))
    init = self._init_hist.get(ck)
    if init is None:
      sd0 = torch.empty(B, 2, device=dev)
      sd0[:, 0] = s_near
      sd0[:, 1] = s_far
      init = (sd0, torch.ones(B, 1, device=dev))
      # entries are never evicted (a captured graph may hold their addresses); with near-plane annealing s_near
      # changes every step, so the table simply stops growing
      if len(self._init_hist) < 8 and not torch.cuda.is_current_stream_capturing():
        self._init_hist[ck] = init
    sdist_prev, w_prev = init

    def draw(key, i, shape, sample):
      # level i's draw: from an explicit dict of draws, or `sample` (torch.rand / randn) from the generator
      if isinstance(rng, dict):
        return rng[key][i].to(dev).reshape(shape).contiguous()
      return sample(shape, device=dev, generator=rng)
    states = []
    for i, lv in enumerate(sched):
      mname = 'NerfMLP_0' if (m.single_mlp or not lv['is_prop']) else 'PropMLP_0'
      mlp = self.mlps[mname]
      st = self._level_state(i, mname, B, lv['S'])
      st.lv = lv
      st.is_prop = lv['is_prop']
      # activations and ReLU masks are kept for a backward pass (and for the Ref-NeRF tangent chain)
      st.keep_acts = loss_config is not None or mlp.plan.density_normals
      jit = None
      if rng is not None:
        jit = draw('jitter', i, (B,) if m.single_jitter else (B, lv['S']), torch.rand)
      u_base, max_jitter = self._u(lv['S'], jit is not None)
      ops.sample_level(sdist_prev, w_prev, lv['S'], dilation=lv['dilation'],
                       use_dilation=lv['use_dilation'], domain=(s_near, s_far), anneal=lv['anneal'],
                       resample_padding=m.resample_padding, jitter=jit, single_jitter=m.single_jitter,
                       u_base=u_base, max_jitter=max_jitter, out=st.sdist, anneal_dev=anneal_dev)
      st.glo_vec = None
      if m.num_glo_features > 0 and not lv['is_prop'] and not zero_glo:
        st.glo_vec = self.params.seg('Embed_0').view(m.num_glo_embeddings, -1)[rays.cam_idx[:, 0].long()]
      st.bneck_noise = None
      if mlp.plan.cfg.bottleneck_noise > 0 and rng is not None and mlp.plan.has_bottleneck:
        st.bneck_noise = draw('bottleneck_noise', i, (B * lv['S'], mlp.plan.cfg.bottleneck_width), torch.randn)
      # levels of an MLP without normals skip the normal losses (the reference raises there instead)
      st.loss_mults = self.level_loss_mults(loss_config, i, batch_rays or B) if (
          loss_config is not None and mlp.plan.has_normals_stage) else None
      if st.loss_mults is not None:
        om, pm, on_pred = st.loss_mults
        if (om > 0 and ((on_pred and not mlp.plan.pred_normals) or (not on_pred and not mlp.plan.density_normals))):
          raise ValueError('Normals cannot be None if orientation loss is on.')
        if pm > 0 and not (mlp.plan.pred_normals and mlp.plan.density_normals):
          raise ValueError('Predicted normals and gradient normals cannot be None if '
                           'predicted normal loss is on.')
      self._mlp_forward(st, mlp, rays, impl=impl, loss_mults=st.loss_mults)
      st.noise = None
      if mlp.plan.cfg.density_noise > 0 and rng is not None:
        st.noise = draw('density_noise', i, (B, lv['S']), torch.randn)
      st.comp_cfg = self._comp_cfg(mlp.plan.cfg)
      # background colour (models.py:240-254): constant, midpoint (rng=None) or per-ray uniform draws
      lo, hi = m.bg_intensity_range
      st.bg_rgb = None
      if lo != hi:
        if rng is None:
          st.comp_cfg['bg_const'] = (lo + hi) / 2
        else:
          st.bg_rgb = (lo + (hi - lo) * draw('bg', i, (B, 3), torch.rand)).contiguous()
      st.comp = ops.composite_fwd(st.raw_density, st.raw_rgb, st.sdist, rays.directions,
                                  rays.near_flat, rays.far_flat, cfg=st.comp_cfg,
                                  density_noise=st.noise, bg_rgb=st.bg_rgb,
                                  rgb_scale=rgb_scale if st.raw_rgb is not None else None,
                                  raw_diffuse=st.heads.get('diffuse'), raw_tint=st.heads.get('tint'),
                                  want_samples=want_samples, want_extras=compute_extras)
      st.rgb_scale = rgb_scale if st.raw_rgb is not None else None
      sdist_prev, w_prev = st.sdist, st.comp['weights']
      states.append(st)
    return states

  def __call__(self, rng, rays, train_frac, compute_extras, zero_glo=True):
    """models.py:75-312.  rng: None (deterministic), a torch.Generator on the device, or a
    dict of explicit draws {'jitter': [per level], 'density_noise': [per level]}."""
    r = self._prep_rays(rays)
    lead = tuple(np.asarray(rays.origins).shape[:-1]) if not isinstance(rays.origins, torch.Tensor) \
        else tuple(rays.origins.shape[:-1])
    return self.call_prepped(rng, r, lead, train_frac, compute_extras, zero_glo)

  def call_prepped(self, rng, r, lead, train_frac, compute_extras, zero_glo=True):
    """`__call__` on rays already flattened on the device (`_prep_rays`): device work only, so a render
    chunk can be captured in a CUDA graph (train_utils.create_render_fn)."""
    states = self.forward_levels(rng, r, train_frac, compute_extras, want_samples=True, zero_glo=zero_glo)
    renderings, ray_history = [], []
    n_vis = self.config.vis_num_rays
    for st in states:
      c = st.comp
      rend = {'rgb': c['rgb'].view(lead + (3,))}
      if compute_extras:
        rend['acc'] = c['acc'].view(lead)
        for j, k in enumerate(['distance_mean', 'distance_percentile_5', 'distance_median',
                               'distance_percentile_95']):
          rend[k] = c['dist'][:, j].contiguous().view(lead)
        w3 = c['weights'][..., None]
        for k, v in (('normals', st.normals), ('normals_pred', st.normals_pred), ('roughness', st.roughness)):
          if v is not None:     # volumetric_rendering extras (render.py:186-189)
            rend[k] = (w3 * v.view(st.B, st.S, -1)).sum(-2).view(lead + (-1,))
        rend['ray_sdist'] = st.sdist[:n_vis].clone()
        rend['ray_weights'] = c['weights'][:n_vis].clone()
        rend['ray_rgbs'] = c['rgb_samples'][:n_vis].clone()
      renderings.append(rend)
      S = st.S
      ray_history.append(dict(
          density=c['density'].view(lead + (S,)), rgb=c['rgb_samples'].view(lead + (S, 3)),
          raw_grad_density=None if st.normals is None else st.rgd.t().reshape(lead + (S, 3)),
          grad_pred=None if 'grad_pred' not in st.heads else st.heads['grad_pred'].view(lead + (S, 3)),
          normals=None if st.normals is None else st.normals.view(lead + (S, 3)),
          normals_pred=None if st.normals_pred is None else st.normals_pred.view(lead + (S, 3)),
          roughness=None if st.roughness is None else st.roughness.view(lead + (S, 1)),
          sdist=st.sdist.clone().view(lead + (S + 1,)), weights=c['weights'].view(lead + (S,))))
    if compute_extras:
      final_rgb = (renderings[-1]['ray_rgbs'] * renderings[-1]['ray_weights'][..., None]).sum(-2)
      for rr in renderings[:-1]:
        rr['ray_rgbs'] = final_rgb[:, None, :].expand(rr['ray_rgbs'].shape).contiguous()
    return renderings, ray_history

  def apply(self, variables, rng, rays, train_frac, compute_extras, zero_glo=True):
    """flax-style entry: model.apply(variables, rng, rays, train_frac=..., compute_extras=...)."""
    if variables is not self.params:
      self.bind(variables)
    return self(rng, rays, train_frac, compute_extras, zero_glo)

  # ------------------------------------------------------------------ backward
  def _mlp_backward(self, st: LevelState, mlp: MLPDevice, rays=None, impl=0, loss_mults=None, stats=None):
    """Accumulates parameter gradients of one level into mlp.grads (fp32).

    The bias gradient of a trunk layer, and of the bottleneck, is the column sum of its weight-gradient GEMM's B
    operand (the stored bf16 dY): `ops.gemm_wgrad` (`bsum`) takes it from the tiles the GEMM stages, with no
    extra pass over HBM.
    """
    plan = mlp.plan
    trunk = plan.by_role('trunk')
    # the trunk's input-gradient chain runs as one launch
    chained = self._use_chain(plan, st.M, impl) and len(trunk) > 1
    if st.bwd is None:
      st.bwd = BwdScratch(plan, st.M, chained, self.device)
    lm = _loss_args(loss_mults)
    if plan.top == 'view':
      self._view_bwd(st, mlp, rays, impl, lm, stats)
    else:
      self._heads_bwd(st, mlp, rays, impl, lm, stats)
    if plan.density_normals:
      self._tangent_bwd(st, mlp, impl)
    self._trunk_bwd(st, mlp, impl, chained)

  def _slab_dgrad(self, st, mlp, slab, impl):
    """d x_last = act'(x_last) * (slab @ wcat_kn^T): one dgrad over the head-gradient slab."""
    ops.gemm(L.GEMM_DGRAD, slab, mlp.wcat_kn, st.bwd.dy[0], m=st.M, n=mlp.plan.cfg.net_width,
             k=mlp.plan.slab_cols, impl=impl, **self._act_grad(mlp.plan, st, -1))

  def _heads_bwd(self, st, mlp, rays, impl, lm, stats):
    """Top of a trunk without a view branch: colourless normals stage, density (or stacked) and narrow heads."""
    plan = mlp.plan
    sc, g = st.bwd, mlp.grads
    d = plan.one('density')
    if plan.normals_stage:
      ops.normals_bwd(st.M, st.S, st.heads.get('grad_pred'), st.rgd, rays.viewdirs, st.comp['weights'], *lm,
                      st.d_raw_density, st.d_heads.get('grad_pred'), st.d_rgd, head_grads=sc.dhead, stats=stats,
                      d_raw_rgb=st.d_raw_rgb if sc.dhead is not None else None)
    # the stacked head splits its weight gradient between the two heads' master matrices
    split = dict(dw2=mlp.W(plan.one('rgb'), g), dw_split=1) if plan.top == 'stacked' else {}
    if plan.slab_cols:
      # d x_last against [w_density | W_grad_pred (| W_rgb)]; the heads' weight and bias gradients follow
      self._slab_dgrad(st, mlp, sc.dhead, impl)
      ops.head_bwd(st.x_last, mlp.w_head, st.d_raw_head, plan.head_n, d.in_pad, dx=None, dw=mlp.W(d, g),
                   db=mlp.b(d, g), **split)
      self._narrow_heads_bwd(st, mlp)
    else:
      # input gradient, weight gradients and bias gradients ([b_density | b_rgb]) in one pass.  Features after a
      # skip are constants: dy holds the hidden columns only
      ops.head_bwd(st.x_last, mlp.w_head, st.d_raw_head, plan.head_n, d.in_pad, dx=sc.dy[0], dw=mlp.W(d, g),
                   db=mlp.b(d, g), dx_cols=plan.cfg.net_width, **split, **self._act_grad(plan, st, -1, head=True))

  def _narrow_heads_bwd(self, st: LevelState, mlp: MLPDevice):
    """Parameter gradients of the narrow heads (x^T d_raw), accumulated into mlp.grads."""
    g = mlp.grads
    for sp in mlp.plan.narrow:
      ops.head_bwd(st.x_last, mlp.w_nk[sp.name], st.d_heads[sp.role], sp.out_dim, sp.in_pad, dx=None,
                   dw=mlp.W(sp, g), db=mlp.b(sp, g))

  def _view_mlp_bwd(self, st, mlp, impl):
    """rgb head and view MLP backward into sc.d_vin[:, :d_vin_cols]: [ d bottleneck (| d direction encoding | d n.v)
    (| d GLO) ] (no activation on vin), the sum of every consumer's contribution."""
    plan = mlp.plan
    sc, g = st.bwd, mlp.grads
    views, r = plan.by_role('view'), plan.one('rgb')
    Wv = plan.cfg.net_width_viewdirs
    n = plan.d_vin_cols
    d_rgb = st.d_raw_rgb.view(st.M, 3)
    if plan.rgb_vin == 'all':
      # no view MLP: the rgb head reads vin, its input gradient is all of d vin
      ops.head_bwd(st.vin, mlp.w_nk[r.name], d_rgb, r.out_dim, r.in_pad, dx=sc.d_vin, dw=mlp.W(r, g), db=mlp.b(r, g),
                   dx_cols=n)
      return
    # the running sum of d vin before view layer 0 adds its part: parts[j % 2] holds contributions 0..j
    parts, j = sc.d_vin_parts, 0
    dcur = sc.dv[0]
    if plan.rgb_vin == 'tail':
      # a view MLP ending on a skip: the head reads [hidden | vin]; the vin columns' gradient is the first part
      ops.head_bwd(st.v_last, mlp.w_nk[r.name], d_rgb, r.out_dim, r.in_pad, dx=dcur, dw=mlp.W(r, g), db=mlp.b(r, g),
                   dxsum=mlp.b(views[-1], g), dx_cols=Wv, dx2=parts[0], **self._act_grad(plan, st, -1, True, True))
      j = 1
    else:
      ops.head_bwd(st.v_last, mlp.w_nk[r.name], d_rgb, r.out_dim, r.in_pad, dx=dcur, dw=mlp.W(r, g), db=mlp.b(r, g),
                   dxsum=mlp.b(views[-1], g), **self._act_grad(plan, st, -1, True, True))
    for i in range(len(views) - 1, -1, -1):
      sp = views[i]
      xin = st.vin if i == 0 else st.vacts[i - 1]
      ops.gemm(L.GEMM_WGRAD, xin, dcur, mlp.W(sp, g), m=sp.in_pad, n=Wv, k=st.M, impl=impl)
      if i > 0:
        if i in plan.view_skips:
          # this layer also consumed vin (skip concat): its contribution, added to the parts so far
          ops.gemm(L.GEMM_DGRAD, dcur, mlp.w_kn[sp.name][Wv:], parts[j % 2], m=st.M, n=plan.vin_pad, k=Wv,
                   addend=parts[(j - 1) % 2] if j else None, impl=impl)
          j += 1
        nxt = sc.dv[1] if dcur is sc.dv[0] else sc.dv[0]
        ops.gemm(L.GEMM_DGRAD, dcur, mlp.w_kn[sp.name], nxt, m=st.M, n=Wv, k=Wv, colsum=mlp.b(views[i - 1], g),
                 impl=impl, **self._act_grad(plan, st, i - 1, view=True))
        dcur = nxt
    # d vin = dcur * Wv0^T (+ the other consumers' parts)
    ops.gemm(L.GEMM_DGRAD, dcur, mlp.w_kn[views[0].name], sc.d_vin[:, :n], m=st.M, n=n, k=Wv,
             addend=parts[(j - 1) % 2][:, :n] if j else None, impl=impl)

  def _view_bwd(self, st, mlp, rays, impl, lm, stats):
    """Top of a trunk with a view branch: view MLP, GLO, Ref-NeRF stage or direction encoding, bottleneck."""
    plan = mlp.plan
    sc, g = st.bwd, mlp.grads
    bt, d = plan.one('bottleneck'), plan.one('density')
    bw = plan.enc_col0
    self._view_mlp_bwd(st, mlp, impl)
    if st.glo_vec is not None:
      # the GLO columns of vin, summed over the samples; read before the Ref-NeRF stage re-uses the slab columns
      g0 = plan.glo_col0
      d_glo = sc.d_vin.view(st.B, st.S, plan.vin_pad)[:, :, g0:g0 + plan.glo_features].float().sum(1)
      self.params.seg('Embed_0', self.params.grads).view(self.mcfg.num_glo_embeddings, -1).index_add_(
          0, rays.cam_idx[:, 0].long(), d_glo)
    if plan.ref_stage:
      ops.refdir_bwd(*self._refdir_args(st, mlp, rays.viewdirs), st.comp['weights'], sc.d_vin, *lm, st.d_raw_density,
                     st.d_heads.get('diffuse'), st.d_heads.get('tint'), st.d_heads.get('grad_pred'),
                     st.d_heads['roughness'].view(st.M) if 'roughness' in st.d_heads else None, st.d_rgd, stats)
      self._narrow_heads_bwd(st, mlp)
    # bottleneck dW + db (models.py:527), then the Dense(1) density head's dW (models.py:460) in a pass of its own:
    # summed inside the GEMM, the weighted x_last tiles take more shared-memory bandwidth from the MMAs than the
    # pass takes HBM time (DESIGN.md section 3)
    if plan.has_bottleneck:
      ops.gemm_wgrad(st.x_last, sc.d_vin[:, :bw], mlp.W(bt, g), m=bt.in_pad, n=bw, k=st.M, bsum=mlp.b(bt, g),
                     impl=impl)
    ops.head_bwd(st.x_last, st.x_last, st.d_raw_density.view(st.M, 1), 1, d.in_pad, dw=mlp.W(d, g).view(-1, 1))
    if plan.ref_stage:
      # d x_last = act'(x_last) * ([d bottleneck | head gradients] @ [W_b | w_heads]^T); without a bottleneck the
      # slab holds the head gradients only
      self._slab_dgrad(st, mlp, sc.d_vin, impl)
    else:
      # d x_last = (dbott * Wb^T + d_raw_density (x) w_density) * act'(x_last)
      ops.gemm(L.GEMM_DGRAD, sc.d_vin[:, :bw], mlp.w_kn[bt.name], sc.dy[0], m=st.M, n=plan.cfg.net_width, k=bw,
               rowv=st.d_raw_density.view(st.M), colv=mlp.colv_density, impl=impl, **self._act_grad(plan, st, -1))
    # bias gradient of the density head: a plain sum of d_raw_density
    mlp.b(d, g).add_(st.d_raw_density.sum())

  def _tangent_bwd(self, st, mlp, impl):
    """Adjoint of the tangent chain: H_last = relu'(x_last) * (d_rgd (x) w_density), three streams.

    A smooth activation starts the chain with H_last = a'(z_last) * T_last, T_last = d_rgd (x) w_density, and adds the
    second-order term a''(z_last) * sum_s T_last u_last into the trunk-top gradient dy[0]; its layers below run
    interleaved with the trunk backward (_trunk_bwd)."""
    plan = mlp.plan
    sc, g = st.bwd, mlp.grads
    W = plan.cfg.net_width
    d = plan.one('density')
    trunk = plan.by_role('trunk')
    hcur, hoth = sc.h[0], sc.h[1]
    relu = plan.act == L.ACT_RELU
    ops.outer_mask(st.d_rgd.view(3 * st.M), mlp.colv_density, st.bits[-1] if relu else None, hcur, rows=3 * st.M,
                   n=W, mask_mod=st.M)
    if not relu:
      self._tangent_second_order(st, mlp, len(trunk) - 1, hcur, sc.dy[0], impl)
    ops.head_bwd(st.t_last, mlp.w_nk[d.name], st.d_rgd.view(3 * st.M, 1), 1, d.in_pad, dx=None,
                 dw=mlp.W(d, g), db=None)
    if not relu:
      return
    for i in range(len(trunk) - 1, -1, -1):
      sp = trunk[i]
      tin = st.tfeat if i == 0 else st.tacts[i - 1]
      ops.gemm(L.GEMM_WGRAD, tin, hcur, mlp.W(sp, g), m=sp.in_pad, n=W, k=3 * st.M, impl=impl)
      if i > 0:
        ops.gemm(L.GEMM_DGRAD, hcur, mlp.w_kn[sp.name], hoth, m=3 * st.M, n=W, k=W,
                 maskbits=st.bits[i - 1], mask_mod=st.M, impl=impl)
        hcur, hoth = hoth, hcur

  def _tangent_second_order(self, st, mlp, i, t_adj, g_out, impl):
    """Trunk layer i of the tangent backward through a smooth activation: t_adj = T_i = dL/dt_i (three streams)
    becomes dL/du_i = a'(z_i) T_i in place, and g_out receives (dy[0], the trunk-top gradient: is added) the
    second-order part of dL/dz_i, a''(z_i) sum_s T_i u_i.  u_i = t_{i-1} W_i is not stored by the forward: it is
    recomputed here from the stored tangent input of the layer (features included after a skip)."""
    plan = mlp.plan
    sc, sp = st.bwd, plan.by_role('trunk')[i]
    tin = st.tfeat if i == 0 else st.tacts[i - 1]
    ops.gemm(L.GEMM_FWD, tin, mlp.w_nk[sp.name], sc.u, m=3 * st.M, n=plan.cfg.net_width, k=sp.in_pad, impl=impl)
    ops.act_tangent_bwd(plan.act, st.zs[i], t_adj, sc.u, t_adj, g_out, accumulate=g_out is sc.dy[0])

  def _trunk_bwd(self, st, mlp, impl, chained):
    """Trunk backward from dy[0] = d loss / d (output of the last trunk layer).  With density normals through a
    smooth activation, the tangent chain (sc.h, from _tangent_bwd) runs here too, one layer ahead: its layer i - 1
    yields the second-order term g that the primal DGRAD into layer i - 1 adds."""
    sc, g = st.bwd, mlp.grads
    plan = mlp.plan
    W = plan.cfg.net_width
    trunk = plan.by_role('trunk')
    nl = len(trunk)
    if chained:
      # dyl[i] = d loss / d (output of trunk layer i); dyl[nl-1] is sc.dy[0], produced at the top of the trunk
      dyl = [sc.dy[nl - 1 - i] for i in range(nl)]
      ops.mlp_chain(self._chain_bwd_desc(st, mlp, dyl))
      for i in range(nl - 1, -1, -1):
        xin = st.feat if i == 0 else st.acts[i - 1]
        ops.gemm_wgrad(xin, dyl[i], mlp.W(trunk[i], g), m=trunk[i].in_pad, n=W, k=st.M, bsum=mlp.b(trunk[i], g),
                       impl=impl)
      return
    cur, other = sc.dy[0], sc.dy[1]
    tangent = plan.density_normals and plan.act != L.ACT_RELU
    hcur, hoth = sc.h if tangent else (None, None)
    for i in range(nl - 1, -1, -1):
      sp = trunk[i]
      xin = st.feat if i == 0 else st.acts[i - 1]
      ops.gemm_wgrad(xin, cur, mlp.W(sp, g), m=sp.in_pad, n=W, k=st.M, bsum=mlp.b(sp, g), impl=impl)
      if tangent:
        tin = st.tfeat if i == 0 else st.tacts[i - 1]
        ops.gemm(L.GEMM_WGRAD, tin, hcur, mlp.W(sp, g), m=sp.in_pad, n=W, k=3 * st.M, impl=impl)
      if i > 0:
        if tangent:
          # T_{i-1} = dL/du_i W_i^T, then dL/du_{i-1} (in place) and the second-order term g of layer i - 1
          ops.gemm(L.GEMM_DGRAD, hcur, mlp.w_kn[sp.name], hoth, m=3 * st.M, n=W, k=W, impl=impl)
          self._tangent_second_order(st, mlp, i - 1, hoth, sc.g, impl)
          hcur, hoth = hoth, hcur
        # only the hidden part of the input carries gradient (features are constants:
        # stop_gradient(sdist), models.py:200-201)
        ops.gemm(L.GEMM_DGRAD, cur, mlp.w_kn[sp.name], other, m=st.M, n=W, k=W, addend=sc.g if tangent else None,
                 impl=impl, **self._act_grad(plan, st, i - 1))
        cur, other = other, cur


def construct_model(rng, rays, config, device=None):
  """models.py:315-338.  `config` is a configs.Bundle; `rng` an int seed (or None -> 0)."""
  bundle = config if isinstance(config, configs.Bundle) else configs.Bundle(config=config)
  model = Model(bundle, device=device)
  seed = 0 if rng is None else (rng if isinstance(rng, int) else int(torch.as_tensor(rng).sum()))
  variables = model.init(seed)
  return model, variables


def render_image(render_fn, rays, rng, config, verbose=True, world_size=1, rank=0):
  """Render all pixels of an image in chunks (models.py:625-706).

  render_fn(rng, chunk_rays) -> (renderings, ray_history) with every rank's rays gathered
  (multinerf_b200.train_utils.create_render_fn).  `rays` leaves are [H, W, n].
  """
  cfg = config.config if isinstance(config, configs.Bundle) else config
  height, width = np.asarray(rays.origins).shape[:2] if not isinstance(rays.origins, torch.Tensor) \
      else rays.origins.shape[:2]
  num_rays = height * width
  flat = rays.map(lambda r: r.reshape((num_rays, -1)))
  chunks = []
  idx0s = range(0, num_rays, cfg.render_chunk_size)
  for i_chunk, idx0 in enumerate(idx0s):
    if verbose and i_chunk % max(1, len(idx0s) // 10) == 0:
      print(f'Rendering chunk {i_chunk}/{len(idx0s)-1}')
    chunk = flat.map(lambda r: r[idx0:idx0 + cfg.render_chunk_size])
    actual = chunk.origins.shape[0]
    rem = actual % world_size
    padding = 0
    if rem != 0:
      padding = world_size - rem
      def pad(r):
        if isinstance(r, torch.Tensor):
          return torch.cat([r, r[-1:].expand(padding, *r.shape[1:])], 0)
        return np.concatenate([r, np.repeat(r[-1:], padding, 0)], 0)
      chunk = chunk.map(pad)
    per = chunk.origins.shape[0] // world_size
    mine = chunk.map(lambda r: r[rank * per:(rank + 1) * per])
    chunk_renderings, _ = render_fn(rng, mine)
    if padding > 0:
      chunk_renderings = [{k: (v[:-padding] if not k.startswith('ray_') else v) for k, v in r.items()}
                          for r in chunk_renderings]
    out = dict(chunk_renderings[-1])
    for k in chunk_renderings[0]:
      if k.startswith('ray_'):
        out[k] = [r[k] for r in chunk_renderings]
    chunks.append(out)
  rendering = {}
  for k in chunks[0]:
    if k.startswith('ray_'):
      rendering[k] = [torch.cat([c[k][i] for c in chunks]) for i in range(len(chunks[0][k]))]
    else:
      z = torch.cat([c[k] for c in chunks])
      rendering[k] = z.reshape((height, width) + tuple(z.shape[1:]))
  keys = [k for k in rendering if k.startswith('ray_')]
  if keys:
    n = rendering[keys[0]][0].shape[0]
    # the reference takes jax.random.permutation(PRNGKey(0)) (threefry, not reproducible here):
    # a fixed numpy permutation plays the same role
    ray_idx = torch.as_tensor(np.random.default_rng(0).permutation(n)[:cfg.vis_num_rays])
    for k in keys:
      rendering[k] = [r[ray_idx.to(r.device)] for r in rendering[k]]
  return rendering
