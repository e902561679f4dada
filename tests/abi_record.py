"""Records the C-ABI calls (`mnrf_*`) the models make, without a GPU: the recorder behind tools/abi_trace.py and
the launch-coverage audit (test_launch_coverage_cpu.py).

`lib.load` is replaced by a fake library that records every call and returns 0, and `lib.ptr` by one that returns
the tensor's address and keeps the tensor alive, so that the CPU allocator cannot hand a freed address to a later
tensor and make the trace depend on the run.  Each call is kept twice:
  - `calls`: the canonical record of tools/abi_trace.py -- symbol, scalar arguments and ctypes descriptors expanded
    field by field, pointers numbered in order of first appearance;
  - `named`: (symbol, {parameter name: value}) with the parameter names of include/mnrf.h, descriptors as dicts of
    their fields and pointers as raw addresses (None for NULL), so that a launch can be classified and planned
    (mnrf_gemm_plan reads addresses only).
A helper module, not a test module.
"""
import contextlib
import ctypes as C
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'mnrf.h')
_BYREF = type(C.byref(C.c_int()))


def _bundles(configs):
  """(name, bundle factory, environment) of every case: each MLP layout and host branch of models.py."""
  def mini360(b):
    b.model.num_prop_samples, b.model.num_nerf_samples = 32, 16
    b.prop_mlp.net_depth, b.prop_mlp.net_width = 2, 64
    b.nerf_mlp.net_depth, b.nerf_mlp.net_width = 6, 128
    b.nerf_mlp.bottleneck_width, b.nerf_mlp.net_width_viewdirs = 64, 64
    return b

  def narrow_blender(b):
    b.prop_mlp.net_width, b.nerf_mlp.net_width = 64, 128
    return b

  def view_independent(b, normals, glo):
    b.model.use_viewdirs = False
    if glo:
      b.model.num_glo_features, b.model.num_glo_embeddings = 4, 3
    if normals:
      normal_losses(b, pred=True)
    return b

  def normal_losses(b, pred, mlps=None):
    c = b.config
    for mlp in mlps or (b.prop_mlp, b.nerf_mlp):
      mlp.disable_density_normals, mlp.enable_pred_normals = False, pred
    c.orientation_loss_mult, c.orientation_coarse_loss_mult = 0.1, 0.01
    c.orientation_loss_target = 'normals_pred' if pred else 'normals'
    if pred:
      c.predicted_normal_loss_mult, c.predicted_normal_coarse_loss_mult = 3e-4, 3e-5
    return b

  def refnerf_density_normals(b):
    b.nerf_mlp.enable_pred_normals = False
    b.config.orientation_loss_target = 'normals'
    b.config.predicted_normal_loss_mult = b.config.predicted_normal_coarse_loss_mult = 0.0
    return b

  def glo(b):
    b.model.num_glo_features, b.model.num_glo_embeddings, b.model.single_mlp = 4, 3, False
    return b

  def glo_refnerf(b):
    glo(b)      # a PropMLP without normals: no normal losses on the proposal levels
    b.config.orientation_coarse_loss_mult = b.config.predicted_normal_coarse_loss_mult = 0.0
    b.nerf_mlp.net_depth_viewdirs = 2      # GLO columns are written through a contiguous view input
    return b

  def noise_bg(b):
    b.nerf_mlp.bottleneck_noise, b.nerf_mlp.density_noise, b.prop_mlp.density_noise = 0.1, 1.0, 1.0
    b.model.bg_intensity_range = (0.0, 1.0)
    return b

  def deep_view(b):
    b.nerf_mlp.net_depth_viewdirs, b.nerf_mlp.skip_layer_dir = 6, 4
    return b

  def single(b):
    b.model.single_mlp = True
    return b

  def robust(b, patch_size=8):
    c = b.config
    c.data_loss_type, c.patch_size, c.enable_robustnerf_loss = 'robustnerf', patch_size, True
    c.robustnerf_inner_patch_size, c.robustnerf_smoothed_filter_size = 4, 3
    return b

  def activation(b, act, mlps=None):
    for mlp in mlps or (b.prop_mlp, b.nerf_mlp):
      mlp.net_activation = act
    return b

  def chunks(b, size=32):
    b.config.train_chunk_size = size     # two passes of the B = 64 rays of run_case
    return b

  def skip_end(b):
    view_independent(b, normals=False, glo=False)
    b.prop_mlp.net_depth = 5
    return b

  def view_layout(b, bottleneck=None, depth=None, skip=None):
    n = b.nerf_mlp
    n.bottleneck_width = n.bottleneck_width if bottleneck is None else bottleneck
    n.net_depth_viewdirs = n.net_depth_viewdirs if depth is None else depth
    n.skip_layer_dir = n.skip_layer_dir if skip is None else skip
    return b

  b360, b256, bref, braw = (configs.bundle_360, configs.bundle_blender_256, configs.bundle_blender_refnerf,
                            configs.bundle_llff_raw)
  return [
      ('360', b360, {}),
      ('360_nochain', b360, {'MNRF_CHAIN': '0'}),
      ('blender_256', b256, {}),
      ('blender_refnerf', bref, {}),
      ('llff_raw', braw, {}),
      ('mini360', lambda: mini360(b360()), {}),
      ('blender_256_narrow', lambda: narrow_blender(b256()), {}),
      ('viewindep_normals_glo', lambda: view_independent(b256(), True, True), {}),
      ('viewindep_plain', lambda: view_independent(b256(), False, False), {}),
      ('viewindep_360', lambda: view_independent(b360(), False, False), {}),
      ('viewindep_narrow_normals_glo', lambda: view_independent(narrow_blender(b256()), True, True), {}),
      ('viewindep_skip_end', lambda: skip_end(narrow_blender(b256())), {}),
      ('prop_normals_pred', lambda: normal_losses(b256(), pred=True), {}),
      ('prop_normals_density', lambda: normal_losses(b256(), pred=False), {}),
      ('prop_normals_narrow', lambda: normal_losses(narrow_blender(b256()), pred=True), {}),
      ('contract_normals', lambda: normal_losses(mini360(b360()), pred=True), {}),
      ('refnerf_density_normals', lambda: refnerf_density_normals(bref()), {}),
      ('glo_360', lambda: glo(b360()), {}),
      ('glo_refnerf', lambda: glo_refnerf(bref()), {}),
      ('noise_bg', lambda: noise_bg(b256()), {}),
      ('deep_view', lambda: deep_view(b256()), {}),
      ('single_mlp', lambda: single(b256()), {}),
      ('robustnerf', lambda: robust(b360()), {}),
      ('refnerf_no_bottleneck', lambda: view_layout(bref(), bottleneck=0), {}),
      ('view_depth0_360', lambda: view_layout(b360(), depth=0), {}),
      ('view_depth0_glo', lambda: view_layout(glo(b256()), depth=0), {}),
      ('view_skips_end_glo', lambda: view_layout(glo(b256()), depth=9, skip=4), {}),
      ('softplus_normals', lambda: activation(normal_losses(b256(), pred=True), 'softplus'), {}),
      ('silu_refnerf', lambda: activation(bref(), 'silu'), {}),
      ('chunks_360', lambda: chunks(b360()), {}),
      # a 32-ray pass holds whole 4 x 4 patches; 8 x 8 patches do not divide it
      ('chunks_robust', lambda: chunks(robust(b360(), patch_size=4)), {}),
  ]


def _mesh_bundles(configs):
  """(name, bundle factory) of the models whose mesh-extraction queries are traced: 360.gin's layout with the
  contraction, reduced (mini360), a one-level blender_256 whose 256-wide trunk runs chained (plumbing), and mini360
  with density normals, whose queries take the tangent encoder (contract_normals)."""
  cases = dict((n, fn) for n, fn, _ in _bundles(configs))

  def plumbing():
    b = configs.bundle_blender_256()
    b.model.num_levels, b.model.num_nerf_samples = 1, 32
    return b
  return [('mini360', cases['mini360']), ('plumbing', plumbing), ('contract_normals', cases['contract_normals'])]


def prototypes(path=HEADER):
  """{symbol: [parameter names]} of every `int mnrf_*(...)` prototype of include/mnrf.h."""
  text = re.sub(r'/\*.*?\*/', ' ', open(path).read(), flags=re.S)
  protos = {}
  for name, params in re.findall(r'\b(?:int|const char\s*\*)\s*(mnrf_\w+)\s*\(([^)]*)\)\s*;', text):
    params = ' '.join(params.split())
    protos[name] = [] if params in ('', 'void') else [re.findall(r'\w+', p)[-1] for p in params.split(',')]
  return protos


def parameter_names(signatures):
  """{symbol: [parameter names]} of the ctypes signatures of lib.py, named by the header's prototypes.  Raises when a
  symbol has no prototype or the two disagree on the argument count."""
  protos = prototypes()
  names = {}
  for sym, (_, args) in signatures.items():
    if sym not in protos:
      raise RuntimeError(f'{sym}: declared in lib.py, but include/mnrf.h has no prototype of it')
    if len(protos[sym]) != len(args):
      raise RuntimeError(f'{sym}: include/mnrf.h declares {len(protos[sym])} parameters, lib.py {len(args)}')
    names[sym] = protos[sym]
  return names


class Recorder:
  """Fake libmnrf: every `mnrf_*` attribute is a function that appends one canonical and one named record and
  returns 0.  names: {symbol: [parameter names]} (parameter_names); None keeps the canonical record only."""

  def __init__(self, names=None):
    self.calls, self.ids, self.alive = [], {}, []
    self.names, self.named = names, []

  def pid(self, addr):
    if not addr:
      return None
    return 'p%d' % self.ids.setdefault(addr, len(self.ids))

  def value(self, v, ctype=None):
    if isinstance(v, _BYREF):
      return self.value(v._obj)
    if isinstance(v, C.Structure):
      return {name: self.value(getattr(v, name), t) for name, t, *_ in v._fields_}
    if isinstance(v, C.Array):
      return [self.value(x, v._type_) for x in v]
    if isinstance(v, C.c_void_p):
      return self.pid(v.value)
    if ctype is C.c_void_p:
      return self.pid(v)
    if isinstance(v, bytes):
      return v.decode()
    if isinstance(v, float):
      return repr(v)
    return v

  @staticmethod
  def raw(v, ctype=None):
    """The argument as the kernel sees it: descriptors as dicts, pointers as addresses (None for NULL)."""
    if isinstance(v, _BYREF):
      return Recorder.raw(v._obj)
    if isinstance(v, C.Structure):
      return {name: Recorder.raw(getattr(v, name), t) for name, t, *_ in v._fields_}
    if isinstance(v, C.Array):
      return [Recorder.raw(x, v._type_) for x in v]
    if isinstance(v, C.c_void_p):
      return v.value or None
    if ctype is C.c_void_p:
      return v or None
    if isinstance(v, (C.c_int32, C.c_int64, C.c_float, C.c_double)):
      return v.value
    return v

  def __getattr__(self, name):
    if not name.startswith('mnrf_'):
      raise AttributeError(name)

    def call(*args):
      self.calls.append([name] + [self.value(a) for a in args])
      if self.names is not None:
        params = self.names[name]
        if len(params) != len(args):
          raise RuntimeError(f'{name} called with {len(args)} arguments; include/mnrf.h declares {len(params)}')
        self.named.append((name, {p: self.raw(a) for p, a in zip(params, args)}))
      return 0
    return call


@contextlib.contextmanager
def recording(lib, env=None, names=None):
  """Run the block with `rec` (yielded) in place of libmnrf: ops.* launches record instead of running, on CPU
  tensors."""
  import torch
  env = env or {}
  rec = Recorder(names)
  saved = {k: os.environ.get(k) for k in env}
  os.environ.update(env)
  patches = [(lib, 'load', lambda build_if_missing=False: rec), (lib, 'check', lambda rc: None),
             (lib, 'require_device', lambda: rec), (lib, 'stream_ptr', lambda: C.c_void_p(0))]

  def ptr(t):
    if t is None:
      return None
    rec.alive.append(t)
    return C.c_void_p(t.data_ptr())
  patches += [(lib, 'ptr', ptr), (torch.cuda, 'is_current_stream_capturing', lambda: False),
              (torch.Tensor, 'pin_memory', lambda self, *a, **k: self)]
  old = [(obj, name, getattr(obj, name)) for obj, name, _ in patches]
  try:
    for obj, name, fn in patches:
      setattr(obj, name, fn)
    yield rec
  finally:
    for obj, name, fn in old:
      setattr(obj, name, fn)
    for k, val in saved.items():
      if val is None:
        os.environ.pop(k, None)
      else:
        os.environ[k] = val


def _result(rec, n_train):
  out = dict(train_calls=n_train, render_calls=len(rec.calls) - n_train, calls=rec.calls)
  if rec.names is not None:
    out['named'] = rec.named
  return out


def run_case(pkg, bundle_fn, env, B=64, names=None):
  """The calls of one train step and one render call of the bundle's model on B synthetic rays.  B=None: the
  configuration's own batch_size.  names (parameter_names): also keep the named records."""
  import torch
  lib, models, train_utils, utils = pkg
  with recording(lib, env, names) as rec:
    bundle = bundle_fn()
    if B is None:
      B = bundle.config.batch_size
    m = bundle.model
    rng = np.random.default_rng(0)
    f = np.float32
    o = rng.normal(size=(B, 3))
    o = o / np.linalg.norm(o, axis=-1, keepdims=True) * 4.0
    d = -o / 4.0 + rng.normal(size=(B, 3)) * 0.1
    v = d / np.linalg.norm(d, axis=-1, keepdims=True)
    extra = {}
    if bundle.config.rawnerf_mode:
      extra = dict(exposure_idx=rng.integers(0, 3, (B, 1)).astype(np.int32),
                   exposure_values=rng.uniform(0.5, 2.0, (B, 1)).astype(f))
    rays = utils.Rays(origins=o.astype(f), directions=(v * rng.uniform(0.8, 1.2, (B, 1))).astype(f),
                      viewdirs=v.astype(f), radii=rng.uniform(5e-4, 1e-3, (B, 1)).astype(f),
                      imageplane=np.zeros((B, 2), f), lossmult=np.ones((B, 1), f),
                      near=np.full((B, 1), bundle.config.near, f), far=np.full((B, 1), bundle.config.far, f),
                      cam_idx=rng.integers(0, 3, (B, 1)).astype(np.int32), **extra)
    model = models.Model(bundle, device='cpu')
    variables = model.init(1)
    S = [m.num_prop_samples] * (m.num_levels - 1) + [m.num_nerf_samples]
    t = lambda *shape: torch.tensor(rng.uniform(0, 1, shape).astype(f))
    draws = {'jitter': [t(B) if m.single_jitter else t(B, s) for s in S],
             'density_noise': [t(B, s) for s in S], 'bg': [t(B, 3) for _ in S],
             'bottleneck_noise': [t(B * s, max(bundle.nerf_mlp.bottleneck_width, 1)) for s in S]}
    step = train_utils.create_train_step(model, bundle.config, use_graph=False)
    batch = utils.Batch(rays=rays, rgb=rng.uniform(0, 1, (B, 3)).astype(f))
    step(draws, train_utils.TrainState(variables), batch, None, 0.5)
    n_train = len(rec.calls)
    model(None, rays, 0.5, True)
    return _result(rec, n_train)


def run_mesh_case(pkg, bundle_fn, N=300, names=None):
  """The calls of mesh extraction's MLP queries (Model.query_density, then Model.query_radiance) on N points of the
  unit ball.  Marching cubes, fusion and post-processing are not traced: under the fake library their scans come
  back empty."""
  lib, models, _, _ = pkg
  with recording(lib, None, names) as rec:
    bundle = bundle_fn()
    rng = np.random.default_rng(1)
    p = rng.uniform(-0.7, 0.7, (N, 3)).astype(np.float32)
    v = rng.normal(size=(N, 3))
    v = (v / np.linalg.norm(v, axis=-1, keepdims=True)).astype(np.float32)
    model = models.Model(bundle, device='cpu')
    model.init(1)
    model.query_density(p, 1e-4)
    model.query_radiance(p, 1e-4, v)
    return _result(rec, len(rec.calls))
