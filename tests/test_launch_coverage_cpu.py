"""Launch-coverage audit: every launch class (tests/launch_classes.py) that the shipped model configurations reach
must be the class of a launch an fp64 test checks.

The model side is the recorded calls (tests/abi_record.py) of one train step and one render call of every case of
abi_record._bundles, traced at B = 64 and at each configuration's own batch_size, and of mesh extraction's MLP
queries.  The fp64 side is the launches the fp64 GPU modules make, taken from the modules themselves (their
`fp64_launches`, run under the same recording library on CPU buffers), so the audit and the GPU tests cannot drift
apart.  Runs without a GPU: the plans come from the library's host-only planners.
"""
import collections
import functools
import importlib

import pytest

import abi_record
import launch_classes

# The fp64 module whose `fp64_launches(ops)` covers each audited entry point.
FP64_MODULES = {
    'mnrf_gemm': 'test_gpu_gemm_matrix',
    'mnrf_gemm_wgrad': 'test_gpu_gemm_matrix',
    'mnrf_head_fwd': 'test_gpu_heads_fp64',
    'mnrf_head_bwd': 'test_gpu_heads_fp64',
}

# Entry points the models reach that this audit does not check yet: their fp64 modules do not expose their launches
# (fp64_launches) and they have no class function, so nothing here says their launches are covered.  This is not a
# list of justified exemptions; each entry leaves when its module gains fp64_launches and its class function.  A
# symbol that is neither here nor in FP64_MODULES fails test_every_traced_entry_point_is_audited.
NOT_AUDITED = {
    s: 'the fp64 module of this kernel does not expose its launches yet'
    for s in ('mnrf_sample_level', 'mnrf_encode', 'mnrf_encode_points', 'mnrf_encode_points_tangent',
              'mnrf_viewdir_enc', 'mnrf_composite_fwd', 'mnrf_composite_bwd', 'mnrf_point_rgb', 'mnrf_mlp_chain',
              'mnrf_clip_adam', 'mnrf_pack_weights_batched', 'mnrf_refdir_fwd',
              'mnrf_refdir_bwd', 'mnrf_normals_fwd', 'mnrf_normals_bwd', 'mnrf_outer_mask', 'mnrf_act_tangent_bwd',
              'mnrf_robust_mask', 'mnrf_quantile')
}


def _pkg():
  from multinerf_b200 import configs, lib, models, train_utils, utils
  return configs, (lib, models, train_utils, utils)


def _names():
  from multinerf_b200 import lib
  return abi_record.parameter_names(lib._SIGNATURES)


@pytest.fixture(scope='module')
def library():
  """The built library: the GEMM classes ask its host-only planner."""
  from multinerf_b200 import lib
  return lib.load()


@functools.lru_cache(maxsize=None)
def model_calls(batch):
  """{case: [(symbol, args)]} of every model case at B = 64 (batch 'small') or its own batch_size ('config'), and
  of the mesh queries (cases 'mesh:<name>')."""
  configs, pkg = _pkg()
  names = _names()
  out = {}
  for name, fn, env in abi_record._bundles(configs):
    out[name] = abi_record.run_case(pkg, fn, env, B=64 if batch == 'small' else None, names=names)['named']
  if batch == 'small':
    for name, fn in abi_record._mesh_bundles(configs):
      out['mesh:' + name] = abi_record.run_mesh_case(pkg, fn, names=names)['named']
  return out


def fp64_calls(modules=None):
  """{module: [(symbol, args)]} of the launches each fp64 module's `fp64_launches` makes."""
  from multinerf_b200 import lib, ops
  out = {}
  for mod in sorted(set(FP64_MODULES.values()) if modules is None else modules):
    with abi_record.recording(lib, names=_names()) as rec:
      importlib.import_module(mod).fp64_launches(ops)
    out[mod] = rec.named
  return out


def classes(calls_by_source):
  """{symbol: {class: set of sources}} of the audited entry points."""
  got = collections.defaultdict(lambda: collections.defaultdict(set))
  for src, calls in calls_by_source.items():
    for sym, args in calls:
      if sym in FP64_MODULES:
        got[sym][launch_classes.classify(sym, args)].add(src)
  return got


def missing(model, fp64):
  """[(symbol, class, model cases)] of the model classes without an fp64 launch of the same class."""
  out = []
  for sym, cls in sorted(model.items()):
    for c, cases in sorted(cls.items(), key=repr):
      if c not in fp64.get(sym, {}):
        out.append((sym, c, sorted(cases)))
  return out


def _report(miss):
  return '\n'.join(f'{sym} {dict(c)} reached by {", ".join(cases)}' for sym, c, cases in miss)


@pytest.fixture(scope='module')
def fp64(library):
  return classes(fp64_calls())


@pytest.mark.parametrize('batch', ['small', 'config'])
def test_model_launches_have_fp64_cases(fp64, batch):
  model = classes(model_calls(batch))
  print(f'\n[launch coverage, batch {batch}] entry point, model classes, fp64 classes')
  for sym in sorted(FP64_MODULES):
    print(f'  {sym:28s} {len(model.get(sym, {})):4d} {len(fp64.get(sym, {})):4d}')
  miss = missing(model, fp64)
  assert not miss, f'launch classes the models reach and no fp64 case checks:\n{_report(miss)}'


def test_every_traced_entry_point_is_audited():
  """A new mnrf_* symbol cannot slip through: every entry point the trace reaches is audited (or listed, with its
  reason, in NOT_AUDITED), and every audited one has a class function."""
  traced = {sym for calls in model_calls('small').values() for sym, _ in calls}
  unknown = traced - set(FP64_MODULES) - set(NOT_AUDITED)
  assert not unknown, f'entry points without a launch class: {sorted(unknown)}'
  assert set(FP64_MODULES) <= set(launch_classes.CLASSES)
  assert not set(FP64_MODULES) & set(NOT_AUDITED)


@pytest.mark.parametrize('module,args,kw', [
    ('test_gpu_gemm_matrix', ('fwd', 38000, 256, 192), {}),
    ('test_gpu_heads_fp64', ('bwd', 2053, 256, 1), dict(out='params', db=False))])
def test_dropping_a_sole_case_fails_the_audit(library, module, args, kw):
  """The audit can fail, and names the class: without the fp64 case that alone covers a class the models reach
  (FWD with bias alone on 256-wide tiles; a head's dW without db), that class and nothing else is reported."""
  mod = importlib.import_module(module)
  i = mod.CASES.index(mod.case(*args, **kw))
  calls = fp64_calls()
  sym, args = calls[module][i]
  lost = launch_classes.classify(sym, args)
  del calls[module][i]
  miss = missing(classes(model_calls('small')), classes(calls))
  assert [(s, c) for s, c, _ in miss] == [(sym, lost)]


def test_parameter_names_match_the_header():
  """Every ctypes signature of lib.py has a prototype in include/mnrf.h with as many parameters."""
  names = _names()
  assert names['mnrf_gemm'][:3] == ['d', 'a', 'b'] and names['mnrf_gemm'][-2:] == ['out', 'stream']
  from multinerf_b200 import lib
  bad = dict(lib._SIGNATURES, mnrf_gemm=(int, lib._SIGNATURES['mnrf_gemm'][1][:-1]))
  with pytest.raises(RuntimeError, match='mnrf_gemm'):
    abi_record.parameter_names(bad)
