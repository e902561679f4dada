"""DGRAD epilogue operand sets of the ping-pong GEMM schedule (gemm_tc_pingpong_kernel, csrc/gemm_tc.cu).

The ping-pong DGRAD has an instance per operand set, which mnrf_gemm_plan reports as `epilogue`: 1 mask bits by TMA
only (the trunk layers), 2 mask bits by TMA and the rank-1 term rowv (x) colv (the NerfMLP bottleneck), 0 the generic
epilogue that tests every optional operand at run time (addend, bf16 mask, mask bits by the epilogue's loads, none).
  test_cases_get_their_set        each case below plans the set it claims (no device needed);
  test_model_launches_get_their_set  every DGRAD of a train step of the full-width 360.gin model gets the set its
                                  operands call for, and the trunk and bottleneck run the fixed sets;
  test_set_same_bits_as_gemm_tc_kernel  each fixed set, at tiles of 128 and 256 columns, with a ragged last row tile
                                  and with mask_mod, equals gemm_tc_kernel (register store) bit for bit and is within
                                  the fp64 bound of tests/gemm_ref.py.
"""
import numpy as np
import pytest
import torch

from test_gpu_gemm_matrix import _bits, case, case_id, layout, plan, run, verify

GENERIC, BITS_TMA, BITS_TMA_RANK1 = 0, 1, 2

# (case, operand set, tile width)
CASES = [
    (case('dgrad', 5000, 1024, 1024, mask='bits'), BITS_TMA, 256),
    (case('dgrad', 5000, 1024, 256, mask='bits', rowv=True), BITS_TMA_RANK1, 256),
    (case('dgrad', 38000, 640, 192, mask='bits'), BITS_TMA, 128),
    (case('dgrad', 38000, 640, 192, mask='bits', rowv=True), BITS_TMA_RANK1, 128),
    (case('dgrad', 3 * 384, 256, 128, mask='bits', rep=3), BITS_TMA, 256),
    (case('dgrad', 3 * 384, 384, 128, mask='bits', rep=3, rowv=True), BITS_TMA_RANK1, 128),
]
# the generic set: any operand besides TMA-loaded mask bits and the rank-1 term
GENERIC_CASES = [
    case('dgrad', 5000, 1024, 256, mask='bits', rowv=True, addend=True),
    case('dgrad', 5000, 1024, 256, mask='bits_odd', rowv=True),
    case('dgrad', 5000, 640, 256, mask='bf16'),
    case('dgrad', 5000, 640, 256),
    case('dgrad', 3 * 200, 256, 128, mask='bits', rep=3),
    case('fwd', 5000, 1024, 512, act='relu', bits=True),
]


def test_cases_get_their_set():
  from multinerf_b200 import ops as ops_mod
  for c, want, bn in CASES:
    v, _ = layout(c, 'cpu', fill=False)
    p = plan(ops_mod, c, v)
    assert (p['pingpong'], p['mask_tma'], p['block_n'], p['epilogue']) == (1, 1, bn, want), (case_id(c), p)
  for c in GENERIC_CASES:
    v, _ = layout(c, 'cpu', fill=False)
    p = plan(ops_mod, c, v)
    assert p['pingpong'] == 1 and p['epilogue'] == GENERIC, (case_id(c), p)


@pytest.fixture(scope='module')
def ops():
  from multinerf_b200 import lib, ops as _ops
  lib.require_device()
  return _ops


@pytest.mark.gpu
def test_model_launches_get_their_set(ops, monkeypatch):
  """One eager train step of the full-width 360.gin model (NerfMLP 8 x 1024 with a bottleneck) on 256 rays, with every
  DGRAD's plan recorded from the arguments it was launched with."""
  from multinerf_b200 import configs, lib as L, models, train_utils, utils
  seen = []
  gemm = ops.gemm

  def recording_gemm(mode, a, b, out, **kw):
    if mode == L.GEMM_DGRAD and kw.get('impl', 0) == 0:
      pk = {k: x for k, x in kw.items() if k != 'impl'}
      seen.append((kw.get('n'), kw.get('k'), kw.get('maskbits') is not None, kw.get('colv') is not None,
                   kw.get('addend') is not None or kw.get('mask') is not None, ops.gemm_plan(mode, a, b, out, **pk)))
    return gemm(mode, a, b, out, **kw)

  monkeypatch.setattr(ops, 'gemm', recording_gemm)
  b = configs.bundle_360()
  B = 256
  rng = np.random.default_rng(0)
  f = np.float32
  d = rng.normal(size=(B, 3))
  d /= np.linalg.norm(d, axis=-1, keepdims=True)
  rays = utils.Rays(origins=rng.uniform(-1, 1, (B, 3)).astype(f), directions=d.astype(f),
                    viewdirs=d.astype(f), radii=np.full((B, 1), 7e-4, f), imageplane=np.zeros((B, 2), f),
                    lossmult=np.ones((B, 1), f), near=np.full((B, 1), 0.2, f), far=np.full((B, 1), 1e6, f),
                    cam_idx=np.zeros((B, 1), np.int32))
  model, variables = models.construct_model(1, rays, b)
  step = train_utils.create_train_step(model, b.config, use_graph=False)
  gen = torch.Generator(device='cuda')
  gen.manual_seed(0)
  batch = utils.Batch(rays=rays, rgb=rng.uniform(0, 1, (B, 3)).astype(f))
  step(gen, train_utils.TrainState(variables), batch, None, 0.5)
  torch.cuda.synchronize()
  counts = {GENERIC: 0, BITS_TMA: 0, BITS_TMA_RANK1: 0}
  for n, k, bits, rank1, other, p in seen:
    want = GENERIC
    if p['pingpong'] and p['mask_tma'] and bits and not other:
      want = BITS_TMA_RANK1 if rank1 else BITS_TMA
    assert p['epilogue'] == want, (n, k, bits, rank1, other, p)
    counts[p['epilogue']] += 1
  # the NerfMLP: 7 trunk layers below the top one (less the skip layer's input split at the concat, which adds the
  # feature part's gradient as an addend) and the bottleneck
  assert counts[BITS_TMA] >= 6 and counts[BITS_TMA_RANK1] >= 1, counts


@pytest.mark.gpu
@pytest.mark.parametrize('c,want,bn', CASES, ids=[f'set{w}-bn{bn}-{case_id(c)}' for c, w, bn in CASES])
def test_set_same_bits_as_gemm_tc_kernel(ops, c, want, bn):
  seed = 11 + c['M'] + c['K']
  v0, bufs, init = run(ops, c, seed)
  verify(c, v0, bufs, init)
  c2 = dict(c, store='reg2')                 # the output two elements off its alignment: gemm_tc_kernel
  v, bufs, init = run(ops, c2, seed)
  assert plan(ops, c2, v)['pingpong'] == 0
  verify(c2, v, bufs, init)
  assert torch.equal(_bits(v['out']), _bits(v0['out'])), f'{case_id(c)}: set {want} differs from gemm_tc_kernel'
