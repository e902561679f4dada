"""FWD epilogue operand sets of the ping-pong GEMM schedule (gemm_tc_pingpong_kernel, csrc/gemm_tc.cu).

The ping-pong FWD has an instance per operand set, which mnrf_gemm_plan reports as `epilogue`: 3 bias + ReLU + mask
bits stored by TMA (trunk and view layers in training), 4 bias + ReLU without mask bits (the same layers in a render),
5 bias alone (the bottleneck), 0 the generic epilogue for any other FWD (no bias, mask words TMA cannot address).
  test_cases_get_their_set          each case below plans the set it claims (no device needed);
  test_model_launches_get_their_set every FWD of a train step and of a render of the full-width 360.gin model gets
                                    the set its operands call for;
  test_set_same_bits_as_gemm_tc_kernel  each fixed set, at tiles of 128 and 256 columns, with a ragged last row tile
                                    and guard rows and columns around every output, writes the same output and mask
                                    words as gemm_tc_kernel (register store) bit for bit, and nothing outside them.
"""
import numpy as np
import pytest
import torch

import gemm_ref as G

GENERIC, BIAS_RELU_BITS, BIAS_RELU, BIAS = 0, 3, 4, 5
RAGGED = 524251          # 4096 row tiles, the last one of 91 rows

# (M, N, K, act, mask bits, operand set, tile width)
CASES = [
    (5000, 1024, 512, 'relu', True, BIAS_RELU_BITS, 256),
    (5000, 640, 192, 'relu', True, BIAS_RELU_BITS, 128),
    (5000, 1024, 1024, 'relu', False, BIAS_RELU, 256),
    (5000, 640, 192, 'relu', False, BIAS_RELU, 128),
    (5000, 256, 1024, 'none', False, BIAS, 256),
    (5000, 384, 192, 'none', False, BIAS, 128),
]


def _buffers(M, N, K, act, bits, device, store='staged', bits_tma=True, bias=True, fill=True):
  """Operands in NaN padding and outputs in sentinel padding, three guard rows above and below each.  store
  'staged': a 16-byte aligned output (the ping-pong kernel); 'reg2': two elements off (gemm_tc_kernel's register
  store).  bits_tma: mask words 16-byte aligned with a row pitch of a multiple of 4 words."""
  nan, sen = ('nan', 'sentinel') if fill else (None, None)
  bf = torch.bfloat16
  v, bufs = {}, {}

  def put(name, shape, dtype, fill_, **kw):
    v[name], bufs[name] = G.embed(shape, dtype, device, fill=fill_, extra_rows=3, **kw)

  put('a', (M, K), bf, nan, extra_cols=16, col0=8)
  put('b', (N, K), bf, nan, extra_cols=16, col0=8)
  put('out', (M, N), bf, sen, extra_cols=16, col0=8 if store == 'staged' else 2)
  if bias:
    put('bias', (N,), torch.float32, nan, extra_cols=4, col0=2)
  if bits:
    if bits_tma:
      put('maskbits', (M, N // 32), torch.int32, sen, extra_cols=8, col0=4)
    else:
      put('maskbits', (M, N // 32), torch.int32, sen, extra_cols=3, col0=1)
  return v, bufs


def _plan(ops, M, N, K, act, v):
  from multinerf_b200 import lib as L
  return ops.gemm_plan(L.GEMM_FWD, v['a'], v['b'], v['out'], m=M, n=N, k=K,
                       act=L.ACT_RELU if act == 'relu' else L.ACT_NONE, bias=v.get('bias'),
                       maskbits=v.get('maskbits'))


def test_cases_get_their_set():
  from multinerf_b200 import ops as ops_mod
  for M, N, K, act, bits, want, bn in CASES:
    v, _ = _buffers(M, N, K, act, bits, 'cpu', fill=False)
    p = _plan(ops_mod, M, N, K, act, v)
    assert (p['pingpong'], p['block_n'], p['epilogue'], p['mask_tma']) == (1, bn, want, int(bits)), (M, N, K, p)
  # the generic set: mask words TMA cannot address, no bias, or mask bits without ReLU
  for kw in (dict(bits=True, bits_tma=False), dict(bits=True, bias=False), dict(bits=False, bias=False)):
    for act in ('relu', 'none'):
      if act == 'none' and kw['bits']:
        continue
      v, _ = _buffers(5000, 1024, 512, act, device='cpu', fill=False, **kw)
      p = _plan(ops_mod, 5000, 1024, 512, act, v)
      assert p['pingpong'] == 1 and p['epilogue'] == GENERIC and p['mask_tma'] == 0, (act, kw, p)
  # on the register store (gemm_tc_kernel) nothing is fixed
  v, _ = _buffers(5000, 1024, 512, 'relu', True, 'cpu', store='reg2', fill=False)
  p = _plan(ops_mod, 5000, 1024, 512, 'relu', v)
  assert (p['pingpong'], p['epilogue'], p['mask_tma']) == (0, GENERIC, 0), p


@pytest.fixture(scope='module')
def ops():
  from multinerf_b200 import lib, ops as _ops
  lib.require_device()
  return _ops


def _record_fwd(ops, monkeypatch):
  """Replace ops.gemm by a wrapper that records (act, bias, mask bits, plan) of every tensor-core FWD launch."""
  from multinerf_b200 import lib as L
  seen = []
  gemm = ops.gemm

  def recording_gemm(mode, a, b, out, **kw):
    if mode == L.GEMM_FWD and kw.get('impl', 0) == 0:
      pk = {k: x for k, x in kw.items() if k != 'impl'}
      seen.append((kw.get('act', L.ACT_NONE), kw.get('bias') is not None, kw.get('maskbits') is not None,
                   ops.gemm_plan(mode, a, b, out, **pk)))
    return gemm(mode, a, b, out, **kw)

  monkeypatch.setattr(ops, 'gemm', recording_gemm)
  return seen


def _check_sets(seen):
  from multinerf_b200 import lib as L
  counts = {s: 0 for s in (GENERIC, BIAS_RELU_BITS, BIAS_RELU, BIAS)}
  for act, bias, bits, p in seen:
    want = GENERIC
    if p['pingpong'] and bias:
      if act == L.ACT_RELU:
        want = BIAS_RELU_BITS if bits and p['mask_tma'] else BIAS_RELU if not bits else GENERIC
      elif act == L.ACT_NONE and not bits:
        want = BIAS
    assert p['epilogue'] == want, (act, bias, bits, p)
    counts[p['epilogue']] += 1
  return counts


def _rays(B, rng):
  from multinerf_b200 import utils
  f = np.float32
  d = rng.normal(size=(B, 3))
  d /= np.linalg.norm(d, axis=-1, keepdims=True)
  return utils.Rays(origins=rng.uniform(-1, 1, (B, 3)).astype(f), directions=d.astype(f),
                    viewdirs=d.astype(f), radii=np.full((B, 1), 7e-4, f), imageplane=np.zeros((B, 2), f),
                    lossmult=np.ones((B, 1), f), near=np.full((B, 1), 0.2, f), far=np.full((B, 1), 1e6, f),
                    cam_idx=np.zeros((B, 1), np.int32))


@pytest.mark.gpu
def test_model_launches_get_their_set(ops, monkeypatch):
  """One eager train step and one render call of the full-width 360.gin model (NerfMLP 8 x 1024 with a bottleneck)
  on 256 rays, with every FWD's plan recorded from the arguments it was launched with."""
  from multinerf_b200 import configs, models, train_utils, utils
  seen = _record_fwd(ops, monkeypatch)
  b = configs.bundle_360()
  B = 256
  rng = np.random.default_rng(0)
  rays = _rays(B, rng)
  model, variables = models.construct_model(1, rays, b)
  step = train_utils.create_train_step(model, b.config, use_graph=False)
  gen = torch.Generator(device='cuda')
  gen.manual_seed(0)
  batch = utils.Batch(rays=rays, rgb=rng.uniform(0, 1, (B, 3)).astype(np.float32))
  step(gen, train_utils.TrainState(variables), batch, None, 0.5)
  torch.cuda.synchronize()
  train = _check_sets(seen)
  # the NerfMLP's 8 trunk layers keep their mask bits for the backward; its bottleneck has a bias and no activation
  assert train[BIAS_RELU_BITS] >= 8 and train[BIAS] >= 1 and train[BIAS_RELU] == 0, train
  seen.clear()
  model(None, rays, 1.0, True)
  torch.cuda.synchronize()
  render = _check_sets(seen)
  # a render keeps no mask bits: the trunk runs the set without them
  assert render[BIAS_RELU] >= 8 and render[BIAS] >= 1 and render[BIAS_RELU_BITS] == 0, render


def _run(ops, M, N, K, act, bits, seed, store):
  from multinerf_b200 import lib as L
  v, bufs = _buffers(M, N, K, act, bits, 'cuda', store=store, bits_tma=store == 'staged')
  g = torch.Generator(device='cuda').manual_seed(seed)
  v['a'].copy_(torch.randn(M, K, generator=g, device='cuda'))
  v['b'].copy_(torch.randn(N, K, generator=g, device='cuda') / K ** 0.5)
  v['bias'].copy_(torch.randn(N, generator=g, device='cuda'))
  # exact zeros and tiny values after the bias: a pre-activation of 0 and a denormal one must give bits 0 and 1
  v['a'][:64].zero_()
  v['bias'][::7] = 0.0
  v['bias'][3::7] = 1e-40
  kw = dict(m=M, n=N, k=K, act=L.ACT_RELU if act == 'relu' else L.ACT_NONE, bias=v['bias'],
            maskbits=v.get('maskbits'))
  p = ops.gemm_plan(L.GEMM_FWD, v['a'], v['b'], v['out'], **kw)
  ops.gemm(L.GEMM_FWD, v['a'], v['b'], v['out'], **kw)
  torch.cuda.synchronize()
  return v, bufs, p


@pytest.mark.gpu
@pytest.mark.parametrize('M', [RAGGED, 38000])
@pytest.mark.parametrize('N,K,act,bits,want,bn', [c[1:] for c in CASES],
                         ids=[f'set{c[5]}-bn{c[6]}-{c[1]}x{c[2]}-{c[3]}{"-bits" if c[4] else ""}' for c in CASES])
def test_set_same_bits_as_gemm_tc_kernel(ops, M, N, K, act, bits, want, bn):
  seed = 5 + N + K
  v, bufs, p = _run(ops, M, N, K, act, bits, seed, 'staged')
  assert (p['pingpong'], p['block_n'], p['epilogue']) == (1, bn, want), p
  for name in ('out', 'maskbits'):
    if name in v:
      assert G.padding_intact(v[name], bufs[name]), f'{name}: a write outside the output'
  v0, bufs0, p0 = _run(ops, M, N, K, act, bits, seed, 'reg2')
  assert p0['pingpong'] == 0 and p0['staged'] == 0, p0
  assert torch.equal(v['out'].view(torch.int16), v0['out'].view(torch.int16)), f'set {want}: output differs'
  if bits:
    assert torch.equal(v['maskbits'], v0['maskbits']), f'set {want}: mask words differ'
    # the zero rows: every bit is that of the bias alone, 0 for a bias of 0 and 1 for a denormal one
    b = v['bias'].cpu()
    want_bits = (b > 0).reshape(N // 32, 32).to(torch.int64) << torch.arange(32)
    words = want_bits.sum(1).to(torch.int64)
    words = torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)
    assert torch.equal(v['maskbits'][:64].cpu(), words.expand(64, -1)), 'mask words of the zero rows'
