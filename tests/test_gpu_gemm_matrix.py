"""Instance matrix of the tensor-core Dense-layer GEMM (csrc/gemm_tc.cu, gemm_tc_act.cu) against fp64.

Every kernel instance the dispatcher can reach -- mode x tile width BN x store path (staged TMA bulk store or
register stores) x smooth activation x WGRAD side sums, and for DGRAD where the mask comes from (bf16 mask, mask
bits by TMA, mask bits by the epilogue's loads) -- is launched by at least one case of CASES with a ragged last row
tile and by at least one with several tiles per persistent CTA; test_every_instance_has_cases asks the library
(mnrf_gemm_plan) which instance each case runs.  Each case checks:
  - every output, z, mask bit and column sum against the fp64 bound of tests/gemm_ref.py;
  - every padding byte around every output buffer unchanged, bitwise;
  - no NaN: every input sits in NaN-filled padding, so a read outside an operand shows.
test_same_bits runs instances that must agree bit for bit on the same data.  test_rejected_arguments checks that each
argument check of the launch raises and writes nothing.  Needs an H100 (test_every_instance_has_cases does not).
fp64_launches makes the launches of test_gemm_case and test_same_bits through the same `launch`, on CPU buffers, for
the launch-coverage audit (test_launch_coverage_cpu.py), which asks that every launch class the models reach has one.
"""
import math

import pytest
import torch

import gemm_ref as G

ACTS = {'none': G.NONE, 'relu': G.RELU, 'softplus': G.SOFTPLUS, 'silu': G.SILU}


@pytest.fixture(scope='module')
def ops():
  from multinerf_b200 import lib, ops as _ops
  lib.require_device()
  return _ops


def case(mode, M, N, K, **kw):
  """One launch.  mode 'fwd' | 'dgrad' | 'wgrad' (WGRAD: M = Mo, K = R).  Options:
    act      'none' | 'relu' | 'softplus' | 'silu'     bias   FWD bias (default on)
    bits     FWD ReLU writes mask bits: True (pitch % 4 != 0: stored from registers) | 'tma' (16-byte aligned
             words, pitch % 4 == 0: stored by TMA from shared memory)
    z        FWD smooth writes z (row pitch > N)
    store    'staged' (16-byte aligned output, pitch % 8 == 0) | 'reg2' (output 2 elements off) | 'reg4' (pitch
             = 4 mod 8): the register store whatever BN
    mask     DGRAD 'none' | 'bf16' | 'bits' (16-byte aligned words, pitch % 4 == 0) | 'bits_odd' (pitch % 4 != 0)
    rep      DGRAD: mask / z rows = M / rep, mask_mod = M / rep (0: no mask_mod)
    rowv, addend, colsum   DGRAD epilogue inputs / output
    side     WGRAD 'none' | 'bsum' | 'both' (bsum and side_aw)
    impl     0 tensor cores, 1 SIMT reference"""
  c = dict(mode=mode, M=M, N=N, K=K, act='none', bias=True, bits=False, z=False, store='staged', mask='none',
           rep=0, rowv=False, addend=False, colsum=False, side='none', impl=0)
  assert set(kw) <= set(c), set(kw) - set(c)
  c.update(kw)
  return c


def case_id(c):
  opts = [k if v is True else f'{k}={v}' for k, v in c.items()
          if k not in ('mode', 'M', 'N', 'K') and v != case('fwd', 1, 1, 1)[k]]
  return '-'.join([c['mode'], f"{c['M']}x{c['N']}x{c['K']}"] + opts)


BIG = 38000              # 297 row tiles, the last one of 112 rows: ragged, and several tiles per CTA at any BN
WAVE = 132 * 128         # one row tile per SM of the H100
WIDTHS = {256: (256, 768, 1024), 128: (128, 384, 640), 64: (64, 192, 320), 32: (32, 96, 160), 16: (16, 48)}
CASES = []
# ---- FWD: every tile width x store path; ReLU with and without mask bits, plain, softplus / SiLU with and without z
for bn, ns in WIDTHS.items():
  stores = ('staged', 'reg2', 'reg4') if bn >= 64 else ('reg2',)
  for i, store in enumerate(stores):
    n = ns[i % len(ns)]
    CASES.append(case('fwd', BIG, n, 192, act='relu', bits=n % 32 == 0 and bn >= 32, store=store))
    CASES.append(case('fwd', (1, 127, 129, 1000)[i], ns[-1], 64, store=store, bias=False))
  CASES.append(case('fwd', WAVE + 1, ns[-1], 1024, act='relu', store=stores[-1]))
for bn in (256, 128, 64):
  n0, n1 = WIDTHS[bn][0], WIDTHS[bn][-1]
  CASES.append(case('fwd', BIG, n1, 192, act='softplus', z=True))
  CASES.append(case('fwd', WAVE - 1, n0, 1536, act='silu', z=True))
  CASES.append(case('fwd', 1000, n1, 64, act='silu'))
  CASES.append(case('fwd', 129, n0, 192, act='softplus'))
# the shapes of test_gemm_fwd (test_gpu_kernels.py) under the fp64 bound: ReLU, bias and mask bits; the SIMT
# reference up to 4096 rows
for m, n, k in [(128, 256, 64), (256, 256, 512), (1000, 128, 320), (384, 1024, 1536), (130, 64, 128),
                (4096, 256, 256), (38000, 256, 64), (10000, 768, 128), (38144, 256, 64), (10240, 1024, 256),
                (512, 512, 128), (512, 1024, 1024), (512, 1024, 1536), (16384, 1024, 512)]:
  for impl in ((0, 1) if m <= 4096 else (0,)):
    CASES.append(case('fwd', m, n, k, act='relu', bits=True, impl=impl))
# ---- DGRAD: every tile width x store path x mask source, and the epilogue inputs
for bn, ns in WIDTHS.items():
  stores = ('staged', 'reg2', 'reg4') if bn >= 64 else ('reg2', 'reg4')
  masks = ('none', 'bf16') + (('bits', 'bits_odd') if bn >= 32 else ())
  for i, store in enumerate(stores):
    for j, mask in enumerate(masks):
      n = ns[(i + j) % len(ns)]
      CASES.append(case('dgrad', BIG if (i + j) % 2 == 0 else WAVE + 1, n, (192, 1024, 64)[(i + j) % 3], mask=mask,
                        store=store, rowv=j % 2 == 1, addend=j >= 2, colsum=n <= 1024))
      CASES.append(case('dgrad', (1, 127, 129, 1000)[j], ns[0], 64, mask=mask, store=store, addend=j == 1,
                        colsum=True))
for bn in (256, 128, 64):
  n0, n1 = WIDTHS[bn][0], WIDTHS[bn][-1]
  CASES.append(case('dgrad', BIG, n1, 192, act='softplus', rowv=True, colsum=True))
  CASES.append(case('dgrad', 3 * 384, n0, 1536, act='silu', rep=3, addend=True, colsum=True))
  CASES.append(case('dgrad', 3 * 200, n1, 64, act='softplus', rep=3, colsum=True))
# mask_mod: a multiple of the 128-row tile (mask bits by TMA at BN >= 128) and not (the epilogue's loads)
for m in (384, 200):
  for n in (256, 320):
    CASES.append(case('dgrad', 3 * m, n, 128, mask='bits', rep=3, colsum=True, store='staged' if n == 256 else 'reg2'))
# the shapes of test_gemm_dgrad (test_gpu_kernels.py) under the fp64 bound (bf16 mask, rowv / colv; mask bits and
# column sums in test_same_bits), and of the column-sum cases where a persistent CTA changes column block
# (N = 640 / 320, test_gpu_gemm_dgrad_epilogue.py)
for m, n, k in [(256, 256, 256), (1000, 1024, 1024), (384, 256, 128), (38000, 256, 256), (10000, 1024, 256),
                (10000, 768, 128), (37888, 256, 256), (10240, 1024, 256), (10240, 768, 128), (512, 1024, 1024),
                (512, 1024, 1536), (16384, 1024, 1024)]:
  for impl in ((0, 1) if m <= 4096 else (0,)):
    CASES.append(case('dgrad', m, n, k, mask='bf16', rowv=True, impl=impl))
for n, mask in [(640, 'bits'), (640, 'bits_odd'), (320, 'bits'), (768, 'bits')]:
  CASES.append(case('dgrad', 20000 if n != 768 else 10000, n, 256 if n != 768 else 128, mask=mask, rowv=n != 768,
                    colsum=True))
# ---- WGRAD: every tile width x side sums; Mo not a multiple of 128, strided fp32 output, ragged last split
for bn, ns in list(WIDTHS.items())[:3]:
  for side in ('none', 'bsum', 'both'):
    CASES.append(case('wgrad', 320, ns[0], 4159, side=side))           # 65 k-blocks, the last of one row
    CASES.append(case('wgrad', 3464, ns[-1], 2049, side=side))         # several tiles per CTA
for r in (1, 15, 37, 64, 65):
  CASES.append(case('wgrad', 200, 128, r, side='both'))
for impl in (0, 1):
  CASES.append(case('wgrad', 320, 256, 1000, side='both', impl=impl))
# ---- the operand sets the models launch (test_launch_coverage_cpu.py): the ping-pong epilogues compiled per operand
# set (FWD bias alone; bias + ReLU + mask bits stored by TMA; DGRAD mask bits by TMA, with and without rowv / colv)
# and the generic epilogue without column sums, each at every tile width the models use
for n in (256, 128, 64):
  CASES.append(case('fwd', BIG, n, 192))
  CASES.append(case('fwd', WAVE + 1, 3 * n, 64, act='relu', bits='tma'))
  CASES.append(case('dgrad', BIG, n, 192))
  CASES.append(case('dgrad', WAVE + 1, n, 192, mask='bits'))
  CASES.append(case('dgrad', BIG, 3 * n, 64, mask='bits', rowv=True))
  CASES.append(case('dgrad', BIG, n, 128, addend=True))
  CASES.append(case('dgrad', 3 * 384, n, 128, mask='bits', rep=3))
CASES.append(case('dgrad', 3 * 200, 128, 128, mask='bits', rep=3))     # mask_mod % 128 != 0: bits by the epilogue
for act in ('softplus', 'silu'):
  CASES.append(case('dgrad', BIG, 256, 192, act=act))
  CASES.append(case('dgrad', WAVE + 1, 256, 128, act=act, addend=True))
  CASES.append(case('dgrad', 3 * 384, 256, 128, act=act, rep=3))
CASES.append(case('dgrad', BIG, 128, 192, act='silu', colsum=True))


# ---------------------------------------------------------------------------------------------- buffers and data
def _words(n):
  return n // 32


def layout(c, device, fill=True):
  """The case's buffers: inputs in NaN padding, outputs in sentinel padding (fill=False: uninitialised, for the
  plan alone).  Returns (views, buffers)."""
  M, N, K = c['M'], c['N'], c['K']
  nan, sen = ('nan', 'sentinel') if fill else (None, None)
  mrows = M // c['rep'] if c['rep'] else M
  v, bufs = {}, {}

  def put(name, shape, dtype, fill_, **kw):
    v[name], bufs[name] = G.embed(shape, dtype, device, fill=fill_, **kw)

  bf = torch.bfloat16
  if c['mode'] == 'wgrad':
    put('a', (K, M), bf, nan, extra_cols=16 + (-M % 8), col0=8)
    put('b', (K, N), bf, nan, extra_cols=16, col0=8)
    put('out', (M, N), torch.float32, sen, extra_cols=6, col0=2)
    if c['side'] != 'none':
      put('bsum', (N,), torch.float32, sen, extra_cols=4, col0=2)
    if c['side'] == 'both':
      put('side_w', (K,), torch.float32, nan, extra_cols=2, col0=1)
      put('side_aw', (M,), torch.float32, sen, extra_cols=4, col0=2)
    return v, bufs
  put('a', (M, K), bf, nan, extra_cols=16, col0=8)
  put('b', (N, K), bf, nan, extra_cols=16, col0=8)
  extra, col0 = {'staged': (16, 8), 'reg2': (16, 2), 'reg4': (12, 4)}[c['store']]
  put('out', (M, N), bf, sen, extra_cols=extra, col0=col0)
  smooth = c['act'] in ('softplus', 'silu')
  if c['mode'] == 'fwd':
    if c['bias']:
      put('bias', (N,), torch.float32, nan, extra_cols=4, col0=2)
    if c['bits'] == 'tma':
      put('maskbits', (M, _words(N)), torch.int32, sen, extra_cols=(-_words(N) % 4) + 8, col0=4)
    elif c['bits']:
      put('maskbits', (M, _words(N)), torch.int32, sen, extra_cols=3, col0=1)
    if c['z']:
      put('z', (M, N), bf, sen, extra_cols=10, col0=2)
    return v, bufs
  if c['rowv']:
    put('rowv', (M,), torch.float32, nan, extra_cols=2, col0=1)
    put('colv', (N,), torch.float32, nan, extra_cols=4, col0=2)
  if c['mask'] == 'bf16':
    put('mask', (mrows, N), bf, nan, extra_cols=6, col0=2)
  elif c['mask'] == 'bits':
    put('maskbits', (mrows, _words(N)), torch.int32, nan, extra_cols=(-_words(N) % 4) + 8, col0=4)
  elif c['mask'] == 'bits_odd':
    w = _words(N)
    put('maskbits', (mrows, w), torch.int32, nan, extra_cols=2 if (w + 2) % 4 else 3, col0=1)
  if smooth:
    put('z', (mrows, N), bf, nan, extra_cols=6, col0=2)
  if c['addend']:
    put('addend', (M, N), bf, nan, extra_cols=6, col0=2)
  if c['colsum']:
    put('colsum', (N,), torch.float32, sen, extra_cols=4, col0=2)
  return v, bufs


def _call_kwargs(c, v):
  kw = dict(m=c['M'], n=c['N'], k=c['K'])
  if c['mode'] == 'wgrad':
    return kw
  kw['act'] = ACTS[c['act']]
  for name in ('bias', 'rowv', 'colv', 'mask', 'maskbits', 'colsum', 'addend', 'z'):
    if name in v:
      kw[name] = v[name]
  if c['rep']:
    kw['mask_mod'] = c['M'] // c['rep']
  return kw


def plan(ops_mod, c, v):
  from multinerf_b200 import lib as L
  kw = _call_kwargs(c, v)
  if c['mode'] == 'wgrad':
    return ops_mod.gemm_plan(L.GEMM_WGRAD, v['a'], v['b'], v['out'], bsum=v.get('bsum'), side_w=v.get('side_w'),
                             side_aw=v.get('side_aw'), **kw)
  mode = L.GEMM_FWD if c['mode'] == 'fwd' else L.GEMM_DGRAD
  return ops_mod.gemm_plan(mode, v['a'], v['b'], v['out'], **kw)


def instance(c, p):
  """The kernel instance a case runs: (mode, BN, staged store, smooth, side sums, DGRAD mask source)."""
  src = ''
  if c['mode'] == 'dgrad' and c['act'] not in ('softplus', 'silu'):
    src = {'none': 'none', 'bf16': 'bf16'}.get(c['mask']) or ('bits_tma' if p['mask_tma'] else 'bits_ldg')
  return (c['mode'], p['block_n'], bool(p['staged']), bool(p['smooth']), bool(p['side']), src)


def _fill(c, v, seed):
  """The case's data, drawn in a fixed order from `seed` so that cases differing only in layout or mask source
  get the same values."""
  M, N, K = c['M'], c['N'], c['K']
  g = torch.Generator(device='cuda').manual_seed(seed)
  dev = 'cuda'

  def normal(*shape, scale=1.0):
    return torch.randn(*shape, generator=g, device=dev) * scale

  mrows = M // c['rep'] if c['rep'] else M
  if c['mode'] == 'wgrad':
    v['a'].copy_(normal(K, M))
    v['b'].copy_(normal(K, N))
    v['out'].copy_(normal(M, N))
    init = {'out': v['out'].clone()}
    if 'bsum' in v:
      v['bsum'].copy_(normal(N))
      init['bsum'] = v['bsum'].clone()
    if 'side_w' in v:
      v['side_w'].copy_(normal(K))
      v['side_aw'].copy_(normal(M))
      init['side_aw'] = v['side_aw'].clone()
    return init
  v['a'].copy_(normal(M, K))
  v['b'].copy_(normal(N, K, scale=1 / math.sqrt(K)))
  bias, rowv, colv = normal(N), normal(M), normal(N)
  maskb = torch.rand(mrows, N, generator=g, device=dev) > 0.4
  mag = normal(mrows, N).abs() + 1e-2
  zin, add, cs = normal(mrows, N, scale=2.0), normal(M, N), normal(N)
  init = {}
  for name, val in (('bias', bias), ('rowv', rowv), ('colv', colv), ('z', zin), ('addend', add)):
    if name in v and not (name == 'z' and c['mode'] == 'fwd'):
      v[name].copy_(val)
  if c['mask'] == 'bf16':
    v['mask'].copy_(torch.where(maskb, mag, -mag))
  elif c['mask'] in ('bits', 'bits_odd'):
    v['maskbits'].copy_(G.pack_bits(maskb))
  if 'colsum' in v:
    v['colsum'].copy_(cs)
    init['colsum'] = cs
  return init


def launch(ops_mod, c, v):
  """The case's one launch on the views of layout(c, ...)."""
  from multinerf_b200 import lib as L
  kw = _call_kwargs(c, v)
  if c['mode'] == 'wgrad':
    if c['side'] == 'none':
      ops_mod.gemm(L.GEMM_WGRAD, v['a'], v['b'], v['out'], impl=c['impl'], **kw)
    else:
      ops_mod.gemm_wgrad(v['a'], v['b'], v['out'], bsum=v.get('bsum'), side_w=v.get('side_w'),
                         side_aw=v.get('side_aw'), impl=c['impl'], **kw)
  else:
    mode = L.GEMM_FWD if c['mode'] == 'fwd' else L.GEMM_DGRAD
    ops_mod.gemm(mode, v['a'], v['b'], v['out'], impl=c['impl'], **kw)


def run(ops_mod, c, seed=0):
  """Launch the case on its data; returns (views, buffers, initial values)."""
  v, bufs = layout(c, 'cuda')
  init = _fill(c, v, seed)
  launch(ops_mod, c, v)
  torch.cuda.synchronize()
  return v, bufs, init


def verify(c, v, bufs, init):
  """fp64 bound of every output, padding intact, no NaN.  Returns the worst err / bound ratio per output."""
  outputs = {'out', 'colsum', 'bsum', 'side_aw'} | ({'maskbits', 'z'} if c['mode'] == 'fwd' else set())
  for name in outputs & set(v):
    assert G.padding_intact(v[name], bufs[name]), f'{name}: a write outside the output'
  worst = {}
  if c['mode'] == 'wgrad':
    ref = G.ref_wgrad(v['a'], v['b'], init=init['out'], bsum_init=init.get('bsum'), side_w=v.get('side_w'),
                      side_aw_init=init.get('side_aw'))
    for name, (val, bound) in ref.items():
      worst[name] = G.check(v[name], val, bound, name)
    return worst
  code = ACTS[c['act']]
  if c['mode'] == 'fwd':
    r = G.ref_fwd(v['a'], v['b'], bias=v.get('bias'), act_code=code)
    worst['out'] = G.check(v['out'], r['out'], r['out_bound'], 'out')
    if 'z' in v:
      worst['z'] = G.check(v['z'], r['z'], r['z_bound'], 'z')
    if 'maskbits' in v:
      G.check_bits(v['maskbits'], v['out'], r['z'], r['pre_bound'], 'mask bits')
    return worst
  r = G.ref_dgrad(v['a'], v['b'], rowv=v.get('rowv'), colv=v.get('colv'), mask=v.get('mask'),
                  maskbits=v.get('maskbits'), mask_mod=c['M'] // c['rep'] if c['rep'] else 0,
                  addend=v.get('addend'), z=v.get('z'), act_code=code)
  worst['out'] = G.check(v['out'], r['out'], r['out_bound'], 'out')
  if 'colsum' in v:
    s, sb = G.colsum_ref(r['out'], r['pre_bound'], init['colsum'], rounded=c['impl'] == 1)
    worst['colsum'] = G.check(v['colsum'], s, sb, 'colsum')
  return worst


@pytest.mark.gpu
@pytest.mark.parametrize('c', CASES, ids=case_id)
def test_gemm_case(ops, c):
  v, bufs, init = run(ops, c, seed=c['M'] + 7 * c['N'] + c['K'])
  inst = instance(c, plan(ops, c, v)) if c['impl'] == 0 else ('simt', c['mode'])
  worst = verify(c, v, bufs, init)
  print(f'\n[gemm err/bound] {inst} {case_id(c)}: ' + ' '.join(f'{k}={x:.3g}' for k, x in worst.items()))


def _bits(t):
  return t.view({torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.int32: torch.int32}[t.dtype])


# Instances that must give the same bits on the same data: (base case, variants, outputs compared bitwise).  Column
# sums use atomics across CTAs: they are checked against the bound, not compared.
SAME_BITS = []
for n in (256, 128, 64):
  SAME_BITS.append((case('fwd', WAVE + 1, n, 192, act='relu', bits=True),
                    [dict(store='reg2'), dict(store='reg4'), dict(bits=False)], ('out', 'maskbits')))
  SAME_BITS.append((case('fwd', 1000, 3 * n, 1024, act='silu', z=True), [dict(z=False)], ('out',)))
  SAME_BITS.append((case('dgrad', BIG, n, 192, mask='bits', rowv=True, addend=True, colsum=True),
                    [dict(store='reg2'), dict(mask='bits_odd'), dict(mask='bf16')], ('out',)))
  SAME_BITS.append((case('dgrad', 3 * 384, n, 128, mask='bits', rep=3, colsum=True),
                    [dict(mask='bits_odd')], ('out',)))
for m, n, k in [(256, 256, 256), (1000, 1024, 1024), (384, 256, 128), (38000, 256, 256), (10000, 1024, 256),
                (10000, 768, 128), (37888, 256, 256), (10240, 1024, 256), (10240, 768, 128), (512, 1024, 1024),
                (512, 1024, 1536), (16384, 1024, 1024)]:
  SAME_BITS.append((case('dgrad', m, n, k, mask='bf16', rowv=True),
                    [dict(mask='bits', colsum=n <= 1024), dict(mask='bits_odd')], ('out',)))


@pytest.mark.gpu
@pytest.mark.parametrize('base,variants,names', SAME_BITS, ids=[case_id(s[0]) for s in SAME_BITS])
def test_same_bits(ops, base, variants, names):
  seed = 1 + base['M'] + base['N']
  v0, bufs, init = run(ops, base, seed)
  verify(base, v0, bufs, init)
  for var in variants:
    c = dict(base, **var)
    v, bufs, init = run(ops, c, seed)
    verify(c, v, bufs, init)
    for name in names:
      if name in v and name in v0:
        assert torch.equal(_bits(v[name]), _bits(v0[name])), f'{name} of {var} differs from {case_id(base)}'


@pytest.mark.gpu
@pytest.mark.parametrize('rep', [3])
@pytest.mark.parametrize('m,n', [(384, 256), (200, 256), (200, 128), (384, 320)])
def test_mask_mod_matches_repeated_masks(ops, m, n, rep):
  """mask_mod = M against the same masks written out three times."""
  c = case('dgrad', rep * m, n, 128, mask='bits', rep=rep, rowv=True)
  v, bufs, init = run(ops, c, seed=m)
  verify(c, v, bufs, init)
  c2 = case('dgrad', rep * m, n, 128, mask='bits', rowv=True)
  v2, bufs2 = layout(c2, 'cuda')
  for name in ('a', 'b', 'rowv', 'colv'):
    v2[name].copy_(v[name])
  v2['maskbits'].copy_(v['maskbits'].repeat(rep, 1))
  from multinerf_b200 import lib as L
  ops.gemm(L.GEMM_DGRAD, v2['a'], v2['b'], v2['out'], **_call_kwargs(c2, v2))
  torch.cuda.synchronize()
  assert torch.equal(_bits(v2['out']), _bits(v['out']))


def fp64_launches(ops_mod):
  """Every launch test_gemm_case and test_same_bits check against fp64, made through `launch` on uninitialised CPU
  buffers of the same layout: under a recording library (tests/abi_record.py) these are the calls the GPU tests
  make, which the launch-coverage audit classifies (test_launch_coverage_cpu.py)."""
  cases = list(CASES) + [dict(base, **var) for base, variants, _ in SAME_BITS for var in [{}] + variants]
  for c in cases:
    v, _ = layout(c, 'cpu', fill=False)
    launch(ops_mod, c, v)


# ---------------------------------------------------------------------------------------------- coverage
def _reachable():
  """Every instance the dispatcher reaches over a grid of descriptors and pointer alignments (mnrf_gemm_plan)."""
  from multinerf_b200 import lib as L, ops as ops_mod
  found = set()
  for mode in ('fwd', 'dgrad', 'wgrad'):
    for n in (16, 32, 64, 128, 256):
      for store in ('staged', 'reg2', 'reg4'):
        for act in ('none', 'relu', 'softplus'):
          for extra in ([dict(mask=m) for m in ('none', 'bf16', 'bits', 'bits_odd')] if mode == 'dgrad' else
                        [dict(side=s) for s in ('none', 'bsum', 'both')] if mode == 'wgrad' else
                        [dict(bits=False), dict(bits=True)]):
            if mode == 'wgrad' and (store != 'staged' or act != 'none'):
              continue
            if mode == 'fwd' and extra['bits'] and (act != 'relu' or n % 32):
              continue
            if mode == 'dgrad' and (extra['mask'] in ('bits', 'bits_odd') and n % 32 or act == 'relu'):
              continue
            c = case(mode, 300, n, 128, act=act, store=store, **extra)
            v, _ = layout(c, 'cpu', fill=False)
            try:
              found.add(instance(c, plan(ops_mod, c, v)))
            except L.MnrfError:
              pass
  return found


def test_every_instance_has_cases():
  """Each reachable instance is the plan of a case with a ragged last row tile and of a case with several tiles per
  persistent CTA (on an H100's 132 SMs; without a device the library plans for 132)."""
  from multinerf_b200 import ops as ops_mod
  reach = _reachable()
  ragged, several = set(), set()
  for c in CASES:
    if c['impl']:
      continue
    v, _ = layout(c, 'cpu', fill=False)
    p = plan(ops_mod, c, v)
    inst = instance(c, p)
    assert inst in reach, f'{case_id(c)} runs {inst}, which the enumeration does not reach'
    if c['M'] % 128:
      ragged.add(inst)
    if p['tiles'] > p['grid']:
      several.add(inst)
  assert not reach - ragged, f'instances without a ragged case: {sorted(reach - ragged)}'
  assert not reach - several, f'instances without a case of several tiles per CTA: {sorted(reach - several)}'


# ---------------------------------------------------------------------------------------------- argument checks
def _bad_calls():
  """(name, builder) pairs; each builder returns (call, buffers that must stay unchanged)."""
  from multinerf_b200 import lib as L
  dev = 'cuda'
  bf = torch.bfloat16

  def t(*shape, dtype=bf):
    return torch.zeros(*shape, dtype=dtype, device=dev)

  def out_buf(m, n, extra=16, col0=8, dtype=bf):
    return G.embed((m, n), dtype, dev, extra_cols=extra, col0=col0, fill='sentinel')

  cases = {}

  def fwd(n=256, k=128, a=None, b=None, out=None, **kw):
    def build():
      o, ob = out or out_buf(256, n)
      aa = a if a is not None else t(256, k)
      bb = b if b is not None else t(n, k)
      return (lambda ops: ops.gemm(L.GEMM_FWD, aa, bb, o, m=256, n=n, k=k, **kw)), [ob]
    return build

  def dgrad(n=256, k=128, **kw):
    def build():
      o, ob = out_buf(256, n)
      extra = {}
      for name, val in list(kw.items()):
        if callable(val):
          extra[name], buf = val()
          if buf is not None:
            extra.setdefault('_bufs', []).append(buf)
        else:
          extra[name] = val
      bufs = extra.pop('_bufs', [])
      return (lambda ops: ops.gemm(L.GEMM_DGRAD, t(256, k), t(n, k), o, m=256, n=n, k=k, **extra)), [ob] + bufs
    return build

  def misaligned(shape, dtype=bf, by=1):
    buf = t(shape[0], shape[1] + by) if len(shape) == 2 else torch.zeros(shape[0] + by, dtype=dtype, device=dev)
    return buf[:, by:] if len(shape) == 2 else buf[by:]

  def colsum_buf(n):
    return lambda: G.embed((n,), torch.float32, dev, extra_cols=4, col0=2, fill='sentinel')

  cases['K % 64'] = fwd(k=96)
  cases['N % 16'] = fwd(n=40)
  cases['A misaligned'] = fwd(a=misaligned((256, 128)))
  cases['A pitch % 8'] = fwd(a=t(256, 132)[:, :128])
  cases['B misaligned'] = fwd(b=misaligned((256, 128)))
  cases['bias misaligned'] = fwd(bias=misaligned((256,), torch.float32))
  cases['out misaligned'] = fwd(out=out_buf(256, 256, col0=1))
  cases['mask bits with N % 32'] = fwd(n=48, act=L.ACT_RELU, maskbits=t(256, 2, dtype=torch.int32))
  cases['mask bits pitch < N / 32'] = fwd(act=L.ACT_RELU, maskbits=t(2048, dtype=torch.int32).as_strided((256, 8),
                                                                                                        (4, 1)))
  cases['smooth act, register store'] = fwd(act=L.ACT_SILU, out=out_buf(256, 256, col0=2))
  cases['smooth act, N % 64'] = fwd(n=32, act=L.ACT_SOFTPLUS)
  cases['smooth act, z misaligned'] = fwd(act=L.ACT_SILU, z=misaligned((256, 256)))
  cases['colsum N > 1024'] = dgrad(n=1088, colsum=colsum_buf(1088))
  cases['addend misaligned'] = dgrad(addend=lambda: (misaligned((256, 256)), None))
  cases['colv misaligned'] = dgrad(rowv=lambda: (torch.zeros(256, device=dev), None),
                                   colv=lambda: (misaligned((256,), torch.float32), None))
  cases['bf16 mask misaligned'] = dgrad(mask=lambda: (misaligned((256, 256)), None))
  cases['smooth DGRAD without z'] = dgrad(act=L.ACT_SILU, colsum=colsum_buf(256))
  # mask_mod is for mask bits and z; the bf16 mask was read at the output row, past the end of a mask of M / 3 rows
  cases['bf16 mask with mask_mod'] = dgrad(mask=lambda: (t(128, 256), None), mask_mod=128, colsum=colsum_buf(256))
  return cases


BAD = ['K % 64', 'N % 16', 'A misaligned', 'A pitch % 8', 'B misaligned', 'bias misaligned', 'out misaligned',
       'mask bits with N % 32', 'mask bits pitch < N / 32', 'smooth act, register store', 'smooth act, N % 64',
       'smooth act, z misaligned', 'colsum N > 1024', 'addend misaligned', 'colv misaligned', 'bf16 mask misaligned',
       'smooth DGRAD without z', 'bf16 mask with mask_mod']


@pytest.mark.gpu
@pytest.mark.parametrize('name', BAD)
def test_rejected_arguments(ops, name):
  from multinerf_b200 import lib as L
  call, bufs = _bad_calls()[name]()
  before = [b.clone() for b in bufs]
  with pytest.raises(L.MnrfError):
    call(ops)
  torch.cuda.synchronize()
  for b0, b in zip(before, bufs):
    assert torch.equal(_bits(b0), _bits(b)), f'{name}: the refused call wrote its output'


@pytest.mark.gpu
@pytest.mark.parametrize('n', [32, 320])
def test_rejected_wgrad(ops, n):
  """WGRAD needs N % 64 == 0 and an 8-byte aligned fp32 output."""
  from multinerf_b200 import lib as L
  x, dy = torch.zeros(128, 256, dtype=torch.bfloat16, device='cuda'), torch.zeros(128, n, dtype=torch.bfloat16,
                                                                                   device='cuda')
  col0 = 2 if n == 32 else 1
  out, buf = G.embed((256, n), torch.float32, 'cuda', extra_cols=4, col0=col0, fill='sentinel')
  before = buf.clone()
  with pytest.raises(L.MnrfError):
    ops.gemm(L.GEMM_WGRAD, x, dy, out, m=256, n=n, k=128)
  torch.cuda.synchronize()
  assert torch.equal(_bits(before), _bits(buf))


# ---------------------------------------------------------------------------------------------- non-finite input
@pytest.mark.gpu
@pytest.mark.parametrize('impl', [0, 1])
@pytest.mark.parametrize('n', [256, 128, 64])
def test_non_finite_rows(ops, n, impl):
  """NaN and +-inf in designated rows of A.  FWD ReLU: a NaN pre-activation stays NaN (torch.relu, jnp.maximum) with
  mask bit 0, +-inf follows fp64.  DGRAD with mask bits: a masked-out element is 0 whatever the sum (a select).
  Every other row equals the clean launch bit for bit."""
  from multinerf_b200 import lib as L
  rows = {5: float('nan'), 130: float('inf'), 131: -float('inf'), 999: float('nan')}
  for mode, c in (('fwd', case('fwd', 1000, n, 192, act='relu', bits=True, impl=impl)),
                  ('dgrad', case('dgrad', 1000, n, 192, mask='bits', impl=impl))):
    v0, _, _ = run(ops, c, seed=n)
    v, bufs = layout(c, 'cuda')
    _fill(c, v, seed=n)
    for r, x in rows.items():
      v['a'][r, 7 + r % 100] = x
    ops.gemm(L.GEMM_FWD if mode == 'fwd' else L.GEMM_DGRAD, v['a'], v['b'], v['out'], impl=impl,
             **_call_kwargs(c, v))
    torch.cuda.synchronize()
    for name in ('out', 'maskbits') if mode == 'fwd' else ('out',):
      assert G.padding_intact(v[name], bufs[name]), name
    idx = sorted(rows)
    others = torch.ones(c['M'], dtype=torch.bool, device='cuda')
    others[idx] = False
    assert torch.equal(_bits(v['out'][others]), _bits(v0['out'][others])), f'{mode}: another row changed'
    a = v['a'][idx]
    if mode == 'fwd':
      r = G.ref_fwd(a, v['b'], bias=v['bias'], act_code=G.RELU)
    else:
      r = G.ref_dgrad(a, v['b'], maskbits=v['maskbits'][idx])
    got = v['out'][idx].double()
    want = r['out'].to(torch.bfloat16).double()
    for what, f in (('NaN', torch.isnan), ('+inf', torch.isposinf), ('-inf', torch.isneginf)):
      assert torch.equal(f(got), f(want)), f'{mode} {what}: {int((f(got) != f(want)).sum())} elements differ'
    if mode == 'fwd':
      assert bool(torch.isnan(got).any()), 'no NaN reached the output'
      bits = G.unpack_bits(v['maskbits'][idx], n)
      assert torch.equal(bits, r['z'] > 0), 'mask bits of the non-finite rows'
    else:
      keep = G.unpack_bits(v['maskbits'][idx], n)
      assert bool((got[~keep] == 0).all()), 'a masked-out element is not 0'
