"""Instance matrix of the narrow heads, column sums, weight packing and clip+Adam (csrc/heads.cu) against fp64.

Every kernel instance the head launchers can reach -- head_fwd_sub_kernel<LPR = 32 / 16 / 8>, head_fwd_kernel,
head_bwd_sub_kernel<N_OUT, LPR, 4, SMOOTH> and head_bwd_kernel<N_OUT, kMaxChunks = 1 / 2 / 4 / 6, SMOOTH> -- is
launched by at least one case with a ragged last block and by at least one whose grid is capped (the forward's
grid-stride loop wraps; the backward's blocks take more than their minimum of rows); test_every_instance_has_cases asks
the library (mnrf_head_plan) which instance each case runs.  Each case checks:
  - every output against the fp64 bound of tests/heads_ref.py;
  - every padding element around every output buffer unchanged, bitwise;
  - no NaN: every input sits in NaN-filled padding, so a read outside an operand shows.
Column sums, weight packing, clip+Adam and the chained trunk's fused head get the same checks.  Needs an H100
(test_every_instance_has_cases does not).  fp64_launches makes the head launches of test_head_case and
test_heads_and_colsum_fp64 through the same `launch`, on CPU buffers, for the launch-coverage audit
(test_launch_coverage_cpu.py), which asks that every head launch class the models reach has one.
"""
import math

import pytest
import torch

import gemm_ref as G
import heads_ref as H

ACTS = {'none': G.NONE, 'relu': G.RELU, 'softplus': G.SOFTPLUS, 'silu': G.SILU}


@pytest.fixture(scope='module')
def ops():
  from multinerf_b200 import lib, ops as _ops
  lib.require_device()
  return _ops


def _bits(t):
  return t.view({torch.bfloat16: torch.int16, torch.float32: torch.int32}[t.dtype])


# ---------------------------------------------------------------------------------------------- head cases
def case(mode, M, K, n_out, **kw):
  """One head launch.  mode 'fwd' | 'bwd'.  Options:
    bias      fwd bias (default on)                   strided   x (and dx, dx2, z) rows with a pitch past K
    act       bwd 'none' | 'relu' | 'softplus' | 'silu'
    out       bwd outputs: 'dx' | 'dx_sum' (dx and dxsum) | 'params' (dx=None) | 'alias' (dx=None, w = x's first row)
    dx_cols   bwd: columns of dx (0: K); the rest go to dx2      split   bwd dw_split (0: none)
    w_off     bwd: w this many elements past a 16-byte boundary
    db        bwd: db given (default on)                 dx2     bwd with dx_cols: dx2 given (default on)"""
  c = dict(mode=mode, M=M, K=K, n_out=n_out, bias=True, strided=False, act='none', out='dx_sum', dx_cols=0, split=0,
           w_off=0, db=True, dx2=True)
  assert set(kw) <= set(c), set(kw) - set(c)
  c.update(kw)
  return c


def case_id(c):
  opts = [k if v is True else f'{k}={v}' for k, v in c.items()
          if k not in ('mode', 'M', 'K', 'n_out') and v != case(c['mode'], 1, 8, 1)[k]]
  return '-'.join([c['mode'], f"{c['M']}x{c['K']}x{c['n_out']}"] + opts)


CASES = []
# ---- forward: the sub kernels (K = 64 / 128 / 256) and the warp-per-row kernel; M = 1, a ragged M, and an M past the
# grid cap (num_sms * 8 blocks: 135168 rows at K = 64, 67584 at 128, 33792 at 256, 8448 on the warp kernel)
FWD_WRAP = {64: 300007, 128: 70001, 256: 34001}
for K in (64, 128, 256, 8, 192, 264, 1024, 1536):
  CASES.append(case('fwd', 1, K, 1 + K % 4, bias=False))
  CASES.append(case('fwd', 1001, K, 3, strided=True))
  CASES.append(case('fwd', 4099, K, 2, bias=K % 3 == 0))
  CASES.append(case('fwd', FWD_WRAP.get(K, 9001), K, 4, strided=K in (256, 1024)))
CASES.append(case('fwd', 3 * 2 ** 20, 256, 1))       # the tangent density head of a 2^20-sample level
CASES.append(case('fwd', 127, 64, 1, bias=False, strided=True))
# ---- backward: every instance (N_OUT x width x SMOOTH) with an M that is ragged against the block's row range and
# past the grid cap (264 blocks of >= 512 rows on the sub kernel, 528 blocks of >= 8 rows on the warp kernel)
BWD_WIDTHS = [(64, 0), (128, 0), (256, 0), (256, 1), (192, 0), (320, 0), (448, 0), (1024, 0), (1536, 0)]
OUTS = {1: dict(out='dx_sum'), 2: dict(out='dx', strided=True), 3: dict(out='dx_sum', split=2, dx_cols=-1),
        4: dict(out='dx_sum', split=1, strided=True)}
for K, w_off in BWD_WIDTHS:
  sub = K in (64, 128, 256) and not w_off
  for n_out in (1, 2, 3, 4):
    for smooth in (False, True):
      act = ('softplus' if n_out % 2 else 'silu') if smooth else ('relu' if n_out % 2 else 'none')
      kw = dict(OUTS[n_out])
      if kw.get('dx_cols') == -1:
        kw['dx_cols'] = K - (32 if K > 64 else 16)
      big = 140001 if sub else 5003
      CASES.append(case('bwd', big, K, n_out, act=act, w_off=w_off, **kw))
  CASES.append(case('bwd', 1, K, 1 + K % 4, act='relu', w_off=w_off))
  CASES.append(case('bwd', 7, K, 3, act='silu', out='dx', split=2, w_off=w_off))
  CASES.append(case('bwd', 1000 if sub else 1001, K, 4, out='params', split=1, w_off=w_off, strided=True))
  CASES.append(case('bwd', 1001, K, 3, act='relu', dx_cols=K - 16, out='dx', split=2, w_off=w_off))
  CASES.append(case('bwd', 2053, K, 1, out='alias', w_off=w_off))
CASES.append(case('bwd', 2 ** 20 + 3, 256, 1, out='alias'))          # the dW-only pass of a Dense(1) head on x
# ---- the output sets the models launch (test_launch_coverage_cpu.py) on contiguous operands: dW alone (no db), the
# parameter gradients alone, dx without dxsum, dx_cols without dx2, and the stacked view-independent heads
for K in (64, 128, 256, 1024):
  CASES.append(case('bwd', 2053 if K != 64 else 24577, K, 1, out='params', db=False))
for K in (64, 256):
  CASES.append(case('bwd', 8195, K, 3, out='params'))
  CASES.append(case('bwd', 4099 if K == 256 else 2049, K, 1, act='relu', out='dx'))
for K in (128, 256, 1024):
  CASES.append(case('bwd', 2049, K, 4, act='relu', out='dx', split=1))
for K in (128, 256):
  CASES.append(case('bwd', 2049, K, 4, out='params', split=1))
CASES.append(case('bwd', 1001, 64, 3, act='relu'))
CASES.append(case('bwd', 8195, 192, 1, act='relu', out='dx', dx_cols=64, dx2=False))
CASES.append(case('bwd', 2049, 320, 3, out='dx', dx_cols=256, dx2=False, strided=True))
CASES.append(case('bwd', 2049, 320, 3, out='dx'))
CASES.append(case('bwd', 2049, 448, 3, act='relu', dx_cols=128))
CASES.append(case('bwd', 2049, 128, 3, act='softplus'))
CASES.append(case('bwd', 8195, 128, 3, act='silu'))


def _embed_flat(shape, dtype, dev, col0, fill):
  """A contiguous [rows, cols] (or [n]) tensor inside a padded 1-D buffer."""
  n = math.prod(shape)
  v, buf = G.embed((n,), dtype, dev, extra_cols=col0 + 16, col0=col0, fill=fill)
  return v.view(*shape), buf


def _intact(view, buf):
  """G.padding_intact, also for a view of _embed_flat's 1-D buffers."""
  return G.padding_intact(view.reshape(-1) if buf.dim() == 1 else view, buf)


def layout(c, device, fill=True):
  """The case's buffers: inputs in NaN padding, outputs in sentinel padding (fill=False: uninitialised, for the
  plan alone).  Returns (views, buffers)."""
  M, K, n = c['M'], c['K'], c['n_out']
  nan, sen = ('nan', 'sentinel') if fill else (None, None)
  bf = torch.bfloat16
  v, bufs = {}, {}

  def put(name, view_buf):
    v[name], bufs[name] = view_buf

  pad = dict(extra_cols=24, col0=8) if c['strided'] else dict(extra_cols=0, col0=0)
  put('x', G.embed((M, K), bf, device, fill=nan, **pad))
  if c['mode'] == 'fwd':
    put('w', _embed_flat((n, K), bf, device, 8, nan))
    if c['bias']:
      put('b', _embed_flat((n,), torch.float32, device, 1, nan))
    put('raw', _embed_flat((M, n), torch.float32, device, 4, sen))
    return v, bufs
  put('w', _embed_flat((n, K), bf, device, 8 + c['w_off'], nan))
  put('draw', _embed_flat((M, n), torch.float32, device, 4, nan))
  cols = c['dx_cols'] or K
  split = c['split'] or n
  put('dw', _embed_flat((K, split), torch.float32, device, 2, sen))
  if split < n:
    put('dw2', _embed_flat((K, n - split), torch.float32, device, 2, sen))
  if c['db']:
    put('db', _embed_flat((n,), torch.float32, device, 2, sen))
  if c['out'] in ('dx', 'dx_sum'):
    put('dx', G.embed((M, cols), bf, device, fill=sen, **pad))
    if cols < K and c['dx2']:
      put('dx2', G.embed((M, K - cols), bf, device, fill=sen, **pad))
    if c['out'] == 'dx_sum':
      put('dxsum', _embed_flat((cols,), torch.float32, device, 2, sen))
  if c['act'] in ('softplus', 'silu'):
    put('z', G.embed((M, cols), bf, device, fill=nan, extra_cols=16 + (K - cols), col0=8))
  if c['out'] == 'alias':
    assert n == 1
    v['w'] = v['x'][0].view(1, K)
  return v, bufs


def plan(ops_mod, c, v):
  return ops_mod.head_plan(v['x'], v['w'], c['n_out'], c['K'], act=ACTS[c['act']], z=v.get('z'), dx=v.get('dx'))


def instance(c, p):
  if c['mode'] == 'fwd':
    return ('fwd', 'sub', p['fwd_lpr']) if p['fwd_kernel'] == 1 else ('fwd', 'warp')
  if p['bwd_kernel'] == 3:
    return ('bwd', 'sub', p['bwd_n_out'], p['bwd_lpr'], bool(p['bwd_smooth']))
  return ('bwd', 'warp', p['bwd_n_out'], p['bwd_chunks'], bool(p['bwd_smooth']))


def shape_flags(c, p):
  """(ragged, capped): the last block (or grid-stride pass) is partial; the grid is at its cap."""
  if c['mode'] == 'fwd':
    rpp = p['fwd_rows_per_pass']
    return c['M'] % rpp != 0, (c['M'] + rpp - 1) // rpp > p['fwd_grid']
  rpb = p['bwd_rows_per_block']
  return c['M'] % rpb != 0, rpb > (512 if p['bwd_kernel'] == 3 else 8)


def _fill(c, v, seed):
  M, K, n = c['M'], c['K'], c['n_out']
  g = torch.Generator(device='cuda').manual_seed(seed)

  def normal(*shape, scale=1.0):
    return torch.randn(*shape, generator=g, device='cuda') * scale

  spread = torch.exp2(torch.randint(-3, 4, (1, K), generator=g, device='cuda').float())
  for r0 in range(0, M, 1 << 18):
    r1 = min(M, r0 + (1 << 18))
    v['x'][r0:r1].copy_(normal(r1 - r0, K) * spread)
  if c['out'] != 'alias':
    v['w'].copy_(normal(n, K, scale=1 / math.sqrt(K)))
  init = {}
  if c['mode'] == 'fwd':
    if 'b' in v:
      v['b'].copy_(normal(n))
    return init
  v['draw'].copy_(normal(M, n))
  if 'z' in v:
    v['z'].copy_(normal(M, v['z'].shape[1], scale=2.0))
  for name in ('dw', 'dw2', 'db', 'dxsum'):
    if name in v:
      v[name].copy_(normal(*v[name].shape))
      init[name] = v[name].clone()
  return init


def launch(ops_mod, c, v):
  """The case's one launch on the views of layout(c, ...)."""
  if c['mode'] == 'fwd':
    ops_mod.head_fwd(v['x'], v['w'], v.get('b'), c['n_out'], c['K'], raw=v['raw'])
  else:
    act = ACTS[c['act']]
    ops_mod.head_bwd(v['x'], v['w'], v['draw'], c['n_out'], c['K'], dx=v.get('dx'), relu_mask=act == G.RELU,
                     dw=v['dw'], db=v.get('db'), dxsum=v.get('dxsum'), dw2=v.get('dw2'), dw_split=c['split'],
                     dx_cols=c['dx_cols'], dx2=v.get('dx2'), act=act if 'z' in v else G.NONE, z=v.get('z'))


def run(ops_mod, c, seed=0):
  v, bufs = layout(c, 'cuda')
  init = _fill(c, v, seed)
  launch(ops_mod, c, v)
  torch.cuda.synchronize()
  return v, bufs, init


def verify(c, v, bufs, init):
  for name in ('raw', 'dx', 'dx2', 'dw', 'dw2', 'db', 'dxsum'):
    if name in v:
      assert _intact(v[name], bufs[name]), f'{name}: a write outside the output'
  if c['mode'] == 'fwd':
    val, bound = H.head_fwd(v['x'], v['w'], v.get('b'))
    return {'raw': G.check(v['raw'], val, bound, 'raw')}
  split = c['split'] or c['n_out']
  dw_init = torch.cat([init['dw']] + ([init['dw2']] if 'dw2' in init else []), 1)
  ref = H.head_bwd(v['x'], v['w'], v['draw'], act=ACTS[c['act']], z=v.get('z'), dx_cols=c['dx_cols'],
                   dw_split=split, dw_init=dw_init, db_init=init.get('db'), dxsum_init=init.get('dxsum'),
                   want_dx='dx' in v)
  worst = {}
  for name, (val, bound) in ref.items():
    if name in v:
      worst[name] = G.check(v[name], val, bound, name)
  return worst


@pytest.mark.gpu
@pytest.mark.parametrize('c', CASES, ids=case_id)
def test_head_case(ops, c):
  v, bufs, init = run(ops, c, seed=c['M'] + 7 * c['K'] + c['n_out'])
  inst = instance(c, plan(ops, c, v))
  worst = verify(c, v, bufs, init)
  print(f'\n[heads err/bound] {inst} {case_id(c)}: ' + ' '.join(f'{k}={x:.3g}' for k, x in worst.items()))


# the shapes the heads were first checked at (fixed tolerances, contiguous operands), now under the fp64 bound
LEGACY_SHAPES = [(1000, 1024, 1), (777, 128, 3), (300, 256, 4), (515, 64, 2), (4099, 256, 1), (1, 128, 3),
                 (70001, 128, 3), (333, 192, 2)]


@pytest.mark.gpu
def test_heads_and_colsum_fp64(ops):
  """Each legacy shape: the forward with a bias, the ReLU-masked backward with dx and dxsum, and the
  parameter-gradient-only backward; then column sums of a [5000, 256] matrix."""
  for M, K, n in LEGACY_SHAPES:
    for c in (case('fwd', M, K, n), case('bwd', M, K, n, act='relu'), case('bwd', M, K, n, out='params')):
      v, bufs, init = run(ops, c, seed=M + K + n)
      verify(c, v, bufs, init)
  _colsum_case(ops, 5000, 256, False)


def fp64_launches(ops_mod):
  """Every launch test_head_case and test_heads_and_colsum_fp64 check against fp64, made through `launch` on
  uninitialised CPU buffers of the same layout, for the launch-coverage audit (test_launch_coverage_cpu.py)."""
  cases = list(CASES) + [c for M, K, n in LEGACY_SHAPES
                         for c in (case('fwd', M, K, n), case('bwd', M, K, n, act='relu'),
                                   case('bwd', M, K, n, out='params'))]
  for c in cases:
    v, _ = layout(c, 'cpu', fill=False)
    launch(ops_mod, c, v)


# ---------------------------------------------------------------------------------------------- coverage
def _reachable():
  """Every instance the launchers reach over a grid of widths, head sizes, activations and w alignments."""
  from multinerf_b200 import lib as L, ops as ops_mod
  found = set()
  for K in range(8, 1537, 8):
    for n in (1, 2, 3, 4):
      for act in ('none', 'relu', 'softplus'):
        for w_off in (0, 1):
          c = case('bwd', 600, K, n, act=act, out='dx', w_off=w_off)
          v, _ = layout(c, 'cpu', fill=False)
          try:
            p = plan(ops_mod, c, v)
          except L.MnrfError:
            continue
          found.add(instance(c, p))
          if p['fwd_kernel']:
            found.add(instance(dict(c, mode='fwd'), p))
  return found


def test_every_instance_has_cases():
  """Each reachable instance is the plan of a case with a ragged last block and of a case whose grid is capped (on
  an H100's 132 SMs; without a device the library plans for 132)."""
  from multinerf_b200 import ops as ops_mod
  reach = _reachable()
  assert len(reach) == 4 + 4 * 3 * 2 + 4 * 4 * 2, sorted(reach)
  ragged, capped = set(), set()
  for c in CASES:
    v, _ = layout(c, 'cpu', fill=False)
    p = plan(ops_mod, c, v)
    inst = instance(c, p)
    assert inst in reach, f'{case_id(c)} runs {inst}, which the enumeration does not reach'
    r, w = shape_flags(c, p)
    if r:
      ragged.add(inst)
    if w:
      capped.add(inst)
  assert not reach - ragged, f'instances without a ragged case: {sorted(reach - ragged)}'
  assert not reach - capped, f'instances without a capped-grid case: {sorted(reach - capped)}'


# ---------------------------------------------------------------------------------------------- column sums
COLSUM = [(m, n, (m + n) % 3 == 0) for n in (8, 256, 1032, 2048) for m in (1, 63, 64, 65, 5000, 10 ** 6)
          if m < 10 ** 6 or n <= 256]


@pytest.mark.gpu
@pytest.mark.parametrize('m,n,strided', COLSUM)
def test_colsum(ops, m, n, strided):
  worst = _colsum_case(ops, m, n, strided)
  print(f'\n[heads err/bound] colsum {m}x{n} strided={strided}: {worst:.3g}')


def _colsum_case(ops, m, n, strided):
  """One mnrf_colsum of an [m, n] matrix onto a non-zero initial value; returns the worst err / bound."""
  pad = dict(extra_cols=24, col0=8) if strided else dict(extra_cols=0, col0=0)
  x, _ = G.embed((m, n), torch.bfloat16, 'cuda', **pad)
  g = torch.Generator(device='cuda').manual_seed(m + n)
  for r0 in range(0, m, 1 << 17):
    r1 = min(m, r0 + (1 << 17))
    x[r0:r1].copy_(torch.randn(r1 - r0, n, generator=g, device='cuda') * 4 + 1)
  out, buf = G.embed((n,), torch.float32, 'cuda', extra_cols=4, col0=2, fill='sentinel')
  out.copy_(torch.randn(n, generator=g, device='cuda'))
  init = out.clone()
  ops.colsum(x, n, out)
  torch.cuda.synchronize()
  assert G.padding_intact(out, buf)
  val, bound = H.colsum(x, init)
  return G.check(out, val, bound, 'colsum')


# ---------------------------------------------------------------------------------------------- weight packing
PACK_SHAPES = [(1, 1), (33, 1), (100, 257), (1536, 1024), (64, 3), (320, 128), (256, 256), (8, 40), (31, 33),
               (32, 32), (65, 7), (128, 1), (1, 300), (257, 100), (96, 4), (1024, 256), (17, 64), (200, 3),
               (40, 40), (512, 129), (3, 3), (127, 255), (2, 1024), (1000, 1), (48, 16), (256, 4), (72, 72),
               (160, 256), (5, 9), (33, 65), (512, 512), (9, 1536), (64, 64), (128, 3), (300, 17), (11, 13),
               (256, 1), (100, 100), (44, 88), (1280, 256)]


@pytest.mark.gpu
def test_pack_weights_batched(ops):
  """One launch over 40 ragged items, some without w_nk and some without w_kn; masters hold exact bf16 ties, fp32
  subnormals, +-0, values that overflow to inf, +-inf and NaN; shadows sit in sentinel buffers."""
  g = torch.Generator(device='cuda').manual_seed(17)
  specials = torch.tensor([1 + 2 ** -8, 1 + 3 * 2 ** -8, -(1 + 2 ** -8), 2 ** -130, -3 * 2 ** -140, 1e-40, 0.0, -0.0,
                           3.4e38, -3.399e38, float('inf'), float('-inf'), float('nan'), 2 ** -126 * (1 + 2 ** -8)],
                          device='cuda')
  layers, shadows = [], []
  for i, (in_pad, out) in enumerate(PACK_SHAPES):
    master, _ = _embed_flat((in_pad, out), torch.float32, 'cuda', 4, 'nan')
    master.copy_(torch.randn(in_pad, out, generator=g, device='cuda') * 2.0 ** (i % 7 - 3))
    idx = torch.randint(0, in_pad * out, (min(in_pad * out, 2 * len(specials)),), generator=g, device='cuda')
    master.view(-1)[idx] = specials.repeat(2)[:idx.numel()]
    nk = None if i % 5 == 3 else _embed_flat((out, in_pad), torch.bfloat16, 'cuda', 8, 'sentinel')
    kn = None if i % 7 == 2 else _embed_flat((in_pad, out), torch.bfloat16, 'cuda', 8, 'sentinel')
    layers.append((master, nk[0] if nk else None, kn[0] if kn else None))
    shadows.append((master, nk, kn))
  ops.pack_weights_batched(ops.pack_table(layers, 'cuda'))
  torch.cuda.synchronize()
  for i, (master, nk, kn) in enumerate(shadows):
    if nk:
      assert _intact(*nk), f'item {i}: w_nk padding'
      assert H.pack_matches(nk[0], master.T.contiguous()), f'item {i} {PACK_SHAPES[i]}: w_nk'
    if kn:
      assert _intact(*kn), f'item {i}: w_kn padding'
      assert H.pack_matches(kn[0], master), f'item {i} {PACK_SHAPES[i]}: w_kn'


# ---------------------------------------------------------------------------------------------- clip + Adam
def adam_case(n, gmn, gmv, scale, dyn, step, special):
  return dict(n=n, grad_max_norm=gmn, grad_max_val=gmv, grad_scale=scale, dyn=dyn, step=step, special=special)


ADAM_CASES = []
for i, n in enumerate((1, 255, 100003, 300007)):
  for j, (gmn, gmv) in enumerate(((1e-3, 0.0), (1e-3, 2e-2), (0.0, 2e-2), (0.0, 0.0))):
    step = (1, 2, 7, 250000)[(i + j) % 4]
    special = ('none', 'nan', 'inf')[(i + 2 * j) % 3] if n > 1 else 'none'
    if special == 'inf' and step == 1 and gmn == 0 and gmv == 0:
      step = 2                                # m / bc1 would sit on the fp32 overflow threshold
    ADAM_CASES.append(adam_case(n, gmn, gmv, (1.0, 0.125)[(i + j) % 2], (i + j) % 3 == 1, step, special))


def _adam_id(c):
  return (f"n{c['n']}-norm{c['grad_max_norm']}-val{c['grad_max_val']}-scale{c['grad_scale']}-"
          f"{'dyn' if c['dyn'] else 'host'}-step{c['step']}-{c['special']}")


def _adam_run(ops, c, seed):
  n = c['n']
  g_ = torch.Generator(device='cuda').manual_seed(seed)
  bufs = {name: G.embed((n,), torch.float32, 'cuda', extra_cols=8, col0=4, fill='sentinel')
          for name in ('p', 'mu', 'nu')}
  grad, _ = G.embed((n,), torch.float32, 'cuda', extra_cols=8, col0=4)
  bufs['p'][0].copy_(torch.randn(n, generator=g_, device='cuda'))
  grad.copy_(torch.randn(n, generator=g_, device='cuda') * 1e-2 *
             torch.exp2(torch.randint(-4, 5, (n,), generator=g_, device='cuda').float()))
  bufs['mu'][0].copy_(torch.randn(n, generator=g_, device='cuda') * 1e-3)
  bufs['nu'][0].copy_(torch.rand(n, generator=g_, device='cuda') * 1e-5)
  if c['special'] == 'nan':
    grad[n // 3] = float('nan')
  elif c['special'] == 'inf':
    grad[n // 3], grad[n // 2 + 1] = float('inf'), float('-inf')
  init = {name: b[0].clone() for name, b in bufs.items()}
  scratch = torch.full((1,), 12345.0, device='cuda')          # garbage: the call zeroes it
  kw = dict(step=c['step'], lr=1.5e-3, beta1=0.9, beta2=0.999, eps=1e-6, grad_max_val=c['grad_max_val'],
            grad_max_norm=c['grad_max_norm'], grad_scale=c['grad_scale'])
  dyn = None
  if c['dyn']:
    t = c['step']
    dyn = torch.tensor([7e-4, 1 - 0.9 ** t, 1 - 0.999 ** t], dtype=torch.float32, device='cuda')
  ops.clip_adam(bufs['p'][0], grad, bufs['mu'][0], bufs['nu'][0], scratch, dyn=dyn, **kw)
  torch.cuda.synchronize()
  ref = H.clip_adam(init['p'], grad, init['mu'], init['nu'], dyn=dyn, **kw)
  return bufs, ref, grad, init


@pytest.mark.gpu
@pytest.mark.parametrize('c', ADAM_CASES, ids=_adam_id)
def test_clip_adam(ops, c):
  bufs, ref, _, _ = _adam_run(ops, c, seed=c['n'] + c['step'])
  worst = {}
  for name, (view, buf) in bufs.items():
    assert G.padding_intact(view, buf), f'{name}: a write outside the buffer'
    worst[name] = H.check_adam(view, *ref[name], name)
  print(f'\n[heads err/bound] clip_adam {_adam_id(c)}: ' + ' '.join(f'{k}={x:.3g}' for k, x in worst.items()))


@pytest.mark.gpu
def test_clip_adam_nan_semantics(ops):
  """train_utils.py:200-218 then :328: jnp.clip and jnp.minimum propagate NaN, so one NaN makes the module's mult
  NaN and the whole module's gradient 0 (the moments decay); without the norm clip only the NaN element is zeroed,
  under a value clip too (0, not -grad_max_val)."""
  b1 = torch.tensor(0.9, dtype=torch.float32)
  for gmv in (0.0, 0.1):
    bufs, _, grad, init = _adam_run(ops, adam_case(100003, 1e-3, gmv, 1.0, False, 7, 'nan'), seed=3)
    assert torch.equal(bufs['mu'][0], b1 * init['mu']), gmv
    assert torch.isfinite(bufs['p'][0]).all()
  bufs, _, grad, init = _adam_run(ops, adam_case(100003, 0.0, 1e-3, 1.0, False, 7, 'nan'), seed=3)
  i = 100003 // 3
  assert float(bufs['mu'][0][i]) == float(b1 * init['mu'][i])
  assert not torch.equal(bufs['mu'][0], b1 * init['mu'])


# ---------------------------------------------------------------------------------------------- chained trunk head
@pytest.mark.gpu
@pytest.mark.parametrize('M', [1000, 16384 + 37])
def test_chain_head_vs_fp64(ops, M):
  """csrc/chain.cu's epilogue head (head_n 4 and 1) is Dense(head_n) on the bf16 activation it stores, fp32
  accumulate: checked against the head_fwd bound on that stored activation."""
  from multinerf_b200 import lib as L
  W, Fpad = 256, 128
  g = torch.Generator(device='cuda').manual_seed(M)
  feat = (torch.rand(M, Fpad, device='cuda', generator=g) * 2 - 1).to(torch.bfloat16)
  ws = [((torch.rand(W, k, device='cuda', generator=g) * 2 - 1) * (6 / k) ** 0.5).to(torch.bfloat16)
        for k in (Fpad, W, W)]
  bs = [torch.rand(W, device='cuda', generator=g) * 0.1 for _ in range(3)]
  hw = ((torch.rand(4, W, device='cuda', generator=g) * 2 - 1) * 0.1).to(torch.bfloat16)
  hb = torch.rand(4, device='cuda', generator=g)
  acts = [torch.empty(M, W, device='cuda', dtype=torch.bfloat16) for _ in range(3)]
  layers = [dict(w=ws[0], bias=bs[0], out=acts[0], n_stream=Fpad // 64, stream_col0=0, stream_kb0=0)]
  layers += [dict(w=ws[i], bias=bs[i], out=acts[i], n_res=4, res_kb0=0) for i in (1, 2)]
  worst = {}
  for head_n in (4, 1):
    out, buf = _embed_flat((M, head_n), torch.float32, 'cuda', 4, 'sentinel')
    ops.mlp_chain(ops.chain_desc(L.CHAIN_FWD, M, layers, stream=feat, stream_cols=Fpad,
                                 head_w=hw[:head_n].float().contiguous(), head_b=hb[:head_n], head_out=out,
                                 head_n=head_n))
    torch.cuda.synchronize()
    assert _intact(out, buf)
    val, bound = H.head_fwd(acts[-1], hw[:head_n], hb[:head_n])
    worst[f'head{head_n}'] = G.check(out, val, bound, f'chain head_n={head_n}')
  print(f'\n[heads err/bound] chain head M={M}: ' + ' '.join(f'{k}={x:.3g}' for k, x in worst.items()))


# ---------------------------------------------------------------------------------------------- argument checks
def _has_alignment_checks(ops):
  """The library refuses a misaligned x before any launch (asked of the host-only plan, so an older library that would
  launch the misaligned access is never called with one)."""
  from multinerf_b200 import lib as L
  x = torch.zeros(64, 72, dtype=torch.bfloat16, device='cuda')
  try:
    ops.head_plan(x[:, 4:68], x[0, 8:72].view(1, 64), 1, 64)
  except L.MnrfError:
    return True
  return False


def _bad_calls():
  """name -> builder returning (call, output buffers that must stay unchanged, misaligned-pointer case)."""
  from multinerf_b200 import lib as L
  dev, bf = 'cuda', torch.bfloat16

  def bwd(K=128, n_out=2, x=None, dx='default', **kw):
    def build():
      xx = x() if x else torch.zeros(256, K, dtype=bf, device=dev)
      w = torch.zeros(n_out, K, dtype=bf, device=dev)
      draw = torch.zeros(256, n_out, device=dev)
      dw, dwb = _embed_flat((K, n_out), torch.float32, dev, 2, 'sentinel')
      db, dbb = _embed_flat((n_out,), torch.float32, dev, 2, 'sentinel')
      bufs = [dwb, dbb]
      extra = {}
      for name, val in kw.items():
        if callable(val):
          extra[name], b = val()
          if b is not None:
            bufs.append(b)
        else:
          extra[name] = val
      d = dx() if callable(dx) else (G.embed((256, K), bf, dev, fill='sentinel') if dx == 'default' else (None, None))
      if d[1] is not None:
        bufs.append(d[1])
      return (lambda ops: ops.head_bwd(xx, w, draw, n_out, K, dx=d[0], dw=dw, db=db, **extra)), bufs
    return build

  def sen(shape, dtype=torch.float32, col0=2):
    return lambda: (_embed_flat(shape, dtype, dev, col0, 'sentinel'))

  def off_out(shape, by):
    def make():
      v, buf = G.embed(shape, bf, dev, extra_cols=8, col0=by, fill='sentinel')
      return v, buf
    return make

  cases = {}
  cases['bwd n_out 5'] = (bwd(n_out=5), False)
  cases['bwd dxsum without dx'] = (bwd(dx=None, dxsum=sen((128,))), False)
  cases['bwd split without dw2'] = (bwd(n_out=3, dw_split=2), False)
  cases['bwd z with relu'] = (bwd(act=L.ACT_RELU, z=lambda: (torch.zeros(256, 128, dtype=bf, device=dev), None)),
                              False)
  cases['bwd K > 1536'] = (bwd(K=1544, n_out=1), False)
  cases['bwd dx_cols % 8'] = (bwd(dx_cols=60), False)
  cases['bwd x misaligned'] = (bwd(x=lambda: G.embed((256, 136), bf, dev, fill='sentinel')[0][:, 4:132]), True)
  cases['bwd dx misaligned'] = (bwd(dx=off_out((256, 128), 4)), True)

  def colsum_mis():
    x = G.embed((256, 64), bf, dev, extra_cols=8, col0=4)[0]
    out, buf = _embed_flat((64,), torch.float32, dev, 2, 'sentinel')
    return (lambda ops: ops.colsum(x, 64, out)), [buf]
  cases['colsum x misaligned'] = (colsum_mis, True)

  def colsum_n():
    x = torch.zeros(256, 68, dtype=bf, device=dev)[:, :60]
    out, buf = _embed_flat((60,), torch.float32, dev, 2, 'sentinel')
    return (lambda ops: ops.colsum(x, 60, out)), [buf]
  cases['colsum N % 8'] = (colsum_n, False)

  def fwd_w_mis():
    x = torch.zeros(256, 64, dtype=bf, device=dev)
    w = torch.zeros(72, dtype=bf, device=dev)[4:68].view(1, 64)
    raw, buf = _embed_flat((256, 1), torch.float32, dev, 4, 'sentinel')
    return (lambda ops: ops.head_fwd(x, w, None, 1, 64, raw=raw)), [buf]
  cases['fwd w misaligned'] = (fwd_w_mis, False)
  return cases


BAD = ['bwd n_out 5', 'bwd dxsum without dx', 'bwd split without dw2', 'bwd z with relu', 'bwd K > 1536',
       'bwd dx_cols % 8', 'bwd x misaligned', 'bwd dx misaligned', 'colsum x misaligned', 'colsum N % 8',
       'fwd w misaligned']


@pytest.mark.gpu
@pytest.mark.parametrize('name', BAD)
def test_rejected_arguments(ops, name):
  from multinerf_b200 import lib as L
  builder, misaligned = _bad_calls()[name]
  if misaligned:
    assert _has_alignment_checks(ops), 'the library does not check pointer alignment: not launching'
  call, bufs = builder()
  torch.cuda.synchronize()
  before = [b.clone() for b in bufs]
  with pytest.raises(L.MnrfError):
    call(ops)
  torch.cuda.synchronize()
  for b0, b in zip(before, bufs):
    assert torch.equal(_bits(b0), _bits(b)), f'{name}: the refused call wrote its output'


def test_head_instance_layout_matches_header():
  """ops.head_plan passes a HeadInstance by reference through a void pointer: its size and field offsets must be
  those of mnrf_head_instance (compiled check)."""
  import ctypes
  import os
  import subprocess
  import tempfile
  from multinerf_b200 import lib as L
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  fields = [name for name, _ in L.HeadInstance._fields_]
  src = ('#include <stdio.h>\n#include <stddef.h>\n#include "mnrf.h"\nint main(){printf("%zu", sizeof(mnrf_head_instance));'
         + ''.join(f'printf(" %zu", offsetof(mnrf_head_instance, {f}));' for f in fields) + 'return 0;}')
  with tempfile.TemporaryDirectory() as td:
    open(os.path.join(td, 'a.c'), 'w').write(src)
    subprocess.run(['gcc', '-I', os.path.join(root, 'include'), os.path.join(td, 'a.c'), '-o', os.path.join(td, 'a')],
                   check=True)
    got = list(map(int, subprocess.run([os.path.join(td, 'a')], capture_output=True, text=True).stdout.split()))
  want = [ctypes.sizeof(L.HeadInstance)] + [getattr(L.HeadInstance, f).offset for f in fields]
  assert got == want


def test_plan_refuses_misaligned_x_and_dx():
  """Host-only: the plan (and so the launch, which runs the same checks) refuses x or dx off a 16-byte boundary and
  takes any w."""
  from multinerf_b200 import lib as L, ops as ops_mod
  buf = torch.zeros(64, 80, dtype=torch.bfloat16)
  x, w = buf[:, :64], buf[0, :64].view(1, 64)
  assert ops_mod.head_plan(x, w, 1, 64)['bwd_kernel'] == L.HEAD_BWD_SUB
  p = ops_mod.head_plan(x, buf[0, 4:68].view(1, 64), 1, 64)
  assert p['bwd_kernel'] == L.HEAD_BWD_WARP and p['bwd_chunks'] == 1 and p['fwd_kernel'] == L.HEAD_NONE
  for bad in (dict(x=buf[:, 4:68]), dict(dx=buf[:, 4:68])):
    with pytest.raises(L.MnrfError):
      ops_mod.head_plan(bad.get('x', x), w, 1, 64, dx=bad.get('dx'))
