"""Case matrix of the layer-chained 256-wide trunk (csrc/chain.cu, mnrf_mlp_chain) against fp64.

Each case is launched on random data, checked against the per-element bound of tests/chain_ref.py, and on exact data
(chain_ref.make_data), checked bit for bit.  Every input is a view inside NaN padding, so a read through a wrong
base, pitch or column offset shows as a NaN; every output sits inside sentinel padding, checked after each launch.
Row counts come from the device's SM count: 1, 63, 64, 65 and 129 rows, two units per SM plus and minus one unit,
and 2^20 - 37.  The forward cases run the train form (every layer stored with its mask words), the render form
(the last layer alone, no mask words) and, where given, a mix of stored layers and mask words: the last two must
equal the train form bit for bit.  Backward cases run with and without column sums and mask words; the fwd_bwd
cases chain a forward launch into the backward launch fed its mask words, as Model._chain_fwd_desc /
_chain_bwd_desc build them.  test_every_schedule_class_has_cases (test_chain_reference_cpu.py) checks that these
cases reach every schedule class.  Also: non-finite rows, zero and subnormal pre-activations, and every argument
check.  Needs an H100.
"""
import os
import time

import numpy as np
import pytest
import torch

import chain_ref as R
import gemm_ref as G

pytestmark = pytest.mark.gpu

W = R.W
SL = R.spec_layer
SMS = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


@pytest.fixture(scope='module')
def ops():
  from multinerf_b200 import lib, ops as _ops
  lib.require_device()
  return _ops


# ---------------------------------------------------------------------------------------------- cases
def trunk(depth, fpad, skip=0, extra_k=0):
  """The forward layers of a models.py trunk: features streamed into layer 0, and into the layer after `skip` as
  weight k-blocks 4.. after the resident ones."""
  nf = fpad // 64
  ls = [SL(n_stream=nf, extra_k=extra_k)]
  for i in range(1, depth):
    if skip and i - 1 == skip:
      ls.append(SL(n_res=4, n_stream=nf, stream_kb0=4, extra_k=extra_k))
    else:
      ls.append(SL(n_res=4, extra_k=extra_k))
  return ls


def bwd_trunk(depth, colsum=True, maskbits=True):
  return [SL(n_stream=4, colsum=colsum, maskbits=maskbits)] + \
      [SL(n_res=4, colsum=colsum, maskbits=maskbits) for _ in range(depth - 2)]


def row_counts(sms):
  return [1, 63, 64, 65, 129, (2 * sms - 1) * 128, (2 * sms + 1) * 128, (1 << 20) - 37]


def cases(sms):
  """The case list for a device of `sms` SMs: dicts of kind ('fwd', 'bwd', 'fwd_bwd'), M, lspecs, stream_cols,
  head_n, head_b, mix (FWD: (out, maskbits) per layer of a third launch) and depth (fwd_bwd)."""
  out = []

  def add(kind, name, M, lspecs=None, stream_cols=0, head_n=1, head_b=True, mix=None, fpad=0, skip=0, depth=0):
    out.append(dict(kind=kind, name=f'{kind}-{name}-M{M}', M=M, lspecs=lspecs, stream_cols=stream_cols,
                    head_n=head_n, head_b=head_b, mix=mix, fpad=fpad, skip=skip, depth=depth))

  # PropMLP of 360.gin (4 x 256, Fpad 512) at every row count
  for M in row_counts(sms):
    add('fwd', 'prop', M, trunk(4, 512), 512)
  # NerfMLP 8 x 256 with the skip after layer 4 (Fpad 128: 4 resident + 2 streamed k-blocks; Fpad 320: 4 + 5, three
  # segments, the ring wraps inside one)
  for M in (65, 8320, 20032):
    add('fwd', 'nerf128', M, trunk(8, 128, skip=4), 128)
  for M in (129, 12345):
    add('fwd', 'nerf320', M, trunk(8, 320, skip=4), 320)
  # the shapes of the earlier per-layer comparisons
  for M, depth, fpad in [(512, 4, 512), (16384, 4, 512), (100352, 4, 512), (1000, 4, 128), (2048, 4, 704),
                         (4096, 2, 64), (777, 1, 192), (4097, 2, 64)]:
    add('fwd', f'd{depth}f{fpad}', M, trunk(depth, fpad), fpad)
  # heads: density + rgb stacked (NH 4), no head, a head without a bias
  add('fwd', 'nh4', 1000, trunk(4, 256), 256, head_n=4)
  add('fwd', 'nh4', (2 * sms + 1) * 128, trunk(8, 128, skip=4), 128, head_n=4)
  add('fwd', 'nohead', 5000, trunk(4, 128), 128, head_n=0)
  add('fwd', 'nohead', 63, trunk(2, 64), 64, head_n=0)
  add('fwd', 'headnobias', 777, trunk(3, 192), 192, head_b=False)
  # operand layouts: features at column 128 of a wider tensor, the resident operand after the streamed k-blocks in
  # the weight columns, a weight pitch past K, a later layer that streams from another column
  lay = [SL(n_stream=4, stream_col0=128, extra_k=64),
         SL(n_res=4, res_kb0=2, n_stream=2, stream_col0=0, stream_kb0=0),
         SL(n_res=4, extra_k=128),
         SL(n_res=4, n_stream=3, stream_col0=320, stream_kb0=5)]
  for M in (64, 3000):
    add('fwd', 'layout', M, lay, 640)
  # the most layers a launch takes
  add('fwd', 'depth8', 9000, trunk(8, 256), 256)
  # mixes of stored layers and mask words
  add('fwd', 'mix', 2000, trunk(4, 128), 128, mix=[(True, False), (False, True), (False, False), (True, True)])
  add('fwd', 'mix', 20032, trunk(8, 128, skip=4), 128,
      mix=[(False, False), (True, False), (False, True), (True, True), (False, False), (True, False), (False, True),
           (True, False)])
  # backward: the model's form (no column sums) and with column sums, at every row count
  for M in row_counts(sms):
    add('bwd', 'model', M, bwd_trunk(4, colsum=False), 256)
    add('bwd', 'colsum', M, bwd_trunk(4), 256)
  for M, depth in [(512, 4), (16384, 4), (100352, 4), (1000, 4), (8320, 8), (640, 2), (4097, 2), (5000, 4)]:
    add('bwd', f'd{depth}', M, bwd_trunk(depth), 256)
  # a later layer that streams (the gradient of a skip layer's features, columns 256..), a layer without mask words
  blay = [SL(n_stream=4, colsum=True), SL(n_res=4, maskbits=False, colsum=True),
          SL(n_res=4, n_stream=2, stream_col0=256, stream_kb0=4, colsum=True, extra_k=64),
          SL(n_res=4, colsum=False)]
  for M in (65, 7000):
    add('bwd', 'layout', M, blay, 384)
  add('bwd', 'nomask', 3000, bwd_trunk(3, maskbits=False), 256)
  add('bwd', 'nomask-nocolsum', 200, bwd_trunk(3, colsum=False, maskbits=False), 256)
  # forward chain, then the backward chain fed its mask words (the model's descriptors)
  for M in ((2 * sms + 1) * 128, (1 << 20) - 37):
    add('fwd_bwd', 'prop', M, fpad=512, depth=4)
  add('fwd_bwd', 'nerf', 20032, fpad=128, skip=4, depth=8)
  add('fwd_bwd', 'nerf', 12345, fpad=320, skip=4, depth=8)
  return out


def launches(c):
  """(mode, lspecs, head_n) of every launch a case makes."""
  if c['kind'] == 'fwd':
    render = [dict(ls, out=i == len(c['lspecs']) - 1, maskbits=False) for i, ls in enumerate(c['lspecs'])]
    res = [(R.FWD, c['lspecs'], c['head_n']), (R.FWD, render, c['head_n'])]
    if c['mix']:
      res.append((R.FWD, [dict(ls, out=o, maskbits=b) for ls, (o, b) in zip(c['lspecs'], c['mix'])], c['head_n']))
    return res
  if c['kind'] == 'bwd':
    return [(R.BWD, c['lspecs'], 0)]
  fwd = trunk(c['depth'], c['fpad'], c['skip'])
  return [(R.FWD, fwd, 1), (R.BWD, bwd_trunk(c['depth'], colsum=False), 0)]


CASES = cases(SMS)


# ---------------------------------------------------------------------------------------------- buffers
def _in(t, extra_cols=16, col0=8):
  """A copy of t inside NaN padding (rows above and below, columns on both sides)."""
  v, buf = G.embed(tuple(t.shape), t.dtype, 'cuda', extra_cols=extra_cols, col0=col0)
  v.copy_(t)
  return v, buf


def _out(shape, dtype, extra_cols, col0):
  return G.embed(shape, dtype, 'cuda', extra_cols=extra_cols, col0=col0, fill='sentinel')


def device_data(d, mode):
  """The case's operands as device views in NaN padding."""
  dd = dict(d)
  dd['stream'] = _in(d['stream'].cuda())[0]
  dd['w'] = [_in(w.cuda())[0] for w in d['w']]
  if mode == R.FWD:
    dd['bias'] = [_in(b.cuda(), extra_cols=4, col0=2)[0] for b in d['bias']]
  else:
    # mask words 4 bytes off an 8-byte boundary: the loads of the backward epilogue at any alignment
    dd['masks'] = [_in(mk.cuda(), extra_cols=3, col0=1)[0] for mk in d['masks']]
  if d.get('head_w') is not None:
    hw, _ = _in(d['head_w'].cuda().reshape(-1), extra_cols=8, col0=4)
    dd['head_w'] = hw.view(d['head_w'].shape)
    dd['head_b'] = _in(d['head_b'].cuda(), extra_cols=2, col0=1)[0] if d.get('head_b') is not None else None
  return dd


def launch(ops, mode, M, lspecs, dd, stream_cols, head_n, *, narrow_bits=False, colsum_init=None):
  """One launch with every output in sentinel padding.  Returns (got, buffers to check)."""
  from multinerf_b200 import lib as L
  outs, bits, colsums, guard = [], [], [], []
  for j, ls in enumerate(lspecs):
    if ls['out']:
      o, ob = _out((M, W), torch.bfloat16, 16, 8)
      outs.append(o)
      guard.append((o, ob))
    else:
      outs.append(None)
    if mode == R.FWD and ls['maskbits']:
      b, bb = _out((M, W // 32), torch.int32, 3 if narrow_bits else 4, 1 if narrow_bits else 2)
      bits.append(b)
      guard.append((b, bb))
    else:
      bits.append(None)
    if mode == R.BWD and ls['colsum']:
      cs, cb = _out((W,), torch.float32, 4, 2)
      cs.copy_(colsum_init[j].cuda())
      colsums.append(cs)
      guard.append((cs, cb))
    else:
      colsums.append(None)
  layers = R.layer_dicts(mode, lspecs, dd, outs=outs, bits=bits, colsums=colsums)
  head = dict()
  hv = None
  if mode == R.FWD and head_n:
    hv, hb = _out((M, head_n), torch.float32, 0, 0)
    guard.append((hv, hb))
    head = dict(head_w=dd['head_w'], head_b=dd.get('head_b'), head_out=hv, head_n=head_n)
  ops.mlp_chain(ops.chain_desc(mode, M, layers, stream=dd['stream'], stream_cols=stream_cols, **head))
  torch.cuda.synchronize()
  for v, buf in guard:
    assert G.padding_intact(v, buf), 'a write outside an output'
  return dict(outs=outs, bits=bits if mode == R.FWD else None, head=hv,
              colsums=colsums if mode == R.BWD else None), layers


def _colsum_init(d, lspecs):
  return [c if ls['colsum'] else None for c, ls in zip(d['colsum_init'], lspecs)] if d['colsum_init'] else None


def _bits(t):
  return t.view({torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.int32: torch.int32}[t.dtype])


def _same(a, b, what):
  assert torch.equal(_bits(a), _bits(b)), f'{what}: differs bitwise from the train form'


def _check(mode, M, layers, dd, got, exact, init=None):
  return R.check_launch(mode, M, layers, dd['stream'], got, exact=exact, head_w=dd.get('head_w'),
                        head_b=dd.get('head_b'), colsum_init=init)


def run_fwd(ops, c, exact, seed):
  M = c['M']
  d = R.make_data(R.FWD, M, c['lspecs'], c['stream_cols'], head_n=c['head_n'], head_b=c['head_b'], exact=exact,
                  seed=seed)
  dd = device_data(d, R.FWD)
  (_, train, nh), (_, render, _), *mix = launches(c)
  got, layers = launch(ops, R.FWD, M, train, dd, c['stream_cols'], nh, narrow_bits=M % 2 == 1)
  worst = _check(R.FWD, M, layers, dd, got, exact)
  for form in [render] + [m[1] for m in mix]:
    g2, _ = launch(ops, R.FWD, M, form, dd, c['stream_cols'], nh)
    for j, ls in enumerate(form):
      if ls['out']:
        _same(g2['outs'][j], got['outs'][j], f'layer {j} output')
      if ls['maskbits']:
        _same(g2['bits'][j], got['bits'][j], f'layer {j} mask words')
    if nh:
      _same(g2['head'], got['head'], 'head')
  return worst


def run_bwd(ops, c, exact, seed):
  M = c['M']
  d = R.make_data(R.BWD, M, c['lspecs'], c['stream_cols'], exact=exact, seed=seed)
  dd = device_data(d, R.BWD)
  init = _colsum_init(d, c['lspecs'])
  got, layers = launch(ops, R.BWD, M, c['lspecs'], dd, c['stream_cols'], 0, colsum_init=init)
  return _check(R.BWD, M, layers, dd, got, exact, init)


def run_fwd_bwd(ops, c, exact, seed):
  """The forward chain, then the backward chain with w_kn = w_nk^T of every layer after the first and the forward
  launch's mask words of the layer before, no column sums (Model._chain_bwd_desc)."""
  M = c['M']
  (_, fwd, _), (_, bwd, _) = launches(c)
  d = R.make_data(R.FWD, M, fwd, c['fpad'], head_n=1, exact=exact, seed=seed)
  dd = device_data(d, R.FWD)
  got, layers = launch(ops, R.FWD, M, fwd, dd, c['fpad'], 1)
  worst = {f'fwd {k}': v for k, v in _check(R.FWD, M, layers, dd, got, exact).items()}
  db = R.make_data(R.BWD, M, bwd, W, exact=exact, seed=seed + 1)
  depth = len(fwd)
  # w_kn [in_pad, 256] of trunk layer i (rows past 256: a skip layer's feature rows, never read)
  db['w'] = [dd['w'][i].T.contiguous() for i in range(depth - 1, 0, -1)]
  db['masks'] = [got['bits'][i - 1] for i in range(depth - 1, 0, -1)]
  dbd = dict(db, stream=_in(db['stream'].cuda())[0], w=[_in(w)[0] for w in db['w']], masks=db['masks'])
  gb, blayers = launch(ops, R.BWD, M, bwd, dbd, W, 0)
  worst.update({f'bwd {k}': v for k, v in _check(R.BWD, M, blayers, dbd, gb, exact).items()})
  return worst


RUN = {'fwd': run_fwd, 'bwd': run_bwd, 'fwd_bwd': run_fwd_bwd}


@pytest.mark.parametrize('c', CASES, ids=[c['name'] for c in CASES])
def test_chain_case(ops, c):
  t0 = time.perf_counter()
  seed = c['M'] + len(c['name'])
  worst = RUN[c['kind']](ops, c, False, seed)
  exact = RUN[c['kind']](ops, c, True, seed)
  assert all(v == 0 for v in exact.values())
  sch = [R.schedule(m, ls, c['M'], SMS, head_n=nh) for m, ls, nh in launches(c)]
  print(f"\n[chain err/bound] {c['name']} units={sch[0]['units']} grid={sch[0]['grid']} segs={sch[0]['segs']}: " +
        ' '.join(f'{k}={v:.3g}' for k, v in worst.items()) +
        f' | exact: bit-equal | {time.perf_counter() - t0:.2f} s')


# ---------------------------------------------------------------------------------------------- non-finite rows
POISON = {3: float('nan'), 200: float('inf'), 201: -float('inf'), 640: float('nan')}   # row -> value


def _classes_match(got, value, what):
  g = got.double()
  for name, f in (('NaN', torch.isnan), ('+inf', lambda t: torch.isposinf(t)), ('-inf', lambda t: torch.isneginf(t))):
    assert torch.equal(f(g), f(value)), f'{what}: {name} elements differ from fp64'


def _check_poisoned_rows(mode, layers, dd, got, rows, init=None):
  """The poisoned rows against fp64 on the kernel's own inputs of those rows: the same NaN and +-inf elements, the
  finite ones inside their bound, mask bits the sign of the pre-activation (0 for NaN)."""
  idx = torch.tensor(rows, device='cuda')
  sub = [dict(ly, maskbits=ly['maskbits'][idx]) if ly.get('maskbits') is not None and mode == R.BWD else ly
         for ly in layers]
  stored = [o[idx] for o in got['outs']]
  for j, r in R.ref_chain(mode, len(rows), sub, dd['stream'][idx], stored=stored, head_w=dd.get('head_w'),
                          head_b=dd.get('head_b')):
    _classes_match(stored[j], r['out'].to(torch.bfloat16).double(), f'layer {j}')
    fin = torch.isfinite(r['out'])
    if fin.any():
      G.check(stored[j][fin], r['out'][fin], r['out_bound'][fin], f'layer {j} finite elements')
    if mode == R.FWD:
      z = r['z']
      bits = G.unpack_bits(got['bits'][j][idx], W)
      nonfin = ~torch.isfinite(z)
      assert torch.equal(bits[nonfin], (z > 0)[nonfin]), f'layer {j}: mask bits of non-finite pre-activations'
      assert not bits[torch.isnan(z)].any(), f'layer {j}: a NaN with its mask bit set'
      if 'head' in r:
        _classes_match(got['head'][idx], r['head'][0], 'head')
    else:
      if layers[j].get('maskbits') is not None:
        keep = G.unpack_bits(layers[j]['maskbits'][idx], W)
        assert bool((stored[j][~keep] == 0).all()), f'layer {j}: a masked-out gradient is not 0'


@pytest.mark.parametrize('mode', ['fwd', 'bwd'])
def test_non_finite_rows(ops, mode):
  """NaN and +-inf in designated rows of the features (FWD) or of dy (BWD), inside the view.  The oracle's contract:
  NaN propagates through the ReLU, a NaN's mask bit is 0, a masked-out gradient is 0 whatever the sum (a select),
  the head of a poisoned row is NaN, and every other row is unaffected, bit for bit."""
  M = 5000
  if mode == 'fwd':
    m_, lspecs, cols = R.FWD, trunk(4, 128), 128
    d = R.make_data(m_, M, lspecs, cols, head_n=1, exact=False, seed=11)
  else:
    m_, lspecs, cols = R.BWD, bwd_trunk(4), 256
    d = R.make_data(m_, M, lspecs, cols, exact=False, seed=12)
  init = _colsum_init(d, lspecs)
  clean, _ = launch(ops, m_, M, lspecs, device_data(d, m_), cols, 1 if mode == 'fwd' else 0, colsum_init=init)
  bad = d['stream'].clone()
  for r, v in POISON.items():
    bad[r, 5 + r % 60] = v
  dd = device_data(dict(d, stream=bad), m_)
  got, layers = launch(ops, m_, M, lspecs, dd, cols, 1 if mode == 'fwd' else 0, colsum_init=init)
  rows = sorted(POISON)
  others = torch.ones(M, dtype=torch.bool, device='cuda')
  others[rows] = False
  for j in range(len(lspecs)):
    _same(got['outs'][j][others], clean['outs'][j][others], f'layer {j}: a row without a non-finite input')
    if mode == 'fwd':
      _same(got['bits'][j][others], clean['bits'][j][others], f'layer {j} mask words of the other rows')
  if mode == 'fwd':
    _same(got['head'][others], clean['head'][others], 'head of the other rows')
    assert bool(torch.isnan(got['head'][rows]).all()), 'the head of a poisoned row is not NaN'
    # layer 0 of the NaN rows: NaN wherever the pre-activation is
    assert bool(torch.isnan(got['outs'][0][3].float()).all()), 'a NaN pre-activation did not stay NaN'
    assert bool((got['bits'][0][3] == 0).all()), 'a NaN pre-activation has its mask bit set'
  _check_poisoned_rows(m_, layers, dd, got, rows)
  if mode == 'bwd':
    for j, r in R.ref_chain(m_, M, layers, dd['stream'], stored=got['outs'], colsum_init=init):
      val, bound = r['colsum']
      _classes_match(got['colsums'][j], val, f'layer {j} colsum')
      fin = torch.isfinite(val)
      G.check(got['colsums'][j][fin], val[fin], bound[fin], f'layer {j} colsum of the finite columns')
  print(f'\n[chain non-finite] {mode}: NaN / +-inf rows {rows} follow the fp64 contract; other rows bit-equal')


def test_model_non_finite_ray_both_paths():
  """One forward pass of the 8 x 256 NerfMLP (chained, MNRF_CHAIN=1, and per-layer GEMMs, MNRF_CHAIN=0) with a
  NaN ray origin: both paths give that ray a NaN colour and agree on the others."""
  from multinerf_b200 import configs, lib, models
  from model_parity import synth_rays
  lib.require_device()
  res = {}
  for chain in ('1', '0'):
    os.environ['MNRF_CHAIN'] = chain
    try:
      bundle = configs.bundle_blender_256()
      bundle.model.num_levels = 1
      bundle.model.num_nerf_samples = 64
      B = 128
      rays, rng = synth_rays(77, B, 2.0, 6.0, unit_cube=False)
      model, _ = models.construct_model(78, rays, bundle)
      rays.origins[5] = np.nan
      rend, _ = model(None, rays, 1.0, False)
      torch.cuda.synchronize()
      res[chain] = torch.as_tensor(np.asarray(rend[-1]['rgb'].cpu() if torch.is_tensor(rend[-1]['rgb'])
                                              else rend[-1]['rgb'])).double()
    finally:
      os.environ.pop('MNRF_CHAIN', None)
  for chain, rgb in res.items():
    assert bool(torch.isnan(rgb[5]).all()), f'MNRF_CHAIN={chain}: the NaN ray has a colour {rgb[5].tolist()}'
    assert bool(torch.isfinite(torch.cat([rgb[:5], rgb[6:]])).all()), f'MNRF_CHAIN={chain}: another ray is not finite'
  keep = torch.ones(res['1'].shape[0], dtype=torch.bool)
  keep[5] = False
  err = float((res['1'][keep] - res['0'][keep]).abs().max())
  assert err < 5e-3, err
  print(f'\n[chain non-finite] model: the NaN ray is NaN on both paths; other rays agree to {err:.2e}')


# ---------------------------------------------------------------------------------------------- zero and subnormal
def test_zero_and_subnormal_pre_activations(ops):
  """Columns with zero weights and a bias of +0, -0, +-2^-140, 2^-134 and 2^-126: the stored activation is the bf16
  rounding of relu(bias), the mask bit the sign of the fp32 pre-activation (set over a stored 0 for 2^-140 and
  2^-134, which round to a bf16 zero)."""
  M = 300
  lspecs = trunk(2, 128)
  d = R.make_data(R.FWD, M, lspecs, 128, head_n=1, exact=False, seed=13)
  special = [0.0, -0.0, 2.0 ** -140, -2.0 ** -140, 2.0 ** -134, 2.0 ** -126]
  for j in range(2):
    cols = torch.arange(len(special)) * 37 + j
    w = d['w'][j].clone()
    used = torch.isfinite(w.float())
    w[cols] = torch.where(used[cols], torch.zeros_like(w[cols]), w[cols])
    d['w'][j] = w
    d['bias'][j] = d['bias'][j].clone()
    d['bias'][j][cols] = torch.tensor(special)
  dd = device_data(d, R.FWD)
  got, layers = launch(ops, R.FWD, M, lspecs, dd, 128, 1)
  R.check_launch(R.FWD, M, layers, dd['stream'], got, exact=False, head_w=dd['head_w'], head_b=dd['head_b'])
  for j in range(2):
    cols = torch.arange(len(special)) * 37 + j
    o = got['outs'][j][:, cols].float().cpu()
    bits = G.unpack_bits(got['bits'][j], W)[:, cols].cpu()
    want = torch.tensor(special).clamp_min(0).to(torch.bfloat16).float()
    assert torch.equal(o, want.expand_as(o)), f'layer {j}: {o[0].tolist()} for biases {special}'
    assert torch.equal(bits, (torch.tensor(special) > 0).expand_as(bits)), f'layer {j}: bits {bits[0].tolist()}'


# ---------------------------------------------------------------------------------------------- argument checks
def _bad_descs():
  """name -> builder of (mode, m, layers, kwargs of chain_desc, desc edits) with small valid tensors otherwise."""
  from multinerf_b200 import lib as L
  dev = 'cuda'
  bf = torch.bfloat16
  x = torch.zeros(512, 512, dtype=bf, device=dev)
  w = torch.zeros(256, 512, dtype=bf, device=dev)
  b = torch.zeros(256, device=dev)
  hw = torch.zeros(4, 256, device=dev)
  mk = torch.zeros(512, 8, dtype=torch.int32, device=dev)
  cs = torch.zeros(256, device=dev)

  def f(n_stream=4, **kw):
    return dict(w=w, bias=b, n_stream=n_stream, **kw)

  S = dict(stream=x, stream_cols=256)
  F, B_ = L.CHAIN_FWD, L.CHAIN_BWD
  c = {
      'bad mode': (7, 512, [f()], S, {}),
      'no layers': (F, 512, [], S, {}),
      f'{R.MAX_LAYERS + 1} layers': (F, 512, [f()] + [f(0, n_res=4)] * R.MAX_LAYERS, S, {}),
      'width 128': (F, 512, [f()], S, {'width': 128}),
      'n_res 2': (F, 512, [f(), f(0, n_res=2)], S, {}),
      'no operand': (F, 512, [f(0)], S, {}),
      'first layer resident': (F, 512, [f(0, n_res=4)], S, {}),
      'weights misaligned': (F, 512, [dict(f(), w=w[:, 1:])], S, {}),
      'weight pitch % 8': (F, 512, [dict(f(), w=torch.zeros(256, 260, dtype=bf, device=dev)[:, :256])], S, {}),
      'weight pitch < K': (F, 512, [f(4, stream_kb0=6)], S, {}),
      'bias misaligned': (F, 512, [dict(f(), bias=b[1:])], S, {}),
      'mask pitch < 8': (F, 512, [dict(f(), maskbits=mk[:, :7].as_strided((512, 7), (7, 1)))], S, {}),
      'BWD with a bias': (B_, 512, [f()], S, {}),
      'FWD without a bias': (F, 512, [dict(w=w, n_stream=4)], S, {}),
      'FWD with colsum': (F, 512, [dict(f(), colsum=cs)], S, {}),
      'output misaligned': (F, 512, [dict(f(), out=x[:, 1:257])], S, {}),
      'output pitch < 256': (F, 512, [dict(f(), out=torch.zeros(512, 200, dtype=bf, device=dev))], S, {}),
      'streamed columns past the tensor': (F, 512, [f(4, stream_col0=64)], S, {}),
      'stream_col0 % 64': (F, 512, [f(2, stream_col0=32)], S, {}),
      'negative stream_col0': (F, 512, [f(4, stream_col0=-64)], S, {}),
      'negative stream_kb0': (F, 512, [f(4, stream_kb0=-1)], S, {}),
      'negative res_kb0': (F, 512, [f(), f(0, n_res=4, res_kb0=-2)], S, {}),
      'stream misaligned': (F, 512, [f()], dict(stream=x[:, 1:257], stream_cols=256), {}),
      'stream_cols % 64': (F, 512, [f(1)], dict(stream=x, stream_cols=96), {}),
      'stream pitch < stream_cols': (F, 512, [f(4, stream_col0=256)],
                                     dict(stream=torch.zeros(512, 256, dtype=bf, device=dev), stream_cols=512), {}),
      'no stream': (F, 512, [f()], dict(stream_cols=256), {}),
      'head in BWD': (B_, 512, [dict(w=w, n_stream=4)], dict(S, head_w=hw[0], head_out=cs), {}),
      'head_n 2': (F, 512, [f()], dict(S, head_w=hw[:2].reshape(-1), head_out=torch.zeros(512, 2, device=dev),
                                       head_n=2), {}),
      'head weights misaligned': (F, 512, [f()], dict(S, head_w=hw.reshape(-1)[1:257], head_out=torch.zeros(512, device=dev)), {}),
      'negative m': (F, -5, [f()], S, {}),
      'm past the int32 rows': (F, 2 ** 31 - 127, [f()], S, {}),
  }
  return c


BAD = ['bad mode', 'no layers', f'{R.MAX_LAYERS + 1} layers', 'width 128', 'n_res 2', 'no operand',
       'first layer resident', 'weights misaligned', 'weight pitch % 8', 'weight pitch < K', 'bias misaligned',
       'mask pitch < 8', 'BWD with a bias', 'FWD without a bias', 'FWD with colsum', 'output misaligned',
       'output pitch < 256', 'streamed columns past the tensor', 'stream_col0 % 64', 'negative stream_col0',
       'negative stream_kb0', 'negative res_kb0', 'stream misaligned', 'stream_cols % 64',
       'stream pitch < stream_cols', 'no stream', 'head in BWD', 'head_n 2', 'head weights misaligned', 'negative m',
       'm past the int32 rows']


@pytest.mark.parametrize('name', BAD)
def test_rejected_descriptor(ops, name):
  """Each argument check of mnrf_mlp_chain raises MnrfError and leaves a sentinel-filled output untouched.  (The
  row-count limit is checked on the host first: no buffer of 2^31 rows is needed.)"""
  from multinerf_b200 import lib as L
  mode, m, layers, kw, edits = _bad_descs()[name]
  o, ob = _out((512, W), torch.bfloat16, 16, 8)
  layers = [dict(ly) for ly in layers]
  for ly in layers:
    ly.setdefault('out', o)
  # more layers than the descriptor holds: num_layers set past them
  d, fl = ops.chain_desc(mode, m, layers[:R.MAX_LAYERS], **kw)
  if len(layers) > R.MAX_LAYERS:
    d.num_layers = len(layers)
  for k, v in edits.items():
    setattr(d, k, v)
  before = ob.clone()
  with pytest.raises(L.MnrfError):
    ops.mlp_chain((d, fl))
  torch.cuda.synchronize()
  assert torch.equal(_bits(ob), _bits(before)), f'{name}: the refused call wrote its output'
