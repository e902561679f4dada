"""The ping-pong schedule of the tensor-core Dense-layer GEMM (gemm_tc_pingpong_kernel in csrc/gemm_tc.cu).

FWD and DGRAD with a staged store, N % 128 == 0, ReLU or no activation and no column sums run each consumer
warpgroup on whole 128 x 128 sub-tiles, alternating.  Every instance of that schedule -- FWD with and without mask
bits, DGRAD with no mask, a bf16 mask, mask bits by TMA and mask bits by the epilogue's loads, at tiles of 128 and
256 columns (one and two sub-tiles per tile) -- runs against the fp64 bound of tests/gemm_ref.py with the padding
and NaN checks of test_gpu_gemm_matrix.py, at three launch shapes:
  one    one tile per CTA and fewer tiles than SMs (at 128 columns the second warpgroup has nothing to do);
  odd    an odd number of sub-tiles on every CTA;
  ragged several tiles per CTA and a ragged last row tile.
test_cases_hit_their_instance asks the library (mnrf_gemm_plan) that each case runs what it claims.  The parity tests
compare the schedule bit for bit with gemm_tc_kernel on the same data: the output two elements off its alignment
(register store), and DGRAD with column sums on.  Needs an H100 (test_cases_hit_their_instance does not).
"""
import pytest
import torch

from test_gpu_gemm_matrix import _bits, case, case_id, layout, plan, run, verify

SMS = 132                # the H100's SMs; without a device the library plans for 132 as well


def _cases():
  out = []
  for bn in (128, 256):
    # odd: 3 tiles on every CTA, so at 128 columns an odd number of sub-tiles and warpgroup 0 runs the last
    shapes = {'one': (128 * 40 + 1, bn), 'odd': (128 * SMS, 3 * bn), 'ragged': (38000, 1024 if bn == 256 else 640)}
    for kind, (m, n) in shapes.items():
      for bits in (False, True):
        out.append((kind, bn, case('fwd', m, n, 192, act='relu', bits=bits)))
      for j, mask in enumerate(('none', 'bf16', 'bits', 'bits_odd')):
        out.append((kind, bn, case('dgrad', m, n, (192, 64, 1024, 128)[j], mask=mask, rowv=True, addend=True)))
    # mask_mod: mask rows = M / 3, a multiple of 128 (mask bits by TMA) and not (the epilogue's loads)
    for m3 in (384, 200):
      for mask in ('bits', 'bits_odd'):
        out.append(('mask_mod', bn, case('dgrad', 3 * m3, bn, 128, mask=mask, rep=3, rowv=m3 == 384,
                                         addend=m3 == 200)))
  return out


CASES = _cases()


def _tiles_per_cta(p):
  return [len(range(b, p['tiles'], p['grid'])) for b in range(p['grid'])]


def test_cases_hit_their_instance():
  """Each case runs the ping-pong schedule at its tile width and mask source, in the launch shape it claims; every
  instance of the schedule has a case of each shape."""
  from multinerf_b200 import ops as ops_mod
  seen = {}
  for kind, bn, c in CASES:
    v, _ = layout(c, 'cpu', fill=False)
    p = plan(ops_mod, c, v)
    assert p['pingpong'] == 1 and p['block_n'] == bn and p['staged'] == 1, (case_id(c), p)
    if c['mask'] in ('bits', 'bits_odd'):
      assert p['mask_tma'] == (c['mask'] == 'bits' and (not c['rep'] or (c['M'] // c['rep']) % 128 == 0)), case_id(c)
    counts = _tiles_per_cta(p)
    if kind == 'one':
      assert p['tiles'] < SMS and set(counts) == {1}, (case_id(c), p)
    elif kind == 'odd':
      assert all(t % 2 == 1 for t in counts), (case_id(c), p)
    elif kind == 'ragged':
      assert c['M'] % 128 and min(counts) > 1, (case_id(c), p)
    src = ('bits_tma' if p['mask_tma'] else 'bits_ldg') if c['mask'] in ('bits', 'bits_odd') else c['mask']
    seen.setdefault((c['mode'], bn, c['bits'], src), set()).add(kind)
  for inst, kinds in seen.items():
    assert {'one', 'odd', 'ragged'} <= kinds, (inst, kinds)


@pytest.fixture(scope='module')
def ops():
  from multinerf_b200 import lib, ops as _ops
  lib.require_device()
  return _ops


@pytest.mark.gpu
@pytest.mark.parametrize('kind,bn,c', CASES, ids=[f'{k}-bn{bn}-{case_id(c)}' for k, bn, c in CASES])
def test_pingpong_case(ops, kind, bn, c):
  v, bufs, init = run(ops, c, seed=c['M'] + 7 * c['N'] + c['K'])
  worst = verify(c, v, bufs, init)
  print(f'\n[pingpong err/bound] {kind} bn={bn} {case_id(c)}: ' + ' '.join(f'{k}={x:.3g}' for k, x in worst.items()))


# (ping-pong case, variant on gemm_tc_kernel, outputs compared bitwise): the NerfMLP shapes -- FWD of layer 0
# (K = 512), of a 1024-wide layer and of the skip layer (K = 1536); DGRAD of a 1024-wide layer with mask bits, and of
# the bottleneck (N = 1024, K = 256) with mask bits and the rank-1 term -- and a 256-wide ragged one
PARITY = []
for k in (512, 1024, 1536):
  PARITY.append((case('fwd', 5000, 1024, k, act='relu', bits=True), dict(store='reg2'), ('out', 'maskbits')))
PARITY.append((case('fwd', 38000, 256, 192, act='none'), dict(store='reg2'), ('out',)))
for k, rowv in ((1024, False), (256, True)):
  PARITY.append((case('dgrad', 5000, 1024, k, mask='bits', rowv=rowv), dict(store='reg2'), ('out',)))
  PARITY.append((case('dgrad', 5000, 1024, k, mask='bits', rowv=rowv), dict(colsum=True), ('out',)))
PARITY.append((case('dgrad', 38000, 256, 192, mask='bits_odd', rowv=True, addend=True), dict(store='reg2'), ('out',)))
PARITY.append((case('dgrad', 38000, 256, 192, mask='bf16', addend=True), dict(colsum=True), ('out',)))


def test_parity_variants_leave_the_schedule():
  from multinerf_b200 import ops as ops_mod
  for base, var, _ in PARITY:
    for c, want in ((base, 1), (dict(base, **var), 0)):
      v, _ = layout(c, 'cpu', fill=False)
      assert plan(ops_mod, c, v)['pingpong'] == want, case_id(c)


@pytest.mark.gpu
@pytest.mark.parametrize('base,var,names', PARITY, ids=[f'{case_id(b)}-vs-{list(v)[0]}' for b, v, _ in PARITY])
def test_same_bits_as_gemm_tc_kernel(ops, base, var, names):
  seed = 3 + base['M'] + base['K']
  v0, bufs, init = run(ops, base, seed)
  verify(base, v0, bufs, init)
  c = dict(base, **var)
  v, bufs, init = run(ops, c, seed)
  verify(c, v, bufs, init)
  for name in names:
    assert torch.equal(_bits(v[name]), _bits(v0[name])), f'{name} of {case_id(c)} differs from the ping-pong schedule'
