"""Ray casting + IPE encoder (mnrf_encode, all three kernels) and mnrf_viewdir_enc (both kernels) against the fp64
reference of tests/encode_ref.py, on every launch plan, sine tier, ray-distance function and output buffer.  Needs an
H100.

Every case checks, element by element and with no outlier fraction: tdist, the fp32 features and the bf16 features of
the fast kernel against their bounds; the feature rows the tangent kernel writes against the same bounds, and against
the fast kernel's rows within twice the bound; zero pad columns; `feat`, `tfeat`, `feat_f32` and `tdist_out` as views
between sentinel pads, which must survive; the same bits of `feat` with and without the optional outputs.  Elements
whose bound says nothing (encode_ref.VACUOUS) are counted, printed per degree, and held to the case's floor on the
checked share.  Each case asserts through encode_ref.plan / tiers that it reaches the launch plan and the sine tiers it
was written for, and prints the plan, the passes per tier and the worst err / bound per degree.

The tangent kernel's tangent rows (d feature / d mean, three streams at rows dir * M + m of tfeat) are checked the same
way against encode_ref.tangent_reference on every `tangent` case, per stream and degree, with their own floor
(`tfloor`, default `floor`): elements are vacuous where the feature is, and on samples within rounding of |x| = 1,
where the contraction's d lift_var jumps.  'unit-shell' puts samples within 2e-6 of that sphere; 'cos-straddle' puts
y below fl32(100 pi) and y + pi/2 above it, so the two halves reduce differently; it shows the bounds sound there
but cannot tell the two reductions apart, whose difference lies far below a bf16 half-ulp.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import encode_ref as ER

pytestmark = pytest.mark.gpu

SENTINEL = -7.25e33
PAD = 37                    # floats of guard on both sides of feat_f32 and tdist_out

_360 = dict(K=21, max_deg=12, raydist='reciprocal', near=0.2, far=1e6, contract=True)
# name: overrides of DEFAULT.  `rays` None: 32 * SMs + 37, one warp per ray.  `reach`: what the plan and the tiers
# must show (checked by reach()).  `floor`: least share of elements with a bound below encode_ref.VACUOUS, set from
# the fp32 emulation of tests/test_encode_reference_cpu.py.
DEFAULT = dict(K=9, min_deg=0, max_deg=8, raydist=None, near=2.0, far=6.0, contract=False, shape='cone', S=32,
               rays=96, no_int=False, origins='unit', radii=(5e-4, 1e-3), sdist='uniform', reach=(), floor=0.98,
               tangent=True)
CASES = {
    '360': dict(_360, reach=('G3', 'nseg>1'), floor=0.95),
    '360-many-rays': dict(_360, max_deg=4, rays=None, reach=('G3', 'nseg1'), tangent=False),
    'blender': dict(K=3, max_deg=16, reach=('G10', 'tier2')),
    'llff': dict(K=3, max_deg=16, near=0.0, far=1.0, shape='cylinder', reach=('G10',)),
    'K9': dict(max_deg=16, reach=('G7', 'tier2')),
    'S1': dict(S=1, reach=('nseg1',)),
    'S5-K9': dict(S=5, reach=('nseg1', 'padded')),
    'S33-K21': dict(_360, max_deg=6, S=33, reach=('short-last',)),
    'S50-K9': dict(S=50, reach=('S%G', 'short-last')),
    'S128': dict(S=128, rays=40),
    'S256': dict(_360, max_deg=4, S=256, rays=24, tangent=False),
    'K3': dict(K=3, S=16, max_deg=6, reach=('G10',)),
    'K32': dict(K=32, S=16, max_deg=6, reach=('G1',)),
    'K33': dict(K=33, S=16, max_deg=6, reach=('G16', 'padded')),
    'min-deg-2': dict(min_deg=2, max_deg=10),
    'log': dict(raydist='log', near=0.5, far=20.0, S=24),
    'exp': dict(raydist='exp', near=0.1, far=3.0, S=24),
    'sqrt': dict(raydist='sqrt', near=0.1, far=9.0, S=24),
    'square': dict(raydist='square', near=0.5, far=5.0, S=24),
    'piecewise': dict(raydist='piecewise', near=0.2, far=50.0, S=24, contract=True),
    'no-integration': dict(max_deg=10, no_int=True),
    'huge-uncontracted': dict(max_deg=16, origins='huge', reach=('tier3',), floor=0.9),
    'mixed-warp': dict(K=3, max_deg=16, near=0.0, far=1.0, shape='cylinder', origins='mixed',
                       reach=('mixed', 'zero', 'padded', 'tier1', 'tier2', 'tier3'), floor=0.95),
    'far-contracted': dict(contract=True, raydist='reciprocal', near=0.2, far=1e6, S=16, rays=48, radii=(0.01, 0.03),
                           sdist='far'),
    # the contraction with cylinders, and without integration (d lift_var = 0), for the tangent rows
    'cylinder-contracted': dict(contract=True, shape='cylinder', near=0.05, far=4.0, radii=(0.01, 0.03), S=16, rays=48),
    'no-integration-contracted': dict(contract=True, no_int=True, near=0.05, far=4.0, radii=(0.01, 0.03), S=16,
                                      rays=48),
    # tangent rows: samples within 1e-6 of |x| = 1, where d lift_var jumps (a share of them within rounding of it)
    'unit-shell': dict(contract=True, near=0.0, far=2.0, origins='zero', sdist='shell', S=16, rays=48, tfloor=0.75,
                       reach=('shell',)),
    # degrees whose y + pi/2 crosses fl32(100 pi) while y stays below it: the two halves reduce differently.  This
    # shows the bounds sound there; it cannot tell the reductions apart (reducing y for the cosine half instead moves
    # the argument by 5.9e-6, some 1e-3 of a tangent element at degree 8, far below its bf16 half-ulp)
    'cos-straddle': dict(K=3, max_deg=12, origins='straddle', reach=('straddle',)),
}


def case(name):
  return dict(DEFAULT, **CASES[name])


def basis_of(K, rng):
  """The two polyhedral bases the models use, or any [K, 3] unit vectors."""
  from multinerf_b200 import geopoly
  if K in (3, 21):
    b = geopoly.generate_basis('octahedron', 1) if K == 3 else geopoly.generate_basis('icosahedron', 2)
    assert b.shape == (K, 3)
    return torch.tensor(b, dtype=torch.float32)
  b = rng.normal(size=(K, 3))
  return torch.tensor(b / np.linalg.norm(b, axis=-1, keepdims=True), dtype=torch.float32)


def make_inputs(name, num_sms, rays=None):
  """(positional fp32 CPU inputs of ops.encode, keyword arguments) of a case; `rays` overrides the case's count."""
  c = case(name)
  rng = np.random.default_rng(sum(name.encode()))
  B = rays or c['rays'] or 32 * num_sms + 37
  S = c['S']
  basis = basis_of(c['K'], rng)
  o = rng.uniform(-1, 1, (B, 3))
  d = rng.normal(size=(B, 3))
  d = d / np.linalg.norm(d, axis=-1, keepdims=True) * rng.uniform(0.8, 1.2, (B, 1))
  if c['origins'] == 'huge':
    o = o * 1.2e4
  elif c['origins'] == 'mixed':
    # one ray in eight 1e4 out along a basis direction, so that its lanes on the directions across it stay small;
    # its neighbours at 1e-3; ray 1 degenerate (origin 0, direction 0): every lifted mean is exactly 0
    o = o * 1e-3
    o[::8] = 1e4 * basis[0].numpy()
    o[1], d[1] = 0, 0
  elif c['origins'] == 'zero':
    o = o * 0
  elif c['origins'] == 'straddle':
    # lm_0 2^8 = fl32(100 pi) - 0.8 +- 0.6 along basis[0]; directions 1e-4 long keep the samples there
    o = basis[0].numpy() * (ER.T32 - 0.8) / 256 * rng.uniform(1 - 2e-3, 1 + 2e-3, (B, 1))
    d = d * 1e-4
  radii = rng.uniform(*c['radii'], B)
  if c['sdist'] == 'shell':
    # t = 2 s: the frustum means lie at |x| = 1 +- 2e-6 (o = 0)
    sdist = np.sort(0.5 / np.linalg.norm(d, axis=-1, keepdims=True) * (1 + rng.uniform(-2e-6, 2e-6, (B, S + 1))), -1)
  elif c['sdist'] == 'far':
    sdist = np.sort(1 - 10 ** rng.uniform(-6.5, 0, (B, S + 1)), -1)
  else:
    sdist = np.sort(rng.uniform(0, 1, (B, S + 1)), -1)
    sdist[:, 0], sdist[:, -1] = 0, 1
  t = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float32)
  pos = (t(sdist), t(o), t(d), t(radii), torch.full((B,), c['near']), torch.full((B,), c['far']), basis)
  kw = dict(min_deg=c['min_deg'], max_deg=c['max_deg'], raydist_fn=c['raydist'], ray_shape=c['shape'],
            warp_contract=c['contract'], disable_integration=c['no_int'])
  return pos, kw


def straddles(ref, min_deg, max_deg):
  """[.., L, K] lifted means whose y = lm 2^l lies below fl32(100 pi) while y + pi/2 does not."""
  y = ref.lm[..., None, :].abs() * 2.0 ** torch.arange(min_deg, max_deg, dtype=torch.float64)[:, None]
  return (y < ER.T32) & (y + 0.5 * np.pi >= ER.T32)


def shell(ref):
  """[3] bool: samples within rounding of |x| = 1 (vacuous tangent rows), and samples with a checked bound within
  1e-6 of it inside and outside."""
  if not hasattr(ref, 'unsure'):
    return torch.zeros(3, dtype=torch.bool)
  d = ref.xnorm - 1
  return torch.stack([ref.unsure.any(), (~ref.unsure & (d < 0) & (d >= -1e-6)).any(),
                      (~ref.unsure & (d > 0) & (d <= 1e-6)).any()])


def reach(name, p, tr, S, ref=None):
  """The case got the launch plan and the sine tiers it was written for."""
  c = case(name)
  for what in c['reach']:
    ok = {'straddle': ref is not None and bool(straddles(ref, c['min_deg'], c['max_deg']).any()),
          'shell': ref is not None and bool(shell(ref).all()),
          'nseg1': p.nseg == 1, 'nseg>1': p.nseg > 1, 'short-last': p.nseg > 1 and p.nseg * p.seg_len != S, 'S%G': S % p.G != 0,
          'padded': bool(tr.padded.any()), 'mixed': bool((tr.mixed & ~tr.unsure).any()),
          'zero': bool(tr.zero.any()), 'tier1': tr.count(1) > 0, 'tier2': tr.count(2) > 0,
          'tier3': int(((tr.rest == 3) & ~tr.unsure).sum()) > 0}.get(what)
    if ok is None:
      ok = p.G == int(what[1:])
    assert ok, f'{name}: does not reach {what} (G {p.G} nseg {p.nseg} seg_len {p.seg_len})'


def report(name, label, got, ref_val, bound, vacuous, K, L):
  """Every non-vacuous element within its bound; returns the printed line with the worst ratio per degree."""
  ratio = (got.double() - ref_val).abs() / bound
  ratio = torch.where(vacuous, torch.zeros_like(ratio), ratio)
  deg = ER.degree_of(K, L)
  worst = [float(ratio[..., deg == l].max()) for l in range(L)]
  vac = [float(vacuous[..., deg == l].double().mean()) for l in range(L)]
  line = (f'{name} {label}: worst err/bound per degree ' + ' '.join(f'{w:.2f}' for w in worst) +
          ' | vacuous share per degree ' + ' '.join(f'{v:.2f}' for v in vac))
  bad = ratio > 1
  if bad.any():
    i = tuple(int(v) for v in np.unravel_index(int(ratio.argmax()), ratio.shape))
    raise AssertionError(f'{line}\n{int(bad.sum())} of {bad.numel()} elements outside their bound; worst at '
                         f'[ray, sample, column] {i} (degree {int(deg[i[2]])}): got {float(got[i])!r}, reference '
                         f'{float(ref_val[i])!r}, bound {float(bound[i]):.3e}')
  return line


@pytest.fixture(scope='module')
def ops():
  from multinerf_b200 import lib, ops as _ops
  lib.require_device()
  return _ops


def _guarded_rows(rows, cols, ld, dtype=torch.bfloat16):
  """A [rows, cols] view with row stride ld into a sentinel-filled buffer with 3 rows before and after."""
  buf = torch.full((rows + 6, ld), 7.0, dtype=dtype, device='cuda')
  return buf[3:3 + rows, :cols], buf


def _rows_intact(buf, rows, cols):
  return bool((buf[:3] == 7).all() and (buf[3 + rows:] == 7).all() and (buf[3:3 + rows, cols:] == 7).all())


@pytest.mark.parametrize('name', list(CASES))
def test_encode_case(ops, name):
  from multinerf_b200 import lib as L
  lib = L.load()
  sms = lib.mnrf_num_sms()
  c = case(name)
  pos, kw = make_inputs(name, sms)
  dev = [t.cuda() for t in pos]
  B, S, K, Ld = pos[0].shape[0], c['S'], c['K'], c['max_deg'] - c['min_deg']
  F = 2 * K * Ld
  cols = (F + 63) // 64 * 64
  M = B * S

  feat, f32, tdist = ops.encode(*dev, **kw, want_f32=True, want_tdist=True)
  assert feat.shape == (M, cols)
  ref = ER.reference(*pos, **kw, tdist=tdist, tangent=c['tangent'])
  p = ER.plan(B, S, K, sms)
  tr = ER.tiers(ref, p, c['min_deg'], c['max_deg'])
  print(f'\n{name}: rays {B} S {S} K {K} L {Ld} | plan G {p.G} nseg {p.nseg} seg_len {p.seg_len} | passes per tier '
        f'1: {tr.count(1)} 2: {tr.count(2)} 3: {tr.count(3)} (unsure {int(tr.unsure.sum())})')
  reach(name, p, tr, S, ref)

  rt = (tdist.cpu().double() - ref.tdist).abs() / ref.tdist_bound
  assert float(rt.max()) <= 1, (name, 'tdist', float(rt.max()), int(rt.argmax()))
  print(f'{name} tdist: worst err/bound {float(rt.max()):.2f}')

  checked = 1 - float(ref.vacuous.double().mean())
  assert checked >= c['floor'], f'{name}: only {checked:.3f} of the elements have a bound that says anything'
  got32 = f32.view(B, S, F).cpu()
  gotbf = feat.view(B, S, cols).float().cpu()
  print(report(name, 'fp32', got32, ref.feat, ref.bound, ref.vacuous, K, Ld))
  print(report(name, 'bf16', gotbf[..., :F], ref.feat, ref.bound_bf16, ref.vacuous, K, Ld))
  assert (got32.to(torch.bfloat16).float() == gotbf[..., :F]).all(), 'bf16 rows are not the rounded fp32 rows'
  assert (gotbf[..., F:] == 0).all(), 'pad columns'

  # the same bits without the optional outputs, into a view of a wider buffer whose surroundings must survive
  view, buf = _guarded_rows(M, cols, cols + 24)
  ops.encode(*dev, **kw, feat=view, feat_cols=cols)
  assert _rows_intact(buf, M, cols), 'wrote outside feat'
  assert torch.equal(view.contiguous().view(torch.int16), feat.view(torch.int16)), 'feat changes with the optional outputs'

  # feat_f32 and tdist_out between sentinel floats, through the C ABI
  fbuf = torch.full((M * F + 2 * PAD,), SENTINEL, device='cuda')
  tbuf = torch.full((B * (S + 1) + 2 * PAD,), SENTINEL, device='cuda')
  feat2 = torch.empty(M, cols, dtype=torch.bfloat16, device='cuda')
  d = L.EncodeDesc(B, S, L.RAYDIST[kw['raydist_fn']], L.RAY_SHAPE[kw['ray_shape']], int(kw['warp_contract']),
                   int(kw['disable_integration']), K, kw['min_deg'], kw['max_deg'], cols, cols)
  L.check(lib.mnrf_encode(C.byref(d), *[L.ptr(t) for t in dev], L.ptr(feat2), L.ptr(fbuf[PAD:]), L.ptr(tbuf[PAD:]),
                          None, 0, L.stream_ptr()))
  for b, inner, what in ((fbuf, f32.view(-1), 'feat_f32'), (tbuf, tdist.view(-1), 'tdist_out')):
    assert (b[:PAD] == SENTINEL).all() and (b[-PAD:] == SENTINEL).all(), f'wrote outside {what}'
    assert torch.equal(b[PAD:-PAD], inner), what
  assert torch.equal(feat2.view(torch.int16), feat.view(torch.int16))

  # the feature rows of the tangent kernel (encode_kernel<contract>): other sine and exp forms, the same bounds
  if c['tangent']:
    tview, tb = _guarded_rows(3 * M, cols, cols + 8)
    fview, fb = _guarded_rows(M, cols, cols + 16)
    ops.encode(*dev, **kw, feat=fview, feat_cols=cols, tfeat=tview)
    assert _rows_intact(tb, 3 * M, cols), 'wrote outside tfeat'
    assert _rows_intact(fb, M, cols), 'wrote outside feat (tangent kernel)'
    gott = fview.float().cpu().view(B, S, cols)
    print(report(name, 'bf16, tangent kernel', gott[..., :F], ref.feat, ref.bound_bf16, ref.vacuous, K, Ld))
    assert (gott[..., F:] == 0).all() and (tview.float()[:, F:] == 0).all(), 'pad columns (tangent kernel)'
    cross = (gott[..., :F] - gotbf[..., :F]).abs().double() / (2 * ref.bound_bf16)
    cross = torch.where(ref.vacuous, torch.zeros_like(cross), cross)
    assert float(cross.max()) <= 1, (name, 'tangent kernel against fast kernel', float(cross.max()))
    print(f'{name} tangent kernel against fast kernel: worst difference / (2 bound) {float(cross.max()):.2f}, '
          f'{float((gott[..., :F] == gotbf[..., :F]).double().mean()):.4f} of the elements bit-equal')
    # the tangent rows d feature / d mean_dir: stream dir at rows dir * M + m
    tchecked = 1 - float(ref.tangent_vacuous.double().mean())
    tfloor = c.get('tfloor', c['floor'])
    assert tchecked >= tfloor, f'{name}: only {tchecked:.3f} of the tangent elements have a bound that says anything'
    gtan = tview.float().cpu().view(3, B, S, cols)[..., :F]
    for a in range(3):
      print(report(name, f'tangent stream {a}', gtan[a], ref.tangent[a], ref.tangent_bound_bf16[a],
                   ref.tangent_vacuous[a], K, Ld))
    print(f'{name} tangent rows: checked share {tchecked:.3f} (floor {tfloor})')


def test_encode_refusals(ops):
  """Argument checks that return before any launch."""
  from multinerf_b200 import lib as L
  pos, kw = make_inputs('S256', 1)
  dev = [t.cuda() for t in pos]
  with pytest.raises(ValueError):
    ops.encode(*dev, **dict(kw, ray_shape='sphere'))
  M, cols = pos[0].shape[0] * 256, 192
  tfeat = torch.full((3 * M, cols), 7.0, dtype=torch.bfloat16, device='cuda')
  feat = torch.full((M, cols), 7.0, dtype=torch.bfloat16, device='cuda')
  with pytest.raises(L.MnrfError, match='shared memory .* too large'):      # tangent kernel, S = 256
    ops.encode(*dev, **kw, feat=feat, feat_cols=cols, tfeat=tfeat)
  with pytest.raises(L.MnrfError, match='take no feat_f32'):
    ops.encode(*dev, **kw, feat=feat, feat_cols=cols, tfeat=tfeat, want_f32=True)
  big = torch.sort(torch.rand(4, 513), -1)[0].cuda()                          # fast kernel, S = 512
  with pytest.raises(L.MnrfError, match='shared memory .* too large'):
    ops.encode(big, *[t[:4].contiguous() for t in dev[1:6]], dev[6], **kw)
  assert (feat == 7).all() and (tfeat == 7).all(), 'a refused call wrote its output'


def _viewdir_enc(ops, deg, S):
  rng = np.random.default_rng(3)
  B, W = 33, 3 + 6 * deg
  v = rng.normal(size=(B, 3)).astype(np.float32)
  v /= np.linalg.norm(v, axis=-1, keepdims=True)
  v = torch.tensor(v)
  enc, bound = ER.pos_enc_reference(v, deg)
  outs = []
  for col0, col_end, ld in ((256, 320, 320), (3, 3 + W, W + 8)):
    out = torch.full((B * S, ld), 7.0, dtype=torch.bfloat16, device='cuda')
    ops.viewdir_enc(v.cuda(), S, deg, out, col0, col_end)
    got = out.float().cpu().view(B, S, ld)
    r = (got[:, :, col0:col0 + W].double() - enc[:, None, :]).abs() / bound[:, None, :]
    assert float(r.max()) <= 1, (deg, S, col0, float(r.max()))
    assert (got[:, :, col0 + W:col_end] == 0).all(), 'columns past 3 + 6 deg'
    assert (got[:, :, :col0] == 7).all() and (got[:, :, col_end:] == 7).all(), 'columns outside the slab'
    print(f'viewdir_enc deg {deg} S {S} slab [{col0}, {col_end}) ld {ld}: worst err/bound {float(r.max()):.2f}')
    outs.append(got[:, :, col0:col0 + W])
  assert torch.equal(outs[0], outs[1]), (deg, S, 'the two kernels differ')


def test_viewdir_enc_both_kernels(ops):
  """The 16-byte row kernel (aligned slab) and the element kernel (col0 = 3, the exact width), deg in {1, 4} and S in
  {1, 5}: values within their bound, zeros past 3 + 6 deg, nothing outside the slab, the two kernels bit-equal."""
  for deg in (1, 4):
    for S in (1, 5):
      _viewdir_enc(ops, deg, S)
