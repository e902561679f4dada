"""tests/refdir_ref.py is sound and sensitive, and the host refuses what the kernels cannot do.  CPU only.

Soundness: `Emul` runs refdir_ref.walk -- the kernels' arithmetic -- in numpy fp32, once with every a * b + c fused
and once with none, with expf / exp2f / sinf / cosf / log1pf moved by their documented error in each direction; the
slab and head-slab stores round to bf16, the zero fill runs to col_end, and the loss statistics go through the
kernels' reduction (per-thread sums over the grid-stride iterations, a 32-lane xor butterfly, one add per warp in a
shuffled order).  Every output lands inside its bound on every case of tests/test_gpu_refdir_fp64.py.

Sensitivity: each plausible kernel bug, applied to the emulation, breaks a non-vacuous bound in at least one case.

Agreement: in float32 the oracle chain reproduces the fp32 oracle; the running-error walk reproduces the oracle's fp64
values; gradcheck passes with each optional input switched on; plan() equals a transcription of the host code.

Refusals: the four entry points, called through ctypes with fake non-null addresses, return an error before any
launch.  They run only where no CUDA device is visible, so that a missing check can never launch.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import refdir_ref as RR
from test_gpu_refdir_fp64 import CASES, DEFAULT, case, enc_width, make_inputs, sweep

F = np.float32
SMS = 132
MCPU = 96


class Emul:
  """The walk's backend of the emulation: numpy fp32, contraction on or off, library functions moved by dirn."""

  def __init__(self, fused, dirn):
    self.fused, self.dirn = fused, dirn

  def inp(self, x):
    return np.asarray(x.detach().cpu().numpy() if torch.is_tensor(x) else x, F)

  def coef(self, c32, c64):
    return self.inp(c32)

  def imul(self, k, x):
    return self.inp(torch.as_tensor(k).float()) * x

  def mask(self, m):
    return m.numpy()

  def cst(self, v64, v32):
    return F(v32)

  def zeros(self, shape):
    return np.zeros(shape, F)

  def fma(self, a, b, c):
    if self.fused:
      return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F)
    return np.asarray(np.asarray(a, F) * np.asarray(b, F), F) + np.asarray(c, F)

  def scale(self, x, p):
    return x * F(p)

  def sqrt(self, x):
    return np.sqrt(x)

  def _lib(self, name, v64):
    return (v64 * (1 + self.dirn * (2 * RR.ULP[name] - 1) * RR.U)).astype(F)

  def exp(self, x):
    with np.errstate(over='ignore'):
      return self._lib('exp', np.exp(np.asarray(x, np.float64)))

  def exp2(self, l):
    return self._lib('exp2', np.float64(2.0 ** l))

  def log1p(self, x):
    return self._lib('log1p', np.log1p(np.asarray(x, np.float64)))

  def sin(self, x):
    return self._lib('sin', np.sin(np.asarray(x, np.float64)))

  def cos(self, x):
    return self._lib('cos', np.cos(np.asarray(x, np.float64)))

  def fmax0(self, x):
    return np.maximum(x, F(0))

  def fmin0(self, x):
    return np.minimum(x, F(0))

  def maxc(self, x, c):
    return np.maximum(x, F(c))

  def abs(self, x):
    return np.abs(x)

  def where(self, c, a, b):
    return np.where(c, a, b).astype(F)

  def col(self, x):
    return x[..., None]

  def cat(self, xs):
    return np.concatenate(xs, -1)

  def clamped(self, g):
    sq = RR._dot(self, g, g)
    c = ~(sq > F(RR.EPS))
    return c, np.zeros_like(c)

  def orient_add(self, p, t_scale, v, a):
    return np.where(p < 0, self.fma(t_scale * p, -v, a), a).astype(F)


def _bf(a):
  return torch.from_numpy(np.ascontiguousarray(a, F)).to(torch.bfloat16).float()


def _reduce(terms, M, num_sms, rng):
  """stats[i] += terms as the kernels sum them: per thread over the grid-stride iterations, a 32-lane xor butterfly,
  one add per warp with a nonzero sum, in a shuffled order."""
  p = RR.plan(M, num_sms)
  t = np.zeros(p.iters * p.threads, F)
  t[:M] = terms
  acc = np.zeros(p.threads, F)
  for j in range(p.iters):
    acc = acc + t[j * p.threads:(j + 1) * p.threads]
  lanes = acc.reshape(-1, 32)
  idx = np.arange(32)
  for o in (16, 8, 4, 2, 1):
    lanes = lanes + lanes[:, idx ^ o]
  total = F(0)
  for w in rng.permutation(lanes.shape[0]):
    if lanes[w, 0] != 0:
      total = F(total + lanes[w, 0])
  return total


def emulate(x, f, fused=True, dirn=1, mut=None, num_sms=SMS):
  """Every output of mnrf_refdir_fwd / _bwd as fp32 (slabs as bf16 values) from the numpy emulation."""
  b = Emul(fused, dirn)
  M = x.v.shape[0]
  W = f['col_end'] - f['col0']
  fw = RR.walk(b, x, f, mut=mut)
  out = {}
  if f['use_pred_normals']:
    out['normals_pred'] = torch.tensor(np.stack(fw.p, -1))
  if f['use_density_normals']:
    out['normals'] = torch.tensor(np.stack(fw.d, -1))
  if f['use_roughness']:
    out['roughness'] = torch.tensor(fw.roughness)
  out['extra_dw'] = torch.tensor(np.broadcast_to(fw.extra_dw, (M,)).copy())
  slab = np.full((M, W), 5.0, F)
  ne = fw.enc.shape[1]
  slab[:, :ne] = fw.enc
  slab[:, ne:W - 1 if mut == 'short_fill' else W] = 0
  out['slab'] = _bf(slab)
  bw = RR.walk(b, x, f, bwd=True, mut=mut)
  rng = np.random.default_rng(0)
  if f['use_pred_normals']:
    out['d_grad_pred'] = torch.tensor(np.stack(bw.d_grad_pred, -1))
  if f['use_density_normals']:
    out['d_raw_grad_density'] = torch.tensor(np.stack(bw.d_raw_grad_density, 0))
  if f['use_roughness']:
    out['d_raw_rough'] = torch.tensor(np.broadcast_to(bw.d_raw_rough, (M,)).copy())
  out['stats_or'] = float(_reduce(np.broadcast_to(bw.st_or, (M,)), M, num_sms, rng))
  out['stats_pn'] = float(_reduce(np.broadcast_to(bw.st_pn, (M,)), M, num_sms, rng))
  h = x.heads
  dif, tint = h.get('diffuse'), h.get('tint')
  if mut == 'swap_heads':
    dif, tint = tint, dif
  out['head'] = RR.head_slab(W, h.get('density'), out.get('d_grad_pred'), dif, tint, out.get('d_raw_rough'))
  return out


OUTPUTS = ('normals_pred', 'normals', 'roughness', 'extra_dw', 'slab', 'd_grad_pred', 'd_raw_rough',
           'd_raw_grad_density')


def broken(ref, got, x):
  """{output: worst err / bound over non-vacuous elements} and whether any bound is broken."""
  worst, bad = {}, False
  for k in OUTPUTS:
    if k not in got:
      continue
    refv = getattr(ref, k)
    r = (got[k].double().reshape(refv.shape) - refv).abs() / getattr(ref, k + '_bound')
    r = torch.where(getattr(ref, k + '_vacuous'), torch.zeros_like(r), r.nan_to_num(nan=math.inf))
    worst[k] = float(r.max()) if r.numel() else 0.0
    bad |= worst[k] > 1
  for k in ('stats_or', 'stats_pn'):
    worst[k] = float(abs(got[k] - float(getattr(ref, k))) / float(getattr(ref, k + '_bound')))
    bad |= worst[k] > 1
  want = RR.head_slab(got['head'].shape[1], x.heads.get('density'), got.get('d_grad_pred'), x.heads.get('diffuse'),
                      x.heads.get('tint'), got.get('d_raw_rough'))
  worst['head'] = 0.0 if torch.equal(got['head'], want) else float('inf')
  bad |= worst['head'] > 1
  return worst, bad


def inputs(name, M=MCPU, num_sms=SMS):
  c = case(name)
  if name == 'M-iter':
    M = 2 * RR.plan(10 ** 9, 1).blocks * 128 + 37           # one SM: 16 blocks, 2 grid-stride iterations
  elif c['M'] is not None:
    M = min(c['M'], M) if c['M'] > 3 else c['M']
  return c, make_inputs(c, M, sum(name.encode()))


@pytest.mark.parametrize('name', list(CASES))
def test_emulation_within_bounds(name):
  c, (x, f) = inputs(name)
  sms = 1 if name == 'M-iter' else SMS
  ref = RR.reference(x, f, num_sms=sms)
  assert ref.chain_gap < 1e-3, (name, 'the running-error walk left the oracle', ref.chain_gap)
  assert not ref.unsure.any()
  for fused in (True, False):
    for dirn in (1, -1):
      got = emulate(x, f, fused, dirn, num_sms=sms)
      worst, bad = broken(ref, got, x)
      assert not bad, (name, fused, dirn, worst)
  ne = ref.enc_width
  print(f'\n{name}: M {x.v.shape[0]} iterations {RR.plan(x.v.shape[0], sms).iters} | worst err/bound ' +
        ' '.join(f'{k} {v:.2f}' for k, v in worst.items()) +
        f' | slab vacuous {float(ref.slab_vacuous[:, :ne].double().mean()):.3f}')
  assert 1 - float(ref.slab_vacuous[:, :ne].double().mean()) >= c['floor']


def test_emulation_within_bounds_sweep():
  n = 0
  for i, over in enumerate(sweep()):
    c = dict(DEFAULT, **over)
    x, f = make_inputs(c, 40, i)
    ref = RR.reference(x, f)
    assert ref.chain_gap < 1e-3, (over, ref.chain_gap)
    worst, bad = broken(ref, emulate(x, f, fused=i % 2 == 0, dirn=1 - 2 * (i % 3 == 0)), x)
    assert not bad, (over, worst)
    n += 1
  assert n >= 100


# mutation: the cases tried, in order
MUTATIONS = {
    'sigma_full': ('kappa-sweep', 'refnerf'), 'conjugate': ('ide-deg2', 'refnerf'), 'e_late': ('ide-deg3', 'refnerf'),
    'dP_no_k': ('ide-deg3', 'refnerf'), 'drop_last_z': ('ide-deg2', 'kappa-sweep'),
    'reflect_plus': ('ide-deg2', 'pe-deg4-refl'), 'ndv_other': ('no-ndv-no-loss', 'refnerf', 'pe-deg4'),
    'project_clamped': ('refnerf', 'M127', 'ide-deg2'), 'orient_flag': ('orient-density', 'density-normals'),
    'no_sigmoid': ('ide-deg2', 'refnerf'), 'swap_heads': ('heads-all',), 'cos_minus': ('pe-deg4', 'pe-deg1'),
    'short_fill': ('ide-deg2',), 'next_weight': ('orient-only', 'prednorm-only'),
}


@pytest.mark.parametrize('mut', list(MUTATIONS))
def test_mutation_is_caught(mut):
  for name in MUTATIONS[mut]:
    c, (x, f) = inputs(name)
    ref = RR.reference(x, f)
    worst, bad = broken(ref, emulate(x, f, mut=mut), x)
    if bad:
      print(f'\n{mut}: caught by {name}: ' + ' '.join(f'{k} {v:.1f}' for k, v in worst.items() if v > 1))
      return
  raise AssertionError(f'{mut}: no case notices')


def test_fp32_oracle_and_extra_dw():
  """In float32 the reference's oracle chain is the fp32 oracle of the former kernel test; extra_dw is autograd of
  the two losses with respect to the weights; the fp64 values are the fp32 ones to fp32 accuracy."""
  from oracle import o_coord
  c, (x, f) = inputs('refnerf', M=64)
  r32 = RR.oracle(x, f, dtype=torch.float32)
  v = x.v
  n_pred = -o_coord.l2_normalize(x.gp)
  n_den = -o_coord.l2_normalize(x.rgd.T)
  rough = torch.nn.functional.softplus(x.rr + f['bias'])
  enc = o_coord.generate_ide_fn(5)(o_coord.reflect(-v, n_pred), rough[:, None])
  assert torch.equal(r32['normals_pred'], n_pred) and torch.equal(r32['normals'], n_den)
  assert torch.allclose(r32['enc'][:, :-1], enc, atol=1e-6, rtol=1e-6)
  om, pm = f['orient_mult'], f['prednorm_mult']
  edw = om * torch.clamp((n_pred * -v).sum(-1), max=0.0) ** 2 + pm * (1.0 - (n_den * n_pred).sum(-1))
  assert torch.allclose(r32['extra_dw'], edw, atol=1e-9, rtol=1e-5)
  r64 = RR.oracle(x, f)
  assert float((r64['enc'] - r32['enc'].double()).abs().max()) < 1e-3


@pytest.mark.parametrize('on', ['none', 'gp', 'rgd', 'rr', 'orient', 'prednorm', 'pe'])
def test_gradcheck(on):
  """torch.autograd.gradcheck of the fp64 oracle chain on a tiny shape, each optional input switched on once."""
  c = dict(DEFAULT, M=6, S=2, deg=2, clamp_rows=False, om=0.0, pm=0.0, pred=1, dens=0, refl=1, ide=1, rough=1)
  c.update({'gp': {}, 'none': dict(refl=0, ndv=0, ide=0, rough=0, deg=1), 'rgd': dict(dens=1),
            'rr': {}, 'orient': dict(om=0.1), 'prednorm': dict(dens=1, pm=3e-4), 'pe': dict(ide=0, rough=0)}[on])
  x, f = make_inputs(c, 6, 3)
  leaves = {k: getattr(x, k).double().requires_grad_(True) for k in ('gp', 'rr', 'rgd') if getattr(x, k) is not None}

  def fn(*vals):
    y = type('X', (), {})()
    y.__dict__.update(x.__dict__)
    for k, t in zip(leaves, vals):
      setattr(y, k, t)
    o = RR.oracle(y, f, graph=True)
    return o['enc'], o['loss_terms']
  assert torch.autograd.gradcheck(fn, tuple(leaves.values()), eps=1e-6, atol=1e-6)


def host_blocks(M, num_sms):
  """The four entry points: int blocks = min((M + 127) / 128, num_sms * 16), 128 threads, grid-stride."""
  blocks = min((M + 127) // 128, num_sms * 16)
  threads = blocks * 128
  iters = 0
  m = 0
  while m < M:
    iters += 1
    m += threads
  return blocks, iters


@pytest.mark.parametrize('M,sms', [(1, 132), (127, 132), (128, 132), (129, 132), (270336, 132), (270337, 132),
                                   (524288, 132), (540709, 132), (4133, 1), (7, 114)])
def test_plan_is_the_hosts(M, sms):
  p = RR.plan(M, sms)
  assert (p.blocks, p.iters) == host_blocks(M, sms)
  assert p.threads == p.blocks * 128 and p.warps == p.blocks * 4


# ---- refusals -----------------------------------------------------------------------------------------------------

FAKE = 1 << 20            # a non-null address that is never dereferenced: every call below returns before a launch


def _lib():
  if torch.cuda.is_available():
    pytest.skip('refusals run only where no check can launch a kernel')
  from multinerf_b200 import lib as L
  try:
    return L, L.load()
  except L.MnrfError as e:
    pytest.skip(f'library not built: {e}')


def _desc(L, **kw):
  d = dict(M=64, num_samples=8, use_pred_normals=1, use_density_normals=1, use_reflections=1, use_ide=1,
           use_n_dot_v=1, use_roughness=1, deg_view=5, ide_n=36, roughness_bias=-1.0, ld=160, col0=64, col_end=160)
  d.update(kw)
  return L.RefdirDesc(*[d[k] for k, _ in L.RefdirDesc._fields_])


def _fwd(L, lib, d, **kw):
  a = dict(mat=FAKE, ml=FAKE, gp=FAKE, rr=FAKE, rgd=FAKE, vd=FAKE, npd=FAKE, nd=FAKE, rough=FAKE, slab=FAKE, om=0.0,
           pm=0.0, oop=1, edw=None)
  a.update(kw)
  return lib.mnrf_refdir_fwd(C.byref(d), a['mat'], a['ml'], a['gp'], a['rr'], a['rgd'], a['vd'], a['npd'], a['nd'],
                             a['rough'], a['slab'], a['om'], a['pm'], a['oop'], a['edw'], None)


def _bwd(L, lib, d, **kw):
  a = dict(mat=FAKE, ml=FAKE, gp=FAKE, rr=FAKE, rgd=FAKE, vd=FAKE, w=FAKE, dslab=FAKE, ld=160, om=0.0, pm=0.0, oop=1,
           drd=None, ddf=None, dti=None, dgp=FAKE, drr=FAKE, drgd=FAKE, stats=FAKE)
  a.update(kw)
  return lib.mnrf_refdir_bwd(C.byref(d), a['mat'], a['ml'], a['gp'], a['rr'], a['rgd'], a['vd'], a['w'], a['dslab'],
                             a['ld'], a['om'], a['pm'], a['oop'], a['drd'], a['ddf'], a['dti'], a['dgp'], a['drr'],
                             a['drgd'], a['stats'], None)


REFUSALS = [
    # (entry, descriptor overrides, argument overrides, message)
    ('both', dict(col_end=64 + 72), {}, 'must hold'),                               # IDE + n.v need 73 columns
    ('both', dict(ld=150, col_end=160), dict(ld=150), 'must hold'),                 # col_end > ld
    ('both', dict(use_ide=0, deg_view=4, col_end=64 + 27), {}, 'must hold'),        # PE + n.v: 28 columns
    ('bwd', dict(use_ide=0, use_reflections=0, use_n_dot_v=0, deg_view=0, col_end=64 + 10), {}, 'must hold'),
    ('bwd', {}, dict(ld=159), 'must hold'),                                         # ld_dslab < col_end
    ('both', dict(deg_view=6, ide_n=36), {}, 'deg_view of at most 5'),
    ('both', dict(deg_view=0, ide_n=0), {}, 'deg_view of at most 5'),
    ('both', dict(deg_view=-1, ide_n=0), {}, 'deg_view of at most 5'),
    ('both', dict(deg_view=4, ide_n=36), {}, 'ide_n 36 does not match deg_view 4'),
    ('both', dict(ide_n=35), {}, 'ide_n 35 does not match'),
    ('both', dict(use_ide=0, deg_view=-1), {}, 'must not be negative'),
    ('both', dict(use_roughness=0), dict(rr=None), 'IDE needs a roughness'),
    ('both', dict(use_pred_normals=0, use_density_normals=0), {}, 'Normals must be computed'),
    ('both', {}, dict(gp=None), 'use_pred_normals needs grad_pred'),
    ('both', {}, dict(rgd=None), 'use_density_normals needs raw_grad_density'),
    ('both', {}, dict(rr=None), 'use_roughness needs raw_rough'),
    ('fwd', {}, dict(rough=None), 'needs the roughness output'),
    ('bwd', {}, dict(drr=None), 'needs d_raw_rough'),
    ('bwd', {}, dict(dgp=None), 'needs d_grad_pred'),
    ('bwd', {}, dict(drgd=None), 'needs d_raw_grad_density'),
    ('both', dict(use_pred_normals=0), dict(om=0.1, oop=1, edw=FAKE), 'orientation loss is on'),
    ('both', dict(use_density_normals=0), dict(om=0.1, oop=0, edw=FAKE), 'orientation loss is on'),
    ('both', dict(use_density_normals=0), dict(pm=1e-3, edw=FAKE), 'predicted normal loss is on'),
    ('both', dict(num_samples=0), {}, 'num_samples must be positive'),
    ('both', {}, dict(ml=None), 'deg_view of at most 5'),
]


@pytest.mark.parametrize('i', range(len(REFUSALS)))
def test_refdir_refusals(i):
  L, lib = _lib()
  entry, dk, ak, msg = REFUSALS[i]
  for e in (('fwd', 'bwd') if entry == 'both' else (entry,)):
    d = _desc(L, **dk)
    args = {k: v for k, v in ak.items() if not (e == 'fwd' and k in ('ld', 'drr', 'dgp', 'drgd'))}
    if e == 'bwd':
      args = {k: v for k, v in args.items() if k not in ('rough', 'edw')}
    rc = (_fwd if e == 'fwd' else _bwd)(L, lib, d, **args)
    err = lib.mnrf_last_error().decode()
    assert rc != 0 and msg in err, (e, dk, ak, rc, err)


def test_refdir_accepts_what_it_should():
  """The checks are no stricter than the kernels: a valid descriptor gets past every one of them (and then fails only
  for want of a device)."""
  L, lib = _lib()
  for e, fn in (('fwd', _fwd), ('bwd', _bwd)):
    for dk in (dict(), dict(use_ide=0, deg_view=10, col_end=64 + 64), dict(deg_view=1, ide_n=2, col_end=64 + 11),
               dict(use_ide=0, use_reflections=0, use_n_dot_v=0, deg_view=0, col_end=64 + 11)):
      fn(L, lib, _desc(L, **dk))
      err = lib.mnrf_last_error().decode()
      assert not any(m in err for m in ('must hold', 'deg_view', 'needs', 'Normals')), (e, dk, err)


@pytest.mark.parametrize('call,msg', [
    ('fwd-orient', 'orientation loss is on'), ('fwd-prednorm', 'predicted normal loss is on'),
    ('bwd-orient', 'orientation loss is on'), ('bwd-prednorm', 'predicted normal loss is on'),
    ('bwd-heads', 'head_grads needs'), ('fwd-none', 'no normals')])
def test_normals_refusals(call, msg):
  L, lib = _lib()
  if call == 'fwd-orient':
    rc = lib.mnrf_normals_fwd(64, 8, None, FAKE, FAKE, None, FAKE, 0.1, 0.0, 1, FAKE, None)
  elif call == 'fwd-prednorm':
    rc = lib.mnrf_normals_fwd(64, 8, FAKE, None, FAKE, FAKE, None, 0.0, 1e-3, 1, FAKE, None)
  elif call == 'fwd-none':
    rc = lib.mnrf_normals_fwd(64, 8, None, None, FAKE, None, None, 0.0, 0.0, 1, None, None)
  elif call == 'bwd-orient':
    rc = lib.mnrf_normals_bwd(64, 8, FAKE, None, FAKE, FAKE, 0.1, 0.0, 0, None, None, 1, FAKE, None, None, 0, FAKE,
                              None)
  elif call == 'bwd-prednorm':
    rc = lib.mnrf_normals_bwd(64, 8, FAKE, None, FAKE, FAKE, 0.0, 1e-3, 1, None, None, 1, FAKE, None, None, 0, FAKE,
                              None)
  else:
    rc = lib.mnrf_normals_bwd(64, 8, None, FAKE, FAKE, FAKE, 0.0, 0.0, 1, FAKE, None, 1, None, FAKE, FAKE, 4, None,
                              None)
  assert rc != 0 and msg in lib.mnrf_last_error().decode()
