"""Proposal resampler (mnrf_sample_level, with d->anneal or a device-side anneal) against the fp64 reference of
tests/sampling_ref.py, on every warp plan, jitter mode, dilation and anneal source.  Needs an H100.

Every case checks: the dilated fenceposts bit for bit; the dilated weights, CDF, interval endpoints and interval
indices against their per-element bounds; with the kernel's own CDF fed back through `cw_in`, indices equal to the
fp64 sorted_interp on that CDF and endpoints within the interpolation's roundings; the same bits of sdist with and
without the index and debug outputs, and through the device-side anneal; inputs that are views into NaN-filled
buffers and an output that is a view between sentinel pads, which must survive.  Each case prints its worst
err / bound ratio.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import sampling_ref as SR

pytestmark = pytest.mark.gpu

F = np.float32
PAD = 37                    # floats of guard on both sides of every input and of the output
SENTINEL = -7.25e33


@pytest.fixture(scope='module')
def ops():
  from multinerf_b200 import lib, ops as _ops
  lib.require_device()
  return _ops


# name: P, S, rays, dilation (0 = none), domain, anneal, padding, jitter mode (0 none, 1 single, 2 per sample),
# weight profile
CASES = {
    'smallest': (1, 2, 1, 0.0, (0.0, 1.0), 1.0, 0.0, 0, 'random'),
    'nb1-dilated': (1, 64, 37, 0.02, (0.0, 1.0), 0.9, 0.0, 1, 'random'),
    'windows-cover-domain': (2, 3, 5, 0.3, (0.0, 1.0), 1.0, 0.0, 2, 'random'),
    'chunk31': (31, 31, 257, 0.0103, (0.0, 1.0), 0.5, 0.0, 1, 'random'),
    'chunk32': (32, 32, 257, 0.0, (0.0, 1.0), 0.5, 0.0, 2, 'random'),
    'chunk33-near': (33, 33, 257, 0.0103, (0.35, 1.0), 0.5, 0.0, 0, 'random'),
    '360-level1': (64, 64, 20000, 0.0103125, (0.0, 1.0), 0.9091, 0.0, 1, 'chained'),
    '360-level2': (64, 32, 20000, 0.0026220703125, (0.0, 1.0), 0.5, 0.0, 1, 'chained'),
    'anneal0': (64, 64, 257, 0.0103, (0.0, 1.0), 0.0, 0.0, 1, 'positive'),
    'anneal0-zeros': (64, 64, 257, 0.0103, (0.0, 1.0), 0.0, 0.0, 1, 'zeros'),
    'peaked-padding': (128, 128, 1000, 0.0, (0.0, 1.0), 1.0, 0.01, 2, 'peaked'),
    'dilation-narrow-zeros': (255, 257, 300, 1e-4, (0.0, 1.0), 1.0, 0.0, 0, 'zeros'),
    'dilation-narrow-dups': (255, 257, 300, 1e-4, (0.0, 1.0), 1.0, 0.0, 0, 'duplicates'),
    'warps2': (1000, 64, 300, 0.003, (0.0, 1.0), 1.0, 0.0, 1, 'random'),
    'P1024': (1024, 32, 64, 0.0, (0.0, 1.0), 1.0, 0.0, 0, 'random'),
    'P1024-nb3070': (1024, 32, 64, 0.001, (0.0, 1.0), 1.0, 0.0, 0, 'random'),
    'warps1': (1024, 12500, 3, 0.0, (0.0, 1.0), 1.0, 0.0, 1, 'random'),
    'stepfun-uniform': (4, 10, 5, 0.0, (-math.inf, math.inf), 1.0, 0.0, 0, 'uniform'),
    # the shapes and settings of the fp32-oracle comparison this file replaces
    'oracle-64-64': (64, 64, 257, 0.0103125, (0.0, 1.0), 0.9091, 0.0, 1, 'duplicates'),
    'oracle-64-32': (64, 32, 257, 0.0026220703125, (0.0, 1.0), 0.9091, 0.0, 1, 'random'),
    'oracle-1-64': (1, 64, 257, 0.0, (0.0, 1.0), 0.9091, 0.01, 1, 'random'),
    'oracle-128-128': (128, 128, 257, 0.0, (0.0, 1.0), 0.9091, 0.01, 2, 'duplicates'),
    'oracle-37-17': (37, 17, 257, 0.02, (0.0, 1.0), 0.9091, 0.0, 2, 'random'),
}


def _density_weights(sdist, bumps):
  """Volume-rendering weights on [B, P+1] intervals of a density made of Gaussian bumps (centre, width, height)."""
  B = sdist.shape[0]
  s = sdist.double().cpu()
  mid, ds = (s[:, 1:] + s[:, :-1]) / 2, s[:, 1:] - s[:, :-1]
  sig = torch.zeros_like(mid)
  for c, wd, a in bumps:
    sig += a * torch.exp(-0.5 * ((mid - c) / wd) ** 2)
  tau = sig * ds
  trans = torch.exp(-torch.cat([torch.zeros(B, 1, dtype=tau.dtype), torch.cumsum(tau, -1)[:, :-1]], -1))
  return ((1 - torch.exp(-tau)) * trans).float()


def _chain(ops, rng, B, levels):
  """The 360.gin schedule's inputs: [near, far] resampled into 64 intervals, then `levels` kernel levels of
  64 samples, each weighted by the same synthetic density of two bumps per ray."""
  bumps = [tuple(torch.tensor(rng.uniform(lo, hi, (B, 1))) for lo, hi in ((0.05, 0.95), (0.01, 0.1), (20, 400)))
           for _ in range(2)]
  t = torch.tensor([[0.0, 1.0]] * B, device='cuda')
  w = torch.ones(B, 1, device='cuda')
  for S, dil in [(64, 0.0)] + [(64, 0.0103125)] * levels:
    jit = torch.tensor(rng.uniform(0, 1, B).astype(F), device='cuda')
    t = ops.sample_level(t, w, S, dilation=dil, use_dilation=dil > 0, anneal=0.9091, jitter=jit)
    w = _density_weights(t, bumps).cuda()
  return t.cpu(), w.cpu()


def make_case(ops, name):
  P, S, B, dil, dom, anneal, pad, jm, prof = CASES[name]
  rng = np.random.default_rng(sum(map(ord, name)))
  if prof == 'chained':
    t, w = _chain(ops, rng, B, 0 if S == 64 else 1)
    te, we = SR.step_functions(rng, 'random', 8, P)
    t[:4], w[:4] = te[:4], we[:4]
  else:
    t, w = SR.step_functions(rng, prof, B, P, domain=dom)
  ub, mj = ops.u_grid(S, jm != 0)
  jit = None
  if jm:
    jit = torch.tensor(rng.uniform(0, 1, (B,) if jm == 1 else (B, S)).astype(F))
    if B >= 8:
      jit[1] = 0          # u = 0 on the ray with a single nonzero bin
  return t, w, S, dict(use_dilation=dil > 0, dilation=dil, domain=dom, anneal=anneal, resample_padding=pad,
                       u_base=ub, max_jitter=mj, jitter=jit, jitter_mode=jm)


def _guarded(x, fill):
  """A CUDA copy of x that is a view into a buffer with PAD elements of `fill` on both sides."""
  buf = torch.full((x.numel() + 2 * PAD,), fill, dtype=x.dtype, device='cuda')
  v = buf[PAD:PAD + x.numel()].view(x.shape)
  v.copy_(x)
  return v, buf


def _pads_intact(buf, fill):
  pads = torch.cat([buf[:PAD], buf[-PAD:]]).cpu()
  return torch.equal(pads.view(torch.int32), torch.full_like(pads, fill).view(torch.int32))


def _bits(x):
  return x.detach().cpu().contiguous().view(torch.int32)


def _launch(ops, t, w, S, cfg, **kw):
  args = dict(dilation=cfg['dilation'], use_dilation=cfg['use_dilation'], domain=cfg['domain'],
              anneal=cfg['anneal'], resample_padding=cfg['resample_padding'], u_base=cfg['u_base'],
              max_jitter=cfg['max_jitter'], jitter=cfg['jitter'], single_jitter=cfg['jitter_mode'] == 1)
  args.update(kw)
  return ops.sample_level(t, w, S, **args)


@pytest.mark.parametrize('name', list(CASES))
def test_sample_level_fp64(ops, name):
  t, w, S, cfg = make_case(ops, name)
  B = w.shape[0]
  tv, tbuf = _guarded(t, math.nan)
  wv, wbuf = _guarded(w, math.nan)
  ubv, ubuf = _guarded(cfg['u_base'], math.nan)
  dev = dict(cfg, u_base=ubv)
  if cfg['jitter'] is not None:
    dev['jitter'], jbuf = _guarded(cfg['jitter'], math.nan)
  out, obuf = _guarded(torch.zeros(B, S + 1), SENTINEL)
  out.fill_(SENTINEL)
  sd, dbg = _launch(ops, tv, wv, S, dev, want_index=True, want_debug=True, out=out)
  torch.cuda.synchronize()
  assert _pads_intact(obuf, SENTINEL), 'wrote outside sdist'

  ref = SR.reference(t, w, S, **cfg)
  worst = SR.ratios(ref, sd, dbg['idx'], dbg['cw'], dbg['tdil'], dbg['wdil'])

  # the same bits without the index / debug outputs, and with anneal read from device memory
  plain = _launch(ops, tv, wv, S, dev)
  only_idx, _ = _launch(ops, tv, wv, S, dev, want_index=True)
  dyn = _launch(ops, tv, wv, S, dev, anneal=1.0,
                anneal_dev=torch.tensor([SR.f32(cfg['anneal'])], device='cuda'))
  for name_, x in (('plain', plain), ('index only', only_idx), ('anneal_dev', dyn)):
    assert torch.equal(_bits(x), _bits(sd)), f'{name_}: sdist bits differ'

  # integer contract: the kernel's own CDF fed back gives the fp64 indices on that CDF
  sd2, dbg2 = _launch(ops, tv, wv, S, dev, cw_in=dbg['cw'].contiguous(), want_index=True)
  ref2 = SR.reference(t, w, S, cw_in=dbg['cw'], **cfg)
  assert torch.equal(dbg2['idx'].cpu().long(), ref2.idx), 'indices on a shared CDF'
  worst['sdist(cw_in)'] = SR.ratios(ref2, sd2)['sdist']
  torch.cuda.synchronize()
  for buf in (tbuf, wbuf, ubuf) + ((jbuf,) if cfg['jitter'] is not None else ()):
    assert torch.isnan(torch.cat([buf[:PAD], buf[-PAD:]])).all()
  print(f'\n{name}: P={w.shape[1]} S={S} rays={B} warps={SR.warp_plan(w.shape[1], S)} '
        f'nan rows={int(ref.nan_row.sum())} worst err/bound ' +
        ' '.join(f'{k}={v:.3g}' for k, v in worst.items()))
  assert all(v <= 1 for v in worst.values()), worst


def test_case_matrix_reaches_every_plan(ops):
  """4-, 2- and 1-warp blocks, the grid-stride loop, every jitter mode, both dilation branches, NaN CDF rows."""
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  plans = {SR.warp_plan(c[0], c[1]) for c in CASES.values()}
  assert plans == {1, 2, 4}, plans
  assert any(c[2] > sms * 16 * SR.warp_plan(c[0], c[1]) for c in CASES.values()), 'no grid-stride case'
  assert {c[7] for c in CASES.values()} == {0, 1, 2}
  assert {c[3] > 0 for c in CASES.values()} == {False, True}


def test_nan_cdf_collapses_onto_first_fencepost(ops):
  """All logits -inf: the CDF's inner knots stay NaN and every sample lands on the first fencepost, as in the
  reference (jnp.minimum keeps the NaN that fminf would drop)."""
  t = torch.tensor([[0.1, 0.3, 0.5, 0.9, 1.0]], device='cuda')
  w = torch.zeros(1, 4, device='cuda')
  sd, dbg = ops.sample_level(t, w, 6, want_index=True, want_debug=True)
  assert torch.isnan(dbg['cw'][0, 1:-1]).all()
  assert torch.equal(sd.cpu(), torch.full((1, 7), 0.1))
  assert torch.equal(dbg['idx'].cpu(), torch.zeros(1, 6, dtype=torch.int32))


def test_stepfun_deterministic(ops):
  """stepfun_test.py: one interval [3, 4], no jitter, unbounded domain -> 11 evenly spaced endpoints."""
  t = torch.tensor([[3.0, 4.0]] * 5).cuda()
  w = torch.ones(5, 1).cuda()
  sd = ops.sample_level(t, w, 10, domain=(-math.inf, math.inf))
  ref = torch.tensor(np.linspace(3, 4, 11)).expand(5, 11)
  assert (sd.cpu().double() - ref).abs().max() <= 4 * 2.0 ** -22
  with pytest.raises(ValueError):
    ops.sample_level(t, w, 1)


def _bad_calls():
  from multinerf_b200 import lib as L
  B, P, S = 8, 4, 6
  t = torch.linspace(0, 1, P + 1).expand(B, P + 1).contiguous().cuda()
  w = torch.full((B, P), 0.25, device='cuda')
  from multinerf_b200 import ops as _ops
  ub = _ops.u_grid(S, False)[0].cuda()

  anneal = torch.ones(1, device='cuda')

  def call(num_prev=P, num_samples=S, jitter_mode=0, null=None):
    out, buf = _guarded(torch.zeros(B, S + 1), SENTINEL)
    out.fill_(SENTINEL)
    d = L.SampleDesc(B, num_prev, num_samples, 0, 0.0, 0.0, 1.0, 1.0, 0.0, jitter_mode, 0.1)
    p = {k: L.ptr(v) for k, v in dict(t=t, w=w, ub=ub, out=out).items()}
    if null:
      p[null] = None

    def run(lib, device_anneal):
      L.check(lib.mnrf_sample_level(C.byref(d), p['t'], p['w'], p['ub'], None,
                                    L.ptr(anneal) if device_anneal else None, None, p['out'], None, None, None, None,
                                    L.stream_ptr()))
    return run, buf
  return {'num_samples 1': lambda: call(num_samples=1), 'num_samples 0': lambda: call(num_samples=0),
          'num_prev 0': lambda: call(num_prev=0), 'num_prev 1025': lambda: call(num_prev=1025),
          'jitter_mode 1 without jitter': lambda: call(jitter_mode=1),
          'jitter_mode 2 without jitter': lambda: call(jitter_mode=2),
          'null sdist_prev': lambda: call(null='t'), 'null w_prev': lambda: call(null='w'),
          'null u_base': lambda: call(null='ub'), 'null sdist_out': lambda: call(null='out')}


BAD = ['num_samples 1', 'num_samples 0', 'num_prev 0', 'num_prev 1025', 'jitter_mode 1 without jitter',
       'jitter_mode 2 without jitter', 'null sdist_prev', 'null w_prev', 'null u_base', 'null sdist_out']


@pytest.mark.parametrize('anneal', ['host anneal', 'device anneal'])
@pytest.mark.parametrize('name', BAD)
def test_rejected_arguments(ops, name, anneal):
  from multinerf_b200 import lib as L
  run, buf = _bad_calls()[name]()
  with pytest.raises(L.MnrfError):
    run(L.load(), anneal == 'device anneal')
  torch.cuda.synchronize()
  assert _pads_intact(buf, SENTINEL) and (buf == SENTINEL).all(), f'{name}: the refused call wrote its output'


def test_zero_rays_with_either_anneal_source(ops):
  from multinerf_b200 import lib as L
  out, buf = _guarded(torch.zeros(4), SENTINEL)
  out.fill_(SENTINEL)
  d = L.SampleDesc(0, 4, 6, 1, 0.01, 0.0, 1.0, 1.0, 0.0, 1, 0.1)
  x = L.ptr(out)
  for anneal_dev in (None, x):       # d->anneal, then the exponent read from the device
    L.check(L.load().mnrf_sample_level(C.byref(d), x, x, x, x, anneal_dev, None, x, None, None, None, None,
                                       L.stream_ptr()))
  torch.cuda.synchronize()
  assert (buf == SENTINEL).all()
