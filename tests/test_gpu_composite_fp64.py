"""Compositing and loss kernels (mnrf_composite_fwd, mnrf_composite_bwd, mnrf_point_rgb) against an fp64 reference
with a bound on every element.

The values are the oracle's chain in float64 differentiated by torch.autograd (composite_ref.grads); the bound of
each element is composite_ref.walk's running error of the kernels' own fp32 arithmetic (see composite_ref.py; its
soundness and sensitivity are shown on the CPU by test_composite_reference_cpu.py).  No outlier fraction: every
element that is not exempt (a branch the kernel takes within rounding of its tie, see the walk) is within its
bound, and each case prints its live fraction (neither exempt nor vacuous) and its worst err / bound.

The case table reaches every sample-count instance (CH = 1, 2, 4, 8) at its edges, every loss type x lossmult
channel count x ray-distance function x rgb activation x opaque / translucent background, every optional input,
interlevel levels of fewer, as many and more fine intervals than a warp has lanes, and 1 ray, fewer rays than a
block has warps, and more rays than a launch has warps.  Inputs sit in front of NaN rows (raw_density / raw_rgb
also as column views of ld 4 and 8), outputs start as NaN inside sentinel padding.  Needs an H100.
"""
import ctypes as C
import itertools
import time

import numpy as np
import pytest
import torch

import composite_ref as R

pytestmark = pytest.mark.gpu

# (near, far) valid for each ray-distance function; ray 3 of a reciprocal batch gets far = 1e6
NEAR_FAR = {None: (2.0, 6.0), 'reciprocal': (0.2, 100.0), 'log': (0.5, 10.0), 'exp': (0.0, 2.0), 'sqrt': (0.0, 4.0),
            'square': (0.5, 3.0), 'piecewise': (0.2, 50.0)}
BASE = dict(density_bias=-1.0, density_noise=0.0, rgb_premultiplier=1.0, rgb_padding=0.001, bg_const=0.7)
SAMPLES = (1, 31, 32, 33, 64, 65, 128, 129, 255, 256)
OPTIONS = ('', 'n', 'b', 's', 'e', 'm', 'r', 'R', 'nbse', 'sr', 'Rm', 'bsRe')
SF = (17, 32, 48, 31, 33, 64, 200, 1)
MANY = -1          # B of the cases with more rays than one launch has warps (from the SM count)
SENTINEL = -12345.0
# the least share of each output's elements that must be live (neither exempt nor vacuous) in every case.  The pixel
# (near 0 on proposal levels, relative to which its bound is wide) and d_raw_density (it cancels to near 0 behind
# opaque samples and on the envelope's empty stretches) have no floor; their live share is printed.
MIN_LIVE = dict(weights=0.5, density=0.9, rgb_samples=0.5, acc=0.5, distance_mean=0.5, d_raw_rgb=0.5, d_rgb_scale=0.5,
                d_raw_diffuse=0.5, d_raw_tint=0.5)


def _cases():
  """(S, B, level, loss type, lossmult channels, raydist, rgb activation, opaque background, options, Sf, ld)
  level 'fine': colour, distortion loss; 'prop': no colour, interlevel loss against a final level of Sf samples.
  options: n density_noise, b bg_rgb, s rgb_scale, e extra_dw, m data_mask, r rgb_mode 1 with a tint, R without.
  ld: floats between samples of raw_density / raw_rgb (0 contiguous, 4 or 8 column views)."""
  out = []
  combos = itertools.product(('mse', 'charb', 'rawnerf'), (1, 3), R.RAYDIST, ('sigmoid', 'safe_exp'), (True, False))
  for i, (loss, lm, rd, act, opaque) in enumerate(combos):
    S = SAMPLES[i % len(SAMPLES)]
    prop = i % 4 == 3
    opts = OPTIONS[(i // 2) % len(OPTIONS)]
    if prop:
      opts = opts.replace('r', '').replace('R', '').replace('s', '')
    Sf = SF[(i // 4) % len(SF)] if prop else 0
    B = (1, 3, 5, 8, 13)[i % 5] if i % 7 else 6
    out.append((S, B, 'prop' if prop else 'fine', loss, lm, rd, act, opaque, opts, Sf, (0, 4, 8)[i % 3]))
  # more rays than one launch has warps: every warp composites several rays and carries its loss partials
  out.append((48, MANY, 'prop', 'mse', 1, 'reciprocal', 'sigmoid', True, 'n', 64, 0))
  out.append((100, MANY, 'fine', 'charb', 3, 'reciprocal', 'sigmoid', False, 'bsr', 0, 4))
  out.append((256, MANY, 'fine', 'rawnerf', 1, 'log', 'safe_exp', False, 'nbsem', 0, 0))
  return out


CASES = _cases()


def many_rays(num_sms):
  """More rays than one launch has warps (num_sms x 16 blocks x 4 warps), and not a multiple of them."""
  return num_sms * 16 * 4 * 2 + 37


def case_id(c):
  S, B, level, loss, lm, rd, act, opaque, opts, Sf, ld = c
  return (f'S{S}-B{"many" if B == MANY else B}-{level}{Sf or ""}-{loss}{lm}-{rd}-{act}-'
          f'{"opaque" if opaque else "translucent"}-{opts or "plain"}-ld{ld}')


def _edge_rays(rng, S, B, raydist, sdist, raw_d, dirs, far):
  """Rays 0-4 of a batch: an empty ray, a ray whose first sample is opaque (T underflows to 0 after it), a ray of
  zero-width intervals (duplicate knots, delta = 0), a ray with far = 1e6 (under the reciprocal warp) and a ray with
  a direction of norm 3."""
  raw_d[0] = -50.0
  raw_d[1] = 30.0
  sdist[1, 1:] = 0.5 + 0.5 * sdist[1, 1:]     # first interval: half the ray
  dirs[1] *= 200.0 / np.linalg.norm(dirs[1])
  if S == 1:
    sdist[2, 1] = sdist[2, 0]
  else:
    sdist[2, 1:S:3] = sdist[2, 0:S - 1:3]
  if raydist == 'reciprocal':
    far[3] = 1e6
  dirs[4] *= 3.0 / np.linalg.norm(dirs[4])


def make(case, seed, num_sms=132):
  """fp32 inputs (CPU tensors, 'inv_denom' included), the composite cfg and the loss settings of one case."""
  S, B, level, loss_type, lm_ch, raydist, act, opaque, opts, Sf, _ = case
  if B == MANY:
    B = many_rays(num_sms)
  rng = np.random.default_rng(seed)
  f = np.float32
  sdist = np.sort(rng.uniform(0, 1, (B, S + 1)), -1)
  sdist[:, 0], sdist[:, -1] = 0, 1
  dup = rng.uniform(size=B) < 0.2                                  # some more duplicate knots
  sdist[dup, S // 2] = sdist[dup, max(S // 2 - 1, 0)]
  raw_d = rng.normal(size=(B, S)) * 3
  # raw densities at the ends of softplus and sigmoid: +-80 and +-1e4 on a few samples of a few rays
  k = rng.uniform(size=(B, S)) < 0.02
  raw_d[k] = rng.choice([80.0, -80.0, 1e4, -1e4], size=int(k.sum()))
  d = rng.normal(size=(B, 3))
  d = d / np.linalg.norm(d, axis=-1, keepdims=True) * rng.uniform(0.8, 1.2, (B, 1))
  near, far = NEAR_FAR[raydist]
  nearv, farv = np.full(B, near), np.full(B, far)
  if B >= 5:
    _edge_rays(rng, S, B, raydist, sdist, raw_d, d, farv)
  inp = dict(raw_density=raw_d, sdist=sdist, directions=d, near=nearv, far=farv,
             target=rng.uniform(0, 1, (B, 3)),
             lossmult=rng.integers(0, 3, (B, lm_ch)) + (rng.uniform(size=(B, lm_ch)) < 0.5) * 0.5)
  inp['lossmult'][0] = 1.0
  rgb = level == 'fine'
  if rgb:
    inp['raw_rgb'] = rng.normal(size=(B, S, 3)) * 1.5
    if act == 'safe_exp' and B >= 5 and S > 1:
      # safe_exp's clamp at 88: on ray 1 behind its opaque first sample (weight exactly 0), so the pixel stays finite
      inp['raw_rgb'][1, 1:, 0] = 100.0
      inp['raw_rgb'][1, 1:, 1] = -100.0
  if 'n' in opts:
    inp['density_noise'] = rng.normal(size=(B, S))
  if 'b' in opts:
    inp['bg_rgb'] = rng.uniform(0, 1, (B, 3))
  if 's' in opts:
    sc = rng.uniform(0.5, 2.0, (B, 3))
    sc[min(3, B - 1), 0] = 0.0                                    # a zero and a negative exposure channel
    sc[min(4, B - 1), 1] = -0.7
    inp['rgb_scale'] = sc
  if 'e' in opts:
    inp['extra_dw'] = rng.normal(size=(B, S)) * 1e-2
  if 'm' in opts:
    inp['data_mask'] = (rng.uniform(size=B) < 0.7).astype(np.float64)
  if 'r' in opts or 'R' in opts:
    inp['raw_diffuse'] = rng.normal(size=(B, S, 3))
    if 'r' in opts:
      inp['raw_tint'] = rng.normal(size=(B, S, 3))
  if level == 'prop':
    # the final level's intervals share about half their knots with this level's (the envelope)
    kk = min(S - 1, Sf // 2)
    own = np.stack([rng.choice(sdist[i, 1:S], kk, replace=False) for i in range(B)]) if kk > 0 else np.zeros((B, 0))
    sf = np.sort(np.concatenate([own, rng.uniform(0, 1, (B, Sf - 1 - kk))], -1), -1)
    inp['sdist_fine'] = np.concatenate([np.zeros((B, 1)), sf, np.ones((B, 1))], -1)
    wf = rng.uniform(0, 1, (B, Sf)) ** 2
    wf[rng.uniform(size=(B, Sf)) < 0.1] = 0.0                      # empty fine intervals
    inp['weights_fine'] = wf / np.maximum(wf.sum(-1, keepdims=True), 1e-12) * 0.9
  if B > 1:
    inp['lossmult'][-1] = 0.0                                      # a ray without data loss
  inp = {k_: torch.tensor(np.asarray(v).astype(f)) for k_, v in inp.items()}
  cfg = dict(BASE, raydist_fn=raydist, opaque_background=opaque, rgb_activation=act,
             rgb_bias=-1.0 if act == 'safe_exp' else 0.0, density_noise=0.5 if 'n' in opts else 0.0,
             rgb_mode=1 if ('r' in opts or 'R' in opts) else 0)
  if act == 'safe_exp':
    cfg['rgb_padding'] = 0.0
  inv_denom = np.float32(1.0 / float(inp['lossmult'].expand(B, 3).double().sum()))
  inp['inv_denom'] = torch.tensor([inv_denom])
  loss = dict(loss_type=loss_type, charb_padding=0.001, data_mult=0.1 if level == 'prop' else (0.5 if seed % 2 else 1.0),
              distortion_mult=0.01 if level == 'fine' else 0.0, interlevel_mult=1.0 if level == 'prop' else 0.0)
  return inp, cfg, loss


# ---- launches through the C ABI, on guarded buffers -----------------------------------------------------------------

class Guarded:
  """A tensor of `shape` inside a buffer of `pad` more rows, filled with `fill`; `view` is what the kernel sees."""

  def __init__(self, shape, fill, pad=2, value=None, ld=0, col=0):
    n = int(np.prod(shape[:2])) if ld else shape[0]
    if ld:
      self.buf = torch.full((n + pad, ld), fill, device='cuda')
      w = int(np.prod(shape[2:])) if len(shape) > 2 else 1
      v = self.buf[:n, col:col + w]
      self.view = v.view(*shape) if len(shape) > 2 else v[:, 0].view(*shape)
    else:
      self.buf = torch.full((n + pad,) + tuple(shape[1:]), fill, device='cuda')
      self.view = self.buf[:n]
    if value is not None:
      self.view.copy_(value)
    self.mask = torch.zeros_like(self.buf, dtype=torch.bool)
    self.mask_view(shape, ld, col, n)
    self.fill = fill

  def mask_view(self, shape, ld, col, n):
    if ld:
      w = int(np.prod(shape[2:])) if len(shape) > 2 else 1
      self.mask[:n, col:col + w] = True
    else:
      self.mask[:n] = True

  def untouched(self):
    out = self.buf[~self.mask]
    return bool((out == self.fill).all()) if not np.isnan(self.fill) else bool(torch.isnan(out).all())


@pytest.fixture(scope='module')
def lib():
  from multinerf_b200 import lib as L
  L.require_device()
  return L, L.load()


def _desc(L, cfg, B, S, ld):
  from multinerf_b200 import ops
  d = ops._cdesc(B, S, **cfg)
  d.ld_density, d.ld_rgb = (ld, ld) if ld else (0, 0)
  return d


def _inputs(inp, ld):
  """Every input in front of NaN rows; raw_density / raw_rgb (and their gradients) as column views when ld."""
  B, S = inp['raw_density'].shape
  g = {}
  for k, v in inp.items():
    if k in ('raw_density', 'raw_rgb') and ld:
      g[k] = Guarded(tuple(v.shape), float('nan'), value=v.cuda(), ld=ld, col=0 if k == 'raw_density' else 1)
    else:
      g[k] = Guarded(tuple(v.shape), float('nan'), value=v.cuda())
  return g


def run_fwd(L, lib, inp, cfg, ld=0, outputs=True):
  B, S = inp['raw_density'].shape
  g = _inputs(inp, ld)
  P = lambda k: L.ptr(g[k].view) if k in g else None
  o = dict(weights=Guarded((B, S), float('nan')), rgb=Guarded((B, 3), float('nan')))
  if outputs:
    o.update(density=Guarded((B, S), float('nan')), rgb_samples=Guarded((B, S, 3), float('nan')),
             acc=Guarded((B,), float('nan')), dist=Guarded((B, 4), float('nan')))
  for v in o.values():
    v.buf[~v.mask] = SENTINEL
    v.fill = SENTINEL
  Q = lambda k: L.ptr(o[k].view) if k in o else None
  d = _desc(L, cfg, B, S, ld)
  rc = lib.mnrf_composite_fwd(C.byref(d), P('raw_density'), P('raw_rgb'), P('density_noise'), P('sdist'),
                              P('directions'), P('near'), P('far'), P('bg_rgb'), P('rgb_scale'), P('raw_diffuse'),
                              P('raw_tint'), Q('weights'), Q('rgb'), Q('density'), Q('rgb_samples'), Q('acc'),
                              Q('dist'), L.stream_ptr())
  L.check(rc)
  torch.cuda.synchronize()
  return o, g


def run_bwd(L, lib, inp, cfg, loss, ld=0, stats0=None, batch_rays=None, rows=None):
  """One backward launch over the rays `rows` (a slice; all by default) of inp.  Returns (outputs, stats)."""
  full_B, S = inp['raw_density'].shape
  if rows is not None:
    inp = {k: (v[rows] if k != 'inv_denom' else v) for k, v in inp.items()}
  B = inp['raw_density'].shape[0]
  g = _inputs(inp, ld)
  P = lambda k: L.ptr(g[k].view) if k in g else None
  o = dict(d_raw_density=Guarded((B, S), float('nan'), ld=ld, col=0))
  if 'raw_rgb' in inp:
    o['d_raw_rgb'] = Guarded((B, S, 3), float('nan'), ld=ld, col=1)
  if 'rgb_scale' in inp:
    o['d_rgb_scale'] = Guarded((B, 3), float('nan'))
  if cfg['rgb_mode'] == 1:
    o['d_raw_diffuse'] = Guarded((B, S, 3), float('nan'))
    o['d_raw_tint'] = Guarded((B, S, 3), float('nan'))
  for v in o.values():
    v.buf[~v.mask] = SENTINEL
    v.fill = SENTINEL
  Q = lambda k: L.ptr(o[k].view) if k in o else None
  stats = Guarded((8,), SENTINEL)
  stats.view.copy_(torch.zeros(8) if stats0 is None else stats0)
  d = L.LossDesc(_desc(L, cfg, B, S, ld), L.LOSS_TYPE[loss['loss_type']], float(loss['charb_padding']),
                 float(loss['data_mult']), float(loss['distortion_mult']), float(loss['interlevel_mult']),
                 inp['weights_fine'].shape[1] if 'weights_fine' in inp else 0, inp['lossmult'].shape[1])
  rc = lib.mnrf_composite_bwd(
      C.byref(d), P('raw_density'), P('raw_rgb'), P('density_noise'), P('sdist'), P('directions'), P('near'), P('far'),
      P('bg_rgb'), P('rgb_scale'), P('raw_diffuse'), P('raw_tint'), P('extra_dw'), P('target'), P('lossmult'),
      P('inv_denom'), P('sdist_fine'), P('weights_fine'), P('data_mask'), Q('d_raw_density'), Q('d_raw_rgb'),
      Q('d_rgb_scale'), Q('d_raw_diffuse'), Q('d_raw_tint'), L.ptr(stats.view),
      int(B if batch_rays is None else batch_rays), L.stream_ptr())
  L.check(rc)
  torch.cuda.synchronize()
  for k, v in g.items():
    assert torch.equal(v.view.cpu(), inp[k].cpu()) or torch.equal(torch.isnan(v.view).cpu(), torch.isnan(inp[k])), \
        f'input {k} was written'
  return o, stats


# ---- the per-element check -------------------------------------------------------------------------------------------

def _check_case(L, lib, case, seed, num_sms):
  S, _, level, loss_type, lm_ch, raydist, act, opaque, opts, Sf, ld = case
  t0 = time.time()
  inp, cfg, loss = make(case, seed, num_sms)
  B = inp['raw_density'].shape[0]
  fo, _ = run_fwd(L, lib, inp, cfg, ld)
  for k, v in fo.items():
    assert v.untouched(), f'{k}: written outside its rows'
  # the optional outputs change nothing of the others
  fn, _ = run_fwd(L, lib, inp, cfg, ld, outputs=False)
  for k in ('weights', 'rgb'):
    assert torch.equal(fn[k].view, fo[k].view), f'{k} differs without the optional outputs'
  bo, st = run_bwd(L, lib, inp, cfg, loss, ld)
  for k, v in list(bo.items()) + [('stats', st)]:
    assert v.untouched(), f'{k}: written outside its rows'
  # the kernel's own decisions: the background weight's branch from its acc, RawNeRF's v < 1 from its pixel
  acc = fo['acc'].view
  dec = dict(bg_on=((1.0 - acc) > 0).cpu(), v_lt1=(fo['rgb'].view < 1).cpu())
  dev = 'cuda' if B > 1000 else 'cpu'
  res = R.reference(inp, cfg, loss, dec, device=dev)
  lines = []
  for name in ('weights', 'density', 'rgb_samples', 'rgb', 'acc'):
    if name == 'rgb_samples' and 'raw_rgb' not in inp:
      assert (fo[name].view == 0).all()
      continue
    lines.append((name,) + R.check(name, fo[name].view, *res[name], min_live=MIN_LIVE.get(name, 0.0)))
  lines.append(('distance_mean',) + R.check('distance_mean', fo['dist'].view[:, 0], *res['distance_mean'],
                                            min_live=MIN_LIVE['distance_mean']))
  R.check_percentiles('percentiles', fo['dist'].view[:, 1:], res)
  for name in ('d_raw_density', 'd_raw_rgb', 'd_rgb_scale', 'd_raw_diffuse', 'd_raw_tint'):
    if name in res:
      lines.append((name,) + R.check(name, bo[name].view, *res[name], min_live=MIN_LIVE.get(name, 0.0)))
  sv, sb, _ = res['stats']
  got = st.view[:4].to(sv.device, torch.float64)
  bad = (got - sv).abs() > sb
  assert not bad.any(), f'stats {got.tolist()} vs {sv.tolist()} bound {sb.tolist()}'
  assert (st.view[4:] == 0).all()
  print(f'{case_id(case)}: ' + ', '.join(f'{n} live {f:.2f} worst {w:.2f}' for n, f, w in lines) +
        f' ({time.time() - t0:.1f}s)')
  return inp, cfg, loss, fo, bo, st


@pytest.mark.parametrize('i', range(len(CASES)), ids=[case_id(c) for c in CASES])
def test_composite_vs_fp64(lib, i):
  L, lb = lib
  _check_case(L, lb, CASES[i], seed=i, num_sms=int(lb.mnrf_num_sms()))


@pytest.mark.parametrize('i', [1, 3, len(CASES) - 2])
def test_two_passes(lib, i):
  """batch_rays > num_rays: the two halves of a batch in two launches, stats starting non-zero, give the one-pass
  launch's per-element outputs bit for bit, and the one-pass stats plus the starting values within bound."""
  L, lb = lib
  case = CASES[i]
  inp, cfg, loss = make(case, seed=i, num_sms=int(lb.mnrf_num_sms()))
  B = inp['raw_density'].shape[0]
  if B < 2:
    inp, cfg, loss = make(case[:1] + (13,) + case[2:], seed=i)
    B = 13
  ld = case[-1]
  one, st1 = run_bwd(L, lb, inp, cfg, loss, ld)
  h = B // 2
  st0 = torch.tensor([0.25, -0.5, 1.5, 3.0, 7.0, -1.0, 2.0, 0.125])
  a, sa = run_bwd(L, lb, inp, cfg, loss, ld, stats0=st0, batch_rays=B, rows=slice(0, h))
  b, sb = run_bwd(L, lb, inp, cfg, loss, ld, stats0=sa.view.cpu(), batch_rays=B, rows=slice(h, B))
  for k in one:
    both = torch.cat([a[k].view, b[k].view])
    assert torch.equal(both, one[k].view), f'{k}: two passes differ from one'
  assert torch.equal(sb.view[4:].cpu(), st0[4:]), 'stats[4:8] were written'
  # stats: the one-pass terms' bound, plus the rounding of every warp's atomicAdd at the scale of the running total,
  # which now starts at st0 (at most one atomic per ray)
  fo, _ = run_fwd(L, lb, inp, cfg, ld)
  dec = dict(bg_on=((1.0 - fo['acc'].view) > 0).cpu(), v_lt1=(fo['rgb'].view < 1).cpu())
  res = R.reference(inp, cfg, loss, dec)
  sv, sbd, _ = res['stats']
  want = sv + st0[:4].double()
  terms = torch.stack([(t.val.abs() + t.err).sum() for t in res['stat_terms']])
  bound = sbd + (B + 2) * R.U * (st0[:4].double().abs() + terms)
  got = sb.view[:4].cpu().double()
  assert ((got - want).abs() <= bound).all(), (got.tolist(), want.tolist(), bound.tolist())


def test_backward_deterministic(lib):
  """The interlevel gradient accumulates through shared-memory atomics: the same launch twice gives the same bits."""
  L, lb = lib
  case = (129, 300, 'prop', 'mse', 1, 'reciprocal', 'sigmoid', True, 'n', 200, 0)
  inp, cfg, loss = make(case, seed=5)
  a, sa = run_bwd(L, lb, inp, cfg, loss)
  b, sb = run_bwd(L, lb, inp, cfg, loss)
  assert torch.equal(a['d_raw_density'].view, b['d_raw_density'].view)


POINT = [(0, 3, 'sigmoid', 0, False), (1, 4, 'safe_exp', 1, True), (1000, 7, 'sigmoid', 1, False),
         (777, 3, 'safe_exp', 0, False), (MANY, 4, 'sigmoid', 1, True), (999, 4, 'safe_exp', 1, False),
         (513, 7, 'sigmoid', 0, False), (65, 3, 'sigmoid', 1, True)]


@pytest.mark.parametrize('M,ld,act,mode,tint', POINT)
def test_point_rgb(lib, M, ld, act, mode, tint):
  """mnrf_point_rgb per element against the colour walk, rows ld_rgb floats apart inside NaN padding."""
  L, lb = lib
  if M == MANY:
    M = int(lb.mnrf_num_sms()) * 16 * 256 + 37
  rng = np.random.default_rng(M + ld)
  raw = torch.tensor(rng.normal(size=(M, 3)).astype(np.float32) * 3)
  if M > 2:
    raw[:2] = torch.tensor([[100.0, -100.0, 88.5], [-1e4, 1e4, 0.0]])
  x = dict(raw_rgb=raw)
  if mode:
    x['raw_diffuse'] = torch.tensor(rng.normal(size=(M, 3)).astype(np.float32) * 2)
    if tint:
      x['raw_tint'] = torch.tensor(rng.normal(size=(M, 3)).astype(np.float32) * 2)
  cfg = dict(BASE, raydist_fn=None, opaque_background=False, rgb_activation=act, rgb_bias=-1.0 if act == 'safe_exp'
             else 0.0, rgb_padding=0.0 if act == 'safe_exp' else 0.001, rgb_mode=mode)
  buf = torch.full((M + 2, ld), float('nan'), device='cuda')
  buf[:M, :3] = raw.cuda()
  gx = {k: Guarded((M, 3), float('nan'), value=v.cuda()) for k, v in x.items() if k != 'raw_rgb'}
  out = Guarded((M, 3), float('nan'))
  out.buf[~out.mask] = SENTINEL
  out.fill = SENTINEL
  from multinerf_b200 import ops
  d = ops._cdesc(M, 1, **cfg)
  rc = lb.mnrf_point_rgb(C.byref(d), M, L.ptr(buf), ld, L.ptr(gx['raw_diffuse'].view) if 'raw_diffuse' in gx else None,
                         L.ptr(gx['raw_tint'].view) if 'raw_tint' in gx else None, L.ptr(out.view), L.stream_ptr())
  L.check(rc)
  torch.cuda.synchronize()
  assert out.untouched()
  assert torch.isnan(buf[M:]).all() and torch.isnan(buf[:M, 3:]).all() and torch.equal(buf[:M, :3].cpu(), raw)
  if M == 0:
    return
  dev = 'cuda' if M > 100000 else 'cpu'
  b = R.Running(dev)
  with torch.no_grad():
    col = R.colour_walk(b, {k: v.to(dev) for k, v in x.items()}, cfg)
    ref = R.colour(x['raw_rgb'].to(dev, torch.float64), cfg,
                   x['raw_diffuse'].to(dev, torch.float64) if 'raw_diffuse' in x else None,
                   x['raw_tint'].to(dev, torch.float64) if 'raw_tint' in x else None)
  gap = (col.c.val - ref).abs()
  bound = R.SLACK * (col.c.err + gap) + R.TINY
  frac, worst = R.check('point_rgb', out.view, ref, bound, col.unsure_lin)
  print(f'point_rgb M {M} ld {ld} {act} mode {mode} tint {tint}: live {frac:.2f} worst {worst:.2f}')


# ---- refusals on the GPU: an error before any launch, and the outputs untouched ------------------------------------

def test_refusals_leave_outputs_untouched(lib):
  L, lb = lib
  import test_composite_reference_cpu as T
  inp, cfg, loss = make((33, 8, 'fine', 'mse', 1, 'reciprocal', 'sigmoid', False, 'r', 0, 0), seed=1)
  for entry, dk, ak, msg in T.REFUSALS:
    names = ('w', 'rgb', 'dens', 'rgbs', 'acc', 'dist', 'drd', 'drgb', 'ddf', 'dti')
    outs = [torch.full((8 * 33 * 3 + 64,), SENTINEL, device='cuda') for _ in names]
    fake = {k: L.ptr(o) for k, o in zip(names, outs)}
    ins = torch.zeros(8 * 33 * 8 + 64, device='cuda')
    for e in (('fwd', 'bwd') if entry == 'both' else (entry,)):
      rc, err = T.call(L, lb, e, dk, ak, real=(L.ptr(ins), fake))
      assert rc != 0 and msg in err, (e, dk, ak, rc, err)
    torch.cuda.synchronize()
    for o in outs:
      assert (o == SENTINEL).all(), (entry, dk, ak)
