"""The Ref-NeRF stage (mnrf_refdir_fwd / mnrf_refdir_bwd) and the colourless normals stage (mnrf_normals_fwd / _bwd)
against the fp64 reference of tests/refdir_ref.py, element by element with no outlier fraction.  Needs an H100.

Every case checks normals_pred, normals, roughness, extra_dw and every slab column against their bounds in the
forward; d_grad_pred, d_raw_rough, d_raw_grad_density and the loss statistics stats[4], stats[5] in the backward; the
11 head-gradient columns bit-equal to bf16 of the kernel's own fp32 outputs and of the passed-through heads, zeros
where a head is absent and to col_end; and sentinels in the slab columns outside [col0, col_end), in the rows around
every output and in the other stats entries, which must survive.  Elements whose bound says nothing
(refdir_ref.VACUOUS) are counted per degree and held to the case's floor.  Each case prints the worst err / bound per
output (per IDE degree for the slab), the vacuous share and the grid-stride iterations it reached.
"""
import itertools
import math

import numpy as np
import pytest
import torch

import refdir_ref as RR

pytestmark = pytest.mark.gpu

SENT = -7.25e33
PAD = 37

DEFAULT = dict(M=129, S=8, pred=1, dens=1, refl=1, ide=1, ndv=1, rough=1, deg=5, bias=-1.0, om=0.1, pm=3e-4, oop=1,
               col0=64, col_end=None, ld=None, kappa=None, gscale=1.0, rgd_scale=30.0, clamp_rows=True,
               heads=('density', 'diffuse'), extra_dw=True, floor=0.9, iters=1)
# name: overrides of DEFAULT.  col_end None: the encoding and 11 head columns rounded up to 8, plus 5 pad columns;
# ld None: col_end.  kappa (lo, hi): roughness drawn log-uniform in [lo, hi].  M None: 2 * blocks * 128 + 37.
CASES = {
    'refnerf': dict(M=296, clamp_rows=False, col_end=192),                      # the two configurations of the
    'viewdir-pe-normals': dict(M=296, ide=0, refl=0, deg=4, clamp_rows=False, col_end=192),   # former kernel test
    'ide-deg1': dict(deg=1), 'ide-deg2': dict(deg=2), 'ide-deg3': dict(deg=3), 'ide-deg4': dict(deg=4),
    'kappa-sweep': dict(kappa=(1e-4, 5.0), M=512, floor=0.85),
    'pe-deg0': dict(ide=0, deg=0), 'pe-deg1': dict(ide=0, deg=1), 'pe-deg4': dict(ide=0, deg=4, refl=0),
    'pe-deg4-refl': dict(ide=0, deg=4), 'pe-deg10': dict(ide=0, deg=10, refl=0), 'pe-deg10-refl': dict(ide=0, deg=10),
    'S1': dict(S=1), 'S7': dict(S=7), 'S64': dict(S=64, M=640),
    'M1': dict(M=1, clamp_rows=False), 'M127': dict(M=127), 'M128': dict(M=128),
    'M-iter': dict(M=None, deg=3, iters=2),
    'col0-0': dict(col0=0), 'col0-3': dict(col0=3), 'col0-256': dict(col0=256),
    'exact-width-ld': dict(col0=5, col_end=5 + 73, ld=5 + 73 + 19),
    'grad-1e-6': dict(gscale=1e-6), 'grad-1e6': dict(gscale=1e6, rgd_scale=1.0),
    'density-normals': dict(pred=0, om=0.1, oop=0, pm=0.0), 'pe-refl-no-rough': dict(ide=0, rough=0, deg=4),
    'no-ndv-no-loss': dict(ndv=0, om=0.0, pm=0.0, extra_dw=False), 'orient-only': dict(pm=0.0),
    'prednorm-only': dict(om=0.0), 'orient-density': dict(oop=0),
    'heads-tint': dict(heads=('tint',)), 'heads-all': dict(heads=('density', 'diffuse', 'tint')),
    'no-bottleneck': dict(col0=0, heads=()),
}


def case(name):
  return dict(DEFAULT, **CASES.get(name, {}))


def flags(c):
  return dict(use_pred_normals=c['pred'], use_density_normals=c['dens'], use_reflections=c['refl'],
              use_ide=c['ide'], use_n_dot_v=c['ndv'], use_roughness=c['rough'], deg_view=c['deg'],
              bias=float(np.float32(c['bias'])), orient_mult=float(np.float32(c['om'] / 37)),
              prednorm_mult=float(np.float32(c['pm'] / 37)), orient_on_pred=c['oop'],
              col0=c['col0'], col_end=c['col_end'])


def enc_width(c):
  return (RR.ide_degree_of(c['deg']).numel() if c['ide'] else 3 + 6 * c['deg']) + c['ndv']


def make_inputs(c, M, seed):
  """(x, f): the fp32 CPU inputs of both entry points and the descriptor / loss fields of a case at M samples."""
  from multinerf_b200 import ref_utils
  from oracle import o_coord
  rng = np.random.default_rng(seed)
  S = c['S']
  B = -(-M // S)
  c = dict(c)
  if c['col_end'] is None:
    c['col_end'] = c['col0'] + (max(enc_width(c), 11) + 7) // 8 * 8 + 5
  f = flags(c)
  f['col_end'] = c['col_end']
  f['ld'] = c['ld'] or c['col_end']
  x = type('X', (), {})()
  v = rng.normal(size=(B, 3))
  x.viewdirs = torch.tensor(v / np.linalg.norm(v, axis=-1, keepdims=True), dtype=torch.float32)
  x.v = x.viewdirs[torch.arange(M) // S]
  gs = c['gscale']
  gp = rng.normal(size=(M, 3)) * gs
  rgd = rng.normal(size=(3, M)) * c['rgd_scale'] * gs
  if c['clamp_rows'] and M >= 3:
    # clamped norms: zero, tiny, and |g|^2 == eps exactly (2^-24 + 2^-24 in every order)
    for row, g in enumerate(([0.0, 0.0, 0.0], [1e-5, -2e-5, 0.5e-5], [2.0 ** -12, 2.0 ** -12, 0.0])):
      gp[row] = g
      rgd[:, (row + 1) % M] = g
  x.gp = torch.tensor(gp, dtype=torch.float32) if c['pred'] else None
  x.rgd = torch.tensor(rgd, dtype=torch.float32) if c['dens'] else None
  if c['kappa']:
    k = np.exp(rng.uniform(np.log(c['kappa'][0]), np.log(c['kappa'][1]), M))
    rr = np.log(np.expm1(k)) - f['bias']
  else:
    rr = rng.normal(size=M)
  x.rr = torch.tensor(rr, dtype=torch.float32) if c['rough'] else None
  x.w = torch.tensor(rng.uniform(0, 0.2, M), dtype=torch.float32)
  W = f['col_end'] - f['col0']
  x.gin = torch.tensor(rng.normal(size=(M, W)), dtype=torch.float32).to(torch.bfloat16).float()
  x.heads = {h: torch.tensor(rng.normal(size=(M,) if h == 'density' else (M, 3)), dtype=torch.float32)
             for h in c['heads']}
  if c['ide']:
    m, l, mat = ref_utils.ide_tables(c['deg'])
    x.m, x.l = torch.tensor(m), torch.tensor(l)
    x.mat = torch.tensor(mat, dtype=torch.float32)
    x.mat64 = torch.tensor(o_coord.ide_tables(c['deg'])[1], dtype=torch.float64)
  else:
    x.m = x.l = x.mat = x.mat64 = None
  return x, f


@pytest.fixture(scope='module')
def ops():
  from multinerf_b200 import lib, ops as _ops
  lib.require_device()
  return _ops


def _guard(n, dtype=torch.float32):
  """A flat view of n elements between PAD sentinels: (view, buffer)."""
  buf = torch.full((n + 2 * PAD,), SENT, dtype=dtype, device='cuda')
  return buf[PAD:PAD + n], buf


def _intact(buf):
  return bool((buf[:PAD] == SENT).all() and (buf[-PAD:] == SENT).all())


def _slab(M, ld, fill):
  """A [M, ld] bf16 slab with 3 sentinel rows (7.0) before and after: (view, buffer)."""
  buf = torch.full((M + 6, ld), 7.0, dtype=torch.bfloat16, device='cuda')
  buf[3:3 + M] = fill
  return buf[3:3 + M], buf


def _ratio(got, ref, bound, vac):
  r = (got.double().cpu() - ref.double().cpu()).abs() / bound.cpu()
  return torch.where(vac.cpu(), torch.zeros_like(r), r.nan_to_num(nan=math.inf))


def run_case(ops, name, c, M, sms, seed, report=True):
  from multinerf_b200 import lib as L
  x, f = make_inputs(c, M, seed)
  W, ld, col0, col_end = f['col_end'] - f['col0'], f['ld'], f['col0'], f['col_end']
  p = RR.plan(M, sms)
  assert p.iters >= c['iters'], (name, p.iters)
  dev = 'cuda' if M > 4096 else 'cpu'
  ref = RR.reference(x, f, num_sms=sms, device=dev)
  assert not ref.unsure.any(), (name, 'a clamp the fp32 orders disagree on')
  desc = ops.refdir_desc(M, c['S'], use_pred_normals=c['pred'], use_density_normals=c['dens'],
                         use_reflections=c['refl'], use_ide=c['ide'], use_n_dot_v=c['ndv'], use_roughness=c['rough'],
                         deg_view=c['deg'], ide_n=0 if x.m is None else len(x.m), roughness_bias=f['bias'], ld=ld,
                         col0=col0, col_end=col_end)
  cu = lambda t: None if t is None else t.contiguous().cuda()
  mat = cu(x.mat)
  ml = None if x.m is None else torch.stack([x.m, x.l]).int().cuda()
  gp, rr, rgd, vd, w = cu(x.gp), cu(x.rr), cu(x.rgd), cu(x.viewdirs), cu(x.w)
  outs = {k: _guard(n) for k, n in (('normals_pred', 3 * M), ('normals', 3 * M), ('roughness', M), ('extra_dw', M))}
  slab, sbuf = _slab(M, ld, 7.0)
  ops.refdir_fwd(desc, mat, ml, gp, rr, rgd, vd, outs['normals_pred'][0] if c['pred'] else None,
                 outs['normals'][0] if c['dens'] else None, outs['roughness'][0] if c['rough'] else None, slab,
                 f['orient_mult'], f['prednorm_mult'], c['oop'], outs['extra_dw'][0] if c['extra_dw'] else None)
  torch.cuda.synchronize()
  lines = []
  for k, (view, buf) in outs.items():
    assert _intact(buf), (name, 'wrote outside', k)
    on = {'normals_pred': c['pred'], 'normals': c['dens'], 'roughness': c['rough'], 'extra_dw': c['extra_dw']}[k]
    if not on:
      assert (view == SENT).all(), (name, k, 'written while off')
      continue
    refv = getattr(ref, k)
    r = _ratio(view.view(refv.shape), refv, getattr(ref, k + '_bound'), getattr(ref, k + '_vacuous'))
    lines.append(f'{k} {float(r.max()):.2f}')
    assert float(r.max()) <= 1, (name, k, float(r.max()), int(r.argmax()))
  got = sbuf.float().cpu()
  assert (got[:3] == 7).all() and (got[3 + M:] == 7).all(), (name, 'slab rows outside M')
  assert (got[3:3 + M, :col0] == 7).all() and (got[3:3 + M, col_end:] == 7).all(), (name, 'slab columns outside')
  rs = _ratio(got[3:3 + M, col0:col_end], ref.slab, ref.slab_bound, ref.slab_vacuous)
  assert float(rs.max()) <= 1, (name, 'slab', float(rs.max()), np.unravel_index(int(rs.argmax()), rs.shape))
  ne = ref.enc_width
  if c['ide']:
    dg = RR.ide_degree_of(c['deg'], c['ndv'])
    per = ' '.join(f'l={l}: {float(rs[:, :ne][:, dg == l].max()):.2f} (vacuous '
                   f'{float(ref.slab_vacuous[:, :ne][:, dg == l].double().mean()):.3f})'
                   for l in sorted(set(dg.tolist()) - {-1}))
  else:
    dg = RR.pe_degree_of(c['deg'], c['ndv'])
    per = f'{float(rs.max()):.2f}'
  lines.append(f'slab {per}')
  checked = 1 - float(ref.slab_vacuous[:, :ne].double().mean())
  assert checked >= c['floor'], (name, 'slab checked share', checked)

  # backward
  dsl, dbuf = _slab(M, ld, 7.0)
  dsl[:, col0:col_end] = x.gin.to(torch.bfloat16).cuda()
  bo = {k: _guard(n) for k, n in (('d_grad_pred', 3 * M), ('d_raw_rough', M), ('d_raw_grad_density', 3 * M))}
  stats = torch.full((8,), SENT, device='cuda')
  stats[4:6] = 0
  hd = {h: cu(t) for h, t in x.heads.items()}
  ops.refdir_bwd(desc, mat, ml, gp, rr, rgd, vd, w, dsl, f['orient_mult'], f['prednorm_mult'], c['oop'],
                 hd.get('density'), hd.get('diffuse'), hd.get('tint'),
                 bo['d_grad_pred'][0] if c['pred'] else None, bo['d_raw_rough'][0] if c['rough'] else None,
                 bo['d_raw_grad_density'][0] if c['dens'] else None, stats)
  torch.cuda.synchronize()
  for k, (view, buf) in bo.items():
    assert _intact(buf), (name, 'wrote outside', k)
    on = {'d_grad_pred': c['pred'], 'd_raw_rough': c['rough'], 'd_raw_grad_density': c['dens']}[k]
    if not on:
      assert (view == SENT).all(), (name, k, 'written while off')
      continue
    refv = getattr(ref, k)
    r = _ratio(view.view(refv.shape), refv, getattr(ref, k + '_bound'), getattr(ref, k + '_vacuous'))
    vac = float(getattr(ref, k + '_vacuous').double().mean())
    lines.append(f'{k} {float(r.max()):.2f} (vacuous {vac:.3f})')
    assert float(r.max()) <= 1, (name, k, float(r.max()), int(r.argmax()))
    assert vac <= 1 - c['floor'], (name, k, 'vacuous share', vac)
  st = stats.cpu()
  assert (st[:4] == SENT).all() and (st[6:] == SENT).all(), (name, 'stats outside [4:6]')
  st = st.double()
  for i, k in ((4, 'stats_or'), (5, 'stats_pn')):
    r = float((st[i] - getattr(ref, k)).abs() / getattr(ref, k + '_bound'))
    lines.append(f'{k} {r:.2f}')
    assert r <= 1, (name, k, float(st[i]), float(getattr(ref, k)))
  db = dbuf.float().cpu()
  assert (db[:3] == 7).all() and (db[3 + M:] == 7).all(), (name, 'd_slab rows outside M')
  assert (db[3:3 + M, :col0] == 7).all() and (db[3:3 + M, col_end:] == 7).all(), (name, 'd_slab columns outside')
  want = RR.head_slab(W, x.heads.get('density'), bo['d_grad_pred'][0].view(M, 3) if c['pred'] else None,
                      x.heads.get('diffuse'), x.heads.get('tint'), bo['d_raw_rough'][0] if c['rough'] else None)
  assert torch.equal(db[3:3 + M, col0:col_end], want), (name, 'head slab')
  if report:
    print(f'\n{name}: M {M} S {c["S"]} blocks {p.blocks} grid-stride iterations {p.iters} | worst err/bound ' +
          ' | '.join(lines))
  return ref


def _sms():
  from multinerf_b200 import lib as L
  return L.load().mnrf_num_sms()


@pytest.mark.parametrize('name', list(CASES))
def test_refdir_case(ops, name):
  c = case(name)
  sms = _sms()
  M = c['M'] or 2 * RR.plan(10 ** 9, sms).blocks * 128 + 37
  ref = run_case(ops, name, c, M, sms, seed=sum(name.encode()))
  if c['kappa']:
    # the l = 8 and l = 16 terms are alive: a real share of their slab elements exceeds 0.05
    dg = RR.ide_degree_of(c['deg'], c['ndv'])
    for l in (8, 16):
      alive = float((ref.slab[:, :dg.numel()][:, dg == l].abs() > 0.05).double().mean())
      print(f'{name}: share of l = {l} slab elements above 0.05: {alive:.3f}')
      assert alive > 0.2, (name, l, alive)


def sweep():
  """Every flag combination the C ABI accepts x orient_on_pred x {no loss, orientation, predicted normal, both}."""
  for pred, dens, refl, ide, ndv, rough in itertools.product((0, 1), repeat=6):
    if (ide and not rough) or ((refl or ndv) and not (pred or dens)):
      continue
    for oop, (om, pm) in itertools.product((0, 1), ((0.0, 0.0), (0.1, 0.0), (0.0, 3e-4), (0.1, 3e-4))):
      if (om and not (pred if oop else dens)) or (pm and not (pred and dens)):
        continue
      yield dict(pred=pred, dens=dens, refl=refl, ide=ide, ndv=ndv, rough=rough, oop=oop, om=om, pm=pm,
                 deg=3 if ide else 2)


def test_refdir_sweep(ops):
  sms = _sms()
  n = 0
  for i, over in enumerate(sweep()):
    c = dict(DEFAULT, **over)
    run_case(ops, f'sweep {over}', c, 129, sms, seed=i, report=False)
    n += 1
  print(f'\nsweep: {n} combinations, every element within its bound')
  assert n >= 100


def test_refdir_per_degree_gradients(ops):
  """The adjoint of one IDE degree at a time (d_slab nonzero on that degree's columns only), roughness from 1e-4 to
  5: worst err / bound of d_grad_pred, d_raw_rough and d_raw_grad_density per degree."""
  from multinerf_b200 import lib as L
  sms = _sms()
  c = dict(DEFAULT, kappa=(1e-4, 5.0), M=256, om=0.0, pm=0.0, heads=())
  x0, f = make_inputs(c, c['M'], 5)
  dg = RR.ide_degree_of(5, True)
  for l in (1, 2, 4, 8, 16):
    x, _ = make_inputs(c, c['M'], 5)
    keep = torch.zeros(x.gin.shape[1], dtype=torch.bool)
    keep[:dg.numel()] = dg == l
    x.gin = torch.where(keep, x.gin, torch.zeros_like(x.gin))
    ref = RR.reference(x, f, num_sms=sms)
    desc = ops.refdir_desc(c['M'], c['S'], use_pred_normals=1, use_density_normals=1, use_reflections=1, use_ide=1,
                           use_n_dot_v=1, use_roughness=1, deg_view=5, ide_n=len(x.m), roughness_bias=f['bias'],
                           ld=f['ld'], col0=f['col0'], col_end=f['col_end'])
    d = torch.zeros(c['M'], f['ld'], dtype=torch.bfloat16, device='cuda')
    d[:, f['col0']:f['col_end']] = x.gin.to(torch.bfloat16).cuda()
    out = [torch.empty(c['M'], 3, device='cuda'), torch.empty(c['M'], device='cuda'), torch.empty(3, c['M'], device='cuda')]
    stats = torch.zeros(8, device='cuda')
    ops.refdir_bwd(desc, x.mat.cuda(), torch.stack([x.m, x.l]).int().cuda(), x.gp.cuda(), x.rr.cuda(), x.rgd.cuda(),
                   x.viewdirs.cuda(), x.w.cuda(), d, 0.0, 0.0, 1, None, None, None, *out, stats)
    torch.cuda.synchronize()
    line = []
    for k, g in zip(('d_grad_pred', 'd_raw_rough', 'd_raw_grad_density'), out):
      r = _ratio(g.cpu(), getattr(ref, k), getattr(ref, k + '_bound'), getattr(ref, k + '_vacuous'))
      vac = float(getattr(ref, k + '_vacuous').double().mean())
      line.append(f'{k} {float(r.max()):.2f} (vacuous {vac:.3f})')
      assert float(r.max()) <= 1, (l, k, float(r.max()))
      # l = 16 from monomials with coefficients up to 9e4: at small roughness a third of its d_grad_pred elements
      # have a bound above a quarter of their value
      assert vac <= (0.5 if l == 16 else 0.15), (l, k, vac)
    print(f'\nIDE degree l = {l} adjoint: worst err/bound ' + ' | '.join(line))


def test_refdir_col_end_one_short_is_refused(ops):
  """A slab physically wide enough whose col_end is one column short of the encoding: refused before any launch,
  the sentinels beyond col_end untouched."""
  from multinerf_b200 import lib as L
  c = case('refnerf')
  x, f = make_inputs(c, 64, 1)
  ne = enc_width(c)
  desc = ops.refdir_desc(64, 8, use_pred_normals=1, use_density_normals=1, use_reflections=1, use_ide=1,
                         use_n_dot_v=1, use_roughness=1, deg_view=5, ide_n=len(x.m), roughness_bias=-1.0, ld=160,
                         col0=64, col_end=64 + ne - 1)
  slab = torch.full((64, 160), 7.0, dtype=torch.bfloat16, device='cuda')
  args = (x.mat.cuda(), torch.stack([x.m, x.l]).int().cuda(), x.gp.cuda(), x.rr.cuda(), x.rgd.cuda(),
          x.viewdirs.cuda())
  with pytest.raises(L.MnrfError, match='must hold'):
    ops.refdir_fwd(desc, *args, torch.empty(64, 3, device='cuda'), torch.empty(64, 3, device='cuda'),
                   torch.empty(64, device='cuda'), slab)
  with pytest.raises(L.MnrfError, match='must hold'):
    ops.refdir_bwd(desc, *args, x.w.cuda(), slab, 0.0, 0.0, 1, None, None, None, torch.empty(64, 3, device='cuda'),
                   torch.empty(64, device='cuda'), torch.empty(3, 64, device='cuda'), torch.zeros(8, device='cuda'))
  torch.cuda.synchronize()
  assert (slab == 7).all(), 'a refused call wrote its slab'


@pytest.mark.parametrize('ld_raw', [1, 4])
def test_normals_stage(ops, ld_raw):
  """mnrf_normals_fwd / _bwd: every pointer combination the host accepts, d_raw_density / d_raw_rgb at a row pitch
  of ld_raw, head_grads 4 and 8 wide, against the same reference; stats untouched when the losses are off."""
  sms = _sms()
  M, S = 300, 6
  n = 0
  for gp_on, rgd_on in ((1, 1), (1, 0), (0, 1)):
    for (om, pm), oop in itertools.product(((0.0, 0.0), (0.1, 0.0), (0.0, 3e-4), (0.1, 3e-4)), (0, 1)):
      if (om and not (gp_on if oop else rgd_on)) or (pm and not (gp_on and rgd_on)):
        continue
      for hw, rgb in ((0, False), (4, False), (8, False), (8, True)):
        if hw and not gp_on:
          continue
        c = dict(DEFAULT, S=S, pred=gp_on, dens=rgd_on, refl=0, ide=0, ndv=0, rough=0, deg=0, om=om, pm=pm,
                 oop=oop, heads=())
        x, f = make_inputs(c, M, n)
        ref = RR.reference(x, dict(f, col_end=f['col0'] + 11), num_sms=sms)
        cu = lambda t: None if t is None else t.contiguous().cuda()
        npd, nbuf = _guard(3 * M)
        nd, dbuf = _guard(3 * M)
        edw, ebuf = _guard(M)
        ops.normals_fwd(M, S, cu(x.gp), cu(x.rgd), cu(x.viewdirs), npd if gp_on else None, nd if rgd_on else None,
                        f['orient_mult'], f['prednorm_mult'], oop, edw)
        raw = torch.tensor(np.random.default_rng(n).normal(size=(M, ld_raw * 4)), dtype=torch.float32).cuda()
        d_rd = raw[:, 0] if ld_raw == 4 else raw[:, 0].contiguous()
        d_rgb = raw[:, 1:4] if ld_raw == 4 else None
        dgp, gbuf = _guard(3 * M)
        drgd, rbuf = _guard(3 * M)
        stats = torch.full((8,), SENT, device='cuda')
        losses = om > 0 or pm > 0
        if losses:
          stats[4:6] = 0
        hg = torch.full((M + 2, max(hw, 1) + 4), 7.0, dtype=torch.bfloat16, device='cuda') if hw else None
        ops.normals_bwd(M, S, cu(x.gp), cu(x.rgd), cu(x.viewdirs), cu(x.w), f['orient_mult'], f['prednorm_mult'],
                        oop, d_rd if hw else None, dgp if gp_on else None, drgd if rgd_on else None,
                        head_grads=hg[1:1 + M, :hw] if hw else None, stats=stats,
                        d_raw_rgb=d_rgb if (rgb and ld_raw == 4) else None)
        torch.cuda.synchronize()
        for buf in (nbuf, dbuf, ebuf, gbuf, rbuf):
          assert _intact(buf)
        checks = [('extra_dw', edw)]
        if gp_on:
          checks += [('normals_pred', npd.view(M, 3)), ('d_grad_pred', dgp.view(M, 3))]
        if rgd_on:
          checks += [('normals', nd.view(M, 3)), ('d_raw_grad_density', drgd.view(3, M))]
        for k, g in checks:
          r = _ratio(g, getattr(ref, k), getattr(ref, k + '_bound'), getattr(ref, k + '_vacuous'))
          assert float(r.max()) <= 1, (gp_on, rgd_on, om, pm, oop, k, float(r.max()))
        st = stats.cpu()
        assert (st[:4] == SENT).all() and (st[6:] == SENT).all()
        st = st.double()
        if losses:
          for i, k in ((4, 'stats_or'), (5, 'stats_pn')):
            assert float((st[i] - getattr(ref, k)).abs()) <= float(getattr(ref, k + '_bound')), (k, float(st[i]))
        else:
          assert (stats.cpu()[4:6] == SENT).all(), 'stats written with the losses off'
        if hw:
          h = hg.float().cpu()
          assert (h[0] == 7).all() and (h[-1] == 7).all() and (h[1:1 + M, hw:] == 7).all(), 'outside head_grads'
          want = torch.zeros(M, hw)
          want[:, 0] = d_rd.cpu()
          want[:, 1:4] = dgp.view(M, 3).cpu()
          if rgb and ld_raw == 4:
            want[:, 4:7] = d_rgb.cpu()
          want = want.to(torch.bfloat16).float()
          if hw == 8 and not (rgb and ld_raw == 4):
            want[:, 4:] = 7.0           # columns 4..7 are written only with d_raw_rgb
          assert torch.equal(h[1:1 + M, :hw], want), (hw, rgb, ld_raw, 'head_grads')
        n += 1
  print(f'\nnormals stage, ld_raw {ld_raw}: {n} pointer combinations within their bounds')
