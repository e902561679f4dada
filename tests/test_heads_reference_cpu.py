"""The fp64 checker of tests/heads_ref.py is sound and sensitive.  CPU only.

Soundness: the arithmetic of csrc/heads.cu emulated in fp32 -- per-lane register partial sums, the 4-, 8-, 16- and
32-lane butterflies of the forward, the per-warp sums, shared-memory atomics and global atomics of the backward in
several orders, fp32 de then round to nearest even into bf16, and the clip+Adam sequence with perturbed powf / sqrtf
-- lands inside the bound for every element.
Sensitivity: each small mutation a launch or indexing bug would make is flagged.
Anchor: the fp64 clip+Adam reference agrees with the oracle's clipping and optax.adam on fp64 inputs.
"""
import pytest
import torch

import gemm_ref as G
import heads_ref as H

ORDERS = ('sequential', 'reversed', 'pairwise', 'per_block')


def _bf16(x):
  return x.to(torch.bfloat16)


def _sum32(t, order, dim=0):
  """fp32 sum of t (fp32) along dim in `order`, rounding after every addition."""
  t = t.float().movedim(dim, 0)
  if order == 'pairwise':
    while t.shape[0] > 1:
      if t.shape[0] % 2:
        t = torch.cat([t, torch.zeros_like(t[:1])])
      t = t[0::2] + t[1::2]
    return t[0] if t.shape[0] else torch.zeros(t.shape[1:])
  acc = torch.zeros(t.shape[1:])
  for i in (range(t.shape[0]) if order != 'reversed' else reversed(range(t.shape[0]))):
    acc = acc + t[i]
  return acc


def _tree32(terms, init, rpb, order):
  """sum over the rows of terms [M, ...] (fp32) onto init the way the backward kernels add them: each block's rows
  [b rpb, (b + 1) rpb) go to eight warps round robin, each warp sums its rows in registers, the warps' partials meet
  in shared-memory atomics, and the blocks' in global atomics on init, in `order` (per_block: sequential within a
  block, the blocks last to first)."""
  m = terms.shape[0]
  blocks = []
  for b0 in range(0, m, rpb):
    blk = terms[b0:b0 + rpb]
    warps = torch.stack([_sum32(blk[w::8], 'sequential') if blk[w::8].shape[0] else torch.zeros(blk.shape[1:])
                         for w in range(8)])
    blocks.append(_sum32(warps, 'sequential' if order == 'per_block' else order))
  parts = torch.stack([init.float()] + (blocks[::-1] if order == 'per_block' else blocks))
  return _sum32(parts, 'sequential' if order == 'per_block' else order)


def _operands(seed, m, k, n_out):
  gen = torch.Generator().manual_seed(seed)
  x = _bf16(torch.randn(m, k, generator=gen) * torch.exp2(torch.randint(-4, 5, (m, k), generator=gen).float()))
  w = _bf16(torch.randn(n_out, k, generator=gen) / k ** 0.5)
  draw = torch.randn(m, n_out, generator=gen) * torch.exp2(torch.randint(-3, 4, (m, n_out), generator=gen).float())
  return x, w, draw, gen


# ---------------------------------------------------------------------------------------------- forward
def _emulate_fwd(x, w, b, lanes, order):
  """head_fwd in fp32: lane j sums the 8-column chunks j, j + lanes, ... (pairs of exact products, in `order` over
  its chunks), then the xor butterfly over `lanes` lanes, then the bias."""
  p = x.float()[:, None, :] * w.float()[None, :, :]                  # [M, n_out, K], exact
  m, n, k = p.shape
  pairs = p.reshape(m, n, k // 2, 2).sum(-1)                          # lo * lo' + hi * hi', one rounding
  chunks = pairs.reshape(m, n, k // 8, 4)
  lane_acc = []
  for j in range(lanes):
    mine = chunks[:, :, j::lanes].reshape(m, n, -1)
    lane_acc.append(_sum32(mine, order, dim=2) if mine.shape[-1] else torch.zeros(m, n))
  acc = torch.stack(lane_acc)                                         # [lanes, M, n_out]
  sh = lanes // 2
  while sh:
    idx = torch.arange(lanes) ^ sh
    acc = acc + acc[idx]
    sh //= 2
  out = acc[0]
  return out + b if b is not None else out


@pytest.mark.parametrize('order', ('sequential', 'reversed', 'pairwise'))
@pytest.mark.parametrize('k,lanes', [(64, 8), (128, 16), (256, 32), (32, 4), (192, 32), (1024, 32), (1536, 32)])
def test_fwd_emulation_inside_bound(k, lanes, order):
  for n_out in (1, 4):
    x, w, _, gen = _operands(k + n_out, 37, k, n_out)
    h = k // 2
    x[:3, h:] = -x[:3, :h]          # rows whose products cancel exactly: the bound is all accumulation error
    w[:, h:] = w[:, :h]
    for b in (None, torch.randn(n_out, generator=gen)):
      val, bound = H.head_fwd(x, w, b)
      G.check(_emulate_fwd(x, w, b, lanes, order), val, bound, f'fwd K={k} lanes={lanes} {order}')


# ---------------------------------------------------------------------------------------------- backward
def _d1_32(code, z, gen):
  """a'(z) with a random relative error of the fast __expf / __fdividef sigmoid."""
  s = torch.sigmoid(z.double())
  d = (torch.rand(z.shape, generator=gen, dtype=torch.float64) * 2 - 1) * (2 + 1.2 * z.double().abs()) * 2.0 ** -23
  s = (s * (1 + d)).float()
  return s * (1 + z.float() * (1 - s)) if code == G.SILU else s


def _emulate_bwd(x, w, draw, *, act, z, dx_cols, split, inits, rpb, order, gen, lanes=1):
  """mnrf_head_bwd in fp32.  Returns dict of outputs (dx, dx2 bf16; dxsum, dw, dw2, db fp32) and the fp32 dx."""
  m, k = x.shape
  n_out = w.shape[0]
  de = torch.zeros(m, k)
  for o in range(n_out):
    de = de + draw[:, o:o + 1] * w[o].float()[None, :]
  dxc = de[:, :dx_cols]
  if act == G.RELU:
    dxc = torch.where(x[:, :dx_cols].float() > 0, dxc, torch.zeros_like(dxc))
  elif act in (G.SOFTPLUS, G.SILU):
    dxc = dxc * _d1_32(act, z[:, :dx_cols], gen)
  out = {'dx': _bf16(dxc)}
  if dx_cols < k:
    out['dx2'] = _bf16(de[:, dx_cols:])
  out['dxsum'] = _tree32(dxc, inits['dxsum'], rpb, order)
  prod = draw[:, None, :] * x.float()[:, :, None]                     # [M, K, n_out], rounded products
  dw = _tree32(prod, inits['dw'], rpb, order)
  out['dw'], out['dw2'] = dw[:, :split], dw[:, split:]
  out['db'] = _tree32(draw * lanes, inits['db'], rpb, order)
  return out, dxc


BWD = [  # (M, K, n_out, act, dx_cols, split, rpb)
    (64, 64, 1, G.NONE, 0, 0, 16), (77, 128, 3, G.RELU, 0, 0, 512), (300, 256, 4, G.RELU, 0, 1, 40),
    (129, 192, 2, G.SOFTPLUS, 0, 0, 8), (45, 320, 4, G.SILU, 256, 2, 9), (33, 1024, 3, G.RELU, 1016, 2, 5),
    (17, 1536, 1, G.SILU, 0, 0, 3), (600, 64, 4, G.NONE, 32, 3, 64)]


@pytest.mark.parametrize('order', ORDERS)
@pytest.mark.parametrize('m,k,n_out,act,dx_cols,split,rpb', BWD)
def test_bwd_emulation_inside_bound(m, k, n_out, act, dx_cols, split, rpb, order):
  x, w, draw, gen = _operands(m + k + n_out + act, m, k, n_out)
  cols = dx_cols or k
  z = _bf16(torch.randn(m, cols, generator=gen) * 3) if act in (G.SOFTPLUS, G.SILU) else None
  inits = dict(dxsum=torch.randn(cols, generator=gen), dw=torch.randn(k, n_out, generator=gen),
               db=torch.randn(n_out, generator=gen))
  sp = split if 0 < split < n_out else n_out
  got, _ = _emulate_bwd(x, w, draw, act=act, z=z, dx_cols=cols, split=sp, inits=inits, rpb=rpb, order=order, gen=gen)
  ref = H.head_bwd(x, w, draw, act=act, z=z, dx_cols=dx_cols, dw_split=split, dw_init=inits['dw'],
                   db_init=inits['db'], dxsum_init=inits['dxsum'])
  assert set(ref) == {'dx', 'dxsum', 'dw', 'db'} | ({'dx2'} if cols < k else set()) | ({'dw2'} if sp < n_out else set())
  for name, (val, bound) in ref.items():
    G.check(got[name], val, bound, f'{name} {order}')


def test_colsum_emulation_inside_bound():
  gen = torch.Generator().manual_seed(3)
  x = _bf16(torch.randn(700, 24, generator=gen) * 8)
  init = torch.randn(24, generator=gen)
  val, bound = H.colsum(x, init)
  for order in ORDERS:
    for rpb in (1, 11, 64, 700):
      G.check(_tree32(x.float(), init, rpb, order), val, bound, f'colsum {order} rpb={rpb}')


# ---------------------------------------------------------------------------------------------- sensitivity
def _flagged(got, value, bound):
  try:
    G.check(got, value, bound, 'mutation')
  except AssertionError:
    return True
  return False


@pytest.fixture(scope='module')
def bwd_case():
  m, k, n_out, rpb = 512, 128, 3, 64
  x, w, draw, gen = _operands(21, m, k, n_out)
  inits = dict(dxsum=torch.randn(96, generator=gen), dw=torch.randn(k, n_out, generator=gen),
               db=torch.randn(n_out, generator=gen))
  kw = dict(act=G.RELU, z=None, dx_cols=96, split=2, inits=inits, rpb=rpb, order='sequential', gen=gen)
  got, dxc = _emulate_bwd(x, w, draw, **kw)
  ref = H.head_bwd(x, w, draw, act=G.RELU, dx_cols=96, dw_split=2, dw_init=inits['dw'], db_init=inits['db'],
                   dxsum_init=inits['dxsum'])
  for name, (val, bound) in ref.items():
    G.check(got[name], val, bound, f'unmutated {name}')
  return dict(x=x, w=w, draw=draw, kw=kw, got=got, dxc=dxc, ref=ref, rpb=rpb)


def test_flags_row_dropped_at_block_boundary(bwd_case):
  c = bwd_case
  keep = torch.ones(c['x'].shape[0], dtype=torch.bool)
  keep[c['rpb'] - 1] = False                 # m_end one short in the first block
  got, _ = _emulate_bwd(c['x'][keep], c['w'], c['draw'][keep], **c['kw'])
  for name in ('dw', 'dw2', 'db', 'dxsum'):
    assert _flagged(got[name], *c['ref'][name]), name


def test_flags_db_once_per_lane(bwd_case):
  c = bwd_case
  got, _ = _emulate_bwd(c['x'], c['w'], c['draw'], lanes=16, **c['kw'])
  assert _flagged(got['db'], *c['ref']['db'])


def test_flags_dw_transposed(bwd_case):
  c = bwd_case
  k = c['x'].shape[0 + 1]
  full = torch.cat([c['got']['dw'], c['got']['dw2']], 1)            # [K, n_out]
  bad = full.T.contiguous().reshape(k, 3)                              # written [n_out, K] into a [K, n_out] buffer
  assert _flagged(bad[:, :2], *c['ref']['dw'])


@pytest.mark.parametrize('shift', [1, -1])
def test_flags_dw_split_off_by_one(bwd_case, shift):
  c = bwd_case
  k = c['x'].shape[1]
  full = torch.cat([c['got']['dw'], c['got']['dw2']], 1)
  split, wrong = 2, 2 + shift
  dw = torch.full((k * split + 2 * k,), float('nan'))
  dw2 = torch.full((k * (3 - split) + 2 * k,), float('nan'))
  for kk in range(k):
    for o in range(3):                       # csrc/heads.cu dw_at with the wrong split
      if o < wrong:
        dw[kk * wrong + o] = full[kk, o]
      else:
        dw2[kk * (3 - wrong) + o - wrong] = full[kk, o]
  bad_dw, bad_dw2 = dw[:k * split].reshape(k, split), dw2[:k * (3 - split)].reshape(k, 3 - split)
  assert _flagged(bad_dw.nan_to_num(1e30), *c['ref']['dw']) or _flagged(bad_dw2.nan_to_num(1e30), *c['ref']['dw2'])


def test_flags_dxsum_of_rounded_or_unmasked_dx():
  m, k, rpb = 64, 64, 8
  x, w, draw, gen = _operands(23, m, k, 2)
  init = torch.zeros(k)
  ref = H.head_bwd(x, w, draw, act=G.RELU, dxsum_init=init)
  _, dxc = _emulate_bwd(x, w, draw, act=G.RELU, z=None, dx_cols=k, split=2,
                        inits=dict(dxsum=init, dw=torch.zeros(k, 2), db=torch.zeros(2)), rpb=rpb, order='sequential',
                        gen=gen)
  G.check(_tree32(dxc, init, rpb, 'sequential'), *ref['dxsum'], 'unmutated')
  assert _flagged(_tree32(_bf16(dxc).float(), init, rpb, 'sequential'), *ref['dxsum'])
  de = draw.float() @ w.float()
  assert _flagged(_tree32(de, init, rpb, 'sequential'), *ref['dxsum'])


def test_flags_masked_dx2(bwd_case):
  c = bwd_case
  x = c['x']
  bad = torch.where(x[:, 96:].float() > 0, c['got']['dx2'].float(), torch.zeros(1))
  assert _flagged(bad, *c['ref']['dx2'])


def test_flags_one_ulp_on_one_dx(bwd_case):
  c = bwd_case
  val, bound = c['ref']['dx']
  got = c['got']['dx']
  # an element the rounding moved away from zero, mid-binade, with a bound below one ulp: one more ulp outward
  up = (got.double().abs() >= val.abs()) & (val.abs() > 0)
  mant = val.abs() / torch.exp2(torch.floor(torch.log2(val.abs().clamp_min(1e-300))))
  cand = up & (mant > 1.1) & (mant < 1.9) & (bound < 0.75 * 2 * G.half_ulp_bf16(val))
  i, j = (int(t) for t in torch.nonzero(cand)[0])
  bad = got.clone()
  bits = bad.view(torch.int16)
  bits[i, j] += 1                            # one ulp further from zero (sign-magnitude)
  assert _flagged(bad, val, bound)


# ---------------------------------------------------------------------------------------------- clip + Adam
def _adam32(p, g, mu, nu, *, step, lr, beta1, beta2, eps, grad_max_val, grad_max_norm, grad_scale, gen, order,
            dyn=None, mutate=None):
  """csrc/heads.cu grad_norm_kernel + clip_adam_kernel in fp32, powf and sqrtf perturbed by a few ulp."""
  def wobble(x, ulps):
    d = (torch.rand((), generator=gen, dtype=torch.float64) * 2 - 1) * ulps * 2.0 ** -24
    return (torch.as_tensor(x, dtype=torch.float64) * (1 + d)).float()
  f = lambda s: torch.tensor(float(s), dtype=torch.float32)
  lr, beta1, beta2, eps, gmv, gmn, scale = map(f, (lr, beta1, beta2, eps, grad_max_val, grad_max_norm, grad_scale))
  v = g * scale
  clip = lambda t: torch.where(torch.isnan(t), t, t.clamp(-gmv, gmv))
  if gmv > 0 and mutate != 'clip_after_norm':
    v = clip(v)
  mult = f(1)
  if gmn > 0:
    nsq = _sum32((v * v)[:, None], order)[0]
    nrm = wobble(torch.sqrt(nsq.double()), 1) if torch.isfinite(nsq) else torch.sqrt(nsq)
    mult = nrm if torch.isnan(nrm) else torch.clamp(gmn / (f(H.EPS32) + nrm), max=1.0)
  v = v * mult
  if gmv > 0 and mutate == 'clip_after_norm':
    v = clip(v)
  v = torch.where(torch.isnan(v), torch.zeros_like(v), v)
  fmax = torch.finfo(torch.float32).max
  if mutate == 'inf_to_zero':
    v = torch.where(torch.isinf(v), torch.zeros_like(v), v)
  else:
    v = torch.where(torch.isinf(v), torch.sign(v) * fmax, v)
  t = step - 1 if mutate == 'step_minus_one' else step
  bc1 = 1 - wobble(float(beta1) ** t, 8)
  bc2 = 1 - wobble(float(beta2) ** t, 8)
  if dyn is not None:
    lr, bc1, bc2 = dyn[0], dyn[1], dyn[2]
  m = beta1 * mu + (1 - beta1) * v
  s = beta2 * nu + (1 - beta2) * v * v
  mh, sh = m / bc1, s / bc2
  rt = torch.sqrt(sh.double())
  rt = (rt * (1 + (torch.rand(rt.shape, generator=gen, dtype=torch.float64) * 2 - 1) * 2.0 ** -24)).float()
  return dict(p=p - lr * mh / (rt + eps), mu=m, nu=s)


def _adam_data(seed, n, special=()):
  gen = torch.Generator().manual_seed(seed)
  p = torch.randn(n, generator=gen)
  g = torch.randn(n, generator=gen) * 1e-2 * torch.exp2(torch.randint(-4, 5, (n,), generator=gen).float())
  mu = torch.randn(n, generator=gen) * 1e-3
  nu = torch.rand(n, generator=gen) * 1e-5
  for i, val in special:
    g[i] = val
  return p, g, mu, nu, gen


ADAM = [dict(grad_max_val=0.0, grad_max_norm=1e-3), dict(grad_max_val=2e-2, grad_max_norm=1e-3),
        dict(grad_max_val=2e-2, grad_max_norm=0.0), dict(grad_max_val=0.0, grad_max_norm=0.0),
        dict(grad_max_val=0.0, grad_max_norm=100.0)]


@pytest.mark.parametrize('order', ('sequential', 'reversed', 'pairwise'))
@pytest.mark.parametrize('step', [1, 2, 7, 250000])
@pytest.mark.parametrize('clip', range(len(ADAM)))
@pytest.mark.parametrize('special', ['none', 'nan', 'inf'])
@pytest.mark.parametrize('scale', [1.0, 0.125])
def test_adam_emulation_inside_bound(order, step, clip, special, scale):
  if special == 'inf' and clip == 3 and step == 1:
    pytest.skip('an infinite gradient without clipping puts m / bc1 on the overflow threshold at step 1')
  n = 513
  sp = {'none': (), 'nan': ((7, float('nan')),), 'inf': ((9, float('inf')), (11, float('-inf')))}[special]
  p, g, mu, nu, gen = _adam_data(step + clip, n, sp)
  kw = dict(step=step, lr=1.5e-3, beta1=0.9, beta2=0.999, eps=1e-6, grad_scale=scale, **ADAM[clip])
  ref = H.clip_adam(p, g, mu, nu, **kw)
  for rep in range(3):
    got = _adam32(p, g, mu, nu, gen=gen, order=order, **kw)
    for name, (val, bound) in ref.items():
      H.check_adam(got[name], val, bound, f'{name} rep {rep}')


def test_adam_dyn_inside_bound():
  p, g, mu, nu, gen = _adam_data(5, 300)
  dyn = torch.tensor([1e-3, 0.271, 0.00599], dtype=torch.float32)
  kw = dict(step=3, lr=5.0, beta1=0.9, beta2=0.999, eps=1e-6, grad_max_val=0.0, grad_max_norm=1e-3)
  ref = H.clip_adam(p, g, mu, nu, dyn=dyn, **kw)
  got = _adam32(p, g, mu, nu, gen=gen, order='sequential', grad_scale=1.0, dyn=dyn, **kw)
  for name, (val, bound) in ref.items():
    H.check_adam(got[name], val, bound, name)
  assert _flagged(_adam32(p, g, mu, nu, gen=gen, order='sequential', grad_scale=1.0, **kw)['p'], *ref['p'])


def test_adam_nan_and_inf_rules():
  p, g, mu, nu, _ = _adam_data(6, 200, ((5, float('nan')),))
  base = dict(step=7, lr=1.5e-3, beta1=0.9, beta2=0.999, eps=1e-6)
  zero = H.clip_adam(p, torch.zeros_like(g), mu, nu, grad_max_val=0.0, grad_max_norm=0.0, **base)
  for gmv in (0.0, 0.1):                      # a NaN anywhere: the whole module's gradient is 0
    r = H.clip_adam(p, g, mu, nu, grad_max_val=gmv, grad_max_norm=1e-3, **base)
    assert torch.equal(r['mu'][0], zero['mu'][0]) and torch.equal(r['p'][0], zero['p'][0])
  r = H.clip_adam(p, g, mu, nu, grad_max_val=1e-3, grad_max_norm=0.0, **base)
  assert float(r['mu'][0][5]) == float(torch.tensor(0.9, dtype=torch.float32)) * float(mu[5])   # NaN -> 0
  assert float(r['mu'][0][6]) != float(torch.tensor(0.9, dtype=torch.float32)) * float(mu[6])
  p, g, mu, nu, _ = _adam_data(6, 200, ((5, float('inf')),))
  r = H.clip_adam(p, g, mu, nu, grad_max_val=0.0, grad_max_norm=1e-3, **base)        # infinite norm: mult = 0
  assert torch.equal(r['mu'][0], zero['mu'][0])
  r = H.clip_adam(p, g, mu, nu, grad_max_val=0.0, grad_max_norm=0.0, **base)         # inf -> FLT_MAX
  assert float(r['nu'][0][5]) == float('inf') and float(r['p'][0][5]) == float(p[5])
  assert float(r['mu'][0][5]) > 1e37


@pytest.mark.parametrize('mutate,clip,special,step', [
    ('step_minus_one', 0, (), 2), ('step_minus_one', 2, (), 3), ('inf_to_zero', 3, ((9, float('inf')),), 7),
    ('clip_after_norm', 1, (), 7)])
def test_flags_adam_mutations(mutate, clip, special, step):
  p, g, mu, nu, gen = _adam_data(8, 513, special)
  kw = dict(step=step, lr=1.5e-3, beta1=0.9, beta2=0.999, eps=1e-6, grad_scale=1.0, **ADAM[clip])
  ref = H.clip_adam(p, g, mu, nu, **kw)
  got = _adam32(p, g, mu, nu, gen=gen, order='sequential', **kw)
  for name, (val, bound) in ref.items():
    H.check_adam(got[name], val, bound, f'unmutated {name}')
  bad = _adam32(p, g, mu, nu, gen=gen, order='sequential', mutate=mutate, **kw)
  flagged = False
  for name, (val, bound) in ref.items():
    try:
      H.check_adam(bad[name], val, bound, name)
    except AssertionError:
      flagged = True
  assert flagged


@pytest.mark.parametrize('clip', range(len(ADAM)))
@pytest.mark.parametrize('step', [1, 6, 250000])
def test_adam_reference_matches_oracle(clip, step):
  """On fp64 inputs, the fp64 reference is the oracle's clip_gradients, nan_to_num and adam_update."""
  from oracle import o_train
  p, g, mu, nu, _ = _adam_data(9 + step, 1000)
  p, g, mu, nu = (t.double() for t in (p, g, mu, nu))
  f32 = lambda s: float(torch.tensor(s, dtype=torch.float32))

  class Cfg:
    adam_beta1, adam_beta2, adam_eps = f32(0.9), f32(0.999), f32(1e-6)
    grad_max_val, grad_max_norm = f32(ADAM[clip]['grad_max_val']), f32(ADAM[clip]['grad_max_norm'])
  gc = torch.nan_to_num(o_train.clip_gradients({'mod': g}, Cfg)['mod'][()])
  p_o, m_o, v_o = o_train.adam_update(p, gc, mu, nu, step - 1, f32(1.5e-3), Cfg)
  r = H.clip_adam(p, g, mu, nu, step=step, lr=1.5e-3, beta1=0.9, beta2=0.999, eps=1e-6, **ADAM[clip])
  for name, want in (('p', p_o), ('mu', m_o), ('nu', v_o)):
    err = (r[name][0] - want).abs() / want.abs().clamp_min(1e-30)
    assert float(err.max()) < 1e-12, (name, float(err.max()))


# ---------------------------------------------------------------------------------------------- packing
def test_pack_matches():
  m = torch.tensor([1.0, 1 + 2 ** -8, 1 + 3 * 2 ** -8, float('nan'), -0.0, 1e-40, 3.4e38, float('-inf')])
  want = m.to(torch.bfloat16)
  assert H.pack_matches(want, m)
  bad = want.clone()
  bad.view(torch.int16)[1] += 1               # a tie rounded away from even
  assert not H.pack_matches(bad, m)
  bad = want.clone()
  bad[4] = 0.0                                # +0 for -0
  assert not H.pack_matches(bad, m)
  ok = want.clone()
  ok.view(torch.int16)[3] = 0x7fc1            # any NaN for a NaN
  assert H.pack_matches(ok, m)
