"""tests/tangent_ref.py is sound and sensitive.  CPU only.

Soundness: `emulate_act` is an fp32 transcription of act_tangent_bwd_kernel on the same padded buffers the GPU cases
use -- rows s M + r of each stream at the operand's own pitch, sigmoid_fast with __expf and __fdividef moved by their
documented error in either direction (the exponential flushed below 2^-126, the quotient 0 above 2^126), act_d1 /
act_d2 in the kernel's order, the three-term sum with and without FMA contraction, prev + a'' gs rounded once or
twice, bf16 stores.  Every element of every case lands inside its bound.  `emulate_outer_mask` is the kernel's
select, and the reference equals it bit for bit.

Sensitivity: each plausible kernel bug, applied to the emulation, is caught on the case meant for it.
"""
import numpy as np
import pytest
import torch

import gemm_ref as GR
import tangent_ref as TR
from test_gpu_tangent_fp64 import ACT_CASES, ACTS, OM_CASES, make_act_inputs, make_om_inputs

ULP = 2.0 ** -23
f32 = torch.float32


def _flat(view, buf):
  """(flat buffer, element offset of the view, pitch)."""
  return buf.view(-1), view.storage_offset() - buf.storage_offset(), view.stride(0)


def _index(off, ld, rows, n):
  return off + rows[:, None] * ld + torch.arange(n)[None, :]


def _read(vb, rows, n):
  flat, off, ld = _flat(*vb)
  idx = _index(off, ld, rows, n)
  inside = (idx >= 0) & (idx < flat.numel())
  return torch.where(inside, flat[idx.clamp(0, flat.numel() - 1)].float(), torch.full_like(idx, float('nan'), dtype=f32))


def _write(vb, rows, vals):
  flat, off, ld = _flat(*vb)
  idx = _index(off, ld, rows, vals.shape[1])
  inside = (idx >= 0) & (idx < flat.numel())
  flat[idx[inside]] = vals[inside].to(flat.dtype)


def _sigmoid_fast(z, dirn):
  """sigmoid_fast in fp32 with __expf and __fdividef moved by their documented error (dirn = +-1)."""
  zd = z.double()
  rel = ((1.5 + 1.173 * zd.abs()) * ULP).clamp(max=0.5)          # an exponential stays positive
  e = (torch.exp(-zd) * (1 + dirn * rel)).to(f32)
  e = torch.where(e < 2.0 ** -126, torch.zeros_like(e), e)                     # ex2.approx.ftz
  d = e + 1                                                                    # fl(1 + E)
  s = (1.0 / d.double() * (1 - dirn * 1.5 * ULP)).to(f32)
  s = torch.where(d == 1, torch.ones_like(s), s)                               # 1 / 1 is exact
  return torch.where(d > 2.0 ** 126, torch.zeros_like(s), s)                   # __fdividef's flush


def _act_d12(code, z, dirn):
  s = _sigmoid_fast(z, dirn)
  q = s * (1 - s)
  if code == GR.SOFTPLUS:
    return s, q
  return s * (1 + z * (1 - s)), q * (2 + z * (1 - 2 * s))


def _fma(a, b, c):
  return (a.double() * b.double() + c.double()).to(f32)


def emulate_act(inp, dirn=1, fma=False, once=False, mut=None):
  """act_tangent_bwd_kernel on the case's buffers (in place where du is T); mutates du and g's buffers."""
  c = inp['case']
  M, N, code = c['M'], c['N'], ACTS[c['act']]
  r = torch.arange(M)
  z = _read(inp['z'], r, N)
  base = (lambda s, vb: s * vb[0].stride(0)) if mut == 'stream_stride_pitch' else (lambda s, vb: s * M)
  T = [_read(inp['t'], base(s, inp['t']) + r, N) for s in range(3)]
  uu = [_read(inp['u'], base(s, inp['u']) + r, N) for s in range(3)]
  d1, d2 = _act_d12(code, z, dirn)
  if mut == 'd1_for_d2':
    d2 = d1
  for s in range(3):
    _write(inp['du'], base(s, inp['du']) + r, (d1 * T[s]).to(torch.bfloat16))
  if mut == 'du_before_read':                      # T read again after du was stored over it
    T = [_read(inp['t'], base(s, inp['t']) + r, N) for s in range(3)]
  gs = torch.zeros_like(z)
  for s in range(2 if mut == 'gs_two_streams' else 3):
    gs = _fma(T[s], uu[s], gs) if fma else gs + T[s] * uu[s]
  prev = _read(inp['g'], r, N) if (c['acc'] or mut == 'prev_when_set') else torch.zeros_like(z)
  g = _fma(d2, gs, prev) if once else prev + d2 * gs
  _write(inp['g'], r, g.to(torch.bfloat16))


def _act_outcome(name, **kw):
  inp = make_act_inputs(name)
  ref = TR.act_tangent_ref(ACTS[inp['case']['act']], inp['z'][0], inp['t'][0], inp['u'][0],
                           inp['g'][0] if inp['case']['acc'] else None)
  emulate_act(inp, **kw)
  out = {}
  for what, view, val, bound in (('du', inp['du'][0], ref[0], ref[1]), ('g', inp['g'][0], ref[2], ref[3])):
    got = view.double()
    ratio = ((got - val).abs() / bound).nan_to_num(nan=np.inf)
    out[what] = ratio
  out['padding'] = GR.padding_intact(*inp['du']) and GR.padding_intact(*inp['g'])
  return out


CPU_ACT = [n for n in ACT_CASES if 'sweep' not in n]


@pytest.mark.parametrize('name', CPU_ACT)
def test_act_emulation_within_bounds(name):
  worst = {}
  for dirn in (1, -1):
    for fma in (False, True):
      for once in (False, True):
        o = _act_outcome(name, dirn=dirn, fma=fma, once=once)
        assert o['padding'], name
        for what in ('du', 'g'):
          w = float(o[what].max())
          assert w <= 1, (name, what, dirn, fma, once, w, np.unravel_index(int(o[what].argmax()), o[what].shape))
          worst[what] = max(worst.get(what, 0.0), w)
  print(f'\n{name}: worst err/bound du {worst["du"]:.3f} g {worst["g"]:.3f}')


def test_bounds_say_something():
  """Where z is ordinary the bound is a few bf16 ulps, not a blanket: |z| <= 8 elements within 2^-6 relative, and
  the special values themselves (|z| up to 1e30) leave du's bound within 2^-6 relative too."""
  inp = make_act_inputs('silu-N64-acc-sep')
  z = inp['z'][0].double().repeat(3, 1)
  du, dub, g, gb = TR.act_tangent_ref(GR.SILU, inp['z'][0], inp['t'][0], inp['u'][0], inp['g'][0])
  rel = dub / du.abs().clamp_min(1e-30)
  ok = (du.abs() > 1e-3)
  assert float(rel[ok].max()) < 2.0 ** -6, float(rel[ok].max())
  big = ok & (z.abs() > 16)
  assert big.any() and float(rel[big].max()) < 2.0 ** -6


def emulate_outer_mask(inp, mut=None):
  c = inp['case']
  rows, n, mod = c['rows'], c['n'], c['mod']
  r = torch.arange(rows)
  rv = inp['rowv'][r % (mod or rows) if (mut == 'rowv_mod' and rows) else r]
  prod = rv[:, None] * inp['colv'][None, :]
  if inp['bits'] is None:
    return prod.to(torch.bfloat16)
  words = inp['bits'].long() & 0xffffffff
  col = torch.arange(n)
  c8 = col // 8 * 8
  shift = (c8 & 31) + (1 if mut == 'mask_shift' else 0)
  w = words[r % mod if mod else r][:, c8 >> 5] >> shift
  bit = (w >> (col - c8)) & 1
  return torch.where(bit.bool(), prod, torch.zeros_like(prod)).to(torch.bfloat16)


@pytest.mark.parametrize('name', list(OM_CASES))
def test_outer_mask_reference_is_the_select(name):
  inp = make_om_inputs(name)
  c = inp['case']
  want = TR.outer_mask_ref(inp['rowv'], inp['colv'], inp['bits'], rows=c['rows'], n=c['n'], mask_mod=c['mod'])
  got = emulate_outer_mask(inp)
  assert torch.equal(got.view(torch.int16), want.view(torch.int16))
  if c['bits'] and c['rows']:
    assert torch.isnan(inp['rowv']).any() and (want.view(torch.int16) == 0).any()
    assert not torch.isnan(want.float()).any(), 'a NaN rowv under a cleared bit must give +0'


# mutation: (kind, the case meant for it)
MUTATIONS = {
    'd1_for_d2': ('act', 'softplus-N64-set-sep'),
    'gs_two_streams': ('act', 'silu-N128-acc-sep'),
    'stream_stride_pitch': ('act', 'silu-N256-set-sep'),
    'prev_when_set': ('act', 'softplus-N8-set-sep'),
    'du_before_read': ('act', 'silu-N64-set-inplace'),
    'mask_shift': ('om', 'bits-mod3'),
    'rowv_mod': ('om', 'bits-mod3'),
}


@pytest.mark.parametrize('mut', list(MUTATIONS))
def test_mutation_is_caught(mut):
  kind, name = MUTATIONS[mut]
  if kind == 'om':
    inp = make_om_inputs(name)
    c = inp['case']
    want = TR.outer_mask_ref(inp['rowv'], inp['colv'], inp['bits'], rows=c['rows'], n=c['n'], mask_mod=c['mod'])
    bad = int((emulate_outer_mask(inp, mut).view(torch.int16) != want.view(torch.int16)).sum())
    assert bad, f'{mut}: {name} does not notice'
    print(f'\n{mut}: caught by {name} on {bad} elements')
    return
  o = _act_outcome(name, mut=mut)
  caught = {w: int((o[w] > 1).sum()) for w in ('du', 'g')}
  assert sum(caught.values()) or not o['padding'], f'{mut}: {name} does not notice'
  print(f'\n{mut}: caught by {name}: elements outside the bound {caught}, padding intact {o["padding"]}')
