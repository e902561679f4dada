"""The trunk's tangent kernels (mnrf_act_tangent_bwd, mnrf_outer_mask) against the fp64 reference of
tests/tangent_ref.py, element by element.  Needs an H100.

act_tangent_bwd: softplus and SiLU, g set and accumulated, du in place (du is T, as the model runs it) and separate;
N in {8, 64, 128, 256, 1024}; a ragged M, and two cases with more rows than one grid-stride sweep covers at 16 blocks
of 256 threads per SM; z over signed zeros, bf16 subnormals, |z| from 16 to 1e30 and SiLU's zeros of a' and a''.
All five operands have their own pitch and sit inside buffers whose padding is NaN (inputs) or a sentinel
(outputs); the padding must survive, the inputs must come back unchanged, and with accumulate = 0 g's view holds
NaN, which a kernel that reads it turns into a non-finite result.  outer_mask is compared bit for bit.  Argument
refusals return before any launch and leave the outputs untouched.

One eager train step of mini_refnerf (softplus, SiLU, ReLU) checks every launch the model makes against the same
references on that launch's own inputs, and how models.py wires them: which buffers they read and write, and in
which order.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import gemm_ref as GR
import tangent_ref as TR
from launch_recorder import Recorder

pytestmark = pytest.mark.gpu

ACTS = {'softplus': GR.SOFTPLUS, 'silu': GR.SILU}
SMS = 132                           # an H100 SXM; the GPU cases size their sweeps by the device's own count


def sweep_chunks(num_sms):
  """8-column chunks one grid-stride sweep of act_tangent_bwd covers: 16 blocks of 256 threads per SM."""
  return num_sms * 16 * 256


def _act_cases():
  cases = {}
  for act in ACTS:
    for N in (8, 64, 128, 256, 1024):
      for acc in (False, True):
        for inplace in (True, False):
          cases[f'{act}-N{N}-{"acc" if acc else "set"}-{"inplace" if inplace else "sep"}'] = dict(
              act=act, N=N, M=331 + N // 8, acc=acc, inplace=inplace)
  # more rows than one sweep of the grid at the device's SM count, ragged against it (M set by case_rows)
  cases['silu-N8-sweep'] = dict(act='silu', N=8, M=None, extra=4097, acc=True, inplace=True)
  cases['softplus-N1024-sweep'] = dict(act='softplus', N=1024, M=None, extra=131, acc=False, inplace=True)
  return cases


def case_rows(c, num_sms=SMS):
  """M of a case; a sweep case has `extra` rows more than one grid-stride sweep covers on num_sms SMs."""
  return c['M'] if c['M'] is not None else sweep_chunks(num_sms) * 8 // c['N'] + c['extra']


ACT_CASES = _act_cases()


def make_act_inputs(name, device='cpu', num_sms=SMS):
  """Buffers of one case: dict of (view, buffer) for z, t, u, du, g and the fp64-exact bf16 inputs.  Pitches:
  z N + 8, T N + 16, u N + 24, du N + 32 (or T's), g N + 40; views start 8 columns in where the pitch allows."""
  c = dict(ACT_CASES[name])
  c['M'] = M = case_rows(c, num_sms)
  N = c['N']
  gen = torch.Generator().manual_seed(sum(name.encode()))
  bf = torch.bfloat16
  z = torch.randn(M, N, generator=gen, dtype=torch.float64) * 3
  sp = TR.special_z()
  idx = torch.randint(0, M * N, (8 * sp.numel(),), generator=gen)
  z.view(-1)[idx] = sp.repeat(8)
  t = torch.randn(3 * M, N, generator=gen, dtype=torch.float64)
  t[torch.randint(0, 3 * M, (M // 10 + 1,), generator=gen)] *= 1e3
  u = torch.randn(3 * M, N, generator=gen, dtype=torch.float64)
  u[torch.randint(0, 3 * M, (M // 10 + 1,), generator=gen)] = 0
  prev = torch.randn(M, N, generator=gen, dtype=torch.float64) * 4
  out = dict(case=c)
  for key, rows, pitch, fill, val in (('z', M, N + 8, 'nan', z), ('t', 3 * M, N + 16, 'sentinel' if c['inplace'] else 'nan', t),
                                      ('u', 3 * M, N + 24, 'nan', u), ('du', 3 * M, N + 32, 'sentinel', None),
                                      ('g', M, N + 40, 'sentinel', prev if c['acc'] else None)):
    if key == 'du' and c['inplace']:
      out['du'] = out['t']
      continue
    view, buf = GR.embed((rows, N), bf, device, extra_cols=pitch - N, col0=8, fill=fill)
    if val is not None:
      view.copy_(val.to(bf))
    elif key == 'g':
      GR._bit_fill(view, GR.NAN_BITS[bf])            # a kernel that reads g with accumulate = 0 gets NaN
    out[key] = (view, buf)
  return out


def act_reference(inp):
  c = inp['case']
  return TR.act_tangent_ref(ACTS[c['act']], inp['z'][0], inp['t'][0], inp['u'][0],
                            inp['g'][0] if c['acc'] else None)


@pytest.fixture(scope='module')
def ops():
  from multinerf_b200 import lib, ops as _ops
  lib.require_device()
  return _ops


@pytest.mark.parametrize('name', list(ACT_CASES))
def test_act_tangent_bwd_case(ops, name):
  from multinerf_b200 import lib as L
  sms = L.load().mnrf_num_sms()
  inp = make_act_inputs(name, 'cuda', sms)
  c = inp['case']
  if 'sweep' in name:
    assert c['M'] * c['N'] // 8 > sweep_chunks(sms), f'{name}: one grid-stride sweep covers all {c["M"]} rows'
  ref = act_reference(inp)          # before the call: in place, du overwrites T
  keep = {k: inp[k][1].clone() for k in ('z', 'u')}
  if not c['inplace']:
    keep['t'] = inp['t'][1].clone()
  ops.act_tangent_bwd(ACTS[c['act']], inp['z'][0], inp['t'][0], inp['u'][0], inp['du'][0], inp['g'][0],
                      accumulate=c['acc'])
  torch.cuda.synchronize()
  wdu = GR.check(inp['du'][0], ref[0], ref[1], f'{name} du')
  wg = GR.check(inp['g'][0], ref[2], ref[3], f'{name} g')
  for k in ('du', 'g'):
    assert GR.padding_intact(*inp[k]), f'{name}: wrote outside {k}'
  for k, b in keep.items():
    assert torch.equal(inp[k][1].view(torch.int16), b.view(torch.int16)), f'{name}: input {k} changed'
  print(f'\n{name}: M {c["M"]} N {c["N"]} | worst err/bound du {wdu:.3f} g {wg:.3f}')


# ------------------------------------------------------------------ outer_mask

OM_CASES = {
    'bits-mod3': dict(rows=3 * 257, n=256, mod=257, bits=True, ld=256 + 40),
    'bits-nomod': dict(rows=300, n=64, mod=0, bits=True, ld=64),
    'bits-n32': dict(rows=3 * 100, n=32, mod=100, bits=True, ld=40),
    'nobits-mod': dict(rows=3 * 129, n=1024, mod=129, bits=False, ld=1024 + 8),
    'nobits': dict(rows=77, n=128, mod=0, bits=False, ld=128),
    'rows0': dict(rows=0, n=256, mod=0, bits=True, ld=264),
}


def make_om_inputs(name, device='cpu'):
  """rowv [rows] with NaN under rows whose mask bits are all clear, colv [n], mask words [mod or rows, n/32 + 3]
  (a third of the rows all clear, the rest random, words past n/32 all set), out (view, buffer) of pitch ld."""
  c = OM_CASES[name]
  gen = torch.Generator().manual_seed(sum(name.encode()))
  rows, n = c['rows'], c['n']
  mrows = c['mod'] or rows
  rowv = torch.randn(rows, generator=gen) * 3
  colv = torch.randn(n, generator=gen)
  bits = None
  if c['bits']:
    keep = torch.rand(mrows, n, generator=gen) < 0.5
    clear = torch.arange(mrows) % 3 == 1
    keep[clear] = False
    bits = GR.pack_bits(keep, n // 32 + 3)
    bits[:, n // 32:] = -1
    r = torch.arange(rows)
    rowv[clear[r % mrows]] = float('nan')
    bits = bits.to(device)
  view, buf = GR.embed((rows, n), torch.bfloat16, device, extra_cols=c['ld'] - n, fill='sentinel')
  return dict(case=c, rowv=rowv.to(device), colv=colv.to(device), bits=bits, out=(view, buf))


@pytest.mark.parametrize('name', list(OM_CASES))
def test_outer_mask_case(ops, name):
  c = OM_CASES[name]
  inp = make_om_inputs(name, 'cuda')
  ops.outer_mask(inp['rowv'], inp['colv'], inp['bits'], inp['out'][0], rows=c['rows'], n=c['n'], mask_mod=c['mod'])
  torch.cuda.synchronize()
  want = TR.outer_mask_ref(inp['rowv'], inp['colv'], inp['bits'], rows=c['rows'], n=c['n'], mask_mod=c['mod'])
  got = inp['out'][0]
  assert torch.equal(got.view(torch.int16), want.view(torch.int16)), \
      f'{name}: {int((got.view(torch.int16) != want.view(torch.int16)).sum())} elements differ in their bits'
  assert GR.padding_intact(*inp['out']), f'{name}: wrote outside out'
  zeros = int((want.view(torch.int16) == 0).sum())
  print(f'\n{name}: rows {c["rows"]} n {c["n"]} mod {c["mod"]} ld {c["ld"]} | bit-equal, {zeros} +0 elements')


# ------------------------------------------------------------------ refusals

def _raw_act(lib, M, n, act, ops_, acc=0):
  """mnrf_act_tangent_bwd with explicit (pointer, pitch) pairs: ops_ = [(tensor or None, pitch)] * 5."""
  from multinerf_b200 import lib as L
  args = []
  for t, ld in ops_:
    args += [None if t is None else C.c_void_p(t), ld]
  return lib.mnrf_act_tangent_bwd(M, n, act, *args, acc, L.stream_ptr())


def test_refusals_leave_outputs_untouched(ops):
  from multinerf_b200 import lib as L
  lib = L.load()
  M, N = 64, 64
  bf = torch.bfloat16
  buf = {k: torch.full((rows, N + 16), 7.0, dtype=bf, device='cuda') for k, rows in
         (('z', M), ('t', 3 * M), ('u', 3 * M), ('du', 3 * M), ('g', M))}
  good = [(buf[k].data_ptr(), N + 16) for k in ('z', 't', 'u', 'du', 'g')]

  def refused(what, M_=M, n=N, act=L.ACT_SILU, args=None, match=None):
    rc = _raw_act(lib, M_, n, act, args or good)
    assert rc != 0, f'act_tangent_bwd accepted {what}'
    msg = lib.mnrf_last_error().decode()
    assert match is None or match in msg, (what, msg)

  for act in (L.ACT_NONE, L.ACT_RELU):
    refused(f'act {act}', act=act, match='not a smooth activation')
  for i, k in enumerate(('z', 't', 'u', 'du', 'g')):
    a = list(good)
    a[i] = (None, N + 16)
    refused(f'null {k}', args=a, match='null pointer')
    a = list(good)
    a[i] = (good[i][0], N + 12)
    refused(f'pitch {N + 12} of {k}', args=a, match='multiples of 8')
    a = list(good)
    a[i] = (good[i][0] + 8, N + 16)
    refused(f'{k} 8 bytes off alignment', args=a, match='16-byte aligned')
  refused('N = 12', n=12, match='multiples of 8')
  torch.cuda.synchronize()
  for k, b in buf.items():
    assert (b == 7).all(), f'a refused act_tangent_bwd wrote {k}'

  out = torch.full((96, 72), 7.0, dtype=bf, device='cuda')
  rowv, colv = torch.ones(96, device='cuda'), torch.ones(64, device='cuda')
  for what, n, ld, ptrs in (('N = 48', 48, 72, None), ('ld = 68', 64, 68, None),
                            ('null rowv', 64, 72, (None, colv, out)), ('null colv', 64, 72, (rowv, None, out)),
                            ('null out', 64, 72, (rowv, colv, None)), ('out 8 bytes off alignment', 64, 72, 'shift')):
    r, cv, o = (rowv, colv, out) if ptrs in (None, 'shift') else ptrs
    if ptrs == 'shift':
      rc = lib.mnrf_outer_mask(95, n, 0, L.ptr(r), L.ptr(cv), None, 0, C.c_void_p(out.data_ptr() + 8), ld,
                               L.stream_ptr())
      assert rc != 0 and 'aligned' in lib.mnrf_last_error().decode(), f'outer_mask accepted {what}'
      continue
    rc = lib.mnrf_outer_mask(96, n, 0, L.ptr(r), L.ptr(cv), None, 0, L.ptr(o), ld, L.stream_ptr())
    assert rc != 0, f'outer_mask accepted {what}'
  torch.cuda.synchronize()
  assert (out == 7).all(), 'a refused outer_mask wrote its output'
  # rows = 0 returns before any check or launch
  assert lib.mnrf_outer_mask(0, 48, 0, None, None, None, 0, None, 68, L.stream_ptr()) == 0


# ------------------------------------------------------------------ the model's launches

@pytest.mark.parametrize('name', ['softplus', 'silu', 'relu'])
def test_refnerf_train_step_tangent_launches(ops, monkeypatch, name):
  """One eager train step of mini_refnerf.  Every outer_mask and act_tangent_bwd launch is checked against the fp64
  reference on its own inputs, and the wiring of models.py is asserted: per level with density normals one outer_mask
  (3M rows, mask_mod M; under ReLU with the mask bits of the last trunk layer), then net_depth second-order launches
  in place, the first (layer net_depth - 1) accumulating into the buffer the head's DGRAD just wrote and the others
  not, layer i reading the z its forward GEMM stored, bit for bit; none under ReLU."""
  from model_parity import level_jitter, mini_refnerf, synth_rays
  from multinerf_b200 import lib as L, models, train_utils, utils
  bundle = mini_refnerf()
  bundle.nerf_mlp.net_activation = bundle.prop_mlp.net_activation = name
  bundle.config.grad_max_norm = bundle.config.grad_max_val = 0.0
  cfg = bundle.nerf_mlp
  B, W, depth = 96, cfg.net_width, cfg.net_depth
  rays, rng = synth_rays(81, B, 2.0, 6.0, unit_cube=False)
  target = rng.uniform(0, 1, (B, 3)).astype(np.float32)
  model, variables = models.construct_model(82, rays, bundle)
  rand = level_jitter(rng, bundle, B)
  rec = Recorder(ops, ('gemm', 'outer_mask', 'act_tangent_bwd'), monkeypatch)
  step_fn = train_utils.create_train_step(model, bundle.config)
  step_fn(rand, train_utils.TrainState(variables), utils.Batch(rays=rays, rgb=target), None, 0.5)
  torch.cuda.synchronize()
  monkeypatch.undo()

  ev = rec.calls

  def kept(c):          # what a trunk layer's FWD GEMM stores for the backward: z or the mask bits
    return next((k for k in ('z', 'maskbits') if c.args.get(k) is not None), None)
  fwd_calls = [c for c in ev if c.fn == 'gemm' and c.args['mode'] == L.GEMM_FWD and c.args['n'] == W and kept(c)]
  # the trunk's forward layers in order, level after level: layer = index mod net_depth
  fwd = {c.args[kept(c)].data_ptr(): (k % depth, c.after[kept(c)]) for k, c in enumerate(fwd_calls)}
  oms = [i for i, c in enumerate(ev) if c.fn == 'outer_mask']
  assert len(oms) == bundle.model.num_levels, f'{len(oms)} outer_mask launches for {bundle.model.num_levels} levels'
  assert len(fwd) == depth * bundle.model.num_levels, 'trunk forward layers that keep z / mask bits'
  worst = {'du': 0.0, 'g': 0.0}
  for j, i0 in enumerate(oms):
    c = ev[i0]
    rowv, colv, bits = c.before['rowv'], c.before['colv'], c.before.get('maskbits')
    rows, n, mod = c.args['rows'], c.args['n'], c.args.get('mask_mod', 0)
    M = rows // 3
    assert n == W and mod == M and rowv.numel() == 3 * M
    want = TR.outer_mask_ref(rowv, colv, bits, rows=rows, n=W, mask_mod=M)
    assert torch.equal(c.after['out'][:rows, :n].view(torch.int16), want.view(torch.int16)), f'level {j}: outer_mask'
    # the buffer the head's DGRAD wrote last before this level's tangent backward
    head = [e.args['out'].data_ptr() for e in ev[:i0] if e.fn == 'gemm' and e.args['mode'] == L.GEMM_DGRAD and
            e.args['m'] == e.args['out'].shape[0] and e.args['n'] == W][-1]
    acts = [e for e in ev[i0 + 1:oms[j + 1] if j + 1 < len(oms) else len(ev)] if e.fn == 'act_tangent_bwd']
    if name == 'relu':
      assert bits is not None and fwd[c.args['maskbits'].data_ptr()][0] == depth - 1, \
          'outer_mask without the last layer\'s bits'
      assert torch.equal(bits, fwd[c.args['maskbits'].data_ptr()][1]), 'mask bits changed since the forward'
      assert not acts, 'second-order launches under ReLU'
      continue
    assert bits is None, 'a smooth activation seeds the tangent chain unmasked'
    assert len(acts) == depth, f'level {j}: {len(acts)} second-order launches for {depth} trunk layers'
    assert [a.args.get('accumulate', False) for a in acts] == [True] + [False] * (depth - 1)
    assert acts[0].args['g'].data_ptr() == head, 'the accumulating launch does not add into the head DGRAD\'s output'
    for k, a in enumerate(acts):
      layer, zf = fwd[a.args['z'].data_ptr()]
      assert layer == depth - 1 - k, f'level {j}: launch {k} reads the z of layer {layer}'
      z, t, u = a.before['z'], a.before['t_adj'], a.before['u']
      prev = a.before['g'] if a.args.get('accumulate', False) else None
      assert torch.equal(z.view(torch.int16), zf.view(torch.int16)), 'z changed since the forward'
      assert a.args['du'].data_ptr() == a.args['t_adj'].data_ptr() and a.args['act'] == ACTS[name]
      du, dub, g, gb = TR.act_tangent_ref(a.args['act'], z, t, u, prev)
      worst['du'] = max(worst['du'], GR.check(a.after['du'], du, dub, f'level {j} layer {layer} du'))
      worst['g'] = max(worst['g'], GR.check(a.after['g'], g, gb, f'level {j} layer {layer} g'))
  n_act = sum(e.fn == 'act_tangent_bwd' for e in ev)
  print(f'\n{name}: {len(oms)} levels, {n_act} second-order launches | worst err/bound '
        f'du {worst["du"]:.3f} g {worst["g"]:.3f}')
