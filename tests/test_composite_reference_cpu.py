"""The reference of the compositing kernels (tests/composite_ref.py) checked on the CPU: torch.autograd.gradcheck at
tiny shapes with each optional input switched on once, and its pixel and data loss against the oracle functions it
reassembles.  The GPU parity test trusts this reference's autograd gradients; this file shows they are right."""
import numpy as np
import pytest
import torch

import composite_ref as R
from oracle import o_render, o_train

CFG = dict(raydist_fn='reciprocal', opaque_background=False, density_bias=-1.0, density_noise=0.0,
           rgb_activation='sigmoid', rgb_premultiplier=1.0, rgb_bias=0.0, rgb_padding=0.001, bg_const=1.0)
LOSS = dict(loss_type='mse', charb_padding=0.001, data_mult=1.0, distortion_mult=0.0, interlevel_mult=0.0)


def _inputs(seed, B=3, S=5, Sf=4, lm_ch=1):
  rng = np.random.default_rng(seed)
  sd = np.sort(rng.uniform(0, 1, (B, S + 1)), -1)
  sd[:, 0], sd[:, -1] = 0, 1
  sf = np.sort(np.concatenate([sd[:, 1:3], rng.uniform(0, 1, (B, Sf - 3))], -1), -1)   # shares two knots
  sf = np.concatenate([np.zeros((B, 1)), sf, np.ones((B, 1))], -1)
  wf = rng.uniform(0, 1, (B, Sf))
  d = rng.normal(size=(B, 3)) * 1.3
  t = lambda x: torch.tensor(np.asarray(x, np.float64))
  return dict(raw_density=t(rng.normal(size=(B, S)) * 2), raw_rgb=t(rng.normal(size=(B, S, 3))), sdist=t(sd),
              directions=t(d), near=t(np.full(B, 0.5)), far=t(np.full(B, 20.0)), target=t(rng.uniform(0, 1, (B, 3))),
              lossmult=t(rng.uniform(0.5, 2, (B, lm_ch))), sdist_fine=t(sf), weights_fine=t(wf / wf.sum(-1, keepdims=True)),
              _rng=rng)


CASES = {
    'plain': {},
    'opaque': dict(cfg=dict(opaque_background=True)),
    'density_noise': dict(cfg=dict(density_noise=0.7), inp=['density_noise']),
    'bg_rgb': dict(inp=['bg_rgb']),
    'rgb_scale': dict(inp=['rgb_scale']),
    'extra_dw': dict(inp=['extra_dw']),
    'data_mask': dict(inp=['data_mask']),
    'tint': dict(cfg=dict(rgb_mode=1), inp=['raw_diffuse', 'raw_tint']),
    'no_tint': dict(cfg=dict(rgb_mode=1), inp=['raw_diffuse']),
    'safe_exp': dict(cfg=dict(rgb_activation='safe_exp', rgb_bias=-1.0, rgb_padding=0.0, raydist_fn='log')),
    'charb_lm3': dict(loss=dict(loss_type='charb'), lm_ch=3),
    'rawnerf': dict(loss=dict(loss_type='rawnerf', data_mult=0.5)),
    'distortion': dict(loss=dict(distortion_mult=0.01)),
    'interlevel': dict(loss=dict(interlevel_mult=1.0), no_rgb=True),
}


def _case(name):
  spec = CASES[name]
  inp = _inputs(sorted(CASES).index(name), lm_ch=spec.get('lm_ch', 1))
  rng = inp.pop('_rng')
  B, S = inp['raw_density'].shape
  t = lambda x: torch.tensor(np.asarray(x, np.float64))
  extra = dict(density_noise=t(rng.normal(size=(B, S))), bg_rgb=t(rng.uniform(0, 1, (B, 3))),
               # one zero and one negative exposure channel: d pixel / d scale is sum_s w_s c_s there too
               rgb_scale=t([[0.0, 1.5, 0.7], [-0.8, 2.0, 1.0], [1.2, 0.3, 0.9]]),
               extra_dw=t(rng.normal(size=(B, S)) * 0.1), data_mask=t([1.0, 0.0, 1.0]),
               raw_diffuse=t(rng.normal(size=(B, S, 3))), raw_tint=t(rng.normal(size=(B, S, 3))))
  for k in spec.get('inp', []):
    inp[k] = extra[k]
  if spec.get('no_rgb'):
    inp['raw_rgb'] = None
  cfg = dict(CFG, **spec.get('cfg', {}))
  loss = dict(LOSS, **spec.get('loss', {}))
  loss['inv_denom'] = 1.0 / float(inp['lossmult'].expand(B, 3).sum())
  return inp, cfg, loss


@pytest.mark.parametrize('name', sorted(CASES))
def test_reference_gradcheck(name):
  inp, cfg, loss = _case(name)
  names = [k for k in R.LEAVES if inp.get(k) is not None]

  def fn(*leaves):
    out = R.composite(dict(inp, **dict(zip(names, leaves))), cfg, loss)
    if loss['loss_type'] == 'rawnerf':
      # the RawNeRF loss weights each residual by a detached 1 / (1e-3 + clip): its gradient is by design not the
      # derivative of its value, so only the pixel and weights are checked here; the loss and its gradient are
      # compared with the oracle's compute_data_loss below
      return out['rgb'], out['weights']
    return out['loss'], out['rgb'], out['weights']
  leaves = tuple(inp[k].clone().requires_grad_(True) for k in names)
  assert torch.autograd.gradcheck(fn, leaves, eps=1e-6, atol=1e-8, rtol=1e-6)


def test_reference_rgb_scale_gradient_at_zero():
  """At a zero exposure channel the scale's gradient is d loss / d pixel * sum_s w_s c_s, not zero."""
  inp, cfg, loss = _case('rgb_scale')
  out, g = R.grads(inp, cfg, loss)
  c = R.colour(inp['raw_rgb'], cfg)
  wc = (out['weights'][..., None] * c).sum(-2)
  dpix = 2 * (out['rgb'] - inp['target']) * inp['lossmult'] * loss['inv_denom']
  torch.testing.assert_close(g['rgb_scale'], dpix * wc, rtol=1e-12, atol=1e-15)
  assert float(g['rgb_scale'][0, 0].abs()) > 1e-3


@pytest.mark.parametrize('loss_type,lm_ch', [('mse', 1), ('charb', 3), ('rawnerf', 3)])
def test_reference_matches_oracle_loss(loss_type, lm_ch):
  """The pixel, the data loss and its gradient are the oracle's volumetric_rendering and compute_data_loss (no
  mask)."""
  inp, cfg, loss = _case('bg_rgb')
  B = inp['raw_density'].shape[0]
  inp['lossmult'] = torch.rand(B, lm_ch, dtype=torch.float64, generator=torch.Generator().manual_seed(lm_ch)) + 0.5
  loss = dict(loss, loss_type=loss_type, inv_denom=1.0 / float(inp['lossmult'].expand(B, 3).sum()))
  out, g = R.grads(inp, cfg, loss)
  r = o_render.volumetric_rendering(out['rgb_samples'], out['weights'], out['t_aug'][:, :-1], inp['bg_rgb'],
                                    inp['far'][:, None], False)
  torch.testing.assert_close(out['rgb'], r['rgb'], rtol=1e-14, atol=1e-15)
  cfg_o = type('C', (), dict(data_loss_type=loss_type, charb_padding=R.f32(0.001), disable_multiscale_loss=False,
                             data_coarse_loss_mult=0.0, data_loss_mult=1.0))
  data, st = o_train.compute_data_loss(inp['target'], [dict(rgb=out['rgb'])], inp['lossmult'], cfg_o)
  torch.testing.assert_close(out['data'], data, rtol=1e-13, atol=0)
  torch.testing.assert_close(out['mse'], st['mses'][0], rtol=1e-13, atol=0)
  # gradient of the oracle's data loss through the same pixel
  leaves = {k: inp[k].detach().requires_grad_(True) for k in ('raw_density', 'raw_rgb')}
  rgb = R.composite(dict(inp, **leaves), cfg)['rgb']
  data_o, _ = o_train.compute_data_loss(inp['target'], [dict(rgb=rgb)], inp['lossmult'], cfg_o)
  g_o = torch.autograd.grad(data_o, list(leaves.values()))
  for k, go in zip(leaves, g_o):
    torch.testing.assert_close(g[k], go, rtol=1e-12, atol=1e-15)


def test_reference_bg_on_pins_the_branch():
  """`bg_on` chooses the background weight's branch whatever acc is (a saturated translucent ray has acc == 1 in
  fp32 and slightly less in fp64)."""
  inp, cfg, loss = _case('plain')
  B = inp['raw_density'].shape[0]
  _, g_on = R.grads(inp, cfg, loss, bg_on=torch.ones(B, dtype=torch.bool))
  _, g_off = R.grads(inp, cfg, loss, bg_on=torch.zeros(B, dtype=torch.bool))
  # with the background on, each weight's gradient loses dpx . bg: the two differ
  assert float((g_on['raw_density'] - g_off['raw_density']).abs().max()) > 1e-6
