"""Generate tests/golden/model_minicontractnormals.npz by EXECUTING the reference's real `Model.__call__`
(internal/models.py) and its orientation / predicted-normal losses (internal/train_utils.py:162-197) under
the jax/flax/gin stand-ins, on a mini unbounded config: reciprocal ray distances and `warp_fn = contract` on
both MLPs, a colourless PropMLP with density and predicted normals, and a Ref-NeRF NerfMLP (density and
predicted normals, reflections, integrated directional encoding, predicted roughness).

The density normals are `value_and_grad` with respect to the world-space mean THROUGH
`coord.track_linearize(contract, ...)` (models.py:441-492, coord.py:39-60), so the warped covariance
J Sigma J^T moves with the mean.  In the stand-in both derivatives are fp64 central differences, the
contraction's nested inside the gradient's.  The inner step is made larger than the stand-in's default here
(see INNER_STEP): the outer difference of a noisy inner difference amplifies its round-off by 1 / (outer
step).  The cones are wide (radii 0.02-0.05) so that the covariance term is a visible part of the normals.

Run in the build container only (needs /root/reference):
    python tests/golden/make_golden_contract_normals.py
The fixture has the key layout of make_golden_prop_normals.py.
"""
import math
import os
import sys
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'standin'))
sys.path.insert(0, '/root/reference')
sys.path.insert(0, HERE)
np.math = math
for missing in ['dm_pix', 'cv2', 'rawpy', 'mediapy', 'optax', 'pycolmap', 'matplotlib', 'tensorflow']:
  try:
    __import__(missing)
  except Exception:  # pylint: disable=broad-except
    sys.modules[missing] = mock.MagicMock()

import gin  # noqa: E402  (the stand-in)
import jax  # noqa: E402
import jax.numpy as jnp  # noqa: E402
from internal import configs as rconfigs  # noqa: E402
from internal import coord, models, train_utils, utils  # noqa: E402
import make_golden_model as mgm  # noqa: E402

F = np.float32
TAG = 'minicontractnormals'
SEED = 7
# relative step of the contraction's central difference, nested inside the gradient's (stand-in default 1e-6).
# Measured against the oracle's autograd (fp32 and fp64 agree to far below this): at 1e-3 the golden's
# density normals are off by up to 0.14, at 1e-2 by up to 0.02 (raw_grad_density within 2 % + 1e-3)
INNER_STEP = 1e-2
SPEC = dict(
    near=0.2, far=1e6, B=12, train_frac=0.6,
    Config=dict(data_loss_type='mse', distortion_loss_mult=0.0, orientation_loss_mult=0.1,
                orientation_loss_target='normals_pred', orientation_coarse_loss_mult=0.01,
                predicted_normal_loss_mult=3e-4, predicted_normal_coarse_loss_mult=3e-5,
                data_coarse_loss_mult=0.1),
    Model=dict(raydist_fn=jnp.reciprocal, num_levels=3, num_prop_samples=8, num_nerf_samples=8,
               single_jitter=False, opaque_background=True),
    PropMLP=dict(warp_fn=coord.contract, net_depth=2, net_width=16, basis_shape='octahedron',
                 basis_subdivisions=1, max_deg_point=12, disable_rgb=True, disable_density_normals=False,
                 enable_pred_normals=True),
    NerfMLP=dict(warp_fn=coord.contract, net_depth=4, net_width=32, bottleneck_width=16, net_width_viewdirs=16,
                 basis_shape='octahedron', basis_subdivisions=1, max_deg_point=12,
                 disable_density_normals=False, enable_pred_normals=True, use_reflections=True,
                 use_directional_enc=True, deg_view=4, enable_pred_roughness=True, density_bias=0.5))


def _rays(rng, B, near, far):
  """Origins at radius 0.3-2 looking roughly through the origin: the first samples of some rays lie inside the
  unit ball, most of every ray outside it."""
  o = rng.normal(size=(B, 3))
  o = o / np.linalg.norm(o, axis=-1, keepdims=True) * rng.uniform(0.3, 2.0, (B, 1))
  d = -o / np.linalg.norm(o, axis=-1, keepdims=True) + rng.normal(size=(B, 3)) * 0.5
  d /= np.linalg.norm(d, axis=-1, keepdims=True)
  v = d.copy()
  d = d * rng.uniform(0.8, 1.2, (B, 1))
  return utils.Rays(origins=o.astype(F), directions=d.astype(F), viewdirs=v.astype(F),
                    radii=rng.uniform(0.02, 0.05, (B, 1)).astype(F), imageplane=np.zeros((B, 2), F),
                    lossmult=np.ones((B, 1), F), near=np.full((B, 1), near, F), far=np.full((B, 1), far, F),
                    cam_idx=np.zeros((B, 1), np.int32))


def _linearize(fn, primal):
  """The stand-in's jax.linearize with the step INNER_STEP * max(1, |primal|)."""
  out = fn(primal)
  p64 = np.asarray(primal, dtype=np.float64)

  def lin(v):
    v64 = np.asarray(v, dtype=np.float64)
    nv = np.linalg.norm(v64, axis=-1, keepdims=True)
    vhat = v64 / np.maximum(nv, 1e-300)
    h = INNER_STEP * np.maximum(1.0, np.linalg.norm(p64, axis=-1, keepdims=True))
    jax._state['x64'] += 1
    try:
      dd = (np.asarray(fn(p64 + h * vhat), dtype=np.float64) -
            np.asarray(fn(p64 - h * vhat), dtype=np.float64)) / (2 * h)
    finally:
      jax._state['x64'] -= 1
    return jax._cast(dd * nv)
  return out, lin


def main():
  rng = np.random.default_rng(SEED)
  spec = SPEC
  gin.clear()
  for cls in ['Model', 'PropMLP', 'NerfMLP']:
    gin.bind(cls, **spec[cls])
  config = rconfigs.Config(**spec['Config'])
  model = models.Model(config=config)
  B = spec['B']
  rays = _rays(rng, B, spec['near'], spec['far'])
  params = mgm._init_params(model, rng, rays)
  out = {'meta_tag': np.array(TAG)}
  for cls in ['Config', 'Model', 'PropMLP', 'NerfMLP']:
    for k, v in spec[cls].items():
      out[f'bind/{cls}/{k}'] = np.array(mgm._name(v))
  out.update({'meta_near': spec['near'], 'meta_far': spec['far'], 'meta_train_frac': spec['train_frac'],
              'meta_inner_step': INNER_STEP})
  for f, v in rays.__dict__.items():
    if v is not None:
      out[f'rays/{f}'] = v
  out.update({'params/' + k: v for k, v in mgm._flatten(params).items()})
  target = rng.uniform(0, 1, (B, 3)).astype(F)
  out['target'] = target
  n = model.num_levels
  with mock.patch.object(jax, 'linearize', _linearize):
    for mode in ['det', 'rand']:
      key = None
      if mode == 'rand':
        draws = []
        for lv in range(n):
          S = model.num_prop_samples if lv < n - 1 else model.num_nerf_samples
          j = rng.uniform(0, 1, (B, S)).astype(F)
          draws.append(j)
          out[f'{mode}/jitter{lv}'] = j
        key = jax.random.Stream(draws)
      renderings, ray_history = model.apply({'params': params}, key, rays, train_frac=spec['train_frac'],
                                            compute_extras=True, zero_glo=False)
      if mode == 'rand':
        assert not key.draws, 'unconsumed random draws'
      for lv, (r, h) in enumerate(zip(renderings, ray_history)):
        for k, v in r.items():
          out[f'{mode}/rend{lv}/{k}'] = np.asarray(v)
        for k, v in h.items():
          if v is not None:
            out[f'{mode}/hist{lv}/{k}'] = np.asarray(v)
        assert h['normals'] is not None and h['normals_pred'] is not None, lv
      batch = utils.Batch(rays=rays, rgb=target)
      data_loss, stats = train_utils.compute_data_loss(batch, renderings, rays, 1.0, config)
      out[f'{mode}/loss_data'] = np.asarray(data_loss)
      out[f'{mode}/mses'] = np.asarray(stats['mses'])
      out[f'{mode}/loss_interlevel'] = np.asarray(train_utils.interlevel_loss(ray_history, config))
      out[f'{mode}/loss_distortion'] = np.asarray(train_utils.distortion_loss(ray_history, config))
      out[f'{mode}/loss_orientation'] = np.asarray(train_utils.orientation_loss(rays, model, ray_history, config))
      out[f'{mode}/loss_pred_normals'] = np.asarray(train_utils.predicted_normal_loss(model, ray_history, config))
      print(mode, 'orientation', float(out[f'{mode}/loss_orientation']),
            'predicted normals', float(out[f'{mode}/loss_pred_normals']))
  path = os.path.join(HERE, f'model_{TAG}.npz')
  np.savez_compressed(path, **{k: np.asarray(v) for k, v in out.items()})
  print(f'model_{TAG}.npz', len(out), 'arrays')


if __name__ == '__main__':
  main()
