"""Generate tests/golden/model_miniviewindep.npz by EXECUTING the reference's real `Model.__call__`
(internal/models.py) and its losses (internal/train_utils.py) under the jax/flax/gin stand-ins, on a mini
bounded two-MLP config with view-independent colour (Model.use_viewdirs = False: the rgb head reads the trunk
output, models.py:512,584), density and predicted normals on both MLPs, both normal losses and GLO vectors
(whose Embed_0 parameter the reference keeps although no layer reads it).

Run where the reference sources are available (the path below):
    python tests/golden/make_golden_view_branch.py
The fixture has the key layout of make_golden_model.py (whose helpers it reuses) without the clip part.
"""
import dataclasses
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
from internal import configs as rconfigs  # noqa: E402
from internal import models, train_utils, utils  # noqa: E402
import make_golden_model as mgm  # noqa: E402

F = np.float32
TAG = 'miniviewindep'
SEED = 7
SPEC = dict(
    near=2.0, far=6.0, rays='sphere', B=12, train_frac=0.6,
    Config=dict(data_loss_type='mse', distortion_loss_mult=0.0, orientation_loss_mult=0.1,
                orientation_loss_target='normals_pred', orientation_coarse_loss_mult=0.01,
                predicted_normal_loss_mult=3e-4, predicted_normal_coarse_loss_mult=3e-5,
                data_coarse_loss_mult=0.1),
    Model=dict(num_levels=3, num_prop_samples=8, num_nerf_samples=8, single_jitter=False, use_viewdirs=False,
               num_glo_features=4, num_glo_embeddings=5),
    PropMLP=dict(net_depth=2, net_width=16, basis_shape='octahedron', basis_subdivisions=1, max_deg_point=16,
                 disable_rgb=True, disable_density_normals=False, enable_pred_normals=True),
    NerfMLP=dict(net_depth=5, net_width=32, bottleneck_width=16, net_width_viewdirs=16, basis_shape='octahedron',
                 basis_subdivisions=1, max_deg_point=16, disable_density_normals=False, enable_pred_normals=True,
                 density_bias=0.5))
CAM_IDX = 5


def main():
  rng = np.random.default_rng(SEED)
  spec = SPEC
  gin.clear()
  for cls in ['Model', 'PropMLP', 'NerfMLP']:
    gin.bind(cls, **spec[cls])
  config = rconfigs.Config(**spec['Config'])
  model = models.Model(config=config)
  B = spec['B']
  rays = mgm._rays(rng, B, spec['near'], spec['far'], spec['rays'])
  rays = dataclasses.replace(rays, cam_idx=rng.integers(0, CAM_IDX, (B, 1)).astype(np.int32))
  params = mgm._init_params(model, rng, rays)
  out = {'meta_tag': np.array(TAG)}
  for cls in ['Config', 'Model', 'PropMLP', 'NerfMLP']:
    for k, v in spec[cls].items():
      out[f'bind/{cls}/{k}'] = np.array(mgm._name(v))
  out.update({'meta_near': spec['near'], 'meta_far': spec['far'], 'meta_train_frac': spec['train_frac']})
  for f, v in rays.__dict__.items():
    if v is not None:
      out[f'rays/{f}'] = v
  out.update({'params/' + k: v for k, v in mgm._flatten(params).items()})
  target = rng.uniform(0, 1, (B, 3)).astype(F)
  out['target'] = target
  n = model.num_levels
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
