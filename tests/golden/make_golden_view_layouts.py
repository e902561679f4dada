"""Generate tests/golden/model_<tag>.npz for the view-branch layouts of the reference MLP by EXECUTING the reference's
real `Model.__call__` (internal/models.py) and its losses (internal/train_utils.py) under the jax/flax/gin stand-ins,
on mini bounded configs:

  mininobottleneck   Ref-NeRF without a bottleneck (bottleneck_width = 0, models.py:526-537): IDE, predicted
                     roughness, diffuse colour, specular tint, n.v, predicted normals and both normal losses; the
                     view MLP reads [IDE | n.v]
  miniviewdepth0     no view MLP (net_depth_viewdirs = 0) with GLO: the rgb head reads [bottleneck | dir enc | GLO]
  miniviewdepth0nb   no view MLP and no bottleneck: rgb = Dense(3)([IDE | n.v])
  miniviewskips      a view MLP with two skips that ends on the second (net_depth_viewdirs = 5, skip_layer_dir = 2),
                     with GLO: the rgb head reads [hidden | view input]

Run where the reference sources are available (the path below):
    python tests/golden/make_golden_view_layouts.py
The fixtures have the key layout of make_golden_model.py (whose helpers this reuses) without the clip part.
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

# Ref-NeRF on one MLP (the shipped blender_refnerf.gin layout at mini widths), both normal losses
REFNERF = dict(
    near=2.0, far=6.0, rays='sphere', B=12, train_frac=0.7, cam_idx=0,
    Config=dict(data_loss_type='mse', distortion_loss_mult=0.0, orientation_loss_mult=0.1,
                orientation_loss_target='normals_pred', predicted_normal_loss_mult=3e-4,
                orientation_coarse_loss_mult=0.01, predicted_normal_coarse_loss_mult=3e-5,
                interlevel_loss_mult=0.0, data_coarse_loss_mult=0.1),
    Model=dict(num_levels=2, single_mlp=True, num_prop_samples=8, num_nerf_samples=8, anneal_slope=0.,
               dilation_multiplier=0., dilation_bias=0., single_jitter=False, resample_padding=0.01),
    PropMLP=dict(),
    NerfMLP=dict(net_depth=5, net_width=32, net_depth_viewdirs=6, net_width_viewdirs=16,
                 basis_shape='octahedron', basis_subdivisions=1, disable_density_normals=False,
                 enable_pred_normals=True, use_directional_enc=True, use_reflections=True, deg_view=5,
                 enable_pred_roughness=True, use_diffuse_color=True, use_specular_tint=True,
                 use_n_dot_v=True, bottleneck_width=0, density_bias=0.5, max_deg_point=16))

# two MLPs, view directions encoded per ray, GLO vectors of five cameras
GLO = dict(
    near=2.0, far=6.0, rays='sphere', B=12, train_frac=0.6, cam_idx=5,
    Config=dict(data_loss_type='mse', distortion_loss_mult=0.0, data_coarse_loss_mult=0.1),
    Model=dict(num_levels=3, num_prop_samples=8, num_nerf_samples=8, single_jitter=False, num_glo_features=4,
               num_glo_embeddings=5),
    PropMLP=dict(net_depth=2, net_width=16, basis_shape='octahedron', basis_subdivisions=1, max_deg_point=16,
                 disable_rgb=True, disable_density_normals=True),
    NerfMLP=dict(net_depth=5, net_width=32, bottleneck_width=16, net_width_viewdirs=16, basis_shape='octahedron',
                 basis_subdivisions=1, max_deg_point=16, disable_density_normals=True, deg_view=3,
                 density_bias=0.5))


def _with(spec, **nerf):
  out = {k: (dict(v) if isinstance(v, dict) else v) for k, v in spec.items()}
  out['NerfMLP'].update(nerf)
  return out


SPECS = {
    'mininobottleneck': (11, REFNERF),
    'miniviewdepth0': (12, _with(GLO, net_depth_viewdirs=0)),
    'miniviewdepth0nb': (13, _with(REFNERF, net_depth_viewdirs=0)),
    'miniviewskips': (14, _with(GLO, net_depth_viewdirs=5, skip_layer_dir=2)),
}


def make(tag):
  seed, spec = SPECS[tag]
  rng = np.random.default_rng(seed)
  gin.clear()
  for cls in ['Model', 'PropMLP', 'NerfMLP']:
    gin.bind(cls, **spec[cls])
  config = rconfigs.Config(**spec['Config'])
  model = models.Model(config=config)
  B = spec['B']
  rays = mgm._rays(rng, B, spec['near'], spec['far'], spec['rays'])
  if spec['cam_idx']:
    rays = dataclasses.replace(rays, cam_idx=rng.integers(0, spec['cam_idx'], (B, 1)).astype(np.int32))
  params = mgm._init_params(model, rng, rays)
  out = {'meta_tag': np.array(tag)}
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
  normals = not spec['NerfMLP'].get('disable_density_normals', True)
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
    batch = utils.Batch(rays=rays, rgb=target)
    data_loss, stats = train_utils.compute_data_loss(batch, renderings, rays, 1.0, config)
    out[f'{mode}/loss_data'] = np.asarray(data_loss)
    out[f'{mode}/mses'] = np.asarray(stats['mses'])
    out[f'{mode}/loss_interlevel'] = np.asarray(train_utils.interlevel_loss(ray_history, config))
    out[f'{mode}/loss_distortion'] = np.asarray(train_utils.distortion_loss(ray_history, config))
    if normals:
      out[f'{mode}/loss_orientation'] = np.asarray(train_utils.orientation_loss(rays, model, ray_history, config))
      out[f'{mode}/loss_pred_normals'] = np.asarray(train_utils.predicted_normal_loss(model, ray_history, config))
    print(tag, mode, 'data loss', float(out[f'{mode}/loss_data']))
  path = os.path.join(HERE, f'model_{tag}.npz')
  np.savez_compressed(path, **{k: np.asarray(v) for k, v in out.items()})
  print(f'model_{tag}.npz', len(out), 'arrays')


def main():
  for tag in (sys.argv[1:] or SPECS):
    make(tag)


if __name__ == '__main__':
  main()
