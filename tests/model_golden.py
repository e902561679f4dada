"""The model fixtures tests/golden/model_<tag>.npz, written by running the reference's models.py and train_utils.py
(tests/golden/make_golden_model.py and its siblings): their configuration, parameters, rays and random draws."""
import os

import numpy as np
import torch

from multinerf_b200 import configs, geopoly
from util import GOLDEN


def load(tag):
  g = np.load(os.path.join(GOLDEN, f'model_{tag}.npz'))
  b = configs.Bundle()
  tgt = {'Config': b.config, 'Model': b.model, 'PropMLP': b.prop_mlp, 'NerfMLP': b.nerf_mlp}
  for k in g.files:
    if k.startswith('bind/'):
      _, cls, attr = k.split('/')
      v = g[k]
      if v.dtype.kind in 'biuf':
        v = v.item() if v.ndim == 0 else tuple(float(x) for x in v)      # e.g. bg_intensity_range
      else:
        v = str(v)
      setattr(tgt[cls], attr, v)
  params = {}
  for k in g.files:
    if k.startswith('params/'):
      d = params
      parts = k.split('/')[1:]
      for p in parts[:-1]:
        d = d.setdefault(p, {})
      d[parts[-1]] = torch.tensor(g[k])

  class R:
    exposure_idx = None
    exposure_values = None
  rays = R()
  for k in g.files:
    if k.startswith('rays/'):
      setattr(rays, k[5:], torch.tensor(g[k]))
  bases = {'nerf': geopoly.generate_basis(b.nerf_mlp.basis_shape, b.nerf_mlp.basis_subdivisions).astype(np.float32)}
  pm = b.nerf_mlp if b.model.single_mlp else b.prop_mlp
  bases['prop'] = geopoly.generate_basis(pm.basis_shape, pm.basis_subdivisions).astype(np.float32)
  return g, b, params, rays, bases


def rand_of(g, mode, n):
  if mode == 'det':
    return None
  r = {'jitter': [torch.tensor(g[f'rand/jitter{i}']) for i in range(n)]}
  if f'rand/density_noise0' in g.files:
    r['density_noise'] = [torch.tensor(g[f'rand/density_noise{i}']) for i in range(n)]
  for name in ('bottleneck_noise', 'bg'):           # present only at the levels that draw them
    if any(f'rand/{name}{i}' in g.files for i in range(n)):
      r[name] = [torch.tensor(g[f'rand/{name}{i}']) if f'rand/{name}{i}' in g.files else None for i in range(n)]
  return r


# per-key tolerances: fp32 throughout; the stand-in's Jacobians are fp64 central differences
TOL = dict(atol=2e-5, rtol=2e-4)
