"""GPU checks of mesh evaluation's edge cases: an empty mesh through render_mesh and evaluate_mesh with every colour
source (all misses, no fault), and the argument checks of ops.mesh_bvh rejecting bad input before any launch."""
import dataclasses
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def mods():
  from multinerf_b200 import lib, mesh, ops
  lib.require_device()
  return ops, mesh


@pytest.mark.parametrize('colour', ['none', 'vertex', 'texture'])
def test_evaluate_empty_mesh(mods, colour, tmp_path):
  ops, mesh = mods
  from multinerf_b200 import configs, datasets
  from test_gpu_mesh import _write_scene
  data = str(tmp_path / 'scene')
  _write_scene(data)
  config = configs.load_config(gin_bindings=[f"Config.data_dir = '{data}'", "Config.dataset_loader = 'blender'",
                                             'Config.near = 1.5', 'Config.far = 5.0']).config
  ds = datasets.load_dataset('test', data, dataclasses.replace(config, render_path=False), device='cuda')
  v = torch.zeros(0, 3, device='cuda')
  f = torch.zeros(0, 3, dtype=torch.int32, device='cuda')
  kw = dict(normals=torch.zeros(0, 3, device='cuda'))
  if colour == 'vertex':
    kw['rgb'] = torch.zeros(0, 3, dtype=torch.uint8, device='cuda')
  elif colour == 'texture':
    uv, tex = mesh.bake_texture(v, f, kw['normals'], 64, lambda p, n: torch.zeros(len(p), 3, dtype=torch.uint8,
                                                                                  device='cuda'))
    kw.update(uv=uv, texture=tex)
  r = mesh.render_mesh(v, f, ops.mesh_bvh(v, f), ds.generate_ray_batch(0).rays, bg=1.0, **kw)
  assert not bool(r['hit'].any()) and bool(torch.isinf(r['distance']).all())
  assert (r['rgb'] is None) == (colour == 'none')
  H, W = ds.height, ds.width
  reference = [(i, torch.full((H, W), 3.0, device='cuda'), torch.ones(H, W, device='cuda'),
                torch.as_tensor(ds.images[i], device='cuda')) for i in range(ds.size)]
  saved = []
  metrics = mesh.evaluate_mesh(v, f, ds, config, reference=reference, bg=1.0, save_fn=lambda i, r: saved.append(i),
                               **kw)
  torch.cuda.synchronize()
  assert saved == list(range(ds.size)) and len(metrics) == ds.size
  for m in metrics:
    assert m['coverage'] == 0 and math.isnan(m['spurious']) and math.isnan(m['depth_abs_rel'])
    assert np.isfinite(m['nerf_psnr'])
    assert ('psnr' in m) == (colour != 'none') and (colour == 'none' or np.isfinite(m['psnr']))


def test_bad_input_is_rejected_before_any_launch(mods):
  ops, _ = mods
  v = torch.tensor([[-1, -1, 0], [1, -1, 0], [0, 1, 0], [0, 0, 1]], dtype=torch.float32, device='cuda')
  f = torch.tensor([[0, 1, 2], [0, 1, 3]], dtype=torch.int32, device='cuda')
  bad_v = v.clone()
  bad_v[3, 1] = float('nan')
  before = ops.LAUNCHES
  for args in ((v, torch.tensor([[0, 1, 4]], dtype=torch.int32, device='cuda')),
               (v, torch.tensor([[0, -1, 2]], dtype=torch.int32, device='cuda')), (bad_v, f)):
    with pytest.raises(ValueError):
      ops.mesh_bvh(*args)
  torch.cuda.synchronize()
  assert ops.LAUNCHES == before
  bvh = ops.mesh_bvh(v, f)
  assert ops.LAUNCHES == before + 4                 # boxes, keys, topology, box fit
  o = torch.tensor([[0.0, 0.0, -1.0]], device='cuda')
  ops.mesh_trace(bvh, o, torch.tensor([[0.0, 0.0, 1.0]], device='cuda'), torch.zeros(1, device='cuda'),
                 torch.full((1,), 10.0, device='cuda'))
  assert ops.LAUNCHES == before + 5
