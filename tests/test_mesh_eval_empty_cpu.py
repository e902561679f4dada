"""mesh.render_mesh on a mesh without faces: every ray misses and nothing is traced or gathered, so the all-miss
render comes back on any device (here the CPU), with vertex colours, normals or a texture given as [0, ...] arrays."""
import math
import os
import sys
from types import SimpleNamespace

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _rays(H=3, W=4):
  g = torch.Generator().manual_seed(0)
  return SimpleNamespace(origins=torch.randn(H, W, 3, generator=g), directions=torch.randn(H, W, 3, generator=g),
                         near=torch.zeros(H, W, 1), far=torch.full((H, W, 1), math.inf))


@pytest.mark.parametrize('colour', ['none', 'vertex', 'texture'])
def test_render_mesh_without_faces_is_all_misses(colour):
  from multinerf_b200 import mesh
  v, f = torch.zeros(0, 3), torch.zeros(0, 3, dtype=torch.int32)
  kw = dict(normals=torch.zeros(0, 3))
  if colour == 'vertex':
    kw['rgb'] = torch.zeros(0, 3, dtype=torch.uint8)
  elif colour == 'texture':
    kw.update(uv=torch.zeros(0, 3, 2), texture=torch.zeros(8, 8, 3, dtype=torch.uint8))
  r = mesh.render_mesh(v, f, None, _rays(), bg=0.25, **kw)
  assert r['hit'].shape == (3, 4) and not bool(r['hit'].any())
  assert r['distance'].shape == (3, 4) and bool(torch.isinf(r['distance']).all())
  assert r['normals'].shape == (3, 4, 3) and bool((r['normals'] == 0).all())
  if colour == 'none':
    assert r['rgb'] is None
  else:
    assert r['rgb'].shape == (3, 4, 3) and bool((r['rgb'] == 0.25).all())
