"""CPU checks of mesh evaluation: the BVH restatement's tree invariants (tests/mesh_trace_ref.py), its brute-force
closest hit against an analytic sphere, Config.mesh_eval parsing and its NDC rejection, and the metric helpers."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import mesh_trace_ref as ref  # noqa: E402


def _soup(n, seed=0, scale=1.0, offset=0.0):
  rng = np.random.default_rng(seed)
  centre = rng.uniform(-1, 1, (n, 1, 3))
  v = (offset + scale * (centre + 0.05 * rng.normal(size=(n, 3, 3)))).astype(np.float32).reshape(-1, 3)
  return v, np.arange(3 * n, dtype=np.int32).reshape(n, 3)


def degenerate_cases():
  """(name, vertices, faces): the inputs the BVH must handle, shared with the GPU test."""
  cases = [('soup', *_soup(300)), ('one_face', *_soup(1)), ('two_faces', *_soup(2))]
  v = np.tile(np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32), (64, 1))
  cases.append(('same_centroid', v, np.arange(192, dtype=np.int32).reshape(64, 3)))
  v, f = _soup(100, seed=1)
  v[3 * np.arange(0, 100, 3) + 1] = v[3 * np.arange(0, 100, 3)]            # every third face has zero area
  cases.append(('zero_area', v, f))
  cases.append(('far_coords', *_soup(200, seed=2, scale=10.0, offset=1e6)))
  return cases


def check_tree(t, F):
  """Every face in exactly one leaf, every box contains its children, every internal node reached, depth <= 63."""
  assert sorted(t['leaf_face'].tolist()) == list(range(F))
  if F < 2:
    return
  ch = t['children']
  assert sorted(ch.reshape(-1).tolist()) == list(range(1, 2 * F - 1))        # each node but the root once
  nb = t['node_box']
  for i in range(F - 1):
    for c in ch[i]:
      assert (nb[i, :3] <= nb[c, :3]).all() and (nb[i, 3:] >= nb[c, 3:]).all()
  assert t['depth'].max() <= 63
  assert (t['parent'][ch[:, 0]] == np.arange(F - 1)).all() and t['parent'][0] == -1


@pytest.mark.parametrize('case', degenerate_cases(), ids=lambda c: c[0])
def test_tree_invariants(case):
  _, v, f = case
  check_tree(ref.build(v, f), len(f))


def test_keys_are_unique_and_quantised():
  v, f = _soup(500, seed=3)
  _, c = ref.face_boxes(v, f)
  k = ref.morton_keys(c)
  assert len(np.unique(k)) == len(k) and (k >= 0).all() and (k >> 62 == 0).all()
  assert ((k & 0xffffffff) == np.arange(len(k))).all()
  # the centroid with the least x, y, z in every axis gets cell 0; the greatest gets 1023
  v = np.array([[0, 0, 0], [0, 0, 0], [0, 0, 0], [1, 2, 3], [1, 2, 3], [1, 2, 3]], np.float32)
  k = ref.morton_keys(ref.face_boxes(v, np.arange(6, dtype=np.int32).reshape(2, 3))[1])
  assert k[0] >> 32 == 0 and k[1] >> 32 == (1 << 30) - 1


def _uv_sphere(n_theta=24, n_phi=48, radius=1.0):
  th = np.linspace(0, np.pi, n_theta + 1)
  ph = np.linspace(0, 2 * np.pi, n_phi, endpoint=False)
  T, P = np.meshgrid(th, ph, indexing='ij')
  v = radius * np.stack([np.sin(T) * np.cos(P), np.sin(T) * np.sin(P), np.cos(T)], -1).reshape(-1, 3)
  idx = np.arange((n_theta + 1) * n_phi).reshape(n_theta + 1, n_phi)
  a, b = idx[:-1], np.roll(idx[:-1], -1, 1)
  c, d = idx[1:], np.roll(idx[1:], -1, 1)
  f = np.concatenate([np.stack([a, c, b], -1).reshape(-1, 3), np.stack([b, c, d], -1).reshape(-1, 3)])
  return v.astype(np.float32), f.astype(np.int32)


def test_brute_force_against_analytic_sphere():
  v, f = _uv_sphere()
  rng = np.random.default_rng(4)
  N = 600
  o = rng.normal(size=(N, 3)) * 0.2 + np.array([0, 0, -4.0])
  target = rng.uniform(-1.2, 1.2, (N, 3)) * np.array([1, 1, 0])
  d = target - o
  face, t, bary, exempt = ref.brute_force(v, f, o, d, np.zeros(N), np.full(N, np.inf))
  # analytic ray / unit-sphere intersection along unnormalised d
  a = (d * d).sum(-1)
  b = 2 * (o * d).sum(-1)
  c = (o * o).sum(-1) - 1
  disc = b * b - 4 * a * c
  hit_true = disc > 0
  t_true = np.where(hit_true, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a), np.inf)
  # the polygonal sphere lies inside the unit sphere, within the sagitta of its largest facet
  sag = 1 - np.cos(np.pi / 24)
  sure = hit_true & (np.sqrt(np.maximum(disc, 0)) / np.sqrt(a) > 2 * np.sqrt(2 * sag))
  assert (face[sure] >= 0).all()
  assert (face[~hit_true] < 0).all()
  hit = face >= 0
  assert (np.abs(t[hit & sure] - t_true[hit & sure]) * np.sqrt(a[hit & sure]) < 3 * sag).all()
  # the hit point lies on the reported face, at the reported barycentrics
  p = o[hit] + t[hit, None] * d[hit]
  q = v[f[face[hit]]].astype(np.float64)
  rec = (1 - bary[hit].sum(-1))[:, None] * q[:, 0] + bary[hit, :1] * q[:, 1] + bary[hit, 1:] * q[:, 2]
  assert np.abs(p - rec).max() < 1e-9
  assert exempt.mean() < 0.2


def test_brute_force_tie_rule_and_interval():
  # two copies of one triangle: the lower index wins; a near beyond it misses; a far before it misses
  v = np.array([[-1, -1, 0], [1, -1, 0], [0, 1, 0]], np.float32)
  f = np.array([[0, 1, 2], [0, 1, 2]], np.int32)
  o = np.array([[0, 0, -1.0]] * 3)
  d = np.array([[0, 0, 1.0]] * 3)
  face, t, _, exempt = ref.brute_force(v, f, o, d, np.array([0, 1.5, 0]), np.array([np.inf, np.inf, 0.5]))
  assert face.tolist() == [0, -1, -1] and t[0] == 1.0
  assert exempt[0]                        # two candidates at the same t


def test_config_mesh_eval_parsing_and_ndc():
  from multinerf_b200 import configs, mesh
  b = configs.load_config([], ['Config.mesh_eval = True'])
  assert b.config.mesh_eval is True and configs.Config().mesh_eval is False

  class Plan:
    warp_fn = None

  class Bundle:
    pass
  for ff in (False, True):
    bb = Bundle()
    bb.config = configs.load_config([], ['Config.mesh_eval = True', f'Config.forward_facing = {ff}']).config
    bb.nerf_mlp = Plan()
    if ff:
      with pytest.raises(ValueError, match='mesh_eval'):
        mesh.validate_config(bb)
    else:
      assert mesh.validate_config(bb) == 'density'


def test_image_metrics_matches_the_evaluate_block():
  """eval_lib.image_metrics against the statements eval_lib.evaluate ran before it was factored out."""
  from multinerf_b200 import configs, eval_lib, image
  import dataclasses
  rng = np.random.default_rng(5)
  rgb, rgb_cc, gt = (rng.uniform(0, 1, (20, 24, 3)) for _ in range(3))
  harness = image.MetricHarness()
  post = lambda z: z ** (1 / 2.2)
  for quant, crop in ((True, 0), (False, 3), (True, 2)):
    config = dataclasses.replace(configs.Config(), eval_quantize_metrics=quant, eval_crop_borders=crop)
    r, rc, g = post(rgb), post(rgb_cc), post(gt)
    if quant:
      r, rc = np.round(r * 255) / 255, np.round(rc * 255) / 255
    if crop > 0:
      r, rc, g = r[crop:-crop, crop:-crop], rc[crop:-crop, crop:-crop], g[crop:-crop, crop:-crop]
    want = [harness(r, g), harness(rc, g)]
    got = eval_lib.image_metrics(config, post, harness, gt, rgb, rgb_cc)
    assert got == want


def test_mesh_metrics_on_fixed_arrays():
  from multinerf_b200 import configs, image, mesh
  import dataclasses
  config = dataclasses.replace(configs.Config(), eval_quantize_metrics=False)
  H, W = 2, 3
  gt = np.full((H, W, 3), 0.5)
  hit = torch.tensor([[True, True, False], [True, False, False]])
  dist = torch.tensor([[1.0, 2.0, np.inf], [4.0, np.inf, np.inf]])
  render = dict(hit=hit, distance=dist, normals=None, rgb=torch.full((H, W, 3), 0.5))
  acc = np.array([[1.0, 0.9, 0.8], [0.1, 0.2, 0.7]])
  dm = np.array([[2.0, 2.0, 3.0], [4.0, 5.0, 6.0]])
  nerf = np.full((H, W, 3), 0.25)
  m = mesh.mesh_metrics(render, gt, config, reference=(dm, acc, nerf))
  assert m['psnr'] == image.MetricHarness()(np.full((H, W, 3), 0.5), gt)['psnr']
  assert m['nerf_psnr'] == pytest.approx(-10 * np.log10(0.0625))
  assert m['coverage'] == pytest.approx(2 / 4)          # acc >= 0.5 at 4 pixels; the mesh hits 2 of them
  assert m['spurious'] == pytest.approx(1 / 3)          # 3 hits, 1 where acc < 0.5
  assert m['depth_abs_rel'] == pytest.approx((0.5 + 0.0) / 2)
  render['rgb'] = None
  m = mesh.mesh_metrics(render, gt, config)
  assert m == {}
  render['hit'] = torch.zeros(H, W, dtype=torch.bool)
  m = mesh.mesh_metrics(render, gt, config, reference=(dm, acc, nerf))
  assert m['coverage'] == 0 and np.isnan(m['spurious']) and np.isnan(m['depth_abs_rel'])
