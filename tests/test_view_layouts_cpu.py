"""The view-branch layouts of the reference MLP, CPU side: no bottleneck (the Ref-NeRF ablation), no view MLP (with
GLO, and without a bottleneck) and a view MLP with several skips that ends on one.  The oracle against the reference's
real `Model.__call__` and losses on mini configs (tests/golden/make_golden_view_layouts.py), and the layer plan of each
layout against the reference's parameter tree: flax names, shapes, parameter counts, and the layout decisions the
forward and backward read."""
import numpy as np
import pytest
import torch

from multinerf_b200 import configs
from multinerf_b200.models import MLPPlan
from model_golden import TOL, load, rand_of
from oracle import o_models, o_train
from util import close

TAGS = ['mininobottleneck', 'miniviewdepth0', 'miniviewdepth0nb', 'miniviewskips']


def _plans(b):
  glo = b.model.num_glo_features
  out = {'NerfMLP_0': MLPPlan(b.nerf_mlp, b.model.use_viewdirs, glo_features=glo)}
  if not b.model.single_mlp:
    out['PropMLP_0'] = MLPPlan(b.prop_mlp, b.model.use_viewdirs)
  return out


@pytest.mark.parametrize('tag', TAGS)
def test_oracle_matches_reference_run(tag):
  g, b, params, rays, bases = load(tag)
  n = b.model.num_levels
  glo = b.model.num_glo_features > 0
  for mode in ['det', 'rand']:
    rend, hist = o_models.model_apply(params, b, bases, rays, float(g['meta_train_frac']), True,
                                      rand=rand_of(g, mode, n), zero_glo=not glo)
    for lv in range(n):
      tag_lv = f'{tag} {mode} level {lv}'
      for k in ('weights', 'density', 'rgb', 'sdist', 'grad_pred', 'normals_pred', 'roughness'):
        if f'{mode}/hist{lv}/{k}' in g.files:
          close(hist[lv][k].detach(), g[f'{mode}/hist{lv}/{k}'], msg=f'{tag_lv} {k}', **TOL)
      for k in ('rgb', 'acc', 'distance_mean', 'distance_median'):
        close(rend[lv][k].detach(), g[f'{mode}/rend{lv}/{k}'], msg=f'{tag_lv} rendered {k}', **TOL)
      for k in ('raw_grad_density', 'normals'):
        if f'{mode}/hist{lv}/{k}' in g.files:
          close(hist[lv][k].detach(), g[f'{mode}/hist{lv}/{k}'], msg=f'{tag_lv} {k}', atol=2e-3, rtol=2e-3)
    data, st = o_train.compute_data_loss(torch.tensor(g['target']), rend, rays.lossmult, b.config)
    close(data.detach(), g[f'{mode}/loss_data'], msg='data loss', atol=1e-6, rtol=1e-4)
    close(st['mses'].detach(), g[f'{mode}/mses'], msg='mses', atol=1e-6, rtol=1e-4)
    if f'{mode}/loss_orientation' in g.files:
      close(torch.as_tensor(o_train.orientation_loss(rays.viewdirs, n, hist, b.config)).detach(),
            g[f'{mode}/loss_orientation'], msg='orientation', atol=1e-7, rtol=1e-3)
      close(torch.as_tensor(o_train.predicted_normal_loss(n, hist, b.config)).detach(),
            g[f'{mode}/loss_pred_normals'], msg='pred normals', atol=1e-7, rtol=2e-2)


@pytest.mark.parametrize('tag', TAGS)
def test_plan_names_layers_like_flax(tag):
  g, b, params, rays, bases = load(tag)
  for mname, plan in _plans(b).items():
    ref = {k: tuple(v['kernel'].shape) for k, v in params[mname].items()}
    assert ref == {s.name: (s.in_dim, s.out_dim) for s in plan.specs}, mname
    assert plan.num_params == sum(v['kernel'].numel() + v['bias'].numel() for v in params[mname].values())
    # flax creation order: Dense_k is the k-th layer of the table
    assert [s.name for s in plan.specs] == [f'Dense_{k}' for k in range(len(plan.specs))]


def test_no_bottleneck_plan():
  g, b, params, rays, bases = load('mininobottleneck')
  plan = _plans(b)['NerfMLP_0']
  cfg = b.nerf_mlp
  assert plan.one('bottleneck') is None and not plan.has_bottleneck and plan.ref_stage
  # the view MLP reads [IDE | n.v]; the 11 head gradients sit in columns [0, 11) of d vin
  assert plan.vin_dim == plan.dir_dim + 1 and plan.enc_col0 == 0
  assert plan.slab_cols == plan.vin_pad and plan.d_vin_cols == plan.vin_pad
  assert sorted(c for _, c in plan.slab_heads) == [0, 1, 4, 7, 10]
  # the heads come straight after the trunk, the first view layer after the roughness head
  roles = [s.role for s in plan.specs]
  assert roles[cfg.net_depth:cfg.net_depth + 6] == ['density', 'grad_pred', 'diffuse', 'tint', 'roughness', 'view']
  assert plan.view_concat_after == [4] and plan.view_skips == [5] and plan.rgb_vin is None
  assert plan.vin_partials == 1


@pytest.mark.parametrize('tag', ['miniviewdepth0', 'miniviewdepth0nb'])
def test_no_view_mlp_plan(tag):
  g, b, params, rays, bases = load(tag)
  plan = _plans(b)['NerfMLP_0']
  r = plan.one('rgb')
  assert not plan.by_role('view') and plan.rgb_vin == 'all' and plan.vin_partials == 0
  assert (r.in_dim, r.in_pad, r.row_map) == (plan.vin_dim, plan.vin_pad, None)
  # the rgb head straight after the bottleneck (or after the last narrow head without one)
  assert plan.specs[-2].role == ('bottleneck' if plan.has_bottleneck else 'roughness') and plan.specs[-1] is r
  if tag == 'miniviewdepth0':
    assert plan.glo_features == 4 and plan.d_vin_cols == plan.vin_pad
    assert plan.vin_dim == b.nerf_mlp.bottleneck_width + 3 + 6 * b.nerf_mlp.deg_view + 4
  else:
    assert plan.vin_dim == plan.dir_dim + 1 and not plan.has_bottleneck


def test_several_view_skips_plan():
  g, b, params, rays, bases = load('miniviewskips')
  plan = _plans(b)['NerfMLP_0']
  Wv, vin = b.nerf_mlp.net_width_viewdirs, plan.vin_dim
  views = plan.by_role('view')
  assert len(views) == 5 and plan.view_concat_after == [2, 4]
  # layer 3 reads [hidden | vin]; layer 4 is the last and a skip, so the rgb head reads [hidden | vin] too
  assert plan.view_skips == [3] and plan.rgb_vin == 'tail' and plan.vin_partials == 2
  expect = np.concatenate([np.arange(Wv), Wv + np.arange(vin)])
  for sp in (views[3], plan.one('rgb')):
    assert (sp.in_dim, sp.in_pad) == (Wv + vin, Wv + plan.vin_pad)
    assert np.array_equal(sp.row_map, expect)
  assert all(sp.row_map is None for sp in (views[0], views[1], views[2], views[4]))


def test_shipped_config_layouts():
  # blender_refnerf.gin without a bottleneck: the bottleneck's parameters go, and the first view layer and the layer
  # after the skip read [IDE | n.v] (73 columns) without the 128 bottleneck columns
  b = configs.bundle_blender_refnerf()
  shipped = MLPPlan(b.nerf_mlp)
  b.nerf_mlp.bottleneck_width = 0
  nb = MLPPlan(b.nerf_mlp)
  bw, Wv, x = 128, b.nerf_mlp.net_width_viewdirs, shipped.x_dim
  assert shipped.num_params - nb.num_params == x * bw + bw + 2 * bw * Wv
  assert (nb.vin_dim, nb.vin_pad) == (73, 128)
  # 360.gin without a view MLP: the rgb head reads [bottleneck | dir enc] (283 columns, K = 320)
  b = configs.bundle_360()
  b.nerf_mlp.net_depth_viewdirs = 0
  p = MLPPlan(b.nerf_mlp)
  assert (p.one('rgb').in_dim, p.one('rgb').in_pad) == (283, 320) and p.rgb_vin == 'all'
  # blender_256.gin with a 9-layer view MLP: skips after layers 4 and 8, the rgb head reads [hidden | vin] (K = 448)
  b = configs.bundle_blender_256()
  b.nerf_mlp.net_depth_viewdirs = 9
  p = MLPPlan(b.nerf_mlp)
  assert p.view_concat_after == [4, 8] and p.view_skips == [5] and p.rgb_vin == 'tail'
  assert p.one('rgb').in_pad == 448
  # and one ending on its only skip: view_skips is empty, the rgb head is the only other consumer of vin
  b.nerf_mlp.net_depth_viewdirs = 5
  p = MLPPlan(b.nerf_mlp)
  assert p.view_concat_after == [4] and p.view_skips == [] and p.rgb_vin == 'tail' and p.vin_partials == 1


def test_ide_without_roughness_still_rejected():
  b = configs.bundle_blender_refnerf()
  b.nerf_mlp.enable_pred_roughness = False
  with pytest.raises(NotImplementedError, match='kappa_inv'):
    MLPPlan(b.nerf_mlp)
