"""View-independent colour (Model.use_viewdirs = False), CPU side: the oracle vs the reference's real
`Model.__call__` and losses on a mini config whose NerfMLP puts its rgb head on the trunk output
(tests/golden/make_golden_view_branch.py), the layer plan of such an MLP, and the colour-branch layouts the
reference itself cannot run, which the plan rejects at construction."""
import pytest
import torch

from multinerf_b200 import configs
from multinerf_b200.models import MLPPlan
from model_golden import TOL, load, rand_of
from oracle import o_models, o_train
from util import close

TAG = 'miniviewindep'


def test_oracle_view_independent_colour_matches_reference_run():
  g, b, params, rays, bases = load(TAG)
  n = b.model.num_levels
  assert not b.model.use_viewdirs and b.model.num_glo_features > 0
  for mode in ['det', 'rand']:
    rend, hist = o_models.model_apply(params, b, bases, rays, float(g['meta_train_frac']), True,
                                      rand=rand_of(g, mode, n), zero_glo=False)
    for lv in range(n):
      tag = f'{mode} level {lv}'
      for k in ('weights', 'density', 'rgb', 'sdist', 'grad_pred', 'normals_pred'):
        close(hist[lv][k].detach(), g[f'{mode}/hist{lv}/{k}'], msg=f'{tag} {k}', **TOL)
      for k in ('rgb', 'acc', 'distance_mean', 'distance_median'):
        close(rend[lv][k].detach(), g[f'{mode}/rend{lv}/{k}'], msg=f'{tag} rendered {k}', **TOL)
      for k in ('raw_grad_density', 'normals'):
        close(hist[lv][k].detach(), g[f'{mode}/hist{lv}/{k}'], msg=f'{tag} {k}', atol=2e-3, rtol=2e-3)
      assert f'{mode}/rend{lv}/roughness' not in g.files
    data, st = o_train.compute_data_loss(torch.tensor(g['target']), rend, rays.lossmult, b.config)
    close(data.detach(), g[f'{mode}/loss_data'], msg='data loss', atol=1e-6, rtol=1e-4)
    close(st['mses'].detach(), g[f'{mode}/mses'], msg='mses', atol=1e-6, rtol=1e-4)
    close(torch.as_tensor(o_train.interlevel_loss(hist, b.config)).detach(), g[f'{mode}/loss_interlevel'],
          msg='interlevel', atol=1e-7, rtol=1e-4)
    close(torch.as_tensor(o_train.orientation_loss(rays.viewdirs, n, hist, b.config)).detach(),
          g[f'{mode}/loss_orientation'], msg='orientation', atol=1e-7, rtol=1e-3)
    close(torch.as_tensor(o_train.predicted_normal_loss(n, hist, b.config)).detach(),
          g[f'{mode}/loss_pred_normals'], msg='pred normals', atol=1e-7, rtol=2e-2)


def test_view_independent_plan_names_layers_like_flax():
  g, b, params, rays, bases = load(TAG)
  glo = b.model.num_glo_features
  for mname, cfg in [('NerfMLP_0', b.nerf_mlp), ('PropMLP_0', b.prop_mlp)]:
    plan = MLPPlan(cfg, b.model.use_viewdirs, glo_features=glo if mname == 'NerfMLP_0' else 0)
    ref = {k: tuple(v['kernel'].shape) for k, v in params[mname].items()}
    assert ref == {s.name: (s.in_dim, s.out_dim) for s in plan.specs}, mname
    assert plan.num_params == sum(v['kernel'].numel() + v['bias'].numel() for v in params[mname].values())
  assert tuple(params['Embed_0']['embedding'].shape) == (b.model.num_glo_embeddings, glo)
  nerf = MLPPlan(b.nerf_mlp, False, glo_features=glo)
  assert nerf.rgb_on_trunk and nerf.normals_stage and not nerf.ref_stage and nerf.normals_head_cols == 64
  assert [s.role for s in nerf.specs[-3:]] == ['density', 'grad_pred', 'rgb']
  assert nerf.one('rgb').in_dim == nerf.x_dim and nerf.one('bottleneck') is None and not nerf.by_role('view')
  # the stacked head's bias block: [b_density | b_rgb] adjacent in the flat buffer
  assert nerf.one('rgb').b_off == nerf.one('density').b_off + 1


def test_view_independent_param_counts_of_shipped_configs():
  # blender_256.gin under Model.use_viewdirs = False: the bottleneck and the view MLP go, Dense(3) reads the trunk
  b = configs.bundle_blender_256()
  shipped = MLPPlan(b.nerf_mlp)
  vi = MLPPlan(b.nerf_mlp, use_viewdirs=False)
  W = b.nerf_mlp.net_width
  assert [s.role for s in vi.specs] == ['trunk'] * b.nerf_mlp.net_depth + ['density', 'rgb']
  assert vi.one('rgb').in_dim == W and vi.num_params == sum(
      s.in_dim * s.out_dim + s.out_dim for s in shipped.specs if s.role in ('trunk', 'density')) + W * 3 + 3
  b = configs.bundle_360()
  vi = MLPPlan(b.nerf_mlp, use_viewdirs=False)
  assert (vi.one('rgb').in_dim, vi.one('rgb').in_pad) == (1024, 1024)


def test_colour_branch_layouts_the_reference_cannot_run_are_rejected():
  b = configs.bundle_blender_256()
  n = b.nerf_mlp
  n.use_diffuse_color = True
  with pytest.raises(ValueError, match='models.py:591'):
    MLPPlan(n, use_viewdirs=False)
  n.use_diffuse_color = False
  n.bottleneck_width = 0
  with pytest.raises(ValueError, match='models.py:552-554'):
    MLPPlan(n)
  n.use_reflections, n.disable_density_normals = True, False
  with pytest.raises(ValueError, match='models.py:567-568'):
    MLPPlan(n, glo_features=4)
  # the Ref-NeRF flags without view directions are accepted, as in the reference: none of their heads is created
  r = configs.bundle_blender_256().nerf_mlp
  r.use_reflections = r.use_n_dot_v = r.enable_pred_roughness = r.use_specular_tint = True
  r.use_directional_enc, r.disable_density_normals = True, False
  plan = MLPPlan(r, use_viewdirs=False)
  assert [s.role for s in plan.specs if s.role not in ('trunk',)] == ['density', 'rgb']
  assert plan.normals_stage and not plan.ref_stage
