"""Normals on a colourless proposal MLP, CPU side: the oracle vs the reference's real `Model.__call__` and
normal losses on a mini bounded config whose PropMLP computes density and predicted normals
(tests/golden/make_golden_prop_normals.py), and the layer plan of such an MLP."""
import torch

from multinerf_b200.models import MLPPlan
from model_golden import TOL, load, rand_of
from oracle import o_models, o_train
from util import close

TAG = 'minipropnormals'


def test_oracle_normals_on_every_level_match_reference_run():
  g, b, params, rays, bases = load(TAG)
  n = b.model.num_levels
  assert b.prop_mlp.disable_rgb and not b.prop_mlp.disable_density_normals and b.prop_mlp.enable_pred_normals
  for mode in ['det', 'rand']:
    rend, hist = o_models.model_apply(params, b, bases, rays, float(g['meta_train_frac']), True,
                                      rand=rand_of(g, mode, n), zero_glo=False)
    for lv in range(n):
      tag = f'{mode} level {lv}'
      close(hist[lv]['weights'].detach(), g[f'{mode}/hist{lv}/weights'], msg=f'{tag} weights', **TOL)
      close(rend[lv]['rgb'].detach(), g[f'{mode}/rend{lv}/rgb'], msg=f'{tag} pixels', **TOL)
      close(hist[lv]['grad_pred'].detach(), g[f'{mode}/hist{lv}/grad_pred'], msg=f'{tag} grad_pred', **TOL)
      close(hist[lv]['normals_pred'].detach(), g[f'{mode}/hist{lv}/normals_pred'], msg=f'{tag} normals_pred', **TOL)
      # golden density normals = fp64 central differences through the MLP (same bound as the model goldens)
      for k in ('raw_grad_density', 'normals'):
        close(hist[lv][k].detach(), g[f'{mode}/hist{lv}/{k}'], msg=f'{tag} {k}', atol=2e-3, rtol=2e-3)
      for k in ('normals', 'normals_pred'):
        close(rend[lv][k].detach(), g[f'{mode}/rend{lv}/{k}'], msg=f'{tag} rendered {k}', atol=2e-3, rtol=2e-3)
    close(torch.as_tensor(o_train.orientation_loss(rays.viewdirs, n, hist, b.config)).detach(),
          g[f'{mode}/loss_orientation'], msg='orientation', atol=1e-7, rtol=1e-3)
    close(torch.as_tensor(o_train.predicted_normal_loss(n, hist, b.config)).detach(),
          g[f'{mode}/loss_pred_normals'], msg='pred normals', atol=1e-7, rtol=2e-2)


def test_colourless_plan_names_layers_like_flax():
  g, b, params, rays, bases = load(TAG)
  for mname, cfg in [('NerfMLP_0', b.nerf_mlp), ('PropMLP_0', b.prop_mlp)]:
    plan = MLPPlan(cfg)
    ref = {k: tuple(v['kernel'].shape) for k, v in params[mname].items()}
    assert ref == {s.name: (s.in_dim, s.out_dim) for s in plan.specs}, mname
  prop = MLPPlan(b.prop_mlp)
  assert prop.normals_stage and not prop.ref_stage and prop.normals_head_cols == 64
  assert prop.one('grad_pred').name == f'Dense_{b.prop_mlp.net_depth + 1}'
  b.prop_mlp.enable_pred_normals = False
  dens_only = MLPPlan(b.prop_mlp)
  assert dens_only.normals_stage and dens_only.normals_head_cols == 0 and dens_only.one('grad_pred') is None
