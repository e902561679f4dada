"""Density normals through the scene contraction, CPU side: the oracle against the reference's real
`Model.__call__` and normal losses on a mini unbounded config (reciprocal ray distances, `warp_fn = contract`
on both MLPs, normals on every level; tests/golden/make_golden_contract_normals.py).

The reference differentiates density with respect to the WORLD-space mean through
coord.track_linearize(contract, mean, cov), so the warped covariance J Sigma J^T depends on the mean too
(models.py:441-492, coord.py:39-60).  The second test drops that term and checks the fixture tells the
difference.
"""
from unittest import mock

import pytest
import torch

from multinerf_b200.models import MLPPlan
from model_golden import TOL, load, rand_of
from oracle import o_coord, o_models, o_train
from util import close

TAG = 'minicontractnormals'
# The golden's gradient is a central difference (outer, step 1e-7) of a central difference (the contraction's
# Jacobian, relative step 1e-2): measured against the oracle's fp32 and fp64 autograd it is off by up to 2 %
# (+ 1e-3) in raw_grad_density and 0.02 in the normals, whose length is clamped where |grad| < sqrt(eps).
TOL_GRAD = dict(atol=2e-3, rtol=3e-2)
TOL_NORMALS = dict(atol=3e-2, rtol=0)


def _apply(g, b, params, rays, bases, mode):
  return o_models.model_apply(params, b, bases, rays, float(g['meta_train_frac']), True,
                              rand=rand_of(g, mode, b.model.num_levels), zero_glo=False)


def _track_linearize_mean_term_only(mean, cov):
  """track_linearize_contract with J treated as a constant inside J Sigma J^T."""
  jac = o_coord.contract_jacobian(mean).detach()
  return o_coord.contract(mean), jac @ cov @ jac.transpose(-1, -2)


@pytest.mark.parametrize('mode', ['det', 'rand'])
def test_oracle_contract_normals_match_reference_run(mode):
  g, b, params, rays, bases = load(TAG)
  n = b.model.num_levels
  assert b.prop_mlp.warp_fn == b.nerf_mlp.warp_fn == 'contract' and b.model.raydist_fn == 'reciprocal'
  rend, hist = _apply(g, b, params, rays, bases, mode)
  for lv in range(n):
    tag = f'{mode} level {lv}'
    close(hist[lv]['weights'].detach(), g[f'{mode}/hist{lv}/weights'], msg=f'{tag} weights', **TOL)
    close(rend[lv]['rgb'].detach(), g[f'{mode}/rend{lv}/rgb'], msg=f'{tag} pixels', **TOL)
    # heads of contracted features: far samples' J Sigma J^T cancels large terms in fp32 (as for density in
    # test_oracle_model_golden.py)
    close(hist[lv]['grad_pred'].detach(), g[f'{mode}/hist{lv}/grad_pred'], msg=f'{tag} grad_pred',
          atol=1e-3, rtol=1e-3)
    close(hist[lv]['normals_pred'].detach(), g[f'{mode}/hist{lv}/normals_pred'], msg=f'{tag} normals_pred',
          atol=2e-3, rtol=2e-3)
    close(hist[lv]['raw_grad_density'].detach(), g[f'{mode}/hist{lv}/raw_grad_density'],
          msg=f'{tag} raw_grad_density', **TOL_GRAD)
    close(hist[lv]['normals'].detach(), g[f'{mode}/hist{lv}/normals'], msg=f'{tag} normals', **TOL_NORMALS)
    close(rend[lv]['normals'].detach(), g[f'{mode}/rend{lv}/normals'], msg=f'{tag} rendered normals',
          **TOL_NORMALS)
  close(torch.as_tensor(o_train.orientation_loss(rays.viewdirs, n, hist, b.config)).detach(),
        g[f'{mode}/loss_orientation'], msg='orientation', atol=1e-7, rtol=1e-3)
  close(torch.as_tensor(o_train.predicted_normal_loss(n, hist, b.config)).detach(),
        g[f'{mode}/loss_pred_normals'], msg='pred normals', atol=1e-7, rtol=2e-2)


def test_fixture_needs_the_covariance_term():
  g, b, params, rays, bases = load(TAG)
  with mock.patch.object(o_coord, 'track_linearize_contract', _track_linearize_mean_term_only):
    _, hist = _apply(g, b, params, rays, bases, 'det')
  for lv in range(b.model.num_levels):
    err = (hist[lv]['normals'].detach() - torch.tensor(g[f'det/hist{lv}/normals'])).abs()
    assert float(err.max()) > 5 * TOL_NORMALS['atol'], (lv, float(err.max()))


def test_contract_plan_with_density_normals():
  _, b, _, _, _ = load(TAG)
  prop, nerf = MLPPlan(b.prop_mlp), MLPPlan(b.nerf_mlp)
  assert prop.density_normals and prop.normals_stage and not prop.ref_stage
  assert nerf.density_normals and nerf.ref_stage
