"""Smooth activations of the Dense layers (MLP.net_activation = softplus | silu, internal/models.py:457,578) on the GPU:
the FWD / DGRAD epilogues that store and read the pre-activation z, the head backward and the second-order term of the
density normals against torch, and the model against the CPU oracle (whose density normals are taken by
torch.autograd with create_graph, so they include the second-order term).  Needs an H100.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from model_parity import (beyond, check_train_step, grad_report, graph_matches_eager, level_jitter, mini360,
                          mini_refnerf, mlp_leaves, pinned_forward, synth_case, synth_rays, train_step, worst)
from util import close

pytestmark = pytest.mark.gpu

ACTS = ['softplus', 'silu']


@pytest.fixture(scope='module')
def mods():
  from multinerf_b200 import lib, models, ops, train_utils
  lib.require_device()
  return models, train_utils, ops, lib


def _bf(x):
  return x.to(torch.bfloat16)


def _act(name):
  return {'softplus': F.softplus, 'silu': F.silu}[name]


def _d1(name, z):
  s = torch.sigmoid(z)
  return s if name == 'softplus' else s * (1 + z * (1 - s))


def _code(lib, name):
  return {'softplus': lib.ACT_SOFTPLUS, 'silu': lib.ACT_SILU}[name]


# ------------------------------------------------------------------ kernels

@pytest.mark.parametrize('name', ACTS)
@pytest.mark.parametrize('N', [64, 128, 256, 1024])
def test_gemm_fwd_writes_activation_and_z(mods, name, N):
  _, _, ops, lib = mods
  M, K = 300, 192
  g = torch.Generator().manual_seed(N)
  a, w = _bf(torch.randn(M, K, generator=g)).cuda(), _bf(torch.randn(N, K, generator=g) * 0.1).cuda()
  bias = torch.randn(N, generator=g).cuda()
  out = torch.empty(M, N, device='cuda', dtype=torch.bfloat16)
  z = torch.empty(M, N, device='cuda', dtype=torch.bfloat16)
  ops.gemm(lib.GEMM_FWD, a, w, out, m=M, n=N, k=K, act=_code(lib, name), bias=bias, z=z)
  zr = a.float() @ w.float().t() + bias
  close(z.float(), zr, atol=2e-2, rtol=1e-2, msg='z')
  close(out.float(), _act(name)(zr), atol=2e-2, rtol=1e-2, msg='a(z)')
  # the render path: no z
  out2 = torch.empty_like(out)
  ops.gemm(lib.GEMM_FWD, a, w, out2, m=M, n=N, k=K, act=_code(lib, name), bias=bias)
  torch.cuda.synchronize()
  assert torch.equal(out, out2)


@pytest.mark.parametrize('name', ACTS)
@pytest.mark.parametrize('opts', ['plain', 'mask_mod', 'rowv_addend_colsum', 'all'])
def test_gemm_dgrad_factor(mods, name, opts):
  """out = a'(z[r mod mask_mod]) * (dY W^T + rowv colv) + addend, colsum of out: factor first, then addend."""
  _, _, ops, lib = mods
  M, N, K = 300, 256, 128
  mod = opts in ('mask_mod', 'all')
  side = opts in ('rowv_addend_colsum', 'all')
  R = 3 * M if mod else M
  g = torch.Generator().manual_seed(7)
  dy, w = _bf(torch.randn(R, K, generator=g)).cuda(), _bf(torch.randn(N, K, generator=g) * 0.1).cuda()
  z = _bf(torch.randn(M, N, generator=g) * 2).cuda()
  rowv, colv = torch.randn(R, generator=g).cuda(), torch.randn(N, generator=g).cuda()
  addend = _bf(torch.randn(R, N, generator=g)).cuda()
  colsum = torch.zeros(N, device='cuda')
  out = torch.empty(R, N, device='cuda', dtype=torch.bfloat16)
  ops.gemm(lib.GEMM_DGRAD, dy, w, out, m=R, n=N, k=K, act=_code(lib, name), z=z, mask_mod=M if mod else 0,
           rowv=rowv if side else None, colv=colv if side else None, addend=addend if side else None,
           colsum=colsum if side else None)
  zr = z.float().repeat(3, 1) if mod else z.float()
  ref = dy.float() @ w.float().t()
  if side:
    ref = ref + rowv[:, None] * colv[None, :]
  ref = _d1(name, zr) * ref
  if side:
    ref = ref + addend.float()
  close(out.float(), ref, atol=3e-2, rtol=1e-2, msg='dgrad')
  if side:
    close(colsum, ref.sum(0), atol=0.5, rtol=1e-3, msg='colsum')


@pytest.mark.parametrize('name', ACTS)
def test_gemm_tensor_cores_match_simt_reference(mods, name):
  _, _, ops, lib = mods
  M, N, K = 8192 + 77, 256, 320
  g = torch.Generator().manual_seed(3)
  a, w = _bf(torch.randn(M, K, generator=g)).cuda(), _bf(torch.randn(N, K, generator=g) * 0.1).cuda()
  bias = torch.randn(N, generator=g).cuda()
  res = []
  for impl in (0, 1):
    out = torch.empty(M, N, device='cuda', dtype=torch.bfloat16)
    z = torch.empty(M, N, device='cuda', dtype=torch.bfloat16)
    ops.gemm(lib.GEMM_FWD, a, w, out, m=M, n=N, k=K, act=_code(lib, name), bias=bias, z=z, impl=impl)
    dx = torch.empty(M, K, device='cuda', dtype=torch.bfloat16)
    cs = torch.zeros(K, device='cuda')
    w_kn = w.t().contiguous()
    ops.gemm(lib.GEMM_DGRAD, out, w_kn, dx, m=M, n=K, k=N, act=_code(lib, name), z=a, colsum=cs, impl=impl)
    torch.cuda.synchronize()
    res.append((out.float(), z.float(), dx.float(), cs))
  for x0, x1, what in zip(res[0], res[1], ['out', 'z', 'dx', 'colsum']):
    close(x0, x1, atol=3e-2 if what != 'colsum' else 5.0, rtol=1e-2, msg=f'impl 0 vs 1: {what}')


@pytest.mark.parametrize('name', ACTS)
@pytest.mark.parametrize('K,n_out', [(256, 1), (128, 3), (256, 4), (320, 1)])
def test_head_bwd_factor(mods, name, K, n_out):
  _, _, ops, lib = mods
  M = 1000
  g = torch.Generator().manual_seed(K + n_out)
  x = _bf(torch.randn(M, K, generator=g)).cuda()
  z = _bf(torch.randn(M, K, generator=g) * 2).cuda()
  w = _bf(torch.randn(n_out, K, generator=g) * 0.1).cuda()
  draw = torch.randn(M, n_out, generator=g).cuda()
  dx = torch.empty(M, K, device='cuda', dtype=torch.bfloat16)
  dw, db, dxsum = torch.zeros(K, n_out, device='cuda'), torch.zeros(n_out, device='cuda'), torch.zeros(K, device='cuda')
  ops.head_bwd(x, w, draw, n_out, K, dx=dx, dw=dw, db=db, dxsum=dxsum, act=_code(lib, name), z=z)
  ref = _d1(name, z.float()) * (draw @ w.float())
  close(dx.float(), ref, atol=2e-2, rtol=1e-2, msg='dx')
  close(dxsum, ref.sum(0), atol=5e-2, rtol=1e-3, msg='dxsum')
  close(dw, x.float().t() @ draw, atol=1e-2, rtol=1e-4, msg='dw')
  close(db, draw.sum(0), atol=1e-3, rtol=1e-5, msg='db')


# ------------------------------------------------------------------ model

def with_act(bundle, nerf, prop=None):
  bundle.nerf_mlp.net_activation = nerf
  bundle.prop_mlp.net_activation = prop or nerf
  bundle.config.grad_max_norm = bundle.config.grad_max_val = 0.0
  return bundle


def wide_trunk(name):
  """blender_256.gin reduced: a 4 x 256 NerfMLP trunk, which the layer-chained kernel would run under ReLU."""
  from multinerf_b200 import configs
  b = configs.bundle_blender_256()
  m, p, n = b.model, b.prop_mlp, b.nerf_mlp
  m.num_prop_samples, m.num_nerf_samples = 32, 16
  p.net_depth, p.net_width = 2, 64
  n.net_depth, n.net_width, n.bottleneck_width, n.net_width_viewdirs = 4, 256, 64, 64
  return with_act(b, name)


def prop_normals(name):
  """Density normals on the colourless PropMLP and on the NerfMLP, with the orientation loss on every level (the
  reference needs normals on each level once the loss is on)."""
  b = wide_trunk(name)
  b.nerf_mlp.net_width = 128
  b.prop_mlp.disable_density_normals = b.nerf_mlp.disable_density_normals = False
  b.config.orientation_loss_mult, b.config.orientation_coarse_loss_mult = 0.1, 0.01
  b.config.orientation_loss_target = 'normals'
  return b


def view_skips(name):
  b = wide_trunk(name)
  b.nerf_mlp.net_width = 128
  b.nerf_mlp.net_depth_viewdirs, b.nerf_mlp.skip_layer_dir = 5, 2      # skips after view layers 2 and 4
  return b


CASES = {'mini360': lambda a: with_act(mini360(), a), 'wide_trunk': wide_trunk, 'prop_normals': prop_normals,
         'view_skips': view_skips}


@pytest.mark.parametrize('name', ACTS)
@pytest.mark.parametrize('case', list(CASES))
def test_train_step_vs_oracle(mods, case, name):
  models, train_utils, _, lib = mods
  bundle = CASES[case](name)
  model = models.Model(bundle)
  for plan in model.plans.values():
    assert plan.act == _code(lib, name)
    assert not model._use_chain(plan, 4096)
  check_train_step(models, train_utils, bundle, 96, 70, (0.2, 0.98))


def test_prop_and_nerf_activations_may_differ(mods):
  models, train_utils, _, lib = mods
  bundle = with_act(mini360(), 'silu', 'softplus')
  model = models.Model(bundle)
  assert (model.plans['NerfMLP_0'].act, model.plans['PropMLP_0'].act) == (lib.ACT_SILU, lib.ACT_SOFTPLUS)
  check_train_step(models, train_utils, bundle, 96, 71, (0.2, 0.98))


def _refnerf_step(models, bundle, seed, colour=True):
  B = 96
  rays, rng = synth_rays(seed, B, 2.0, 6.0, unit_cube=False)
  target = rng.uniform(0, 1, (B, 3)).astype(np.float32)
  model, variables = models.construct_model(seed + 1, rays, bundle)
  rand = level_jitter(rng, bundle, B)
  t = train_step(model, variables, bundle, rays, target, rand, 0.5)
  for k in ['orientation', 'predicted_normals']:
    lo = float(t.stats_o['losses'][k].detach())
    assert abs(t.stats['losses'][k] - lo) < 0.05 * abs(lo) + 1e-7, (k, t.stats['losses'][k], lo)
  report, zero = grad_report(model, t.grads_o, mlp_leaves(model, modules=['NerfMLP_0']))
  # without a data loss the colour branch gets no gradient
  assert not zero if colour else not any(zero.values()), zero
  print(f'worst leaves (rel, cos): {worst(report)}')
  return model, rays, rand, t, report


@pytest.mark.parametrize('name', ACTS)
def test_refnerf_vs_oracle(mods, name):
  """mini_refnerf: density and predicted normals, IDE, orientation and predicted-normal losses; forward (normals
  included) and one train step."""
  models, _, _, _ = mods
  bundle = with_act(mini_refnerf(), name)
  B, S = 96, 16
  rays, rng = synth_rays(72, B, 2.0, 6.0, unit_cube=False)
  model, _ = models.construct_model(73, rays, bundle)
  rand = level_jitter(rng, bundle, B)

  def normals(i, st, h):
    cosn = (st.normals.cpu().view(B, S, 3) * h['normals']).sum(-1)
    assert float((cosn > 0.98).float().mean()) > 0.97, float((cosn > 0.98).float().mean())
  pinned_forward(model, bundle, rays, rand, dens=(0.08, 4e-3), pixel=1.5e-2, samples=4e-2, level=normals)
  _, _, _, t, report = _refnerf_step(models, bundle, 74)
  close(t.stats['mses'], t.stats_o['mses'].detach(), atol=2e-3, rtol=3e-2, msg='mses')
  bad = beyond(report, 0.2, 0.98)
  assert not bad, (bad, report)


@pytest.mark.parametrize('name', ACTS)
def test_second_order_term_drives_trunk_gradient(mods, name):
  """No data loss, only the orientation and predicted-normal losses on the density normals: the trunk's gradient is
  then mostly the second-order term a''(z) sum_s T u.  Without it the trunk kernels' gradients are far off the
  oracle's."""
  models, _, _, _ = mods
  bundle = with_act(mini_refnerf(), name)
  c = bundle.config
  c.data_loss_mult = c.data_coarse_loss_mult = 0.0
  c.orientation_loss_target = 'normals'
  model, _, _, _, report = _refnerf_step(models, bundle, 75, colour=False)
  trunk = [k for k in report if k[1] in {sp.name for sp in model.plans['NerfMLP_0'].by_role('trunk')}]
  assert trunk
  # with the term the worst trunk leaf is at (0.13, 0.991) (SiLU), without it every trunk leaf is beyond
  # (0.29, 0.96)
  bad = beyond({k: report[k] for k in trunk}, 0.2, 0.98)
  assert not bad, (bad, worst(report))


def test_render_image_matches_forward(mods):
  """render_image (chunks in CUDA graphs, no pre-activations stored) against the eager forward, and the forward
  against the oracle."""
  models, train_utils, _, _ = mods
  from model_parity import image_rays
  bundle = with_act(mini360(), 'silu')
  bundle.config.render_chunk_size = 256
  bundle.config.vis_num_rays = 8
  H, W = 19, 23
  rays = image_rays(H, W)
  model, state, render_eval_pfn, _, _ = train_utils.setup_model(bundle, 3)
  out = models.render_image(lambda rng, r: render_eval_pfn(state.params, 1.0, None, r), rays, None, bundle,
                            verbose=False)
  rend, _ = model(None, rays.map(lambda a: a.reshape(H * W, -1)), 1.0, False)
  torch.cuda.synchronize()
  close(out['rgb'].reshape(-1, 3), rend[-1]['rgb'], atol=2e-3, rtol=0, msg='render_image vs forward')
  rays_b, rand, _ = synth_case(bundle, 96, 76, 0.2, 1e6)
  pinned_forward(model, bundle, rays_b, rand, dens=(0.08, 4e-3), pixel=1.5e-2, samples=1.5e-2)


def test_cuda_graph_matches_eager(mods):
  models, train_utils, _, _ = mods
  bundle = with_act(mini_refnerf(), 'softplus')
  B = 96
  rng = np.random.default_rng(77)
  batches = []
  for _ in range(4):
    rays, _ = synth_rays(int(rng.integers(1 << 30)), B, 2.0, 6.0, unit_cube=False)
    batches.append((rays, rng.uniform(0, 1, (B, 3)).astype(np.float32), level_jitter(rng, bundle, B)))
  graph_matches_eager(models, train_utils, bundle, batches, 78)
