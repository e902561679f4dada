"""View-independent colour (Model.use_viewdirs = False) on the GPU: the rgb head on the trunk output, stacked with
the density head as one 4-output head (csrc/chain.cu epilogue head for chained 256-wide trunks, mnrf_head_fwd /
mnrf_head_bwd with n_out = 4 for per-layer trunks), against the CPU oracle.  Needs an H100.

Reference: internal/models.py:512 (no view branch without view directions), :584 (rgb = act(Dense(3)(x))).
"""
import numpy as np
import pytest
import torch

from model_parity import (bases, check_train_step, graph_matches_eager, oracle_rays, pinned_forward, synth_case,
                          synth_rays, torch_tree)
from oracle import o_models
from util import close

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def mods():
  from multinerf_b200 import lib, models, train_utils
  lib.require_device()
  return models, train_utils


def mini_view_independent(normals=True, glo=True):
  """A reduced blender_256.gin under Model.use_viewdirs = False (widths multiples of 64); normals: density and
  predicted normals on both MLPs with both normal losses; glo: GLO vectors (kept, unused by any layer)."""
  from multinerf_b200 import configs
  b = configs.bundle_blender_256()
  c, m, p, n = b.config, b.model, b.prop_mlp, b.nerf_mlp
  m.use_viewdirs = False
  m.num_prop_samples, m.num_nerf_samples = 32, 16
  p.net_depth, p.net_width = 2, 64
  n.net_depth, n.net_width = 5, 128          # skip after layer 4: the heads read [hidden | features]
  if glo:
    m.num_glo_features, m.num_glo_embeddings = 4, 3
  if normals:
    for mlp in (p, n):
      mlp.disable_density_normals, mlp.enable_pred_normals = False, True
    c.orientation_loss_mult, c.orientation_coarse_loss_mult, c.orientation_loss_target = 0.1, 0.01, 'normals_pred'
    c.predicted_normal_loss_mult, c.predicted_normal_coarse_loss_mult = 3e-4, 3e-5
  c.grad_max_norm = c.grad_max_val = 0.0
  return b


def fullwidth_view_independent(name):
  from multinerf_b200 import configs
  b = configs.bundle_blender_256() if name == 'blender_256' else configs.bundle_360()
  b.model.use_viewdirs = False
  b.config.grad_max_norm = b.config.grad_max_val = 0.0
  return b


def _forward_vs_oracle(models, bundle, B, seed, dens_lim, pix_atol):
  if bundle.model.raydist_fn is None or bundle.config.far < 100:
    rays, rand, _ = synth_case(bundle, B, seed, 2.0, 6.0, unit_cube=False)
  else:
    rays, rand, _ = synth_case(bundle, B, seed, 0.2, 1e6)
  model, _ = models.construct_model(seed + 1, rays, bundle)
  assert model.plans['NerfMLP_0'].rgb_on_trunk
  # sample positions pinned to the oracle's: each level's MLP and heads in isolation
  rend_o, _ = pinned_forward(model, bundle, rays, rand, dens=dens_lim, pixel=pix_atol, samples=pix_atol)
  rend, hist = model(rand, rays, 0.5, True)
  torch.cuda.synchronize()
  assert all('roughness' not in r_ for r_ in rend)
  close(rend[-1]['rgb'], rend_o[-1]['rgb'], atol=3e-2, rtol=0, msg='final pixel end-to-end')
  return model


def test_construction_and_flax_tree(mods):
  models, _ = mods
  for bundle in (mini_view_independent(), mini_view_independent(False, False),
                 fullwidth_view_independent('blender_256'), fullwidth_view_independent('360')):
    model = models.Model(bundle)
    model.init(0)
    tree = model.export_flax()
    nerf = tree['NerfMLP_0']
    last = sorted(nerf, key=lambda s: int(s.split('_')[1]))[-1]
    assert nerf[last]['kernel'].shape == (model.plans['NerfMLP_0'].x_dim, 3)
    assert ('Embed_0' in tree) == (bundle.model.num_glo_features > 0)
    assert model.num_params() == sum(v['kernel'].size + v['bias'].size for k, t in tree.items() if k != 'Embed_0'
                                     for v in t.values())
    # the tree round-trips through init(flax_params=...) (stacked head weights and the shared bias block)
    m2 = models.Model(bundle)
    m2.init(flax_params=tree)
    t2 = m2.export_flax()
    for mname in model.plans:
      for k, v in tree[mname].items():
        assert np.array_equal(v['kernel'], t2[mname][k]['kernel']) and np.array_equal(v['bias'], t2[mname][k]['bias'])
    rays, _ = synth_rays(0, 4, 2.0, 6.0, unit_cube=False)
    o_models.model_apply(torch_tree(tree), bundle, bases(model), oracle_rays(rays), 0.5, False)


@pytest.mark.parametrize('normals', [False, True])
def test_forward_vs_oracle(mods, normals):
  models, _ = mods
  _forward_vs_oracle(models, mini_view_independent(normals), 96, 10, (0.08, 4e-3), 1.5e-2)


@pytest.mark.parametrize('normals', [False, True])
def test_train_step_vs_oracle(mods, normals):
  models, train_utils = mods
  bundle = mini_view_independent(normals)
  check_train_step(models, train_utils, bundle, 96, 20, (0.2, 0.98))
  # GLO vectors feed no layer without view directions: their gradient is zero, as in the reference
  model, variables = models.construct_model(3, synth_rays(0, 8, 2.0, 6.0, unit_cube=False)[0], bundle)
  from multinerf_b200 import utils
  rays, rng = synth_rays(21, 64, 2.0, 6.0, unit_cube=False)
  rays.cam_idx[:] = 1
  step = train_utils.create_train_step(model, bundle.config, use_graph=False)
  state = train_utils.TrainState(variables)
  step(None, state, utils.Batch(rays=rays, rgb=rng.uniform(0, 1, (64, 3)).astype(np.float32)), None, 0.5)
  torch.cuda.synchronize()
  assert float(variables.seg('Embed_0', variables.grads).abs().max()) == 0.0


@pytest.mark.parametrize('name', ['blender_256', '360'])
def test_fullwidth_forward_vs_oracle(mods, name):
  models, _ = mods
  bundle = fullwidth_view_independent(name)
  model = _forward_vs_oracle(models, bundle, 64, 30, (0.1, 5e-3), 1.5e-2)
  M = 64 * bundle.model.num_nerf_samples
  assert model._use_chain(model.plans['NerfMLP_0'], M) == (name == 'blender_256')


@pytest.mark.parametrize('name', ['blender_256', '360'])
def test_fullwidth_train_step_vs_oracle(mods, name):
  # blender_256: chained 256-wide trunk, the stacked head in its epilogue; 360: per-layer 1024-wide trunk, the
  # stacked mnrf_head_fwd / mnrf_head_bwd at K = 1024.  Bounds of the shipped full-width train-step tests.
  models, train_utils = mods
  lim = (0.3, 0.95) if name == 'blender_256' else (0.2, 0.98)
  check_train_step(models, train_utils, fullwidth_view_independent(name), 128, 40, lim)


def test_colourless_trunk_ending_on_skip_train_step_vs_oracle(mods):
  """A PropMLP whose last trunk layer is a skip layer (its density head reads [hidden | features]) and that has no
  predicted normals: the head's input gradient covers the hidden columns only."""
  models, train_utils = mods
  bundle = mini_view_independent(normals=False, glo=False)
  bundle.prop_mlp.net_depth = 5
  assert models.MLPPlan(bundle.prop_mlp).last_has_feat
  check_train_step(models, train_utils, bundle, 96, 25, (0.2, 0.98))


def test_chained_trunk_matches_per_layer(mods, monkeypatch):
  """blender_256 under use_viewdirs = False: the 4-output head in the chain's epilogue vs the per-layer GEMMs and
  one mnrf_head_fwd launch (MNRF_CHAIN=0), forward renderings and one step's gradients."""
  models, train_utils = mods
  from multinerf_b200 import utils
  bundle = fullwidth_view_independent('blender_256')
  B = 256
  rays, rng = synth_rays(5, B, 2.0, 6.0, unit_cube=False)
  target = rng.uniform(0, 1, (B, 3)).astype(np.float32)
  out = []
  for chain in ('1', '0'):
    monkeypatch.setenv('MNRF_CHAIN', chain)
    model, variables = models.construct_model(9, rays, bundle)
    rend, _ = model(None, rays, 0.5, False)
    step = train_utils.create_train_step(model, bundle.config, use_graph=False)
    state = train_utils.TrainState(variables)
    variables.grads.zero_()
    _, stats, _ = step(None, state, utils.Batch(rays=rays, rgb=target), None, 0.5)
    torch.cuda.synchronize()
    stats.materialize()
    out.append((rend[-1]['rgb'].clone(), stats['loss'], model.export_grads_flax()))
  (r1, l1, g1), (r0, l0, g0) = out
  close(r1, r0, atol=2e-3, rtol=0, msg='pixels chained vs per-layer')
  assert abs(l1 - l0) < 1e-3 * max(1.0, abs(l0)), (l1, l0)
  for name in ('Dense_8', 'Dense_9'):        # density and rgb heads of the 8-layer NerfMLP
    for leaf in ('kernel', 'bias'):
      a, b = torch.tensor(g1['NerfMLP_0'][name][leaf]), torch.tensor(g0['NerfMLP_0'][name][leaf])
      assert float((a - b).norm() / b.norm()) < 2e-2, (name, leaf)


def test_cuda_graph_matches_eager(mods):
  models, train_utils = mods
  B, steps = 192, 5
  rng = np.random.default_rng(33)
  batches = []
  for _ in range(steps):
    rays, _ = synth_rays(int(rng.integers(1 << 30)), B, 2.0, 6.0, unit_cube=False)
    rand = {'jitter': [torch.tensor(rng.uniform(0, 1, (B,)).astype(np.float32)) for _ in range(2)]}
    batches.append((rays, rng.uniform(0, 1, (B, 3)).astype(np.float32), rand))
  graph_matches_eager(models, train_utils, mini_view_independent(), batches, 6)


@pytest.mark.parametrize('M', [512, 1000, 16384])
def test_chain_four_output_head_vs_head_fwd(mods, M):
  """The chain's epilogue head with head_n = 4 against mnrf_head_fwd (n_out = 4) on the chain's own output."""
  from multinerf_b200 import lib as L, ops
  W, Fpad = 256, 128
  g = torch.Generator(device='cuda')
  g.manual_seed(M)
  feat = (torch.rand(M, Fpad, device='cuda', generator=g) * 2 - 1).to(torch.bfloat16)
  ws = [((torch.rand(W, k, device='cuda', generator=g) * 2 - 1) * (6 / k) ** 0.5).to(torch.bfloat16)
        for k in (Fpad, W, W)]
  bs = [torch.rand(W, device='cuda', generator=g) * 0.1 for _ in range(3)]
  hw = ((torch.rand(4, W, device='cuda', generator=g) * 2 - 1) * 0.1).to(torch.bfloat16)
  hb = torch.rand(4, device='cuda', generator=g)
  acts = [torch.empty(M, W, device='cuda', dtype=torch.bfloat16) for _ in range(3)]
  layers = [dict(w=ws[0], bias=bs[0], out=acts[0], n_stream=Fpad // 64, stream_col0=0, stream_kb0=0)]
  layers += [dict(w=ws[i], bias=bs[i], out=acts[i], n_res=4, res_kb0=0) for i in (1, 2)]
  head = torch.full((M, 4), -3.0, device='cuda')
  ops.mlp_chain(ops.chain_desc(L.CHAIN_FWD, M, layers, stream=feat, stream_cols=Fpad, head_w=hw.float().contiguous(),
                               head_b=hb, head_out=head, head_n=4))
  ref = ops.head_fwd(acts[-1], hw, hb, 4, W)
  # density-only instance on the same operands: its output is column 0 of the stacked head
  head1 = torch.zeros(M, device='cuda')
  ops.mlp_chain(ops.chain_desc(L.CHAIN_FWD, M, layers, stream=feat, stream_cols=Fpad,
                               head_w=hw[0].float().contiguous(), head_b=hb[:1], head_out=head1))
  torch.cuda.synchronize()
  close(head, ref, atol=2e-3, rtol=2e-3, msg='stacked head vs head_fwd')
  assert torch.equal(head[:, 0], head1)


def test_stacked_head_backward_vs_separate_heads(mods):
  """mnrf_head_bwd with n_out = 4 and a split weight gradient against the two heads' own backward launches."""
  from multinerf_b200 import ops
  g = torch.Generator(device='cuda')
  g.manual_seed(3)
  for M, K in ((5000, 256), (3000, 1024), (2000, 384)):
    x = torch.relu(torch.randn(M, K, device='cuda', generator=g)).to(torch.bfloat16)
    w = (torch.randn(4, K, device='cuda', generator=g) * 0.05).to(torch.bfloat16)
    draw = torch.randn(M, 4, device='cuda', generator=g)
    dx, dw1, dw3, db, dxs = (torch.zeros(M, K, device='cuda', dtype=torch.bfloat16), torch.zeros(K, 1, device='cuda'),
                             torch.zeros(K, 3, device='cuda'), torch.zeros(4, device='cuda'), torch.zeros(K, device='cuda'))
    dxc = 256 if K == 384 else K        # a head on [hidden | features]: input gradient of the hidden part only
    ops.head_bwd(x, w, draw, 4, K, dx=dx, relu_mask=True, dw=dw1, dw2=dw3, dw_split=1, db=db, dxsum=dxs,
                 dx_cols=dxc if dxc < K else 0)
    e1, e3, eb1, eb3 = (torch.zeros(K, 1, device='cuda'), torch.zeros(K, 3, device='cuda'), torch.zeros(1, device='cuda'),
                        torch.zeros(3, device='cuda'))
    ops.head_bwd(x, w[:1].contiguous(), draw[:, :1].contiguous(), 1, K, dw=e1, db=eb1)
    ops.head_bwd(x, w[1:].contiguous(), draw[:, 1:].contiguous(), 3, K, dw=e3, db=eb3)
    torch.cuda.synchronize()
    close(dw1, e1, atol=1e-2, rtol=1e-3, msg=f'density dW K={K}')
    close(dw3, e3, atol=1e-2, rtol=1e-3, msg=f'rgb dW K={K}')
    close(db, torch.cat([eb1, eb3]), atol=1e-2, rtol=1e-4, msg='db')
    ref_dx = (draw @ w.float()) * (x.float() > 0)
    ref_dx[:, dxc:] = 0
    close(dx.float(), ref_dx, atol=1e-2, rtol=1e-2, msg='dx')
    close(dxs, dx.float().sum(0), atol=0.5, rtol=1e-2, msg='dxsum')
    assert not dxs[dxc:].any()


@pytest.mark.parametrize('name', ['blender_256', '360'])
def test_launch_count(mods, name):
  """The rgb head of a view-independent model costs no launch: its NerfMLP level runs exactly the launches of the same
  MLP without colour (one head launch forward, one backward), and fewer than the shipped model's."""
  models, train_utils = mods
  from multinerf_b200 import configs, ops, utils
  B = 256
  rays, rng = synth_rays(7, B, 2.0, 6.0, unit_cube=False) if name == 'blender_256' else synth_rays(7, B, 0.2, 1e6)
  target = rng.uniform(0, 1, (B, 3)).astype(np.float32)
  counts = {}
  for variant in ('shipped', 'view_independent', 'colourless'):
    bundle = fullwidth_view_independent(name)
    bundle.model.use_viewdirs = variant == 'shipped'
    bundle.nerf_mlp.disable_rgb = variant == 'colourless'
    model, variables = models.construct_model(0, rays, bundle)
    r = model._prep_rays(rays)
    states = model.forward_levels(None, r, 0.5, False, False, loss_config=bundle.config)
    st = states[-1]
    mlp = model.mlps[st.mname]
    n0 = ops.LAUNCHES
    model._mlp_forward(st, mlp, r)
    n1 = ops.LAUNCHES
    st.d_raw_density.normal_()
    if st.d_raw_rgb is not None:
      st.d_raw_rgb.normal_()
    model._mlp_backward(st, mlp, r)
    counts[variant] = (n1 - n0, ops.LAUNCHES - n1)
    torch.cuda.synchronize()
    step = train_utils.create_train_step(model, bundle.config, use_graph=False)
    n2 = ops.LAUNCHES
    step(None, train_utils.TrainState(variables), utils.Batch(rays=rays, rgb=target), None, 0.5)
    counts[variant] += (ops.LAUNCHES - n2,)
  print(name, counts)
  assert counts['view_independent'][:2] == counts['colourless'][:2], counts
  chained = name == 'blender_256'
  depth = 8
  # forward: encode + (one chain launch | 8 GEMMs + the stacked head)
  assert counts['view_independent'][0] == (2 if chained else 2 + depth), counts
  assert counts['view_independent'][2] < counts['shipped'][2], counts
