"""The render path through the real kernels (models.py:625-706 render_image over
train_utils.py:377-396 render_eval_pfn): a chunked image render must equal one direct
Model.__call__ on the same rays, keep the reference's output keys/shapes, and agree with the oracle.
Needs an H100.  The N-GPU all-gather variant is tools/render_check.py (needs torchrun)."""
import pytest
import torch

from model_parity import bases, image_rays, mini360, oracle_rays, torch_tree
from oracle import o_models
from util import close

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('which', ['mini360', 'full360'])
def test_render_image_equals_direct_call(which):
  from multinerf_b200 import configs, lib, models, train_utils
  lib.require_device()
  bundle = mini360() if which == 'mini360' else configs.bundle_360()
  H, W = (37, 53) if which == 'mini360' else (48, 64)          # 1961 rays: ragged last chunk | 3072 rays
  bundle.config.render_chunk_size = 512 if which == 'mini360' else 1024
  bundle.config.vis_num_rays = 8
  rays = image_rays(H, W)
  model, state, render_eval_pfn, _, _ = train_utils.setup_model(bundle, 3)
  render_fn = lambda rng, r: render_eval_pfn(state.params, 1.0, None, r)
  out = models.render_image(render_fn, rays, None, bundle, verbose=False)
  torch.cuda.synchronize()
  flat = rays.map(lambda a: a.reshape(H * W, -1))
  rend, hist = model(None, flat, 1.0, True)
  torch.cuda.synchronize()
  assert out['rgb'].shape == (H, W, 3) and out['acc'].shape == (H, W)
  for k in ('rgb', 'acc', 'distance_mean', 'distance_median', 'distance_percentile_5', 'distance_percentile_95'):
    # rays are independent: chunking must not change a single bit
    assert torch.equal(out[k].reshape(rend[-1][k].shape), rend[-1][k]), k
  # the CUDA-graph render function (one captured graph per chunk shape, ragged last chunk eager)
  gfn = train_utils.create_render_fn(model, use_graph=True)
  out_g = models.render_image(lambda rng, r: gfn(state.params, 1.0, None, r), rays, None, bundle, verbose=False)
  torch.cuda.synchronize()
  for k in ('rgb', 'acc', 'distance_mean', 'distance_median'):
    assert torch.equal(out_g[k], out[k]), ('graph replay', k)
  for a, b in zip(out_g['ray_sdist'], out['ray_sdist']):
    assert torch.equal(a, b)
  # ray_* bundles: one entry per level, vis_num_rays rays each (models.py:696-705)
  for k in ('ray_sdist', 'ray_weights', 'ray_rgbs'):
    assert len(out[k]) == bundle.model.num_levels and out[k][-1].shape[0] == 8, (k, out[k][-1].shape)
  assert torch.isfinite(out['rgb']).all() and float(out['rgb'].min()) >= 0.0


def test_render_image_vs_oracle():
  """A small image through render_image vs the oracle's deterministic Model.__call__ (rng=None)."""
  from multinerf_b200 import lib, models, train_utils
  lib.require_device()
  bundle = mini360()
  H, W = 12, 20
  bundle.config.render_chunk_size = 100
  rays = image_rays(H, W, focal=30.0)
  model, state, render_eval_pfn, _, _ = train_utils.setup_model(bundle, 5)
  out = models.render_image(lambda rng, r: render_eval_pfn(state.params, 1.0, None, r), rays, None, bundle,
                            verbose=False)
  flat = rays.map(lambda a: a.reshape(H * W, -1))
  with torch.no_grad():
    rend_o, _ = o_models.model_apply(torch_tree(model.export_flax()), bundle, bases(model), oracle_rays(flat), 1.0,
                                     True, rand=None, bf16=True)
  close(out['rgb'].reshape(H * W, 3), rend_o[-1]['rgb'], atol=2e-2, rtol=0, msg='rendered image vs oracle')
  close(out['acc'].reshape(H * W), rend_o[-1]['acc'], atol=2e-2, rtol=0, msg='acc vs oracle')
