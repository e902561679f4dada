"""Side sums of the tensor-core weight-gradient GEMM (mnrf_gemm_wgrad): the bias gradient bsum[N] += sum_r dY[r, :]
and the Dense(1) head gradient side_aw[Mo] += sum_r side_w[r] X[r, :], both taken from the operand tiles the GEMM
stages, against fp64 sums of the same bf16 operands.  Needs an H100."""
import math

import numpy as np
import pytest
import torch

from util import close

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ops():
  from multinerf_b200 import lib, ops as _ops
  lib.require_device()
  return _ops


def _colsum64(t, w=None, chunk=1 << 16):
  """fp64 column sums of a [R, C] bf16 tensor (weighted by w[R] if given), chunked to bound the fp64 copy."""
  out = torch.zeros(t.shape[1], dtype=torch.float64, device=t.device)
  for r0 in range(0, t.shape[0], chunk):
    blk = t[r0:r0 + chunk].double()
    out += blk.sum(0) if w is None else w[r0:r0 + chunk].double() @ blk
  return out


def _operands(R, Mo, N, seed):
  g = torch.Generator(device='cuda')
  g.manual_seed(seed)
  x = torch.randn(R, Mo, device='cuda', generator=g).bfloat16()
  dy = (torch.randn(R, N, device='cuda', generator=g) * 0.1).bfloat16()
  w = torch.randn(R, device='cuda', generator=g)
  return x, dy, w


# the NerfMLP trunk ([1024, 1024], 4 R-splits per output tile; R ragged), the bottleneck ([1024, 256] with the density
# head's dW), the PropMLP trunk ([256, 256] and [512, 256] at 2 x 524288 rows, many splits), narrow and ragged tiles
@pytest.mark.parametrize('R,Mo,N', [(524251, 1024, 1024), (524288, 1024, 256), (1048576, 256, 256),
                                    (1048576, 512, 256), (65536, 320, 128), (4099, 1280, 64)])
def test_fused_sums_vs_fp64(ops, R, Mo, N):
  x, dy, w = _operands(R, Mo, N, R + Mo + N)
  out = torch.zeros(Mo, N, device='cuda')
  bsum = torch.full((N,), 0.5, device='cuda')
  aw = torch.full((Mo,), -0.25, device='cuda')
  ops.gemm_wgrad(x, dy, out, m=Mo, n=N, k=R, bsum=bsum, side_w=w, side_aw=aw)
  torch.cuda.synchronize()
  tol = 2e-3 * math.sqrt(R)
  close(bsum, _colsum64(dy) + 0.5, atol=1e-4 * math.sqrt(R), rtol=1e-5, msg='bsum')
  close(aw, _colsum64(x, w) - 0.25, atol=tol, rtol=1e-5, msg='side_aw')
  ref = torch.zeros(Mo, N, dtype=torch.float64, device='cuda')
  for r0 in range(0, R, 1 << 16):
    ref += x[r0:r0 + (1 << 16)].double().T @ dy[r0:r0 + (1 << 16)].double()
  close(out, ref, atol=tol * 0.1, rtol=1e-4, msg='weight gradient')


@pytest.mark.parametrize('R,Mo,N', [(524251, 1024, 1024), (1048576, 256, 256), (37, 64, 64)])
def test_each_side_sum_alone(ops, R, Mo, N):
  x, dy, w = _operands(R, Mo, N, 7 * R + N)
  bsum = torch.zeros(N, device='cuda')
  o1 = torch.zeros(Mo, N, device='cuda')
  ops.gemm_wgrad(x, dy, o1, m=Mo, n=N, k=R, bsum=bsum)
  aw = torch.zeros(Mo, device='cuda')
  o2 = torch.zeros(Mo, N, device='cuda')
  ops.gemm_wgrad(x, dy, o2, m=Mo, n=N, k=R, side_w=w, side_aw=aw)
  torch.cuda.synchronize()
  close(bsum, _colsum64(dy), atol=1e-4 * math.sqrt(R), rtol=1e-5, msg='bsum only')
  close(aw, _colsum64(x, w), atol=2e-3 * math.sqrt(R), rtol=1e-5, msg='side_w only')
  close(o1, o2, atol=2e-3 * math.sqrt(R), rtol=1e-4, msg='weight gradient, bsum-only vs side_w-only launch')


def test_weight_gradient_unchanged_by_side_sums(ops):
  """With one R-split per output tile (11 x 12 = 132 tiles of 128 x 256) every output element takes exactly one
  fp32 reduction, so the weight gradient must be bit-identical with and without side sums."""
  from multinerf_b200 import lib as L
  R, Mo, N = 6000, 1408, 3072
  x, dy, w = _operands(R, Mo, N, 11)
  plain = torch.full((Mo, N), 0.125, device='cuda')
  ops.gemm(L.GEMM_WGRAD, x, dy, plain, m=Mo, n=N, k=R)
  fused = torch.full((Mo, N), 0.125, device='cuda')
  bsum, aw = torch.zeros(N, device='cuda'), torch.zeros(Mo, device='cuda')
  ops.gemm_wgrad(x, dy, fused, m=Mo, n=N, k=R, bsum=bsum, side_w=w, side_aw=aw)
  torch.cuda.synchronize()
  assert torch.equal(plain, fused)
  close(bsum, _colsum64(dy), atol=1e-4 * math.sqrt(R), rtol=1e-5, msg='bsum')
  close(aw, _colsum64(x, w), atol=2e-3 * math.sqrt(R), rtol=1e-5, msg='side_aw')


def test_model_bias_gradients_are_column_sums_of_stored_dy(ops, monkeypatch):
  """One backward of every level of the full-width 360.gin model: the bias gradient of each trunk layer and of the
  bottleneck is the fp64 column sum of the bf16 dY its weight-gradient GEMM reads."""
  from multinerf_b200 import configs, models
  from model_parity import synth_rays
  bundle = configs.bundle_360()
  B = 256
  rays, _ = synth_rays(3, B, 0.2, 1e6)
  model, _ = models.construct_model(0, rays, bundle)
  r = model._prep_rays(rays)
  states = model.forward_levels(None, r, 0.5, False, False, loss_config=bundle.config)
  real = ops.gemm_wgrad
  for st in states:
    mlp = model.mlps[st.mname]
    model._mlp_forward(st, mlp, r)
    st.d_raw_density.normal_()
    if st.d_raw_rgb is not None:
      st.d_raw_rgb.normal_()
    seen = {}

    def recording(x, dy, out, *, m, n, k, bsum=None, **kw):
      if bsum is not None:
        ref = _colsum64(dy[:k, :n])
        key = bsum.data_ptr()
        seen[key] = (bsum, seen[key][1] + ref if key in seen else ref)
      return real(x, dy, out, m=m, n=n, k=k, bsum=bsum, **kw)

    monkeypatch.setattr(ops, 'gemm_wgrad', recording)
    mlp.grads.zero_()
    model._mlp_backward(st, mlp, r)
    torch.cuda.synchronize()
    monkeypatch.setattr(ops, 'gemm_wgrad', real)
    trunk = mlp.plan.by_role('trunk')
    want = {mlp.b(sp, mlp.grads).data_ptr() for sp in trunk + mlp.plan.by_role('bottleneck')}
    assert want <= set(seen), (st.mname, len(want), len(seen))
    for bsum, ref in seen.values():
      close(bsum, ref, atol=1e-4 * math.sqrt(st.M), rtol=1e-5, msg=f'{st.mname} bias gradient')
