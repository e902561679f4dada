"""Parity of each CUDA entry point (through the C ABI) against the CPU oracle.  Needs an H100.

Tolerances: integer indices bit-exact given the same CDF; fp32 stages atol=rtol=1e-5 unless a
comment says why not; bf16 tensor-core GEMMs are compared against the same product evaluated
in fp32 from the bf16-rounded operands (error = accumulation order + one output rounding).
"""
import math

import numpy as np
import pytest
import torch

from composite_ref import CFG, oracle_composite
from oracle import o_coord, o_math, o_render
from util import close, kernel_rays

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ops():
  from multinerf_b200 import lib, ops as _ops
  lib.require_device()
  return _ops


@pytest.mark.parametrize('S,opaque,raydist,near,far,act', [
    (32, True, 'reciprocal', 0.2, 1e6, 'sigmoid'), (64, True, 'reciprocal', 0.2, 1e6, 'sigmoid'),
    (128, False, None, 2.0, 6.0, 'sigmoid'), (48, False, None, 0.0, 1.0, 'safe_exp')])
def test_composite_fwd_vs_oracle(ops, S, opaque, raydist, near, far, act):
  rng = np.random.default_rng(S)
  B = 130
  cfg = dict(CFG, raydist_fn=raydist, opaque_background=opaque, rgb_activation=act,
             rgb_bias=-5.0 if act == 'safe_exp' else 0.0, rgb_padding=0.0 if act == 'safe_exp' else 0.001)
  _, d, _ = kernel_rays(rng, B)
  sdist = torch.tensor(np.sort(rng.uniform(0, 1, (B, S + 1)).astype(np.float32), -1))
  sdist[:, 0], sdist[:, -1] = 0, 1
  raw_d = torch.tensor(rng.normal(size=(B, S)).astype(np.float32) * 3)
  raw_d[0] = -50
  raw_d[1] = 30
  raw_rgb = torch.tensor(rng.normal(size=(B, S, 3)).astype(np.float32))
  nearv, farv = torch.full((B, 1), near), torch.full((B, 1), far)
  w_o, r_o, dens_o, rgb_o = oracle_composite(raw_d, raw_rgb, sdist, d, nearv, farv, cfg, extras=True)
  out = ops.composite_fwd(raw_d.cuda(), raw_rgb.cuda(), sdist.cuda(), d.cuda(), nearv[:, 0].contiguous().cuda(),
                          farv[:, 0].contiguous().cuda(), cfg=cfg, want_samples=True, want_extras=True)
  close(out['density'], dens_o, msg='density')
  close(out['rgb_samples'], rgb_o, msg='rgb samples')
  close(out['weights'], w_o, atol=1e-6, rtol=1e-5, msg='weights')
  close(out['rgb'], r_o['rgb'], msg='pixel')
  close(out['acc'], r_o['acc'], msg='acc')
  dist = out['dist'].cpu()
  close(dist[:, 0], r_o['distance_mean'], rtol=2e-5, atol=1e-5, msg='distance_mean')
  # percentiles are piecewise-linear in the CDF; a knot within rounding of p moves the answer by a
  # whole interval, so compare through the CDF (|cdf(t_gpu) - p| small) on top of the bulk check
  for i, k in enumerate(['distance_percentile_5', 'distance_median', 'distance_percentile_95']):
    ref = r_o[k]
    rel = ((dist[:, 1 + i] - ref).abs() / ref.abs().clamp(min=1e-6))
    assert (rel < 1e-3).float().mean() > 0.97, (k, rel.max())
  # PropMLP levels: rgb = 0
  w_o2, r_o2, _, _ = oracle_composite(raw_d, None, sdist, d, nearv, farv, cfg)
  out2 = ops.composite_fwd(raw_d.cuda(), None, sdist.cuda(), d.cuda(), nearv[:, 0].contiguous().cuda(),
                           farv[:, 0].contiguous().cuda(), cfg=cfg)
  close(out2['rgb'], r_o2['rgb'], msg='prop pixel')


@pytest.mark.parametrize('level,loss_type,S', [('fine', 'charb', 32), ('prop', 'mse', 64),
                                              ('fine', 'mse', 128), ('fine', 'rawnerf', 32)])
def test_composite_bwd_vs_oracle_autograd(ops, level, loss_type, S):
  from oracle import o_train
  rng = np.random.default_rng(11)
  B, Sf = 70, 32
  cfg = dict(CFG)
  _, d, _ = kernel_rays(rng, B)

  def mk_sdist(n):
    s = torch.tensor(np.sort(rng.uniform(0, 1, (B, n + 1)).astype(np.float32), -1))
    s[:, 0], s[:, -1] = 0, 1
    return s
  sdist = mk_sdist(S)
  raw_d = torch.tensor(rng.normal(size=(B, S)).astype(np.float32) * 2, requires_grad=True)
  raw_rgb = None if level == 'prop' else torch.tensor(rng.normal(size=(B, S, 3)).astype(np.float32),
                                                     requires_grad=True)
  nearv, farv = torch.full((B, 1), 0.2), torch.full((B, 1), 1e6)
  target = torch.tensor(rng.uniform(0, 1, (B, 3)).astype(np.float32))
  lossmult = torch.tensor(rng.integers(0, 2, (B, 3)).astype(np.float32)) if loss_type == 'rawnerf' \
      else torch.ones(B, 1)
  sdist_f = mk_sdist(Sf)
  w_f = torch.tensor(rng.uniform(0, 1, (B, Sf)).astype(np.float32))
  w_f = w_f / w_f.sum(-1, keepdim=True) * 0.9

  class Cfg:
    data_loss_type = loss_type
    charb_padding = 0.001
    disable_multiscale_loss = False
    data_coarse_loss_mult = 0.1
    data_loss_mult = 1.0
    interlevel_loss_mult = 1.0
    distortion_loss_mult = 0.01
  w_o, r_o, _, _ = oracle_composite(raw_d, raw_rgb, sdist, d, nearv, farv, cfg)
  lm = lossmult.expand(B, 3)
  data, st = o_train.compute_data_loss(target, [r_o], lm, Cfg)   # single level -> data_loss_mult
  data_mult = 1.0
  if level == 'prop':
    data = data * 0.1
    data_mult = 0.1
    hist = [dict(sdist=sdist, weights=w_o), dict(sdist=sdist_f, weights=w_f)]
    extra = o_train.interlevel_loss(hist, Cfg)
    dist_mult, inter_mult = 0.0, 1.0
  else:
    extra = o_train.distortion_loss([dict(sdist=sdist, weights=w_o)], Cfg)
    dist_mult, inter_mult = 0.01, 0.0
  loss = data + extra
  grads = torch.autograd.grad(loss, [raw_d] + ([raw_rgb] if raw_rgb is not None else []))
  stats = torch.zeros(8, device='cuda')
  inv_denom = (1.0 / lm.sum()).reshape(1).cuda()
  g_d, g_rgb = ops.composite_bwd(
      raw_d.detach().cuda(), None if raw_rgb is None else raw_rgb.detach().cuda(), sdist.cuda(), d.cuda(),
      nearv[:, 0].contiguous().cuda(), farv[:, 0].contiguous().cuda(), target.cuda(), lossmult.contiguous().cuda(),
      inv_denom, stats, cfg=cfg, loss_type=loss_type, charb_padding=0.001, data_mult=data_mult,
      distortion_mult=dist_mult, interlevel_mult=inter_mult,
      sdist_fine=sdist_f.cuda() if level == 'prop' else None,
      weights_fine=w_f.cuda() if level == 'prop' else None)
  scale = float(grads[0].abs().max())
  close(g_d, grads[0], atol=2e-5 * scale, rtol=2e-4, msg='d raw_density')
  if raw_rgb is not None:
    close(g_rgb, grads[1], atol=2e-5 * float(grads[1].abs().max()), rtol=2e-4, msg='d raw_rgb')
  st_gpu = stats.cpu()
  close(st_gpu[0], data.detach(), rtol=1e-4, atol=1e-7, msg='data loss')
  close(st_gpu[1], st['mses'][0].detach(), rtol=1e-4, atol=1e-7, msg='mse')
  close(st_gpu[2] + st_gpu[3], extra.detach(), rtol=1e-4, atol=1e-7, msg='regulariser')


def _bf(x):
  return torch.tensor(x).to(torch.bfloat16)


@pytest.mark.parametrize('impl', [1, 0])
@pytest.mark.parametrize('M,N,K', [(128, 256, 64), (256, 256, 512), (1000, 128, 320), (384, 1024, 1536),
                                   (130, 64, 128), (4096, 256, 256), (38000, 256, 64), (10000, 768, 128),
                                   # whole 256-row units, several tiles per CTA
                                   (38144, 256, 64), (10240, 1024, 256), (512, 512, 128),
                                   # the 360.gin NerfMLP layer shapes (K = 1024 and the skip layer's 1536)
                                   (512, 1024, 1024), (512, 1024, 1536), (16384, 1024, 512)])
def test_gemm_fwd(ops, impl, M, N, K):
  from multinerf_b200 import lib as L
  rng = np.random.default_rng(M + N + K)
  a = _bf(rng.normal(size=(M, K)).astype(np.float32))
  w = _bf(rng.normal(size=(N, K)).astype(np.float32) / math.sqrt(K))
  bias = torch.tensor(rng.normal(size=(N,)).astype(np.float32))
  ref = torch.relu(a.float() @ w.float().T + bias)
  out = torch.full((M, N + 64), -3.0, dtype=torch.bfloat16, device='cuda')   # strided output view
  bits = torch.full((M, N // 32), -1, dtype=torch.int32, device='cuda')
  ops.gemm(L.GEMM_FWD, a.cuda(), w.cuda(), out[:, :N], m=M, n=N, k=K, act=L.ACT_RELU, bias=bias.cuda(),
           maskbits=bits, impl=impl)
  torch.cuda.synchronize()
  close(out[:, :N].float(), ref.to(torch.bfloat16).float(), atol=2e-2, rtol=1.6e-2, msg=f'fwd impl={impl}')
  assert (out[:, N:] == -3).all()
  # 1-bit ReLU mask == (stored activation > 0), bit j of word w <-> column 32w + j
  got = ((bits.cpu().long()[:, :, None] >> torch.arange(32)) & 1).reshape(M, N).bool()
  assert torch.equal(got, out[:, :N].float().cpu() > 0)
  # no activation, no bias, no mask output
  out2 = torch.empty(M, N, dtype=torch.bfloat16, device='cuda')
  ops.gemm(L.GEMM_FWD, a.cuda(), w.cuda(), out2, m=M, n=N, k=K, impl=impl)
  close(out2.float(), (a.float() @ w.float().T).to(torch.bfloat16).float(), atol=2e-2, rtol=1.6e-2, msg='fwd plain')


@pytest.mark.parametrize('impl', [1, 0])
@pytest.mark.parametrize('M,N,K', [(256, 256, 256), (1000, 1024, 1024), (384, 256, 128),
                                   # several tiles per persistent CTA: row inputs prefetched a tile ahead,
                                   # column sums resident in registers (N=768: 3 column blocks, not resident)
                                   (38000, 256, 256), (10000, 1024, 256), (10000, 768, 128),
                                   # M % 256 == 0
                                   (37888, 256, 256), (10240, 1024, 256), (10240, 768, 128),
                                   # the long reductions of the 360.gin NerfMLP (K = 1024 / 1536)
                                   (512, 1024, 1024), (512, 1024, 1536), (16384, 1024, 1024)])
def test_gemm_dgrad(ops, impl, M, N, K):
  from multinerf_b200 import lib as L
  rng = np.random.default_rng(M + 7 * N + K)
  dy = _bf(rng.normal(size=(M, K)).astype(np.float32))           # reduction over the layer's outputs
  w_kn = _bf(rng.normal(size=(N, K)).astype(np.float32) / math.sqrt(K))   # [in, out]
  mask = _bf(rng.normal(size=(M, N)).astype(np.float32))
  rowv = torch.tensor(rng.normal(size=(M,)).astype(np.float32))
  colv = torch.tensor(rng.normal(size=(N,)).astype(np.float32))
  ref = (dy.float() @ w_kn.float().T + rowv[:, None] * colv[None, :]) * (mask.float() > 0)
  out = torch.empty(M, N, dtype=torch.bfloat16, device='cuda')
  ops.gemm(L.GEMM_DGRAD, dy.cuda(), w_kn.cuda(), out, m=M, n=N, k=K, rowv=rowv.cuda(), colv=colv.cuda(),
           mask=mask.cuda(), impl=impl)
  torch.cuda.synchronize()
  close(out.float(), ref.to(torch.bfloat16).float(), atol=3e-2, rtol=1.6e-2, msg=f'dgrad impl={impl}')
  # same mask as packed bits
  mb = (mask.float() > 0).reshape(M, N // 32, 32).long()
  words = (mb << torch.arange(32)).sum(-1)
  words = torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)
  out2 = torch.empty(M, N, dtype=torch.bfloat16, device='cuda')
  cs = torch.full((N,), 3.0, device='cuda')
  ops.gemm(L.GEMM_DGRAD, dy.cuda(), w_kn.cuda(), out2, m=M, n=N, k=K, rowv=rowv.cuda(), colv=colv.cuda(),
           maskbits=words.cuda(), colsum=cs, impl=impl)
  torch.cuda.synchronize()
  close(out2.float(), ref.to(torch.bfloat16).float(), atol=3e-2, rtol=1.6e-2, msg=f'dgrad bits impl={impl}')
  # fused bias gradient = column sums of the (fp32, pre-rounding) output, accumulated into cs
  close(cs, ref.sum(0) + 3.0, atol=2e-2 * math.sqrt(M), rtol=2e-3, msg=f'dgrad colsum impl={impl}')
  out3 = torch.empty(M, N, dtype=torch.bfloat16, device='cuda')
  ops.gemm(L.GEMM_DGRAD, dy.cuda(), w_kn.cuda(), out3, m=M, n=N, k=K, impl=impl)
  close(out3.float(), (dy.float() @ w_kn.float().T).to(torch.bfloat16).float(), atol=3e-2, rtol=1.6e-2, msg='dgrad plain')


@pytest.mark.parametrize('impl', [1, 0])
@pytest.mark.parametrize('R,Mo,N', [(64, 128, 256), (4096, 512, 256), (8192, 320, 128), (2048, 1536, 1024),
                                    (1024, 64, 64), (65536, 256, 256),
                                    # sample counts that are not a multiple of the 64-row reduction block
                                    (2080, 128, 256), (1000, 256, 256), (37, 64, 64)])
def test_gemm_wgrad(ops, impl, R, Mo, N):
  from multinerf_b200 import lib as L
  rng = np.random.default_rng(R + Mo + N)
  x = _bf(rng.normal(size=(R, Mo)).astype(np.float32))
  dy = _bf(rng.normal(size=(R, N)).astype(np.float32))
  ref = x.float().T @ dy.float()
  out = torch.ones(Mo, N, device='cuda')          # accumulates into existing contents
  ops.gemm(L.GEMM_WGRAD, x.cuda(), dy.cuda(), out, m=Mo, n=N, k=R, impl=impl)
  torch.cuda.synchronize()
  close(out, ref + 1.0, atol=2e-3 * math.sqrt(R), rtol=1e-4, msg=f'wgrad impl={impl}')


@pytest.mark.parametrize('impl', [1, 0])
@pytest.mark.parametrize('R,Mo,N', [(65536, 256, 256), (4096, 512, 256), (8192, 1024, 1024), (16384, 1280, 256),
                                    (2080, 128, 256), (1000, 320, 128), (37, 64, 64), (5000, 256, 64)])
def test_gemm_wgrad_side_sums(ops, impl, R, Mo, N):
  """mnrf_gemm_wgrad: the weight gradient plus the bias gradient (column sums of dY) and the gradient of a
  Dense(1) head on the same activation, both taken from the operand tiles of the main loop."""
  rng = np.random.default_rng(R + 3 * Mo + N)
  x = _bf(rng.normal(size=(R, Mo)).astype(np.float32))
  dy = _bf(rng.normal(size=(R, N)).astype(np.float32))
  w = torch.tensor(rng.normal(size=(R,)).astype(np.float32))
  out = torch.ones(Mo, N, device='cuda')
  bsum = torch.full((N,), 2.0, device='cuda')
  aw = torch.full((Mo,), -1.0, device='cuda')
  ops.gemm_wgrad(x.cuda(), dy.cuda(), out, m=Mo, n=N, k=R, bsum=bsum, side_w=w.cuda(), side_aw=aw, impl=impl)
  torch.cuda.synchronize()
  close(out, x.float().T @ dy.float() + 1.0, atol=2e-3 * math.sqrt(R), rtol=1e-4, msg=f'wgrad impl={impl}')
  close(bsum, dy.float().sum(0) + 2.0, atol=2e-3 * math.sqrt(R), rtol=1e-4, msg=f'bias gradient impl={impl}')
  close(aw, (x.float() * w[:, None]).sum(0) - 1.0, atol=2e-3 * math.sqrt(R), rtol=1e-4, msg=f'head dW impl={impl}')
  # each side sum alone
  b2 = torch.zeros(N, device='cuda')
  o2 = torch.zeros(Mo, N, device='cuda')
  ops.gemm_wgrad(x.cuda(), dy.cuda(), o2, m=Mo, n=N, k=R, bsum=b2, impl=impl)
  close(b2, dy.float().sum(0), atol=2e-3 * math.sqrt(R), rtol=1e-4, msg='bias gradient alone')
  close(o2, x.float().T @ dy.float(), atol=2e-3 * math.sqrt(R), rtol=1e-4, msg='wgrad with bsum only')
  a3 = torch.zeros(Mo, device='cuda')
  o3 = torch.zeros(Mo, N, device='cuda')
  ops.gemm_wgrad(x.cuda(), dy.cuda(), o3, m=Mo, n=N, k=R, side_w=w.cuda(), side_aw=a3, impl=impl)
  close(a3, (x.float() * w[:, None]).sum(0), atol=2e-3 * math.sqrt(R), rtol=1e-4, msg='head dW alone')
  # strided operands (the activation lives inside a wider buffer)
  xb = torch.zeros(R, Mo + 64, dtype=torch.bfloat16, device='cuda')
  xb[:, :Mo] = x.cuda()
  b4 = torch.zeros(N, device='cuda')
  o4 = torch.zeros(Mo, N, device='cuda')
  ops.gemm_wgrad(xb[:, :Mo], dy.cuda(), o4, m=Mo, n=N, k=R, bsum=b4, impl=impl)
  close(o4, x.float().T @ dy.float(), atol=2e-3 * math.sqrt(R), rtol=1e-4, msg='strided x')


def test_composite_diffuse_specular_mode(ops):
  """rgb_mode 1 (Ref-NeRF, models.py:588-602): value and gradients vs oracle autograd."""
  from oracle import o_train
  rng = np.random.default_rng(31)
  B, S = 50, 32
  cfg = dict(CFG, raydist_fn=None, opaque_background=False, density_bias=0.5, rgb_mode=1)
  _, d, _ = kernel_rays(rng, B)
  sdist = torch.tensor(np.sort(rng.uniform(0, 1, (B, S + 1)).astype(np.float32), -1))
  nearv, farv = torch.full((B, 1), 2.0), torch.full((B, 1), 6.0)
  leaves = [torch.tensor(rng.normal(size=sh).astype(np.float32) * sc, requires_grad=True)
            for sh, sc in [((B, S), 2.0), ((B, S, 3), 1.0), ((B, S, 3), 1.5), ((B, S, 3), 1.0)]]
  raw_d, raw_rgb, raw_dif, raw_tint = leaves
  extra = torch.tensor(rng.normal(size=(B, S)).astype(np.float32) * 1e-3)
  target = torch.tensor(rng.uniform(0, 1, (B, 3)).astype(np.float32))

  def colour(raw_rgb, raw_dif, raw_tint):
    spec = torch.sigmoid(raw_tint) * torch.sigmoid(raw_rgb)
    lin = spec + torch.sigmoid(raw_dif - math.log(3.0))
    return torch.clamp(o_math.linear_to_srgb(lin), 0.0, 1.0) * (1 + 2 * 0.001) - 0.001
  _, s_to_t = o_coord.construct_ray_warps(None, nearv, farv)
  tdist = s_to_t(sdist)
  dens = torch.nn.functional.softplus(raw_d + 0.5)
  w = o_render.compute_alpha_weights(dens, tdist, d)[0]
  c = colour(raw_rgb, raw_dif, raw_tint)
  pix = o_render.volumetric_rendering(c, w, tdist, 1.0, farv, False)['rgb']
  loss = ((pix - target) ** 2).sum() / (3 * B) + (w * extra).sum()
  grads = torch.autograd.grad(loss, leaves)
  out = ops.composite_fwd(raw_d.detach().cuda(), raw_rgb.detach().cuda(), sdist.cuda(), d.cuda(),
                          nearv[:, 0].contiguous().cuda(), farv[:, 0].contiguous().cuda(), cfg=cfg,
                          raw_diffuse=raw_dif.detach().cuda(), raw_tint=raw_tint.detach().cuda(), want_samples=True)
  close(out['rgb_samples'], c.detach(), msg='diffuse+specular colour')
  close(out['rgb'], pix.detach(), msg='pixel')
  stats = torch.zeros(8, device='cuda')
  d_dif = torch.empty(B, S, 3, device='cuda')
  d_tint = torch.empty(B, S, 3, device='cuda')
  g_d, g_rgb = ops.composite_bwd(
      raw_d.detach().cuda(), raw_rgb.detach().cuda(), sdist.cuda(), d.cuda(), nearv[:, 0].contiguous().cuda(),
      farv[:, 0].contiguous().cuda(), target.cuda(), torch.ones(B, 1).cuda(), torch.tensor([1.0 / (3 * B)]).cuda(),
      stats, cfg=cfg, loss_type='mse', charb_padding=0.001, data_mult=1.0, distortion_mult=0.0, interlevel_mult=0.0,
      raw_diffuse=raw_dif.detach().cuda(), raw_tint=raw_tint.detach().cuda(), extra_dw=extra.cuda(),
      d_raw_diffuse=d_dif, d_raw_tint=d_tint)
  for got, ref, name in [(g_d, grads[0], 'd raw_density'), (g_rgb, grads[1], 'd raw_rgb'),
                         (d_dif, grads[2], 'd raw_diffuse'), (d_tint, grads[3], 'd raw_tint')]:
    close(got, ref, atol=2e-5 * float(ref.abs().max()), rtol=3e-4, msg=name)


@pytest.mark.parametrize('on_pred', [True, False])
def test_normals_stage_matches_refdir_stage(ops, on_pred):
  """The colourless stage (mnrf_normals_fwd/bwd) and the Ref-NeRF stage share their normals and normal-loss
  arithmetic: with a zero direction-encoding gradient both give the same bits."""
  rng = np.random.default_rng(43)
  B, S = 37, 8
  M = B * S
  v = rng.normal(size=(B, 3)).astype(np.float32)
  v /= np.linalg.norm(v, axis=-1, keepdims=True)
  vt = torch.tensor(v).cuda()
  gp = torch.tensor(rng.normal(size=(M, 3)).astype(np.float32))
  rgd = torch.tensor(rng.normal(size=(3, M)).astype(np.float32) * 30.0)
  gp[0] = 0.0          # clamped norms
  rgd[:, 1] = 0.0
  gp, rgd = gp.cuda(), rgd.cuda()
  w = torch.tensor(rng.uniform(0, 0.2, M).astype(np.float32)).cuda()
  drd = torch.tensor(rng.normal(size=M).astype(np.float32)).cuda()
  om, pm = 0.1 / B, 3e-4 / B
  col0, ld = 64, 128
  desc = ops.refdir_desc(M, S, use_pred_normals=True, use_density_normals=True, use_reflections=False,
                         use_ide=False, use_n_dot_v=False, use_roughness=False, deg_view=4, ide_n=0,
                         roughness_bias=0.0, ld=ld, col0=col0, col_end=ld)
  outs = []
  for stage in ('refdir', 'normals'):
    npd, nd_, edw = torch.empty(M, 3, device='cuda'), torch.empty(M, 3, device='cuda'), torch.empty(M, device='cuda')
    d_gp, d_rgd = torch.empty(M, 3, device='cuda'), torch.empty(3, M, device='cuda')
    stats = torch.zeros(8, device='cuda')
    if stage == 'refdir':
      slab = torch.empty(M, ld, dtype=torch.bfloat16, device='cuda')
      ops.refdir_fwd(desc, None, None, gp, None, rgd, vt, npd, nd_, None, slab, om, pm, on_pred, edw)
      d_slab = torch.zeros(M, ld, dtype=torch.bfloat16, device='cuda')
      ops.refdir_bwd(desc, None, None, gp, None, rgd, vt, w, d_slab, om, pm, on_pred, drd, None, None, d_gp, None,
                     d_rgd, stats)
      heads = d_slab[:, col0:col0 + 4]
    else:
      ops.normals_fwd(M, S, gp, rgd, vt, npd, nd_, om, pm, on_pred, edw)
      head_grads = torch.zeros(M, 64, dtype=torch.bfloat16, device='cuda')
      ops.normals_bwd(M, S, gp, rgd, vt, w, om, pm, on_pred, drd, d_gp, d_rgd, head_grads=head_grads, stats=stats)
      heads = head_grads[:, :4]
    outs.append(dict(normals_pred=npd, normals=nd_, extra_dw=edw, d_grad_pred=d_gp, d_raw_grad_density=d_rgd,
                     heads=heads, stats=stats[4:6]))
  torch.cuda.synchronize()
  ref, got = outs
  assert (ref['extra_dw'] > 0).any() and (ref['stats'] > 0).all()
  for k in ('normals_pred', 'normals', 'extra_dw', 'd_grad_pred', 'd_raw_grad_density', 'heads'):
    assert torch.equal(got[k], ref[k]), k
  close(got['stats'].cpu(), ref['stats'].cpu(), atol=0, rtol=1e-6, msg='loss stats')


def test_outer_mask_and_gemm_mask_mod_addend(ops):
  from multinerf_b200 import lib as L
  rng = np.random.default_rng(51)
  M, N, K = 256, 128, 192
  bits = torch.tensor(rng.integers(-2 ** 31, 2 ** 31, (M, N // 32)), dtype=torch.int32)
  maskb = ((bits.long()[:, :, None] >> torch.arange(32)) & 1).reshape(M, N).bool()
  rowv = torch.tensor(rng.normal(size=3 * M).astype(np.float32))
  colv = torch.tensor(rng.normal(size=N).astype(np.float32))
  out = torch.empty(3 * M, N, dtype=torch.bfloat16, device='cuda')
  ops.outer_mask(rowv.cuda(), colv.cuda(), bits.cuda(), out, rows=3 * M, n=N, mask_mod=M)
  ref = (rowv[:, None] * colv[None, :]) * maskb.repeat(3, 1)
  close(out.float(), ref.to(torch.bfloat16).float(), atol=0, rtol=0, msg='outer_mask')
  for impl in [1, 0]:
    a = _bf(rng.normal(size=(3 * M, K)).astype(np.float32))
    w = _bf(rng.normal(size=(N, K)).astype(np.float32) / math.sqrt(K))
    add = _bf(rng.normal(size=(3 * M, N)).astype(np.float32))
    o2 = torch.empty(3 * M, N, dtype=torch.bfloat16, device='cuda')
    ops.gemm(L.GEMM_DGRAD, a.cuda(), w.cuda(), o2, m=3 * M, n=N, k=K, maskbits=bits.cuda(), mask_mod=M,
             addend=add.cuda(), impl=impl)
    ref2 = (a.float() @ w.float().T) * maskb.repeat(3, 1) + add.float()
    close(o2.float(), ref2.to(torch.bfloat16).float(), atol=3e-2, rtol=1.6e-2, msg=f'mask_mod+addend impl={impl}')
