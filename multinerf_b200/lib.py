"""ctypes binding of libmnrf_b200.so (the C ABI declared in include/mnrf.h).

PyTorch supplies device memory and streams only; every kernel that runs is ours.  The
library is built in-tree by multinerf_b200/build.py; loading fails loudly when it is
missing -- there is no CPU or eager fallback.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# MNRF_LIB: an alternative build of the same library (kernel timing experiments, tools/build_variant.sh)
LIB_PATH = os.environ.get('MNRF_LIB') or os.path.join(_HERE, 'libmnrf_b200.so')


class MnrfError(RuntimeError):
  pass


class SampleDesc(C.Structure):
  _fields_ = [('num_rays', C.c_int32), ('num_prev', C.c_int32), ('num_samples', C.c_int32),
              ('use_dilation', C.c_int32), ('dilation', C.c_float), ('domain_lo', C.c_float),
              ('domain_hi', C.c_float), ('anneal', C.c_float), ('resample_padding', C.c_float),
              ('jitter_mode', C.c_int32), ('max_jitter', C.c_float)]


class EncodeDesc(C.Structure):
  _fields_ = [('num_rays', C.c_int32), ('num_samples', C.c_int32), ('raydist_fn', C.c_int32),
              ('ray_shape', C.c_int32), ('warp_contract', C.c_int32),
              ('disable_integration', C.c_int32), ('basis_k', C.c_int32), ('min_deg', C.c_int32),
              ('max_deg', C.c_int32), ('ld_feat', C.c_int32), ('feat_cols', C.c_int32)]


class GemmDesc(C.Structure):
  _fields_ = [('mode', C.c_int32), ('act', C.c_int32), ('m', C.c_int64), ('n', C.c_int32),
              ('k', C.c_int32), ('lda', C.c_int64), ('ldb', C.c_int64), ('ldc', C.c_int64),
              ('ldmask', C.c_int64), ('ldmaskbits', C.c_int64), ('ldadd', C.c_int64),
              ('mask_mod', C.c_int64),
              ('impl', C.c_int32)]


class GemmInstance(C.Structure):
  _fields_ = [('block_n', C.c_int32), ('staged', C.c_int32), ('mask_tma', C.c_int32), ('smooth', C.c_int32),
              ('side', C.c_int32), ('splits', C.c_int32), ('tiles', C.c_int32), ('grid', C.c_int32),
              ('pingpong', C.c_int32), ('epilogue', C.c_int32)]


class HeadInstance(C.Structure):
  _fields_ = [('fwd_kernel', C.c_int32), ('fwd_lpr', C.c_int32), ('fwd_grid', C.c_int32), ('bwd_kernel', C.c_int32),
              ('bwd_n_out', C.c_int32), ('bwd_lpr', C.c_int32), ('bwd_chunks', C.c_int32), ('bwd_smooth', C.c_int32),
              ('bwd_grid', C.c_int32), ('reserved', C.c_int32), ('fwd_rows_per_pass', C.c_int64),
              ('bwd_rows_per_block', C.c_int64)]


class CompositeDesc(C.Structure):
  _fields_ = [('num_rays', C.c_int32), ('num_samples', C.c_int32), ('raydist_fn', C.c_int32),
              ('opaque_background', C.c_int32), ('density_bias', C.c_float),
              ('density_noise', C.c_float), ('rgb_act', C.c_int32), ('rgb_premult', C.c_float),
              ('rgb_bias', C.c_float), ('rgb_padding', C.c_float), ('bg_const', C.c_float),
              ('rgb_mode', C.c_int32), ('ld_density', C.c_int32), ('ld_rgb', C.c_int32)]


class LossDesc(C.Structure):
  _fields_ = [('c', CompositeDesc), ('loss_type', C.c_int32), ('charb_padding', C.c_float),
              ('data_mult', C.c_float), ('distortion_mult', C.c_float),
              ('interlevel_mult', C.c_float), ('num_samples_fine', C.c_int32),
              ('lossmult_channels', C.c_int32)]


class RobustDesc(C.Structure):
  _fields_ = [('num_rays', C.c_int32), ('patch_size', C.c_int32), ('inner_patch_size', C.c_int32),
              ('filter_size', C.c_int32), ('enable', C.c_int32), ('smoothed_thresh', C.c_float),
              ('patch_thresh', C.c_float)]


class RefdirDesc(C.Structure):
  _fields_ = [('M', C.c_int64), ('num_samples', C.c_int32), ('use_pred_normals', C.c_int32),
              ('use_density_normals', C.c_int32), ('use_reflections', C.c_int32), ('use_ide', C.c_int32),
              ('use_n_dot_v', C.c_int32), ('use_roughness', C.c_int32), ('deg_view', C.c_int32),
              ('ide_n', C.c_int32), ('roughness_bias', C.c_float), ('ld', C.c_int32), ('col0', C.c_int32),
              ('col_end', C.c_int32)]


class CameraDesc(C.Structure):
  _fields_ = [('num_rays', C.c_int32), ('num_cameras', C.c_int32), ('camtype', C.c_int32),
              ('has_distortion', C.c_int32), ('k1', C.c_float), ('k2', C.c_float), ('k3', C.c_float),
              ('k4', C.c_float), ('p1', C.c_float), ('p2', C.c_float), ('undistort_eps', C.c_float),
              ('undistort_iters', C.c_int32), ('has_ndc', C.c_int32), ('ndc_p02', C.c_float),
              ('ndc_p12', C.c_float), ('ndc_near', C.c_float)]


class SphericalDesc(C.Structure):
  _fields_ = [('height', C.c_int32), ('width', C.c_int32), ('camtoworld', C.c_double * 12)]


class PackItem(C.Structure):
  _fields_ = [('master', C.c_void_p), ('w_nk', C.c_void_p), ('w_kn', C.c_void_p), ('in_pad', C.c_int32),
              ('out', C.c_int32), ('tile0', C.c_int32), ('reserved', C.c_int32)]


CHAIN_MAX_LAYERS = 8
CHAIN_FWD, CHAIN_BWD = 0, 1


class ChainLayer(C.Structure):
  _fields_ = [('w', C.c_void_p), ('ldw', C.c_int64), ('bias', C.c_void_p), ('maskbits', C.c_void_p),
              ('ldmaskbits', C.c_int64), ('colsum', C.c_void_p), ('out', C.c_void_p), ('ldo', C.c_int64),
              ('n_stream', C.c_int32), ('stream_col0', C.c_int32), ('stream_kb0', C.c_int32),
              ('n_res', C.c_int32), ('res_kb0', C.c_int32), ('reserved', C.c_int32)]


class ChainDesc(C.Structure):
  _fields_ = [('mode', C.c_int32), ('num_layers', C.c_int32), ('width', C.c_int32), ('stream_cols', C.c_int32),
              ('m', C.c_int64), ('stream', C.c_void_p), ('ldstream', C.c_int64), ('head_w', C.c_void_p),
              ('head_b', C.c_void_p), ('head_out', C.c_void_p), ('head_n', C.c_int32), ('reserved', C.c_int32),
              ('layer', ChainLayer * CHAIN_MAX_LAYERS)]


class AdamDesc(C.Structure):
  _fields_ = [('n', C.c_int64), ('grad_max_val', C.c_float), ('grad_max_norm', C.c_float),
              ('lr', C.c_float), ('beta1', C.c_float), ('beta2', C.c_float), ('eps', C.c_float),
              ('step', C.c_int32), ('grad_scale', C.c_float)]


RAYDIST = {None: 0, 'none': 0, 'reciprocal': 1, 'log': 2, 'exp': 3, 'sqrt': 4, 'square': 5,
           'piecewise': 6}
RAY_SHAPE = {'cone': 0, 'cylinder': 1}
RGB_ACT = {'sigmoid': 0, 'safe_exp': 1}
LOSS_TYPE = {'mse': 0, 'charb': 1, 'rawnerf': 2}
GEMM_FWD, GEMM_DGRAD, GEMM_WGRAD = 0, 1, 2
ACT_NONE, ACT_RELU, ACT_SOFTPLUS, ACT_SILU = 0, 1, 2, 3
SMOOTH_ACTS = (ACT_SOFTPLUS, ACT_SILU)

_P = C.c_void_p
_SIGNATURES = {
    'mnrf_abi_version': (C.c_int, []),
    'mnrf_last_error': (C.c_char_p, []),
    'mnrf_device_ok': (C.c_int, []),
    'mnrf_num_sms': (C.c_int, []),
    'mnrf_sample_level': (C.c_int, [C.POINTER(SampleDesc)] + [_P] * 12),
    'mnrf_encode': (C.c_int, [C.POINTER(EncodeDesc)] + [_P] * 11 + [C.c_int32, _P]),
    'mnrf_viewdir_enc': (C.c_int, [C.c_int32, C.c_int32, C.c_int32, _P, _P, C.c_int32, C.c_int32,
                                   C.c_int32, _P]),
    'mnrf_gemm': (C.c_int, [C.POINTER(GemmDesc)] + [_P] * 10 + [C.c_int64, _P, _P]),
    'mnrf_gemm_wgrad': (C.c_int, [C.POINTER(GemmDesc)] + [_P] * 7),
    'mnrf_gemm_plan': (C.c_int, [C.POINTER(GemmDesc)] + [_P] * 10 + [C.c_int64] + [_P] * 4 +
                       [C.POINTER(GemmInstance)]),
    'mnrf_mlp_chain': (C.c_int, [C.POINTER(ChainDesc), _P]),
    'mnrf_mlp_chain_max_layers': (C.c_int, []),
    'mnrf_head_fwd': (C.c_int, [C.c_int64, C.c_int32, C.c_int32, _P, C.c_int64, _P, _P, _P, _P]),
    'mnrf_head_bwd': (C.c_int, [C.c_int64, C.c_int32, C.c_int32, _P, C.c_int64, _P, _P, _P, C.c_int64, C.c_int32,
                                _P, C.c_int64, _P, _P, C.c_int32, _P, _P, C.c_int32, _P, C.c_int64, _P]),
    # the plan is written to a host HeadInstance, passed by reference (ops.head_plan)
    'mnrf_head_plan': (C.c_int, [C.c_int64, C.c_int32, C.c_int32, _P, _P, C.c_int32, _P, _P, _P]),
    'mnrf_colsum': (C.c_int, [C.c_int64, C.c_int32, _P, C.c_int64, _P, _P]),
    'mnrf_composite_fwd': (C.c_int, [C.POINTER(CompositeDesc)] + [_P] * 18),
    'mnrf_composite_bwd': (C.c_int, [C.POINTER(LossDesc)] + [_P] * 24 + [C.c_int32, _P]),
    'mnrf_robust_mask': (C.c_int, [C.POINTER(RobustDesc)] + [_P] * 7 + [C.c_int32, _P]),
    'mnrf_quantile': (C.c_int, [C.c_int32, C.c_float, _P, _P, _P]),
    'mnrf_refdir_fwd': (C.c_int, [C.POINTER(RefdirDesc)] + [_P] * 10 + [C.c_float, C.c_float, C.c_int32, _P, _P]),
    'mnrf_refdir_bwd': (C.c_int, [C.POINTER(RefdirDesc)] + [_P] * 8 + [C.c_int32, C.c_float, C.c_float, C.c_int32] +
                        [_P] * 8),
    'mnrf_normals_fwd': (C.c_int, [C.c_int64, C.c_int32] + [_P] * 5 + [C.c_float, C.c_float, C.c_int32, _P, _P]),
    'mnrf_normals_bwd': (C.c_int, [C.c_int64, C.c_int32] + [_P] * 4 + [C.c_float, C.c_float, C.c_int32] + [_P] * 2 +
                         [C.c_int64] + [_P] * 3 +
                         [C.c_int64, _P, _P]),
    'mnrf_outer_mask': (C.c_int,[C.c_int64, C.c_int32, C.c_int64, _P, _P, _P, C.c_int64, _P, C.c_int64, _P]),
    'mnrf_act_tangent_bwd': (C.c_int, [C.c_int64, C.c_int32, C.c_int32] + [_P, C.c_int64] * 5 + [C.c_int32, _P]),
    'mnrf_pixels_to_rays': (C.c_int, [C.POINTER(CameraDesc)] + [_P] * 11),
    'mnrf_spherical_rays': (C.c_int, [C.POINTER(SphericalDesc)] + [_P] * 6),
    'mnrf_clip_adam': (C.c_int, [C.POINTER(AdamDesc)] + [_P] * 7),
    'mnrf_pack_weights_batched': (C.c_int, [C.c_int32, _P, C.c_int32, _P]),
    'mnrf_encode_points': (C.c_int, [C.POINTER(EncodeDesc), _P, C.c_float, _P, _P, _P, _P]),
    'mnrf_marching_cubes': (C.c_int, [C.c_int32] * 4 + [_P, C.c_float] + [_P] * 7),
    'mnrf_encode_points_tangent': (C.c_int, [C.POINTER(EncodeDesc), _P, C.c_float, _P, _P, _P, C.c_int32, _P]),
    'mnrf_point_rgb': (C.c_int, [C.POINTER(CompositeDesc), C.c_int64, _P, C.c_int32, _P, _P, _P, _P]),
    'mnrf_mc_normals': (C.c_int, [C.c_int32] * 3 + [_P, C.c_float] + [_P] * 4),
    'mnrf_tsdf_integrate': (C.c_int, [C.POINTER(CameraDesc)] + [C.c_int32] * 3 + [C.c_double] * 4 + [C.c_int32] * 3 +
                            [_P] * 5 + [C.c_float] + [_P] * 5),
    'mnrf_tsdf_integrate_contracted': (C.c_int, [C.POINTER(CameraDesc)] + [C.c_int32] * 3 + [C.c_double] * 4 +
                                       [C.c_int32] * 3 + [_P] * 5 + [C.c_float] + [_P] * 5),
    'mnrf_mesh_uncontract': (C.c_int, [C.c_int64] + [_P] * 5),
    'mnrf_mesh_components': (C.c_int, [C.c_int32, C.c_int64, _P, _P, _P]),
    'mnrf_points_view_count': (C.c_int, [C.POINTER(CameraDesc), C.c_int64, _P, C.c_int32, C.c_int32, C.c_int32,
                                         _P, _P, _P, _P]),
    'mnrf_mesh_quadrics': (C.c_int, [C.c_int32, C.c_int64] + [_P] * 4 + [C.c_int64] + [_P] * 6),
    'mnrf_mesh_edge_cost': (C.c_int, [C.c_int32, C.c_int64, C.c_int64] + [_P] * 12),
    'mnrf_mesh_collapse_select': (C.c_int, [C.c_int32, C.c_int64, C.c_int64] + [_P] * 7),
    'mnrf_mesh_collapse_apply': (C.c_int, [C.c_int32, C.c_int64, C.c_int64] + [_P] * 13),
    'mnrf_mesh_texture_raster': (C.c_int, [C.c_int32, C.c_int64, _P, _P, _P, C.c_int32] + [_P] * 5),
    'mnrf_mesh_bvh': (C.c_int, [C.c_int32, C.c_int32, C.c_int64] + [_P] * 12),
    'mnrf_mesh_trace': (C.c_int, [C.c_int64] + [_P] * 4 + [C.c_int64] + [_P] * 9),
}
MC_COUNT, MC_EMIT = 0, 1
BVH_BOXES, BVH_KEYS, BVH_TREE = 0, 1, 2
HEAD_NONE, HEAD_FWD_SUB, HEAD_FWD_WARP, HEAD_BWD_SUB, HEAD_BWD_WARP = 0, 1, 2, 3, 4
EXPORTED = tuple(_SIGNATURES)

_lib = None


def load(build_if_missing=False):
  """dlopen the library (optionally building it first); raises MnrfError if unavailable."""
  global _lib
  if _lib is not None:
    return _lib
  if not os.path.exists(LIB_PATH):
    if build_if_missing:
      from . import build as _build
      _build.build()
    else:
      raise MnrfError(f'{LIB_PATH} is missing: run `python -m multinerf_b200.build` '
                      '(there is no CPU fallback)')
  lib = C.CDLL(LIB_PATH)
  for name, (res, args) in _SIGNATURES.items():
    fn = getattr(lib, name)          # AttributeError if the .so lacks a declared symbol
    fn.restype = res
    fn.argtypes = args
  if lib.mnrf_abi_version() != 2:
    raise MnrfError('ABI version mismatch')
  _lib = lib
  return lib


def ptr(t):
  """Device pointer of a tensor (None -> NULL).  Tensors must be contiguous CUDA tensors."""
  if t is None:
    return None
  if not t.is_cuda:
    raise MnrfError('mnrf kernels take CUDA tensors only (no CPU path)')
  return C.c_void_p(t.data_ptr())


def stream_ptr():
  return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def check(rc):
  if rc != 0:
    raise MnrfError(load().mnrf_last_error().decode())


def require_device():
  lib = load()
  if not torch.cuda.is_available():
    raise MnrfError('no CUDA device: the mnrf hot path has no CPU fallback')
  if not lib.mnrf_device_ok():
    raise MnrfError(lib.mnrf_last_error().decode())
  return lib
