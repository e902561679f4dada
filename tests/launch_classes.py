"""Launch classes: each recorded `mnrf_*` call (abi_record.Recorder.named) mapped to the tuple of everything its kernel
branches on -- descriptor flags and modes, which optional operands are null, and the plan the library picks -- and
nothing that only sizes the launch.  test_launch_coverage_cpu.py asks that every class the models reach is also the
class of a launch an fp64 test makes.  A helper module, not a test module.

Each entry point has one function `<symbol without mnrf_>(args, plan)` -> tuple of (field, value) pairs; `plan` is
the library's own host-only planner for that entry point (PLANS) where it has one.  The comment above each function says
which kernel branch each field selects: that comment is what the function is checked against.
"""
import ctypes as C


def _null(*ptrs):
  return tuple(p is None for p in ptrs)


# ---------------------------------------------------------------------------------------------- dense-layer GEMM
def gemm_plan(sym, a):
  """The instance mnrf_gemm_plan picks for a recorded mnrf_gemm / mnrf_gemm_wgrad call (host only: without a device
  the library plans for 132 SMs, an H100 SXM's count).  Raises for arguments the launch refuses."""
  from multinerf_b200 import lib as L
  lib = L.load()
  d = L.GemmDesc(**{k: v for k, v in a['d'].items()})
  p = lambda name: C.c_void_p(a[name]) if a.get(name) else None
  plan = L.GemmInstance()
  if sym == 'mnrf_gemm':
    args = [p(n) for n in ('a', 'b', 'bias', 'rowv', 'colv', 'mask', 'maskbits', 'colsum', 'addend', 'z')]
    args += [a['ldz'], p('out'), None, None, None]
  else:
    args = [p('a'), p('b')] + [None] * 8 + [0, p('out'), p('bsum'), p('side_w'), p('side_aw')]
  rc = lib.mnrf_gemm_plan(C.byref(d), *args, C.byref(plan))
  if rc:
    raise RuntimeError(f'{sym}: mnrf_gemm_plan refuses the call: {lib.mnrf_last_error().decode()}')
  return {name: int(getattr(plan, name)) for name, _ in L.GemmInstance._fields_}


# mnrf_gemm (csrc/gemm_tc.cu, gemm_tc_act.cu):
#   mode     FWD / DGRAD kernel body (kDgrad), or WGRAD: the cooperative WGRAD instance without side sums (the
#            instance mnrf_gemm_wgrad runs when bsum and side_aw are NULL)
#   act      epilogue activation: ReLU mask, none, or the smooth a(z) / a'(z) path
#   impl     0 tensor cores, 1 the SIMT reference kernel (gemm_ref.cu)
#   null     which of bias, rowv, colv, mask, maskbits, colsum, addend, z are NULL: each is a run-time operand test of
#            the generic epilogue (EPI_GENERIC), and bias / maskbits / rowv-colv also pick the compiled ping-pong
#            epilogue below
#   mask_mod mask_mod > 0: mask-bit and z rows are taken modulo mask_mod (the tangent streams of density normals)
#   plan     block_n (tile width template BN), staged (TMA bulk store through shared memory, or register stores),
#            mask_tma (DGRAD: mask bits loaded by TMA with the operands; FWD: stored by TMA), smooth (the softplus /
#            SiLU epilogue instance), pingpong (gemm_tc_pingpong_kernel or the cooperative kernel) and epilogue (the
#            ping-pong epilogue operand set compiled into the instance).  The plan is not asked for impl 1.
# The row pitches are not part of the class: the kernel reads them only through the TMA descriptors and the store
# addresses, and where alignment changes the path the plan's `staged` and `mask_tma` say so.
def gemm(a, plan):
  d = a['d']
  cls = (('mode', d['mode']), ('act', d['act']), ('impl', d['impl']),
         ('null', _null(a['bias'], a['rowv'], a['colv'], a['mask'], a['maskbits'], a['colsum'], a['addend'],
                        a['z'])),
         ('mask_mod', d['mask_mod'] > 0))
  if d['impl'] == 0:
    p = plan('mnrf_gemm', a)
    cls += (('plan', tuple(p[k] for k in ('block_n', 'staged', 'mask_tma', 'smooth', 'pingpong', 'epilogue'))),)
  return cls


# mnrf_gemm_wgrad (csrc/gemm_tc.cu, the WGRAD instance of the cooperative kernel):
#   impl     0 tensor cores, 1 SIMT reference (side sums as separate passes)
#   null     bsum (bias-gradient side sum) and side_w / side_aw (the Dense(1) head's dW side sum): the producer
#            warpgroup's side-sum warps run only for non-null outputs
#   plan     block_n (tile width template BN) and side (the side-sum instance); splits only sizes the reduction
def gemm_wgrad(a, plan):
  d = a['d']
  cls = (('impl', d['impl']), ('null', _null(a['bsum'], a['side_w'], a['side_aw'])))
  if d['impl'] == 0:
    p = plan('mnrf_gemm_wgrad', a)
    cls += (('plan', (p['block_n'], p['side'])),)
  return cls


# ---------------------------------------------------------------------------------------------- narrow heads
def head_plan(sym, a):
  """The instances mnrf_head_plan picks for a recorded mnrf_head_fwd / mnrf_head_bwd call (host only).  Raises for
  arguments the backward launch refuses."""
  from multinerf_b200 import lib as L
  lib = L.load()
  p = lambda name: C.c_void_p(a[name]) if a.get(name) else None
  plan = L.HeadInstance()
  if sym == 'mnrf_head_fwd':
    rc = lib.mnrf_head_plan(a['m'], a['k'], a['n_out'], p('x'), p('w'), 0, None, None, C.byref(plan))
  else:
    rc = lib.mnrf_head_plan(a['m'], a['k'], a['n_out'], p('x'), p('w'), a['act'], p('z'), p('dx'), C.byref(plan))
  if rc:
    raise RuntimeError(f'{sym}: mnrf_head_plan refuses the call: {lib.mnrf_last_error().decode()}')
  return {name: int(getattr(plan, name)) for name, _ in L.HeadInstance._fields_}


# mnrf_head_fwd (csrc/heads.cu):
#   null     b is NULL: the bias add is skipped
#   strided  ldx > k: rows of x are read at a pitch past the columns (both kernels index x + m * ldx)
#   plan     fwd_kernel (head_fwd_sub_kernel, K <= 256 in whole 16-byte lanes, or the warp-per-row head_fwd_kernel) and
#            fwd_lpr (the sub kernel's LPR template: lanes per row).  n_out is a run-time loop bound of both kernels.
def head_fwd(a, plan):
  p = plan('mnrf_head_fwd', a)
  return (('null', _null(a['b'])), ('strided', a['ldx'] > a['k']), ('plan', (p['fwd_kernel'], p['fwd_lpr'])))


# mnrf_head_bwd (csrc/heads.cu):
#   act      the factor on dx: none, the ReLU mask x > 0, or a'(z) (the SMOOTH template, also in the plan)
#   null     which of dx, z, dw, dw2, db, dxsum, dx2 are NULL: each output is written only when given
#   split    0 < dw_split < n_out: dW split between dw and dw2
#   dx_cols  0 < dx_cols < k: dx and dxsum cover the first dx_cols columns, dx2 the rest
#   strided  ldx > k, and lddx > dx_cols (or k) when dx is given: row pitches past the columns
#   plan     bwd_kernel (head_bwd_sub_kernel or the warp-per-row head_bwd_kernel), bwd_n_out (template N_OUT), bwd_lpr
#            (the sub kernel's LPR), bwd_chunks (the warp kernel's kMaxChunks) and bwd_smooth (template SMOOTH)
def head_bwd(a, plan):
  p = plan('mnrf_head_bwd', a)
  cols = a['dx_cols'] or a['k']
  return (('act', a['act']), ('null', _null(a['dx'], a['z'], a['dw'], a['dw2'], a['db'], a['dxsum'], a['dx2'])),
          ('split', 0 < a['dw_split'] < a['n_out']), ('dx_cols', 0 < a['dx_cols'] < a['k']),
          ('strided', a['ldx'] > a['k'] or (a['dx'] is not None and a['lddx'] > cols)),
          ('plan', tuple(p[k] for k in ('bwd_kernel', 'bwd_n_out', 'bwd_lpr', 'bwd_chunks', 'bwd_smooth'))))


CLASSES = {'mnrf_gemm': gemm, 'mnrf_gemm_wgrad': gemm_wgrad, 'mnrf_head_fwd': head_fwd, 'mnrf_head_bwd': head_bwd}
PLANS = {'mnrf_gemm': gemm_plan, 'mnrf_gemm_wgrad': gemm_plan, 'mnrf_head_fwd': head_plan, 'mnrf_head_bwd': head_plan}


def classify(sym, args):
  """The launch class of one named record."""
  return CLASSES[sym](args, PLANS.get(sym))
