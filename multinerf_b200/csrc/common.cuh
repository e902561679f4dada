// Internal helpers shared by the kernels of libmnrf_b200.so (sm_90a only).
#pragma once

#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/mnrf.h"

namespace mnrf {

void set_error(const char* fmt, ...);

#define MNRF_CHECK(cond, ...)            \
  do {                                   \
    if (!(cond)) {                       \
      ::mnrf::set_error(__VA_ARGS__);    \
      return 1;                          \
    }                                    \
  } while (0)

#define MNRF_CUDA(expr)                                                               \
  do {                                                                                \
    cudaError_t _e = (expr);                                                          \
    if (_e != cudaSuccess) {                                                          \
      ::mnrf::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),       \
                        __FILE__, __LINE__);                                          \
      return 2;                                                                       \
    }                                                                                 \
  } while (0)

#define MNRF_LAUNCH_CHECK() MNRF_CUDA(cudaGetLastError())

constexpr float kEps = 1.1920929e-07f;        // jnp.finfo(float32).eps
constexpr float kEpsSq = 1.4210855e-14f;      // eps**2 (stepfun.py:89,121)
constexpr unsigned kFull = 0xffffffffu;

// ReLU that keeps a NaN, as torch.relu and jnp.maximum do (fmaxf returns the other operand): one max.NaN.f32
__device__ __forceinline__ float relu_nan(float x) {
  float r;
  asm("max.NaN.f32 %0, %1, 0f00000000;" : "=f"(r) : "f"(x));
  return r;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(kFull, v, o));
  return v;
}
// Inclusive prefix sum across the 32 lanes.
__device__ __forceinline__ float warp_scan_incl(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    float n = __shfl_up_sync(kFull, v, o);
    if (lane >= o) v += n;
  }
  return v;
}
// Inclusive suffix sum across the 32 lanes.
__device__ __forceinline__ float warp_scan_incl_rev(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    float n = __shfl_down_sync(kFull, v, o);
    if (lane + o < 32) v += n;
  }
  return v;
}

__device__ __forceinline__ float softplus_f(float x) {
  // jax.nn.softplus = logaddexp(x, 0) = max(x,0) + log1p(exp(-|x|))
  return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x)));
}
__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + expf(-x)); }

// Smooth activations of the Dense layers (MNRF_ACT_SOFTPLUS | MNRF_ACT_SILU) and their first two derivatives:
//   softplus: a = logaddexp(z, 0),  a' = s,                 a'' = s (1 - s)
//   silu:     a = z s,              a' = s (1 + z (1 - s)),  a'' = s (1 - s) (2 + z (1 - 2 s)),     s = sigmoid(z)
// They run in GEMM epilogues, once per output element, and their results are rounded to bf16: the hardware
// exp / log / reciprocal approximations (relative error ~1e-6) keep the epilogue short.
__device__ __forceinline__ float sigmoid_fast(float z) { return __fdividef(1.f, 1.f + __expf(-z)); }
__device__ __forceinline__ float act_fwd(int act, float z) {
  return act == MNRF_ACT_SILU ? z * sigmoid_fast(z) : fmaxf(z, 0.f) + __logf(1.f + __expf(-fabsf(z)));
}
__device__ __forceinline__ float act_d1(int act, float z) {
  const float s = sigmoid_fast(z);
  return act == MNRF_ACT_SILU ? s * (1.f + z * (1.f - s)) : s;
}
__device__ __forceinline__ float act_d2(int act, float z) {
  const float s = sigmoid_fast(z), q = s * (1.f - s);
  return act == MNRF_ACT_SILU ? q * (2.f + z * (1.f - 2.f * s)) : q;
}

// math.safe_sin (math.py:26-38): sin(|x| < 100*pi ? x : x mod 100*pi), Python-style mod.
__device__ __forceinline__ float safe_sin_f(float x) {
  const float t = 314.159271240234375f;  // fl32(100*pi)
  if (!(fabsf(x) < t)) {
    float r = fmodf(x, t);
    if (r != 0.f && (r < 0.f)) r += t;
    x = r;
  }
  return sinf(x);
}

// rintf for |v| < 2^22 without the conversion pipe: adding 1.5 * 2^23 rounds v to an integer (nearest-even, the
// add's own rounding) and the subtraction is exact.  FRND shares the quarter-rate unit with MUFU.SIN / MUFU.EX2,
// which the IPE inner loop already keeps busy three instructions out of every ~30.
__device__ __forceinline__ float rint_small(float v) {
  return __fsub_rn(__fadd_rn(v, 12582912.f), 12582912.f);
}

// Same function for the bulk of the IPE features (1.3e9 evaluations per 360.gin step):
//  * x mod fl32(100*pi) is reproduced EXACTLY without fmodf: k = floor(x/t) may be off by one, the
//    remainder x - k*t is exact in one FMA (fmod results are representable), and the +-t fix-up is
//    exact for the same reason;
//  * sin of the reduced argument (|r| < 100*pi): Cody-Waite reduction by 2*pi (hi + lo, two FMAs)
//    then MUFU.SIN (|arg| <= pi: abs error 2^-21.4).  Total abs error < 1e-6 (parity bar: 1e-5).
// sin(x) for |x| < 100*pi (the caller guarantees it): Cody-Waite by 2*pi, then MUFU.SIN
__device__ __forceinline__ float sin_below_100pi(float x) {
  const float q = rint_small(__fmul_rn(x, 0.15915494309189535f));
  float r = __fmaf_rn(-q, 6.2831854820251465f, x);
  r = __fmaf_rn(q, 1.7484555e-7f, r);      // 2*pi = 6.2831854820251465 - 1.7484555e-7
  return __sinf(r);
}
__device__ __forceinline__ float safe_sin_fast(float x) {
  const float t = 314.159271240234375f;  // fl32(100*pi)
  if (!(fabsf(x) < t)) {
    float k = floorf(__fmul_rn(x, 1.f / t));
    float r = __fmaf_rn(-k, t, x);
    if (r < 0.f) r = __fadd_rn(r, t);
    else if (r >= t) r = __fsub_rn(r, t);
    x = r;
  }
  return sin_below_100pi(x);
}

// safe_sin for |x| < 2^22 * 100*pi (1.3e9), without branches.  The large-argument path of safe_sin_fast diverges
// (lanes above and below 100*pi, then the two +-t fix-ups), and at the high IPE degrees nearly every warp takes it:
// that path executes several times the instructions per (direction, degree) step of the check-free one.  Here the
// remainder is taken with k = rint(x / t) instead of floor (the remainder x - k t is exact in one FMA either way;
// a negative one is fixed up by + t, which is exact too), and a select keeps x itself below 100*pi -- the reference
// reduces only when |x| >= 100*pi, and fl32(100*pi) != 100*pi, so reducing a small x would change it by 6e-6.
__device__ __forceinline__ float safe_sin_nobranch(float x) {
  const float t = 314.159271240234375f;  // fl32(100*pi)
  const float k = rint_small(__fmul_rn(x, 1.f / t));
  float r = __fmaf_rn(-k, t, x);
  r = r < 0.f ? __fadd_rn(r, t) : r;
  return sin_below_100pi(fabsf(x) < t ? x : r);
}

// sin and cos of the same reduced argument (the cosine is d/dx safe_sin(x), used by the tangent
// features of the density-normal chain).
__device__ __forceinline__ void safe_sincos_fast(float x, float& sn, float& cs) {
  const float t = 314.159271240234375f;
  if (!(fabsf(x) < t)) {
    float k = floorf(__fmul_rn(x, 1.f / t));
    float r = __fmaf_rn(-k, t, x);
    if (r < 0.f) r = __fadd_rn(r, t);
    else if (r >= t) r = __fsub_rn(r, t);
    x = r;
  }
  const float q = rint_small(__fmul_rn(x, 0.15915494309189535f));
  float r = __fmaf_rn(-q, 6.2831854820251465f, x);
  r = __fmaf_rn(q, 1.7484555e-7f, r);
  sn = __sinf(r);
  cs = __cosf(r);
}

// s_to_t of coord.construct_ray_warps (coord.py:63-99) for one value.
__device__ __forceinline__ float fwd_raydist(int fn, float x) {
  switch (fn) {
    case MNRF_RAYDIST_RECIPROCAL: return 1.f / x;
    case MNRF_RAYDIST_LOG: return logf(x);
    case MNRF_RAYDIST_EXP: return expf(x);
    case MNRF_RAYDIST_SQRT: return sqrtf(x);
    case MNRF_RAYDIST_SQUARE: return x * x;
    case MNRF_RAYDIST_PIECEWISE: return x < 1.f ? 0.5f * x : 1.f - 0.5f / x;
    default: return x;
  }
}
__device__ __forceinline__ float inv_raydist(int fn, float x) {
  switch (fn) {
    case MNRF_RAYDIST_RECIPROCAL: return 1.f / x;
    case MNRF_RAYDIST_LOG: return expf(x);
    case MNRF_RAYDIST_EXP: return logf(x);
    case MNRF_RAYDIST_SQRT: return x * x;
    case MNRF_RAYDIST_SQUARE: return sqrtf(x);
    case MNRF_RAYDIST_PIECEWISE: return x < 0.5f ? 2.f * x : 0.5f / (1.f - x);
    default: return x;
  }
}
__device__ __forceinline__ float s_to_t(int fn, float s, float s_near, float s_far) {
  // fn_inv(s * s_far + (1 - s) * s_near), products and sum rounded separately like XLA's
  // unfused elementwise graph.
  return inv_raydist(fn, __fadd_rn(__fmul_rn(s, s_far), __fmul_rn(__fsub_rn(1.f, s), s_near)));
}

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }

inline int ceil_div(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

}  // namespace mnrf
