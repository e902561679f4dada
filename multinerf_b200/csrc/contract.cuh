// The scene contraction of unbounded scenes (coord.contract, coord.py:21-27) as point maps: contract, its inverse and
// its Jacobian.  One copy, included by the encoder (encode.cu: tangent rows of points that are already contracted)
// and by mesh.cu (the contracted-space TSDF fusion and the mapping of contracted meshes back to world space).
//
// contract(x) = x for |x| <= 1, (2 - 1 / r) x / r with r = |x| outside.  It maps the world onto the open ball of
// radius 2.  Its Jacobian J = dy/dx is symmetric: J = s (I - P) + q P with P = xh xh^T, xh = x / r, s = 2/r - 1/r^2
// and q = 1/r^2 outside the unit ball, and J = I inside (as contract_terms in encode.cu writes it).
#pragma once

#include "common.cuh"

namespace mnrf {

// y = contract(x), with |x|^2 clamped to eps as the reference clamps it
__device__ __forceinline__ void contract_point(const float x[3], float y[3]) {
  const float m = fmaxf(kEps, x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
  const float scale = m <= 1.f ? 1.f : (2.f * sqrtf(m) - 1.f) / m;
#pragma unroll
  for (int i = 0; i < 3; ++i) y[i] = scale * x[i];
}

// x = inv_contract(z) for |z| < 2: z inside the unit ball, z / (r (2 - r)) outside.  The reference writes the
// denominator 2 r - r^2, which loses the bits of 2 - r to cancellation near r = 2; r (2 - r) keeps them.  r is
// clamped to the largest float below 2, so a point whose fp32 norm rounds up to 2 still maps to a finite x.
__device__ __forceinline__ void inv_contract_point(const float z[3], float x[3]) {
  const float m = fmaxf(kEps, z[0] * z[0] + z[1] * z[1] + z[2] * z[2]);
  float scale = 1.f;
  if (m > 1.f) {
    const float r = fminf(sqrtf(m), 1.99999988f);             // 2 - 2^-23
    scale = 1.f / (r * (2.f - r));
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) x[i] = scale * z[i];
}

// The Jacobian of contract at world point x as (s, q, xh): J = s (I - P) + q P, P = xh xh^T.  Inside the unit ball
// s = q = 1 and xh = 0.
__device__ __forceinline__ void contract_jacobian(const float x[3], float& s, float& q, float xh[3]) {
  const float m = fmaxf(kEps, x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
  s = 1.f; q = 1.f;
  xh[0] = xh[1] = xh[2] = 0.f;
  if (m <= 1.f) return;
  const float r = sqrtf(m);
  const float ir = 1.f / r;
#pragma unroll
  for (int i = 0; i < 3; ++i) xh[i] = x[i] * ir;
  s = 2.f / r - 1.f / m;
  q = 1.f / m;
}

// J v for the Jacobian (s, q, xh) of contract_jacobian: s (v - (xh.v) xh) + q (xh.v) xh
__device__ __forceinline__ void contract_jacobian_apply(float s, float q, const float xh[3], const float v[3],
                                                        float out[3]) {
  const float beta = xh[0] * v[0] + xh[1] * v[1] + xh[2] * v[2];
#pragma unroll
  for (int i = 0; i < 3; ++i) out[i] = s * (v[i] - beta * xh[i]) + (q * beta) * xh[i];
}

}  // namespace mnrf
