// SIMT reference GEMM (bring-up / test cross-check of the wgmma kernel at sizes the CPU oracle
// cannot reach) and the mnrf_gemm dispatcher.  Same contract as gemm_tc.cu, no tensor cores.
#include <algorithm>

#include "common.cuh"

namespace mnrf {

int gemm_tc_launch(const mnrf_gemm_desc* d, const mnrf_bf16* a, const mnrf_bf16* b, const float* bias,
                   const float* rowv, const float* colv, const mnrf_bf16* mask, uint32_t* maskbits,
                   float* colsum, const mnrf_bf16* addend, void* out, cudaStream_t stream, float* bsum,
                   const float* side_w, float* side_aw, mnrf_bf16* z, int64_t ldz);

__device__ __forceinline__ float ldbf(const __nv_bfloat16* p) { return __bfloat162float(*p); }

// FWD/DGRAD: out[m,n] = sum_k A[m,k] * B[n,k]   (16x16 tiles)
__global__ void gemm_ref_nt_kernel(mnrf_gemm_desc d, const __nv_bfloat16* __restrict__ a,
                                   const __nv_bfloat16* __restrict__ b, const float* __restrict__ bias,
                                   const float* __restrict__ rowv, const float* __restrict__ colv,
                                   const __nv_bfloat16* __restrict__ mask, uint32_t* __restrict__ maskbits,
                                   const __nv_bfloat16* __restrict__ addend, __nv_bfloat16* __restrict__ out,
                                   __nv_bfloat16* __restrict__ z, int64_t ldz) {
  __shared__ float sa[16][17], sb[16][17];
  const int64_t m = (int64_t)blockIdx.y * 16 + threadIdx.y;
  const int n = blockIdx.x * 16 + threadIdx.x;
  float acc = 0.f;
  for (int k0 = 0; k0 < d.k; k0 += 16) {
    int64_t am = (int64_t)blockIdx.y * 16 + threadIdx.y;
    int bn = blockIdx.x * 16 + threadIdx.y;
    sa[threadIdx.y][threadIdx.x] = (am < d.m && k0 + threadIdx.x < d.k) ? ldbf(a + am * d.lda + k0 + threadIdx.x) : 0.f;
    sb[threadIdx.y][threadIdx.x] = (bn < d.n && k0 + threadIdx.x < d.k) ? ldbf(b + (int64_t)bn * d.ldb + k0 + threadIdx.x) : 0.f;
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) acc += sa[threadIdx.y][kk] * sb[threadIdx.x][kk];
    __syncthreads();
  }
  if (m >= d.m || n >= d.n) return;
  if (d.mode == MNRF_GEMM_FWD) {
    if (bias) acc += bias[n];
    if (d.act == MNRF_ACT_RELU) {
      acc = relu_nan(acc);
      if (maskbits && acc > 0.f) atomicOr(&maskbits[m * d.ldmaskbits + (n >> 5)], 1u << (n & 31));
    } else if (d.act == MNRF_ACT_SOFTPLUS || d.act == MNRF_ACT_SILU) {
      if (z) z[m * ldz + n] = __float2bfloat16(acc);
      acc = act_fwd(d.act, acc);
    }
  } else {
    if (rowv) acc += rowv[m] * colv[n];
    if (z) {
      acc *= act_d1(d.act, ldbf(z + (d.mask_mod > 0 ? m % d.mask_mod : m) * ldz + n));
    } else if (maskbits) {
      const int64_t mrow = d.mask_mod > 0 ? m % d.mask_mod : m;
      if (!((maskbits[mrow * d.ldmaskbits + (n >> 5)] >> (n & 31)) & 1u)) acc = 0.f;
    } else if (mask && !(ldbf(mask + m * d.ldmask + n) > 0.f)) {
      acc = 0.f;
    }
    if (addend) acc += ldbf(addend + m * d.ldadd + n);
  }
  out[m * d.ldc + n] = __float2bfloat16(acc);
}

// WGRAD: out[mo,n] += sum_r A[r,mo] * B[r,n]
__global__ void gemm_ref_tn_kernel(mnrf_gemm_desc d, const __nv_bfloat16* __restrict__ a,
                                   const __nv_bfloat16* __restrict__ b, float* __restrict__ out,
                                   int r_per_block) {
  const int64_t mo = (int64_t)blockIdx.y * 16 + threadIdx.y;
  const int n = blockIdx.x * 16 + threadIdx.x;
  const int64_t r0 = (int64_t)blockIdx.z * r_per_block, r1 = min((int64_t)d.k, r0 + r_per_block);
  __shared__ float sa[16][17], sb[16][17];
  float acc = 0.f;
  for (int64_t rr = r0; rr < r1; rr += 16) {
    int64_t r = rr + threadIdx.y;
    int64_t amo = (int64_t)blockIdx.y * 16 + threadIdx.x;
    sa[threadIdx.y][threadIdx.x] = (r < r1 && amo < d.m) ? ldbf(a + r * d.lda + amo) : 0.f;
    sb[threadIdx.y][threadIdx.x] = (r < r1 && n < d.n) ? ldbf(b + r * d.ldb + n) : 0.f;
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) acc += sa[kk][threadIdx.y] * sb[kk][threadIdx.x];
    __syncthreads();
  }
  if (mo < d.m && n < d.n) atomicAdd(&out[mo * d.ldc + n], acc);
}

}  // namespace mnrf

extern "C" int mnrf_gemm(const mnrf_gemm_desc* d, const mnrf_bf16* a, const mnrf_bf16* b, const float* bias,
                         const float* rowv, const float* colv, const mnrf_bf16* mask, uint32_t* maskbits,
                         float* colsum, const mnrf_bf16* addend, mnrf_bf16* z, int64_t ldz, void* out,
                         mnrf_stream stream) {
  using namespace mnrf;
  if (d && (d->m == 0 || d->n == 0 || d->k == 0)) return 0;   // empty operand: nothing to compute or accumulate
  MNRF_CHECK(d && a && b && out, "mnrf_gemm: null pointer");
  MNRF_CHECK(d->mode >= 0 && d->mode <= 2, "mnrf_gemm: unknown mode %d", d->mode);
  if (d->act == MNRF_ACT_SOFTPLUS || d->act == MNRF_ACT_SILU) {
    MNRF_CHECK(d->mode == MNRF_GEMM_FWD || d->mode == MNRF_GEMM_DGRAD, "mnrf_gemm: a smooth activation is FWD or DGRAD");
    MNRF_CHECK(d->mode == MNRF_GEMM_FWD || z, "mnrf_gemm: the DGRAD of a smooth activation needs z");
    MNRF_CHECK(!z || ldz >= d->n, "mnrf_gemm: ldz %lld < N %d", (long long)ldz, d->n);
    MNRF_CHECK(!mask && !maskbits, "mnrf_gemm: a smooth activation takes z, not a ReLU mask");
  } else {
    MNRF_CHECK(!z, "mnrf_gemm: z is the pre-activation of a smooth activation, act %d is not one", d->act);
  }
  MNRF_CHECK((rowv == nullptr) == (colv == nullptr), "mnrf_gemm: rowv and colv come together");
  // the bf16 mask has a row per output row (mask_mod is for the 1-bit masks and z of the stacked tangent streams)
  MNRF_CHECK(!mask || d->mask_mod == 0, "mnrf_gemm: mask_mod applies to maskbits and z, not to a bf16 mask");
  if (d->m == 0 || d->n == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  if (colsum) MNRF_CHECK(d->mode == MNRF_GEMM_DGRAD, "mnrf_gemm: colsum is a DGRAD output");
  if (addend) MNRF_CHECK(d->mode == MNRF_GEMM_DGRAD, "mnrf_gemm: addend is a DGRAD input");
  if (d->impl == 0)
    return gemm_tc_launch(d, a, b, bias, rowv, colv, mask, maskbits, colsum, addend, out, s, nullptr, nullptr, nullptr,
                          z, ldz);
  dim3 block(16, 16);
  if (d->mode != MNRF_GEMM_WGRAD) {
    dim3 grid((d->n + 15) / 16, (unsigned)((d->m + 15) / 16));
    if (maskbits && d->mode == MNRF_GEMM_FWD && d->act == MNRF_ACT_RELU) {
      // the reference kernel ORs bits in: clear the words of this [M, N/32] block first
      MNRF_CUDA(cudaMemset2DAsync(maskbits, d->ldmaskbits * 4, 0, (size_t)(d->n / 32) * 4, d->m, s));
    }
    gemm_ref_nt_kernel<<<grid, block, 0, s>>>(*d, reinterpret_cast<const __nv_bfloat16*>(a),
                                               reinterpret_cast<const __nv_bfloat16*>(b), bias, rowv, colv,
                                               reinterpret_cast<const __nv_bfloat16*>(mask), maskbits,
                                               reinterpret_cast<const __nv_bfloat16*>(addend),
                                               reinterpret_cast<__nv_bfloat16*>(out),
                                               reinterpret_cast<__nv_bfloat16*>(z), ldz);
    MNRF_LAUNCH_CHECK();
    if (colsum) {   // reference path: sum the (bf16-rounded) output in a second pass
      if (int rc = mnrf_colsum(d->m, d->n, reinterpret_cast<const mnrf_bf16*>(out), d->ldc, colsum, stream)) return rc;
    }
  } else {
    int splits = (int)std::max<int64_t>(1, std::min<int64_t>(64, d->k / 4096));
    int rpb = (int)(((d->k + splits - 1) / splits + 15) / 16 * 16);
    splits = (d->k + rpb - 1) / rpb;
    dim3 grid((d->n + 15) / 16, (unsigned)((d->m + 15) / 16), splits);
    gemm_ref_tn_kernel<<<grid, block, 0, s>>>(*d, reinterpret_cast<const __nv_bfloat16*>(a),
                                               reinterpret_cast<const __nv_bfloat16*>(b),
                                               reinterpret_cast<float*>(out), rpb);
  }
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_gemm_wgrad(const mnrf_gemm_desc* d, const mnrf_bf16* a, const mnrf_bf16* b, float* bsum,
                               const float* side_w, float* side_aw, float* out, mnrf_stream stream) {
  using namespace mnrf;
  if (d && (d->m == 0 || d->n == 0 || d->k == 0)) return 0;
  MNRF_CHECK(d && a && b && out, "mnrf_gemm_wgrad: null pointer");
  MNRF_CHECK(d->mode == MNRF_GEMM_WGRAD, "mnrf_gemm_wgrad: mode must be MNRF_GEMM_WGRAD");
  MNRF_CHECK((side_w == nullptr) == (side_aw == nullptr), "mnrf_gemm_wgrad: side_w and side_aw come together");
  // tensor cores: one launch, the side sums taken from the operand tiles the main loop stages
  if (d->impl == 0) return gemm_tc_launch(d, a, b, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, out,
                                          (cudaStream_t)stream, bsum, side_w, side_aw, nullptr, 0);
  // SIMT reference: the weight gradient, then the side sums as separate passes over the same operands
  if (int rc = mnrf_gemm(d, a, b, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0, out,
                         stream))
    return rc;
  if (bsum)
    if (int rc = mnrf_colsum(d->k, d->n, b, d->ldb, bsum, stream)) return rc;
  if (side_aw)      // side_aw[m] += sum_r side_w[r] * A[r, m]  ==  the dW of a Dense(1) head on A with draw = side_w
    if (int rc = mnrf_head_bwd(d->k, (int32_t)d->m, 1, a, d->lda, a, side_w, nullptr, 0, MNRF_ACT_NONE, nullptr, 0,
                               side_aw, nullptr, 0, nullptr, nullptr, 0, nullptr, 0, stream))
      return rc;
  return 0;
}
