// Narrow Dense heads (1-4 outputs), bias-gradient column sums, weight repacking, clip+Adam.
//
// Heads replace the Dense(1) density head models.py:460, Dense(3) rgb head :585 and the other
// <=4-wide heads (:495,515,518,521); they are HBM-bound row reductions (16-byte loads; rows of up to 256
// inputs: K/8 lanes per row and four rows in flight per lane -- head_*_sub_kernel; wider rows: one warp per
// row), not GEMM-shaped work.  Optimizer: train_utils.clip_gradients
// train_utils.py:200-218 + nan_to_num :328 + optax.adam (restated, see oracle/o_train.py).
#include <algorithm>

#include "common.cuh"

namespace mnrf {

constexpr int kMaxHead = 4;

// raw[m, o] = sum_k x[m,k] * w[o,k] + b[o]
__global__ void __launch_bounds__(256)
head_fwd_kernel(int64_t M, int K, int n_out, const __nv_bfloat16* __restrict__ x, int64_t ldx,
                const __nv_bfloat16* __restrict__ w, const float* __restrict__ b,
                float* __restrict__ raw) {
  extern __shared__ __align__(16) unsigned char smraw[];
  __nv_bfloat16* sw = reinterpret_cast<__nv_bfloat16*>(smraw);   // [n_out][K]
  for (int i = threadIdx.x; i < n_out * K; i += blockDim.x) sw[i] = w[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int64_t m = (int64_t)blockIdx.x * nw + wib; m < M; m += (int64_t)gridDim.x * nw) {
    const uint4* xr = reinterpret_cast<const uint4*>(x + m * ldx);
    float acc[kMaxHead] = {0.f, 0.f, 0.f, 0.f};
    for (int c = lane; c < K / 8; c += 32) {
      uint4 v = xr[c];
      uint32_t vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int o = 0; o < kMaxHead; ++o) {
        if (o < n_out) {
          const uint4 wv = reinterpret_cast<const uint4*>(sw + (size_t)o * K)[c];
          uint32_t ww[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
          for (int q = 0; q < 4; ++q)
            acc[o] += bf16_lo(vv[q]) * bf16_lo(ww[q]) + bf16_hi(vv[q]) * bf16_hi(ww[q]);
        }
      }
    }
#pragma unroll
    for (int o = 0; o < kMaxHead; ++o) {
      if (o < n_out) {
        float s = warp_sum(acc[o]);
        if (lane == 0) raw[m * n_out + o] = s + (b ? b[o] : 0.f);
      }
    }
  }
}

// element (k, o) of dW in the fp32 master layout: outputs [0, split) in dw [K, split], the rest in dw2 (mnrf.h)
__device__ __forceinline__ float* dw_at(float* dw, float* dw2, int split, int n_out, int k, int o) {
  return o < split ? dw + (size_t)k * split + o : dw2 + (size_t)k * (n_out - split) + (o - split);
}

// dx[m,k] = relu'(x[m,k]) * sum_o draw[m,o] w[o,k] for k < dx_cols (SMOOTH: a'(z[m,k]) in place of relu'(x[m,k]));  dx2[m,k-dx_cols] = sum_o draw[m,o] w[o,k] for
// k >= dx_cols (optional);  dw[k,o] += sum_m draw[m,o] x[m,k];  db[o] += sum_m draw[m,o]
template <int N_OUT, int kMaxChunks, bool SMOOTH>
__global__ void __launch_bounds__(256)
head_bwd_kernel(int64_t M, int K, const __nv_bfloat16* __restrict__ x, int64_t ldx,
                const __nv_bfloat16* __restrict__ w, const float* __restrict__ draw,
                __nv_bfloat16* __restrict__ dx, int64_t lddx, int relu_mask,
                float* __restrict__ dw, float* __restrict__ dw2, int dw_split, float* __restrict__ db,
                float* __restrict__ dxsum, int dx_cols, __nv_bfloat16* __restrict__ dx2, int64_t lddx2,
                int64_t rows_per_block, int act, const __nv_bfloat16* __restrict__ z, int64_t ldz) {
  extern __shared__ __align__(16) unsigned char smraw[];
  constexpr int n_out = N_OUT;
  float* sdw = reinterpret_cast<float*>(smraw);                                   // [n_out][K] fp32
  __nv_bfloat16* sw = reinterpret_cast<__nv_bfloat16*>(sdw + (size_t)n_out * K);  // [n_out][K]
  for (int i = threadIdx.x; i < n_out * K; i += blockDim.x) { sw[i] = w[i]; sdw[i] = 0.f; }
  __syncthreads();
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int64_t m_begin = (int64_t)blockIdx.x * rows_per_block;
  const int64_t m_end = min(M, m_begin + rows_per_block);
  // Each lane owns the 8-column chunks c = lane, lane+32, ...: it accumulates their dw in
  // registers across the rows of this warp and flushes once into shared memory.
  float racc[N_OUT][kMaxChunks][8];
#pragma unroll
  for (int o = 0; o < N_OUT; ++o)
#pragma unroll
    for (int q = 0; q < kMaxChunks; ++q)
#pragma unroll
      for (int e = 0; e < 8; ++e) racc[o][q][e] = 0.f;
  float dbacc[N_OUT];
#pragma unroll
  for (int o = 0; o < N_OUT; ++o) dbacc[o] = 0.f;
  float xsum[kMaxChunks][8];       // column sums of dx over this thread's rows
#pragma unroll
  for (int q = 0; q < kMaxChunks; ++q)
#pragma unroll
    for (int e = 0; e < 8; ++e) xsum[q][e] = 0.f;
  for (int64_t m = m_begin + wib; m < m_end; m += nw) {
    float g[N_OUT];
#pragma unroll
    for (int o = 0; o < N_OUT; ++o) g[o] = draw[m * n_out + o];
    const uint4* xr = reinterpret_cast<const uint4*>(x + m * ldx);
    uint4* dxr = dx ? reinterpret_cast<uint4*>(dx + m * lddx) : nullptr;
    __nv_bfloat16* dx2r = dx2 ? dx2 + m * lddx2 : nullptr;
#pragma unroll
    for (int q = 0; q < kMaxChunks; ++q) {
      int c = lane + 32 * q;
      if (c < K / 8) {
        uint4 v = xr[c];
        uint32_t vv[4] = {v.x, v.y, v.z, v.w};
        float xe[8], de[8];
#pragma unroll
        for (int p = 0; p < 4; ++p) { xe[2 * p] = bf16_lo(vv[p]); xe[2 * p + 1] = bf16_hi(vv[p]); }
#pragma unroll
        for (int e = 0; e < 8; ++e) de[e] = 0.f;
#pragma unroll
        for (int o = 0; o < N_OUT; ++o) {
          const uint4 wv = reinterpret_cast<const uint4*>(sw + (size_t)o * K)[c];
          uint32_t ww[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
          for (int p = 0; p < 4; ++p) {
            de[2 * p] += g[o] * bf16_lo(ww[p]);
            de[2 * p + 1] += g[o] * bf16_hi(ww[p]);
          }
#pragma unroll
          for (int e = 0; e < 8; ++e) racc[o][q][e] += g[o] * xe[e];
        }
        if (dxr && c * 8 < dx_cols) {
          if constexpr (SMOOTH) {
            const uint4 zv = *reinterpret_cast<const uint4*>(z + m * ldz + c * 8);
            const uint32_t zz[4] = {zv.x, zv.y, zv.z, zv.w};
#pragma unroll
            for (int p = 0; p < 4; ++p) {
              de[2 * p] *= act_d1(act, bf16_lo(zz[p]));
              de[2 * p + 1] *= act_d1(act, bf16_hi(zz[p]));
            }
          } else if (relu_mask) {
#pragma unroll
            for (int e = 0; e < 8; ++e) de[e] = xe[e] > 0.f ? de[e] : 0.f;
          }
#pragma unroll
          for (int e = 0; e < 8; ++e) xsum[q][e] += de[e];
          uint4 o4;
          o4.x = pack_bf16(de[0], de[1]); o4.y = pack_bf16(de[2], de[3]);
          o4.z = pack_bf16(de[4], de[5]); o4.w = pack_bf16(de[6], de[7]);
          dxr[c] = o4;
        } else if (dx2r && c * 8 >= dx_cols) {
          // columns past dx_cols: unmasked, not summed (the input tail a skip concatenation appended)
          uint4 o4;
          o4.x = pack_bf16(de[0], de[1]); o4.y = pack_bf16(de[2], de[3]);
          o4.z = pack_bf16(de[4], de[5]); o4.w = pack_bf16(de[6], de[7]);
          reinterpret_cast<uint4*>(dx2r + (c * 8 - dx_cols))[0] = o4;
        }
      }
    }
    if (lane == 0) {
#pragma unroll
      for (int o = 0; o < N_OUT; ++o) dbacc[o] += g[o];
    }
  }
#pragma unroll
  for (int o = 0; o < N_OUT; ++o) {
#pragma unroll
    for (int q = 0; q < kMaxChunks; ++q) {
      int c = lane + 32 * q;
      if (c < K / 8) {
#pragma unroll
        for (int e = 0; e < 8; ++e) atomicAdd(&sdw[(size_t)o * K + c * 8 + e], racc[o][q][e]);
      }
    }
    if (lane == 0 && db && dbacc[o] != 0.f) atomicAdd(&db[o], dbacc[o]);
  }
  if (dxsum) {
    // reuse the dw staging buffer's first K floats once dw has been flushed
    __syncthreads();
    if (dw) for (int i = threadIdx.x; i < n_out * K; i += blockDim.x) {
      int o = i / K, k = i - o * K;
      atomicAdd(dw_at(dw, dw2, dw_split, n_out, k, o), sdw[i]);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < K; i += blockDim.x) sdw[i] = 0.f;
    __syncthreads();
#pragma unroll
    for (int q = 0; q < kMaxChunks; ++q) {
      int c = lane + 32 * q;
      if (c < K / 8) {
#pragma unroll
        for (int e = 0; e < 8; ++e) atomicAdd(&sdw[c * 8 + e], xsum[q][e]);
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < dx_cols; i += blockDim.x) atomicAdd(&dxsum[i], sdw[i]);
    return;
  }
  __syncthreads();
  // dw is in the master layout [K, n_out] (row-major), the staging buffer is [n_out][K]
  if (dw) for (int i = threadIdx.x; i < n_out * K; i += blockDim.x) {
    int o = i / K, k = i - o * K;
    atomicAdd(dw_at(dw, dw2, dw_split, n_out, k, o), sdw[i]);
  }
}

// Narrow inputs (K = 64 or 128: the rgb head on the view MLP's output): a row is only LPR = K/8 sixteen-byte chunks,
// so a warp-per-row mapping leaves half (or three quarters) of the lanes idle and one load in flight per warp.  Here
// a warp covers 32/LPR rows per pass and U passes per iteration (U independent 16-byte loads per lane in flight);
// row sums are butterfly reductions over the LPR lanes of a row (the same additions, in the same order, as the
// full-warp butterfly of head_fwd_kernel with its idle lanes contributing zeros).
template <int LPR, int U>
__global__ void __launch_bounds__(256)
head_fwd_sub_kernel(int64_t M, int n_out, const __nv_bfloat16* __restrict__ x, int64_t ldx,
                    const __nv_bfloat16* __restrict__ w, const float* __restrict__ b, float* __restrict__ raw) {
  constexpr int K = LPR * 8, RW = 32 / LPR;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int sub = lane / LPR, c = lane % LPR;
  float wv[kMaxHead][8];
#pragma unroll
  for (int o = 0; o < kMaxHead; ++o) {
    uint4 t = make_uint4(0u, 0u, 0u, 0u);
    if (o < n_out) t = __ldg(reinterpret_cast<const uint4*>(w + (size_t)o * K) + c);
    const uint32_t tt[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) { wv[o][2 * q] = bf16_lo(tt[q]); wv[o][2 * q + 1] = bf16_hi(tt[q]); }
  }
  float bv[kMaxHead];
#pragma unroll
  for (int o = 0; o < kMaxHead; ++o) bv[o] = (b && o < n_out) ? __ldg(b + o) : 0.f;
  const int64_t step = (int64_t)gridDim.x * nw * (RW * U);
  for (int64_t m0 = ((int64_t)blockIdx.x * nw + wib) * (RW * U); m0 < M; m0 += step) {
    uint4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t row = m0 + u * RW + sub;
      v[u] = row < M ? __ldg(reinterpret_cast<const uint4*>(x + row * ldx) + c) : make_uint4(0u, 0u, 0u, 0u);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t row = m0 + u * RW + sub;
      const uint32_t vv[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
      for (int o = 0; o < kMaxHead; ++o) {
        if (o < n_out) {
          float acc = 0.f;
#pragma unroll
          for (int q = 0; q < 4; ++q) acc += bf16_lo(vv[q]) * wv[o][2 * q] + bf16_hi(vv[q]) * wv[o][2 * q + 1];
#pragma unroll
          for (int sh = LPR / 2; sh > 0; sh >>= 1) acc += __shfl_xor_sync(kFull, acc, sh);
          if (c == 0 && row < M) raw[row * n_out + o] = acc + bv[o];
        }
      }
    }
  }
}

template <int N_OUT, int LPR, int U, bool SMOOTH>
__global__ void __launch_bounds__(256)
head_bwd_sub_kernel(int64_t M, const __nv_bfloat16* __restrict__ x, int64_t ldx,
                    const __nv_bfloat16* __restrict__ w, const float* __restrict__ draw,
                    __nv_bfloat16* __restrict__ dx, int64_t lddx, int relu_mask,
                    float* __restrict__ dw, float* __restrict__ dw2, int dw_split, float* __restrict__ db,
                    float* __restrict__ dxsum, int dx_cols, __nv_bfloat16* __restrict__ dx2, int64_t lddx2,
                    int64_t rows_per_block, int act, const __nv_bfloat16* __restrict__ z, int64_t ldz) {
  constexpr int K = LPR * 8, RW = 32 / LPR;
  __shared__ float sdw[N_OUT * K];
  __shared__ float sxs[K];
  for (int i = threadIdx.x; i < N_OUT * K; i += blockDim.x) sdw[i] = 0.f;
  for (int i = threadIdx.x; i < K; i += blockDim.x) sxs[i] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int sub = lane / LPR, c = lane % LPR;
  float wv[N_OUT][8];
#pragma unroll
  for (int o = 0; o < N_OUT; ++o) {
    const uint4 t = __ldg(reinterpret_cast<const uint4*>(w + (size_t)o * K) + c);
    const uint32_t tt[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) { wv[o][2 * q] = bf16_lo(tt[q]); wv[o][2 * q + 1] = bf16_hi(tt[q]); }
  }
  float racc[N_OUT][8], dbacc[N_OUT], xsum[8];
#pragma unroll
  for (int o = 0; o < N_OUT; ++o) {
    dbacc[o] = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) racc[o][e] = 0.f;
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) xsum[e] = 0.f;
  const int64_t m_begin = (int64_t)blockIdx.x * rows_per_block;
  const int64_t m_end = min(M, m_begin + rows_per_block);
  for (int64_t m0 = m_begin + (int64_t)wib * (RW * U); m0 < m_end; m0 += (int64_t)nw * (RW * U)) {
    uint4 v[U];
    float g[U][N_OUT];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t row = m0 + u * RW + sub;
      const bool ok = row < m_end;
      v[u] = ok ? __ldg(reinterpret_cast<const uint4*>(x + row * ldx) + c) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
      for (int o = 0; o < N_OUT; ++o) g[u][o] = ok ? __ldg(draw + row * N_OUT + o) : 0.f;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t row = m0 + u * RW + sub;
      const uint32_t vv[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
      float xe[8], de[8];
#pragma unroll
      for (int q = 0; q < 4; ++q) { xe[2 * q] = bf16_lo(vv[q]); xe[2 * q + 1] = bf16_hi(vv[q]); }
#pragma unroll
      for (int e = 0; e < 8; ++e) de[e] = 0.f;
#pragma unroll
      for (int o = 0; o < N_OUT; ++o) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          de[e] += g[u][o] * wv[o][e];
          racc[o][e] += g[u][o] * xe[e];
        }
        if (c == 0) dbacc[o] += g[u][o];
      }
      if (dx && row < m_end && c * 8 < dx_cols) {
        if constexpr (SMOOTH) {
          const uint4 zv = __ldg(reinterpret_cast<const uint4*>(z + row * ldz) + c);
          const uint32_t zz[4] = {zv.x, zv.y, zv.z, zv.w};
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            de[2 * q] *= act_d1(act, bf16_lo(zz[q]));
            de[2 * q + 1] *= act_d1(act, bf16_hi(zz[q]));
          }
        } else if (relu_mask) {
#pragma unroll
          for (int e = 0; e < 8; ++e) de[e] = xe[e] > 0.f ? de[e] : 0.f;
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) xsum[e] += de[e];
        uint4 o4;
        o4.x = pack_bf16(de[0], de[1]); o4.y = pack_bf16(de[2], de[3]);
        o4.z = pack_bf16(de[4], de[5]); o4.w = pack_bf16(de[6], de[7]);
        reinterpret_cast<uint4*>(dx + row * lddx)[c] = o4;
      } else if (dx2 && row < m_end && c * 8 >= dx_cols) {
        uint4 o4;
        o4.x = pack_bf16(de[0], de[1]); o4.y = pack_bf16(de[2], de[3]);
        o4.z = pack_bf16(de[4], de[5]); o4.w = pack_bf16(de[6], de[7]);
        reinterpret_cast<uint4*>(dx2 + row * lddx2 + (c * 8 - dx_cols))[0] = o4;
      }
    }
  }
#pragma unroll
  for (int o = 0; o < N_OUT; ++o) {
#pragma unroll
    for (int e = 0; e < 8; ++e) atomicAdd(&sdw[o * K + c * 8 + e], racc[o][e]);
    if (c == 0 && db && dbacc[o] != 0.f) atomicAdd(&db[o], dbacc[o]);
  }
  if (dxsum) {
#pragma unroll
    for (int e = 0; e < 8; ++e) atomicAdd(&sxs[c * 8 + e], xsum[e]);
  }
  __syncthreads();
  // dw is in the master layout [K, n_out] (row-major), the staging buffer is [n_out][K]
  if (dw) for (int i = threadIdx.x; i < N_OUT * K; i += blockDim.x) {
    const int o = i / K, k = i - o * K;
    atomicAdd(dw_at(dw, dw2, dw_split, N_OUT, k, o), sdw[i]);
  }
  if (dxsum) for (int i = threadIdx.x; i < dx_cols; i += blockDim.x) atomicAdd(&dxsum[i], sxs[i]);
}

// out[n] += sum_m x[m, n]
__global__ void __launch_bounds__(256)
colsum_kernel(int64_t M, int N, const __nv_bfloat16* __restrict__ x, int64_t ldx,
              float* __restrict__ out, int64_t rows_per_block) {
  // thread t owns columns [8t, 8t+8) (16-byte loads); blockDim.x * 8 >= N is enforced by the
  // launcher through a 2-D grid over column slabs.
  const int col = (blockIdx.y * blockDim.x + threadIdx.x) * 8;
  if (col >= N) return;
  const int64_t m0 = (int64_t)blockIdx.x * rows_per_block, m1 = min(M, m0 + rows_per_block);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const __nv_bfloat16* base = x + col;
  int64_t m = m0;
  constexpr int U = 8;                     // independent 16-byte loads in flight per thread
  for (; m + U <= m1; m += U) {
    uint4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) v[u] = __ldg(reinterpret_cast<const uint4*>(base + (m + u) * ldx));
#pragma unroll
    for (int u = 0; u < U; ++u) {
      uint32_t vv[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
      for (int p = 0; p < 4; ++p) { acc[2 * p] += bf16_lo(vv[p]); acc[2 * p + 1] += bf16_hi(vv[p]); }
    }
  }
  for (; m < m1; ++m) {
    uint4 v = __ldg(reinterpret_cast<const uint4*>(base + m * ldx));
    uint32_t vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int p = 0; p < 4; ++p) { acc[2 * p] += bf16_lo(vv[p]); acc[2 * p + 1] += bf16_hi(vv[p]); }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) atomicAdd(&out[col + e], acc[e]);
}

// One launch for every layer: blockIdx.x is a global tile number, the owning layer is found by a
// binary search over the items' first tiles.
__global__ void pack_weights_batched_kernel(int count, const mnrf_pack_item* __restrict__ items) {
  __shared__ float tile[32][33];
  int lo = 0, hi = count - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (items[mid].tile0 <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const mnrf_pack_item it = items[lo];
  const int tiles_n = (it.out + 31) / 32;
  const int t = blockIdx.x - it.tile0;
  const int k0 = (t / tiles_n) * 32, n0 = (t % tiles_n) * 32;
  const int in_pad = it.in_pad, out = it.out;
  __nv_bfloat16* w_nk = reinterpret_cast<__nv_bfloat16*>(it.w_nk);
  __nv_bfloat16* w_kn = reinterpret_cast<__nv_bfloat16*>(it.w_kn);
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    int k = k0 + r, n = n0 + threadIdx.x;
    float v = (k < in_pad && n < out) ? it.master[(size_t)k * out + n] : 0.f;
    tile[r][threadIdx.x] = v;
    if (w_kn && k < in_pad && n < out) w_kn[(size_t)k * out + n] = __float2bfloat16(v);
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    int n = n0 + r, k = k0 + threadIdx.x;
    if (w_nk && n < out && k < in_pad) w_nk[(size_t)n * in_pad + k] = __float2bfloat16(tile[threadIdx.x][r]);
  }
}

__global__ void __launch_bounds__(256)
grad_norm_kernel(int64_t n, const float* __restrict__ g, float scale, float max_val,
                 float* __restrict__ norm_sq) {
  float acc = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float v = g[i] * scale;
    // jnp.clip propagates NaN (fminf/fmaxf would drop it): a NaN anywhere makes the module norm NaN
    if (max_val > 0.f && v == v) v = fminf(fmaxf(v, -max_val), max_val);
    acc += v * v;
  }
  acc = warp_sum(acc);
  __shared__ float part[8];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? part[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) atomicAdd(norm_sq, v);
  }
}

__global__ void __launch_bounds__(256)
clip_adam_kernel(mnrf_adam_desc d, float* __restrict__ p, const float* __restrict__ g,
                 float* __restrict__ mu, float* __restrict__ nu, const float* __restrict__ norm_sq,
                 const float* __restrict__ dyn) {
  // train_utils.py:200-218 then :328: value clip, mult = min(1, max_norm / (eps + norm)), mult * g,
  // nan_to_num.  jnp.minimum / jnp.clip propagate NaN, so a NaN anywhere in the module makes mult NaN
  // and the whole module's update zero; an infinite norm gives mult = 0.
  float mult = 1.f;
  if (d.grad_max_norm > 0.f) {
    const float nrm = sqrtf(*norm_sq);
    mult = (nrm != nrm) ? nrm : fminf(1.f, d.grad_max_norm / (kEps + nrm));
  }
  float bc1 = 1.f - powf(d.beta1, (float)d.step);
  float bc2 = 1.f - powf(d.beta2, (float)d.step);
  if (dyn) { d.lr = dyn[0]; bc1 = dyn[1]; bc2 = dyn[2]; }
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < d.n; i += (int64_t)gridDim.x * blockDim.x) {
    float v = g[i] * d.grad_scale;
    if (d.grad_max_val > 0.f && v == v) v = fminf(fmaxf(v, -d.grad_max_val), d.grad_max_val);
    v *= mult;
    // jnp.nan_to_num: nan -> 0, +-inf -> +-max float
    if (isnan(v)) v = 0.f;
    else if (isinf(v)) v = v > 0.f ? 3.4028235e38f : -3.4028235e38f;
    float m = d.beta1 * mu[i] + (1.f - d.beta1) * v;
    float s = d.beta2 * nu[i] + (1.f - d.beta2) * v * v;
    mu[i] = m;
    nu[i] = s;
    float mh = m / bc1, sh = s / bc2;
    p[i] = p[i] - d.lr * mh / (sqrtf(sh) + d.eps);
  }
}

// The launch choices of mnrf_head_fwd / mnrf_head_bwd after their argument checks (mnrf_head_plan reports them).
static void head_fwd_plan(int64_t m, int k, mnrf_head_instance* p) {
  if (k == 256 || k == 128 || k == 64) {
    // rows of one / half / a quarter of a warp's 16-byte chunks: 4 independent loads in flight per lane
    p->fwd_kernel = MNRF_HEAD_FWD_SUB;
    p->fwd_lpr = k / 8;
    p->fwd_rows_per_pass = 8 * (256 / k) * 4;
  } else {
    p->fwd_kernel = MNRF_HEAD_FWD_WARP;
    p->fwd_lpr = 0;
    p->fwd_rows_per_pass = 8;
  }
  p->fwd_grid = (int)std::min<int64_t>((m + p->fwd_rows_per_pass - 1) / p->fwd_rows_per_pass,
                                       (int64_t)mnrf_num_sms() * 8);
}

static void head_bwd_plan(int64_t m, int k, int n_out, const mnrf_bf16* w, bool smooth, mnrf_head_instance* p) {
  p->bwd_n_out = n_out;
  p->bwd_smooth = smooth;
  if ((k == 256 || k == 128 || k == 64) && ((uintptr_t)w % 16) == 0) {
    // rows of one / half / a quarter of a warp's 16-byte chunks (see head_bwd_sub_kernel)
    // every block ends with n_out*K + K global atomics on the same addresses: two blocks per SM keep enough loads
    // in flight (8 warps x 4 x 512 B each) without serialising the flush
    p->bwd_kernel = MNRF_HEAD_BWD_SUB;
    p->bwd_lpr = k / 8;
    p->bwd_chunks = 0;
    p->bwd_grid = (int)std::min<int64_t>((m + 511) / 512, (int64_t)mnrf_num_sms() * 2);
    p->bwd_rows_per_block = ((m + p->bwd_grid - 1) / p->bwd_grid + 7) / 8 * 8;
    return;
  }
  const int chunks = (k / 8 + 31) / 32;
  p->bwd_kernel = MNRF_HEAD_BWD_WARP;
  p->bwd_lpr = 0;
  p->bwd_chunks = chunks <= 1 ? 1 : chunks <= 2 ? 2 : chunks <= 4 ? 4 : 6;
  p->bwd_grid = (int)std::min<int64_t>((m + 7) / 8, (int64_t)mnrf_num_sms() * 4);
  p->bwd_rows_per_block = (m + p->bwd_grid - 1) / p->bwd_grid;
}

// The checks of mnrf_head_bwd on the arguments mnrf_head_plan takes as well.
static int head_bwd_check(int k, int n_out, const mnrf_bf16* x, const mnrf_bf16* w, int act, const mnrf_bf16* z,
                          const mnrf_bf16* dx) {
  MNRF_CHECK(x && w, "mnrf_head_bwd: null pointer");
  MNRF_CHECK(n_out >= 1 && n_out <= kMaxHead, "mnrf_head_bwd: n_out %d not in [1,4]", n_out);
  MNRF_CHECK(k % 8 == 0 && k <= 1536, "mnrf_head_bwd: K must be a multiple of 8 and <= 1536");
  // both kernels read the rows of x, and write those of dx, in 16-byte chunks
  MNRF_CHECK(((uintptr_t)x % 16) == 0 && ((uintptr_t)dx % 16) == 0, "mnrf_head_bwd: x and dx must be 16-byte aligned");
  MNRF_CHECK(act >= MNRF_ACT_NONE && act <= MNRF_ACT_SILU, "mnrf_head_bwd: unknown act %d", act);
  const bool smooth = act == MNRF_ACT_SOFTPLUS || act == MNRF_ACT_SILU;
  MNRF_CHECK(smooth || !z, "mnrf_head_bwd: z is the pre-activation of a smooth activation, act %d is not one", act);
  MNRF_CHECK(!smooth || (z && dx && ((uintptr_t)z % 16) == 0),
             "mnrf_head_bwd: a smooth activation needs dx and a 16-byte aligned z");
  return 0;
}

}  // namespace mnrf

extern "C" int mnrf_head_fwd(int64_t m, int32_t k, int32_t n_out, const mnrf_bf16* x, int64_t ldx,
                             const mnrf_bf16* w, const float* b, float* raw, mnrf_stream stream) {
  using namespace mnrf;
  if (m == 0) return 0;
  MNRF_CHECK(x && w && raw, "mnrf_head_fwd: null pointer");
  MNRF_CHECK(n_out >= 1 && n_out <= kMaxHead, "mnrf_head_fwd: n_out %d not in [1,4]", n_out);
  MNRF_CHECK(k % 8 == 0 && ldx % 8 == 0 && ((uintptr_t)x % 16) == 0 && ((uintptr_t)w % 16) == 0,
             "mnrf_head_fwd: K/ld must be multiples of 8 and pointers 16-byte aligned");
  mnrf_head_instance p = {};
  head_fwd_plan(m, k, &p);
  if (p.fwd_kernel == MNRF_HEAD_FWD_SUB) {
#define MNRF_HFS(LPR_)                                                                                 \
  head_fwd_sub_kernel<LPR_, 4><<<p.fwd_grid, 256, 0, (cudaStream_t)stream>>>(                           \
      m, n_out, reinterpret_cast<const __nv_bfloat16*>(x), ldx, reinterpret_cast<const __nv_bfloat16*>(w), b, raw)
    if (p.fwd_lpr == 32) MNRF_HFS(32); else if (p.fwd_lpr == 16) MNRF_HFS(16); else MNRF_HFS(8);
    MNRF_LAUNCH_CHECK();
    return 0;
  }
  size_t smem = (size_t)n_out * k * 2;
  head_fwd_kernel<<<p.fwd_grid, 256, smem, (cudaStream_t)stream>>>(
      m, k, n_out, reinterpret_cast<const __nv_bfloat16*>(x), ldx,
      reinterpret_cast<const __nv_bfloat16*>(w), b, raw);
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_head_bwd(int64_t m, int32_t k, int32_t n_out, const mnrf_bf16* x, int64_t ldx,
                             const mnrf_bf16* w, const float* draw, mnrf_bf16* dx, int64_t lddx, int32_t act,
                             const mnrf_bf16* z_, int64_t ldz, float* dw, float* dw2, int32_t dw_split, float* db,
                             float* dxsum, int32_t dx_cols, mnrf_bf16* dx2, int64_t lddx2, mnrf_stream stream) {
  using namespace mnrf;
  const __nv_bfloat16* z = reinterpret_cast<const __nv_bfloat16*>(z_);
  if (m == 0) return 0;
  MNRF_CHECK(draw, "mnrf_head_bwd: null pointer");
  if (int rc = head_bwd_check(k, n_out, x, w, act, z_, dx)) return rc;
  MNRF_CHECK(!dxsum || dx, "mnrf_head_bwd: dxsum needs dx");
  MNRF_CHECK(ldx % 8 == 0 && (!dx || lddx % 8 == 0), "mnrf_head_bwd: the pitches of x and dx must be multiples of 8");
  if (dw_split <= 0 || dw_split >= n_out) dw_split = n_out;
  if (dx_cols <= 0) dx_cols = k;
  MNRF_CHECK(dx_cols <= k && dx_cols % 8 == 0, "mnrf_head_bwd: dx_cols must be a multiple of 8 and <= K");
  MNRF_CHECK(!dx2 || (dx_cols < k && lddx2 % 8 == 0 && ((uintptr_t)dx2 % 16) == 0),
             "mnrf_head_bwd: dx2 needs dx_cols < K, a pitch that is a multiple of 8 and a 16-byte aligned pointer");
  MNRF_CHECK(dw_split == n_out || (dw && dw2), "mnrf_head_bwd: a split weight gradient needs dw and dw2");
  const bool smooth = act == MNRF_ACT_SOFTPLUS || act == MNRF_ACT_SILU;
  MNRF_CHECK(!smooth || ldz % 8 == 0, "mnrf_head_bwd: the pitch of z must be a multiple of 8");
  // the kernels take the ReLU mask as a flag of its own and `act` for the smooth derivative only
  const int32_t relu_mask = act == MNRF_ACT_RELU;
  if (!smooth) act = MNRF_ACT_NONE;
  mnrf_head_instance p = {};
  head_bwd_plan(m, k, n_out, w, smooth, &p);
  const int64_t rpb = p.bwd_rows_per_block;
  if (p.bwd_kernel == MNRF_HEAD_BWD_SUB) {
#define MNRF_HBS2(NO, LPR_, SM_)                                                                        \
  head_bwd_sub_kernel<NO, LPR_, 4, SM_><<<p.bwd_grid, 256, 0, (cudaStream_t)stream>>>(                  \
      m, reinterpret_cast<const __nv_bfloat16*>(x), ldx, reinterpret_cast<const __nv_bfloat16*>(w), draw, \
      reinterpret_cast<__nv_bfloat16*>(dx), lddx, relu_mask, dw, dw2, dw_split, db, dxsum, dx_cols,      \
      reinterpret_cast<__nv_bfloat16*>(dx2), lddx2, rpb, act, z, ldz)
#define MNRF_HBS(NO, LPR_) do { if (p.bwd_smooth) MNRF_HBS2(NO, LPR_, true); else MNRF_HBS2(NO, LPR_, false); } while (0)
#define MNRF_HBS_N(NO) do { if (p.bwd_lpr == 32) MNRF_HBS(NO, 32); else if (p.bwd_lpr == 16) MNRF_HBS(NO, 16); else MNRF_HBS(NO, 8); } while (0)
    switch (p.bwd_n_out) {
      case 1: MNRF_HBS_N(1); break;
      case 2: MNRF_HBS_N(2); break;
      case 3: MNRF_HBS_N(3); break;
      default: MNRF_HBS_N(4); break;
    }
    MNRF_LAUNCH_CHECK();
    return 0;
  }
  size_t smem = (size_t)n_out * k * (4 + 2);
  MNRF_CHECK(smem <= 48 * 1024, "mnrf_head_bwd: n_out*K too large for the shared-memory staging");
#define MNRF_HB2(NO, CK, SM_)                                                                   \
  head_bwd_kernel<NO, CK, SM_><<<p.bwd_grid, 256, smem, (cudaStream_t)stream>>>(                \
      m, k, reinterpret_cast<const __nv_bfloat16*>(x), ldx, reinterpret_cast<const __nv_bfloat16*>(w), \
      draw, reinterpret_cast<__nv_bfloat16*>(dx), lddx, relu_mask, dw, dw2, dw_split, db, dxsum, dx_cols, \
      reinterpret_cast<__nv_bfloat16*>(dx2), lddx2, rpb, act, z, ldz)
#define MNRF_HB(NO, CK) do { if (p.bwd_smooth) MNRF_HB2(NO, CK, true); else MNRF_HB2(NO, CK, false); } while (0)
#define MNRF_HB_N(NO)                                      \
  do {                                                     \
    if (p.bwd_chunks == 1) MNRF_HB(NO, 1);                 \
    else if (p.bwd_chunks == 2) MNRF_HB(NO, 2);            \
    else if (p.bwd_chunks == 4) MNRF_HB(NO, 4);            \
    else MNRF_HB(NO, 6);                                   \
  } while (0)
  switch (p.bwd_n_out) {
    case 1: MNRF_HB_N(1); break;
    case 2: MNRF_HB_N(2); break;
    case 3: MNRF_HB_N(3); break;
    default: MNRF_HB_N(4); break;
  }
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_head_plan(int64_t m, int32_t k, int32_t n_out, const mnrf_bf16* x, const mnrf_bf16* w,
                              int32_t act, const mnrf_bf16* z, const mnrf_bf16* dx, mnrf_head_instance* plan) {
  using namespace mnrf;
  MNRF_CHECK(plan, "mnrf_head_plan: null pointer");
  MNRF_CHECK(m > 0, "mnrf_head_plan: m must be positive (an empty launch runs no kernel)");
  if (int rc = head_bwd_check(k, n_out, x, w, act, z, dx)) return rc;
  *plan = mnrf_head_instance{};
  if (((uintptr_t)w % 16) == 0) head_fwd_plan(m, k, plan);
  head_bwd_plan(m, k, n_out, w, act == MNRF_ACT_SOFTPLUS || act == MNRF_ACT_SILU, plan);
  return 0;
}

extern "C" int mnrf_colsum(int64_t m, int32_t n, const mnrf_bf16* x, int64_t ldx, float* out,
                           mnrf_stream stream) {
  using namespace mnrf;
  if (m == 0) return 0;
  MNRF_CHECK(x && out, "mnrf_colsum: null pointer");
  MNRF_CHECK(n % 8 == 0 && ldx % 8 == 0 && ((uintptr_t)x % 16) == 0,
             "mnrf_colsum: N and ld must be multiples of 8 and x 16-byte aligned");
  const int threads = 128;
  dim3 grid;
  grid.y = (n / 8 + threads - 1) / threads;
  int bx = std::max(1, mnrf_num_sms() * 16 / (int)grid.y);
  bx = (int)std::min<int64_t>(bx, (m + 63) / 64);
  grid.x = bx;
  int64_t rpb = (m + bx - 1) / bx;
  colsum_kernel<<<grid, threads, 0, (cudaStream_t)stream>>>(
      m, n, reinterpret_cast<const __nv_bfloat16*>(x), ldx, out, rpb);
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_pack_weights_batched(int32_t count, const mnrf_pack_item* items, int32_t total_tiles,
                                         mnrf_stream stream) {
  using namespace mnrf;
  if (count == 0 || total_tiles == 0) return 0;
  MNRF_CHECK(items && count > 0 && total_tiles > 0, "mnrf_pack_weights_batched: null item table");
  pack_weights_batched_kernel<<<total_tiles, dim3(32, 8), 0, (cudaStream_t)stream>>>(count, items);
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_clip_adam(const mnrf_adam_desc* d, float* params, const float* grads, float* mu,
                              float* nu, float* norm_sq_scratch, const float* dyn, mnrf_stream stream) {
  using namespace mnrf;
  MNRF_CHECK(d && params && grads && mu && nu && norm_sq_scratch, "mnrf_clip_adam: null pointer");
  MNRF_CHECK(d->step >= 1, "mnrf_clip_adam: step is the 1-based update count");
  if (d->n == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  int blocks = (int)std::min<int64_t>((d->n + 255) / 256, (int64_t)mnrf_num_sms() * 8);
  MNRF_CUDA(cudaMemsetAsync(norm_sq_scratch, 0, sizeof(float), s));
  if (d->grad_max_norm > 0.f) {
    grad_norm_kernel<<<blocks, 256, 0, s>>>(d->n, grads, d->grad_scale, d->grad_max_val, norm_sq_scratch);
    MNRF_LAUNCH_CHECK();
  }
  clip_adam_kernel<<<blocks, 256, 0, s>>>(*d, params, grads, mu, nu, norm_sq_scratch, dyn);
  MNRF_LAUNCH_CHECK();
  return 0;
}
