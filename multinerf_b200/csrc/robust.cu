// RobustNeRF (robustnerf.py:8-115): the per-patch outlier mask of data_loss_type 'robustnerf', and the
// exact linear-interpolated quantile of the per-pixel errors that becomes the next step's inlier threshold.
//
// Mask: one CTA per patch, one thread per pixel (rays are patch-major [patch, y, x]).  The inlier bits live
// in shared memory for the f x f box filter (separable, zero padding at the patch border) and the patch
// counts come from __syncthreads_count.  Every comparison the reference makes on a mean of 0/1 values is
// made on fl32(count / size), which is what a float32 sum of 0/1 values (exact below 2^24) divided by the
// size rounds to.  The box filter's reference is a convolution with weights fl32(1/f^2); its sum of k such
// weights may land one ulp away from fl32(k/f^2), so when 1 - smoothed_inlier_quantile is exactly
// representable as k/f^2 (e.g. f = 5 and q = 0.8: 5/25) the two can disagree on ">" for that k.  The
// kernel's rule is fl32(k/f^2) > fl32(1 - q), i.e. such a tie is NOT an inlier neighbourhood.
//
// Quantile: one CTA, radix select over the order-preserving uint32 image of the floats (four 8-bit digit
// passes find the lo-th smallest, one more pass the next larger value), then jnp.quantile's 'linear'
// formula in fp32.  Any NaN in the input gives NaN.
#include "common.cuh"

namespace mnrf {

constexpr int kMaxPatchPixels = 1024;

__global__ void __launch_bounds__(1024)
robust_mask_kernel(mnrf_robust_desc d, const float* __restrict__ rgb, const float* __restrict__ target,
                   const float* __restrict__ threshold, float* __restrict__ mask, float* __restrict__ err_out,
                   uint32_t* __restrict__ counts, float* __restrict__ stats, int batch_rays) {
  __shared__ uint8_t inl[kMaxPatchPixels];
  __shared__ uint16_t rowcnt[kMaxPatchPixels];
  const int p = d.patch_size, pp = p * p;
  const int t = threadIdx.x;
  const bool live = t < pp;
  const int y = live ? t / p : 0, x = live ? t - y * p : 0;
  const int64_t ray = (int64_t)blockIdx.x * pp + t;
  const float thr = *threshold;

  // error_per_pixel = mean(resid_sq, -1): ((r0 + r1) + r2) / 3, each step rounded (no contraction)
  float e = 0.f;
  if (live) {
    float r[3];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const float dv = __fsub_rn(rgb[ray * 3 + ch], target[ray * 3 + ch]);
      r[ch] = __fmul_rn(dv, dv);
    }
    e = __fdiv_rn(__fadd_rn(__fadd_rn(r[0], r[1]), r[2]), 3.0f);
    err_out[ray] = e;
  }
  const int is_inl = live && (e < thr);

  int nb = 0, pix = 0, in_patch = 0, m = 1;
  if (d.enable) {
    inl[t] = (uint8_t)is_inl;
    __syncthreads();
    const int h = d.filter_size / 2;
    if (live) {
      int c = 0;
      for (int dx = -h; dx <= h; ++dx) {
        const int xx = x + dx;
        if (xx >= 0 && xx < p) c += inl[y * p + xx];
      }
      rowcnt[t] = (uint16_t)c;
    }
    __syncthreads();
    if (live) {
      int c = 0;
      for (int dy = -h; dy <= h; ++dy) {
        const int yy = y + dy;
        if (yy >= 0 && yy < p) c += rowcnt[yy * p + x];
      }
      nb = __fdiv_rn((float)c, (float)(d.filter_size * d.filter_size)) > d.smoothed_thresh;
      pix = nb || is_inl;
    }
    const int patch_cnt = __syncthreads_count(pix);
    const bool patch_ok = __fdiv_rn((float)patch_cnt, (float)pp) > d.patch_thresh;
    const int lo = (p - d.inner_patch_size) / 2;
    const bool inner = live && y >= lo && y < lo + d.inner_patch_size && x >= lo && x < lo + d.inner_patch_size;
    in_patch = patch_ok && inner;
    m = in_patch || pix;
  }
  if (live) mask[ray] = m ? 1.f : 0.f;

  if (stats == nullptr) return;
  // per-rank means of is_inlier_loss, has_inlier_neighbors, is_inlier_patch, mask: exact integer counts,
  // then the last CTA divides once by the batch's ray count and leaves the counters zeroed for the next launch
  const int c0 = __syncthreads_count(is_inl), c1 = __syncthreads_count(nb);
  const int c2 = __syncthreads_count(in_patch), c3 = __syncthreads_count(live && m);
  if (t == 0) {
    atomicAdd(&counts[0], (uint32_t)c0);
    atomicAdd(&counts[1], (uint32_t)c1);
    atomicAdd(&counts[2], (uint32_t)c2);
    atomicAdd(&counts[3], (uint32_t)c3);
    __threadfence();
    const uint32_t ticket = atomicAdd(&counts[4], 1u);
    if (ticket == gridDim.x - 1) {
      __threadfence();
      const float n = (float)batch_rays;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t c = atomicExch(&counts[k], 0u);
        if (d.enable || k == 3) stats[1 + k] += __fdiv_rn((float)c, n);
      }
      atomicExch(&counts[4], 0u);
    }
  }
}

__device__ __forceinline__ uint32_t float_key(float v) {
  const uint32_t u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_float(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

constexpr int kQThreads = 1024;

__global__ void __launch_bounds__(kQThreads)
quantile_kernel(int n, float q, const float* __restrict__ x, float* __restrict__ out) {
  __shared__ uint32_t hist[256];
  __shared__ uint32_t s_prefix, s_rank, s_less, s_bin_cnt;
  const int t = threadIdx.x;
  // jnp.quantile 'linear': n and q in fp32, qn = q * (n - 1), lo = floor, hi = ceil, w = qn - lo
  const float qn = __fmul_rn(q, __fsub_rn((float)n, 1.f));
  const float flo = floorf(qn), fhi = ceilf(qn);
  const float w = __fsub_rn(qn, flo);
  const int lo = min(max((int)flo, 0), n - 1), hi = min(max((int)fhi, 0), n - 1);

  if (t == 0) { s_prefix = 0; s_rank = (uint32_t)lo; s_less = 0; }
  int has_nan = 0;
  uint32_t mask_hi = 0;             // bits of the key fixed by the passes so far
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    for (int i = t; i < 256; i += kQThreads) hist[i] = 0;
    __syncthreads();
    const uint32_t prefix = s_prefix;
    for (int i = t; i < n; i += kQThreads) {
      const float v = x[i];
      if (pass == 0 && isnan(v)) has_nan = 1;
      const uint32_t k = float_key(v);
      if ((k & mask_hi) == prefix) atomicAdd(&hist[(k >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (t == 0) {
      // the bin that holds rank s_rank among the elements matching the prefix
      uint32_t r = s_rank, acc = 0;
      int b = 0;
      for (; b < 255; ++b) {
        if (acc + hist[b] > r) break;
        acc += hist[b];
      }
      s_rank = r - acc;
      s_less += acc;
      s_bin_cnt = hist[b];
      s_prefix = prefix | ((uint32_t)b << shift);
    }
    mask_hi |= 255u << shift;
    __syncthreads();
  }
  if (__syncthreads_or(has_nan)) {
    if (t == 0) *out = NAN;
    return;
  }
  const uint32_t key_lo = s_prefix;
  // elements equal to x[lo] occupy ranks [s_less, s_less + s_bin_cnt): x[hi] is x[lo] unless hi is past them
  const bool need_next = hi != lo && (uint32_t)hi >= s_less + s_bin_cnt;
  uint32_t next = 0xffffffffu;
  if (need_next) {
    for (int i = t; i < n; i += kQThreads) {
      const uint32_t k = float_key(x[i]);
      if (k > key_lo && k < next) next = k;
    }
    __shared__ uint32_t s_min;
    if (t == 0) s_min = 0xffffffffu;
    __syncthreads();
    for (int o = 16; o > 0; o >>= 1) next = min(next, __shfl_xor_sync(kFull, next, o));
    if ((t & 31) == 0) atomicMin(&s_min, next);
    __syncthreads();
    next = s_min;
  }
  if (t == 0) {
    const float vlo = key_float(key_lo);
    const float vhi = need_next ? key_float(next) : vlo;
    *out = __fadd_rn(__fmul_rn(vlo, __fsub_rn(1.f, w)), __fmul_rn(vhi, w));
  }
}

}  // namespace mnrf

extern "C" int mnrf_robust_mask(const mnrf_robust_desc* d, const float* rgb, const float* target,
                                const float* threshold, float* mask, float* error_per_pixel, uint32_t* counts,
                                float* stats, int32_t batch_rays, mnrf_stream stream) {
  using namespace mnrf;
  MNRF_CHECK(d && rgb && target && threshold && mask && error_per_pixel, "mnrf_robust_mask: null pointer");
  MNRF_CHECK(!stats || counts, "mnrf_robust_mask: stats need the counts workspace");
  const int p = d->patch_size;
  MNRF_CHECK(p >= 1 && p * p <= kMaxPatchPixels, "mnrf_robust_mask: patch_size %d (need p*p <= %d)", p,
             kMaxPatchPixels);
  MNRF_CHECK(d->num_rays >= 0 && d->num_rays % (p * p) == 0,
             "mnrf_robust_mask: num_rays %d is not a multiple of patch_size^2 = %d", d->num_rays, p * p);
  if (d->enable) {
    MNRF_CHECK(d->inner_patch_size >= 0 && d->inner_patch_size <= p,
               "mnrf_robust_mask: inner_patch_size %d > patch_size %d", d->inner_patch_size, p);
    MNRF_CHECK(d->filter_size >= 1 && d->filter_size % 2 == 1 && d->filter_size <= p,
               "mnrf_robust_mask: filter_size %d must be odd and <= patch_size %d", d->filter_size, p);
  }
  MNRF_CHECK(batch_rays >= d->num_rays, "mnrf_robust_mask: batch_rays %d < num_rays %d", batch_rays,
             d->num_rays);
  if (d->num_rays == 0) return 0;
  const int threads = (p * p + 31) / 32 * 32;
  robust_mask_kernel<<<d->num_rays / (p * p), threads, 0, (cudaStream_t)stream>>>(
      *d, rgb, target, threshold, mask, error_per_pixel, counts, stats, batch_rays);
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_quantile(int32_t n, float q, const float* x, float* out, mnrf_stream stream) {
  using namespace mnrf;
  MNRF_CHECK(x && out, "mnrf_quantile: null pointer");
  MNRF_CHECK(n >= 1 && n < (1 << 24), "mnrf_quantile: n = %d (need 1 <= n < 2^24)", n);
  MNRF_CHECK(q >= 0.f && q <= 1.f, "mnrf_quantile: q = %g outside [0, 1]", (double)q);
  quantile_kernel<<<1, kQThreads, 0, (cudaStream_t)stream>>>(n, q, x, out);
  MNRF_LAUNCH_CHECK();
  return 0;
}
