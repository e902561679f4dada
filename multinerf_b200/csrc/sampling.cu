// Hierarchical proposal resampling: one warp owns one ray.
//
// Replaces (reference file:line) stepfun.max_dilate_weights stepfun.py:116-128, the [1:-1]
// trim models.py:170-171, the annealed logits models.py:183-185 and
// stepfun.sample_intervals stepfun.py:214-263 (softmax -> integrate_weights -> sorted_interp
// math.py:108-127 -> midpoints with reflected, domain-clamped ends).
//
// HBM traffic per ray (level 1 of 360.gin): reads 65+64 floats, writes 65 floats (+64 int32
// when the index is requested) -- little next to the dependent binary searches and shuffle scans per ray, so the
// kernel is expected to be latency / issue bound rather than HBM-bound.
#include "common.cuh"

namespace mnrf {

// Number of elements of a sorted array `a[0..n)` that are <  x (lower) / <= x (upper).
__device__ __forceinline__ int count_lt(const float* a, int n, float x) {
  int lo = 0, hi = n;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (a[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}
__device__ __forceinline__ int count_le(const float* a, int n, float x) {
  int lo = 0, hi = n;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (a[mid] <= x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// Shared-memory plan per warp (floats):  t[P+1] t0[P] t1[P] p[P] | td[3P+1] wd[3P] cw[3P+1] c[S]
__global__ void __launch_bounds__(128)
sample_level_kernel(mnrf_sample_desc d, const float* __restrict__ sdist_prev,
                    const float* __restrict__ w_prev, const float* __restrict__ u_base,
                    const float* __restrict__ jitter, const float* __restrict__ cw_in,
                    float* __restrict__ sdist_out, int32_t* __restrict__ idx_out,
                    float* __restrict__ cw_out, float* __restrict__ tdil_out,
                    float* __restrict__ wdil_out, const float* __restrict__ anneal_dev) {
  extern __shared__ float smem[];
  if (anneal_dev) d.anneal = *anneal_dev;
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int P = d.num_prev, S = d.num_samples;
  const int nmax = 3 * P + 1;
  const int per_warp = (P + 1) + 3 * P + nmax + nmax + nmax + S;
  float* base = smem + (size_t)wib * per_warp;
  float* t = base;                 // P+1
  float* t0 = t + (P + 1);         // P
  float* t1 = t0 + P;              // P
  float* p = t1 + P;               // P
  float* td = p + P;               // nmax  (merged / final fenceposts)
  float* wd = td + nmax;           // nmax  (weights, later softmax numerators)
  float* cw = wd + nmax;           // nmax
  float* cen = cw + nmax;          // S

  const int warps_per_block = blockDim.x >> 5;
  for (int ray = blockIdx.x * warps_per_block + wib; ray < d.num_rays;
       ray += gridDim.x * warps_per_block) {
    const float* tp = sdist_prev + (size_t)ray * (P + 1);
    const float* wp = w_prev + (size_t)ray * P;
    int nb;  // number of bins of the step function we resample from
    for (int i = lane; i <= P; i += 32) t[i] = tp[i];
    __syncwarp();
    if (d.use_dilation) {
      // weight_to_pdf, shifted copies
      for (int i = lane; i < P; i += 32) {
        float dt = __fsub_rn(t[i + 1], t[i]);
        p[i] = __fdiv_rn(wp[i], fmaxf(kEpsSq, dt));
        t0[i] = __fsub_rn(t[i], d.dilation);
        t1[i] = __fadd_rn(t[i + 1], d.dilation);
      }
      __syncwarp();
      // 3-way merge == jnp.sort(concat[t, t0, t1]) (values identical; ties broken by list id)
      for (int i = lane; i <= P; i += 32) {
        float x = t[i];
        int r = i + count_lt(t0, P, x) + count_lt(t1, P, x);
        td[r] = fminf(fmaxf(x, d.domain_lo), d.domain_hi);
      }
      for (int i = lane; i < P; i += 32) {
        float x = t0[i];
        int r = i + count_le(t, P + 1, x) + count_lt(t1, P, x);
        td[r] = fminf(fmaxf(x, d.domain_lo), d.domain_hi);
        x = t1[i];
        r = i + count_le(t, P + 1, x) + count_le(t0, P, x);
        td[r] = fminf(fmaxf(x, d.domain_lo), d.domain_hi);
      }
      __syncwarp();
      // windowed max of p over {i : t0[i] <= x < t1[i]} = [count_le(t1,x), count_le(t0,x)-1]
      float part = 0.f;
      for (int j = lane; j < 3 * P; j += 32) {
        float x = td[j];
        int ilo = count_le(t1, P, x);
        int ihi = count_le(t0, P, x) - 1;
        float m = 0.f;
        for (int i = ilo; i <= ihi; ++i) m = fmaxf(m, p[i]);
        float w = __fmul_rn(m, __fsub_rn(td[j + 1], x));   // pdf_to_weight
        wd[j] = w;
        part += w;
      }
      float tot = warp_sum(part);
      float denom = fmaxf(kEpsSq, tot);
      __syncwarp();
      // renormalise and trim [1:-1]: fenceposts td[1..3P-1], weights wd[1..3P-2]
      nb = 3 * P - 2;
      float keep_t = 0.f, keep_w = 0.f;
      // shift down by one in place (each lane reads before anyone writes a lower index of
      // the same stride class: do it through registers in two phases)
      for (int j0 = 0; j0 < nb + 1; j0 += 32) {
        int j = j0 + lane;
        if (j < nb + 1) keep_t = td[j + 1];
        if (j < nb) keep_w = __fdiv_rn(wd[j + 1], denom);
        __syncwarp();
        if (j < nb + 1) td[j] = keep_t;
        if (j < nb) wd[j] = keep_w;
        __syncwarp();
      }
    } else {
      nb = P;
      for (int i = lane; i <= P; i += 32) td[i] = t[i];
      for (int i = lane; i < P; i += 32) wd[i] = wp[i];
      __syncwarp();
    }
    if (tdil_out) for (int i = lane; i <= nb; i += 32) tdil_out[(size_t)ray * (nb + 1) + i] = td[i];
    if (wdil_out) for (int i = lane; i < nb; i += 32) wdil_out[(size_t)ray * nb + i] = wd[i];

    if (cw_in) {
      for (int i = lane; i <= nb; i += 32) cw[i] = cw_in[(size_t)ray * (nb + 1) + i];
      __syncwarp();
    } else {
      // logits = where(dt > 0, anneal * log(w + pad), -inf); softmax; CDF
      float mx = -INFINITY;
      for (int i = lane; i < nb; i += 32) {
        float lg = (td[i + 1] > td[i])
                       ? __fmul_rn(d.anneal, logf(__fadd_rn(wd[i], d.resample_padding)))
                       : -INFINITY;
        wd[i] = lg;
        mx = fmaxf(mx, lg);
      }
      mx = warp_max(mx);
      float se = 0.f;
      for (int i = lane; i < nb; i += 32) {
        float e = expf(__fsub_rn(wd[i], mx));
        wd[i] = e;
        se += e;
      }
      se = warp_sum(se);
      __syncwarp();
      // cw = [0, min(1, cumsum(w[:-1])), 1]: lane L owns a contiguous chunk (sequential adds
      // inside it), chunk offsets come from a warp shuffle scan of the chunk sums.  The min keeps
      // a NaN (all logits -inf, or anneal 0 times log 0) as jnp.minimum does, where fminf would
      // drop it: the samples of such a ray then collapse onto td[0], as in the reference.
      const int chunk = (nb + 31) / 32;
      const int b0 = lane * chunk;
      float local = 0.f;
      for (int i = b0; i < b0 + chunk && i < nb; ++i) {
        float w = __fdiv_rn(wd[i], se);
        wd[i] = w;
        local += w;
      }
      float incl = warp_scan_incl(local, lane);
      float run = __shfl_up_sync(kFull, incl, 1);
      if (lane == 0) run = 0.f;
      for (int i = b0; i < b0 + chunk && i < nb - 1; ++i) {
        run += wd[i];
        cw[i + 1] = run > 1.f ? 1.f : run;
      }
      if (lane == 0) { cw[0] = 0.f; cw[nb] = 1.f; }
      __syncwarp();
    }
    if (cw_out) for (int i = lane; i <= nb; i += 32) cw_out[(size_t)ray * (nb + 1) + i] = cw[i];

    // inverse CDF at u (sorted_interp in index form)
    for (int s = lane; s < S; s += 32) {
      float u = u_base[s];
      if (d.jitter_mode == 1) u = __fadd_rn(u, __fmul_rn(jitter[ray], d.max_jitter));
      else if (d.jitter_mode == 2) u = __fadd_rn(u, __fmul_rn(jitter[(size_t)ray * S + s], d.max_jitter));
      int cnt = count_le(cw, nb + 1, u);          // #{cw <= u} in [0, nb+1]
      int i0 = max(cnt - 1, 0), i1 = min(cnt, nb);
      float x0 = cw[i0], x1 = cw[i1], f0 = td[i0], f1 = td[i1];
      float off = __fdiv_rn(__fsub_rn(u, x0), __fsub_rn(x1, x0));
      if (isnan(off)) off = 0.f;
      off = fminf(fmaxf(off, 0.f), 1.f);
      cen[s] = __fadd_rn(f0, __fmul_rn(off, __fsub_rn(f1, f0)));
      if (idx_out) idx_out[(size_t)ray * S + s] = cnt - 1;
    }
    __syncwarp();
    // intervals spanning the midpoints, ends reflected and clamped to the domain
    float* out = sdist_out + (size_t)ray * (S + 1);
    for (int s = lane; s <= S; s += 32) {
      float v;
      if (s == 0) {
        float mid0 = __fmul_rn(__fadd_rn(cen[1], cen[0]), 0.5f);
        v = fmaxf(d.domain_lo, __fsub_rn(__fmul_rn(2.f, cen[0]), mid0));
      } else if (s == S) {
        float midl = __fmul_rn(__fadd_rn(cen[S - 1], cen[S - 2]), 0.5f);
        v = fminf(d.domain_hi, __fsub_rn(__fmul_rn(2.f, cen[S - 1]), midl));
      } else {
        v = __fmul_rn(__fadd_rn(cen[s], cen[s - 1]), 0.5f);
      }
      out[s] = v;
    }
    __syncwarp();
  }
}

}  // namespace mnrf

extern "C" int mnrf_sample_level(const mnrf_sample_desc* d, const float* sdist_prev,
                                 const float* w_prev, const float* u_base, const float* jitter,
                                 const float* anneal_dev, const float* cw_in, float* sdist_out,
                                 int32_t* idx_out, float* cw_out, float* tdil_out, float* wdil_out,
                                 mnrf_stream stream) {
  using namespace mnrf;
  if (d && d->num_rays == 0) return 0;
  MNRF_CHECK(d && sdist_prev && w_prev && u_base && sdist_out, "mnrf_sample_level: null pointer");
  MNRF_CHECK(d->num_samples > 1, "num_samples must be > 1, is %d.", d->num_samples);
  MNRF_CHECK(d->num_prev >= 1 && d->num_prev <= 1024, "mnrf_sample_level: num_prev %d out of range",
             d->num_prev);
  MNRF_CHECK(d->jitter_mode == 0 || jitter, "mnrf_sample_level: jitter_mode %d needs jitter",
             d->jitter_mode);
  if (d->num_rays == 0) return 0;
  const int P = d->num_prev, S = d->num_samples;
  const int nmax = 3 * P + 1;
  const size_t per_warp = (size_t)((P + 1) + 3 * P + 3 * nmax + S) * sizeof(float);
  int warps = 4;
  while (warps > 1 && per_warp * warps > 200 * 1024) warps >>= 1;
  MNRF_CHECK(per_warp * warps <= 227 * 1024, "mnrf_sample_level: step function too large");
  const size_t smem = per_warp * warps;
  MNRF_CUDA(cudaFuncSetAttribute(sample_level_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)smem));
  int blocks = ceil_div(d->num_rays, warps);
  const int max_blocks = mnrf_num_sms() * 16;
  if (blocks > max_blocks) blocks = max_blocks;
  sample_level_kernel<<<blocks, warps * 32, smem, (cudaStream_t)stream>>>(
      *d, sdist_prev, w_prev, u_base, jitter, cw_in, sdist_out, idx_out, cw_out, tdil_out, wdil_out,
      anneal_dev);
  MNRF_LAUNCH_CHECK();
  return 0;
}
