// Alpha-weight compositing, its adjoint, and the per-ray losses: one warp owns one ray.
//
// Forward replaces (reference file:line): density/rgb activations models.py:506,584-602;
// render.compute_alpha_weights render.py:130-151 (exclusive-prefix transmittance scan with
// warp shuffles); render.volumetric_rendering render.py:154-213 incl. distance_mean and the
// weighted percentiles stepfun.py:298-308.
// Backward fuses train_utils.compute_data_loss train_utils.py:72-136, interlevel_loss
// :139-150 (stepfun.lossfun_outer stepfun.py:64-86), distortion_loss :153-159
// (stepfun.lossfun_distortion stepfun.py:266-276 in its O(S) prefix-sum form) with the
// adjoint of the compositing (SURVEY Appendix B; checked against oracle autograd).
//
// Lane L owns the CH contiguous samples [L*CH, L*CH+CH): scans are lane-local + shuffle.
#include "common.cuh"

namespace mnrf {

template <int CH>
struct RayState {
  float a[CH];      // density * delta (inf on the opaque last sample)
  float T[CH];      // transmittance before the sample
  float w[CH];      // alpha * T
  float dens_in[CH];  // raw + bias (+ noise): argument of softplus
  float delta[CH];
  float c[CH][3];   // activated + padded colour, times the per-ray exposure scale
  float z[CH][3];   // premult * raw + bias (argument of the rgb activation)
  float sc[3];      // per-ray rgb scale (RawNeRF exposure, models.py:257-267); 1 if absent
  float zd[CH][3];  // Ref-NeRF: raw diffuse colour (pre-activation), rgb_mode 1
  float zt[CH][3];  // Ref-NeRF: raw specular tint (pre-activation), rgb_mode 1
  float acc;        // sum of w
};

__device__ __forceinline__ float rgb_act(int kind, float z) {
  return kind == MNRF_RGB_SAFE_EXP ? expf(fminf(z, 88.f)) : sigmoid_f(z);
}
// image.linear_to_srgb (image.py:48-56) and its derivative
__device__ __forceinline__ float lin2srgb(float x) {
  return x <= 0.0031308f ? (323.f / 25.f) * x : (211.f * powf(fmaxf(kEps, x), 5.f / 12.f) - 11.f) / 200.f;
}
__device__ __forceinline__ float lin2srgb_grad(float x) {
  if (x <= 0.0031308f) return 323.f / 25.f;
  return x > kEps ? (211.f / 200.f) * (5.f / 12.f) * powf(x, -7.f / 12.f) : 0.f;
}
constexpr float kLog3 = 1.09861228866810969f;

// colour of one channel: returns c (before the per-ray scale); mode 1 = diffuse + tinted specular
__device__ __forceinline__ float colour_fwd(const mnrf_composite_desc& d, float z, float zd, float zt,
                                            bool has_tint) {
  float a = rgb_act(d.rgb_act, z);
  if (d.rgb_mode == 1) {
    float t = has_tint ? sigmoid_f(zt) : 0.5f;
    float lin = t * a + sigmoid_f(zd - kLog3);
    a = fminf(fmaxf(lin2srgb(lin), 0.f), 1.f);
  }
  return a * (1.f + 2.f * d.rgb_padding) - d.rgb_padding;
}

__device__ __forceinline__ float rgb_act_grad(int kind, float z) {
  if (kind == MNRF_RGB_SAFE_EXP) return expf(fminf(z, 88.f));
  float s = sigmoid_f(z);
  return s * (1.f - s);
}

// floats between consecutive samples of raw_density / raw_rgb and of their gradients (mnrf.h)
__device__ __forceinline__ size_t ld_density(const mnrf_composite_desc& d) { return d.ld_density ? d.ld_density : 1; }
__device__ __forceinline__ size_t ld_rgb(const mnrf_composite_desc& d) { return d.ld_rgb ? d.ld_rgb : 3; }

template <int CH>
__device__ __forceinline__ void ray_forward(const mnrf_composite_desc& d, int ray, int lane,
                                            const float* __restrict__ raw_density,
                                            const float* __restrict__ raw_rgb,
                                            const float* __restrict__ density_noise,
                                            const float* __restrict__ rgb_scale,
                                            const float* __restrict__ raw_diffuse,
                                            const float* __restrict__ raw_tint,
                                            const float* tds, float dnorm, RayState<CH>& st) {
  const int S = d.num_samples;
  float local = 0.f;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) st.sc[ch] = rgb_scale ? rgb_scale[ray * 3 + ch] : 1.f;
#pragma unroll
  for (int j = 0; j < CH; ++j) {
    int s = lane * CH + j;
    bool ok = s < S;
    float raw = ok ? raw_density[((size_t)ray * S + s) * ld_density(d)] : 0.f;
    if (density_noise && ok) raw += d.density_noise * density_noise[(size_t)ray * S + s];
    float din = raw + d.density_bias;
    st.dens_in[j] = din;
    float dens = softplus_f(din);
    float dl = ok ? (tds[s + 1] - tds[s]) * dnorm : 0.f;
    st.delta[j] = dl;
    float a = ok ? dens * dl : 0.f;
    if (d.opaque_background && s == S - 1) a = INFINITY;
    st.a[j] = a;
    if (s < S - 1) local += a;   // the last a never enters a prefix that is used
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      float z = 0.f, c = 0.f, zd = 0.f, zt = 0.f;
      if (raw_rgb && ok) {
        const size_t ci = ((size_t)ray * S + s) * 3 + ch;
        z = d.rgb_premult * raw_rgb[((size_t)ray * S + s) * ld_rgb(d) + ch] + d.rgb_bias;
        if (d.rgb_mode == 1) {
          zd = raw_diffuse[ci];
          if (raw_tint) zt = raw_tint[ci];
        }
        c = colour_fwd(d, z, zd, zt, raw_tint != nullptr) * st.sc[ch];
      }
      st.z[j][ch] = z;
      st.zd[j][ch] = zd;
      st.zt[j][ch] = zt;
      st.c[j][ch] = c;
    }
  }
  float incl = warp_scan_incl(local, lane);
  float run = __shfl_up_sync(kFull, incl, 1);
  if (lane == 0) run = 0.f;
  float accp = 0.f;
#pragma unroll
  for (int j = 0; j < CH; ++j) {
    int s = lane * CH + j;
    float T = expf(-run);
    float alpha = 1.f - expf(-st.a[j]);
    float w = (s < S) ? alpha * T : 0.f;
    st.T[j] = T;
    st.w[j] = w;
    accp += w;
    run += st.a[j];
  }
  st.acc = warp_sum(accp);
}

// Loads tdist = s_to_t(sdist) of one ray into shared memory (S+1 floats).
__device__ __forceinline__ void load_tdist(int fn, int ray, int S, int lane,
                                           const float* __restrict__ sdist,
                                           const float* __restrict__ near,
                                           const float* __restrict__ far, float* tds) {
  const float s_near = fwd_raydist(fn, near[ray]);
  const float s_far = fwd_raydist(fn, far[ray]);
  for (int i = lane; i <= S; i += 32)
    tds[i] = s_to_t(fn, sdist[(size_t)ray * (S + 1) + i], s_near, s_far);
  __syncwarp();
}

template <int CH>
__global__ void __launch_bounds__(128)
composite_fwd_kernel(mnrf_composite_desc d, const float* __restrict__ raw_density,
                     const float* __restrict__ raw_rgb, const float* __restrict__ density_noise,
                     const float* __restrict__ sdist, const float* __restrict__ directions,
                     const float* __restrict__ near, const float* __restrict__ far,
                     const float* __restrict__ bg_rgb, const float* __restrict__ rgb_scale,
                     const float* __restrict__ raw_diffuse, const float* __restrict__ raw_tint,
                     float* __restrict__ weights,
                     float* __restrict__ rgb_out, float* __restrict__ density_out,
                     float* __restrict__ rgb_samples, float* __restrict__ acc_out,
                     float* __restrict__ dist_out) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int S = d.num_samples;
  float* tds = smem + (size_t)wib * (2 * S + 4);   // tdist[S+1] then cw[S+2] (extras)
  float* cws = tds + (S + 1);
  for (int ray = blockIdx.x * nw + wib; ray < d.num_rays; ray += gridDim.x * nw) {
    load_tdist(d.raydist_fn, ray, S, lane, sdist, near, far, tds);
    const float dx = directions[ray * 3], dy = directions[ray * 3 + 1], dz = directions[ray * 3 + 2];
    const float dnorm = sqrtf(dx * dx + dy * dy + dz * dz);
    RayState<CH> st;
    ray_forward<CH>(d, ray, lane, raw_density, raw_rgb, density_noise, rgb_scale, raw_diffuse, raw_tint, tds,
                    dnorm, st);
    float px[3] = {0.f, 0.f, 0.f};
    float elog = 0.f;
#pragma unroll
    for (int j = 0; j < CH; ++j) {
      int s = lane * CH + j;
      if (s < S) {
        weights[(size_t)ray * S + s] = st.w[j];
        if (density_out) density_out[(size_t)ray * S + s] = softplus_f(st.dens_in[j]);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
          px[ch] += st.w[j] * st.c[j][ch];
          if (rgb_samples) rgb_samples[((size_t)ray * S + s) * 3 + ch] = st.c[j][ch];
        }
        if (dist_out) elog += st.w[j] * logf(0.5f * (tds[s] + tds[s + 1]));
      }
    }
    const float bg_w = fmaxf(0.f, 1.f - st.acc);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      float v = warp_sum(px[ch]);
      float bg = bg_rgb ? bg_rgb[ray * 3 + ch] : d.bg_const;
      if (lane == 0) rgb_out[ray * 3 + ch] = v + bg_w * bg;
    }
    if (acc_out && lane == 0) acc_out[ray] = st.acc;
    if (dist_out) {
      // distance_mean (render.py:193-198)
      elog = warp_sum(elog);
      float dm = expf(elog / fmaxf(kEps, st.acc));
      if (isnan(dm)) dm = 0.f;                       // nan_to_num's 2nd positional arg is `copy`
      if (isinf(dm)) dm = dm > 0 ? 3.4028235e38f : -3.4028235e38f;
      dm = fminf(fmaxf(dm, tds[0]), tds[S]);
      // percentiles of (t ∪ far, w ∪ bg_w): cw = [0, min(1, cumsum(w)), 1]  (S+2 entries)
      float local = 0.f;
#pragma unroll
      for (int j = 0; j < CH; ++j) local += st.w[j];
      float incl = warp_scan_incl(local, lane);
      float run = __shfl_up_sync(kFull, incl, 1);
      if (lane == 0) run = 0.f;
#pragma unroll
      for (int j = 0; j < CH; ++j) {
        int s = lane * CH + j;
        run += st.w[j];
        if (s < S) cws[s + 1] = fminf(1.f, run);
      }
      if (lane == 0) { cws[0] = 0.f; cws[S + 1] = 1.f; }
      __syncwarp();
      if (lane < 3) {
        const float p = lane == 0 ? 0.05f : (lane == 1 ? 0.5f : 0.95f);
        const int n = S + 2;
        // np.interp: index of the right neighbour = #{cw <= p}, clamped to [1, n-1]
        int lo = 0, hi = n;
        while (lo < hi) { int mid = (lo + hi) >> 1; if (cws[mid] <= p) lo = mid + 1; else hi = mid; }
        int i1 = min(max(lo, 1), n - 1), i0 = i1 - 1;
        float x0 = cws[i0], x1 = cws[i1];
        float far_t = far[ray];
        float f0 = i0 <= S ? tds[i0] : far_t, f1 = i1 <= S ? tds[i1] : far_t;
        float dxp = x1 - x0;
        float v = dxp == 0.f ? f0 : f0 + (f1 - f0) / dxp * (p - x0);
        dist_out[ray * 4 + 1 + lane] = v;
      }
      if (lane == 0) dist_out[ray * 4] = dm;
      __syncwarp();
    }
    __syncwarp();
  }
}

// ----------------------------------------------------------------------------------------
template <int CH>
__global__ void __launch_bounds__(128)
composite_bwd_kernel(mnrf_loss_desc L, const float* __restrict__ raw_density,
                     const float* __restrict__ raw_rgb, const float* __restrict__ density_noise,
                     const float* __restrict__ sdist, const float* __restrict__ directions,
                     const float* __restrict__ near, const float* __restrict__ far,
                     const float* __restrict__ bg_rgb, const float* __restrict__ rgb_scale,
                     const float* __restrict__ raw_diffuse, const float* __restrict__ raw_tint,
                     const float* __restrict__ extra_dw, const float* __restrict__ target_rgb,
                     const float* __restrict__ lossmult, const float* __restrict__ inv_denom_p,
                     const float* __restrict__ sdist_fine, const float* __restrict__ weights_fine,
                     const float* __restrict__ data_mask,
                     float* __restrict__ d_raw_density, float* __restrict__ d_raw_rgb,
                     float* __restrict__ d_rgb_scale, float* __restrict__ d_raw_diffuse,
                     float* __restrict__ d_raw_tint, float* __restrict__ stats, int batch_rays) {
  extern __shared__ float smem[];
  const mnrf_composite_desc& d = L.c;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int S = d.num_samples, Sf = L.num_samples_fine;
  // per warp: tdist[S+1] | senv[S+1] | cy[S+1] | D[S+2]
  float* tds = smem + (size_t)wib * (4 * S + 6);
  float* senv = tds + (S + 1);
  float* cy = senv + (S + 1);
  float* D = cy + (S + 1);
  const float inv_denom = *inv_denom_p;
  // the distortion and interlevel losses are means over the step's whole batch (batch_rays), of which this launch
  // may be one pass
  const float invB = 1.f / (float)batch_rays;
  float st_data = 0.f, st_mse = 0.f, st_dist = 0.f, st_inter = 0.f;

  for (int ray = blockIdx.x * nw + wib; ray < d.num_rays; ray += gridDim.x * nw) {
    load_tdist(d.raydist_fn, ray, S, lane, sdist, near, far, tds);
    const float dx = directions[ray * 3], dy = directions[ray * 3 + 1], dz = directions[ray * 3 + 2];
    const float dnorm = sqrtf(dx * dx + dy * dy + dz * dz);
    RayState<CH> st;
    ray_forward<CH>(d, ray, lane, raw_density, raw_rgb, density_noise, rgb_scale, raw_diffuse, raw_tint, tds,
                    dnorm, st);

    // ---- pixel and data loss ------------------------------------------------------------
    float px[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < CH; ++j)
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) px[ch] += st.w[j] * st.c[j][ch];
    const float bg_w = fmaxf(0.f, 1.f - st.acc);
    const float bg_on = (1.f - st.acc) > 0.f ? 1.f : 0.f;
    float dpx[3], bgc[3], wc[3];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      bgc[ch] = bg_rgb ? bg_rgb[ray * 3 + ch] : d.bg_const;
      wc[ch] = warp_sum(px[ch]);                      // sum_s w_s c_s (scaled colour)
      float v = wc[ch] + bg_w * bgc[ch];
      float tgt = target_rgb[ray * 3 + ch];
      float lm = lossmult[L.lossmult_channels == 3 ? ray * 3 + ch : ray];
      float resid = v - tgt;
      float g, lv;
      if (L.loss_type == MNRF_LOSS_MSE) {
        lv = resid * resid;
        g = 2.f * resid;
      } else if (L.loss_type == MNRF_LOSS_CHARB) {
        lv = sqrtf(resid * resid + L.charb_padding * L.charb_padding);
        g = resid / lv;
      } else {
        float clip = fminf(1.f, v);
        float rc = clip - tgt;
        float sc = 1.f / (1e-3f + clip);
        lv = rc * rc * sc * sc;
        g = v < 1.f ? 2.f * rc * sc * sc : 0.f;
      }
      if (data_mask) {                                // robustnerf: resid_sq * mask (a constant for autodiff)
        const float m = data_mask[ray];
        lv *= m;
        g *= m;
      }
      dpx[ch] = L.data_mult * lm * g * inv_denom;
      // d pixel / d scale = sum_s w_s c_unscaled_s = (sum_s w_s c_s) / scale.  A zero scale (RawNeRF exposure
      // value times 1 + offset) leaves no scaled colour to divide: sum the unscaled colours again (warp-uniform).
      float wcu = 0.f;
      if (d_rgb_scale && st.sc[ch] == 0.f && raw_rgb) {
#pragma unroll
        for (int j = 0; j < CH; ++j)
          wcu += st.w[j] * colour_fwd(d, st.z[j][ch], st.zd[j][ch], st.zt[j][ch], raw_tint != nullptr);
        wcu = warp_sum(wcu);
      }
      if (lane == 0) {
        st_data += L.data_mult * lm * lv * inv_denom;
        st_mse += lm * resid * resid * inv_denom;
        if (d_rgb_scale) d_rgb_scale[ray * 3 + ch] = st.sc[ch] != 0.f ? dpx[ch] * wc[ch] / st.sc[ch] : dpx[ch] * wcu;
      }
    }

    // ---- dL/dw from the pixel ------------------------------------------------------------
    float g[CH];
#pragma unroll
    for (int j = 0; j < CH; ++j) {
      g[j] = 0.f;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) g[j] += dpx[ch] * (st.c[j][ch] - bg_on * bgc[ch]);
      if (extra_dw) {        // orientation / predicted-normal losses (train_utils.py:162-197)
        int s = lane * CH + j;
        if (s < S) g[j] += extra_dw[(size_t)ray * S + s];
      }
    }

    // ---- distortion loss (final level) in normalised s-space ---------------------------
    if (L.distortion_mult > 0.f) {
      const float* sr = sdist + (size_t)ray * (S + 1);
      float m[CH], dl[CH], lw = 0.f, lwm = 0.f;
#pragma unroll
      for (int j = 0; j < CH; ++j) {
        int s = lane * CH + j;
        float s0 = s < S ? sr[s] : 0.f, s1 = s < S ? sr[s + 1] : 0.f;
        m[j] = 0.5f * (s0 + s1);
        dl[j] = s1 - s0;
        lw += st.w[j];
        lwm += st.w[j] * m[j];
      }
      float iw = warp_scan_incl(lw, lane), iwm = warp_scan_incl(lwm, lane);
      float totw = __shfl_sync(kFull, iw, 31), totwm = __shfl_sync(kFull, iwm, 31);
      float pw = __shfl_up_sync(kFull, iw, 1), pwm = __shfl_up_sync(kFull, iwm, 1);
      if (lane == 0) { pw = 0.f; pwm = 0.f; }
      float lossp = 0.f;
#pragma unroll
      for (int j = 0; j < CH; ++j) {
        // prefix (exclusive) = (pw, pwm); suffix (exclusive) = total - prefix - own
        float sw = totw - pw - st.w[j], swm = totwm - pwm - st.w[j] * m[j];
        float inter_i = m[j] * pw - pwm + swm - m[j] * sw;       // sum_j w_j |m_i - m_j|
        lossp += st.w[j] * inter_i + st.w[j] * st.w[j] * dl[j] * (1.f / 3.f);
        g[j] += L.distortion_mult * invB * (2.f * inter_i + (2.f / 3.f) * st.w[j] * dl[j]);
        pw += st.w[j];
        pwm += st.w[j] * m[j];
      }
      lossp = warp_sum(lossp);
      if (lane == 0) st_dist += L.distortion_mult * invB * lossp;
    }

    // ---- interlevel loss (this is a proposal level; envelope = own step function) -----
    if (L.interlevel_mult > 0.f) {
      const float* se = sdist + (size_t)ray * (S + 1);
      for (int i = lane; i <= S; i += 32) { senv[i] = se[i]; D[i] = 0.f; }
      if (lane == 0) D[S + 1] = 0.f;
      // cy = [0, cumsum(w_env)]
      float lw = 0.f;
#pragma unroll
      for (int j = 0; j < CH; ++j) lw += st.w[j];
      float iw = warp_scan_incl(lw, lane);
      float run = __shfl_up_sync(kFull, iw, 1);
      if (lane == 0) { run = 0.f; cy[0] = 0.f; }
#pragma unroll
      for (int j = 0; j < CH; ++j) {
        int s = lane * CH + j;
        run += st.w[j];
        if (s < S) cy[s + 1] = run;
      }
      __syncwarp();
      const float* cf = sdist_fine + (size_t)ray * (Sf + 1);
      const float* wf = weights_fine + (size_t)ray * Sf;
      const float scale = L.interlevel_mult / ((float)batch_rays * (float)Sf);
      float lossp = 0.f;
      for (int i = lane; i < Sf; i += 32) {
        float t0 = cf[i], t1 = cf[i + 1], w = wf[i];
        // idx_lo(t0) = max{j : senv[j] <= t0} (0 if none); idx_hi(t1) = min{j : senv[j] > t1} (S if none)
        int lo = 0, hi = S + 1;
        while (lo < hi) { int mid = (lo + hi) >> 1; if (senv[mid] <= t0) lo = mid + 1; else hi = mid; }
        int idx_lo = max(lo - 1, 0);
        lo = 0; hi = S + 1;
        while (lo < hi) { int mid = (lo + hi) >> 1; if (senv[mid] <= t1) lo = mid + 1; else hi = mid; }
        int idx_hi = min(lo, S);
        float w_outer = cy[idx_hi] - cy[idx_lo];
        float ex = fmaxf(0.f, w - w_outer);
        lossp += ex * ex / (w + kEps);
        float gi = -2.f * ex / (w + kEps) * scale;     // dL/dw_outer
        if (gi != 0.f && idx_hi > idx_lo) {
          atomicAdd(&D[idx_lo], gi);                   // d cy[hi]/d w_j = [j < hi]; range [lo, hi)
          atomicAdd(&D[idx_hi], -gi);
        }
      }
      lossp = warp_sum(lossp);
      if (lane == 0) st_inter += scale * lossp;
      __syncwarp();
      // grad wrt w_env[j] = sum_{k<=j} D[k]
      float ld = 0.f;
#pragma unroll
      for (int j = 0; j < CH; ++j) { int s = lane * CH + j; if (s < S) ld += D[s]; }
      float idd = warp_scan_incl(ld, lane);
      float rd = __shfl_up_sync(kFull, idd, 1);
      if (lane == 0) rd = 0.f;
#pragma unroll
      for (int j = 0; j < CH; ++j) {
        int s = lane * CH + j;
        if (s < S) { rd += D[s]; g[j] += rd; }
      }
      __syncwarp();
    }

    // ---- compositing adjoint: dL/da_k = g_k e^{-a_k} T_k - sum_{i>k} g_i w_i -----------
    float lgw = 0.f;
#pragma unroll
    for (int j = 0; j < CH; ++j) lgw += g[j] * st.w[j];
    float sfx = warp_scan_incl_rev(lgw, lane) - lgw;   // lanes after this one
    float after = sfx;
#pragma unroll
    for (int j = CH - 1; j >= 0; --j) {
      int s = lane * CH + j;
      if (s < S) {
        float da;
        if (isinf(st.a[j])) da = 0.f;
        else da = g[j] * expf(-st.a[j]) * st.T[j] - after;
        float dd = da * st.delta[j] * sigmoid_f(st.dens_in[j]);
        d_raw_density[((size_t)ray * S + s) * ld_density(d)] = dd;
        if (d_raw_rgb) {
#pragma unroll
          for (int ch = 0; ch < 3; ++ch) {
            const size_t ci = ((size_t)ray * S + s) * 3 + ch;
            const size_t ri = ((size_t)ray * S + s) * ld_rgb(d) + ch;
            // dL/d(colour before padding and scale)
            const float gc = dpx[ch] * st.w[j] * st.sc[ch] * (1.f + 2.f * d.rgb_padding);
            const float da = rgb_act_grad(d.rgb_act, st.z[j][ch]) * d.rgb_premult;
            if (d.rgb_mode == 1) {
              const float a = rgb_act(d.rgb_act, st.z[j][ch]);
              const float t = raw_tint ? sigmoid_f(st.zt[j][ch]) : 0.5f;
              const float dl = sigmoid_f(st.zd[j][ch] - kLog3);
              const float lin = t * a + dl;
              const float sr = lin2srgb(lin);
              const float glin = (sr > 0.f && sr < 1.f) ? gc * lin2srgb_grad(lin) : 0.f;
              d_raw_rgb[ri] = glin * t * da;
              d_raw_diffuse[ci] = glin * dl * (1.f - dl);
              if (d_raw_tint) d_raw_tint[ci] = raw_tint ? glin * a * t * (1.f - t) : 0.f;
            } else {
              d_raw_rgb[ri] = gc * da;
            }
          }
        }
      }
      after += g[j] * st.w[j];
    }
    __syncwarp();
  }
  if (lane == 0) {
    if (st_data != 0.f) atomicAdd(&stats[0], st_data);
    if (st_mse != 0.f) atomicAdd(&stats[1], st_mse);
    if (st_dist != 0.f) atomicAdd(&stats[2], st_dist);
    if (st_inter != 0.f) atomicAdd(&stats[3], st_inter);
  }
}

// The activated, padded colour of each of M independent samples: ray_forward's colour without compositing and
// without the per-ray scale (one thread per sample; raw_rgb rows ld_rgb floats apart)
__global__ void __launch_bounds__(256)
point_rgb_kernel(mnrf_composite_desc d, int64_t M, const float* __restrict__ raw_rgb, int ld_rgb,
                 const float* __restrict__ raw_diffuse, const float* __restrict__ raw_tint, float* __restrict__ rgb_out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < M; i += (int64_t)gridDim.x * blockDim.x) {
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const float z = d.rgb_premult * raw_rgb[i * ld_rgb + ch] + d.rgb_bias;
      float zd = 0.f, zt = 0.f;
      if (d.rgb_mode == 1) {
        zd = raw_diffuse[i * 3 + ch];
        if (raw_tint) zt = raw_tint[i * 3 + ch];
      }
      rgb_out[i * 3 + ch] = colour_fwd(d, z, zd, zt, raw_tint != nullptr);
    }
  }
}

// The descriptor fields both entry points branch on: anything else would silently take some other branch (an unknown
// rgb_mode composites as mode 0) or read rows that overlap (ld_rgb 1 or 2).  ld 0 means the contiguous default.
static int check_desc(const char* fn, const mnrf_composite_desc& d) {
  MNRF_CHECK(d.num_rays >= 0, "%s: negative num_rays %d", fn, d.num_rays);
  MNRF_CHECK(d.raydist_fn >= MNRF_RAYDIST_NONE && d.raydist_fn <= MNRF_RAYDIST_PIECEWISE, "%s: unknown raydist_fn %d",
             fn, d.raydist_fn);
  MNRF_CHECK(d.rgb_act == MNRF_RGB_SIGMOID || d.rgb_act == MNRF_RGB_SAFE_EXP, "%s: unknown rgb_act %d", fn, d.rgb_act);
  MNRF_CHECK(d.rgb_mode == 0 || d.rgb_mode == 1, "%s: unknown rgb_mode %d", fn, d.rgb_mode);
  MNRF_CHECK(d.ld_density >= 0, "%s: negative ld_density %d", fn, d.ld_density);
  MNRF_CHECK(d.ld_rgb == 0 || d.ld_rgb >= 3, "%s: ld_rgb %d overlaps the rgb rows (0 or >= 3)", fn, d.ld_rgb);
  return 0;
}

}  // namespace mnrf

#define MNRF_DISPATCH_CH(S, CALL)                         \
  do {                                                    \
    if ((S) <= 32) { constexpr int CH = 1; CALL; }        \
    else if ((S) <= 64) { constexpr int CH = 2; CALL; }   \
    else if ((S) <= 128) { constexpr int CH = 4; CALL; }  \
    else { constexpr int CH = 8; CALL; }                  \
  } while (0)

extern "C" int mnrf_composite_fwd(const mnrf_composite_desc* d, const float* raw_density,
                                  const float* raw_rgb, const float* density_noise,
                                  const float* sdist, const float* directions, const float* near,
                                  const float* far, const float* bg_rgb, const float* rgb_scale,
                                  const float* raw_diffuse, const float* raw_tint,
                                  float* weights, float* rgb_out, float* density_out,
                                  float* rgb_samples, float* acc, float* dist, mnrf_stream stream) {
  using namespace mnrf;
  MNRF_CHECK(d, "mnrf_composite_fwd: null descriptor");
  if (check_desc("mnrf_composite_fwd", *d)) return 1;
  if (d->num_rays == 0) return 0;
  MNRF_CHECK(raw_density && sdist && directions && near && far && weights && rgb_out,
             "mnrf_composite_fwd: null pointer");
  MNRF_CHECK(d->num_samples >= 1 && d->num_samples <= 256, "mnrf_composite_fwd: num_samples %d not in [1, 256]",
             d->num_samples);
  MNRF_CHECK(d->rgb_mode == 0 || (raw_rgb && raw_diffuse), "mnrf_composite_fwd: rgb_mode 1 needs raw_diffuse");
  const int nw = 4;
  size_t smem = (size_t)nw * (2 * d->num_samples + 4) * sizeof(float);
  int blocks = ceil_div(d->num_rays, nw);
  int maxb = mnrf_num_sms() * 16;
  if (blocks > maxb) blocks = maxb;
  MNRF_DISPATCH_CH(d->num_samples, (composite_fwd_kernel<CH><<<blocks, nw * 32, smem, (cudaStream_t)stream>>>(
      *d, raw_density, raw_rgb, density_noise, sdist, directions, near, far, bg_rgb, rgb_scale, raw_diffuse,
      raw_tint, weights, rgb_out, density_out, rgb_samples, acc, dist)));
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_point_rgb(const mnrf_composite_desc* d, int64_t M, const float* raw_rgb, int32_t ld_rgb,
                              const float* raw_diffuse, const float* raw_tint, float* rgb_out, mnrf_stream stream) {
  using namespace mnrf;
  MNRF_CHECK(d, "mnrf_point_rgb: null descriptor");
  MNRF_CHECK(M >= 0, "mnrf_point_rgb: negative sample count %lld", (long long)M);
  if (M == 0) return 0;
  MNRF_CHECK(raw_rgb && rgb_out, "mnrf_point_rgb: null pointer");
  MNRF_CHECK(ld_rgb >= 3, "mnrf_point_rgb: ld_rgb %d < 3", ld_rgb);
  MNRF_CHECK(d->rgb_act == MNRF_RGB_SIGMOID || d->rgb_act == MNRF_RGB_SAFE_EXP, "mnrf_point_rgb: unknown rgb_act %d",
             d->rgb_act);
  MNRF_CHECK(d->rgb_mode == 0 || d->rgb_mode == 1, "mnrf_point_rgb: unknown rgb_mode %d", d->rgb_mode);
  MNRF_CHECK(d->rgb_mode == 0 || raw_diffuse, "mnrf_point_rgb: rgb_mode 1 needs raw_diffuse");
  const int64_t maxb = (int64_t)mnrf_num_sms() * 16;
  const int blocks = (int)((M + 255) / 256 < maxb ? (M + 255) / 256 : maxb);
  point_rgb_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(*d, M, raw_rgb, ld_rgb, raw_diffuse, raw_tint, rgb_out);
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_composite_bwd(const mnrf_loss_desc* d, const float* raw_density, const float* raw_rgb,
                                  const float* density_noise, const float* sdist, const float* directions,
                                  const float* near, const float* far, const float* bg_rgb, const float* rgb_scale,
                                  const float* raw_diffuse, const float* raw_tint, const float* extra_dw,
                                  const float* target_rgb, const float* lossmult, const float* inv_denom,
                                  const float* sdist_fine, const float* weights_fine, const float* data_mask,
                                  float* d_raw_density, float* d_raw_rgb, float* d_rgb_scale,
                                  float* d_raw_diffuse, float* d_raw_tint, float* stats, int32_t batch_rays,
                                  mnrf_stream stream) {
  using namespace mnrf;
  MNRF_CHECK(d, "mnrf_composite_bwd: null descriptor");
  if (check_desc("mnrf_composite_bwd", d->c)) return 1;
  if (d->c.num_rays == 0) return 0;
  MNRF_CHECK(raw_density && sdist && directions && near && far && target_rgb && lossmult &&
             inv_denom && d_raw_density && stats, "mnrf_composite_bwd: null pointer");
  MNRF_CHECK(d->c.rgb_mode == 0 || (raw_rgb && d_raw_rgb && raw_diffuse && d_raw_diffuse && (!raw_tint || d_raw_tint)),
             "mnrf_composite_bwd: rgb_mode 1 needs raw_rgb / d_raw_rgb and raw_diffuse / d_raw_diffuse (and d_raw_tint "
             "with raw_tint)");
  MNRF_CHECK(d->c.num_samples >= 1 && d->c.num_samples <= 256, "mnrf_composite_bwd: num_samples %d not in [1, 256]",
             d->c.num_samples);
  MNRF_CHECK(d->interlevel_mult == 0.f || (sdist_fine && weights_fine && d->num_samples_fine >= 1),
             "mnrf_composite_bwd: interlevel loss needs the final level's sdist/weights (num_samples_fine %d)",
             d->num_samples_fine);
  MNRF_CHECK(d->lossmult_channels == 1 || d->lossmult_channels == 3, "lossmult_channels must be 1 or 3");
  MNRF_CHECK(d->loss_type >= 0 && d->loss_type <= 2, "unknown data_loss_type");
  MNRF_CHECK(batch_rays >= d->c.num_rays, "mnrf_composite_bwd: batch_rays %d < num_rays %d", batch_rays,
             d->c.num_rays);
  const int nw = 4;
  size_t smem = (size_t)nw * (4 * d->c.num_samples + 6) * sizeof(float);
  int blocks = ceil_div(d->c.num_rays, nw);
  int maxb = mnrf_num_sms() * 16;
  if (blocks > maxb) blocks = maxb;
  MNRF_DISPATCH_CH(d->c.num_samples, (composite_bwd_kernel<CH><<<blocks, nw * 32, smem, (cudaStream_t)stream>>>(
      *d, raw_density, raw_rgb, density_noise, sdist, directions, near, far, bg_rgb, rgb_scale, raw_diffuse,
      raw_tint, extra_dw, target_rgb, lossmult, inv_denom, sdist_fine, weights_fine, data_mask, d_raw_density,
      d_raw_rgb, d_rgb_scale, d_raw_diffuse, d_raw_tint, stats, batch_rays)));
  MNRF_LAUNCH_CHECK();
  return 0;
}
