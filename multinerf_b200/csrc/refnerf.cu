// Ref-NeRF per-sample stage between the spatial trunk and the directional MLP, and its adjoint.
//
// Forward replaces (reference file:line): normals / normals_pred = -l2_normalize(.)
// models.py:488-499 + ref_utils.l2_normalize ref_utils.py:40-42; roughness models.py:520-523;
// ref_utils.reflect ref_utils.py:22-37 (models.py:545); the integrated directional encoding
// ref_utils.generate_ide_fn ref_utils.py:98-159 or coord.pos_enc for plain view directions;
// n.v models.py:560-563.  It writes the bf16 direction-encoding slab of the view-MLP input.
// Backward fuses the adjoint of all of the above with train_utils.orientation_loss
// train_utils.py:162-178 and train_utils.predicted_normal_loss :181-197.
// One thread per sample: HBM-bound elementwise work.
#include <algorithm>

#include "common.cuh"

namespace mnrf {

constexpr int kIdeMax = 36;     // (m,l) pairs at deg_view = 5
constexpr int kZMax = 17;       // z^0 .. z^16

struct IdeTab {                 // staged in shared memory
  float mat[kZMax * kIdeMax];   // [k][i]
  float sigma[kIdeMax];
  int m[kIdeMax];
  int n, zdeg;
};

__device__ __forceinline__ void load_tab(IdeTab* s, const float* __restrict__ mat, const int* __restrict__ ml,
                                         int n, int zdeg) {
  for (int i = threadIdx.x; i < zdeg * n; i += blockDim.x) s->mat[i] = mat[i];
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    s->m[i] = ml[i];
    int l = ml[n + i];
    s->sigma[i] = 0.5f * (float)l * (float)(l + 1);
  }
  if (threadIdx.x == 0) { s->n = n; s->zdeg = zdeg; }
  __syncthreads();
}

// -x / sqrt(max(|x|^2, eps))
__device__ __forceinline__ void neg_normalize(const float g[3], float out[3], float& s, bool& clamped) {
  float sq = g[0] * g[0] + g[1] * g[1] + g[2] * g[2];
  clamped = !(sq > kEps);
  s = sqrtf(fmaxf(sq, kEps));
  out[0] = -g[0] / s; out[1] = -g[1] / s; out[2] = -g[2] / s;
}
// adjoint of neg_normalize: given a = dL/dout, returns dL/dg
__device__ __forceinline__ void neg_normalize_bwd(const float out[3], float s, bool clamped, const float a[3],
                                                  float dg[3]) {
  if (clamped) { dg[0] = -a[0] / s; dg[1] = -a[1] / s; dg[2] = -a[2] / s; return; }
  // out = -ghat:  d out/d g = -(I - ghat ghat^T)/s = -(I - out out^T)/s
  float dot = out[0] * a[0] + out[1] * a[1] + out[2] * a[2];
#pragma unroll
  for (int i = 0; i < 3; ++i) dg[i] = -(a[i] - out[i] * dot) / s;
}

struct RefDesc {
  int64_t M;
  int S;                       // samples per ray (viewdirs are per ray)
  int use_pred_normals, use_density_normals, use_reflections, use_ide, use_n_dot_v, use_roughness;
  int deg_view;
  float roughness_bias;
  int ld, col0, col_end;       // bf16 slab [M, ld], columns [col0, col_end)
};

struct RefLoss {
  float orient_mult, prednorm_mult;   // already divided by the number of rays
  int orient_on_pred;                 // orientation_loss_target == 'normals_pred'
};

// The normals and normal-loss arithmetic shared by the Ref-NeRF stage (refdir_*) and the colourless stage
// (normals_*).  Both stages must produce the same bits for the same inputs, so each piece exists once.

// One sample's normals_pred (p) and normals (d), zero when off, with the norms they were divided by
// and whether those norms were clamped.
struct Normals {
  float p[3], d[3];
  float s_p, s_d;
  bool cl_p, cl_d;
};

__device__ __forceinline__ void load_viewdir(const float* __restrict__ viewdirs, int S, int64_t m, float v[3]) {
  const int ray = (int)(m / S);
  v[0] = viewdirs[ray * 3]; v[1] = viewdirs[ray * 3 + 1]; v[2] = viewdirs[ray * 3 + 2];
}

// normals_pred = -l2_normalize(grad_pred), normals = -l2_normalize(raw_grad_density); each is stored when its
// output pointer is given
__device__ __forceinline__ Normals load_normals(int64_t M, int64_t m, bool use_p, bool use_d,
                                                const float* __restrict__ grad_pred,
                                                const float* __restrict__ raw_grad_density /* [3, M] */,
                                                float* __restrict__ normals_pred, float* __restrict__ normals) {
  Normals n{{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}, 1.f, 1.f, false, false};
  if (use_p) {
    const float g[3] = {grad_pred[m * 3], grad_pred[m * 3 + 1], grad_pred[m * 3 + 2]};
    neg_normalize(g, n.p, n.s_p, n.cl_p);
    if (normals_pred) { normals_pred[m * 3] = n.p[0]; normals_pred[m * 3 + 1] = n.p[1]; normals_pred[m * 3 + 2] = n.p[2]; }
  }
  if (use_d) {
    const float g[3] = {raw_grad_density[m], raw_grad_density[M + m], raw_grad_density[2 * M + m]};
    neg_normalize(g, n.d, n.s_d, n.cl_d);
    if (normals) { normals[m * 3] = n.d[0]; normals[m * 3 + 1] = n.d[1]; normals[m * 3 + 2] = n.d[2]; }
  }
  return n;
}

// -(n . v) for the normal the orientation loss reads.  Selected by value, not through a pointer into the two
// arrays (which would put them on the stack).
__device__ __forceinline__ float orient_p(const Normals& n, bool op, const float v[3]) {
  return -((op ? n.p[0] : n.d[0]) * v[0] + (op ? n.p[1] : n.d[1]) * v[1] + (op ? n.p[2] : n.d[2]) * v[2]);
}

// d(orientation + predicted-normal loss)/d(weight of this sample): pure forward quantities
__device__ __forceinline__ float loss_dw(const Normals& n, const float v[3], const RefLoss& L) {
  float dw = 0.f;
  if (L.orient_mult > 0.f) {
    float pm = fminf(0.f, orient_p(n, L.orient_on_pred, v));
    dw += L.orient_mult * pm * pm;
  }
  if (L.prednorm_mult > 0.f) dw += L.prednorm_mult * (1.f - (n.d[0] * n.p[0] + n.d[1] * n.p[1] + n.d[2] * n.p[2]));
  return dw;
}

// The two losses at weight w: values added to st_or / st_pn, adjoints with respect to the normals to a_p / a_d
// (the weights are differentiated through extra_dw)
__device__ __forceinline__ void loss_bwd(const Normals& n, const float v[3], float w, const RefLoss& L, float a_p[3],
                                         float a_d[3], float& st_or, float& st_pn) {
  if (L.orient_mult > 0.f) {
    const bool op = L.orient_on_pred;
    float p = orient_p(n, op, v);
    float pm = fminf(0.f, p);
    st_or += L.orient_mult * w * pm * pm;
    if (p < 0.f) {
      // a += t * -v, fused explicitly: with the destination chosen by a branch the compiler does not always
      // contract a product that both adds share
      const float t = L.orient_mult * w * 2.f * p;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        if (op) a_p[i] = fmaf(t, -v[i], a_p[i]); else a_d[i] = fmaf(t, -v[i], a_d[i]);
      }
    }
  }
  if (L.prednorm_mult > 0.f) {
    float dot = n.d[0] * n.p[0] + n.d[1] * n.p[1] + n.d[2] * n.p[2];
    st_pn += L.prednorm_mult * w * (1.f - dot);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      a_p[i] += -L.prednorm_mult * w * n.d[i];
      a_d[i] += -L.prednorm_mult * w * n.p[i];
    }
  }
}

// Adjoint of load_normals: stores d grad_pred and d raw_grad_density [3, M] of the enabled normals and returns
// d grad_pred (zero when off) in dgp
__device__ __forceinline__ void normals_adjoint(const Normals& n, bool use_p, bool use_d, int64_t M, int64_t m,
                                                const float a_p[3], const float a_d[3], float* __restrict__ d_grad_pred,
                                                float* __restrict__ d_raw_grad_density, float dgp[3]) {
  dgp[0] = dgp[1] = dgp[2] = 0.f;
  if (use_p) {
    neg_normalize_bwd(n.p, n.s_p, n.cl_p, a_p, dgp);
    d_grad_pred[m * 3] = dgp[0]; d_grad_pred[m * 3 + 1] = dgp[1]; d_grad_pred[m * 3 + 2] = dgp[2];
  }
  if (use_d) {
    float dg[3];
    neg_normalize_bwd(n.d, n.s_d, n.cl_d, a_d, dg);
    d_raw_grad_density[m] = dg[0]; d_raw_grad_density[M + m] = dg[1]; d_raw_grad_density[2 * M + m] = dg[2];
  }
}

// stats[4] += orientation loss, stats[5] += predicted-normal loss, one atomic per warp
__device__ __forceinline__ void add_loss_stats(float st_or, float st_pn, float* stats) {
  st_or = warp_sum(st_or);
  st_pn = warp_sum(st_pn);
  if ((threadIdx.x & 31) == 0) {
    if (st_or != 0.f) atomicAdd(&stats[4], st_or);
    if (st_pn != 0.f) atomicAdd(&stats[5], st_pn);
  }
}

__global__ void __launch_bounds__(128)
refdir_fwd_kernel(RefDesc d, const float* __restrict__ ide_mat, const int* __restrict__ ide_ml, int ide_n,
                  const float* __restrict__ grad_pred, const float* __restrict__ raw_rough,
                  const float* __restrict__ raw_grad_density /* [3, M] */, const float* __restrict__ viewdirs,
                  float* __restrict__ normals_pred, float* __restrict__ normals, float* __restrict__ roughness,
                  __nv_bfloat16* __restrict__ slab, RefLoss L, float* __restrict__ extra_dw) {
  __shared__ IdeTab tab;
  if (d.use_ide) load_tab(&tab, ide_mat, ide_ml, ide_n, (1 << (d.deg_view - 1)) + 1);
  for (int64_t m = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; m < d.M; m += (int64_t)gridDim.x * blockDim.x) {
    float v[3];
    load_viewdir(viewdirs, d.S, m, v);
    const Normals nrm = load_normals(d.M, m, d.use_pred_normals, d.use_density_normals, grad_pred, raw_grad_density,
                                     normals_pred, normals);
    const bool up = d.use_pred_normals;
    const float n[3] = {up ? nrm.p[0] : nrm.d[0], up ? nrm.p[1] : nrm.d[1], up ? nrm.p[2] : nrm.d[2]};
    float kappa = 0.f;
    if (d.use_roughness) {
      kappa = softplus_f(raw_rough[m] + d.roughness_bias);
      roughness[m] = kappa;
    }
    if (extra_dw) extra_dw[m] = loss_dw(nrm, v, L);
    const float ndv = n[0] * v[0] + n[1] * v[1] + n[2] * v[2];
    float dir[3] = {v[0], v[1], v[2]};
    if (d.use_reflections) {
      // reflect(-v, n) = 2 (n . -v) n + v
#pragma unroll
      for (int i = 0; i < 3; ++i) dir[i] = v[i] - 2.f * ndv * n[i];
    }
    __nv_bfloat16* out = slab + m * (int64_t)d.ld + d.col0;
    int c = 0;
    if (d.use_ide) {
      float zp[kZMax];
      zp[0] = 1.f;
      for (int k = 1; k < tab.zdeg; ++k) zp[k] = zp[k - 1] * dir[2];
      // (x + iy)^m by repeated multiplication; pairs are listed with m increasing inside each l
      for (int i = 0; i < tab.n; ++i) {
        float P = 0.f;
        for (int k = 0; k < tab.zdeg; ++k) P += zp[k] * tab.mat[k * tab.n + i];
        float cr = 1.f, ci = 0.f;
        for (int q = 0; q < tab.m[i]; ++q) { float t = cr * dir[0] - ci * dir[1]; ci = cr * dir[1] + ci * dir[0]; cr = t; }
        float A = expf(-tab.sigma[i] * kappa);
        out[i] = __float2bfloat16(cr * P * A);
        out[tab.n + i] = __float2bfloat16(ci * P * A);
      }
      c = 2 * tab.n;
    } else {
      // coord.pos_enc(dir, 0, deg_view, append_identity=True)
      out[0] = __float2bfloat16(dir[0]); out[1] = __float2bfloat16(dir[1]); out[2] = __float2bfloat16(dir[2]);
      for (int half = 0; half < 2; ++half)
        for (int l = 0; l < d.deg_view; ++l)
          for (int ch = 0; ch < 3; ++ch) {
            float x = dir[ch] * exp2f((float)l);
            out[3 + half * 3 * d.deg_view + l * 3 + ch] = __float2bfloat16(sinf(half ? x + 1.57079637050628662109375f : x));
          }
      c = 3 + 6 * d.deg_view;
    }
    if (d.use_n_dot_v) out[c++] = __float2bfloat16(ndv);
    for (; d.col0 + c < d.col_end; ++c) out[c] = __float2bfloat16(0.f);
  }
}

__global__ void __launch_bounds__(128)
refdir_bwd_kernel(RefDesc d, RefLoss L, const float* __restrict__ ide_mat, const int* __restrict__ ide_ml, int ide_n,
                  const float* __restrict__ grad_pred, const float* __restrict__ raw_rough,
                  const float* __restrict__ raw_grad_density, const float* __restrict__ viewdirs,
                  const float* __restrict__ weights, __nv_bfloat16* __restrict__ d_slab, int ld_dslab,
                  const float* __restrict__ d_raw_density, const float* __restrict__ d_raw_diffuse,
                  const float* __restrict__ d_raw_tint,
                  float* __restrict__ d_grad_pred, float* __restrict__ d_raw_rough,
                  float* __restrict__ d_raw_grad_density /* [3, M] */,
                  float* __restrict__ stats /* [4]=orientation, [5]=pred normals */) {
  __shared__ IdeTab tab;
  if (d.use_ide) load_tab(&tab, ide_mat, ide_ml, ide_n, (1 << (d.deg_view - 1)) + 1);
  float st_or = 0.f, st_pn = 0.f;
  for (int64_t m = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; m < d.M; m += (int64_t)gridDim.x * blockDim.x) {
    float v[3];
    load_viewdir(viewdirs, d.S, m, v);
    const Normals nrm = load_normals(d.M, m, d.use_pred_normals, d.use_density_normals, grad_pred, raw_grad_density,
                                     nullptr, nullptr);
    const bool up = d.use_pred_normals;
    const float n[3] = {up ? nrm.p[0] : nrm.d[0], up ? nrm.p[1] : nrm.d[1], up ? nrm.p[2] : nrm.d[2]};
    float kappa = 0.f, rin = 0.f;
    if (d.use_roughness) { rin = raw_rough[m] + d.roughness_bias; kappa = softplus_f(rin); }
    const float ndv = n[0] * v[0] + n[1] * v[1] + n[2] * v[2];
    float dir[3] = {v[0], v[1], v[2]};
    if (d.use_reflections) {
#pragma unroll
      for (int i = 0; i < 3; ++i) dir[i] = v[i] - 2.f * ndv * n[i];
    }
    // ---- adjoint of the direction encoding: u = dL/d dir, dkappa
    const __nv_bfloat16* gin = d_slab + m * (int64_t)ld_dslab + d.col0;
    float u[3] = {0.f, 0.f, 0.f}, dkappa = 0.f;
    int c = 0;
    if (d.use_ide) {
      float zp[kZMax];
      zp[0] = 1.f;
      for (int k = 1; k < tab.zdeg; ++k) zp[k] = zp[k - 1] * dir[2];
      for (int i = 0; i < tab.n; ++i) {
        float P = 0.f, dP = 0.f;
        for (int k = 0; k < tab.zdeg; ++k) {
          float co = tab.mat[k * tab.n + i];
          P += zp[k] * co;
          if (k > 0) dP += (float)k * zp[k - 1] * co;
        }
        const int mi = tab.m[i];
        float cr = 1.f, ci = 0.f, er = 0.f, ei = 0.f;      // c = (x+iy)^m, e = m (x+iy)^(m-1)
        for (int q = 0; q < mi; ++q) {
          if (q == mi - 1) { er = (float)mi * cr; ei = (float)mi * ci; }
          float t = cr * dir[0] - ci * dir[1]; ci = cr * dir[1] + ci * dir[0]; cr = t;
        }
        const float A = expf(-tab.sigma[i] * kappa);
        const float gr = __bfloat162float(gin[i]), gi = __bfloat162float(gin[tab.n + i]);
        dkappa += -tab.sigma[i] * A * P * (gr * cr + gi * ci);
        u[2] += A * dP * (gr * cr + gi * ci);
        u[0] += A * P * (gr * er + gi * ei);
        u[1] += A * P * (-gr * ei + gi * er);
      }
      c = 2 * tab.n;
    } else {
      u[0] = __bfloat162float(gin[0]); u[1] = __bfloat162float(gin[1]); u[2] = __bfloat162float(gin[2]);
      for (int half = 0; half < 2; ++half)
        for (int l = 0; l < d.deg_view; ++l)
          for (int ch = 0; ch < 3; ++ch) {
            float sc = exp2f((float)l);
            float x = dir[ch] * sc;
            float g = __bfloat162float(gin[3 + half * 3 * d.deg_view + l * 3 + ch]);
            u[ch] += g * cosf(half ? x + 1.57079637050628662109375f : x) * sc;
          }
      c = 3 + 6 * d.deg_view;
    }
    float a_n[3] = {0.f, 0.f, 0.f};     // dL/d n (normals_to_use)
    if (d.use_n_dot_v) {
      float gq = __bfloat162float(gin[c]);
#pragma unroll
      for (int i = 0; i < 3; ++i) a_n[i] += gq * v[i];
    }
    if (d.use_reflections) {
      // dir = v - 2 (n.v) n  ->  dL/dn = -2 (u.n) v - 2 (n.v) u
      float un = u[0] * n[0] + u[1] * n[1] + u[2] * n[2];
#pragma unroll
      for (int i = 0; i < 3; ++i) a_n[i] += -2.f * un * v[i] - 2.f * ndv * u[i];
    }
    float a_p[3] = {0.f, 0.f, 0.f}, a_d[3] = {0.f, 0.f, 0.f};
    if (d.use_pred_normals) { a_p[0] = a_n[0]; a_p[1] = a_n[1]; a_p[2] = a_n[2]; }
    else { a_d[0] = a_n[0]; a_d[1] = a_n[1]; a_d[2] = a_n[2]; }
    loss_bwd(nrm, v, weights[m], L, a_p, a_d, st_or, st_pn);
    float hg[11];                        // head gradients, in the column order of Wcat (models.py layout)
#pragma unroll
    for (int i = 0; i < 11; ++i) hg[i] = 0.f;
    hg[0] = d_raw_density ? d_raw_density[m] : 0.f;
    normals_adjoint(nrm, d.use_pred_normals, d.use_density_normals, d.M, m, a_p, a_d, d_grad_pred, d_raw_grad_density,
                    hg + 1);
    if (d_raw_diffuse) { hg[4] = d_raw_diffuse[m * 3]; hg[5] = d_raw_diffuse[m * 3 + 1]; hg[6] = d_raw_diffuse[m * 3 + 2]; }
    if (d_raw_tint) { hg[7] = d_raw_tint[m * 3]; hg[8] = d_raw_tint[m * 3 + 1]; hg[9] = d_raw_tint[m * 3 + 2]; }
    if (d.use_roughness) { hg[10] = dkappa * sigmoid_f(rin); d_raw_rough[m] = hg[10]; }
    // the consumed direction-encoding gradient columns are re-used for the head gradients: together
    // with the bottleneck gradient in columns [0, col0) they form the A operand of one dgrad GEMM
    __nv_bfloat16* hs = d_slab + m * (int64_t)ld_dslab + d.col0;
#pragma unroll
    for (int i = 0; i < 11; ++i) hs[i] = __float2bfloat16(hg[i]);
    for (int i = 11; d.col0 + i < d.col_end; ++i) hs[i] = __float2bfloat16(0.f);
  }
  add_loss_stats(st_or, st_pn, stats);
}

// Colourless form of the stage: an MLP with disable_rgb (a proposal MLP) whose normals feed only the
// orientation / predicted-normal losses and the renderings.  The normals and loss pieces of refdir_fwd/bwd, no
// direction encoding.  A NULL grad_pred / raw_grad_density switches that normal off, and viewdirs / weights are
// read only when a loss needs them.
__global__ void __launch_bounds__(128)
normals_fwd_kernel(int64_t M, int S, const float* __restrict__ grad_pred,
                   const float* __restrict__ raw_grad_density /* [3, M] */, const float* __restrict__ viewdirs,
                   float* __restrict__ normals_pred, float* __restrict__ normals, RefLoss L,
                   float* __restrict__ extra_dw) {
  for (int64_t m = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; m < M; m += (int64_t)gridDim.x * blockDim.x) {
    const Normals nrm = load_normals(M, m, grad_pred != nullptr, raw_grad_density != nullptr, grad_pred,
                                     raw_grad_density, normals_pred, normals);
    if (extra_dw) {
      float v[3] = {0.f, 0.f, 0.f};
      if (L.orient_mult > 0.f) load_viewdir(viewdirs, S, m, v);
      extra_dw[m] = loss_dw(nrm, v, L);
    }
  }
}

__global__ void __launch_bounds__(128)
normals_bwd_kernel(int64_t M, int S, RefLoss L, const float* __restrict__ grad_pred,
                   const float* __restrict__ raw_grad_density, const float* __restrict__ viewdirs,
                   const float* __restrict__ weights, const float* __restrict__ d_raw_density,
                   const float* __restrict__ d_raw_rgb, int64_t ld_raw, float* __restrict__ d_grad_pred, float* __restrict__ d_raw_grad_density /* [3, M] */,
                   __nv_bfloat16* __restrict__ head_grads, int64_t ld_head_grads,
                   float* __restrict__ stats /* [4]=orientation, [5]=pred normals */) {
  float st_or = 0.f, st_pn = 0.f;
  for (int64_t m = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; m < M; m += (int64_t)gridDim.x * blockDim.x) {
    const bool use_p = grad_pred != nullptr, use_d = raw_grad_density != nullptr;
    const Normals nrm = load_normals(M, m, use_p, use_d, grad_pred, raw_grad_density, nullptr, nullptr);
    float a_p[3] = {0.f, 0.f, 0.f}, a_d[3] = {0.f, 0.f, 0.f};
    if (L.orient_mult > 0.f || L.prednorm_mult > 0.f) {
      const float w = weights[m];      // issued before the ray index's division, which hides its latency
      float v[3] = {0.f, 0.f, 0.f};
      if (L.orient_mult > 0.f) load_viewdir(viewdirs, S, m, v);
      loss_bwd(nrm, v, w, L, a_p, a_d, st_or, st_pn);
    }
    float dgp[3];
    normals_adjoint(nrm, use_p, use_d, M, m, a_p, a_d, d_grad_pred, d_raw_grad_density, dgp);
    if (head_grads) {
      // [d raw_density | d grad_pred]: the A operand of the dgrad GEMM into the trunk against [w_density | W_grad_pred]
      __nv_bfloat16* hs = head_grads + m * ld_head_grads;
      *reinterpret_cast<uint32_t*>(hs) = pack_bf16(d_raw_density[m * ld_raw], dgp[0]);
      *reinterpret_cast<uint32_t*>(hs + 2) = pack_bf16(dgp[1], dgp[2]);
      if (d_raw_rgb) {
        // [.. | d raw_rgb]: the rgb head of a view-independent model reads the same trunk output
        const float* g = d_raw_rgb + m * ld_raw;
        *reinterpret_cast<uint32_t*>(hs + 4) = pack_bf16(g[0], g[1]);
        *reinterpret_cast<uint32_t*>(hs + 6) = pack_bf16(g[2], 0.f);
      }
    }
  }
  if (stats) add_loss_stats(st_or, st_pn, stats);
}

// out[r, n] (bf16) = mask(r mod mod, n) ? rowv[r] * colv[n] : 0     (start of the tangent backward chain)
__global__ void outer_mask_kernel(int64_t R, int N, int64_t mod, const float* __restrict__ rowv,
                                  const float* __restrict__ colv, const uint32_t* __restrict__ maskbits,
                                  int64_t ldmb, __nv_bfloat16* __restrict__ out, int64_t ldo) {
  const int64_t total = R * (N / 8);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i / (N / 8);
    int c8 = (int)(i - r * (N / 8)) * 8;
    float rv = rowv[r];
    uint32_t bits = maskbits ? maskbits[(mod ? r % mod : r) * ldmb + (c8 >> 5)] >> (c8 & 31) : 0xffu;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = ((bits >> e) & 1u) ? rv * colv[c8 + e] : 0.f;
    uint4 o;
    o.x = pack_bf16(v[0], v[1]); o.y = pack_bf16(v[2], v[3]); o.z = pack_bf16(v[4], v[5]); o.w = pack_bf16(v[6], v[7]);
    *reinterpret_cast<uint4*>(out + r * ldo + c8) = o;
  }
}

// One trunk layer of the tangent backward through a smooth activation (mnrf.h): per [row, 8 columns] of z,
//   du_s = a'(z) T_s,   g (+)= a''(z) sum_s T_s u_s        (s = the three tangent streams, rows m, M + m, 2M + m)
// du may alias T: each thread reads its T chunk of every stream before it writes the same chunk of du.
__global__ void __launch_bounds__(256)
act_tangent_bwd_kernel(int64_t M, int N, int act, const __nv_bfloat16* __restrict__ z, int64_t ldz,
                       const __nv_bfloat16* t_adj, int64_t ldt, const __nv_bfloat16* __restrict__ u, int64_t ldu,
                       __nv_bfloat16* du, int64_t lddu, __nv_bfloat16* __restrict__ g, int64_t ldg, int accumulate) {
  const int64_t total = M * (N / 8);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / (N / 8);
    const int c8 = (int)(i - r * (N / 8)) * 8;
    const uint4 zv = __ldg(reinterpret_cast<const uint4*>(z + r * ldz + c8));
    uint4 tv[3], uv[3];
#pragma unroll
    for (int s = 0; s < 3; ++s) {
      tv[s] = *reinterpret_cast<const uint4*>(t_adj + (s * M + r) * ldt + c8);
      uv[s] = __ldg(reinterpret_cast<const uint4*>(u + (s * M + r) * ldu + c8));
    }
    float zf[8], d1[8], gs[8];
    const uint32_t zw[4] = {zv.x, zv.y, zv.z, zv.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) { zf[2 * q] = bf16_lo(zw[q]); zf[2 * q + 1] = bf16_hi(zw[q]); }
#pragma unroll
    for (int e = 0; e < 8; ++e) { d1[e] = act_d1(act, zf[e]); gs[e] = 0.f; }
#pragma unroll
    for (int s = 0; s < 3; ++s) {
      const uint32_t tw[4] = {tv[s].x, tv[s].y, tv[s].z, tv[s].w}, uw[4] = {uv[s].x, uv[s].y, uv[s].z, uv[s].w};
      uint32_t o[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float t0 = bf16_lo(tw[q]), t1 = bf16_hi(tw[q]);
        gs[2 * q] += t0 * bf16_lo(uw[q]);
        gs[2 * q + 1] += t1 * bf16_hi(uw[q]);
        o[q] = pack_bf16(d1[2 * q] * t0, d1[2 * q + 1] * t1);
      }
      *reinterpret_cast<uint4*>(du + (s * M + r) * lddu + c8) = make_uint4(o[0], o[1], o[2], o[3]);
    }
    float prev[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (accumulate) {
      const uint4 gv = *reinterpret_cast<const uint4*>(g + r * ldg + c8);
      const uint32_t gw[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) { prev[2 * q] = bf16_lo(gw[q]); prev[2 * q + 1] = bf16_hi(gw[q]); }
    }
    uint32_t o[4];
#pragma unroll
    for (int q = 0; q < 4; ++q)
      o[q] = pack_bf16(prev[2 * q] + act_d2(act, zf[2 * q]) * gs[2 * q],
                       prev[2 * q + 1] + act_d2(act, zf[2 * q + 1]) * gs[2 * q + 1]);
    *reinterpret_cast<uint4*>(g + r * ldg + c8) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// Host checks shared by mnrf_refdir_fwd and mnrf_refdir_bwd: the IDE tables, the normals and roughness the flags
// switch on, the normals the losses read, and the slab columns [col0, col_end) within a row of `ld` holding
// `min_cols` (the encoding in the forward, the encoding and the 11 head gradients in the backward).  Returns the
// MNRF_CHECK code.
inline int check_refdir(const char* fn, const mnrf_refdir_desc* d, const float* ide_mat, const int32_t* ide_ml,
                        const float* grad_pred, const float* raw_grad_density, const float* raw_rough,
                        float orient_mult, float prednorm_mult, int32_t orient_on_pred, bool losses, int64_t ld,
                        bool bwd) {
  MNRF_CHECK(d->num_samples > 0, "%s: num_samples must be positive", fn);
  MNRF_CHECK(!d->use_ide || (ide_mat && ide_ml && d->deg_view >= 1 && d->deg_view <= 5),
             "Only deg_view of at most 5 is numerically stable.");
  int ide_n = 0;
  for (int i = 0; d->use_ide && i < d->deg_view; ++i) ide_n += (1 << i) + 1;
  MNRF_CHECK(!d->use_ide || d->ide_n == ide_n, "%s: ide_n %d does not match deg_view %d (%d (m, l) pairs)", fn,
             d->ide_n, d->deg_view, ide_n);
  MNRF_CHECK(d->use_ide || d->deg_view >= 0, "%s: deg_view must not be negative", fn);
  MNRF_CHECK(!d->use_ide || d->use_roughness, "%s: the IDE needs a roughness (kappa_inv)", fn);
  MNRF_CHECK(d->use_pred_normals || d->use_density_normals || !(d->use_reflections || d->use_n_dot_v),
             "Normals must be computed for reflection directions.");
  MNRF_CHECK(!d->use_pred_normals || grad_pred, "%s: use_pred_normals needs grad_pred", fn);
  MNRF_CHECK(!d->use_density_normals || raw_grad_density, "%s: use_density_normals needs raw_grad_density", fn);
  MNRF_CHECK(!d->use_roughness || raw_rough, "%s: use_roughness needs raw_rough", fn);
  MNRF_CHECK(!losses || !(orient_mult > 0.f) || (orient_on_pred ? d->use_pred_normals : d->use_density_normals),
             "Normals cannot be None if orientation loss is on.");
  MNRF_CHECK(!losses || !(prednorm_mult > 0.f) || (d->use_pred_normals && d->use_density_normals),
             "Predicted normals and gradient normals cannot be None if predicted normal loss is on.");
  const int64_t enc = (d->use_ide ? 2 * (int64_t)ide_n : 3 + 6 * (int64_t)d->deg_view) + (d->use_n_dot_v ? 1 : 0);
  const int64_t min_cols = bwd ? std::max<int64_t>(enc, 11) : enc;
  MNRF_CHECK(d->col0 >= 0 && (int64_t)d->col_end - d->col0 >= min_cols && d->col_end <= ld,
             "%s: the slab columns [%d, %d) of a row of %lld must hold %lld columns", fn, d->col0, d->col_end,
             (long long)ld, (long long)min_cols);
  return 0;
}

}  // namespace mnrf

extern "C" int mnrf_refdir_fwd(const mnrf_refdir_desc* d, const float* ide_mat, const int32_t* ide_ml,
                               const float* grad_pred, const float* raw_rough, const float* raw_grad_density,
                               const float* viewdirs, float* normals_pred, float* normals, float* roughness,
                               mnrf_bf16* slab, float orient_mult, float prednorm_mult, int32_t orient_on_pred,
                               float* extra_dw, mnrf_stream stream) {
  using namespace mnrf;
  if (d && d->M == 0) return 0;
  MNRF_CHECK(d && viewdirs && slab, "mnrf_refdir_fwd: null pointer");
  if (check_refdir("mnrf_refdir_fwd", d, ide_mat, ide_ml, grad_pred, raw_grad_density, raw_rough, orient_mult,
                   prednorm_mult, orient_on_pred, extra_dw != nullptr, d->ld, false))
    return 1;
  MNRF_CHECK(!d->use_roughness || roughness, "mnrf_refdir_fwd: use_roughness needs the roughness output");
  if (d->M == 0) return 0;
  RefDesc r{d->M, d->num_samples, d->use_pred_normals, d->use_density_normals, d->use_reflections, d->use_ide,
            d->use_n_dot_v, d->use_roughness, d->deg_view, d->roughness_bias, d->ld, d->col0, d->col_end};
  int blocks = (int)std::min<int64_t>((d->M + 127) / 128, (int64_t)mnrf_num_sms() * 16);
  refdir_fwd_kernel<<<blocks, 128, 0, (cudaStream_t)stream>>>(
      r, ide_mat, ide_ml, d->ide_n, grad_pred, raw_rough, raw_grad_density, viewdirs, normals_pred, normals,
      roughness, reinterpret_cast<__nv_bfloat16*>(slab), RefLoss{orient_mult, prednorm_mult, orient_on_pred},
      extra_dw);
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_refdir_bwd(const mnrf_refdir_desc* d, const float* ide_mat, const int32_t* ide_ml,
                               const float* grad_pred, const float* raw_rough, const float* raw_grad_density,
                               const float* viewdirs, const float* weights, mnrf_bf16* d_slab,
                               int32_t ld_dslab, float orient_mult, float prednorm_mult, int32_t orient_on_pred,
                               const float* d_raw_density, const float* d_raw_diffuse, const float* d_raw_tint,
                               float* d_grad_pred, float* d_raw_rough, float* d_raw_grad_density,
                               float* stats, mnrf_stream stream) {
  using namespace mnrf;
  if (d && d->M == 0) return 0;
  MNRF_CHECK(d && viewdirs && weights && d_slab && stats, "mnrf_refdir_bwd: null pointer");
  if (check_refdir("mnrf_refdir_bwd", d, ide_mat, ide_ml, grad_pred, raw_grad_density, raw_rough, orient_mult,
                   prednorm_mult, orient_on_pred, true, ld_dslab, true))
    return 1;
  MNRF_CHECK(!d->use_roughness || d_raw_rough, "mnrf_refdir_bwd: use_roughness needs d_raw_rough");
  MNRF_CHECK(!d->use_pred_normals || d_grad_pred, "mnrf_refdir_bwd: use_pred_normals needs d_grad_pred");
  MNRF_CHECK(!d->use_density_normals || d_raw_grad_density,
             "mnrf_refdir_bwd: use_density_normals needs d_raw_grad_density");
  if (d->M == 0) return 0;
  RefDesc r{d->M, d->num_samples, d->use_pred_normals, d->use_density_normals, d->use_reflections, d->use_ide,
            d->use_n_dot_v, d->use_roughness, d->deg_view, d->roughness_bias, d->ld, d->col0, d->col_end};
  RefLoss L{orient_mult, prednorm_mult, orient_on_pred};
  int blocks = (int)std::min<int64_t>((d->M + 127) / 128, (int64_t)mnrf_num_sms() * 16);
  refdir_bwd_kernel<<<blocks, 128, 0, (cudaStream_t)stream>>>(
      r, L, ide_mat, ide_ml, d->ide_n, grad_pred, raw_rough, raw_grad_density, viewdirs, weights,
      reinterpret_cast<__nv_bfloat16*>(d_slab), ld_dslab, d_raw_density, d_raw_diffuse, d_raw_tint, d_grad_pred,
      d_raw_rough, d_raw_grad_density, stats);
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_outer_mask(int64_t rows, int32_t n, int64_t mask_mod, const float* rowv, const float* colv,
                               const uint32_t* maskbits, int64_t ldmaskbits, mnrf_bf16* out, int64_t ldo,
                               mnrf_stream stream) {
  using namespace mnrf;
  if (rows == 0) return 0;
  MNRF_CHECK(rowv && colv && out, "mnrf_outer_mask: null pointer");
  MNRF_CHECK(n % 32 == 0 && ldo % 8 == 0, "mnrf_outer_mask: N %% 32 == 0 and ld %% 8 == 0 required");
  MNRF_CHECK((reinterpret_cast<uintptr_t>(out) & 15) == 0, "mnrf_outer_mask: out must be 16-byte aligned");
  int64_t total = rows * (n / 8);
  int blocks = (int)std::min<int64_t>((total + 255) / 256, (int64_t)mnrf_num_sms() * 16);
  outer_mask_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(rows, n, mask_mod, rowv, colv, maskbits, ldmaskbits,
                                                            reinterpret_cast<__nv_bfloat16*>(out), ldo);
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_normals_fwd(int64_t M, int32_t num_samples, const float* grad_pred, const float* raw_grad_density,
                                const float* viewdirs, float* normals_pred, float* normals, float orient_mult,
                                float prednorm_mult, int32_t orient_on_pred, float* extra_dw, mnrf_stream stream) {
  using namespace mnrf;
  if (M == 0) return 0;
  MNRF_CHECK(grad_pred || raw_grad_density, "mnrf_normals_fwd: no normals to compute");
  MNRF_CHECK(!grad_pred == !normals_pred && !raw_grad_density == !normals, "mnrf_normals_fwd: null pointer");
  MNRF_CHECK(!extra_dw || !(orient_mult > 0.f) || (viewdirs && (orient_on_pred ? grad_pred : raw_grad_density)),
             "Normals cannot be None if orientation loss is on.");
  MNRF_CHECK(!extra_dw || !(prednorm_mult > 0.f) || (grad_pred && raw_grad_density),
             "Predicted normals and gradient normals cannot be None if predicted normal loss is on.");
  MNRF_CHECK(num_samples > 0, "mnrf_normals_fwd: num_samples must be positive");
  int blocks = (int)std::min<int64_t>((M + 127) / 128, (int64_t)mnrf_num_sms() * 16);
  normals_fwd_kernel<<<blocks, 128, 0, (cudaStream_t)stream>>>(
      M, num_samples, grad_pred, raw_grad_density, viewdirs, normals_pred, normals,
      RefLoss{orient_mult, prednorm_mult, orient_on_pred}, extra_dw);
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_normals_bwd(int64_t M, int32_t num_samples, const float* grad_pred, const float* raw_grad_density,
                                const float* viewdirs, const float* weights, float orient_mult, float prednorm_mult,
                                int32_t orient_on_pred, const float* d_raw_density, const float* d_raw_rgb,
                                int64_t ld_raw, float* d_grad_pred, float* d_raw_grad_density, mnrf_bf16* head_grads,
                                int64_t ld_head_grads, float* stats, mnrf_stream stream) {
  using namespace mnrf;
  if (M == 0) return 0;
  MNRF_CHECK(grad_pred || raw_grad_density, "mnrf_normals_bwd: no normals to differentiate");
  MNRF_CHECK(!grad_pred == !d_grad_pred && !raw_grad_density == !d_raw_grad_density, "mnrf_normals_bwd: null pointer");
  const bool losses = orient_mult > 0.f || prednorm_mult > 0.f;
  MNRF_CHECK(!losses || (weights && stats), "mnrf_normals_bwd: the losses need weights and a stats row");
  MNRF_CHECK(!(orient_mult > 0.f) || (viewdirs && (orient_on_pred ? grad_pred : raw_grad_density)),
             "Normals cannot be None if orientation loss is on.");
  MNRF_CHECK(!(prednorm_mult > 0.f) || (grad_pred && raw_grad_density),
             "Predicted normals and gradient normals cannot be None if predicted normal loss is on.");
  MNRF_CHECK(!head_grads || (grad_pred && d_raw_density && ld_head_grads >= 4 && ld_head_grads % 2 == 0 &&
                             (reinterpret_cast<uintptr_t>(head_grads) & 3) == 0),
             "mnrf_normals_bwd: head_grads needs grad_pred, d_raw_density and 4 aligned columns");
  MNRF_CHECK(!d_raw_rgb || (head_grads && ld_head_grads >= 8), "mnrf_normals_bwd: d_raw_rgb needs 8 head_grads columns");
  if (ld_raw <= 0) ld_raw = 1;
  MNRF_CHECK(num_samples > 0, "mnrf_normals_bwd: num_samples must be positive");
  int blocks = (int)std::min<int64_t>((M + 127) / 128, (int64_t)mnrf_num_sms() * 16);
  normals_bwd_kernel<<<blocks, 128, 0, (cudaStream_t)stream>>>(
      M, num_samples, RefLoss{orient_mult, prednorm_mult, orient_on_pred}, grad_pred, raw_grad_density, viewdirs,
      weights, d_raw_density, d_raw_rgb, ld_raw, d_grad_pred, d_raw_grad_density,
      reinterpret_cast<__nv_bfloat16*>(head_grads),
      ld_head_grads, losses ? stats : nullptr);
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_act_tangent_bwd(int64_t M, int32_t n, int32_t act, const mnrf_bf16* z, int64_t ldz,
                                    const mnrf_bf16* t_adj, int64_t ldt, const mnrf_bf16* u, int64_t ldu, mnrf_bf16* du,
                                    int64_t lddu, mnrf_bf16* g, int64_t ldg, int32_t accumulate, mnrf_stream stream) {
  using namespace mnrf;
  if (M == 0) return 0;
  MNRF_CHECK(z && t_adj && u && du && g, "mnrf_act_tangent_bwd: null pointer");
  MNRF_CHECK(act == MNRF_ACT_SOFTPLUS || act == MNRF_ACT_SILU, "mnrf_act_tangent_bwd: act %d is not a smooth activation",
             act);
  MNRF_CHECK(n % 8 == 0 && ldz % 8 == 0 && ldt % 8 == 0 && ldu % 8 == 0 && lddu % 8 == 0 && ldg % 8 == 0,
             "mnrf_act_tangent_bwd: N and every pitch must be multiples of 8");
  MNRF_CHECK(((uintptr_t)z | (uintptr_t)t_adj | (uintptr_t)u | (uintptr_t)du | (uintptr_t)g) % 16 == 0,
             "mnrf_act_tangent_bwd: pointers must be 16-byte aligned");
  const int64_t total = M * (n / 8);
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, (int64_t)mnrf_num_sms() * 16);
  act_tangent_bwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(
      M, n, act, reinterpret_cast<const __nv_bfloat16*>(z), ldz, reinterpret_cast<const __nv_bfloat16*>(t_adj), ldt,
      reinterpret_cast<const __nv_bfloat16*>(u), ldu, reinterpret_cast<__nv_bfloat16*>(du), lddu,
      reinterpret_cast<__nv_bfloat16*>(g), ldg, accumulate);
  MNRF_LAUNCH_CHECK();
  return 0;
}
