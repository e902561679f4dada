// Ray casting + integrated positional encoding: one warp owns one ray, loops over its samples.
//
// Replaces (reference file:line): coord.construct_ray_warps s_to_t coord.py:63-99;
// render.cast_rays render.py:103-127 -> conical_frustum_to_gaussian :44-78 (stable form) /
// cylinder_to_gaussian :81-100 -> lift_gaussian :21-41 (diag=False, models.py:213);
// coord.contract + track_linearize coord.py:21-60 (closed-form Jacobian, SURVEY App. B);
// coord.lift_and_diagonalize :129-133; coord.integrated_pos_enc :107-126 with
// math.safe_sin math.py:26-38.  Also coord.pos_enc :136-147 for the view directions.
//
// Output: bf16 feature rows written straight into the MLP's input buffer (row stride
// ld_feat), staged through shared memory so that each lane stores 16 B.
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "contract.cuh"

namespace mnrf {

struct Gauss {
  float mean[3];
  float cov[3][3];
};

__device__ __forceinline__ void cast_one(int ray_shape, float t0, float t1, const float o[3],
                                         const float dvec[3], float radius, Gauss& g) {
  float t_mean, t_var, r_var;
  if (ray_shape == MNRF_RAY_CONE) {
    float mu = (t0 + t1) / 2.f;
    float hw = (t1 - t0) / 2.f;
    float hw2 = hw * hw, mu2 = mu * mu;
    float hw4 = hw2 * hw2;
    float denom = fmaxf(kEps, 3.f * mu2 + hw2);
    t_mean = mu + (2.f * mu * hw2) / denom;
    t_var = hw2 / 3.f - (4.f / 15.f) * hw4 * (12.f * mu2 - hw2) / (denom * denom);
    r_var = mu2 / 4.f + (5.f / 12.f) * hw2 - (4.f / 15.f) * hw4 / denom;
    r_var = r_var * (radius * radius);
  } else {
    t_mean = (t0 + t1) / 2.f;
    r_var = (radius * radius) / 4.f;
    float dt = t1 - t0;
    t_var = (dt * dt) / 12.f;
  }
  float dmag = fmaxf(1e-10f, dvec[0] * dvec[0] + dvec[1] * dvec[1] + dvec[2] * dvec[2]);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    g.mean[i] = dvec[i] * t_mean + o[i];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      float d_outer = dvec[i] * dvec[j];
      float null_outer = (i == j ? 1.f : 0.f) - dvec[i] * (dvec[j] / dmag);
      g.cov[i][j] = t_var * d_outer + r_var * null_outer;
    }
  }
}

__device__ __forceinline__ void contract_gauss(Gauss& g) {
  float x0 = g.mean[0], x1 = g.mean[1], x2 = g.mean[2];
  float m = fmaxf(kEps, x0 * x0 + x1 * x1 + x2 * x2);
  if (m <= 1.f) return;
  float r = sqrtf(m);
  float scale = (2.f * r - 1.f) / m;
  float s = 2.f / r - 1.f / m;
  float c = 2.f / (m * m) - 2.f / (m * r);
  float x[3] = {x0, x1, x2};
  float J[3][3], T[3][3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) J[i][j] = (i == j ? s : 0.f) + c * x[i] * x[j];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      T[i][j] = J[i][0] * g.cov[0][j] + J[i][1] * g.cov[1][j] + J[i][2] * g.cov[2][j];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      g.cov[i][j] = T[i][0] * J[j][0] + T[i][1] * J[j][1] + T[i][2] * J[j][2];
#pragma unroll
  for (int i = 0; i < 3; ++i) g.mean[i] = scale * x[i];
}

// Tangent rows through the contraction.  z = s x and Sigma' = J Sigma J^T.  With r = |x|, xh = x / r and
// P = xh xh^T, outside the unit ball J = s (I - P) + q P with s = 2/r - 1/r^2 and q = 1/r^2 (inside: J = I).
// For a basis vector b write beta = xh.b, b_t = b - beta xh, u = J b = s b_t + q beta xh and v = Sigma u
// (pre-warp Sigma), gamma = xh.v, v_t = v - gamma xh.  The lifted mean and variance move with world axis a as
//   d(b.z)/dx_a          = u_a
//   d(b^T Sigma' b)/dx_a = 2 [ xh_a (s_r (b_t.v) + q_r beta gamma) + s_r (beta (v_t)_a + gamma (b_t)_a) ]
// with s_r = ds/dr = -2 (r - 1) / r^3 (which is also (q - s) / r, the factor of dP/dx) and q_r = -2 / r^3, both 0
// inside the ball.  Every term there is of the size of the result: written with c = 2/r^4 - 2/r^3 in
// J = s I + c x x^T instead, the terms grow with r against their sum and fp32 loses the variance term from
// |x| ~ 1e3 on.  Phase A keeps xh (0 inside the ball), the pre-warp Sigma (6 unique entries) and (s, q, s_r, q_r)
// beside the warped Gaussian.
struct ContractTerms {
  float xh[3], cov[6], s, q, s_r, q_r;
};

__device__ __forceinline__ void contract_terms(const Gauss& g, ContractTerms& t) {
  const float x0 = g.mean[0], x1 = g.mean[1], x2 = g.mean[2];
  t.cov[0] = g.cov[0][0]; t.cov[1] = g.cov[0][1]; t.cov[2] = g.cov[0][2];
  t.cov[3] = g.cov[1][1]; t.cov[4] = g.cov[1][2]; t.cov[5] = g.cov[2][2];
  const float m = fmaxf(kEps, x0 * x0 + x1 * x1 + x2 * x2);
  t.xh[0] = t.xh[1] = t.xh[2] = 0.f;
  t.s = 1.f; t.q = 1.f; t.s_r = 0.f; t.q_r = 0.f;
  if (m <= 1.f) return;
  const float r = sqrtf(m);
  const float ir = 1.f / r;
  t.xh[0] = x0 * ir; t.xh[1] = x1 * ir; t.xh[2] = x2 * ir;
  t.s = 2.f / r - 1.f / m;
  t.q = 1.f / m;
  t.q_r = -2.f / (m * r);
  t.s_r = (r - 1.f) * t.q_r;
}

// smem: basis[3K] (block) | per warp: tdist[S+1] | gauss[S][stride] | lift_mean[K] | lift_var[K] |
//       (Contract: d lift_mean[3][K] | d lift_var[3][K]) | row[feat_cols] bf16 | 3 tangent rows
constexpr int kGaussStride = 13;   // 12 floats (mean 3 + cov 9), padded against bank conflicts
constexpr int kContractStride = 25;   // + xh 3, pre-warp cov 6, (s, q, s_r, q_r) 4: odd against bank conflicts

// Phase A of the general encoder for one Gaussian: stores it at gp (stride floats: kGaussStride, or kContractStride
// with the terms of the tangent rows through the contraction ahead of the warp), contracted when d.warp_contract.
template <bool Contract>
__device__ __forceinline__ void store_gauss(const mnrf_encode_desc& d, Gauss& g, float* gp) {
  if (Contract) {
    ContractTerms t;
    contract_terms(g, t);
#pragma unroll
    for (int i = 0; i < 3; ++i) gp[12 + i] = t.xh[i];
#pragma unroll
    for (int i = 0; i < 6; ++i) gp[15 + i] = t.cov[i];
    gp[21] = t.s; gp[22] = t.q; gp[23] = t.s_r; gp[24] = t.q_r;
  }
  if (d.warp_contract) contract_gauss(g);
  gp[0] = g.mean[0]; gp[1] = g.mean[1]; gp[2] = g.mean[2];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) gp[3 + i * 3 + j] = g.cov[i][j];
}

// The general encoder's per-warp shared memory: lift scratch and staged rows
struct TangentScratch {
  float *lm, *lv, *dlm, *dlv;      // lifted mean / variance [K]; Contract: their derivatives [dir][K]
  __nv_bfloat16 *row, *trow;       // feature row, then (tfeat) three tangent rows, trow_elems apart
  int trow_elems, row_bytes;
};

// Phase B of the general encoder for one Gaussian (stored at gp by store_gauss): lift onto the basis, then write
// feature row m (bf16, fp32 copy when feat_f32 is given) and, with tfeat, the tangent rows dir * M_total + m,
// d feature / d mean_dir.  Shared by the ray and the point encoder.
template <bool Contract>
__device__ __forceinline__ void gauss_tangent_rows(const mnrf_encode_desc& d, const float* gp, const float* sb,
                                                   const TangentScratch& ws, size_t m, size_t M_total,
                                                   __nv_bfloat16* __restrict__ feat, float* __restrict__ feat_f32,
                                                   __nv_bfloat16* __restrict__ tfeat, int ld_tfeat, int lane) {
  const int K = d.basis_k, L = d.max_deg - d.min_deg, KL = K * L;
  float* lm = ws.lm;
  float* lv = ws.lv;
  float* dlm = ws.dlm;
  float* dlv = ws.dlv;
  __nv_bfloat16* row = ws.row;
  __nv_bfloat16* trow = ws.trow;
  const int trow_elems = ws.trow_elems, row_bytes = ws.row_bytes;
  // (l, k) of feature f = l*K + k advance by 32 features per iteration without integer division
  const int q32 = 32 / K, r32 = 32 - q32 * K;
  const int l_first = lane / K, k_first = lane - l_first * K;
  for (int k = lane; k < K; k += 32) {
    float b0 = sb[k * 3 + 0], b1 = sb[k * 3 + 1], b2 = sb[k * 3 + 2];
    lm[k] = gp[0] * b0 + gp[1] * b1 + gp[2] * b2;
    float c0 = gp[3] * b0 + gp[4] * b1 + gp[5] * b2;
    float c1 = gp[6] * b0 + gp[7] * b1 + gp[8] * b2;
    float c2 = gp[9] * b0 + gp[10] * b1 + gp[11] * b2;
    lv[k] = d.disable_integration ? 0.f : (b0 * c0 + b1 * c1 + b2 * c2);
    if (Contract) {
      const float b[3] = {b0, b1, b2};
      const float* xh = gp + 12;
      const float* cv = gp + 15;                 // xx xy xz yy yz zz
      const float sj = gp[21], qj = gp[22], s_r = gp[23], q_r = gp[24];
      const float beta = xh[0] * b0 + xh[1] * b1 + xh[2] * b2;
      float bt[3], u[3], v[3], vt[3];
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        bt[i] = b[i] - beta * xh[i];
        u[i] = sj * bt[i] + (qj * beta) * xh[i];
      }
      v[0] = cv[0] * u[0] + cv[1] * u[1] + cv[2] * u[2];
      v[1] = cv[1] * u[0] + cv[3] * u[1] + cv[4] * u[2];
      v[2] = cv[2] * u[0] + cv[4] * u[1] + cv[5] * u[2];
      const float gamma = xh[0] * v[0] + xh[1] * v[1] + xh[2] * v[2];
#pragma unroll
      for (int i = 0; i < 3; ++i) vt[i] = v[i] - gamma * xh[i];
      const float btv = bt[0] * v[0] + bt[1] * v[1] + bt[2] * v[2];
      const float radial = s_r * btv + q_r * (beta * gamma);
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        dlm[a * K + k] = u[a];
        dlv[a * K + k] = d.disable_integration ? 0.f
                                               : 2.f * (xh[a] * radial + s_r * (beta * vt[a] + gamma * bt[a]));
      }
    }
  }
  __syncwarp();
  int l = l_first, k = k_first;
  for (int f = lane; f < KL; f += 32) {
    const float sc = __int_as_float((127 + d.min_deg + l) << 23);       // 2^(min_deg + l)
    float y = lm[k] * sc;
    float v = lv[k] * (sc * sc);
    float e = __expf(-0.5f * v);
    float fs, fc;
    if (tfeat) {
      // d/d mean_dir of e * safe_sin(lm * sc) = e * cos(reduced arg) * sc * basis[k][dir]
      float s0, c0, s1, c1;
      safe_sincos_fast(y, s0, c0);
      safe_sincos_fast(y + 1.57079637050628662109375f, s1, c1);
      fs = e * s0;
      fc = e * s1;
      if (Contract) {
        // d feature = e cos(y) sc d lift_mean - 1/2 sc^2 feature d lift_var
        const float esc = e * sc, hsc2 = 0.5f * (sc * sc);
#pragma unroll
        for (int dir = 0; dir < 3; ++dir) {
          const float dm = dlm[dir * K + k] * esc, dvar = dlv[dir * K + k] * hsc2;
          trow[dir * trow_elems + f] = __float2bfloat16(c0 * dm - fs * dvar);
          trow[dir * trow_elems + KL + f] = __float2bfloat16(c1 * dm - fc * dvar);
        }
      } else {
#pragma unroll
        for (int dir = 0; dir < 3; ++dir) {
          const float bk = sb[k * 3 + dir] * sc * e;
          trow[dir * trow_elems + f] = __float2bfloat16(c0 * bk);
          trow[dir * trow_elems + KL + f] = __float2bfloat16(c1 * bk);
        }
      }
    } else {
      fs = e * safe_sin_fast(y);
      fc = e * safe_sin_fast(y + 1.57079637050628662109375f);
    }
    row[f] = __float2bfloat16(fs);
    row[KL + f] = __float2bfloat16(fc);
    if (feat_f32) {
      feat_f32[m * (2 * KL) + f] = fs;
      feat_f32[m * (2 * KL) + KL + f] = fc;
    }
    k += r32;
    l += q32;
    if (k >= K) { k -= K; l += 1; }
  }
  __syncwarp();
  const uint4* src = reinterpret_cast<const uint4*>(row);
  uint4* dst = reinterpret_cast<uint4*>(feat + m * (size_t)d.ld_feat);
  for (int c = lane; c < row_bytes / 16; c += 32) dst[c] = src[c];
  if (tfeat) {
#pragma unroll
    for (int dir = 0; dir < 3; ++dir) {
      const uint4* ts = reinterpret_cast<const uint4*>(trow + dir * trow_elems);
      uint4* td = reinterpret_cast<uint4*>(tfeat + ((size_t)dir * M_total + m) * (size_t)ld_tfeat);
      for (int c = lane; c < row_bytes / 16; c += 32) td[c] = ts[c];
    }
  }
  __syncwarp();
}

template <bool Contract>
__global__ void __launch_bounds__(256)
encode_kernel(mnrf_encode_desc d, const float* __restrict__ sdist,
              const float* __restrict__ origins, const float* __restrict__ directions,
              const float* __restrict__ radii, const float* __restrict__ near,
              const float* __restrict__ far, const float* __restrict__ basis,
              __nv_bfloat16* __restrict__ feat, float* __restrict__ feat_f32,
              float* __restrict__ tdist_out, __nv_bfloat16* __restrict__ tfeat, int ld_tfeat) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int S = d.num_samples, K = d.basis_k;
  float* sb = reinterpret_cast<float*>(smem_raw);                 // basis [K][3]
  const int row_bytes = ((d.feat_cols * 2 + 15) / 16) * 16;
  constexpr int stride = Contract ? kContractStride : kGaussStride;
  const int per_warp_f = (S + 1) + S * stride + (Contract ? 8 : 2) * K;
  float* wbase = sb + 3 * K + (size_t)wib * per_warp_f;
  float* tds = wbase;
  float* gs = tds + (S + 1);
  TangentScratch ws;
  ws.lm = gs + S * stride;
  ws.lv = ws.lm + K;
  ws.dlm = ws.lv + K;
  ws.dlv = ws.dlm + 3 * K;
  unsigned char* rows = smem_raw + (((size_t)(3 * K + nw * per_warp_f) * 4 + 15) / 16) * 16;
  const int rows_per_warp = tfeat ? 4 : 1;        // feature row + three tangent rows
  ws.row = reinterpret_cast<__nv_bfloat16*>(rows + (size_t)wib * rows_per_warp * row_bytes);
  ws.trow = reinterpret_cast<__nv_bfloat16*>(reinterpret_cast<unsigned char*>(ws.row) + row_bytes);
  ws.trow_elems = row_bytes / 2;
  ws.row_bytes = row_bytes;
  const size_t M_total = (size_t)d.num_rays * d.num_samples;

  for (int i = threadIdx.x; i < 3 * K; i += blockDim.x) sb[i] = basis[i];
  __syncthreads();
  for (int i = lane; i < d.feat_cols * rows_per_warp; i += 32)
    ws.row[i + (i / d.feat_cols) * (ws.trow_elems - d.feat_cols)] = __float2bfloat16(0.f);

  for (int ray = blockIdx.x * nw + wib; ray < d.num_rays; ray += gridDim.x * nw) {
    const float o[3] = {origins[ray * 3 + 0], origins[ray * 3 + 1], origins[ray * 3 + 2]};
    const float dv[3] = {directions[ray * 3 + 0], directions[ray * 3 + 1], directions[ray * 3 + 2]};
    const float radius = radii[ray];
    const float s_near = fwd_raydist(d.raydist_fn, near[ray]);
    const float s_far = fwd_raydist(d.raydist_fn, far[ray]);
    for (int i = lane; i <= S; i += 32) {
      float t = s_to_t(d.raydist_fn, sdist[(size_t)ray * (S + 1) + i], s_near, s_far);
      tds[i] = t;
      if (tdist_out) tdist_out[(size_t)ray * (S + 1) + i] = t;
    }
    __syncwarp();
    // phase A: one lane per sample -- Gaussian of the frustum, contracted
    for (int s = lane; s < S; s += 32) {
      Gauss g;
      cast_one(d.ray_shape, tds[s], tds[s + 1], o, dv, radius, g);
      store_gauss<Contract>(d, g, gs + s * stride);
    }
    __syncwarp();
    // phase B: per sample, lift onto the basis and emit the 2*K*L features
    for (int s = 0; s < S; ++s)
      gauss_tangent_rows<Contract>(d, gs + s * stride, sb, ws, (size_t)ray * S + s, M_total, feat, feat_f32, tfeat,
                                   ld_tfeat, lane);
  }
}

// Phase A of the point encoder for a Gaussian whose mean is already a contracted point p (warp_contract 2): the
// Gaussian is stored as it is, and the terms of the tangent rows are those of the contraction at x = inv_contract(p)
// with s_r = q_r = 0, so phase B writes d feature / d p times J(x) = d feature / d x with the footprint held fixed in
// contracted space: the lifted variance does not move.
__device__ __forceinline__ void store_contracted_gauss(const Gauss& g, float* gp) {
  float x[3], s, q, xh[3];
  inv_contract_point(g.mean, x);
  contract_jacobian(x, s, q, xh);
#pragma unroll
  for (int i = 0; i < 3; ++i) gp[12 + i] = xh[i];
  gp[15] = g.cov[0][0]; gp[16] = g.cov[0][1]; gp[17] = g.cov[0][2];
  gp[18] = g.cov[1][1]; gp[19] = g.cov[1][2]; gp[20] = g.cov[2][2];
  gp[21] = s; gp[22] = q; gp[23] = 0.f; gp[24] = 0.f;
  gp[0] = g.mean[0]; gp[1] = g.mean[1]; gp[2] = g.mean[2];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) gp[3 + i * 3 + j] = g.cov[i][j];
}

// Point form with tangent rows: the Gaussian of point i has mean points[i] and covariance var * I.  One warp takes
// 32 points at a time, one lane per point in phase A, then the general encoder's phase B point by point.
// Contracted (with Contract): the points are already contracted (store_contracted_gauss).
template <bool Contract, bool Contracted = false>
__global__ void __launch_bounds__(256)
encode_points_tangent_kernel(mnrf_encode_desc d, const float* __restrict__ points, float var,
                             const float* __restrict__ basis, __nv_bfloat16* __restrict__ feat,
                             __nv_bfloat16* __restrict__ tfeat, int ld_tfeat) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int K = d.basis_k;
  float* sb = reinterpret_cast<float*>(smem_raw);                 // basis [K][3]
  const int row_bytes = ((d.feat_cols * 2 + 15) / 16) * 16;
  constexpr int stride = Contract ? kContractStride : kGaussStride;
  const int per_warp_f = 32 * stride + (Contract ? 8 : 2) * K;
  float* gs = sb + 3 * K + (size_t)wib * per_warp_f;
  TangentScratch ws;
  ws.lm = gs + 32 * stride;
  ws.lv = ws.lm + K;
  ws.dlm = ws.lv + K;
  ws.dlv = ws.dlm + 3 * K;
  unsigned char* rows = smem_raw + (((size_t)(3 * K + nw * per_warp_f) * 4 + 15) / 16) * 16;
  ws.row = reinterpret_cast<__nv_bfloat16*>(rows + (size_t)wib * 4 * row_bytes);
  ws.trow = reinterpret_cast<__nv_bfloat16*>(reinterpret_cast<unsigned char*>(ws.row) + row_bytes);
  ws.trow_elems = row_bytes / 2;
  ws.row_bytes = row_bytes;
  const size_t N = (size_t)d.num_rays;

  for (int i = threadIdx.x; i < 3 * K; i += blockDim.x) sb[i] = basis[i];
  __syncthreads();
  for (int i = lane; i < d.feat_cols * 4; i += 32)
    ws.row[i + (i / d.feat_cols) * (ws.trow_elems - d.feat_cols)] = __float2bfloat16(0.f);

  const int64_t num_groups = ((int64_t)N + 31) / 32;
  for (int64_t grp = (int64_t)blockIdx.x * nw + wib; grp < num_groups; grp += (int64_t)gridDim.x * nw) {
    const int64_t p0 = grp * 32;
    const int g = (int)min((int64_t)32, (int64_t)N - p0);
    __syncwarp();
    if (lane < g) {
      Gauss ga;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        ga.mean[i] = points[(p0 + lane) * 3 + i];
#pragma unroll
        for (int j = 0; j < 3; ++j) ga.cov[i][j] = i == j ? var : 0.f;
      }
      if (Contracted)
        store_contracted_gauss(ga, gs + lane * stride);
      else
        store_gauss<Contract>(d, ga, gs + lane * stride);
    }
    __syncwarp();
    for (int s = 0; s < g; ++s)
      gauss_tangent_rows<Contract>(d, gs + s * stride, sb, ws, (size_t)p0 + s, N, feat, nullptr, tfeat, ld_tfeat,
                                   lane);
  }
}

// Fast path (no tangent rows): work items are (sample, basis direction) pairs, G samples at a time so
// that G*K items fill whole 32-lane passes (K = 21: G = 3 -> 63 of 64 slots).  A lane lifts its own
// (mean, variance) onto its basis direction and walks the L degrees by exact doubling
// (y *= 2, var *= 4 give bit-identical values to lm * 2^l, lv * 4^l), so the inner loop carries no
// shared-memory exchange, no warp sync and no index arithmetic.  Rows are staged in shared memory
// and leave as 16-byte stores.
__device__ __forceinline__ float ex2_ftz(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

// The Gaussian-to-feature tail of the fast path, shared by the ray and the point encoders: lifts the g <= G
// Gaussians at gs (kGaussStride floats apart, shared memory) onto the basis and writes their feature rows m0 ..
// m0 + g - 1 (bf16, staged in `row`, G rows of row_elems; fp32 copy when feat_f32 is given).
__device__ __forceinline__ void gauss_feature_rows(const mnrf_encode_desc& d, int g, const float* gs,
                                                   const float* sb, __nv_bfloat16* row, int row_elems, size_t m0,
                                                   __nv_bfloat16* __restrict__ feat, float* __restrict__ feat_f32,
                                                   int lane) {
  const int K = d.basis_k, L = d.max_deg - d.min_deg, KL = K * L;
  const float sc0 = __int_as_float((127 + d.min_deg) << 23);       // 2^min_deg
  const float sc_top = exp2f((float)(L + 1));                      // bound on the growth of |y| over the degrees (+ pi/2)
  const int chunks = row_elems / 8;
  for (int j0 = 0; j0 < g * K; j0 += 32) {
    // uniform trip count (warp-wide max below): lanes past the last item redo it and store the same values
    const int j = min(j0 + lane, g * K - 1);
    const int sl = j / K;
    const int k = j - sl * K;
    const float* gp = gs + sl * kGaussStride;
    const float b0 = sb[k * 3 + 0], b1 = sb[k * 3 + 1], b2 = sb[k * 3 + 2];
    const float lm = gp[0] * b0 + gp[1] * b1 + gp[2] * b2;
    const float c0 = gp[3] * b0 + gp[4] * b1 + gp[5] * b2;
    const float c1 = gp[6] * b0 + gp[7] * b1 + gp[8] * b2;
    const float c2 = gp[9] * b0 + gp[10] * b1 + gp[11] * b2;
    const float lv = d.disable_integration ? 0.f : (b0 * c0 + b1 * c1 + b2 * c2);
    float y = lm * sc0;
    float v = lv * (sc0 * sc0);
    __nv_bfloat16* rp = row + sl * row_elems + k;
    float* fp = feat_f32 ? feat_f32 + (m0 + sl) * (size_t)(2 * KL) + k : nullptr;
    // Leading degrees for which EVERY lane's |y| and |y + pi/2| stay below 100*pi need none of safe_sin's
    // large-argument handling (two compare-and-branch pairs with their reconvergence barriers per degree, a
    // fifth of the loop's instructions): |y| 2^l <= 311  <=>  l <= floor(log2(311 / |y|)), read off the exponent.
    const float ymax = warp_max(fabsf(y));
    int n_fast = ((__float_as_int(__fdividef(311.f, ymax)) >> 23) & 0xff) - 126;
    n_fast = min(max(n_fast, 0), L);
    int l = 0;
#pragma unroll 4
    for (; l < n_fast; ++l) {
      // exp(-v/2): (-0.5 v) is exact, so one multiply by -0.5*log2(e) rounds like __expf's own
      const float e = ex2_ftz(v * -0.72134751081466674805f);
      const float fs = e * sin_below_100pi(y);
      const float fc = e * sin_below_100pi(y + 1.57079637050628662109375f);
      rp[l * K] = __float2bfloat16(fs);
      rp[KL + l * K] = __float2bfloat16(fc);
      if (fp) { fp[l * K] = fs; fp[KL + l * K] = fc; }
      y = y * 2.f;
      v = v * 4.f;
    }
    // remaining degrees: the branch-free large-argument form while every argument stays below its 1.3e9 limit
    // (warp-uniform test), the general one otherwise
    if (ymax * sc_top < 1e9f) {
#pragma unroll 4
      for (; l < L; ++l) {
        const float e = ex2_ftz(v * -0.72134751081466674805f);
        const float fs = e * safe_sin_nobranch(y);
        const float fc = e * safe_sin_nobranch(y + 1.57079637050628662109375f);
        rp[l * K] = __float2bfloat16(fs);
        rp[KL + l * K] = __float2bfloat16(fc);
        if (fp) { fp[l * K] = fs; fp[KL + l * K] = fc; }
        y = y * 2.f;
        v = v * 4.f;
      }
    }
    for (; l < L; ++l) {
      const float e = ex2_ftz(v * -0.72134751081466674805f);
      const float fs = e * safe_sin_fast(y);
      const float fc = e * safe_sin_fast(y + 1.57079637050628662109375f);
      rp[l * K] = __float2bfloat16(fs);
      rp[KL + l * K] = __float2bfloat16(fc);
      if (fp) { fp[l * K] = fs; fp[KL + l * K] = fc; }
      y = y * 2.f;
      v = v * 4.f;
    }
  }
  __syncwarp();
  for (int r = 0; r < g; ++r) {
    const uint4* src = reinterpret_cast<const uint4*>(row + r * row_elems);
    uint4* dst = reinterpret_cast<uint4*>(feat + (m0 + r) * (size_t)d.ld_feat);
    for (int c = lane; c < chunks; c += 32) dst[c] = src[c];
  }
  __syncwarp();
}

// Samples per group of the fast path: fill the 32-lane passes over (sample, direction) items as fully as possible.
static int encode_group_size(int basis_k, int max_g) {
  int G = 1;
  double best = 0.0;
  for (int g = 1; g <= 16 && g <= max_g; ++g) {
    const int items = g * basis_k;
    const double eff = (double)items / (32.0 * ((items + 31) / 32));
    if (eff > best + 1e-9) { best = eff; G = g; }
  }
  return G;
}

// A ray may be split into `nseg` segments of `seg_len` samples (a multiple of G), one warp each: with few rays per
// launch (a 2048-ray shard of an 8-GPU step) one warp per ray leaves most of the machine idle.
__global__ void __launch_bounds__(256, 4)
encode_fast_kernel(mnrf_encode_desc d, int G, int nseg, int seg_len, const float* __restrict__ sdist,
                   const float* __restrict__ origins, const float* __restrict__ directions,
                   const float* __restrict__ radii, const float* __restrict__ near,
                   const float* __restrict__ far, const float* __restrict__ basis,
                   __nv_bfloat16* __restrict__ feat, float* __restrict__ feat_f32,
                   float* __restrict__ tdist_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int S = d.num_samples, K = d.basis_k;
  float* sb = reinterpret_cast<float*>(smem_raw);                 // basis [K][3]
  const int row_bytes = ((d.feat_cols * 2 + 15) / 16) * 16;
  const int row_elems = row_bytes / 2;
  const int per_warp_f = (S + 1) + S * kGaussStride;
  float* tds = sb + 3 * K + (size_t)wib * per_warp_f;
  float* gs = tds + (S + 1);
  unsigned char* rows = smem_raw + (((size_t)(3 * K + nw * per_warp_f) * 4 + 15) / 16) * 16;
  __nv_bfloat16* row = reinterpret_cast<__nv_bfloat16*>(rows + (size_t)wib * G * row_bytes);

  for (int i = threadIdx.x; i < 3 * K; i += blockDim.x) sb[i] = basis[i];
  __syncthreads();
  for (int i = lane; i < G * row_elems; i += 32) row[i] = __float2bfloat16(0.f);   // zero pad columns once

  const int64_t num_items = (int64_t)d.num_rays * nseg;
  for (int64_t item = (int64_t)blockIdx.x * nw + wib; item < num_items; item += (int64_t)gridDim.x * nw) {
    const int ray = (int)(item / nseg);
    const int s_begin = (int)(item - (int64_t)ray * nseg) * seg_len;
    const int s_end = min(S, s_begin + seg_len);
    const float o[3] = {origins[ray * 3 + 0], origins[ray * 3 + 1], origins[ray * 3 + 2]};
    const float dv[3] = {directions[ray * 3 + 0], directions[ray * 3 + 1], directions[ray * 3 + 2]};
    const float radius = radii[ray];
    const float s_near = fwd_raydist(d.raydist_fn, near[ray]);
    const float s_far = fwd_raydist(d.raydist_fn, far[ray]);
    __syncwarp();
    for (int i = s_begin + lane; i <= s_end; i += 32) {
      float t = s_to_t(d.raydist_fn, sdist[(size_t)ray * (S + 1) + i], s_near, s_far);
      tds[i] = t;
      if (tdist_out) tdist_out[(size_t)ray * (S + 1) + i] = t;
    }
    __syncwarp();
    // phase A: one lane per sample -- Gaussian of the frustum, contracted
    for (int s = s_begin + lane; s < s_end; s += 32) {
      Gauss g;
      cast_one(d.ray_shape, tds[s], tds[s + 1], o, dv, radius, g);
      if (d.warp_contract) contract_gauss(g);
      float* gp = gs + s * kGaussStride;
      gp[0] = g.mean[0]; gp[1] = g.mean[1]; gp[2] = g.mean[2];
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) gp[3 + i * 3 + j] = g.cov[i][j];
    }
    __syncwarp();
    // phase B: G samples at a time
    for (int s0 = s_begin; s0 < s_end; s0 += G)
      gauss_feature_rows(d, min(G, s_end - s0), gs + s0 * kGaussStride, sb, row, row_elems, (size_t)ray * S + s0,
                         feat, feat_f32, lane);
  }
}

// Point form: the Gaussian of point i has mean points[i] and covariance var * I.  One warp encodes G points at a
// time through the fast path's tail.
__global__ void __launch_bounds__(256, 4)
encode_points_kernel(mnrf_encode_desc d, int G, const float* __restrict__ points, float var,
                     const float* __restrict__ basis, __nv_bfloat16* __restrict__ feat, float* __restrict__ feat_f32) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int K = d.basis_k;
  float* sb = reinterpret_cast<float*>(smem_raw);                 // basis [K][3]
  const int row_bytes = ((d.feat_cols * 2 + 15) / 16) * 16;
  const int row_elems = row_bytes / 2;
  float* gs = sb + 3 * K + (size_t)wib * G * kGaussStride;
  unsigned char* rows = smem_raw + (((size_t)(3 * K + nw * G * kGaussStride) * 4 + 15) / 16) * 16;
  __nv_bfloat16* row = reinterpret_cast<__nv_bfloat16*>(rows + (size_t)wib * G * row_bytes);

  for (int i = threadIdx.x; i < 3 * K; i += blockDim.x) sb[i] = basis[i];
  __syncthreads();
  for (int i = lane; i < G * row_elems; i += 32) row[i] = __float2bfloat16(0.f);   // zero pad columns once

  const int64_t num_groups = ((int64_t)d.num_rays + G - 1) / G;
  for (int64_t grp = (int64_t)blockIdx.x * nw + wib; grp < num_groups; grp += (int64_t)gridDim.x * nw) {
    const int64_t p0 = grp * G;
    const int g = (int)min((int64_t)G, (int64_t)d.num_rays - p0);
    __syncwarp();
    if (lane < g) {
      Gauss ga;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        ga.mean[i] = points[(p0 + lane) * 3 + i];
#pragma unroll
        for (int j = 0; j < 3; ++j) ga.cov[i][j] = i == j ? var : 0.f;
      }
      if (d.warp_contract) contract_gauss(ga);
      float* gp = gs + lane * kGaussStride;
      gp[0] = ga.mean[0]; gp[1] = ga.mean[1]; gp[2] = ga.mean[2];
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) gp[3 + i * 3 + j] = ga.cov[i][j];
    }
    __syncwarp();
    gauss_feature_rows(d, g, gs, sb, row, row_elems, (size_t)p0, feat, feat_f32, lane);
  }
}

__global__ void viewdir_enc_kernel(int num_rays, int S, int deg, const float* __restrict__ viewdirs,
                                   __nv_bfloat16* __restrict__ out, int ld, int col0, int col_end) {
  // one thread per (row, column) of the [col0, col_end) slab; consecutive threads -> columns
  const int width = col_end - col0;
  const size_t total = (size_t)num_rays * S * width;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    size_t rowi = i / width;
    int c = (int)(i - rowi * width);
    int ray = (int)(rowi / S);
    float v = 0.f;
    if (c < 3) {
      v = viewdirs[ray * 3 + c];
    } else if (c < 3 + 6 * deg) {
      int f = c - 3;
      int half = f / (3 * deg);
      f -= half * 3 * deg;
      int l = f / 3, ch = f - l * 3;
      float x = viewdirs[ray * 3 + ch] * exp2f((float)l);
      v = sinf(half ? x + 1.57079637050628662109375f : x);   // plain sin (coord.py:143-144)
    }
    out[rowi * (size_t)ld + col0 + c] = __float2bfloat16(v);
  }
}

// Same values, computed ONCE per ray (they do not depend on the sample) and replicated over the ray's S rows with
// 16-byte stores: one warp per ray, the slab row staged in shared memory.  Needs a 16-byte aligned slab.
__global__ void __launch_bounds__(256)
viewdir_enc_rows_kernel(int num_rays, int S, int deg, const float* __restrict__ viewdirs,
                        __nv_bfloat16* __restrict__ out, int ld, int col0, int col_end) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int width = col_end - col0;                 // multiple of 8
  const int chunks = width / 8;                     // 16-byte chunks per row
  __nv_bfloat16* row = reinterpret_cast<__nv_bfloat16*>(smem_raw) + (size_t)wib * width;
  for (int ray = blockIdx.x * nw + wib; ray < num_rays; ray += gridDim.x * nw) {
    __syncwarp();
    for (int c = lane; c < width; c += 32) {
      float v = 0.f;
      if (c < 3) {
        v = viewdirs[ray * 3 + c];
      } else if (c < 3 + 6 * deg) {
        int f = c - 3;
        const int half = f / (3 * deg);
        f -= half * 3 * deg;
        const int l = f / 3, ch = f - l * 3;
        const float x = viewdirs[ray * 3 + ch] * exp2f((float)l);
        v = sinf(half ? x + 1.57079637050628662109375f : x);   // plain sin (coord.py:143-144)
      }
      row[c] = __float2bfloat16(v);
    }
    __syncwarp();
    const uint4* src = reinterpret_cast<const uint4*>(row);
    __nv_bfloat16* dst0 = out + (size_t)ray * S * (size_t)ld + col0;
    for (int i = lane; i < S * chunks; i += 32) {
      const int r = i / chunks, c = i - r * chunks;
      reinterpret_cast<uint4*>(dst0 + (size_t)r * ld)[c] = src[c];
    }
  }
}

}  // namespace mnrf

extern "C" int mnrf_encode(const mnrf_encode_desc* d, const float* sdist, const float* origins,
                           const float* directions, const float* radii, const float* near,
                           const float* far, const float* basis, mnrf_bf16* feat_bf16,
                           float* feat_f32, float* tdist_out, mnrf_bf16* tfeat, int32_t ld_tfeat,
                           mnrf_stream stream) {
  using namespace mnrf;
  if (d && d->num_rays == 0) return 0;            // nothing to do (and empty tensors carry null pointers)
  MNRF_CHECK(d && sdist && origins && directions && radii && near && far && basis && feat_bf16,
             "mnrf_encode: null pointer");
  if (tfeat) {
    MNRF_CHECK(!feat_f32 && !tdist_out, "mnrf_encode: the tangent features take no feat_f32 / tdist_out");
    MNRF_CHECK(ld_tfeat >= d->feat_cols && ld_tfeat % 8 == 0 && ((uintptr_t)tfeat % 16) == 0,
               "mnrf_encode: tangent rows must be 16-byte aligned");
  }
  MNRF_CHECK(d->ray_shape == MNRF_RAY_CONE || d->ray_shape == MNRF_RAY_CYLINDER,
             "ray_shape must be 'cone' or 'cylinder'");
  MNRF_CHECK(d->warp_contract == 0 || d->warp_contract == 1, "mnrf_encode: warp_contract %d: want 0 or 1",
             d->warp_contract);
  const int KL2 = 2 * d->basis_k * (d->max_deg - d->min_deg);
  MNRF_CHECK(d->feat_cols >= KL2 && d->ld_feat >= d->feat_cols, "mnrf_encode: feat_cols %d < 2KL %d or ld %d",
             d->feat_cols, KL2, d->ld_feat);
  MNRF_CHECK(d->feat_cols % 8 == 0 && d->ld_feat % 8 == 0 && ((uintptr_t)feat_bf16 % 16) == 0,
             "mnrf_encode: feature rows must be 16-byte aligned");
  if (d->num_rays == 0) return 0;
  int nw = 8;
  const int row_bytes = ((d->feat_cols * 2 + 15) / 16) * 16;
  int blocks = ceil_div(d->num_rays, nw);
  const int max_blocks = mnrf_num_sms() * 8;
  if (blocks > max_blocks) blocks = max_blocks;
  if (!tfeat) {
    const int G = encode_group_size(d->basis_k, d->num_samples);
    size_t smem = (((size_t)(3 * d->basis_k + nw * ((d->num_samples + 1) + d->num_samples * kGaussStride)) * 4 + 15) / 16) * 16 +
                  (size_t)nw * G * row_bytes;
    MNRF_CHECK(smem <= 200 * 1024, "mnrf_encode: shared memory %zu too large", smem);
    MNRF_CUDA(cudaFuncSetAttribute(encode_fast_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    // segments per ray: enough warps to fill the machine ~4 deep when the launch has few rays
    const int64_t want_warps = (int64_t)mnrf_num_sms() * nw * 4;
    int nseg = (int)std::min<int64_t>((want_warps + d->num_rays - 1) / d->num_rays, std::max(1, d->num_samples / (2 * G)));
    nseg = std::max(1, nseg);
    int seg_len = (d->num_samples + nseg - 1) / nseg;
    seg_len = (seg_len + G - 1) / G * G;
    nseg = (d->num_samples + seg_len - 1) / seg_len;
    blocks = (int)std::min<int64_t>(((int64_t)d->num_rays * nseg + nw - 1) / nw, max_blocks);
    encode_fast_kernel<<<blocks, nw * 32, smem, (cudaStream_t)stream>>>(
        *d, G, nseg, seg_len, sdist, origins, directions, radii, near, far, basis,
        reinterpret_cast<__nv_bfloat16*>(feat_bf16), feat_f32, tdist_out);
    MNRF_LAUNCH_CHECK();
    return 0;
  }
  const bool contract = d->warp_contract != 0;
  const int stride = contract ? kContractStride : kGaussStride;
  size_t smem = (((size_t)(3 * d->basis_k + nw * ((d->num_samples + 1) + d->num_samples * stride +
                                                   (contract ? 8 : 2) * d->basis_k)) * 4 + 15) / 16) * 16 +
                (size_t)nw * row_bytes * (tfeat ? 4 : 1);
  MNRF_CHECK(smem <= 200 * 1024, "mnrf_encode: shared memory %zu too large", smem);
  auto kernel = contract ? encode_kernel<true> : encode_kernel<false>;
  MNRF_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<blocks, nw * 32, smem, (cudaStream_t)stream>>>(
      *d, sdist, origins, directions, radii, near, far, basis,
      reinterpret_cast<__nv_bfloat16*>(feat_bf16), feat_f32, tdist_out,
      reinterpret_cast<__nv_bfloat16*>(tfeat), ld_tfeat);
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_encode_points(const mnrf_encode_desc* d, const float* points, float var, const float* basis,
                                  mnrf_bf16* feat_bf16, float* feat_f32, mnrf_stream stream) {
  using namespace mnrf;
  MNRF_CHECK(d, "mnrf_encode_points: null descriptor");
  MNRF_CHECK(d->num_rays >= 0, "mnrf_encode_points: negative point count %d", d->num_rays);
  if (d->num_rays == 0) return 0;
  MNRF_CHECK(points && basis && feat_bf16, "mnrf_encode_points: null pointer");
  MNRF_CHECK(d->num_samples == 1 && d->raydist_fn == 0 && d->ray_shape == 0,
             "mnrf_encode_points: num_samples must be 1 and raydist_fn, ray_shape 0 (got %d, %d, %d)",
             d->num_samples, d->raydist_fn, d->ray_shape);
  MNRF_CHECK(var >= 0.f, "mnrf_encode_points: var %g < 0", var);
  MNRF_CHECK(d->warp_contract >= 0 && d->warp_contract <= 2, "mnrf_encode_points: warp_contract %d: want 0, 1 or 2",
             d->warp_contract);
  mnrf_encode_desc dd = *d;
  if (dd.warp_contract == 2) dd.warp_contract = 0;      // already contracted: the feature rows of mode 0
  MNRF_CHECK(d->basis_k > 0 && d->max_deg > d->min_deg, "mnrf_encode_points: empty encoding");
  const int KL2 = 2 * d->basis_k * (d->max_deg - d->min_deg);
  MNRF_CHECK(d->feat_cols >= KL2 && d->ld_feat >= d->feat_cols, "mnrf_encode_points: feat_cols %d < 2KL %d or ld %d",
             d->feat_cols, KL2, d->ld_feat);
  MNRF_CHECK(d->feat_cols % 8 == 0 && d->ld_feat % 8 == 0 && ((uintptr_t)feat_bf16 % 16) == 0,
             "mnrf_encode_points: feature rows must be 16-byte aligned");
  const int nw = 8;
  const int G = encode_group_size(d->basis_k, 16);
  const int row_bytes = ((d->feat_cols * 2 + 15) / 16) * 16;
  const size_t smem = (((size_t)(3 * d->basis_k + nw * G * kGaussStride) * 4 + 15) / 16) * 16 +
                      (size_t)nw * G * row_bytes;
  MNRF_CHECK(smem <= 200 * 1024, "mnrf_encode_points: shared memory %zu too large", smem);
  MNRF_CUDA(cudaFuncSetAttribute(encode_points_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t groups = ((int64_t)d->num_rays + G - 1) / G;
  const int blocks = (int)std::min<int64_t>((groups + nw - 1) / nw, (int64_t)mnrf_num_sms() * 8);
  encode_points_kernel<<<blocks, nw * 32, smem, (cudaStream_t)stream>>>(
      dd, G, points, var, basis, reinterpret_cast<__nv_bfloat16*>(feat_bf16), feat_f32);
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_encode_points_tangent(const mnrf_encode_desc* d, const float* points, float var,
                                          const float* basis, mnrf_bf16* feat_bf16, mnrf_bf16* tfeat_bf16,
                                          int32_t ld_tfeat, mnrf_stream stream) {
  using namespace mnrf;
  MNRF_CHECK(d, "mnrf_encode_points_tangent: null descriptor");
  MNRF_CHECK(d->num_rays >= 0, "mnrf_encode_points_tangent: negative point count %d", d->num_rays);
  if (d->num_rays == 0) return 0;
  MNRF_CHECK(points && basis && feat_bf16 && tfeat_bf16, "mnrf_encode_points_tangent: null pointer");
  MNRF_CHECK(d->num_samples == 1 && d->raydist_fn == 0 && d->ray_shape == 0,
             "mnrf_encode_points_tangent: num_samples must be 1 and raydist_fn, ray_shape 0 (got %d, %d, %d)",
             d->num_samples, d->raydist_fn, d->ray_shape);
  MNRF_CHECK(var >= 0.f && std::isfinite(var), "mnrf_encode_points_tangent: var %g is not finite and >= 0", var);
  MNRF_CHECK(d->basis_k > 0 && d->max_deg > d->min_deg, "mnrf_encode_points_tangent: empty encoding");
  const int KL2 = 2 * d->basis_k * (d->max_deg - d->min_deg);
  MNRF_CHECK(d->feat_cols >= KL2 && d->ld_feat >= d->feat_cols,
             "mnrf_encode_points_tangent: feat_cols %d < 2KL %d or ld %d", d->feat_cols, KL2, d->ld_feat);
  MNRF_CHECK(d->feat_cols % 8 == 0 && d->ld_feat % 8 == 0 && ((uintptr_t)feat_bf16 % 16) == 0,
             "mnrf_encode_points_tangent: feature rows must be 16-byte aligned");
  MNRF_CHECK(ld_tfeat >= d->feat_cols && ld_tfeat % 8 == 0 && ((uintptr_t)tfeat_bf16 % 16) == 0,
             "mnrf_encode_points_tangent: tangent rows must be 16-byte aligned");
  MNRF_CHECK(d->warp_contract >= 0 && d->warp_contract <= 2,
             "mnrf_encode_points_tangent: warp_contract %d: want 0, 1 or 2", d->warp_contract);
  const int nw = 8;
  const bool contract = d->warp_contract != 0;
  const int stride = contract ? kContractStride : kGaussStride;
  const int row_bytes = ((d->feat_cols * 2 + 15) / 16) * 16;
  const size_t smem = (((size_t)(3 * d->basis_k + nw * (32 * stride + (contract ? 8 : 2) * d->basis_k)) * 4 + 15) /
                       16) * 16 + (size_t)nw * 4 * row_bytes;
  MNRF_CHECK(smem <= 200 * 1024, "mnrf_encode_points_tangent: shared memory %zu too large", smem);
  auto kernel = d->warp_contract == 2 ? encode_points_tangent_kernel<true, true>
              : contract              ? encode_points_tangent_kernel<true>
                                      : encode_points_tangent_kernel<false>;
  MNRF_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t groups = ((int64_t)d->num_rays + 31) / 32;
  const int blocks = (int)std::min<int64_t>((groups + nw - 1) / nw, (int64_t)mnrf_num_sms() * 8);
  kernel<<<blocks, nw * 32, smem, (cudaStream_t)stream>>>(*d, points, var, basis,
                                                          reinterpret_cast<__nv_bfloat16*>(feat_bf16),
                                                          reinterpret_cast<__nv_bfloat16*>(tfeat_bf16), ld_tfeat);
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_viewdir_enc(int32_t num_rays, int32_t num_samples, int32_t deg,
                                const float* viewdirs, mnrf_bf16* out, int32_t ld, int32_t col0,
                                int32_t col_end, mnrf_stream stream) {
  using namespace mnrf;
  if (num_rays == 0) return 0;
  MNRF_CHECK(viewdirs && out, "mnrf_viewdir_enc: null pointer");
  MNRF_CHECK(col_end - col0 >= 3 + 6 * deg && col_end <= ld, "mnrf_viewdir_enc: slab [%d,%d) too small for deg %d",
             col0, col_end, deg);
  if (num_rays == 0) return 0;
  if ((col_end - col0) % 8 == 0 && col0 % 8 == 0 && ld % 8 == 0 && ((uintptr_t)out % 16) == 0) {
    const int nw = 8;
    const int blocks_r = std::min((num_rays + nw - 1) / nw, mnrf_num_sms() * 8);
    viewdir_enc_rows_kernel<<<blocks_r, nw * 32, (size_t)nw * (col_end - col0) * 2, (cudaStream_t)stream>>>(
        num_rays, num_samples, deg, viewdirs, reinterpret_cast<__nv_bfloat16*>(out), ld, col0, col_end);
    MNRF_LAUNCH_CHECK();
    return 0;
  }
  size_t total = (size_t)num_rays * num_samples * (col_end - col0);
  int blocks = (int)((total + 255) / 256);
  int maxb = mnrf_num_sms() * 16;
  if (blocks > maxb) blocks = maxb;
  viewdir_enc_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(
      num_rays, num_samples, deg, viewdirs, reinterpret_cast<__nv_bfloat16*>(out), ld, col0, col_end);
  MNRF_LAUNCH_CHECK();
  return 0;
}
