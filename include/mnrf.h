/* mnrf.h -- C ABI of the H100-native MultiNeRF per-ray core (libmnrf_b200.so).
 *
 * The reference (google-research/multinerf) has NO native boundary: its operator API is
 * the Python signature `Model.__call__` (internal/models.py:75-312) plus the free
 * functions of internal/{stepfun,render,coord}.py, all lowered by XLA.  This header is
 * the boundary a maintainer would bind instead (ctypes stub in INTEGRATION.md); each entry
 * names the reference code it replaces.
 *
 * Conventions
 *  - every pointer is a DEVICE pointer owned by the caller (fp32 row-major, samples on the
 *    last axis, unless a parameter says bf16); entries only write their declared outputs;
 *  - entries enqueue work on `stream` and return immediately: no allocation, no host
 *    synchronisation, no global mutable state (except the tensor-map encoder lookup);
 *  - return 0 on success, non-zero on error; the message is in mnrf_last_error()
 *    (thread-local).  Python-side config errors of the reference (ValueError at trace
 *    time) stay Python-side; the ABI reports shape / alignment / launch failures;
 *  - bf16 buffers are raw uint16 storage (`mnrf_bf16`);
 *  - WORKSPACE POLICY: no entry needs scratch beyond its declared arguments (every intermediate is an
 *    argument the caller allocates: per-level activation / mask / gradient buffers are sized from the
 *    shapes documented per entry), so there are no `*_workspace_bytes` queries; kernels keep their
 *    staging in shared memory / registers.  The Python host (multinerf_b200/models.py `_level_state`)
 *    allocates each buffer once per (level, shape) and never frees it while a captured graph lives.
 */
#ifndef MNRF_H_
#define MNRF_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef uint16_t mnrf_bf16;
typedef void* mnrf_stream;   /* cudaStream_t */

#define MNRF_ABI_VERSION 2

/* ---- library ------------------------------------------------------------------------- */
int mnrf_abi_version(void);
const char* mnrf_last_error(void);
/* 1 if the current device is sm_90 (H100) and the wgmma/TMA path can run. */
int mnrf_device_ok(void);
int mnrf_num_sms(void);

/* ---- hierarchical resampling ---------------------------------------------------------
 * Replaces, for one level: stepfun.max_dilate_weights (stepfun.py:116-128) + the [1:-1]
 * trim (models.py:170-171) + the annealed logits (models.py:183-185) + stepfun.
 * sample_intervals (stepfun.py:214-263: softmax, integrate_weights, sorted_interp
 * math.py:108-127, midpoints).  One warp owns one ray.
 *   sdist_prev [B, P+1], w_prev [B, P]           previous step function
 *   u_base     [S]      host-computed linspace grid of stepfun.py:194-206
 *   jitter     raw U[0,1): NULL | [B] (single_jitter) | [B, S]
 *   anneal_dev optional device scalar: the annealing exponent is read from anneal_dev[0] at run time
 *              instead of d->anneal, so that a captured CUDA graph can be replayed while train_frac
 *              advances (models.py:174-179)
 *   cw_in      optional [B, P'+1] CDF to use instead of the internally computed one
 *              (P' = 3P-2 with dilation, else P) -- lets tests pin the integer search
 *   sdist_out  [B, S+1]
 *   idx_out    optional int32 [B, S]: interval index #{cw <= u} - 1 (bit-exact contract)
 *   cw_out     optional [B, P'+1]; tdil_out/wdil_out optional [B, P'+1] / [B, P'] (trimmed)
 */
typedef struct {
  int32_t num_rays, num_prev, num_samples;
  int32_t use_dilation;
  float dilation, domain_lo, domain_hi;
  float anneal, resample_padding;
  int32_t jitter_mode;      /* 0 none, 1 per ray, 2 per sample */
  float max_jitter;
} mnrf_sample_desc;

int mnrf_sample_level(const mnrf_sample_desc* d, const float* sdist_prev, const float* w_prev,
                      const float* u_base, const float* jitter, const float* anneal_dev, const float* cw_in,
                      float* sdist_out, int32_t* idx_out, float* cw_out, float* tdil_out,
                      float* wdil_out, mnrf_stream stream);

/* ---- ray casting + integrated positional encoding ------------------------------------
 * Replaces coord.construct_ray_warps s_to_t (coord.py:63-99), render.cast_rays
 * (render.py:103-127, diag=False), coord.track_linearize(contract) (coord.py:21-60),
 * coord.lift_and_diagonalize (:129-133) and coord.integrated_pos_enc (:107-126).
 *   sdist [B, S+1]; origins/directions [B,3]; radii/near/far [B]; basis [K,3]
 *   feat_bf16  [B*S, ld_feat] row stride in elements; columns [2KL, feat_cols) zero-filled
 *   feat_f32   optional [B*S, 2KL] (fp32 copy for parity tests)
 *   tdist_out  optional [B, S+1]
 *   tfeat_bf16 optional: the tangent features d(feature)/d(mean_x|y|z) as three stacked bf16 blocks
 *              tfeat[dir*B*S + m, ld_tfeat] (input of the forward-mode density-normal chain that replaces
 *              vmap(value_and_grad(predict_density)), models.py:473-492).  The derivative is taken with respect
 *              to the world-space mean: with warp_contract it runs through the contraction, including the
 *              dependence of the warped covariance J Sigma J^T on the mean (coord.track_linearize,
 *              coord.py:39-60).  ld_tfeat >= feat_cols, a multiple of 8, tfeat 16-byte aligned; refused
 *              together with feat_f32 or tdist_out.
 */
enum { MNRF_RAYDIST_NONE = 0, MNRF_RAYDIST_RECIPROCAL, MNRF_RAYDIST_LOG, MNRF_RAYDIST_EXP,
       MNRF_RAYDIST_SQRT, MNRF_RAYDIST_SQUARE, MNRF_RAYDIST_PIECEWISE };
enum { MNRF_RAY_CONE = 0, MNRF_RAY_CYLINDER = 1 };

typedef struct {
  int32_t num_rays, num_samples;
  int32_t raydist_fn, ray_shape, warp_contract, disable_integration;
  int32_t basis_k, min_deg, max_deg;
  int32_t ld_feat, feat_cols;
} mnrf_encode_desc;

int mnrf_encode(const mnrf_encode_desc* d, const float* sdist, const float* origins,
                const float* directions, const float* radii, const float* near,
                const float* far, const float* basis, mnrf_bf16* feat_bf16, float* feat_f32,
                float* tdist_out, mnrf_bf16* tfeat_bf16, int32_t ld_tfeat, mnrf_stream stream);

/* Point form of the encoder: the MLP input of the Gaussian with mean points[i] and covariance var * I, in place of
 * a cast ray interval (density queries on a grid, multinerf_b200/mesh.py).  The same contraction (covariance through
 * the Jacobian when warp_contract), lift onto the basis and IPE (lifted variance 0 with disable_integration) as
 * mnrf_encode, and the same bf16 rows:
 *   d->num_rays = point count N; d->num_samples must be 1, d->raydist_fn and d->ray_shape 0
 *   points [N, 3]; var >= 0; basis [K, 3]
 *   feat_bf16 [N, ld_feat], columns [2KL, feat_cols) zero-filled; feat_f32 optional [N, 2KL]
 */
int mnrf_encode_points(const mnrf_encode_desc* d, const float* points, float var, const float* basis,
                       mnrf_bf16* feat_bf16, float* feat_f32, mnrf_stream stream);

/* mnrf_encode_points plus the tangent rows d feature / d point (the input of the density-normal chain, as
 * mnrf_encode's tfeat_bf16): the same feature rows, and tfeat_bf16[dir * N + i, ld_tfeat] = d feat_i / d point_i[dir],
 * through the contraction and the dependence of its covariance on the mean when warp_contract.  var finite and
 * >= 0; ld_tfeat >= feat_cols, a multiple of 8, tfeat_bf16 16-byte aligned.
 * warp_contract = 2 (here and in mnrf_encode_points; mnrf_encode takes 0 or 1): the points are already contracted
 * (|p| < 2; meshes extracted in contracted space, multinerf_b200/mesh.py).  The Gaussians (p, var * I) are encoded as
 * they are, so the feature rows are those of warp_contract = 0; the tangent rows are the derivatives with respect to
 * the world point x = inv_contract(p) with the footprint held fixed in contracted space: mode 0's rows times
 * J(x) = d contract / dx (symmetric), tfeat[dir] = sum_b d feat / d p_b J[b][dir]. */
int mnrf_encode_points_tangent(const mnrf_encode_desc* d, const float* points, float var, const float* basis,
                               mnrf_bf16* feat_bf16, mnrf_bf16* tfeat_bf16, int32_t ld_tfeat, mnrf_stream stream);

/* View-direction positional encoding, coord.pos_enc (coord.py:136-147) with
 * append_identity, broadcast over the S samples of each ray (models.py:550-554) and
 * written as bf16 into columns [col0, col0 + 3 + 6*deg) of a [B*S, ld] buffer; columns up
 * to col_end are zero-filled. */
int mnrf_viewdir_enc(int32_t num_rays, int32_t num_samples, int32_t deg, const float* viewdirs,
                     mnrf_bf16* out, int32_t ld, int32_t col0, int32_t col_end,
                     mnrf_stream stream);

/* ---- dense layers on wgmma --------------------------------------------------------------
 * One Dense layer of models.py:436-437,455-460 (y = act(x W + b)) and its two backward
 * GEMMs, bf16 operands, fp32 accumulation in registers.
 *   mode FWD  : out[M,N] bf16 = act(A[M,K] * Bt[N,K]^T + bias[N])           (A, Bt K-major)
 *   mode DGRAD: out[M,N] bf16 = (A[M,K] * Bt[N,K]^T + rowv[M]*colv[N]) masked by mask[M,N]>0
 *               (or by the 1-bit `maskbits`)
 *               (A = dY, Bt = W in [in,out] layout; mask = stored activation; all optional)
 *   mode WGRAD: out[Mo,N] fp32 += A[R,Mo]^T * B[R,N]   (A = X, B = dY, both row-major with
 *               the reduction index R on rows: "MN-major" operands), split over R, fp32 atomics
 * All leading dimensions are in elements.  FWD / DGRAD: K must be a multiple of 64 and N a multiple
 * of 16.  WGRAD: R may be any count (the last 64-row reduction block is zero-filled past R) and N a
 * multiple of 64.  M-tiles are 128 rows; M (Mo) may be any count.
 */
enum { MNRF_GEMM_FWD = 0, MNRF_GEMM_DGRAD = 1, MNRF_GEMM_WGRAD = 2 };
/* Activations of the Dense layers (MLP.net_activation, models.py:457,578): SOFTPLUS is jax.nn.softplus
 * (logaddexp(z, 0)), SILU is jax.nn.silu (z * sigmoid(z)). */
enum { MNRF_ACT_NONE = 0, MNRF_ACT_RELU = 1, MNRF_ACT_SOFTPLUS = 2, MNRF_ACT_SILU = 3 };

typedef struct {
  int32_t mode, act;
  int64_t m;          /* rows of the output (FWD/DGRAD: samples; WGRAD: `in` features) */
  int32_t n, k;       /* output columns; reduction length (WGRAD: number of samples R) */
  int64_t lda, ldb, ldc, ldmask;
  int64_t ldmaskbits; /* row pitch of `maskbits` in 32-bit words */
  int64_t ldadd;      /* row pitch of `addend` */
  int64_t mask_mod;   /* > 0: mask row = output row mod mask_mod (the 3 stacked tangent streams of the
                         density-normal chain share the primal's ReLU masks); 0: mask row = output row.
                         Applies to `maskbits` and z; a bf16 `mask` with mask_mod > 0 is refused */
  int32_t impl;       /* 0 = wgmma (product path);   1 = SIMT reference kernel (bring-up/tests) */
} mnrf_gemm_desc;

/* maskbits (optional): 1-bit ReLU masks, word w of row m covers columns [32w, 32w+32).  FWD with
 * MNRF_ACT_RELU writes them (bit = output > 0); DGRAD reads them instead of the bf16 `mask`
 * (16x less mask traffic).  The caller zero-fills nothing: every word of the tile is written.
 * colsum (optional, DGRAD only): colsum[N] += column sums of the output, i.e. the bias gradient
 * of the layer whose activation masks this dgrad; reduced from the epilogue registers (fp32,
 * before the bf16 rounding of the stored output) -- no separate pass over dY.
 * addend (optional, DGRAD only): out += addend[M, ldadd] (bf16), added after the mask -- the second
 * gradient contribution to an input consumed twice (skip connection of the view MLP).
 * z / ldz: the pre-activation of a smooth activation (d->act = MNRF_ACT_SOFTPLUS or MNRF_ACT_SILU; refused with any
 * other act).  The backward needs a'(z) (and, for density normals, a''(z)), which the output h = a(z) does not give
 * back for SiLU, so the forward stores z itself in place of mask bits:
 *   mode FWD  : out[M,N] = a(z), z = A Bt^T + bias;  z[M, ldz] (optional, bf16) receives z
 *   mode DGRAD: out[M,N] = a'(z[r]) * (A Bt^T + rowv colv) + addend, with z row r = output row mod d->mask_mod (when
 *               > 0: the three tangent streams share the primal's z); colsum[N] += column sums of out
 * A smooth activation takes FWD or DGRAD only, z (required for DGRAD) with ldz >= N, and no `mask` / `maskbits`; N
 * must be a multiple of 64 and `out` 16-byte aligned with a row pitch that is a multiple of 8 on the tensor-core path
 * (impl 0). */
int mnrf_gemm(const mnrf_gemm_desc* d, const mnrf_bf16* a, const mnrf_bf16* b, const float* bias,
              const float* rowv, const float* colv, const mnrf_bf16* mask, uint32_t* maskbits,
              float* colsum, const mnrf_bf16* addend, mnrf_bf16* z, int64_t ldz, void* out, mnrf_stream stream);

/* Weight gradient with side sums computed from the operand tiles the main loop stages (by the three warps of
 * the producer warpgroup that issue no loads), so the bias gradient and the gradient of a Dense(1) head on the
 * same activation cost no extra pass over HBM; one launch (impl = 1, the SIMT reference, runs them as separate
 * passes).  They do cost shared-memory bandwidth the MMAs use (DESIGN.md section 3):
 *   out[Mo,N] += A[R,Mo]^T B[R,N]                       (as mnrf_gemm, mode MNRF_GEMM_WGRAD; A = X, B = dY)
 *   bsum[N]   += sum_r B[r, :]                          (optional: bias gradient of the layer)
 *   side_aw[Mo] += sum_r side_w[r] * A[r, :]            (optional: dW of a Dense(1) head reading X, with
 *                                                        side_w = its d(raw output), models.py:460) */
int mnrf_gemm_wgrad(const mnrf_gemm_desc* d, const mnrf_bf16* a, const mnrf_bf16* b, float* bsum,
                    const float* side_w, float* side_aw, float* out, mnrf_stream stream);

/* The kernel instance and launch shape the tensor-core path (impl 0) of mnrf_gemm / mnrf_gemm_wgrad chooses for
 * these arguments, which take the places they have there (bsum / side_w / side_aw: mnrf_gemm_wgrad; null where the
 * call has none).  Host-only: no pointer is dereferenced
 * and nothing is launched.  Returns nonzero, with the launch's error message, for arguments the launch refuses. */
typedef struct {
  int32_t block_n;    /* output tile width BN: 256, 128, 64, 32 or 16 */
  int32_t staged;     /* 1: the bf16 output goes through shared memory and TMA bulk stores; 0: register stores */
  int32_t mask_tma;   /* mask bits by TMA: DGRAD 1 loaded with the operands, 0 loaded by the epilogue (or none);
                         FWD 1 stored from shared memory by the epilogue set 3, 0 stored from registers (or none) */
  int32_t smooth;     /* softplus / SiLU epilogue */
  int32_t side;       /* WGRAD side sums (bsum / side_aw) */
  int32_t splits;     /* reduction splits (WGRAD; 1 otherwise) */
  int32_t tiles;      /* work items: row blocks x column blocks x splits */
  int32_t grid;       /* persistent CTAs */
  int32_t pingpong;   /* FWD / DGRAD: 1 each consumer warpgroup runs whole 128 x 128 sub-tiles of the 128 x block_n
                         tiles, alternating, so one's epilogue runs under the other's MMAs; 0 both run each tile */
  int32_t epilogue;   /* ping-pong epilogue operand set, compiled into its instance.  DGRAD: 1 mask bits by TMA
                         only, 2 mask bits by TMA and the rank-1 term rowv (x) colv.  FWD: 3 bias + ReLU + mask bits
                         stored by TMA, 4 bias + ReLU without mask bits, 5 bias alone.  0 any operands, tested at run
                         time (also every other instance) */
} mnrf_gemm_instance;
int mnrf_gemm_plan(const mnrf_gemm_desc* d, const mnrf_bf16* a, const mnrf_bf16* b, const float* bias,
                   const float* rowv, const float* colv, const mnrf_bf16* mask, const uint32_t* maskbits,
                   const float* colsum, const mnrf_bf16* addend, const mnrf_bf16* z, int64_t ldz, const void* out,
                   const float* bsum, const float* side_w, const float* side_aw, mnrf_gemm_instance* plan);

/* ---- layer-chained 256-wide MLP trunk ------------------------------------------------------
 * ONE persistent launch walks 512-row units of samples through all Dense layers of a 256-wide trunk
 * (forward; models.py:441-465 incl. the skip concat) or through its whole input-gradient chain
 * (backward, the dgrad side of jax.value_and_grad, train_utils.py:316-317).  Activations stay in
 * shared memory between layers and are written out once per layer (for the weight-gradient GEMMs);
 * accumulators live in registers; weights stream from L2 (csrc/chain.cu).
 *
 * A layer multiplies up to two operands, both in 64-column k-blocks:
 *   resident  -- the previous layer's output held in shared memory: n_res = 4 k-blocks (0 for the
 *                first layer), against weight k-blocks [res_kb0, res_kb0 + 4);
 *   streamed  -- n_stream k-blocks of the `stream` tensor (columns stream_col0 + 64 s), against weight
 *                k-blocks [stream_kb0, stream_kb0 + n_stream): the IPE features of layer 0 and of a
 *                skip layer (forward), the incoming gradient of the first chained layer (backward).
 * `w` is K-major [256, ldw] bf16: the forward operand w_nk [out, in_pad] or the dgrad operand
 * w_kn [in_pad(first 256 rows used), out].
 *   FWD: out = relu(acc + bias) (bf16), maskbits written (1 bit per output, as mnrf_gemm);
 *        head_w/head_b/head_out (optional): head_out[m, o] = <bf16(out_last[m, :]), head_w[o, :]> + head_b[o]
 *        for o < head_n, computed in the last layer's epilogue: the Dense(1) density head of models.py:460
 *        (head_n = 1), or that head stacked with the Dense(3) rgb head of a view-independent model
 *        (use_viewdirs = False, models.py:584; head_n = 4, head_out [m, 4] = [raw_density | raw_rgb]).
 *   BWD: out = acc masked by maskbits (read; NULL = no mask); colsum[256] += column sums of out (the
 *        bias gradient of the layer whose activation the mask came from).
 * `out` may be NULL (FWD only: the activation is not needed later).  m is any row count; rows past m
 * are zero-filled on load and clipped on store.
 */
#define MNRF_CHAIN_MAX_LAYERS 8
enum { MNRF_CHAIN_FWD = 0, MNRF_CHAIN_BWD = 1 };

typedef struct {
  const mnrf_bf16* w;
  int64_t ldw;
  const float* bias;
  uint32_t* maskbits;
  int64_t ldmaskbits;         /* in 32-bit words */
  float* colsum;
  mnrf_bf16* out;
  int64_t ldo;
  int32_t n_stream, stream_col0, stream_kb0;
  int32_t n_res, res_kb0;
  int32_t reserved;
} mnrf_chain_layer;

typedef struct {
  int32_t mode, num_layers;
  int32_t width;              /* must be 256 */
  int32_t stream_cols;        /* columns of `stream` (multiple of 64) */
  int64_t m;                  /* sample rows */
  const mnrf_bf16* stream;    /* [m, ldstream] bf16 */
  int64_t ldstream;
  const float* head_w;        /* [head_n, 256] fp32 or NULL */
  const float* head_b;        /* [head_n] fp32 or NULL */
  float* head_out;            /* [m, head_n] fp32 */
  int32_t head_n;             /* 1 or 4 (0 reads as 1) */
  int32_t reserved;
  mnrf_chain_layer layer[MNRF_CHAIN_MAX_LAYERS];
} mnrf_chain_desc;

int mnrf_mlp_chain(const mnrf_chain_desc* d, mnrf_stream stream);
int mnrf_mlp_chain_max_layers(void);

/* ---- small heads (N <= 4 outputs): density / rgb / predicted normals ---------------------
 * raw[M, n_out] = X[M, K](bf16) * W[n_out, K](bf16) + b, fp32 accumulate; models.py:460,585.
 * Backward: dX[M, K] (bf16, multiplied by the derivative of the activation `act` that produced X; optional
 * accumulate is not provided -- the trunk adds the density term through mnrf_gemm's rowv/colv),
 * dW[K, n_out] += (the fp32 master layout [in, out]), db[n_out] += (fp32 atomics);
 * dxsum[K] += column sums of dX (optional: bias gradient of the layer that produced X).
 * 0 < dw_split < n_out splits dW between two master matrices: outputs [0, dw_split) go to
 * dw [K, dw_split], outputs [dw_split, n_out) to dw2 [K, n_out - dw_split] (the density and rgb heads
 * of a view-independent model run as one stacked head; their weights live apart).  dx_cols (0: K) limits dX and
 * dxsum to the first dx_cols columns (a head reading [hidden | features] needs the gradient of the hidden part only).
 * dx2 (optional, needs dx_cols < K): dx2[M, K - dx_cols] (bf16, row pitch lddx2) receives the input gradient of
 * columns [dx_cols, K), never multiplied by the activation derivative and not summed into dxsum -- the rgb head of a
 * view MLP that ends on a skip layer reads [hidden | view input], and the second part is its contribution to the view
 * input's gradient.
 * act: the factor applied to dx[m, k] for k < dx_cols (dxsum sums the factored dx):
 *   MNRF_ACT_NONE                      none
 *   MNRF_ACT_RELU                      the ReLU mask X > 0
 *   MNRF_ACT_SOFTPLUS | MNRF_ACT_SILU  a'(z[m, k]), z [M, ldz] bf16 the pre-activation of the layer that produced X
 *                                      (mnrf_gemm FWD); needs dx, ldz a multiple of 8 and z 16-byte aligned
 * z is refused with any other act.
 * x (and dx) are read (written) in 16-byte chunks: both launches need them 16-byte aligned, with pitches that are
 * multiples of 8.  The forward needs w 16-byte aligned too; the backward takes any w.
 */
int mnrf_head_fwd(int64_t m, int32_t k, int32_t n_out, const mnrf_bf16* x, int64_t ldx,
                  const mnrf_bf16* w, const float* b, float* raw, mnrf_stream stream);
int mnrf_head_bwd(int64_t m, int32_t k, int32_t n_out, const mnrf_bf16* x, int64_t ldx,
                  const mnrf_bf16* w, const float* draw, mnrf_bf16* dx, int64_t lddx,
                  int32_t act, const mnrf_bf16* z, int64_t ldz, float* dw, float* dw2, int32_t dw_split,
                  float* db, float* dxsum, int32_t dx_cols, mnrf_bf16* dx2, int64_t lddx2, mnrf_stream stream);

/* The kernel instances and launch shapes mnrf_head_fwd and mnrf_head_bwd choose for these arguments (the ones the
 * choice depends on; x, w, z and dx take their places in the launches).  Host-only: no pointer is dereferenced and
 * nothing is launched.  Returns nonzero, with the backward launch's error message, for arguments mnrf_head_bwd
 * refuses; fwd_kernel is MNRF_HEAD_NONE where mnrf_head_fwd alone refuses them (w not 16-byte aligned). */
enum { MNRF_HEAD_NONE = 0, MNRF_HEAD_FWD_SUB = 1, MNRF_HEAD_FWD_WARP = 2, MNRF_HEAD_BWD_SUB = 3,
       MNRF_HEAD_BWD_WARP = 4 };
typedef struct {
  int32_t fwd_kernel;         /* MNRF_HEAD_FWD_SUB (head_fwd_sub_kernel) or MNRF_HEAD_FWD_WARP (head_fwd_kernel) */
  int32_t fwd_lpr;            /* sub kernel: lanes per row, K / 8 (32, 16 or 8); 0 otherwise */
  int32_t fwd_grid;           /* blocks */
  int32_t bwd_kernel;         /* MNRF_HEAD_BWD_SUB (head_bwd_sub_kernel) or MNRF_HEAD_BWD_WARP (head_bwd_kernel) */
  int32_t bwd_n_out;          /* template N_OUT */
  int32_t bwd_lpr;            /* sub kernel: lanes per row, K / 8; 0 otherwise */
  int32_t bwd_chunks;         /* warp-per-row kernel: kMaxChunks, 16-byte chunks per lane (1, 2, 4 or 6); 0 otherwise */
  int32_t bwd_smooth;         /* SMOOTH template flag: dx *= a'(z) */
  int32_t bwd_grid;           /* blocks */
  int32_t reserved;
  int64_t fwd_rows_per_pass;  /* rows one block covers per pass of its grid-stride loop */
  int64_t bwd_rows_per_block; /* rows of each block's range (the last block's may be shorter) */
} mnrf_head_instance;
int mnrf_head_plan(int64_t m, int32_t k, int32_t n_out, const mnrf_bf16* x, const mnrf_bf16* w, int32_t act,
                   const mnrf_bf16* z, const mnrf_bf16* dx, mnrf_head_instance* plan);

/* Column sums of a bf16 matrix into fp32 (bias gradients): out[N] += sum_m x[m, :].  x 16-byte aligned, N and ldx
 * multiples of 8. */
int mnrf_colsum(int64_t m, int32_t n, const mnrf_bf16* x, int64_t ldx, float* out,
                mnrf_stream stream);

/* ---- compositing ------------------------------------------------------------------------
 * Forward: density activation (models.py:506) + rgb activation/padding (models.py:584-602)
 * + render.compute_alpha_weights (render.py:130-151) + render.volumetric_rendering
 * (render.py:154-213).  One warp owns one ray.
 *   raw_density [B,S]; raw_rgb [B,S,3] or NULL (PropMLP: disable_rgb -> rgb = 0); ld_density / ld_rgb
 *   are the floats between consecutive samples of raw_density / raw_rgb and of their gradients (0: 1 and 3),
 *   so a stacked head's [B*S, 4] output is read and its gradient written in place (ld 4 for both)
 *   density_noise optional [B,S] N(0,1) draws (models.py:462-464)
 *   sdist [B,S+1]; directions [B,3]; near/far [B]; bg: scalar or NULL->bg_rgb [B,3]
 *   rgb_scale optional [B,3]: per-ray colour scale applied to the sample colours (RawNeRF
 *   exposure_values x learned exposure scaling, models.py:257-267)
 *   outputs: weights [B,S]; rgb_out [B,3]; optional density_out [B,S], rgb_samples [B,S,3]
 *   extras (compute_extras): acc [B], dist [B,4] = (mean, p5, median, p95) or NULL
 */
enum { MNRF_RGB_SIGMOID = 0, MNRF_RGB_SAFE_EXP = 1 };

typedef struct {
  int32_t num_rays, num_samples;
  int32_t raydist_fn, opaque_background;
  float density_bias, density_noise;
  int32_t rgb_act;
  float rgb_premult, rgb_bias, rgb_padding;
  float bg_const;
  int32_t rgb_mode;         /* 0: colour = act(raw_rgb); 1: diffuse + specular (models.py:588-599):
                               clip(linear_to_srgb(tint * act(raw_rgb) + sigmoid(raw_diffuse - log 3)), 0, 1),
                               tint = sigmoid(raw_tint) or 0.5 when raw_tint is NULL */
  int32_t ld_density, ld_rgb;
} mnrf_composite_desc;

int mnrf_composite_fwd(const mnrf_composite_desc* d, const float* raw_density,
                       const float* raw_rgb, const float* density_noise, const float* sdist,
                       const float* directions, const float* near, const float* far,
                       const float* bg_rgb, const float* rgb_scale, const float* raw_diffuse,
                       const float* raw_tint, float* weights, float* rgb_out,
                       float* density_out, float* rgb_samples, float* acc, float* dist,
                       mnrf_stream stream);

/* The activated, padded colour of M independent samples, as mnrf_composite_fwd's rgb_samples without compositing
 * and without a per-sample scale (colours of points, e.g. mesh vertices).  Reads d's rgb_act, rgb_premult, rgb_bias,
 * rgb_padding and rgb_mode only.
 *   raw_rgb [M, ld_rgb] (ld_rgb >= 3: 4 reads the rgb columns of a stacked [density | rgb] head in place, passed at
 *   its column 1); raw_diffuse [M, 3] with rgb_mode 1; raw_tint [M, 3] or NULL; rgb_out [M, 3] */
int mnrf_point_rgb(const mnrf_composite_desc* d, int64_t M, const float* raw_rgb, int32_t ld_rgb,
                   const float* raw_diffuse, const float* raw_tint, float* rgb_out, mnrf_stream stream);

/* Losses + compositing backward for one level (train_utils.py:72-159 + the adjoint of
 * render.py:130-213).  Fuses: data loss (mse | charb | rawnerf) on this level's pixel,
 * distortion loss (final level), interlevel loss (proposal levels, against the final
 * level's (sdist, weights)), then the alpha-compositing adjoint, the density-activation
 * and rgb-activation derivatives.
 *   outputs: d_raw_density [B,S]; d_raw_rgb [B,S,3] or NULL; stats[8] += (fp32 atomics):
 *     [0] data loss (already weighted by data_mult)  [1] mse  [2] distortion  [3] interlevel
 *   data_mask  optional [B] fp32 per-ray 0/1 weight on the data loss (data_loss_type 'robustnerf',
 *              train_utils.py:104-108): the data-loss value and its gradient of ray r are multiplied by
 *              data_mask[r]; the mse stat (stats[1]) stays unmasked.  NULL: unmasked.
 *   batch_rays the ray count the distortion and interlevel means divide by (>= num_rays): num_rays for a one-pass
 *              step; the whole batch for one pass of a train step that runs its batch in several passes, so each
 *              pass adds its share to stats and every per-sample gradient equals the one-pass step's.
 */
enum { MNRF_LOSS_MSE = 0, MNRF_LOSS_CHARB = 1, MNRF_LOSS_RAWNERF = 2 };

typedef struct {
  mnrf_composite_desc c;
  int32_t loss_type;
  float charb_padding;
  float data_mult;          /* data_loss_mult (final) or data_coarse_loss_mult (proposal) */
  float distortion_mult;    /* 0 on proposal levels */
  float interlevel_mult;    /* 0 on the final level */
  int32_t num_samples_fine; /* S of the final level (interlevel) */
  int32_t lossmult_channels;/* 1 or 3 */
} mnrf_loss_desc;

int mnrf_composite_bwd(const mnrf_loss_desc* d, const float* raw_density, const float* raw_rgb,
                       const float* density_noise, const float* sdist, const float* directions,
                       const float* near, const float* far, const float* bg_rgb,
                       const float* rgb_scale, const float* raw_diffuse, const float* raw_tint,
                       const float* extra_dw /* [B,S] added to dL/dweights, or NULL */,
                       const float* target_rgb,
                       const float* lossmult, const float* inv_denom /* device scalar */,
                       const float* sdist_fine, const float* weights_fine, const float* data_mask,
                       float* d_raw_density, float* d_raw_rgb, float* d_rgb_scale /* [B,3] or NULL */,
                       float* d_raw_diffuse, float* d_raw_tint, float* stats, int32_t batch_rays,
                       mnrf_stream stream);

/* ---- RobustNeRF mask and inlier threshold (robustnerf.py:8-115) ------------------------------
 * mnrf_robust_mask: one CTA per patch; rays are patch-major [num_rays / p^2, p, p].
 *   rgb, target [B,3]; threshold: device scalar (the previous step's loss_threshold; strict "<")
 *   mask [B] fp32 0/1 (all ones when enable == 0); error_per_pixel [B] = mean over the 3 channels of
 *   (rgb - target)^2, rounded as ((r0 + r1) + r2) / 3
 *   stats (optional): stats[1..4] += per-rank means of is_inlier_loss, has_inlier_neighbors,
 *   is_inlier_patch, mask (only mask when enable == 0), as count / batch_rays; needs `counts`, a uint32[5]
 *   workspace that is zero before the first launch and that every launch leaves zero.
 *   batch_rays (>= num_rays): num_rays for a one-pass step; the whole batch for one pass of a step over several,
 *   so the passes of a step add up to the batch's means.
 * Requires p*p <= 1024, num_rays a multiple of p*p, and (enable) inner_patch_size <= p, odd filter_size <= p.
 * Comparisons on neighbourhood / patch means use fl32(count / size) > fl32(1 - quantile); see csrc/robust.cu
 * for the tie rule of the box filter.
 * mnrf_quantile: out[0] = jnp.quantile(x[0:n], q) ('linear'), computed in fp32 as
 *   qn = q * (n - 1), lo = floor(qn), hi = ceil(qn), w = qn - lo, x_(lo) * (1 - w) + x_(hi) * w
 * (x_(i) = i-th smallest); NaN if any x is NaN.  One CTA, no workspace; 1 <= n < 2^24. */
typedef struct {
  int32_t num_rays;
  int32_t patch_size, inner_patch_size, filter_size;
  int32_t enable;
  float smoothed_thresh;    /* fl32(1 - robustnerf_smoothed_inlier_quantile) */
  float patch_thresh;       /* fl32(1 - robustnerf_inner_patch_inlier_quantile) */
} mnrf_robust_desc;

int mnrf_robust_mask(const mnrf_robust_desc* d, const float* rgb, const float* target, const float* threshold,
                     float* mask, float* error_per_pixel, uint32_t* counts, float* stats, int32_t batch_rays,
                     mnrf_stream stream);
int mnrf_quantile(int32_t n, float q, const float* x, float* out, mnrf_stream stream);

/* ---- Ref-NeRF per-sample stage ---------------------------------------------------------------
 * Between the spatial trunk and the directional MLP: normals_pred / normals = -l2_normalize(.)
 * (models.py:488-499, ref_utils.py:40-42), roughness = softplus(raw + bias) (models.py:520-523),
 * refdirs = reflect(-viewdirs, normals) (ref_utils.py:22-37, models.py:545), the integrated
 * directional encoding (ref_utils.generate_ide_fn ref_utils.py:98-159; ide_mat [l_max+1, ide_n]
 * fp32 and ide_ml int32 [2, ide_n] = (m | l) come from multinerf_b200/ref_utils.py) or coord.pos_enc,
 * and n.v (models.py:560-563).  Writes the bf16 slab [col0, col_end) of the view-MLP input.
 * raw_grad_density / d_raw_grad_density are direction-major [3, M].
 * Backward adds train_utils.orientation_loss (:162-178) and predicted_normal_loss (:181-197):
 * orient_mult / prednorm_mult are the level's multipliers divided by the number of rays;
 * extra_dw [M] (forward) receives d(loss)/d(weights) of those two terms; stats[4], stats[5] their
 * values.  After consuming d_slab[:, col0:col_end) (the gradient of the encoding), the backward
 * overwrites those columns with the 11 head gradients (raw_density, grad_pred x3, raw_diffuse x3,
 * raw_tint x3, raw_roughness; bf16, zero-padded) so that [bottleneck grad | head grads] is the A
 * operand of a single dgrad GEMM into the trunk.
 */
typedef struct {
  int64_t M;
  int32_t num_samples;
  int32_t use_pred_normals, use_density_normals, use_reflections, use_ide, use_n_dot_v, use_roughness;
  int32_t deg_view, ide_n;
  float roughness_bias;
  int32_t ld, col0, col_end;
} mnrf_refdir_desc;

int mnrf_refdir_fwd(const mnrf_refdir_desc* d, const float* ide_mat, const int32_t* ide_ml,
                    const float* grad_pred, const float* raw_rough, const float* raw_grad_density,
                    const float* viewdirs, float* normals_pred, float* normals, float* roughness,
                    mnrf_bf16* slab, float orient_mult, float prednorm_mult, int32_t orient_on_pred,
                    float* extra_dw /* [M] or NULL */, mnrf_stream stream);
int mnrf_refdir_bwd(const mnrf_refdir_desc* d, const float* ide_mat, const int32_t* ide_ml,
                    const float* grad_pred, const float* raw_rough, const float* raw_grad_density,
                    const float* viewdirs, const float* weights, mnrf_bf16* d_slab,
                    int32_t ld_dslab, float orient_mult, float prednorm_mult, int32_t orient_on_pred,
                    const float* d_raw_density, const float* d_raw_diffuse, const float* d_raw_tint,
                    float* d_grad_pred, float* d_raw_rough, float* d_raw_grad_density,
                    float* stats, mnrf_stream stream);
/* Colourless form of the stage, for an MLP with disable_rgb (a proposal MLP) whose normals only feed
 * the losses and the renderings: the normals, extra_dw and the loss adjoint of mnrf_refdir_fwd/bwd,
 * with no direction encoding.  grad_pred [M, 3] (with normals_pred / d_grad_pred) and
 * raw_grad_density [3, M] (with normals / d_raw_grad_density) may each be NULL, not both.
 * viewdirs [M / num_samples, 3] are read only for the orientation loss; weights and stats only when a
 * multiplier is > 0 (stats[4], stats[5] as above).  head_grads (optional, bf16 [M, ld_head_grads]):
 * the backward writes [d_raw_density | d_grad_pred] to its columns 0..3 and leaves the others alone, so
 * a zero-filled [M, 64] buffer is the A operand of one dgrad GEMM into the trunk against the K-major
 * [w_density | W_grad_pred | 0].  d_raw_rgb (optional, with head_grads: the rgb head of a view-independent
 * model on the same trunk) goes to columns 4..6, against [w_density | W_grad_pred | W_rgb | 0].  Sample m of
 * d_raw_density / d_raw_rgb is at m * ld_raw (0 reads as 1). */
int mnrf_normals_fwd(int64_t M, int32_t num_samples, const float* grad_pred, const float* raw_grad_density,
                     const float* viewdirs, float* normals_pred, float* normals, float orient_mult,
                     float prednorm_mult, int32_t orient_on_pred, float* extra_dw /* [M] or NULL */,
                     mnrf_stream stream);
int mnrf_normals_bwd(int64_t M, int32_t num_samples, const float* grad_pred, const float* raw_grad_density,
                     const float* viewdirs, const float* weights, float orient_mult, float prednorm_mult,
                     int32_t orient_on_pred, const float* d_raw_density, const float* d_raw_rgb, int64_t ld_raw,
                     float* d_grad_pred, float* d_raw_grad_density, mnrf_bf16* head_grads, int64_t ld_head_grads,
                     float* stats, mnrf_stream stream);
/* out[r, n] bf16 = maskbit(r mod mask_mod, n) ? rowv[r] * colv[n] : 0 -- the first dY of the
 * density-normal (tangent) backward chain.  N a multiple of 32, ld a multiple of 8, out 16-byte aligned. */
int mnrf_outer_mask(int64_t rows, int32_t n, int64_t mask_mod, const float* rowv, const float* colv,
                    const uint32_t* maskbits, int64_t ldmaskbits, mnrf_bf16* out, int64_t ldo,
                    mnrf_stream stream);
/* One trunk layer of the density-normal backward through a smooth activation a (act = MNRF_ACT_SOFTPLUS |
 * MNRF_ACT_SILU).  With z [M, N] the layer's pre-activation, T = dL/dt and u = t_in W the tangent before the
 * activation factor (t = a'(z) u), both three stacked streams [3M, N]:
 *   du[s*M + m, n] = a'(z[m, n]) T[s*M + m, n]                              dL/du, bf16; du may be T (in place)
 *   g[m, n]        = a''(z[m, n]) sum_s T[s*M + m, n] u[s*M + m, n]          the second-order part of dL/dz, bf16
 *                    (accumulate != 0: added to g's contents), fp32 arithmetic
 * N must be a multiple of 8, every pitch a multiple of 8 and every pointer 16-byte aligned. */
int mnrf_act_tangent_bwd(int64_t M, int32_t n, int32_t act, const mnrf_bf16* z, int64_t ldz, const mnrf_bf16* t_adj,
                         int64_t ldt, const mnrf_bf16* u, int64_t ldu, mnrf_bf16* du, int64_t lddu, mnrf_bf16* g,
                         int64_t ldg, int32_t accumulate, mnrf_stream stream);

/* ---- ray generation (the step before the path; SURVEY 8(f) row 1) --------------------------
 * camera_utils.pixels_to_rays (camera_utils.py:522-636) + the camera gather of
 * camera_utils.cast_ray_batch (:639-688), as the reference runs it on the device when
 * Config.cast_rays_in_train_step is set (train_utils.py:266-268): half-pixel offset, inverse
 * intrinsics, optional radial/tangential undistortion (_radial_and_tangential_undistort
 * :478-513, Newton steps), optional fisheye model, OpenCV->OpenGL flip, camera rotation,
 * optional NDC projection (convert_to_ndc :32-97), mip-NeRF cone radii from the dx/dy neighbours.
 * pixtocams [num_cameras, 3, 3] and camtoworlds [num_cameras, 3, 4] are row-major fp32;
 * cam_idx may be NULL when num_cameras == 1.  Outputs are [num_rays, 3|3|3|1|2] fp32.
 * Fisheye: sin(theta) / theta is 1 on the optical axis (theta = 0), where the reference's 0 / 0 gives NaN rays.
 */
#define MNRF_CAM_PERSPECTIVE 0
#define MNRF_CAM_FISHEYE 1
typedef struct {
  int32_t num_rays;
  int32_t num_cameras;
  int32_t camtype;
  int32_t has_distortion;
  float k1, k2, k3, k4, p1, p2;
  float undistort_eps;        /* 1e-9 in the reference */
  int32_t undistort_iters;    /* 10 in the reference */
  int32_t has_ndc;
  float ndc_p02, ndc_p12;     /* pixtocam_ndc[0][2], pixtocam_ndc[1][2] */
  float ndc_near;             /* 1.0 in the reference */
} mnrf_camera_desc;

int mnrf_pixels_to_rays(const mnrf_camera_desc* d, const int32_t* pix_x, const int32_t* pix_y,
                        const int32_t* cam_idx, const float* pixtocams, const float* camtoworlds,
                        float* origins, float* directions, float* viewdirs, float* radii,
                        float* imageplane, mnrf_stream stream);

/* camera_utils.cast_spherical_rays (camera_utils.py:716-763): an equirectangular 360-degree panorama of
 * height x width pixels, the render_camtype = 'pano' path of datasets.py:486-492.  Computed in fp64 as the
 * reference does: grid nodes theta = linspace(0, 2 pi, width + 1), phi = linspace(0, pi, height + 1) (numpy's
 * rounding: node k = k * (stop / n), the last node exactly stop); pixel (x, y) looks along node (x, y),
 * R [-sin(phi) sin(theta), cos(phi), sin(phi) cos(theta)] with R = camtoworld[:3, :3], not normalised;
 * radii from the differences to nodes (x+1, y) and (x, y+1) as in mnrf_pixels_to_rays; origins = the
 * camera position; imageplane = 0.  viewdirs = directions.
 * Outputs are [height * width, 3|3|3|1|2] fp32, row-major with y outer; 64-bit ray indices. */
typedef struct {
  int32_t height, width;
  double camtoworld[12];      /* [3, 4] row-major, by value: no device copy of the pose */
} mnrf_spherical_desc;

int mnrf_spherical_rays(const mnrf_spherical_desc* d, float* origins, float* directions, float* viewdirs,
                        float* radii, float* imageplane, mnrf_stream stream);

/* ---- optimizer ---------------------------------------------------------------------------
 * train_utils.clip_gradients (train_utils.py:200-218: value clip, then global-norm clip with
 * eps in the denominator), nan_to_num (:328) and optax.adam on one flat fp32 parameter
 * group (one top-level module).  norm_sq_scratch: device float[1], zeroed by the call.
 * dyn (optional): (lr, 1-beta1^t, 1-beta2^t) read from device memory dyn[0..2] instead of computed from d
 * (graph replay).
 */
typedef struct {
  int64_t n;
  float grad_max_val, grad_max_norm;
  float lr, beta1, beta2, eps;
  int32_t step;             /* 1-based update count t */
  float grad_scale;         /* multiplies the raw gradient first (1/world_size for pmean) */
} mnrf_adam_desc;

int mnrf_clip_adam(const mnrf_adam_desc* d, float* params, const float* grads, float* mu,
                   float* nu, float* norm_sq_scratch, const float* dyn, mnrf_stream stream);

/* fp32 master [in_pad, out] (row-major) -> bf16 shadows: w_nk [out, in_pad] (K-major operand
 * of the forward GEMM) and w_kn [in_pad, out] (K-major operand of the dgrad GEMM), for `count` layers
 * in one launch (the optimizer epilogue of a train step).  `items` is a
 * DEVICE array of mnrf_pack_item, ordered as the layers' 32x32 tiles are numbered: item i owns tiles
 * [tile0, tile0 + ceil(out/32) * ceil(in_pad/32)), tile0 of item i+1 = the end of item i;
 * total_tiles = the end of the last item. */
typedef struct {
  const float* master;
  mnrf_bf16* w_nk;          /* may be NULL */
  mnrf_bf16* w_kn;          /* may be NULL */
  int32_t in_pad, out;
  int32_t tile0;
  int32_t reserved;
} mnrf_pack_item;

int mnrf_pack_weights_batched(int32_t count, const mnrf_pack_item* items, int32_t total_tiles,
                              mnrf_stream stream);

/* ---- mesh extraction -----------------------------------------------------------------------
 * Marching cubes on an fp32 grid [nz, ny, nx] (each side in [2, 1024]); a point is inside when its value is
 * > level.  Point p = (z * ny + y) * nx + x owns the edges leaving it along +x, +y, +z (edge id 3 p + axis) and
 * the cell whose lowest corner it is (cell id p).  No reference counterpart (the reference has no mesh export).
 *   phase COUNT: edge_cut [3 N] uint8 = 1 where the edge crosses the level; cell_tris [N] uint8 = triangles of the
 *                cell (0 where p starts no cell).  N = nx * ny * nz.
 *   phase EMIT:  edge_scan [3 N] / tri_scan [N] int64: inclusive scans of edge_cut / cell_tris (V, F = their last
 *                elements); writes vertices [V, 3] (x, y, z in grid units: the linear crossing on the edge), one
 *                per cut edge in edge order, and faces [F, 3] int32 (V < 2^31) in cell order, wound so that normals
 *                point from inside to outside.
 * The mesh of a level set that stays off the grid boundary is closed and consistently wound.
 * A NaN grid point is unobserved: a cell with a NaN corner has no triangles, an edge with a NaN end is not cut, and
 * an edge is cut only if at least one cell it borders has eight non-NaN corners, so every vertex is used by a face.
 * On grids without NaN the output does not depend on this rule.
 */
enum { MNRF_MC_COUNT = 0, MNRF_MC_EMIT = 1 };
int mnrf_marching_cubes(int32_t phase, int32_t nx, int32_t ny, int32_t nz, const float* grid, float level,
                        uint8_t* edge_cut, uint8_t* cell_tris, const int64_t* edge_scan, const int64_t* tri_scan,
                        float* vertices, int32_t* faces, mnrf_stream stream);

/* Vertex normals of a marching-cubes mesh: after phase EMIT, with the same grid, level, edge_cut and edge_scan,
 * writes normals [V, 3], one unit vector per cut edge at the edge's rank -- the order of EMIT's vertices, so
 * normals[i] belongs to vertices[i].  The gradient of the grid at each end of the edge is taken by central
 * differences (one-sided on the grid boundary), the two are interpolated with the vertex's t, and the normal is
 * -g / |g|: from dense to empty space, the side the faces' winding faces.  The difference is one-sided next to a
 * NaN neighbour too; where both neighbours along an axis are NaN or missing, or g is zero or not finite, the normal
 * is the edge's direction from its inside end to its outside end.  Cells are cubes, so the normals hold in world
 * space too. */
int mnrf_mc_normals(int32_t nx, int32_t ny, int32_t nz, const float* grid, float level, const uint8_t* edge_cut,
                    const int64_t* edge_scan, float* normals, mnrf_stream stream);

/* Truncated signed-distance fusion of rendered depth maps into the grid points lo + h (x, y, z) of an [nz, ny, nx]
 * grid (each side in [2, 1024]; the points are rounded to fp32 from fp64, as mesh.density_grid places them).
 * cam: the camera model -- camtype, has_distortion, k1..k4, p1, p2 are read; num_cameras is the number of
 * camera-to-pixel matrices (1, shared, or num_views); has_ndc must be 0; the other fields are not read.
 * worldtocams [num_views, 3, 4]: world -> camera (OpenGL axes, the inverse of camtoworld); camtopixs
 * [num_cameras, 3, 3]: the inverse of pixtocam; depth, acc [num_views, height, width] fp32: each view's median
 * distance and opacity, distances in the units of the rays' directions; rgb [num_views, height, width, 3] or NULL.
 * State, updated in place: tsdf, weight [nz * ny * nx]; with rgb, color_sum [N, 3] and color_weight [N].
 * Per point and view, in view order: the view is skipped when the point has no pixel (behind a perspective camera,
 * theta = pi of a fisheye), its pixel (floor(u), floor(v)) is off the image or the depth is not finite.
 * d = depth - t (t: the point's parameter along its pixel's ray) where acc >= 0.5, +inf otherwise (the median
 * distance sits at `far`); skipped when d < -tau; else tsdf = (weight tsdf + min(d, tau) / tau) / (weight + 1),
 * weight += 1, and where |d| <= tau, color_sum += rgb, color_weight += 1.  One thread per point, no atomics: the
 * state depends on the views and their order, not on how they are split into calls. */
int mnrf_tsdf_integrate(const mnrf_camera_desc* cam, int32_t nx, int32_t ny, int32_t nz, double x0, double y0,
                        double z0, double h, int32_t num_views, int32_t height, int32_t width,
                        const float* worldtocams, const float* camtopixs, const float* depth, const float* acc,
                        const float* rgb, float tau, float* tsdf, float* weight, float* color_sum,
                        float* color_weight, mnrf_stream stream);

/* mnrf_tsdf_integrate on a grid in the contracted space of an unbounded scene (coord.contract; Config.mesh_space =
 * 'contracted'), with the same arguments, state and rules except: lo, h and tau are in contracted units; a grid point p
 * with |p| >= 2 (no world preimage) is left untouched, so its weight stays 0; the other points are projected at
 * x = inv_contract(p), and where acc >= 0.5, d = sign(depth - t) |contract(s) - p| with s = o + (x - o) depth / t the
 * pixel's surface point on the ray through x (o: the camera centre of the view's worldtocam). */
int mnrf_tsdf_integrate_contracted(const mnrf_camera_desc* cam, int32_t nx, int32_t ny, int32_t nz, double x0,
                                   double y0, double z0, double h, int32_t num_views, int32_t height, int32_t width,
                                   const float* worldtocams, const float* camtopixs, const float* depth,
                                   const float* acc, const float* rgb, float tau, float* tsdf, float* weight,
                                   float* color_sum, float* color_weight, mnrf_stream stream);

/* A mesh extracted in contracted space, back to world space: world_points[i] = inv_contract(points[i]) (z inside the
 * unit ball, z / (r (2 - r)) with r = |z| outside; |z| < 2 for a finite result), points [n, 3] fp32.  normals [n, 3] or
 * NULL (then world_normals NULL too): level-set normals in contracted space; world_normals[i] is the unit vector
 * along J(x) normals[i], J = d contract / dx at x = world_points[i] (symmetric: a gradient's pullback), or, where
 * that is zero or not finite, along normals[i], else (0, 0, 1). */
int mnrf_mesh_uncontract(int64_t n, const float* points, const float* normals, float* world_points,
                         float* world_normals, mnrf_stream stream);

/* Connected components of a triangle mesh (mesh cleaning, mesh.clean_mesh): the graph whose nodes are the
 * num_vertices vertices and whose edges are the edges of the num_faces faces [num_faces, 3] int32.  Every index must
 * lie in [0, num_vertices); the kernel does not check (ops.mesh_components does, on the device, before the call).
 * Writes labels [num_vertices] int32: each vertex's label is the smallest vertex index of its component, so a vertex
 * no face uses is its own label.  Union-find in three grid-stride passes with no host synchronisation: labels[v] = v;
 * hook (per face, join v0 with v1 and v0 with v2: find both roots, atomicCAS the larger root's parent from itself to
 * the smaller, retry on failure, path halving on the way); compress (labels[v] = v's root, walked without halving
 * stores, so every store of this pass is a root).  Parents only move to smaller indices, so the
 * labels are bit-deterministic whatever the thread schedule.  Degenerate and duplicate faces are fine.
 * No reference counterpart. */
int mnrf_mesh_components(int32_t num_vertices, int64_t num_faces, const int32_t* faces, int32_t* labels,
                         mnrf_stream stream);

/* For each of n points [n, 3] fp32 (world coordinates), the number of views whose image it lands on:
 * counts [n] int32.  Views and the camera as mnrf_tsdf_integrate reads them (cam: camtype perspective or fisheye,
 * has_distortion, k1..k4, p1, p2; num_cameras = 1 or num_views camera-to-pixel matrices; has_ndc must be 0;
 * worldtocams [num_views, 3, 4], camtopixs [num_cameras, 3, 3]).  A point lands on a view when it has a pixel there
 * (not behind a perspective camera, not at theta = pi of a fisheye) and that pixel (floor(u), floor(v)) lies in
 * [0, width) x [0, height): the rule mnrf_tsdf_integrate applies before it reads a pixel, from the same device
 * function.  Frustum only: occlusion is not considered.  One thread per point; deterministic.
 * No reference counterpart. */
int mnrf_points_view_count(const mnrf_camera_desc* cam, int64_t n, const float* points, int32_t num_views,
                           int32_t height, int32_t width, const float* worldtocams, const float* camtopixs,
                           int32_t* counts, mnrf_stream stream);

/* ---- mesh simplification by quadric edge collapse (mesh.simplify_mesh) -----------------------------------------
 * Parallel greedy quadric edge collapse (Garland and Heckbert 1997) in rounds.  No reference counterpart.  The
 * mesh: num_vertices vertices [V, 3] fp32 and num_faces faces [F, 3] int32; every face index lies in [0, V) and no
 * face repeats an index (mesh.simplify_mesh checks both on the device before the first call); V < 2^31.
 * The topology of the current faces, rebuilt by the caller before each round (mesh.mesh_topology):
 *   edges [E, 2] int32: the unique undirected edges (a, b), a < b, sorted by (a, b); E < 2^32, so an edge index
 *     fits the low 32 bits of a key;
 *   edge_off [E + 1] int64, edge_face [edge_off[E]] int32: the faces of edge e, ascending, at
 *     edge_face[edge_off[e] .. edge_off[e + 1]) (its face count is the difference);
 *   vf_off [V + 1] int64, vf_face [3 F] int32: the faces at vertex v, ascending, at vf_face[vf_off[v] .. vf_off[v + 1]).
 * A quadric is 10 fp64 values (aa, ab, ac, ad, bb, bc, bd, cc, cd, dd) of w (a, b, c, d)^T (a, b, c, d) for the
 * plane a x + b y + c z + d = 0 of unit normal (a, b, c) and weight w.  All geometry is fp64 in registers; the kernels
 * are compiled without FMA contraction, so their results are bit-reproducible from the stated operations
 * (tests/mesh_simplify_ref.py restates them).  The only atomics are atomicOr of flag bits and atomicMin of keys, so
 * every output is bit-deterministic. */

/* quadrics [V, 10] fp64: per vertex, the sum in this order of the plane quadric of each face at it (in face order),
 * weighted by the face's area (0 for a zero-area face), then of each boundary edge at it (in edge order): the plane
 * containing the edge and perpendicular to its face, weighted by 1000 |e|^2 (kBoundaryWeight).  The boundary edges
 * (the edges in exactly one face) of the current faces: boundary_edges [nb, 2] int32 in edge order, boundary_face
 * [nb] int32 their faces, vb_off [V + 1] int64 and vb_edge [2 nb] int32 the boundary edges at each vertex,
 * ascending. */
int mnrf_mesh_quadrics(int32_t num_vertices, int64_t num_faces, const float* vertices, const int32_t* faces,
                       const int64_t* vf_off, const int32_t* vf_face, int64_t num_boundary,
                       const int32_t* boundary_edges, const int32_t* boundary_face, const int64_t* vb_off,
                       const int32_t* vb_edge, double* quadrics, mnrf_stream stream);

/* Per edge e = (a, b): positions [E, 3] fp32, where a collapse of e puts the survivor, and keys [E] uint64.
 * Q = Q_a + Q_b; the position solves A v = -(q_ad, q_bd, q_cd) (A the upper 3x3 of Q) by cofactors unless
 * |det A| <= 1e-10 max|A_ij|^3 (kDetRel) or the solution lies farther than |b - a| from the midpoint; then it is the
 * cheapest of a, b and the midpoint (rounded to fp32), ties to the earlier.  The solution is rounded to fp32 before
 * its cost v^T Q v is taken; the cost is clamped to >= 0.  key = (fp32 bits of the cost, rounded to nearest) << 32 | e
 * when the edge may be collapsed, UINT64_MAX when not.  It may be collapsed when: it has 1 or 2 faces; neither end
 * touches an edge of more than 2 faces; it is not an edge of 2 faces whose ends are both on the boundary; at most 24
 * faces (kMaxValence) are at each end; every common neighbour of a and b is an apex of one of its faces, and no two
 * faces (a, x, y) and (b, x, y) exist; the collapse leaves a face of star(a) u star(b); and each face with exactly
 * one of a, b, that corner moved to the position, keeps a nonzero normal n' with n'.n > 0 where its normal n is
 * nonzero.  flags [V] int32 is scratch (bit 0: on the boundary, bit 1: on an edge of more than 2 faces). */
int mnrf_mesh_edge_cost(int32_t num_vertices, int64_t num_faces, int64_t num_edges, const float* vertices,
                        const int32_t* faces, const double* quadrics, const int32_t* edges, const int64_t* edge_off,
                        const int32_t* edge_face, const int64_t* vf_off, const int32_t* vf_face, int32_t* flags,
                        uint64_t* keys, float* positions, mnrf_stream stream);

/* selected [E] uint8 = 1 for the edges a round collapses: with vmin[v] the least key of the edges at v, fmin[f] the
 * least vmin of f's corners and rmin[v] the least fmin of the faces at v, edge (a, b) is selected when its key is
 * not UINT64_MAX and rmin[a] == rmin[b] == key.  No face touches two selected edges, and the least key is always
 * selected.  vmin, rmin [V] uint64 are scratch (they end holding those minima). */
int mnrf_mesh_collapse_select(int32_t num_vertices, int64_t num_faces, int64_t num_edges, const int32_t* faces,
                              const int32_t* edges, const uint64_t* keys, uint64_t* vmin, uint64_t* rmin,
                              uint8_t* selected, mnrf_stream stream);

/* Collapses each edge e = (a, b) with collapse[e] != 0, in place; the collapsed edges must be selected ones (a
 * subset of mnrf_mesh_collapse_select's, on the same topology and positions).  a survives: vertices[a] =
 * positions[e], quadrics[a] = Q_a + Q_b; with normals [V, 3] (may be NULL), normals[a] = the normalised
 * (1 - t) n_a + t n_b, t = clamp((p - a).(b - a) / |b - a|^2, 0, 1) (0 when a = b), unchanged when the blend is
 * zero.  The faces of e get face_alive[f] = 0 (every other face 1); in the other faces at b, b becomes a, so
 * the winding is kept.  b keeps its (now unused) entries. */
int mnrf_mesh_collapse_apply(int32_t num_vertices, int64_t num_faces, int64_t num_edges, const uint8_t* collapse,
                             const int32_t* edges, const int64_t* edge_off, const int32_t* edge_face,
                             const int64_t* vf_off, const int32_t* vf_face, const float* positions, float* vertices,
                             double* quadrics, float* normals, int32_t* faces, uint8_t* face_alive,
                             mnrf_stream stream);

/* ---- texture atlas of a mesh (mesh.bake_texture) ----------------------------------------------------------------
 * Per-face charts packed two faces per square cell of an S x S atlas (S = size, in [4, 16384]): n = ceil(sqrt(ceil(F
 * / 2))) cells per row, c = floor(S / n) texels per cell side, c >= 4 required (so at most 2 floor(S / 4)^2 faces);
 * cell k (row-major) holds faces 2k (A) and 2k + 1 (B) and starts at texel ((k % n) c, (k / n) c).  In the cell's
 * texel units, texel (i, j) centred at (i + 0.5, j + 0.5), a face's corners 0, 1, 2 are o, o + (d, 0), o + (0, d):
 * A has o = (0.5, 0.5), d = c - 3; B has o = (c - 0.5, c - 0.5), d = 2 - c.  Texel (i, j) belongs to A when
 * i + j + 2 <= c, else to B (to A when the cell has no B).  A bilinear sample inside a face's triangle reads only
 * texels its face owns, so no face bleeds into another at mip level 0.
 * Inputs: num_vertices vertices [V, 3] fp32, num_faces faces [F, 3] int32 (every index in [0, V); the kernel does not
 * check, ops.mesh_texture_raster does, on the device, before the call), vertex normals [V, 3] fp32.
 * Outputs: uv [F, 3, 2] fp32, each corner (u, v) in atlas texel units (u along a row, v down the rows; half-integers,
 * exact); and, for each texel t of the used cells, ceil(F / 2) c^2 of them, cell-major and row-major within a cell:
 * texel_index [T] int32 = row * S + column in the atlas, points [T, 3] = w0 p0 + w1 p1 + w2 p2 and texel_normals
 * [T, 3], where (w1, w2) are the owner's barycentrics (the texel centre's offset from o over d) clamped to the
 * triangle (w >= 0, then onto the hypotenuse w1 = clamp((w1 - w2 + 1) / 2, 0, 1), w2 = 1 - w1 when w1 + w2 > 1) and
 * w0 = 1 - w1 - w2: the nearest point of the triangle.  The normal is the unit w0 n0 + w1 n1 + w2 n2; where that is
 * zero, the face's unit (p1 - p0) x (p2 - p0); where that is zero too, (0, 0, 1).  A corner's texel has its vertex as
 * its point exactly.  fp32, no FMA contraction; deterministic.  No reference counterpart. */
int mnrf_mesh_texture_raster(int32_t num_vertices, int64_t num_faces, const float* vertices, const int32_t* faces,
                             const float* normals, int32_t size, float* uv, int32_t* texel_index, float* points,
                             float* texel_normals, mnrf_stream stream);

/* ---- closest-hit ray casting into a mesh (mesh.evaluate_mesh; csrc/mesh_trace.cu) ---------------------------------
 * A linear BVH over the faces (Karras 2012) and one thread per ray tracing it.  No reference counterpart.
 * The mesh: num_vertices vertices [V, 3] fp32, all finite, and num_faces faces [F, 3] int32 with every index in [0, V)
 * and 1 <= F < 2^30 (the kernels do not check; ops.mesh_bvh checks both on the device before the first call, and
 * handles F = 0 and F = 1 on the host: a one-face tree is its leaf, with no nodes).
 *   phase BOXES: face_boxes [F, 6] fp32 = (min xyz, max xyz) of each face's corners, and centroids [F, 3] fp32 =
 *                ((v0 + v1) + v2) / 3 per axis, each operation rounded to nearest.
 *   phase KEYS:  with centroid_bounds [6] fp32 = (min xyz, max xyz) of the centroids (on the device): keys [F] int64
 *                = morton << 32 | face, morton the 30-bit interleave (x highest) of each axis' cell
 *                floor(clamp((c - lo) / (hi - lo), 0, 1) * 1024) clamped to 1023 (0 where hi == lo).
 *   phase TREE:  with sorted_keys [F] int64 ascending, F >= 2: nodes [F - 1, 16] (fp32 with int32 children), parent
 *                [2 F - 1] int32, leaf_face [F] int32; counters [F - 1] int32 is scratch, zeroed by the call.  Node
 *                c < F - 1 is internal (0 is the root, whose parent is -1); node c >= F - 1 is leaf c - (F - 1), in
 *                key order, holding face leaf_face[c - (F - 1)] = sorted_keys[c - (F - 1)] & 0xffffffff.  Internal
 *                node i: floats [0, 6) and [6, 12) the boxes (min xyz, max xyz) of its left and right child, [12, 14)
 *                the children (int32), [14, 16) zero.  Children by Karras's split of the sorted keys; a leaf's box
 *                is its face's box, an internal node's the min / max of its children's.  The keys have 62
 *                significant bits and the common prefix grows at every level, so the depth is at most 63.
 * No rounding in the tree phase: the result is bit-reproducible (tests/mesh_trace_ref.py restates it).  Phases
 * BOXES and TREE read the inputs only on the device; none synchronises the host. */
enum { MNRF_BVH_BOXES = 0, MNRF_BVH_KEYS = 1, MNRF_BVH_TREE = 2 };
int mnrf_mesh_bvh(int32_t phase, int32_t num_vertices, int64_t num_faces, const float* vertices, const int32_t* faces,
                  float* face_boxes, float* centroids, const float* centroid_bounds, int64_t* keys,
                  const int64_t* sorted_keys, float* nodes, int32_t* parent, int32_t* leaf_face, int32_t* counters,
                  mnrf_stream stream);

/* Closest hit of each of num_rays rays: origins, directions [N, 3], near, far [N] fp32 (as Rays holds them).  Only
 * hits with near <= t <= far count, t the parameter along `directions` (not normalised).  The tree of mnrf_mesh_bvh
 * (nodes: NULL allowed when F = 1) on the same vertices and faces.  Outputs: hit_face [N] int32 (-1 for a miss),
 * hit_t [N] fp32 (+inf for a miss), hit_bary [N, 2] fp32, the barycentrics of corners faces[f, 1] and faces[f, 2]
 * (0 for a miss).  Among the faces tested the closest hit is the least (t, face), and the traversal is a fixed
 * function of the tree, so two runs on the same mesh are bit-identical.  A box is skipped when its fp32 entry
 * distance exceeds the best t, with no downward widening: where two faces' t tie exactly, a tree over the same faces
 * in another order can settle on the other one.  Ray/box: slab test, far bound widened by 1 + 2 gamma(3) rounded up
 * to a float (Ize 2013).  Ray/triangle: watertight
 * (Woop, Benthin and Wald 2013), a shear onto the dominant axis of the direction, fp32 edge functions recomputed in
 * fp64 when one is exactly 0, so a ray through a shared edge or vertex hits at least one of the faces there.  A ray
 * with a non-finite origin or direction component, a zero direction, a NaN near or far, or near > far misses.
 * Depth-first with a 64-entry stack per thread; should a push find it full, the ray ends as a miss and error_flag
 * (int32, device) is or-ed with 1: the caller reads it back.  fp32, no FMA contraction; no atomics but the flag. */
int mnrf_mesh_trace(int64_t num_rays, const float* origins, const float* directions, const float* near,
                    const float* far, int64_t num_faces, const float* nodes, const int32_t* leaf_face,
                    const float* vertices, const int32_t* faces, int32_t* hit_face, float* hit_t, float* hit_bary,
                    int32_t* error_flag, mnrf_stream stream);

#ifdef __cplusplus
}
#endif
#endif  /* MNRF_H_ */
