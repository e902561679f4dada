// Dense layers of the PropMLP / NerfMLP on Hopper tensor cores (sm_90a): persistent, warp-specialised GEMM
// with TMA-staged operands, wgmma.mma_async accumulating in registers and a fused epilogue.  Replaces nn.Dense
// (+ReLU, + skip-concat as a wider K) of models.py:436-437,455-460,527,577 and the dgrad / wgrad GEMMs
// jax.value_and_grad derives from them (train_utils.py:316-317).
//
//   warpgroup 0   : TMA producer (one thread) -- cp.async.bulk.tensor.2d into an operand ring of 128 x 64 A and
//                   BN x 64 B k-blocks; WGRAD with side sums: warps 1-3 sum the staged tiles (bias gradient,
//                   Dense(1) head gradient) while the consumers multiply them; gives its registers up (setmaxnreg) to
//   warpgroups 1-2: consumers -- each issues wgmma m64nBNk16 for 64 of the tile's 128 rows, keeps the fp32
//                   accumulators in registers and runs the epilogue from them: bias/ReLU/mask bits | rank-1 term,
//                   mask, addend, column sums | fp32 vector reductions.
//
// Operand layouts (all bf16, 128-byte swizzle):
//   FWD / DGRAD : A[M,K] and B[N,K] are K-major (reduction index contiguous);
//   WGRAD       : A = X[R,Mo] and B = dY[R,N] are "MN-major" (reduction index R on rows):
//                 out[Mo,N] += X^T dY, split over R with fp32 vector reductions.
#include <cuda.h>

#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "tc_common.cuh"

namespace mnrf {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;          // 64 bf16 = one 128-byte swizzle span
constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;        // 16 KiB
constexpr int NUM_THREADS = 384;
constexpr int CS_MAX = 1024;         // widest output the fused DGRAD column sums are offered for
// operand ring depth per tile width: 192 KB of the 227 KB of shared memory
constexpr int gemm_stages(int bn) { return bn == 256 ? 4 : bn == 128 ? 6 : 8; }
// TS: the bf16 output is staged in shared memory and written by TMA bulk stores, which leave coalesced full lines
// and run while the epilogue and the next tile's main loop do.  Each consumer warpgroup stages its 64 x BN tile one
// [64 rows x 64 cols] block (8 KB, 128-byte swizzle) at a time through a ring of staging blocks: two where the
// tile has an even number of blocks and the shared memory has room (FWD: DGRAD holds column sums and mask words),
// else one.
constexpr int STAGING_BLOCK_BYTES = 64 * 128;
constexpr int staging_blocks(int mode, int bn, bool ts) {
  return !ts ? 0 : (mode == MNRF_GEMM_FWD && bn >= 128) ? 2 : 1;
}
// DGRAD: mask words per row of a tile's TMA-loaded mask block.  A box row must be a multiple of 16 bytes and start
// 16-byte aligned, so tiles narrower than 128 columns load their mask words in the epilogue instead.
constexpr int mask_words(int bn) { return bn >= 128 ? bn / 32 : 0; }
constexpr int MASK_BUFS = 2;         // mask blocks in flight: the producer loads tile t+1's during tile t's epilogue
// DGRAD: per-consumer-warp column sums [8][BN] fp32, then MASK_BUFS mask blocks [128 rows][mask_words] uint32
constexpr int dgrad_smem_bytes(int bn) { return 8 * bn * 4 + MASK_BUFS * BLOCK_M * mask_words(bn) * 4; }
// WGRAD side sums: warps 1-3 of the producer warpgroup, 8 columns (one 16-byte chunk) per thread, whose partial sums
// meet in an fp32 scratch of [96 threads][8] once per tile
constexpr int SIDE_SCRATCH = 96 * 8;
constexpr int smem_bytes(int mode, int bn, bool ts, bool side) {
  return gemm_stages(bn) * (A_STAGE_BYTES + bn * BLOCK_K * 2) + 2 * staging_blocks(mode, bn, ts) * STAGING_BLOCK_BYTES +
         (mode == MNRF_GEMM_DGRAD ? dgrad_smem_bytes(bn) : 0) + (side ? SIDE_SCRATCH * 4 : 0) + 256 /*barriers*/ +
         1024 /*align*/;
}

struct GemmParams {
  int mode, act;
  int64_t m;                  // output rows
  int n, k;                   // output cols, reduction length
  int num_m_blocks, num_n_blocks, num_splits, kblocks_per_split, num_k_blocks;
  int64_t ldc, ldmask;        // SMOOTH instances: ldmask is the row pitch of z
  const float* bias;
  const float* rowv;
  const float* colv;
  const __nv_bfloat16* mask;  // SMOOTH instances (a smooth activation has no mask): the pre-activation z, which FWD
                              // writes (optional) and DGRAD multiplies by a'(z) (row = output row, mod mask_mod if > 0)
  uint32_t* maskbits;         // FWD+ReLU: written (1 bit per output, word = 32 columns); DGRAD: read
  int64_t ldmaskbits;         // in 32-bit words
  int64_t mask_mod;           // > 0: mask row = output row mod mask_mod
  int mask_tma;               // DGRAD: the producer loads each tile's mask words by TMA (else the epilogue's __ldg)
  const __nv_bfloat16* addend;  // DGRAD: out += addend[M, ldadd] (second contribution to a shared input)
  int64_t ldadd;
  float* colsum;              // DGRAD: colsum[N] += column sums of the output (bias gradient of the
                              // layer that produced the masking activation)
  float* bsum;                // WGRAD side sums (optional): bsum[N] += sum_r B[r, :]
  const float* side_w;        //   and side_aw[Mo] += sum_r side_w[r] * A[r, :]
  float* side_aw;
  void* out;
};

// Work item `tile` of the persistent loop: its column block, row block and the k-blocks [kb0, kb1) of its split
struct Tile {
  int n_blk, m_blk, kb0, kb1;
};
__device__ __forceinline__ Tile decode_tile(const GemmParams& p, int tile) {
  const int n_blk = tile % p.num_n_blocks;
  const int rest = tile / p.num_n_blocks;
  const int m_blk = rest % p.num_m_blocks;
  const int split = rest / p.num_m_blocks;
  const int kb0 = split * p.kblocks_per_split;
  return {n_blk, m_blk, kb0, min(p.num_k_blocks, kb0 + p.kblocks_per_split)};
}

// WGRAD side sums of one operand, run by NT threads of the producer warpgroup (t = 0..NT-1) beside the consumers:
//   B (WEIGHTED = false): out = bsum,    out[n_blk * BN + col]  += sum_r B[r, col]
//   A (WEIGHTED = true):  out = side_aw, out[m_blk * 128 + col] += sum_r side_w[r] A[r, col]
// Tile (m_blk, n_blk) sums, of every k-block it stages, the B rows r % num_m_blocks == m_blk and the A rows
// r % num_n_blocks == n_blk: every row of every (n-block, k-block) B tile and (m-block, k-block) A tile is summed
// once across the grid, and each stage costs the same few shared-memory reads.  (Summing whole k-blocks on every
// num_m_blocks-th stage instead holds those stages for longer than the MMAs take: under the wgmma traffic a shared
// load here takes a few hundred cycles.)  The threads wait on every stage as the consumers do and release it once
// read (empty_bar counts their warps).  MN-major stage layout: atoms of [64 r x 64 mn], the 16-byte chunk c of row r
// at chunk c ^ (r & 7).  Thread t owns the 8 columns of chunk t % CHUNKS, in fp32 registers (this warpgroup runs at 40
// registers a thread), and flushes them once per tile through `scratch`: the row groups meet there and one reduction
// per column leaves.  Rows past R are zero-filled by TMA; side_w is read as 0 there.
template <int STAGES, int STAGE_BYTES, int CHUNKS, int NT, bool WEIGHTED>
__device__ __forceinline__ void wgrad_side_sums(const GemmParams& p, int t, uint32_t ring, uint64_t* full_bar,
                                                uint64_t* empty_bar, uint32_t scratch) {
  constexpr int G = NT / CHUNKS;                     // row groups
  constexpr int COLS = CHUNKS * 8;
  static_assert(NT % CHUNKS == 0 && NT % 32 == 0, "side-sum warps tile the chunks");
  const int lane = t & 31;
  const int c = t % CHUNKS, g0 = t / CHUNKS;
  // chunk c in row 0 of a stage: the ring is 1024-byte aligned, so the swizzle is an XOR on address bits 4-6
  ring += (c >> 3) * (BLOCK_K * 128) + ((c & 7) << 4);
  const int total_tiles = p.num_m_blocks * p.num_n_blocks * p.num_splits;
  const int every = WEIGHTED ? p.num_n_blocks : p.num_m_blocks;
  const int step = every * G;                        // row stride of a thread
  uint32_t slot = 0;                                 // k-blocks consumed: stage slot % STAGES
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const auto [n_blk, m_blk, kb0, kb1] = decode_tile(p, tile);
    const int own = WEIGHTED ? n_blk : m_blk;        // first row of each k-block this tile sums
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
    for (int kb = kb0; kb < kb1; ++kb, ++slot) {
      float wlo = 0.f, whi = 0.f;                    // A: side_w of the k-block's 64 rows, two per lane
      if (WEIGHTED) {
        const int r0 = kb * BLOCK_K + lane;
        if (r0 < p.k) wlo = __ldg(p.side_w + r0);
        if (r0 + 32 < p.k) whi = __ldg(p.side_w + r0 + 32);
      }
      mbar_wait(&full_bar[slot % STAGES], (slot / STAGES) & 1, 6);
      const uint32_t base = ring + (slot % STAGES) * STAGE_BYTES;
      // the same trip count on every lane (the weights come by shuffle); B one row at a time, A two: deeper
      // unrolling spills
#pragma unroll(WEIGHTED ? 2 : 1)
      for (int r0 = own; r0 < BLOCK_K; r0 += step) {
        const int r = r0 + every * g0;
        float w = 1.f;                               // B: fma with 1 is the plain sum
        if (WEIGHTED) {                              // (the source lane's value cannot depend on this lane's r)
          const float wl = __shfl_sync(0xffffffffu, wlo, r & 31), wh = __shfl_sync(0xffffffffu, whi, r & 31);
          w = r < 32 ? wl : wh;
        }
        if (r < BLOCK_K) {
          const uint4 v = ld_shared_v4((base + r * 128) ^ ((r & 7) << 4));
          const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            acc[2 * q] = fmaf(w, bf16_lo(u[q]), acc[2 * q]);
            acc[2 * q + 1] = fmaf(w, bf16_hi(u[q]), acc[2 * q + 1]);
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[slot % STAGES]);
    }
    if (own < BLOCK_K && kb0 < kb1) {                // the same on all NT threads
      // thread t's partials at t * 8: row group g of column col sits at g * COLS + col
      if (NT > 32) named_bar_sync(4, NT); else __syncwarp();   // the previous flush has read the scratch
#pragma unroll
      for (int e = 0; e < 8; ++e) st_shared_u32(scratch + (t * 8 + e) * 4, __float_as_uint(acc[e]));
      if (NT > 32) named_bar_sync(4, NT); else __syncwarp();
      const int64_t col0 = WEIGHTED ? (int64_t)m_blk * BLOCK_M : (int64_t)n_blk * COLS;
      float* out = WEIGHTED ? p.side_aw : p.bsum;
      for (int col = t; col < COLS; col += NT) {
        if (WEIGHTED && col0 + col >= p.m) break;    // columns past Mo are never written
        float sum = 0.f;
#pragma unroll
        for (int g = 0; g < G; ++g) sum += __uint_as_float(ld_shared_u32(scratch + (g * COLS + col) * 4));
        atomicAdd(out + col0 + col, sum);
      }
    }
  }
}

// MNRF_GEMM_CLOCKS: a build for measurement only.  The first thread of each consumer warpgroup of CTA 0 of
// gemm_tc_pingpong_kernel splits its clock64() time into the classes below and adds them to g_gemm_clk[warpgroup]
// at the end of the launch (mnrf_gemm_clocks reads them).  Without it GemmClk is empty and tick() compiles to nothing.
enum { GK_TURN, GK_FULL, GK_MMA, GK_EPI_LOOP, GK_EPI_SYNC, GK_MASK, GK_N };
#ifdef MNRF_GEMM_CLOCKS
__device__ unsigned long long g_gemm_clk[2][GK_N];
struct GemmClk {
  long long t[GK_N] = {};
  long long last = 0;
  __device__ __forceinline__ void start() { last = clock64(); }
  __device__ __forceinline__ void tick(int k) {
    const long long now = clock64();
    t[k] += now - last;
    last = now;
  }
};
#else
struct GemmClk {
  __device__ __forceinline__ void start() {}
  __device__ __forceinline__ void tick(int) {}
};
#endif

// Epilogue operand sets of the ping-pong kernel (mnrf_gemm_instance.epilogue), one instance each, so the model's
// FWDs and DGRADs run an epilogue that tests no optional operand; the generic set tests each at run time.
//   DGRAD: mask bits by TMA (the trunk), and with the rank-1 term (the bottleneck);
//   FWD:   bias + ReLU + mask bits stored by TMA (trunk and view layers in training), bias + ReLU (the same layers
//          in a render), bias alone (the bottleneck).
enum {
  EPI_GENERIC = 0, EPI_BITS_TMA = 1, EPI_BITS_TMA_RANK1 = 2,
  EPI_FWD_BIAS_RELU_BITS = 3, EPI_FWD_BIAS_RELU = 4, EPI_FWD_BIAS = 5
};
constexpr bool epi_fwd(int ops) { return ops >= EPI_FWD_BIAS_RELU_BITS; }

// The FWD / DGRAD epilogue of one consumer warpgroup, from the accumulator fragment of wgmma m64nNC (per thread:
// acc[4i + 2h + e] is row 16*warp + lane/4 + 8h, column 8i + 2*(lane%4) + e of the warpgroup's 64 x NC block):
// FWD bias, then ReLU and mask bits or a smooth a(z) | DGRAD rank-1 term, mask bits (from the TMA-loaded mask block
// at m_tile if mask_tma, else from global memory), bf16 mask or a'(z), addend and, if do_cs, column sums into the
// warp's shared-memory slice at cs_lane.  An operand set OPS other than EPI_GENERIC fixes which of these are
// present at compile time; the FWD sets read the bias of columns [ncol0, ncol0 + NC) from shared memory at bias_s,
// and EPI_FWD_BIAS_RELU_BITS builds the mask words of the tile's 128 rows in the [128 rows x MW words] block at
// m_tile, which the call for rows [64, 128) writes out with one bulk store by tmap_m along with its last output
// block.  The block is rows [r0, r0 + 64) of the 128-row tile m_blk and columns
// [ncol0, ncol0 + NC); warpgroup wg (0 or 1) owns named barrier 2 + wg and staging blocks [wg * SB, wg * SB + SB).
// TS: the bf16 output goes through a ring of SB (1 to 3) staging blocks of [64 rows x 64 cols], one TMA bulk store
// per 64 columns; else it is stored from registers.  SB = 3 carries the ring position `sblk` across calls (a
// call stages two or four blocks); with SB = 1 or 2 block j of a call uses staging block j % SB.
template <int MODE, int NC, bool TS, int SB, bool SMOOTH, int OPS = EPI_GENERIC>
__device__ __forceinline__ void gemm_epilogue(const GemmParams& p, const CUtensorMap* tmap_c, const float (&acc)[NC / 2],
                                              int m_blk, int r0, int ncol0, int wg, uint8_t* smem_c, bool mask_tma,
                                              uint32_t m_tile, bool do_cs, uint32_t cs_lane, int& sblk, GemmClk& clk,
                                              const CUtensorMap* tmap_m = nullptr, uint32_t bias_s = 0) {
  constexpr int MW = mask_words(NC);
  static_assert(OPS == EPI_GENERIC || ((MODE == MNRF_GEMM_FWD) == epi_fwd(OPS) && TS && !SMOOTH && MW > 0),
                "fixed operand sets are FWD / DGRAD epilogues of the staged store with mask words by TMA");
  constexpr bool kFixed = OPS != EPI_GENERIC;
  constexpr bool kFwdFixed = kFixed && epi_fwd(OPS);
  const bool has_rowv = kFixed ? OPS == EPI_BITS_TMA_RANK1 : p.rowv != nullptr;
  const bool has_bits = kFixed ? OPS == EPI_FWD_BIAS_RELU_BITS || !kFwdFixed : p.maskbits != nullptr;
  const bool bits_tma = kFixed || mask_tma;
  const bool has_mask = !kFixed && p.mask != nullptr;
  const bool has_addend = !kFixed && p.addend != nullptr;
  const bool has_bias = kFixed || p.bias != nullptr;
  const bool relu = kFixed ? OPS != EPI_FWD_BIAS : p.act == MNRF_ACT_RELU;
  const int lane = threadIdx.x & 31;
  const int r_in = r0 + (16 * ((threadIdx.x >> 5) & 3) + (lane >> 2));   // this thread's row (h = 0) in the tile
  const int cq = 2 * (lane & 3);
  const bool leader = (threadIdx.x & 127) == 0;   // TS: issues and waits on the warpgroup's bulk stores
  // TS: this thread's row (h = 0) in the warpgroup's first staging block
  const uint32_t c_row = smem_u32(smem_c) + wg * (SB * STAGING_BLOCK_BYTES) + (r_in - r0) * 128 + (cq << 1);
  const uint32_t m_row = m_tile + r_in * (MW * 4);
  int64_t rows[2];
  bool row_ok[2];
  float rv[2] = {0.f, 0.f};
  const uint32_t* mrow[2] = {nullptr, nullptr};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    rows[h] = (int64_t)m_blk * BLOCK_M + r_in + 8 * h;
    row_ok[h] = rows[h] < p.m;
    if (MODE == MNRF_GEMM_DGRAD && row_ok[h]) {
      if (has_rowv) rv[h] = p.rowv[rows[h]];
      if (has_bits && !bits_tma)
        mrow[h] = p.maskbits + (p.mask_mod > 0 ? rows[h] % p.mask_mod : rows[h]) * p.ldmaskbits;
    }
  }
  uint32_t bits[2] = {0u, 0u};
  uint32_t mw[2] = {0u, 0u};                    // DGRAD mask bits: the rows' words of the current 32 columns
#pragma unroll
  for (int i = 0; i < NC / 8; ++i) {
    const int col = ncol0 + 8 * i + cq;
    const int sb = SB == 3 ? sblk : (i >> 3) & (SB - 1);   // TS: the block's staging block
    if (TS && SB == 1 && (i & 7) == 0) {
      // the previous bulk store must have finished reading the staging block
      clk.tick(GK_EPI_LOOP);
      if (leader) tma_store_wait_read<0>();
      named_bar_sync(2 + wg, 128);
      clk.tick(GK_EPI_SYNC);
    }
    if (MODE == MNRF_GEMM_DGRAD && has_bits && (i & 3) == 0) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
        mw[h] = bits_tma ? ld_shared_u32(m_row + (8 * h * MW + (i >> 2)) * 4)
                         : row_ok[h] ? __ldg(mrow[h] + (col >> 5)) : 0u;
    }
    float v[2][2];
#pragma unroll
    for (int h = 0; h < 2; ++h) { v[h][0] = acc[4 * i + 2 * h]; v[h][1] = acc[4 * i + 2 * h + 1]; }
    if (MODE == MNRF_GEMM_FWD) {
      if (has_bias) {
        const float2 b = kFwdFixed ? ld_shared_f2(bias_s + (8 * i + cq) * 4)
                                   : __ldg(reinterpret_cast<const float2*>(p.bias + col));
#pragma unroll
        for (int h = 0; h < 2; ++h) { v[h][0] += b.x; v[h][1] += b.y; }
      }
      if constexpr (SMOOTH) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (p.mask && row_ok[h])
            *reinterpret_cast<uint32_t*>(const_cast<__nv_bfloat16*>(p.mask) + rows[h] * p.ldmask + col) =
                pack_bf16(v[h][0], v[h][1]);
          v[h][0] = act_fwd(p.act, v[h][0]);
          v[h][1] = act_fwd(p.act, v[h][1]);
        }
      } else if (relu) {
        // bit 8 * (i % 4) + e of this thread's share of the word: shifted by cq once the word is complete
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            v[h][e] = relu_nan(v[h][e]);
            bits[h] |= (v[h][e] > 0.f ? 1u : 0u) << (8 * (i & 3) + e);
          }
      }
    } else {
      float2 cv = make_float2(0.f, 0.f);
      if (has_rowv) cv = __ldg(reinterpret_cast<const float2*>(p.colv + col));
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (has_rowv) { v[h][0] += rv[h] * cv.x; v[h][1] += rv[h] * cv.y; }
        if constexpr (SMOOTH) {
          if (row_ok[h]) {
            const int64_t zr = p.mask_mod > 0 ? rows[h] % p.mask_mod : rows[h];
            const uint32_t zz = __ldg(reinterpret_cast<const unsigned int*>(p.mask + zr * p.ldmask + col));
            v[h][0] *= act_d1(p.act, bf16_lo(zz));
            v[h][1] *= act_d1(p.act, bf16_hi(zz));
          }
        } else if (has_bits) {
          if (!((mw[h] >> (col & 31)) & 1u)) v[h][0] = 0.f;
          if (!((mw[h] >> ((col + 1) & 31)) & 1u)) v[h][1] = 0.f;
        } else if (has_mask && row_ok[h]) {
          const uint32_t mm = __ldg(reinterpret_cast<const unsigned int*>(p.mask + rows[h] * p.ldmask + col));
          if (!(bf16_lo(mm) > 0.f)) v[h][0] = 0.f;
          if (!(bf16_hi(mm) > 0.f)) v[h][1] = 0.f;
        }
        if (has_addend && row_ok[h]) {
          const uint32_t aa = __ldg(reinterpret_cast<const unsigned int*>(p.addend + rows[h] * p.ldadd + col));
          v[h][0] += bf16_lo(aa);
          v[h][1] += bf16_hi(aa);
        }
      }
      if (do_cs) {
        // column sums over the warp's 16 rows (rows past M hold zeros: zero-filled A tile, rv = 0).  The first
        // butterfly step swaps halves: lane bit 2 keeps column col + bit 2, so the two columns share the
        // remaining steps and one slice word.  Each sum is added in the same pairwise order as a butterfly per
        // column.  Lanes 0-7 own 8 distinct words of the warp's own slice: a plain load and store.
        const bool hi = (lane >> 2) & 1;
        const float s0 = v[0][0] + v[1][0], s1 = v[0][1] + v[1][1];
        float t = (hi ? s1 : s0) + __shfl_xor_sync(0xffffffffu, hi ? s0 : s1, 4);
        t += __shfl_xor_sync(0xffffffffu, t, 8);
        t += __shfl_xor_sync(0xffffffffu, t, 16);
        if (lane < 8) {
          const uint32_t a = cs_lane + 8 * i * 4;
          st_shared_u32(a, __float_as_uint(__uint_as_float(ld_shared_u32(a)) + t));
        }
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (TS) {
        // staging block sb, row r_in - r0 + 8h, 16-byte chunk (i % 8) ^ (row % 8), byte 2 * cq
        st_shared_u32(c_row + sb * STAGING_BLOCK_BYTES + h * (8 * 128) + (((i & 7) ^ ((lane >> 2) & 7)) << 4),
                      pack_bf16(v[h][0], v[h][1]));
      } else if (row_ok[h]) {
        *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(p.out) + rows[h] * p.ldc + col) =
            pack_bf16(v[h][0], v[h][1]);
      }
    }
    if (MODE == MNRF_GEMM_FWD && relu && has_bits && (i & 3) == 3) {
      // one 32-column mask word per row: the four lanes of a quad hold its 32 bits between them.  The fixed set
      // builds the tile's words in shared memory (rows past M included: the bulk store clips them).
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        bits[h] <<= cq;
        bits[h] |= __shfl_xor_sync(0xffffffffu, bits[h], 1);
        bits[h] |= __shfl_xor_sync(0xffffffffu, bits[h], 2);
        if ((lane & 3) == ((i >> 2) & 3)) {
          if (kFwdFixed) st_shared_u32(m_row + (8 * h * MW + (i >> 2)) * 4, bits[h]);
          else if (row_ok[h]) p.maskbits[rows[h] * p.ldmaskbits + (col >> 5)] = bits[h];
        }
        bits[h] = 0u;
      }
    }
    if (TS && (i & 7) == 7) {
      fence_proxy_async();                      // generic-proxy writes -> visible to the bulk store (async proxy)
      clk.tick(GK_EPI_LOOP);
      // SB >= 2: the store of block j - SB + 1, in the staging block that block j + 1 overwrites, has been read
      if (SB >= 2 && leader) tma_store_wait_read<SB - 2>();
      named_bar_sync(2 + wg, 128);
      if (leader) {                             // TMA clips the rows past M
        tma_store_2d(tmap_c, smem_c + (wg * SB + sb) * STAGING_BLOCK_BYTES, ncol0 + 8 * (i & ~7),
                     (int)((int64_t)m_blk * BLOCK_M + r0));
        // the tile's mask words are complete once the second half's last block is staged
        if (OPS == EPI_FWD_BIAS_RELU_BITS && i == NC / 8 - 1 && r0 == BLOCK_M - 64)
          tma_store_2d(tmap_m, m_tile, ncol0 / 32, m_blk * BLOCK_M);
        tma_store_commit();
      }
      if (SB == 3) sblk = sblk == 2 ? 0 : sblk + 1;
      clk.tick(GK_EPI_SYNC);
    }
  }
}

// SMOOTH: the epilogue of a softplus / SiLU layer (p.act): FWD stores z and applies a(z), DGRAD multiplies by a'(z)
// where the ReLU instances handle mask bits.  Separate instances, so the ReLU ones keep their code.
template <int MODE, int BN, bool TS, bool SIDE, bool SMOOTH = false>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               const __grid_constant__ CUtensorMap tmap_c, const __grid_constant__ CUtensorMap tmap_m,
               const GemmParams p) {
  constexpr int STAGES = gemm_stages(BN);
  constexpr int B_STAGE = BN * BLOCK_K * 2;
  constexpr bool kWgrad = (MODE == MNRF_GEMM_WGRAD);
  constexpr bool kDgrad = (MODE == MNRF_GEMM_DGRAD);
  constexpr int NACC = BN / 2;
  constexpr int SB = staging_blocks(MODE, BN, TS);
  constexpr int MW = mask_words(BN);
  static_assert(SB < 2 || (BN / 64) % 2 == 0, "block j of every tile must use staging block j % SB");
  static_assert(!SIDE || kWgrad, "side sums are a WGRAD feature");
  static_assert(!SMOOTH || (TS && !kWgrad), "smooth activations are FWD / DGRAD epilogues of the staged store");
  extern __shared__ uint8_t smem_dyn[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * A_STAGE_BYTES;
  uint8_t* smem_c = smem_b + STAGES * B_STAGE;                                   // TS: [2 warpgroups][SB] blocks
  // DGRAD: column sums of the current n-block, one private [BN] slice per consumer warp, then the mask blocks
  // (offsets stay multiples of 128 bytes, as TMA destinations need)
  float* cs_s = reinterpret_cast<float*>(smem_c + 2 * SB * STAGING_BLOCK_BYTES);  // [8][BN]
  float* side_s = cs_s;                                                          // WGRAD: [SIDE_SCRATCH]
  uint32_t* mask_s = reinterpret_cast<uint32_t*>(cs_s + (kDgrad ? 8 * BN : SIDE ? SIDE_SCRATCH : 0));  // [MASK_BUFS][BLOCK_M][MW]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(mask_s + (kDgrad ? MASK_BUFS * BLOCK_M * MW : 0));  // [STAGES]
  uint64_t* empty_bar = full_bar + STAGES;                                       // [STAGES]
  uint64_t* mask_full = empty_bar + STAGES;                                      // [MASK_BUFS]
  uint64_t* mask_empty = mask_full + MASK_BUFS;                                  // [MASK_BUFS]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  const int total_tiles = p.num_m_blocks * p.num_n_blocks * p.num_splits;
  const bool do_cs = kDgrad && p.colsum != nullptr;
  const bool mask_tma = kDgrad && p.mask_tma;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_b);
    if (TS) prefetch_tmap(&tmap_c);
    if (mask_tma) prefetch_tmap(&tmap_m);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      // one arrival per consumer warp and side-sum warp
      mbar_init(&empty_bar[i], 8 + (!SIDE ? 0 : !p.side_aw ? 3 : p.bsum ? 3 : 2));
    }
    for (int i = 0; i < MASK_BUFS; ++i) {
      mbar_init(&mask_full[i], 1);
      mbar_init(&mask_empty[i], 8);
    }
    fence_barrier_init();
  }
  if (do_cs)
    for (int i = threadIdx.x; i < 8 * BN; i += NUM_THREADS) cs_s[i] = 0.f;
  __syncthreads();
  // Programmatic dependent launch: nothing above touched global memory, everything below may.
  pdl_launch_dependents();
  pdl_wait();

  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      const uint32_t stage_bytes = A_STAGE_BYTES + B_STAGE;
      uint32_t stage = 0, phase = 0;
      for (int tile = blockIdx.x, it = 0; tile < total_tiles; tile += gridDim.x, ++it) {
        const auto [n_blk, m_blk, kb0, kb1] = decode_tile(p, tile);
        if (mask_tma) {
          // the tile's [128 rows x MW words] of mask bits; with mask_mod (a multiple of 128) the tile's rows map to
          // 128 consecutive mask rows.  Rows past the end are zero-filled.
          const int mb = it % MASK_BUFS;
          mbar_wait(&mask_empty[mb], ((it / MASK_BUFS) & 1) ^ 1, 4);
          mbar_expect_tx(&mask_full[mb], BLOCK_M * MW * 4);
          const int64_t r0 = (int64_t)m_blk * BLOCK_M;
          tma_load_2d(mask_s + mb * (BLOCK_M * MW), &tmap_m, &mask_full[mb], n_blk * (BN / 32),
                      (int)(p.mask_mod > 0 ? r0 % p.mask_mod : r0));
        }
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1, 1);
          mbar_expect_tx(&full_bar[stage], stage_bytes);
          uint8_t* sa = smem_a + stage * A_STAGE_BYTES;
          uint8_t* sb = smem_b + stage * B_STAGE;
          if (!kWgrad) {
            // K-major: box = [64 k][rows]
            tma_load_2d(sa, &tmap_a, &full_bar[stage], kb * BLOCK_K, m_blk * BLOCK_M);
            tma_load_2d(sb, &tmap_b, &full_bar[stage], kb * BLOCK_K, n_blk * BN);
          } else {
            // MN-major: one box per 64-wide MN atom = [64 mn][64 r], atoms BLOCK_K*128 bytes apart
#pragma unroll
            for (int a = 0; a < BLOCK_M / 64; ++a)
              tma_load_2d(sa + a * (BLOCK_K * 128), &tmap_a, &full_bar[stage], m_blk * BLOCK_M + a * 64, kb * BLOCK_K);
#pragma unroll
            for (int a = 0; a < BN / 64; ++a)
              tma_load_2d(sb + a * (BLOCK_K * 128), &tmap_b, &full_bar[stage], n_blk * BN + a * 64, kb * BLOCK_K);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    } else if (SIDE && warp > 0) {
      // ===================== WGRAD side sums =====================
      // bsum alone: warps 1-3.  With side_aw, whose A rows of every k-block are all read when N is one tile wide
      // (the bottleneck): warp 1 bsum, warps 2-3 side_aw.
      const uint32_t scratch = smem_u32(side_s);
      if (!p.side_aw) {
        wgrad_side_sums<STAGES, B_STAGE, BN / 8, 96, false>(p, threadIdx.x - 32, smem_u32(smem_b), full_bar, empty_bar,
                                                            scratch);
      } else if (warp >= 2) {
        wgrad_side_sums<STAGES, A_STAGE_BYTES, BLOCK_M / 8, 64, true>(p, threadIdx.x - 64, smem_u32(smem_a), full_bar,
                                                                      empty_bar, scratch + 32 * 8 * 4);
      } else if (p.bsum) {
        wgrad_side_sums<STAGES, B_STAGE, BN / 8, 32, false>(p, lane, smem_u32(smem_b), full_bar, empty_bar, scratch);
      }
    }
  } else {
    // ===================== consumers: MMA + epilogue =====================
    setmaxnreg_inc<232>();
    const int c = wg - 1;                       // rows [64c, 64c + 64) of each 128-row tile
    const int w = warp & 3;
    const int r_in = 64 * c + 16 * w + (lane >> 2);
    const int cq = 2 * (lane & 3);
    uint32_t stage = 0, phase = 0;
    float acc[NACC];
    // DGRAD: this warp's column-sum slice, at the column pair of lanes 0-7 after the butterfly below
    const uint32_t cs_lane = smem_u32(cs_s) + ((warp - 4) * BN + cq + ((lane >> 2) & 1)) * 4;
    for (int tile = blockIdx.x, it = 0; tile < total_tiles; tile += gridDim.x, ++it) {
      const auto [n_blk, m_blk, kb0, kb1] = decode_tile(p, tile);
      int prev = -1;
      fence_acc(acc);
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase, 3);
        const uint32_t sa = smem_u32(smem_a + stage * A_STAGE_BYTES);
        const uint32_t sb = smem_u32(smem_b + stage * B_STAGE);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / WGMMA_K; ++k) {
          uint64_t adesc, bdesc;
          if (!kWgrad) {
            adesc = make_smem_desc(sa + c * (64 * 128) + k * (WGMMA_K * 2), 0, 1024);
            bdesc = make_smem_desc(sb + k * (WGMMA_K * 2), 0, 1024);
          } else {
            adesc = make_smem_desc(sa + c * (BLOCK_K * 128) + k * (WGMMA_K * 128), BLOCK_K * 128, 1024);
            bdesc = make_smem_desc(sb + k * (WGMMA_K * 128), BLOCK_K * 128, 1024);
          }
          Wgmma<BN, kWgrad ? 1 : 0, kWgrad ? 1 : 0>::mma(acc, adesc, bdesc, (kb > kb0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();                        // the k-block before this one has been read: release its slot
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = (int)stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      fence_acc(acc);
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);

      const int ncol0 = n_blk * BN;
      if (MODE == MNRF_GEMM_WGRAD) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int64_t row = (int64_t)m_blk * BLOCK_M + r_in + 8 * h;
          if (row >= p.m) continue;
          float* dst = reinterpret_cast<float*>(p.out) + row * p.ldc + ncol0 + cq;
#pragma unroll
          for (int i = 0; i < BN / 8; ++i) atomicAdd(reinterpret_cast<float2*>(dst + 8 * i), make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]));
        }
        continue;
      }
      if (mask_tma) mbar_wait(&mask_full[it % MASK_BUFS], (it / MASK_BUFS) & 1, 5);
      int sblk = 0;                             // not read: SB < 3
      GemmClk clk;                              // the split covers the ping-pong kernel only
      clk.start();
      gemm_epilogue<MODE, BN, TS, SB, SMOOTH>(p, &tmap_c, acc, m_blk, 64 * c, ncol0, c, smem_c, mask_tma,
                                              smem_u32(mask_s) + (it % MASK_BUFS) * (BLOCK_M * MW * 4), do_cs, cs_lane,
                                              sblk, clk);
      if (mask_tma) {                           // this warp has read its mask words: the buffer may be refilled
        __syncwarp();
        if (lane == 0) mbar_arrive(&mask_empty[it % MASK_BUFS]);
      }
      const int next = tile + (int)gridDim.x;
      if (do_cs && (next >= total_tiles || next % p.num_n_blocks != n_blk)) {
        // the n-block's sums are complete: add the eight slices in warp order, one global reduction per column,
        // and clear the slices for the next n-block
        named_bar_sync(1, 2 * 128);
        for (int j = threadIdx.x - 128; j < BN; j += 2 * 128) {
          float s = 0.f;
#pragma unroll
          for (int sw = 0; sw < 8; ++sw) {
            s += cs_s[sw * BN + j];
            cs_s[sw * BN + j] = 0.f;
          }
          atomicAdd(p.colsum + ncol0 + j, s);
        }
        named_bar_sync(1, 2 * 128);
      }
    }
    if (TS && (threadIdx.x & 127) == 0) tma_store_wait_all();
  }
}

// ---------------------------------------------------------------------------- ping-pong schedule (FWD / DGRAD)
// gemm_tc_kernel runs both consumer warpgroups through the main loop and then through the epilogue together, so the
// tensor cores idle for the whole epilogue (a third to two thirds of a tile's time at the NerfMLP shapes).  Here each
// consumer warpgroup owns whole 128 x 128 sub-tiles instead: the CTA's tiles (the same 128 x BN tiles in the same
// order as gemm_tc_kernel) are cut into BN / 128 column sub-tiles, numbered it = 0, 1, ... in order, and warpgroup
// it & 1 runs sub-tile it.  An ordered hand-off (mma_turn) lets a warpgroup issue its sub-tile's wgmmas only once the
// other has issued all of the previous sub-tile's, so one warpgroup's epilogue runs under the other's MMAs.  Each
// output still accumulates its k-blocks in order through the same k16 steps: the outputs equal gemm_tc_kernel's bit
// for bit.  Staged store only; no column sums, no smooth activation.
constexpr int PP_BN = 128;             // sub-tile width
constexpr int PP_STAGES = 5;           // operand ring: 5 x 32 KB
// staging blocks per warpgroup (a sub-tile stages 4 blocks of 64 x 64).  DGRAD: three, so that before the bulk
// store of block j the leader waits only for block j - 2's to have been read, not for block j - 1's, issued just
// before.  FWD keeps two: with three, its 1024-wide layers measured slower (DESIGN.md section 3).
constexpr int pp_staging_blocks(int mode) { return mode == MNRF_GEMM_DGRAD ? 3 : 2; }
// Mask blocks of [128 rows x 4 words], sub-tile it in buffer it % PP_MASK_BUFS (warpgroup it & 1 owns buffers
// it & 1 and (it & 1) + 2).  DGRAD, loaded by TMA: four, so that the producer loads sub-tile it + 2's mask and
// operands while sub-tile it's epilogue still reads its mask block.  FWD with mask bits, built by the epilogue and
// stored by TMA: two per warpgroup, so that sub-tile it + 2 builds its words while sub-tile it's bulk store may
// still read them; the leader's wait for block 0 of sub-tile it + 2's output covers that store before it + 4.
// The FWD sets then keep each warpgroup's sub-tile bias, [PP_BN] fp32.
constexpr int PP_MASK_BUFS = 4;
constexpr int pp_smem_bytes(int mode, int ops) {
  return PP_STAGES * (A_STAGE_BYTES + PP_BN * BLOCK_K * 2) + 2 * pp_staging_blocks(mode) * STAGING_BLOCK_BYTES +
         (mode == MNRF_GEMM_DGRAD || ops == EPI_FWD_BIAS_RELU_BITS ? PP_MASK_BUFS * BLOCK_M * mask_words(PP_BN) * 4
                                                                   : 0) +
         (epi_fwd(ops) ? 2 * PP_BN * 4 : 0) + 256 /*barriers*/ + 1024 /*align*/;
}

// Accumulator fragments of the two wgmma m64n128 of a sub-tile (per consumer thread): acc[g][4i + 2h + e] is row
// 64g + 16*warp + lane/4 + 8h, column 8i + 2*(lane%4) + e of the warpgroup's 128 x 128 sub-tile.  OPS: the
// epilogue operand set.
template <int MODE, int BN, int OPS>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_tc_pingpong_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                        const __grid_constant__ CUtensorMap tmap_c, const __grid_constant__ CUtensorMap tmap_m,
                        const GemmParams p) {
  constexpr int STAGES = PP_STAGES;
  constexpr int B_STAGE = PP_BN * BLOCK_K * 2;
  constexpr int SUB = BN / PP_BN;        // sub-tiles per tile
  constexpr int MW = mask_words(PP_BN);
  constexpr int SB = pp_staging_blocks(MODE);
  constexpr bool kDgrad = (MODE == MNRF_GEMM_DGRAD);
  constexpr bool kFwdFixed = epi_fwd(OPS);                         // bias from shared memory
  constexpr bool kFwdBits = OPS == EPI_FWD_BIAS_RELU_BITS;         // mask words stored by TMA
  static_assert(MODE != MNRF_GEMM_WGRAD && (BN == 128 || BN == 256), "FWD / DGRAD tiles of 128 or 256 columns");
  extern __shared__ uint8_t smem_dyn[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * A_STAGE_BYTES;
  uint8_t* smem_c = smem_b + STAGES * B_STAGE;                                   // [2 warpgroups][SB] blocks
  uint32_t* mask_s = reinterpret_cast<uint32_t*>(smem_c + 2 * SB * STAGING_BLOCK_BYTES);  // [PP_MASK_BUFS][BLOCK_M][MW]
  float* bias_s = reinterpret_cast<float*>(mask_s + (kDgrad || kFwdBits ? PP_MASK_BUFS * BLOCK_M * MW : 0));  // [2][PP_BN]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(bias_s + (kFwdFixed ? 2 * PP_BN : 0));  // [STAGES]
  uint64_t* empty_bar = full_bar + STAGES;                                       // [STAGES]
  uint64_t* mask_full = empty_bar + STAGES;                                      // [PP_MASK_BUFS]
  uint64_t* mask_empty = mask_full + PP_MASK_BUFS;                               // [PP_MASK_BUFS]
  uint64_t* mma_turn = mask_empty + PP_MASK_BUFS;                               // [2]: warpgroup c may issue

  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  const int total_tiles = p.num_m_blocks * p.num_n_blocks;
  const int nk = p.num_k_blocks;         // k-blocks of every sub-tile
  const bool mask_tma = kDgrad && (OPS != EPI_GENERIC || p.mask_tma);

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_b);
    prefetch_tmap(&tmap_c);
    if (mask_tma || kFwdBits) prefetch_tmap(&tmap_m);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 4);     // the 4 warps of the warpgroup that consumes the stage
    }
    for (int i = 0; i < PP_MASK_BUFS; ++i) {
      mbar_init(&mask_full[i], 1);
      mbar_init(&mask_empty[i], 4);
    }
    for (int i = 0; i < 2; ++i) mbar_init(&mma_turn[i], 4);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  if (wg == 0) {
    // ===================== TMA producer: the sub-tiles' k-blocks in order, into one ring =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      uint32_t stage = 0, phase = 0;
      int it = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int n_blk = tile % p.num_n_blocks;
        const int m_blk = tile / p.num_n_blocks;
        for (int s = 0; s < SUB; ++s, ++it) {
          const int ncol0 = n_blk * BN + s * PP_BN;
          if (mask_tma) {
            // the sub-tile's [128 rows x MW words] of mask bits (mask_mod, a multiple of 128: 128 consecutive
            // mask rows); rows past the end are zero-filled
            const int mb = it % PP_MASK_BUFS;
            mbar_wait(&mask_empty[mb], ((it / PP_MASK_BUFS) & 1) ^ 1, 4);
            mbar_expect_tx(&mask_full[mb], BLOCK_M * MW * 4);
            const int64_t r0 = (int64_t)m_blk * BLOCK_M;
            tma_load_2d(mask_s + mb * (BLOCK_M * MW), &tmap_m, &mask_full[mb], ncol0 / 32,
                        (int)(p.mask_mod > 0 ? r0 % p.mask_mod : r0));
          }
          for (int kb = 0; kb < nk; ++kb) {
            mbar_wait(&empty_bar[stage], phase ^ 1, 1);
            mbar_expect_tx(&full_bar[stage], A_STAGE_BYTES + B_STAGE);
            tma_load_2d(smem_a + stage * A_STAGE_BYTES, &tmap_a, &full_bar[stage], kb * BLOCK_K, m_blk * BLOCK_M);
            tma_load_2d(smem_b + stage * B_STAGE, &tmap_b, &full_bar[stage], kb * BLOCK_K, ncol0);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else {
    // ===================== consumers: warpgroup c runs sub-tiles it = c, c + 2, ... =====================
    setmaxnreg_inc<232>();
    const int c = wg - 1;
    float acc[2][64];
    int sblk = 0;                                // SB = 3: the warpgroup's next staging block
    GemmClk clk;
    clk.start();
    for (int it = c; ; it += 2) {                // sub-tile it: column block it % SUB of the CTA's tile it / SUB
      const int tile = blockIdx.x + (it / SUB) * (int)gridDim.x;
      if (tile >= total_tiles) break;
      const int s = it % SUB;
      const int n_blk = tile % p.num_n_blocks;
      const int m_blk = tile / p.num_n_blocks;
      const int ncol0 = n_blk * BN + s * PP_BN;
      // FWD sets: one bias value of the sub-tile per thread, loaded under the main loop
      const float bias_v = kFwdFixed ? __ldg(p.bias + ncol0 + (threadIdx.x & 127)) : 0.f;
      // the ring slots of this sub-tile: the producer fills nk per sub-tile, in order
      const uint32_t slot = (uint32_t)it * (uint32_t)nk;
      uint32_t stage = slot % STAGES, phase = (slot / STAGES) & 1;
      clk.tick(GK_EPI_LOOP);
      // the other warpgroup has issued every wgmma of sub-tile it - 1
      if (it > 0) mbar_wait(&mma_turn[c], ((it - 1) >> 1) & 1, 7);
      clk.tick(GK_TURN);
      int prev = -1;
      fence_acc(acc[0]);
      fence_acc(acc[1]);
      for (int kb = 0; kb < nk; ++kb) {
        mbar_wait(&full_bar[stage], phase, 3);
        clk.tick(GK_FULL);
        const uint32_t sa = smem_u32(smem_a + stage * A_STAGE_BYTES);
        const uint32_t sb = smem_u32(smem_b + stage * B_STAGE);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / WGMMA_K; ++k) {
          const uint64_t bdesc = make_smem_desc(sb + k * (WGMMA_K * 2), 0, 1024);
#pragma unroll
          for (int g = 0; g < 2; ++g)
            Wgmma<PP_BN, 0, 0>::mma(acc[g], make_smem_desc(sa + g * (64 * 128) + k * (WGMMA_K * 2), 0, 1024), bdesc,
                                    (kb > 0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();                        // the k-block before this one has been read: release its slot
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = (int)stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
        clk.tick(GK_MMA);
      }
      // every wgmma of this sub-tile is issued: the other warpgroup's next sub-tile may start
      if (blockIdx.x + ((it + 1) / SUB) * (int)gridDim.x < total_tiles) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&mma_turn[c ^ 1]);
      }
      wgmma_wait<0>();
      fence_acc(acc[0]);
      fence_acc(acc[1]);
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      clk.tick(GK_MMA);

      // ---- epilogue: rows [64g, 64g + 64) of the sub-tile from acc[0], one 64 x 64 staging block per 8 columns.
      // A rolled loop that moves acc[1] into acc[0] for its second pass: unrolled, nvcc hoists the second half's
      // loads into the first and the DGRAD instances spill 2.4 KB.
      const uint32_t m_base = smem_u32(mask_s) + (it % PP_MASK_BUFS) * (BLOCK_M * MW * 4);
      if (mask_tma) mbar_wait(&mask_full[it % PP_MASK_BUFS], (it / PP_MASK_BUFS) & 1, 5);
      // FWD sets: the bias into the warpgroup's slice.  Every read of the previous sub-tile's bias came before the
      // warpgroup's last named barrier of that epilogue; the barrier here orders the writes before this one's reads.
      const uint32_t bias_wg = smem_u32(bias_s) + c * (PP_BN * 4);
      if (kFwdFixed) {
        st_shared_u32(bias_wg + (threadIdx.x & 127) * 4, __float_as_uint(bias_v));
        named_bar_sync(2 + c, 128);
      }
      clk.tick(GK_MASK);
#pragma unroll 1
      for (int g = 0; g < 2; ++g) {
        gemm_epilogue<MODE, PP_BN, true, SB, false, OPS>(p, &tmap_c, acc[0], m_blk, 64 * g, ncol0, c, smem_c, mask_tma,
                                                         m_base, false, 0, sblk, clk, &tmap_m, bias_wg);
#pragma unroll
        for (int e = 0; e < 64; ++e) acc[0][e] = acc[1][e];   // rows [64, 128) next
      }
      if (mask_tma) {                           // this warp has read its mask words: the buffer may be refilled
        __syncwarp();
        if (lane == 0) mbar_arrive(&mask_empty[it % PP_MASK_BUFS]);
      }
    }
    if ((threadIdx.x & 127) == 0) tma_store_wait_all();
#ifdef MNRF_GEMM_CLOCKS
    clk.tick(GK_EPI_SYNC);
    if (blockIdx.x == 0 && (threadIdx.x & 127) == 0)
      for (int k = 0; k < GK_N; ++k) atomicAdd(&g_gemm_clk[c][k], (unsigned long long)clk.t[k]);
#endif
  }
}

// ------------------------------------------------------------------------------------ host
template <int MODE, int BN, int OPS = EPI_GENERIC>
static int launch_gemm_tc_pingpong(int grid, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc,
                                   const CUtensorMap& tm, const GemmParams& p, cudaStream_t stream) {
  constexpr int kSmem = pp_smem_bytes(MODE, OPS);
  static_assert(kSmem <= 232448, "shared memory budget");
  return launch_tc<gemm_tc_pingpong_kernel<MODE, BN, OPS>>(grid, NUM_THREADS, kSmem, stream, ta, tb, tc, tm, p);
}

// DGRAD ping-pong at tile width BN, in the instance of its epilogue operand set
template <int BN>
static int launch_dgrad_pingpong(int ops, int grid, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc,
                                 const CUtensorMap& tm, const GemmParams& p, cudaStream_t stream) {
  switch (ops) {
    case EPI_BITS_TMA:
      return launch_gemm_tc_pingpong<MNRF_GEMM_DGRAD, BN, EPI_BITS_TMA>(grid, ta, tb, tc, tm, p, stream);
    case EPI_BITS_TMA_RANK1:
      return launch_gemm_tc_pingpong<MNRF_GEMM_DGRAD, BN, EPI_BITS_TMA_RANK1>(grid, ta, tb, tc, tm, p, stream);
  }
  return launch_gemm_tc_pingpong<MNRF_GEMM_DGRAD, BN>(grid, ta, tb, tc, tm, p, stream);
}

// FWD ping-pong at tile width BN, in the instance of its epilogue operand set
template <int BN>
static int launch_fwd_pingpong(int ops, int grid, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc,
                               const CUtensorMap& tm, const GemmParams& p, cudaStream_t stream) {
  switch (ops) {
    case EPI_FWD_BIAS_RELU_BITS:
      return launch_gemm_tc_pingpong<MNRF_GEMM_FWD, BN, EPI_FWD_BIAS_RELU_BITS>(grid, ta, tb, tc, tm, p, stream);
    case EPI_FWD_BIAS_RELU:
      return launch_gemm_tc_pingpong<MNRF_GEMM_FWD, BN, EPI_FWD_BIAS_RELU>(grid, ta, tb, tc, tm, p, stream);
    case EPI_FWD_BIAS:
      return launch_gemm_tc_pingpong<MNRF_GEMM_FWD, BN, EPI_FWD_BIAS>(grid, ta, tb, tc, tm, p, stream);
  }
  return launch_gemm_tc_pingpong<MNRF_GEMM_FWD, BN>(grid, ta, tb, tc, tm, p, stream);
}

template <int MODE, int BN, bool TS, bool SIDE, bool SMOOTH = false>
static int launch_gemm_tc(int grid, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc,
                          const CUtensorMap& tm, const GemmParams& p, cudaStream_t stream) {
  constexpr int kSmem = smem_bytes(MODE, BN, TS, SIDE);
  static_assert(kSmem <= 232448, "shared memory budget");
  return launch_tc<gemm_tc_kernel<MODE, BN, TS, SIDE, SMOOTH>>(grid, NUM_THREADS, kSmem, stream, ta, tb, tc, tm, p);
}

// The SMOOTH instances are compiled in a translation unit of their own (gemm_tc_act.cu): instantiated beside the
// ReLU ones, they change how nvcc optimises the ReLU DGRAD instances.
int gemm_tc_smooth_launch(int mode, int block_n, int grid, const CUtensorMap& ta, const CUtensorMap& tb,
                          const CUtensorMap& tc, const GemmParams& p, cudaStream_t stream);

#ifndef MNRF_GEMM_TC_SMOOTH_UNIT
static int pick_block_n(int n) {
  const int cands[] = {256, 128, 64, 32, 16};
  for (int c : cands)
    if (n % c == 0) return c;
  return 0;
}

// The host-side choices of gemm_tc_launch, after every argument check: tile width, store path, where DGRAD's mask
// bits come from, instance family, reduction splits and grid, and the tile counts of the launch parameters `p`.
// Dereferences nothing (mnrf_gemm_plan).
static int gemm_tc_plan(const mnrf_gemm_desc* d, const mnrf_bf16* a, const mnrf_bf16* b, const float* bias,
                        const float* colv, const mnrf_bf16* mask, const uint32_t* maskbits, const float* colsum,
                        const mnrf_bf16* addend, const void* out, const float* bsum, const float* side_w,
                        const float* side_aw, const mnrf_bf16* z, int64_t ldz, mnrf_gemm_instance* plan,
                        GemmParams* p) {
  // K-major modes: the reduction index is the contiguous one and layers are padded to 64.  WGRAD reduces
  // over the sample rows, any count: the last 64-row block is zero-filled by TMA past the tensor's end.
  MNRF_CHECK(d->mode == MNRF_GEMM_WGRAD || d->k % BLOCK_K == 0,
             "mnrf_gemm(tc): reduction length %d must be a multiple of %d", d->k, BLOCK_K);
  MNRF_CHECK(d->lda % 8 == 0 && d->ldb % 8 == 0 && ((uintptr_t)a % 16) == 0 && ((uintptr_t)b % 16) == 0,
             "mnrf_gemm(tc): operands must be 16-byte aligned with ld %% 8 == 0");
  const int block_n = pick_block_n(d->n);
  MNRF_CHECK(block_n > 0, "mnrf_gemm(tc): N=%d must be a multiple of 16", d->n);
  if (d->mode == MNRF_GEMM_WGRAD)
    MNRF_CHECK(block_n >= 64, "mnrf_gemm(tc): WGRAD needs N %% 64 == 0 (MN-major 128-byte atoms), N=%d", d->n);
  if (addend) MNRF_CHECK(d->mode == MNRF_GEMM_DGRAD && d->ldadd % 2 == 0 && ((uintptr_t)addend % 4) == 0,
                         "mnrf_gemm(tc): addend is a DGRAD input with 4-byte aligned rows");
  if (colsum) MNRF_CHECK(d->mode == MNRF_GEMM_DGRAD && d->n <= CS_MAX,
                         "mnrf_gemm(tc): colsum is a DGRAD output of at most %d columns", CS_MAX);
  const bool side = bsum != nullptr || side_aw != nullptr;
  if (side) MNRF_CHECK(d->mode == MNRF_GEMM_WGRAD && (side_w == nullptr) == (side_aw == nullptr),
                       "mnrf_gemm(tc): side sums are WGRAD outputs; side_w and side_aw come together");
  if (maskbits) {
    MNRF_CHECK(d->mode != MNRF_GEMM_WGRAD, "mnrf_gemm(tc): maskbits make no sense for WGRAD");
    MNRF_CHECK(d->n % 32 == 0 && block_n % 32 == 0 && d->ldmaskbits * 32 >= d->n,
               "mnrf_gemm(tc): maskbits need N %% 32 == 0 and ldmaskbits >= N/32");
  }
  const bool smooth = d->mode != MNRF_GEMM_WGRAD && (d->act == MNRF_ACT_SOFTPLUS || d->act == MNRF_ACT_SILU);
  if (smooth) {
    MNRF_CHECK(!maskbits && !mask, "mnrf_gemm(tc): a smooth activation takes z, not a ReLU mask");
    MNRF_CHECK(d->mode == MNRF_GEMM_FWD || z, "mnrf_gemm(tc): the DGRAD of a smooth activation needs z");
    MNRF_CHECK(!z || (ldz % 2 == 0 && ((uintptr_t)z % 4) == 0), "mnrf_gemm(tc): z must be 4-byte aligned");
  }
  if (bias) MNRF_CHECK(((uintptr_t)bias % 8) == 0, "mnrf_gemm(tc): bias must be 8-byte aligned");
  if (colv) MNRF_CHECK(((uintptr_t)colv % 8) == 0, "mnrf_gemm(tc): colv must be 8-byte aligned");
  const int workers = mnrf_num_sms();
  const int num_m_blocks = (int)((d->m + BLOCK_M - 1) / BLOCK_M);
  const int num_n_blocks = d->n / block_n;
  const int num_k_blocks = (d->k + BLOCK_K - 1) / BLOCK_K;
  int num_splits = 1;
  if (d->mode == MNRF_GEMM_WGRAD) {
    // Split the reduction over the sample rows so that (output tiles x splits) work items fill whole rounds of the
    // workers -- with the FEWEST splits that do: every work item ends in an fp32 reduction pass over its output
    // tile, and for a one-tile weight gradient (PropMLP 256 x 256) those passes all hit the same 256 KB of L2.
    const int out_tiles = num_m_blocks * num_n_blocks;
    const int max_splits = std::min(std::max(1, (2 * workers) / out_tiles), num_k_blocks);
    int splits = max_splits;
    for (int sp = 1; sp <= max_splits; ++sp) {
      const int items = out_tiles * sp;
      const int rounds = (items + workers - 1) / workers;
      if (items * 100 >= rounds * workers * 95) { splits = sp; break; }
    }
    num_splits = splits;
  }
  const int kblocks_per_split = (num_k_blocks + num_splits - 1) / num_splits;
  num_splits = (num_k_blocks + kblocks_per_split - 1) / kblocks_per_split;
  if (d->mode != MNRF_GEMM_WGRAD) {
    MNRF_CHECK(d->ldc % 2 == 0 && ((uintptr_t)out % 4) == 0, "mnrf_gemm(tc): bf16 output must be 4-byte aligned");
    if (mask) MNRF_CHECK(d->ldmask % 2 == 0 && ((uintptr_t)mask % 4) == 0, "mnrf_gemm(tc): mask must be 4-byte aligned");
  } else {
    MNRF_CHECK(d->ldc % 2 == 0 && ((uintptr_t)out % 8) == 0, "mnrf_gemm(tc): fp32 output must be 8-byte aligned");
  }
  // The bf16 output goes through the staged bulk store when its tiles are whole 128-byte swizzle spans and TMA can
  // address it (16-byte aligned base and row pitch); otherwise the epilogue stores from registers.
  const bool ts = d->mode != MNRF_GEMM_WGRAD && block_n >= 64 && ((uintptr_t)out % 16) == 0 && d->ldc % 8 == 0;
  // the smooth epilogues exist for the staged store only: every hidden layer is a multiple of 64 wide
  MNRF_CHECK(!smooth || ts, "mnrf_gemm(tc): a smooth activation needs N %% 64 == 0 and a 16-byte aligned output "
             "with a row pitch that is a multiple of 8");
  // Mask words can move by TMA when the tile is at least 128 columns wide and the words are a TMA-addressable array
  // (16-byte aligned base and row pitch).  DGRAD loads them so when the mask rows of a 128-row tile are 128
  // consecutive rows; otherwise the epilogue loads them itself.
  const bool bits_tma_ok = maskbits && mask_words(block_n) > 0 && d->ldmaskbits % 4 == 0 &&
                           ((uintptr_t)maskbits % 16) == 0;
  bool mask_tma = d->mode == MNRF_GEMM_DGRAD && bits_tma_ok && (d->mask_mod == 0 || d->mask_mod % BLOCK_M == 0);
  // FWD and DGRAD run the ping-pong schedule (gemm_tc_pingpong_kernel) wherever it has an epilogue: staged store,
  // whole 128-column sub-tiles, ReLU or no activation, no column sums.
  const bool pingpong = d->mode != MNRF_GEMM_WGRAD && ts && d->n % PP_BN == 0 && !smooth && !colsum;
  // The ping-pong epilogue's operand set.  DGRAD: mask bits by TMA, with or without the rank-1 term (rowv and colv
  // come together).  FWD with a bias: ReLU with mask bits the epilogue stores by TMA, ReLU without mask bits, or no
  // activation and no mask bits; FWD mask bits are stored by TMA only in that set.  Any other combination runs the
  // generic one.
  int epilogue = EPI_GENERIC;
  if (pingpong && d->mode == MNRF_GEMM_DGRAD && mask_tma && !mask && !addend)
    epilogue = colv ? EPI_BITS_TMA_RANK1 : EPI_BITS_TMA;
  if (pingpong && d->mode == MNRF_GEMM_FWD && bias) {
    if (d->act == MNRF_ACT_RELU)
      epilogue = !maskbits ? EPI_FWD_BIAS_RELU : bits_tma_ok ? EPI_FWD_BIAS_RELU_BITS : EPI_GENERIC;
    else if (d->act == MNRF_ACT_NONE && !maskbits)
      epilogue = EPI_FWD_BIAS;
    mask_tma = epilogue == EPI_FWD_BIAS_RELU_BITS;
  }
  const int tiles = num_m_blocks * num_n_blocks * num_splits;
  plan->block_n = block_n;
  plan->staged = ts;
  plan->mask_tma = mask_tma;
  plan->smooth = smooth;
  plan->side = side;
  plan->splits = num_splits;
  plan->tiles = tiles;
  plan->grid = std::min(tiles, workers);
  plan->pingpong = pingpong;
  plan->epilogue = epilogue;
  p->num_m_blocks = num_m_blocks;
  p->num_n_blocks = num_n_blocks;
  p->num_k_blocks = num_k_blocks;
  p->num_splits = num_splits;
  p->kblocks_per_split = kblocks_per_split;
  return 0;
}

// FWD / DGRAD through the register store, at every tile width
template <int MODE>
static int launch_register_store(int block_n, int grid, const CUtensorMap& ta, const CUtensorMap& tb,
                                 const CUtensorMap& tc, const CUtensorMap& tm, const GemmParams& p,
                                 cudaStream_t stream) {
  switch (block_n) {
    case 256: return launch_gemm_tc<MODE, 256, false, false>(grid, ta, tb, tc, tm, p, stream);
    case 128: return launch_gemm_tc<MODE, 128, false, false>(grid, ta, tb, tc, tm, p, stream);
    case 64: return launch_gemm_tc<MODE, 64, false, false>(grid, ta, tb, tc, tm, p, stream);
    case 32: return launch_gemm_tc<MODE, 32, false, false>(grid, ta, tb, tc, tm, p, stream);
    case 16: return launch_gemm_tc<MODE, 16, false, false>(grid, ta, tb, tc, tm, p, stream);
  }
  set_error("mnrf_gemm(tc): no register-store instance at BN=%d", block_n);
  return 1;
}

// Launches the instance of a plan.  Only the combinations gemm_tc_plan produces have one: FWD and DGRAD with the
// staged store at BN >= 128 run the ping-pong kernel unless the activation is smooth or DGRAD has column sums, and
// WGRAD needs BN >= 64.
static int launch_gemm_tc_plan(int mode, const mnrf_gemm_instance& plan, const CUtensorMap& ta, const CUtensorMap& tb,
                               const CUtensorMap& tc, const CUtensorMap& tm, const GemmParams& p,
                               cudaStream_t stream) {
  const int bn = plan.block_n, grid = plan.grid;
  const bool fwd = mode == MNRF_GEMM_FWD;
  if (plan.pingpong) {
    if (bn == 256)
      return fwd ? launch_fwd_pingpong<256>(plan.epilogue, grid, ta, tb, tc, tm, p, stream)
                 : launch_dgrad_pingpong<256>(plan.epilogue, grid, ta, tb, tc, tm, p, stream);
    if (bn == 128)
      return fwd ? launch_fwd_pingpong<128>(plan.epilogue, grid, ta, tb, tc, tm, p, stream)
                 : launch_dgrad_pingpong<128>(plan.epilogue, grid, ta, tb, tc, tm, p, stream);
  } else if (plan.smooth) {
    return gemm_tc_smooth_launch(mode, bn, grid, ta, tb, tc, p, stream);
  } else if (mode == MNRF_GEMM_WGRAD) {
    if (bn == 256)
      return plan.side ? launch_gemm_tc<MNRF_GEMM_WGRAD, 256, false, true>(grid, ta, tb, tc, tm, p, stream)
                       : launch_gemm_tc<MNRF_GEMM_WGRAD, 256, false, false>(grid, ta, tb, tc, tm, p, stream);
    if (bn == 128)
      return plan.side ? launch_gemm_tc<MNRF_GEMM_WGRAD, 128, false, true>(grid, ta, tb, tc, tm, p, stream)
                       : launch_gemm_tc<MNRF_GEMM_WGRAD, 128, false, false>(grid, ta, tb, tc, tm, p, stream);
    if (bn == 64)
      return plan.side ? launch_gemm_tc<MNRF_GEMM_WGRAD, 64, false, true>(grid, ta, tb, tc, tm, p, stream)
                       : launch_gemm_tc<MNRF_GEMM_WGRAD, 64, false, false>(grid, ta, tb, tc, tm, p, stream);
  } else if (!plan.staged) {
    return fwd ? launch_register_store<MNRF_GEMM_FWD>(bn, grid, ta, tb, tc, tm, p, stream)
               : launch_register_store<MNRF_GEMM_DGRAD>(bn, grid, ta, tb, tc, tm, p, stream);
  } else if (bn == 64) {
    return fwd ? launch_gemm_tc<MNRF_GEMM_FWD, 64, true, false>(grid, ta, tb, tc, tm, p, stream)
               : launch_gemm_tc<MNRF_GEMM_DGRAD, 64, true, false>(grid, ta, tb, tc, tm, p, stream);
  } else if (!fwd) {   // DGRAD with column sums
    if (bn == 256) return launch_gemm_tc<MNRF_GEMM_DGRAD, 256, true, false>(grid, ta, tb, tc, tm, p, stream);
    if (bn == 128) return launch_gemm_tc<MNRF_GEMM_DGRAD, 128, true, false>(grid, ta, tb, tc, tm, p, stream);
  }
  set_error("mnrf_gemm(tc): no kernel instance for mode %d, BN=%d, staged %d, side sums %d", mode, bn, plan.staged,
            plan.side);
  return 1;
}

int gemm_tc_launch(const mnrf_gemm_desc* d, const mnrf_bf16* a, const mnrf_bf16* b, const float* bias,
                   const float* rowv, const float* colv, const mnrf_bf16* mask, uint32_t* maskbits,
                   float* colsum, const mnrf_bf16* addend, void* out, cudaStream_t stream, float* bsum,
                   const float* side_w, float* side_aw, mnrf_bf16* z, int64_t ldz) {
  mnrf_gemm_instance plan;
  GemmParams p{};
  if (int rc = gemm_tc_plan(d, a, b, bias, colv, mask, maskbits, colsum, addend, out, bsum, side_w, side_aw, z, ldz,
                            &plan, &p))
    return rc;
  const int block_n = plan.block_n;
  const bool ts = plan.staged;
  p.mode = d->mode; p.act = d->act; p.m = d->m; p.n = d->n; p.k = d->k;
  p.ldc = d->ldc; p.ldmask = d->ldmask;
  p.bias = bias; p.rowv = rowv; p.colv = colv;
  p.mask = reinterpret_cast<const __nv_bfloat16*>(mask);
  p.out = out;
  p.maskbits = maskbits;
  p.ldmaskbits = d->ldmaskbits;
  p.mask_mod = d->mask_mod;
  p.addend = reinterpret_cast<const __nv_bfloat16*>(addend);
  p.ldadd = d->ldadd;
  p.colsum = colsum;
  p.bsum = bsum; p.side_w = side_w; p.side_aw = side_aw;
  if (plan.smooth) {
    p.mask = reinterpret_cast<const __nv_bfloat16*>(z);
    p.ldmask = ldz;
  }
  p.mask_tma = plan.mask_tma;
  CUtensorMap ta, tb, tc;
  if (d->mode != MNRF_GEMM_WGRAD) {
    if (make_tmap(&ta, a, d->m, d->k, d->lda, BLOCK_K, BLOCK_M)) return 1;
    if (make_tmap(&tb, b, d->n, d->k, d->ldb, BLOCK_K, plan.pingpong ? PP_BN : block_n)) return 1;
  } else {
    // A = X[R, Mo], B = dY[R, N]; reduction index on rows
    if (make_tmap(&ta, a, d->k, d->m, d->lda, 64, BLOCK_K)) return 1;
    if (make_tmap(&tb, b, d->k, d->n, d->ldb, 64, BLOCK_K)) return 1;
  }
  if (ts) {
    if (make_tmap(&tc, out, d->m, d->n, d->ldc, 64, 64)) return 1;
  } else {
    tc = tb;   // not read
  }
  // DGRAD loads [128 rows x words] blocks of the mask words by it, FWD stores them (FWD ignores mask_mod)
  CUtensorMap tm = tb;   // not read unless p.mask_tma
  if (p.mask_tma &&
      make_tmap(&tm, maskbits, d->mode == MNRF_GEMM_DGRAD && d->mask_mod > 0 ? d->mask_mod : d->m, d->n / 32,
                d->ldmaskbits,
                mask_words(plan.pingpong ? PP_BN : block_n), BLOCK_M, CU_TENSOR_MAP_DATA_TYPE_UINT32, 4,
                CU_TENSOR_MAP_SWIZZLE_NONE))
    return 1;
  if (plan.grid == 0) return 0;
  if (int rc = launch_gemm_tc_plan(d->mode, plan, ta, tb, tc, tm, p, stream)) return rc;
  MNRF_LAUNCH_CHECK();
  return 0;
}
#endif  // MNRF_GEMM_TC_SMOOTH_UNIT

}  // namespace mnrf

#ifndef MNRF_GEMM_TC_SMOOTH_UNIT
extern "C" int mnrf_gemm_plan(const mnrf_gemm_desc* d, const mnrf_bf16* a, const mnrf_bf16* b, const float* bias,
                              const float* rowv, const float* colv, const mnrf_bf16* mask, const uint32_t* maskbits,
                              const float* colsum, const mnrf_bf16* addend, const mnrf_bf16* z, int64_t ldz,
                              const void* out, const float* bsum, const float* side_w, const float* side_aw,
                              mnrf_gemm_instance* plan) {
  MNRF_CHECK(d && plan, "mnrf_gemm_plan: null pointer");
  MNRF_CHECK((rowv == nullptr) == (colv == nullptr), "mnrf_gemm: rowv and colv come together");
  MNRF_CHECK(!mask || d->mask_mod == 0, "mnrf_gemm: mask_mod applies to maskbits and z, not to a bf16 mask");
  mnrf::GemmParams p;
  return mnrf::gemm_tc_plan(d, a, b, bias, colv, mask, maskbits, colsum, addend, out, bsum, side_w, side_aw, z, ldz,
                            plan, &p);
}

#ifdef MNRF_GEMM_CLOCKS
// measurement build only: read (and clear) the ping-pong kernel's clock64() classes, [warpgroup][class], summed since
// the last call
extern "C" int mnrf_gemm_clocks(unsigned long long* out) {
  unsigned long long zero[2 * mnrf::GK_N] = {};
  if (cudaDeviceSynchronize() != cudaSuccess) return 1;
  if (cudaMemcpyFromSymbol(out, mnrf::g_gemm_clk, sizeof(zero)) != cudaSuccess) return 1;
  return cudaMemcpyToSymbol(mnrf::g_gemm_clk, zero, sizeof(zero)) != cudaSuccess;
}
#endif
#endif
