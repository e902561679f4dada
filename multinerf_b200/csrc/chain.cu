// Layer-chained 256-wide MLP trunk on Hopper tensor cores (sm_90a): ONE persistent launch walks row blocks of
// samples through ALL Dense layers of a trunk (forward) or through its whole input-gradient chain (backward).
// Replaces the per-layer launches of models.py:441-465 (`x = dense_layer(net_width)(x); x = net_activation(x)`,
// skip-concat as extra K blocks) and of the matching reverse-mode chain, for the 256-wide MLPs (PropMLP of
// 360.gin; PropMLP/NerfMLP of the blender / llff / Ref-NeRF / RawNeRF configs).
//
// Why: a 256-wide layer has 128 FLOP per byte of activation traffic when every layer reads its input from HBM
// and writes its output back -- below the H100's machine balance (~295 FLOP/B) -- so per-layer kernels are
// HBM-bound.  Here the activations of a row block stay in shared memory between layers (they are written out
// only where a later pass needs them), accumulators live in registers, weights stream from L2 through a TMA ring.
//
// Work decomposition (per CTA):
//   unit    = 128 sample rows; consumer warpgroup c owns rows [64c, 64c + 64) and a 64 x 256 fp32 accumulator;
//   layer   = wgmma 64 x 256 x K per warpgroup, then an epilogue that turns the accumulator into the next layer's
//             A operand in shared memory (SWIZZLE_128B K-major, 4 k-blocks) and, where asked, bulk-stores it;
//   weights : k-blocks [256 N rows x 64 K] stream from L2 through a ring of four 32 KB slots, once per unit for both
//             warpgroups (128 KB per 256 x 256 layer and 128 rows);
//   streamed: a STREAMED operand (IPE features of layer 0 / of a skip layer, or the incoming gradient of the
//             backward chain) travels as [64 rows x 64] blocks, one per warpgroup and k-block, through a ring of
//             three 8 KB blocks of its own.
//
// Schedule: a layer's k-blocks are cut into segments of at most CH_SEG k-blocks (a resident 256-wide layer is one
// segment) and the two consumer warpgroups take turns segment by segment (`turn`, as mma_turn of
// gemm_tc_pingpong_kernel): warpgroup 0 issues a segment's wgmmas for its rows, hands over, warpgroup 1 issues the
// same segment for its rows.  After a layer's last segment a warpgroup runs its epilogue while the other still has
// that segment's MMAs on the tensor cores.  Every output accumulates the same k-blocks through the same k16 steps,
// whoever issues when.
//
//   warpgroup 0   : TMA producer (one thread)
//   warpgroups 1-2: consumers (wgmma + epilogue + bulk stores of their own rows)
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "tc_common.cuh"

namespace mnrf {

constexpr int CH_W = 256;                   // layer width: N of every MMA, K of the resident operand
constexpr int CH_ROWS = 128;                // rows of a unit
constexpr int CH_KBLK = CH_ROWS * 128;      // one [128 rows x 64 bf16] k-block, SWIZZLE_128B
constexpr int CH_WBLK = CH_W * 128;         // one [256 rows x 64 bf16] weight k-block
constexpr int CH_RING = 4;                  // weight slots
constexpr int CH_SEG = CH_W / 64;           // k-blocks of a segment (at most): one resident layer
constexpr int CH_SBLK = 64 * 128;           // one warpgroup's [64 rows x 64 bf16] block of the streamed operand
constexpr int CH_SRING = 3;                 // streamed-operand blocks
constexpr int CH_ACT = 4 * CH_KBLK;         // a 128 x 256 bf16 activation block = 4 k-blocks
constexpr int CH_THREADS = 384;
constexpr int CH_MAX_LAYERS = MNRF_CHAIN_MAX_LAYERS;
constexpr int CH_AUX = CH_MAX_LAYERS * CH_W * 4;   // FWD: the biases of every layer; BWD: the column sums
constexpr int CH_SMEM = CH_ACT + CH_RING * CH_WBLK + CH_SRING * CH_SBLK + CH_AUX + 256 /*barriers*/ + 1024 /*align*/;
static_assert(CH_SMEM <= 232448, "shared memory budget");
// Why the hand-off cannot deadlock.  The producer issues its loads in one fixed order: segment by segment, and
// within a segment the weight k-blocks each followed by warpgroup 0's streamed block, then warpgroup 1's streamed
// blocks.  Warpgroup 0 consumes a prefix of that order and warpgroup 1 the rest, so a load never waits for a slot
// whose occupant needs a LATER load to be consumed.  What remains is the turn: warpgroup 1 may start segment s only
// when warpgroup 0 has issued all of it, and a weight slot is freed only when both have consumed it (`wempty`
// counts 8 warps), so warpgroup 0 needs every weight k-block of segment s in a slot at the same time.  That holds
// because a segment has at most CH_SEG <= CH_RING k-blocks: the slot a k-block of segment s wants was last used
// by a k-block of an EARLIER segment, which warpgroup 1 consumes on a turn that depends on earlier segments only.
// A hand-off per layer with more k-blocks than slots would hang; the segment length is a constant, not a
// property of the launch.  Slots are released when the wgmmas that read them have completed, before any wait on
// `turn`, so a release never depends on the other warpgroup.
static_assert(CH_SEG >= 1 && CH_SEG <= CH_RING, "a segment must fit in the weight ring");

struct alignas(64) ChainMaps {
  CUtensorMap stream;
  CUtensorMap w[CH_MAX_LAYERS];
  CUtensorMap out[CH_MAX_LAYERS];
};

struct ChainLayer {
  int n_stream, stream_col0, stream_kb0;
  int n_res, res_kb0;
  int store;
  const float* bias;
  uint32_t* maskbits;
  int64_t ldmaskbits;
  float* colsum;
};

struct ChainParams {
  int num_layers;
  int64_t m;
  int64_t num_units;
  ChainLayer layer[CH_MAX_LAYERS];
  const float* head_w;      // FWD: [NH][256] narrow head on the last layer's output, fp32 copy of the bf16 rows
  const float* head_b;      //   (NH = 1: the density head; 4: density + rgb of a view-independent model)
  float* head_out;          // [m][NH]
};

// two fp32 -> packed bf16x2 with ReLU in the conversion (one instruction for both lanes)
__device__ __forceinline__ uint32_t pack_bf16_relu(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.relu.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// Read-only shared data (the biases, written once before the unit loop): not volatile, so the compiler may move
// the load ahead of the epilogue's shared-memory stores.
__device__ __forceinline__ float2 ld_shared_const_f2(uint32_t addr) {
  float2 v;
  asm("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
  return v;
}

// MNRF_CHAIN_CLOCKS: a build for measurement only.  The first thread of consumer warpgroup 1 of CTA 0 splits its
// clock64() time into the classes below and adds them to g_chain_clk at the end of the launch.
enum { CK_TURN, CK_FULL, CK_MMA, CK_EPI_SYNC, CK_EPI_LOOP, CK_EPI_TAIL, CK_N };
#ifdef MNRF_CHAIN_CLOCKS
__device__ unsigned long long g_chain_clk[CK_N];
#define CH_CLK(k) do { const long long t_ = clock64(); clk[k] += t_ - clk_t; clk_t = t_; } while (0)
#else
#define CH_CLK(k) do { } while (0)
#endif

// MODE 0: forward  -- epilogue = + bias, ReLU, 1-bit masks out, bf16 activation to smem (+ HBM), density head
// MODE 1: backward -- epilogue = x ReLU mask (bits in), bias-gradient column sums, bf16 gradient to smem + HBM
// NH: outputs of the forward head (1 or 4)
template <int MODE, int NH>
__global__ void __launch_bounds__(CH_THREADS, 1)
mlp_chain_kernel(const __grid_constant__ ChainMaps maps, const ChainParams p) {
  extern __shared__ uint8_t smem_dyn[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  uint8_t* act = smem;                                     // [4 k-blocks][128 rows][128 B]
  uint8_t* wring = act + CH_ACT;                           // [CH_RING] weight k-blocks
  uint8_t* sring = wring + CH_RING * CH_WBLK;              // [CH_SRING] streamed-operand blocks
  float* aux = reinterpret_cast<float*>(sring + CH_SRING * CH_SBLK);   // [CH_MAX_LAYERS][CH_W] biases / column sums
  uint64_t* wfull = reinterpret_cast<uint64_t*>(aux + CH_MAX_LAYERS * CH_W);   // [CH_RING]
  uint64_t* wempty = wfull + CH_RING;                      // [CH_RING]: both warpgroups have consumed the slot
  uint64_t* sfull = wempty + CH_RING;                      // [CH_SRING]
  uint64_t* sempty = sfull + CH_SRING;                     // [CH_SRING]: the block's warpgroup has consumed it
  uint64_t* turn = sempty + CH_SRING;                      // [2]: warpgroup c may issue its next segment

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    bool any_stream = false;
    for (int j = 0; j < p.num_layers; ++j) {
      prefetch_tmap(&maps.w[j]);
      if (p.layer[j].store) prefetch_tmap(&maps.out[j]);
      any_stream |= p.layer[j].n_stream > 0;
    }
    if (any_stream) prefetch_tmap(&maps.stream);
    for (int i = 0; i < CH_RING; ++i) { mbar_init(&wfull[i], 1); mbar_init(&wempty[i], 8); }
    for (int i = 0; i < CH_SRING; ++i) { mbar_init(&sfull[i], 1); mbar_init(&sempty[i], 4); }
    for (int i = 0; i < 2; ++i) mbar_init(&turn[i], 4);
    fence_barrier_init();
  }
  if (MODE == 1)
    for (int i = threadIdx.x; i < CH_MAX_LAYERS * CH_W; i += CH_THREADS) aux[i] = 0.f;
  __syncthreads();
  // programmatic dependent launch (see tc_common.cuh): persistent grid, no global access above this line
  pdl_launch_dependents();
  pdl_wait();
  if (MODE == 0) {
    // the biases do not change within a launch: one copy per CTA, read from shared memory in every epilogue
    for (int i = threadIdx.x; i < p.num_layers * CH_W; i += CH_THREADS) aux[i] = __ldg(p.layer[i / CH_W].bias + i % CH_W);
    __syncthreads();
  }

  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      uint32_t wslot = 0, wphase = 0, sslot = 0, sphase = 0;
      for (int64_t unit = blockIdx.x; unit < p.num_units; unit += gridDim.x) {
        const int row0 = (int)(unit * CH_ROWS);
        for (int j = 0; j < p.num_layers; ++j) {
          const ChainLayer& L = p.layer[j];
          const int nk = L.n_res + L.n_stream;
          for (int s0 = 0; s0 < nk; s0 += CH_SEG) {
            const int s1 = min(s0 + CH_SEG, nk);
            // c = 0: the segment's weights, each with warpgroup 0's streamed block; c = 1: warpgroup 1's blocks
            for (int c = 0; c < 2; ++c)
              for (int s = s0; s < s1; ++s) {
                const bool streamed = s >= L.n_res;
                const int si = s - L.n_res;
                if (c == 0) {
                  mbar_wait(&wempty[wslot], wphase ^ 1, 1);
                  mbar_expect_tx(&wfull[wslot], CH_WBLK);
                  tma_load_2d(wring + wslot * CH_WBLK, &maps.w[j], &wfull[wslot],
                              (streamed ? L.stream_kb0 + si : L.res_kb0 + s) * 64, 0);
                  if (++wslot == CH_RING) { wslot = 0; wphase ^= 1; }
                }
                if (streamed) {
                  mbar_wait(&sempty[sslot], sphase ^ 1, 2);
                  mbar_expect_tx(&sfull[sslot], CH_SBLK);
                  tma_load_2d(sring + sslot * CH_SBLK, &maps.stream, &sfull[sslot], L.stream_col0 + si * 64, row0 + 64 * c);
                  if (++sslot == CH_SRING) { sslot = 0; sphase ^= 1; }
                }
              }
          }
          // The streamed blocks come from HBM and the ring holds three of them: have the next unit's first-layer
          // blocks on their way into L2 while this unit computes.
          if (j == 0 && L.n_stream > 0 && unit + gridDim.x < p.num_units)
            for (int si = 0; si < L.n_stream; ++si)
              for (int c = 0; c < 2; ++c)
                tma_prefetch_2d(&maps.stream, L.stream_col0 + si * 64, (int)((unit + gridDim.x) * CH_ROWS) + 64 * c);
        }
      }
    }
  } else {
    // ===================== consumers =====================
    setmaxnreg_inc<232>();
    const int c = wg - 1;
    const int w = warp & 3;
    const int r_in = 64 * c + 16 * w + (lane >> 2);      // rows r_in and r_in + 8 of the unit
    const int q = lane & 3;
    const int cq = 2 * q;
    const uint32_t wring_s = smem_u32(wring), sring_s = smem_u32(sring), act_s = smem_u32(act);
    const uint32_t aux_s = smem_u32(aux);
    const bool lead = (threadIdx.x & 127) == 0;          // issues this warpgroup's bulk stores
    uint32_t wslot = 0, wphase = 0;
    uint32_t spos = 0;                                   // streamed blocks loaded before this segment (both warpgroups')
    uint32_t seg = 0;                                    // segments before this one
#ifdef MNRF_CHAIN_CLOCKS
    long long clk[CK_N] = {};
    long long clk_t = clock64();
#endif
    float acc[CH_W / 2];
    for (int64_t unit = blockIdx.x; unit < p.num_units; unit += gridDim.x) {
      int64_t rows[2];
      bool row_ok[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        rows[h] = unit * CH_ROWS + r_in + 8 * h;
        row_ok[h] = rows[h] < p.m;
      }
      for (int j = 0; j < p.num_layers; ++j) {
        const ChainLayer& L = p.layer[j];
        const bool last = (j == p.num_layers - 1);
        const bool do_head = (MODE == 0) && last && p.head_w != nullptr;
        // Mask words of the two rows: the four lanes of a quad hold a row's eight words between them, lane q the
        // words 2q and 2q + 1.  BWD loads them here, so the loads complete under the main loop; FWD gathers them
        // in the epilogue and stores a row's 32 bytes as one sector after it.
        uint32_t mw[2][2] = {{0u, 0u}, {0u, 0u}};
        if (MODE == 1 && L.maskbits) {
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (row_ok[h]) mw[h][e] = __ldg(L.maskbits + rows[h] * L.ldmaskbits + 2 * q + e);
        }
        // ---- main loop: the resident operand (the previous layer's output), then the streamed k-blocks -- the
        // order of the weight columns of a skip layer, so the fp32 sums round like the per-layer GEMM's
        const int nk = L.n_res + L.n_stream;
        fence_acc(acc);
        for (int s0 = 0; s0 < nk; s0 += CH_SEG, ++seg) {
          const int s1 = min(s0 + CH_SEG, nk);
          const int ns = s1 - max(s0, L.n_res);          // streamed k-blocks of this segment (<= 0: none)
          uint32_t sp = spos + (c && ns > 0 ? ns : 0);
          if (ns > 0) spos += 2 * ns;
          // my turn: warpgroup 0 follows warpgroup 1's previous segment, warpgroup 1 follows warpgroup 0's this one
          if (c == 1) mbar_wait(&turn[1], seg & 1, 7);
          else if (seg > 0) mbar_wait(&turn[0], (seg - 1) & 1, 7);
          CH_CLK(CK_TURN);
          int prev_w = -1, prev_s = -1;
          for (int s = s0; s < s1; ++s) {
            const bool streamed = s >= L.n_res;
            mbar_wait(&wfull[wslot], wphase, 3);
            uint32_t a0 = act_s + s * CH_KBLK + c * (64 * 128);
            int cur_s = -1;
            if (streamed) {
              cur_s = (int)(sp % CH_SRING);
              mbar_wait(&sfull[cur_s], (sp / CH_SRING) & 1, 4);
              a0 = sring_s + cur_s * CH_SBLK;
              ++sp;
            }
            CH_CLK(CK_FULL);
            const uint32_t b0 = wring_s + wslot * CH_WBLK;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 64 / WGMMA_K; ++k)
              Wgmma<CH_W, 0, 0>::mma(acc, make_smem_desc(a0 + k * (WGMMA_K * 2), 0, 1024),
                                     make_smem_desc(b0 + k * (WGMMA_K * 2), 0, 1024), (s > 0 || k > 0) ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<1>();
            if (lane == 0) {
              if (prev_w >= 0) mbar_arrive(&wempty[prev_w]);
              if (prev_s >= 0) mbar_arrive(&sempty[prev_s]);
            }
            prev_w = (int)wslot;
            prev_s = cur_s;
            if (++wslot == CH_RING) { wslot = 0; wphase ^= 1; }
          }
          // every wgmma of the segment is issued: the other warpgroup may issue its next one
          __syncwarp();
          if (lane == 0) mbar_arrive(&turn[c ^ 1]);
          wgmma_wait<0>();
          if (lane == 0) {
            mbar_arrive(&wempty[prev_w]);
            if (prev_s >= 0) mbar_arrive(&sempty[prev_s]);
          }
          CH_CLK(CK_MMA);
        }
        fence_acc(acc);

        // ---- epilogue: the accumulator becomes the next layer's A operand (this warpgroup's 64 rows of `act`)
        // the previous bulk store of these rows must have finished reading them
        if (lead) tma_store_wait_read<0>();
        named_bar_sync(1 + c, 128);
        CH_CLK(CK_EPI_SYNC);
        uint32_t bits[2] = {0u, 0u};
        float hdot[NH][2];
#pragma unroll
        for (int o = 0; o < NH; ++o) hdot[o][0] = hdot[o][1] = 0.f;
#pragma unroll
        for (int i = 0; i < CH_W / 8; ++i) {
          const int col = 8 * i + cq;
          float v[2][2];
#pragma unroll
          for (int h = 0; h < 2; ++h) { v[h][0] = acc[4 * i + 2 * h]; v[h][1] = acc[4 * i + 2 * h + 1]; }
          uint32_t o[2];
          if (MODE == 0) {
            const float2 b = ld_shared_const_f2(aux_s + (j * CH_W + col) * 4);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              v[h][0] += b.x;
              v[h][1] += b.y;
              // ReLU is folded into the bf16 conversion (a NaN stays NaN, with mask bit 0); the mask is the sign of
              // the fp32 pre-activation: stored > 0 implies the bit, and a set bit over a stored 0 only where the
              // pre-activation is in (0, 2^-134], which rounds to a bf16 zero
              bits[h] |= ((v[h][0] > 0.f ? 1u : 0u) | (v[h][1] > 0.f ? 2u : 0u)) << (col & 31);
              o[h] = pack_bf16_relu(v[h][0], v[h][1]);
            }
            if (do_head) {
              // Dense(NH) on the bf16-rounded activation, fp32 accumulate (what the head kernel computes)
#pragma unroll
              for (int oo = 0; oo < NH; ++oo) {
                const float2 hw = __ldg(reinterpret_cast<const float2*>(p.head_w + oo * CH_W + col));
#pragma unroll
                for (int h = 0; h < 2; ++h) hdot[oo][h] += bf16_lo(o[h]) * hw.x + bf16_hi(o[h]) * hw.y;
              }
            }
          } else {
            if (L.maskbits && (i & 3) == 0) {
              // the 32-column word of this group of four steps, from the quad's lane that loaded it
#pragma unroll
              for (int h = 0; h < 2; ++h)
                bits[h] = __shfl_sync(0xffffffffu, mw[h][(i >> 2) & 1], (lane & ~3) | (i >> 3));
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              if (L.maskbits) {
                if (!((bits[h] >> (col & 31)) & 1u)) v[h][0] = 0.f;
                if (!((bits[h] >> ((col + 1) & 31)) & 1u)) v[h][1] = 0.f;
              }
              o[h] = pack_bf16(v[h][0], v[h][1]);
            }
            if (L.colsum) {
              // column sums over the warp's 16 rows (rows past M hold zeros: zero-filled operand, zero mask)
              float s0 = v[0][0] + v[1][0], s1 = v[0][1] + v[1][1];
#pragma unroll
              for (int sh = 4; sh < 32; sh <<= 1) {
                s0 += __shfl_xor_sync(0xffffffffu, s0, sh);
                s1 += __shfl_xor_sync(0xffffffffu, s1, sh);
              }
              if (lane < 4) { atomicAdd(aux + j * CH_W + col, s0); atomicAdd(aux + j * CH_W + col + 1, s1); }
            }
          }
          // K-major SWIZZLE_128B k-block (the layout TMA produces and wgmma / the bulk store consume)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = r_in + 8 * h;
            st_shared_u32(act_s + (col >> 6) * CH_KBLK + r * 128 + ((((col & 63) >> 3) ^ (r & 7)) << 4) + (cq << 1), o[h]);
          }
          if (MODE == 0 && (i & 3) == 3) {
            // one 32-column mask word per row: the four lanes of a quad hold its 32 bits between them
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              bits[h] |= __shfl_xor_sync(0xffffffffu, bits[h], 1);
              bits[h] |= __shfl_xor_sync(0xffffffffu, bits[h], 2);
              if (q == (i >> 3)) mw[h][(i >> 2) & 1] = bits[h];
              bits[h] = 0u;
            }
          }
        }
        CH_CLK(CK_EPI_LOOP);
        fence_proxy_async();                // generic-proxy writes -> visible to wgmma / TMA (async proxy)
        named_bar_sync(1 + c, 128);
        CH_CLK(CK_EPI_SYNC);
        if (lead && L.store) {
#pragma unroll
          for (int kb = 0; kb < 4; ++kb)
            tma_store_2d(&maps.out[j], act + kb * CH_KBLK + c * (64 * 128), kb * 64, (int)(unit * CH_ROWS) + 64 * c);
          tma_store_commit();
        }
        if (MODE == 0 && L.maskbits) {
          // a quad writes a row's 32 bytes: one full sector where the rows are 8-byte aligned
          const bool wide = (((uintptr_t)L.maskbits | (uintptr_t)(L.ldmaskbits * 4)) & 7) == 0;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (!row_ok[h]) continue;
            uint32_t* dst = L.maskbits + rows[h] * L.ldmaskbits + 2 * q;
            if (wide) *reinterpret_cast<uint2*>(dst) = make_uint2(mw[h][0], mw[h][1]);
            else { dst[0] = mw[h][0]; dst[1] = mw[h][1]; }
          }
        }
        if (do_head) {
#pragma unroll
          for (int oo = 0; oo < NH; ++oo)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              hdot[oo][h] += __shfl_xor_sync(0xffffffffu, hdot[oo][h], 1);
              hdot[oo][h] += __shfl_xor_sync(0xffffffffu, hdot[oo][h], 2);
              if (q == 0 && row_ok[h])
                p.head_out[rows[h] * NH + oo] = hdot[oo][h] + (p.head_b ? __ldg(p.head_b + oo) : 0.f);
            }
        }
        CH_CLK(CK_EPI_TAIL);
      }
    }
    if (lead) tma_store_wait_all();
#ifdef MNRF_CHAIN_CLOCKS
    if (blockIdx.x == 0 && threadIdx.x == 256)
      for (int k = 0; k < CK_N; ++k) atomicAdd(&g_chain_clk[k], (unsigned long long)clk[k]);
#endif
    if (MODE == 1) {
      named_bar_sync(3, 256);             // both consumer warpgroups are done with the shared sums
      for (int jj = 0; jj < p.num_layers; ++jj) {
        if (!p.layer[jj].colsum) continue;
        for (int i = threadIdx.x - 128; i < CH_W; i += 256) atomicAdd(p.layer[jj].colsum + i, aux[jj * CH_W + i]);
      }
    }
  }
}

}  // namespace mnrf

extern "C" int mnrf_mlp_chain_max_layers(void) { return mnrf::CH_MAX_LAYERS; }

#ifdef MNRF_CHAIN_CLOCKS
// measurement build only: read (and clear) the clock64() classes summed since the last call
extern "C" int mnrf_chain_clocks(unsigned long long* out) {
  unsigned long long zero[mnrf::CK_N] = {};
  if (cudaDeviceSynchronize() != cudaSuccess) return 1;
  if (cudaMemcpyFromSymbol(out, mnrf::g_chain_clk, sizeof(zero)) != cudaSuccess) return 1;
  return cudaMemcpyToSymbol(mnrf::g_chain_clk, zero, sizeof(zero)) != cudaSuccess;
}
#endif

extern "C" int mnrf_mlp_chain(const mnrf_chain_desc* d, mnrf_stream stream_) {
  using namespace mnrf;
  cudaStream_t stream = (cudaStream_t)stream_;
  MNRF_CHECK(d, "mnrf_mlp_chain: null descriptor");
  // the TMA row coordinates of a unit are int32
  MNRF_CHECK(d->m >= 0 && (d->m + CH_ROWS - 1) / CH_ROWS * CH_ROWS <= INT32_MAX,
             "mnrf_mlp_chain: m must be in [0, %d], got %lld", INT32_MAX / CH_ROWS * CH_ROWS, (long long)d->m);
  if (d->m == 0) return 0;
  MNRF_CHECK(d->mode == MNRF_CHAIN_FWD || d->mode == MNRF_CHAIN_BWD, "mnrf_mlp_chain: bad mode %d", d->mode);
  MNRF_CHECK(d->num_layers >= 1 && d->num_layers <= CH_MAX_LAYERS, "mnrf_mlp_chain: 1..%d layers, got %d",
             CH_MAX_LAYERS, d->num_layers);
  MNRF_CHECK(d->width == CH_W, "mnrf_mlp_chain: layer width must be %d, got %d", CH_W, d->width);
  const int sms = mnrf_num_sms();
  ChainMaps maps;
  memset(&maps, 0, sizeof(maps));
  ChainParams p{};
  p.num_layers = d->num_layers;
  p.m = d->m;
  p.num_units = (d->m + CH_ROWS - 1) / CH_ROWS;
  bool any_stream = false;
  for (int j = 0; j < d->num_layers; ++j) {
    const mnrf_chain_layer& s = d->layer[j];
    ChainLayer& L = p.layer[j];
    MNRF_CHECK(s.n_res == 0 || s.n_res == CH_W / 64, "mnrf_mlp_chain: layer %d: n_res must be 0 or %d", j, CH_W / 64);
    MNRF_CHECK(s.n_stream >= 0 && (s.n_stream > 0 || s.n_res > 0), "mnrf_mlp_chain: layer %d has no operand", j);
    MNRF_CHECK(s.stream_col0 >= 0 && s.stream_kb0 >= 0 && s.res_kb0 >= 0,
               "mnrf_mlp_chain: layer %d: negative column or k-block offset", j);
    MNRF_CHECK(j > 0 || s.n_res == 0, "mnrf_mlp_chain: the first layer has no resident operand");
    MNRF_CHECK(s.w && ((uintptr_t)s.w % 16) == 0 && s.ldw % 8 == 0, "mnrf_mlp_chain: layer %d: weights must be 16-byte aligned", j);
    const int kblocks = std::max(s.n_stream > 0 ? s.stream_kb0 + s.n_stream : 0, s.n_res > 0 ? s.res_kb0 + s.n_res : 0);
    MNRF_CHECK(s.ldw >= (int64_t)kblocks * 64, "mnrf_mlp_chain: layer %d: weight pitch %lld < K %d", j, (long long)s.ldw, kblocks * 64);
    L.n_stream = s.n_stream; L.stream_col0 = s.stream_col0; L.stream_kb0 = s.stream_kb0;
    L.n_res = s.n_res; L.res_kb0 = s.res_kb0;
    L.store = s.out ? 1 : 0;
    L.bias = s.bias; L.maskbits = s.maskbits; L.ldmaskbits = s.ldmaskbits; L.colsum = s.colsum;
    if (s.bias) MNRF_CHECK(((uintptr_t)s.bias % 8) == 0, "mnrf_mlp_chain: layer %d: bias must be 8-byte aligned", j);
    if (s.maskbits)
      MNRF_CHECK(s.ldmaskbits >= CH_W / 32, "mnrf_mlp_chain: layer %d: maskbits rows must hold >= %d words", j, CH_W / 32);
    if (d->mode == MNRF_CHAIN_BWD) MNRF_CHECK(!s.bias, "mnrf_mlp_chain: bias is a forward input");
    else MNRF_CHECK(s.bias && !s.colsum, "mnrf_mlp_chain: layer %d: the forward chain takes a bias and no colsum", j);
    // K-major weights [256 rows, K]: box = [64 k][256 rows]
    if (make_tmap(&maps.w[j], s.w, CH_W, (int64_t)kblocks * 64, s.ldw, 64, CH_W)) return 1;
    if (s.out) {
      MNRF_CHECK(((uintptr_t)s.out % 16) == 0 && s.ldo % 8 == 0 && s.ldo >= CH_W, "mnrf_mlp_chain: layer %d: output alignment", j);
      // each consumer warpgroup stores its own 64 rows
      if (make_tmap(&maps.out[j], s.out, d->m, CH_W, s.ldo, 64, 64)) return 1;
    }
    any_stream |= s.n_stream > 0;
    if (s.n_stream > 0)
      MNRF_CHECK(s.stream_col0 % 64 == 0 && s.stream_col0 + s.n_stream * 64 <= d->stream_cols,
                 "mnrf_mlp_chain: layer %d: streamed columns [%d, %d) outside the stream tensor (%d columns)", j,
                 s.stream_col0, s.stream_col0 + s.n_stream * 64, d->stream_cols);
  }
  if (any_stream) {
    MNRF_CHECK(d->stream && ((uintptr_t)d->stream % 16) == 0 && d->ldstream % 8 == 0 && d->stream_cols % 64 == 0,
               "mnrf_mlp_chain: streamed operand must be 16-byte aligned with a multiple of 64 columns");
    MNRF_CHECK(d->ldstream >= d->stream_cols, "mnrf_mlp_chain: stream pitch %lld < %d columns",
               (long long)d->ldstream, d->stream_cols);
    // each consumer warpgroup waits on its own 64 rows
    if (make_tmap(&maps.stream, d->stream, d->m, d->stream_cols, d->ldstream, 64, CH_ROWS / 2)) return 1;
  }
  p.head_w = d->head_w; p.head_b = d->head_b; p.head_out = d->head_out;
  const int head_n = d->head_n ? d->head_n : 1;
  if (d->head_w) MNRF_CHECK(d->mode == MNRF_CHAIN_FWD && d->head_out && ((uintptr_t)d->head_w % 16) == 0,
                            "mnrf_mlp_chain: the head is a forward output (16-byte aligned weights)");
  MNRF_CHECK(head_n == 1 || (head_n == 4 && d->head_w), "mnrf_mlp_chain: head_n must be 1 or 4, got %d", head_n);
  const int grid = (int)std::min<int64_t>(p.num_units, sms);
  const int rc = d->mode == MNRF_CHAIN_BWD ? launch_tc<mlp_chain_kernel<1, 1>>(grid, CH_THREADS, CH_SMEM, stream, maps, p)
                 : head_n == 4             ? launch_tc<mlp_chain_kernel<0, 4>>(grid, CH_THREADS, CH_SMEM, stream, maps, p)
                                           : launch_tc<mlp_chain_kernel<0, 1>>(grid, CH_THREADS, CH_SMEM, stream, maps, p);
  if (rc) return rc;
  MNRF_LAUNCH_CHECK();
  return 0;
}
