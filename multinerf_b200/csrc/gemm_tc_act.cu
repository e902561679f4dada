// The smooth-activation (softplus / SiLU) instances of the Dense-layer GEMM of gemm_tc.cu, in a translation unit of
// their own so that the ReLU instances compile to the same code as without them.  gemm_tc.cu's gemm_tc_launch checks
// the arguments and builds the parameters and tensor maps; this unit only picks the instance.
#define MNRF_GEMM_TC_SMOOTH_UNIT
#include "gemm_tc.cu"

namespace mnrf {

int gemm_tc_smooth_launch(int mode, int block_n, int grid, const CUtensorMap& ta, const CUtensorMap& tb,
                          const CUtensorMap& tc, const GemmParams& p, cudaStream_t stream) {
  // the staged bulk store (TS) only: gemm_tc_launch checked that the output allows it
#define MNRF_LAUNCH_SMOOTH(MODE_, BN_) launch_gemm_tc<MODE_, BN_, true, false, true>(grid, ta, tb, tc, tb, p, stream)
  if (mode == MNRF_GEMM_FWD) {
    return block_n == 256   ? MNRF_LAUNCH_SMOOTH(MNRF_GEMM_FWD, 256)
           : block_n == 128 ? MNRF_LAUNCH_SMOOTH(MNRF_GEMM_FWD, 128)
                            : MNRF_LAUNCH_SMOOTH(MNRF_GEMM_FWD, 64);
  }
  return block_n == 256   ? MNRF_LAUNCH_SMOOTH(MNRF_GEMM_DGRAD, 256)
         : block_n == 128 ? MNRF_LAUNCH_SMOOTH(MNRF_GEMM_DGRAD, 128)
                          : MNRF_LAUNCH_SMOOTH(MNRF_GEMM_DGRAD, 64);
#undef MNRF_LAUNCH_SMOOTH
}

}  // namespace mnrf
