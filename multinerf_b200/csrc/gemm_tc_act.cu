// The smooth-activation (softplus / SiLU) instances of the Dense-layer GEMM of gemm_tc.cu, in a translation unit of
// their own so that the ReLU instances compile to the same code as without them.  gemm_tc.cu's gemm_tc_launch checks
// the arguments and builds the parameters and tensor maps; this unit only picks the instance.
#define MNRF_GEMM_TC_SMOOTH_UNIT
#include "gemm_tc.cu"

namespace mnrf {

int gemm_tc_smooth_launch(int mode, int block_n, int grid, const CUtensorMap& ta, const CUtensorMap& tb,
                          const CUtensorMap& tc, const GemmParams& p, cudaStream_t stream) {
  // the staged bulk store (TS) only: gemm_tc_launch checked that the output allows it
  const bool fwd = mode == MNRF_GEMM_FWD;
  switch (block_n) {
    case 256:
      return fwd ? launch_gemm_tc<MNRF_GEMM_FWD, 256, true, false, true>(grid, ta, tb, tc, tb, p, stream)
                 : launch_gemm_tc<MNRF_GEMM_DGRAD, 256, true, false, true>(grid, ta, tb, tc, tb, p, stream);
    case 128:
      return fwd ? launch_gemm_tc<MNRF_GEMM_FWD, 128, true, false, true>(grid, ta, tb, tc, tb, p, stream)
                 : launch_gemm_tc<MNRF_GEMM_DGRAD, 128, true, false, true>(grid, ta, tb, tc, tb, p, stream);
    case 64:
      return fwd ? launch_gemm_tc<MNRF_GEMM_FWD, 64, true, false, true>(grid, ta, tb, tc, tb, p, stream)
                 : launch_gemm_tc<MNRF_GEMM_DGRAD, 64, true, false, true>(grid, ta, tb, tc, tb, p, stream);
  }
  set_error("mnrf_gemm(tc): no smooth-activation instance at BN=%d", block_n);
  return 1;
}

}  // namespace mnrf
