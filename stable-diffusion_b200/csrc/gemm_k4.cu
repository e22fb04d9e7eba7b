// gemm_tc_kernel instantiations of epilogue KIND 4 (see gemm_kernel.cuh)
#include "gemm_kernel.cuh"

namespace sdb {
int launch_gemm_kind4(int bn, int cg, const TmapPack& tm, const GemmArgs& p, cudaStream_t st) {
  return launch_gemm_kind<4>(bn, cg, tm, p, st);
}
}  // namespace sdb
