// Tap-GEMM kernels of tile width BN = 256 (see tapgemm_tc_kernel.cuh).
#include "tapgemm_tc_kernel.cuh"

namespace aero {
KernelFn tapgemm_tc_kernels_bn256(bool f16a, bool f16o, int amode, bool res, bool stats) { return pick_kernel_bn<256>(f16a, f16o, amode, res, stats); }
}  // namespace aero
