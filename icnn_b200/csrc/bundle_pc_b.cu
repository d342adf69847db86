// K2 predictor-corrector path: instantiation for 8 warps per sample (see bundle_pc.cu).
#include "bundle_pc_kernel.cuh"
namespace icnn {
cudaError_t launch_pc_8x2(const PcArgs& a, const PcConfig& c, int B, cudaStream_t st) { return launch_pc<8, 2, true>(a, c, B, st); }
}  // namespace icnn
