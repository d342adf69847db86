// K2 predictor-corrector path: instantiations for 16 warps per sample (see bundle_pc.cu).
#include "bundle_pc_kernel.cuh"
namespace icnn {
cudaError_t launch_pc_16x2(const PcArgs& a, const PcConfig& c, int B, cudaStream_t st) { return launch_pc<16, 2, true>(a, c, B, st); }
cudaError_t launch_pc_16x4(const PcArgs& a, const PcConfig& c, int B, cudaStream_t st) { return launch_pc<16, 4, true>(a, c, B, st); }
}  // namespace icnn
