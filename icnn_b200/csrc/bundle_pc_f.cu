// K2 predictor-corrector path: the three-n-vector instantiation (V3, see bundle_pc_kernel.cuh): two 8-warp samples
// per SM at n_y = 4096 (C5).
#include "bundle_pc_kernel.cuh"
namespace icnn {
cudaError_t launch_pc_v3_8x4(const PcArgs& a, const PcConfig& c, int B, cudaStream_t st) { return launch_pc<8, 4, true, true>(a, c, B, st); }
}  // namespace icnn
