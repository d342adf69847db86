// The parts of the GD training backward (gd_backward.cu) that the bundle-entropy training gradient
// (train_grad.cu) runs as well: one accumulate-mode iteration of gd_backward (primal forward, tangent
// forward, primal backward with the gradient accumulations) is that gradient for a block of feed rows.
#pragma once
#include "common.cuh"

namespace icnn {

struct GdbLayout {
  size_t Z[ICNN_MAX_LAYERS], Zt[ICNN_MAX_LAYERS], Dacc[ICNN_MAX_LAYERS], dl[2], y, v, g, a, f, tc, total;
  size_t wpart;   // wgrad_part_bytes() (wgrad.cuh): the weight-gradient GEMMs' partial tiles, independent of B
  bool use_tc;
  // stored-pattern mode (single pass): per-iteration stores and the phase-2 scratch
  bool stored;
  size_t kap, Zs[ICNN_MAX_LAYERS], Ds[ICNN_MAX_LAYERS], As[ICNN_MAX_LAYERS], Zts[ICNN_MAX_LAYERS], Ty[ICNN_MAX_LAYERS];
  size_t P_hi, P_lo, Pk, Sout;
};

// float64 accumulators of the weight gradients (train_grad.cu): when given, the weight-gradient GEMMs sum in
// float64 into these instead of into the float32 dWy / dWz of icnn_gd_grads
struct GdbW64 { double* dWy[ICNN_MAX_LAYERS + 1]; double* dWz[ICNN_MAX_LAYERS + 1]; };

// Accumulate mode of gdb_iteration.  c != nullptr (train_grad.cu): once the tangent forward is done,
// Zt_l <- c o Z_l + Zt_l (per-row scale c), so that the backward accumulates with the combined operand.
// w64 != nullptr: dWz accumulates in float64 (GdbW64).
struct GdbAcc { const icnn_gd_grads* gr; float kappa; const float* c; const GdbW64* w64; };

bool gdb_use_tc(const icnn_picnn* h, int B);
GdbLayout gdb_layout(const icnn_picnn* h, int B, int nIter);
int gdb_iteration(const icnn_picnn* h, const icnn_gates* gt, float* ws, const GdbLayout& lo, const GdbAcc* acc,
                  int store_it, float store_kappa, cudaStream_t st);
// y-gate terms from the accumulated Delta_l (ws + lo.Dacc[l]) and the direction av [B, n]:
//   dWy_l += (av o cy_l)^T Delta_l,  dcy_l += av o (Delta_l Wy_l^T);  output layer Delta_L = ksum
// (w64 != nullptr: dWy accumulates in float64, GdbW64)
int gdb_ygate_stage(const icnn_picnn* h, const icnn_gates* gt, float* ws, const GdbLayout& lo, const float* av,
                    const icnn_gd_grads* gr, float ksum, const GdbW64* w64, cudaStream_t st);

// dst[r, j] += c[r] * src[r, j] for r < rows, j < w
void launch_row_axpy(float* dst, const float* src, const float* c, long long rows, int w, cudaStream_t st);

// Adjoint weights of the nIter gradient evaluations of the unrolled momentum-GD loop (gd_backward.cu's header), on
// the host in double:  c_N = 1 + m,  c_i = m c_{i+1} + 1,  kappa[i] = float(-lr c_{i+1})  for i < nIter.
// Returns the double sum of the float kappa[i], i = 0..nIter-1 in that order (0 for nIter = 0).
inline double gd_kappa(int nIter, float lr, float momentum, float* kappa) {
  double c = 1.0 + (double)momentum;   // c_{i+1} of i = nIter - 1
  for (int i = nIter - 1; i >= 0; --i) {
    kappa[i] = (float)(-(double)lr * c);
    c = (double)momentum * c + 1.0;
  }
  double ksum = 0.0;
  for (int i = 0; i < nIter; ++i) ksum += (double)kappa[i];
  return ksum;
}

}  // namespace icnn
