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
// dL != nullptr (td_grad.cu): the output adjoint of row r is dL[r] instead of 1.  There is no tangent forward: the
// accumulations take the primal Z_l as their operand, and the output-layer terms are scaled by dL per row.  The
// caller scales delta_{L-1} by dL between gdb_forward and gdb_backward (dL depends on f).
struct GdbAcc { const icnn_gd_grads* gr; float kappa; const float* c; const GdbW64* w64; const float* dL = nullptr; };

// The argument checks of the FC training entries (icnn_gd_backward, icnn_train_grad, icnn_td_grad): no affine (RL)
// input wrapper, a non-empty batch, and every per-layer gradient buffer the layers use (dd only with need_dd).
// ICNN_OK, or the error code with the error set; entry names the entry point in the message.
int gdb_check_args(const icnn_picnn* h, const icnn_gates* gates, const icnn_train_grads& gr, bool need_dd,
                   const char* entry);

// The float64 weight-gradient accumulators (train_grad.cu, td_grad.cu): dWy_0..L, then dWz_1..L, in one buffer of
// gdb_w64_doubles(h) doubles.  gdb_w64_bind points a GdbW64 into it and zeroes it on st; gdb_w64_round writes the
// sums, rounded once, into the float32 dWy / dWz of gr.
size_t gdb_w64_doubles(const icnn_picnn* h);
int gdb_w64_bind(const icnn_picnn* h, double* base, GdbW64* w, cudaStream_t st);
int gdb_w64_round(const icnn_picnn* h, const GdbW64& w, const icnn_train_grads* gr, cudaStream_t st);

// tensor-core buffers of the GD training backward (picnn_tc.cu): their floats for a B-row batch, with b's pointers
// set from base when b != nullptr; and the (a o cy_l) columns of the tangent operands
size_t picnn_gdb_tc_ws_floats(const icnn_picnn* h, int B, GdbTcBufs* b, float* base);
void picnn_gdb_tc_gate_a(const icnn_picnn* h, const icnn_gates* gt, const float* a, const GdbTcBufs& b, cudaStream_t st);

bool gdb_use_tc(const icnn_picnn* h, int B);
GdbLayout gdb_layout(const icnn_picnn* h, int B, int nIter);
int gdb_iteration(const icnn_picnn* h, const icnn_gates* gt, float* ws, const GdbLayout& lo, const GdbAcc* acc,
                  int store_it, float store_kappa, cudaStream_t st);
// the two halves of gdb_iteration: the forward (and the tangent forward) through the output layer, which leaves
// f at ws + lo.f and delta_{L-1} in the plain buffer ws + lo.dl[0] (tensor-core path: also its TF32 hi/lo split in
// the first delta slot of picnn_gdb_tc_ws_floats); then the backward with the accumulations
int gdb_forward(const icnn_picnn* h, const icnn_gates* gt, float* ws, const GdbLayout& lo, const GdbAcc* acc,
                int store_it, float store_kappa, cudaStream_t st);
int gdb_backward(const icnn_picnn* h, const icnn_gates* gt, float* ws, const GdbLayout& lo, const GdbAcc* acc,
                 int store_it, float store_kappa, cudaStream_t st);
// y-gate terms from the accumulated Delta_l (ws + lo.Dacc[l]) and the direction av [B, n]:
//   dWy_l += (av o cy_l)^T Delta_l,  dcy_l += av o (Delta_l Wy_l^T);  output layer Delta_L = ksum (times dL[row]
// when dL != nullptr)   (w64 != nullptr: dWy accumulates in float64, GdbW64)
int gdb_ygate_stage(const icnn_picnn* h, const icnn_gates* gt, float* ws, const GdbLayout& lo, const float* av,
                    const icnn_gd_grads* gr, float ksum, const GdbW64* w64, const float* dL, cudaStream_t st);

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
