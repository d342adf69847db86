// The convolutional PICNN handle and the f / df/dy pass of conv_picnn.cu as seen by the training gradient
// (conv_train_grad.cu), which runs that pass per feed row and reads the per-layer values it leaves in the workspace.
#pragma once
#include "tc_gemm.cuh"

namespace icnn {

struct ConvGeom {
  int C, k, s, Cp;            // out channels, kernel, stride, in channels of the z part (C_{l-1}; 0 at l = 0)
  int Hi, Wi, Ho, Wo;         // input / output grid
  int pt, pl;                 // 'SAME' padding before (top, left); the rest goes after
  int K;                      // k^2 (Cp + 1)
};

}  // namespace icnn

struct icnn_conv_picnn {
  int H, W, Lc, Ld;
  int fcs[ICNN_MAX_LAYERS];
  icnn::ConvGeom g[ICNN_MAX_LAYERS];
  int flat;                   // H_Lc * W_Lc * C_{Lc-1}: width of the first dense layer's input
  // conv l: Wf [C, ld4(K)] (forward B operand), Wb [K, ld4(C)] (backward B operand); dense hidden layer j (index
  // Lc + j): Wf [w, ld4(in)], Wb [in, ld4(w)]; all TF32 hi/lo
  float* Wf_hi[2 * ICNN_MAX_LAYERS]; float* Wf_lo[2 * ICNN_MAX_LAYERS];
  float* Wb_hi[2 * ICNN_MAX_LAYERS]; float* Wb_lo[2 * ICNN_MAX_LAYERS];
  float* wout;                // [in] weights of the width-1 output layer
  float* red[ICNN_MAX_LAYERS];  // [k^2 + 1]: Wred_l then bred_l
  int in_w(int j) const { return j == 0 ? flat : fcs[j - 1]; }   // input width of dense layer j
};

namespace icnn {

// what conv_fg leaves in its workspace (all [rows, ...] of the B rows it ran)
struct ConvWs {
  float* Ah[ICNN_MAX_LAYERS]; float* Al[ICNN_MAX_LAYERS]; float* Z[ICNN_MAX_LAYERS];
  float* dh[ICNN_MAX_LAYERS]; float* dl[ICNN_MAX_LAYERS];            // delta_l, the GEMM operand [M_l, ld4(C_l)]
  float* r[ICNN_MAX_LAYERS]; float* rho[ICNN_MAX_LAYERS];            // l >= 1: [B, H_l W_l]
  float* cols;                                                       // [M_l, K_l], the largest layer
  float* fAh[ICNN_MAX_LAYERS]; float* fAl[ICNN_MAX_LAYERS]; float* fZ[ICNN_MAX_LAYERS];   // dense hidden layers
  float* fdh[ICNN_MAX_LAYERS]; float* fdl[ICNN_MAX_LAYERS];
  float* th; float* tl;                                              // delta_{Lc-1} at pitch C before repitching
};

// floats of workspace for B rows; with base != nullptr also the buffer addresses
size_t conv_ws_floats(const icnn_conv_picnn* h, int B, float* base, ConvWs* w);

// f and df/dy of B rows (icnn_conv_picnn_fg).  eout != nullptr: eout[l] [B H_l W_l, C_{l-1} + 1] receives the
// un-gated adjoints [e_z | e_r] = conv_l^T(delta_l; [Wz_l | Wy_l]) of every conv layer
int conv_fg(const icnn_conv_picnn* h, const icnn_gates* gt, const float* y32, float* f, float* g,
            long long g_row_stride, const int* perm, const int* count, int KS, void* workspace, const int* skip,
            cudaStream_t st, float* const* eout = nullptr);

// the gated im2col of conv layer g (TF32 hi/lo, row pitch ld4(K)) and the first dense layer's gated operand
void conv_im2col_gate_launch(const float* Z, const float* cz, const float* r, const float* cy, const ConvGeom& g,
                             int B, float* hi, float* lo, cudaStream_t st);
void conv_gate_split_launch(const float* Z, const float* cz, int B, int w, float* hi, float* lo, int ld,
                            cudaStream_t st);

}  // namespace icnn
