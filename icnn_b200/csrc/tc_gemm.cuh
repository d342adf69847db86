// The 3xTF32 wgmma GEMM of picnn_tc.cu as seen by the other translation units that launch it (conv_picnn.cu,
// conv_train_grad.cu):
//   C[M,N] = A[M,K] * B[N,K]^T, both operands K-major, pre-split TF32 hi/lo, row pitches multiples of 4 floats,
// with the fused epilogues selected by TcArgs::mode.
#pragma once
#include "common.cuh"

namespace icnn {

struct TcArgs {
  int M, N, K;
  int ch;    // half k-blocks per accumulation chunk (>= 1), set by launch_tc_gemm
  int mode;  // 0 forward, 1 backward, 2 plain store C = acc, 3 x-path gates
  // forward epilogue: Z = act(acc + D); optional next-layer operand A'_{next}[:, 0:N] = Z o Cz_next (hi/lo)
  const float* D; float* Z; float alpha;
  const float* Cz_next; float* nxt_hi; float* nxt_lo; int nxt_ld;
  // backward epilogue: columns < N0 -> delta_prev = act'(Zprev) o Cz o acc (hi/lo, row pitch dprev_ld); else g += ...
  int N0; const float* Zprev; const float* Cz; float* dprev_hi; float* dprev_lo; int dprev_ld;
  const float* Cy; float* g; long long g_row_stride; const int* perm; const int* count; int KS; int n;
  float g_scale;
  float* C;  // mode 2: the self test and the conv PICNN's plain GEMMs (conv_picnn.cu, conv_train_grad.cu)
  // training gradients (GDB instantiation only): the GD training backward (gd_backward.cu) and the bundle-entropy
  // gradient (train_grad.cu) through picnn_tc.cu's GDB layer GEMMs; conv_train_grad.cu launches with tangent = 1:
  //   mode 0 with tangent != 0: Z = act'(D) o acc (D holds the primal activation), no bias
  //   mode 1: optional plain copy of delta_prev, dCz += kappa * Ztprev o acc, Dacc += kappa * delta_prev
  //   mode 0 with tangent == 2 (stored-pattern phase): Z = act'(Zmask) o (acc + D[(row % drow_mod), :])
  //   mode 1: optional plain copy of the pre-gating product acc (acc_plain, [M, N0])
  int tangent; float* dprev_plain; float* dCz; const float* Ztprev; float* Dacc; float kappa;
  const float* Zmask; int drow_mod; float* acc_plain;
  // mode 3 (x-path gate GEMM): out = acc + bias[col]; up to 4 column ranges [rbeg[r], rbeg[r+1]) each with
  // its own ReLU flag and destination (row pitch rld[r]); range 0 may instead be written as a TF32
  // hi/lo pair (the next u-layer operand)
  int nr; int rbeg[5]; int rrelu[4]; float* rdst[4]; int rld[4]; float* r0_hi; float* r0_lo; const float* bias;
  const int* skip_if_zero;
};

// Enqueues one GEMM on st (tile variant / split-K chosen as in picnn_tc.cu, or pinned by icnn_tc_set_tuning).
// lda / ldb: row pitches of A and B in floats (multiples of 4).  ICNN_OK or an ICNN_E_* code with the error set.
int launch_tc_gemm(const float* Ah, const float* Al, long long lda, const float* Bh, const float* Bl, long long ldb,
                   TcArgs a, cudaStream_t st, bool gdb = false);

// momentum GD update y, v <- (multi-label-cls/icnn-back.py:122-128) over N elements (picnn_simt.cu)
void gd_update_launch(float* y, float* v, const float* g, long long N, float lr, float mom, cudaStream_t st);

}  // namespace icnn
