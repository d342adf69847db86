// Shared helpers for libicnn_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>

#include "../../include/icnn_b200.h"

#define ICNN_MAX_LAYERS 8

namespace icnn {

void set_error(const char* fmt, ...);

#define ICNN_CUDA_CHECK(expr)                                                        \
  do {                                                                               \
    cudaError_t _e = (expr);                                                         \
    if (_e != cudaSuccess) {                                                         \
      icnn::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return ICNN_E_CUDA;                                                            \
    }                                                                                \
  } while (0)

#define ICNN_REQUIRE(cond, msg)                                        \
  do {                                                                 \
    if (!(cond)) {                                                     \
      icnn::set_error("%s:%d: invalid argument: %s", __FILE__, __LINE__, msg); \
      return ICNN_E_INVALID;                                           \
    }                                                                  \
  } while (0)

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }
// streaming multiprocessors of the current device (132 on an H100 SXM): the grid-size heuristics aim at it
static inline int device_sms() {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    return 132;
  return sms;
}
#ifdef __CUDACC__
// optional per-outer-iteration statistics (icnn_bundle_bufs::iter_stats), totals over samples
__device__ __forceinline__ void stat_add(double* st, int t, int idx, double v) {
  if (st) atomicAdd(st + (size_t)t * ICNN_NSTAT + idx, v);
}
// y log y + (1 - y) log(1 - y) with 0 log 0 = 0  (negative entropy of one coordinate, ebundle-vs-gd.py:38-41)
__device__ __forceinline__ double neg_entropy(double y) {
  double a = 0.0;
  if (y > 0.0) a += y * log(y);
  if (y < 1.0) a += (1.0 - y) * log(1.0 - y);
  return a;
}
#endif
// leading dimension padded to 4 floats: 16-byte row pitch for TMA; the pad columns lie outside the
// tensor map's extent (TMA zero-fills them), so they are never read and need no initialisation
static inline int ld4(int k) { return (k + 3) & ~3; }

// buffers of the GD training backward on the tensor-core GEMMs (layout owned by gd_backward.cu)
struct GdbTcBufs {
  float* y; float* g;
  float* Z[ICNN_MAX_LAYERS]; float* Zt[ICNN_MAX_LAYERS]; float* Dacc[ICNN_MAX_LAYERS];
  float* Ah[ICNN_MAX_LAYERS]; float* Al[ICNN_MAX_LAYERS];     // primal K-concatenated operands (TF32 hi/lo)
  float* Ath[ICNN_MAX_LAYERS]; float* Atl[ICNN_MAX_LAYERS];   // tangent operands
  float* dh[2]; float* dl[2]; float* dp[2];                   // delta: hi / lo / plain, ping-pong
  // backward-epilogue extras (all optional)
  float* dstore[ICNN_MAX_LAYERS];   // plain delta_l goes here instead of dp[] (stored-pattern mode)
  float* astore[ICNN_MAX_LAYERS];   // plain pre-gating product delta_l Wz_l^T
  float* dcz[ICNN_MAX_LAYERS + 1];  // dcz_l += kappa zt_{l-1} o (delta_l Wz_l^T)
  bool acc_delta;                   // Dacc_{l-1} += kappa delta_{l-1}
  bool want_plain;                  // write plain delta_{l-1} (into dstore or dp)
  float kappa;
};

}  // namespace icnn

// Library-owned weight descriptor.
struct icnn_picnn {
  int n, L;
  int hidden[ICNN_MAX_LAYERS];
  float alpha;
  // Wcat[i], i = 0..L : [(s_{i-1} + n), s_i] row-major = [Wz_i ; Wy_i]  (s_{-1} = 0, s_L = 1)
  float* Wcat[ICNN_MAX_LAYERS + 1];
  // tensor-core path (picnn_tc.cu), hidden layers only: TF32 hi/lo splits of Wcat_i as stored
  // ([K_f, s_i]: K-major B operand of the backward GEMM) and transposed ([s_i, K_f]: forward)
  float* Wb_hi[ICNN_MAX_LAYERS]; float* Wb_lo[ICNN_MAX_LAYERS];
  float* Wf_hi[ICNN_MAX_LAYERS]; float* Wf_lo[ICNN_MAX_LAYERS];
  bool use_tc;
  // x-path (gate precompute) weights: per source s = 0..L the N-concatenated, transposed, hi/lo-split
  // [Wu_s | Wzu_s | Wyu_s | Wzx_s] and the matching bias vector
  int m; bool has_xpath;
  float* Xw_hi[ICNN_MAX_LAYERS + 1]; float* Xw_lo[ICNN_MAX_LAYERS + 1]; float* Xbias[ICNN_MAX_LAYERS + 1];
  int xN[ICNN_MAX_LAYERS + 1]; int xK[ICNN_MAX_LAYERS + 1];
  int width(int i) const { return i < L ? hidden[i] : 1; }
  int prev(int i) const { return i == 0 ? 0 : hidden[i - 1]; }
};
