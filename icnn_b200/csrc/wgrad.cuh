// The weight gradient every training path ends in (gd_backward.cu, train_grad.cu through gdb.cuh, conv_train_grad.cu):
//   C[m, n] (+)= kappa * sum_row (A o G)[row, m] D[row, n]
// an FP32 FFMA reduction over a long row dimension into a small output.  64 x 64 output tiles, 16 rows per stage,
// 4 x 4 register micro-tiles; both operands are read along their contiguous dimension.
//
// The rows are split into P parts (wgrad_parts): CTA z of a tile sums the 16-row tiles [nk z / P, nk (z+1) / P) in
// ascending order from zero.  P == 1 stores straight into C; P > 1 writes the partial tiles to WgradArgs::part and
// wgrad_reduce_kernel adds them in rank order, v = 0 + part_0 + ... + part_{P-1}.  No atomics: every call gives the
// same bits.
//
// Acc = double (WgradArgs::C64): every product of two floats is exact in float64 and the sums over the rows and the
// parts are float64, so the result depends on how the rows are split only through the order of float64 additions.
#pragma once
#include "common.cuh"

namespace icnn {

constexpr int WG_T = 64, WG_BK = 16, WG_PAD = 4;

struct WgradArgs {
  int M, N, Kb;                               // C is [M, N]; reduction over Kb rows
  const float* A; const float* G; int lda;    // A (optionally gated by G) [Kb, lda]
  const float* D; const float* Dlo; int ldd;  // D [Kb, ldd], + Dlo in float32 when given (a TF32 hi/lo pair);
                                              // D == nullptr: a column of ones (N == 1)
  float* C; int ldc; float kappa;             // C = fmaf(kappa, v, C)
  double* C64;                                // optional: C64 += (double)kappa * v in float64 (C unused)
  void* part;                                 // wgrad_part_bytes() of scratch for the partial tiles of P > 1
};

// Parts of the row split: start at 1 and double while the grid stays under twice the SMs and each part keeps at
// least 8 row tiles, up to 1024.  So tiles * P < 4 SMs whenever P > 1, which bounds the partials.
static inline int wgrad_parts(int tiles, int Kb, int sms) {
  const int nk = (Kb + WG_BK - 1) / WG_BK;
  int P = 1;
  while (P < 1024 && (long long)tiles * P < 2LL * sms && nk / (P * 2) >= 4) P *= 2;
  return P;
}
// bytes of WgradArgs::part: the float64 partial tiles of any launch (tiles * P < 4 SMs)
static inline size_t wgrad_part_bytes() { return (size_t)4 * device_sms() * WG_T * WG_T * sizeof(double); }

__device__ __forceinline__ float wg_madd(float x, float y, float acc) { return fmaf(x, y, acc); }
__device__ __forceinline__ double wg_madd(float x, float y, double acc) { return fma((double)x, (double)y, acc); }
__device__ __forceinline__ void wg_store(const WgradArgs& a, int m, int nn, float v) {
  float* c = a.C + (long long)m * a.ldc + nn;
  *c = fmaf(a.kappa, v, *c);
}
__device__ __forceinline__ void wg_store(const WgradArgs& a, int m, int nn, double v) {
  a.C64[(long long)m * a.ldc + nn] += (double)a.kappa * v;
}

template <typename Acc>
static __global__ void __launch_bounds__(256) wgrad_kernel(WgradArgs a) {
  __shared__ __align__(16) float As[2][WG_BK][WG_T + WG_PAD];
  __shared__ __align__(16) float Bs[2][WG_BK][WG_T + WG_PAD];
  const int t = threadIdx.x;
  const int P = gridDim.z;
  const int m0 = blockIdx.y * WG_T, n0 = blockIdx.x * WG_T;
  const int ty = t / 16, tx = t % 16;
  const int l_k = t / 16, l_c = (t % 16) * 4;

  float ra[4], rb[4];
  auto load_tiles = [&](int b0) {
    const int b = b0 + l_k;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int m = m0 + l_c + i, nn = n0 + l_c + i;
      float va = 0.f, vb = 0.f;
      if (b < a.Kb) {
        if (m < a.M) {
          va = a.A[(long long)b * a.lda + m];
          if (a.G) va *= a.G[(long long)b * a.lda + m];
        }
        if (nn < a.N) {
          const long long o = (long long)b * a.ldd + nn;
          vb = a.D ? a.D[o] : 1.f;
          if (a.Dlo) vb += a.Dlo[o];
        }
      }
      ra[i] = va; rb[i] = vb;
    }
  };
  auto store_tiles = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 4; ++i) { As[buf][l_k][l_c + i] = ra[i]; Bs[buf][l_k][l_c + i] = rb[i]; }
  };

  Acc acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = Acc(0);

  const int nk_all = (a.Kb + WG_BK - 1) / WG_BK;
  const int kt0 = (int)(((long long)nk_all * blockIdx.z) / P);
  const int nk = (int)(((long long)nk_all * (blockIdx.z + 1)) / P) - kt0;
  if (nk > 0) { load_tiles(kt0 * WG_BK); store_tiles(0); }
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) load_tiles((kt0 + kt + 1) * WG_BK);
#pragma unroll
    for (int k = 0; k < WG_BK; ++k) {
      const float4 av = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 bv = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float aa[4] = {av.x, av.y, av.z, av.w};
      const float bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = wg_madd(aa[i], bb[j], acc[i][j]);
    }
    if (kt + 1 < nk) store_tiles(buf ^ 1);
    __syncthreads();
  }

  Acc* part = static_cast<Acc*>(a.part) + (long long)blockIdx.z * a.M * a.N;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= a.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int nn = n0 + tx * 4 + j;
      if (nn >= a.N) continue;
      if (P == 1) wg_store(a, m, nn, acc[i][j]);
      else part[(long long)m * a.N + nn] = acc[i][j];
    }
  }
}

// the P partial [M, N] tiles summed in rank order, then stored as the P == 1 path stores
template <typename Acc>
static __global__ void wgrad_reduce_kernel(WgradArgs a, int P) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long MN = (long long)a.M * a.N;
  if (i >= MN) return;
  const Acc* part = static_cast<const Acc*>(a.part);
  Acc v = Acc(0);
  for (int z = 0; z < P; ++z) v += part[z * MN + i];
  wg_store(a, (int)(i / a.N), (int)(i % a.N), v);
}

static inline cudaError_t launch_wgrad(const WgradArgs& a, cudaStream_t st) {
  const int gx = cdiv(a.N, WG_T), gy = cdiv(a.M, WG_T);
  const int P = wgrad_parts(gx * gy, a.Kb, device_sms());
  const dim3 grid(gx, gy, P);
  const unsigned gr = (unsigned)(((long long)a.M * a.N + 255) / 256);
  if (a.C64) {
    wgrad_kernel<double><<<grid, 256, 0, st>>>(a);
    if (P > 1) wgrad_reduce_kernel<double><<<gr, 256, 0, st>>>(a, P);
  } else {
    wgrad_kernel<float><<<grid, 256, 0, st>>>(a);
    if (P > 1) wgrad_reduce_kernel<float><<<gr, 256, 0, st>>>(a, P);
  }
  return cudaPeekAtLastError();
}

}  // namespace icnn
