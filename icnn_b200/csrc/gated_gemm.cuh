// Gated FP32 GEMM with fused PICNN epilogues and cluster split-K (shared by picnn_simt.cu and
// gd_backward.cu).  See picnn_simt.cu for the recurrence it evaluates.
#pragma once
#include "common.cuh"

#include <cooperative_groups.h>

namespace icnn {

namespace cg = cooperative_groups;

struct GemmArgs {
  int M, N, K0, K1;
  const float* A0; const float* G0; int lda0;
  const float* A1; const float* G1; int lda1;
  float a1_scale, a1_shift;
  const float* W; int ldw;
  // forward epilogue
  const float* D; float* Z; float alpha;
  // backward epilogue
  int N0; const float* Zprev; const float* Cz; float* dprev;
  const float* Cy; float* g; long long g_row_stride; const int* perm; const int* count; int KS; int n;
  float g_scale;
  const int* skip_if_zero;
  // MODE 2 (tangent forward): Z = act'(Zmask) o acc
  const float* Zmask;
  // MODE 1 extras for the GD backward pass (gd_backward.cu), all optional:
  //   dCz  += kappa * Ztprev o acc          (acc = delta_i Wz_i^T before gating)
  //   Dacc += kappa * delta_{i-1}
  float* dCz; const float* Ztprev; float* Dacc; float kappa;
};

constexpr int BM = 64, BN = 64, BK = 16, PAD = 4;

__device__ __forceinline__ float* g_row_ptr(const GemmArgs& a, int m) {
  if (a.perm == nullptr) return a.g + (long long)m * a.g_row_stride;
  int slot = a.perm[(long long)m * a.KS + a.count[m]];
  return a.g + ((long long)m * a.KS + slot) * a.n;
}

// One output element of the fused epilogue (shared by the register and the split-K paths).
template <int MODE>
__device__ __forceinline__ void epilogue_elem(const GemmArgs& a, int m, int nn, float acc, float* grow) {
  if (MODE == 0) {
    const float v = acc + a.D[(long long)m * a.N + nn];
    a.Z[(long long)m * a.N + nn] = v > 0.f ? v : a.alpha * v;
  } else if (MODE == 2) {
    const long long idx = (long long)m * a.N + nn;
    a.Z[idx] = a.Zmask ? (a.Zmask[idx] > 0.f ? 1.f : a.alpha) * acc : acc;   // Zmask == nullptr: plain product
  } else {
    if (nn < a.N0) {
      const long long idx = (long long)m * a.N0 + nn;
      const float da = a.Zprev[idx] > 0.f ? 1.f : a.alpha;
      const float dp = da * a.Cz[idx] * acc;
      a.dprev[idx] = dp;
      if (a.dCz) a.dCz[idx] = fmaf(a.kappa * a.Ztprev[idx], acc, a.dCz[idx]);
      if (a.Dacc) a.Dacc[idx] = fmaf(a.kappa, dp, a.Dacc[idx]);
    } else {
      const int e = nn - a.N0;
      grow[e] = fmaf(a.g_scale * a.Cy[(long long)m * a.n + e], acc, grow[e]);
    }
  }
}

// MODE 0: forward (W is [K, N]);  MODE 1: backward (W is [N, K], K = K0, no second segment);
// MODE 2: MODE 0's product with the tangent epilogue (no bias, activation pattern taken from Zmask)
// Split-K: gridDim.z = S CTAs of one thread-block cluster share an output tile; each reduces a
// K-slice, the partial tiles are summed through distributed shared memory (rank r owns BM/S rows
// of the tile for the reduction + epilogue).  S = 1 is the plain kernel.
template <int MODE>
__global__ void __launch_bounds__(256) gated_gemm_kernel(GemmArgs a) {
  if (a.skip_if_zero != nullptr && *a.skip_if_zero == 0) return;
  __shared__ __align__(16) float smem_f[2 * BK * (BM + PAD) + 2 * BK * (BN + PAD)];
  float (*As)[BK][BM + PAD] = reinterpret_cast<float (*)[BK][BM + PAD]>(smem_f);
  float (*Bs)[BK][BN + PAD] = reinterpret_cast<float (*)[BK][BN + PAD]>(smem_f + 2 * BK * (BM + PAD));
  const int t = threadIdx.x;
  const int S = gridDim.z;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int K = a.K0 + a.K1;
  const int ty = t / 16, tx = t % 16;

  // loader coordinates
  const int a_row = t / 4, a_k = (t % 4) * 4;  // A tile: 64 rows x 16 k
  const int b_k = t / 16, b_n = (t % 16) * 4;  // fwd W tile: 16 k x 64 n
  const int bt_n = t / 4, bt_k = (t % 4) * 4;  // bwd W tile: 64 n x 16 k

  float ra[4], rb[4];
  auto load_tiles = [&](int k0) {
    const int m = m0 + a_row;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int kk = k0 + a_k + i;
      float v = 0.f;
      if (m < a.M && kk < K) {
        if (kk < a.K0) {
          v = a.A0[(long long)m * a.lda0 + kk];
          if (a.G0) v *= a.G0[(long long)m * a.lda0 + kk];
        } else {
          const int k1 = kk - a.K0;
          v = fmaf(a.a1_scale, a.A1[(long long)m * a.lda1 + k1], a.a1_shift);
          if (a.G1) v *= a.G1[(long long)m * a.lda1 + k1];
        }
      }
      ra[i] = v;
    }
    if (MODE != 1) {
      const int kk = k0 + b_k;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int nn = n0 + b_n + i;
        rb[i] = (kk < K && nn < a.N) ? a.W[(long long)kk * a.ldw + nn] : 0.f;
      }
    } else {
      const int nn = n0 + bt_n;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int kk = k0 + bt_k + i;
        rb[i] = (kk < K && nn < a.N) ? a.W[(long long)nn * a.ldw + kk] : 0.f;
      }
    }
  };
  auto store_tiles = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 4; ++i) As[buf][a_k + i][a_row] = ra[i];
    if (MODE != 1) {
#pragma unroll
      for (int i = 0; i < 4; ++i) Bs[buf][b_k][b_n + i] = rb[i];
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) Bs[buf][bt_k + i][bt_n] = rb[i];
    }
  };

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const int nk_all = (K + BK - 1) / BK;
  const int kt0 = (int)(((long long)nk_all * blockIdx.z) / S);
  const int nk = (int)(((long long)nk_all * (blockIdx.z + 1)) / S) - kt0;
  if (nk > 0) { load_tiles(kt0 * BK); store_tiles(0); }
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) load_tiles((kt0 + kt + 1) * BK);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 av = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 bv = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float aa[4] = {av.x, av.y, av.z, av.w};
      const float bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(aa[i], bb[j], acc[i][j]);
    }
    if (kt + 1 < nk) store_tiles(buf ^ 1);
    __syncthreads();
  }

  if (S == 1) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int m = m0 + ty * 4 + i;
      if (m >= a.M) continue;
      float* grow = (MODE == 1) ? g_row_ptr(a, m) : nullptr;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int nn = n0 + tx * 4 + j;
        if (nn < a.N) epilogue_elem<MODE>(a, m, nn, acc[i][j], grow);
      }
    }
    return;
  }
  // ---- split-K: partial tile -> own shared memory -> DSMEM reduction ----
  cg::cluster_group cluster = cg::this_cluster();
  float (*Ps)[BN + 1] = reinterpret_cast<float (*)[BN + 1]>(smem_f);   // [BM][BN+1] floats fit
  static_assert(BM * (BN + 1) <= 2 * BK * (BM + PAD) + 2 * BK * (BN + PAD), "partial tile must fit");
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) Ps[ty * 4 + i][tx * 4 + j] = acc[i][j];
  cluster.sync();
  const int rank = (int)cluster.block_rank();
  const int r_lo = (BM * rank) / S, r_hi = (BM * (rank + 1)) / S;
  for (int idx = t; idx < (r_hi - r_lo) * BN; idx += 256) {
    const int rr = r_lo + idx / BN, cc = idx % BN;
    float v = 0.f;
    for (int q = 0; q < S; ++q) {
      const float* rp = cluster.map_shared_rank(&Ps[rr][cc], q);
      v += *rp;
    }
    const int m = m0 + rr, nn = n0 + cc;
    if (m < a.M && nn < a.N) {
      float* grow = (MODE == 1 && nn >= a.N0) ? g_row_ptr(a, m) : nullptr;
      epilogue_elem<MODE>(a, m, nn, v, grow);
    }
  }
  cluster.sync();   // keep every CTA's partial tile alive until all ranks have read it
}

// Launch with a (1,1,S) thread-block cluster; S chosen so that the grid covers the chip at least
// ~2x while every CTA keeps >= 4 k-tiles.
template <int MODE>
static cudaError_t launch_gemm(const GemmArgs& a, cudaStream_t st) {
  const int gx = cdiv(a.N, BN), gy = cdiv(a.M, BM);
  const int nk = cdiv(a.K0 + a.K1, BK);
  int S = 1;
  const int target = 2 * device_sms();
  while (S < 8 && gx * gy * S < target && nk / (S * 2) >= 4) S *= 2;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(gx, gy, S);
  cfg.blockDim = dim3(256);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 1; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = S;
  cfg.attrs = attr; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, gated_gemm_kernel<MODE>, a);
}

// momentum GD update, multi-label-cls/icnn-back.py:122-128
static __global__ void gd_update_kernel(float* y, float* v, const float* g, long long N, float lr, float mom) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= N) return;
  const float vp = v[i];
  const float vn = mom * vp - lr * g[i];
  y[i] = y[i] - mom * vp + (1.f + mom) * vn;
  v[i] = vn;
}

}  // namespace icnn
