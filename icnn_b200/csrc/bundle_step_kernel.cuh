// K2: one outer iteration of the bundle-entropy method for every unfinished sample.
//
// Restates on the GPU the per-sample loop body of the reference's three solveBatch copies
// (paths relative to the locuslab/icnn repository):
//   lib/bundle_entropy.py:211-237        append row, SVD rank stop, pdipm_pc (:5-78), prune lam<=1e-8
//   lib/bundle_entropy_dual.py:148-174   append, rank stop, proj_newton_logistic (:15-85), prune lam<=0
//   RL/src/bundle_entropy.py:106-131     append, Newton (:14-83), clip [.03,.97], |dy|<1e-6 stop
//
// Work decomposition: a GROUP of WPS warps owns one sample (WPS = 1 for small n_y: eight samples
// per CTA; WPS = 8: one CTA per sample).  Bundle rows G_j (float32, written by K1 straight into
// the sample's free slot) are streamed coalesced along n_y; every reduction over n_y is
// accumulated in FP64, the k x k algebra (k <= KS) is FP64 in shared memory and is executed by
// warp 0 of the group.  Three access patterns cover every variant:
//   column pass : thread owns columns e, loops rows j      ->  n-vector  = G^T w      (k loads/col)
//   row pass    : warp owns rows j, lanes stride columns   ->  k-vector  = G v       (shuffle reduce)
//   gram pass   : warp owns 4x4 blocks of the k x k output ->  G diag(w) G^T         (shuffle reduce)
#pragma once
#include "common.cuh"

#include <cooperative_groups.h>

#include <cstdlib>

namespace cg = cooperative_groups;

namespace icnn {

struct StepArgs {
  icnn_bundle_bufs b;
  icnn_bundle_cfg c;
  int t;
  int npad;  // doubles reserved per n-vector in shared memory (local column slice)
  int ld;    // leading dimension of the k x k matrices
  int nloc;  // columns owned by one CTA (= n when the sample is not split over a cluster)
  int gpitch;  // floats per resident G row in shared memory, 0 = rows are streamed from L2
};

constexpr int NKVEC = 20;  // k-vectors per group in shared memory

__host__ __device__ inline size_t xb_doubles(int KS, int ld) { return ((size_t)KS * ld + 2 * KS + 8 + 1) & ~(size_t)1; }

__host__ __device__ inline size_t group_smem_doubles(int npad, int KS, int ld, int wps, int gpitch, int cs) {
  // 3 n-vectors, 2 matrices, NKVEC k-vectors, reduction scratch, scalars,
  // [cluster export buffer: M + 2 k-vectors + 8 scalars], [resident G rows: KS x gpitch floats]
  size_t d = (size_t)3 * npad + (size_t)2 * KS * ld + (size_t)NKVEC * KS + 4 * wps + 16;
  if (cs > 1) d += xb_doubles(KS, ld);
  d += ((size_t)KS * gpitch + 1) / 2;
  return (d + 1) & ~(size_t)1;
}

// generic float load: bundle rows are either streamed from global memory or resident in shared memory
__device__ __forceinline__ float ldf(const float* p) { return *p; }

template <int WPS, int CS = 1>
struct Grp {
  int tid, lane, warp, gid;
  double* red;  // [4*WPS]
  double* xb;   // cluster export buffer (CS > 1): [KS*ld + 2*KS + 8]
  static constexpr int T = WPS * 32;

  // ---- reductions over the whole sample = group, then (CS > 1) the CTAs of the cluster.  Every
  // CTA combines the CS partials in rank order, so all CTAs hold bit-identical results and take
  // identical branches.
  __device__ __forceinline__ double cfold(double v, int op) const {
    if (CS == 1) return v;
    cg::cluster_group cl = cg::this_cluster();
    if (tid == 0) xb[0] = v;
    cl.sync();
    double r = *cl.map_shared_rank(xb, 0);
#pragma unroll
    for (int q = 1; q < CS; ++q) {
      const double o = *cl.map_shared_rank(xb, q);
      r = (op == 0) ? r + o : (op == 1) ? fmin(r, o) : fmax(r, o);
    }
    cl.sync();
    return r;
  }
  // two minima in one exchange (the step bounds of y and 1-y)
  __device__ __forceinline__ void cmin2(double& a, double& b) const {
    a = wmin(a); b = wmin(b);
    if (WPS > 1) {
      if (lane == 0) { red[warp] = a; red[WPS + warp] = b; }
      sync();
      double ra = red[0], rb = red[WPS];
#pragma unroll
      for (int w = 1; w < WPS; ++w) { ra = fmin(ra, red[w]); rb = fmin(rb, red[WPS + w]); }
      sync();
      a = ra; b = rb;
    }
    if (CS > 1) { a = cfold(a, 1); b = cfold(b, 1); }
  }
  __device__ __forceinline__ double csum(double v) const { return cfold(sum(v), 0); }
  __device__ __forceinline__ double cmin(double v) const { return cfold(min(v), 1); }
  __device__ __forceinline__ double cmax(double v) const { return cfold(max(v), 2); }
  // in-place cluster sum of up to three shared-memory segments (one exchange)
  __device__ __forceinline__ void cvsum(double* p0, int l0, double* p1 = nullptr, int l1 = 0,
                                        double* p2 = nullptr, int l2 = 0) const {
    if (CS == 1) return;
    cg::cluster_group cl = cg::this_cluster();
    sync();
    for (int i = tid; i < l0; i += T) xb[i] = p0[i];
    for (int i = tid; i < l1; i += T) xb[l0 + i] = p1[i];
    for (int i = tid; i < l2; i += T) xb[l0 + l1 + i] = p2[i];
    cl.sync();
    const int tot = l0 + l1 + l2;
    for (int i = tid; i < tot; i += T) {
      double r = 0.0;
#pragma unroll
      for (int q = 0; q < CS; ++q) r += *cl.map_shared_rank(xb + i, q);
      if (i < l0) p0[i] = r; else if (i < l0 + l1) p1[i - l0] = r; else p2[i - l0 - l1] = r;
    }
    cl.sync();
  }

  __device__ __forceinline__ void sync() const {
    if (WPS == 1) __syncwarp();
    else if (WPS >= 8) __syncthreads();      // the group is the whole CTA (256 or 512 threads)
    else asm volatile("bar.sync %0, %1;" ::"r"(gid + 1), "r"(WPS * 32) : "memory");
  }
  static __device__ __forceinline__ double wsum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
  }
  static __device__ __forceinline__ double wmin(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
  }
  static __device__ __forceinline__ double wmax(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
  }
  // all-reduce over the group; every thread gets the result
  __device__ __forceinline__ double sum(double v) const {
    v = wsum(v);
    if (WPS == 1) return v;
    if (lane == 0) red[warp] = v;
    sync();
    double r = 0.0;
#pragma unroll
    for (int w = 0; w < WPS; ++w) r += red[w];
    sync();
    return r;
  }
  __device__ __forceinline__ double min(double v) const {
    v = wmin(v);
    if (WPS == 1) return v;
    if (lane == 0) red[warp] = v;
    sync();
    double r = red[0];
#pragma unroll
    for (int w = 1; w < WPS; ++w) r = fmin(r, red[w]);
    sync();
    return r;
  }
  __device__ __forceinline__ double max(double v) const {
    v = wmax(v);
    if (WPS == 1) return v;
    if (lane == 0) red[warp] = v;
    sync();
    double r = red[0];
#pragma unroll
    for (int w = 1; w < WPS; ++w) r = fmax(r, red[w]);
    sync();
    return r;
  }
};

// ---- k x k dense algebra, executed by ONE warp (lane-parallel over rows), FP64 in smem -------

// In-place lower Cholesky of the symmetric matrix A (full storage, leading dim ld), left-looking,
// lane r owns rows r and r+32.  invd[c] = 1 / L[c][c].  Returns false on a non-positive /
// non-finite pivot.  One __syncwarp per column; pivots travel by shuffle, not shared memory.
// K32 (k <= 32): lane r owns row r only -- the r + 32 halves and the (c < 32) selects compile away (this one-warp
// stage is issue-bound: ncu counted 460 warp instructions per row of k in the general form).
template <bool K32>
__device__ __forceinline__ bool warp_cholesky_t(double* A, double* invd, int k, int ld, int lane) {
  bool ok = true;
  const int r0 = lane, r1 = lane + 32;
  for (int c = 0; c < k; ++c) {
    double s0 = 0.0, s1 = 0.0;
    if (r0 >= c && r0 < k) {
      s0 = A[r0 * ld + c];
      for (int p = 0; p < c; ++p) s0 = fma(-A[r0 * ld + p], A[c * ld + p], s0);
    }
    if (!K32) {
      if (r1 >= c && r1 < k) {
        s1 = A[r1 * ld + c];
        for (int p = 0; p < c; ++p) s1 = fma(-A[r1 * ld + p], A[c * ld + p], s1);
      }
    }
    const double piv = K32 ? __shfl_sync(0xffffffffu, s0, c) : __shfl_sync(0xffffffffu, (c < 32) ? s0 : s1, c & 31);
    if (!(piv > 0.0) || !isfinite(piv)) { ok = false; break; }
    const double inv = rsqrt(piv);
    if (r0 > c && r0 < k) A[r0 * ld + c] = s0 * inv;
    if (!K32) { if (r1 > c && r1 < k) A[r1 * ld + c] = s1 * inv; }
    if (lane == 0) { A[c * ld + c] = piv * inv; invd[c] = inv; }
    __syncwarp();
  }
  __syncwarp();
  return ok;
}
__device__ inline bool warp_cholesky(double* A, double* invd, int k, int ld, int lane) {
  return k <= 32 ? warp_cholesky_t<true>(A, invd, k, ld, lane) : warp_cholesky_t<false>(A, invd, k, ld, lane);
}

// Solve L L^T X = B in place for NR right-hand sides held in shared memory (rhs[q][0..k)).
// The running vectors live in registers (lane r owns rows r, r+32) and the pivots are broadcast
// by shuffle, so a substitution step costs one shuffle + one FMA of latency instead of two
// shared-memory round trips.
template <int NR, bool K32>
__device__ __forceinline__ void warp_chol_solve_t(const double* L, const double* invd, int k, int ld,
                                                  double* const (&rhs)[NR], int lane) {
  const int r0 = lane, r1 = lane + 32;
  double b0[NR], b1[NR];
#pragma unroll
  for (int q = 0; q < NR; ++q) {
    b0[q] = (r0 < k) ? rhs[q][r0] : 0.0;
    b1[q] = (!K32 && r1 < k) ? rhs[q][r1] : 0.0;
  }
  for (int i = 0; i < k; ++i) {  // forward: L x = b
    const double di = invd[i];
    const double l0 = (r0 > i && r0 < k) ? L[r0 * ld + i] : 0.0;
    const double l1 = (!K32 && r1 > i && r1 < k) ? L[r1 * ld + i] : 0.0;
#pragma unroll
    for (int q = 0; q < NR; ++q) {
      const double xi = (K32 ? __shfl_sync(0xffffffffu, b0[q], i) : __shfl_sync(0xffffffffu, (i < 32) ? b0[q] : b1[q], i & 31)) * di;
      b0[q] = (r0 == i) ? xi : fma(-l0, xi, b0[q]);
      if (!K32) b1[q] = (r1 == i) ? xi : fma(-l1, xi, b1[q]);
    }
  }
  for (int i = k - 1; i >= 0; --i) {  // backward: L^T x = b
    const double di = invd[i];
    const double l0 = (r0 < i) ? L[i * ld + r0] : 0.0;
    const double l1 = (!K32 && r1 < i) ? L[i * ld + r1] : 0.0;
#pragma unroll
    for (int q = 0; q < NR; ++q) {
      const double xi = (K32 ? __shfl_sync(0xffffffffu, b0[q], i) : __shfl_sync(0xffffffffu, (i < 32) ? b0[q] : b1[q], i & 31)) * di;
      b0[q] = (r0 == i) ? xi : fma(-l0, xi, b0[q]);
      if (!K32) b1[q] = (r1 == i) ? xi : fma(-l1, xi, b1[q]);
    }
  }
#pragma unroll
  for (int q = 0; q < NR; ++q) {
    if (r0 < k) rhs[q][r0] = b0[q];
    if (!K32) { if (r1 < k) rhs[q][r1] = b1[q]; }
  }
  __syncwarp();
}
template <int NR>
__device__ inline void warp_chol_solve(const double* L, const double* invd, int k, int ld,
                                       double* const (&rhs)[NR], int lane) {
  if (k <= 32) warp_chol_solve_t<NR, true>(L, invd, k, ld, rhs, lane);
  else warp_chol_solve_t<NR, false>(L, invd, k, ld, rhs, lane);
}

// step length keeping v + a dv >= 0  (lib/bundle_entropy.py:158-163), over a k-vector, one warp
__device__ inline double warp_max_step(const double* v, const double* dv, int k, int lane) {
  double a = 1e300;
  bool any = false;
  for (int j = lane; j < k; j += 32)
    if (dv[j] < 0.0) { a = fmin(a, -v[j] / dv[j]); any = true; }
  a = Grp<1>::wmin(a);
  any = __any_sync(0xffffffffu, any);
  return any ? a : 1.0;
}

__device__ __forceinline__ double softplus_d(double x) {  // lib/bundle_entropy_dual.py:6-12
  return x > 1.0 ? log1p(exp(-x)) + x : log1p(exp(x));
}

// ---- G passes -----------------------------------------------------------------------------

// column pass core: acc[c] = sum_j G_j[e_c] * w[j] for this thread's CHN columns
// e_c = cb + c*T + tid.  The row loop is outermost so w[j] and the row pointer are read from
// shared memory once per CHN global loads.  PRED: guard e_c < n (ragged tail only).
template <int T, int CHN, bool PRED>
__device__ __forceinline__ void col_dots(const float* const* rowp, int k, int n, int cb, int tid,
                                         const double* w, double (&acc)[CHN]) {
#pragma unroll
  for (int c = 0; c < CHN; ++c) acc[c] = 0.0;
  // several rows in flight per thread: the row loads are L2-latency bound
#pragma unroll (CHN >= 8 ? 2 : 4)
  for (int j = 0; j < k; ++j) {
    const float* p = rowp[j] + cb + tid;
    const double wj = w[j];
    float v[CHN];
#pragma unroll
    for (int c = 0; c < CHN; ++c) v[c] = (!PRED || cb + c * T + tid < n) ? ldf(p + c * T) : 0.f;
#pragma unroll
    for (int c = 0; c < CHN; ++c) acc[c] = fma((double)v[c], wj, acc[c]);
  }
}

template <int T, int CHN, bool PRED, class F>
__device__ __forceinline__ void col_chunk(const float* const* rowp, int k, int n, int cb, int tid,
                                          const double* w, F&& f) {
  double acc[CHN];
  col_dots<T, CHN, PRED>(rowp, k, n, cb, tid, w, acc);
#pragma unroll
  for (int c = 0; c < CHN; ++c) {
    const int e = cb + c * T + tid;
    if (!PRED || e < n) f(e, acc[c]);
  }
}

// column pass: for every column e, f(e, sum_j G_j[e] w[j]).  8 columns per thread per chunk while
// they last, then 4 / 2 / 1, then one predicated chunk for the ragged tail.
template <int T, class F>
__device__ __forceinline__ void col_pass(const float* const* rowp, int k, int n, int tid,
                                         const double* w, F&& f) {
  int cb = 0;
  for (; cb + 8 * T <= n; cb += 8 * T) col_chunk<T, 8, false>(rowp, k, n, cb, tid, w, f);
  if (cb + 4 * T <= n) { col_chunk<T, 4, false>(rowp, k, n, cb, tid, w, f); cb += 4 * T; }
  if (cb + 2 * T <= n) { col_chunk<T, 2, false>(rowp, k, n, cb, tid, w, f); cb += 2 * T; }
  if (cb + T <= n) { col_chunk<T, 1, false>(rowp, k, n, cb, tid, w, f); cb += T; }
  if (cb < n) col_chunk<T, 1, true>(rowp, k, n, cb, tid, w, f);
}

// FP64 tensor-core MMA, D(8x8) += A(8x4) * B(4x8).  Fragments (PTX ISA, m8n8k4 .f64):
// A: lane holds A[lane/4][lane%4];  B: lane holds B[lane%4][lane/4];  C/D: lane holds
// C[lane/4][2*(lane%4) + {0,1}].
__device__ __forceinline__ void dmma884(double& d0, double& d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}

// gram pass (fallback, any n): warp owns 4x4 blocks of M = G diag(w) G^T, lanes stride columns.
template <int WPS, class G>
__device__ inline void gram_pass_simt(const G& g, const float* const* rowp, int k, int n,
                                      const double* w, double* M, int ld, int widx, int nw) {
  const int kb = (k + 3) >> 2;
  const int nblk = kb * (kb + 1) / 2;
  for (int blk = (widx < 0 ? nblk : widx); blk < nblk; blk += nw) {
    int bi = 0, rem = blk;
    while (rem >= kb - bi) { rem -= kb - bi; ++bi; }
    const int bj = bi + rem;
    const float* ri[4];
    const float* rj[4];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      ri[a] = rowp[min(bi * 4 + a, k - 1)];
      rj[a] = rowp[min(bj * 4 + a, k - 1)];
    }
    double acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
    for (int e = g.lane; e < n; e += 32) {
      const double we = w[e];
      double vi[4], vj[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) { vi[a] = (double)ldf(ri[a] + e) * we; vj[a] = (double)ldf(rj[a] + e); }
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = fma(vi[a], vj[b], acc[a][b]);
    }
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const double v = Grp<WPS>::wsum(acc[a][b]);
        const int i = bi * 4 + a, j = bj * 4 + b;
        if (g.lane == 0 && i < k && j < k) { M[i * ld + j] = v; M[j * ld + i] = v; }
      }
  }
}

// gram pass on the FP64 tensor cores (n % 4 == 0): every warp sweeps its own 16-column groups
// for a rectangle of 8x8 tiles (row blocks a0..a0+NA-1 x b0..b0+NB-1; TRI: a0 == b0 and only the
// upper triangle), so each row of the rectangle is read once per sweep with one 128-bit load
// per lane per row block -- lane (r, q) = (lane/4, lane%4) gets columns 4q..4q+3 of row
// 8*blk + r, which are its A/B fragment elements for four consecutive k-steps (the four columns
// of a k-step may be any four, as long as A, B and w agree).  Warp partials are then added into
// M in warp order (deterministic).
template <int WPS, int NA, int NB, bool TRI, class G>
__device__ inline void gram_sweep(const G& g, const float* const* rowp, int k, int n,
                                  const double* w, double* M, int ld, int a0, int b0, int widx, int nw) {
  constexpr int NT = TRI ? NA * (NA + 1) / 2 : NA * NB;
  constexpr int NL = TRI ? NB : NA + NB;   // row blocks to load (TRI: A and B blocks coincide)
  double acc[NT][2];
#pragma unroll
  for (int t = 0; t < NT; ++t) acc[t][0] = acc[t][1] = 0.0;
  const int r = g.lane >> 2, q = g.lane & 3;
  const float* rp[NL];
  bool rok[NL];
#pragma unroll
  for (int b = 0; b < NL; ++b) {
    const int blk = TRI ? (b0 + b) : (b < NA ? a0 + b : b0 + (b - NA));
    const int row = blk * 8 + r;
    rok[b] = row < k;
    rp[b] = rowp[rok[b] ? row : k - 1] + 4 * q;
  }
  const int ngrp = (n + 15) >> 4;
  for (int gi = (widx < 0 ? ngrp : widx); gi < ngrp; gi += nw) {
    const int col = gi * 16 + 4 * q;
    const bool cv = col < n;  // n % 4 == 0: the whole float4 is in or out
    float4 v[NL];
#pragma unroll
    for (int b = 0; b < NL; ++b)
      v[b] = (cv && rok[b]) ? *reinterpret_cast<const float4*>(rp[b] + gi * 16) : make_float4(0.f, 0.f, 0.f, 0.f);
    double wv[4];
    if (cv) {
      const double2 w01 = *reinterpret_cast<const double2*>(w + col);
      const double2 w23 = *reinterpret_cast<const double2*>(w + col + 2);
      wv[0] = w01.x; wv[1] = w01.y; wv[2] = w23.x; wv[3] = w23.y;
    } else {
      wv[0] = wv[1] = wv[2] = wv[3] = 0.0;
    }
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      double f[NL];
#pragma unroll
      for (int b = 0; b < NL; ++b)
        f[b] = (double)((s == 0) ? v[b].x : (s == 1) ? v[b].y : (s == 2) ? v[b].z : v[b].w);
      int t = 0;
#pragma unroll
      for (int i = 0; i < NA; ++i) {
        const double af = f[i] * wv[s];   // A fragment carries the weight
#pragma unroll
        for (int j = TRI ? i : 0; j < NB; ++j) { dmma884(acc[t][0], acc[t][1], af, f[TRI ? j : NA + j]); ++t; }
      }
    }
  }
  // ordered accumulation of the warp partials into M (symmetric fill)
  for (int wi = 0; wi < nw; ++wi) {
    if (widx == wi) {
      int t = 0;
#pragma unroll
      for (int i = 0; i < NA; ++i)
#pragma unroll
        for (int j = TRI ? i : 0; j < NB; ++j) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int ii = (a0 + i) * 8 + r, jj = (b0 + j) * 8 + 2 * q + h;
            if (ii < k && jj < k && (!(TRI && i == j) || jj >= ii)) {
              const double val = (wi == 0 ? 0.0 : M[ii * ld + jj]) + acc[t][h];
              M[ii * ld + jj] = val;
              M[jj * ld + ii] = val;
            }
          }
          ++t;
        }
    }
    g.sync();
  }
}

template <int WPS, int NB, class G>
__device__ inline void gram_rect_pair(const G& g, const float* const* rowp, int k, int n,
                                      const double* w, double* M, int ld, int widx, int nw) {
  gram_sweep<WPS, 2, NB, false>(g, rowp, k, n, w, M, ld, 0, 4, widx, nw);
  gram_sweep<WPS, 2, NB, false>(g, rowp, k, n, w, M, ld, 2, 4, widx, nw);
}

// Warps widx = 0..nw-1 of the group sweep the Gram (the others -- widx < 0 -- only take part in the
// barriers), so that a row pass can run on the remaining warps at the same time.
template <int WPS, class G>
__device__ inline void gram_pass(const G& g, const float* const* rowp, int k, int n,
                                 const double* w, double* M, int ld, int widx, int nw) {
  if ((n & 3) != 0) { gram_pass_simt<WPS>(g, rowp, k, n, w, M, ld, widx, nw); g.sync(); return; }
  const int rb = (k + 7) >> 3;   // <= 8 (KS <= 64)
  if (rb == 1) gram_sweep<WPS, 1, 1, true>(g, rowp, k, n, w, M, ld, 0, 0, widx, nw);
  else if (rb == 2) gram_sweep<WPS, 2, 2, true>(g, rowp, k, n, w, M, ld, 0, 0, widx, nw);
  else if (rb == 3) gram_sweep<WPS, 3, 3, true>(g, rowp, k, n, w, M, ld, 0, 0, widx, nw);
  else {
    gram_sweep<WPS, 4, 4, true>(g, rowp, k, n, w, M, ld, 0, 0, widx, nw);
    if (rb > 4) {   // rows 32..k-1: second triangle + the 4 x (rb-4) rectangle in two halves
      const int r2 = rb - 4;
      if (r2 == 1) { gram_sweep<WPS, 1, 1, true>(g, rowp, k, n, w, M, ld, 4, 4, widx, nw); gram_rect_pair<WPS, 1>(g, rowp, k, n, w, M, ld, widx, nw); }
      else if (r2 == 2) { gram_sweep<WPS, 2, 2, true>(g, rowp, k, n, w, M, ld, 4, 4, widx, nw); gram_rect_pair<WPS, 2>(g, rowp, k, n, w, M, ld, widx, nw); }
      else if (r2 == 3) { gram_sweep<WPS, 3, 3, true>(g, rowp, k, n, w, M, ld, 4, 4, widx, nw); gram_rect_pair<WPS, 3>(g, rowp, k, n, w, M, ld, widx, nw); }
      else { gram_sweep<WPS, 4, 4, true>(g, rowp, k, n, w, M, ld, 4, 4, widx, nw); gram_rect_pair<WPS, 4>(g, rowp, k, n, w, M, ld, widx, nw); }
    }
  }
}

// ---- the step kernel ----------------------------------------------------------------------

// CS > 1: the sample is split over a thread-block cluster of CS CTAs by columns (WPS == 8); each
// CTA keeps its column slice of the bundle rows RESIDENT in shared memory (A.gpitch > 0), runs
// the column / row / Gram passes on its slice and exchanges the partial sums through distributed
// shared memory; the k x k algebra is replicated in every CTA.
// WPS == 16: one 512-thread CTA per sample, for n_y so large that shared memory allows a single CTA
// per SM anyway (C5: n_y = 4096) -- twice the threads on the passes.
template <int WPS, int MINB, int CS>
__global__ void __launch_bounds__(WPS == 16 ? 512 : 256, MINB) bundle_step_kernel(StepArgs A) {
  const icnn_bundle_bufs& b = A.b;
  const icnn_bundle_cfg& cf = A.c;
  if (b.nactive[A.t] == 0) return;
  extern __shared__ __align__(16) double smem_d[];
  constexpr int GPB = (WPS >= 8) ? 1 : 8 / WPS;  // groups per block
  constexpr int T = WPS * 32;
  static_assert(CS == 1 || WPS == 8, "a cluster-split sample owns whole CTAs");
  Grp<WPS, CS> g;
  g.tid = threadIdx.x % T;
  g.lane = threadIdx.x & 31;
  g.warp = g.tid >> 5;
  g.gid = threadIdx.x / T;
  constexpr int NWG = (WPS >= 2) ? WPS / 2 : 1;                  // warps that sweep the Gram
  const int WIDX = (WPS == 1) ? 0 : (g.warp < NWG ? g.warp : -1);
  const int crank = (CS == 1) ? 0 : (int)cg::this_cluster().block_rank();
  const int u = (CS == 1) ? blockIdx.x * GPB + g.gid : (int)(blockIdx.x / CS);
  if (u >= b.B) return;
  if (b.finished[u]) return;

  const int nglob = b.n, KS = b.KS, ld = A.ld, npad = A.npad;
  const int c0 = crank * A.nloc;                       // first column of this CTA's slice
  const int n = ::min(A.nloc, nglob - c0);             // columns of the slice ("n" below is LOCAL)
  const bool lead = (crank == 0);                      // the CTA that writes per-sample scalars
  double* base = smem_d + (size_t)g.gid * group_smem_doubles(npad, KS, ld, WPS, A.gpitch, CS);
  double* yv = base;            // n-vectors
  double* rv = yv + npad;
  double* dv = rv + npad;
  double* M = dv + npad;        // k x k
  double* Lm = M + (size_t)KS * ld;
  double* kv = Lm + (size_t)KS * ld;
  double* hk = kv + 0 * KS;     // offsets h_j (logical order)
  double* zk = kv + 1 * KS;     // lambda / z
  double* sk = kv + 2 * KS;
  double* rdk = kv + 3 * KS;
  double* qk = kv + 4 * KS;
  double* rk = kv + 5 * KS;
  double* dza = kv + 6 * KS;
  double* dsa = kv + 7 * KS;
  double* dzc = kv + 8 * KS;
  double* invd = kv + 9 * KS;   // 1 / diag(L)
  double* w1 = kv + 10 * KS;
  double* ck = kv + 11 * KS;
  double* gk = kv + 12 * KS;   // gradient
  double* g0 = kv + 13 * KS;
  double* dk = kv + 14 * KS;   // Newton direction
  double* lnk = kv + 15 * KS;  // trial lambda
  double* yk = kv + 16 * KS;   // change of variables y (lambda with pivot set to 1)
  double* ek = kv + 17 * KS;   // e vector
  double* tk = kv + 18 * KS;   // temp
  const float** rowp = reinterpret_cast<const float**>(kv + 19 * KS);  // row pointers (k <= KS)
  g.red = kv + (size_t)NKVEC * KS;
  double* sc = g.red + 4 * WPS;  // 16 scalars
  int* isc = reinterpret_cast<int*>(sc + 12);  // 8 ints
  g.xb = sc + 16;
  float* Gs = reinterpret_cast<float*>(g.xb + (CS > 1 ? xb_doubles(KS, ld) : 0));

  const int k0 = b.count[u];
  const int k = k0 + 1;
  const int* permu = b.perm + (size_t)u * KS;
  float* Gu = b.G + (size_t)u * KS * nglob + c0;
  double* hu = b.h + (size_t)u * KS;
  double* lamu = b.lam + (size_t)u * KS;
  double* rsu = b.rsum + (size_t)u * KS;
  double* gramu = b.gram + (size_t)u * KS * KS;
  double* yu = b.y + (size_t)u * nglob + c0;
  const int slot_new = permu[k0];

  if (A.gpitch > 0) {
    // stage this CTA's slice of the k active rows into shared memory: the only global read of the
    // bundle in this launch (every pass below then runs out of shared memory)
    const int gp = A.gpitch;
    if ((n & 3) == 0 && (nglob & 3) == 0) {
      const int n4 = n >> 2;
      for (int idx = g.tid; idx < k * n4; idx += T) {
        const int j = idx / n4, c = idx - j * n4;
        reinterpret_cast<float4*>(Gs + (size_t)j * gp)[c] =
            reinterpret_cast<const float4*>(Gu + (size_t)permu[j] * nglob)[c];
      }
    } else {
      for (int idx = g.tid; idx < k * n; idx += T) {
        const int j = idx / n, c = idx - j * n;
        Gs[(size_t)j * gp + c] = Gu[(size_t)permu[j] * nglob + c];
      }
    }
    for (int j = g.tid; j < k; j += T) rowp[j] = Gs + (size_t)j * gp;
  } else {
    for (int j = g.tid; j < k; j += T) rowp[j] = Gu + (size_t)permu[j] * nglob;
  }
  if (g.tid == 0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) isc[i] = 0;
  }
  g.sync();
  const float* gnew = rowp[k0];

  // ---- append: h = f - g.y ; row sum ; unweighted Gram row ; xs copy ; non-finite guard ------
  {
    double hs = 0.0, rs = 0.0, bad = 0.0, ent = 0.0;
    double* ysrow = b.ys ? b.ys + ((size_t)u * KS + slot_new) * nglob + c0 : nullptr;
    for (int e = g.tid; e < n; e += T) {
      const double ge = (double)gnew[e];
      const double ye = yu[e];
      hs = fma(ge, ye, hs);
      rs += ge;
      if (!isfinite(ge)) bad = 1.0;
      if (ysrow) __stcs(ysrow + e, ye);   // write-only during the solve: streaming store, keeps the bundle rows in L2
      if (b.iter_stats) ent += neg_entropy(ye);
    }
    if (b.iter_stats) ent = g.csum(ent);
    hs = g.csum(hs);
    rs = g.csum(rs);
    bad = g.cmax(bad);
    const double fu = b.f64 ? b.f64[u] : (double)b.f[u];
    if (g.tid == 0 && lead) { stat_add(b.iter_stats, A.t, 0, 1.0); stat_add(b.iter_stats, A.t, 6, fu + ent); }
    if (bad > 0.0 || !isfinite(fu)) {
      if (g.tid == 0 && lead) { b.status[u] = ICNN_ST_NONFINITE; b.finished[u] = 1; b.nIters[u] = A.t - 1; stat_add(b.iter_stats, A.t, 5, 1.0); }
      return;
    }
    // Gram row of the new row against all active rows (row pass), plus exact-duplicate detection
    for (int j = g.warp; j < k; j += WPS) {
      const float* rj = rowp[j];
      double acc = 0.0;
      int diff = 0;
      for (int e = g.lane; e < n; e += 32) {
        const float a = ldf(rj + e), c = gnew[e];
        acc = fma((double)a, (double)c, acc);
        diff |= (a != c);
      }
      acc = Grp<WPS>::wsum(acc);
      diff = __any_sync(0xffffffffu, diff);
      if (g.lane == 0) { tk[j] = acc; ek[j] = diff ? 1.0 : 0.0; }
    }
    if (g.tid == 0 && lead) { hu[slot_new] = fu - hs; rsu[slot_new] = rs; }
    g.sync();
    g.cvsum(tk, k, ek, k);     // Gram row and per-row "differs somewhere" counts over all slices
    if (g.tid == 0) {
      int dup = 0;
      for (int j = 0; j < k0; ++j) dup |= (ek[j] == 0.0);
      isc[0] = dup;
      sc[10] = fu - hs;        // h and row sum of the new row (identical in every CTA)
      sc[11] = rs;
    }
    g.sync();
  }
  // NOTE: control flow below is group-uniform: every decision is read from shared memory after
  // a group barrier (or is the result of a group-wide reduction).
  bool dependent = false;
  if (cf.variant != ICNN_VARIANT_RL) {
    // ---- dependency test (stands in for np.linalg.matrix_rank, lib/bundle_entropy.py:219) ----
    // distance of the new row from the span of the active rows, computed explicitly (with one
    // step of iterative refinement in the gray zone), relative to the largest row norm.
    if (k > nglob) dependent = true;
    else if (k0 > 0) {
      if (g.warp == 0) {
        for (int i = g.lane; i < k0; i += 32)
          for (int j = 0; j < k0; ++j) Lm[i * ld + j] = gramu[(size_t)permu[i] * KS + permu[j]];
        for (int j = g.lane; j < k0; j += 32) rk[j] = tk[j];
        __syncwarp();
        const bool ok = warp_cholesky(Lm, invd, k0, ld, g.lane);
        if (ok) { double* const r1[1] = {rk}; warp_chol_solve<1>(Lm, invd, k0, ld, r1, g.lane); }
        double md = tk[k0];
        for (int j = g.lane; j < k0; j += 32) md = fmax(md, gramu[(size_t)permu[j] * KS + permu[j]]);
        md = Grp<1>::wmax(md);
        if (g.lane == 0) { isc[1] = ok ? 1 : 0; sc[9] = md; }
        __syncwarp();
      }
      g.sync();
      const double maxdiag = sc[9];
      if (isc[0]) dependent = true;          // exact duplicate of an active row
      else if (!isc[1]) dependent = false;   // Gram of the active rows too ill-conditioned to
                                             // factor: near- (not exactly) dependent rows, which
                                             // the reference's float64 SVD test keeps as well
      else {
        const double thr2 = cf.rank_tol * cf.rank_tol * maxdiag;
        for (int rep = 0; rep < 2; ++rep) {
          // residual res = (rep ? res : gnew) - sum_j c_j G_j
          double p = 0.0;
          col_pass<T>(rowp, k0, n, g.tid, rk, [&](int e, double a) {
            const double r = (rep ? rv[e] : (double)gnew[e]) - a;
            rv[e] = r;
            p = fma(r, r, p);
          });
          p = g.csum(p);
          if (p <= thr2) { dependent = true; break; }
          // clearly independent (relative distance > 1e-4), or already refined once
          if (rep == 1 || p > 1e-8 * maxdiag) break;
          // gray zone: one step of iterative refinement, c' = M^-1 (G res)
          g.sync();
          for (int j = g.warp; j < k0; j += WPS) {
            double acc = 0.0;
            for (int e = g.lane; e < n; e += 32) acc = fma((double)ldf(rowp[j] + e), rv[e], acc);
            acc = Grp<WPS>::wsum(acc);
            if (g.lane == 0) rk[j] = acc;
          }
          g.sync();
          g.cvsum(rk, k0);
          if (g.warp == 0) { double* const r1[1] = {rk}; warp_chol_solve<1>(Lm, invd, k0, ld, r1, g.lane); }
          g.sync();
        }
      }
    } else {
      dependent = !(tk[0] > 0.0);  // a zero first row has rank 0 < 1
    }
    if (dependent) {
      // pop the row, mark finished, nIters = t-1 (lib/bundle_entropy.py:220-225); y unchanged
      if (g.tid == 0 && lead) { b.status[u] = ICNN_ST_RANK_STOP; b.finished[u] = 1; b.nIters[u] = A.t - 1; stat_add(b.iter_stats, A.t, 5, 1.0); }
      return;
    }
  }
  // commit the Gram row
  if (lead)
    for (int j = g.tid; j < k; j += T) {
      gramu[(size_t)slot_new * KS + permu[j]] = tk[j];
      gramu[(size_t)permu[j] * KS + slot_new] = tk[j];
    }
  for (int j = g.tid; j < k; j += T) hk[j] = (j == k0) ? sc[10] : hu[permu[j]];
  g.sync();

  int inner_its = 0;
  int fail = 0;

  if (cf.solver == ICNN_SOLVER_PC) {
    // =====================  Mehrotra predictor-corrector, lib/bundle_entropy.py:5-78  ==========
    const int maxit = cf.max_inner > 0 ? cf.max_inner : 20;
    for (int e = g.tid; e < n; e += T) yv[e] = 0.5;
    for (int j = g.tid; j < k; j += T) { zk[j] = 1.0 / k; sk[j] = 1.0; }
    if (g.tid == 0) sc[0] = 1.0;  // t
    g.sync();
    for (int it = 0; it < maxit; ++it) {
      // column pass: ry = log y - log(1-y) + G^T z ; D = y(1-y) = 1/(1/y + 1/(1-y))
      double pr = 0.0;
      col_pass<T>(rowp, k, n, g.tid, zk, [&](int e, double a) {
        const double ye = yv[e];
        const double r = log(ye / (1.0 - ye)) + a;   // = log y - log(1-y): one log + one division
        rv[e] = r;
        dv[e] = ye * (1.0 - ye);
        pr = fma(r, r, pr);
      });
      pr = g.sum(pr);   // local; (contains the barrier that publishes rv / dv)
      if (WPS == 1) __syncwarp();
      // row pass (rd = G y + h - t + s ; q = G D ry) on the upper half of the group's warps while
      // the lower half sweeps the weighted Gram on the FP64 tensor cores (both only read G, y, D, ry)
      // Rows are taken four at a time per warp: four independent loads per element (the loop is
      // L2-latency bound) and one read of y, D, ry for the four rows.
      {
        const int rw = (WPS == 1) ? 0 : g.warp - NWG, nrw = (WPS == 1) ? 1 : WPS - NWG;
        for (int j0 = 4 * rw; j0 < k && rw >= 0; j0 += 4 * nrw) {
          const float* rj[4];
#pragma unroll
          for (int r = 0; r < 4; ++r) rj[r] = rowp[::min(j0 + r, k - 1)];
          double a1[4] = {0.0, 0.0, 0.0, 0.0}, a2[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll 2
          for (int e = g.lane; e < n; e += 32) {
            float gv[4];
#pragma unroll
            for (int r = 0; r < 4; ++r) gv[r] = ldf(rj[r] + e);
            const double ye = yv[e], te = dv[e] * rv[e];
#pragma unroll
            for (int r = 0; r < 4; ++r) { a1[r] = fma((double)gv[r], ye, a1[r]); a2[r] = fma((double)gv[r], te, a2[r]); }
          }
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const double s1 = Grp<WPS>::wsum(a1[r]), s2 = Grp<WPS>::wsum(a2[r]);
            if (g.lane == 0 && j0 + r < k) { rdk[j0 + r] = s1; qk[j0 + r] = s2; }   // column sums only; h - t + s is added below
          }
        }
      }
      gram_pass<WPS>(g, rowp, k, n, dv, M, ld, WIDX, NWG);
      g.sync();
      if (CS > 1) {   // one exchange: M, (G y, G D ry) and the squared residual norm
        if (g.tid == 0) sc[11] = pr;
        g.cvsum(M, k * ld, rdk, 2 * KS, sc + 11, 1);
        pr = sc[11];
      }
      if (g.warp == 0) {
        const int lane = g.lane;
        for (int j = lane; j < k; j += 32) rdk[j] = ((rdk[j] + hk[j]) - sc[0]) + sk[j];   // rd = G y + h - t + s
        __syncwarp();
        double zs = 0.0, dr = 0.0;
        for (int j = lane; j < k; j += 32) { zs += zk[j]; dr = fma(rdk[j], rdk[j], dr); }
        zs = Grp<1>::wsum(zs);
        dr = Grp<1>::wsum(dr);
        const double rt = 1.0 - zs;
        const bool conv = (sqrt(pr + rt * rt) < 1e-8 && sqrt(dr) < 1e-8);
        if (conv) {
          if (lane == 0) isc[2] = 1;
        } else {
          for (int i = lane; i < k; i += 32) {
            for (int j = 0; j < k; ++j) Lm[i * ld + j] = M[i * ld + j];
            Lm[i * ld + i] += sk[i] / zk[i];
          }
          __syncwarp();
          const bool ok = warp_cholesky(Lm, invd, k, ld, lane);
          if (!ok) { if (lane == 0) isc[3] = 1; }
          else {
            // two right-hand sides in one sweep: w1 = M^-1 1, dza = M^-1 r with
            // r = rd - G D ry - (s/z) rc, rc = z  ->  r = rd - q - s.   Then
            // dt = (r.w1 - rt)/sum(w1) and dz_aff = M^-1 (r - dt 1) = M^-1 r - dt w1.
            for (int j = lane; j < k; j += 32) { w1[j] = 1.0; dza[j] = rdk[j] - qk[j] - sk[j]; rk[j] = dza[j]; }
            __syncwarp();
            double* const r2[2] = {w1, dza};
            warp_chol_solve<2>(Lm, invd, k, ld, r2, lane);
            double w1s = 0.0, rw = 0.0;
            for (int j = lane; j < k; j += 32) { w1s += w1[j]; rw = fma(rk[j], w1[j], rw); }
            w1s = Grp<1>::wsum(w1s);
            rw = Grp<1>::wsum(rw);
            const double dt = (rw - rt) / w1s;
            for (int j = lane; j < k; j += 32) {
              dza[j] = fma(-dt, w1[j], dza[j]);
              dsa[j] = -(sk[j] / zk[j]) * (zk[j] + dza[j]);
            }
            if (lane == 0) { sc[2] = dt; sc[3] = w1s; }
          }
        }
        __syncwarp();
      }
      g.sync();
      if (isc[2]) break;
      if (isc[3]) { fail = 1; break; }
      inner_its = it + 1;
      // column pass: dy_aff = -D (ry + G^T dz_aff) ; get_step(y, dy) and get_step(1-y, -dy)
      double st = 1e300, st2 = 1e300;
      col_pass<T>(rowp, k, n, g.tid, dza, [&](int e, double a) {
        const double dy = -dv[e] * (rv[e] + a);
        rv[e] = dy;  // rv now holds dy_aff
        const double ye = yv[e];
        // get_step(y, dy) / get_step(1-y, -dy): one division serves whichever bound applies
        const double ratio = (dy < 0.0 ? -ye : 1.0 - ye) / dy;
        if (dy < 0.0) st = fmin(st, ratio);
        if (dy > 0.0) st2 = fmin(st2, ratio);
      });
      g.cmin2(st, st2);
      st = fmin(st > 1e299 ? 1.0 : st, st2 > 1e299 ? 1.0 : st2);
      if (g.warp == 0) {
        const int lane = g.lane;
        double alpha = fmin(fmin(warp_max_step(zk, dza, k, lane), warp_max_step(sk, dsa, k, lane)),
                            fmin(st, 1.0));
        double num = 0.0, den = 0.0;
        for (int j = lane; j < k; j += 32) {
          num = fma(sk[j] + alpha * dsa[j], zk[j] + alpha * dza[j], num);
          den = fma(sk[j], zk[j], den);
        }
        num = Grp<1>::wsum(num);
        den = Grp<1>::wsum(den);
        const double sg = num / den;
        const double sig = sg * sg * sg;
        const double mu = den / k;
        // corrector: ry = rt = rd = 0, rc = -(mu sig - ds_aff dz_aff)/s  ->  r = -(s/z) rc
        for (int j = lane; j < k; j += 32) {
          const double rc = -(mu * sig - dsa[j] * dza[j]) / sk[j];
          tk[j] = rc;
          rk[j] = -(sk[j] / zk[j]) * rc;
          dzc[j] = rk[j];
        }
        __syncwarp();
        double* const r1[1] = {dzc};
        warp_chol_solve<1>(Lm, invd, k, ld, r1, lane);   // dzc = M^-1 r
        double rw = 0.0;
        for (int j = lane; j < k; j += 32) rw = fma(rk[j], w1[j], rw);
        rw = Grp<1>::wsum(rw);
        const double dtc = rw / sc[3];
        for (int j = lane; j < k; j += 32) {
          dzc[j] = fma(-dtc, w1[j], dzc[j]);      // M^-1 (r - dt_c 1)
          const double dscj = -(sk[j] / zk[j]) * (tk[j] + dzc[j]);
          dza[j] += dzc[j];   // total dz
          dsa[j] += dscj;     // total ds
        }
        if (lane == 0) sc[2] += dtc;  // total dt
        __syncwarp();
      }
      g.sync();
      // column pass: dy = dy_aff - D G^T dz_cor ; step bounds
      st = 1e300; st2 = 1e300;
      col_pass<T>(rowp, k, n, g.tid, dzc, [&](int e, double a) {
        const double dy = rv[e] - dv[e] * a;
        rv[e] = dy;
        const double ye = yv[e];
        // get_step(y, dy) / get_step(1-y, -dy): one division serves whichever bound applies
        const double ratio = (dy < 0.0 ? -ye : 1.0 - ye) / dy;
        if (dy < 0.0) st = fmin(st, ratio);
        if (dy > 0.0) st2 = fmin(st2, ratio);
      });
      g.cmin2(st, st2);
      st = fmin(st > 1e299 ? 1.0 : st, st2 > 1e299 ? 1.0 : st2);
      if (g.warp == 0) {
        const int lane = g.lane;
        double a = fmin(fmin(warp_max_step(sk, dsa, k, lane), warp_max_step(zk, dza, k, lane)), st);
        a = fmax(0.0, fmin(1.0, 0.99 * a));
        __syncwarp();
        for (int j = lane; j < k; j += 32) { sk[j] += a * dsa[j]; zk[j] += a * dza[j]; }
        if (lane == 0) { sc[0] += a * sc[2]; sc[4] = a; }
        __syncwarp();
      }
      g.sync();
      const double a = sc[4];
      for (int e = g.tid; e < n; e += T) yv[e] = fma(a, rv[e], yv[e]);
      g.sync();
    }
  } else {
    // =====================  dual projected Newton  ============================================
    // lib/bundle_entropy_dual.py:15-85 ; RL deltas RL/src/bundle_entropy.py:14-83
    const bool rl = (cf.variant == ICNN_VARIANT_RL);
    const int maxit = cf.max_inner > 0 ? cf.max_inner : (rl ? 20 : 100);
    const int maxback = rl ? 10 : 50;
    if (k == 1) {
      if (g.tid == 0) zk[0] = 1.0;  // lam = [1]  (:166-168)
      g.sync();
    } else {
      for (int j = g.tid; j < k; j += T) { zk[j] = 1.0 / k; ck[j] = ((j == k0) ? sc[11] : rsu[permu[j]]) + hk[j]; ek[j] = 1.0; }
      g.sync();
      bool done = false;
      for (int it = 0; it < maxit && !done; ++it) {
        inner_its = it + 1;
        // column pass: a = G^T lam ; z = sigma(a) ; F = -c.lam + sum softplus(a)
        double fs = 0.0;
        col_pass<T>(rowp, k, n, g.tid, zk, [&](int e, double a) {
          const double ze = 1.0 / (1.0 + exp(-a));
          yv[e] = ze;
          dv[e] = ze * (1.0 - ze);
          fs += softplus_d(a);
        });
        fs = g.csum(fs);
        if (WPS == 1) __syncwarp();
        // row pass: grad = -c + G z  (upper half of the warps; the lower half sweeps the Gram)
        for (int j = (WPS == 1 ? 0 : g.warp - NWG); j < k && j >= 0; j += (WPS == 1 ? 1 : WPS - NWG)) {
          const float* rj = rowp[j];
          double acc = 0.0;
          for (int e = g.lane; e < n; e += 32) acc = fma((double)ldf(rj + e), yv[e], acc);
          acc = Grp<WPS>::wsum(acc);
          if (g.lane == 0) gk[j] = acc;   // G z (column sums only); -c is added below
        }
        gram_pass<WPS>(g, rowp, k, n, dv, M, ld, WIDX, NWG);
        g.sync();
        g.cvsum(M, k * ld, gk, k);
        for (int j = g.tid; j < k; j += T) gk[j] -= ck[j];   // grad = -c + G z
        g.sync();
        if (g.warp == 0) {
          const int lane = g.lane;
          // F, pivot p = argmax lam (first maximum, np.argmax)
          double cl = 0.0;
          for (int j = lane; j < k; j += 32) cl = fma(ck[j], zk[j], cl);
          cl = Grp<1>::wsum(cl);
          const double F = fs - cl;
          double best = -1e300; int bi = 0;
          for (int j = lane; j < k; j += 32) if (zk[j] > best) { best = zk[j]; bi = j; }
          for (int o = 16; o > 0; o >>= 1) {
            const double ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
          }
          const int p = bi;
          // change of variables, reduced gradient / Hessian, bound set
          for (int j = lane; j < k; j += 32) {
            yk[j] = (j == p) ? 1.0 : zk[j];
            ek[j] = (j == p) ? 0.0 : 1.0;
          }
          __syncwarp();
          for (int j = lane; j < k; j += 32) g0[j] = gk[j] - ek[j] * gk[p];
          __syncwarp();
          // free list in tk (indices as doubles), built serially by lane 0 (k <= 64)
          if (lane == 0) {
            int nf = 0;
            for (int j = 0; j < k; ++j) {
              const bool bound = (j == p) || (yk[j] <= 1e-12 && g0[j] > 0.0);
              if (!bound) { tk[nf++] = (double)j; }
            }
            isc[4] = nf;
          }
          __syncwarp();
          const int nfree = isc[4];
          double gn = 0.0;
          for (int a = lane; a < nfree; a += 32) { const double v = g0[(int)tk[a]]; gn = fma(v, v, gn); }
          gn = Grp<1>::wsum(gn);
          if (sqrt(gn) < 1e-10) {
            if (lane == 0) isc[5] = 1;  // converged: return lam
          } else {
            // H0 on the free set: H0[a][b] = H[i][j] - H[j][p] - H[i][p] + H[p][p]  (e_i = e_j = 1)
            for (int a = lane; a < nfree; a += 32) {
              const int i = (int)tk[a];
              for (int c2 = 0; c2 < nfree; ++c2) {
                const int j = (int)tk[c2];
                Lm[a * ld + c2] = M[i * ld + j] - M[j * ld + p] - M[i * ld + p] + M[p * ld + p];
              }
              rk[a] = -g0[i];
            }
            __syncwarp();
            const bool ok = warp_cholesky(Lm, invd, nfree, ld, lane);
            if (!ok) {
              if (lane == 0) isc[5] = 2;  // solve failure (RL: break; dual: flagged)
            } else {
              double* const r1[1] = {rk};
              warp_chol_solve<1>(Lm, invd, nfree, ld, r1, lane);
              for (int j = lane; j < k; j += 32) dk[j] = 0.0;
              __syncwarp();
              double dg = 0.0, dmax = 0.0;
              for (int a = lane; a < nfree; a += 32) {
                const int i = (int)tk[a];
                dk[i] = rk[a];
                dg = fma(rk[a], g0[i], dg);
                dmax = fmax(dmax, fabs(rk[a]));
              }
              dg = Grp<1>::wsum(dg);
              dmax = Grp<1>::wmax(dmax);
              if (lane == 0) {
                isc[5] = 0;
                sc[5] = F; sc[6] = dg; sc[7] = dmax;
                sc[8] = rl ? fmin(1.0 / dmax, 1.0) : 1.0;  // tau
                isc[6] = p;
              }
            }
          }
          __syncwarp();
        }
        g.sync();
        if (isc[5] == 1) { inner_its = it; break; }
        if (isc[5] == 2) { fail = 1; break; }
        const int p = isc[6];
        // projected backtracking line search
        bool ret_now = false;
        for (int bt = 0; bt < maxback; ++bt) {
          const double tau = sc[8];
          if (g.warp == 0) {
            const int lane = g.lane;
            double es = 0.0;
            for (int j = lane; j < k; j += 32) {
              double yn = fmax(yk[j] + tau * dk[j], 0.0);
              if (j == p) yn = 1.0;
              lnk[j] = yn;
              es = fma(ek[j], yn, es);
            }
            es = Grp<1>::wsum(es);
            __syncwarp();
            if (lane == 0) lnk[p] = 1.0 - es;
            __syncwarp();
          }
          g.sync();
          bool accept = false;
          if (lnk[p] >= 0.0) {
            if (cf.line_search) {
              double fs2 = 0.0;
              col_pass<T>(rowp, k, n, g.tid, lnk, [&](int e, double a) { fs2 += softplus_d(a); });
              fs2 = g.csum(fs2);
              double cl = 0.0;
              for (int j = 0; j < k; ++j) cl = fma(ck[j], lnk[j], cl);
              const double Fn = fs2 - cl;
              accept = Fn < sc[5] + tau * 1e-5 * sc[6];
            } else {
              accept = true;
            }
          }
          if (accept) break;
          const bool small = rl ? (tau * sc[7] < 1e-10) : (tau < 1e-10);
          if (small) { ret_now = true; break; }
          g.sync();
          if (g.tid == 0) sc[8] = tau * 0.5;
          g.sync();
        }
        g.sync();
        for (int j = g.tid; j < k; j += T) zk[j] = lnk[j];
        g.sync();
        if (ret_now) done = true;
      }
    }
    // y = 1 / (1 + exp(G^T lam))   (:165 / :168)
    col_pass<T>(rowp, k, n, g.tid, zk, [&](int e, double a) { yv[e] = 1.0 / (1.0 + exp(a)); });
    g.sync();
  }

  // ---- commit: y, lambda, prune, bookkeeping -------------------------------------------------
  double maxdiff = 0.0, bad = 0.0;
  const bool rl = (cf.variant == ICNN_VARIANT_RL);
  for (int e = g.tid; e < n; e += T) {
    double ye = yv[e];
    if (rl) ye = fmin(fmax(ye, 0.03), 0.97);  // RL/src/bundle_entropy.py:118,123
    if (!isfinite(ye)) bad = 1.0;
    maxdiff = fmax(maxdiff, fabs(yu[e] - ye));
    yu[e] = ye;
    b.y32[(size_t)u * nglob + c0 + e] = (float)ye;
  }
  if (rl) maxdiff = g.cmax(maxdiff);
  bad = g.cmax(bad);
  if (g.tid == 0 && lead) {
    // prune (keep lam > thr), rebuild perm: kept slots, then dropped, then the old free tail
    int nk = 0, nd = 0;
    int dropped[64], oldp[64];
    int* pw = b.perm + (size_t)u * KS;
    for (int j = 0; j < k; ++j) oldp[j] = pw[j];
    for (int j = 0; j < k; ++j) {
      const double lj = zk[j];
      if (lj > cf.prune_thr) { pw[nk++] = oldp[j]; lamu[oldp[j]] = lj; }
      else dropped[nd++] = oldp[j];
    }
    for (int j = 0; j < nd; ++j) pw[nk + j] = dropped[j];
    b.count[u] = nk;
    int fin = 0;
    int stt = ICNN_ST_RUNNING;
    if (fail || b.status[u] == ICNN_ST_SOLVE_FAIL) stt = ICNN_ST_SOLVE_FAIL;   // sticky: an earlier failed inner solve stays visible
    if (bad > 0.0) { stt = ICNN_ST_NONFINITE; fin = 1; }
    if (rl && maxdiff < 1e-6) { fin = 1; if (stt == ICNN_ST_RUNNING) stt = ICNN_ST_CONVERGED; }
    b.status[u] = stt;
    if (fin) b.finished[u] = 1;
    else atomicAdd(&b.nactive[A.t + 1], 1);
    if (b.newton_its) b.newton_its[u] += inner_its;
    if (b.ksum) b.ksum[u] += k;
    if (b.iter_stats) {
      stat_add(b.iter_stats, A.t, 1, (double)k);
      stat_add(b.iter_stats, A.t, 2, (double)inner_its);
      stat_add(b.iter_stats, A.t, 3, (double)inner_its * k * k);
      stat_add(b.iter_stats, A.t, 4, (double)inner_its * k);
      if (fin) stat_add(b.iter_stats, A.t, 5, 1.0);
    }
  }
}


// ---- launch helper shared by the translation units that instantiate the kernel --------------------
struct K2Config { int wps, cs, nloc, gpitch, npad, ld; size_t smem; };

template <int WPS, int CS>
static cudaError_t launch_k2(const StepArgs& a, const K2Config& c, int B, cudaStream_t st) {
  // register budget: 3 CTAs / SM (80 registers) for the small groups and for WPS = 8 when the
  // shared-memory footprint allows it; the 128-register build otherwise
  void (*kern)(StepArgs);
  if constexpr (WPS == 16) kern = bundle_step_kernel<16, 1, CS>;
  else if constexpr (CS > 1) kern = bundle_step_kernel<WPS, 2, CS>;
  else if constexpr (WPS == 8) kern = (c.smem * 3 <= 225 * 1024) ? bundle_step_kernel<8, 3, 1> : bundle_step_kernel<8, 2, 1>;
  else kern = bundle_step_kernel<WPS, 3, 1>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c.smem);
  if (e != cudaSuccess) return e;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(CS == 1 ? cdiv(B, WPS >= 8 ? 1 : 8 / WPS) : B * CS));
  cfg.blockDim = dim3(WPS == 16 ? 512 : 256);
  cfg.dynamicSmemBytes = c.smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CS; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, a);
}

}  // namespace icnn
