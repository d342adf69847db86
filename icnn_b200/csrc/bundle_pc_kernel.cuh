// K2, Mehrotra predictor-corrector path (solver = ICNN_SOLVER_PC): two sweeps over the bundle rows per
// interior-point iteration instead of five.
//
// Same algorithm, start and stopping rule as the reference's pdipm_pc (lib/bundle_entropy.py:5-78)
// and the same per-sample loop body as bundle_step_kernel (append, dependency test, prune:
// lib/bundle_entropy.py:211-237); what changes is how the O(k n) work of one iteration is organised:
//
//   sweep A (FP64 tensor cores, DMMA m8n8k4): ONE pass gives the weighted Gram  M0 = G D G^T  and, as two
//       pseudo-rows of the same sweep, q = G (D o ry) and w = G y  (the row pass of the old kernel);
//   k x k stage (warp 0): rd, stopping test, Cholesky of M = M0 + diag(s/z), then FOUR solves
//       M^-1 {1, r_aff, mu/z, r_q}.  The corrector right-hand side is affine in sigma,
//       r_cor = sigma (mu/z) - ds_aff o dz_aff / z   (lib/bundle_entropy.py:61-63 with rc = -(mu sigma - ds dz)/s),
//       so dz_cor = sigma dz_p + dz_q with dz_p, dz_q known BEFORE sigma is;
//   sweep B (column pass, three right-hand sides at once): v1 = G^T dz_aff, v2 = G^T dz_p, v3 = G^T dz_q.
//       v1 gives dy_aff and the affine step bound -> sigma; then dy = -D (ry + v1 + sigma v2 + v3) needs no
//       further pass over G.  v2 stays in registers (the thread that produced a column consumes it).
//   u = G^T z is maintained incrementally (u += alpha (v1 + sigma v2 + v3)), so ry = logit(y) + u costs one
//       log per element per iteration and no pass.
//
// Shared memory per sample: 4 n-vectors (y, u, ry|du, v1+v3|dy), ONE packed lower-triangular k x k matrix,
// 18 k-vectors.  All reductions over n_y and all k x k algebra are FP64, as in the reference.
//
// V3 build (three n-vectors: y, ry, v1+v3|du): for n_y where four FP64 n-vectors leave room for ONE sample per SM
// (n_y = 4096: 128 KB) the kernel is latency-bound on that one sample's serial stages (the one-warp k x k
// factor/solves, the tree sums); with three vectors and 12 aliased k-vectors a sample needs <= 113 KB, so TWO
// 8-warp samples are resident per SM and one sample's serial stage overlaps the other's sweeps.  u = G^T z is
// not stored: u_old = ry_old - logit(y_old) is recovered in the update (one more log per element per
// interior-point iteration), and dy = -D (ry + du) is recomputed there from the stored du (same expression,
// same inputs -> the same bits as the value the step bound was taken from).
#pragma once
#include "bundle_step_kernel.cuh"

namespace icnn {

struct PcArgs {
  icnn_bundle_bufs b;
  icnn_bundle_cfg c;
  int t;
  int npad;  // doubles reserved per n-vector
  int flags; // exploration knobs (bundle_pc.cu): bit 0 = general k x k stage even for k <= 32, bit 1 = plain stores for xs
};

constexpr int PC_NKV = 18;
constexpr int PC_NKV_V3 = 12;   // V3: tk / ek / rk (append + dependency test, commit) alias dza / dzp / dzq (IPM only)

__host__ __device__ inline size_t pc_group_doubles(int npad, int KS, int wps, bool gv = false, bool v3 = false) {
  size_t d = (gv ? (size_t)0 : (size_t)(v3 ? 3 : 4) * npad) + (size_t)KS * (KS + 1) / 2 +
             (size_t)(v3 ? PC_NKV_V3 : PC_NKV) * KS + KS /* row pointers */ +
             8 * wps /* two reduction buffers */ + 16 /* scalars */ + 4 /* 8 ints */;
  return (d + 1) & ~(size_t)1;
}

__device__ __forceinline__ int lidx(int r, int c) { return r * (r + 1) / 2 + c; }   // packed lower, c <= r

// In-place lower Cholesky of a packed symmetric matrix; lane r owns rows r and r + 32 (k <= 64).  The
// dot product of a column step runs on four independent accumulators (the FP64 FMA chain is the
// critical path of this one-warp stage).
__device__ __forceinline__ double chol_dot(const double* a, const double* b, int c) {
  double t0 = 0.0, t1 = 0.0, t2 = 0.0, t3 = 0.0;
  int p = 0;
  for (; p + 3 < c; p += 4) {
    t0 = fma(a[p], b[p], t0);
    t1 = fma(a[p + 1], b[p + 1], t1);
    t2 = fma(a[p + 2], b[p + 2], t2);
    t3 = fma(a[p + 3], b[p + 3], t3);
  }
  for (; p < c; ++p) t0 = fma(a[p], b[p], t0);
  return (t0 + t1) + (t2 + t3);
}
// K32: k <= 32 -> lane r owns row r only; the second-row paths (r + 32) and the (i < 32) selects compile away.
// The one-warp k x k stage is latency- AND issue-bound (ncu, C5: 9.2k warp instructions per stage at k = 20, IPC 0.27,
// a quarter of the kernel's time with the other warps parked at the barrier behind it), so the common k <= 32 case
// gets its own lean instantiation.
template <bool K32>
__device__ __forceinline__ bool warp_cholesky_impl(double* L, double* invd, int k, int lane) {
  bool ok = true;
  const int r0 = lane, r1 = lane + 32;
  const int o0 = lidx(r0, 0), o1 = lidx(r1, 0);
  for (int c = 0; c < k; ++c) {
    const int oc = lidx(c, 0);
    double s0 = 0.0, s1 = 0.0;
    if (r0 >= c && r0 < k) s0 = L[o0 + c] - chol_dot(L + o0, L + oc, c);
    if (!K32) { if (r1 >= c && r1 < k) s1 = L[o1 + c] - chol_dot(L + o1, L + oc, c); }
    const double piv = K32 ? __shfl_sync(0xffffffffu, s0, c) : __shfl_sync(0xffffffffu, (c < 32) ? s0 : s1, c & 31);
    if (!(piv > 0.0) || !isfinite(piv)) { ok = false; break; }
    const double inv = rsqrt(piv);
    if (r0 > c && r0 < k) L[o0 + c] = s0 * inv;
    if (!K32) { if (r1 > c && r1 < k) L[o1 + c] = s1 * inv; }
    if (lane == 0) { L[oc + c] = piv * inv; invd[c] = inv; }
    __syncwarp();
  }
  __syncwarp();
  return ok;
}
__device__ inline bool warp_cholesky_p(double* L, double* invd, int k, int lane) {
  return k <= 32 ? warp_cholesky_impl<true>(L, invd, k, lane) : warp_cholesky_impl<false>(L, invd, k, lane);
}

// L L^T X = B for NR right-hand sides held in registers (lane r owns rows r, r + 32), pivots by shuffle.
template <int NR, bool K32>
__device__ __forceinline__ void warp_chol_solve_impl(const double* L, const double* invd, int k, double (&b0)[NR],
                                                     double (&b1)[NR], int lane) {
  const int r0 = lane, r1 = lane + 32;
  const int o0 = lidx(r0, 0), o1 = lidx(r1, 0);
  for (int i = 0; i < k; ++i) {
    const double di = invd[i];
    const double l0 = (r0 > i && r0 < k) ? L[o0 + i] : 0.0;
    const double l1 = (!K32 && r1 > i && r1 < k) ? L[o1 + i] : 0.0;
#pragma unroll
    for (int q = 0; q < NR; ++q) {
      const double xi = (K32 ? __shfl_sync(0xffffffffu, b0[q], i) : __shfl_sync(0xffffffffu, (i < 32) ? b0[q] : b1[q], i & 31)) * di;
      b0[q] = (r0 == i) ? xi : fma(-l0, xi, b0[q]);
      if (!K32) b1[q] = (r1 == i) ? xi : fma(-l1, xi, b1[q]);
    }
  }
  for (int i = k - 1; i >= 0; --i) {
    const double di = invd[i];
    const int oi = lidx(i, 0);
    const double l0 = (r0 < i) ? L[oi + r0] : 0.0;
    const double l1 = (!K32 && r1 < i) ? L[oi + r1] : 0.0;
#pragma unroll
    for (int q = 0; q < NR; ++q) {
      const double xi = (K32 ? __shfl_sync(0xffffffffu, b0[q], i) : __shfl_sync(0xffffffffu, (i < 32) ? b0[q] : b1[q], i & 31)) * di;
      b0[q] = (r0 == i) ? xi : fma(-l0, xi, b0[q]);
      if (!K32) b1[q] = (r1 == i) ? xi : fma(-l1, xi, b1[q]);
    }
  }
}
template <int NR>
__device__ inline void warp_chol_solve_p(const double* L, const double* invd, int k, double (&b0)[NR],
                                         double (&b1)[NR], int lane) {
  if (k <= 32) warp_chol_solve_impl<NR, true>(L, invd, k, b0, b1, lane);
  else warp_chol_solve_impl<NR, false>(L, invd, k, b0, b1, lane);
}

// get_step (lib/bundle_entropy.py:158-163) over a k-vector whose elements j = lane, lane + 32 sit in registers
__device__ __forceinline__ double step2(double v0, double d0, bool ok0, double v1, double d1, bool ok1) {
  double a = 1e300;
  bool any = false;
  if (ok0 && d0 < 0.0) { a = -v0 / d0; any = true; }
  if (ok1 && d1 < 0.0) { a = fmin(a, -v1 / d1); any = true; }
  a = Grp<1>::wmin(a);
  any = __any_sync(0xffffffffu, any);
  return any ? a : 1.0;
}

// group-wide reductions with ONE barrier each: consecutive reductions alternate between two scratch
// buffers, so the next write of a buffer is separated from its last read by the barrier in between.
template <int WPS>
struct PcRed {
  double* red;  // [2][4 * WPS]
  int par;
  template <class G>
  __device__ __forceinline__ double sum(const G& g, double v) {
    v = Grp<WPS>::wsum(v);
    if (WPS == 1) { __syncwarp(); return v; }   // the reduction doubles as the barrier that publishes the n-vectors
    double* r = red + par * 4 * WPS;
    par ^= 1;
    if (g.lane == 0) r[g.warp] = v;
    g.sync();
    double a = 0.0;
#pragma unroll
    for (int w = 0; w < WPS; ++w) a += r[w];
    return a;
  }
  template <class G>
  __device__ __forceinline__ void min2(const G& g, double& a, double& b) {
    a = Grp<WPS>::wmin(a);
    b = Grp<WPS>::wmin(b);
    if (WPS == 1) { __syncwarp(); return; }
    double* r = red + par * 4 * WPS;
    par ^= 1;
    if (g.lane == 0) { r[g.warp] = a; r[WPS + g.warp] = b; }
    g.sync();
    double ra = r[0], rb = r[WPS];
#pragma unroll
    for (int w = 1; w < WPS; ++w) { ra = fmin(ra, r[w]); rb = fmin(rb, r[WPS + w]); }
    a = ra; b = rb;
  }
};

// D = y (1 - y) = 1 / (1/y + 1/(1-y))  (lib/bundle_entropy.py:18), one FMA; the same expression everywhere
__device__ __forceinline__ double dweight(double y) { return fma(-y, y, y); }

// ---- sweep A: weighted Gram + the two pseudo-rows on the FP64 tensor cores --------------------------
// Sweep rows: R = 0 -> pseudo-row whose A-fragment value is D_j ry_j  (result row 0:  q = G (D o ry)),
//             R = 1 -> pseudo-row whose A-fragment value is y_j       (result row 1:  w = G y),
//             R >= 2 -> bundle row R - 2 (A fragment G D, B fragment G).
// Row blocks of 8, tiles (a0 + i, b0 + j); TRI: a0 == b0, upper triangle of tiles only.  Lane (r, q) =
// (lane / 4, lane % 4) loads columns 4q..4q+3 of row 8 blk + r of a 16-column group: its A/B fragment
// elements for four consecutive k-steps.  The n-vectors are padded to a multiple of 16 doubles with finite
// values, so only the loads of G are predicated.  The warp partials are summed by a fixed tree through a
// scratch n-vector (deterministic), and warp 0 stores the result (packed matrix / q / w).
// VEC: rows are 16-byte aligned (n % 4 == 0) -> one 128-bit load per row block.
template <int WPS, int NA, int NB, bool TRI, bool PSEUDO, bool VEC, bool GVL, class G>
__device__ __forceinline__ void gram_sweep_pc(const G& g, const float* const* rowp, int k, int n, const double* yv,
                                              const double* rv, double* Lp, double* qk, double* wk, double* scratch,
                                              int scap, int a0, int b0) {
  constexpr int NT = TRI ? NA * (NA + 1) / 2 : NA * NB;
  constexpr int NL = TRI ? NB : NA + NB;
  double acc[NT][2];
#pragma unroll
  for (int t = 0; t < NT; ++t) acc[t][0] = acc[t][1] = 0.0;
  const int r = g.lane >> 2, q = g.lane & 3;
  const float* rp[NL];
  bool rok[NL];
#pragma unroll
  for (int b = 0; b < NL; ++b) {
    const int blk = TRI ? (b0 + b) : (b < NA ? a0 + b : b0 + (b - NA));
    const int row = blk * 8 + r - 2;
    rok[b] = row >= 0 && row < k;
    rp[b] = rowp[rok[b] ? row : 0] + 4 * q;
  }
  const bool ps = PSEUDO && r < 2;   // block 0 is the first loaded block; this lane carries a pseudo-row there
  const double* yq = yv + 4 * q;
  const double* rq = rv + 4 * q;
  const int ngrp = (n + 15) >> 4;
  // Two 16-column groups per loop trip when the tile set is small: both groups' row loads are issued before
  // the tensor-core work (one sample's sweep is otherwise a chain of L2 round trips); with 8+ tiles of
  // accumulators the second set of row registers would spill.
  constexpr int NG = (NT <= 6) ? 2 : 1;
#pragma unroll 1
  for (int gi = g.warp; gi < ngrp; gi += NG * WPS) {
    float4 v[NG][NL];
    double2 yl[GVL ? NG : 1][2], rl[GVL ? NG : 1][2];   // GVL: y / ry come from L2 as well -> issued with the row loads
#pragma unroll
    for (int u = 0; u < NG; ++u) {
      const int gu = gi + u * WPS;
      const int off = gu * 16;
      const int col = off + 4 * q;
      const bool gv = (u == 0) || gu < ngrp;
      if (GVL) {
        const int og = gv ? off : 0;
        yl[GVL ? u : 0][0] = *reinterpret_cast<const double2*>(yq + og);
        yl[GVL ? u : 0][1] = *reinterpret_cast<const double2*>(yq + og + 2);
        if (PSEUDO && ps && r == 0) {
          rl[GVL ? u : 0][0] = *reinterpret_cast<const double2*>(rq + og);
          rl[GVL ? u : 0][1] = *reinterpret_cast<const double2*>(rq + og + 2);
        }
      }
#pragma unroll
      for (int b = 0; b < NL; ++b) {
        v[u][b] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (VEC) {
          if (gv && rok[b] && col < n) v[u][b] = *reinterpret_cast<const float4*>(rp[b] + off);
        } else if (gv && rok[b]) {
          const float* p = rp[b] + off;
          if (col < n) v[u][b].x = p[0];
          if (col + 1 < n) v[u][b].y = p[1];
          if (col + 2 < n) v[u][b].z = p[2];
          if (col + 3 < n) v[u][b].w = p[3];
        }
      }
    }
#pragma unroll
    for (int u = 0; u < NG; ++u) {
      const int gu = gi + u * WPS;
      if (u > 0 && gu >= ngrp) break;
      const int off = gu * 16;
      const double2 ya = GVL ? yl[GVL ? u : 0][0] : *reinterpret_cast<const double2*>(yq + off);
      const double2 yb = GVL ? yl[GVL ? u : 0][1] : *reinterpret_cast<const double2*>(yq + off + 2);
      double dd[4] = {dweight(ya.x), dweight(ya.y), dweight(yb.x), dweight(yb.y)};
      double pa[4] = {0.0, 0.0, 0.0, 0.0};
      if (PSEUDO && ps) {
        if (r == 0) {
          const double2 ra = GVL ? rl[GVL ? u : 0][0] : *reinterpret_cast<const double2*>(rq + off);
          const double2 rb = GVL ? rl[GVL ? u : 0][1] : *reinterpret_cast<const double2*>(rq + off + 2);
          pa[0] = dd[0] * ra.x; pa[1] = dd[1] * ra.y; pa[2] = dd[2] * rb.x; pa[3] = dd[3] * rb.y;
        } else {
          pa[0] = ya.x; pa[1] = ya.y; pa[2] = yb.x; pa[3] = yb.y;
        }
      }
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        double f[NL];
#pragma unroll
        for (int b = 0; b < NL; ++b)
          f[b] = (double)((s == 0) ? v[u][b].x : (s == 1) ? v[u][b].y : (s == 2) ? v[u][b].z : v[u][b].w);
        int t = 0;
#pragma unroll
        for (int i = 0; i < NA; ++i) {
          // pseudo lanes have f[0] = 0 (no bundle row), the others pa = 0: one FMA selects the A value
          const double af = (PSEUDO && i == 0) ? fma(f[0], dd[s], pa[s]) : f[i] * dd[s];
#pragma unroll
          for (int j = TRI ? i : 0; j < NB; ++j) { dmma884(acc[t][0], acc[t][1], af, f[TRI ? j : NA + j]); ++t; }
        }
      }
    }
  }
  // ---- deterministic tree sum of the warp partials through the scratch vector
  if (WPS > 1) {
    constexpr int SLAB = NT * 64;
    const int cap = scap / SLAB;
    g.sync();   // scratch is free: its last readers (previous sweep / previous phase) are done
    if (cap >= 1) {
      int active = WPS;
      while (active > 1) {
        const int m = ::min(cap, active >> 1);
        if (g.warp >= active - m && g.warp < active) {
          double* sl = scratch + (size_t)(g.warp - (active - m)) * SLAB + g.lane;
#pragma unroll
          for (int t = 0; t < NT; ++t) { sl[(2 * t) * 32] = acc[t][0]; sl[(2 * t + 1) * 32] = acc[t][1]; }
        }
        g.sync();
        if (g.warp >= active - 2 * m && g.warp < active - m) {
          const double* sl = scratch + (size_t)(g.warp - (active - 2 * m)) * SLAB + g.lane;
#pragma unroll
          for (int t = 0; t < NT; ++t) { acc[t][0] += sl[(2 * t) * 32]; acc[t][1] += sl[(2 * t + 1) * 32]; }
        }
        active -= m;
        if (active > 1) g.sync();
      }
    } else {
      // scratch too small for one slab (tiny n_y): ordered accumulation straight into the outputs
      for (int wi = 1; wi < WPS; ++wi) {
        if (g.warp == wi) {
          int t = 0;
#pragma unroll
          for (int i = 0; i < NA; ++i)
#pragma unroll
            for (int j = TRI ? i : 0; j < NB; ++j) {
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int ii = (a0 + i) * 8 + r, jj = (b0 + j) * 8 + 2 * q + h;
                if (jj >= 2 && jj < k + 2) {
                  if (ii < 2) { if (PSEUDO && i == 0) { double* d = (ii == 0 ? qk : wk) + (jj - 2); *d = (wi == 1 ? 0.0 : *d) + acc[t][h]; } }
                  else if (ii < k + 2 && (!(TRI && i == j) || jj >= ii)) { double* d = Lp + lidx(jj - 2, ii - 2); *d = (wi == 1 ? 0.0 : *d) + acc[t][h]; }
                }
              }
              ++t;
            }
        }
        g.sync();
      }
    }
  }
  if (g.warp == 0) {
    const bool addin = (WPS > 1) && (scap / (NT * 64) < 1);   // ordered path left the other warps' sum in place
    int t = 0;
#pragma unroll
    for (int i = 0; i < NA; ++i)
#pragma unroll
      for (int j = TRI ? i : 0; j < NB; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int ii = (a0 + i) * 8 + r, jj = (b0 + j) * 8 + 2 * q + h;
          if (jj >= 2 && jj < k + 2) {
            if (ii < 2) {
              if (PSEUDO && i == 0) { double* d = (ii == 0 ? qk : wk) + (jj - 2); *d = (addin ? *d : 0.0) + acc[t][h]; }
            } else if (ii < k + 2 && (!(TRI && i == j) || jj >= ii)) {
              double* d = Lp + lidx(jj - 2, ii - 2);
              *d = (addin ? *d : 0.0) + acc[t][h];
            }
          }
        }
        ++t;
      }
    __syncwarp();
  }
}

template <int WPS, int NB, bool VEC, bool GVL, class G>
__device__ __forceinline__ void gram_rect_pair_pc(const G& g, const float* const* rowp, int k, int n, const double* yv,
                                                  const double* rv, double* Lp, double* qk, double* wk, double* sx, int scap) {
  gram_sweep_pc<WPS, 2, NB, false, true, VEC, GVL>(g, rowp, k, n, yv, rv, Lp, qk, wk, sx, scap, 0, 4);
  gram_sweep_pc<WPS, 2, NB, false, false, VEC, GVL>(g, rowp, k, n, yv, rv, Lp, qk, wk, sx, scap, 2, 4);
}

// k + 2 sweep rows in rb = ceil((k + 2) / 8) <= 8 row blocks (k <= 62).  On return warp 0 has stored M0, q, w.
template <int WPS, bool VEC, bool GVL, class G>
__device__ __forceinline__ void gram_pass_pc(const G& g, const float* const* rowp, int k, int n, const double* yv,
                                             const double* rv, double* Lp, double* qk, double* wk, double* sx, int scap) {
  const int rb = (k + 2 + 7) >> 3;
  if (rb == 1) gram_sweep_pc<WPS, 1, 1, true, true, VEC, GVL>(g, rowp, k, n, yv, rv, Lp, qk, wk, sx, scap, 0, 0);
  else if (rb == 2) gram_sweep_pc<WPS, 2, 2, true, true, VEC, GVL>(g, rowp, k, n, yv, rv, Lp, qk, wk, sx, scap, 0, 0);
  else if (rb == 3) gram_sweep_pc<WPS, 3, 3, true, true, VEC, GVL>(g, rowp, k, n, yv, rv, Lp, qk, wk, sx, scap, 0, 0);
  else {
    gram_sweep_pc<WPS, 4, 4, true, true, VEC, GVL>(g, rowp, k, n, yv, rv, Lp, qk, wk, sx, scap, 0, 0);
    if (rb > 4) {
      const int r2 = rb - 4;
      if (r2 == 1) { gram_sweep_pc<WPS, 1, 1, true, false, VEC, GVL>(g, rowp, k, n, yv, rv, Lp, qk, wk, sx, scap, 4, 4); gram_rect_pair_pc<WPS, 1, VEC, GVL>(g, rowp, k, n, yv, rv, Lp, qk, wk, sx, scap); }
      else if (r2 == 2) { gram_sweep_pc<WPS, 2, 2, true, false, VEC, GVL>(g, rowp, k, n, yv, rv, Lp, qk, wk, sx, scap, 4, 4); gram_rect_pair_pc<WPS, 2, VEC, GVL>(g, rowp, k, n, yv, rv, Lp, qk, wk, sx, scap); }
      else if (r2 == 3) { gram_sweep_pc<WPS, 3, 3, true, false, VEC, GVL>(g, rowp, k, n, yv, rv, Lp, qk, wk, sx, scap, 4, 4); gram_rect_pair_pc<WPS, 3, VEC, GVL>(g, rowp, k, n, yv, rv, Lp, qk, wk, sx, scap); }
      else { gram_sweep_pc<WPS, 4, 4, true, false, VEC, GVL>(g, rowp, k, n, yv, rv, Lp, qk, wk, sx, scap, 4, 4); gram_rect_pair_pc<WPS, 4, VEC, GVL>(g, rowp, k, n, yv, rv, Lp, qk, wk, sx, scap); }
    }
  }
}

// ---- sweep B: column pass with NR right-hand sides, four columns per thread per chunk ----------------
// VEC: columns cb + 4 tid + {0..3} (one 128-bit load per row);  else columns cb + tid + T {0..3}.
template <int T, bool VEC>
__device__ __forceinline__ int pc_col(int cb, int tid, int c) { return VEC ? cb + 4 * tid + c : cb + tid + c * T; }

template <int T, int NR, bool VEC>
__device__ __forceinline__ void col_dots_pc(const float* const* rowp, int k, int n, int cb, int tid,
                                            const double* const (&w)[NR], double (&acc)[NR][4]) {
#pragma unroll
  for (int q = 0; q < NR; ++q)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[q][c] = 0.0;
  const bool in0 = VEC ? (cb + 4 * tid < n) : (cb + tid < n);
  const bool full = VEC ? in0 : (cb + tid + 3 * T < n);
#pragma unroll 4
  for (int j = 0; j < k; ++j) {
    const float* p = rowp[j];
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (VEC) {
      if (in0) { const float4 x = *reinterpret_cast<const float4*>(p + cb + 4 * tid); v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w; }
    } else {
#pragma unroll
      for (int c = 0; c < 4; ++c) if (full || cb + tid + c * T < n) v[c] = p[cb + tid + c * T];
    }
#pragma unroll
    for (int q = 0; q < NR; ++q) {
      const double wq = w[q][j];
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[q][c] = fma((double)v[c], wq, acc[q][c]);
    }
  }
}

// running minimum of num / den over candidates (num >= 0, den > 0) without dividing: a/b < n/d  <=>  a d < n b.
// Start (n, d) = (1, 0) = +inf.
__device__ __forceinline__ void ratio_min(double& nm, double& dn, double a, double b) {
  if (a * dn < nm * b) { nm = a; dn = b; }
}

// ---- k x k stage (one warp): rd, stopping test, Cholesky of M = M0 + diag(s/z), the four solves ------------------
// K32: k <= 32, every lane owns at most one element / row (the j + 32 halves compile away).
struct PcKxk {
  double* Lp; double* invd; const double* zc; const double* scur; const double* wk; const double* hk; const double* qk;
  double* dza; double* dzp; double* dzq; double* dsa; double* sc; int* isc;
};
template <bool K32>
__device__ __forceinline__ void pc_kxk_stage(const PcKxk& io, int k, int lane, double pr) {
  double* Lp = io.Lp;
  const int j0 = lane, j1 = lane + 32;
  const bool v0 = j0 < k, v1ok = !K32 && j1 < k;
  const double tt = io.sc[0];
  const double z0 = v0 ? io.zc[j0] : 0.0, z1 = v1ok ? io.zc[j1] : 0.0;
  const double s0 = v0 ? io.scur[j0] : 0.0, s1 = v1ok ? io.scur[j1] : 0.0;
  const double rd0 = v0 ? ((io.wk[j0] + io.hk[j0]) - tt) + s0 : 0.0;    // rd = G y + h - t + s
  const double rd1 = v1ok ? ((io.wk[j1] + io.hk[j1]) - tt) + s1 : 0.0;
  const double zs = Grp<1>::wsum(z0 + z1);
  const double dr = Grp<1>::wsum(fma(rd0, rd0, rd1 * rd1));
  const double rt = 1.0 - zs;
  const bool conv = (sqrt(pr + rt * rt) < 1e-8 && sqrt(dr) < 1e-8);
  if (conv) {
    if (lane == 0) io.isc[2] = 1;
  } else {
    if (v0) Lp[lidx(j0, j0)] += s0 / z0;
    if (v1ok) Lp[lidx(j1, j1)] += s1 / z1;
    __syncwarp();
    const bool ok = warp_cholesky_impl<K32>(Lp, io.invd, k, lane);
    if (!ok) { if (lane == 0) io.isc[3] = 1; }
    else {
      const double mu = Grp<1>::wsum(fma(s0, z0, s1 * z1)) / k;
      // three right-hand sides in one sweep: 1, r_aff = rd - G D ry - s  (rc = z), mu / z
      const double ra0 = v0 ? rd0 - io.qk[j0] - s0 : 0.0, ra1 = v1ok ? rd1 - io.qk[j1] - s1 : 0.0;
      const double rp0 = v0 ? mu / z0 : 0.0, rp1 = v1ok ? mu / z1 : 0.0;
      double b0[3] = {v0 ? 1.0 : 0.0, ra0, rp0}, b1[3] = {v1ok ? 1.0 : 0.0, ra1, rp1};
      warp_chol_solve_impl<3, K32>(Lp, io.invd, k, b0, b1, lane);
      const double w1s = Grp<1>::wsum(b0[0] + b1[0]);
      const double dta = (Grp<1>::wsum(fma(ra0, b0[0], ra1 * b1[0])) - rt) / w1s;
      const double dtp = Grp<1>::wsum(fma(rp0, b0[0], rp1 * b1[0])) / w1s;
      const double da0 = fma(-dta, b0[0], b0[1]), da1 = fma(-dta, b1[0], b1[1]);   // dz_aff
      const double dp0 = fma(-dtp, b0[0], b0[2]), dp1 = fma(-dtp, b1[0], b1[2]);   // dz_p
      const double dsa0 = v0 ? -(s0 / z0) * (z0 + da0) : 0.0, dsa1 = v1ok ? -(s1 / z1) * (z1 + da1) : 0.0;
      // r_q = -(ds_aff o dz_aff) / z
      const double rq0 = v0 ? -(dsa0 * da0) / z0 : 0.0, rq1 = v1ok ? -(dsa1 * da1) / z1 : 0.0;
      double c0[1] = {rq0}, c1[1] = {rq1};
      warp_chol_solve_impl<1, K32>(Lp, io.invd, k, c0, c1, lane);
      const double dtq = Grp<1>::wsum(fma(rq0, b0[0], rq1 * b1[0])) / w1s;
      if (v0) { io.dza[j0] = da0; io.dzp[j0] = dp0; io.dzq[j0] = fma(-dtq, b0[0], c0[0]); io.dsa[j0] = dsa0; }
      if (v1ok) { io.dza[j1] = da1; io.dzp[j1] = dp1; io.dzq[j1] = fma(-dtq, b1[0], c1[0]); io.dsa[j1] = dsa1; }
      if (lane == 0) { io.sc[1] = dta; io.sc[2] = dtp; io.sc[3] = dtq; }
    }
  }
  __syncwarp();
}

// ---- the kernel ----------------------------------------------------------------------------------------
// One CTA of WPS warps per sample (the block scheduler balances the SMs at sample granularity: with several
// samples per CTA the last, partly filled wave costs a whole extra round);  NCH = chunks of 4 T columns per
// thread (n <= 4 T NCH);  R80: 80-register build (768 threads / SM) instead of 128 registers (512 / SM).
// GV: the four n-vectors of a sample live in the caller's scratch (icnn_bundle_bufs::vec_ws, L2-resident) instead of
// shared memory: shared memory per sample drops to the k x k part, so the samples in flight per SM are bounded by
// registers / threads only and the one-warp k x k stage of one sample overlaps the sweeps of the others.
template <int WPS, int NCH, bool R80, bool VEC, bool GV = false, bool V3 = false>
__global__ void __launch_bounds__(WPS * 32, WPS == 16 ? 1 : (R80 ? 24 : 16) / WPS) bundle_pc_kernel(PcArgs A) {
  static_assert(!(GV && V3), "V3 is a shared-memory layout");
  const icnn_bundle_bufs& b = A.b;
  const icnn_bundle_cfg& cf = A.c;
  if (b.nactive[A.t] == 0) return;
  extern __shared__ __align__(16) double smem_d[];
  constexpr int GPB = 1;
  constexpr int T = WPS * 32;
  static_assert(NCH == 1 || NCH == 2 || NCH == 4, "NCH");
  Grp<WPS, 1> g;
  g.tid = threadIdx.x % T;
  g.lane = threadIdx.x & 31;
  g.warp = g.tid >> 5;
  g.gid = threadIdx.x / T;
  const int u = blockIdx.x * GPB + g.gid;
  if (u >= b.B) return;
  if (b.finished[u]) return;

  const int n = b.n, KS = b.KS, npad = A.npad;
  double* base = smem_d + (size_t)g.gid * pc_group_doubles(npad, KS, WPS, GV, V3);
  double* yv = GV ? b.vec_ws + (size_t)u * 4 * npad : base;
  double* uv = V3 ? nullptr : yv + npad;   // V3: u is not stored (recovered as ry - logit(y) in the update)
  double* rv = V3 ? yv + npad : uv + npad;   // ry, then du (V3: ry only)
  double* xv = rv + npad;   // v1 + v3, then dy (V3: then du) ; scratch of the dependency test and of the sweep-A tree sum
  double* Lp = GV ? base : xv + npad;   // packed lower k x k
  double* kv = Lp + (size_t)KS * (KS + 1) / 2;
#define PCKV(i) (kv + (i) * KS)
  double* hk = PCKV(0);
  double* wk = PCKV(5);    // G y
  double* qk = PCKV(6);    // G (D o ry)
  double* dza = PCKV(7);
  double* dzp = PCKV(8);
  double* dzq = PCKV(9);
  double* dsa = PCKV(10);
  double* invd = PCKV(11);
  // V3: these three live in the append / dependency test and (tk) the commit only; dza / dzp / dzq in the IPM loop only
  double* tk = PCKV(V3 ? 7 : 12);
  double* ek = PCKV(V3 ? 8 : 13);
  double* rk = PCKV(V3 ? 9 : 14);
  const float** rowp = reinterpret_cast<const float**>(kv + (size_t)(V3 ? PC_NKV_V3 : PC_NKV) * KS);
  PcRed<WPS> red;
  red.red = reinterpret_cast<double*>(rowp + KS);
  red.par = 0;
  g.red = red.red;              // Grp's own two-barrier reductions (append / dependency test) share the scratch
  double* sc = red.red + 8 * WPS;
  int* isc = reinterpret_cast<int*>(sc + 16);

  const int k0 = b.count[u];
  const int k = k0 + 1;
  const int* permu = b.perm + (size_t)u * KS;
  float* Gu = b.G + (size_t)u * KS * n;
  double* hu = b.h + (size_t)u * KS;
  double* lamu = b.lam + (size_t)u * KS;
  double* rsu = b.rsum + (size_t)u * KS;
  double* gramu = b.gram + (size_t)u * KS * KS;
  double* yu = b.y + (size_t)u * n;
  const int slot_new = permu[k0];

  for (int j = g.tid; j < k; j += T) rowp[j] = Gu + (size_t)permu[j] * n;
  if (g.tid == 0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) isc[i] = 0;
  }
  g.sync();
  const float* gnew = rowp[k0];

  // ---- append: h = f - g.y ; row sum ; unweighted Gram row ; xs copy ; non-finite guard  (lib/bundle_entropy.py:207,215-217)
  {
    double hs = 0.0, rs = 0.0, bad = 0.0, ent = 0.0;
    double* ysrow = b.ys ? b.ys + ((size_t)u * KS + slot_new) * n : nullptr;
    for (int e = g.tid; e < n; e += T) {
      const double ge = (double)gnew[e];
      const double ye = yu[e];
      hs = fma(ge, ye, hs);
      rs += ge;
      if (!isfinite(ge)) bad = 1.0;
      if (ysrow) { if (A.flags & 2) ysrow[e] = ye; else __stcs(ysrow + e, ye); }   // write-only during the solve: streaming store
      if (b.iter_stats) ent += neg_entropy(ye);
    }
    if (b.iter_stats) ent = g.sum(ent);
    hs = g.sum(hs);
    rs = g.sum(rs);
    bad = g.max(bad);
    const double fu = b.f64 ? b.f64[u] : (double)b.f[u];
    if (g.tid == 0) { stat_add(b.iter_stats, A.t, 0, 1.0); stat_add(b.iter_stats, A.t, 6, fu + ent); }
    if (bad > 0.0 || !isfinite(fu)) {
      if (g.tid == 0) { b.status[u] = ICNN_ST_NONFINITE; b.finished[u] = 1; b.nIters[u] = A.t - 1; stat_add(b.iter_stats, A.t, 5, 1.0); }
      return;
    }
    for (int j = g.warp; j < k; j += WPS) {
      const float* rj = rowp[j];
      double acc = 0.0;
      int diff = 0;
      for (int e = g.lane; e < n; e += 32) {
        const float a = rj[e], c = gnew[e];
        acc = fma((double)a, (double)c, acc);
        diff |= (a != c);
      }
      acc = Grp<WPS>::wsum(acc);
      diff = __any_sync(0xffffffffu, diff);
      if (g.lane == 0) { tk[j] = acc; ek[j] = diff ? 1.0 : 0.0; }
    }
    if (g.tid == 0) { hu[slot_new] = fu - hs; rsu[slot_new] = rs; sc[10] = fu - hs; sc[11] = rs; }
    g.sync();
    if (g.tid == 0) {
      int dup = 0;
      for (int j = 0; j < k0; ++j) dup |= (ek[j] == 0.0);
      isc[0] = dup;
    }
    g.sync();
  }
  // ---- dependency test (stands in for np.linalg.matrix_rank, lib/bundle_entropy.py:219): as bundle_step_kernel
  bool dependent = false;
  if (k > n) dependent = true;
  else if (k0 > 0) {
    if (g.warp == 0) {
      for (int i = g.lane; i < k0; i += 32)
        for (int j = 0; j <= i; ++j) Lp[lidx(i, j)] = gramu[(size_t)permu[i] * KS + permu[j]];
      __syncwarp();
      const bool ok = warp_cholesky_p(Lp, invd, k0, g.lane);
      if (ok) {
        double b0[1] = {g.lane < k0 ? tk[g.lane] : 0.0}, b1[1] = {g.lane + 32 < k0 ? tk[g.lane + 32] : 0.0};
        warp_chol_solve_p<1>(Lp, invd, k0, b0, b1, g.lane);
        if (g.lane < k0) rk[g.lane] = b0[0];
        if (g.lane + 32 < k0) rk[g.lane + 32] = b1[0];
      }
      double md = tk[k0];
      for (int j = g.lane; j < k0; j += 32) md = fmax(md, gramu[(size_t)permu[j] * KS + permu[j]]);
      md = Grp<1>::wmax(md);
      if (g.lane == 0) { isc[1] = ok ? 1 : 0; sc[9] = md; }
      __syncwarp();
    }
    g.sync();
    const double maxdiag = sc[9];
    if (isc[0]) dependent = true;
    else if (!isc[1]) dependent = false;
    else {
      const double thr2 = cf.rank_tol * cf.rank_tol * maxdiag;
      for (int rep = 0; rep < 2; ++rep) {
        double p = 0.0;
        col_pass<T>(rowp, k0, n, g.tid, rk, [&](int e, double a) {
          const double r = (rep ? xv[e] : (double)gnew[e]) - a;
          xv[e] = r;
          p = fma(r, r, p);
        });
        p = g.sum(p);
        if (p <= thr2) { dependent = true; break; }
        if (rep == 1 || p > 1e-8 * maxdiag) break;
        g.sync();
        for (int j = g.warp; j < k0; j += WPS) {
          double acc = 0.0;
          for (int e = g.lane; e < n; e += 32) acc = fma((double)rowp[j][e], xv[e], acc);
          acc = Grp<WPS>::wsum(acc);
          if (g.lane == 0) rk[j] = acc;
        }
        g.sync();
        if (g.warp == 0) {
          double b0[1] = {g.lane < k0 ? rk[g.lane] : 0.0}, b1[1] = {g.lane + 32 < k0 ? rk[g.lane + 32] : 0.0};
          warp_chol_solve_p<1>(Lp, invd, k0, b0, b1, g.lane);
          if (g.lane < k0) rk[g.lane] = b0[0];
          if (g.lane + 32 < k0) rk[g.lane + 32] = b1[0];
        }
        g.sync();
      }
    }
  } else {
    dependent = !(tk[0] > 0.0);
  }
  if (dependent) {
    if (g.tid == 0) { b.status[u] = ICNN_ST_RANK_STOP; b.finished[u] = 1; b.nIters[u] = A.t - 1; stat_add(b.iter_stats, A.t, 5, 1.0); }
    return;
  }
  for (int j = g.tid; j < k; j += T) {
    gramu[(size_t)slot_new * KS + permu[j]] = tk[j];
    gramu[(size_t)permu[j] * KS + slot_new] = tk[j];
    hk[j] = (j == k0) ? sc[10] : hu[permu[j]];
    PCKV(1)[j] = 1.0 / k;   // z
    PCKV(3)[j] = 1.0;       // s
  }
  if (g.tid == 0) sc[0] = 1.0;  // t
  // pads of the n-vectors the tensor-core sweep reads: y = 0.5, ry = 0 (finite; the G loads there are zero)
  for (int e = n + g.tid; e < npad; e += T) { yv[e] = 0.5; rv[e] = 0.0; }
  g.sync();

  // =====================  Mehrotra predictor-corrector, lib/bundle_entropy.py:5-78  =====================
  const int maxit = cf.max_inner > 0 ? cf.max_inner : 20;
  int inner_its = 0, fail = 0;
  int zsel = 0;   // z lives in k-vector 1 + zsel, s in 3 + zsel; the update writes the other buffer
  // y = 0.5 (logit = 0), u = G^T z0, ry = u
  double pr = 0.0;
  {
    const double* const w1r[1] = {PCKV(1)};
#pragma unroll 1
    for (int ch = 0; ch < NCH; ++ch) {
      const int cb = ch * 4 * T;
      if (cb >= n) break;
      double acc[1][4];
      col_dots_pc<T, 1, VEC>(rowp, k, n, cb, g.tid, w1r, acc);
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int e = pc_col<T, VEC>(cb, g.tid, c);
        if (e < n) { yv[e] = 0.5; if (!V3) uv[e] = acc[0][c]; rv[e] = acc[0][c]; pr = fma(acc[0][c], acc[0][c], pr); }
      }
    }
  }
  pr = red.sum(g, pr);
  const int j0 = g.lane, j1 = g.lane + 32;
  const bool v0 = j0 < k, v1ok = j1 < k;
#pragma unroll 1
  for (int it = 0; it < maxit; ++it) {
    double* zc = PCKV(1 + zsel);
    double* scur = PCKV(3 + zsel);
    // ---- sweep A (warp 0 ends up holding M0, q, w in shared memory)
    gram_pass_pc<WPS, VEC, GV>(g, rowp, k, n, yv, rv, Lp, qk, wk, xv, npad);
    // ---- k x k stage
    if (g.warp == 0) {
      const PcKxk io{Lp, invd, zc, scur, wk, hk, qk, dza, dzp, dzq, dsa, sc, isc};
      if (k <= 32 && !(A.flags & 1)) pc_kxk_stage<true>(io, k, g.lane, pr);
      else pc_kxk_stage<false>(io, k, g.lane, pr);
    }
    g.sync();
    if (isc[2]) break;
    if (isc[3]) { fail = 1; break; }
    inner_its = it + 1;
    // ---- sweep B: v1 = G^T dz_aff, v2 = G^T dz_p, v3 = G^T dz_q ; dy_aff = -D (ry + v1) and its step bounds
    double x2a[4], x2b[4], x2c[4], x2d[4];   // v2 of this thread's columns, per chunk (NCH <= 4)
    double n1 = 1.0, d1 = 0.0, n2 = 1.0, d2 = 0.0;   // min over dy<0 of y/(-dy); min over dy>0 of (1-y)/dy
    {
      const double* const w3[3] = {dza, dzp, dzq};
#pragma unroll 1
      for (int ch = 0; ch < NCH; ++ch) {
        const int cb = ch * 4 * T;
        if (cb >= n) break;
        double acc[3][4];
        col_dots_pc<T, 3, VEC>(rowp, k, n, cb, g.tid, w3, acc);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int e = pc_col<T, VEC>(cb, g.tid, c);
          if (e < n) {
            const double ye = yv[e];
            const double dy = -dweight(ye) * (rv[e] + acc[0][c]);
            if (dy < 0.0) ratio_min(n1, d1, ye, -dy);          // get_step(y, dy)
            if (dy > 0.0) ratio_min(n2, d2, 1.0 - ye, dy);     // get_step(1-y, -dy)
            xv[e] = acc[0][c] + acc[2][c];
          }
          const double v2 = acc[1][c];
          if (ch == 0) x2a[c] = v2; else if (ch == 1) x2b[c] = v2; else if (ch == 2) x2c[c] = v2; else x2d[c] = v2;
        }
      }
    }
    double st = d1 > 0.0 ? n1 / d1 : 1e300, st2 = d2 > 0.0 ? n2 / d2 : 1e300;
    red.min2(g, st, st2);
    st = fmin(st > 1e299 ? 1.0 : st, st2 > 1e299 ? 1.0 : st2);
    // ---- sigma and the combined direction (every warp, redundantly: lanes own elements j, j + 32)
    const double z0 = v0 ? zc[j0] : 0.0, z1 = v1ok ? zc[j1] : 0.0;
    const double s0 = v0 ? scur[j0] : 0.0, s1 = v1ok ? scur[j1] : 0.0;
    const double da0 = v0 ? dza[j0] : 0.0, da1 = v1ok ? dza[j1] : 0.0;
    const double dsa0 = v0 ? dsa[j0] : 0.0, dsa1 = v1ok ? dsa[j1] : 0.0;
    double dz0, dz1, ds0, ds1, dtt, sig;
    {
      const double alpha = fmin(fmin(step2(z0, da0, v0, z1, da1, v1ok), step2(s0, dsa0, v0, s1, dsa1, v1ok)), fmin(st, 1.0));
      const double num = Grp<1>::wsum(fma(s0 + alpha * dsa0, z0 + alpha * da0, (s1 + alpha * dsa1) * (z1 + alpha * da1)));
      const double den = Grp<1>::wsum(fma(s0, z0, s1 * z1));
      const double sg = num / den;
      sig = sg * sg * sg;
      const double mu = den / k;
      const double dzc0 = v0 ? fma(sig, dzp[j0], dzq[j0]) : 0.0, dzc1 = v1ok ? fma(sig, dzp[j1], dzq[j1]) : 0.0;
      const double rc0 = v0 ? -(mu * sig - dsa0 * da0) / s0 : 0.0, rc1 = v1ok ? -(mu * sig - dsa1 * da1) / s1 : 0.0;
      dz0 = da0 + dzc0; dz1 = da1 + dzc1;
      ds0 = v0 ? dsa0 - (s0 / z0) * (rc0 + dzc0) : 0.0;
      ds1 = v1ok ? dsa1 - (s1 / z1) * (rc1 + dzc1) : 0.0;
      dtt = sc[1] + fma(sig, sc[2], sc[3]);
    }
    // ---- dy = -D (ry + v1 + sigma v2 + v3), step bounds; du = v1 + sigma v2 + v3
    n1 = 1.0; d1 = 0.0; n2 = 1.0; d2 = 0.0;
#pragma unroll 1
    for (int ch = 0; ch < NCH; ++ch) {
      const int cb = ch * 4 * T;
      if (cb >= n) break;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int e = pc_col<T, VEC>(cb, g.tid, c);
        const double v2 = (ch == 0) ? x2a[c] : (ch == 1) ? x2b[c] : (ch == 2) ? x2c[c] : x2d[c];
        if (e < n) {
          const double ye = yv[e];
          const double du = fma(sig, v2, xv[e]);
          const double dy = -dweight(ye) * (rv[e] + du);
          if (dy < 0.0) ratio_min(n1, d1, ye, -dy);
          if (dy > 0.0) ratio_min(n2, d2, 1.0 - ye, dy);
          if (V3) xv[e] = du;            // ry stays in rv; dy is recomputed in the update
          else { xv[e] = dy; rv[e] = du; }
        }
      }
    }
    st = d1 > 0.0 ? n1 / d1 : 1e300; st2 = d2 > 0.0 ? n2 / d2 : 1e300;
    red.min2(g, st, st2);
    st = fmin(st > 1e299 ? 1.0 : st, st2 > 1e299 ? 1.0 : st2);
    double a = fmin(fmin(step2(s0, ds0, v0, s1, ds1, v1ok), step2(z0, dz0, v0, z1, dz1, v1ok)), st);
    a = fmax(0.0, fmin(1.0, 0.99 * a));
    if (g.warp == 0) {   // the other warps may still be reading z / s: write the other buffer
      double* zn = PCKV(2 - zsel);
      double* snew = PCKV(4 - zsel);
      if (v0) { zn[j0] = fma(a, dz0, z0); snew[j0] = fma(a, ds0, s0); }
      if (v1ok) { zn[j1] = fma(a, dz1, z1); snew[j1] = fma(a, ds1, s1); }
      if (g.lane == 0) sc[0] += a * dtt;
    }
    zsel ^= 1;
    // ---- y += a dy ; u += a du ; ry = logit(y) + u
    pr = 0.0;
#pragma unroll 1
    for (int ch = 0; ch < NCH; ++ch) {
      const int cb = ch * 4 * T;
      if (cb >= n) break;
      // one warp per sample: keep the log / division body rolled (ncu, C3: 36 % of the warp cycles were
      // instruction-fetch stalls with the 4x unrolled body; many small CTAs at different code positions per SM)
#pragma unroll (WPS == 1 ? 1 : 4)
      for (int c = 0; c < 4; ++c) {
        const int e = pc_col<T, VEC>(cb, g.tid, c);
        if (e < n) {
          if (V3) {
            const double yo = yv[e], ro = rv[e], du = xv[e];
            const double dy = -dweight(yo) * (ro + du);            // the expression of the pass above, same inputs
            const double uo = ro - log(yo / (1.0 - yo));           // u = ry - logit(y)
            const double ye = fma(a, dy, yo);
            const double ue = fma(a, du, uo);
            const double r = log(ye / (1.0 - ye)) + ue;
            yv[e] = ye; rv[e] = r;
            pr = fma(r, r, pr);
          } else {
            const double ye = fma(a, xv[e], yv[e]);
            const double ue = fma(a, rv[e], uv[e]);
            const double r = log(ye / (1.0 - ye)) + ue;
            yv[e] = ye; uv[e] = ue; rv[e] = r;
            pr = fma(r, r, pr);
          }
        }
      }
    }
    pr = red.sum(g, pr);   // the barrier also publishes y / ry / z / s for the next sweep
  }
  g.sync();
  const double* zfin = PCKV(1 + zsel);

  // ---- commit: y, lambda, prune (lam > thr), bookkeeping  (lib/bundle_entropy.py:228,234-237) -----------
  double bad = 0.0;
  for (int e = g.tid; e < n; e += T) {
    const double ye = yv[e];
    if (!isfinite(ye)) bad = 1.0;
    yu[e] = ye;
    b.y32[(size_t)u * n + e] = (float)ye;
  }
  bad = g.max(bad);
  if (g.tid == 0) {
    int nk = 0, nd = 0;
    int* oldp = reinterpret_cast<int*>(tk);      // two int scratch arrays of KS entries in one k-vector
    int* dropped = oldp + KS;
    int* pw = b.perm + (size_t)u * KS;
    for (int j = 0; j < k; ++j) oldp[j] = pw[j];
    for (int j = 0; j < k; ++j) {
      const double lj = zfin[j];
      if (lj > cf.prune_thr) { pw[nk++] = oldp[j]; lamu[oldp[j]] = lj; }
      else dropped[nd++] = oldp[j];
    }
    for (int j = 0; j < nd; ++j) pw[nk + j] = dropped[j];
    b.count[u] = nk;
    int fin = 0;
    int stt = ICNN_ST_RUNNING;
    if (fail || b.status[u] == ICNN_ST_SOLVE_FAIL) stt = ICNN_ST_SOLVE_FAIL;   // sticky: an earlier failed inner solve stays visible
    if (bad > 0.0) { stt = ICNN_ST_NONFINITE; fin = 1; }
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
#undef PCKV
}

struct PcConfig { int wps, nch, npad, minb; bool vec, gv, v3; size_t smem; };

template <int WPS, int NCH, bool VEC, bool GV = false, bool V3 = false>
static cudaError_t launch_pc(const PcArgs& a, const PcConfig& c, int B, cudaStream_t st) {
  void (*kern)(PcArgs);
  if constexpr (V3) kern = bundle_pc_kernel<WPS, NCH, false, VEC, false, true>;   // 128-register build, two CTAs per SM
  else if constexpr (WPS == 16) kern = bundle_pc_kernel<16, NCH, false, VEC, GV>;
  else kern = (c.minb >= 3) ? bundle_pc_kernel<WPS, NCH, true, VEC, GV> : bundle_pc_kernel<WPS, NCH, false, VEC, GV>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c.smem);
  if (e != cudaSuccess) return e;
  if constexpr (V3) {   // the whole point is two 113 KB samples per SM: ask for the largest shared-memory carve-out
    e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) return e;
  }
  kern<<<(unsigned)B, WPS * 32, c.smem, st>>>(a);
  return cudaGetLastError();
}

}  // namespace icnn
