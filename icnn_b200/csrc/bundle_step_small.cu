// K2 for tiny problems (n_y <= 8, at most 10 bundle slots): ONE THREAD PER SAMPLE.
//
// Same algorithm, same buffers and same semantics as bundle_step.cu (the reference's
// lib/bundle_entropy.py:211-237, lib/bundle_entropy_dual.py:148-174, RL/src/bundle_entropy.py:106-131),
// but with a whole sample's bundle (<= 8 x 8) in one thread's registers / local memory: at the RL
// dimensions (HalfCheetah: n_y = 6, 65 536 replay samples, BASELINE.json configs[3]) a warp per
// sample leaves 26 of 32 lanes idle in every pass and spends its time in shuffles and barriers.
#include "common.cuh"

namespace icnn {

struct SmallArgs {
  icnn_bundle_bufs b;
  icnn_bundle_cfg c;
  int t;
};

constexpr int NM = 8;  // max n_y
constexpr int KM = 10; // max rows (KS <= 10: covers min(nIter, n) + 1 for n_y <= 8)

__device__ __forceinline__ double softplus_s(double x) { return x > 1.0 ? log1p(exp(-x)) + x : log1p(exp(x)); }

// in-place lower Cholesky of A (k x k, full symmetric storage); false on a non-positive pivot
__device__ inline bool chol_s(double (&A)[KM][KM], int k) {
  for (int c = 0; c < k; ++c) {
    double s = A[c][c];
    for (int p = 0; p < c; ++p) s = fma(-A[c][p], A[c][p], s);
    if (!(s > 0.0) || !isfinite(s)) return false;
    const double inv = rsqrt(s);
    A[c][c] = s * inv;
    for (int r = c + 1; r < k; ++r) {
      double v = A[r][c];
      for (int p = 0; p < c; ++p) v = fma(-A[r][p], A[c][p], v);
      A[r][c] = v * inv;
    }
  }
  return true;
}
__device__ inline void chol_solve_s(const double (&L)[KM][KM], int k, double (&b)[KM]) {
  for (int i = 0; i < k; ++i) {
    double v = b[i];
    for (int p = 0; p < i; ++p) v = fma(-L[i][p], b[p], v);
    b[i] = v / L[i][i];
  }
  for (int i = k - 1; i >= 0; --i) {
    double v = b[i];
    for (int p = i + 1; p < k; ++p) v = fma(-L[p][i], b[p], v);
    b[i] = v / L[i][i];
  }
}
__device__ inline double max_step_s(const double* v, const double* dv, int k) {  // lib/bundle_entropy.py:158-163
  double a = 1e300; bool any = false;
  for (int j = 0; j < k; ++j) if (dv[j] < 0.0) { a = fmin(a, -v[j] / dv[j]); any = true; }
  return any ? a : 1.0;
}

__global__ void __launch_bounds__(128) bundle_step_small_kernel(SmallArgs A) {
  const icnn_bundle_bufs& b = A.b;
  const icnn_bundle_cfg& cf = A.c;
  if (b.nactive[A.t] == 0) return;
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= b.B || b.finished[u]) return;
  const int n = b.n, KS = b.KS;
  const int k0 = b.count[u], k = k0 + 1;
  int* permu = b.perm + (size_t)u * KS;
  const float* Gu = b.G + (size_t)u * KS * n;
  double* hu = b.h + (size_t)u * KS;
  double* lamu = b.lam + (size_t)u * KS;
  double* rsu = b.rsum + (size_t)u * KS;
  double* gramu = b.gram + (size_t)u * KS * KS;
  double* yu = b.y + (size_t)u * n;
  int sl[KM];
  for (int j = 0; j < k; ++j) sl[j] = permu[j];
  const int slot_new = sl[k0];

  double G[KM][NM], y[NM];
  for (int j = 0; j < k; ++j)
    for (int e = 0; e < n; ++e) G[j][e] = (double)Gu[(size_t)sl[j] * n + e];
  for (int e = 0; e < n; ++e) y[e] = yu[e];

  // ---- append ----
  double hs = 0.0, rs = 0.0;
  bool bad = false;
  for (int e = 0; e < n; ++e) { hs = fma(G[k0][e], y[e], hs); rs += G[k0][e]; bad |= !isfinite(G[k0][e]); }
  const double fu = b.f64 ? b.f64[u] : (double)b.f[u];
  if (b.iter_stats) {
    double ent = 0.0;
    for (int e = 0; e < n; ++e) ent += neg_entropy(y[e]);
    stat_add(b.iter_stats, A.t, 0, 1.0);
    stat_add(b.iter_stats, A.t, 6, fu + ent);
  }
  if (b.ys) { double* ysrow = b.ys + ((size_t)u * KS + slot_new) * n; for (int e = 0; e < n; ++e) ysrow[e] = y[e]; }
  if (bad || !isfinite(fu)) { b.status[u] = ICNN_ST_NONFINITE; b.finished[u] = 1; b.nIters[u] = A.t - 1; stat_add(b.iter_stats, A.t, 5, 1.0); return; }
  double tk[KM];
  bool dup = false;
  for (int j = 0; j < k; ++j) {
    double acc = 0.0; bool diff = false;
    for (int e = 0; e < n; ++e) { acc = fma(G[j][e], G[k0][e], acc); diff |= (G[j][e] != G[k0][e]); }
    tk[j] = acc;
    if (j < k0 && !diff) dup = true;
  }
  double hk[KM];
  hu[slot_new] = fu - hs; rsu[slot_new] = rs;
  for (int j = 0; j < k0; ++j) hk[j] = hu[sl[j]];
  hk[k0] = fu - hs;

  // ---- dependency test (lib / dual) ----
  if (cf.variant != ICNN_VARIANT_RL) {
    bool dependent = false;
    if (k > n) dependent = true;
    else if (k0 > 0) {
      if (dup) dependent = true;
      else {
        double L[KM][KM], c[KM];
        double maxdiag = tk[k0];
        for (int i = 0; i < k0; ++i) {
          for (int j = 0; j < k0; ++j) L[i][j] = gramu[(size_t)sl[i] * KS + sl[j]];
          c[i] = tk[i];
          maxdiag = fmax(maxdiag, L[i][i]);
        }
        if (chol_s(L, k0)) {   // else: near-dependent active rows, kept like the float64 SVD test does
          chol_solve_s(L, k0, c);
          const double thr2 = cf.rank_tol * cf.rank_tol * maxdiag;
          double res[NM];
          for (int rep = 0; rep < 2; ++rep) {
            double p = 0.0;
            for (int e = 0; e < n; ++e) {
              double r = rep ? res[e] : G[k0][e];
              for (int j = 0; j < k0; ++j) r = fma(-c[j], G[j][e], r);
              res[e] = r;
              p = fma(r, r, p);
            }
            if (p <= thr2) { dependent = true; break; }
            if (rep == 1 || p > 1e-8 * maxdiag) break;
            for (int j = 0; j < k0; ++j) { double acc = 0.0; for (int e = 0; e < n; ++e) acc = fma(G[j][e], res[e], acc); c[j] = acc; }
            chol_solve_s(L, k0, c);
          }
        }
      }
    } else dependent = !(tk[0] > 0.0);
    if (dependent) { b.status[u] = ICNN_ST_RANK_STOP; b.finished[u] = 1; b.nIters[u] = A.t - 1; stat_add(b.iter_stats, A.t, 5, 1.0); return; }
  }
  for (int j = 0; j < k; ++j) { gramu[(size_t)slot_new * KS + sl[j]] = tk[j]; gramu[(size_t)sl[j] * KS + slot_new] = tk[j]; }

  double ynew[NM], z[KM];
  int inner_its = 0, fail = 0;
  if (cf.solver == ICNN_SOLVER_PC) {
    // ---- Mehrotra predictor-corrector, lib/bundle_entropy.py:5-78 ----
    const int maxit = cf.max_inner > 0 ? cf.max_inner : 20;
    double s[KM], t = 1.0;
    for (int e = 0; e < n; ++e) ynew[e] = 0.5;
    for (int j = 0; j < k; ++j) { z[j] = 1.0 / k; s[j] = 1.0; }
    for (int it = 0; it < maxit; ++it) {
      double ry[NM], D[NM], rd[KM], q[KM];
      double pr = 0.0, zs = 0.0, dr = 0.0;
      for (int e = 0; e < n; ++e) {
        double a = 0.0;
        for (int j = 0; j < k; ++j) a = fma(G[j][e], z[j], a);
        ry[e] = log(ynew[e] / (1.0 - ynew[e])) + a;
        D[e] = ynew[e] * (1.0 - ynew[e]);
        pr = fma(ry[e], ry[e], pr);
      }
      for (int j = 0; j < k; ++j) {
        double a1 = 0.0, a2 = 0.0;
        for (int e = 0; e < n; ++e) { a1 = fma(G[j][e], ynew[e], a1); a2 = fma(G[j][e], D[e] * ry[e], a2); }
        rd[j] = ((a1 + hk[j]) - t) + s[j];
        q[j] = a2;
        zs += z[j];
        dr = fma(rd[j], rd[j], dr);
      }
      const double rt = 1.0 - zs;
      if (sqrt(pr + rt * rt) < 1e-8 && sqrt(dr) < 1e-8) break;
      inner_its = it + 1;
      double M[KM][KM], w1[KM], r[KM], dza[KM], dsa[KM];
      for (int i = 0; i < k; ++i)
        for (int j = 0; j <= i; ++j) {
          double acc = 0.0;
          for (int e = 0; e < n; ++e) acc = fma(G[i][e] * D[e], G[j][e], acc);
          M[i][j] = acc; M[j][i] = acc;
        }
      for (int j = 0; j < k; ++j) M[j][j] += s[j] / z[j];
      if (!chol_s(M, k)) { fail = 1; break; }
      double w1s = 0.0, rw = 0.0;
      for (int j = 0; j < k; ++j) { w1[j] = 1.0; r[j] = rd[j] - q[j] - s[j]; dza[j] = r[j]; }
      chol_solve_s(M, k, w1);
      chol_solve_s(M, k, dza);
      for (int j = 0; j < k; ++j) { w1s += w1[j]; rw = fma(r[j], w1[j], rw); }
      double dt = (rw - rt) / w1s;
      for (int j = 0; j < k; ++j) { dza[j] = fma(-dt, w1[j], dza[j]); dsa[j] = -(s[j] / z[j]) * (z[j] + dza[j]); }
      double dy[NM];
      double st = 1e300, st2 = 1e300;
      for (int e = 0; e < n; ++e) {
        double a = 0.0;
        for (int j = 0; j < k; ++j) a = fma(G[j][e], dza[j], a);
        dy[e] = -D[e] * (ry[e] + a);
        const double ratio = (dy[e] < 0.0 ? -ynew[e] : 1.0 - ynew[e]) / dy[e];
        if (dy[e] < 0.0) st = fmin(st, ratio);
        if (dy[e] > 0.0) st2 = fmin(st2, ratio);
      }
      st = fmin(st > 1e299 ? 1.0 : st, st2 > 1e299 ? 1.0 : st2);
      const double alpha = fmin(fmin(max_step_s(z, dza, k), max_step_s(s, dsa, k)), fmin(st, 1.0));
      double num = 0.0, den = 0.0;
      for (int j = 0; j < k; ++j) { num = fma(s[j] + alpha * dsa[j], z[j] + alpha * dza[j], num); den = fma(s[j], z[j], den); }
      const double sg = num / den, sig = sg * sg * sg, mu = den / k;
      double rc[KM], dzc[KM];
      rw = 0.0;
      for (int j = 0; j < k; ++j) {
        rc[j] = -(mu * sig - dsa[j] * dza[j]) / s[j];
        r[j] = -(s[j] / z[j]) * rc[j];
        dzc[j] = r[j];
      }
      chol_solve_s(M, k, dzc);
      for (int j = 0; j < k; ++j) rw = fma(r[j], w1[j], rw);
      const double dtc = rw / w1s;
      for (int j = 0; j < k; ++j) {
        dzc[j] = fma(-dtc, w1[j], dzc[j]);
        const double dscj = -(s[j] / z[j]) * (rc[j] + dzc[j]);
        dza[j] += dzc[j];
        dsa[j] += dscj;
      }
      dt += dtc;
      st = 1e300; st2 = 1e300;
      for (int e = 0; e < n; ++e) {
        double a = 0.0;
        for (int j = 0; j < k; ++j) a = fma(G[j][e], dzc[j], a);
        dy[e] = dy[e] - D[e] * a;
        const double ratio = (dy[e] < 0.0 ? -ynew[e] : 1.0 - ynew[e]) / dy[e];
        if (dy[e] < 0.0) st = fmin(st, ratio);
        if (dy[e] > 0.0) st2 = fmin(st2, ratio);
      }
      st = fmin(st > 1e299 ? 1.0 : st, st2 > 1e299 ? 1.0 : st2);
      double a = fmin(fmin(max_step_s(s, dsa, k), max_step_s(z, dza, k)), st);
      a = fmax(0.0, fmin(1.0, 0.99 * a));
      for (int j = 0; j < k; ++j) { s[j] += a * dsa[j]; z[j] += a * dza[j]; }
      t += a * dt;
      for (int e = 0; e < n; ++e) ynew[e] = fma(a, dy[e], ynew[e]);
    }
  } else {
    // ---- dual projected Newton, lib/bundle_entropy_dual.py:15-85 ; RL/src/bundle_entropy.py:14-83 ----
    const bool rl = (cf.variant == ICNN_VARIANT_RL);
    const int maxit = cf.max_inner > 0 ? cf.max_inner : (rl ? 20 : 100);
    const int maxback = rl ? 10 : 50;
    if (k == 1) z[0] = 1.0;
    else {
      double c[KM];
      for (int j = 0; j < k; ++j) { z[j] = 1.0 / k; c[j] = ((j == k0) ? rs : rsu[sl[j]]) + hk[j]; }
      bool done = false;
      for (int it = 0; it < maxit && !done; ++it) {
        inner_its = it + 1;
        double zz[NM], w[NM], gk[KM], H[KM][KM];
        double fs = 0.0, cl = 0.0;
        for (int e = 0; e < n; ++e) {
          double a = 0.0;
          for (int j = 0; j < k; ++j) a = fma(G[j][e], z[j], a);
          zz[e] = 1.0 / (1.0 + exp(-a));
          w[e] = zz[e] * (1.0 - zz[e]);
          fs += softplus_s(a);
        }
        for (int j = 0; j < k; ++j) {
          double acc = 0.0;
          for (int e = 0; e < n; ++e) acc = fma(G[j][e], zz[e], acc);
          gk[j] = acc - c[j];
          cl = fma(c[j], z[j], cl);
          for (int i = 0; i <= j; ++i) {
            double hh = 0.0;
            for (int e = 0; e < n; ++e) hh = fma(G[j][e] * w[e], G[i][e], hh);
            H[j][i] = hh; H[i][j] = hh;
          }
        }
        const double F = fs - cl;
        int p = 0;
        for (int j = 1; j < k; ++j) if (z[j] > z[p]) p = j;          // first maximum (np.argmax)
        double yk[KM], ek[KM], g0[KM], dk[KM];
        int fl[KM], nf = 0;
        for (int j = 0; j < k; ++j) { yk[j] = (j == p) ? 1.0 : z[j]; ek[j] = (j == p) ? 0.0 : 1.0; }
        for (int j = 0; j < k; ++j) g0[j] = gk[j] - ek[j] * gk[p];
        double gn = 0.0;
        for (int j = 0; j < k; ++j) {
          const bool bound = (j == p) || (yk[j] <= 1e-12 && g0[j] > 0.0);
          if (!bound) { fl[nf++] = j; gn = fma(g0[j], g0[j], gn); }
        }
        if (sqrt(gn) < 1e-10) { inner_its = it; break; }
        double H0[KM][KM], rr[KM];
        for (int a = 0; a < nf; ++a) {
          const int i = fl[a];
          for (int c2 = 0; c2 < nf; ++c2) { const int j = fl[c2]; H0[a][c2] = H[i][j] - H[j][p] - H[i][p] + H[p][p]; }
          rr[a] = -g0[i];
        }
        if (!chol_s(H0, nf)) { fail = 1; break; }
        chol_solve_s(H0, nf, rr);
        double dg = 0.0, dmax = 0.0;
        for (int j = 0; j < k; ++j) dk[j] = 0.0;
        for (int a = 0; a < nf; ++a) { dk[fl[a]] = rr[a]; dg = fma(rr[a], g0[fl[a]], dg); dmax = fmax(dmax, fabs(rr[a])); }
        double tau = rl ? fmin(1.0 / dmax, 1.0) : 1.0;
        double ln[KM];
        bool ret_now = false;
        for (int bt = 0; bt < maxback; ++bt) {
          double es = 0.0;
          for (int j = 0; j < k; ++j) { double yn = fmax(yk[j] + tau * dk[j], 0.0); if (j == p) yn = 1.0; ln[j] = yn; es = fma(ek[j], yn, es); }
          ln[p] = 1.0 - es;
          bool accept = false;
          if (ln[p] >= 0.0) {
            if (cf.line_search) {
              double fs2 = 0.0, cl2 = 0.0;
              for (int e = 0; e < n; ++e) { double a = 0.0; for (int j = 0; j < k; ++j) a = fma(G[j][e], ln[j], a); fs2 += softplus_s(a); }
              for (int j = 0; j < k; ++j) cl2 = fma(c[j], ln[j], cl2);
              accept = (fs2 - cl2) < F + tau * 1e-5 * dg;
            } else accept = true;
          }
          if (accept) break;
          if (rl ? (tau * dmax < 1e-10) : (tau < 1e-10)) { ret_now = true; break; }
          tau *= 0.5;
        }
        for (int j = 0; j < k; ++j) z[j] = ln[j];
        if (ret_now) done = true;
      }
    }
    for (int e = 0; e < n; ++e) {
      double a = 0.0;
      for (int j = 0; j < k; ++j) a = fma(G[j][e], z[j], a);
      ynew[e] = 1.0 / (1.0 + exp(a));
    }
  }

  // ---- commit ----
  const bool rl = (cf.variant == ICNN_VARIANT_RL);
  double maxdiff = 0.0;
  bool nf_bad = false;
  for (int e = 0; e < n; ++e) {
    double ye = ynew[e];
    if (rl) ye = fmin(fmax(ye, 0.03), 0.97);
    nf_bad |= !isfinite(ye);
    maxdiff = fmax(maxdiff, fabs(y[e] - ye));
    yu[e] = ye;
    b.y32[(size_t)u * n + e] = (float)ye;
  }
  int nk = 0, nd = 0, dropped[KM];
  for (int j = 0; j < k; ++j) {
    if (z[j] > cf.prune_thr) { permu[nk++] = sl[j]; lamu[sl[j]] = z[j]; }
    else dropped[nd++] = sl[j];
  }
  for (int j = 0; j < nd; ++j) permu[nk + j] = dropped[j];
  b.count[u] = nk;
  int fin = 0, stt = ICNN_ST_RUNNING;
  if (fail || b.status[u] == ICNN_ST_SOLVE_FAIL) stt = ICNN_ST_SOLVE_FAIL;   // sticky: an earlier failed inner solve stays visible
  if (nf_bad) { stt = ICNN_ST_NONFINITE; fin = 1; }
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

bool bundle_step_small_ok(int n, int KS) { return n <= NM && KS <= KM; }

int bundle_step_small_launch(const icnn_bundle_cfg* cfg, const icnn_bundle_bufs* b, int t, cudaStream_t st) {
  SmallArgs a;
  a.b = *b; a.c = *cfg; a.t = t;
  bundle_step_small_kernel<<<cdiv(b->B, 128), 128, 0, st>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_error("bundle_step_small launch: %s", cudaGetErrorString(e)); return ICNN_E_CUDA; }
  return ICNN_OK;
}

}  // namespace icnn
