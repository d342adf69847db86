// K3: argmin differentiation (see bundle_step_kernel.cuh for the shared group / G-pass helpers).
#include "bundle_step_kernel.cuh"

namespace icnn {

// ---- K3: argmin differentiation ---------------------------------------------------------------
// Differentiates y* through the KKT system of the final bundle model (SURVEY.md section 8f row 1):
//   crossEntrGrad  multi-label-cls/icnn_ebundle.py:390-417   (loss 1)
//   mseGrad        completion/icnn_ebundle.py:493-522          (loss 0)
// and assembles the per-bundle-point pairs of train_step_fd (multi-label-cls/icnn_ebundle.py:296-314):
//   v_i = lam_i * cy + clam_i * (yN - ys_i),  c_i = clam_i.
// Same group-per-sample decomposition and the same G passes as the bundle step.

// general (k+1)x(k+1) solve, LU with partial pivoting (np.linalg.solve), one warp, in place
__device__ inline bool warp_lu_solve(double* A, int m, int ld, double* rhs, int lane) {
  for (int c = 0; c < m; ++c) {
    double best = -1.0; int bi = c;
    for (int r = c + lane; r < m; r += 32) { const double v = fabs(A[r * ld + c]); if (v > best) { best = v; bi = r; } }
    for (int o = 16; o > 0; o >>= 1) {
      const double ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if (!(best > 0.0) || !isfinite(best)) return false;
    if (bi != c) {
      for (int j = lane; j < m; j += 32) { const double t = A[c * ld + j]; A[c * ld + j] = A[bi * ld + j]; A[bi * ld + j] = t; }
      if (lane == 0) { const double t = rhs[c]; rhs[c] = rhs[bi]; rhs[bi] = t; }
    }
    __syncwarp();
    const double piv = A[c * ld + c];
    const double rc = rhs[c];
    for (int r = c + 1 + lane; r < m; r += 32) {
      const double f = A[r * ld + c] / piv;
      for (int j = c + 1; j < m; ++j) A[r * ld + j] = fma(-f, A[c * ld + j], A[r * ld + j]);
      rhs[r] = fma(-f, rc, rhs[r]);
    }
    __syncwarp();
  }
  for (int i = m - 1; i >= 0; --i) {
    const double xi = rhs[i] / A[i * ld + i];
    __syncwarp();
    for (int r = lane; r < i; r += 32) rhs[r] = fma(-A[r * ld + i], xi, rhs[r]);
    if (lane == 0) rhs[i] = xi;
    __syncwarp();
  }
  return true;
}

struct GradArgs {
  icnn_bundle_bufs b;
  int loss;  // 0 mse, 1 cross-entropy
  const double* trueY;
  double* cy; double* clam; double* ct; double* V;
  int npad, ld;
};

template <int WPS>
__global__ void __launch_bounds__(256, 2) argmin_grad_kernel(GradArgs A) {
  const icnn_bundle_bufs& b = A.b;
  extern __shared__ __align__(16) double smem_d[];
  constexpr int GPB = 8 / WPS;
  constexpr int T = WPS * 32;
  Grp<WPS, 1> g;
  g.tid = threadIdx.x % T; g.lane = threadIdx.x & 31; g.warp = g.tid >> 5; g.gid = threadIdx.x / T;
  const int u = blockIdx.x * GPB + g.gid;
  if (u >= b.B) return;
  const int n = b.n, KS = b.KS, ld = A.ld, npad = A.npad;
  const int KA = KS + 1;
  double* base = smem_d + (size_t)g.gid * (((size_t)3 * npad + (size_t)2 * KA * ld + 4 * KA + 4 * WPS + 8 + 1) & ~(size_t)1);
  double* yv = base; double* rv = yv + npad; double* dv = rv + npad;
  double* M = dv + npad; double* Am = M + (size_t)KA * ld;
  double* bk = Am + (size_t)KA * ld; double* lamk = bk + KA; double* clk = lamk + KA;
  const float** rowp = reinterpret_cast<const float**>(clk + KA);
  g.red = reinterpret_cast<double*>(rowp + KA) ; g.xb = nullptr;
  int* flag = reinterpret_cast<int*>(g.red + 4 * WPS);

  const int k = b.count[u];
  const int* permu = b.perm + (size_t)u * KS;
  const double* yu = b.y + (size_t)u * n;
  const double* tu = A.trueY + (size_t)u * n;
  double* cyu = A.cy + (size_t)u * n;
  if (k == 0) {
    for (int e = g.tid; e < n; e += T) cyu[e] = 0.0;
    if (g.tid == 0) A.ct[u] = 0.0;
    return;
  }
  for (int j = g.tid; j < k; j += T) { rowp[j] = b.G + ((size_t)u * KS + permu[j]) * n; lamk[j] = b.lam[(size_t)u * KS + permu[j]]; }
  for (int e = g.tid; e < n; e += T) {
    const double y = yu[e], ty = tu[e];
    double y_, dl;
    if (A.loss == 1) { y_ = fmin(fmax(y, 1e-8), 1.0 - 1e-8); dl = ty / y_ - (1.0 - ty) / (1.0 - y_); }
    else { y_ = y; dl = -(y - ty); }
    yv[e] = y;
    dv[e] = 1.0 / (1.0 / y_ + 1.0 / (1.0 - y_));   // zinv
    rv[e] = dl;
  }
  g.sync();
  // b = G (zinv o dl) ; M = G diag(zinv) G^T
  for (int j = g.warp; j < k; j += WPS) {
    const float* rj = rowp[j];
    double acc = 0.0;
    for (int e = g.lane; e < n; e += 32) acc = fma((double)ldf(rj + e), dv[e] * rv[e], acc);
    acc = Grp<WPS>::wsum(acc);
    if (g.lane == 0) bk[j] = acc;
  }
  gram_pass<WPS>(g, rowp, k, n, dv, M, ld, g.warp, WPS);
  g.sync();
  if (g.warp == 0) {
    const int lane = g.lane, m = k + 1;
    for (int i = lane; i < m; i += 32)
      for (int j = 0; j < m; ++j)
        Am[i * ld + j] = (i < k && j < k) ? M[i * ld + j] : ((i == k && j == k) ? 0.0 : 1.0);
    if (lane == 0) bk[k] = 0.0;
    __syncwarp();
    const bool ok = warp_lu_solve(Am, m, ld, bk, lane);
    if (lane == 0) flag[0] = ok ? 0 : 1;
    __syncwarp();
  }
  g.sync();
  if (flag[0]) {   // singular KKT system: the reference raises LinAlgError; report NaNs
    for (int e = g.tid; e < n; e += T) cyu[e] = nan("");
    if (g.tid == 0) A.ct[u] = nan("");
    return;
  }
  for (int j = g.tid; j < k; j += T) { clk[j] = bk[j]; A.clam[(size_t)u * KS + j] = bk[j]; }
  if (g.tid == 0) A.ct[u] = bk[k];
  g.sync();
  // cy = zinv o dl - (G o zinv)^T clam ; zero where y is exactly 0 or 1
  col_pass<T>(rowp, k, n, g.tid, clk, [&](int e, double a) {
    const double y = yv[e];
    double c = dv[e] * rv[e] - dv[e] * a;
    if (y == 0.0 || y == 1.0) c = 0.0;
    cyu[e] = c;
    rv[e] = c;
  });
  g.sync();
  if (A.V != nullptr && b.ys != nullptr) {
    for (int i = 0; i < k; ++i) {
      const double li = lamk[i], ci = clk[i];
      const double* ysi = b.ys + ((size_t)u * KS + permu[i]) * n;
      double* Vi = A.V + ((size_t)u * KS + i) * n;
      for (int e = g.tid; e < n; e += T) Vi[e] = li * rv[e] + ci * (yv[e] - ysi[e]);
    }
  }
}

int argmin_grad_launch(const icnn_bundle_bufs* b, int loss, const double* trueY, double* cy, double* clam,
                       double* ct, double* V, cudaStream_t st) {
  GradArgs a;
  a.b = *b; a.loss = loss; a.trueY = trueY; a.cy = cy; a.clam = clam; a.ct = ct; a.V = V;
  a.npad = (b->n + 3) & ~3;
  a.ld = (b->KS + 1) | 1;
  const int n = b->n;
  int wps = n <= 128 ? 1 : (n <= 512 ? 2 : (n <= 1024 ? 4 : 8));
  const int KA = b->KS + 1;
  auto smem_of = [&](int w) {
    return sizeof(double) * ((((size_t)3 * a.npad + (size_t)2 * KA * a.ld + 4 * KA + 4 * w + 8 + 1) & ~(size_t)1)) * (8 / w);
  };
  // 8 / wps samples share a CTA: when their k x k systems do not fit side by side (large KS at small n_y), the
  // sample gets more warps and the CTA fewer samples
  while (wps < 8 && smem_of(wps) > 227 * 1024) wps *= 2;
  const size_t smem = smem_of(wps);
  if (smem > 227 * 1024) { set_error("argmin_grad: shared memory %zu B exceeds 227 KB", smem); return ICNN_E_UNSUPPORTED; }
  void (*kern)(GradArgs) = wps == 1 ? argmin_grad_kernel<1> : wps == 2 ? argmin_grad_kernel<2> : wps == 4 ? argmin_grad_kernel<4> : argmin_grad_kernel<8>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) { set_error("argmin_grad smem attr: %s", cudaGetErrorString(e)); return ICNN_E_CUDA; }
  kern<<<cdiv(b->B, 8 / wps), 256, smem, st>>>(a);
  e = cudaGetLastError();
  if (e != cudaSuccess) { set_error("argmin_grad launch: %s", cudaGetErrorString(e)); return ICNN_E_CUDA; }
  return ICNN_OK;
}

}  // namespace icnn
