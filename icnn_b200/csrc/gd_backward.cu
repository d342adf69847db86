// d loss / d theta through the unrolled momentum-GD inner loop (SURVEY.md section 8f row 4).
//
// Replaces what TensorFlow's double backprop evaluates for
//   opt.compute_gradients(self.mse_, self.theta_)        multi-label-cls/icnn-back.py:120-139
//                                                        completion/icnn.back.py:133-156
// on the graph that unrolls nIter steps  v' = m v - lr dE/dy(y),  y' = y - m v + (1+m) v'.
//
// The ReLU / leaky-ReLU energy is piecewise linear in y, so the Hessian term vanishes and the
// adjoint of every gradient evaluation g_i is kappa_i * a with a = dl/dy_N and
//   c_N = 1+m, c_i = m c_{i+1} + 1, kappa_i = -lr c_{i+1}.
// dl/dtheta = sum_i kappa_i d/dtheta <g_i, a>; with iterate i's activation pattern fixed, <g_i, a> is
// the output of the linear tangent network  zt_l = act'(pre_l) o ((zt_{l-1} o cz_l) Wz_l + (a o cy_l) Wy_l)
// whose backprop multipliers are the primal delta_l (derivation and torch-autograd pin:
// oracle/gd_grad_np.py, tests/test_oracle_gd_grad.py).  Per layer l:
//   dWy_l = (a o cy_l)^T Delta_l,  dcy_l = a o (Delta_l Wy_l^T),   Delta_l = sum_i kappa_i delta_l^(i)
//   dWz_l = sum_i kappa_i (zt_{l-1}^(i) o cz_l)^T delta_l^(i)
//   dcz_l = sum_i kappa_i zt_{l-1}^(i) o (delta_l^(i) Wz_l^T)
//
// Single-pass mode (tensor-core path, stores within ICNN_GDB_STORE_GB): the GD loop runs once; the
// GDB epilogues of tc_gemm_kernel keep Z_l^(i), delta_l^(i) and delta_l^(i) Wz_l^T of every iteration
// in HBM and accumulate Delta_l (kappa does not depend on a).  With a known, Ty_l = (a o cy_l) Wy_l is
// iteration-independent, zt_0^(i) = act'(Z_0^(i)) o Ty_0 is elementwise, and per hidden layer ONE
// wgmma GEMM over all iterations (M = nIter*B) gives zt_l, ONE weight-gradient GEMM (K = nIter*B)
// gives dWz_l, and tangent_stage_kernel reduces dcz_l over the iterations.
// Two-pass mode (fallback; also the FP32 FFMA path for B < 64): pass 1 -> y_N, pass 2 replays the
// deterministic loop (bit-identical iterates) with, per iteration, the tangent forward (the same
// gated product with the activation pattern of the primal Z_l), the dcz / Delta accumulation fused
// into the backward epilogue, and one weight-gradient GEMM per Wz_l.
// The weight-gradient GEMMs are wgrad.cuh's (FP32 FFMA, rows split over CTAs and the parts summed in a
// fixed order: no atomics, deterministic); their partial tiles go to GdbLayout::wpart.
#include "gated_gemm.cuh"
#include "gdb.cuh"
#include "wgrad.cuh"

#include <cstdlib>
#include <vector>

namespace icnn {

size_t picnn_simt_ws_floats(const icnn_picnn* h, int B, size_t* zoff, size_t* doff);
size_t picnn_gdb_tc_ws_floats(const icnn_picnn* h, int B, GdbTcBufs* b, float* base);
void picnn_gdb_tc_gate_a(const icnn_picnn* h, const icnn_gates* gt, const float* a, const GdbTcBufs& b, cudaStream_t st);
int picnn_gdb_tc_forward(const icnn_picnn* h, const icnn_gates* gt, const GdbTcBufs& b, bool tangent, cudaStream_t st);
int picnn_gdb_tc_backward_layer(const icnn_picnn* h, const icnn_gates* gt, const GdbTcBufs& b, int i, int cur,
                                cudaStream_t st);
int picnn_gdb_tc_stored_tangent(const icnn_picnn* h, int l, long long M, int B, const float* P_hi, const float* P_lo,
                                const float* Ty, const float* Zs, float* Zt, cudaStream_t st);
void out_layer_launch(const icnn_picnn* h, const icnn_gates* gt, const float* Zlast, const float* y32, float* f,
                      float* delta, float* delta_hi, float* delta_lo, float* g, long long g_row_stride,
                      const int* perm, const int* count, int KS, const int* skip, cudaStream_t st);

// dst[r, j] += c[r] * src[r, j]
__global__ void row_axpy_kernel(float* dst, const float* src, const float* c, long long N, int w) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < N) dst[i] = fmaf(c[i / w], src[i], dst[i]);
}

void launch_row_axpy(float* dst, const float* src, const float* c, long long rows, int w, cudaStream_t st) {
  const long long N = rows * w;
  if (N > 0) row_axpy_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(dst, src, c, N, w);
}

// dst += kappa * src
__global__ void axpy_kernel(float* dst, const float* src, float kappa, long long N) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < N) dst[i] = fmaf(kappa, src[i], dst[i]);
}
// dst[b, j] += kappa * rs[b] * src[b, j] * w[j]   (rs == nullptr: 1)
__global__ void rowbcast_fma_kernel(float* dst, const float* src, const float* w, const float* rs, float kappa,
                                    long long N, int width) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < N) dst[i] = fmaf((rs ? kappa * rs[i / width] : kappa) * src[i], w[i % width], dst[i]);
}
// a = scale * (y - trueY)      (d/dy_N of scale/2 * sum (y_N - trueY)^2)
__global__ void mse_grad_kernel(float* a, const float* y, const float* trueY, float scale, long long N) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < N) a[i] = scale * (y[i] - trueY[i]);
}

// Stored-pattern phase, per (sample b, unit j of layer l-1), looping over the nIter stored iterations:
//   zt_i = zt_{l-1}^(i)[b, j]   (layer 0: act'(Zs_0^(i)) * Ty_0, later layers: read from Zt_st)
//   hidden layer l:  dcz_l[b, j] = sum_i kappa_i zt_i As_l^(i)[b, j];   P^(i)[b, j] = zt_i cz_l[b, j]
//                    (TF32 hi/lo operand of the batched tangent GEMM, and kappa_i * P plain for the
//                    batched weight-gradient GEMM)
//   output layer:    S[b, j] = sum_i kappa_i zt_i;   dcz_L[b, j] = S wz_L[j]
struct StageArgs {
  int B, S, nIter; float alpha;
  const float* kappa;        // device [nIter]
  const float* Zs; const float* Ty;   // on-the-fly zt (layer 0) when Zt_st == nullptr
  const float* Zt_st;
  const float* As;           // hidden layer: stored delta_l Wz_l^T; nullptr = output layer
  const float* cz; const float* wz;
  float* dcz; float* Sout;
  float* P_hi; float* P_lo; int ldp; float* Pk;
};
__global__ void tangent_stage_kernel(StageArgs a) {
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long BS = (long long)a.B * a.S;
  if (idx >= BS) return;
  const int b = (int)(idx / a.S), j = (int)(idx % a.S);
  const float ty = a.Zt_st ? 0.f : a.Ty[idx];
  const float czv = a.cz ? a.cz[idx] : 0.f;
  float acc = 0.f;
  for (int i = 0; i < a.nIter; ++i) {
    const long long off = (long long)i * BS + idx;
    const float zt = a.Zt_st ? a.Zt_st[off] : (a.Zs[off] > 0.f ? 1.f : a.alpha) * ty;
    const float k = a.kappa[i];
    if (a.As) {
      acc = fmaf(k * zt, a.As[off], acc);
      const float p = zt * czv;
      const float h = tf32_rn(p);
      const long long o = ((long long)i * a.B + b) * a.ldp + j;
      a.P_hi[o] = h;
      a.P_lo[o] = tf32_rn(p - h);
      a.Pk[off] = k * p;
    } else {
      acc = fmaf(k, zt, acc);
    }
  }
  if (a.As) a.dcz[idx] = acc;
  else { a.dcz[idx] = acc * a.wz[j]; a.Sout[idx] = acc; }
}

// tensor-core GEMMs (3xTF32) for the forward / tangent / backward products once a 128-row tile fills;
// ICNN_GDB=simt keeps the FP32 FFMA kernels
bool gdb_use_tc(const icnn_picnn* h, int B) {
  const char* v = getenv("ICNN_GDB");
  return h->use_tc && B >= 64 && !(v && v[0] == 's');
}

// Single pass with the activation patterns, deltas and pre-gating products of every iteration kept in
// HBM (then every iteration-independent product is hoisted and the rest is batched over the
// iterations) when that store fits ICNN_GDB_STORE_GB (default 24) GiB; ICNN_GDB=twopass disables it.
static bool gdb_want_stored(const icnn_picnn* h, int B, int nIter, size_t store_floats) {
  const char* v = getenv("ICNN_GDB");
  if (!gdb_use_tc(h, B) || nIter < 1 || (v && v[0] == 't')) return false;
  double cap = 24.0;
  if (const char* c = getenv("ICNN_GDB_STORE_GB")) cap = atof(c);
  return (double)store_floats * 4.0 <= cap * 1073741824.0;
}

GdbLayout gdb_layout(const icnn_picnn* h, int B, int nIter) {
  GdbLayout lo{};
  size_t off = 0;
  auto take = [&](size_t nfl) { size_t o = off; off += (nfl + 63) & ~(size_t)63; return o; };
  int smax = 0;
  for (int i = 0; i < h->L; ++i) smax = h->hidden[i] > smax ? h->hidden[i] : smax;
  for (int i = 0; i < h->L; ++i) {
    lo.Z[i] = take((size_t)B * h->hidden[i]);
    lo.Zt[i] = take((size_t)B * h->hidden[i]);
    lo.Dacc[i] = take((size_t)B * h->hidden[i]);
  }
  lo.dl[0] = take((size_t)B * smax); lo.dl[1] = take((size_t)B * smax);
  lo.y = take((size_t)B * h->n); lo.v = take((size_t)B * h->n); lo.g = take((size_t)B * h->n);
  lo.a = take((size_t)B * h->n); lo.f = take((size_t)B);
  lo.wpart = take(wgrad_part_bytes() / sizeof(float));
  lo.tc = off;
  lo.use_tc = gdb_use_tc(h, B);
  if (lo.use_tc) off += picnn_gdb_tc_ws_floats(h, B, nullptr, nullptr);
  {
    const size_t base = off, R = (size_t)(nIter > 0 ? nIter : 1) * B;
    int spmax = 1;
    for (int i = 1; i <= h->L; ++i) spmax = h->prev(i) > spmax ? h->prev(i) : spmax;
    lo.kap = take((size_t)(nIter > 0 ? nIter : 1));
    for (int i = 0; i < h->L; ++i) {
      lo.Zs[i] = take(R * h->hidden[i]);
      lo.Ds[i] = take(R * h->hidden[i]);
      lo.Ty[i] = take((size_t)B * h->hidden[i]);
      if (i > 0) { lo.As[i] = take(R * h->prev(i)); lo.Zts[i] = take(R * h->hidden[i]); }
    }
    lo.P_hi = take(R * ld4(spmax)); lo.P_lo = take(R * ld4(spmax)); lo.Pk = take(R * spmax);
    lo.Sout = take((size_t)B * h->hidden[h->L - 1]);
    lo.stored = gdb_want_stored(h, B, nIter, off - base);
    if (!lo.stored) off = base;
  }
  lo.total = off;
  return lo;
}

#define GDB_LAUNCH(expr, what)                                                                   \
  do {                                                                                           \
    cudaError_t _le = (expr);                                                                    \
    if (_le != cudaSuccess) { set_error("%s launch: %s", what, cudaGetErrorString(_le)); return ICNN_E_CUDA; } \
  } while (0)

// The buffers of the tensor-core GEMMs of one iteration, with the optional epilogue accumulations / stores.
static GdbTcBufs gdb_tc_bufs(const icnn_picnn* h, const icnn_gates* gt, float* ws, const GdbLayout& lo,
                             const GdbAcc* acc, int store_it, float store_kappa) {
  const int B = gt->B, L = h->L;
  GdbTcBufs tb{};
  tb.y = ws + lo.y; tb.g = ws + lo.g; tb.dp[0] = ws + lo.dl[0]; tb.dp[1] = ws + lo.dl[1];
  const bool primal_op = acc && acc->dL;   // td_grad: the accumulations take Z_l where the tangent pass takes Zt_l
  for (int i = 0; i < L; ++i) {
    tb.Z[i] = ws + lo.Z[i]; tb.Zt[i] = ws + (primal_op ? lo.Z[i] : lo.Zt[i]); tb.Dacc[i] = ws + lo.Dacc[i];
  }
  if (acc) {
    tb.want_plain = true; tb.acc_delta = true; tb.kappa = acc->kappa;
    for (int i = 1; i < L; ++i) tb.dcz[i] = acc->gr->dcz[i];
  }
  if (store_it >= 0) {
    tb.want_plain = true; tb.acc_delta = true; tb.kappa = store_kappa;
    for (int i = 0; i < L; ++i) {
      const size_t r = (size_t)store_it * B;
      tb.Z[i] = ws + lo.Zs[i] + r * h->hidden[i];
      tb.dstore[i] = ws + lo.Ds[i] + r * h->hidden[i];
      if (i > 0) tb.astore[i] = ws + lo.As[i] + r * h->prev(i);
    }
  }
  picnn_gdb_tc_ws_floats(h, B, &tb, ws + lo.tc);
  return tb;
}

// One GD iteration's primal forward + backward.  acc != nullptr: also the tangent forward and the
// gradient accumulations (pass 2 of the two-pass mode).  store_it >= 0 (stored-pattern mode, tensor-core
// path only): the primal pass writes Z_l, delta_l and delta_l Wz_l^T of this iteration into the stores
// and accumulates Delta_l += kappa delta_l.  (GdbAcc: gdb.cuh)
int gdb_iteration(const icnn_picnn* h, const icnn_gates* gt, float* ws, const GdbLayout& lo,
                  const GdbAcc* acc, int store_it, float store_kappa, cudaStream_t st) {
  const int rc = gdb_forward(h, gt, ws, lo, acc, store_it, store_kappa, st);
  return rc ? rc : gdb_backward(h, gt, ws, lo, acc, store_it, store_kappa, st);
}

int gdb_forward(const icnn_picnn* h, const icnn_gates* gt, float* ws, const GdbLayout& lo, const GdbAcc* acc,
                int store_it, float store_kappa, cudaStream_t st) {
  const int B = gt->B, n = h->n, L = h->L;
  float* y = ws + lo.y; float* g = ws + lo.g; float* f = ws + lo.f; float* av = ws + lo.a;
  const bool tangent = acc && !acc->dL;
  GdbTcBufs tb{};
  if (lo.use_tc) {
    tb = gdb_tc_bufs(h, gt, ws, lo, acc, store_it, store_kappa);
    int rc = picnn_gdb_tc_forward(h, gt, tb, tangent, st);
    if (rc) return rc;
  }
  for (int i = 0; i < L && !lo.use_tc; ++i) {
    GemmArgs a{};
    a.M = B; a.N = h->hidden[i]; a.K0 = h->prev(i); a.K1 = n;
    a.A0 = i ? ws + lo.Z[i - 1] : nullptr; a.G0 = i ? gt->cz[i] : nullptr; a.lda0 = a.K0;
    a.A1 = y; a.G1 = gt->cy[i]; a.lda1 = n; a.a1_scale = 1.f; a.a1_shift = 0.f;
    a.W = h->Wcat[i]; a.ldw = a.N; a.D = gt->d[i]; a.Z = ws + lo.Z[i]; a.alpha = h->alpha;
    GDB_LAUNCH(launch_gemm<0>(a, st), "gd_backward forward");
    if (tangent) {   // tangent layer: same product on (zt_{i-1}, a), pattern of Z_i, no bias
      a.A0 = i ? ws + lo.Zt[i - 1] : nullptr; a.A1 = av; a.D = nullptr;
      a.Zmask = ws + lo.Z[i]; a.Z = ws + lo.Zt[i];
      GDB_LAUNCH(launch_gemm<2>(a, st), "gd_backward tangent");
    }
  }
  if (acc && acc->c)   // train_grad: the backward accumulates with c o Z_l + Zt_l in place of the tangent
    for (int i = 0; i < L; ++i) launch_row_axpy(ws + lo.Zt[i], ws + lo.Z[i], acc->c, B, h->hidden[i], st);
  float* dlast = store_it >= 0 ? tb.dstore[L - 1] : ws + lo.dl[0];     // plain delta_{L-1}
  out_layer_launch(h, gt, lo.use_tc ? tb.Z[L - 1] : ws + lo.Z[L - 1], y, f, dlast, lo.use_tc ? tb.dh[0] : nullptr,
                   lo.use_tc ? tb.dl[0] : nullptr, g, n, nullptr, nullptr, 0, nullptr, st);
  return ICNN_OK;
}

int gdb_backward(const icnn_picnn* h, const icnn_gates* gt, float* ws, const GdbLayout& lo, const GdbAcc* acc,
                 int store_it, float store_kappa, cudaStream_t st) {
  const int B = gt->B, L = h->L;
  float* g = ws + lo.g;
  float* dl[2] = {ws + lo.dl[0], ws + lo.dl[1]};
  GdbTcBufs tb{};
  if (lo.use_tc) tb = gdb_tc_bufs(h, gt, ws, lo, acc, store_it, store_kappa);
  // the backward's accumulation operand of layer i: the tangent Zt_i, or with GdbAcc::dL the primal Z_i
  auto zt = [&](int i) { return ws + (acc && acc->dL ? lo.Z[i] : lo.Zt[i]); };
  const int sl = h->hidden[L - 1];
  const long long NL = (long long)B * sl;
  if (store_it >= 0) axpy_kernel<<<(unsigned)((NL + 255) / 256), 256, 0, st>>>(ws + lo.Dacc[L - 1], tb.dstore[L - 1],
                                                                                store_kappa, NL);
  if (acc) {
    const float kp = acc->kappa;
    axpy_kernel<<<(unsigned)((NL + 255) / 256), 256, 0, st>>>(ws + lo.Dacc[L - 1], dl[0], kp, NL);
    rowbcast_fma_kernel<<<(unsigned)((NL + 255) / 256), 256, 0, st>>>(acc->gr->dcz[L], zt(L - 1), h->Wcat[L], acc->dL,
                                                                      kp, NL, sl);
    WgradArgs w{};   // dWz_L [s_{L-1}, 1] += kappa * sum_b zt_{L-1} o cz_L delta_L   (delta_L = 1, or dL[b])
    w.M = sl; w.N = 1; w.Kb = B; w.A = zt(L - 1); w.G = gt->cz[L]; w.lda = sl; w.D = acc->dL; w.ldd = 1;
    w.C = acc->gr->dWz[L]; w.ldc = 1; w.kappa = kp; w.C64 = acc->w64 ? acc->w64->dWz[L] : nullptr;
    w.part = ws + lo.wpart;
    GDB_LAUNCH(launch_wgrad(w, st), "gd_backward wgrad(L)");
  }
  int cur = 0;
  for (int i = L - 1; i >= 0; --i) {
    if (acc && i > 0) {   // dWz_i += kappa (zt_{i-1} o cz_i)^T delta_i
      WgradArgs w{};
      w.M = h->prev(i); w.N = h->hidden[i]; w.Kb = B; w.A = zt(i - 1); w.G = gt->cz[i]; w.lda = w.M;
      w.D = dl[cur]; w.ldd = w.N; w.C = acc->gr->dWz[i]; w.ldc = w.N; w.kappa = acc->kappa;
      w.C64 = acc->w64 ? acc->w64->dWz[i] : nullptr; w.part = ws + lo.wpart;
      GDB_LAUNCH(launch_wgrad(w, st), "gd_backward wgrad");
    }
    if (lo.use_tc) {
      int rc = picnn_gdb_tc_backward_layer(h, gt, tb, i, cur, st);
      if (rc) return rc;
      cur ^= 1;
      continue;
    }
    GemmArgs a{};
    a.M = B; a.N0 = h->prev(i); a.N = a.N0 + h->n; a.K0 = h->hidden[i]; a.K1 = 0;
    a.A0 = dl[cur]; a.lda0 = a.K0; a.W = h->Wcat[i]; a.ldw = a.K0; a.alpha = h->alpha;
    a.Zprev = i ? ws + lo.Z[i - 1] : nullptr; a.Cz = i ? gt->cz[i] : nullptr; a.dprev = dl[cur ^ 1];
    a.Cy = gt->cy[i]; a.g = g; a.g_row_stride = h->n; a.n = h->n; a.g_scale = 1.f;
    if (acc && i > 0) {
      a.dCz = acc->gr->dcz[i]; a.Ztprev = zt(i - 1); a.Dacc = ws + lo.Dacc[i - 1]; a.kappa = acc->kappa;
    }
    GDB_LAUNCH(launch_gemm<1>(a, st), "gd_backward backward");
    cur ^= 1;
  }
  return ICNN_OK;
}

int gdb_ygate_stage(const icnn_picnn* h, const icnn_gates* gt, float* ws, const GdbLayout& lo, const float* av,
                    const icnn_gd_grads* gr, float ksum, const GdbW64* w64, const float* dL, cudaStream_t st) {
  const int B = gt->B, n = h->n, L = h->L;
  const long long N = (long long)B * n;
  for (int l = 0; l < L; ++l) {
    WgradArgs w{};
    w.M = n; w.N = h->hidden[l]; w.Kb = B; w.A = av; w.G = gt->cy[l]; w.lda = n;
    w.D = ws + lo.Dacc[l]; w.ldd = w.N; w.C = gr->dWy[l]; w.ldc = w.N; w.kappa = 1.f;
    w.C64 = w64 ? w64->dWy[l] : nullptr; w.part = ws + lo.wpart;
    GDB_LAUNCH(launch_wgrad(w, st), "gd_backward wgrad(Wy)");
    GemmArgs a{};   // dcy_l = a o (Delta_l Wy_l^T): the backward GEMM against the Wy rows of Wcat_l
    a.M = B; a.N0 = 0; a.N = n; a.K0 = h->hidden[l]; a.K1 = 0; a.A0 = ws + lo.Dacc[l]; a.lda0 = a.K0;
    a.W = h->Wcat[l] + (size_t)h->prev(l) * h->hidden[l]; a.ldw = a.K0; a.alpha = h->alpha;
    a.Cy = av; a.g = gr->dcy[l]; a.g_row_stride = n; a.n = n; a.g_scale = 1.f;
    GDB_LAUNCH(launch_gemm<1>(a, st), "gd_backward dcy");
  }
  // output layer: Delta_L = ksum for every row (times dL[row] when given)
  WgradArgs w{};
  w.M = n; w.N = 1; w.Kb = B; w.A = av; w.G = gt->cy[L]; w.lda = n; w.D = dL; w.ldd = 1;
  w.C = gr->dWy[L]; w.ldc = 1; w.kappa = ksum; w.C64 = w64 ? w64->dWy[L] : nullptr; w.part = ws + lo.wpart;
  GDB_LAUNCH(launch_wgrad(w, st), "gd_backward wgrad(Wy_L)");
  rowbcast_fma_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(gr->dcy[L], av, h->Wcat[L] + h->hidden[L - 1], dL,
                                                                  ksum, N, n);
  return ICNN_OK;
}

}  // namespace icnn

using namespace icnn;

extern "C" size_t icnn_gd_backward_workspace_bytes(const icnn_picnn_t* h, int32_t B, int32_t nIter) {
  if (!h || B <= 0 || nIter < 0) return 0;
  return sizeof(float) * gdb_layout(h, B, nIter).total;
}

extern "C" int icnn_gd_backward(const icnn_picnn_t* h, const icnn_gates* gates, const float* y0,
                                const float* trueY, float loss_scale, int32_t nIter, float lr, float momentum,
                                float* yN, const icnn_gd_grads* gr, void* workspace, void* stream) {
  ICNN_REQUIRE(h && gates && y0 && trueY && yN && gr && workspace, "null pointer");
  ICNN_REQUIRE(gates->B > 0 && nIter >= 0, "empty batch or nIter < 0");
  if (gates->in_scale != 1.f || gates->in_shift != 0.f || gates->g_scale != 1.f) {
    set_error("icnn_gd_backward: the affine (RL) input wrapper is not on this path");
    return ICNN_E_UNSUPPORTED;
  }
  const int B = gates->B, n = h->n, L = h->L;
  for (int l = 0; l <= L; ++l)
    ICNN_REQUIRE(gr->dWy[l] && gr->dcy[l] && (l == 0 || (gr->dWz[l] && gr->dcz[l])), "null gradient buffer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const GdbLayout lo = gdb_layout(h, B, nIter);
  float* ws = static_cast<float*>(workspace);
  const long long N = (long long)B * n;
  const unsigned gN = (unsigned)((N + 255) / 256);

  // adjoint weights of the nIter gradient evaluations
  std::vector<float> kappa(nIter > 0 ? nIter : 1, 0.f);
  const double ksum = gd_kappa(nIter, lr, momentum, kappa.data());

  // outputs and accumulators start from zero
  for (int l = 0; l <= L; ++l) {
    const size_t sl = (size_t)h->width(l), sp = (size_t)h->prev(l);
    ICNN_CUDA_CHECK(cudaMemsetAsync(gr->dWy[l], 0, sizeof(float) * n * sl, st));
    ICNN_CUDA_CHECK(cudaMemsetAsync(gr->dcy[l], 0, sizeof(float) * N, st));
    if (l > 0) {
      ICNN_CUDA_CHECK(cudaMemsetAsync(gr->dWz[l], 0, sizeof(float) * sp * sl, st));
      ICNN_CUDA_CHECK(cudaMemsetAsync(gr->dcz[l], 0, sizeof(float) * (size_t)B * sp, st));
    }
    if (l < L) ICNN_CUDA_CHECK(cudaMemsetAsync(ws + lo.Dacc[l], 0, sizeof(float) * (size_t)B * sl, st));
  }

  const float* av = ws + lo.a;
  if (lo.stored) {
    // ---- single pass: the GD loop with per-iteration stores, then the batched tangent phase ----
    // (pageable source: the call returns once kappa has been staged, so the vector may go out of scope)
    ICNN_CUDA_CHECK(cudaMemcpyAsync(ws + lo.kap, kappa.data(), sizeof(float) * nIter, cudaMemcpyHostToDevice, st));
    ICNN_CUDA_CHECK(cudaMemcpyAsync(ws + lo.y, y0, sizeof(float) * N, cudaMemcpyDeviceToDevice, st));
    ICNN_CUDA_CHECK(cudaMemsetAsync(ws + lo.v, 0, sizeof(float) * N, st));
    for (int it = 0; it < nIter; ++it) {
      int rc = gdb_iteration(h, gates, ws, lo, nullptr, it, kappa[it], st);
      if (rc) return rc;
      gd_update_kernel<<<gN, 256, 0, st>>>(ws + lo.y, ws + lo.v, ws + lo.g, N, lr, momentum);
    }
    ICNN_CUDA_CHECK(cudaMemcpyAsync(yN, ws + lo.y, sizeof(float) * N, cudaMemcpyDeviceToDevice, st));
    mse_grad_kernel<<<gN, 256, 0, st>>>(ws + lo.a, ws + lo.y, trueY, loss_scale, N);
    const long long R = (long long)nIter * B;
    for (int l = 0; l < L; ++l) {   // Ty_l = (a o cy_l) Wy_l: independent of the iteration
      GemmArgs a{};
      a.M = B; a.N = h->hidden[l]; a.K0 = 0; a.K1 = n; a.A1 = av; a.G1 = gates->cy[l]; a.lda1 = n;
      a.a1_scale = 1.f; a.a1_shift = 0.f; a.W = h->Wcat[l] + (size_t)h->prev(l) * h->hidden[l]; a.ldw = a.N;
      a.Zmask = nullptr; a.Z = ws + lo.Ty[l]; a.alpha = h->alpha;
      GDB_LAUNCH(launch_gemm<2>(a, st), "gd_backward Ty");
    }
    for (int l = 1; l <= L; ++l) {
      const int sp = h->prev(l);
      const long long BS = (long long)B * sp;
      StageArgs sa{};
      sa.B = B; sa.S = sp; sa.nIter = nIter; sa.alpha = h->alpha; sa.kappa = ws + lo.kap;
      if (l == 1) { sa.Zs = ws + lo.Zs[0]; sa.Ty = ws + lo.Ty[0]; } else sa.Zt_st = ws + lo.Zts[l - 1];
      sa.dcz = gr->dcz[l];
      if (l < L) {
        sa.As = ws + lo.As[l]; sa.cz = gates->cz[l];
        sa.P_hi = ws + lo.P_hi; sa.P_lo = ws + lo.P_lo; sa.ldp = ld4(sp); sa.Pk = ws + lo.Pk;
      } else {
        sa.wz = h->Wcat[L]; sa.Sout = ws + lo.Sout;
      }
      tangent_stage_kernel<<<(unsigned)((BS + 255) / 256), 256, 0, st>>>(sa);
      WgradArgs w{};
      if (l < L) {
        int rc = picnn_gdb_tc_stored_tangent(h, l, R, B, ws + lo.P_hi, ws + lo.P_lo, ws + lo.Ty[l], ws + lo.Zs[l],
                                             ws + lo.Zts[l], st);
        if (rc) return rc;
        // dWz_l = sum_i kappa_i (zt_{l-1}^(i) o cz_l)^T delta_l^(i): one GEMM with K = nIter * B
        w.M = sp; w.N = h->hidden[l]; w.Kb = (int)R; w.A = ws + lo.Pk; w.G = nullptr; w.lda = sp;
        w.D = ws + lo.Ds[l]; w.ldd = w.N; w.C = gr->dWz[l]; w.ldc = w.N; w.kappa = 1.f;
      } else {   // dWz_L[j] = sum_b S[b, j] cz_L[b, j]
        w.M = sp; w.N = 1; w.Kb = B; w.A = ws + lo.Sout; w.G = gates->cz[L]; w.lda = sp; w.D = nullptr; w.ldd = 1;
        w.C = gr->dWz[L]; w.ldc = 1; w.kappa = 1.f;
      }
      w.part = ws + lo.wpart;
      GDB_LAUNCH(launch_wgrad(w, st), "gd_backward wgrad (stored)");
    }
  } else
  for (int pass = 0; pass < 2; ++pass) {
    ICNN_CUDA_CHECK(cudaMemcpyAsync(ws + lo.y, y0, sizeof(float) * N, cudaMemcpyDeviceToDevice, st));
    ICNN_CUDA_CHECK(cudaMemsetAsync(ws + lo.v, 0, sizeof(float) * N, st));
    for (int it = 0; it < nIter; ++it) {
      GdbAcc acc{gr, kappa[it], nullptr, nullptr};
      int rc = gdb_iteration(h, gates, ws, lo, pass ? &acc : nullptr, -1, 0.f, st);
      if (rc) return rc;
      gd_update_kernel<<<gN, 256, 0, st>>>(ws + lo.y, ws + lo.v, ws + lo.g, N, lr, momentum);
    }
    if (pass == 0) {
      ICNN_CUDA_CHECK(cudaMemcpyAsync(yN, ws + lo.y, sizeof(float) * N, cudaMemcpyDeviceToDevice, st));
      mse_grad_kernel<<<gN, 256, 0, st>>>(ws + lo.a, ws + lo.y, trueY, loss_scale, N);
      if (lo.use_tc) {
        GdbTcBufs tb{};
        picnn_gdb_tc_ws_floats(h, B, &tb, ws + lo.tc);
        picnn_gdb_tc_gate_a(h, gates, ws + lo.a, tb, st);
      }
    }
  }

  if (nIter > 0) {
    int rc = gdb_ygate_stage(h, gates, ws, lo, av, gr, (float)ksum, nullptr, nullptr, st);
    if (rc) return rc;
  }
  ICNN_CUDA_CHECK(cudaGetLastError());
  return ICNN_OK;
}
