// TD training gradient of the RL agent (SURVEY.md section 8f: the training step after Agent.adam).
//
// Replaces optim_q.compute_gradients(loss_q) (RL/src/icnn.py:107-108) of the default '--icnn_opt adam' agent
// (RL/src/icnn.py:55-93, the minibatch step Agent.train :304-323) for the y-path of the online network:
//   negQ_entr = negQ(obs, act) - H(act),  q_entr = -negQ_entr                                      (:59-62)
//   q_target_entr = -(negQ_target(ob2, act2) - H(act2))                                            (:69-75)
//   y = term ? rew : rew + discount q_target_entr,  y = min(q_entr + 1, max(q_entr - 1, y))        (:78-81)
//   td = q_entr - y,  ms_td_error = mean(td^2)                                                     (:82, :90)
// with H(a) = -sum_j p log p + (1 - p) log(1 - p), p = clip((a + 1) / 2, 1e-4, 1 - 1e-4) (:455-458).  y is under
// stop_gradient, so d ms_td_error / d negQ_u = c_u = -2 td_u / B, and the gradient is that of sum_u c_u negQ_u:
// K1's backward with the output seed delta_L = c_u instead of 1.  Every delta_l is then c o delta_l and
//   dWy_l = sum_u (act o cy_l)^T delta_l    dcy_l = act o (delta_l Wy_l^T)
//   dWz_l = sum_u (z_{l-1} o cz_l)^T delta_l    dcz_l = z_{l-1} o (delta_l Wz_l^T)    dd_l = delta_l
// which is icnn_train_grad at Y = act, V = 0 and one row per sample, without its tangent network (V = 0 makes it
// zero), its per-row gate gather and its segmented sums, and with c taken from the same forward.
//
// Launch sequence: the primal forward of gdb_forward (3xTF32 wgmma GEMMs for B >= 64, FP32 FFMA below) gives
// negQ = f; td_seed_kernel forms td and c per sample and scales delta_{L-1} (and its TF32 hi/lo split) by c;
// gdb_backward runs the backward GEMMs with the GDB accumulation epilogue on the primal Z_l (GdbAcc::dL);
// gdb_ygate_stage adds the y-gate terms.  dWy / dWz are summed in float64 (GdbW64) and rounded once; the loss is a
// fixed-order float64 sum.  No atomics: every call gives the same bits.
#include "gdb.cuh"
#include "train_rows.cuh"
#include "wgrad.cuh"

namespace icnn {

size_t picnn_gdb_tc_ws_floats(const icnn_picnn* h, int B, GdbTcBufs* b, float* base);

constexpr int TD_MAX_B = 65536;          // the C4 minibatch; the whole batch runs as one block of rows
constexpr int TD_LOSS_THREADS = 1024;

struct TdLayout {
  size_t w64, n64;   // bytes / doubles: float64 accumulators of dWy_0..L, dWz_1..L (in that order)
  size_t c;          // bytes: c [B] floats
  size_t gdb;        // bytes: gdb_layout(h, B, 0) floats from here
  GdbLayout lo;
  size_t total;
};

static TdLayout td_layout(const icnn_picnn* h, int B) {
  TdLayout t{};
  auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
  size_t bytes = 0;
  for (int l = 0; l <= h->L; ++l) t.n64 += (size_t)h->width(l) * (h->n + h->prev(l));
  t.w64 = bytes; bytes += al(sizeof(double) * t.n64);
  t.c = bytes; bytes += al(sizeof(float) * (size_t)B);
  t.gdb = bytes;
  t.lo = gdb_layout(h, B, 0);
  t.total = bytes + sizeof(float) * t.lo.total;
  return t;
}

// -sum_j [p log p + (1 - p) log(1 - p)] of one action row, p = clip((a + 1) / 2, 1e-4, 1 - 1e-4), over a warp
__device__ __forceinline__ double td_entropy(const float* a, int n, int lane) {
  double s = 0.0;
  for (int j = lane; j < n; j += 32) {
    const double p = fmin(fmax(((double)a[j] + 1.0) / 2.0, 1e-4), 1.0 - 1e-4);
    s += p * log(p) + (1.0 - p) * log(1.0 - p);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return -s;
}

struct TdArgs {
  int B, n, S;                              // S = s_{L-1}
  const float* f;                           // negQ(obs, act) [B] (K1 forward)
  const float* act; const float* act2;      // [B, n]
  const float* negq_t; const float* rew; const uint8_t* term;
  float discount;
  float* td; float* c;                      // [B]
  float* delta; float* delta_hi; float* delta_lo; int delta_ld;   // delta_{L-1} [B, S] (hi / lo: tensor-core path)
};

// one warp per sample: the TD target and error, c = -2 td / B, and delta_{L-1} <- c delta_{L-1}
__global__ void __launch_bounds__(256) td_seed_kernel(TdArgs a) {
  const int u = (int)((blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (u >= a.B) return;
  const double h1 = td_entropy(a.act + (long long)u * a.n, a.n, lane);
  const double h2 = td_entropy(a.act2 + (long long)u * a.n, a.n, lane);
  const double q = -((double)a.f[u] - h1);
  const double qt = -((double)a.negq_t[u] - h2);
  double y = a.term[u] ? (double)a.rew[u] : (double)a.rew[u] + (double)a.discount * qt;
  y = fmin(q + 1.0, fmax(q - 1.0, y));
  const double td = q - y;
  const float cu = (float)(-2.0 * td / a.B);
  if (lane == 0) { a.td[u] = (float)td; a.c[u] = cu; }
  for (int j = lane; j < a.S; j += 32) {
    const long long idx = (long long)u * a.S + j;
    const float dl = cu * a.delta[idx];
    a.delta[idx] = dl;
    if (a.delta_hi) {
      const float hh = tf32_rn(dl);
      const long long o = (long long)u * a.delta_ld + j;
      a.delta_hi[o] = hh;
      a.delta_lo[o] = tf32_rn(dl - hh);
    }
  }
}

// loss = mean(td^2) in float64: thread t sums rows t, t + T, ... in order, then a fixed tree over the threads
__global__ void __launch_bounds__(TD_LOSS_THREADS) td_loss_kernel(const float* td, int B, double* loss) {
  __shared__ double red[TD_LOSS_THREADS];
  double s = 0.0;
  for (int i = threadIdx.x; i < B; i += TD_LOSS_THREADS) s += (double)td[i] * (double)td[i];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int w = TD_LOSS_THREADS / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) *loss = red[0] / B;
}

}  // namespace icnn

using namespace icnn;

extern "C" size_t icnn_td_grad_workspace_bytes(const icnn_picnn_t* h, int32_t B) {
  if (!h || B <= 0 || B > TD_MAX_B) return 0;
  return td_layout(h, B).total;
}

extern "C" int icnn_td_grad(const icnn_picnn_t* h, const icnn_gates* gates, const float* act, const float* negq_target,
                            const float* act2, const float* rew, const uint8_t* term, float discount, float* td,
                            double* loss, const icnn_train_grads* gr, void* workspace, void* stream) {
  ICNN_REQUIRE(h && gates && act && negq_target && act2 && rew && term && td && loss && gr && workspace,
               "null pointer");
  ICNN_REQUIRE(gr->dWy && gr->dWz && gr->dcy && gr->dcz && gr->dd, "null gradient array");
  ICNN_REQUIRE(gates->B > 0, "empty batch");
  if (gates->B > TD_MAX_B) {
    set_error("icnn_td_grad: B = %d is above %d; split the minibatch", gates->B, TD_MAX_B);
    return ICNN_E_INVALID;
  }
  if (gates->in_scale != 1.f || gates->in_shift != 0.f || gates->g_scale != 1.f) {
    set_error("icnn_td_grad: the affine (RL bundle) input wrapper is not on this path; bind obs without it");
    return ICNN_E_UNSUPPORTED;
  }
  const int B = gates->B, n = h->n, L = h->L;
  for (int l = 0; l <= L; ++l)
    ICNN_REQUIRE(gr->dWy[l] && gr->dcy[l] && gr->dd[l] && (l == 0 || (gr->dWz[l] && gr->dcz[l])),
                 "null gradient buffer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const TdLayout t = td_layout(h, B);
  const GdbLayout& lo = t.lo;
  char* wsb = static_cast<char*>(workspace);
  float* c = reinterpret_cast<float*>(wsb + t.c);
  float* ws = reinterpret_cast<float*>(wsb + t.gdb);
  double* acc64 = reinterpret_cast<double*>(wsb + t.w64);
  GdbW64 w64{};
  {
    size_t o = 0;
    for (int l = 0; l <= L; ++l) { w64.dWy[l] = acc64 + o; o += (size_t)n * h->width(l); }
    for (int l = 1; l <= L; ++l) { w64.dWz[l] = acc64 + o; o += (size_t)h->prev(l) * h->width(l); }
  }
  // accumulated outputs and accumulators start from zero (dWy / dWz and dd are written whole at the end)
  ICNN_CUDA_CHECK(cudaMemsetAsync(acc64, 0, sizeof(double) * t.n64, st));
  for (int l = 0; l <= L; ++l) {
    ICNN_CUDA_CHECK(cudaMemsetAsync(gr->dcy[l], 0, sizeof(float) * (size_t)B * n, st));
    if (l > 0) ICNN_CUDA_CHECK(cudaMemsetAsync(gr->dcz[l], 0, sizeof(float) * (size_t)B * h->prev(l), st));
    if (l < L) ICNN_CUDA_CHECK(cudaMemsetAsync(ws + lo.Dacc[l], 0, sizeof(float) * (size_t)B * h->width(l), st));
  }
  ICNN_CUDA_CHECK(cudaMemcpyAsync(ws + lo.y, act, sizeof(float) * (size_t)B * n, cudaMemcpyDeviceToDevice, st));

  const icnn_gd_grads rg{gr->dWy, gr->dWz, gr->dcy, gr->dcz};
  GdbAcc acc{&rg, 1.f, nullptr, &w64};
  acc.dL = c;
  int rc = gdb_forward(h, gates, ws, lo, &acc, -1, 0.f, st);
  if (rc) return rc;

  TdArgs ta{};
  ta.B = B; ta.n = n; ta.S = h->hidden[L - 1]; ta.f = ws + lo.f; ta.act = act; ta.act2 = act2;
  ta.negq_t = negq_target; ta.rew = rew; ta.term = term; ta.discount = discount; ta.td = td; ta.c = c;
  ta.delta = ws + lo.dl[0]; ta.delta_ld = ld4(ta.S);
  if (lo.use_tc) {
    GdbTcBufs tb{};
    picnn_gdb_tc_ws_floats(h, B, &tb, ws + lo.tc);
    ta.delta_hi = tb.dh[0]; ta.delta_lo = tb.dl[0];
  }
  td_seed_kernel<<<cdiv(B, 8), 256, 0, st>>>(ta);
  td_loss_kernel<<<1, TD_LOSS_THREADS, 0, st>>>(td, B, loss);
  ICNN_CUDA_CHECK(cudaGetLastError());

  rc = gdb_backward(h, gates, ws, lo, &acc, -1, 0.f, st);
  if (rc) return rc;
  rc = gdb_ygate_stage(h, gates, ws, lo, ws + lo.y, &rg, 1.f, &w64, c, st);
  if (rc) return rc;

  // dd_l = delta_l (the accumulated Dacc_l of the single pass; delta_L = c), and the float64 sums rounded once
  for (int l = 0; l < L; ++l)
    ICNN_CUDA_CHECK(cudaMemcpyAsync(gr->dd[l], ws + lo.Dacc[l], sizeof(float) * (size_t)B * h->width(l),
                                    cudaMemcpyDeviceToDevice, st));
  ICNN_CUDA_CHECK(cudaMemcpyAsync(gr->dd[L], c, sizeof(float) * (size_t)B, cudaMemcpyDeviceToDevice, st));
  for (int l = 0; l <= L; ++l) {
    const long long Ny = (long long)n * h->width(l), Nz = (long long)h->prev(l) * h->width(l);
    round_to_float_kernel<<<(unsigned)((Ny + 255) / 256), 256, 0, st>>>(gr->dWy[l], w64.dWy[l], Ny);
    if (l > 0) round_to_float_kernel<<<(unsigned)((Nz + 255) / 256), 256, 0, st>>>(gr->dWz[l], w64.dWz[l], Nz);
  }
  ICNN_CUDA_CHECK(cudaGetLastError());
  return ICNN_OK;
}
