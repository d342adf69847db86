// Bundle-entropy training gradient d F / d theta (SURVEY.md section 8f row 1: the step after K3).
//
// Replaces opt.compute_gradients(F_, theta_)            multi-label-cls/icnn_ebundle.py:153-156
// on the surrogate F_ = c E(x, y) + sum_j v_j dE/dy_j    multi-label-cls/icnn_ebundle.py:148
// fed one row per (sample, bundle point) by train_step_fd (:296-314): y = bundle point y_r, v = v_r, c = c_r.
//
// The ReLU / leaky-ReLU energy is piecewise linear in y, so with row r's activation pattern fixed v . dE/dy is
// the output of the linear tangent network of gd_backward.cu driven by v, and its backprop multipliers are the
// primal delta_l of E (delta_L = 1); c E backpropagates with the same delta_l.  With
//   yhat = c y + v,   zhat_{l-1} = c z_{l-1} + zt_{l-1}
// every row contributes (oracle/bundle_grad_np.py derives it from the layer recurrences)
//   dWy_l += (yhat o cy_l)^T delta_l          dcy_l[u] += yhat o (delta_l Wy_l^T)
//   dWz_l += (zhat_{l-1} o cz_l)^T delta_l    dcz_l[u] += zhat_{l-1} o (delta_l Wz_l^T)
//                                             dd_l[u]  += c delta_l
// That is one accumulate-mode iteration of gd_backward (gdb_iteration with kappa = 1) at y = y_r and a = v_r,
// with Zt replaced by zhat once the tangent forward is done (GdbAcc::c) and a replaced by yhat before the y-gate
// stage -- the same 3xTF32 wgmma GEMMs (rows >= 64) or FP32 FFMA kernels (fewer rows, or ICNN_GDB=simt).
//
// Rows are processed in chunks cut at sample boundaries, so the workspace is bounded (ICNN_TRAIN_WS_GB, default
// 2 GiB; ICNN_TRAIN_CHUNK forces the rows per chunk).  New device code here is only: the gather of each chunk's
// per-row gates from the per-sample gates, the c-scaled row axpy that forms zhat and yhat, and the segmented sum
// of per-row gate adjoints into the per-sample outputs (one thread per output element walks its sample's rows in
// order: deterministic, no atomics).  dWy / dWz are summed over the rows and the chunks in float64 (the
// weight-gradient GEMM's float64 variant, GdbW64) and rounded once at the end: the rows of a sample partly cancel
// (its c sum to zero), so float32 sums would make the result depend on where the chunks are cut.
#include "gdb.cuh"
#include "train_rows.cuh"
#include "wgrad.cuh"

namespace icnn {

struct TgLayout {
  size_t off, row_u;          // bytes: device copy of row_offsets, row -> sample map
  size_t w64;                 // bytes: the float64 weight-gradient accumulators (gdb_w64_bind)
  size_t gdb;                 // bytes: gdb_layout(h, cap, 0) floats from here
  GdbLayout lo;
  size_t cy[ICNN_MAX_LAYERS + 1], cz[ICNN_MAX_LAYERS + 1], d[ICNN_MAX_LAYERS + 1];   // per-row gates (floats)
  size_t dcy[ICNN_MAX_LAYERS + 1], dcz[ICNN_MAX_LAYERS + 1];                          // per-row gate adjoints
  size_t total;               // bytes
  long long cap;              // rows per chunk
};

static size_t tg_floats(const icnn_picnn* h, long long cap, TgLayout* t) {
  size_t off = 0;
  auto take = [&](size_t nfl) { size_t o = off; off += (nfl + 63) & ~(size_t)63; return o; };
  const size_t rows = (size_t)cap, n = (size_t)h->n;
  for (int l = 0; l <= h->L; ++l) {
    const size_t cy = take(rows * n), cz = l ? take(rows * h->prev(l)) : 0, d = take(rows * h->width(l));
    const size_t dcy = take(rows * n), dcz = l ? take(rows * h->prev(l)) : 0;
    if (t) { t->cy[l] = cy; t->cz[l] = cz; t->d[l] = d; t->dcy[l] = dcy; t->dcz[l] = dcz; }
  }
  return off;
}

// rows per chunk: ICNN_TRAIN_CHUNK if set, else what fits ICNN_TRAIN_WS_GB (at least 64, at most R); the
// weight-gradient partials are one fixed region, not per row
static long long tg_chunk_rows(const icnn_picnn* h, long long R) {
  const long long probe = 1024;
  const size_t fl = gdb_layout(h, (int)probe, 0).total - wgrad_part_bytes() / sizeof(float) + tg_floats(h, probe, nullptr);
  return chunk_rows(4.0 * (double)fl / probe, R);
}

static TgLayout tg_layout(const icnn_picnn* h, int B, long long R) {
  TgLayout t{};
  auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
  t.cap = tg_chunk_rows(h, R);
  size_t bytes = 0;
  t.off = bytes; bytes += al(sizeof(long long) * ((size_t)B + 1));
  t.row_u = bytes; bytes += al(sizeof(int) * (size_t)t.cap);
  t.w64 = bytes; bytes += al(sizeof(double) * gdb_w64_doubles(h));
  t.gdb = bytes;
  if (t.cap > 0) {
    t.lo = gdb_layout(h, (int)t.cap, 0);
    const size_t base = t.lo.total;
    tg_floats(h, t.cap, &t);
    for (int l = 0; l <= h->L; ++l) {
      t.cy[l] += base; t.cz[l] += base; t.d[l] += base; t.dcy[l] += base; t.dcz[l] += base;
    }
    bytes += sizeof(float) * (base + tg_floats(h, t.cap, nullptr));
  }
  t.total = bytes;
  return t;
}

size_t gdb_w64_doubles(const icnn_picnn* h) {
  size_t n64 = 0;
  for (int l = 0; l <= h->L; ++l) n64 += (size_t)h->width(l) * (h->n + h->prev(l));
  return n64;
}

int gdb_w64_bind(const icnn_picnn* h, double* base, GdbW64* w, cudaStream_t st) {
  ICNN_CUDA_CHECK(cudaMemsetAsync(base, 0, sizeof(double) * gdb_w64_doubles(h), st));
  *w = GdbW64{};
  size_t o = 0;
  for (int l = 0; l <= h->L; ++l) { w->dWy[l] = base + o; o += (size_t)h->n * h->width(l); }
  for (int l = 1; l <= h->L; ++l) { w->dWz[l] = base + o; o += (size_t)h->prev(l) * h->width(l); }
  return ICNN_OK;
}

int gdb_w64_round(const icnn_picnn* h, const GdbW64& w, const icnn_train_grads* gr, cudaStream_t st) {
  for (int l = 0; l <= h->L; ++l) {
    const long long Ny = (long long)h->n * h->width(l), Nz = (long long)h->prev(l) * h->width(l);
    round_to_float_kernel<<<(unsigned)((Ny + 255) / 256), 256, 0, st>>>(gr->dWy[l], w.dWy[l], Ny);
    if (l > 0) round_to_float_kernel<<<(unsigned)((Nz + 255) / 256), 256, 0, st>>>(gr->dWz[l], w.dWz[l], Nz);
  }
  ICNN_CUDA_CHECK(cudaGetLastError());
  return ICNN_OK;
}

}  // namespace icnn

using namespace icnn;

extern "C" size_t icnn_train_grad_workspace_bytes(const icnn_picnn_t* h, int32_t B, int64_t R) {
  if (!h || B <= 0 || R < 0 || R > INT32_MAX) return 0;
  return tg_layout(h, B, R).total;
}

extern "C" int icnn_train_grad(const icnn_picnn_t* h, const icnn_gates* gates, const int64_t* row_offsets,
                               const float* Y, const float* V, const float* c, const icnn_train_grads* gr,
                               void* workspace, void* stream) {
  ICNN_REQUIRE(h && gates && row_offsets && gr && workspace, "null pointer");
  if (const int rc = gdb_check_args(h, gates, *gr, true, "icnn_train_grad")) return rc;
  const int B = gates->B, n = h->n, L = h->L;
  const long long R = check_row_offsets(row_offsets, B, Y && V && c);
  if (R < 0) return (int)R;
  cudaStream_t st = static_cast<cudaStream_t>(stream);

  for (int l = 0; l <= L; ++l) {   // outputs: accumulated over the chunks from zero
    const size_t sl = (size_t)h->width(l), sp = (size_t)h->prev(l);
    ICNN_CUDA_CHECK(cudaMemsetAsync(gr->dWy[l], 0, sizeof(float) * n * sl, st));
    ICNN_CUDA_CHECK(cudaMemsetAsync(gr->dcy[l], 0, sizeof(float) * (size_t)B * n, st));
    ICNN_CUDA_CHECK(cudaMemsetAsync(gr->dd[l], 0, sizeof(float) * (size_t)B * sl, st));
    if (l > 0) {
      ICNN_CUDA_CHECK(cudaMemsetAsync(gr->dWz[l], 0, sizeof(float) * sp * sl, st));
      ICNN_CUDA_CHECK(cudaMemsetAsync(gr->dcz[l], 0, sizeof(float) * (size_t)B * sp, st));
    }
  }
  if (R == 0) return ICNN_OK;

  const TgLayout t = tg_layout(h, B, R);
  char* wsb = static_cast<char*>(workspace);
  long long* off_d = reinterpret_cast<long long*>(wsb + t.off);
  int* row_u = reinterpret_cast<int*>(wsb + t.row_u);
  float* ws = reinterpret_cast<float*>(wsb + t.gdb);
  // (pageable source: the call returns once the offsets have been staged)
  ICNN_CUDA_CHECK(cudaMemcpyAsync(off_d, row_offsets, sizeof(long long) * ((size_t)B + 1), cudaMemcpyHostToDevice, st));
  GdbW64 w64;
  if (const int rc = gdb_w64_bind(h, reinterpret_cast<double*>(wsb + t.w64), &w64, st)) return rc;

  // per-row views of the chunk: gates and the gate-adjoint outputs of gdb_iteration
  float *cy[ICNN_MAX_LAYERS + 1], *cz[ICNN_MAX_LAYERS + 1], *dd[ICNN_MAX_LAYERS + 1];
  float *dcy[ICNN_MAX_LAYERS + 1], *dcz[ICNN_MAX_LAYERS + 1];
  for (int l = 0; l <= L; ++l) {
    cy[l] = ws + t.cy[l]; dd[l] = ws + t.d[l]; dcy[l] = ws + t.dcy[l];
    cz[l] = l ? ws + t.cz[l] : nullptr; dcz[l] = l ? ws + t.dcz[l] : nullptr;
  }
  icnn_gates gt{};
  gt.cy = cy; gt.cz = cz; gt.d = dd; gt.in_scale = 1.f; gt.in_shift = 0.f; gt.g_scale = 1.f;
  const icnn_gd_grads rg{gr->dWy, gr->dWz, dcy, dcz};

  long long r0 = 0;
  int u0 = 0;
  while (r0 < R) {
    long long r1;
    int u1;
    next_chunk(row_offsets, B, R, t.cap, r0, &u0, &r1, &u1);
    const int rows = (int)(r1 - r0);

    GdbLayout lo = t.lo;
    lo.use_tc = lo.use_tc && gdb_use_tc(h, rows);
    gt.B = rows;
    launch_row_sample(row_u, off_d, u0, u1, r0, rows, st);
    for (int l = 0; l <= L; ++l) {
      const long long Nn = (long long)rows * n, Nd = (long long)rows * h->width(l), Nz = (long long)rows * h->prev(l);
      launch_gather_rows(cy[l], gates->cy[l], row_u, rows, n, st);
      launch_gather_rows(dd[l], gates->d[l], row_u, rows, h->width(l), st);
      if (l > 0) launch_gather_rows(cz[l], gates->cz[l], row_u, rows, h->prev(l), st);
      ICNN_CUDA_CHECK(cudaMemsetAsync(dcy[l], 0, sizeof(float) * Nn, st));
      if (l > 0) ICNN_CUDA_CHECK(cudaMemsetAsync(dcz[l], 0, sizeof(float) * Nz, st));
      if (l < L) ICNN_CUDA_CHECK(cudaMemsetAsync(ws + lo.Dacc[l], 0, sizeof(float) * Nd, st));
    }
    ICNN_LAUNCH_CHECK(cudaGetLastError(), "train_grad gather");
    ICNN_CUDA_CHECK(cudaMemcpyAsync(ws + lo.y, Y + r0 * n, sizeof(float) * rows * n, cudaMemcpyDeviceToDevice, st));
    ICNN_CUDA_CHECK(cudaMemcpyAsync(ws + lo.a, V + r0 * n, sizeof(float) * rows * n, cudaMemcpyDeviceToDevice, st));
    if (lo.use_tc) {   // the (v o cy_l) columns of the tangent operands
      GdbTcBufs tb{};
      picnn_gdb_tc_ws_floats(h, rows, &tb, ws + lo.tc);
      picnn_gdb_tc_gate_a(h, &gt, ws + lo.a, tb, st);
    }
    const GdbAcc acc{&rg, 1.f, c + r0, &w64};
    int rc = gdb_iteration(h, &gt, ws, lo, &acc, -1, 0.f, st);
    if (rc) return rc;
    launch_row_axpy(ws + lo.a, ws + lo.y, c + r0, rows, n, st);   // yhat = c y + v
    rc = gdb_ygate_stage(h, &gt, ws, lo, ws + lo.a, &rg, 1.f, &w64, nullptr, st);
    if (rc) return rc;

    // per-row gate adjoints -> per-sample outputs; dd_l = sum_r c_r delta_l (delta_L = 1)
    for (int l = 0; l <= L; ++l) {
      const int wl = h->width(l), pl = h->prev(l);
      const SegView one{nullptr, nullptr, 0, 1, 0, 0};
      launch_segsum_prod(gr->dcy[l], SegView{dcy[l], nullptr, n, n, 0, 0}, one, nullptr, n, off_d, u0, u1, r0, r1, st);
      if (l > 0)
        launch_segsum_prod(gr->dcz[l], SegView{dcz[l], nullptr, pl, pl, 0, 0}, one, nullptr, pl, off_d, u0, u1, r0, r1,
                           st);
      launch_segsum_prod(gr->dd[l], l < L ? SegView{ws + lo.Dacc[l], nullptr, wl, wl, 0, 0} : one, one, c, wl, off_d,
                         u0, u1, r0, r1, st);
    }
    ICNN_LAUNCH_CHECK(cudaGetLastError(), "train_grad segmented sum");
    r0 = r1;
  }
  return gdb_w64_round(h, w64, gr, st);   // the float64 weight-gradient sums, rounded once
}
