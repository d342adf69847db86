// Bundle-entropy training gradient d F / d theta of the convolutional PICNN (the image-completion energy).
//
// Replaces compute_gradients(F_, theta_)                  completion/icnn_ebundle.py:129-140
// on the surrogate F_ = c E(x, y) + sum_j v_j dE/dy_j     (:129-130)
// fed one row per (sample, bundle point) by train_step_fd (:315-335): y = bundle point y_r, v = v_r, c = c_r.
//
// ReLU makes E piecewise linear in y: with row r's activation pattern fixed, delta_l and rho_l (notation of
// conv_picnn.cu) do not depend on y, so v . dE/dy is the output of the linear tangent network driven by v and its
// backprop multipliers are the primal delta_l / rho_l.  Per row, conv_fg at y = Y_r gives r_l, z_l, delta_l, rho_l
// and (col2im, eout) the un-gated adjoints [e_z,l | e_r,l] = conv_l^T(delta_l; [Wz_l | Wy_l]); the tangent forward
//   rt_0 = V_r,  rt_{l+1} = conv_l(rt_l; Wred_l)                                   (no bias)
//   conv:  zt_l = relu'(z_l) o conv_l([zt_{l-1} o cz_l | rt_l o cy_l]; Wcat_l)       (no d)
//   dense: zt_i = relu'(z_i) o ((zt_{i-1} o cz_i) Wz_i)
// is the forward's gated im2col and the GEMM with the tangent epilogue (TcArgs::tangent = 1).  With the hats
// zhat_l = c_r z_l + zt_l, rhat_l = c_r r_l + rt_l, summed over all rows
//   dWcat_l = im2col([zhat_{l-1} o cz_l | rhat_l o cy_l])^T delta_l    (-> 'z{l}_zu_proj/W', 'z{l}_yu/W')
//   dWz_i   = (zhat_{i-1} o cz_i)^T delta_i                           (delta = 1 at the width-1 output)
//   dWred_l[tap] = sum_o rhat_l[in(o, tap)] rho_{l+1}[o],  dbred_l = c_r sum_o rho_{l+1}[o]    (l < Lc - 1)
// and summed over each sample's rows
//   dcz_l = zhat_{l-1} o e_z,l,  dcy_l = rhat_l o e_r,l,  dd_l = c_r delta_l
// (dense layers: e_z,i = delta_i Wz_i^T, recomputed by one plain GEMM per hidden dense layer; the output layer's is
// its weight vector).
//
// Rows are processed in chunks cut at sample boundaries (train_rows.cuh; ICNN_TRAIN_WS_GB / ICNN_TRAIN_CHUNK as in
// train_grad.cu).  Every weight gradient is summed in float64 -- each product of two floats is exact -- over the
// rows and the chunks, and rounded once: a sample's c sum to zero, so float32 sums would depend on the chunk cut; in
// float64 a different cut only reorders additions, and the results agree up to the final rounding.
// The per-sample outputs are float64 sums over a sample's rows, rounded once per chunk: only a sample with more rows
// than a chunk holds (split over chunks, as in train_grad.cu) sees more than one rounding.
// The weight gradients are wgrad.cuh's GEMM in float64 with delta's TF32 hi/lo pair as D + Dlo.  A conv layer's
// reduction is long (rows H_{l+1} W_{l+1}) and its output small (K_l x C_l), so wgrad_parts splits it over the rows
// into enough CTAs to fill the machine and the float64 partials are summed in a fixed order: no atomics, the same
// result on every call.
//
// The GD training backward of the same net (icnn_conv_gd_backward, completion/icnn.back.py:133-156) is this gradient
// on other rows: with a = dloss/dy_N and kappa_i of gd_backward.cu's derivation (the conv energy is piecewise linear
// in y too), dloss/dtheta = sum_{i < N} d/dtheta <dE/dy(x, y_i), kappa_i a>, i.e. one row per (sample, GD step) with
// Y = y_i, V = kappa_i a, c = 0.  It runs the GD loop of icnn_conv_gd_solve keeping the iterates, forms the rows
// and calls icnn_conv_train_grad on them; with c = 0 the hats are the tangents and dd, dbred come back zero.
#include "conv_picnn.cuh"
#include "gdb.cuh"
#include "train_rows.cuh"
#include "wgrad.cuh"

#include <vector>

namespace icnn {

int conv_check_gates(const icnn_conv_picnn* h, const icnn_gates* gt);

static inline unsigned nb(long long n) { return (unsigned)((n + 255) / 256); }

// r_{l+1} tangent: conv(r_l; Wred_l) without the bias, taps in yred_kernel's order
static __global__ void yred_tangent_kernel(const float* r, float* rn, const float* red, ConvGeom g, int B) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)B * g.Ho * g.Wo) return;
  const int ox = (int)(i % g.Wo), oy = (int)((i / g.Wo) % g.Ho), b = (int)(i / ((long long)g.Wo * g.Ho));
  const float* rb = r + (long long)b * g.Hi * g.Wi;
  float acc = 0.f;
  for (int ky = 0; ky < g.k; ++ky) {
    const int iy = oy * g.s - g.pt + ky;
    if (iy < 0 || iy >= g.Hi) continue;
    for (int kx = 0; kx < g.k; ++kx) {
      const int ix = ox * g.s - g.pl + kx;
      if (ix < 0 || ix >= g.Wi) continue;
      acc = fmaf(red[ky * g.k + kx], rb[iy * g.Wi + ix], acc);
    }
  }
  rn[i] = acc;
}

// A[m, t (Cp+1) + c] = (c < Cp ? Z o cz : r o cy) at tap t of output pixel m (0 in the padding), float, pitch K
static __global__ void im2col_plain_kernel(const float* Z, const float* cz, const float* r, const float* cy,
                                           ConvGeom g, int B, float* A) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long M = (long long)B * g.Ho * g.Wo;
  if (i >= M * g.K) return;
  const long long m = i / g.K;
  const int kk = (int)(i % g.K);
  const int ox = (int)(m % g.Wo), oy = (int)((m / g.Wo) % g.Ho), b = (int)(m / ((long long)g.Wo * g.Ho));
  const int t = kk / (g.Cp + 1), c = kk % (g.Cp + 1);
  const int iy = oy * g.s - g.pt + t / g.k, ix = ox * g.s - g.pl + t % g.k;
  float v = 0.f;
  if (iy >= 0 && iy < g.Hi && ix >= 0 && ix < g.Wi) {
    const long long p = ((long long)b * g.Hi + iy) * g.Wi + ix;
    v = c < g.Cp ? Z[p * g.Cp + c] * cz[p * g.Cp + c] : r[p] * cy[p];
  }
  A[i] = v;
}

// y_red gradients of conv layer g from the rows' rhat_l [rows, Hi Wi] and rho_{l+1} [rows, Ho Wo]; CTA (t, z) sums
// the output pixels [Mo z / P, Mo (z+1) / P) into part[z][t]:
//   t < k^2: rhat_l[in(o, t)] rho_{l+1}[o] (0 in the padding);  t = k^2: c_row rho_{l+1}[o]
static __global__ void __launch_bounds__(256) yred_grad_kernel(const float* rhat, const float* rho, const float* c,
                                                               ConvGeom g, long long Mo, double* part) {
  __shared__ double red[256];
  const int t = blockIdx.x, T = g.k * g.k, P = gridDim.y, z = blockIdx.y, hw = g.Ho * g.Wo;
  const long long b0 = Mo * z / P, b1 = Mo * (z + 1) / P;
  double acc = 0.0;
  for (long long o = b0 + threadIdx.x; o < b1; o += 256) {
    const long long row = o / hw;
    const int q = (int)(o % hw), oy = q / g.Wo, ox = q % g.Wo;
    double v;
    if (t == T) {
      v = (double)c[row];
    } else {
      const int iy = oy * g.s - g.pt + t / g.k, ix = ox * g.s - g.pl + t % g.k;
      if (iy < 0 || iy >= g.Hi || ix < 0 || ix >= g.Wi) continue;
      v = (double)rhat[(row * g.Hi + iy) * g.Wi + ix];
    }
    acc = fma(v, (double)rho[o], acc);
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[(long long)z * (T + 1) + t] = red[0];
}

// dWcat [K, N] (float64) -> 'z{l}_zu_proj/W' [taps, Cp, N] and 'z{l}_yu/W' [taps, 1, N]: the inverse of
// conv_pack_kernel's row order kk = t (Cp + 1) + c
static __global__ void conv_unpack_kernel(const double* acc, int taps, int Cp, int N, float* Wz, float* Wy) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)taps * (Cp + 1) * N) return;
  const int kk = (int)(i / N), o = (int)(i % N), t = kk / (Cp + 1), c = kk % (Cp + 1);
  const float v = (float)acc[i];
  if (c < Cp) Wz[((long long)t * Cp + c) * N + o] = v;
  else Wy[(long long)t * N + o] = v;
}

// ---- workspace --------------------------------------------------------------------------------------------------
struct CtgLayout {
  size_t off, row_u, acc64, part64, fl;   // bytes
  size_t n64;                             // doubles
  size_t aw[2 * ICNN_MAX_LAYERS], ared[ICNN_MAX_LAYERS];   // doubles into acc64: dWcat_l / dWz_i, y_red l
  // floats from fl: conv_fg's workspace, per-row gates, e_l, tangents, dense e_z, f and g scratch
  size_t cws, cy[2 * ICNN_MAX_LAYERS], cz[2 * ICNN_MAX_LAYERS], d[2 * ICNN_MAX_LAYERS], e[ICNN_MAX_LAYERS];
  size_t zt[2 * ICNN_MAX_LAYERS], rt[ICNN_MAX_LAYERS], ez[2 * ICNN_MAX_LAYERS], f, g, nfl;
  long long cap;
  size_t total;
};

static int yred_parts(long long Mo) {
  const long long p = (Mo + 4095) / 4096;
  return (int)(p < 1 ? 1 : p > 64 ? 64 : p);
}

// per-row floats (without conv_fg's workspace) for cap rows; fills t's float offsets when t != nullptr
static size_t ctg_floats(const icnn_conv_picnn* h, long long cap, CtgLayout* t) {
  size_t off = 0;
  auto take = [&](size_t nfl) { const size_t o = off; off += (nfl + 63) & ~(size_t)63; return o; };
  const size_t R = (size_t)cap;
  CtgLayout tmp{};
  CtgLayout& o = t ? *t : tmp;
  for (int l = 0; l < h->Lc; ++l) {
    const ConvGeom& g = h->g[l];
    const size_t pin = (size_t)g.Hi * g.Wi, pout = (size_t)g.Ho * g.Wo;
    o.cy[l] = take(R * pin);
    o.cz[l] = l ? take(R * pin * g.Cp) : 0;
    o.d[l] = take(R * pout * g.C);
    o.e[l] = take(R * pin * (g.Cp + 1));
    o.zt[l] = take(R * pout * g.C);
    o.rt[l] = take(R * pin);
  }
  for (int j = 0; j < h->Ld; ++j) {
    const int i = h->Lc + j;
    o.cz[i] = take(R * h->in_w(j));
    o.d[i] = take(R * h->fcs[j]);
    if (j + 1 < h->Ld) { o.zt[i] = take(R * h->fcs[j]); o.ez[i] = take(R * h->in_w(j)); }
  }
  o.f = take(R);
  o.g = take(R * h->H * h->W);
  return off;
}

static CtgLayout ctg_layout(const icnn_conv_picnn* h, int B, long long R) {
  CtgLayout t{};
  auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
  {
    const long long probe = 256;
    ConvWs w{};
    const double per_row = 4.0 * (double)(conv_ws_floats(h, (int)probe, nullptr, &w) + ctg_floats(h, probe, nullptr)) / probe;
    t.cap = chunk_rows(per_row, R);
  }
  size_t n64 = 0, npart = wgrad_part_bytes() / sizeof(double);   // the y_red partials share the region
  for (int l = 0; l < h->Lc; ++l) {
    const ConvGeom& g = h->g[l];
    t.aw[l] = n64; n64 += (size_t)g.K * g.C;
    if (l + 1 < h->Lc) {
      t.ared[l] = n64; n64 += (size_t)g.k * g.k + 1;
      const size_t p = (size_t)yred_parts(t.cap * g.Ho * g.Wo) * (g.k * g.k + 1);
      npart = p > npart ? p : npart;
    }
  }
  for (int j = 0; j < h->Ld; ++j) { t.aw[h->Lc + j] = n64; n64 += (size_t)h->in_w(j) * h->fcs[j]; }
  t.n64 = n64;
  size_t bytes = 0;
  t.off = bytes; bytes += al(sizeof(long long) * ((size_t)B + 1));
  t.row_u = bytes; bytes += al(sizeof(int) * (size_t)t.cap);
  t.acc64 = bytes; bytes += al(sizeof(double) * n64);
  t.part64 = bytes; bytes += al(sizeof(double) * npart);
  t.fl = bytes;
  if (t.cap > 0) {
    ConvWs w{};
    t.cws = 0;
    const size_t cw = conv_ws_floats(h, (int)t.cap, nullptr, &w);
    t.nfl = ctg_floats(h, t.cap, &t);
    const size_t base = (cw + 63) & ~(size_t)63;
    for (int i = 0; i < h->Lc + h->Ld; ++i) {
      t.cy[i] += base; t.cz[i] += base; t.d[i] += base; t.zt[i] += base; t.ez[i] += base;
      if (i < h->Lc) { t.e[i] += base; t.rt[i] += base; }
    }
    t.f += base; t.g += base;
    bytes += sizeof(float) * (base + t.nfl);
  }
  t.total = bytes;
  return t;
}

// every per-layer buffer of icnn_conv_train_grads the layers use is given
static int ctg_check_buffers(const icnn_conv_picnn* h, const icnn_conv_train_grads* gr) {
  const int Lc = h->Lc, NL = h->Lc + h->Ld;
  for (int i = 0; i < NL; ++i) {
    ICNN_REQUIRE(gr->dd[i] && (i == 0 || (gr->dWz[i] && gr->dcz[i])), "null gradient buffer");
    ICNN_REQUIRE(i >= Lc || (gr->dWy[i] && gr->dcy[i]), "null gradient buffer");
    ICNN_REQUIRE(i + 1 >= Lc || (gr->dWred[i] && gr->dbred[i]), "null gradient buffer");
  }
  return ICNN_OK;
}

// ---- the GD training backward (icnn_conv_gd_backward) -------------------------------------------------------------
// Its rows are one per (sample u, GD step i), sample-major: row u nIter + i holds Y = y_i[u], V = kappa_i a[u], c = 0,
// so the row offsets are u nIter and the gradient is icnn_conv_train_grad on them.

// V[u, i, :] = kappa_i a[u, :] with a = loss_scale (yN - trueY): one subtraction and one multiply for a, one
// multiply for V; c [B nIter] = 0
static __global__ void gd_seed_kernel(float* V, float* c, const float* yN, const float* trueY, const float* kappa,
                                      float loss_scale, int nIter, int n, long long N) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= N) return;
  const long long row = i / n, u = row / nIter;
  const int j = (int)(i % n), it = (int)(row % nIter);
  const float a = loss_scale * (yN[u * n + j] - trueY[u * n + j]);
  V[i] = kappa[it] * a;
  if (j == 0) c[row] = 0.f;
}

// bytes: the trajectory Y [B nIter, n], V [B nIter, n], c [B nIter], kappa [nIter], the GD loop's v, g [B, n] and
// f [B]; then one region that the loop's conv_fg workspace and, after the loop, icnn_conv_train_grad's share
struct CgdLayout { size_t Y, V, c, kap, v, g, f, ws, total; };

static CgdLayout cgd_layout(const icnn_conv_picnn* h, int B, int nIter) {
  auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
  const size_t R = (size_t)B * nIter, n = (size_t)h->H * h->W;
  CgdLayout t{};
  size_t bytes = 0;
  auto take = [&](size_t nb_) { const size_t o = bytes; bytes += al(nb_ > 0 ? nb_ : 4); return o; };
  t.Y = take(sizeof(float) * R * n);
  t.V = take(sizeof(float) * R * n);
  t.c = take(sizeof(float) * R);
  t.kap = take(sizeof(float) * (size_t)nIter);
  t.v = take(sizeof(float) * B * n);
  t.g = take(sizeof(float) * B * n);
  t.f = take(sizeof(float) * B);
  ConvWs w{};
  const size_t fgb = sizeof(float) * conv_ws_floats(h, B, nullptr, &w), tgb = ctg_layout(h, B, (long long)R).total;
  t.ws = take(fgb > tgb ? fgb : tgb);
  t.total = bytes;
  return t;
}

}  // namespace icnn

using namespace icnn;

extern "C" size_t icnn_conv_train_grad_workspace_bytes(const icnn_conv_picnn_t* h, int32_t B, int64_t R) {
  if (!h || B <= 0 || R < 0 || R > INT32_MAX) return 0;
  return ctg_layout(h, B, R).total;
}

extern "C" int icnn_conv_train_grad(const icnn_conv_picnn_t* h, const icnn_gates* gates, const int64_t* row_offsets,
                                    const float* Y, const float* V, const float* c, const icnn_conv_train_grads* gr,
                                    void* workspace, void* stream) {
  ICNN_REQUIRE(h && gates && row_offsets && gr && workspace, "null pointer");
  ICNN_REQUIRE(gr->dWz && gr->dWy && gr->dWred && gr->dbred && gr->dcy && gr->dcz && gr->dd, "null gradient array");
  int rc = conv_check_gates(h, gates);
  if (rc) return rc;
  const int B = gates->B, Lc = h->Lc, Ld = h->Ld, NL = Lc + Ld, n = h->H * h->W;
  const long long R = check_row_offsets(row_offsets, B, Y && V && c);
  if (R < 0) return (int)R;
  if ((rc = ctg_check_buffers(h, gr))) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);

  // outputs: the per-sample ones accumulate over the chunks from zero
  for (int l = 0; l < Lc; ++l) {
    const ConvGeom& g = h->g[l];
    ICNN_CUDA_CHECK(cudaMemsetAsync(gr->dcy[l], 0, sizeof(float) * (size_t)B * g.Hi * g.Wi, st));
    ICNN_CUDA_CHECK(cudaMemsetAsync(gr->dd[l], 0, sizeof(float) * (size_t)B * g.Ho * g.Wo * g.C, st));
    if (l) ICNN_CUDA_CHECK(cudaMemsetAsync(gr->dcz[l], 0, sizeof(float) * (size_t)B * g.Hi * g.Wi * g.Cp, st));
  }
  for (int j = 0; j < Ld; ++j) {
    ICNN_CUDA_CHECK(cudaMemsetAsync(gr->dcz[Lc + j], 0, sizeof(float) * (size_t)B * h->in_w(j), st));
    ICNN_CUDA_CHECK(cudaMemsetAsync(gr->dd[Lc + j], 0, sizeof(float) * (size_t)B * h->fcs[j], st));
  }

  const CtgLayout t = ctg_layout(h, B, R);
  char* wsb = static_cast<char*>(workspace);
  long long* off_d = reinterpret_cast<long long*>(wsb + t.off);
  int* row_u = reinterpret_cast<int*>(wsb + t.row_u);
  double* acc64 = reinterpret_cast<double*>(wsb + t.acc64);
  double* part64 = reinterpret_cast<double*>(wsb + t.part64);
  float* fl = reinterpret_cast<float*>(wsb + t.fl);
  ICNN_CUDA_CHECK(cudaMemsetAsync(acc64, 0, sizeof(double) * t.n64, st));
  // (pageable source: the call returns once the offsets have been staged)
  ICNN_CUDA_CHECK(cudaMemcpyAsync(off_d, row_offsets, sizeof(long long) * ((size_t)B + 1), cudaMemcpyHostToDevice, st));

  if (R > 0) {
    float *cy[2 * ICNN_MAX_LAYERS] = {}, *cz[2 * ICNN_MAX_LAYERS] = {}, *dd[2 * ICNN_MAX_LAYERS] = {};
    float *e[ICNN_MAX_LAYERS] = {}, *zt[2 * ICNN_MAX_LAYERS] = {}, *rt[ICNN_MAX_LAYERS] = {};
    float* ez[2 * ICNN_MAX_LAYERS] = {};
    for (int i = 0; i < NL; ++i) {
      dd[i] = fl + t.d[i];
      cz[i] = (i > 0) ? fl + t.cz[i] : nullptr;
      if (i < Lc) { cy[i] = fl + t.cy[i]; e[i] = fl + t.e[i]; rt[i] = fl + t.rt[i]; zt[i] = fl + t.zt[i]; }
      else if (i + 1 < NL) { zt[i] = fl + t.zt[i]; ez[i] = fl + t.ez[i]; }
    }
    float* fbuf = fl + t.f;
    float* gbuf = fl + t.g;
    icnn_gates gt{};
    gt.cy = cy; gt.cz = cz; gt.d = dd; gt.in_scale = 1.f; gt.in_shift = 0.f; gt.g_scale = 1.f;

    long long r0 = 0;
    int u0 = 0;
    while (r0 < R) {
      long long r1;
      int u1;
      next_chunk(row_offsets, B, R, t.cap, r0, &u0, &r1, &u1);
      const int rows = (int)(r1 - r0);
      ConvWs w{};     // conv_fg's buffers as it lays them out for this chunk's rows
      conv_ws_floats(h, rows, fl + t.cws, &w);
      const float* Yc = Y + r0 * n;
      const float* cc = c + r0;
      gt.B = rows;

      // ---- per-row gates ----
      launch_row_sample(row_u, off_d, u0, u1, r0, rows, st);
      auto gather = [&](float* dst, const float* src, long long wdt) { launch_gather_rows(dst, src, row_u, rows, wdt, st); };
      for (int l = 0; l < Lc; ++l) {
        const ConvGeom& g = h->g[l];
        gather(cy[l], gates->cy[l], (long long)g.Hi * g.Wi);
        if (l) gather(cz[l], gates->cz[l], (long long)g.Hi * g.Wi * g.Cp);
        gather(dd[l], gates->d[l], (long long)g.Ho * g.Wo * g.C);
      }
      for (int j = 0; j < Ld; ++j) {
        gather(cz[Lc + j], gates->cz[Lc + j], h->in_w(j));
        gather(dd[Lc + j], gates->d[Lc + j], h->fcs[j]);
      }
      ICNN_LAUNCH_CHECK(cudaGetLastError(), "conv_train_grad gather");

      // ---- primal: f, df/dy and the un-gated conv adjoints e_l ----
      if ((rc = conv_fg(h, &gt, Yc, fbuf, gbuf, n, nullptr, nullptr, 0, fl + t.cws, nullptr, st, e))) return rc;

      // ---- tangent forward on V (the forward operands Ah / Al are free again) ----
      ICNN_CUDA_CHECK(cudaMemcpyAsync(rt[0], V + r0 * n, sizeof(float) * (size_t)rows * n, cudaMemcpyDeviceToDevice, st));
      for (int l = 0; l < Lc; ++l) {
        const ConvGeom& G = h->g[l];
        if (l + 1 < Lc) yred_tangent_kernel<<<nb((long long)rows * G.Ho * G.Wo), 256, 0, st>>>(rt[l], rt[l + 1], h->red[l], G, rows);
        conv_im2col_gate_launch(l ? zt[l - 1] : nullptr, cz[l], rt[l], cy[l], G, rows, w.Ah[l], w.Al[l], st);
        TcArgs a{};
        a.M = rows * G.Ho * G.Wo; a.N = G.C; a.K = G.K; a.mode = 0; a.tangent = 1; a.D = w.Z[l]; a.Z = zt[l];
        a.alpha = 0.f;
        if ((rc = launch_tc_gemm(w.Ah[l], w.Al[l], ld4(G.K), h->Wf_hi[l], h->Wf_lo[l], ld4(G.K), a, st, true))) return rc;
      }
      for (int j = 0; j + 1 < Ld; ++j) {
        const int in = h->in_w(j), wj = h->fcs[j];
        if (j == 0) conv_gate_split_launch(zt[Lc - 1], cz[Lc], rows, in, w.fAh[0], w.fAl[0], ld4(in), st);
        TcArgs a{};
        a.M = rows; a.N = wj; a.K = in; a.mode = 0; a.tangent = 1; a.D = w.fZ[j]; a.Z = zt[Lc + j]; a.alpha = 0.f;
        if (j + 2 < Ld) { a.Cz_next = cz[Lc + j + 1]; a.nxt_hi = w.fAh[j + 1]; a.nxt_lo = w.fAl[j + 1]; a.nxt_ld = ld4(wj); }
        if ((rc = launch_tc_gemm(w.fAh[j], w.fAl[j], ld4(in), h->Wf_hi[Lc + j], h->Wf_lo[Lc + j], ld4(in), a, st, true))) return rc;
      }
      // ---- dense e_z = delta Wz^T (the backward GEMM without its gating epilogue) ----
      for (int j = 0; j + 1 < Ld; ++j) {
        const int in = h->in_w(j), wj = h->fcs[j];
        TcArgs a{};
        a.M = rows; a.N = in; a.K = wj; a.mode = 2; a.C = ez[Lc + j];
        if ((rc = launch_tc_gemm(w.fdh[j], w.fdl[j], ld4(wj), h->Wb_hi[Lc + j], h->Wb_lo[Lc + j], ld4(wj), a, st))) return rc;
      }
      // ---- hats: zhat = c z + zt, rhat = c r + rt ----
      for (int l = 0; l < Lc; ++l) {
        const ConvGeom& G = h->g[l];
        launch_row_axpy(zt[l], w.Z[l], cc, rows, G.Ho * G.Wo * G.C, st);
        launch_row_axpy(rt[l], l ? w.r[l] : Yc, cc, rows, G.Hi * G.Wi, st);
      }
      for (int j = 0; j + 1 < Ld; ++j) launch_row_axpy(zt[Lc + j], w.fZ[j], cc, rows, h->fcs[j], st);
      ICNN_LAUNCH_CHECK(cudaGetLastError(), "conv_train_grad tangent");

      // ---- weight gradients (float64 over the rows) ----
      for (int l = 0; l < Lc; ++l) {
        const ConvGeom& G = h->g[l];
        const long long M = (long long)rows * G.Ho * G.Wo;
        im2col_plain_kernel<<<nb(M * G.K), 256, 0, st>>>(l ? zt[l - 1] : nullptr, cz[l], rt[l], cy[l], G, rows, w.Ah[l]);
        WgradArgs a{};
        a.M = G.K; a.N = G.C; a.Kb = (int)M; a.A = w.Ah[l]; a.lda = G.K;
        a.D = w.dh[l]; a.Dlo = w.dl[l]; a.ldd = ld4(G.C); a.C64 = acc64 + t.aw[l]; a.ldc = G.C; a.kappa = 1.f;
        a.part = part64;
        launch_wgrad(a, st);
        ICNN_LAUNCH_CHECK(cudaGetLastError(), "conv_train_grad weight gradient");
        if (l + 1 < Lc) {   // acc += the y_red partials in rank order: the reduce of an M = 1 weight gradient
          WgradArgs r{};
          r.M = 1; r.N = G.k * G.k + 1; r.C64 = acc64 + t.ared[l]; r.ldc = r.N; r.kappa = 1.f; r.part = part64;
          const int P = yred_parts(M);
          yred_grad_kernel<<<dim3(r.N, P), 256, 0, st>>>(rt[l], w.rho[l + 1], cc, G, M, part64);
          wgrad_reduce_kernel<double><<<nb(r.N), 256, 0, st>>>(r, P);
          ICNN_LAUNCH_CHECK(cudaGetLastError(), "conv_train_grad y_red gradient");
        }
      }
      for (int j = 0; j < Ld; ++j) {
        const int i = Lc + j;
        WgradArgs a{};
        a.M = h->in_w(j); a.N = h->fcs[j]; a.Kb = rows; a.A = zt[i - 1]; a.G = cz[i]; a.lda = a.M;
        if (j + 1 < Ld) { a.D = w.fdh[j]; a.Dlo = w.fdl[j]; a.ldd = ld4(h->fcs[j]); }
        a.C64 = acc64 + t.aw[i]; a.ldc = a.N; a.kappa = 1.f; a.part = part64;
        launch_wgrad(a, st);
        ICNN_LAUNCH_CHECK(cudaGetLastError(), "conv_train_grad weight gradient");
      }

      // ---- per-sample gate adjoints ----
      auto seg = [&](float* out, SegView a, SegView ev, const float* scale, long long wdt) {
        launch_segsum_prod(out, a, ev, scale, wdt, off_d, u0, u1, r0, r1, st);
      };
      const SegView one{nullptr, nullptr, 0, 1, 0, 0};
      for (int l = 0; l < Lc; ++l) {
        const ConvGeom& G = h->g[l];
        const long long pin = (long long)G.Hi * G.Wi, pout = (long long)G.Ho * G.Wo, er = pin * (G.Cp + 1);
        if (l) seg(gr->dcz[l], SegView{zt[l - 1], nullptr, pin * G.Cp, (int)(pin * G.Cp), 0, 0},
                   SegView{e[l], nullptr, er, G.Cp, G.Cp + 1, 0}, nullptr, pin * G.Cp);
        seg(gr->dcy[l], SegView{rt[l], nullptr, pin, (int)pin, 0, 0}, SegView{e[l], nullptr, er, 1, G.Cp + 1, G.Cp},
            nullptr, pin);
        seg(gr->dd[l], SegView{w.dh[l], w.dl[l], pout * ld4(G.C), G.C, ld4(G.C), 0}, one, c, pout * G.C);
      }
      for (int j = 0; j < Ld; ++j) {
        const int i = Lc + j, in = h->in_w(j), wj = h->fcs[j];
        const SegView zp{zt[i - 1], nullptr, in, in, 0, 0};
        if (j + 1 < Ld) {
          seg(gr->dcz[i], zp, SegView{ez[i], nullptr, in, in, 0, 0}, nullptr, in);
          seg(gr->dd[i], SegView{w.fdh[j], w.fdl[j], ld4(wj), wj, 0, 0}, one, c, wj);
        } else {
          seg(gr->dcz[i], zp, SegView{h->wout, nullptr, 0, in, 0, 0}, nullptr, in);
          seg(gr->dd[i], one, one, c, 1);
        }
      }
      ICNN_LAUNCH_CHECK(cudaGetLastError(), "conv_train_grad segmented sum");
      r0 = r1;
    }
  }

  // ---- the float64 weight-gradient sums, rounded once ----
  for (int l = 0; l < Lc; ++l) {
    const ConvGeom& G = h->g[l];
    conv_unpack_kernel<<<nb((long long)G.K * G.C), 256, 0, st>>>(acc64 + t.aw[l], G.k * G.k, G.Cp, G.C,
                                                                   l ? gr->dWz[l] : nullptr, gr->dWy[l]);
    if (l + 1 < Lc) {
      round_to_float_kernel<<<nb(G.k * G.k), 256, 0, st>>>(gr->dWred[l], acc64 + t.ared[l], G.k * G.k);
      round_to_float_kernel<<<1, 32, 0, st>>>(gr->dbred[l], acc64 + t.ared[l] + G.k * G.k, 1);
    }
  }
  for (int j = 0; j < Ld; ++j) {
    const long long N = (long long)h->in_w(j) * h->fcs[j];
    round_to_float_kernel<<<nb(N), 256, 0, st>>>(gr->dWz[Lc + j], acc64 + t.aw[Lc + j], N);
  }
  ICNN_LAUNCH_CHECK(cudaGetLastError(), "conv_train_grad round");
  return ICNN_OK;
}

extern "C" size_t icnn_conv_gd_backward_workspace_bytes(const icnn_conv_picnn_t* h, int32_t B, int32_t nIter) {
  if (!h || B <= 0 || nIter < 0 || (long long)B * nIter > INT32_MAX) return 0;
  return cgd_layout(h, B, nIter).total;
}

extern "C" int icnn_conv_gd_backward(const icnn_conv_picnn_t* h, const icnn_gates* gates, const float* y0,
                                     const float* trueY, float loss_scale, int32_t nIter, float lr, float momentum,
                                     float* yN, const icnn_conv_train_grads* gr, void* workspace, void* stream) {
  ICNN_REQUIRE(h && gates && y0 && trueY && yN && gr && workspace, "null pointer");
  ICNN_REQUIRE(gr->dWz && gr->dWy && gr->dWred && gr->dbred && gr->dcy && gr->dcz && gr->dd, "null gradient array");
  ICNN_REQUIRE(nIter >= 0, "nIter < 0");
  int rc = conv_check_gates(h, gates);
  if (rc) return rc;
  const int B = gates->B, n = h->H * h->W;
  ICNN_REQUIRE((long long)B * nIter <= INT32_MAX, "B * nIter is more than 2^31 - 1 rows");
  if ((rc = ctg_check_buffers(h, gr))) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const CgdLayout t = cgd_layout(h, B, nIter);
  char* wsb = static_cast<char*>(workspace);
  float* Y = reinterpret_cast<float*>(wsb + t.Y);
  float* V = reinterpret_cast<float*>(wsb + t.V);
  float* c = reinterpret_cast<float*>(wsb + t.c);
  float* kap = reinterpret_cast<float*>(wsb + t.kap);
  float* v = reinterpret_cast<float*>(wsb + t.v);
  float* g = reinterpret_cast<float*>(wsb + t.g);
  float* f = reinterpret_cast<float*>(wsb + t.f);
  void* ws = wsb + t.ws;
  const long long N = (long long)B * n, RN = N * nIter;

  // ---- the GD loop of icnn_conv_gd_solve in yN, recording y_i at row u nIter + i before step i ----
  ICNN_CUDA_CHECK(cudaMemcpyAsync(yN, y0, sizeof(float) * N, cudaMemcpyDeviceToDevice, st));
  ICNN_CUDA_CHECK(cudaMemsetAsync(v, 0, sizeof(float) * N, st));
  for (int it = 0; it < nIter; ++it) {
    ICNN_CUDA_CHECK(cudaMemcpy2DAsync(Y + (size_t)it * n, sizeof(float) * (size_t)nIter * n, yN, sizeof(float) * n,
                                      sizeof(float) * n, B, cudaMemcpyDeviceToDevice, st));
    if ((rc = conv_fg(h, gates, yN, f, g, n, nullptr, nullptr, 0, ws, nullptr, st))) return rc;
    gd_update_launch(yN, v, g, N, lr, momentum, st);
  }

  // ---- row seeds V = kappa_i a, c = 0 ----
  std::vector<float> kappa(nIter > 0 ? nIter : 1, 0.f);
  gd_kappa(nIter, lr, momentum, kappa.data());
  if (nIter > 0) {
    // (pageable source: the call returns once kappa has been staged)
    ICNN_CUDA_CHECK(cudaMemcpyAsync(kap, kappa.data(), sizeof(float) * nIter, cudaMemcpyHostToDevice, st));
    gd_seed_kernel<<<nb(RN), 256, 0, st>>>(V, c, yN, trueY, kap, loss_scale, nIter, n, RN);
    ICNN_LAUNCH_CHECK(cudaGetLastError(), "conv_train_grad GD row seeds");
  }

  // ---- the training gradient of those rows: sample u owns rows [u nIter, (u + 1) nIter) ----
  std::vector<int64_t> off((size_t)B + 1);
  for (int u = 0; u <= B; ++u) off[u] = (int64_t)u * nIter;
  return icnn_conv_train_grad(h, gates, off.data(), Y, V, c, gr, ws, stream);
}
