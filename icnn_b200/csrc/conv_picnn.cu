// Convolutional PICNN f and df/dy (the image-completion energy, completion/icnn_ebundle.py:337-452) on the
// 3xTF32 wgmma GEMM of picnn_tc.cu.
//
//   r_0 = y ;  r_{l+1} = conv_l(r_l; Wred_l) + bred_l                          (1 channel)
//   conv l:   a_l = conv_l([z_{l-1} o cz_l | r_l o cy_l]; [Wz_l | Wy_l]) + d_l,  z_l = relu(a_l)   (no z part at l = 0)
//   dense i:  a_i = (flatNHWC(z_{i-1}) o cz_i) Wz_i + d_i,  z_i = relu(a_i);  the width-1 output is f
// and the backward
//   delta_out = 1 ;  dense: delta_{i-1} = relu'(a_{i-1}) o cz_i o (Wz_i delta_i)
//   conv l:   [e_z | e_r] = conv_l^T(delta_l; [Wz_l | Wy_l]),  delta_{l-1} = relu'(a_{l-1}) o cz_l o e_z
//             rho_l = cy_l o e_r + conv_l^T(rho_{l+1}; Wred_l),  rho_{Lc} = 0,  g = rho_0
//
// Each conv layer is ONE GEMM over K = k^2 (C_{l-1} + 1): the two convolutions of a layer share kernel size, stride
// and output grid, so their weights are concatenated along K per tap (the TensorFlow layout [k, k, c_in, c_out]
// flattened, with the y channel appended to every tap), like K1's Wcat = [Wz; Wy].
//   forward:  gated im2col producer -> A hi/lo [M_l, K_l] -> GEMM (epilogue: + d_l, ReLU -> z_l)
//   backward: GEMM delta_l Wcat_l^T -> columns [M_l, K_l] -> col2im GATHER: every input position sums the output
//             windows covering it in a fixed order (no atomics: bit-reproducible), fused with relu' o cz (delta_{l-1}
//             as the next GEMM's hi/lo operand), cy o e_r and the transposed y_red convolution
// The dense layers are K1's GEMMs with their epilogues; the width-1 output is a per-sample reduction.
#include "conv_picnn.cuh"

#include <cstring>

namespace icnn {

// ---- weight packing ---------------------------------------------------------------------------------------------
// Wcat[kk, o], kk = t (Cp + ych) + c over taps t and input channels c (c = Cp: the y channel when ych = 1):
// Wz [taps, Cp, N] (TF layout) and Wy [taps, 1, N].  Writes both orientations, TF32 hi/lo.
__global__ void conv_pack_kernel(const float* Wz, const float* Wy, int taps, int Cp, int ych, int N, float* bhi,
                                 float* blo, int ldb, float* fhi, float* flo, int ldf) {
  const int K = taps * (Cp + ych);
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)K * N) return;
  const int kk = (int)(i / N), o = (int)(i % N);
  const int t = kk / (Cp + ych), c = kk % (Cp + ych);
  const float w = c < Cp ? Wz[((long long)t * Cp + c) * N + o] : Wy[(long long)t * N + o];
  const float h = tf32_rn(w), l = tf32_rn(w - h);
  bhi[(long long)kk * ldb + o] = h; blo[(long long)kk * ldb + o] = l;
  fhi[(long long)o * ldf + kk] = h; flo[(long long)o * ldf + kk] = l;
}

// ---- forward ----------------------------------------------------------------------------------------------------
// r_{l+1} = conv(r_l; Wred_l) + bred_l, one thread per output pixel, taps in row-major order
__global__ void yred_kernel(const float* r, float* rn, const float* red, ConvGeom g, int B, const int* skip) {
  if (skip != nullptr && *skip == 0) return;
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
  rn[i] = acc + red[g.k * g.k];
}

// gated im2col: A[m, t (Cp+1) + c] = (c < Cp ? z_{l-1} o cz_l : r_l o cy_l) at the input position tap t of output
// pixel m reads (0 in the padding), TF32 hi/lo with row pitch ld4(K)
__global__ void im2col_gate_kernel(const float* Z, const float* cz, const float* r, const float* cy, ConvGeom g,
                                   int B, float* hi, float* lo, const int* skip) {
  if (skip != nullptr && *skip == 0) return;
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
  const float h = tf32_rn(v);
  const long long o = m * ((g.K + 3) & ~3) + kk;     // ld4(K)
  hi[o] = h;
  lo[o] = tf32_rn(v - h);
}

// A[b, e] = Z[b, e] cz[b, e] as TF32 hi/lo with row pitch ld (the first dense layer's operand)
__global__ void gate_split_kernel(const float* Z, const float* cz, int B, int w, float* hi, float* lo, int ld,
                                  const int* skip) {
  if (skip != nullptr && *skip == 0) return;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)B * w) return;
  const float v = Z[i] * cz[i], h = tf32_rn(v);
  const long long o = (i / w) * ld + i % w;
  hi[o] = h;
  lo[o] = tf32_rn(v - h);
}

// width-1 output layer, one CTA per sample: f = (z o cz) . w + d, and its backward seed
// delta = relu'(z) o cz o w as TF32 hi/lo; element e of the sample goes to row (b R + e / rw), column e % rw, pitch ld
// (R = S / rw rows per sample: a dense [B, S] operand has rw = S, a conv feature map [B hw, C] has rw = C)
__global__ void __launch_bounds__(256) conv_out_kernel(const float* Z, const float* cz, const float* w, const float* d,
                                                       int S, int rw, int ld, float* f, float* dhi, float* dlo,
                                                       const int* skip) {
  if (skip != nullptr && *skip == 0) return;
  __shared__ float red[8];
  const int b = blockIdx.x;
  float acc = 0.f;
  for (int e = threadIdx.x; e < S; e += 256) {
    const long long idx = (long long)b * S + e;
    const float z = Z[idx], c = cz[idx] * w[e];
    acc = fmaf(z, c, acc);
    const float dl = z > 0.f ? c : 0.f, h = tf32_rn(dl);
    const long long o = ((long long)b * (S / rw) + e / rw) * ld + e % rw;
    dhi[o] = h;
    dlo[o] = tf32_rn(dl - h);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += red[i];
    f[b] = s + d[b];
  }
}

// [R, C] hi/lo pairs with pitch C -> pitch ld (the last conv layer's delta when C is not a multiple of 4)
__global__ void repitch_kernel(const float* shi, const float* slo, float* dhi, float* dlo, long long R, int C, int ld,
                               const int* skip) {
  if (skip != nullptr && *skip == 0) return;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= R * C) return;
  const long long o = (i / C) * ld + i % C;
  dhi[o] = shi[i];
  dlo[o] = slo[i];
}

// ---- backward ---------------------------------------------------------------------------------------------------
// col2im gather of conv layer l, one thread per (input pixel p, channel c <= Cp):
//   e = sum over the output windows covering p (oy, then ox ascending) of cols[window, tap (Cp+1) + c]
//   c < Cp:  delta_{l-1}[p, c] = relu'(z_{l-1}) cz_l e            -> TF32 hi/lo, row pitch ld4(Cp)
//   c = Cp:  rho_l[p] = cy_l e + sum over the same windows of rho_{l+1} Wred_l[tap]   -> rho (l > 0) or the g row
//   eout != nullptr (training gradient, conv_train_grad.cu): eout[p, c] = e, the un-gated adjoint [e_z | e_r]
__global__ void col2im_kernel(const float* cols, ConvGeom g, int B, const float* Zp, const float* cz, float* dhi,
                              float* dlo, const float* cy, const float* rho_next, const float* wred, float* rho,
                              float* gout, long long g_row_stride, const int* perm, const int* count, int KS, int n,
                              float* eout, const int* skip) {
  if (skip != nullptr && *skip == 0) return;
  const int CC = g.Cp + 1;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)B * g.Hi * g.Wi * CC) return;
  const long long p = i / CC;
  const int c = (int)(i % CC);
  const int ix = (int)(p % g.Wi), iy = (int)((p / g.Wi) % g.Hi), b = (int)(p / ((long long)g.Wi * g.Hi));
  // output rows oy with 0 <= iy + pt - oy s < k
  const int ty = iy + g.pt, tx = ix + g.pl;
  const int oy0 = ty - g.k + 1 > 0 ? (ty - g.k + g.s) / g.s : 0, oy1 = min(g.Ho - 1, ty / g.s);
  const int ox0 = tx - g.k + 1 > 0 ? (tx - g.k + g.s) / g.s : 0, ox1 = min(g.Wo - 1, tx / g.s);
  const bool ych = c == g.Cp;
  float e = 0.f, rr = 0.f;
  for (int oy = oy0; oy <= oy1; ++oy) {
    const int ky = ty - oy * g.s;
    for (int ox = ox0; ox <= ox1; ++ox) {
      const int kx = tx - ox * g.s;
      const long long mo = ((long long)b * g.Ho + oy) * g.Wo + ox;
      e += cols[mo * g.K + (ky * g.k + kx) * CC + c];
      if (ych && rho_next) rr = fmaf(rho_next[mo], wred[ky * g.k + kx], rr);
    }
  }
  if (eout) eout[i] = e;
  if (!ych) {
    const long long idx = p * g.Cp + c;
    const float v = Zp[idx] > 0.f ? cz[idx] * e : 0.f, h = tf32_rn(v);
    const long long o = p * ((g.Cp + 3) & ~3) + c;    // ld4(Cp)
    dhi[o] = h;
    dlo[o] = tf32_rn(v - h);
  } else {
    const float v = fmaf(cy[p], e, rr);
    if (rho) {
      rho[p] = v;
    } else {
      float* grow = perm == nullptr ? gout + (long long)b * g_row_stride
                                    : gout + ((long long)b * KS + perm[(long long)b * KS + count[b]]) * n;
      grow[iy * g.Wi + ix] = v;
    }
  }
}

// ---- workspace ----------------------------------------------------------------------------------------------------
// floats of workspace for B rows; with base != nullptr also the buffer addresses
size_t conv_ws_floats(const icnn_conv_picnn* h, int B, float* base, ConvWs* w) {
  size_t off = 0;
  auto take = [&](size_t nfl) { const size_t o = off; off += (nfl + 63) & ~(size_t)63; return base ? base + o : nullptr; };
  size_t cmax = 0;
  for (int l = 0; l < h->Lc; ++l) {
    const ConvGeom& g = h->g[l];
    const size_t M = (size_t)B * g.Ho * g.Wo;
    w->Ah[l] = take(M * ld4(g.K)); w->Al[l] = take(M * ld4(g.K)); w->Z[l] = take(M * g.C);
    w->dh[l] = take(M * ld4(g.C)); w->dl[l] = take(M * ld4(g.C));
    w->r[l] = l ? take((size_t)B * g.Hi * g.Wi) : nullptr;
    w->rho[l] = l ? take((size_t)B * g.Hi * g.Wi) : nullptr;
    cmax = M * g.K > cmax ? M * g.K : cmax;
  }
  w->cols = take(cmax);
  for (int j = 0; j + 1 < h->Ld; ++j) {
    w->fAh[j] = take((size_t)B * ld4(h->in_w(j))); w->fAl[j] = take((size_t)B * ld4(h->in_w(j)));
    w->fZ[j] = take((size_t)B * h->fcs[j]);
    w->fdh[j] = take((size_t)B * ld4(h->fcs[j])); w->fdl[j] = take((size_t)B * ld4(h->fcs[j]));
  }
  const bool rp = h->Ld > 1 && h->g[h->Lc - 1].C % 4 != 0;
  w->th = rp ? take((size_t)B * h->flat) : nullptr;
  w->tl = rp ? take((size_t)B * h->flat) : nullptr;
  return off;
}

static inline unsigned nblk(long long n) { return (unsigned)((n + 255) / 256); }

int conv_fg(const icnn_conv_picnn* h, const icnn_gates* gt, const float* y32, float* f, float* g,
            long long g_row_stride, const int* perm, const int* count, int KS, void* workspace, const int* skip,
            cudaStream_t st, float* const* eout) {
  const int B = gt->B, Lc = h->Lc, Ld = h->Ld, n = h->H * h->W;
  ConvWs w{};
  conv_ws_floats(h, B, static_cast<float*>(workspace), &w);
  int rc;
  // ---- forward: conv layers ----
  for (int l = 0; l < Lc; ++l) {
    const ConvGeom& G = h->g[l];
    const float* r = l ? w.r[l] : y32;
    if (l + 1 < Lc)   // r_{Lc} is never used
      yred_kernel<<<nblk((long long)B * G.Ho * G.Wo), 256, 0, st>>>(r, w.r[l + 1], h->red[l], G, B, skip);
    const long long M = (long long)B * G.Ho * G.Wo;
    im2col_gate_kernel<<<nblk(M * G.K), 256, 0, st>>>(l ? w.Z[l - 1] : nullptr, gt->cz[l], r, gt->cy[l], G, B,
                                                      w.Ah[l], w.Al[l], skip);
    TcArgs a{};
    a.M = (int)M; a.N = G.C; a.K = G.K; a.mode = 0; a.D = gt->d[l]; a.Z = w.Z[l]; a.alpha = 0.f; a.skip_if_zero = skip;
    if ((rc = launch_tc_gemm(w.Ah[l], w.Al[l], ld4(G.K), h->Wf_hi[l], h->Wf_lo[l], ld4(G.K), a, st))) return rc;
  }
  // ---- forward: dense hidden layers ----
  const ConvGeom& GL = h->g[Lc - 1];
  const float* Zlast = w.Z[Lc - 1];
  for (int j = 0; j + 1 < Ld; ++j) {
    const int in = h->in_w(j), wj = h->fcs[j];
    if (j == 0)
      gate_split_kernel<<<nblk((long long)B * in), 256, 0, st>>>(Zlast, gt->cz[Lc], B, in, w.fAh[0], w.fAl[0], ld4(in), skip);
    TcArgs a{};
    a.M = B; a.N = wj; a.K = in; a.mode = 0; a.D = gt->d[Lc + j]; a.Z = w.fZ[j]; a.alpha = 0.f; a.skip_if_zero = skip;
    if (j + 2 < Ld) { a.Cz_next = gt->cz[Lc + j + 1]; a.nxt_hi = w.fAh[j + 1]; a.nxt_lo = w.fAl[j + 1]; a.nxt_ld = ld4(wj); }
    if ((rc = launch_tc_gemm(w.fAh[j], w.fAl[j], ld4(in), h->Wf_hi[Lc + j], h->Wf_lo[Lc + j], ld4(in), a, st))) return rc;
    Zlast = w.fZ[j];
  }
  // ---- width-1 output and its backward seed ----
  {
    const int S = h->in_w(Ld - 1);
    float *sh, *sl;
    int rw, ld;
    if (Ld > 1) { sh = w.fdh[Ld - 2]; sl = w.fdl[Ld - 2]; rw = S; ld = ld4(S); }
    else { sh = w.dh[Lc - 1]; sl = w.dl[Lc - 1]; rw = GL.C; ld = ld4(GL.C); }
    conv_out_kernel<<<B, 256, 0, st>>>(Zlast, gt->cz[Lc + Ld - 1], h->wout, gt->d[Lc + Ld - 1], S, rw, ld, f, sh, sl, skip);
  }
  // ---- backward: dense hidden layers ----
  for (int j = Ld - 2; j >= 0; --j) {
    const int in = h->in_w(j), wj = h->fcs[j];
    TcArgs a{};
    a.M = B; a.N0 = in; a.N = in; a.K = wj; a.mode = 1; a.alpha = 0.f; a.n = 0; a.g_scale = 1.f; a.skip_if_zero = skip;
    a.Cz = gt->cz[Lc + j];
    if (j > 0) {
      a.Zprev = w.fZ[j - 1]; a.dprev_hi = w.fdh[j - 1]; a.dprev_lo = w.fdl[j - 1]; a.dprev_ld = ld4(in);
    } else {   // delta of the last conv layer's map: [B, flat] = [B hw, C] at pitch C
      a.Zprev = w.Z[Lc - 1]; a.dprev_ld = in;
      a.dprev_hi = w.th ? w.th : w.dh[Lc - 1]; a.dprev_lo = w.tl ? w.tl : w.dl[Lc - 1];
    }
    if ((rc = launch_tc_gemm(w.fdh[j], w.fdl[j], ld4(wj), h->Wb_hi[Lc + j], h->Wb_lo[Lc + j], ld4(wj), a, st))) return rc;
  }
  if (w.th)
    repitch_kernel<<<nblk((long long)B * h->flat), 256, 0, st>>>(w.th, w.tl, w.dh[Lc - 1], w.dl[Lc - 1],
                                                                 (long long)B * GL.Ho * GL.Wo, GL.C, ld4(GL.C), skip);
  // ---- backward: conv layers ----
  for (int l = Lc - 1; l >= 0; --l) {
    const ConvGeom& G = h->g[l];
    const long long M = (long long)B * G.Ho * G.Wo;
    TcArgs a{};
    a.M = (int)M; a.N = G.K; a.K = G.C; a.mode = 2; a.C = w.cols; a.skip_if_zero = skip;
    if ((rc = launch_tc_gemm(w.dh[l], w.dl[l], ld4(G.C), h->Wb_hi[l], h->Wb_lo[l], ld4(G.C), a, st))) return rc;
    col2im_kernel<<<nblk((long long)B * G.Hi * G.Wi * (G.Cp + 1)), 256, 0, st>>>(
        w.cols, G, B, l ? w.Z[l - 1] : nullptr, gt->cz[l], l ? w.dh[l - 1] : nullptr, l ? w.dl[l - 1] : nullptr,
        gt->cy[l], l + 1 < Lc ? w.rho[l + 1] : nullptr, h->red[l], l ? w.rho[l] : nullptr, g, g_row_stride, perm,
        count, KS, n, eout ? eout[l] : nullptr, skip);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_error("conv_picnn_fg launch: %s", cudaGetErrorString(e)); return ICNN_E_CUDA; }
  return ICNN_OK;
}

void conv_im2col_gate_launch(const float* Z, const float* cz, const float* r, const float* cy, const ConvGeom& g,
                             int B, float* hi, float* lo, cudaStream_t st) {
  im2col_gate_kernel<<<nblk((long long)B * g.Ho * g.Wo * g.K), 256, 0, st>>>(Z, cz, r, cy, g, B, hi, lo, nullptr);
}

void conv_gate_split_launch(const float* Z, const float* cz, int B, int w, float* hi, float* lo, int ld,
                            cudaStream_t st) {
  gate_split_kernel<<<nblk((long long)B * w), 256, 0, st>>>(Z, cz, B, w, hi, lo, ld, nullptr);
}

int conv_check_gates(const icnn_conv_picnn* h, const icnn_gates* gt) {
  ICNN_REQUIRE(gt->B > 0, "empty batch");
  ICNN_REQUIRE(gt->cy && gt->cz && gt->d, "null gate array");
  ICNN_REQUIRE(gt->in_scale == 1.f && gt->in_shift == 0.f && gt->g_scale == 1.f,
               "the conv PICNN has no affine input wrapper: in_scale, in_shift, g_scale must be (1, 0, 1)");
  for (int l = 0; l < h->Lc + h->Ld; ++l) {
    ICNN_REQUIRE(gt->d[l], "null gate d");
    ICNN_REQUIRE(l >= h->Lc || gt->cy[l], "null gate cy on a conv layer");
    ICNN_REQUIRE(l == 0 || gt->cz[l], "null gate cz");
  }
  return ICNN_OK;
}

}  // namespace icnn

using namespace icnn;

extern "C" int icnn_conv_picnn_destroy(icnn_conv_picnn_t* h) {
  if (!h) return ICNN_OK;
  for (int i = 0; i < 2 * ICNN_MAX_LAYERS; ++i)
    for (float* p : {h->Wf_hi[i], h->Wf_lo[i], h->Wb_hi[i], h->Wb_lo[i]})
      if (p) cudaFree(p);
  for (int l = 0; l < ICNN_MAX_LAYERS; ++l)
    if (h->red[l]) cudaFree(h->red[l]);
  if (h->wout) cudaFree(h->wout);
  delete h;
  return ICNN_OK;
}

extern "C" int icnn_conv_picnn_create(const icnn_conv_picnn_desc* d, icnn_conv_picnn_t** out, void* stream) {
  ICNN_REQUIRE(d && out, "null descriptor");
  ICNN_REQUIRE(d->H >= 1 && d->W >= 1, "H and W must be positive");
  ICNN_REQUIRE(d->Lc >= 1 && d->Lc <= ICNN_MAX_LAYERS, "Lc must be in [1, 8]");
  ICNN_REQUIRE(d->Ld >= 1 && d->Ld <= ICNN_MAX_LAYERS, "Ld must be in [1, 8]");
  ICNN_REQUIRE(d->C && d->k && d->s && d->fcs && d->Wz && d->Wy && d->Wred && d->bred, "null array");
  ICNN_REQUIRE(d->fcs[d->Ld - 1] == 1, "the last dense layer must have width 1");
  for (int l = 0; l < d->Lc; ++l) {
    ICNN_REQUIRE(d->C[l] >= 1 && d->k[l] >= 1 && d->s[l] >= 1, "conv (C, k, s) must be positive");
    ICNN_REQUIRE(d->Wy[l] && d->Wred[l] && d->bred[l] && (l == 0 || d->Wz[l]), "null conv weight pointer");
  }
  for (int j = 0; j < d->Ld; ++j) {
    ICNN_REQUIRE(d->fcs[j] >= 1, "dense widths must be positive");
    ICNN_REQUIRE(d->Wz[d->Lc + j], "null dense weight pointer");
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  icnn_conv_picnn* h = new icnn_conv_picnn();
  memset(h, 0, sizeof(*h));
  h->H = d->H; h->W = d->W; h->Lc = d->Lc; h->Ld = d->Ld;
  for (int j = 0; j < d->Ld; ++j) h->fcs[j] = d->fcs[j];
  int Hi = d->H, Wi = d->W, Cp = 0;
  for (int l = 0; l < d->Lc; ++l) {
    ConvGeom& g = h->g[l];
    g.C = d->C[l]; g.k = d->k[l]; g.s = d->s[l]; g.Cp = Cp; g.Hi = Hi; g.Wi = Wi;
    g.Ho = (Hi + g.s - 1) / g.s; g.Wo = (Wi + g.s - 1) / g.s;
    const int th = (g.Ho - 1) * g.s + g.k - Hi, tw = (g.Wo - 1) * g.s + g.k - Wi;
    g.pt = th > 0 ? th / 2 : 0; g.pl = tw > 0 ? tw / 2 : 0;
    g.K = g.k * g.k * (Cp + 1);
    Hi = g.Ho; Wi = g.Wo; Cp = g.C;
  }
  h->flat = Hi * Wi * Cp;
  auto alloc = [&](float** p, size_t nfl) { return cudaMalloc(p, sizeof(float) * nfl) == cudaSuccess; };
  bool ok = true;
  for (int l = 0; l < d->Lc && ok; ++l) {
    const ConvGeom& g = h->g[l];
    ok = alloc(&h->Wb_hi[l], (size_t)g.K * ld4(g.C)) && alloc(&h->Wb_lo[l], (size_t)g.K * ld4(g.C)) &&
         alloc(&h->Wf_hi[l], (size_t)g.C * ld4(g.K)) && alloc(&h->Wf_lo[l], (size_t)g.C * ld4(g.K)) &&
         alloc(&h->red[l], (size_t)g.k * g.k + 1);
    if (!ok) break;
    conv_pack_kernel<<<nblk((long long)g.K * g.C), 256, 0, st>>>(d->Wz[l], d->Wy[l], g.k * g.k, g.Cp, 1, g.C,
                                                                 h->Wb_hi[l], h->Wb_lo[l], ld4(g.C), h->Wf_hi[l],
                                                                 h->Wf_lo[l], ld4(g.K));
    cudaMemcpyAsync(h->red[l], d->Wred[l], sizeof(float) * g.k * g.k, cudaMemcpyDeviceToDevice, st);
    cudaMemcpyAsync(h->red[l] + g.k * g.k, d->bred[l], sizeof(float), cudaMemcpyDeviceToDevice, st);
  }
  for (int j = 0; j + 1 < d->Ld && ok; ++j) {
    const int in = h->in_w(j), wj = h->fcs[j], i = d->Lc + j;
    ok = alloc(&h->Wb_hi[i], (size_t)in * ld4(wj)) && alloc(&h->Wb_lo[i], (size_t)in * ld4(wj)) &&
         alloc(&h->Wf_hi[i], (size_t)wj * ld4(in)) && alloc(&h->Wf_lo[i], (size_t)wj * ld4(in));
    if (!ok) break;
    conv_pack_kernel<<<nblk((long long)in * wj), 256, 0, st>>>(d->Wz[i], nullptr, 1, in, 0, wj, h->Wb_hi[i],
                                                               h->Wb_lo[i], ld4(wj), h->Wf_hi[i], h->Wf_lo[i], ld4(in));
  }
  if (ok) {
    const int in = h->in_w(d->Ld - 1);
    ok = alloc(&h->wout, in);
    if (ok) cudaMemcpyAsync(h->wout, d->Wz[d->Lc + d->Ld - 1], sizeof(float) * in, cudaMemcpyDeviceToDevice, st);
  }
  if (!ok) { icnn_conv_picnn_destroy(h); set_error("cudaMalloc conv weights failed"); return ICNN_E_CUDA; }
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) { icnn_conv_picnn_destroy(h); set_error("conv_picnn_create: %s", cudaGetErrorString(e)); return ICNN_E_CUDA; }
  *out = h;
  return ICNN_OK;
}

extern "C" size_t icnn_conv_picnn_workspace_bytes(const icnn_conv_picnn_t* h, int32_t B) {
  if (!h || B <= 0) return 0;
  ConvWs w{};
  return sizeof(float) * conv_ws_floats(h, B, nullptr, &w);
}

extern "C" int icnn_conv_picnn_fg(const icnn_conv_picnn_t* h, const icnn_gates* gates, const float* y32, float* f,
                                  float* g, int64_t g_row_stride, const int32_t* perm, const int32_t* count,
                                  int32_t KS, void* workspace, const int32_t* skip_if_zero, void* stream) {
  ICNN_REQUIRE(h && gates && y32 && f && g && workspace, "null pointer");
  ICNN_REQUIRE((perm == nullptr) == (count == nullptr), "perm and count go together");
  int rc = conv_check_gates(h, gates);
  if (rc) return rc;
  return conv_fg(h, gates, y32, f, g, g_row_stride, perm, count, KS, workspace, skip_if_zero,
                 static_cast<cudaStream_t>(stream));
}

extern "C" int icnn_conv_solve_batch_fused(const icnn_conv_picnn_t* h, const icnn_gates* gates,
                                           const icnn_bundle_cfg* cfg, const icnn_bundle_bufs* b, void* workspace,
                                           void* stream) {
  ICNN_REQUIRE(h && gates && cfg && b && workspace, "null pointer");
  ICNN_REQUIRE(gates->B == b->B, "gates.B != bufs.B");
  ICNN_REQUIRE(h->H * h->W == b->n, "H * W != bufs.n");
  ICNN_REQUIRE(cfg->nIter >= 1, "nIter < 1");
  ICNN_REQUIRE(b->KS >= 2, "KS < 2");
  int rc = conv_check_gates(h, gates);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if ((rc = icnn_bundle_init(b, cfg->nIter, stream))) return rc;
  for (int t = 0; t < cfg->nIter; ++t) {
    if ((rc = conv_fg(h, gates, b->y32, b->f, b->G, 0, b->perm, b->count, b->KS, workspace, b->nactive + t, st))) return rc;
    if ((rc = icnn_bundle_step(cfg, b, t, stream))) return rc;
  }
  return ICNN_OK;
}

extern "C" int icnn_conv_gd_solve(const icnn_conv_picnn_t* h, const icnn_gates* gates, float* y32, float* v, float* g,
                                  float* f_out, int32_t nIter, float lr, float momentum, void* workspace,
                                  void* stream) {
  ICNN_REQUIRE(h && gates && y32 && v && g && f_out && workspace, "null pointer");
  ICNN_REQUIRE(nIter >= 0, "nIter < 0");
  int rc = conv_check_gates(h, gates);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int n = h->H * h->W;
  const long long N = (long long)gates->B * n;
  ICNN_CUDA_CHECK(cudaMemsetAsync(v, 0, sizeof(float) * N, st));
  for (int it = 0; it < nIter; ++it) {
    if ((rc = conv_fg(h, gates, y32, f_out, g, n, nullptr, nullptr, 0, workspace, nullptr, st))) return rc;
    gd_update_launch(y32, v, g, N, lr, momentum, st);
  }
  if ((rc = conv_fg(h, gates, y32, f_out, g, n, nullptr, nullptr, 0, workspace, nullptr, st))) return rc;
  ICNN_CUDA_CHECK(cudaGetLastError());
  return ICNN_OK;
}
