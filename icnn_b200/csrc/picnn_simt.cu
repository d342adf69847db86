// K1 (baseline): fully-connected PICNN energy f and df/dy for a whole minibatch, FP32 FFMA.
//
// Restates on the GPU what the reference evaluates through TensorFlow:
//   forward   multi-label-cls/icnn_ebundle.py:349-387, RL/src/icnn.py:356-404
//   gradient  tf.gradients(E_, y_)  (multi-label-cls/icnn_ebundle.py:146)
//
//   a_i = (z_{i-1} o cz_i) Wz_i + (y o cy_i) Wy_i + d_i ,  z_i = act(a_i) (i < L),  f = a_L
//   delta_L = 1 ;  g += cy_i o (delta_i Wy_i^T) ;  delta_{i-1} = act'(a_{i-1}) o cz_i o (delta_i Wz_i^T)
//
// Each hidden layer is one gated GEMM against Wcat_i = [Wz_i ; Wy_i] (forward: K-concatenated,
// backward: the same buffer read transposed), with the per-sample gates applied while the A tile
// is staged and bias/activation/act'-mask/g-accumulate fused into the epilogue.  The width-1
// output layer and its backward seed are a warp-per-sample kernel (shuffle reduction).
// This FP32 kernel is the accuracy anchor for the wgmma path (picnn_tc.cu).
#include "gated_gemm.cuh"

#include <cstdlib>

namespace icnn {

struct OutArgs {
  int M, S, n;                  // S = s_{L-1}
  const float* Z; const float* Cz;      // [M, S]
  const float* y; const float* Cy;      // [M, n]
  const float* D;                        // [M]
  const float* w;                        // [S + n]  = [wz_L ; wy_L]
  float in_scale, in_shift, g_scale, alpha;
  float* f; float* delta;                // [M], [M, S]
  float* delta_hi; float* delta_lo; int delta_ld;   // optional TF32 hi/lo split of delta (tensor-core path, row pitch ld4(S))
  float* g; long long g_row_stride; const int* perm; const int* count; int KS;
  const int* skip_if_zero;
};

// TPS threads per sample (32 = a warp, 256 = a CTA for small batches where a warp per sample is
// latency-bound): f = d_L + (z o cz_L).wz_L + (y o cy_L).wy_L ; seeds delta_{L-1} and g.
template <int TPS>
__global__ void __launch_bounds__(256) out_layer_kernel(OutArgs a) {
  if (a.skip_if_zero != nullptr && *a.skip_if_zero == 0) return;
  __shared__ float red[8];
  const int m = (int)((blockIdx.x * (long long)blockDim.x + threadIdx.x) / TPS);
  const int tl = threadIdx.x % TPS;
  const int lane = threadIdx.x & 31;
  const bool mv = m < a.M;
  float acc = 0.f;
  if (mv) {
    for (int j = tl; j < a.S; j += TPS) {
      const long long idx = (long long)m * a.S + j;
      const float z = a.Z[idx], c = a.Cz[idx] * a.w[j];
      acc = fmaf(z, c, acc);
      const float dl = (z > 0.f ? 1.f : a.alpha) * c;
      if (a.delta) a.delta[idx] = dl;
      if (a.delta_hi) {
        // TF32 hi/lo with round-to-nearest on both parts
        const float h = tf32_rn(dl);
        const long long o = (long long)m * a.delta_ld + j;
        a.delta_hi[o] = h;
        a.delta_lo[o] = tf32_rn(dl - h);
      }
    }
    float* grow;
    if (a.perm == nullptr) grow = a.g + (long long)m * a.g_row_stride;
    else grow = a.g + ((long long)m * a.KS + a.perm[(long long)m * a.KS + a.count[m]]) * a.n;
    for (int e = tl; e < a.n; e += TPS) {
      const long long idx = (long long)m * a.n + e;
      const float c = a.Cy[idx] * a.w[a.S + e];
      acc = fmaf(fmaf(a.in_scale, a.y[idx], a.in_shift), c, acc);
      grow[e] = a.g_scale * c;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (TPS == 32) {
    if (mv && lane == 0) a.f[m] = acc + a.D[m];
  } else {   // TPS == 256: one sample per CTA, fixed-order sum of the 8 warp partials
    if (lane == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0 && mv) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) s += red[w];
      a.f[m] = s + a.D[m];
    }
  }
}

__global__ void concat_rows_kernel(float* dst, const float* top, long long ntop, const float* bot,
                                   long long nbot) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < ntop) dst[i] = top[i];
  else if (i < ntop + nbot) dst[i] = bot[i - ntop];
}

// workspace layout: Z_0..Z_{L-1} [B, s_i], then two delta buffers [B, smax]
size_t picnn_simt_ws_floats(const icnn_picnn* h, int B, size_t* zoff, size_t* doff) {
  size_t off = 0;
  int smax = 0;
  for (int i = 0; i < h->L; ++i) {
    if (zoff) zoff[i] = off;
    off += (size_t)B * h->hidden[i];
    off = (off + 63) & ~(size_t)63;
    smax = h->hidden[i] > smax ? h->hidden[i] : smax;
  }
  if (doff) { doff[0] = off; doff[1] = off + (((size_t)B * smax + 63) & ~(size_t)63); }
  off += 2 * (((size_t)B * smax + 63) & ~(size_t)63);
  return off;
}

void out_layer_launch(const icnn_picnn* h, const icnn_gates* gt, const float* Zlast, const float* y32, float* f,
                      float* delta, float* delta_hi, float* delta_lo, float* g, long long g_row_stride,
                      const int* perm, const int* count, int KS, const int* skip, cudaStream_t st) {
  const int B = gt->B, L = h->L;
  OutArgs o{};
  o.M = B; o.S = h->hidden[L - 1]; o.n = h->n; o.Z = Zlast; o.Cz = gt->cz[L]; o.y = y32; o.Cy = gt->cy[L];
  o.D = gt->d[L]; o.w = h->Wcat[L]; o.in_scale = gt->in_scale; o.in_shift = gt->in_shift;
  o.g_scale = gt->g_scale; o.alpha = h->alpha; o.f = f; o.delta = delta; o.delta_hi = delta_hi; o.delta_lo = delta_lo; o.delta_ld = ld4(o.S);
  o.g = g; o.g_row_stride = g_row_stride; o.perm = perm; o.count = count; o.KS = KS; o.skip_if_zero = skip;
  if (B <= 2048) out_layer_kernel<256><<<B, 256, 0, st>>>(o);          // few samples: a CTA each
  else out_layer_kernel<32><<<cdiv(B * 32, 256), 256, 0, st>>>(o);
}

// host launcher of gd_update_kernel for the other translation units (conv_picnn.cu; declared in tc_gemm.cuh)
void gd_update_launch(float* y, float* v, const float* g, long long N, float lr, float mom, cudaStream_t st) {
  gd_update_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(y, v, g, N, lr, mom);
}

bool picnn_tc_supported(const icnn_picnn* h);
int picnn_tc_prepare_weights(icnn_picnn* h, cudaStream_t st);
void picnn_tc_free_weights(icnn_picnn* h);
void picnn_xpath_free(icnn_picnn* h);
size_t picnn_tc_ws_floats(const icnn_picnn* h, int B, size_t* aoff, size_t* doff);
int picnn_fg_tc(const icnn_picnn* h, const icnn_gates* gt, const float* y32, float* f, float* g,
                long long g_row_stride, const int* perm, const int* count, int KS, void* workspace,
                const int* skip, cudaStream_t st);

int picnn_fg_simt(const icnn_picnn* h, const icnn_gates* gt, const float* y32, float* f, float* g,
                  long long g_row_stride, const int* perm, const int* count, int KS, void* workspace,
                  const int* skip, cudaStream_t st) {
  const int B = gt->B, n = h->n, L = h->L;
  size_t zoff[ICNN_MAX_LAYERS], doff[2];
  picnn_simt_ws_floats(h, B, zoff, doff);
  float* ws = static_cast<float*>(workspace);
  float* Z[ICNN_MAX_LAYERS];
  for (int i = 0; i < L; ++i) Z[i] = ws + zoff[i];
  float* dl[2] = {ws + doff[0], ws + doff[1]};

  for (int i = 0; i < L; ++i) {  // forward hidden layers
    GemmArgs a{};
    a.M = B; a.N = h->hidden[i]; a.K0 = h->prev(i); a.K1 = n;
    a.A0 = i ? Z[i - 1] : nullptr; a.G0 = i ? gt->cz[i] : nullptr; a.lda0 = a.K0;
    a.A1 = y32; a.G1 = gt->cy[i]; a.lda1 = n; a.a1_scale = gt->in_scale; a.a1_shift = gt->in_shift;
    a.W = h->Wcat[i]; a.ldw = a.N;
    a.D = gt->d[i]; a.Z = Z[i]; a.alpha = h->alpha; a.skip_if_zero = skip;
    cudaError_t le = launch_gemm<0>(a, st);
    if (le != cudaSuccess) { set_error("gated_gemm<0> launch: %s", cudaGetErrorString(le)); return ICNN_E_CUDA; }
  }
  out_layer_launch(h, gt, Z[L - 1], y32, f, dl[0], nullptr, nullptr, g, g_row_stride, perm, count, KS, skip, st);
  int cur = 0;
  for (int i = L - 1; i >= 0; --i) {  // backward hidden layers
    GemmArgs a{};
    a.M = B; a.N0 = h->prev(i); a.N = a.N0 + n; a.K0 = h->hidden[i]; a.K1 = 0;
    a.A0 = dl[cur]; a.G0 = nullptr; a.lda0 = a.K0;
    a.W = h->Wcat[i]; a.ldw = a.K0; a.alpha = h->alpha;
    a.Zprev = i ? Z[i - 1] : nullptr; a.Cz = i ? gt->cz[i] : nullptr; a.dprev = dl[cur ^ 1];
    a.Cy = gt->cy[i]; a.g = g; a.g_row_stride = g_row_stride; a.perm = perm; a.count = count; a.KS = KS;
    a.n = n; a.g_scale = gt->g_scale; a.skip_if_zero = skip;
    cudaError_t le = launch_gemm<1>(a, st);
    if (le != cudaSuccess) { set_error("gated_gemm<1> launch: %s", cudaGetErrorString(le)); return ICNN_E_CUDA; }
    cur ^= 1;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_error("picnn_fg launch: %s", cudaGetErrorString(e)); return ICNN_E_CUDA; }
  return ICNN_OK;
}

// K1 dispatch: wgmma path once there are enough rows to fill a 128-row tile, FP32 FFMA path
// otherwise.  ICNN_K1=simt at handle creation keeps everything on the FFMA path.
int picnn_fg_dispatch(const icnn_picnn* h, const icnn_gates* gt, const float* y32, float* f, float* g,
                      long long g_row_stride, const int* perm, const int* count, int KS, void* workspace,
                      const int* skip, cudaStream_t st) {
  if (h->use_tc && gt->B >= 64)
    return picnn_fg_tc(h, gt, y32, f, g, g_row_stride, perm, count, KS, workspace, skip, st);
  return picnn_fg_simt(h, gt, y32, f, g, g_row_stride, perm, count, KS, workspace, skip, st);
}

}  // namespace icnn

using namespace icnn;

extern "C" int icnn_picnn_create(const icnn_picnn_desc* d, icnn_picnn_t** out, void* stream) {
  ICNN_REQUIRE(d && out, "null descriptor");
  ICNN_REQUIRE(d->L >= 1 && d->L <= ICNN_MAX_LAYERS, "L must be in [1, 8]");
  ICNN_REQUIRE(d->n >= 1, "n must be positive");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  icnn_picnn* h = new icnn_picnn();
  h->n = d->n; h->L = d->L; h->alpha = d->alpha;
  for (int i = 0; i < d->L; ++i) {
    if (d->hidden[i] < 1) { delete h; set_error("hidden width must be positive"); return ICNN_E_INVALID; }
    h->hidden[i] = d->hidden[i];
  }
  for (int i = 0; i <= d->L; ++i) h->Wcat[i] = nullptr;
  for (int i = 0; i < ICNN_MAX_LAYERS; ++i) h->Wb_hi[i] = h->Wb_lo[i] = h->Wf_hi[i] = h->Wf_lo[i] = nullptr;
  h->use_tc = false;
  h->m = 0; h->has_xpath = false;
  for (int i = 0; i <= ICNN_MAX_LAYERS; ++i) h->Xw_hi[i] = h->Xw_lo[i] = h->Xbias[i] = nullptr;
  for (int i = 0; i <= d->L; ++i) {
    const long long si = h->width(i), sp = h->prev(i);
    const long long ntop = sp * si, nbot = (long long)h->n * si;
    if (!d->Wy[i] || (i > 0 && !d->Wz[i])) { icnn_picnn_destroy(h); set_error("null weight pointer, layer %d", i); return ICNN_E_INVALID; }
    cudaError_t e = cudaMalloc(&h->Wcat[i], sizeof(float) * (ntop + nbot));
    if (e != cudaSuccess) { icnn_picnn_destroy(h); set_error("cudaMalloc weights: %s", cudaGetErrorString(e)); return ICNN_E_CUDA; }
    const long long tot = ntop + nbot;
    concat_rows_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(h->Wcat[i], d->Wz[i], ntop, d->Wy[i], nbot);
  }
  {
    const char* k1 = getenv("ICNN_K1");
    const bool want = !(k1 && k1[0] == 's');
    if (want && picnn_tc_supported(h)) {
      int rc = picnn_tc_prepare_weights(h, st);
      if (rc) { icnn_picnn_destroy(h); return rc; }
      h->use_tc = true;
    } else if (k1 && k1[0] == 't') {
      icnn_picnn_destroy(h); set_error("ICNN_K1=tc but cuTensorMapEncodeTiled is unavailable"); return ICNN_E_UNSUPPORTED;
    }
  }
  cudaError_t e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) { icnn_picnn_destroy(h); set_error("picnn_create: %s", cudaGetErrorString(e)); return ICNN_E_CUDA; }
  *out = h;
  return ICNN_OK;
}

extern "C" int icnn_picnn_destroy(icnn_picnn_t* h) {
  if (!h) return ICNN_OK;
  for (int i = 0; i <= h->L && i <= ICNN_MAX_LAYERS; ++i)
    if (h->Wcat[i]) cudaFree(h->Wcat[i]);
  picnn_tc_free_weights(h);
  picnn_xpath_free(h);
  delete h;
  return ICNN_OK;
}

extern "C" size_t icnn_picnn_workspace_bytes(const icnn_picnn_t* h, int32_t B) {
  if (!h || B <= 0) return 0;
  return sizeof(float) * (picnn_simt_ws_floats(h, B, nullptr, nullptr) +
                          (h->use_tc ? picnn_tc_ws_floats(h, B, nullptr, nullptr) : 0));
}

extern "C" int icnn_picnn_fg(const icnn_picnn_t* h, const icnn_gates* gates, const float* y32, float* f,
                             float* g, int64_t g_row_stride, const int32_t* perm, const int32_t* count,
                             int32_t KS, void* workspace, const int32_t* skip_if_zero, void* stream) {
  ICNN_REQUIRE(h && gates && y32 && f && g && workspace, "null pointer");
  ICNN_REQUIRE(gates->B > 0, "empty batch");
  ICNN_REQUIRE((perm == nullptr) == (count == nullptr), "perm and count go together");
  return picnn_fg_dispatch(h, gates, y32, f, g, g_row_stride, perm, count, KS, workspace, skip_if_zero,
                           static_cast<cudaStream_t>(stream));
}

extern "C" int icnn_gd_solve(const icnn_picnn_t* h, const icnn_gates* gates, float* y32, float* v, float* g,
                             float* f_out, int32_t nIter, float lr, float momentum, void* workspace,
                             void* stream) {
  ICNN_REQUIRE(h && gates && y32 && v && g && f_out && workspace, "null pointer");
  ICNN_REQUIRE(nIter >= 0, "nIter < 0");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long N = (long long)gates->B * h->n;
  ICNN_CUDA_CHECK(cudaMemsetAsync(v, 0, sizeof(float) * N, st));
  for (int it = 0; it < nIter; ++it) {
    int rc = picnn_fg_dispatch(h, gates, y32, f_out, g, h->n, nullptr, nullptr, 0, workspace, nullptr, st);
    if (rc) return rc;
    gd_update_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(y32, v, g, N, lr, momentum);
  }
  int rc = picnn_fg_dispatch(h, gates, y32, f_out, g, h->n, nullptr, nullptr, 0, workspace, nullptr, st);
  if (rc) return rc;
  ICNN_CUDA_CHECK(cudaGetLastError());
  return ICNN_OK;
}
