// K2 host side: buffer init, launch configuration, C-ABI entries.  The kernel template and its
// helpers live in bundle_step_kernel.cuh; the cluster-split instantiations in
// bundle_step_cluster.cu, K3 in argmin_grad.cu (three translation units so that `make -j` compiles
// the instantiations in parallel).
#include "bundle_step_kernel.cuh"

namespace icnn {

int argmin_grad_launch(const icnn_bundle_bufs* b, int loss, const double* trueY, double* cy, double* clam,
                       double* ct, double* V, cudaStream_t st);

__global__ void bundle_init_kernel(icnn_bundle_bufs b, int nIterMax, int nIterDefault) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long tot = (long long)b.B * b.KS;
  if (i < tot) b.perm[i] = (int)(i % b.KS);
  if (i < b.B) {
    b.count[i] = 0; b.status[i] = 0; b.finished[i] = 0; b.nIters[i] = nIterDefault;
    if (b.newton_its) b.newton_its[i] = 0;
    if (b.ksum) b.ksum[i] = 0;
  }
  if (i <= nIterMax) b.nactive[i] = (i == 0) ? b.B : 0;
  if (b.iter_stats && i < (long long)nIterMax * ICNN_NSTAT) b.iter_stats[i] = 0.0;
}

__global__ void y_round_kernel(const double* y, float* y32, long long N) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < N) y32[i] = (float)y[i];
}

__global__ void put_fg_kernel(icnn_bundle_bufs b, const float* f, const float* gsrc) {
  const int u = blockIdx.x;
  const int slot = b.perm[(size_t)u * b.KS + b.count[u]];
  float* dst = b.G + ((size_t)u * b.KS + slot) * b.n;
  for (int e = threadIdx.x; e < b.n; e += blockDim.x) dst[e] = gsrc[(size_t)u * b.n + e];
  if (threadIdx.x == 0) b.f[u] = f[u];
}

__global__ void put_fg64_kernel(icnn_bundle_bufs b, const double* f, const double* gsrc, double* f64) {
  const int u = blockIdx.x;
  const int slot = b.perm[(size_t)u * b.KS + b.count[u]];
  float* dst = b.G + ((size_t)u * b.KS + slot) * b.n;
  for (int e = threadIdx.x; e < b.n; e += blockDim.x) dst[e] = (float)gsrc[(size_t)u * b.n + e];
  if (threadIdx.x == 0) { b.f[u] = (float)f[u]; f64[u] = f[u]; }
}

// Launch configuration: warps per sample (WPS), cluster size over columns (CS) and whether the
// sample's rows are kept resident in shared memory.
//   n <= 192: 1 warp / sample, <= 512: 2, <= 1024: 4, else 8 (one CTA per column slice);
//   resident rows whenever KS x slice fits next to the work vectors; the sample is split over
//   CS = 2/4/8 CTAs of a cluster when one CTA cannot hold it (or to get two CTAs per SM).
static bool k2_fits(int n, int KS, int wps, int cs, bool resident, size_t limit, K2Config* out) {
  K2Config c;
  c.wps = wps; c.cs = cs;
  c.nloc = (cs == 1) ? n : (((n + cs - 1) / cs + 3) & ~3);
  if (cs > 1 && (long long)c.nloc * (cs - 1) >= n) return false;      // an empty slice
  c.npad = (c.nloc + 3) & ~3;
  c.ld = KS | 1;
  c.gpitch = 0;
  if (resident) { const int p4 = (c.nloc + 3) & ~3; c.gpitch = p4 + ((16 - (p4 & 31)) & 31); }   // = 16 mod 32 floats
  c.smem = sizeof(double) * group_smem_doubles(c.npad, KS, c.ld, wps, c.gpitch, cs) * (wps >= 8 ? 1 : 8 / wps);
  if (c.smem > limit) return false;
  // register budget of launch_k2: 80 registers (3 CTAs / SM) for the small groups and for 8 warps when shared memory
  // lets three CTAs share an SM, else 128; clusters 2 CTAs / SM, 16 warps one
  c.minb = wps == 16 ? 1 : cs > 1 ? 2 : wps == 8 ? (c.smem * 3 <= 225 * 1024 ? 3 : 2) : 3;
  *out = c;
  return true;
}

static int pick_k2(int n, int KS, K2Config* out) {
  // measured (K2 ms per solveBatch): n=159 (C3) WPS 1: 6.8, 2: 7.9;  n=512 (T) 1: 12.8, 2: 9.3, 4: 12.9;
  // n=2048 (C2) 4: 41.7, 8: 19.4
  int wps = n <= 192 ? 1 : (n <= 512 ? 2 : (n <= 1024 ? 4 : 8));
  bool pinned = false;   // a valid ICNN_K2_WPS: no fall back to more warps below
  if (const char* v = getenv("ICNN_K2_WPS")) {   // any value set (even an invalid one) skips the 16-warp upgrade
    const int w = atoi(v);
    if (w == 1 || w == 2 || w == 4 || w == 8 || w == 16) { wps = w; pinned = true; }
  } else if (wps == 8) {   // a single CTA per SM fits anyway -> give the sample 16 warps
    K2Config probe;
    if (k2_fits(n, KS, 8, 1, false, 227 * 1024, &probe) && probe.smem > 113 * 1024) wps = 16;
  }
  int want_cs = 0;
  if (const char* v = getenv("ICNN_K2_CS")) want_cs = atoi(v);
  // Resident rows / cluster split are OFF by default: they lost to streaming the rows from L2 on every
  // configuration when measured on an earlier GPU (not re-measured on H100) -- the per-sample solve is a
  // latency-bound FP64 chain, and what hides it is the number of samples in flight per SM, which
  // residency divides by 3-5.
  const char* rv = getenv("ICNN_K2_RESIDENT");
  const bool allow_res = (rv && rv[0] == '1');
  const size_t big = 200 * 1024, half = 110 * 1024;
  if (want_cs == 1 || want_cs == 2 || want_cs == 4 || want_cs == 8) {
    if (k2_fits(n, KS, want_cs > 1 ? 8 : wps, want_cs, allow_res, big, out)) return ICNN_OK;
    if (want_cs == 1 && k2_fits(n, KS, wps, 1, false, 227 * 1024, out)) return ICNN_OK;
    set_error("bundle_step: ICNN_K2_CS=%d does not fit (n=%d, KS=%d)", want_cs, n, KS);
    return ICNN_E_UNSUPPORTED;
  }
  if (allow_res) {
    if (k2_fits(n, KS, wps, 1, true, half, out)) return ICNN_OK;                 // resident, >= 2 CTAs / SM
    if (wps == 8 || n > 1024) {
      for (int cs = 2; cs <= 8; cs *= 2) if (k2_fits(n, KS, 8, cs, true, half, out)) return ICNN_OK;
      if (k2_fits(n, KS, 8, 1, true, big, out)) return ICNN_OK;
      for (int cs = 2; cs <= 8; cs *= 2) if (k2_fits(n, KS, 8, cs, true, big, out)) return ICNN_OK;
    } else if (k2_fits(n, KS, wps, 1, true, big, out)) return ICNN_OK;
  }
  if (k2_fits(n, KS, wps, 1, false, 227 * 1024, out)) return ICNN_OK;               // rows streamed from L2
  // 1 / 2 / 4 warps put 8 / 4 / 2 samples in one CTA; when their k x k matrices do not fit side by side (KS > ~36 at
  // n_y <= 192, KS > 62 at n_y <= 512) the sample gets more warps and the CTA fewer samples
  for (int w = wps * 2; !pinned && w <= 8; w *= 2)
    if (k2_fits(n, KS, w, 1, false, 227 * 1024, out)) return ICNN_OK;
  set_error("bundle_step: shared memory does not fit (n=%d, KS=%d)", n, KS);
  return ICNN_E_UNSUPPORTED;
}

bool bundle_step_small_ok(int n, int KS);

// The whole dispatch of one bundle step: tiny problems take one thread per sample (bundle_step_small.cu;
// ICNN_K2_SMALL=0 forces the group kernels); the PC solver takes the two-sweep kernel where pick_pc accepts the
// shape (ICNN_K2_PC=legacy keeps the five-sweep kernel); everything else takes the five-sweep kernel (pick_k2).
int k2_plan(int n, int KS, int solver, K2Plan* out) {
  K2Plan p = {};
  const char* sv = getenv("ICNN_K2_SMALL");
  if (!(sv && sv[0] == '0') && bundle_step_small_ok(n, KS)) { p.family = K2_SMALL; *out = p; return ICNN_OK; }
  if (KS > 64) { set_error("bundle_step: KS=%d > 64 unsupported", KS); return ICNN_E_UNSUPPORTED; }
  if (solver == ICNN_SOLVER_PC) {
    const char* v = getenv("ICNN_K2_PC");
    if (!(v && v[0] == 'l') && pick_pc(n, KS, &p.pc)) { p.family = K2_TWO_SWEEP; *out = p; return ICNN_OK; }
  }
  const int rc = pick_k2(n, KS, &p.k2);
  if (rc) return rc;
  p.family = K2_FIVE_SWEEP;
  *out = p;
  return ICNN_OK;
}

void k2_plan_record(const K2Plan& p, int n, int32_t out[ICNN_K2_PLAN_LEN]) {
  for (int i = 0; i < ICNN_K2_PLAN_LEN; ++i) out[i] = 0;
  out[0] = p.family;
  if (p.family == K2_TWO_SWEEP) {
    out[1] = p.pc.wps; out[2] = p.pc.nch; out[3] = p.pc.v3; out[4] = p.pc.vec;
    out[6] = pc_launch_minb(p.pc); out[7] = (int32_t)p.pc.smem;
  } else if (p.family == K2_FIVE_SWEEP) {
    out[1] = p.k2.wps; out[2] = p.k2.cs; out[4] = (n & 3) == 0; out[5] = p.k2.gpitch > 0;
    out[6] = p.k2.minb; out[7] = (int32_t)p.k2.smem;
  }
}

// icnn_k2_last_launch: the record of the calling thread's most recent K2 enqueue
static thread_local int32_t g_k2_last[ICNN_K2_PLAN_LEN] = {-1, 0, 0, 0, 0, 0, 0, 0};

cudaError_t bundle_step_cluster_launch(const StepArgs& a, const K2Config& c, int B, cudaStream_t st);
int bundle_step_small_launch(const icnn_bundle_cfg* cfg, const icnn_bundle_bufs* b, int t, cudaStream_t st);

int bundle_pc_launch(const icnn_bundle_cfg* cfg, const icnn_bundle_bufs* b, int t, const PcConfig& c, cudaStream_t st);

static int five_sweep_launch(const icnn_bundle_cfg* cfg, const icnn_bundle_bufs* b, int t, const K2Config& c,
                             cudaStream_t st) {
  StepArgs a;
  a.b = *b; a.c = *cfg; a.t = t;
  a.npad = c.npad; a.ld = c.ld; a.nloc = c.nloc; a.gpitch = c.gpitch;
  cudaError_t e;
  if (c.cs > 1) e = bundle_step_cluster_launch(a, c, b->B, st);     // bundle_step_cluster.cu
  else if (c.wps == 1) e = launch_k2<1, 1>(a, c, b->B, st);
  else if (c.wps == 2) e = launch_k2<2, 1>(a, c, b->B, st);
  else if (c.wps == 4) e = launch_k2<4, 1>(a, c, b->B, st);
  else if (c.wps == 16) e = launch_k2<16, 1>(a, c, b->B, st);
  else e = launch_k2<8, 1>(a, c, b->B, st);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) { set_error("bundle_step launch (wps=%d cs=%d smem=%zu): %s", c.wps, c.cs, c.smem, cudaGetErrorString(e)); return ICNN_E_CUDA; }
  return ICNN_OK;
}

int bundle_step_launch(const icnn_bundle_cfg* cfg, const icnn_bundle_bufs* b, int t, cudaStream_t st) {
  K2Plan p;
  int rc = k2_plan(b->n, b->KS, cfg->solver, &p);
  if (rc) return rc;
  if (p.family == K2_SMALL) rc = bundle_step_small_launch(cfg, b, t, st);
  else if (p.family == K2_TWO_SWEEP) rc = bundle_pc_launch(cfg, b, t, p.pc, st);   // bundle_pc_kernel.cuh
  else rc = five_sweep_launch(cfg, b, t, p.k2, st);                                 // bundle_step_kernel.cuh
  if (rc == ICNN_OK) k2_plan_record(p, b->n, g_k2_last);
  return rc;
}

}  // namespace icnn

using namespace icnn;

static int check_bufs(const icnn_bundle_bufs* b) {
  ICNN_REQUIRE(b, "null bufs");
  ICNN_REQUIRE(b->B > 0 && b->n > 0 && b->KS >= 2, "bad B / n / KS");
  ICNN_REQUIRE(b->y && b->y32 && b->f && b->G && b->h && b->lam && b->rsum && b->gram && b->perm &&
                   b->count && b->status && b->finished && b->nIters && b->nactive,
               "null buffer in icnn_bundle_bufs");
  return ICNN_OK;
}

extern "C" int icnn_bundle_init(const icnn_bundle_bufs* b, int32_t nIterMax, void* stream) {
  int rc = check_bufs(b);
  if (rc) return rc;
  ICNN_REQUIRE(nIterMax >= 1, "nIterMax < 1");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  long long tot = (long long)b->B * b->KS;
  if (tot < nIterMax + 1) tot = nIterMax + 1;
  if (tot < (long long)nIterMax * ICNN_NSTAT) tot = (long long)nIterMax * ICNN_NSTAT;
  bundle_init_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(*b, nIterMax, nIterMax);
  const long long N = (long long)b->B * b->n;
  y_round_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(b->y, b->y32, N);
  ICNN_CUDA_CHECK(cudaGetLastError());
  return ICNN_OK;
}

extern "C" int icnn_bundle_put_fg(const icnn_bundle_bufs* b, const float* f, const float* g, void* stream) {
  int rc = check_bufs(b);
  if (rc) return rc;
  ICNN_REQUIRE(f && g, "null f/g");
  put_fg_kernel<<<b->B, 128, 0, static_cast<cudaStream_t>(stream)>>>(*b, f, g);
  ICNN_CUDA_CHECK(cudaGetLastError());
  return ICNN_OK;
}

extern "C" int icnn_bundle_put_fg_f64(const icnn_bundle_bufs* b, const double* f, const double* g, void* stream) {
  int rc = check_bufs(b);
  if (rc) return rc;
  ICNN_REQUIRE(f && g, "null f/g");
  ICNN_REQUIRE(b->f64, "icnn_bundle_put_fg_f64 needs bufs.f64");
  put_fg64_kernel<<<b->B, 128, 0, static_cast<cudaStream_t>(stream)>>>(*b, f, g, const_cast<double*>(b->f64));
  ICNN_CUDA_CHECK(cudaGetLastError());
  return ICNN_OK;
}

extern "C" int icnn_argmin_grad(const icnn_bundle_bufs* b, int32_t loss, const double* trueY, double* cy,
                                double* clam, double* ct, double* V, void* stream) {
  int rc = check_bufs(b);
  if (rc) return rc;
  ICNN_REQUIRE(loss == 0 || loss == 1, "loss must be 0 (mse) or 1 (cross-entropy)");
  ICNN_REQUIRE(trueY && cy && clam && ct, "null pointer");
  ICNN_REQUIRE(b->KS <= 63, "KS > 63 unsupported");
  return argmin_grad_launch(b, loss, trueY, cy, clam, ct, V, static_cast<cudaStream_t>(stream));
}

extern "C" int icnn_bundle_step(const icnn_bundle_cfg* cfg, const icnn_bundle_bufs* b, int32_t t, void* stream) {
  int rc = check_bufs(b);
  if (rc) return rc;
  ICNN_REQUIRE(cfg, "null cfg");
  ICNN_REQUIRE(cfg->variant >= 0 && cfg->variant <= 2, "bad variant");
  ICNN_REQUIRE(cfg->solver == ICNN_SOLVER_PC || cfg->solver == ICNN_SOLVER_NEWTON, "bad solver");
  ICNN_REQUIRE(cfg->variant == ICNN_VARIANT_LIB || cfg->solver == ICNN_SOLVER_NEWTON,
               "dual / rl variants use the Newton solver");
  ICNN_REQUIRE(t >= 0, "t < 0");
  return bundle_step_launch(cfg, b, t, static_cast<cudaStream_t>(stream));
}

extern "C" int icnn_k2_plan(int32_t n, int32_t KS, int32_t solver, int32_t variant, int32_t out[ICNN_K2_PLAN_LEN]) {
  ICNN_REQUIRE(out, "null pointer");
  ICNN_REQUIRE(n > 0 && KS >= 2, "bad n / KS");
  ICNN_REQUIRE(variant >= 0 && variant <= 2, "bad variant");
  ICNN_REQUIRE(solver == ICNN_SOLVER_PC || solver == ICNN_SOLVER_NEWTON, "bad solver");
  ICNN_REQUIRE(variant == ICNN_VARIANT_LIB || solver == ICNN_SOLVER_NEWTON, "dual / rl variants use the Newton solver");
  K2Plan p;
  const int rc = k2_plan(n, KS, solver, &p);
  if (rc) return rc;
  k2_plan_record(p, n, out);
  return ICNN_OK;
}

extern "C" int icnn_k2_last_launch(int32_t out[ICNN_K2_PLAN_LEN]) {
  ICNN_REQUIRE(out, "null pointer");
  for (int i = 0; i < ICNN_K2_PLAN_LEN; ++i) out[i] = g_k2_last[i];
  return ICNN_OK;
}
