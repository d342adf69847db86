// K2 predictor-corrector path: launch configuration + the one-warp instantiations; the larger groups are
// instantiated in bundle_pc_b.cu / bundle_pc_c.cu / bundle_pc_f.cu so that `make -j` compiles them in parallel.
#include "bundle_pc_kernel.cuh"

#include <cstdio>
#include <cstdlib>

namespace icnn {

#define ICNN_PC_DECL(NAME) cudaError_t launch_pc_##NAME(const PcArgs& a, const PcConfig& c, int B, cudaStream_t st)
ICNN_PC_DECL(1x1); ICNN_PC_DECL(1x2);
ICNN_PC_DECL(1x1_scalar); ICNN_PC_DECL(1x2_scalar);   // n_y % 4 != 0 (rows not 16-byte aligned): scalar row loads
ICNN_PC_DECL(8x2);                                    // bundle_pc_b.cu
ICNN_PC_DECL(16x2); ICNN_PC_DECL(16x4);               // bundle_pc_c.cu
ICNN_PC_DECL(v3_8x4);                                 // three n-vectors per sample (V3, bundle_pc_f.cu)

ICNN_PC_DECL(1x1) { return launch_pc<1, 1, true>(a, c, B, st); }
ICNN_PC_DECL(1x2) { return launch_pc<1, 2, true>(a, c, B, st); }
ICNN_PC_DECL(1x1_scalar) { return launch_pc<1, 1, false>(a, c, B, st); }
ICNN_PC_DECL(1x2_scalar) { return launch_pc<1, 2, false>(a, c, B, st); }

// What the tests switch, read at every launch (they change a variable between two solves of one process, or in the
// middle of one).  Each selects the reference a test compares the default against:
//   ICNN_PC_V3=0           four-vector 16-warp build at 2048 < n_y <= 4096 (test_three_vector_pc_kernel_matches_four_vector)
//   ICNN_PC_LEGACY=1       sweep A at rb = 5 as the multi-sweep composition (tests/test_gpu_k2_passes.py)
//   ICNN_PC_PREFETCH="a,b" L2 prefetch distances of the V3 row sweeps, "0,0" = off (tests/test_gpu_k2_prefetch.py)
//   ICNN_PC_SEED=0         sweep A at it = 0 and the dependency residual pass always
//                          (tests/test_gpu_k2_seed.py)
//   ICNN_PC_TWOLOG=1       V3 update with two logs, ry_new = logit(y_new) + (ry_old - logit(y_old)) + a du
//                          (tests/test_gpu_k2_onelog.py)
struct PcTestEnv { bool v3, split5, seed, twolog; int pfa, pfb; };
static PcTestEnv pc_test_env() {
  // prefetch defaults: sweep A one loop trip ahead, sweep B eight rows ahead (chosen per setting with
  // tools/k2_profile.py at C5 on H100, DESIGN.md §3 "Row passes")
  PcTestEnv e = {true, false, true, false, 1, 8};
  if (const char* v = getenv("ICNN_PC_V3")) e.v3 = v[0] != '0';
  if (const char* v = getenv("ICNN_PC_LEGACY")) e.split5 = v[0] == '1';
  if (const char* v = getenv("ICNN_PC_SEED")) e.seed = v[0] != '0';
  if (const char* v = getenv("ICNN_PC_TWOLOG")) e.twolog = v[0] == '1';
  if (const char* v = getenv("ICNN_PC_PREFETCH")) {
    int pa = 0, pb = 0;
    if (sscanf(v, "%d,%d", &pa, &pb) == 2 && pa >= 0 && pa <= 8 && pb >= 0 && pb <= 64) { e.pfa = pa; e.pfb = pb; }
  }
  return e;
}

// The thread that owns a column in sweep B keeps v2 in registers, so n <= 128 * WPS * NCH.
static bool pc_fits(int n, int KS, int wps, int nch, bool v3, PcConfig* out) {
  if (n > 128 * wps * nch) return false;
  PcConfig c;
  c.wps = wps; c.nch = nch; c.v3 = v3;
  c.npad = (n + 15) & ~15;   // the tensor-core sweep reads whole 16-column groups of the n-vectors
  c.vec = (n & 3) == 0;
  if (!c.vec && wps > 1) return false;
  c.smem = sizeof(double) * pc_group_doubles(c.npad, KS, wps, v3);
  if (c.smem > 227 * 1024) return false;
  if (v3) {   // only worth it when at least two samples fit an SM (228 KB, 1 KB reserved per CTA)
    if (!c.vec || 2 * (c.smem + 1024) > 228 * 1024) return false;
    c.minb = 2;
  } else if (wps == 16) c.minb = 1;
  else if (wps == 1) c.minb = 2;   // one warp per sample: the 128-register build (no spills) wins (C3 4.5 vs 5.2 ms)
  else   // 80-register build (768 threads / SM) when shared memory lets that many samples be resident, else 128 registers
    c.minb = (c.smem + 1024) * (24 / wps) <= 228 * 1024 ? 3 : 2;
  *out = c;
  return true;
}

// The two-sweep kernel where it wins (small and very large n_y), the five-sweep kernel in between.  Chosen by K2 time
// per solveBatch, measured per shape (DESIGN.md §3 "Dispatch"):
//          n_y <= 128    1 warp,  1 chunk
//    128 < n_y <= 256    1 warp,  2 chunks
//    256 < n_y <= 1024   five-sweep kernel
//   1024 < n_y <= 2048   8 warps, 2 chunks   (n_y % 4 == 0, else five-sweep)
//   2048 < n_y <= 4096   V3: 8 warps, 4 chunks when two samples fit an SM, else 16 warps, 2 chunks
//   4096 < n_y           16 warps, 4 chunks
// false: the shape takes the five-sweep kernel (also whenever shared memory does not fit).  Part of k2_plan
// (bundle_step.cu), which reads ICNN_K2_PC first.
bool pick_pc(int n, int KS, PcConfig* out) {
  const bool allow_v3 = pc_test_env().v3;
  if (KS > 62) return false;   // k + 2 sweep rows in <= 8 row blocks
  if (n <= 128) return pc_fits(n, KS, 1, 1, false, out);
  if (n <= 256) return pc_fits(n, KS, 1, 2, false, out);
  if (n <= 1024) return false;
  if (n <= 2048) return pc_fits(n, KS, 8, 2, false, out);
  if (n <= 4096) return (allow_v3 && pc_fits(n, KS, 8, 4, true, out)) || pc_fits(n, KS, 16, 2, false, out);
  return pc_fits(n, KS, 16, 4, false, out);
}

// enqueues the two-sweep build c (from pick_pc)
int bundle_pc_launch(const icnn_bundle_cfg* cfg, const icnn_bundle_bufs* b, int t, const PcConfig& c, cudaStream_t st) {
  const PcTestEnv env = pc_test_env();
  PcArgs a;
  a.b = *b; a.c = *cfg; a.t = t; a.npad = c.npad;
  a.split5 = env.split5; a.seed = env.seed; a.twolog = env.twolog; a.pfa = env.pfa; a.pfb = env.pfb;
  cudaError_t e;
  if (c.v3) e = launch_pc_v3_8x4(a, c, b->B, st);
  else if (c.wps == 16) e = c.nch == 2 ? launch_pc_16x2(a, c, b->B, st) : launch_pc_16x4(a, c, b->B, st);
  else if (c.wps == 8) e = launch_pc_8x2(a, c, b->B, st);
  else if (c.vec) e = c.nch == 1 ? launch_pc_1x1(a, c, b->B, st) : launch_pc_1x2(a, c, b->B, st);
  else e = c.nch == 1 ? launch_pc_1x1_scalar(a, c, b->B, st) : launch_pc_1x2_scalar(a, c, b->B, st);
  if (e != cudaSuccess) {
    set_error("bundle_pc launch (wps=%d nch=%d v3=%d smem=%zu): %s", c.wps, c.nch, (int)c.v3, c.smem, cudaGetErrorString(e));
    return ICNN_E_CUDA;
  }
  return ICNN_OK;
}

}  // namespace icnn
