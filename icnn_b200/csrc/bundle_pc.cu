// K2 predictor-corrector path: launch configuration + instantiations (WPS = 1, 2); the larger groups are
// instantiated in bundle_pc_b.cu / bundle_pc_c.cu so that `make -j` compiles them in parallel.
#include "bundle_pc_kernel.cuh"

#include <cstdio>
#include <cstdlib>

namespace icnn {

#define ICNN_PC_DECL(W, N) cudaError_t launch_pc_##W##_##N(const PcArgs& a, const PcConfig& c, int B, cudaStream_t st)
ICNN_PC_DECL(1, 1); ICNN_PC_DECL(1, 2); ICNN_PC_DECL(1, 4); ICNN_PC_DECL(2, 1); ICNN_PC_DECL(2, 2);
ICNN_PC_DECL(4, 1); ICNN_PC_DECL(4, 2); ICNN_PC_DECL(8, 1); ICNN_PC_DECL(8, 2);
ICNN_PC_DECL(16, 1); ICNN_PC_DECL(16, 2); ICNN_PC_DECL(16, 4);
// n-vectors in the caller's scratch instead of shared memory (bundle_pc_e.cu): W = 200 + warps
ICNN_PC_DECL(201, 4); ICNN_PC_DECL(202, 2); ICNN_PC_DECL(204, 2); ICNN_PC_DECL(208, 4); ICNN_PC_DECL(208, 2);
// three n-vectors per sample (V3, bundle_pc_f.cu): two samples per SM at n_y = 4096: W = 300 + warps
ICNN_PC_DECL(308, 4); ICNN_PC_DECL(304, 4);
// n_y % 4 != 0 (rows not 16-byte aligned): scalar row loads, small groups only (bundle_pc_d.cu)
ICNN_PC_DECL(101, 1); ICNN_PC_DECL(101, 2); ICNN_PC_DECL(102, 1); ICNN_PC_DECL(102, 2);

ICNN_PC_DECL(1, 1) { return launch_pc<1, 1, true>(a, c, B, st); }
ICNN_PC_DECL(1, 2) { return launch_pc<1, 2, true>(a, c, B, st); }
ICNN_PC_DECL(1, 4) { return launch_pc<1, 4, true>(a, c, B, st); }
ICNN_PC_DECL(2, 1) { return launch_pc<2, 1, true>(a, c, B, st); }
ICNN_PC_DECL(2, 2) { return launch_pc<2, 2, true>(a, c, B, st); }

static bool pc_fits(const icnn_bundle_bufs* b, int wps, int nch, PcConfig* out, bool gv = false, bool v3 = false) {
  if (b->n > 128 * wps * nch) return false;
  PcConfig c;
  c.wps = wps; c.nch = nch; c.gv = gv; c.v3 = v3;
  c.npad = (b->n + 15) & ~15;   // the tensor-core sweep reads whole 16-column groups of the n-vectors
  c.vec = (b->n & 3) == 0;
  if (!c.vec && wps > 2) return false;
  c.smem = sizeof(double) * pc_group_doubles(c.npad, b->KS, wps, gv, v3);
  if (c.smem > 227 * 1024) return false;
  if (v3) {   // only worth it when at least two samples fit an SM (228 KB, 1 KB reserved per CTA)
    if (!c.vec || 2 * (c.smem + 1024) > 228 * 1024) return false;
    c.minb = 2;
    *out = c;
    return true;
  }
  // 80-register build (768 threads / SM) when shared memory lets that many samples be resident, else 128 registers
  c.minb = (wps == 16) ? 1 : ((c.smem + 1024) * (24 / wps) <= 228 * 1024 ? 3 : 2);
  if (wps == 1) c.minb = 2;   // one warp per sample: the 128-register build (no spills) wins (C3 4.5 vs 5.2 ms)
  if (const char* v = getenv("ICNN_PC_MINB")) { if (v[0] == '2') c.minb = 2; }   // tuning knob: 128-register build
  *out = c;
  return true;
}

// Threads per sample by n_y (measured per shape, see DESIGN.md K2): the thread that owns a column in
// sweep B keeps v2 in registers, so n <= 128 * WPS * NCH.
static bool pick_pc(const icnn_bundle_bufs* b, PcConfig* out) {
  const int n = b->n;
  if (b->KS > 62) return false;   // k + 2 sweep rows in <= 8 row blocks
  // Chosen by K2 time per solveBatch, measured per shape on an earlier GPU (not re-measured on H100):
  // -> the two-sweep kernel where it wins (small and very large n_y), the five-sweep kernel in between.
  int wps, nch;
  if (n <= 128) { wps = 1; nch = 1; }
  else if (n <= 256) { wps = 1; nch = 2; }
  else if (n <= 512) { wps = 2; nch = 2; }
  else if (n <= 1024) { wps = 4; nch = 2; }
  else if (n <= 2048) { wps = 8; nch = 2; }
  else if (n <= 4096) { wps = 16; nch = 2; }
  else { wps = 16; nch = 4; }
  // ICNN_PC_GV=<warps>: n-vectors in global scratch (exploration / measured dispatch below)
  if (const char* v = getenv("ICNN_PC_GV")) {
    const int w = atoi(v);
    if (b->vec_ws && (n & 3) == 0) {
      if (w == 1 && n <= 512) return pc_fits(b, 1, 4, out, true);
      if (w == 2 && n <= 512) return pc_fits(b, 2, 2, out, true);
      if (w == 4 && n <= 1024) return pc_fits(b, 4, 2, out, true);
      if (w == 8 && n <= 2048) return pc_fits(b, 8, 2, out, true);
      if (w == 8 && n <= 4096) return pc_fits(b, 8, 4, out, true);
    }
  }
  // three-vector build: ICNN_PC_V3=0 disables it, =1 also tries it for 1024 < n_y <= 2048 (exploration)
  {
    const char* v3 = getenv("ICNN_PC_V3");
    const bool off = v3 && v3[0] == '0', force = v3 && v3[0] == '1';
    if (!off && !getenv("ICNN_PC_WPS") && (n & 3) == 0) {
      if (n > 2048 && n <= 4096 && pc_fits(b, 8, 4, out, false, true)) return true;
      if (force && n > 1024 && n <= 2048 && pc_fits(b, 4, 4, out, false, true)) return true;
    }
  }
  // 256 < n_y <= 1024 stays on the five-sweep kernel (a tie within the run-to-run spread); with the lean k <= 32 stage
  // the two-sweep kernel won at n_y = 2048 (ICNN_PC_5SWEEP=1 restores the old choice)
  if (n > 256 && n <= 1024 && !getenv("ICNN_PC_WPS")) return false;
  if (n > 1024 && n <= 2048 && getenv("ICNN_PC_5SWEEP") && !getenv("ICNN_PC_WPS")) return false;
  if (const char* v = getenv("ICNN_PC_WPS")) {
    const int w = atoi(v);
    if (w == 1 || w == 2 || w == 4 || w == 8 || w == 16) {
      wps = w;
      nch = (n <= 128 * w) ? 1 : (n <= 256 * w ? 2 : 4);
    }
  }
  if (nch == 4 && wps != 16 && wps != 1) return false;
  return pc_fits(b, wps, nch, out);
}

// returns ICNN_E_UNSUPPORTED when the shape has to take the streaming kernel of bundle_step_kernel.cuh
int bundle_pc_launch(const icnn_bundle_cfg* cfg, const icnn_bundle_bufs* b, int t, cudaStream_t st) {
  PcConfig c;
  if (!pick_pc(b, &c)) return ICNN_E_UNSUPPORTED;
  PcArgs a;
  a.b = *b; a.c = *cfg; a.t = t; a.npad = c.npad;
  a.flags = 0;
  if (const char* v = getenv("ICNN_PC_FLAGS")) a.flags = atoi(v);
  if (const char* v = getenv("ICNN_PC_LEGACY")) { if (v[0] == '1') a.flags |= 4; }
  // L2 prefetch distances of the V3 row sweeps: sweep A one loop trip ahead, sweep B eight rows ahead (chosen per
  // setting with tools/k2_profile.py at C5 on H100, DESIGN.md §3 "Row passes").  ICNN_PC_PREFETCH="a,b" overrides them
  // at every launch ("0,0" = off), so settings can be compared in one process.
  a.pfa = 1; a.pfb = 8;
  if (const char* v = getenv("ICNN_PC_PREFETCH")) {
    int pa = 0, pb = 0;
    if (sscanf(v, "%d,%d", &pa, &pb) == 2 && pa >= 0 && pa <= 8 && pb >= 0 && pb <= 64) { a.pfa = pa; a.pfb = pb; }
  }
  cudaError_t e;
  const int key = (c.v3 ? 3000 : 0) + (c.gv ? 2000 : 0) + (c.vec ? 0 : 1000) + c.wps * 10 + c.nch;
  switch (key) {
    case 3084: e = launch_pc_308_4(a, c, b->B, st); break;
    case 3044: e = launch_pc_304_4(a, c, b->B, st); break;
    case 2014: e = launch_pc_201_4(a, c, b->B, st); break;
    case 2022: e = launch_pc_202_2(a, c, b->B, st); break;
    case 2042: e = launch_pc_204_2(a, c, b->B, st); break;
    case 2082: e = launch_pc_208_2(a, c, b->B, st); break;
    case 2084: e = launch_pc_208_4(a, c, b->B, st); break;
    case 1011: e = launch_pc_101_1(a, c, b->B, st); break;
    case 1012: e = launch_pc_101_2(a, c, b->B, st); break;
    case 1021: e = launch_pc_102_1(a, c, b->B, st); break;
    case 1022: e = launch_pc_102_2(a, c, b->B, st); break;
    case 11: e = launch_pc_1_1(a, c, b->B, st); break;
    case 12: e = launch_pc_1_2(a, c, b->B, st); break;
    case 14: e = launch_pc_1_4(a, c, b->B, st); break;
    case 21: e = launch_pc_2_1(a, c, b->B, st); break;
    case 22: e = launch_pc_2_2(a, c, b->B, st); break;
    case 41: e = launch_pc_4_1(a, c, b->B, st); break;
    case 42: e = launch_pc_4_2(a, c, b->B, st); break;
    case 81: e = launch_pc_8_1(a, c, b->B, st); break;
    case 82: e = launch_pc_8_2(a, c, b->B, st); break;
    case 161: e = launch_pc_16_1(a, c, b->B, st); break;
    case 162: e = launch_pc_16_2(a, c, b->B, st); break;
    case 164: e = launch_pc_16_4(a, c, b->B, st); break;
    default: return ICNN_E_UNSUPPORTED;
  }
  if (e != cudaSuccess) {
    set_error("bundle_pc launch (wps=%d nch=%d v3=%d smem=%zu): %s", c.wps, c.nch, (int)c.v3, c.smem, cudaGetErrorString(e));
    return ICNN_E_CUDA;
  }
  return ICNN_OK;
}

}  // namespace icnn
