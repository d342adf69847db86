// Phase-timer build of the V3 two-sweep K2 kernel (bundle_pc_kernel.cuh with ICNN_PC_PHASES), compiled by
// tools/k2_phases.py into a shared object of its own; the library never contains it.
#define ICNN_PC_PHASES
#include "bundle_pc_kernel.cuh"

using namespace icnn;

// One K2 launch of the V3 build (8 warps, 4 chunks) for outer iteration t; ph: [nIter][PC_NPH][PC_PH_SLOTS] cycles.
// pfa / pfb: the prefetch distances (the library's defaults are 1, 8: bundle_pc.cu, pc_test_env).
extern "C" int k2ph_launch(const icnn_bundle_cfg* cfg, const icnn_bundle_bufs* b, int t, unsigned long long* ph,
                           int pfa, int pfb, void* stream) {
  PcArgs a;
  a.b = *b; a.c = *cfg; a.t = t; a.npad = (b->n + 15) & ~15;
  a.pfa = pfa; a.pfb = pfb; a.split5 = false; a.seed = true; a.twolog = false; a.ph = ph;
  PcConfig c;
  c.wps = 8; c.nch = 4; c.npad = a.npad; c.minb = 2; c.vec = true; c.v3 = true;
  c.smem = sizeof(double) * pc_group_doubles(a.npad, b->KS, 8, true);
  return (int)launch_pc<8, 4, true, true>(a, c, b->B, static_cast<cudaStream_t>(stream));
}

extern "C" int k2ph_nph() { return PC_NPH; }
extern "C" int k2ph_slots() { return PC_PH_SLOTS; }
