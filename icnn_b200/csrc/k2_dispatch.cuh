// K2 dispatch: which kernel build one bundle step launches, decided on the host from (n_y, KS, solver) and the launch
// environment variables, without launching anything.  bundle_step_launch (bundle_step.cu) enqueues exactly the build
// k2_plan returns, and icnn_k2_plan / icnn_k2_last_launch report it (include/icnn_b200.h).
#pragma once
#include <cstddef>
#include <cstdint>

#include "../../include/icnn_b200.h"

namespace icnn {

// two-sweep predictor-corrector kernel (bundle_pc_kernel.cuh): warps per sample, column chunks per thread, the
// minBlocks the build asks for (3 = 80-register build), 16-byte row loads, three n-vectors, dynamic shared memory
struct PcConfig { int wps, nch, npad, minb; bool vec, v3; size_t smem; };

// five-sweep kernel (bundle_step_kernel.cuh): warps per sample, cluster size, columns per CTA, resident-row pitch
// (0 = rows streamed from L2), n-vector pitch, k x k leading dimension, __launch_bounds__ minBlocks, shared memory
struct K2Config { int wps, cs, nloc, gpitch, npad, ld, minb; size_t smem; };

// 80-register build of the two-sweep kernel: only for 2 / 4 / 8 warps without V3 when three CTAs fit an SM
inline bool pc_r80(const PcConfig& c) { return !(c.v3 || c.wps == 16 || c.wps == 1) && c.minb >= 3; }
// second __launch_bounds__ argument of the two-sweep instantiation launch_pc picks for c
inline int pc_launch_minb(const PcConfig& c) { return c.wps == 16 ? 1 : (pc_r80(c) ? 24 : 16) / c.wps; }

enum K2Family { K2_SMALL = 0, K2_TWO_SWEEP = 1, K2_FIVE_SWEEP = 2 };

struct K2Plan {
  int family;
  PcConfig pc;   // K2_TWO_SWEEP
  K2Config k2;   // K2_FIVE_SWEEP
};

// ICNN_OK and the build, or ICNN_E_UNSUPPORTED with the error message set (the launch would fail the same way).
int k2_plan(int n, int KS, int solver, K2Plan* out);
// the icnn_k2_plan record of p at n_y = n
void k2_plan_record(const K2Plan& p, int n, int32_t out[ICNN_K2_PLAN_LEN]);

// two-sweep part of the dispatch (bundle_pc.cu): false = the shape takes the five-sweep kernel
bool pick_pc(int n, int KS, PcConfig* out);

}  // namespace icnn
