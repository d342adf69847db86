// K1 (tensor-core path): PICNN f and df/dy with Hopper warpgroup MMA (wgmma.mma_async, tf32 inputs,
// 3xTF32 split for FP32-level accuracy), operands staged by TMA into 128B-swizzled shared memory,
// accumulators in registers, fused epilogues.
//
// Same math as picnn_simt.cu (multi-label-cls/icnn_ebundle.py:349-387,146; RL/src/icnn.py:356-404):
//   forward  layer i : Z_i   = act( A'_i  Wcat_i + d_i ),   A'_i = [Z_{i-1} o cz_i | (s y + t) o cy_i]
//   backward layer i : [delta_{i-1} | g +=] = delta_i Wcat_i^T  with the gate / act' epilogues
// Every GEMM is  C[M,N] = A[M,K] * B[N,K]^T  with BOTH operands K-major (the library keeps the
// weights in both orientations; wgmma takes tf32 operands K-major only), each operand pre-split into
// hi = tf32(x) and lo = x - hi:
//   C = A_hi B_hi + A_hi B_lo + A_lo B_hi     (three wgmma per k-step into one FP32 accumulator)
// Plain TF32 (10-bit mantissa) moves y* by 1e-3..1e-2 (SURVEY.md section 7, hard part 2); the split
// restores ~2^-21 relative error.
//
// Kernel anatomy (288 threads, one 128 x BN output tile per CTA):
//   warps 0..7  two consumer warpgroups; warpgroup g owns tile rows 64g..64g+63.  Per 32-wide k-block
//               it issues 12 wgmma m64nBNk8 (4 k-steps x {hi*hi, hi*lo, lo*hi}) and releases the stage;
//               afterwards every warp runs the fused epilogue on the 16 rows its accumulators hold
//   warp 8      TMA producer: cp.async.bulk.tensor.2d of A_hi/A_lo/B_hi/B_lo boxes (32 fp32 = 128 B
//               wide) into an NST-stage ring, mbarrier expect_tx
#include "common.cuh"

#include <cuda.h>
#include <cooperative_groups.h>

#include <cstdlib>
#include <cstring>

namespace cg = cooperative_groups;

namespace icnn {

// ---------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t ok;
  uint32_t spins = 0;
  do {
    if (++spins > (1u << 28)) __trap();   // a lost transaction would otherwise hang the GPU
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
  } while (!ok);
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
// one lane of a converged warp, chosen by the hardware (elect.sync): unlike `lane == 0`, ptxas knows that exactly one
// thread runs the guarded region, so the single-thread TMA issue is emitted straight instead of inside a loop over
// the active lanes
__device__ __forceinline__ bool elect_one_sync() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}
// the 256 threads of the two consumer warpgroups (named barrier 1; the producer warp never joins it)
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accesses of accumulator registers across the asynchronous MMA
template <int R>
__device__ __forceinline__ void fence_operands(float (&d)[R]) {
#pragma unroll
  for (int j = 0; j < R; ++j) asm volatile("" : "+f"(d[j])::"memory");
}
// D[64 x N] (+)= A[smem desc] * B[smem desc]^T, tf32 inputs, FP32 accumulator in registers of the
// issuing warpgroup; scale_d = 0 overwrites D.  Fragment of thread (warp w of the warpgroup, lane l):
//   d[4j + 2i + c] = D[16w + l/4 + 8i][8j + 2(l%4) + c]
__device__ __forceinline__ void wgmma_tf32(float (&d)[32], uint64_t adesc, uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
      "}, %32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(scale_d) : "memory");
}
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t adesc, uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
      "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
      "}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(scale_d) : "memory");
}

// shared-memory matrix descriptor (sm_90 wgmma), K-major operand, 128-byte swizzle, rows of 128 B,
// 8-row atoms of 1024 B: start>>4 [0,14), LBO>>4 [16,30) (unused: the K extent of a stage is one
// swizzle span), SBO>>4 [32,46) = 1024 B between 8-row atoms, layout SWIZZLE_128B = 1 at [62,64).
// Every operand buffer starts on a 1024-byte boundary, so the base-offset field stays 0.
__device__ __forceinline__ uint64_t make_kmajor_sw128_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)((1024 >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// TF32 split with round-to-nearest on both parts: hi = rn_tf32(x), lo = rn_tf32(x - hi), both exactly
// representable in TF32 (the tensor core would otherwise TRUNCATE its inputs), so
// |x - (hi + lo)| <= 2^-22 |x|  (measured: gates/f/g errors 2-4x lower than with truncation).
__device__ __forceinline__ float tf32_rn(float x) { return __uint_as_float((__float_as_uint(x) + 0x00001000u) & 0xFFFFE000u); }
__device__ __forceinline__ float tf32_hi(float x) { return tf32_rn(x); }
__device__ __forceinline__ float tf32_lo(float x, float hi) { return tf32_rn(x - hi); }

// ---------------------------------------------------------------------------------------------
// the GEMM kernel
// ---------------------------------------------------------------------------------------------
constexpr int TC_BM = 128;
constexpr int TC_BK = 32;  // fp32 elements per stage row = one 128-byte swizzle span
constexpr int TC_HALF = TC_BK / 16;   // k-steps (K = 8 each) per half k-block
constexpr int TC_CH = 1;   // default half k-blocks per accumulation chunk (K = 16: 6 MMAs into the chunk accumulator before
                           // the RN add into the running sum); TcArgs::ch carries the value a launch uses (ICNN_TC_CH,
                           // read once: accuracy/speed exploration)
constexpr int TC_CONSUMER_WARPS = 8;
constexpr int TC_THREADS = 32 * (TC_CONSUMER_WARPS + 1);

struct TcArgs {
  int M, N, K;
  int ch;    // half k-blocks per accumulation chunk (>= 1), set by launch_tc_gemm
  int mode;  // 0 forward, 1 backward, 2 plain store (self test)
  // forward epilogue: Z = act(acc + D); optional next-layer operand A'_{next}[:, 0:N] = Z o Cz_next (hi/lo)
  const float* D; float* Z; float alpha;
  const float* Cz_next; float* nxt_hi; float* nxt_lo; int nxt_ld;
  // backward epilogue: columns < N0 -> delta_prev = act'(Zprev) o Cz o acc (hi/lo, row pitch dprev_ld); else g += ...
  int N0; const float* Zprev; const float* Cz; float* dprev_hi; float* dprev_lo; int dprev_ld;
  const float* Cy; float* g; long long g_row_stride; const int* perm; const int* count; int KS; int n;
  float g_scale;
  float* C;  // mode 2
  // GD training backward (GDB instantiation only, gd_backward.cu):
  //   mode 0 with tangent != 0: Z = act'(D) o acc (D holds the primal activation), no bias
  //   mode 1: optional plain copy of delta_prev, dCz += kappa * Ztprev o acc, Dacc += kappa * delta_prev
  //   mode 0 with tangent == 2 (stored-pattern phase): Z = act'(Zmask) o (acc + D[(row % drow_mod), :])
  //   mode 1: optional plain copy of the pre-gating product acc (acc_plain, [M, N0])
  int tangent; float* dprev_plain; float* dCz; const float* Ztprev; float* Dacc; float kappa;
  const float* Zmask; int drow_mod; float* acc_plain;
  // mode 3 (x-path gate GEMM): out = acc + bias[col]; up to 4 column ranges [rbeg[r], rbeg[r+1]) each with
  // its own ReLU flag and destination (row pitch rld[r]); range 0 may instead be written as a TF32
  // hi/lo pair (the next u-layer operand)
  int nr; int rbeg[5]; int rrelu[4]; float* rdst[4]; int rld[4]; float* r0_hi; float* r0_lo; const float* bias;
  const int* skip_if_zero;
};

template <int BN, int NST_>
struct TcSmem {
  static constexpr int NST = NST_;
  static constexpr int A_BYTES = TC_BM * 128;
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;
  static constexpr int BAR_OFF = NST * STAGE_BYTES;
  static constexpr int TOTAL = BAR_OFF + 256 + 1024;  // + alignment slack
  // the finished [TC_BM][BN + 1] tile is staged for the epilogue in the idle ring
  static_assert(TC_BM * (BN + 1) * 4 <= BAR_OFF, "epilogue tile does not fit the ring");
};

// <128,3>: one CTA / SM (194 KB);  <64,4>: one CTA / SM, deeper ring for small grids;
// <64,2>: two CTAs / SM (98 KB each) so that one CTA's epilogue overlaps the other's main loop.
template <int BN, int NST_, bool GDB = false>
__global__ void __launch_bounds__(TC_THREADS, (BN == 64 && NST_ == 2) ? 2 : 1)
tc_gemm_kernel(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
               const __grid_constant__ CUtensorMap tmBh, const __grid_constant__ CUtensorMap tmBl, TcArgs a) {
  if (a.skip_if_zero != nullptr && *a.skip_if_zero == 0) return;
  using SM = TcSmem<BN, NST_>;
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment (128B swizzle atoms) as an OFFSET into the shared array, so that every address below keeps
  // the shared address space
  const uint32_t smem_pad = ((smem_u32(smem_raw) + 1023u) & ~1023u) - smem_u32(smem_raw);
  uint8_t* smem = smem_raw + smem_pad;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + SM::BAR_OFF);
  uint64_t* empty = full + SM::NST;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.y * TC_BM, n0 = blockIdx.x * BN;
  // split-K: gridDim.z = S CTAs of one cluster share the output tile, each reduces a K-slice into its
  // own accumulators; the partial tiles are summed through distributed shared memory below
  const int S = gridDim.z;
  const int nkb_all = (a.K + TC_BK - 1) / TC_BK;
  const int kb0 = (int)(((long long)nkb_all * blockIdx.z) / S);
  const int nkb = (int)(((long long)nkb_all * (blockIdx.z + 1)) / S) - kb0;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmAh); tma_prefetch_desc(&tmAl); tma_prefetch_desc(&tmBh); tma_prefetch_desc(&tmBl);
    // a stage is free again once each of the eight consumer warps has seen its MMAs complete
    for (int s = 0; s < SM::NST; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], TC_CONSUMER_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == TC_CONSUMER_WARPS) {
    // ---- producer ----
    if (elect_one_sync()) {
      for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % SM::NST;
        const uint32_t ph = (kb / SM::NST) & 1;
        mbar_wait(&empty[s], ph ^ 1);
        mbar_expect_tx(&full[s], SM::STAGE_BYTES);
        uint8_t* st = smem + s * SM::STAGE_BYTES;
        const int kc = (kb0 + kb) * TC_BK;
        tma_load_2d(st, &tmAh, &full[s], kc, m0);
        tma_load_2d(st + SM::A_BYTES, &tmAl, &full[s], kc, m0);
        tma_load_2d(st + 2 * SM::A_BYTES, &tmBh, &full[s], kc, n0);
        tma_load_2d(st + 2 * SM::A_BYTES + SM::B_BYTES, &tmBl, &full[s], kc, n0);
      }
    }
    __syncwarp();
    // every thread of the cluster takes part in both cluster barriers of the split-K epilogue
    if (S > 1) { cg::this_cluster().sync(); cg::this_cluster().sync(); }
    return;
  }

  // ---- consumers: main loop ----
  // Chunked accumulation.  The tensor core does not round its FP32 accumulator to nearest at every MMA, which
  // leaves a systematic relative bias per accumulation (tools/tc_bias_probe.py) that compounds through the layers
  // and moves y* over 50 bundle iterations.  The reduction is therefore cut into CHUNKS of a.ch half k-blocks: the
  // products of one chunk (hi*hi and the 2^-11 smaller cross terms) go into the wgmma accumulator `frag`, which
  // is then added into the FP32 running sum `run` with round-to-nearest adds.
  // Each half-block waits for its own MMAs (wait_group 0) before the next is issued: the tensor core of an SM is
  // kept busy by the other warpgroup and the second CTA, not by a deeper MMA pipeline within one warpgroup.
  const int wg = warp >> 2;   // consumer warpgroup: tile rows 64 wg .. 64 wg + 63
  float run[BN / 2], frag[BN / 2];
#pragma unroll
  for (int j = 0; j < BN / 2; ++j) { run[j] = 0.f; frag[j] = 0.f; }
  {
    const int CH = a.ch;
    for (int kb = 0; kb < nkb; ++kb) {
      const int s = kb % SM::NST;
      const uint32_t ph = (kb / SM::NST) & 1;
      mbar_wait(&full[s], ph);
      const uint32_t st = smem_u32(smem + s * SM::STAGE_BYTES);
      const uint32_t arow = (uint32_t)(wg * (SM::A_BYTES / 2));   // 64 rows x 128 B
      const uint64_t dAh = make_kmajor_sw128_desc(st + arow);
      const uint64_t dAl = make_kmajor_sw128_desc(st + SM::A_BYTES + arow);
      const uint64_t dBh = make_kmajor_sw128_desc(st + 2 * SM::A_BYTES);
      const uint64_t dBl = make_kmajor_sw128_desc(st + 2 * SM::A_BYTES + SM::B_BYTES);
      // two half-blocks of K = 16 (TC_HALF k-steps each); chunk c covers half-blocks c*CH .. c*CH + CH - 1
#pragma unroll
      for (int hb = 0; hb < 2; ++hb) {
        const int h = 2 * kb + hb;
        const int first = (h % CH) == 0;
        fence_operands(frag);
        wgmma_fence();
        // the 2^-11 smaller cross terms first, then the hi*hi products: an accumulation truncates at the
        // accumulator's magnitude, so only the hi*hi steps add a truncation at full size
#pragma unroll
        for (int k = 0; k < TC_HALF; ++k) {
          const uint64_t adv = (uint64_t)(((hb * TC_HALF + k) * 8 * 4) >> 4);  // +32 B per k-step inside the swizzle span
          wgmma_tf32(frag, dAh + adv, dBl + adv, (first && k == 0) ? 0 : 1);
          wgmma_tf32(frag, dAl + adv, dBh + adv, 1);
        }
#pragma unroll
        for (int k = 0; k < TC_HALF; ++k) {
          const uint64_t adv = (uint64_t)(((hb * TC_HALF + k) * 8 * 4) >> 4);
          wgmma_tf32(frag, dAh + adv, dBh + adv, 1);
        }
        wgmma_commit();
        wgmma_wait0();
        fence_operands(frag);
        if ((h + 1) % CH == 0 || h + 1 == 2 * nkb) {
#pragma unroll
          for (int j = 0; j < BN / 2; ++j) run[j] += frag[j];
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);   // this warp's share of the stage has been read
    }
  }

  // ---- epilogue: registers -> [TC_BM][BN + 1] tile in the idle ring -> fused epilogue -> global ----
  // Warp w holds tile rows 16w..16w+15 (warpgroup w/4, warp w%4 of it).  Global traffic wants one row per
  // warp instruction (lanes = consecutive columns), so the accumulators go through shared memory first.
  consumer_sync();   // both warpgroups are done reading the ring
  float* P = reinterpret_cast<float*>(smem);
  constexpr int PP = BN + 1;
  {
    const int rb = warp * 16 + (lane >> 2), cb = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int c = 0; c < 2; ++c) P[(rb + 8 * i) * PP + 8 * j + cb + c] = run[4 * j + 2 * i + c];
  }
  if (S > 1) {
    // ---- split-K epilogue: DSMEM sum of the cluster's partial tiles -> fused epilogue ----
    // (every CTA of the cluster reaches both cluster barriers: the producer warp calls them above)
    cg::this_cluster().sync();
    cg::cluster_group cl = cg::this_cluster();
    const int rank = (int)cl.block_rank();
    const int rlo = (TC_BM * rank) / S, rhi = (TC_BM * (rank + 1)) / S;
    for (int rr = rlo + warp; rr < rhi; rr += TC_CONSUMER_WARPS) {   // this warp's rows of the CTA's row slice
      const int m = m0 + rr;
      if (m >= a.M) break;
      float* grow = nullptr;
      if (a.mode == 1)
        grow = (a.perm == nullptr) ? a.g + (long long)m * a.g_row_stride
                                   : a.g + ((long long)m * a.KS + a.perm[(long long)m * a.KS + a.count[m]]) * a.n;
      for (int c = lane; c < BN; c += 32) {
        const int nn = n0 + c;
        if (nn >= a.N) break;
        float acc = 0.f;
        for (int qq = 0; qq < S; ++qq) acc += *cl.map_shared_rank(P + rr * PP + c, qq);
        if (a.mode == 0) {
          const long long idx = (long long)m * a.N + nn;
          float dv;
          if (GDB && a.tangent == 2) dv = __ldg(a.D + (long long)(m % a.drow_mod) * a.N + nn);
          else dv = __ldg(a.D + idx);
          const float x = acc + dv;
          float z = x > 0.f ? x : a.alpha * x;
          if constexpr (GDB) {
            if (a.tangent == 1) z = (dv > 0.f ? 1.f : a.alpha) * acc;
            else if (a.tangent == 2) z = (__ldg(a.Zmask + idx) > 0.f ? 1.f : a.alpha) * x;
          }
          a.Z[idx] = z;
          if (a.nxt_hi) {
            const float p = z * __ldg(a.Cz_next + idx);
            const float h = tf32_hi(p);
            a.nxt_hi[(long long)m * a.nxt_ld + nn] = h;
            a.nxt_lo[(long long)m * a.nxt_ld + nn] = tf32_lo(p, h);
          }
        } else {
          if (nn < a.N0) {
            const long long idx = (long long)m * a.N0 + nn;
            const float da = __ldg(a.Zprev + idx) > 0.f ? 1.f : a.alpha;
            const float p = da * __ldg(a.Cz + idx) * acc;
            const float h = tf32_hi(p);
            a.dprev_hi[(long long)m * a.dprev_ld + nn] = h;
            a.dprev_lo[(long long)m * a.dprev_ld + nn] = tf32_lo(p, h);
            if constexpr (GDB) {
              if (a.dprev_plain) a.dprev_plain[idx] = p;
              if (a.acc_plain) a.acc_plain[idx] = acc;
              if (a.dCz) a.dCz[idx] = fmaf(a.kappa * __ldg(a.Ztprev + idx), acc, a.dCz[idx]);
              if (a.Dacc) a.Dacc[idx] = fmaf(a.kappa, p, a.Dacc[idx]);
            }
          } else {
            const int e = nn - a.N0;
            grow[e] = fmaf(a.g_scale * __ldg(a.Cy + (long long)m * a.n + e), acc, grow[e]);
          }
        }
      }
    }
    cg::this_cluster().sync();   // partial tiles stay alive until every rank has read them
    return;
  }
  __syncwarp();   // each warp reads back only the rows it wrote
  // bundle-slot row pointer of row 16 warp + lane (backward mode, lanes 0..15), broadcast by shuffle
  unsigned long long growp = 0;
  if (a.mode == 1 && lane < 16) {
    const int mr = m0 + warp * 16 + lane;
    if (mr < a.M) {
      float* gp = (a.perm == nullptr) ? a.g + (long long)mr * a.g_row_stride
                                      : a.g + ((long long)mr * a.KS + a.perm[(long long)mr * a.KS + a.count[mr]]) * a.n;
      growp = reinterpret_cast<unsigned long long>(gp);
    }
  }
#pragma unroll
  for (int c0 = 0; c0 < BN; c0 += 32) {
    if (n0 + c0 >= a.N) break;          // warp-uniform: whole chunk out of range
    const int nn = n0 + c0 + lane;                     // this lane's column for the whole chunk
    const bool nv = nn < a.N;
    // rows in groups of RG: issue every global load of the group first (they are independent
    // and L2-latency bound), then compute and store
    constexpr int RG = 8;
    for (int r0 = 0; r0 < 16; r0 += RG) {
      if (m0 + warp * 16 + r0 >= a.M) break;           // warp-uniform
      float acc[RG], in0[RG], in1[RG];
      float in2[GDB ? RG : 1], in3[GDB ? RG : 1], in4[GDB ? RG : 1];
      unsigned long long gp[RG];
#pragma unroll
      for (int i = 0; i < RG; ++i) {
        const int m = m0 + warp * 16 + r0 + i;
        acc[i] = P[(warp * 16 + r0 + i) * PP + c0 + lane];
        gp[i] = __shfl_sync(0xffffffffu, growp, r0 + i);
        in0[i] = 0.f; in1[i] = 0.f;
        if (nv && m < a.M) {
          if (a.mode == 0) {
            const long long idx = (long long)m * a.N + nn;
            if (GDB && a.tangent == 2) {
              in0[i] = __ldg(a.D + (long long)(m % a.drow_mod) * a.N + nn);
              in1[i] = __ldg(a.Zmask + idx);
            } else {
              in0[i] = __ldg(a.D + idx);
              if (a.nxt_hi) in1[i] = __ldg(a.Cz_next + idx);
            }
          } else if (a.mode == 3) {
            in0[i] = __ldg(a.bias + nn);
          } else if (a.mode == 1) {
            if (nn < a.N0) {
              const long long idx = (long long)m * a.N0 + nn;
              in0[i] = __ldg(a.Zprev + idx);
              in1[i] = __ldg(a.Cz + idx);
              if constexpr (GDB) {
                if (a.dCz) { in2[i] = __ldg(a.Ztprev + idx); in3[i] = a.dCz[idx]; }
                if (a.Dacc) in4[i] = a.Dacc[idx];
              }
            } else {
              const int e = nn - a.N0;
              in0[i] = __ldg(a.Cy + (long long)m * a.n + e);
              in1[i] = reinterpret_cast<const float*>(gp[i])[e];
            }
          }
        }
      }
#pragma unroll
      for (int i = 0; i < RG; ++i) {
        const int m = m0 + warp * 16 + r0 + i;
        if (!nv || m >= a.M) continue;
        if (a.mode == 0) {
          const long long idx = (long long)m * a.N + nn;
          const float x = acc[i] + in0[i];
          float z = x > 0.f ? x : a.alpha * x;
          if constexpr (GDB) {
            if (a.tangent == 1) z = (in0[i] > 0.f ? 1.f : a.alpha) * acc[i];
            else if (a.tangent == 2) z = (in1[i] > 0.f ? 1.f : a.alpha) * x;
          }
          a.Z[idx] = z;
          if (a.nxt_hi) {
            const float p = z * in1[i];
            const float h = tf32_hi(p);
            a.nxt_hi[(long long)m * a.nxt_ld + nn] = h;
            a.nxt_lo[(long long)m * a.nxt_ld + nn] = tf32_lo(p, h);
          }
        } else if (a.mode == 1) {
          if (nn < a.N0) {
            const float da = in0[i] > 0.f ? 1.f : a.alpha;
            const float p = da * in1[i] * acc[i];
            const float h = tf32_hi(p);
            a.dprev_hi[(long long)m * a.dprev_ld + nn] = h;
            a.dprev_lo[(long long)m * a.dprev_ld + nn] = tf32_lo(p, h);
            if constexpr (GDB) {
              const long long idx = (long long)m * a.N0 + nn;
              if (a.dprev_plain) a.dprev_plain[idx] = p;
              if (a.acc_plain) a.acc_plain[idx] = acc[i];
              if (a.dCz) a.dCz[idx] = fmaf(a.kappa * in2[i], acc[i], in3[i]);
              if (a.Dacc) a.Dacc[idx] = fmaf(a.kappa, p, in4[i]);
            }
          } else {
            const int e = nn - a.N0;
            reinterpret_cast<float*>(gp[i])[e] = fmaf(a.g_scale * in0[i], acc[i], in1[i]);
          }
        } else if (a.mode == 3) {
          int r = 0;
#pragma unroll
          for (int t = 1; t < 4; ++t) if (t < a.nr && nn >= a.rbeg[t]) r = t;
          float v = acc[i] + in0[i];
          if (a.rrelu[r]) v = fmaxf(v, 0.f);
          const int c = nn - a.rbeg[r];
          if (r == 0 && a.r0_hi) {
            const float h = tf32_hi(v);
            a.r0_hi[(long long)m * a.rld[0] + c] = h;
            a.r0_lo[(long long)m * a.rld[0] + c] = tf32_lo(v, h);
          } else {
            a.rdst[r][(long long)m * a.rld[r] + c] = v;
          }
        } else {
          a.C[(long long)m * a.N + nn] = acc[i];
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// elementwise helpers
// ---------------------------------------------------------------------------------------------
// A'_i[:, off + e] = ((s*y + t) o cy_i)[e] split into hi/lo, for all layers in one launch
struct GateYArgs {
  int B, n, L;
  const float* y; float sc, sh;
  const float* cy[ICNN_MAX_LAYERS]; float* hi[ICNN_MAX_LAYERS]; float* lo[ICNN_MAX_LAYERS];
  int ld[ICNN_MAX_LAYERS]; int off[ICNN_MAX_LAYERS];
  const int* skip_if_zero;
};
__global__ void gate_y_kernel(GateYArgs a) {
  if (a.skip_if_zero != nullptr && *a.skip_if_zero == 0) return;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)a.B * a.n) return;
  const int m = (int)(i / a.n), e = (int)(i % a.n);
  const float yy = fmaf(a.sc, a.y[i], a.sh);
  for (int l = 0; l < a.L; ++l) {
    const float p = yy * a.cy[l][i];
    const float h = tf32_hi(p);
    a.hi[l][(long long)m * a.ld[l] + a.off[l] + e] = h;
    a.lo[l][(long long)m * a.ld[l] + a.off[l] + e] = tf32_lo(p, h);
  }
}

// src [R, C] dense -> hi/lo [R, C] with row pitch ld
__global__ void split_tf32_kernel(const float* src, float* hi, float* lo, long long R, int C, int ld) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= R * C) return;
  const long long o = (i / C) * ld + (i % C);
  const float x = src[i], h = tf32_hi(x);
  hi[o] = h;
  lo[o] = tf32_lo(x, h);
}
// dst[c, r] = src[r, c] split hi/lo   (src [R, C] row-major -> dst [C, R] with row pitch ldr)
__global__ void transpose_split_kernel(const float* src, float* hi, float* lo, int R, int C, int ldr) {
  __shared__ float tile[32][33];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (r < R && c < C) ? src[(long long)r * C + c] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (c < C && r < R) {
      const float x = tile[threadIdx.x][i], h = tf32_hi(x);
      hi[(long long)c * ldr + r] = h;
      lo[(long long)c * ldr + r] = tf32_lo(x, h);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// Tensor maps are pure functions of (base, rows, cols, pitch, box): the weights of a handle and the workspace
// operands of a bound minibatch see the same tuples on every iteration of every solveBatch, so the encoded
// descriptors are kept in a small per-thread table instead of calling cuTensorMapEncodeTiled four times per GEMM
// launch (VERDICT r01: 480 encodes per C2 solveBatch).  Direct-mapped, 256 entries, overwritten on collision.
struct TmapKey { const void* base; long long rows, cols, ld; int box; };
struct TmapSlot { TmapKey k; CUtensorMap tm; bool valid; };
static thread_local TmapSlot g_tmap_cache[256];

static int make_tmap_uncached(CUtensorMap* tm, const float* base, long long rows, long long cols, long long ld, int box_rows);

// 2-D fp32 tensor [rows, cols] (cols contiguous, row pitch ld floats), box = [box_rows, 32 cols], 128B swizzle
static int make_tmap(CUtensorMap* tm, const float* base, long long rows, long long cols, long long ld, int box_rows) {
  unsigned long long hsh = reinterpret_cast<unsigned long long>(base) >> 6;
  hsh ^= (unsigned long long)rows * 0x9E3779B97F4A7C15ull ^ (unsigned long long)cols * 0xC2B2AE3D27D4EB4Full ^
         (unsigned long long)ld * 0x165667B19E3779F9ull ^ (unsigned long long)box_rows;
  TmapSlot& sl = g_tmap_cache[(hsh ^ (hsh >> 17) ^ (hsh >> 31)) & 255];
  if (sl.valid && sl.k.base == base && sl.k.rows == rows && sl.k.cols == cols && sl.k.ld == ld && sl.k.box == box_rows) {
    *tm = sl.tm;
    return ICNN_OK;
  }
  const int rc = make_tmap_uncached(tm, base, rows, cols, ld, box_rows);
  if (rc == ICNN_OK) { sl.k = TmapKey{base, rows, cols, ld, box_rows}; sl.tm = *tm; sl.valid = true; }
  return rc;
}

static int make_tmap_uncached(CUtensorMap* tm, const float* base, long long rows, long long cols, long long ld, int box_rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled unavailable"); return ICNN_E_CUDA; }
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstr[1] = {(cuuint64_t)ld * sizeof(float)};
  cuuint32_t box[2] = {(cuuint32_t)TC_BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), gdim, gstr, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld ld=%lld", (int)r, rows, cols, ld); return ICNN_E_CUDA; }
  return ICNN_OK;
}

template <int BN, int NST_, bool GDB = false>
static cudaError_t launch_tc_variant(const CUtensorMap& tAh, const CUtensorMap& tAl, const CUtensorMap& tBh,
                                     const CUtensorMap& tBl, const TcArgs& a, int splitk, cudaStream_t st) {
  // per device / context attribute: set on every launch (a process-wide "done" flag would leave every device but
  // the first without it; the call is a host-side table update, ~1 us)
  {
    cudaError_t e = cudaFuncSetAttribute(tc_gemm_kernel<BN, NST_, GDB>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         TcSmem<BN, NST_>::TOTAL);
    if (e != cudaSuccess) return e;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(cdiv(a.N, BN), cdiv(a.M, TC_BM), splitk);
  cfg.blockDim = dim3(TC_THREADS);
  cfg.dynamicSmemBytes = TcSmem<BN, NST_>::TOTAL;
  cfg.stream = st;
  cudaLaunchAttribute lattr[1];
  lattr[0].id = cudaLaunchAttributeClusterDimension;
  lattr[0].val.clusterDim.x = 1; lattr[0].val.clusterDim.y = 1; lattr[0].val.clusterDim.z = splitk;
  cfg.attrs = lattr; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, tc_gemm_kernel<BN, NST_, GDB>, tAh, tAl, tBh, tBl, a);
}

static int launch_tc_gemm(const float* Ah, const float* Al, long long lda, const float* Bh, const float* Bl, long long ldb,
                          TcArgs a, cudaStream_t st, bool gdb = false) {
  const int gy = cdiv(a.M, TC_BM);
  // tile choice: 64-wide tiles; two CTAs per SM (the epilogue of one overlaps the main loop of the
  // other) once there are >= 2 tiles per SM, else one CTA per SM with a 4-deep ring.
  // ICNN_TC_CFG=128|64x4|64x2 forces a variant.
  const int sms = device_sms();
  int cfg = (cdiv(a.N, 64) * gy >= 2 * sms) ? 2 : 1;
  static const int env_cfg = [] {     // tuning knobs are read once per process, not per launch
    const char* v = getenv("ICNN_TC_CFG");
    if (!v) return -1;
    return !strcmp(v, "128") ? 0 : !strcmp(v, "64x4") ? 1 : !strcmp(v, "64x2") ? 2 : -1;
  }();
  static const int env_splitk = [] {
    const char* v = getenv("ICNN_TC_SPLITK");
    const int w = v ? atoi(v) : 0;
    return (w == 1 || w == 2 || w == 4 || w == 8) ? w : 0;
  }();
  static const int env_ch = [] {
    const char* v = getenv("ICNN_TC_CH");
    const int w = v ? atoi(v) : 0;
    return (w >= 1 && w <= 64) ? w : TC_CH;
  }();
  a.ch = env_ch;
  if (env_cfg >= 0) cfg = env_cfg;
  if (gdb && cfg == 0) cfg = 1;
  const int BN = cfg == 0 ? 128 : 64;
  CUtensorMap tAh, tAl, tBh, tBl;
  int rc;
  if ((rc = make_tmap(&tAh, Ah, a.M, a.K, lda, TC_BM))) return rc;
  if ((rc = make_tmap(&tAl, Al, a.M, a.K, lda, TC_BM))) return rc;
  if ((rc = make_tmap(&tBh, Bh, a.N, a.K, ldb, BN))) return rc;
  if ((rc = make_tmap(&tBl, Bl, a.N, a.K, ldb, BN))) return rc;
  // split-K over a cluster when the tile grid leaves most of the chip idle (C2: 4 row tiles)
  int splitk = 1;
  if (cfg == 1 && (a.mode == 0 || a.mode == 1)) {
    const int tiles = cdiv(a.N, 64) * gy, nkb = cdiv(a.K, TC_BK);
    while (splitk < 8 && tiles * splitk * 2 <= sms && nkb / (splitk * 2) >= 4) splitk *= 2;
    if (env_splitk) splitk = env_splitk;
  }
  cudaError_t e;
  if (gdb)   // GD training backward: the 64-wide variants with the tangent / accumulation epilogue
    e = cfg == 2 ? launch_tc_variant<64, 2, true>(tAh, tAl, tBh, tBl, a, 1, st)
                 : launch_tc_variant<64, 4, true>(tAh, tAl, tBh, tBl, a, cfg == 1 ? splitk : 1, st);
  else
    e = cfg == 0 ? launch_tc_variant<128, 3>(tAh, tAl, tBh, tBl, a, 1, st)
      : cfg == 1 ? launch_tc_variant<64, 4>(tAh, tAl, tBh, tBl, a, splitk, st)
                 : launch_tc_variant<64, 2>(tAh, tAl, tBh, tBl, a, 1, st);
  if (e != cudaSuccess) { set_error("tc_gemm launch: %s", cudaGetErrorString(e)); return ICNN_E_CUDA; }
  return ICNN_OK;
}

// Every shape is accepted: TMA needs 16-byte row pitches, so every library-owned operand (packed
// weights, K-concatenated activations, delta) is laid out with its leading dimension padded to 4
// floats (ld4); the tensor maps keep the true extents, so the pad is never read.
bool picnn_tc_supported(const icnn_picnn* h) {
  (void)h;
  return get_encode() != nullptr;
}

int picnn_tc_prepare_weights(icnn_picnn* h, cudaStream_t st) {
  for (int i = 0; i < h->L; ++i) {  // hidden layers only; the width-1 output layer stays on the SIMT kernel
    const int si = h->hidden[i], kf = h->prev(i) + h->n;
    // Wb: [kf, si] pitch ld4(si) (backward B operand); Wf: [si, kf] pitch ld4(kf) (forward B operand)
    for (float** p : {&h->Wb_hi[i], &h->Wb_lo[i], &h->Wf_hi[i], &h->Wf_lo[i]}) {
      const bool wb = (p == &h->Wb_hi[i] || p == &h->Wb_lo[i]);
      const size_t bytes = sizeof(float) * (wb ? (size_t)kf * ld4(si) : (size_t)si * ld4(kf));
      cudaError_t e = cudaMalloc(p, bytes);
      if (e != cudaSuccess) { set_error("cudaMalloc tc weights: %s", cudaGetErrorString(e)); return ICNN_E_CUDA; }
    }
    const long long N = (long long)kf * si;
    split_tf32_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(h->Wcat[i], h->Wb_hi[i], h->Wb_lo[i], kf, si, ld4(si));
    dim3 tb(32, 8), tg(cdiv(si, 32), cdiv(kf, 32));
    transpose_split_kernel<<<tg, tb, 0, st>>>(h->Wcat[i], h->Wf_hi[i], h->Wf_lo[i], kf, si, ld4(kf));
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_error("tc weight prep: %s", cudaGetErrorString(e)); return ICNN_E_CUDA; }
  return ICNN_OK;
}

void picnn_tc_free_weights(icnn_picnn* h) {
  for (int i = 0; i < ICNN_MAX_LAYERS; ++i)
    for (float** p : {&h->Wb_hi[i], &h->Wb_lo[i], &h->Wf_hi[i], &h->Wf_lo[i]})
      if (*p) { cudaFree(*p); *p = nullptr; }
}

// extra workspace (floats) after the SIMT part: per hidden layer A'_i hi/lo [B, s_{i-1}+n] (pitch ld4);
// delta hi/lo x2 (pitch ld4)
size_t picnn_tc_ws_floats(const icnn_picnn* h, int B, size_t* aoff, size_t* doff) {
  size_t off = 0;
  int smax = 0;
  auto al = [](size_t v) { return (v + 63) & ~(size_t)63; };
  for (int i = 0; i < h->L; ++i) {
    const size_t sz = al((size_t)B * ld4(h->prev(i) + h->n));
    if (aoff) { aoff[2 * i] = off; aoff[2 * i + 1] = off + sz; }
    off += 2 * sz;
    smax = h->hidden[i] > smax ? h->hidden[i] : smax;
  }
  const size_t dsz = al((size_t)B * ld4(smax));
  if (doff) for (int j = 0; j < 4; ++j) doff[j] = off + j * dsz;
  off += 4 * dsz;
  return off;
}

void out_layer_launch(const icnn_picnn* h, const icnn_gates* gt, const float* Zlast, const float* y32, float* f,
                      float* delta, float* delta_hi, float* delta_lo, float* g, long long g_row_stride,
                      const int* perm, const int* count, int KS, const int* skip, cudaStream_t st);
size_t picnn_simt_ws_floats(const icnn_picnn* h, int B, size_t* zoff, size_t* doff);

int picnn_fg_tc(const icnn_picnn* h, const icnn_gates* gt, const float* y32, float* f, float* g,
                long long g_row_stride, const int* perm, const int* count, int KS, void* workspace,
                const int* skip, cudaStream_t st) {
  const int B = gt->B, n = h->n, L = h->L;
  size_t zoff[ICNN_MAX_LAYERS], sdoff[2], aoff[2 * ICNN_MAX_LAYERS], doff[4];
  const size_t simt = picnn_simt_ws_floats(h, B, zoff, sdoff);
  picnn_tc_ws_floats(h, B, aoff, doff);
  float* ws = static_cast<float*>(workspace);
  float* tcw = ws + simt;
  float* Z[ICNN_MAX_LAYERS];
  float *Ah[ICNN_MAX_LAYERS], *Al[ICNN_MAX_LAYERS];
  for (int i = 0; i < L; ++i) { Z[i] = ws + zoff[i]; Ah[i] = tcw + aoff[2 * i]; Al[i] = tcw + aoff[2 * i + 1]; }
  float* dh[2] = {tcw + doff[0], tcw + doff[2]};
  float* dl[2] = {tcw + doff[1], tcw + doff[3]};

  {  // (s y + t) o cy_i for every hidden layer, straight into the K-concatenated operands
    GateYArgs ga{};
    ga.B = B; ga.n = n; ga.L = L; ga.y = y32; ga.sc = gt->in_scale; ga.sh = gt->in_shift; ga.skip_if_zero = skip;
    for (int i = 0; i < L; ++i) { ga.cy[i] = gt->cy[i]; ga.hi[i] = Ah[i]; ga.lo[i] = Al[i]; ga.ld[i] = ld4(h->prev(i) + n); ga.off[i] = h->prev(i); }
    const long long N = (long long)B * n;
    gate_y_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(ga);
  }
  for (int i = 0; i < L; ++i) {
    TcArgs a{};
    a.M = B; a.N = h->hidden[i]; a.K = h->prev(i) + n; a.mode = 0;
    a.D = gt->d[i]; a.Z = Z[i]; a.alpha = h->alpha; a.skip_if_zero = skip;
    if (i + 1 < L) { a.Cz_next = gt->cz[i + 1]; a.nxt_hi = Ah[i + 1]; a.nxt_lo = Al[i + 1]; a.nxt_ld = ld4(h->hidden[i] + n); }
    int rc = launch_tc_gemm(Ah[i], Al[i], ld4(a.K), h->Wf_hi[i], h->Wf_lo[i], ld4(a.K), a, st);
    if (rc) return rc;
  }
  out_layer_launch(h, gt, Z[L - 1], y32, f, nullptr, dh[0], dl[0], g, g_row_stride, perm, count, KS, skip, st);
  int cur = 0;
  for (int i = L - 1; i >= 0; --i) {
    TcArgs a{};
    a.M = B; a.N0 = h->prev(i); a.N = a.N0 + n; a.K = h->hidden[i]; a.mode = 1; a.alpha = h->alpha;
    a.Zprev = i ? Z[i - 1] : nullptr; a.Cz = i ? gt->cz[i] : nullptr; a.dprev_hi = dh[cur ^ 1]; a.dprev_lo = dl[cur ^ 1]; a.dprev_ld = ld4(a.N0);
    a.Cy = gt->cy[i]; a.g = g; a.g_row_stride = g_row_stride; a.perm = perm; a.count = count; a.KS = KS; a.n = n;
    a.g_scale = gt->g_scale; a.skip_if_zero = skip;
    int rc = launch_tc_gemm(dh[cur], dl[cur], ld4(a.K), h->Wb_hi[i], h->Wb_lo[i], ld4(a.K), a, st);
    if (rc) return rc;
    cur ^= 1;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_error("picnn_fg_tc launch: %s", cudaGetErrorString(e)); return ICNN_E_CUDA; }
  return ICNN_OK;
}

// ---- GD training backward on the tensor-core GEMMs (gd_backward.cu orchestrates) -----------------------
size_t picnn_gdb_tc_ws_floats(const icnn_picnn* h, int B, GdbTcBufs* b, float* base) {
  size_t off = 0;
  auto take = [&](size_t nfl) { size_t o = off; off += (nfl + 63) & ~(size_t)63; return base ? base + o : nullptr; };
  int smax = 0;
  for (int i = 0; i < h->L; ++i) {
    const size_t sz = (size_t)B * ld4(h->prev(i) + h->n);
    float* p0 = take(sz); float* p1 = take(sz); float* p2 = take(sz); float* p3 = take(sz);
    if (b) { b->Ah[i] = p0; b->Al[i] = p1; b->Ath[i] = p2; b->Atl[i] = p3; }
    smax = h->hidden[i] > smax ? h->hidden[i] : smax;
  }
  for (int j = 0; j < 2; ++j) {
    float* p0 = take((size_t)B * ld4(smax)); float* p1 = take((size_t)B * ld4(smax));
    if (b) { b->dh[j] = p0; b->dl[j] = p1; }
  }
  return off;
}

static void gdb_gate(const icnn_picnn* h, const icnn_gates* gt, const float* v, float* const* hi, float* const* lo,
                     cudaStream_t st) {
  GateYArgs ga{};
  ga.B = gt->B; ga.n = h->n; ga.L = h->L; ga.y = v; ga.sc = 1.f; ga.sh = 0.f; ga.skip_if_zero = nullptr;
  for (int i = 0; i < h->L; ++i) {
    ga.cy[i] = gt->cy[i]; ga.hi[i] = hi[i]; ga.lo[i] = lo[i]; ga.ld[i] = ld4(h->prev(i) + h->n); ga.off[i] = h->prev(i);
  }
  const long long N = (long long)gt->B * h->n;
  gate_y_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(ga);
}

// the (a o cy_i) columns of the tangent operands: constant over the GD iterations
void picnn_gdb_tc_gate_a(const icnn_picnn* h, const icnn_gates* gt, const float* a, const GdbTcBufs& b, cudaStream_t st) {
  gdb_gate(h, gt, a, b.Ath, b.Atl, st);
}

// primal forward of every hidden layer at b.y (and, with tangent, the tangent layers on direction a)
int picnn_gdb_tc_forward(const icnn_picnn* h, const icnn_gates* gt, const GdbTcBufs& b, bool tangent, cudaStream_t st) {
  const int B = gt->B, n = h->n, L = h->L;
  gdb_gate(h, gt, b.y, b.Ah, b.Al, st);
  for (int i = 0; i < L; ++i) {
    TcArgs a{};
    a.M = B; a.N = h->hidden[i]; a.K = h->prev(i) + n; a.mode = 0;
    a.D = gt->d[i]; a.Z = b.Z[i]; a.alpha = h->alpha;
    if (i + 1 < L) { a.Cz_next = gt->cz[i + 1]; a.nxt_hi = b.Ah[i + 1]; a.nxt_lo = b.Al[i + 1]; a.nxt_ld = ld4(h->hidden[i] + n); }
    int rc = launch_tc_gemm(b.Ah[i], b.Al[i], ld4(a.K), h->Wf_hi[i], h->Wf_lo[i], ld4(a.K), a, st, true);
    if (rc) return rc;
    if (tangent) {
      a.tangent = 1; a.D = b.Z[i]; a.Z = b.Zt[i];
      if (i + 1 < L) { a.nxt_hi = b.Ath[i + 1]; a.nxt_lo = b.Atl[i + 1]; }
      rc = launch_tc_gemm(b.Ath[i], b.Atl[i], ld4(a.K), h->Wf_hi[i], h->Wf_lo[i], ld4(a.K), a, st, true);
      if (rc) return rc;
    }
  }
  return ICNN_OK;
}

// backward GEMM of hidden layer i: delta_i (hi/lo in slot cur) -> delta_{i-1} (slot cur^1: hi/lo, optionally
// plain) and g; the optional accumulations / plain stores of GdbTcBufs run in the epilogue
int picnn_gdb_tc_backward_layer(const icnn_picnn* h, const icnn_gates* gt, const GdbTcBufs& b, int i, int cur,
                                cudaStream_t st) {
  TcArgs a{};
  a.M = gt->B; a.N0 = h->prev(i); a.N = a.N0 + h->n; a.K = h->hidden[i]; a.mode = 1; a.alpha = h->alpha;
  a.Zprev = i ? b.Z[i - 1] : nullptr; a.Cz = i ? gt->cz[i] : nullptr;
  a.dprev_hi = b.dh[cur ^ 1]; a.dprev_lo = b.dl[cur ^ 1]; a.dprev_ld = ld4(a.N0);
  a.Cy = gt->cy[i]; a.g = b.g; a.g_row_stride = h->n; a.n = h->n; a.g_scale = 1.f;
  if (i > 0) {
    if (b.want_plain) a.dprev_plain = b.dstore[i - 1] ? b.dstore[i - 1] : b.dp[cur ^ 1];
    a.acc_plain = b.astore[i];
    if (b.dcz[i]) { a.dCz = b.dcz[i]; a.Ztprev = b.Zt[i - 1]; }
    if (b.acc_delta) a.Dacc = b.Dacc[i - 1];
    a.kappa = b.kappa;
  }
  return launch_tc_gemm(b.dh[cur], b.dl[cur], ld4(a.K), h->Wb_hi[i], h->Wb_lo[i], ld4(a.K), a, st, true);
}

// stored-pattern phase, hidden layer l >= 1, all nIter iterations in one GEMM (M = nIter * B rows):
//   Zt[r, :] = act'(Zs[r, :]) o (P[r, :] Wz_l + Ty[r % B, :]),   P = zt_{l-1} o cz_l (TF32 hi/lo, pitch ld4)
int picnn_gdb_tc_stored_tangent(const icnn_picnn* h, int l, long long M, int B, const float* P_hi, const float* P_lo,
                                const float* Ty, const float* Zs, float* Zt, cudaStream_t st) {
  TcArgs a{};
  a.M = (int)M; a.N = h->hidden[l]; a.K = h->prev(l); a.mode = 0; a.tangent = 2; a.alpha = h->alpha;
  a.D = Ty; a.drow_mod = B; a.Zmask = Zs; a.Z = Zt;
  // Wf_l is [s_l, s_{l-1} + n] K-major: its first s_{l-1} columns are Wz_l^T
  return launch_tc_gemm(P_hi, P_lo, ld4(a.K), h->Wf_hi[l], h->Wf_lo[l], ld4(h->prev(l) + h->n), a, st, true);
}

// ---- x-path (gate precompute, SURVEY.md section 8f row 2) -------------------------------------------
// One GEMM per source activation P_s (P_0 = x, P_s = u_{s-1}) against the N-concatenated weights
//   [Wu_s | Wzu_s | Wyu_s | Wzx_s]   (multi-label-cls/icnn_ebundle.py:339-347,354-356,363-365,372-373)
// kept transposed ([N_total, K], K-major) and TF32 hi/lo split; bias, ReLU and the scatter into
// u / cz / cy / d are fused into the epilogue (mode 3).
int picnn_xpath_prepare(icnn_picnn* h, int m, const float* const* Wu, const float* const* bu,
                        const float* const* Wzu, const float* const* bzu, const float* const* Wyu,
                        const float* const* byu, const float* const* Wzx, const float* const* bzx, cudaStream_t st) {
  const int L = h->L, n = h->n;
  h->m = m;
  for (int s = 0; s <= L; ++s) {
    const int K = s == 0 ? m : h->hidden[s - 1];
    const int wu = s < L ? h->hidden[s] : 0, wzu = s >= 1 ? h->hidden[s - 1] : 0, wd = h->width(s);
    const int Nt = wu + wzu + n + wd;
    h->xN[s] = Nt; h->xK[s] = K;
    for (float** p : {&h->Xw_hi[s], &h->Xw_lo[s]})
      if (cudaMalloc(p, sizeof(float) * (size_t)Nt * ld4(K)) != cudaSuccess) { set_error("cudaMalloc x-path weights"); return ICNN_E_CUDA; }
    if (cudaMalloc(&h->Xbias[s], sizeof(float) * Nt) != cudaSuccess) { set_error("cudaMalloc x-path bias"); return ICNN_E_CUDA; }
    int off = 0;
    auto put = [&](const float* W, const float* bvec, int width) {   // W [K, width] row-major -> rows off.. of [Nt, K]
      if (width == 0) return;
      dim3 tb(32, 8), tg(cdiv(width, 32), cdiv(K, 32));
      transpose_split_kernel<<<tg, tb, 0, st>>>(W, h->Xw_hi[s] + (size_t)off * ld4(K), h->Xw_lo[s] + (size_t)off * ld4(K), K, width, ld4(K));
      cudaMemcpyAsync(h->Xbias[s] + off, bvec, sizeof(float) * width, cudaMemcpyDeviceToDevice, st);
      off += width;
    };
    if (s < L) put(Wu[s], bu[s], wu);
    if (s >= 1) put(Wzu[s], bzu[s], wzu);
    put(Wyu[s], byu[s], n);
    put(Wzx[s], bzx[s], wd);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_error("x-path prepare: %s", cudaGetErrorString(e)); return ICNN_E_CUDA; }
  h->has_xpath = true;
  return ICNN_OK;
}

void picnn_xpath_free(icnn_picnn* h) {
  for (int s = 0; s <= ICNN_MAX_LAYERS; ++s)
    for (float** p : {&h->Xw_hi[s], &h->Xw_lo[s], &h->Xbias[s]})
      if (*p) { cudaFree(*p); *p = nullptr; }
}

// workspace (floats): x hi/lo [B, m], u_s hi/lo [B, s_s] for s < L (row pitch ld4)
size_t picnn_xpath_ws_floats(const icnn_picnn* h, int B, size_t* off) {
  size_t o = 0;
  auto al = [](size_t v) { return (v + 63) & ~(size_t)63; };
  for (int s = 0; s <= h->L; ++s) {
    const size_t sz = al((size_t)B * ld4(s == 0 ? h->m : h->hidden[s - 1]));
    if (off) { off[2 * s] = o; off[2 * s + 1] = o + sz; }
    o += 2 * sz;
  }
  return o;
}

int picnn_gates_tc(const icnn_picnn* h, const float* x, int B, float* const* cz, float* const* cy, float* const* d,
                   void* workspace, cudaStream_t st) {
  const int L = h->L, n = h->n;
  size_t off[2 * (ICNN_MAX_LAYERS + 1)];
  picnn_xpath_ws_floats(h, B, off);
  float* ws = static_cast<float*>(workspace);
  split_tf32_kernel<<<(unsigned)(((long long)B * h->m + 255) / 256), 256, 0, st>>>(x, ws + off[0], ws + off[1], B, h->m, ld4(h->m));
  for (int s = 0; s <= L; ++s) {
    const int wu = s < L ? h->hidden[s] : 0, wzu = s >= 1 ? h->hidden[s - 1] : 0, wd = h->width(s);
    TcArgs a{};
    a.M = B; a.N = h->xN[s]; a.K = h->xK[s]; a.mode = 3; a.bias = h->Xbias[s];
    int r = 0, c = 0;
    a.rbeg[0] = 0;
    if (s < L) {   // u_s = (relu for s < L-1)(P Wu + bu): only needed as the next GEMM's hi/lo operand
      a.rrelu[r] = (s < L - 1); a.rdst[r] = nullptr; a.rld[r] = ld4(wu); a.r0_hi = ws + off[2 * (s + 1)]; a.r0_lo = ws + off[2 * (s + 1) + 1];
      c += wu; a.rbeg[++r] = c;
    }
    if (s >= 1) { a.rrelu[r] = 1; a.rdst[r] = cz[s]; a.rld[r] = wzu; c += wzu; a.rbeg[++r] = c; }
    a.rrelu[r] = 0; a.rdst[r] = cy[s]; a.rld[r] = n; c += n; a.rbeg[++r] = c;
    a.rrelu[r] = 0; a.rdst[r] = d[s]; a.rld[r] = wd; c += wd; a.rbeg[++r] = c;
    a.nr = r;
    int rc = launch_tc_gemm(ws + off[2 * s], ws + off[2 * s + 1], ld4(a.K), h->Xw_hi[s], h->Xw_lo[s], ld4(a.K), a, st);
    if (rc) return rc;
  }
  return ICNN_OK;
}

}  // namespace icnn

using namespace icnn;

extern "C" int icnn_picnn_set_xpath(icnn_picnn_t* h, int32_t m, const float* const* Wu, const float* const* bu,
                                    const float* const* Wzu, const float* const* bzu, const float* const* Wyu,
                                    const float* const* byu, const float* const* Wzx, const float* const* bzx,
                                    void* stream) {
  ICNN_REQUIRE(h && Wu && bu && Wzu && bzu && Wyu && byu && Wzx && bzx, "null pointer");
  ICNN_REQUIRE(m >= 1, "m must be positive");
  if (!h->use_tc) { set_error("x-path kernel needs the tensor-core path (ICNN_K1=simt build of the handle)"); return ICNN_E_UNSUPPORTED; }
  if (h->has_xpath) picnn_xpath_free(h);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = picnn_xpath_prepare(h, m, Wu, bu, Wzu, bzu, Wyu, byu, Wzx, bzx, st);
  if (rc) return rc;
  ICNN_CUDA_CHECK(cudaStreamSynchronize(st));
  return ICNN_OK;
}

extern "C" size_t icnn_picnn_gates_workspace_bytes(const icnn_picnn_t* h, int32_t B) {
  if (!h || !h->has_xpath || B <= 0) return 0;
  return sizeof(float) * picnn_xpath_ws_floats(h, B, nullptr);
}

extern "C" int icnn_picnn_gates(const icnn_picnn_t* h, const float* x, int32_t B, float* const* cz,
                                float* const* cy, float* const* d, void* workspace, void* stream) {
  ICNN_REQUIRE(h && x && cz && cy && d && workspace, "null pointer");
  ICNN_REQUIRE(B > 0, "empty batch");
  if (!h->has_xpath) { set_error("icnn_picnn_set_xpath was not called"); return ICNN_E_INVALID; }
  return picnn_gates_tc(h, x, B, cz, cy, d, workspace, static_cast<cudaStream_t>(stream));
}

// Self test of the tensor-core GEMM: C[M,N] = A[M,K] * B[N,K]^T (3xTF32), all device, row-major.
// scratch: (2*M + 2*N) * ((K+3)&~3) floats.
extern "C" int icnn_tc_gemm_selftest(const float* A, const float* B, float* C, int32_t M, int32_t N, int32_t K,
                                     float* scratch, void* stream) {
  ICNN_REQUIRE(A && B && C && scratch, "null pointer");
  ICNN_REQUIRE(M > 0 && N > 0 && K > 0, "empty problem");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int ld = ld4(K);
  float* Ah = scratch; float* Al = Ah + (size_t)M * ld; float* Bh = Al + (size_t)M * ld; float* Bl = Bh + (size_t)N * ld;
  split_tf32_kernel<<<(unsigned)(((long long)M * K + 255) / 256), 256, 0, st>>>(A, Ah, Al, M, K, ld);
  split_tf32_kernel<<<(unsigned)(((long long)N * K + 255) / 256), 256, 0, st>>>(B, Bh, Bl, N, K, ld);
  TcArgs a{};
  a.M = M; a.N = N; a.K = K; a.mode = 2; a.C = C;
  return launch_tc_gemm(Ah, Al, ld, Bh, Bl, ld, a, st);
}
