/*
 * icnn_b200 -- C ABI of the H100-native ICNN inner-loop library (libicnn_b200.so).
 *
 * Drop-in boundary for ONE hot path of locuslab/icnn: argmin_y f(x, y; theta) by the
 * bundle-entropy method and by unrolled momentum gradient descent.  The reference is pure
 * Python/numpy/TensorFlow and has no FFI of its own; each entry point below names the reference
 * function (path:line in the locuslab/icnn repository) whose work it replaces.  The Python side
 * (icnn_b200/_capi.py, ctypes) is the binding a maintainer of the reference would add -- see
 * INTEGRATION.md.
 *
 * Conventions
 *   - plain C types only; every pointer marked "device" is a CUDA device pointer owned by the
 *     caller (the Python layer allocates them as torch tensors); "host" pointers are host memory.
 *   - all calls are asynchronous on the caller-supplied cudaStream_t (passed as void*).
 *   - return value: 0 = ok, < 0 = error (ICNN_E_*); icnn_last_error() gives the message.
 *   - nothing here falls back to the CPU: without a CUDA device every compute call fails.
 *   - row-major everywhere; fully-connected weights are [in, out] (tflearn fully_connected).
 */
#ifndef ICNN_B200_H
#define ICNN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ICNN_ABI_VERSION 3

#define ICNN_OK 0
#define ICNN_E_INVALID (-1)  /* bad argument */
#define ICNN_E_CUDA (-2)     /* CUDA runtime error */
#define ICNN_E_UNSUPPORTED (-3)

/* per-sample status written by the bundle step */
#define ICNN_ST_RUNNING 0    /* still iterating (or stopped by the iteration cap) */
#define ICNN_ST_RANK_STOP 2  /* new row linearly dependent -> finished (lib/bundle_entropy.py:219-225) */
#define ICNN_ST_SOLVE_FAIL 3 /* Cholesky/Newton breakdown (RL/src/bundle_entropy.py:55-62 swallows it) */
#define ICNN_ST_NONFINITE 4  /* NaN/Inf met in f, g or the solve */
#define ICNN_ST_CONVERGED 5  /* RL: max|dy| < 1e-6 -> finished (RL/src/bundle_entropy.py:125-126) */

/* variant = which of the reference's three copies of solveBatch is reproduced */
#define ICNN_VARIANT_LIB 0  /* lib/bundle_entropy.py:192-242        */
#define ICNN_VARIANT_DUAL 1 /* lib/bundle_entropy_dual.py:129-179   */
#define ICNN_VARIANT_RL 2   /* RL/src/bundle_entropy.py:85-136      */

/* per-sample subproblem solver */
#define ICNN_SOLVER_PC 0     /* Mehrotra predictor-corrector, lib/bundle_entropy.py:5-78           */
#define ICNN_SOLVER_NEWTON 1 /* dual projected Newton, lib/bundle_entropy_dual.py:15-85 (+RL :14-83) */

typedef struct icnn_picnn icnn_picnn_t; /* opaque: device copies of the y-path weights */

/* y-path weights of a fully-connected PICNN (multi-label-cls/icnn_ebundle.py:316-388,
 * RL/src/icnn.py:325-404).  z-layers i = 0..L, widths hidden[0..L-1], output width 1. */
typedef struct {
  int32_t n;             /* n_y                                                        */
  int32_t L;             /* number of hidden z-layers (>= 1)                           */
  const int32_t* hidden; /* host [L]                                                   */
  float alpha;           /* leaky-ReLU slope; 0 = ReLU                                 */
  const float* const* Wy; /* host [L+1] of device ptrs; Wy[i] is [n, s_i]   ('z{i}_yu/W')      */
  const float* const* Wz; /* host [L+1] of device ptrs; Wz[i] is [s_{i-1}, s_i], Wz[0] = NULL
                             ('z{i}_zu_proj/W', >= 0)                                   */
} icnn_picnn_desc;

/* x-path products, constant over the inner loop (multi-label-cls/icnn_ebundle.py:354-373):
 * cy[i] [B, n], cz[i] [B, s_{i-1}] (cz[0] = NULL), d[i] [B, s_i]; host arrays of L+1 device ptrs.
 * in_scale/in_shift/g_scale implement the RL wrapper (RL/src/icnn.py:148-153): the network sees
 * in_scale*y + in_shift and the returned gradient is multiplied by g_scale ((1,0,1) otherwise). */
typedef struct {
  int32_t B;
  const float* const* cy;
  const float* const* cz;
  const float* const* d;
  float in_scale, in_shift, g_scale;
} icnn_gates;

/* Bundle state for B samples, all device memory, caller-owned.  Rows live in PHYSICAL slots;
 * perm[u, 0..count[u]) lists the active slots in the reference's list order and
 * perm[u, count[u]] is the free slot the next gradient row is written to. */
typedef struct {
  int32_t B, n, KS;  /* KS = slot capacity >= max active rows + 1 (<= 64: nIter <= 63)    */
  double* y;         /* [B, n]      iterate (float64, like the reference's x)          */
  float* y32;        /* [B, n]      iterate rounded for the fg kernel                  */
  float* f;          /* [B]         f(y) of the current iterate                        */
  float* G;          /* [B, KS, n]  gradient rows (the reference's A / G)              */
  double* ys;        /* [B, KS, n]  iterates the rows were taken at (xs); may be NULL  */
  double* h;         /* [B, KS]     offsets (b / h), by slot                           */
  double* lam;       /* [B, KS]     multipliers, by slot                               */
  double* rsum;      /* [B, KS]     row sums of G, by slot                             */
  double* gram;      /* [B, KS, KS] unweighted Gram of the rows, by slot               */
  int32_t* perm;     /* [B, KS]                                                        */
  int32_t* count;    /* [B]                                                            */
  int32_t* status;   /* [B]  ICNN_ST_*                                                 */
  int32_t* finished; /* [B]  0/1                                                       */
  int32_t* nIters;   /* [B]  the reference's nIters list                               */
  int32_t* nactive;  /* [nIterMax+1] unfinished samples entering iteration t           */
  int32_t* newton_its; /* [B] accumulated inner (IPM / Newton) iterations, diagnostics */
  int32_t* ksum;     /* [B] sum over executed iterations of the active row count k_t
                        (algorithmic-bytes accounting for the roofline, SURVEY.md section 8d) */
  const double* f64; /* [B] optional (may be NULL): f(y) in float64.  When set, h = f - g.y is formed from
                        it instead of the float32 f -- callback mode with a float64 fg, whose f the
                        reference keeps in float64 (lib/bundle_entropy.py:205-207)                      */
  double* iter_stats; /* [nIterMax, ICNN_NSTAT] optional (may be NULL): per-outer-iteration totals over the
                        samples solved in that iteration, accumulated with atomics (SURVEY.md section 5:
                        what the reference prints / plots per iteration, ebundle-vs-gd.py:94-99):
                        [0] samples entering the solve   [1] sum of active rows k      [2] sum of inner
                        (IPM / Newton) iterations        [3] sum of inner_its * k^2    [4] sum of inner_its * k
                        [5] samples stopped in this iteration (rank / convergence / non-finite)
                        [6] sum of f(y_t) - H(y_t) over the samples entering the iteration (0 log 0 = 0)
                        [7] reserved                                                                  */
  double* vec_ws;    /* optional (may be NULL): device scratch of B * 4 * ((n + 15) & ~15) doubles.  When set, the
                        predictor-corrector kernel may keep a sample's four n-vectors (y, u, ry, dy) there (L2-resident)
                        instead of in shared memory, which multiplies the samples in flight per SM (DESIGN.md K2)    */
} icnn_bundle_bufs;
#define ICNN_NSTAT 8

typedef struct {
  int32_t variant;     /* ICNN_VARIANT_*                                               */
  int32_t solver;      /* ICNN_SOLVER_*  (LIB: PC or NEWTON; DUAL/RL: NEWTON)           */
  int32_t line_search; /* Newton Armijo line search: 0/1 (reference: dual 0, rl 1)      */
  int32_t max_inner;   /* inner iteration cap; 0 = reference default (20 / 100 / 20)    */
  double prune_thr;    /* keep rows with lam > thr (1e-8 lib, 0 dual/rl)                */
  double rank_tol;     /* relative distance below which a new row counts as dependent   */
  int32_t nIter;       /* requested outer iterations (for nIters bookkeeping)           */
  int32_t reserved;
} icnn_bundle_cfg;

const char* icnn_last_error(void);
int icnn_abi_version(void);
/* number of CUDA devices visible, or <0 */
int icnn_device_count(void);

/* ---- K1: PICNN energy + gradient ------------------------------------------------------- */
/* replaces: the TF graph behind fg()  (multi-label-cls/icnn_ebundle.py:133,146,218-221;
 * RL/src/icnn.py:127,150-153).  Copies the weights into library-owned device buffers. */
int icnn_picnn_create(const icnn_picnn_desc* desc, icnn_picnn_t** out, void* stream);
int icnn_picnn_destroy(icnn_picnn_t* h);
/* bytes of caller-provided device scratch icnn_picnn_fg needs for B rows */
size_t icnn_picnn_workspace_bytes(const icnn_picnn_t* h, int32_t B);
/* f[u] = f(x_u, y_u), g row u = df/dy.  Row u of g goes to
 *   g + u*g_row_stride                                   if perm == NULL
 *   g + (u*KS + perm[u*KS + count[u]])*n                 otherwise (free slot of the bundle)
 * skip_if_zero (device int*, may be NULL): the launch is a no-op when *skip_if_zero == 0. */
int icnn_picnn_fg(const icnn_picnn_t* h, const icnn_gates* gates, const float* y32, float* f,
                  float* g, int64_t g_row_stride, const int32_t* perm, const int32_t* count,
                  int32_t KS, void* workspace, const int32_t* skip_if_zero, void* stream);

/* ---- x-path gate precompute (SURVEY.md section 8f, row 2) ------------------------------------------ */
/* replaces: the u-path and gate fully-connected layers of Model.f / Agent.negQ
 * (multi-label-cls/icnn_ebundle.py:339-347,354-356,363-365,372-373), evaluated once per solveBatch.
 * set_xpath hands the library the x-path weights (host arrays of device pointers, [in, out] layout;
 * Wu/bu: L entries, the others L+1, Wzu[0]/bzu[0] ignored); gates() then fills cz/cy/d for a
 * minibatch x [B, m] with one wgmma GEMM per source activation (bias, ReLU and the scatter into
 * the outputs fused into the epilogue).  ICNN_E_UNSUPPORTED when a width is not a multiple of 4. */
int icnn_picnn_set_xpath(icnn_picnn_t* h, int32_t m, const float* const* Wu, const float* const* bu,
                         const float* const* Wzu, const float* const* bzu, const float* const* Wyu,
                         const float* const* byu, const float* const* Wzx, const float* const* bzx,
                         void* stream);
size_t icnn_picnn_gates_workspace_bytes(const icnn_picnn_t* h, int32_t B);
int icnn_picnn_gates(const icnn_picnn_t* h, const float* x, int32_t B, float* const* cz, float* const* cy,
                     float* const* d, void* workspace, void* stream);

/* ---- K2: bundle-entropy step ------------------------------------------------------------- */
/* replaces: the per-sample loop body of solveBatch, lib/bundle_entropy.py:211-237 (and the dual /
 * RL copies), including pdipm_pc :5-78 / proj_newton_logistic. */
int icnn_bundle_init(const icnn_bundle_bufs* b, int32_t nIterMax, void* stream);
/* callback mode: scatter a dense g [B, n] (device, float32) into the free slots and f [B] */
int icnn_bundle_put_fg(const icnn_bundle_bufs* b, const float* f, const float* g, void* stream);
/* same for a float64 fg (the reference keeps whatever dtype fg returns and forms b = f - sum(g x) in
 * float64, lib/bundle_entropy.py:205-207): rows are rounded to the float32 row storage, f is kept in
 * float64 in b->f64 (which must be set) so that the cut offset h = f - g.y is formed from the float64 f. */
int icnn_bundle_put_fg_f64(const icnn_bundle_bufs* b, const double* f, const double* g, void* stream);
/* one outer iteration t for every unfinished sample: append row, dependency test, solve,
 * y update, prune.  f and the new row must already be in place. */
int icnn_bundle_step(const icnn_bundle_cfg* cfg, const icnn_bundle_bufs* b, int32_t t, void* stream);

/* ---- K3: argmin differentiation (SURVEY.md section 8f, row 1) ------------------------------------ */
/* replaces: crossEntrGrad (multi-label-cls/icnn_ebundle.py:390-417, loss = 1) / mseGrad
 * (completion/icnn_ebundle.py:493-522, loss = 0) and the (v, c) assembly of train_step_fd
 * (multi-label-cls/icnn_ebundle.py:296-314), on the final bundle state of a solve.
 * trueY [B, n] f64; outputs cy [B, n], clam [B, KS] (list order), ct [B], optional
 * V [B, KS, n] with V[u, i] = lam_i * cy + clam_i * (y* - ys_i)  (all device, f64). */
int icnn_argmin_grad(const icnn_bundle_bufs* b, int32_t loss, const double* trueY, double* cy,
                     double* clam, double* ct, double* V, void* stream);

/* ---- fused loops --------------------------------------------------------------------------- */
/* replaces: solveBatch end to end (lib/bundle_entropy.py:192-242) with fg = the PICNN handle:
 * nIter x (K1, K2) enqueued back to back on the stream, no host round trip; iterations after
 * every sample has finished are device-side no-ops (the reference returns early, :239). */
int icnn_solve_batch_fused(const icnn_picnn_t* h, const icnn_gates* gates, const icnn_bundle_cfg* cfg,
                           const icnn_bundle_bufs* b, void* workspace, void* stream);
/* The same loop as a CUDA graph (SURVEY.md section 7 step 5, "CUDA graph or persistent kernel"): the
 * reference crosses host<->device once per iteration (lib/bundle_entropy.py:204-205); here the
 * 2 + nIter*(2L+3) launches of icnn_solve_batch_fused are captured ONCE and replayed with a single
 * cudaGraphLaunch per solveBatch.  create() captures on a private stream (nothing executes); every device
 * pointer reachable from (h, gates, b, workspace) and the values of cfg are baked in, so launch() is only
 * valid while those buffers are alive and at the same addresses (the Python layer keys its cache on them).
 * nodes() = kernel nodes in the graph (= gpu launches replayed per call). */
typedef struct icnn_loop_graph icnn_loop_graph_t;
int icnn_loop_graph_create(const icnn_picnn_t* h, const icnn_gates* gates, const icnn_bundle_cfg* cfg,
                           const icnn_bundle_bufs* b, void* workspace, icnn_loop_graph_t** out);
int icnn_loop_graph_launch(icnn_loop_graph_t* g, void* stream);
int64_t icnn_loop_graph_nodes(const icnn_loop_graph_t* g);
int icnn_loop_graph_destroy(icnn_loop_graph_t* g);
/* replaces: the unrolled momentum-GD inner loop, multi-label-cls/icnn-back.py:116-131
 * (= completion/icnn.back.py:133-147).  y32 [B,n] in/out, v [B,n] scratch, f_out [B] = f(y_n). */
int icnn_gd_solve(const icnn_picnn_t* h, const icnn_gates* gates, float* y32, float* v, float* g,
                  float* f_out, int32_t nIter, float lr, float momentum, void* workspace,
                  void* stream);

/* ---- training backward of the unrolled GD loop (SURVEY.md section 8f, row 4) ------------------------ */
/* replaces: TensorFlow's double backprop behind opt.compute_gradients(self.mse_, self.theta_) on the
 * graph that unrolls the momentum-GD loop (multi-label-cls/icnn-back.py:120-139,
 * completion/icnn.back.py:133-156).  Runs the loop from y0 [B,n] (f32), writes y_N to yN [B,n], takes
 * a = loss_scale * (y_N - trueY) as d loss / d y_N (mse_ = reduce_mean(square(yn - trueY)):
 * loss_scale = 2/(B n); completion: 2*255^2/(B n)) and returns d loss / d (y-path weights and gates):
 *   dWy[l] [n, s_l], dWz[l] [s_{l-1}, s_l], dcy[l] [B, n], dcz[l] [B, s_{l-1}]   (l = 0..L; [0] of
 *   dWz/dcz unused; the additive gate d_l gets no gradient).  All buffers device f32, overwritten.
 * The x-path parameters follow from (dcy, dcz) by ordinary dense-layer backprop on the caller's side.
 * workspace = icnn_gd_backward_workspace_bytes(h, B, nIter) device bytes (it includes, when it fits
 * ICNN_GDB_STORE_GB, the per-iteration stores of the single-pass mode).  The affine RL wrapper is not
 * supported here (ICNN_E_UNSUPPORTED). */
typedef struct {
  float* const* dWy;
  float* const* dWz;
  float* const* dcy;
  float* const* dcz;
} icnn_gd_grads;
size_t icnn_gd_backward_workspace_bytes(const icnn_picnn_t* h, int32_t B, int32_t nIter);
int icnn_gd_backward(const icnn_picnn_t* h, const icnn_gates* gates, const float* y0, const float* trueY,
                     float loss_scale, int32_t nIter, float lr, float momentum, float* yN,
                     const icnn_gd_grads* grads, void* workspace, void* stream);

/* ---- RL Adam argmin (SURVEY.md section 8f, row 3) -------------------------------------------------- */
/* replaces: Agent.adam (RL/src/icnn.py:160-215) applied to [negQ - entropy(act), d/dact]
 * (RL/src/icnn.py:60-63,127-131,455-458): batched Adam on the actions with best-so-far tracking and
 * the rolling-average stop, looped on the device (the stop flag is read back every 16 iterations).
 * gates must be bound WITHOUT the affine wrapper (the network sees act in [-1,1] directly).
 * act_best [B, n] f64 and f_best [B] f64 are outputs; iters_out (host) gets the reference's iteration
 * count; scratch = icnn_adam_workspace_bytes(B, n) device bytes, workspace = icnn_picnn_workspace_bytes. */
size_t icnn_adam_workspace_bytes(int32_t B, int32_t n);
int icnn_adam_solve(const icnn_picnn_t* h, const icnn_gates* gates, double* act_best, double* f_best,
                    int32_t max_iter, int32_t* iters_out, void* scratch, void* workspace, void* stream);

/* ---- diagnostics ------------------------------------------------------------------------------ */
/* Self test of the wgmma / TMA GEMM the tensor-core K1 path is built from:
 * C[M,N] = A[M,K] * B[N,K]^T with the 3xTF32 split (all row-major device buffers, K % 4 == 0;
 * scratch holds 2*M*K + 2*N*K floats). */
int icnn_tc_gemm_selftest(const float* A, const float* B, float* C, int32_t M, int32_t N, int32_t K,
                          float* scratch, void* stream);
/* FP64 tensor-core throughput probe: every warp of a full-chip grid issues `iters` x 8 independent
 * mma.m8n8k4.f64 (the instruction K2's weighted-Gram sweep is built from); *flops_out (host) = FLOPs the
 * launch performs, sink (device, 1 double) keeps the result alive.  bench.py times it with CUDA events to
 * get the denominator of K2's roofline (MEASURED_PEAKS.json has no FP64 entry). */
int icnn_fp64_mma_probe(int32_t iters, double* sink, double* flops_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ICNN_B200_H */
