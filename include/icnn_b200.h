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

/* 7: icnn_bundle_bufs ends at iter_stats (the vec_ws scratch pointer of version 6 is gone; 19 pointers)
 * 8: the conv PICNN training gradient (icnn_conv_train_grads, icnn_conv_train_grad)
 * 9: the conv PICNN GD training backward (icnn_conv_gd_backward) */
#define ICNN_ABI_VERSION 9

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

/* ---- bundle-entropy training gradient (SURVEY.md section 8f, row 1: the step after K3) ---------------- */
/* replaces: opt.compute_gradients(F_, theta_) (multi-label-cls/icnn_ebundle.py:154) on the surrogate
 *   F_ = c * E(x, y) + sum_j v_j dE/dy_j          (multi-label-cls/icnn_ebundle.py:148)
 * fed the train_step_fd rows (:296-314) in CSR form: sample u owns rows row_offsets[u] .. row_offsets[u+1]
 * (host int64 [B+1], row_offsets[0] = 0, non-decreasing, R = row_offsets[B]) of Y [R, n] (bundle points),
 * V [R, n] and c [R] (all device f32, the reference's float32 placeholders :129-131); row r sees the gates of
 * its sample (the bound minibatch's row u).  Returns d (sum of F_ over all rows) / d (y-path weights and gates):
 *   dWy[l] [n, s_l], dWz[l] [s_{l-1}, s_l]   summed over every row
 *   dcy[l] [B, n], dcz[l] [B, s_{l-1}], dd[l] [B, s_l]   per sample (summed over the sample's rows)
 * for l = 0..L ([0] of dWz/dcz unused).  All buffers device f32, overwritten.  The x-path parameters follow from
 * (dcy, dcz, dd) by dense-layer backprop on the caller's side.  workspace =
 * icnn_train_grad_workspace_bytes(h, B, R) device bytes; rows are processed in chunks, so it does not grow with R
 * beyond ICNN_TRAIN_WS_GB (default 2) GiB.  The affine RL wrapper is not supported (ICNN_E_UNSUPPORTED): the
 * RL code's bundle path is disabled in the reference (RL/src/icnn.py:84). */
typedef struct {
  float* const* dWy;
  float* const* dWz;
  float* const* dcy;
  float* const* dcz;
  float* const* dd;
} icnn_train_grads;
size_t icnn_train_grad_workspace_bytes(const icnn_picnn_t* h, int32_t B, int64_t R);
int icnn_train_grad(const icnn_picnn_t* h, const icnn_gates* gates, const int64_t* row_offsets, const float* Y,
                    const float* V, const float* c, const icnn_train_grads* grads, void* workspace, void* stream);

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

/* ---- convolutional PICNN (the image-completion energy) ------------------------------------------ */
/* replaces: the TF graph behind fg() of the completion experiment, Model.f (completion/icnn_ebundle.py:337-452,
 * = completion/icnn.back.py:276-396) with E_ / dE_dy_ (:118-120).  Images are H x W, y and x are [B, H*W] in
 * row-major H x W order, feature maps NHWC.  Conv z-layers l = 0..Lc-1 with (C[l], k[l], s[l]) and TensorFlow
 * 'SAME' padding (H_{l+1} = ceil(H_l / s_l), the odd pad at the end), then dense z-layers of widths fcs[0..Ld-1],
 * fcs[Ld-1] = 1 (the energy).  Weight layouts are TensorFlow's (host arrays of device pointers):
 *   Wz[l]   conv l:  [k, k, C_{l-1}, C_l]  ('z{l}_zu_proj/W', >= 0; Wz[0] = NULL)
 *           dense:   [in, out]             ('z{i}_zu_proj/W', in = flat size of z_{i-1}, NHWC order)
 *   Wy[l]   [k, k, 1, C_l]  ('z{l}_yu/W'),  Wred[l] [k, k, 1, 1], bred[l] [1]  ('z{l}_y_red/W|b'), l < Lc
 * The gates are an icnn_gates over Lc + Ld layers (x-path products, computed once per minibatch):
 *   conv l:   cy[l] [B, H_l, W_l], cz[l] [B, H_l, W_l, C_{l-1}] (cz[0] = NULL), d[l] [B, H_{l+1}, W_{l+1}, C_l]
 *   dense i:  cy[i] = NULL, cz[i] [B, in_i], d[i] [B, fcs]
 *   in_scale, in_shift, g_scale must be (1, 0, 1). */
typedef struct icnn_conv_picnn icnn_conv_picnn_t; /* opaque: packed device copies of the y-path weights */
typedef struct {
  int32_t H, W;
  int32_t Lc;             /* conv z-layers, 1..8                                         */
  const int32_t* C;       /* host [Lc] output channels                                   */
  const int32_t* k;       /* host [Lc] kernel sizes                                      */
  const int32_t* s;       /* host [Lc] strides                                           */
  int32_t Ld;             /* dense z-layers including the width-1 output, 1..8           */
  const int32_t* fcs;     /* host [Ld] widths, fcs[Ld-1] = 1                             */
  const float* const* Wz; /* host [Lc + Ld]                                              */
  const float* const* Wy; /* host [Lc]                                                   */
  const float* const* Wred; /* host [Lc]                                                 */
  const float* const* bred; /* host [Lc]                                                 */
} icnn_conv_picnn_desc;
int icnn_conv_picnn_create(const icnn_conv_picnn_desc* desc, icnn_conv_picnn_t** out, void* stream);
int icnn_conv_picnn_destroy(icnn_conv_picnn_t* h);
/* bytes of caller-provided device scratch icnn_conv_picnn_fg needs for B rows */
size_t icnn_conv_picnn_workspace_bytes(const icnn_conv_picnn_t* h, int32_t B);
/* f and df/dy with the argument list and g-row placement of icnn_picnn_fg (n = H*W). */
int icnn_conv_picnn_fg(const icnn_conv_picnn_t* h, const icnn_gates* gates, const float* y32, float* f,
                       float* g, int64_t g_row_stride, const int32_t* perm, const int32_t* count,
                       int32_t KS, void* workspace, const int32_t* skip_if_zero, void* stream);
/* replaces: solveBatch (lib/bundle_entropy.py:192-242) as the completion script calls it with this energy
 * (completion/icnn_ebundle.py:218-226): icnn_bundle_init + nIter x (icnn_conv_picnn_fg, icnn_bundle_step). */
int icnn_conv_solve_batch_fused(const icnn_conv_picnn_t* h, const icnn_gates* gates, const icnn_bundle_cfg* cfg,
                                const icnn_bundle_bufs* b, void* workspace, void* stream);
/* replaces: the unrolled momentum-GD inner loop of completion/icnn.back.py:133-147 on this energy; the
 * arguments are those of icnn_gd_solve. */
int icnn_conv_gd_solve(const icnn_conv_picnn_t* h, const icnn_gates* gates, float* y32, float* v, float* g,
                       float* f_out, int32_t nIter, float lr, float momentum, void* workspace, void* stream);

/* replaces: compute_gradients(F_, theta_) of the completion experiment (completion/icnn_ebundle.py:129-140) on
 * F_ = c E(x, y) + sum_j v_j dE/dy_j, summed over the train_step_fd rows (:315-335), for this energy.  The rows
 * and the gates follow icnn_train_grad: row_offsets (host, [B + 1], CSR), Y, V [R, H*W], c [R] device f32, gates
 * the per-sample gates of the minibatch.  Outputs (host arrays of device f32 pointers, all overwritten):
 *   dWz[Lc + Ld]   conv l: [k, k, C_{l-1}, C_l] (dWz[0] unused), dense: [in, out]       summed over every row
 *   dWy[Lc]        [k, k, 1, C_l]
 *   dWred[Lc]      [k, k, 1, 1], dbred[Lc] [1]; entry Lc-1 unused (r_{Lc} feeds nothing)
 *   dcy[Lc], dcz[Lc + Ld] (dcz[0] unused), dd[Lc + Ld]   per sample, in the gate layouts above
 * The x-path parameters follow from (dcy, dcz, dd) by backprop through the gates on the caller's side.
 * workspace = icnn_conv_train_grad_workspace_bytes(h, B, R) device bytes; rows are processed in chunks bounded as
 * for icnn_train_grad (ICNN_TRAIN_WS_GB, default 2 GiB; ICNN_TRAIN_CHUNK). */
typedef struct {
  float* const* dWz;
  float* const* dWy;
  float* const* dWred;
  float* const* dbred;
  float* const* dcy;
  float* const* dcz;
  float* const* dd;
} icnn_conv_train_grads;
size_t icnn_conv_train_grad_workspace_bytes(const icnn_conv_picnn_t* h, int32_t B, int64_t R);
int icnn_conv_train_grad(const icnn_conv_picnn_t* h, const icnn_gates* gates, const int64_t* row_offsets,
                         const float* Y, const float* V, const float* c, const icnn_conv_train_grads* grads,
                         void* workspace, void* stream);
/* replaces: TensorFlow's double backprop behind opt.compute_gradients(self.mse_, self.theta_) of the completion
 * experiment's back-optimisation mode (completion/icnn.back.py:133-156) for this energy: the nIter unrolled
 * momentum-GD steps of icnn_conv_gd_solve (lr = 0.01, momentum = 0.9 at :133-134) from y0 [B, H*W], then
 * mse_ = reduce_mean(square(255 (yn_ - trueY))) (:149).  The arguments are those of icnn_gd_backward: y_N goes to yN
 * [B, H*W] (bit-identical to icnn_conv_gd_solve with the same arguments), a = loss_scale (y_N - trueY) is d loss /
 * d y_N (completion: loss_scale = 2 255^2 / (B H W)).  Outputs in the icnn_conv_train_grads layouts, all overwritten:
 * d loss / d (y-path weights) summed over the batch, and the per-sample gate adjoints dcy, dcz; dd and dbred come
 * back zero (the additive gates do not enter dE/dy, and TensorFlow's graph gives the y_red bias a zero gradient).
 * The gradient is that of icnn_conv_train_grad on one row per (sample, step): the rows are chunked the same way.
 * workspace = icnn_conv_gd_backward_workspace_bytes(h, B, nIter) device bytes: the trajectory and the row seeds
 * (2 B nIter H W floats) plus the chunked gradient's workspace; 0 for arguments it cannot size (B * nIter must be
 * at most 2^31 - 1 rows).  nIter = 0 gives yN = y0 and zero gradients. */
size_t icnn_conv_gd_backward_workspace_bytes(const icnn_conv_picnn_t* h, int32_t B, int32_t nIter);
int icnn_conv_gd_backward(const icnn_conv_picnn_t* h, const icnn_gates* gates, const float* y0, const float* trueY,
                          float loss_scale, int32_t nIter, float lr, float momentum, float* yN,
                          const icnn_conv_train_grads* grads, void* workspace, void* stream);

/* ---- diagnostics ------------------------------------------------------------------------------ */
/* Self test of the wgmma / TMA GEMM the tensor-core K1 path is built from:
 * C[M,N] = A[M,K] * B[N,K]^T with the 3xTF32 split (all row-major device buffers, any M, N, K >= 1;
 * scratch holds (2*M + 2*N) * ((K + 3) & ~3) floats: the split operands, rows padded to 4 floats). */
int icnn_tc_gemm_selftest(const float* A, const float* B, float* C, int32_t M, int32_t N, int32_t K,
                          float* scratch, void* stream);
/* Pins the tensor-core GEMM's tuning for every later launch in the process (all threads), on top of the
 * ICNN_TC_CFG / ICNN_TC_SPLITK / ICNN_TC_CH environment variables; -1 = automatic / default.
 *   cfg: 0 = 128-wide tiles, 3-stage ring; 1 = 64-wide, 4 stages; 2 = 64-wide, 2 stages (two CTAs per SM)
 *   splitk: 1, 2, 4 or 8 (applies only to cfg 1 and to the GEMMs with a split-K epilogue, not the x-path gates)
 *   ch: 1..64 half k-blocks (K = 16 each) per round-to-nearest accumulation chunk
 * The GD training backward has no 128-wide variant and runs cfg 0 as cfg 1.  Out-of-range values return
 * ICNN_E_INVALID and leave the current setting unchanged. */
int icnn_tc_set_tuning(int32_t cfg, int32_t splitk, int32_t ch);
/* out (host, 5 int32) = {tile width BN, ring stages, split-K factor, chunk length, mode} of the calling thread's
 * most recent tensor-core GEMM launch (mode 0 forward, 1 backward, 2 self test, 3 x-path gates; -1 = none yet). */
int icnn_tc_last_launch(int32_t out[5]);
/* Which K2 build icnn_bundle_step launches for a problem of n_y = n with KS bundle slots, decided on the host from
 * the shape, the solver and the launch environment variables (read at every call, as at every launch); nothing is
 * enqueued and no device is touched.  variant / solver are checked as icnn_bundle_step checks them.  A shape no
 * build fits returns ICNN_E_UNSUPPORTED with the message the launch would set.  out (host, ICNN_K2_PLAN_LEN int32):
 *   out[0] kernel family: 0 thread-per-sample (bundle_step_small), 1 two-sweep PC kernel, 2 five-sweep kernel
 *   out[1] warps per sample (0 for the thread-per-sample kernel)
 *   out[2] column chunks per thread (two-sweep) or CTAs per cluster (five-sweep; 1 = no cluster); 0 otherwise
 *   out[3] 1 = two-sweep V3 build (three n-vectors per sample)
 *   out[4] 1 = 16-byte row loads / tensor-core Gram (n_y % 4 == 0), 0 = scalar row loads / SIMT Gram
 *   out[5] 1 = bundle rows resident in shared memory (five-sweep ICNN_K2_RESIDENT=1), 0 = streamed from L2
 *   out[6] minBlocks of the instantiation's __launch_bounds__ (0 = none given)
 *   out[7] dynamic shared memory per CTA in bytes */
#define ICNN_K2_PLAN_LEN 8
int icnn_k2_plan(int32_t n, int32_t KS, int32_t solver, int32_t variant, int32_t out[ICNN_K2_PLAN_LEN]);
/* out (host, ICNN_K2_PLAN_LEN int32) = the icnn_k2_plan record of the calling thread's most recent K2 enqueue
 * (icnn_bundle_step, the fused loop or a loop-graph capture); out[0] = -1 and zeros when there was none yet. */
int icnn_k2_last_launch(int32_t out[ICNN_K2_PLAN_LEN]);
/* FP64 tensor-core throughput probe: every warp of a full-chip grid issues `iters` x 8 independent
 * mma.m8n8k4.f64 (the instruction K2's weighted-Gram sweep is built from); *flops_out (host) = FLOPs the
 * launch performs, sink (device, 1 double) keeps the result alive.  bench.py times it with CUDA events to
 * get the denominator of K2's roofline (MEASURED_PEAKS.json has no FP64 entry). */
int icnn_fp64_mma_probe(int32_t iters, double* sink, double* flops_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ICNN_B200_H */
