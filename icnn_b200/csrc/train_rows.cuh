// Row bookkeeping shared by the training gradients (train_grad.cu, conv_train_grad.cu): feed rows come in CSR order
// (sample u owns rows [off[u], off[u + 1])) and are processed in chunks cut at sample boundaries.
#pragma once
#include "common.cuh"

#include <cstdlib>

namespace icnn {

static __global__ void round_to_float_kernel(float* dst, const double* src, long long N) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < N) dst[i] = (float)src[i];
}

// sample of each chunk row: the u in [u0, u1) with off[u] <= r0 + i < off[u + 1]
static __global__ void row_sample_kernel(int* row_u, const long long* off, int u0, int u1, long long r0, int rows) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows) return;
  const long long r = r0 + i;
  int lo = u0, hi = u1 - 1;   // largest u with off[u] <= r
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= r) lo = mid; else hi = mid - 1;
  }
  row_u[i] = lo;
}

// dst[i, j] = src[row_u[i], j]
static __global__ void gather_rows_kernel(float* dst, const float* src, const int* row_u, long long N, int w) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < N) dst[i] = src[(long long)row_u[i / w] * w + i % w];
}

// element (r, j) of a per-row array: hi[r rs + (j / grp) gs + j % grp + goff] (+ lo at the same index);
// hi == nullptr: 1.  SegView{p, nullptr, w, w, 0, 0} is a plain [rows, w] array.
struct SegView {
  const float* hi; const float* lo; long long rs; int grp, gs, goff;
};
__device__ __forceinline__ double seg_at(const SegView& v, long long r, int j) {
  if (!v.hi) return 1.0;
  const long long i = r * v.rs + (long long)(j / v.grp) * v.gs + j % v.grp + v.goff;
  return v.lo ? (double)(v.hi[i] + v.lo[i]) : (double)v.hi[i];
}

// out[u, j] += sum over the rows r of sample u inside [r0, r1) of scale[r] a(r - r0, j) e(r - r0, j) (scale ==
// nullptr: 1), rows in order.  Accumulated in float64: the bundle multipliers c of a sample sum to zero (the KKT
// row of ones), so e.g. dd_L = sum_r c_r is pure cancellation and a float32 sum of O(|c|) terms would leave
// rounding noise larger than the result.
static __global__ void segsum_prod_kernel(float* out, SegView a, SegView e, const float* scale, int w,
                                          const long long* off, int u0, int u1, long long r0, long long r1) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)(u1 - u0) * w) return;
  const int u = u0 + (int)(i / w), j = (int)(i % w);
  const long long ra = off[u] > r0 ? off[u] : r0, rb = off[u + 1] < r1 ? off[u + 1] : r1;
  double acc = 0.0;
  for (long long r = ra; r < rb; ++r) {
    const double v = seg_at(a, r - r0, j) * seg_at(e, r - r0, j);
    acc = scale ? fma((double)scale[r], v, acc) : acc + v;
  }
  out[(long long)u * w + j] = (float)((double)out[(long long)u * w + j] + acc);
}

// launches over one chunk (256 threads per block): rows rows from r0, samples [u0, u1)
static inline void launch_row_sample(int* row_u, const long long* off, int u0, int u1, long long r0, int rows,
                                     cudaStream_t st) {
  row_sample_kernel<<<cdiv(rows, 256), 256, 0, st>>>(row_u, off, u0, u1, r0, rows);
}
// dst [rows, w] = the rows of src [B, w] of each chunk row's sample
static inline void launch_gather_rows(float* dst, const float* src, const int* row_u, int rows, long long w,
                                      cudaStream_t st) {
  const long long N = (long long)rows * w;
  gather_rows_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(dst, src, row_u, N, (int)w);
}
static inline void launch_segsum_prod(float* out, SegView a, SegView e, const float* scale, long long w,
                                      const long long* off, int u0, int u1, long long r0, long long r1,
                                      cudaStream_t st) {
  const long long N = (long long)(u1 - u0) * w;
  segsum_prod_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(out, a, e, scale, (int)w, off, u0, u1, r0, r1);
}

// The CSR row offsets of B > 0 samples: row_offsets[0] = 0, non-decreasing, at most 2^31 - 1 rows, and the row
// inputs given (have_rows) when there are rows.  Returns R = row_offsets[B], or ICNN_E_INVALID with the error set.
static inline long long check_row_offsets(const int64_t* row_offsets, int B, bool have_rows) {
  ICNN_REQUIRE(row_offsets[0] == 0, "row_offsets[0] != 0");
  for (int u = 0; u < B; ++u) ICNN_REQUIRE(row_offsets[u + 1] >= row_offsets[u], "row_offsets decreasing");
  const long long R = row_offsets[B];
  ICNN_REQUIRE(R <= INT32_MAX, "more than 2^31 - 1 rows");
  ICNN_REQUIRE(R == 0 || have_rows, "null row input");
  return R;
}

// rows per chunk: ICNN_TRAIN_CHUNK if set, else what fits ICNN_TRAIN_WS_GB (default 2) GiB at bytes_per_row
// (at least 64, at most R)
static inline long long chunk_rows(double bytes_per_row, long long R) {
  if (const char* v = getenv("ICNN_TRAIN_CHUNK")) {
    const long long c = atoll(v);
    if (c > 0) return c < R ? c : R;
  }
  double gb = 2.0;
  if (const char* v = getenv("ICNN_TRAIN_WS_GB")) gb = atof(v);
  long long c = (long long)(gb * 1073741824.0 / bytes_per_row);
  if (c < 64) c = 64;
  return c < R ? c : R;
}

// the chunk after row r0 < R: *u0 advances to the first sample with rows left; rows [r0, *r1) of samples
// [*u0, *u1).  Balanced chunks: k = ceil(rest / cap) pieces of about rest / k rows, cut at the first sample boundary
// past that size that still fits the cap; a single sample longer than the cap is split
static inline void next_chunk(const int64_t* row_offsets, int B, long long R, long long cap, long long r0, int* u0,
                              long long* r1_out, int* u1_out) {
  while (row_offsets[*u0 + 1] <= r0) ++*u0;
  const long long rest = R - r0, k = (rest + cap - 1) / cap, target = (rest + k - 1) / k;
  long long r1 = r0;
  int u1 = *u0;
  while (u1 < B && row_offsets[u1 + 1] - r0 <= cap && r1 - r0 < target) r1 = row_offsets[++u1];
  if (r1 == r0) { r1 = r0 + cap; u1 = *u0 + 1; }
  else while (u1 < B && row_offsets[u1] < r1) ++u1;   // (u1 = one past the last sample with rows in the chunk)
  *r1_out = r1;
  *u1_out = u1;
}

}  // namespace icnn
