// lbfgs_dev.cu -- device-resident batched L-BFGS-B driver for binary columns and multinomial candidates.
//
// Replaces the host loop scipy/optimize/_lbfgsb_py.py:406-437 (setulb reverse communication)
// that each of the reference's tasks runs inside estimator.fit (ref search.py:230); the
// optimiser arithmetic is csrc/lbfgs_core.h.  Per round:
//   lb_step_kernel    : gather the entry's partial sums -> f, g (float64, adds the L2 term as
//                       SK/linear_model/_linear_loss.py:350,356-361), advance the state machine
//   lb_compact_kernel : rebuild the list of still-running problems (stable order)
//   lb_export_kernel  : cast the new trial points to fp32 (SK/_linear_loss.py:216-217) into the
//                       active-slot weight matrix for the next evaluation
#include "skd_internal.h"

namespace skd {

constexpr int LB_THREADS = 128;

// One CTA per problem: reductions over the CTA's four warps.
struct CtaPar {
  static constexpr int PER_CTA = 1;   // problems per LB_THREADS-thread CTA
  double* red;  // shared, >= 4 doubles
  __device__ __forceinline__ int tid() const { return threadIdx.x; }
  __device__ __forceinline__ int nthr() const { return LB_THREADS; }
  __device__ __forceinline__ void sync() const { __syncthreads(); }
  __device__ __forceinline__ double block_sum(double v) const {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();  // protect red from the previous reduction's readers
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    return (red[0] + red[1]) + (red[2] + red[3]);
  }
  __device__ __forceinline__ double dot(const double* a, const double* b, int n) const {
    double acc = 0.0;
    for (int i = threadIdx.x; i < n; i += LB_THREADS) acc += a[i] * b[i];
    return block_sum(acc);
  }
  __device__ __forceinline__ double amax(const double* a, int n) const {
    double m = 0.0;
    for (int i = threadIdx.x; i < n; i += LB_THREADS) m = fmax(m, fabs(a[i]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    return fmax(fmax(red[0], red[1]), fmax(red[2], red[3]));
  }
};

// One WARP per column: no block barriers, reductions by shuffles.  The optimiser's vector
// operations are a few hundred elements long; a 128-thread CTA spent most of its time in the two
// barriers of every reduction.
struct WarpPar {
  static constexpr int PER_CTA = LB_THREADS / 32;
  double* red;  // not used: the reductions are shuffles
  __device__ __forceinline__ int tid() const { return threadIdx.x & 31; }
  __device__ __forceinline__ int nthr() const { return 32; }
  __device__ __forceinline__ void sync() const { __syncwarp(); }
  __device__ __forceinline__ double block_sum(double v) const {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
  }
  __device__ __forceinline__ double dot(const double* a, const double* b, int n) const {
    double acc = 0.0;
    for (int i = threadIdx.x & 31; i < n; i += 32) acc += a[i] * b[i];
    return block_sum(acc);
  }
  __device__ __forceinline__ double amax(const double* a, int n) const {
    double m = 0.0;
    for (int i = threadIdx.x & 31; i < n; i += 32) m = fmax(m, fabs(a[i]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    return m;
  }
};

// f, g of active entry a from the evaluation partials, added in chunk order, with the L2 term in float64 as
// SK/linear_model/_linear_loss.py:349-372 forms it (penalty on the weights only): loss = sum(loss_i) / n +
// 0.5 * l2 * ||W||^2, grad[k, :d] = G^T X / n + l2 * W, grad[k, d] = sum_i G / n for the K class rows of the
// problem (slot a * K + k).  fmask: the problem's feature mask or null.
template <class Par>
__device__ __forceinline__ double gather_fg(const Par& P, int a, int n_act, int K, int nz_used, int d, int ldx,
                                            int fit_intercept, const double* __restrict__ lossp,
                                            const double* __restrict__ gsump, const float* __restrict__ gradp,
                                            const double* __restrict__ gradr, const double* __restrict__ gscale,
                                            const uint8_t* __restrict__ fmask, double l2, double inv_n,
                                            const double* x, double* g) {
  const int dp = d + 1;
  const size_t n_slots = (size_t)n_act * K;
  double lsum = 0.0;
  for (int z = 0; z < nz_used; ++z) lsum += lossp[(size_t)z * n_act + a];
  double wsq = 0.0;
  for (int idx = P.tid(); idx < K * dp; idx += P.nthr()) {
    const int k = idx / dp, j = idx - k * dp;
    const size_t s = (size_t)a * K + k;
    double acc = 0.0;
    if (j == d) {
      for (int z = 0; z < nz_used; ++z) acc += gsump[(size_t)z * n_slots + s];
      g[idx] = fit_intercept ? acc * inv_n : 0.0;
      continue;
    }
    // the partials are added in chunk order (the result must not depend on anything else); eight
    // loads are put in flight at a time, the additions stay sequential
    int z = 0;
    if (gradr) { acc = gradr[s * ldx + j]; z = nz_used; }   // already reduced by lb_reduce_kernel
    for (; z + 8 <= nz_used; z += 8) {
      float v[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) v[q] = gradp[((size_t)(z + q) * n_slots + s) * ldx + j];
#pragma unroll
      for (int q = 0; q < 8; ++q) acc += (double)v[q];
    }
    for (; z < nz_used; ++z) acc += (double)gradp[((size_t)z * n_slots + s) * ldx + j];
    const double xk = x[idx];
    if (gscale) acc *= gscale[j];
    // acc * inv_n + l2 * xk with one product fused into the sum: the penalty's for binary columns, the data
    // term's for multinomial candidates (the roundings each kind's fits have always had)
    const double gk = K == 1 ? __fma_rn(l2, xk, __dmul_rn(acc, inv_n)) : __fma_rn(acc, inv_n, __dmul_rn(l2, xk));
    // a feature masked out of this problem (DistFeatureEliminator) keeps weight 0 in every class row: with a
    // zero gradient entry every L-BFGS direction is 0 there, i.e. the fit on the remaining columns of X
    g[idx] = (fmask && !fmask[j]) ? 0.0 : gk;
    wsq += xk * xk;
  }
  wsq = P.block_sum(wsq);
  return lsum * inv_n + 0.5 * l2 * wsq;
}

// Sum of the per-chunk gradient partials of every (slot, feature) in chunk order, float64, one
// thread per element: the whole device streams the partial array once (one column's optimiser warp
// alone cannot pull its 147 KB fast enough).  Same additions in the same order as gather_fg's loop.
// Binary columns only (one slot per entry).
__global__ void __launch_bounds__(256)
lb_reduce_kernel(const float* __restrict__ gradp, int nz, int n_act, int ldx, const int32_t* __restrict__ n_act_dev,
                 double* __restrict__ gradr) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t total = (int64_t)min(n_act, (int)*n_act_dev) * ldx;
  if (e >= total) return;
  const size_t stride = (size_t)n_act * ldx;
  double acc = 0.0;
  int z = 0;
  for (; z + 8 <= nz; z += 8) {
    float v[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) v[q] = gradp[(size_t)(z + q) * stride + e];
#pragma unroll
    for (int q = 0; q < 8; ++q) acc += (double)v[q];
  }
  for (; z < nz; ++z) acc += (double)gradp[(size_t)z * stride + e];
  gradr[e] = acc;
}

// Test / diagnostic entries: objective and gradient of every problem at caller-supplied points xin [B][n].  The
// partials are indexed by active entry, the problem's constants, point and outputs by slot[a].col.
__global__ void __launch_bounds__(LB_THREADS)
lb_gather_kernel(const SlotMeta* __restrict__ slot, int n_act, int K, int nz_used, int d, int ldx, int fit_intercept,
                 const double* __restrict__ lossp, const double* __restrict__ gsump,
                 const float* __restrict__ gradp, const double* __restrict__ gscale,
                 const uint8_t* __restrict__ fmask, const double* __restrict__ l2v,
                 const double* __restrict__ inv_nv, const double* __restrict__ xin,
                 double* __restrict__ fout, double* __restrict__ gout) {
  __shared__ double red[8];
  const int a = blockIdx.x;
  if (a >= n_act) return;
  const int col = slot[a].col;
  if (col < 0) return;   // padding slot of the fold-grouped layout
  const size_t n = (size_t)K * (d + 1);
  CtaPar P{red};
  const double f = gather_fg(P, a, n_act, K, nz_used, d, ldx, fit_intercept, lossp, gsump, gradp, nullptr, gscale,
                             fmask ? fmask + (size_t)col * d : nullptr, l2v[col], inv_nv[col], xin + col * n,
                             gout + col * n);
  if (threadIdx.x == 0) fout[col] = f;
}

__global__ void lb_init_kernel(LbfgsScalars* sc, double* vec, size_t stride, int B, int n, int m, int maxiter,
                               int maxls, double pgtol, double ftol, SlotMeta* slot, const int32_t* col_fold,
                               const int32_t* col_pos, const int32_t* col_neg1, int32_t* n_evals, int32_t* n_act) {
  const int col = blockIdx.x;
  if (col >= B) return;
  double* base = vec + (size_t)col * stride;
  for (size_t i = threadIdx.x; i < stride; i += blockDim.x) base[i] = 0.0;
  if (threadIdx.x == 0) {
    LbfgsScalars s;
    lbfgs_init(s, n, m, maxiter, maxls, pgtol, ftol);
    sc[col] = s;
    if (slot) {   // dense layout: entry i = problem i (the grouped layout is uploaded by the host)
      SlotMeta sm;
      sm.col = col; sm.fold = col_fold[col]; sm.pos = col_pos ? col_pos[col] : 0; sm.pad = col_neg1 ? col_neg1[col] : 0;
      slot[col] = sm;
      if (col == 0) *n_act = B;
    }
    n_evals[col] = 0;
  }
}

// f, g, then one step of the optimiser state machine.  WarpPar: one warp per entry, four per CTA (binary
// columns); CtaPar: one CTA per entry (multinomial candidates).  The policy fixes the order of the dot products.
template <class Par>
__global__ void __launch_bounds__(LB_THREADS)
lb_step_kernel(LbfgsScalars* sc, double* vec, size_t stride, const SlotMeta* slot, int n_act,
               const int32_t* __restrict__ n_act_dev, int K, int nz_used, int d, int ldx, int fit_intercept,
               const double* __restrict__ lossp, const double* __restrict__ gsump, const float* __restrict__ gradp,
               const double* __restrict__ gradr, const double* __restrict__ gscale,
               const uint8_t* __restrict__ fmask, const double* __restrict__ l2v, const double* __restrict__ inv_nv,
               int32_t* n_evals) {
  __shared__ double red[8];
  const int a = blockIdx.x * Par::PER_CTA + threadIdx.x / (LB_THREADS / Par::PER_CTA);
  // n_act (host) may be a stale upper bound when several rounds are enqueued per host round trip:
  // the partial sums are indexed with it, the live slot count is the device's
  if (a >= n_act || a >= *n_act_dev) return;
  const int col = slot[a].col;
  if (col < 0) return;   // padding slot of the fold-grouped layout
  LbfgsScalars st = sc[col];
  const int n = st.n, m = st.m;
  LbfgsVectors v = lbfgs_col_vectors(vec + (size_t)col * stride, n, m);
  Par P{red};
  const double f = gather_fg(P, a, n_act, K, nz_used, d, ldx, fit_intercept, lossp, gsump, gradp, gradr, gscale,
                             fmask ? fmask + (size_t)col * d : nullptr, l2v[col], inv_nv[col], v.x, v.g);
  P.sync();
  lbfgs_advance(P, st, v, f);
  P.sync();
  if (P.tid() == 0) {
    sc[col] = st;
    n_evals[col] += 1;
  }
}

// Exclusive prefix sum of keep over the CTA, in thread order; total receives the CTA's sum.  wsum: shared, 32
// ints; the caller synchronises before the next call writes it again.
__device__ __forceinline__ int block_scan(int keep, int* wsum, int& total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int x = keep;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) wsum[wid] = x;
  __syncthreads();
  if (wid == 0) {
    int w = (lane < (int)(blockDim.x >> 5)) ? wsum[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    wsum[lane] = w;  // inclusive
  }
  __syncthreads();
  total = wsum[(blockDim.x >> 5) - 1];
  return x - keep + (wid > 0 ? wsum[wid - 1] : 0);
}

// Stable in-place compaction of the active list (single CTA).
__global__ void lb_compact_kernel(const LbfgsScalars* sc, SlotMeta* slot, int n_act_in, int32_t* n_act_out,
                                  int32_t* n_run_out, int32_t* hist) {
  __shared__ int wsum[32];
  __shared__ int base_s;
  const int tid = threadIdx.x;
  if (tid == 0) base_s = 0;
  { const int live = *n_act_out; if (live < n_act_in) n_act_in = live; }   // host value may be a stale upper bound
  __syncthreads();
  for (int start = 0; start < n_act_in; start += blockDim.x) {
    int i = start + tid;
    SlotMeta sm;
    int keep = 0;
    if (i < n_act_in) {
      sm = slot[i];
      keep = sc[sm.col].status == LB_RUNNING ? 1 : 0;
    }
    int total;
    const int prefix = block_scan(keep, wsum, total);
    int base = base_s;
    __syncthreads();
    if (keep) slot[base + prefix] = sm;
    if (tid == 0) base_s = base + total;
    __syncthreads();
  }
  if (tid == 0) {
    *n_act_out = base_s;
    if (n_run_out) *n_run_out = base_s;
    if (hist) { hist[0] = base_s; hist[1] = base_s; }   // per-round record
  }
}

// Fold-grouped compaction (single CTA).  Input: slots grouped by fold in 128-aligned segments
// (padding entries col = -1).  Output, in place: the still-running columns of every fold, in
// their old order, each fold segment padded again to a multiple of 128.
__global__ void lb_compact_grouped_kernel(const LbfgsScalars* sc, SlotMeta* slot, int n_in,
                                          int32_t* n_slots_out, int32_t* n_run_out, int32_t* hist) {
  __shared__ int cnt[130];       // kept per fold key (key = fold + 1, fold in [-1, 127])
  __shared__ int base[130];      // output base per fold key
  __shared__ int before[130];    // kept in earlier fold keys
  __shared__ int wsum[32];
  __shared__ int run_s;
  const int tid = threadIdx.x;
  for (int i = tid; i < 130; i += blockDim.x) cnt[i] = 0;
  if (tid == 0) run_s = 0;
  { const int live = *n_slots_out; if (live < n_in) n_in = live; }         // host value may be a stale upper bound
  __syncthreads();
  for (int i = tid; i < n_in; i += blockDim.x) {
    const SlotMeta sm = slot[i];
    if (sm.col >= 0 && sc[sm.col].status == LB_RUNNING) atomicAdd(&cnt[sm.fold + 1], 1);
  }
  __syncthreads();
  if (tid == 0) {
    int b = 0, k = 0;
    for (int f = 0; f < 130; ++f) { base[f] = b; before[f] = k; b += (cnt[f] + 127) / 128 * 128; k += cnt[f]; }
    *n_slots_out = b;
    *n_run_out = k;
    if (hist) { hist[0] = b; hist[1] = k; }   // per-round record (read back once at the end)
  }
  __syncthreads();
  // ordered scatter: global rank of a kept entry minus the kept entries of earlier folds
  for (int start = 0; start < n_in; start += blockDim.x) {
    const int i = start + tid;
    SlotMeta sm;
    int keep = 0;
    if (i < n_in) { sm = slot[i]; keep = (sm.col >= 0 && sc[sm.col].status == LB_RUNNING) ? 1 : 0; }
    int total;
    const int rank = run_s + block_scan(keep, wsum, total);
    __syncthreads();
    if (keep) slot[base[sm.fold + 1] + rank - before[sm.fold + 1]] = sm;
    if (tid == 0) run_s += total;
    __syncthreads();
  }
  // padding
  for (int f = 0; f < 130; ++f) {
    const int lo = base[f] + cnt[f], hi = base[f] + (cnt[f] + 127) / 128 * 128;
    for (int i = lo + tid; i < hi; i += blockDim.x) {
      SlotMeta sm; sm.col = -1; sm.fold = f - 1; sm.pos = -1; sm.pad = 0;
      slot[i] = sm;
    }
  }
}

// Points of the active entries as fp32 slot rows (SK/_linear_loss.py:216-217 casts the same way): one CTA per
// slot a * K + k, row k of the point of problem slot[a].col in x (pitch x_stride).
__global__ void lb_export_kernel(const double* x, size_t x_stride, const SlotMeta* slot, const int32_t* n_act, int K,
                                 int d, int ldx, size_t bias_off, float* W) {
  const int a = blockIdx.x / K, k = blockIdx.x - a * K;
  if (a >= *n_act) return;
  const double* xr = x + (size_t)slot[a].col * x_stride + (size_t)k * (d + 1);
  const size_t s = (size_t)a * K + k;
  for (int j = threadIdx.x; j < ldx; j += blockDim.x) W[s * ldx + j] = j < d ? (float)xr[j] : 0.f;
  if (threadIdx.x == 0) W[bias_off + s] = (float)xr[d];
}

__global__ void lb_finish_kernel(const LbfgsScalars* sc, const double* vec, size_t stride, int B, int n,
                                 float* coef, int32_t* niter, int32_t* status, double* loss) {
  const int col = blockIdx.x;
  if (col >= B) return;
  const double* x = vec + (size_t)col * stride;
  for (int k = threadIdx.x; k < n; k += blockDim.x) coef[(size_t)col * n + k] = (float)x[k];
  if (threadIdx.x == 0) {
    const LbfgsScalars& s = sc[col];
    niter[col] = s.nit < s.maxiter ? s.nit : s.maxiter;
    status[col] = s.status;
    loss[col] = s.f;
  }
}

int lbfgs_alloc(Ctx* c, Scratch& sx, LbfgsBatch& b, int slot_cap, bool with_n_run) {
  b.stride = lbfgs_col_doubles(b.n, LBFGS_M);
  SKD_CUDA(c, sx.alloc(&b.sc, (size_t)b.B));
  SKD_CUDA(c, sx.alloc(&b.vec, (size_t)b.B * b.stride));
  SKD_CUDA(c, sx.alloc(&b.l2, (size_t)b.B));
  SKD_CUDA(c, sx.alloc(&b.inv_n, (size_t)b.B));
  SKD_CUDA(c, sx.alloc(&b.n_evals, (size_t)b.B));
  if (slot_cap > 0) {
    SKD_CUDA(c, sx.alloc(&b.slot, (size_t)slot_cap));
    SKD_CUDA(c, sx.alloc(&b.n_act, 1));
    if (with_n_run) SKD_CUDA(c, sx.alloc(&b.n_run, 1));
  }
  return 0;
}

// fp32 rows [B * K x ldx] then bias [B * K]
static size_t export_bias_offset(const Ctx* c, const LbfgsBatch& b) { return (size_t)b.B * b.K * c->ldx; }

int lbfgs_init(Ctx* c, LbfgsBatch& b, const int32_t* col_fold, const int32_t* col_pos, const int32_t* col_neg1,
               double tol, int max_iter, int maxls, double ftol) {
  lb_init_kernel<<<b.B, 128, 0, c->stream>>>(b.sc, b.vec, b.stride, b.B, b.n, LBFGS_M, max_iter, maxls, tol, ftol,
                                             col_fold ? b.slot : nullptr, col_fold, col_pos, col_neg1, b.n_evals,
                                             b.n_act);
  c->launches += 1;
  // initial iterate w0 = 0 (SK/linear_model/_logistic.py:443)
  if (b.W)
    SKD_CUDA(c, cudaMemsetAsync(b.W, 0, (export_bias_offset(c, b) + (size_t)b.B * b.K) * sizeof(float), c->stream));
  SKD_CUDA(c, cudaGetLastError());
  return 0;
}

int lbfgs_enqueue(Ctx* c, LbfgsBatch& b, int n_act_in, int nz_used, int fit_intercept, int32_t* hist,
                  LogregWork* tc) {
  const int d = (int)c->d;
  // many partials per slot (tensor-core path): reduce them with the whole device first
  const double* gradr = (b.gradr && nz_used > 8) ? b.gradr : nullptr;
  if (gradr) {
    const int64_t total = (int64_t)n_act_in * b.ldw;
    lb_reduce_kernel<<<(unsigned)((total + 255) / 256), 256, 0, c->stream>>>(b.gradp, nz_used, n_act_in, b.ldw, b.n_act,
                                                                          b.gradr);
    c->launches += 1;
  }
  if (b.K == 1)
    lb_step_kernel<WarpPar><<<(n_act_in + WarpPar::PER_CTA - 1) / WarpPar::PER_CTA, LB_THREADS, 0, c->stream>>>(
        b.sc, b.vec, b.stride, b.slot, n_act_in, b.n_act, b.K, nz_used, d, b.ldw, fit_intercept, b.lossp, b.gsump,
        b.gradp, gradr, b.gscale, b.fmask, b.l2, b.inv_n, b.n_evals);
  else
    lb_step_kernel<CtaPar><<<n_act_in, LB_THREADS, 0, c->stream>>>(
        b.sc, b.vec, b.stride, b.slot, n_act_in, b.n_act, b.K, nz_used, d, b.ldw, fit_intercept, b.lossp, b.gsump,
        b.gradp, gradr, b.gscale, b.fmask, b.l2, b.inv_n, b.n_evals);
  if (b.grouped) lb_compact_grouped_kernel<<<1, 1024, 0, c->stream>>>(b.sc, b.slot, n_act_in, b.n_act, b.n_run, hist);
  else lb_compact_kernel<<<1, 1024, 0, c->stream>>>(b.sc, b.slot, n_act_in, b.n_act, b.n_run, hist);
  c->launches += 2;
  if (tc) {
    if (tc_export(c, *tc, n_act_in, nullptr, fit_intercept)) return 1;
  } else {
    lb_export_kernel<<<n_act_in * b.K, 128, 0, c->stream>>>(b.vec, b.stride, b.slot, b.n_act, b.K, d, (int)c->ldx,
                                                           export_bias_offset(c, b), b.W);
    c->launches += 1;
  }
  SKD_CUDA(c, cudaGetLastError());
  return 0;
}

int lbfgs_run(Ctx* c, LbfgsBatch& b, int n_act, int fit_intercept, int max_iter, int32_t* hist, LogregWork* tc,
              const std::function<int(int n_act, long round, int* nz_used)>& eval, long* rounds_out) {
  const long max_rounds = lbfgs_max_rounds(max_iter);
  long rounds = 0;
  int n_run = b.B;
  // Several optimiser rounds are enqueued per host round trip: the kernels read the live slot count on the
  // device, the host's n_act is only an upper bound that sizes the grids and strides.
  while (n_run > 0) {
    for (int q = 0; q < LBFGS_ROUNDS_PER_SYNC; ++q) {
      int nz_used = b.nz;
      if (eval(n_act, rounds, &nz_used)) return 1;
      if (lbfgs_enqueue(c, b, n_act, nz_used, fit_intercept, hist ? hist + 2 * rounds : nullptr, tc)) return 1;
      if (++rounds > max_rounds) return fail(c, "device L-BFGS-B: round limit exceeded (internal error)");
    }
    int32_t na = 0, nr = 0;
    SKD_CUDA(c, cudaMemcpyAsync(&na, b.n_act, sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
    if (b.n_run) SKD_CUDA(c, cudaMemcpyAsync(&nr, b.n_run, sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
    SKD_CUDA(c, cudaStreamSynchronize(c->stream));
    c->d2h += (b.n_run ? 2 : 1) * sizeof(int32_t);
    n_act = na;
    n_run = b.n_run ? nr : na;
  }
  if (rounds_out) *rounds_out = rounds;
  return 0;
}

int lbfgs_export_points(Ctx* c, LbfgsBatch& b, int n_act_upper, const double* dx) {
  lb_export_kernel<<<n_act_upper * b.K, 128, 0, c->stream>>>(dx, (size_t)b.n, b.slot, b.n_act, b.K, (int)c->d,
                                                            (int)c->ldx, export_bias_offset(c, b), b.W);
  c->launches += 1;
  SKD_CUDA(c, cudaGetLastError());
  return 0;
}

int lbfgs_gather(Ctx* c, LbfgsBatch& b, int n_act, int nz_used, int fit_intercept, const double* dx, double* df,
                 double* dg) {
  lb_gather_kernel<<<n_act, LB_THREADS, 0, c->stream>>>(b.slot, n_act, b.K, nz_used, (int)c->d, b.ldw, fit_intercept,
                                                        b.lossp, b.gsump, b.gradp, b.gscale, b.fmask, b.l2, b.inv_n,
                                                        dx, df, dg);
  c->launches += 1;
  SKD_CUDA(c, cudaGetLastError());
  return 0;
}

int lbfgs_result(Ctx* c, Scratch& sx, LbfgsBatch& b, int64_t b0, float* coef_out, int32_t* n_iter_out,
                 int32_t* status_out, double* loss_out, int32_t* n_evals_out) {
  const int B = b.B;
  float* dcoef; int32_t *dniter, *dstatus; double* dloss;
  SKD_CUDA(c, sx.alloc(&dcoef, (size_t)B * b.n));
  SKD_CUDA(c, sx.alloc(&dniter, (size_t)B));
  SKD_CUDA(c, sx.alloc(&dstatus, (size_t)B));
  SKD_CUDA(c, sx.alloc(&dloss, (size_t)B));
  lb_finish_kernel<<<B, 128, 0, c->stream>>>(b.sc, b.vec, b.stride, B, b.n, dcoef, dniter, dstatus, dloss);
  c->launches += 1;
  SKD_CUDA(c, cudaGetLastError());
  SKD_CUDA(c, cudaMemcpyAsync(coef_out + b0 * b.n, dcoef, (size_t)B * b.n * sizeof(float), cudaMemcpyDeviceToHost,
                              c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(n_iter_out + b0, dniter, B * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(status_out + b0, dstatus, B * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
  if (loss_out)
    SKD_CUDA(c, cudaMemcpyAsync(loss_out + b0, dloss, B * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  if (n_evals_out)
    SKD_CUDA(c, cudaMemcpyAsync(n_evals_out + b0, b.n_evals, B * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
  c->d2h += (int64_t)B * (b.n * 4 + 20);
  return 0;
}

}  // namespace skd
