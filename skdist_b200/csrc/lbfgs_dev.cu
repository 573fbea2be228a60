// lbfgs_dev.cu -- device-resident batched L-BFGS-B driver: one CTA per active column.
//
// Replaces the host loop scipy/optimize/_lbfgsb_py.py:406-437 (setulb reverse communication)
// that each of the reference's tasks runs inside estimator.fit (ref search.py:230); the
// optimiser arithmetic is csrc/lbfgs_core.h.  Per round:
//   lb_step_kernel    : gather the slot's partial sums -> f, g (float64, adds the L2 term as
//                       SK/linear_model/_linear_loss.py:350,356-361), advance the state machine
//   lb_compact_kernel : rebuild the list of still-running columns (stable order)
//   lb_export_kernel  : cast the new trial points to fp32 (SK/_linear_loss.py:216-217) into the
//                       active-slot weight matrix for the next evaluation
#include "skd_internal.h"

namespace skd {

constexpr int LB_THREADS = 128;

struct CtaPar {
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

__device__ __forceinline__ LbfgsVectors col_vectors(double* base, int n, int m) {
  LbfgsVectors v;
  double* p = base;
  v.x = p; p += n;
  v.g = p; p += n;
  v.t = p; p += n;
  v.r = p; p += n;
  v.d = p; p += n;
  v.S = p; p += (size_t)m * n;
  v.Y = p; p += (size_t)m * n;
  v.rho = p; p += m;
  v.alpha = p;
  return v;
}


// f, g of slot s from the evaluation partials, with the L2 term added in float64 exactly as
// SK/linear_model/_linear_loss.py:349-361 does (penalty on the weights only).
template <class Par>
__device__ __forceinline__ double gather_fg(const Par& P, int s, int n_act, int nz_used, int d,
                                            int ldx, int fit_intercept,
                                            const double* __restrict__ lossp,
                                            const double* __restrict__ gsump,
                                            const float* __restrict__ gradp,
                                            const double* __restrict__ gscale, double l2,
                                            double inv_n, const double* x, double* g,
                                            const uint8_t* __restrict__ fmask = nullptr,
                                            const double* __restrict__ gradr = nullptr) {
  double lsum = 0.0, gsum = 0.0;
  for (int z = 0; z < nz_used; ++z) {
    lsum += lossp[(size_t)z * n_act + s];
    gsum += gsump[(size_t)z * n_act + s];
  }
  double wsq = 0.0;
  for (int k = P.tid(); k < d; k += P.nthr()) {
    double acc = 0.0;
    // the partials are added in chunk order (the result must not depend on anything else); eight
    // loads are put in flight at a time, the additions stay sequential
    int z = 0;
    if (gradr) { acc = gradr[(size_t)s * ldx + k]; z = nz_used; }   // already reduced by lb_reduce_kernel
    for (; z + 8 <= nz_used; z += 8) {
      float v[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) v[q] = gradp[((size_t)(z + q) * n_act + s) * ldx + k];
#pragma unroll
      for (int q = 0; q < 8; ++q) acc += (double)v[q];
    }
    for (; z < nz_used; ++z) acc += (double)gradp[((size_t)z * n_act + s) * ldx + k];
    double xk = x[k];
    if (gscale) acc *= gscale[k];
    // a feature masked out of this column (DistFeatureEliminator) keeps weight 0: with a zero
    // gradient entry every L-BFGS direction is 0 there, i.e. the fit on the remaining columns of X
    g[k] = (fmask && !fmask[k]) ? 0.0 : acc * inv_n + l2 * xk;
    wsq += xk * xk;
  }
  if (P.tid() == 0) g[d] = fit_intercept ? gsum * inv_n : 0.0;
  wsq = P.block_sum(wsq);
  return lsum * inv_n + 0.5 * l2 * wsq;
}

// Sum of the per-chunk gradient partials of every (slot, feature) in chunk order, float64, one
// thread per element: the whole device streams the partial array once (one column's optimiser CTA
// alone cannot pull its 147 KB fast enough).  Same additions in the same order as gather_fg's loop.
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

// Diagnostic / test entry: objective and gradient of every column at caller-supplied points.  The
// partials are indexed by slot, the column's constants, point and outputs by slot[s].col.
__global__ void __launch_bounds__(LB_THREADS)
lb_gather_kernel(int n_act, int nz_used, int d, int ldx, int fit_intercept, const SlotMeta* __restrict__ slot,
                 const double* __restrict__ lossp, const double* __restrict__ gsump,
                 const float* __restrict__ gradp, const double* __restrict__ gscale,
                 const double* __restrict__ l2v,
                 const double* __restrict__ inv_nv, const double* __restrict__ xin,
                 double* __restrict__ fout, double* __restrict__ gout) {
  __shared__ double red[8];
  const int s = blockIdx.x;
  if (s >= n_act) return;
  const int col = slot[s].col;
  if (col < 0) return;   // padding slot of the fold-grouped layout
  CtaPar P{red};
  double f = gather_fg(P, s, n_act, nz_used, d, ldx, fit_intercept, lossp, gsump, gradp, gscale,
                       l2v[col], inv_nv[col], xin + (size_t)col * (d + 1), gout + (size_t)col * (d + 1));
  if (threadIdx.x == 0) fout[col] = f;
}

__global__ void lb_init_kernel(LbfgsScalars* sc, double* vec, size_t vec_stride, int B, int n,
                               int m, int maxiter, int maxls, double pgtol, double ftol,
                               SlotMeta* slot, const int32_t* col_fold, const int32_t* col_pos,
                               const int32_t* col_neg1, int32_t* n_evals, int32_t* n_act) {
  int col = blockIdx.x;
  if (col >= B) return;
  double* base = vec + (size_t)col * vec_stride;
  for (size_t i = threadIdx.x; i < vec_stride; i += blockDim.x) base[i] = 0.0;
  if (threadIdx.x == 0) {
    LbfgsScalars s;
    lbfgs_init(s, n, m, maxiter, maxls, pgtol, ftol);
    sc[col] = s;
    if (slot) {   // dense layout: slot i = column i (the grouped layout is uploaded by the host)
      SlotMeta sm;
      sm.col = col; sm.fold = col_fold[col]; sm.pos = col_pos[col]; sm.pad = col_neg1 ? col_neg1[col] : 0;
      slot[col] = sm;
      if (col == 0) *n_act = B;
    }
    n_evals[col] = 0;
  }
}

// one warp per slot, four slots per CTA
__global__ void __launch_bounds__(LB_THREADS)
lb_step_kernel(LbfgsScalars* sc, double* vec, size_t vec_stride, const SlotMeta* slot, int n_act,
               int nz_used, int d, int ldx, int fit_intercept, const double* __restrict__ lossp,
               const double* __restrict__ gsump, const float* __restrict__ gradp,
               const double* __restrict__ gscale,
               const double* __restrict__ l2v, const double* __restrict__ inv_nv,
               int32_t* n_evals, const uint8_t* __restrict__ fmask, const int32_t* __restrict__ n_act_dev,
               const double* __restrict__ gradr) {
  const int s = blockIdx.x * (LB_THREADS / 32) + (threadIdx.x >> 5);
  // n_act (host) may be a stale upper bound when several rounds are enqueued per host round trip:
  // the partial sums are indexed with it, the live slot count is the device's
  if (s >= n_act || s >= *n_act_dev) return;
  const int col = slot[s].col;
  if (col < 0) return;   // padding slot of the fold-grouped layout
  LbfgsScalars st = sc[col];
  const int n = st.n, m = st.m;
  LbfgsVectors v = col_vectors(vec + (size_t)col * vec_stride, n, m);
  WarpPar P;
  const double l2 = l2v[col], inv_n = inv_nv[col];
  double f = gather_fg(P, s, n_act, nz_used, d, ldx, fit_intercept, lossp, gsump, gradp, gscale, l2,
                       inv_n, v.x, v.g, fmask ? fmask + (size_t)col * d : nullptr, gradr);
  __syncwarp();
  lbfgs_advance(P, st, v, f);
  __syncwarp();
  if (P.tid() == 0) {
    sc[col] = st;
    n_evals[col] += 1;
  }
}

// Stable in-place compaction of the active slot list (single CTA).
__global__ void lb_compact_kernel(const LbfgsScalars* sc, SlotMeta* slot, int n_act_in,
                                  int32_t* n_act_out, int32_t* n_act_host) {
  __shared__ int wsum[32];
  __shared__ int base_s;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
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
    // block exclusive scan of keep
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
    int prefix = x - keep + (wid > 0 ? wsum[wid - 1] : 0);
    int total = wsum[(blockDim.x >> 5) - 1];
    int base = base_s;
    __syncthreads();
    if (keep) slot[base + prefix] = sm;
    if (tid == 0) base_s = base + total;
    __syncthreads();
  }
  if (tid == 0) {
    *n_act_out = base_s;
    if (n_act_host) { n_act_host[0] = base_s; n_act_host[1] = base_s; }   // per-round record
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
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
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
    int x = keep;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) wsum[wid] = x;
    __syncthreads();
    if (wid == 0) {
      int w = (lane < (int)(blockDim.x >> 5)) ? wsum[lane] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
      wsum[lane] = w;
    }
    __syncthreads();
    const int rank = run_s + x - keep + (wid > 0 ? wsum[wid - 1] : 0);
    const int total = wsum[(blockDim.x >> 5) - 1];
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

__global__ void lb_export_kernel(const LbfgsScalars* sc, const double* vec, size_t vec_stride,
                                 const SlotMeta* slot, const int32_t* n_act, int d, int ldx,
                                 int Bcap, float* Wact) {
  const int s = blockIdx.x;
  if (s >= *n_act) return;
  const int col = slot[s].col;
  const double* x = vec + (size_t)col * vec_stride;
  for (int k = threadIdx.x; k < ldx; k += blockDim.x)
    Wact[(size_t)s * ldx + k] = k < d ? (float)x[k] : 0.f;
  if (threadIdx.x == 0) Wact[(size_t)Bcap * ldx + s] = (float)x[d];
}

__global__ void lb_finish_kernel(const LbfgsScalars* sc, const double* vec, size_t vec_stride,
                                 int B, int d, float* coef, int32_t* niter, int32_t* status,
                                 double* loss) {
  const int col = blockIdx.x;
  if (col >= B) return;
  const double* x = vec + (size_t)col * vec_stride;
  for (int k = threadIdx.x; k <= d; k += blockDim.x) coef[(size_t)col * (d + 1) + k] = (float)x[k];
  if (threadIdx.x == 0) {
    const LbfgsScalars& s = sc[col];
    niter[col] = s.nit < s.maxiter ? s.nit : s.maxiter;
    status[col] = s.status;
    loss[col] = s.f;
  }
}

int lbfgs_dev_init(Ctx* c, LogregWork& w, int fit_intercept, double tol, int max_iter, int maxls, double ftol) {
  const int m = 10;
  lb_init_kernel<<<w.B, 128, 0, c->stream>>>(w.sc, w.vec, w.vec_stride, w.B, w.dp, m, max_iter,
                                             maxls, tol, ftol, w.grouped ? nullptr : w.slot, w.col_fold,
                                             w.col_pos, w.col_neg1, w.n_evals, w.n_act);
  // initial iterate is w0 = 0 (SK/linear_model/_logistic.py:443): export zeros
  c->launches += 1;
  if (w.use_tc) {
    if (tc_export(c, w, w.grouped ? w.slot_cap : w.B, nullptr, fit_intercept)) return 1;
  } else {
    SKD_CUDA(c, cudaMemsetAsync(w.Wact, 0, ((size_t)w.B * c->ldx + w.B) * sizeof(float), c->stream));
  }
  SKD_CUDA(c, cudaGetLastError());
  return 0;
}

// One optimiser round on the stream, no host synchronisation: advance every live column, rebuild the
// slot list, export the new trial points.  n_act_in may be a stale upper bound of the live slot count
// (the kernels read the device-side count); hist (may be null) receives {slots, running} of the round.
int lbfgs_dev_enqueue(Ctx* c, LogregWork& w, int n_act_in, int nz_used, int fit_intercept, int32_t* hist) {
  const int d = (int)c->d, ldx = (int)c->ldx;
  if (w.gradr && nz_used > 8) {   // many partials per slot (tensor-core path): reduce them with the whole device first
    const int64_t total = (int64_t)n_act_in * w.ldw;
    lb_reduce_kernel<<<(unsigned)((total + 255) / 256), 256, 0, c->stream>>>(w.gradp, nz_used, n_act_in, w.ldw, w.n_act,
                                                                          w.gradr);
    c->launches += 1;
  }
  lb_step_kernel<<<(n_act_in + LB_THREADS / 32 - 1) / (LB_THREADS / 32), LB_THREADS, 0, c->stream>>>(
      w.sc, w.vec, w.vec_stride, w.slot, n_act_in, nz_used, d, w.ldw, fit_intercept, w.lossp,
      w.gsump, w.gradp, w.gscale, w.l2, w.inv_n, w.n_evals, w.fmask, w.n_act,
      (w.gradr && nz_used > 8) ? w.gradr : nullptr);
  if (w.grouped) lb_compact_grouped_kernel<<<1, 1024, 0, c->stream>>>(w.sc, w.slot, n_act_in, w.n_act, w.n_run, hist);
  else lb_compact_kernel<<<1, 1024, 0, c->stream>>>(w.sc, w.slot, n_act_in, w.n_act, hist);
  c->launches += 2;
  if (w.use_tc) {
    if (tc_export(c, w, n_act_in, nullptr, fit_intercept)) return 1;
  } else {
    lb_export_kernel<<<n_act_in, 128, 0, c->stream>>>(w.sc, w.vec, w.vec_stride, w.slot, w.n_act, d,
                                                      ldx, w.B, w.Wact);
    c->launches += 1;
  }
  SKD_CUDA(c, cudaGetLastError());
  return 0;
}

// Host round trip: current slot count and number of running columns.
int lbfgs_dev_readback(Ctx* c, LogregWork& w, int* n_act_out, int* n_run_out) {
  int32_t na = 0, nr = 0;
  SKD_CUDA(c, cudaMemcpyAsync(&na, w.n_act, sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
  if (w.grouped) SKD_CUDA(c, cudaMemcpyAsync(&nr, w.n_run, sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  c->d2h += 2 * sizeof(int32_t);
  *n_act_out = na;
  *n_run_out = w.grouped ? nr : na;
  return 0;
}

int lbfgs_dev_gather(Ctx* c, LogregWork& w, int n_act, int nz_used, int fit_intercept,
                     const double* dx, double* df, double* dg) {
  lb_gather_kernel<<<n_act, LB_THREADS, 0, c->stream>>>(n_act, nz_used, (int)c->d, w.ldw,
                                                        fit_intercept, w.slot, w.lossp, w.gsump, w.gradp,
                                                        w.gscale, w.l2, w.inv_n, dx, df, dg);
  c->launches += 1;
  SKD_CUDA(c, cudaGetLastError());
  return 0;
}

int lbfgs_dev_finish(Ctx* c, LogregWork& w, float* dcoef, int32_t* dniter, int32_t* dstatus,
                     double* dloss) {
  lb_finish_kernel<<<w.B, 128, 0, c->stream>>>(w.sc, w.vec, w.vec_stride, w.B, (int)c->d, dcoef,
                                               dniter, dstatus, dloss);
  c->launches += 1;
  SKD_CUDA(c, cudaGetLastError());
  return 0;
}

// ---- multinomial problems: one CTA per active candidate, K * dp variables ------------------
// f, g of active candidate a from the evaluation partials, added in chunk order (SK/linear_model/_linear_loss.py:349-372,
// multiclass branch: loss = sum(loss_i) / n + 0.5 * l2 * ||W||^2, grad[:, :d] = G^T X / n + l2 * W,
// grad[:, d] = sum_i G / n).  fmask: the candidate's feature mask or null.
template <class Par>
__device__ __forceinline__ double mn_gather_fg(const Par& P, int a, int n_act_in, int K, int d, int ldx, int nz,
                                               int fit_intercept, const double* __restrict__ lossp,
                                               const double* __restrict__ gsump, const float* __restrict__ gradp,
                                               double l2, double inv_n, const double* x, double* g,
                                               const uint8_t* __restrict__ fmask) {
  const int dp = d + 1, n = K * dp;
  const size_t n_slots = (size_t)n_act_in * K;
  double lsum = 0.0;
  for (int z = 0; z < nz; ++z) lsum += lossp[(size_t)z * n_act_in + a];
  double wsq = 0.0;
  for (int idx = P.tid(); idx < n; idx += P.nthr()) {
    const int k = idx / dp, j = idx - k * dp;
    const size_t slot = (size_t)a * K + k;
    double acc = 0.0;
    if (j < d) {
      for (int z = 0; z < nz; ++z) acc += (double)gradp[((size_t)z * n_slots + slot) * ldx + j];
      const double xk = x[idx];
      // a feature masked out of this candidate keeps weight 0 in every class row (zero gradient entry)
      g[idx] = (fmask && !fmask[j]) ? 0.0 : acc * inv_n + l2 * xk;
      wsq += xk * xk;
    } else {
      for (int z = 0; z < nz; ++z) acc += gsump[(size_t)z * n_slots + slot];
      g[idx] = fit_intercept ? acc * inv_n : 0.0;
    }
  }
  wsq = P.block_sum(wsq);
  return lsum * inv_n + 0.5 * l2 * wsq;
}

// f, g, then one step of the optimiser state machine.
__global__ void __launch_bounds__(LB_THREADS)
mn_step_kernel(LbfgsScalars* sc, double* vec, size_t vec_stride, const SlotMeta* cand, int n_act_in,
               const int32_t* __restrict__ n_act_dev, int K, int d, int ldx, int nz, int fit_intercept,
               const double* __restrict__ lossp, const double* __restrict__ gsump,
               const float* __restrict__ gradp, const double* __restrict__ l2v,
               const double* __restrict__ inv_nv, int32_t* n_evals, const uint8_t* __restrict__ fmask) {
  __shared__ double red[8];
  const int a = blockIdx.x;
  if (a >= n_act_in || a >= *n_act_dev) return;
  const int col = cand[a].col;
  LbfgsScalars st = sc[col];
  const int n = st.n, m = st.m;
  LbfgsVectors v = col_vectors(vec + (size_t)col * vec_stride, n, m);
  CtaPar P{red};
  const double f = mn_gather_fg(P, a, n_act_in, K, d, ldx, nz, fit_intercept, lossp, gsump, gradp, l2v[col],
                                inv_nv[col], v.x, v.g, fmask ? fmask + (size_t)col * d : nullptr);
  __syncthreads();
  lbfgs_advance(P, st, v, f);
  __syncthreads();
  if (threadIdx.x == 0) {
    sc[col] = st;
    n_evals[col] += 1;
  }
}

// Test entry: objective and gradient of every active candidate at caller points xin [B][K][dp]; the partials
// are indexed by active index, the constants, point and outputs by cand[a].col.
__global__ void __launch_bounds__(LB_THREADS)
mn_gather_kernel(const SlotMeta* cand, int n_act_in, int K, int d, int ldx, int nz, int fit_intercept,
                 const double* __restrict__ lossp, const double* __restrict__ gsump,
                 const float* __restrict__ gradp, const double* __restrict__ l2v,
                 const double* __restrict__ inv_nv, const uint8_t* __restrict__ fmask,
                 const double* __restrict__ xin, double* __restrict__ fout, double* __restrict__ gout) {
  __shared__ double red[8];
  const int a = blockIdx.x;
  if (a >= n_act_in) return;
  const int col = cand[a].col;
  const size_t n = (size_t)K * (d + 1);
  CtaPar P{red};
  const double f = mn_gather_fg(P, a, n_act_in, K, d, ldx, nz, fit_intercept, lossp, gsump, gradp, l2v[col],
                                inv_nv[col], xin + col * n, gout + col * n, fmask ? fmask + (size_t)col * d : nullptr);
  if (threadIdx.x == 0) fout[col] = f;
}

__global__ void mn_init_kernel(LbfgsScalars* sc, double* vec, size_t vec_stride, int B, int n, int m,
                               int maxiter, int maxls, double pgtol, double ftol, SlotMeta* cand,
                               const int32_t* col_fold, int32_t* n_evals, int32_t* n_act) {
  const int col = blockIdx.x;
  if (col >= B) return;
  double* base = vec + (size_t)col * vec_stride;
  for (size_t i = threadIdx.x; i < vec_stride; i += blockDim.x) base[i] = 0.0;
  if (threadIdx.x == 0) {
    LbfgsScalars s;
    lbfgs_init(s, n, m, maxiter, maxls, pgtol, ftol);
    sc[col] = s;
    SlotMeta sm;
    sm.col = col; sm.fold = col_fold[col]; sm.pos = 0; sm.pad = 0;
    cand[col] = sm;
    n_evals[col] = 0;
    if (col == 0) *n_act = B;
  }
}

// trial points of the active candidates as fp32 slot rows (SK/_linear_loss.py:216-217 casts the same way)
__global__ void mn_export_kernel(const double* vec, size_t vec_stride, const SlotMeta* cand,
                                 const int32_t* n_act, int K, int d, int ldx, size_t bias_off, float* W) {
  const int a = blockIdx.x / K, k = blockIdx.x - a * K;
  if (a >= *n_act) return;
  const double* x = vec + (size_t)cand[a].col * vec_stride + (size_t)k * (d + 1);
  const size_t slot = (size_t)a * K + k;
  for (int j = threadIdx.x; j < ldx; j += blockDim.x) W[slot * ldx + j] = j < d ? (float)x[j] : 0.f;
  if (threadIdx.x == 0) W[bias_off + slot] = (float)x[d];
}

__global__ void mn_finish_kernel(const LbfgsScalars* sc, const double* vec, size_t vec_stride, int B, int n,
                                 float* coef, int32_t* niter, int32_t* status, double* loss) {
  const int col = blockIdx.x;
  if (col >= B) return;
  const double* x = vec + (size_t)col * vec_stride;
  for (int k = threadIdx.x; k < n; k += blockDim.x) coef[(size_t)col * n + k] = (float)x[k];
  if (threadIdx.x == 0) {
    const LbfgsScalars& s = sc[col];
    niter[col] = s.nit < s.maxiter ? s.nit : s.maxiter;
    status[col] = s.status;
    loss[col] = s.f;
  }
}

int multi_lbfgs_init(Ctx* c, MultiWork& w, const int32_t* d_col_fold, double tol, int max_iter, int maxls,
                     double ftol) {
  const int m = 10;
  mn_init_kernel<<<w.B, 128, 0, c->stream>>>(w.sc, w.vec, w.vec_stride, w.B, w.K * w.dp, m, max_iter, maxls,
                                             tol, ftol, w.cand, d_col_fold, w.n_evals, w.n_act);
  c->launches += 1;
  // w0 = 0 (SK/linear_model/_logistic.py:443)
  SKD_CUDA(c, cudaMemsetAsync(w.W, 0, ((size_t)w.B * w.K * c->ldx + (size_t)w.B * w.K) * sizeof(float), c->stream));
  SKD_CUDA(c, cudaGetLastError());
  return 0;
}

int multi_lbfgs_enqueue(Ctx* c, MultiWork& w, int n_act_in, int fit_intercept, int32_t* hist) {
  const int d = (int)c->d, ldx = (int)c->ldx;
  mn_step_kernel<<<n_act_in, LB_THREADS, 0, c->stream>>>(w.sc, w.vec, w.vec_stride, w.cand, n_act_in, w.n_act,
                                                         w.K, d, ldx, w.nz, fit_intercept, w.lossp, w.gsump,
                                                         w.gradp, w.l2, w.inv_n, w.n_evals, w.fmask);
  lb_compact_kernel<<<1, 1024, 0, c->stream>>>(w.sc, w.cand, n_act_in, w.n_act, hist);
  mn_export_kernel<<<n_act_in * w.K, 128, 0, c->stream>>>(w.vec, w.vec_stride, w.cand, w.n_act, w.K, d, ldx,
                                                          (size_t)w.B * w.K * ldx, w.W);
  c->launches += 3;
  SKD_CUDA(c, cudaGetLastError());
  return 0;
}

// caller points dx [B][K][dp] (device, float64) to the fp32 slot rows, by the export of the optimiser's trial points
int multi_export_points(Ctx* c, MultiWork& w, const double* dx) {
  mn_export_kernel<<<w.B * w.K, 128, 0, c->stream>>>(dx, (size_t)w.K * w.dp, w.cand, w.n_act, w.K, (int)c->d,
                                                     (int)c->ldx, (size_t)w.B * w.K * c->ldx, w.W);
  c->launches += 1;
  SKD_CUDA(c, cudaGetLastError());
  return 0;
}

int multi_gather(Ctx* c, MultiWork& w, int fit_intercept, const double* dx, double* df, double* dg) {
  mn_gather_kernel<<<w.B, LB_THREADS, 0, c->stream>>>(w.cand, w.B, w.K, (int)c->d, (int)c->ldx, w.nz, fit_intercept,
                                                      w.lossp, w.gsump, w.gradp, w.l2, w.inv_n, w.fmask, dx, df, dg);
  c->launches += 1;
  SKD_CUDA(c, cudaGetLastError());
  return 0;
}

int multi_lbfgs_finish(Ctx* c, MultiWork& w, float* dcoef, int32_t* dniter, int32_t* dstatus, double* dloss) {
  mn_finish_kernel<<<w.B, 128, 0, c->stream>>>(w.sc, w.vec, w.vec_stride, w.B, w.K * w.dp, dcoef, dniter,
                                               dstatus, dloss);
  c->launches += 1;
  SKD_CUDA(c, cudaGetLastError());
  return 0;
}

}  // namespace skd
