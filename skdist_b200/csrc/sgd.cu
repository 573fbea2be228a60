// sgd.cu -- exact-order column-batched SGD: every one-vs-rest label column at once.
//
// Replaces K invocations of the reference's `_fit_binary` (ref multiclass.py:109-152) with
// estimator = SGDClassifier: SK/linear_model/_stochastic_gradient.py:387-515 (fit_binary) ->
// SK/linear_model/_sgd_fast.pyx.tp:274-640 (_plain_sgd32) with WeightVector32
// (SK/utils/_weight_vector.pyx.tp) and the Fisher-Yates / xorshift shuffle
// (SK/utils/_seq_dataset.pyx.tp:137-145, SK/utils/_random.pxd:20-34).
//
// SGD is sequential in the samples but independent across label columns.  Columns form order groups:
// every column of a group walks the group's rows in the group's shuffled order (one-vs-rest: one group
// of all rows; a search: one group per (fold, seed)), with its own alpha.  One WARP owns one column: its d float32
// weights live in registers (d/32 per lane) for the whole epoch and the warp walks the shuffled
// rows, reproducing the reference's arithmetic operation by operation (sgd_replay.h), so fits are
// bit-identical to scikit-learn.  No tensor cores: the work per sample is two length-d vector
// operations per column, bound by the FP64 pipe and L2 latency.  Large hinge problems run their
// epochs on the tensor cores instead (sgd_tc.cu); sgd_fit below drives both.
#include <math.h>
#include <stdio.h>

#include <algorithm>
#include <chrono>
#include <memory>
#include <stdlib.h>

#include "sgd_replay.h"

namespace skd {

enum { SGD_HINGE = 0 };

enum { SGD_LR_OPTIMAL = 0, SGD_LR_CONSTANT = 1, SGD_LR_INVSCALING = 2 };

// per-sample learning rate and weight-decay factor of one epoch of the tensor-core path (one alpha for every
// column): "optimal" and "constant" (invscaling is evaluated on the host, see sgd_fit)
__global__ void sgd_schedule_kernel(int64_t n, double t0, double alpha, double optimal_init,
                                    int lr_type, double eta0, double* __restrict__ eta,
                                    float* __restrict__ cfac) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double t = t0 + (double)i;
  const double e = lr_type == SGD_LR_OPTIMAL ? 1.0 / (alpha * (optimal_init + t - 1.0)) : eta0;
  eta[i] = e;
  cfac[i] = (float)fmax(0.0, __dsub_rn(1.0, __dmul_rn(e, alpha)));  // w.scale(max(0, 1 - eta*alpha)) arg as float
}

// "invscaling": eta0 / pow(t, power_t) with the C library's pow, the one scikit-learn's Cython loop calls.  CUDA's
// double pow is only accurate to 2 ulp, and a different eta moves the float64 intercept.  cfac: the tensor-core
// path's decay factors (the warp kernels form them per column)
static void sgd_invscaling_schedule(int64_t n, double t0, double alpha, double eta0, double power_t, double* eta,
                                    float* cfac) {
  for (int64_t i = 0; i < n; ++i) {
    const double e = eta0 / pow(t0 + (double)i, power_t);
    eta[i] = e;
    if (cfac) cfac[i] = (float)fmax(0.0, 1.0 - e * alpha);
  }
}

// learning rate of sample i of an epoch that starts at t = t0 (1 + epochs done * n_g), for a column with
// `alpha` and `oi` = optimal_init: "optimal" 1.0 / (alpha * (optimal_init + t - 1.0)) in the C expression's
// order and rounding (no contraction), "constant" eta0, "invscaling" the host's table of the column's group
__device__ __forceinline__ double sgd_rate(const SgdFit& f, const double* etab, int64_t i, double t0, double alpha,
                                           double oi) {
  if (f.lr_type == SGD_LR_OPTIMAL)
    return __ddiv_rn(1.0, __dmul_rn(alpha, __dsub_rn(__dadd_rn(oi, __dadd_rn(t0, (double)i)), 1.0)));
  if (f.lr_type == SGD_LR_CONSTANT) return f.eta0;
  return __ldg(etab + i);
}

// w.scale(max(0, 1 - eta * alpha)): the argument as float
__device__ __forceinline__ float sgd_decay(double e, double alpha) {
  return (float)fmax(0.0, __dsub_rn(1.0, __dmul_rn(e, alpha)));
}

// log_loss, one sample at a time
template <int DPL>
__global__ void __launch_bounds__(128)
sgd_epoch_kernel(const float* __restrict__ X, int ldx, int d, const int32_t* __restrict__ ycls, const SgdFit f,
                 int n_active) {
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int a = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (a >= n_active) return;
  const int col = f.active[a];
  const int pos = f.col_pos[col];
  const int g = f.col_group[col];
  const int64_t g0 = f.goff[g], n = f.goff[g + 1] - g0;        // the group's rows
  const int32_t* __restrict__ order = f.order + g0;
  const double* etab = f.eta ? f.eta + g0 : nullptr;
  const double alpha = f.col_alpha[col], oi = f.col_oi[col];
  float* __restrict__ W = f.W;
  const int ldw = f.ldw;
  SgdState st = f.state[col];
  const double t0 = st.t;
  float w[DPL];
#pragma unroll
  for (int j = 0; j < DPL; ++j) {
    const int k = lane + 32 * j;
    w[j] = k < d ? W[(size_t)col * ldw + k] : 0.f;
  }
  double wscale = st.wscale, sq_norm = st.sq_norm, intercept = st.intercept;
  double objective_sum = 0.0;

  // software pipeline: everything sample i+1 needs (row index, features, label) is requested while
  // sample i is processed, so the per-sample dependency chain never waits on L2.  The step sizes of 32
  // samples are formed at once, lane l the one of sample i + l, and broadcast one per sample.
  float xn[DPL];
  int row = __ldg(order);
  int r_nxt = n > 1 ? __ldg(order + 1) : 0;
#pragma unroll
  for (int j = 0; j < DPL; ++j) {
    const int k = lane + 32 * j;
    xn[j] = k < ldx ? __ldg(X + (size_t)row * ldx + k) : 0.f;
  }
  int yc_n = ycls[row];
  double e_lane = 0.0;
  for (int64_t i = 0; i < n; ++i) {
    if ((i & 31) == 0) e_lane = i + lane < n ? sgd_rate(f, etab, i + lane, t0, alpha, oi) : 0.0;
    float x[DPL];
#pragma unroll
    for (int j = 0; j < DPL; ++j) x[j] = xn[j];
    const double y01 = (yc_n == pos) ? 1.0 : 0.0;
    const double e = __shfl_sync(FULL, e_lane, (int)(i & 31));
    const float c = sgd_decay(e, alpha);
    if (i + 1 < n) {
      row = r_nxt;
      r_nxt = i + 2 < n ? __ldg(order + i + 2) : 0;
#pragma unroll
      for (int j = 0; j < DPL; ++j) {
        const int k = lane + 32 * j;
        xn[j] = k < ldx ? __ldg(X + (size_t)row * ldx + k) : 0.f;
      }
      yc_n = ycls[row];
    }
    // p = w.dot(x) + intercept          (WeightVector32.dot)
    double acc = 0.0;
#pragma unroll
    for (int j = 0; j < DPL; ++j) acc += (double)__fmul_rn(w[j], x[j]);
    acc = warp_sum(acc);
    const double p = (double)(float)(acc * wscale) + intercept;
    // CyHalfBinomialLoss on y in {0,1} (SK/_loss/_loss.pyx.tp:256-266,686-725)
    double l1p, dloss;
    if (p <= -37.0) l1p = exp(p);
    else if (p <= -2.0) l1p = log1p(exp(p));
    else if (p <= 18.0) l1p = log(__dadd_rn(1.0, exp(p)));
    else if (p <= 33.3) l1p = __dadd_rn(p, exp(-p));
    else l1p = p;
    const double cur_loss = __dsub_rn(l1p, __dmul_rn(y01, p));
    if (p > -37.0) {
      const double et = exp(-p);
      dloss = __ddiv_rn(__dsub_rn(1.0 - y01, __dmul_rn(y01, et)), __dadd_rn(1.0, et));
    } else {
      dloss = __dsub_rn(exp(p), y01);
    }
    const float normf = (float)sqrt(sq_norm);
    objective_sum = __dadd_rn(objective_sum,
                              __dadd_rn(cur_loss, __dmul_rn(alpha, __dmul_rn(0.5, (double)__fmul_rn(normf, normf)))));
    if (dloss < -1e12) dloss = -1e12; else if (dloss > 1e12) dloss = 1e12;
    const double update = -e * dloss;
    // w.scale(c)
    wscale *= (double)c;
    sq_norm *= (double)__fmul_rn(c, c);
    if (wscale < 1e-6) {
      sgd_reset_wscale<DPL>(w, wscale);
      wscale = 1.0;
    }
    if (update != 0.0) {
      double q;
      sq_norm = sgd_add<DPL>(w, x, update, wscale, f.fit_intercept, intercept, q);
    }
  }
#pragma unroll
  for (int j = 0; j < DPL; ++j) {
    const int k = lane + 32 * j;
    if (k < d) W[(size_t)col * ldw + k] = w[j];
  }
  st.wscale = wscale; st.sq_norm = sq_norm; st.intercept = intercept;
  sgd_end_epoch<DPL>(st, w, intercept, objective_sum, n, f.tol, f.n_iter_no_change);
  if (lane == 0) f.state[col] = st;
}

// Hinge loss, speculative blocks.  With hinge loss a sample whose margin y*p exceeds 1 changes
// nothing but the lazy scale (wscale, sq_norm) and the objective sum -- scalars.  The warp therefore
// computes the dot products of the next T = 16 samples against the CURRENT weights at once
// (independent FMAs, all loads in flight together), reduces them with a butterfly, and then walks
// the 16 samples in order doing only the scalar recurrence; the first margin violator (or a
// reset_wscale) applies its weight update exactly as _plain_sgd32 does and the block restarts
// behind it.  Every value is computed by the same operations in the same order as one sample at a
// time, so the result stays bit-identical to scikit-learn; only the waiting changes.
template <int DPL>
__global__ void __launch_bounds__(128)
sgd_epoch_spec_kernel(const float* __restrict__ X, int ldx, int d, const int32_t* __restrict__ ycls, const SgdFit f,
                      int n_active) {
  constexpr int T = 16;                                                        // samples per block
  constexpr int S = (32 / DPL) < 1 ? 1 : ((32 / DPL) > 8 ? 8 : (32 / DPL));   // samples per load batch (2 S DPL floats in flight)
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int a = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (a >= n_active) return;
  const int col = f.active[a];
  const int pos = f.col_pos[col];
  const int g = f.col_group[col];
  const int64_t g0 = f.goff[g], n = f.goff[g + 1] - g0;        // the group's rows
  const int32_t* __restrict__ order = f.order + g0;
  const double* etab = f.eta ? f.eta + g0 : nullptr;
  const double alpha = f.col_alpha[col], oi = f.col_oi[col];
  float* __restrict__ W = f.W;
  const int ldw = f.ldw;
  SgdState st = f.state[col];
  const double t0 = st.t;
  float w[DPL];
#pragma unroll
  for (int j = 0; j < DPL; ++j) {
    const int k = lane + 32 * j;
    w[j] = k < d ? W[(size_t)col * ldw + k] : 0.f;
  }
  double wscale = st.wscale, sq_norm = st.sq_norm, intercept = st.intercept;
  double objective_sum = 0.0;

  int64_t i0 = 0;
  while (i0 < n) {
    const int Te = (int)((n - i0) < T ? (n - i0) : T);
    // lane t < Te owns the metadata of sample i0 + t
    int row_l = 0;
    double y_l = 0.0, e_l = 0.0;
    float c_l = 0.f;
    if (lane < Te) {
      row_l = __ldg(order + i0 + lane);
      e_l = sgd_rate(f, etab, i0 + lane, t0, alpha, oi);
      c_l = sgd_decay(e_l, alpha);
      y_l = (ycls[row_l] == pos) ? 1.0 : -1.0;
    }
    // dot products of all block samples with the current weights
    double part[T];
#pragma unroll
    for (int t = 0; t < T; ++t) part[t] = 0.0;
    float xb[2][S][DPL];
#pragma unroll
    for (int s2 = 0; s2 < S; ++s2) {
      const int r = __shfl_sync(FULL, row_l, s2);
#pragma unroll
      for (int j = 0; j < DPL; ++j) {
        const int k = lane + 32 * j;
        xb[0][s2][j] = k < ldx ? __ldg(X + (size_t)r * ldx + k) : 0.f;
      }
    }
#pragma unroll
    for (int b = 0; b < T / S; ++b) {
      if (b + 1 < T / S) {
#pragma unroll
        for (int s2 = 0; s2 < S; ++s2) {
          const int r = __shfl_sync(FULL, row_l, (b + 1) * S + s2);
#pragma unroll
          for (int j = 0; j < DPL; ++j) {
            const int k = lane + 32 * j;
            xb[(b + 1) & 1][s2][j] = k < ldx ? __ldg(X + (size_t)r * ldx + k) : 0.f;
          }
        }
      }
#pragma unroll
      for (int s2 = 0; s2 < S; ++s2)
#pragma unroll
        for (int j = 0; j < DPL; ++j) part[b * S + s2] += (double)__fmul_rn(w[j], xb[b & 1][s2][j]);
    }
    // butterfly reduce-scatter: afterwards lane L holds the full sum of sample L >> 1
#pragma unroll
    for (int half = T / 2, m = 16; half >= 1; half >>= 1, m >>= 1) {
      const bool up = (lane & m) != 0;
#pragma unroll
      for (int q = 0; q < half; ++q) {
        const double send = up ? part[q] : part[q + half];
        const double keep = up ? part[q + half] : part[q];
        part[q] = keep + __shfl_xor_sync(FULL, send, m);
      }
    }
    const double mysum = part[0] + __shfl_xor_sync(FULL, part[0], 1);

    // ---- ordered walk over the block, restructured so that only what is inherently serial is serial:
    //  A. the lazy-scale recurrences wscale *= c_t, sq_norm *= c_t^2 (two chains of 16 dependent
    //     multiplies, evaluated redundantly by every lane; lane t keeps the values BEFORE sample t);
    //  B. lane t evaluates sample t: prediction, margin, loss and objective term;
    //  C. the first event (margin violator or reset_wscale) is found with one ballot;
    //  D. the objective terms of samples 0..event are added in order;
    //  E. the event's weight update is applied exactly as one sample at a time.
    float c_all[T];
#pragma unroll
    for (int q = 0; q < T; ++q) c_all[q] = __shfl_sync(FULL, c_l, q);
    double my_ws = wscale, my_sq = sq_norm;        // state before this lane's sample
    double my_ws_after = wscale, my_sq_after = sq_norm;
    {
      double ws = wscale, sq = sq_norm;
#pragma unroll
      for (int q = 0; q < T; ++q) {
        if (lane == q) { my_ws = ws; my_sq = sq; }
        ws *= (double)c_all[q];
        sq *= (double)__fmul_rn(c_all[q], c_all[q]);
        if (lane == q) { my_ws_after = ws; my_sq_after = sq; }
      }
    }
    const double acc_l = __shfl_sync(FULL, mysum, (2 * lane) & 31);   // lane t < 16: dot of sample t
    const double p_l = (double)(float)(acc_l * my_ws) + intercept;
    const double z_l = p_l * y_l;
    const bool viol_l = lane < Te && z_l <= 1.0;
    const bool reset_l = lane < Te && my_ws_after < 1e-6;
    const double loss_l = viol_l ? 1.0 - z_l : 0.0;
    const float normf_l = (float)sqrt(my_sq);
    const double term_l = __dadd_rn(loss_l, __dmul_rn(alpha, __dmul_rn(0.5, (double)__fmul_rn(normf_l, normf_l))));
    const unsigned evmask = __ballot_sync(FULL, viol_l || reset_l);
    const int ev = evmask ? __ffs(evmask) - 1 : -1;        // first event sample, -1: none in this block
    const int last = ev >= 0 ? ev : Te - 1;                // samples 0..last are consumed
    {
      double terms[T];
#pragma unroll
      for (int q = 0; q < T; ++q) terms[q] = __shfl_sync(FULL, term_l, q);
#pragma unroll
      for (int q = 0; q < T; ++q)
        if (q <= last) objective_sum = __dadd_rn(objective_sum, terms[q]);
    }
    wscale = __shfl_sync(FULL, my_ws_after, last);
    sq_norm = __shfl_sync(FULL, my_sq_after, last);
    if (ev >= 0) {
      const bool is_reset = (evmask >> ev) & 1u ? __shfl_sync(FULL, (int)reset_l, ev) != 0 : false;
      const bool is_viol = __shfl_sync(FULL, (int)viol_l, ev) != 0;
      if (is_reset) {
        sgd_reset_wscale<DPL>(w, wscale);
        wscale = 1.0;
      }
      if (is_viol) {
        const double y = __shfl_sync(FULL, y_l, ev);
        const double e = __shfl_sync(FULL, e_l, ev);
        const double update = -e * (-y);
        if (update != 0.0) {
          const int r = __shfl_sync(FULL, row_l, ev);
          float x[DPL];
#pragma unroll
          for (int j2 = 0; j2 < DPL; ++j2) {
            const int k = lane + 32 * j2;
            x[j2] = k < ldx ? __ldg(X + (size_t)r * ldx + k) : 0.f;
          }
          double q;
          sq_norm = sgd_add<DPL>(w, x, update, wscale, f.fit_intercept, intercept, q);
        }
      }
    }
    const int t = last + 1;
    i0 += t;
  }
#pragma unroll
  for (int j = 0; j < DPL; ++j) {
    const int k = lane + 32 * j;
    if (k < d) W[(size_t)col * ldw + k] = w[j];
  }
  st.wscale = wscale; st.sq_norm = sq_norm; st.intercept = intercept;
  sgd_end_epoch<DPL>(st, w, intercept, objective_sum, n, f.tol, f.n_iter_no_change);
  if (lane == 0) f.state[col] = st;
}

// w.reset_wscale() at the end of _plain_sgd, then export
__global__ void sgd_finish_kernel(const float* __restrict__ W, int ldw, int d, const SgdState* __restrict__ state,
                                  int B, float* __restrict__ coef, double* __restrict__ intercept,
                                  int32_t* __restrict__ n_iter, double* __restrict__ t_out,
                                  int32_t* __restrict__ status) {
  const int col = blockIdx.x;
  if (col >= B) return;
  const float wf = (float)state[col].wscale;
  for (int k = threadIdx.x; k < d; k += blockDim.x) coef[(size_t)col * d + k] = __fmul_rn(W[(size_t)col * ldw + k], wf);
  if (threadIdx.x == 0) {
    intercept[col] = state[col].intercept;
    n_iter[col] = state[col].n_iter;
    t_out[col] = state[col].t;
    status[col] = state[col].status;
  }
}

static inline uint32_t xorshift_rand_r(uint32_t* seed) {   // SK/utils/_random.pxd:20-34
  if (*seed == 0) *seed = 1;
  *seed ^= (uint32_t)(*seed << 13);
  *seed ^= (uint32_t)(*seed >> 17);
  *seed ^= (uint32_t)(*seed << 5);
  return *seed % ((uint32_t)2147483647 + 1);
}

// Fisher-Yates with the SAME seed every epoch, applied to the evolving order (SK/utils/_seq_dataset.pyx.tp:137-145)
static void sgd_shuffle(int32_t* order, int64_t n, uint32_t seed) {
  for (int64_t i = 0; i < n - 1; ++i) {
    int64_t j = i + xorshift_rand_r(&seed) % (uint32_t)(n - i);
    std::swap(order[i], order[j]);
  }
}

// one epoch on the warp-per-column kernels: speculative blocks for hinge, one sample at a time for log_loss
static cudaError_t launch_epoch(Ctx* c, const SgdFit& f, int loss, int n_active) {
  const int grid = (n_active + 3) / 4;
#define SGD_CASE(D)                                                                                              \
  case D:                                                                                                        \
    if (loss == SGD_HINGE)                                                                                       \
      sgd_epoch_spec_kernel<D><<<grid, 128, 0, c->stream>>>(c->X, (int)c->ldx, (int)c->d, c->ycls, f, n_active); \
    else                                                                                                         \
      sgd_epoch_kernel<D><<<grid, 128, 0, c->stream>>>(c->X, (int)c->ldx, (int)c->d, c->ycls, f, n_active);      \
    break;
  switch (f.dpl) {
    SGD_CASE(1) SGD_CASE(2) SGD_CASE(4) SGD_CASE(8) SGD_CASE(16) SGD_CASE(32)
    default: return cudaErrorInvalidValue;
  }
#undef SGD_CASE
  return cudaGetLastError();
}

// The one SGD driver.  B columns in G order groups: column j fits the rows of group col_group[j] with
// col_alpha[j] / col_oi[j]; group g walks grows[goff[g] .. goff[g+1]) and shuffles that list with gseed[g]
// every epoch.  allow_tc: the caller is the one-group, one-alpha fit over all n rows in row order, which
// may run on the tensor cores.
static int sgd_fit(Ctx* c, int B, const int32_t* col_pos, const int32_t* col_group, const double* col_alpha,
                   const double* col_oi, int G, const int64_t* goff, const int32_t* grows, const uint32_t* gseed,
                   bool allow_tc, int loss, int fit_intercept, int max_iter, double tol, int shuffle, int lr_type,
                   double eta0, double power_t, int n_iter_no_change, float* coef_out, double* intercept_out,
                   int32_t* n_iter_out, double* t_out, int32_t* status_out) {
  const int64_t N = goff[G];     // rows of all groups
  const int d = (int)c->d;
  if (d > 1024) return fail(c, "sgd: device path supports d <= 1024");
  SgdFit f;
  f.B = B;
  f.dpl = 1;
  while (f.dpl * 32 < d) f.dpl *= 2;
  f.ldw = f.dpl * 32;
  f.alpha = col_alpha[0]; f.tol = tol; f.eta0 = eta0;
  f.fit_intercept = fit_intercept; f.n_iter_no_change = n_iter_no_change; f.lr_type = lr_type;
  Scratch sx(c);
  std::unique_ptr<SgdTc> tc;
  if (allow_tc && sgd_tc_supported(c, loss, shuffle)) tc.reset(new SgdTc(c));   // hinge: blocked-exact, same results
  // per-sample tables: the tensor-core path reads eta and cfac; the warp kernels only invscaling's eta
  const bool tables = tc || lr_type == SGD_LR_INVSCALING;
  float* W; SgdState* state; int32_t *order, *active, *dpos, *dgrp; double *eta = nullptr, *dalpha, *doi;
  int64_t* dgoff; float* cfac = nullptr;
  float* dcoef; double *dint, *dt; int32_t *dniter, *dstatus;
  SKD_CUDA(c, sx.alloc(&W, (size_t)B * f.ldw));
  SKD_CUDA(c, sx.alloc(&state, (size_t)B));
  SKD_CUDA(c, sx.alloc(&order, (size_t)N));
  SKD_CUDA(c, sx.alloc(&active, (size_t)B));
  SKD_CUDA(c, sx.alloc(&dpos, (size_t)B));
  SKD_CUDA(c, sx.alloc(&dgrp, (size_t)B));
  SKD_CUDA(c, sx.alloc(&dalpha, (size_t)B));
  SKD_CUDA(c, sx.alloc(&doi, (size_t)B));
  SKD_CUDA(c, sx.alloc(&dgoff, (size_t)G + 1));
  if (tables) SKD_CUDA(c, sx.alloc(&eta, (size_t)N));
  if (tc) SKD_CUDA(c, sx.alloc(&cfac, (size_t)N));
  SKD_CUDA(c, sx.alloc(&dcoef, (size_t)B * d));
  SKD_CUDA(c, sx.alloc(&dint, (size_t)B));
  SKD_CUDA(c, sx.alloc(&dt, (size_t)B));
  SKD_CUDA(c, sx.alloc(&dniter, (size_t)B));
  SKD_CUDA(c, sx.alloc(&dstatus, (size_t)B));
  f.W = W; f.state = state; f.col_pos = dpos; f.col_group = dgrp; f.col_alpha = dalpha; f.col_oi = doi;
  f.goff = dgoff; f.order = order; f.active = active; f.eta = eta; f.cfac = cfac;
  SKD_CUDA(c, cudaMemsetAsync(W, 0, (size_t)B * f.ldw * sizeof(float), c->stream));
  std::vector<SgdState> hs(B);
  for (auto& s : hs) { s.wscale = 1.0; s.sq_norm = 0.0; s.intercept = 0.0; s.best_objective = INFINITY; s.t = 1.0;
                       s.no_improve = 0; s.done = 0; s.n_iter = 0; s.status = 3; s.objective_sum = 0.0; }
  SKD_CUDA(c, cudaMemcpyAsync(state, hs.data(), (size_t)B * sizeof(SgdState), cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(dpos, col_pos, (size_t)B * 4, cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(dgrp, col_group, (size_t)B * 4, cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(dalpha, col_alpha, (size_t)B * 8, cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(doi, col_oi, (size_t)B * 8, cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(dgoff, goff, (size_t)(G + 1) * 8, cudaMemcpyHostToDevice, c->stream));
  c->h2d += (int64_t)B * 24 + (int64_t)(G + 1) * 8;
  if (tc && tc->init(c, f)) return 1;
  std::vector<int32_t> hact(B), hord(grows, grows + N);
  std::vector<double> heta(tables ? N : 0);
  std::vector<float> hcfac(tc && lr_type == SGD_LR_INVSCALING ? N : 0);
  std::vector<char> grun(G);     // groups with a running column
  for (int j = 0; j < B; ++j) hact[j] = j;
  int n_active = B;
  const char* trace_env = getenv("SKDIST_B200_TRACE");
  const bool trace = trace_env && trace_env[0] == '2';
  for (int epoch = 0; epoch < max_iter && n_active > 0; ++epoch) {
    auto tw0 = std::chrono::steady_clock::now();
    std::fill(grun.begin(), grun.end(), 0);
    for (int a = 0; a < n_active; ++a) grun[col_group[hact[a]]] = 1;
    if (shuffle)
      for (int g = 0; g < G; ++g)
        if (grun[g]) sgd_shuffle(hord.data() + goff[g], goff[g + 1] - goff[g], gseed[g]);
    const bool new_order = shuffle || epoch == 0;
    if (new_order) {
      SKD_CUDA(c, cudaMemcpyAsync(order, hord.data(), (size_t)N * 4, cudaMemcpyHostToDevice, c->stream));
      c->h2d += N * 4;
    }
    SKD_CUDA(c, cudaMemcpyAsync(active, hact.data(), (size_t)n_active * 4, cudaMemcpyHostToDevice, c->stream));
    auto tw1 = std::chrono::steady_clock::now();
    if (lr_type == SGD_LR_INVSCALING) {     // the host's pow, group by group (t0 = 1 + epoch * n_g)
      for (int g = 0; g < G; ++g)
        if (grun[g]) {
          const int64_t ng = goff[g + 1] - goff[g];
          sgd_invscaling_schedule(ng, 1.0 + (double)epoch * (double)ng, f.alpha, eta0, power_t, heta.data() + goff[g],
                                  tc ? hcfac.data() + goff[g] : nullptr);
        }
      SKD_CUDA(c, cudaMemcpyAsync(eta, heta.data(), (size_t)N * 8, cudaMemcpyHostToDevice, c->stream));
      c->h2d += N * 8;
      if (tc) {
        SKD_CUDA(c, cudaMemcpyAsync(cfac, hcfac.data(), (size_t)N * 4, cudaMemcpyHostToDevice, c->stream));
        c->h2d += N * 4;
      }
    } else if (tc) {
      sgd_schedule_kernel<<<(unsigned)((N + 255) / 256), 256, 0, c->stream>>>(N, 1.0 + (double)epoch * (double)N, f.alpha,
                                                                             col_oi[0], lr_type, eta0, eta, cfac);
      c->launches += 1;
    }
    if (tc) {
      if (tc->epoch(c, f, epoch, n_active, new_order, trace)) return 1;
    } else {
      cudaError_t e = launch_epoch(c, f, loss, n_active);
      c->launches += 1;
      if (e != cudaSuccess) return fail(c, std::string("sgd epoch launch: ") + cudaGetErrorString(e));
    }
    SKD_CUDA(c, cudaMemcpyAsync(hs.data(), state, (size_t)B * sizeof(SgdState), cudaMemcpyDeviceToHost, c->stream));
    SKD_CUDA(c, cudaStreamSynchronize(c->stream));
    c->d2h += (int64_t)B * sizeof(SgdState);
    if (trace) {
      auto tw2 = std::chrono::steady_clock::now();
      fprintf(stderr, "[skd trace] %s epoch %3d active %5d host shuffle %7.2f ms device %8.2f ms\n", tc ? "sgd-tc" : "sgd",
              epoch, n_active, std::chrono::duration<double, std::milli>(tw1 - tw0).count(),
              std::chrono::duration<double, std::milli>(tw2 - tw1).count());
    }
    n_active = 0;
    for (int j = 0; j < B; ++j)     // compacted across groups: columns of different groups stop at different epochs
      if (!hs[j].done) hact[n_active++] = j;
  }
  if (tc && trace) tc->print_counters();
  sgd_finish_kernel<<<B, 128, 0, c->stream>>>(W, f.ldw, d, state, B, dcoef, dint, dniter, dt, dstatus);
  c->launches += 1;
  SKD_CUDA(c, cudaGetLastError());
  SKD_CUDA(c, cudaMemcpyAsync(coef_out, dcoef, (size_t)B * d * 4, cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(intercept_out, dint, (size_t)B * 8, cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(n_iter_out, dniter, (size_t)B * 4, cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(t_out, dt, (size_t)B * 8, cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(status_out, dstatus, (size_t)B * 4, cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  c->d2h += (int64_t)B * (d * 4 + 24);
  return 0;
}

// one-vs-rest: every column in one group of all n rows in row order, one alpha
int sgd_fit_batch(Ctx* c, int B, const int32_t* col_pos, int loss, double alpha, int fit_intercept,
                  int max_iter, double tol, int shuffle, uint32_t seed, int lr_type, double eta0,
                  double power_t, double optimal_init, int n_iter_no_change, float* coef_out,
                  double* intercept_out, int32_t* n_iter_out, double* t_out, int32_t* status_out) {
  const int64_t n = c->n;
  std::vector<int32_t> grp(B, 0), rows(n);
  std::vector<double> al(B, alpha), oi(B, optimal_init);
  for (int64_t i = 0; i < n; ++i) rows[i] = (int32_t)i;
  const int64_t goff[2] = {0, n};
  return sgd_fit(c, B, col_pos, grp.data(), al.data(), oi.data(), 1, goff, rows.data(), &seed, true, loss,
                 fit_intercept, max_iter, tol, shuffle, lr_type, eta0, power_t, n_iter_no_change, coef_out,
                 intercept_out, n_iter_out, t_out, status_out);
}

int sgd_fit_groups(Ctx* c, int B, const int32_t* col_pos, const int32_t* col_group, const double* col_alpha,
                   const double* col_oi, int G, const int64_t* goff, const int32_t* grows, const uint32_t* gseed,
                   int loss, int fit_intercept, int max_iter, double tol, int shuffle, int lr_type, double eta0,
                   double power_t, int n_iter_no_change, float* coef_out, double* intercept_out,
                   int32_t* n_iter_out, double* t_out, int32_t* status_out) {
  return sgd_fit(c, B, col_pos, col_group, col_alpha, col_oi, G, goff, grows, gseed, false, loss, fit_intercept,
                 max_iter, tol, shuffle, lr_type, eta0, power_t, n_iter_no_change, coef_out, intercept_out,
                 n_iter_out, t_out, status_out);
}

}  // namespace skd
