// sgd_replay.h -- the pieces of scikit-learn's exact-order SGD that every SGD kernel replays
// (sgd.cu: one warp per label column; sgd_tc.cu: blocked-exact on the tensor cores).
//
// SK/linear_model/_sgd_fast.pyx.tp:274-640 (_plain_sgd32) with WeightVector32
// (SK/utils/_weight_vector.pyx.tp).  One warp owns one label column and keeps its d float32 weights
// in registers, d/32 per lane (w[j] is feature lane + 32 j).  Every helper reproduces the reference
// operation by operation: float32 products accumulated in float64, float32 lazy scale `wscale`,
// float64 norm / intercept / objective, weight update w = float(double(w) + double(x) * q).  The helpers
// take the lazy scale as a value: the warp kernels pass their running wscale, sgd_scan_kernel the
// host's replay of the scale chain.
#pragma once
#include <cuda_fp16.h>
#include <math.h>

#include "skd_internal.h"

namespace skd {

// per label column, carried from epoch to epoch (and from block to block on the tensor-core path)
struct SgdState {
  double wscale, sq_norm, intercept, best_objective, t;
  int32_t no_improve, done, n_iter, status;
  double objective_sum;   // objective of the current epoch so far (sgd_scan_kernel: across blocks; 0 between epochs)
};

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// w.reset_wscale(): sscal by float(wscale); the caller sets wscale = 1
template <int DPL>
__device__ __forceinline__ void sgd_reset_wscale(float (&w)[DPL], double wscale) {
  const float wf = (float)wscale;
#pragma unroll
  for (int j = 0; j < DPL; ++j) w[j] = __fmul_rn(w[j], wf);
}

// w.add(x, update) for update != 0 at lazy scale wscale, then intercept += update if fit_intercept.
// Returns the new sq_norm; q is the step applied to the stored weights, float(update) / float(wscale).
template <int DPL>
__device__ __forceinline__ double sgd_add(float (&w)[DPL], const float (&x)[DPL], double update, double wscale,
                                          int fit_intercept, double& intercept, double& q) {
  const float cf = (float)update, wsf = (float)wscale;
  q = (double)__fdiv_rn(cf, wsf);
  double acc2 = 0.0;
#pragma unroll
  for (int j = 0; j < DPL; ++j) {
    w[j] = (float)fma((double)x[j], q, (double)w[j]);
    acc2 += (double)__fmul_rn(w[j], w[j]);
  }
  acc2 = warp_sum(acc2);
  if (fit_intercept) intercept += update;
  return acc2 * (double)__fmul_rn(wsf, wsf);
}

// end of epoch (SK/linear_model/_sgd_fast.pyx.tp:570-628): every lane of the warp calls it with the column's
// weights and intercept after the epoch's n samples; st.wscale / sq_norm / intercept are the caller's
template <int DPL>
__device__ __forceinline__ void sgd_end_epoch(SgdState& st, const float (&w)[DPL], double intercept, double objective_sum,
                                              int64_t n, double tol, int n_iter_no_change) {
  bool finite = isfinite(intercept);
#pragma unroll
  for (int j = 0; j < DPL; ++j) finite = finite && isfinite(w[j]);
  finite = __all_sync(0xffffffffu, finite);
  st.t += (double)n;
  st.n_iter += 1;
  if (!finite) { st.done = 1; st.status = 5; }
  else {
    const double obj = objective_sum / (double)n;
    if (tol > -INFINITY && obj > st.best_objective - tol) st.no_improve += 1; else st.no_improve = 0;
    if (obj < st.best_objective) st.best_objective = obj;
    if (st.no_improve >= n_iter_no_change) { st.done = 1; st.status = 1; }
  }
  st.objective_sum = 0.0;
}

// What one fit shares between its epochs and between the two paths (device pointers).  The columns form
// order groups: group g walks its own n_g rows order[goff[g] .. goff[g+1]) (its own shuffle), and column j
// belongs to group col_group[j] with its own alpha.  The tensor-core path runs one group of all n rows with
// one alpha and reads the per-sample tables eta / cfac; the warp kernels form each column's rates themselves.
struct SgdFit {
  int B, dpl, ldw;          // columns; weights per lane; leading dimension of W (32 * dpl)
  float* W;                 // [B x ldw] stored weights (times wscale = the coefficients)
  SgdState* state;          // [B]
  const int32_t* col_pos;   // [B] positive class of each column
  const int32_t* col_group; // [B] order group of each column
  const double* col_alpha;  // [B] alpha of each column
  const double* col_oi;     // [B] its optimal_init ("optimal" rate)
  const int64_t* goff;      // [G + 1] start of each group's rows in order (and in eta)
  const int32_t* order;     // [goff[G]] sample order of the epoch, group by group
  const int32_t* active;    // [n_active] columns still running
  const double* eta;        // [goff[G]] learning rate of each sample of the epoch (tensor cores; warp kernels: invscaling only)
  const float* cfac;        // [n] its weight-decay factor max(0, 1 - eta * alpha), as float (tensor cores only)
  double alpha, tol, eta0;  // alpha: the tensor-core path's one alpha
  int fit_intercept, n_iter_no_change, lr_type;
};

// whether a fit runs its epochs on SgdTc: hinge, d <= 1024 and n >= 2 blocks of samples, unless
// SKDIST_B200_SGD_KERNEL=tc|simt chooses
bool sgd_tc_supported(const Ctx* c, int loss, int shuffle);

// Blocked-exact hinge epochs on the tensor cores (sgd_tc.cu).  Created once per fit: row norms and the
// power-of-two scale of X, the fp16 copies of X and W, the S / G products, the tensor maps, a second
// stream for G and the events that order the two streams.
struct SgdTc {
  explicit SgdTc(Ctx* c) : sx(c) {}
  ~SgdTc();
  int init(Ctx* c, const SgdFit& f);
  // one epoch after the schedule kernel has filled eta / cfac: permute X when `new_order`, replay the
  // lazy-scale chain on the host, export W, then per block of samples the S / G products and the scan
  int epoch(Ctx* c, const SgdFit& f, int epoch, int n_active, bool new_order, bool trace);
  void print_counters();   // screened / exact / violating sample visits of the whole fit and the scans whose
                           // violator log filled up (SKDIST_B200_TRACE=2)

  Scratch sx;
  int dpad = 0, kpad = 0, n_g = 0;
  int64_t npad = 0;
  size_t gemm_smem = 0;
  float sxs = 1.f, inv_sx = 1.f, inv_sx2 = 1.f;
  double wscale_epoch = 1.0;   // lazy scale at the start of the epoch (identical for all running columns)
  double* dws = nullptr;
  float *xnorm = nullptr, *xnorm_p = nullptr, *S = nullptr, *G[2] = {nullptr, nullptr};
  int32_t* ycls_p = nullptr;
  __half *Xp = nullptr, *Wp = nullptr;
  float2* wmeta[2] = {nullptr, nullptr};
  int2* gtiles = nullptr;
  unsigned long long* counters = nullptr;
  CUtensorMap map_x, map_w;
  cudaStream_t sB = nullptr;
  cudaEvent_t ev_perm = nullptr, ev_g[2] = {nullptr, nullptr}, ev_scan[2] = {nullptr, nullptr};
  cudaEvent_t ev_t[3] = {nullptr, nullptr, nullptr};
  std::vector<float> hcfac;
  std::vector<double> hws;
};

}  // namespace skd
