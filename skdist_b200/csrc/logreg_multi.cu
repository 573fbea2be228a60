// logreg_multi.cu -- batched multinomial logistic regression (more than two classes).
//
// What LogisticRegression(solver="lbfgs").fit does for a multiclass target, for every
// (candidate, fold) of a search at once (ref search.py:228-230 -> SK/linear_model/_logistic.py:523-547,
// 584-598):  minimise  mean_i[ logsumexp(z_i) - z_{i, y_i} ] + 0.5 * l2 * ||W||^2,  z_i = W x_i + b,
// l2 = 1 / (C * n_train), intercepts unpenalised, L-BFGS-B from W = 0.
//
// One optimiser problem per candidate with K * (d + 1) variables (lbfgs_dev.cu lb_step_kernel); the
// evaluation treats the K class rows of every active candidate as K slots of one fp32 slot matrix:
//   simt_raw_prediction  Z = X W^T + b                       (fp32 FMA, SK/_linear_loss.py:219)
//   mn_pointwise_kernel  per training row: softmax, loss, p - onehot in place of Z
//                        (CyHalfMultinomialLoss.loss_gradient, SK/_loss/_loss.pyx.tp:1293-1327,
//                        sum_exp_minus_max :269-305, float32 in / float32 out like the reference)
//   mn_colsum_kernel     sum_i G[i][slot]  (intercept gradient, SK/_linear_loss.py:368-370)
//   simt_backward        G^T X             (SK/_linear_loss.py:364)
// Rows are split into a FIXED number of chunks that depends on n alone and the per-chunk partial
// sums are added in chunk order, so a candidate's result does not depend on what else is in the
// batch.  Held-out rows of a candidate get a zero pointwise gradient (fold mask, no copies of X).
//
// First CUDA path of this objective: fp32 CUDA cores (the binary objective's tensor-core kernel does
// not cover it yet, DESIGN.md "multinomial").
#include <algorithm>

#include "skd_internal.h"

namespace skd {

// One CTA per (active candidate, row chunk); a thread owns whole rows.
__global__ void __launch_bounds__(256)
mn_pointwise_kernel(float* __restrict__ G, int ldg, int64_t n, int64_t rpc, int K,
                    const SlotMeta* __restrict__ cand, const int32_t* __restrict__ n_act_dev, int n_act_in,
                    const int32_t* __restrict__ ycls, const int8_t* __restrict__ fold,
                    double* __restrict__ lossp, const float* __restrict__ cw) {
  __shared__ double red[8];
  const int a = blockIdx.x, z = blockIdx.y;
  if (a >= *n_act_dev) return;
  const int f = cand[a].fold;
  const float* wk = cw ? cw + (size_t)cand[a].col * K : nullptr;   // class weights of the candidate
  const int64_t row_begin = (int64_t)z * rpc;
  int64_t row_end = row_begin + rpc;
  if (row_end > n) row_end = n;
  double acc = 0.0;
  for (int64_t r = row_begin + threadIdx.x; r < row_end; r += 256) {
    float* zr = G + r * ldg + (size_t)a * K;
    const int y = ycls[r];
    const bool train = (f < 0 || !fold || (int)fold[r] != f) && y >= 0 && y < K;
    if (!train) {
      for (int k = 0; k < K; ++k) zr[k] = 0.f;
      continue;
    }
    float mx = zr[0];
    for (int k = 1; k < K; ++k) { const float v = zr[k]; if (mx < v) mx = v; }
    double sum = 0.0;
    for (int k = 0; k < K; ++k) sum += (double)(float)exp((double)zr[k] - (double)mx);
    const float sum_f = (float)sum;
    float loss = (float)(log((double)sum_f) + (double)mx);
    loss -= zr[y];
    if (wk) {   // sample weight of the row: float32 products, as SK/_loss/_loss.pyx.tp:1348-1350
      const float sw = wk[y];
      for (int k = 0; k < K; ++k) {
        float p = (float)exp((double)zr[k] - (double)mx);
        p /= sum_f;
        zr[k] = (p - (k == y ? 1.f : 0.f)) * sw;
      }
      loss *= sw;
    } else {
      for (int k = 0; k < K; ++k) {
        float p = (float)exp((double)zr[k] - (double)mx);
        p /= sum_f;
        zr[k] = p - (k == y ? 1.f : 0.f);
      }
    }
    acc += (double)loss;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0)
    lossp[(size_t)z * n_act_in + a] = ((red[0] + red[1]) + (red[2] + red[3])) + ((red[4] + red[5]) + (red[6] + red[7]));
}

// gsump[z][slot] = sum over the rows of chunk z of G[i][slot]; 64 slots x 4 row lanes per CTA
__global__ void __launch_bounds__(256)
mn_colsum_kernel(const float* __restrict__ G, int ldg, int64_t n, int64_t rpc, int n_slots,
                 double* __restrict__ gsump) {
  __shared__ double part[4][64];
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
  const int s = blockIdx.x * 64 + tx, z = blockIdx.y;
  const int64_t row_begin = (int64_t)z * rpc;
  int64_t row_end = row_begin + rpc;
  if (row_end > n) row_end = n;
  double acc = 0.0;
  if (s < n_slots)
    for (int64_t r = row_begin + ty; r < row_end; r += 4) acc += (double)G[r * ldg + s];
  part[ty][tx] = acc;
  __syncthreads();
  if (ty == 0 && s < n_slots)
    gsump[(size_t)z * n_slots + s] = (part[0][tx] + part[1][tx]) + (part[2][tx] + part[3][tx]);
}

// confusion counts conf[b][true class][predicted class] of argmax_k z (first maximum, like
// numpy.argmax in LinearClassifierMixin.predict, SK/linear_model/_base.py:351-374) on the rows
// selected by the candidate's scoring code (score_code_selects).
// Every count-based multiclass metric (accuracy, precision / recall / f1 with any averaging,
// balanced accuracy) is a function of this matrix.  SMEM = 1: the CTA counts in shared memory first.
template <int SMEM>
__global__ void __launch_bounds__(256)
mn_confusion_kernel(const float* __restrict__ Z, int ldz, int64_t n, int64_t rpc, int K, int B,
                    const int32_t* __restrict__ code, const int32_t* __restrict__ ycls,
                    const int8_t* __restrict__ fold, unsigned long long* __restrict__ conf) {
  extern __shared__ unsigned int sconf[];
  const int b = blockIdx.x, z = blockIdx.y;
  const int cd = code[b];
  const int KK = K * K;
  if (SMEM) {
    for (int i = threadIdx.x; i < KK; i += 256) sconf[i] = 0u;
    __syncthreads();
  }
  unsigned long long* out = conf + (size_t)b * KK;
  const int64_t row_begin = (int64_t)z * rpc;
  int64_t row_end = row_begin + rpc;
  if (row_end > n) row_end = n;
  for (int64_t r = row_begin + threadIdx.x; r < row_end; r += 256) {
    const int fd = fold ? (int)fold[r] : -1;
    const bool test = score_code_selects(cd, fd);
    const int y = ycls[r];
    if (!test || y < 0 || y >= K) continue;
    const float* zr = Z + r * ldz + (size_t)b * K;
    int best = 0;
    float mx = zr[0];
    for (int k = 1; k < K; ++k) { const float v = zr[k]; if (v > mx) { mx = v; best = k; } }
    if (SMEM) atomicAdd(&sconf[y * K + best], 1u);
    else atomicAdd(&out[y * K + best], 1ull);
  }
  if (SMEM) {
    __syncthreads();
    for (int i = threadIdx.x; i < KK; i += 256)
      if (sconf[i]) atomicAdd(&out[i], (unsigned long long)sconf[i]);
  }
}

// fixed row chunking: depends on n alone
static void multi_chunks(int64_t n, int* nz, int64_t* rpc) {
  int want = (int)std::min<int64_t>(64, (n + 63) / 64);
  if (want < 1) want = 1;
  int64_t r = (n + want - 1) / want;
  r = (r + 63) / 64 * 64;
  *rpc = r;
  *nz = (int)((n + r - 1) / r);
}

static int64_t candidates_per_pass(const Ctx* c, int K, int nz) {
  // bound the raw-prediction matrix (n x slots fp32) and the gradient partials (nz x slots x ldx fp32)
  const double budget = 6.0e9;
  const double per_cand = 4.0 * K * ((double)c->n + (double)nz * (double)c->ldx);
  int64_t b = (int64_t)(budget / per_cand);
  return b < 1 ? 1 : b;
}

// Device buffers of one pass over candidates b0 .. b0 + Bb - 1 and the uploads of their constants (l2, inv_n,
// held-out folds into *d_fold, feature masks, class weights), shared by multi_fit and multi_loss_grad.
static int multi_pass_setup(Ctx* c, Scratch& sx, MultiWork& w, int64_t b0, int Bb, int K, int nz, int64_t rpc,
                            const double* l2, const double* inv_n, const int32_t* col_fold, const uint8_t* fmask,
                            const float* cw, int32_t** d_fold) {
  const int64_t n = c->n, ldx = c->ldx;
  LbfgsBatch& b = w.lb;
  b.B = Bb; b.K = K; b.n = K * ((int)c->d + 1); b.nz = nz; b.ldw = (int)ldx;
  w.rpc = rpc;
  const size_t slots = (size_t)Bb * K;
  w.ldg = (int)((slots + 63) / 64 * 64);
  if (lbfgs_alloc(c, sx, b, Bb, false)) return 1;
  SKD_CUDA(c, sx.alloc(d_fold, (size_t)Bb));
  SKD_CUDA(c, sx.alloc(&b.W, slots * ldx + slots));
  SKD_CUDA(c, sx.alloc(&w.G, (size_t)n * w.ldg));
  SKD_CUDA(c, sx.alloc(&b.lossp, (size_t)nz * Bb));
  SKD_CUDA(c, sx.alloc(&b.gsump, (size_t)nz * slots));
  SKD_CUDA(c, sx.alloc(&b.gradp, (size_t)nz * slots * ldx));
  SKD_CUDA(c, cudaMemcpyAsync(b.l2, l2 + b0, Bb * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(b.inv_n, inv_n + b0, Bb * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(*d_fold, col_fold + b0, Bb * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
  c->h2d += (int64_t)Bb * 20;
  if (fmask) {     // per-candidate feature masks (DistFeatureEliminator): masked weights stay exactly 0
    SKD_CUDA(c, sx.alloc(&b.fmask, (size_t)Bb * c->d));
    SKD_CUDA(c, cudaMemcpyAsync(b.fmask, fmask + (size_t)b0 * c->d, (size_t)Bb * c->d, cudaMemcpyHostToDevice, c->stream));
    c->h2d += (int64_t)Bb * c->d;
  }
  if (cw) {
    float* dcw;
    SKD_CUDA(c, sx.alloc(&dcw, (size_t)Bb * K));
    SKD_CUDA(c, cudaMemcpyAsync(dcw, cw + (size_t)b0 * K, (size_t)Bb * K * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    c->h2d += (int64_t)Bb * K * 4;
    w.cw = dcw;
  }
  return 0;
}

// One evaluation of the n_act active candidates at the slot rows in w.lb.W: raw predictions, pointwise loss and
// gradient in place, per-chunk intercept and weight gradient partials (lossp, gsump, gradp of w.lb).
static int multi_eval(Ctx* c, MultiWork& w, int n_act) {
  const LbfgsBatch& b = w.lb;
  const size_t slots = (size_t)b.B * b.K;
  const int ns = n_act * b.K;
  if (simt_raw_prediction(c, ns, b.W, b.W + slots * c->ldx, w.G, w.ldg)) return 1;
  mn_pointwise_kernel<<<dim3(n_act, b.nz), 256, 0, c->stream>>>(w.G, w.ldg, c->n, w.rpc, b.K, b.slot, b.n_act, n_act,
                                                               c->ycls, c->fold, b.lossp, w.cw);
  mn_colsum_kernel<<<dim3((ns + 63) / 64, b.nz), 256, 0, c->stream>>>(w.G, w.ldg, c->n, w.rpc, ns, b.gsump);
  c->launches += 2;
  return simt_backward(c, w.G, w.ldg, ns, b.nz, w.rpc, b.gradp);
}

int multi_fit(Ctx* c, int B, int K, const double* l2, const double* inv_n, const int32_t* col_fold, int fit_intercept,
              double tol, int max_iter, const uint8_t* fmask, const float* cw, float* coef_out,
              int32_t* n_iter_out, int32_t* status_out, double* loss_out, int32_t* n_evals_out) {
  int nz;
  int64_t rpc;
  multi_chunks(c->n, &nz, &rpc);
  const int64_t per_pass = candidates_per_pass(c, K, nz);
  for (int64_t b0 = 0; b0 < B; b0 += per_pass) {
    const int Bb = (int)std::min<int64_t>(per_pass, B - b0);
    Scratch sx(c);
    MultiWork w;
    int32_t* d_fold;
    if (multi_pass_setup(c, sx, w, b0, Bb, K, nz, rpc, l2, inv_n, col_fold, fmask, cw, &d_fold)) return 1;
    if (lbfgs_init(c, w.lb, d_fold, nullptr, nullptr, tol, max_iter)) return 1;
    if (lbfgs_run(c, w.lb, Bb, fit_intercept, max_iter, nullptr, nullptr,
                  [&](int n_act, long, int*) { return multi_eval(c, w, n_act); }, nullptr))
      return 1;
    if (lbfgs_result(c, sx, w.lb, b0, coef_out, n_iter_out, status_out, loss_out, n_evals_out)) return 1;
    SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  }
  return 0;
}

// Objective and gradient at caller points w_in [B][K][d+1] (float64): the passes, set-up, evaluation and
// gather of multi_fit's first round, with every candidate active in column order.
int multi_loss_grad(Ctx* c, int B, int K, const double* l2, const double* inv_n, const int32_t* col_fold,
                    int fit_intercept, const uint8_t* fmask, const float* cw, const double* w_in, double* loss_out,
                    double* grad_out) {
  const int dp = (int)c->d + 1;
  int nz;
  int64_t rpc;
  multi_chunks(c->n, &nz, &rpc);
  const int64_t per_pass = candidates_per_pass(c, K, nz);
  for (int64_t b0 = 0; b0 < B; b0 += per_pass) {
    const int Bb = (int)std::min<int64_t>(per_pass, B - b0);
    Scratch sx(c);
    MultiWork w;
    int32_t* d_fold;
    if (multi_pass_setup(c, sx, w, b0, Bb, K, nz, rpc, l2, inv_n, col_fold, fmask, cw, &d_fold)) return 1;
    std::vector<SlotMeta> hc(Bb);
    for (int j = 0; j < Bb; ++j) { hc[j].col = j; hc[j].fold = col_fold[b0 + j]; hc[j].pos = 0; hc[j].pad = 0; }
    double *dx, *df, *dg;
    const size_t nvar = (size_t)Bb * K * dp;
    SKD_CUDA(c, sx.alloc(&dx, nvar));
    SKD_CUDA(c, sx.alloc(&df, (size_t)Bb));
    SKD_CUDA(c, sx.alloc(&dg, nvar));
    SKD_CUDA(c, cudaMemcpyAsync(w.lb.slot, hc.data(), Bb * sizeof(SlotMeta), cudaMemcpyHostToDevice, c->stream));
    SKD_CUDA(c, cudaMemcpyAsync(w.lb.n_act, &Bb, sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    SKD_CUDA(c, cudaMemcpyAsync(dx, w_in + (size_t)b0 * K * dp, nvar * sizeof(double), cudaMemcpyHostToDevice,
                                c->stream));
    c->h2d += (int64_t)Bb * sizeof(SlotMeta) + 4 + (int64_t)nvar * 8;
    if (lbfgs_export_points(c, w.lb, Bb, dx)) return 1;
    if (multi_eval(c, w, Bb)) return 1;
    if (lbfgs_gather(c, w.lb, Bb, nz, fit_intercept, dx, df, dg)) return 1;
    SKD_CUDA(c, cudaMemcpyAsync(loss_out + b0, df, Bb * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    SKD_CUDA(c, cudaMemcpyAsync(grad_out + (size_t)b0 * K * dp, dg, nvar * sizeof(double), cudaMemcpyDeviceToHost,
                                c->stream));
    SKD_CUDA(c, cudaStreamSynchronize(c->stream));
    c->d2h += (int64_t)Bb * 8 + (int64_t)nvar * 8;
  }
  return 0;
}

int multi_score(Ctx* c, int B, int K, const float* coef, const int32_t* col_fold, int64_t* conf_out) {
  const int64_t n = c->n, d = c->d, ldx = c->ldx;
  const int dp = (int)d + 1;
  const size_t KK = (size_t)K * K;
  int nz;
  int64_t rpc;
  multi_chunks(n, &nz, &rpc);
  const int64_t per_pass = candidates_per_pass(c, K, 0);
  for (int64_t b0 = 0; b0 < B; b0 += per_pass) {
    const int Bb = (int)std::min<int64_t>(per_pass, B - b0);
    const size_t slots = (size_t)Bb * K;
    Scratch sx(c);
    float *dW, *Z;
    int32_t* dcode;
    unsigned long long* dconf;
    const int ldz = (int)slots;
    if (pack_coef(c, sx, (int)slots, coef + (size_t)b0 * K * dp, d, ldx, &dW)) return 1;
    SKD_CUDA(c, sx.alloc(&Z, (size_t)n * ldz));
    SKD_CUDA(c, sx.alloc(&dcode, (size_t)Bb));
    SKD_CUDA(c, sx.alloc(&dconf, (size_t)Bb * KK));
    SKD_CUDA(c, cudaMemcpyAsync(dcode, col_fold + b0, Bb * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    SKD_CUDA(c, cudaMemsetAsync(dconf, 0, (size_t)Bb * KK * sizeof(unsigned long long), c->stream));
    if (simt_raw_prediction(c, (int)slots, dW, dW + slots * ldx, Z, ldz)) return 1;
    const size_t smem = KK * sizeof(unsigned int);
    if (smem <= 48 * 1024)
      mn_confusion_kernel<1><<<dim3(Bb, nz), 256, smem, c->stream>>>(Z, ldz, n, rpc, K, Bb, dcode, c->ycls, c->fold, dconf);
    else
      mn_confusion_kernel<0><<<dim3(Bb, nz), 256, 0, c->stream>>>(Z, ldz, n, rpc, K, Bb, dcode, c->ycls, c->fold, dconf);
    c->launches += 1;
    SKD_CUDA(c, cudaGetLastError());
    SKD_CUDA(c, cudaMemcpyAsync(conf_out + (size_t)b0 * KK, dconf, (size_t)Bb * KK * sizeof(int64_t),
                                cudaMemcpyDeviceToHost, c->stream));
    SKD_CUDA(c, cudaStreamSynchronize(c->stream));
    c->d2h += (int64_t)Bb * KK * 8;
  }
  return 0;
}

// ---- log loss of the predicted probabilities (scoring="neg_log_loss") --------------------------------
// log_loss(y_test, predict_proba(X_test)) of SK/metrics/_classification.py: probabilities = softmax of
// the decision values (binary: [1 - expit(z), expit(z)], SK/linear_model/_logistic.py:1617-1625), clipped to
// [eps, 1 - eps] with eps = float32 epsilon (predict_proba returns float32 for float32 X), summed as
// -log p_true.  K == 1: binary columns, true class = (ycls == pos[b]).  Partials per (chunk, column) in
// double, added in chunk order by the host.
__global__ void __launch_bounds__(256)
mn_logloss_kernel(const float* __restrict__ Z, int ldz, int64_t n, int64_t rpc, int K, int B,
                  const int32_t* __restrict__ code, const int32_t* __restrict__ pos,
                  const int32_t* __restrict__ ycls, const int8_t* __restrict__ fold,
                  double* __restrict__ lossp, unsigned long long* __restrict__ count) {
  __shared__ double red[8];
  __shared__ unsigned long long redn[8];
  const int b = blockIdx.x, z = blockIdx.y;
  const int cd = code[b];
  const double eps = 1.1920928955078125e-07;     // numpy.finfo(float32).eps
  const int64_t row_begin = (int64_t)z * rpc;
  int64_t row_end = row_begin + rpc;
  if (row_end > n) row_end = n;
  double acc = 0.0;
  unsigned long long nn = 0;
  for (int64_t r = row_begin + threadIdx.x; r < row_end; r += 256) {
    const int fd = fold ? (int)fold[r] : -1;
    if (!score_code_selects(cd, fd)) continue;
    const int y = ycls[r];
    double p;
    if (K == 1) {
      // binary: p1 = expit(z) as float32, p0 = 1 - p1 in float32 (SK/linear_model/_base.py:438-440) --
      // the cancellation in 1 - p1 is part of what the reference scores
      // scipy's float32 expit is 1 / (1 + expf(-z)) in float arithmetic; each rounding is reproduced
      const float e = (float)exp(-(double)Z[r * ldz + b]);
      const float p1 = __fdiv_rn(1.0f, __fadd_rn(1.0f, e));
      p = (double)((y == pos[b]) ? p1 : __fsub_rn(1.0f, p1));
    } else {
      if (y < 0 || y >= K) continue;
      const float* zr = Z + r * ldz + (size_t)b * K;
      float mx = zr[0];
      for (int k = 1; k < K; ++k) mx = fmaxf(mx, zr[k]);
      double sum = 0.0;
      for (int k = 0; k < K; ++k) sum += exp((double)zr[k] - (double)mx);
      p = (double)(float)(exp((double)zr[y] - (double)mx) / sum);      // predict_proba is float32
    }
    p = fmin(fmax(p, eps), 1.0 - eps);
    acc -= log(p);
    nn += 1;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    acc += __shfl_xor_sync(0xffffffffu, acc, o);
    nn += __shfl_xor_sync(0xffffffffu, nn, o);
  }
  if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5] = acc; redn[threadIdx.x >> 5] = nn; }
  __syncthreads();
  if (threadIdx.x == 0) {
    lossp[(size_t)z * B + b] = ((red[0] + red[1]) + (red[2] + red[3])) + ((red[4] + red[5]) + (red[6] + red[7]));
    unsigned long long t = 0;
    for (int i = 0; i < 8; ++i) t += redn[i];
    if (t) atomicAdd(&count[b], t);
  }
}

// K == 1: coef [B][d+1] binary columns with col_pos; K >= 2: coef [B][K][d+1]
int logloss_batch(Ctx* c, int B, int K, const float* coef, const int32_t* col_fold, const int32_t* col_pos,
                  double* loss_sum_out, int64_t* count_out) {
  const int64_t n = c->n, d = c->d, ldx = c->ldx;
  const int dp = (int)d + 1;
  int nz;
  int64_t rpc;
  multi_chunks(n, &nz, &rpc);
  const int64_t per_pass = candidates_per_pass(c, K, 0);
  for (int64_t b0 = 0; b0 < B; b0 += per_pass) {
    const int Bb = (int)std::min<int64_t>(per_pass, B - b0);
    const size_t slots = (size_t)Bb * K;
    Scratch sx(c);
    float *dW, *Z;
    int32_t *dcode, *dpos = nullptr;
    double* dloss;
    unsigned long long* dcount;
    const int ldz = (int)slots;
    if (pack_coef(c, sx, (int)slots, coef + (size_t)b0 * K * dp, d, ldx, &dW)) return 1;
    SKD_CUDA(c, sx.alloc(&Z, (size_t)n * ldz));
    SKD_CUDA(c, sx.alloc(&dcode, (size_t)Bb));
    SKD_CUDA(c, sx.alloc(&dpos, (size_t)Bb));
    SKD_CUDA(c, sx.alloc(&dloss, (size_t)nz * Bb));
    SKD_CUDA(c, sx.alloc(&dcount, (size_t)Bb));
    SKD_CUDA(c, cudaMemcpyAsync(dcode, col_fold + b0, Bb * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    if (col_pos) SKD_CUDA(c, cudaMemcpyAsync(dpos, col_pos + b0, Bb * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    SKD_CUDA(c, cudaMemsetAsync(dcount, 0, Bb * sizeof(unsigned long long), c->stream));
    if (simt_raw_prediction(c, (int)slots, dW, dW + slots * ldx, Z, ldz)) return 1;
    mn_logloss_kernel<<<dim3(Bb, nz), 256, 0, c->stream>>>(Z, ldz, n, rpc, K, Bb, dcode, dpos, c->ycls, c->fold, dloss,
                                                          dcount);
    c->launches += 1;
    SKD_CUDA(c, cudaGetLastError());
    std::vector<double> hl((size_t)nz * Bb);
    SKD_CUDA(c, cudaMemcpyAsync(hl.data(), dloss, hl.size() * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    SKD_CUDA(c, cudaMemcpyAsync(count_out + b0, dcount, Bb * sizeof(int64_t), cudaMemcpyDeviceToHost, c->stream));
    SKD_CUDA(c, cudaStreamSynchronize(c->stream));
    c->d2h += (int64_t)hl.size() * 8 + (int64_t)Bb * 8;
    for (int j = 0; j < Bb; ++j) {
      double sum = 0.0;
      for (int z = 0; z < nz; ++z) sum += hl[(size_t)z * Bb + j];
      loss_sum_out[b0 + j] = sum;
    }
  }
  return 0;
}

}  // namespace skd
