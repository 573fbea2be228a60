// auc.cu -- ranked counts of linear classifiers on their held-out rows: ROC-AUC (one-vs-rest, one-vs-one) and
// average precision.
//
// The reference scores a fitted clone with scorer(estimator, X_test, y_test) (ref search.py:264,
// utils.py:45-72).  For the ranking scorers (roc_auc, roc_auc_ovr[_weighted], roc_auc_ovo[_weighted],
// average_precision) every score is a function of one or more SEGMENTS: a set of rows, a positive flag per
// row and one fp32 score per row.
//   binary column (n_classes == 1)  the selected rows; positive = (ycls == col_pos); score = s
//   one-vs-rest (n_classes = K >= 3) one segment per class k: the selected rows; positive = (y == k); score s_k
//   one-vs-one  (K >= 3)            one segment per ordered pair (a, b), a != b: the selected rows with
//                                   y in {a, b}; positive = (y == a); score s_a.  A row lands in 2(K - 1)
//                                   segments.  Segment a * (K - 1) + (b < a ? b : b - 1).
// The area under the ROC curve with trapezoidal interpolation (SK/metrics/_ranking.py) of a segment equals
// the Mann-Whitney statistic
//   U = #{(p, q): s_p > s_q} + 0.5 * #{(p, q): s_p == s_q},  p positive rows, q negative rows,
//   auc = U / (n_pos * n_neg),
// which is computed here in INTEGERS (2U), so it does not depend on any summation order.  The uninterpolated
// average precision of precision_recall_curve(drop_intermediate=False) is, over the tie groups g of the
// segment in descending score order,
//   ap = sum_g pos_g * tp_g / (tp_g + fp_g) / n_pos,  tp_g / fp_g = positives / negatives scoring >= group g,
// and 0 for a segment without positives (scikit-learn's value there).
//   rank_key_kernel   one 64-bit key per (segment, row): segment id (bits 33..63) | order-preserving image of
//                     the fp32 score (bits 1..32) | label bit (negatives sort first inside a tie)
//   cub::DeviceRadixSort::SortKeys over all keys of a block of fits
//   rank_count_kernel one CTA per segment walks its sorted run: for every positive row the negatives at or
//                     below it (prefix count) and the rows of its tie group (two binary searches):
//                     2U = 2 * sum(prefix) - sum(tied negatives); the same searches give tp_g and fp_g.
//                     ap is summed in double per thread in row order, then over a fixed tree: deterministic.
// Scores (score_kind):
//   RANK_DECISION      the fp32 decision values of the CUDA-core path (simt_raw_prediction), as the
//                      reference's decision_function computes them in fp32
//   RANK_NEG_DECISION  their negation: scikit-learn's _get_response_values negates the decision values when
//                      the scorer's pos_label is classes_[0]
//   RANK_PROBA         float32 predict_proba of LogisticRegression on float32 X.  Binary: _predict_proba_lr's
//                      expit 1 / (1 + exp(-z)) in float32.  Multiclass: sklearn.utils.extmath.softmax in
//                      float32 -- subtract the row max, exp, numpy's pairwise row sum (8 accumulators), one
//                      division.  Every fp32 operation is rounded as numpy rounds it (no contraction); exp is
//                      exp() in double rounded once to float, i.e. correctly rounded, where numpy's SIMD expf
//                      is within 4 ulp of it.  A probability therefore differs from scikit-learn's by at most
//                      (K + 10) * 2^-23 of its value (K = 1 for binary): 4 from each exp in the quotient, one
//                      rounding per term of the sum that can go the other way, one for the division.
//                      Only pairs of rows whose probabilities lie closer than that can rank differently;
//                      saturated probabilities (exactly 1.0f once the decision gap exceeds about 17) are
//                      reproduced exactly, so their ties count 1/2 as in scikit-learn.
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>

#include "skd_internal.h"

namespace skd {

__device__ __forceinline__ unsigned int ordered_bits(float z) {
  if (z == 0.f) z = 0.f;                       // -0.0 and +0.0 are one value
  const unsigned int b = __float_as_uint(z);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ float exp_rn(float x) { return (float)exp((double)x); }

// numpy's float32 add.reduce of a contiguous row of n <= 128 terms (pairwise_sum: a plain loop below 8 terms,
// else 8 accumulators, a fixed tree, then the tail); term k = exp(z[k] - mx)
__device__ float softmax_row_sum(const float* __restrict__ z, int n, float mx) {
  if (n < 8) {
    float s = 0.f;
    for (int k = 0; k < n; ++k) s = __fadd_rn(s, exp_rn(__fsub_rn(z[k], mx)));
    return s;
  }
  float r[8];
#pragma unroll
  for (int q = 0; q < 8; ++q) r[q] = exp_rn(__fsub_rn(z[q], mx));
  int i = 8;
  for (; i < n - (n % 8); i += 8) {
#pragma unroll
    for (int q = 0; q < 8; ++q) r[q] = __fadd_rn(r[q], exp_rn(__fsub_rn(z[i + q], mx)));
  }
  float s = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])),
                      __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
  for (; i < n; ++i) s = __fadd_rn(s, exp_rn(__fsub_rn(z[i], mx)));
  return s;
}

__device__ __forceinline__ unsigned long long rank_key(int64_t seg, float s, bool pos) {
  return ((unsigned long long)seg << 33) | ((unsigned long long)ordered_bits(s) << 1) | (pos ? 1ull : 0ull);
}

// Keys of the t-th selected row of every fit in `fits`: keys[kbase[j] + t * kpr + q], q < kpr keys per row
// (1 binary, K one-vs-rest, 2(K - 1) one-vs-one).  Z: decision values, fit j's K' values at Z[r * ldz + j * K'].
__global__ void __launch_bounds__(256)
rank_key_kernel(const float* __restrict__ Z, int ldz, const int64_t* __restrict__ rows, int64_t n_rows,
                const int32_t* __restrict__ fits, int n_fits, const int64_t* __restrict__ kbase,
                const int32_t* __restrict__ ycls, const int32_t* __restrict__ pos, int K, int pairs, int kind,
                unsigned long long* __restrict__ keys) {
  const int jf = blockIdx.y;
  if (jf >= n_fits) return;
  const int j = fits[jf];                      // fit index inside this block of fits
  for (int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x; t < n_rows; t += (int64_t)gridDim.x * 256) {
    const int64_t r = rows[t];
    const int y = ycls[r];
    if (K == 1) {                              // binary column
      const float z = Z[r * ldz + j];
      float s = kind == RANK_NEG_DECISION ? -z : z;
      if (kind == RANK_PROBA) s = __fdiv_rn(1.0f, __fadd_rn(1.0f, exp_rn(-z)));
      keys[kbase[j] + t] = rank_key(j, s, y == pos[j]);
      continue;
    }
    const float* zr = Z + r * ldz + (int64_t)j * K;
    float mx = 0.f, sum = 1.f;
    if (kind == RANK_PROBA) {
      mx = zr[0];
      for (int k = 1; k < K; ++k) mx = fmaxf(mx, zr[k]);
      sum = softmax_row_sum(zr, K, mx);
    }
    auto score = [&](int k) {
      if (kind == RANK_PROBA) return __fdiv_rn(exp_rn(__fsub_rn(zr[k], mx)), sum);
      return kind == RANK_NEG_DECISION ? -zr[k] : zr[k];
    };
    unsigned long long* out = keys + kbase[j] + t * (pairs ? 2 * (K - 1) : K);
    if (!pairs) {
      for (int k = 0; k < K; ++k) out[k] = rank_key((int64_t)j * K + k, score(k), y == k);
    } else {
      // (y, b): positive with score s_y; (b, y): negative with score s_b
      const int64_t seg0 = (int64_t)j * K * (K - 1);
      const float sy = score(y);
      int q = 0;
      for (int b = 0; b < K; ++b) {
        if (b == y) continue;
        out[q++] = rank_key(seg0 + (int64_t)y * (K - 1) + (b < y ? b : b - 1), sy, true);
        out[q++] = rank_key(seg0 + (int64_t)b * (K - 1) + (y < b ? y : y - 1), score(b), false);
      }
    }
  }
}

__device__ __forceinline__ int64_t lower_bound_u64(const unsigned long long* a, int64_t n, unsigned long long v) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (a[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// out[3 s .. 3 s + 2] = {2U, n_pos, n_neg}, ap[s] = average precision of segment s of the sorted keys
__global__ void __launch_bounds__(256)
rank_count_kernel(const unsigned long long* __restrict__ keys, int64_t total, int n_seg, long long* __restrict__ out,
                  double* __restrict__ ap_out) {
  __shared__ long long s_cnt[256];
  __shared__ long long s_red[2][8];
  __shared__ double s_ap[8];
  const int sg = blockIdx.x;
  if (sg >= n_seg) return;
  const int64_t b0 = lower_bound_u64(keys, total, (unsigned long long)sg << 33);
  const int64_t len = lower_bound_u64(keys, total, (unsigned long long)(sg + 1) << 33) - b0;
  const unsigned long long* a = keys + b0;
  const int64_t per = (len + 255) / 256;
  int64_t b = (int64_t)threadIdx.x * per;
  if (b > len) b = len;
  int64_t e = b + per;
  if (e > len) e = len;
  long long negs = 0;
  for (int64_t i = b; i < e; ++i) negs += (long long)(~a[i] & 1ull);
  s_cnt[threadIdx.x] = negs;
  __syncthreads();
  for (int o = 1; o < 256; o <<= 1) {          // inclusive scan of the per-thread negative counts
    const long long v = threadIdx.x >= o ? s_cnt[threadIdx.x - o] : 0;
    __syncthreads();
    s_cnt[threadIdx.x] += v;
    __syncthreads();
  }
  const long long N = s_cnt[255], P = (long long)len - N;
  long long neg_before = s_cnt[threadIdx.x] - negs;   // negatives in front of this thread's run
  long long sum_prefix = 0, sum_ties = 0, n_pos = 0;
  double ap = 0.0, last_prec = 0.0;
  unsigned long long last_base = ~0ull;
  long long last_ties = 0;
  for (int64_t i = b; i < e; ++i) {
    const unsigned long long k = a[i];
    if (k & 1ull) {
      // negatives sort first inside a tie group, so every negative at or below this row is in front of it
      const unsigned long long base = k & ~1ull;
      if (base != last_base) {
        const int64_t g0 = lower_bound_u64(a, len, base), g1 = lower_bound_u64(a, len, base | 1ull);
        last_base = base;
        last_ties = (long long)(g1 - g0);
        const long long neg_below = neg_before - last_ties;          // negatives under the group
        const long long tp = P - ((long long)g0 - neg_below), fp = N - neg_below;
        last_prec = (double)tp / (double)(tp + fp);
      }
      sum_prefix += neg_before;
      sum_ties += last_ties;
      n_pos += 1;
      ap += last_prec;
    } else {
      neg_before += 1;
    }
  }
  long long v[2] = {2 * sum_prefix - sum_ties, n_pos};
#pragma unroll
  for (int q = 0; q < 2; ++q) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[q] += __shfl_xor_sync(0xffffffffu, v[q], o);
    if ((threadIdx.x & 31) == 0) s_red[q][threadIdx.x >> 5] = v[q];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ap += __shfl_xor_sync(0xffffffffu, ap, o);
  if ((threadIdx.x & 31) == 0) s_ap[threadIdx.x >> 5] = ap;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long u2 = 0, np = 0;
    for (int w = 0; w < 8; ++w) { u2 += s_red[0][w]; np += s_red[1][w]; }
    out[3 * (int64_t)sg + 0] = u2;
    out[3 * (int64_t)sg + 1] = np;
    out[3 * (int64_t)sg + 2] = (long long)len - np;
    const double sum = ((s_ap[0] + s_ap[1]) + (s_ap[2] + s_ap[3])) + ((s_ap[4] + s_ap[5]) + (s_ap[6] + s_ap[7]));
    ap_out[sg] = np > 0 ? sum / (double)np : 0.0;
  }
}

int rank_segments(int K, int pairs) { return K == 1 ? 1 : (pairs ? K * (K - 1) : K); }

// col_fold: scoring codes of skd_linear_score_batch.  K == 1: coef [B][d+1] binary columns with col_pos;
// K >= 3: coef [B][K][d+1].  Outputs [B][rank_segments(K, pairs)]; ap_out may be null.
int rank_batch(Ctx* c, int B, int K, const float* coef, const int32_t* col_fold, const int32_t* col_pos, int kind,
               int pairs, int64_t* u2_out, int64_t* n_pos_out, int64_t* n_neg_out, double* ap_out) {
  const int64_t n = c->n, ldx = c->ldx;
  const int Kz = K == 1 ? 1 : K;                        // decision values per fit
  const int S = rank_segments(K, pairs);                // segments per fit
  const int kpr = K == 1 ? 1 : (pairs ? 2 * (K - 1) : K);   // keys per selected row
  // row selection lists, one per distinct code
  std::vector<int32_t> codes(col_fold, col_fold + B);
  std::sort(codes.begin(), codes.end());
  codes.erase(std::unique(codes.begin(), codes.end()), codes.end());
  if (!c->h_fold.empty() && (int64_t)c->h_fold.size() != n) return fail(c, "skd_linear_rank_batch: fold ids out of date");
  std::vector<std::vector<int64_t>> lists(codes.size());
  for (size_t q = 0; q < codes.size(); ++q) {
    const int cd = codes[q];
    for (int64_t r = 0; r < n; ++r) {
      const int fd = c->h_fold.empty() ? -1 : (int)c->h_fold[r];
      if (score_code_selects(cd, fd)) lists[q].push_back(r);
    }
  }
  auto list_of = [&](int cd) { return (size_t)(std::lower_bound(codes.begin(), codes.end(), cd) - codes.begin()); };
  // blocks of fits: bound the decision matrix (n x fits x K' fp32), the keys (2 x 8 B per key) and the
  // segments (4096 per block where a fit has no more: 12 bits of segment id keep the sorted key width at 45
  // bits, so the radix sort makes no more passes over the keys than it needs)
  size_t max_rows = 1;
  for (auto& l : lists) max_rows = std::max(max_rows, l.size());
  int per = (int)std::max<double>(1.0, std::min({2.0e9 / (4.0 * (double)n * Kz),
                                                 3.0e9 / (16.0 * (double)max_rows * kpr), 4096.0 / S}));
  for (int b0 = 0; b0 < B; b0 += per) {
    const int Bb = std::min(per, B - b0);
    const int n_seg = Bb * S;
    Scratch sx(c);
    std::vector<int64_t> kbase(Bb + 1, 0);
    for (int j = 0; j < Bb; ++j) kbase[j + 1] = kbase[j] + (int64_t)lists[list_of(col_fold[b0 + j])].size() * kpr;
    const int64_t total = kbase[Bb];
    float *dW, *Z;
    int64_t* dkbase;
    int32_t* dpos;
    unsigned long long *k0, *k1;
    long long* dout;
    double* dap;
    const size_t slots = (size_t)Bb * Kz;
    if (pack_coef(c, sx, (int)slots, coef + (size_t)b0 * Kz * (c->d + 1), c->d, ldx, &dW)) return 1;
    SKD_CUDA(c, sx.alloc(&Z, (size_t)n * slots));
    SKD_CUDA(c, sx.alloc(&dkbase, (size_t)Bb + 1));
    SKD_CUDA(c, sx.alloc(&dpos, (size_t)Bb));
    SKD_CUDA(c, sx.alloc(&k0, (size_t)std::max<int64_t>(total, 1)));
    SKD_CUDA(c, sx.alloc(&k1, (size_t)std::max<int64_t>(total, 1)));
    SKD_CUDA(c, sx.alloc(&dout, (size_t)3 * n_seg));
    SKD_CUDA(c, sx.alloc(&dap, (size_t)n_seg));
    SKD_CUDA(c, cudaMemcpyAsync(dkbase, kbase.data(), kbase.size() * sizeof(int64_t), cudaMemcpyHostToDevice, c->stream));
    if (K == 1)
      SKD_CUDA(c, cudaMemcpyAsync(dpos, col_pos + b0, Bb * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    if (simt_raw_prediction(c, (int)slots, dW, dW + slots * ldx, Z, (int)slots)) return 1;
    // keys, one launch per selection list (the fits that use it)
    std::vector<int64_t*> drows(codes.size(), nullptr);
    std::vector<int32_t*> dfits(codes.size(), nullptr);
    std::vector<std::vector<int32_t>> hfits(codes.size());
    for (int j = 0; j < Bb; ++j) hfits[list_of(col_fold[b0 + j])].push_back(j);
    for (size_t q = 0; q < codes.size(); ++q) {
      if (hfits[q].empty() || lists[q].empty()) continue;
      SKD_CUDA(c, sx.alloc(&drows[q], lists[q].size()));
      SKD_CUDA(c, sx.alloc(&dfits[q], hfits[q].size()));
      SKD_CUDA(c, cudaMemcpyAsync(drows[q], lists[q].data(), lists[q].size() * sizeof(int64_t), cudaMemcpyHostToDevice, c->stream));
      SKD_CUDA(c, cudaMemcpyAsync(dfits[q], hfits[q].data(), hfits[q].size() * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
      const int gx = (int)std::min<int64_t>(1024, ((int64_t)lists[q].size() + 255) / 256);
      for (size_t c0 = 0; c0 < hfits[q].size(); c0 += 65535) {
        const int nf = (int)std::min<size_t>(65535, hfits[q].size() - c0);
        rank_key_kernel<<<dim3(gx, nf), 256, 0, c->stream>>>(Z, (int)slots, drows[q], (int64_t)lists[q].size(),
                                                             dfits[q] + c0, nf, dkbase, c->ycls, dpos, K, pairs, kind,
                                                             k0);
        c->launches += 1;
      }
    }
    SKD_CUDA(c, cudaGetLastError());
    const unsigned long long* sorted = k0;
    if (total > 0) {
      int seg_bits = 1;
      while ((1 << seg_bits) < n_seg) ++seg_bits;
      size_t tmp_bytes = 0;
      SKD_CUDA(c, cub::DeviceRadixSort::SortKeys(nullptr, tmp_bytes, k0, k1, total, 0, 33 + seg_bits, c->stream));
      uint8_t* tmp;
      SKD_CUDA(c, sx.alloc(&tmp, tmp_bytes + 16));
      SKD_CUDA(c, cub::DeviceRadixSort::SortKeys(tmp, tmp_bytes, k0, k1, total, 0, 33 + seg_bits, c->stream));
      c->launches += 1;
      sorted = k1;
    }
    rank_count_kernel<<<n_seg, 256, 0, c->stream>>>(sorted, total, n_seg, dout, dap);
    c->launches += 1;
    SKD_CUDA(c, cudaGetLastError());
    std::vector<long long> hout((size_t)3 * n_seg);
    SKD_CUDA(c, cudaMemcpyAsync(hout.data(), dout, hout.size() * sizeof(long long), cudaMemcpyDeviceToHost, c->stream));
    if (ap_out)
      SKD_CUDA(c, cudaMemcpyAsync(ap_out + (size_t)b0 * S, dap, (size_t)n_seg * sizeof(double), cudaMemcpyDeviceToHost,
                                  c->stream));
    SKD_CUDA(c, cudaStreamSynchronize(c->stream));
    c->d2h += (int64_t)hout.size() * 8 + (ap_out ? (int64_t)n_seg * 8 : 0);
    for (int s = 0; s < n_seg; ++s) {
      u2_out[(size_t)b0 * S + s] = hout[3 * (size_t)s + 0];
      n_pos_out[(size_t)b0 * S + s] = hout[3 * (size_t)s + 1];
      n_neg_out[(size_t)b0 * S + s] = hout[3 * (size_t)s + 2];
    }
  }
  return 0;
}

// ROC-AUC counts of binary columns on their fp32 decision values (skd_linear_auc_batch)
int auc_batch(Ctx* c, int B, const float* coef, const int32_t* col_fold, const int32_t* col_pos,
              int64_t* u2_out, int64_t* n_pos_out, int64_t* n_neg_out) {
  return rank_batch(c, B, 1, coef, col_fold, col_pos, RANK_DECISION, 0, u2_out, n_pos_out, n_neg_out, nullptr);
}

}  // namespace skd
