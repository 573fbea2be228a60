// auc.cu -- area under the ROC curve of B linear binary classifiers on their held-out rows.
//
// The reference scores a fitted clone with scorer(estimator, X_test, y_test) (ref search.py:264,
// utils.py:45-72); with scoring="roc_auc" (the reference's own examples/search/basic_usage.py) that is
// roc_auc_score(y_test, decision_function(X_test)).  For a binary target the area under the ROC
// curve with trapezoidal interpolation (SK/metrics/_ranking.py) equals the Mann-Whitney statistic
//   U = #{(p, q): z_p > z_q} + 0.5 * #{(p, q): z_p == z_q},  p positive rows, q negative rows,
//   auc = U / (n_pos * n_neg),
// which is computed here in INTEGERS (2U), so the result does not depend on any summation order:
//   auc_key_kernel   one 64-bit key per (column, selected row): column id | order-preserving image of
//                    the fp32 decision value | label bit (negatives sort first inside a tie)
//   cub::DeviceRadixSort::SortKeys over all keys of a block of columns (45 key bits at most)
//   auc_count_kernel one CTA per column walks its sorted segment: for every positive row the number
//                    of negatives at or below it (prefix count) and the negatives of its tie group
//                    (two binary searches); 2U = 2 * sum(prefix) - sum(ties)
// Decision values are the fp32 products of the CUDA-core path (simt_decision), as the reference's
// decision_function computes them in fp32.
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>

#include "skd_internal.h"

namespace skd {

__device__ __forceinline__ unsigned int ordered_bits(float z) {
  if (z == 0.f) z = 0.f;                       // -0.0 and +0.0 are one value
  const unsigned int b = __float_as_uint(z);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// keys[off[j] + t] for the t-th selected row of column j (rows of one selection list)
__global__ void __launch_bounds__(256)
auc_key_kernel(const float* __restrict__ dec, int ldd, int col0, const int64_t* __restrict__ rows, int64_t n_rows,
               const int32_t* __restrict__ cols, int n_cols, const int64_t* __restrict__ off,
               const int32_t* __restrict__ ycls, const int32_t* __restrict__ pos,
               unsigned long long* __restrict__ keys) {
  const int jc = blockIdx.y;
  if (jc >= n_cols) return;
  const int j = cols[jc];                      // column index inside this block of columns
  const int p = pos[j];
  for (int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x; t < n_rows; t += (int64_t)gridDim.x * 256) {
    const int64_t r = rows[t];
    const float z = dec[r * ldd + col0 + j];
    const unsigned long long lab = (ycls[r] == p) ? 1ull : 0ull;
    keys[off[j] + t] = ((unsigned long long)j << 33) | ((unsigned long long)ordered_bits(z) << 1) | lab;
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

// out[j] = {2U, n_pos, n_neg} of the sorted segment of column j
__global__ void __launch_bounds__(256)
auc_count_kernel(const unsigned long long* __restrict__ keys, const int64_t* __restrict__ off, int B,
                 long long* __restrict__ out) {
  __shared__ long long s_cnt[256];
  __shared__ long long s_red[3][8];
  const int j = blockIdx.x;
  if (j >= B) return;
  const unsigned long long* a = keys + off[j];
  const int64_t len = off[j + 1] - off[j];
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
  long long neg_before = s_cnt[threadIdx.x] - negs;   // negatives in front of this thread's run
  long long sum_prefix = 0, sum_ties = 0, n_pos = 0;
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
      }
      sum_prefix += neg_before;
      sum_ties += last_ties;
      n_pos += 1;
    } else {
      neg_before += 1;
    }
  }
  long long v[3] = {2 * sum_prefix - sum_ties, n_pos, 0};
#pragma unroll
  for (int q = 0; q < 2; ++q) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[q] += __shfl_xor_sync(0xffffffffu, v[q], o);
    if ((threadIdx.x & 31) == 0) s_red[q][threadIdx.x >> 5] = v[q];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    long long u2 = 0, np = 0;
    for (int w = 0; w < 8; ++w) { u2 += s_red[0][w]; np += s_red[1][w]; }
    out[3 * j + 0] = u2;
    out[3 * j + 1] = np;
    out[3 * j + 2] = (long long)len - np;
  }
}

// col_fold: scoring codes of skd_linear_score_batch.  u2_out / n_pos_out / n_neg_out: [B].
int auc_batch(Ctx* c, int B, const float* coef, const int32_t* col_fold, const int32_t* col_pos,
              int64_t* u2_out, int64_t* n_pos_out, int64_t* n_neg_out) {
  const int64_t n = c->n, ldx = c->ldx;
  // row selection lists, one per distinct code
  std::vector<int32_t> codes(col_fold, col_fold + B);
  std::sort(codes.begin(), codes.end());
  codes.erase(std::unique(codes.begin(), codes.end()), codes.end());
  if (!c->h_fold.empty() && (int64_t)c->h_fold.size() != n) return fail(c, "skd_linear_auc_batch: fold ids out of date");
  std::vector<std::vector<int64_t>> lists(codes.size());
  for (size_t q = 0; q < codes.size(); ++q) {
    const int cd = codes[q];
    for (int64_t r = 0; r < n; ++r) {
      const int fd = c->h_fold.empty() ? -1 : (int)c->h_fold[r];
      if (score_code_selects(cd, fd)) lists[q].push_back(r);
    }
  }
  auto list_of = [&](int cd) { return (size_t)(std::lower_bound(codes.begin(), codes.end(), cd) - codes.begin()); };
  // blocks of columns: bound the decision matrix (n x cols fp32) and the keys (2 x 8 B per selected row)
  size_t max_rows = 1;
  for (auto& l : lists) max_rows = std::max(max_rows, l.size());
  int per = (int)std::max<double>(1.0, std::min(2.0e9 / (4.0 * (double)n), 3.0e9 / (16.0 * (double)max_rows)));
  per = std::min(per, 4096);                   // 12 bits of column id in the key
  for (int b0 = 0; b0 < B; b0 += per) {
    const int Bb = std::min(per, B - b0);
    Scratch sx(c);
    std::vector<int64_t> off(Bb + 1, 0);
    for (int j = 0; j < Bb; ++j) off[j + 1] = off[j] + (int64_t)lists[list_of(col_fold[b0 + j])].size();
    const int64_t total = off[Bb];
    float *dW, *dec;
    int64_t* doff;
    int32_t* dpos;
    unsigned long long *k0, *k1;
    long long* dout;
    if (pack_coef(c, sx, Bb, coef + (size_t)b0 * (c->d + 1), c->d, ldx, &dW)) return 1;
    SKD_CUDA(c, sx.alloc(&dec, (size_t)n * Bb));
    SKD_CUDA(c, sx.alloc(&doff, (size_t)Bb + 1));
    SKD_CUDA(c, sx.alloc(&dpos, (size_t)Bb));
    SKD_CUDA(c, sx.alloc(&k0, (size_t)std::max<int64_t>(total, 1)));
    SKD_CUDA(c, sx.alloc(&k1, (size_t)std::max<int64_t>(total, 1)));
    SKD_CUDA(c, sx.alloc(&dout, (size_t)3 * Bb));
    SKD_CUDA(c, cudaMemcpyAsync(doff, off.data(), off.size() * sizeof(int64_t), cudaMemcpyHostToDevice, c->stream));
    SKD_CUDA(c, cudaMemcpyAsync(dpos, col_pos + b0, Bb * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    if (simt_decision(c, Bb, dW, dec)) return 1;
    // keys, one launch per selection list (the columns that use it)
    std::vector<int64_t*> drows(codes.size(), nullptr);
    std::vector<int32_t*> dcols(codes.size(), nullptr);
    std::vector<std::vector<int32_t>> hcols(codes.size());
    for (int j = 0; j < Bb; ++j) hcols[list_of(col_fold[b0 + j])].push_back(j);
    for (size_t q = 0; q < codes.size(); ++q) {
      if (hcols[q].empty() || lists[q].empty()) continue;
      SKD_CUDA(c, sx.alloc(&drows[q], lists[q].size()));
      SKD_CUDA(c, sx.alloc(&dcols[q], hcols[q].size()));
      SKD_CUDA(c, cudaMemcpyAsync(drows[q], lists[q].data(), lists[q].size() * sizeof(int64_t), cudaMemcpyHostToDevice, c->stream));
      SKD_CUDA(c, cudaMemcpyAsync(dcols[q], hcols[q].data(), hcols[q].size() * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
      const int gx = (int)std::min<int64_t>(1024, ((int64_t)lists[q].size() + 255) / 256);
      for (size_t c0 = 0; c0 < hcols[q].size(); c0 += 65535) {
        const int nc = (int)std::min<size_t>(65535, hcols[q].size() - c0);
        auc_key_kernel<<<dim3(gx, nc), 256, 0, c->stream>>>(dec, Bb, 0, drows[q], (int64_t)lists[q].size(), dcols[q] + c0, nc,
                                                            doff, c->ycls, dpos, k0);
        c->launches += 1;
      }
    }
    SKD_CUDA(c, cudaGetLastError());
    const unsigned long long* sorted = k0;
    if (total > 0) {
      int col_bits = 1;
      while ((1 << col_bits) < Bb) ++col_bits;
      size_t tmp_bytes = 0;
      SKD_CUDA(c, cub::DeviceRadixSort::SortKeys(nullptr, tmp_bytes, k0, k1, total, 0, 33 + col_bits, c->stream));
      uint8_t* tmp;
      SKD_CUDA(c, sx.alloc(&tmp, tmp_bytes + 16));
      SKD_CUDA(c, cub::DeviceRadixSort::SortKeys(tmp, tmp_bytes, k0, k1, total, 0, 33 + col_bits, c->stream));
      c->launches += 1;
      sorted = k1;
    }
    auc_count_kernel<<<Bb, 256, 0, c->stream>>>(sorted, doff, Bb, dout);
    c->launches += 1;
    SKD_CUDA(c, cudaGetLastError());
    std::vector<long long> hout((size_t)3 * Bb);
    SKD_CUDA(c, cudaMemcpyAsync(hout.data(), dout, hout.size() * sizeof(long long), cudaMemcpyDeviceToHost, c->stream));
    SKD_CUDA(c, cudaStreamSynchronize(c->stream));
    c->d2h += (int64_t)hout.size() * 8;
    for (int j = 0; j < Bb; ++j) {
      u2_out[b0 + j] = hout[3 * j + 0];
      n_pos_out[b0 + j] = hout[3 * j + 1];
      n_neg_out[b0 + j] = hout[3 * j + 2];
    }
  }
  return 0;
}

}  // namespace skd
