// predict.cu -- streaming batched linear inference  out[i, j] = x_i . coef_j + intercept_j.
//
// Replaces the per-Arrow-batch `model.predict(vals)` that the reference wraps in a Spark
// pandas_udf (ref skdist/distribute/predict.py:160-179; _get_vals transposes the column batch,
// :59-71).  HBM-bound: 4*d bytes read per row for 2*d*B FLOPs, so one warp per row with float4
// loads; up to 8 models share one pass over the rows.
#include "skd_internal.h"

namespace skd {

constexpr size_t PREDICT_CACHE_BYTES = 48 * 1024;   // shared-memory weight cache of predict_kernel

// CACHED: the NB weight rows are copied to shared memory once per CTA; otherwise (rows wider than the
// cache) every warp reads them from global memory, where they stay L2-resident.
template <int NB, bool CACHED>
__global__ void __launch_bounds__(256)
predict_kernel(const float* __restrict__ X, int64_t m, int ldx, int d, const float* __restrict__ W /*[NB][ldx]*/,
               const float* __restrict__ bias, float* __restrict__ out, int ldo, int col0) {
  extern __shared__ float sw[];   // NB * ldx
  if (CACHED) {
    for (int i = threadIdx.x; i < NB * ldx; i += blockDim.x) sw[i] = W[i];
    __syncthreads();
  }
  const float* wsrc = CACHED ? sw : W;
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int64_t r = (int64_t)blockIdx.x * wpb + (threadIdx.x >> 5); r < m; r += (int64_t)gridDim.x * wpb) {
    const float4* row = reinterpret_cast<const float4*>(X + r * ldx);
    float acc[NB];
#pragma unroll
    for (int b = 0; b < NB; ++b) acc[b] = 0.f;
    for (int q = lane; q < ldx / 4; q += 32) {
      const float4 x = __ldg(row + q);
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        const float4* wp = reinterpret_cast<const float4*>(wsrc + b * ldx + q * 4);
        const float4 w = CACHED ? *wp : __ldg(wp);
        acc[b] = fmaf(x.x, w.x, fmaf(x.y, w.y, fmaf(x.z, w.z, fmaf(x.w, w.w, acc[b]))));
      }
    }
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      float v = acc[b];
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) out[r * ldo + col0 + b] = v + bias[b];
    }
  }
  (void)d;
}

int predict_cache_rows(int64_t ldx) {
  return (int)std::min<int64_t>(8, (int64_t)PREDICT_CACHE_BYTES / (ldx * (int64_t)sizeof(float)));
}

template <bool CACHED>
static void predict_launch(Ctx* c, int nb, const float* dX, int64_t m, int ldx, int d, const float* w,
                           const float* bias, float* dout, int B, int b0) {
  const int grid = c->sm_count * 8;
  const size_t smem = CACHED ? (size_t)nb * ldx * sizeof(float) : 0;
  switch (nb) {
    case 8: predict_kernel<8, CACHED><<<grid, 256, smem, c->stream>>>(dX, m, ldx, d, w, bias, dout, B, b0); break;
    case 4: predict_kernel<4, CACHED><<<grid, 256, smem, c->stream>>>(dX, m, ldx, d, w, bias, dout, B, b0); break;
    case 2: predict_kernel<2, CACHED><<<grid, 256, smem, c->stream>>>(dX, m, ldx, d, w, bias, dout, B, b0); break;
    default: predict_kernel<1, CACHED><<<grid, 256, smem, c->stream>>>(dX, m, ldx, d, w, bias, dout, B, b0); break;
  }
}

// dX: [m x ldx] device rows (ldx % 4 == 0, zero padded), dW: [B x ldx] + bias[B] packed as in
// pack_coef (weights then bias block), dout: [m x B].  Each pass takes the largest of 8/4/2/1 models
// that are left and fit the weight cache; rows wider than the cache run uncached, up to 8 models a pass.
int predict_device(Ctx* c, const float* dX, int64_t m, int ldx, int d, int B, const float* dW, float* dout) {
  if (m <= 0) return 0;
  const int cache_rows = predict_cache_rows(ldx);
  for (int b0 = 0; b0 < B;) {
    const int cap = std::min(B - b0, cache_rows > 0 ? cache_rows : 8);
    const int nb = cap >= 8 ? 8 : (cap >= 4 ? 4 : (cap >= 2 ? 2 : 1));
    const float* w = dW + (size_t)b0 * ldx;
    const float* bias = dW + (size_t)B * ldx + b0;
    if (cache_rows > 0) predict_launch<true>(c, nb, dX, m, ldx, d, w, bias, dout, B, b0);
    else predict_launch<false>(c, nb, dX, m, ldx, d, w, bias, dout, B, b0);
    c->launches += 1;
    b0 += nb;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(c, std::string("predict launch: ") + cudaGetErrorString(e));
  return 0;
}

// ---- forest inference ----------------------------------------------------------------------
// One thread per row walks every tree from its root (children_left == -1 marks a leaf) and adds
// the leaf's class fractions in tree order (float64).  The walk is a chain of dependent loads of
// 16-byte node records; rows are independent, so thousands of walks are in flight per SM and the
// top levels of every tree stay in L2.
struct __align__(16) FNode {
  int32_t left, right, feature, pad;
};

template <int CMAX>
__global__ void __launch_bounds__(256)
forest_predict_kernel(const float* __restrict__ X, int64_t m, int ldx, int n_trees,
                      const int64_t* __restrict__ tree_offset, const FNode* __restrict__ node,
                      const double* __restrict__ threshold, const double* __restrict__ value, int C,
                      double* __restrict__ out) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= m) return;
  const float* x = X + r * ldx;
  double acc[CMAX > 0 ? CMAX : 1];
#pragma unroll
  for (int c = 0; c < CMAX; ++c) acc[c] = 0.0;
  for (int t = 0; t < n_trees; ++t) {
    const int64_t base = tree_offset[t];
    int64_t k = base;
    FNode nd = node[k];
    while (nd.left != -1) {
      const double v = (double)__ldg(x + nd.feature);
      k = base + (v <= threshold[k] ? nd.left : nd.right);
      nd = node[k];
    }
    const double* val = value + k * C;
    if (CMAX > 0) {
#pragma unroll
      for (int c = 0; c < CMAX; ++c)
        if (c < C) acc[c] += val[c];
    } else {
      for (int c = 0; c < C; ++c) out[r * C + c] += val[c];   // many classes: accumulate in place (zeroed by the host)
    }
  }
  if (CMAX > 0) {
    const double inv = (double)n_trees;
#pragma unroll
    for (int c = 0; c < CMAX; ++c)
      if (c < C) out[r * C + c] = acc[c] / inv;
  } else {
    for (int c = 0; c < C; ++c) out[r * C + c] /= (double)n_trees;
  }
}

int forest_predict_device(Ctx* c, const float* dX, int64_t m, int ldx, int n_trees, const int64_t* d_off,
                          const void* d_node, const double* d_thr, const double* d_val, int C, double* d_out) {
  if (m <= 0) return 0;
  const unsigned grid = (unsigned)((m + 255) / 256);
  const FNode* nd = (const FNode*)d_node;
  if (C <= 2) forest_predict_kernel<2><<<grid, 256, 0, c->stream>>>(dX, m, ldx, n_trees, d_off, nd, d_thr, d_val, C, d_out);
  else if (C <= 8) forest_predict_kernel<8><<<grid, 256, 0, c->stream>>>(dX, m, ldx, n_trees, d_off, nd, d_thr, d_val, C, d_out);
  else if (C <= 32) forest_predict_kernel<32><<<grid, 256, 0, c->stream>>>(dX, m, ldx, n_trees, d_off, nd, d_thr, d_val, C, d_out);
  else {
    cudaMemsetAsync(d_out, 0, (size_t)m * C * sizeof(double), c->stream);
    forest_predict_kernel<0><<<grid, 256, 0, c->stream>>>(dX, m, ldx, n_trees, d_off, nd, d_thr, d_val, C, d_out);
  }
  c->launches += 1;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(c, std::string("forest predict launch: ") + cudaGetErrorString(e));
  return 0;
}

}  // namespace skd
