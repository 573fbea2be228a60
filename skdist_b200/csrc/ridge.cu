// ridge.cu -- batched Ridge cross-validation: every (alpha, fold) column from ONE pass over X.
//
// Replaces, for all columns at once, what each reference task runs (ref search.py:230 ->
// Ridge.fit): centring (SK/linear_model/_base.py:189-199), A = Xc^T Xc and Xc^T yc by sgemm
// (SK/linear_model/_ridge.py:215-221), scipy.linalg.solve(assume_a="pos") (:223-234).
// The reference recomputes the same Gram matrix for every alpha and every fold; here
//       colsum / colmean         : global shifts mu = mean(X) and yg = mean(y) (with an intercept;
//                                  0 without), float64 slab partials added in slab order
//   K4  gram_kernel / xty_kernel : per-fold-block  S_f = X_f^T X_f,  v_f = X_f^T y_f,  s_f = sum x,
//                                  sum y, sum y^2  in one pass, all on x - mu and y - yg (rows visited
//                                  fold by fold through a permutation; fp32 products summed per block of
//                                  16 rows, fp32 over the blocks of a chunk of <= 2048 rows, float64
//                                  across chunks)
//       ridge_prepare_kernel     : training statistics of fold f = total - block f, centred in
//                                  float64:  A_f = S - n xbar xbar^T,  b_f = v - n xbar ybar; the
//                                  intercept's ybar gets yg back
//   K5  ridge_solve_kernel       : one CTA per (alpha, fold): A_f + alpha I -> fp32 Cholesky in
//                                  shared memory (packed lower triangle) -> two triangular solves
//                                  (the arithmetic class of LAPACK sposv)
// Scoring (K6) is the r2 epilogue of the evaluation kernels (logreg_simt.cu MODE_R2 / logreg_tc.cu TC_R2).
#include "skd_internal.h"

namespace skd {

constexpr int GR_T = 64;     // tile edge
constexpr int GR_K = 16;     // rows per inner step
constexpr int GR_CHUNK = 2048;

struct GramChunk {
  int64_t start;  // offset into perm
  int32_t len;
  int32_t fold;
};

// The packed Cholesky factor and the right-hand side of one column live in shared memory; the largest
// d whose buffer fits the 226 KB the solve kernel opts into is 338 (230 516 B; d = 339 needs 231 876 B).
constexpr size_t ridge_smem_bytes(int64_t d) { return ((size_t)d * (d + 1) / 2 + (size_t)d) * sizeof(float); }
constexpr int RIDGE_MAX_D = 338;
constexpr size_t RIDGE_SMEM_CAP = 226 * 1024;
static_assert(ridge_smem_bytes(RIDGE_MAX_D) <= RIDGE_SMEM_CAP && ridge_smem_bytes(RIDGE_MAX_D + 1) > RIDGE_SMEM_CAP,
              "RIDGE_MAX_D must be the largest d whose solve buffer fits RIDGE_SMEM_CAP");
constexpr int CS_SLAB = 4096;  // rows per column-sum partial

// Global column means of X and, in column d, the mean of y: float64 partials over 4096-row slabs,
// added in slab order by colmean_kernel (so mu and the target shift are the same on every run).
// All block statistics below are taken on x - mu and y - ybar_g, so that "S - n xbar xbar^T" and
// "v - n xbar ybar" never cancel leading digits on uncentred features or targets (the reference
// centres X and y before forming X^T X and X^T y, SK/linear_model/_base.py:196-199).
__global__ void colsum_kernel(const float* __restrict__ X, const float* __restrict__ y, int64_t n, int ldx, int d,
                              double* __restrict__ part /*[slab][d + 1]*/) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k > d) return;
  const int64_t r0 = (int64_t)blockIdx.y * CS_SLAB, r1 = r0 + CS_SLAB < n ? r0 + CS_SLAB : n;
  double a = 0.0;
  if (k < d)
    for (int64_t r = r0; r < r1; ++r) a += (double)X[r * ldx + k];
  else
    for (int64_t r = r0; r < r1; ++r) a += (double)y[r];
  part[(size_t)blockIdx.y * (d + 1) + k] = a;
}
// mu[0..ldx) = column means (0 on the padding), mu[ldx] = mean of y
__global__ void colmean_kernel(const double* __restrict__ part, int nslab, int64_t n, int d, int ldx,
                               float* __restrict__ mu) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k > ldx) return;
  if (k >= d && k < ldx) { mu[k] = 0.f; return; }
  const int col = k < d ? k : d;
  double a = 0.0;
  for (int s = 0; s < nslab; ++s) a += part[(size_t)s * (d + 1) + col];
  mu[k] = (float)(a / (double)n);
}

// Partial Gram of one chunk for one (ti <= tj) tile pair: Gp[(chunk * npairs + pair)][64][64]
__global__ void __launch_bounds__(256, 4)   // 64 registers: four CTAs per SM
gram_kernel(const float* __restrict__ X, int ldx, const float* __restrict__ mu,
            const int32_t* __restrict__ perm, const GramChunk* __restrict__ chunks, int ntile,
            float* __restrict__ Gp) {
  __shared__ float As[GR_K][GR_T + 4];
  __shared__ float Bs[GR_K][GR_T + 4];
  // pair index -> (ti, tj), ti <= tj
  int pair = blockIdx.x, ti = 0, rem = pair;
  while (rem >= ntile - ti) { rem -= ntile - ti; ++ti; }
  const int tj = ti + rem;
  const int npairs = ntile * (ntile + 1) / 2;
  const GramChunk ch = chunks[blockIdx.y];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int r0 = 0; r0 < ch.len; r0 += GR_K) {
    {
      int r = tid >> 4, q = (tid & 15) * 4;
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
      if (r0 + r < ch.len) {
        const float* row = X + (int64_t)perm[ch.start + r0 + r] * ldx;
        if (ti * GR_T + q < ldx) {
          a = *reinterpret_cast<const float4*>(row + ti * GR_T + q);
          const float4 m = *reinterpret_cast<const float4*>(mu + ti * GR_T + q);
          a.x -= m.x; a.y -= m.y; a.z -= m.z; a.w -= m.w;
        }
        if (tj * GR_T + q < ldx) {
          b = *reinterpret_cast<const float4*>(row + tj * GR_T + q);
          const float4 m = *reinterpret_cast<const float4*>(mu + tj * GR_T + q);
          b.x -= m.x; b.y -= m.y; b.z -= m.z; b.w -= m.w;
        }
      }
      *reinterpret_cast<float4*>(&As[r][q]) = a;
      *reinterpret_cast<float4*>(&Bs[r][q]) = b;
    }
    __syncthreads();
    // products of the 16 rows summed on their own, then added to the chunk sum: the fp32 rounding error
    // grows with 16 + len/16 additions instead of len (sequentially over 2048 rows it exceeds that of a
    // float32 GEMM and shows in the coefficients)
    float blk[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) blk[i][j] = 0.f;
#pragma unroll
    for (int k = 0; k < GR_K; ++k) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[k][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[k][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) blk[i][j] = fmaf(a[i], b[j], blk[i][j]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] += blk[i][j];
    __syncthreads();
  }
  float* out = Gp + ((size_t)blockIdx.y * npairs + pair) * (GR_T * GR_T);
#pragma unroll
  for (int i = 0; i < 4; ++i)
    *reinterpret_cast<float4*>(out + (ty * 4 + i) * GR_T + tx * 4) =
        make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
}

// (X - mu)^T (y - yg), sum (x - mu) per chunk (threads over features), sum (y - yg) / sum (y - yg)^2 per
// chunk.  yg = mu[ldx] is the global mean of y with an intercept and 0 without one: the fp32 products
// and chunk sums then carry the spread of y, not its offset.
__global__ void __launch_bounds__(256)
xty_kernel(const float* __restrict__ X, int ldx, int d, const float* __restrict__ mu,
           const float* __restrict__ y,
           const int32_t* __restrict__ perm, const GramChunk* __restrict__ chunks,
           float* __restrict__ vp /*[chunk][ldx]*/, float* __restrict__ sp /*[chunk][ldx]*/,
           double* __restrict__ yp /*[chunk][2]*/) {
  __shared__ double red[2][8];
  const GramChunk ch = chunks[blockIdx.x];
  const float yg = mu[ldx];
  for (int k0 = 0; k0 < ldx; k0 += 256) {
    const int k = k0 + threadIdx.x;
    float av = 0.f, as = 0.f;
    if (k < ldx) {
      for (int r0 = 0; r0 < ch.len; r0 += GR_K) {     // blocks of 16 rows, as gram_kernel
        const int r1 = r0 + GR_K < ch.len ? r0 + GR_K : ch.len;
        float bv = 0.f, bs = 0.f;
        for (int r = r0; r < r1; ++r) {
          const int32_t row = perm[ch.start + r];
          const float xv = X[(int64_t)row * ldx + k] - mu[k];
          bv = fmaf(xv, y[row] - yg, bv);
          bs += xv;
        }
        av += bv;
        as += bs;
      }
      vp[(size_t)blockIdx.x * ldx + k] = av;
      sp[(size_t)blockIdx.x * ldx + k] = as;
    }
  }
  double sy = 0.0, syy = 0.0;
  for (int r = threadIdx.x; r < ch.len; r += 256) {
    const double v = (double)(y[perm[ch.start + r]] - yg);
    sy += v;
    syy += v * v;
  }
  for (int o = 16; o > 0; o >>= 1) {
    sy += __shfl_xor_sync(0xffffffffu, sy, o);
    syy += __shfl_xor_sync(0xffffffffu, syy, o);
  }
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = sy; red[1][threadIdx.x >> 5] = syy; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0, b = 0.0;
    for (int i = 0; i < 8; ++i) { a += red[0][i]; b += red[1][i]; }
    yp[(size_t)blockIdx.x * 2] = a;
    yp[(size_t)blockIdx.x * 2 + 1] = b;
  }
}

// Per-fold block statistics in float64: S[f][dG x dG] (full symmetric), v[f][dG], s[f][dG],
// ys[f] = {sum y, sum y^2, count}
__global__ void gram_reduce_kernel(const float* __restrict__ Gp, const float* __restrict__ vp,
                                   const float* __restrict__ sp, const double* __restrict__ yp,
                                   const GramChunk* __restrict__ chunks, int nchunks, int ntile, int ldx,
                                   int n_folds, double* __restrict__ S, double* __restrict__ v,
                                   double* __restrict__ s, double* __restrict__ ys) {
  const int dG = ntile * GR_T;
  const int npairs = ntile * (ntile + 1) / 2;
  const int f = blockIdx.y;
  // Gram entries
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < (int64_t)npairs * GR_T * GR_T;
       e += (int64_t)gridDim.x * blockDim.x) {
    const int pair = (int)(e / (GR_T * GR_T)), within = (int)(e % (GR_T * GR_T));
    int ti = 0, rem = pair;
    while (rem >= ntile - ti) { rem -= ntile - ti; ++ti; }
    const int tj = ti + rem;
    double acc = 0.0;
    for (int c = 0; c < nchunks; ++c)
      if (chunks[c].fold == f) acc += (double)Gp[((size_t)c * npairs + pair) * (GR_T * GR_T) + within];
    const int r = ti * GR_T + within / GR_T, cc = tj * GR_T + within % GR_T;
    S[((size_t)f * dG + r) * dG + cc] = acc;
    S[((size_t)f * dG + cc) * dG + r] = acc;
  }
  if (blockIdx.x == 0) {
    for (int k = threadIdx.x; k < dG; k += blockDim.x) {
      double av = 0.0, as = 0.0;
      if (k < ldx)
        for (int c = 0; c < nchunks; ++c)
          if (chunks[c].fold == f) { av += (double)vp[(size_t)c * ldx + k]; as += (double)sp[(size_t)c * ldx + k]; }
      v[(size_t)f * dG + k] = av;
      s[(size_t)f * dG + k] = as;
    }
    if (threadIdx.x == 0) {
      double a = 0.0, b = 0.0, cnt = 0.0;
      for (int c = 0; c < nchunks; ++c)
        if (chunks[c].fold == f) { a += yp[(size_t)c * 2]; b += yp[(size_t)c * 2 + 1]; cnt += chunks[c].len; }
      ys[f * 3] = a; ys[f * 3 + 1] = b; ys[f * 3 + 2] = cnt;
    }
  }
  (void)n_folds;
}

// Training statistics for "hold out fold h" (h == n_folds: hold out nothing), centred.
// A[h][dG x dG] fp32, b[h][dG] fp32, xbar[h][dG] fp32, misc[h] = {ybar, n_train}.  The block sums are on
// y - yg; centring removes yg from b, and misc gets it back so that ybar is the mean of the original y.
__global__ void ridge_prepare_kernel(const double* __restrict__ S, const double* __restrict__ v,
                                     const double* __restrict__ s, const double* __restrict__ ys,
                                     const float* __restrict__ mu, int ldx,
                                     int n_folds, int dG, int fit_intercept, float* __restrict__ A,
                                     float* __restrict__ b, float* __restrict__ xbar,
                                     double* __restrict__ misc) {
  const int h = blockIdx.y;
  double ntr = 0.0, sy = 0.0;
  for (int f = 0; f < n_folds; ++f)
    if (f != h) { ntr += ys[f * 3 + 2]; sy += ys[f * 3]; }
  const double ybar = fit_intercept && ntr > 0 ? sy / ntr : 0.0;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < (int64_t)dG * dG;
       e += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(e / dG), c = (int)(e % dG);
    double acc = 0.0, sr = 0.0, sc = 0.0;
    for (int f = 0; f < n_folds; ++f)
      if (f != h) {
        acc += S[((size_t)f * dG + r) * dG + c];
        sr += s[(size_t)f * dG + r];
        sc += s[(size_t)f * dG + c];
      }
    if (fit_intercept && ntr > 0) acc -= sr * sc / ntr;   // S - n xbar xbar^T
    A[(size_t)h * dG * dG + e] = (float)acc;
    if (c == 0) {
      double vv = 0.0;
      for (int f = 0; f < n_folds; ++f)
        if (f != h) vv += v[(size_t)f * dG + r];
      if (fit_intercept && ntr > 0) vv -= sr * ybar;      // v - n xbar ybar
      b[(size_t)h * dG + r] = (float)vv;
      // statistics are on x - mu: the training mean in original coordinates is mu + mean(x - mu).
      // Without an intercept nothing may be shifted: the host passes mu == 0 in that case.
      xbar[(size_t)h * dG + r] = fit_intercept && ntr > 0 ? (float)((double)(r < ldx ? mu[r] : 0.f) + sr / ntr) : 0.f;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    misc[h * 2] = fit_intercept && ntr > 0 ? ybar + (double)mu[ldx] : 0.0;
    misc[h * 2 + 1] = ntr;
  }
}

// One CTA per column: fp32 Cholesky of (A_h + alpha I) on the packed lower triangle in shared
// memory, then L z = b, L^T w = z.  coef_out[col][0..d) weights, [d] intercept.
__global__ void __launch_bounds__(256)
ridge_solve_kernel(const float* __restrict__ A, const float* __restrict__ bvec,
                   const float* __restrict__ xbar, const double* __restrict__ misc, int dG, int d,
                   const double* __restrict__ alpha, const int32_t* __restrict__ col_hold,
                   int fit_intercept, float* __restrict__ coef_out, int32_t* __restrict__ status) {
  extern __shared__ float sm[];
  float* L = sm;                                   // packed lower: L[i*(i+1)/2 + j], j <= i
  float* w = sm + (size_t)d * (d + 1) / 2;         // d
  __shared__ float piv;
  __shared__ int bad;
  const int col = blockIdx.x, h = col_hold[col];
  const float al = (float)alpha[col];
  const float* Ah = A + (size_t)h * dG * dG;
  if (threadIdx.x == 0) bad = 0;
  for (int e = threadIdx.x; e < d * d; e += blockDim.x) {
    int i = e / d, j = e % d;
    if (j <= i) L[i * (i + 1) / 2 + j] = Ah[(size_t)i * dG + j] + (i == j ? al : 0.f);
  }
  for (int i = threadIdx.x; i < d; i += blockDim.x) w[i] = bvec[(size_t)h * dG + i];
  __syncthreads();
  // right-looking Cholesky
  for (int j = 0; j < d; ++j) {
    if (threadIdx.x == 0) {
      float p = L[j * (j + 1) / 2 + j];
      if (!(p > 0.f)) { bad = 1; p = 1.f; }
      piv = sqrtf(p);
      L[j * (j + 1) / 2 + j] = piv;
    }
    __syncthreads();
    const float inv = 1.f / piv;
    for (int i = j + 1 + threadIdx.x; i < d; i += blockDim.x) L[i * (i + 1) / 2 + j] *= inv;
    __syncthreads();
    // trailing update: for i > j, j < k <= i: L[i][k] -= L[i][j] * L[k][j]   (rows dealt cyclically)
    for (int i = j + 1 + threadIdx.x; i < d; i += blockDim.x) {
      const float lij = L[i * (i + 1) / 2 + j];
      float* Li = L + i * (i + 1) / 2;
      for (int k = j + 1; k <= i; ++k) Li[k] = fmaf(-lij, L[k * (k + 1) / 2 + j], Li[k]);
    }
    __syncthreads();
  }
  // forward substitution L z = b (column oriented), then L^T w = z
  for (int j = 0; j < d; ++j) {
    if (threadIdx.x == 0) w[j] /= L[j * (j + 1) / 2 + j];
    __syncthreads();
    const float zj = w[j];
    for (int i = j + 1 + threadIdx.x; i < d; i += blockDim.x) w[i] = fmaf(-L[i * (i + 1) / 2 + j], zj, w[i]);
    __syncthreads();
  }
  for (int j = d - 1; j >= 0; --j) {
    if (threadIdx.x == 0) w[j] /= L[j * (j + 1) / 2 + j];
    __syncthreads();
    const float wj = w[j];
    for (int i = threadIdx.x; i < j; i += blockDim.x) w[i] = fmaf(-L[j * (j + 1) / 2 + i], wj, w[i]);
    __syncthreads();
  }
  // intercept = ybar - xbar . w   (SK/linear_model/_base.py _set_intercept)
  __shared__ float red[8];
  float part = 0.f;
  for (int i = threadIdx.x; i < d; i += blockDim.x) {
    coef_out[(size_t)col * (d + 1) + i] = w[i];
    part = fmaf(xbar[(size_t)h * dG + i], w[i], part);
  }
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = part;
  __syncthreads();
  if (threadIdx.x == 0) {
    float dot = 0.f;
    for (int i = 0; i < 8; ++i) dot += red[i];
    coef_out[(size_t)col * (d + 1) + d] = fit_intercept ? (float)misc[h * 2] - dot : 0.f;
    status[col] = bad ? 4 : 1;
  }
}

// Host driver.  hold[j] in [0, n_folds) = held-out fold of column j, or n_folds for "none".
int ridge_fit_batch(Ctx* c, int B, const double* alpha, const int32_t* hold, int fit_intercept,
                    float* coef_out, int32_t* status_out) {
  const int64_t n = c->n;
  const int d = (int)c->d, ldx = (int)c->ldx;
  if (!c->yreal) return fail(c, "ridge: stage real-valued targets first (skd_stage_targets)");
  const int ntile = (d + GR_T - 1) / GR_T, dG = ntile * GR_T;
  if (d > RIDGE_MAX_D) return fail(c, "ridge: device path supports d <= 338 (Cholesky in shared memory)");
  const size_t smem = ridge_smem_bytes(d);
  const int n_folds = c->fold ? c->n_folds : 1;
  // host: permutation of rows by fold + chunk table (chunks never straddle a fold)
  std::vector<int8_t> hfold;
  if (c->fold) {
    hfold.resize(n);
    SKD_CUDA(c, cudaMemcpy(hfold.data(), c->fold, (size_t)n, cudaMemcpyDeviceToHost));
  }
  std::vector<int64_t> cnt(n_folds, 0), off(n_folds + 1, 0);
  for (int64_t i = 0; i < n; ++i) cnt[c->fold ? hfold[i] : 0]++;
  for (int f = 0; f < n_folds; ++f) off[f + 1] = off[f] + cnt[f];
  std::vector<int32_t> perm(n);
  {
    std::vector<int64_t> pos(off.begin(), off.end() - 1);
    for (int64_t i = 0; i < n; ++i) perm[pos[c->fold ? hfold[i] : 0]++] = (int32_t)i;
  }
  std::vector<GramChunk> chunks;
  for (int f = 0; f < n_folds; ++f)
    for (int64_t s0 = off[f]; s0 < off[f + 1]; s0 += GR_CHUNK)
      chunks.push_back({s0, (int32_t)std::min<int64_t>(GR_CHUNK, off[f + 1] - s0), f});
  const int nchunks = (int)chunks.size(), npairs = ntile * (ntile + 1) / 2;

  Scratch sx(c);
  int32_t* dperm; GramChunk* dchunks; float *Gp, *vp, *sp; double* yp;
  double *S, *v, *s, *ys, *misc; float *A, *bv, *xbar;
  double* dalpha; int32_t* dhold; float* dcoef; int32_t* dstatus;
  // mu[0..ldx): feature shift, mu[ldx]: target shift; all zero without an intercept
  double* colpart; float* mu;
  const int nslab = (int)((n + CS_SLAB - 1) / CS_SLAB);
  SKD_CUDA(c, sx.alloc(&mu, (size_t)ldx + 1));
  SKD_CUDA(c, cudaMemsetAsync(mu, 0, ((size_t)ldx + 1) * sizeof(float), c->stream));
  if (fit_intercept) {
    SKD_CUDA(c, sx.alloc(&colpart, (size_t)nslab * (d + 1)));
    colsum_kernel<<<dim3((d + 1 + 127) / 128, (unsigned)nslab), 128, 0, c->stream>>>(c->X, c->yreal, n, ldx, d, colpart);
    colmean_kernel<<<(ldx + 1 + 127) / 128, 128, 0, c->stream>>>(colpart, nslab, n, d, ldx, mu);
    c->launches += 2;
  }
  SKD_CUDA(c, sx.alloc(&dperm, (size_t)n));
  SKD_CUDA(c, sx.alloc(&dchunks, (size_t)nchunks));
  SKD_CUDA(c, sx.alloc(&Gp, (size_t)nchunks * npairs * GR_T * GR_T));
  SKD_CUDA(c, sx.alloc(&vp, (size_t)nchunks * ldx));
  SKD_CUDA(c, sx.alloc(&sp, (size_t)nchunks * ldx));
  SKD_CUDA(c, sx.alloc(&yp, (size_t)nchunks * 2));
  SKD_CUDA(c, sx.alloc(&S, (size_t)n_folds * dG * dG));
  SKD_CUDA(c, sx.alloc(&v, (size_t)n_folds * dG));
  SKD_CUDA(c, sx.alloc(&s, (size_t)n_folds * dG));
  SKD_CUDA(c, sx.alloc(&ys, (size_t)n_folds * 3));
  SKD_CUDA(c, sx.alloc(&A, (size_t)(n_folds + 1) * dG * dG));
  SKD_CUDA(c, sx.alloc(&bv, (size_t)(n_folds + 1) * dG));
  SKD_CUDA(c, sx.alloc(&xbar, (size_t)(n_folds + 1) * dG));
  SKD_CUDA(c, sx.alloc(&misc, (size_t)(n_folds + 1) * 2));
  SKD_CUDA(c, sx.alloc(&dalpha, (size_t)B));
  SKD_CUDA(c, sx.alloc(&dhold, (size_t)B));
  SKD_CUDA(c, sx.alloc(&dcoef, (size_t)B * (d + 1)));
  SKD_CUDA(c, sx.alloc(&dstatus, (size_t)B));
  SKD_CUDA(c, cudaMemcpyAsync(dperm, perm.data(), (size_t)n * 4, cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(dchunks, chunks.data(), (size_t)nchunks * sizeof(GramChunk), cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(dalpha, alpha, (size_t)B * 8, cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(dhold, hold, (size_t)B * 4, cudaMemcpyHostToDevice, c->stream));
  c->h2d += n * 4 + (int64_t)B * 12;

  gram_kernel<<<dim3(npairs, nchunks), 256, 0, c->stream>>>(c->X, ldx, mu, dperm, dchunks, ntile, Gp);
  xty_kernel<<<nchunks, 256, 0, c->stream>>>(c->X, ldx, d, mu, c->yreal, dperm, dchunks, vp, sp, yp);
  gram_reduce_kernel<<<dim3(64, n_folds), 256, 0, c->stream>>>(Gp, vp, sp, yp, dchunks, nchunks, ntile, ldx,
                                                              n_folds, S, v, s, ys);
  ridge_prepare_kernel<<<dim3(64, n_folds + 1), 256, 0, c->stream>>>(S, v, s, ys, mu, ldx, n_folds, dG, fit_intercept,
                                                                    A, bv, xbar, misc);
  static size_t attr_bytes = 0;
  if (smem > attr_bytes) {
    SKD_CUDA(c, cudaFuncSetAttribute(ridge_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_bytes = smem;
  }
  ridge_solve_kernel<<<B, 256, smem, c->stream>>>(A, bv, xbar, misc, dG, d, dalpha, dhold, fit_intercept,
                                                  dcoef, dstatus);
  c->launches += 5;
  SKD_CUDA(c, cudaGetLastError());
  SKD_CUDA(c, cudaMemcpyAsync(coef_out, dcoef, (size_t)B * (d + 1) * 4, cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(status_out, dstatus, (size_t)B * 4, cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  c->d2h += (int64_t)B * (d + 2) * 4;
  return 0;
}

}  // namespace skd
