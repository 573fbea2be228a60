// logreg_simt.cu -- fp32 CUDA-core evaluation of the batched logistic objective.
//
// General-shape path (any d, any B) and the accuracy reference for the tensor-core path.
// Replaces, per L-BFGS evaluation and for all active columns at once,
//   SK/linear_model/_linear_loss.py:291-379  LinearModelLoss.loss_gradient
//     raw = X @ w32 + b32                         (:219)   -> fwd_kernel K-loop (fp32 FMA)
//     closs_grad_half_binomial in double          (SK/_loss/_loss.pyx.tp:728-751) -> epilogue
//     X.T @ grad_pointwise                        (:356)   -> bwd_kernel (fp32 FMA)
//     sum(grad_pointwise)                         (:361)   -> gsump
// and the scorer's decision_function / accuracy (ref search.py:264).
//
// Layout: X [n x ldx] fp32 row-major, ldx = d rounded up to 16 (zero padded);
// W of the active slots [n_act x ldx] (zero padded) + bias[n_act]; G [n x ldg].
// Partials are written per row chunk z and summed in a fixed order by the consumer, so a
// run is bit-reproducible.
#include "skd_internal.h"

namespace skd {

constexpr int TM = 64;   // rows per tile
constexpr int TN = 64;   // slots per tile
constexpr int TK = 16;

enum { MODE_FIT = 0, MODE_SCORE = 1, MODE_DECISION = 2, MODE_R2 = 3 };

// sklearn's closs_grad_half_binomial (SK/_loss/_loss.pyx.tp:728-751), evaluated in double.
__device__ __forceinline__ void loss_grad_half_binomial(double y, double raw, double& loss,
                                                        double& grad) {
  if (raw <= -37.0) {
    double e = exp(raw);
    loss = e - y * raw;
    grad = e - y;
  } else if (raw <= -2.0) {
    double e = exp(raw);
    loss = log1p(e) - y * raw;
    grad = ((1.0 - y) * e - y) / (1.0 + e);
  } else if (raw <= 18.0) {
    double e = exp(-raw);
    loss = log1p(e) + (1.0 - y) * raw;
    grad = ((1.0 - y) - y * e) / (1.0 + e);
  } else {
    double e = exp(-raw);
    loss = e + (1.0 - y) * raw;
    grad = ((1.0 - y) - y * e) / (1.0 + e);
  }
}

template <int MODE>
__global__ void __launch_bounds__(256)
fwd_kernel(const float* __restrict__ X, int64_t n, int ldx, const float* __restrict__ W,
           const float* __restrict__ bias, const SlotMeta* __restrict__ slot, int n_act,
           const int32_t* __restrict__ ycls, const int8_t* __restrict__ fold,
           int64_t rows_per_chunk, float* __restrict__ G, int ldg, double* __restrict__ lossp,
           double* __restrict__ gsump, int64_t* __restrict__ correct, int64_t* __restrict__ count,
           float* __restrict__ dec, int ldd, const float* __restrict__ yreal,
           const uint32_t* __restrict__ ybits = nullptr, const uint32_t* __restrict__ mbits = nullptr,
           long long rb_words = 0, const float2* __restrict__ cw = nullptr,
           const float* __restrict__ roww = nullptr) {
  __shared__ float As[TK][TM + 4];
  __shared__ float Bs[TK][TN + 4];
  __shared__ double red[16][TN + 1];

  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int s0 = blockIdx.x * TN;
  const int z = blockIdx.y;
  const int64_t row_begin = (int64_t)z * rows_per_chunk;
  int64_t row_end = row_begin + rows_per_chunk;
  if (row_end > n) row_end = n;

  // per-thread slot metadata for its 4 slots
  int sfold[4], spos[4], sneg1[4], scol[4];
  float sb[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    int s = s0 + tx * 4 + j;
    sfold[j] = -100; spos[j] = -100; sneg1[j] = 0; sb[j] = 0.f; scol[j] = 0;
    if (s < n_act) {
      sb[j] = bias[s];
      if (MODE != MODE_DECISION) { sfold[j] = slot[s].fold; spos[j] = slot[s].pos; sneg1[j] = slot[s].pad; scol[j] = slot[s].col; }
    }
  }
  double acc_loss[4] = {0, 0, 0, 0}, acc_g[4] = {0, 0, 0, 0};
  long long acc_c[4] = {0, 0, 0, 0}, acc_n[4] = {0, 0, 0, 0};

  for (int64_t r0 = row_begin; r0 < row_end; r0 += TM) {
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int k0 = 0; k0 < ldx; k0 += TK) {
      {  // A tile: 64 rows x 16 k, one float4 per thread
        int r = tid >> 2, kq = (tid & 3) * 4;
        int64_t gr = r0 + r;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (gr < row_end) v = *reinterpret_cast<const float4*>(X + gr * ldx + k0 + kq);
        As[kq + 0][r] = v.x; As[kq + 1][r] = v.y; As[kq + 2][r] = v.z; As[kq + 3][r] = v.w;
        int s = s0 + r;
        float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
        if (s < n_act) w = *reinterpret_cast<const float4*>(W + (int64_t)s * ldx + k0 + kq);
        Bs[kq + 0][r] = w.x; Bs[kq + 1][r] = w.y; Bs[kq + 2][r] = w.z; Bs[kq + 3][r] = w.w;
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < TK; ++k) {
        float a[4], b[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = As[k][ty * 4 + i];
#pragma unroll
        for (int j = 0; j < 4; ++j) b[j] = Bs[k][tx * 4 + j];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
      __syncthreads();
    }
    // epilogue
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int64_t gr = r0 + ty * 4 + i;
      bool rvalid = gr < row_end;
      int yc = -1, fd = -1;
      float yr = 0.f;
      if (MODE != MODE_DECISION && rvalid) {
        if (MODE == MODE_R2) yr = yreal[gr];
        else yc = ycls[gr];
        if (fold) fd = (int)fold[gr];
      }
      float gout[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float raw = acc[i][j] + sb[j];
        gout[j] = 0.f;
        if (MODE == MODE_FIT) {
          bool train = rvalid && (fd != sfold[j] || sfold[j] < 0) && sfold[j] != -100 &&
                       (sneg1[j] == 0 || yc == spos[j] || yc == sneg1[j] - 1);   // one-vs-one: only the pair's rows
          bool ypos = yc == spos[j];
          if (train && (ybits || mbits) && scol[j] >= 0) {    // staged row bit matrices (multilabel targets, sampled negatives)
            const size_t wi = (size_t)scol[j] * rb_words + (size_t)(gr >> 5);
            const unsigned sh = (unsigned)(gr & 31);
            if (mbits) train = (mbits[wi] >> sh) & 1u;
            if (ybits) ypos = (ybits[wi] >> sh) & 1u;
          }
          if (train) {
            double y = ypos ? 1.0 : 0.0;
            double l, g;
            loss_grad_half_binomial(y, (double)raw, l, g);
            if (cw) {   // the row's weight times the double results (SK/_loss/_loss.pyx.tp:1083-1084): its class
                        // weight times its sample weight, a float32 product as SK/linear_model/_logistic.py:436 forms it
              const float2 wc = cw[scol[j]];
              const float cwl = ypos ? wc.y : wc.x;
              const double sw = (double)(roww ? cwl * roww[gr] : cwl);
              l *= sw;
              g *= sw;
            }
            float lf = (float)l, gf = (float)g;   // sklearn stores both as float32
            acc_loss[j] += (double)lf;
            acc_g[j] += (double)gf;
            gout[j] = gf;
          }
        } else if (MODE == MODE_SCORE) {
          bool test = rvalid && sfold[j] != -100 && score_code_selects(sfold[j], fd);
          if (test) {
            bool pred = raw > 0.f;
            bool y = (yc == spos[j]);
            acc_c[j] += (pred == y) ? 1 : 0;
            acc_n[j] += 1;
          }
        } else if (MODE == MODE_R2) {
          bool test = rvalid && sfold[j] != -100 && score_code_selects(sfold[j], fd);
          if (test) {
            double r = (double)yr - (double)raw;
            acc_loss[j] += r * r;
            acc_n[j] += 1;
          }
        } else {
          gout[j] = raw;
        }
      }
      if (MODE == MODE_FIT && rvalid) {
        *reinterpret_cast<float4*>(G + gr * ldg + s0 + tx * 4) =
            make_float4(gout[0], gout[1], gout[2], gout[3]);
      }
      if (MODE == MODE_DECISION && rvalid) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          int s = s0 + tx * 4 + j;
          if (s < n_act) dec[gr * ldd + s] = gout[j];
        }
      }
    }
  }
  if (MODE == MODE_DECISION) return;
  // reduce the per-thread accumulators over ty (16 threads share a slot quadruple)
  for (int pass = 0; pass < 2; ++pass) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      double v;
      if (MODE == MODE_FIT) v = pass == 0 ? acc_loss[j] : acc_g[j];
      else if (MODE == MODE_R2) v = pass == 0 ? acc_loss[j] : (double)acc_n[j];
      else v = pass == 0 ? (double)acc_c[j] : (double)acc_n[j];
      red[ty][tx * 4 + j] = v;
    }
    __syncthreads();
    if (tid < TN) {
      double sum = 0.0;
#pragma unroll
      for (int t = 0; t < 16; ++t) sum += red[t][tid];
      int s = s0 + tid;
      if (s < n_act) {
        if (MODE == MODE_FIT) {
          if (pass == 0) lossp[(int64_t)z * n_act + s] = sum;
          else gsump[(int64_t)z * n_act + s] = sum;
        } else if (MODE == MODE_R2) {
          if (pass == 0) atomicAdd(&lossp[s], sum);      // sum of squared residuals per slot
          else atomicAdd((unsigned long long*)&count[s], (unsigned long long)(sum + 0.5));
        } else {
          if (pass == 0) atomicAdd((unsigned long long*)&correct[s], (unsigned long long)(sum + 0.5));
          else atomicAdd((unsigned long long*)&count[s], (unsigned long long)(sum + 0.5));
        }
      }
    }
    __syncthreads();
  }
}

// gradp[z][s][k] = sum_{i in chunk z} G[i][s] * X[i][k]
__global__ void __launch_bounds__(256)
bwd_kernel(const float* __restrict__ X, int64_t n, int ldx, const float* __restrict__ G, int ldg,
           int n_act, int64_t rows_per_chunk, float* __restrict__ gradp) {
  __shared__ float Gs[TK][TN + 4];
  __shared__ float Xs[TK][TM + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;  // tx -> k quad, ty -> slot quad
  const int k0 = blockIdx.x * 64;
  const int s0 = blockIdx.y * TN;
  const int z = blockIdx.z;
  const int64_t row_begin = (int64_t)z * rows_per_chunk;
  int64_t row_end = row_begin + rows_per_chunk;
  if (row_end > n) row_end = n;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int64_t r0 = row_begin; r0 < row_end; r0 += TK) {
    {
      int r = tid >> 4, q = (tid & 15) * 4;  // 16 rows x 64 cols, float4 each
      int64_t gr = r0 + r;
      float4 g = make_float4(0.f, 0.f, 0.f, 0.f), x = make_float4(0.f, 0.f, 0.f, 0.f);
      if (gr < row_end) {
        g = *reinterpret_cast<const float4*>(G + gr * ldg + s0 + q);
        if (k0 + q < ldx) x = *reinterpret_cast<const float4*>(X + gr * ldx + k0 + q);
      }
      *reinterpret_cast<float4*>(&Gs[r][q]) = g;
      *reinterpret_cast<float4*>(&Xs[r][q]) = x;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < TK; ++k) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = Gs[k][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Xs[k][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int s = s0 + ty * 4 + i;
    if (s >= n_act) continue;
    int k = k0 + tx * 4;
    if (k < ldx) {
      *reinterpret_cast<float4*>(gradp + ((int64_t)z * n_act + s) * ldx + k) =
          make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
    }
  }
}

static void pick_chunks(Ctx* c, int64_t n, int n_act, int max_nz, int* nz, int64_t* rows_per_chunk) {
  int ctiles = (n_act + TN - 1) / TN;
  int want = (4 * c->sm_count + ctiles - 1) / ctiles;
  if (want < 1) want = 1;
  if (want > max_nz) want = max_nz;
  int64_t rpc = (n + want - 1) / want;
  rpc = ((rpc + TM - 1) / TM) * TM;
  if (rpc < TM) rpc = TM;
  *nz = (int)((n + rpc - 1) / rpc);
  *rows_per_chunk = rpc;
}

int simt_eval(Ctx* c, LogregWork& w, int n_act, int* nz_used) {
  *nz_used = 0;
  if (n_act <= 0) return 0;
  int nz;
  int64_t rpc;
  pick_chunks(c, c->n, n_act, w.lb.nz, &nz, &rpc);
  const int ldx = (int)c->ldx;
  // SlotMeta / W are indexed by slot; G uses ldg columns.  Process slot ranges so that the
  // grid covers [0, n_act).
  dim3 gf((n_act + TN - 1) / TN, nz);
  fwd_kernel<MODE_FIT><<<gf, 256, 0, c->stream>>>(
      c->X, c->n, ldx, w.lb.W, w.lb.W + (size_t)w.lb.B * ldx /*bias block*/, w.lb.slot, n_act, c->ycls,
      c->fold, rpc, w.G, w.ldg, w.lb.lossp, w.lb.gsump, nullptr, nullptr, nullptr, 0, nullptr, w.ybits, w.mbits,
      (long long)w.rb_words, w.cw, w.cw ? w.roww : nullptr);
  dim3 gb((ldx + 63) / 64, (n_act + TN - 1) / TN, nz);
  bwd_kernel<<<gb, 256, 0, c->stream>>>(c->X, c->n, ldx, w.G, w.ldg, n_act, rpc, w.lb.gradp);
  c->launches += 2;
  *nz_used = nz;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(c, std::string("simt_eval launch: ") + cudaGetErrorString(e));
  return 0;
}

int simt_score(Ctx* c, int B, const float* dW, const SlotMeta* dslot, int64_t* dcorrect,
               int64_t* dcount) {
  int nz;
  int64_t rpc;
  pick_chunks(c, c->n, B, 4096, &nz, &rpc);
  const int ldx = (int)c->ldx;
  dim3 g((B + TN - 1) / TN, nz);
  fwd_kernel<MODE_SCORE><<<g, 256, 0, c->stream>>>(
      c->X, c->n, ldx, dW, dW + (size_t)B * ldx, dslot, B, c->ycls, c->fold, rpc, nullptr, 0,
      nullptr, nullptr, dcorrect, dcount, nullptr, 0, nullptr);
  c->launches += 1;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(c, std::string("simt_score launch: ") + cudaGetErrorString(e));
  return 0;
}

// sum of squared residuals and row counts per slot (regression scoring; fold codes as simt_score)
int simt_r2(Ctx* c, int B, const float* dW, const SlotMeta* dslot, double* dsse, int64_t* dcount) {
  int nz;
  int64_t rpc;
  pick_chunks(c, c->n, B, 4096, &nz, &rpc);
  const int ldx = (int)c->ldx;
  dim3 g((B + TN - 1) / TN, nz);
  fwd_kernel<MODE_R2><<<g, 256, 0, c->stream>>>(
      c->X, c->n, ldx, dW, dW + (size_t)B * ldx, dslot, B, nullptr, c->fold, rpc, nullptr, 0, dsse,
      nullptr, nullptr, dcount, nullptr, 0, c->yreal);
  c->launches += 1;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(c, std::string("simt_r2 launch: ") + cudaGetErrorString(e));
  return 0;
}

int simt_decision(Ctx* c, int B, const float* dW, float* dout) {
  int nz;
  int64_t rpc;
  pick_chunks(c, c->n, B, 4096, &nz, &rpc);
  const int ldx = (int)c->ldx;
  dim3 g((B + TN - 1) / TN, nz);
  // slot metadata is unused in decision mode except for bounds; pass a dummy pointer-safe array
  fwd_kernel<MODE_DECISION><<<g, 256, 0, c->stream>>>(
      c->X, c->n, ldx, dW, dW + (size_t)B * ldx, nullptr, B, c->ycls, c->fold, rpc, nullptr, 0,
      nullptr, nullptr, nullptr, nullptr, dout, B, nullptr);
  c->launches += 1;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(c, std::string("simt_decision launch: ") + cudaGetErrorString(e));
  return 0;
}

// Z = X W^T + b for an arbitrary slot matrix (multinomial path: K slots per candidate)
int simt_raw_prediction(Ctx* c, int n_slots, const float* dW, const float* dbias, float* dout, int ldd) {
  int nz;
  int64_t rpc;
  pick_chunks(c, c->n, n_slots, 4096, &nz, &rpc);
  dim3 g((n_slots + TN - 1) / TN, nz);
  fwd_kernel<MODE_DECISION><<<g, 256, 0, c->stream>>>(
      c->X, c->n, (int)c->ldx, dW, dbias, nullptr, n_slots, c->ycls, c->fold, rpc, nullptr, 0,
      nullptr, nullptr, nullptr, nullptr, dout, ldd, nullptr);
  c->launches += 1;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(c, std::string("simt_raw_prediction launch: ") + cudaGetErrorString(e));
  return 0;
}

// gradp[z][slot][k] = sum over the rows of chunk z of G[i][slot] * X[i][k]; ldg must be a multiple of 64
int simt_backward(Ctx* c, const float* G, int ldg, int n_slots, int nz, int64_t rpc, float* gradp) {
  const int ldx = (int)c->ldx;
  dim3 gb((ldx + 63) / 64, (n_slots + TN - 1) / TN, nz);
  bwd_kernel<<<gb, 256, 0, c->stream>>>(c->X, c->n, ldx, G, ldg, n_slots, rpc, gradp);
  c->launches += 1;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(c, std::string("simt_backward launch: ") + cudaGetErrorString(e));
  return 0;
}

}  // namespace skd
