// sgd_tc.cu -- hinge-loss SGD for every one-vs-rest label column, blocked-exact on the tensor cores.
//
// Same contract as sgd.cu (it replaces K runs of the reference's `_fit_binary`, ref
// multiclass.py:109-152, estimator = SGDClassifier; SK/linear_model/_sgd_fast.pyx.tp:274-640
// `_plain_sgd32`) and the same results bit for bit.  What changes is where the 4*n*d flops per
// column and epoch are spent.
//
// With hinge loss a sample whose margin y*p exceeds 1 changes only scalars (lazy scale, norm,
// objective); about 1 sample in 200 is a margin violator.  So the dot products of a block of
// T = 2048 shuffled samples with the weights the block starts from are ONE dense product
//     S = X_T W^T        [T x K]   (all label columns at once)
// and a violator j inside the block changes later margins of its column by q_j * (x_j . x_t),
// one entry of the block's Gram matrix
//     G = X_T X_T^T      [T x T]   (shared by all columns).
// Both run on the tensor cores in fp16 (sgd_gemm_kernel: TMA -> 128B-swizzled shared memory ->
// wgmma 64x128x16, two warpgroups per 128 x 128 tile, fp32 accumulators in registers), X permuted into the epoch's shuffled order and
// scaled by a power of two once per epoch.  They are used for SCREENING only: sgd_scan_kernel (one
// warp per column, its float32 weights in registers like sgd.cu) walks the block in order and
// declares a sample a non-violator only if its approximate margin clears 1 by more than a rigorous
// error bound (2^-9 * |w| * |x| covers the fp16 operand rounding and the fp32 accumulation); every
// other sample gets the exact float32-product / float64-sum dot product of sgd.cu, and every
// update is applied exactly as `_plain_sgd32` does.  Scalar recurrences (float64 norm and objective
// in sample order) are kept operation for operation.  Hence identical coefficients, intercepts and
// n_iter_, at tensor-core cost for 99 % of the samples.  sgd_fit_batch (sgd.cu) runs the fit and
// hands each epoch to SgdTc::epoch.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "sgd_replay.h"
#include "tc_ptx.h"

namespace skd {

constexpr int ST_T = 2048;           // samples per block
constexpr int ST_TILE = 128;
constexpr int ST_STAGES = 4;         // TMA ring: [A chunk | B chunk] of 128 rows x 64 fp16 each
constexpr int ST_VMAX = 96;          // in-block violators a column can log before it falls back to exact dots
constexpr float ST_KAPPA = 0.001953125f;   // 2^-9

// ------------------------------------------------------------------------------------------
// C = A B^T for fp16 row-major operands [rows x K] (K-major), fp32 accumulation in registers.
// One 128 x 128 output tile per CTA, two warpgroups of 64 output rows each (wgmma m64n128k16);
// thread 0 also streams the K chunks through a TMA ring of ST_STAGES slots.
// Tiles [0, n_s): S tile (sample tile mi, column group ni), stored transposed S[col][sample];
// tiles [n_s, n_s + n_g): Gram tile (mi <= ni) stored G[j][t].
// ------------------------------------------------------------------------------------------
struct SgdGemmParams {
  float* S;            // [kpad][T]
  float* G;            // [T][T]
  int row0;            // first row of the block in the permuted matrix
  int n_s, n_colgroups;
  int n_g;
  const int2* gtiles;  // [n_g] (mi, ni)
  int kchunks;         // dpad / 64
};

struct __align__(8) SgdGemmBars {
  uint64_t full[ST_STAGES];
  uint64_t empty[ST_STAGES];
};

constexpr int ST_THREADS = 256;

__global__ void __launch_bounds__(ST_THREADS, 1)
sgd_gemm_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                const SgdGemmParams prm) {
  extern __shared__ uint8_t smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;                   // warpgroup: output rows [64 wg, 64 wg + 64) of the tile
  uint8_t* base = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  constexpr uint32_t CHUNK = ST_TILE * 128;          // 128 rows x 64 fp16
  constexpr uint32_t STAGE = 2 * CHUNK;
  SgdGemmBars* bars = reinterpret_cast<SgdGemmBars*>(base + ST_STAGES * STAGE);
  if (threadIdx.x == 0) {
    for (int i = 0; i < ST_STAGES; ++i) { mbar_init(&bars->full[i], 1); mbar_init(&bars->empty[i], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int tile = blockIdx.x;
  const bool is_g = tile >= prm.n_s;
  int mi, ni;
  if (!is_g) { mi = tile / prm.n_colgroups; ni = tile % prm.n_colgroups; }
  else { const int2 t = prm.gtiles[tile - prm.n_s]; mi = t.x; ni = t.y; }
  const int arow = prm.row0 + mi * ST_TILE;
  const int brow = is_g ? prm.row0 + ni * ST_TILE : ni * ST_TILE;
  const CUtensorMap* bmap = is_g ? &map_x : &map_w;

  // chunk kc goes to slot kc % ST_STAGES once both warpgroups are done with chunk kc - ST_STAGES
  auto issue = [&](int kc) {
    const uint32_t sl = kc % ST_STAGES;
    if (kc >= ST_STAGES) mbar_wait(&bars->empty[sl], ((kc / ST_STAGES) - 1) & 1, 500);
    mbar_expect_tx(&bars->full[sl], STAGE);
    tma_load_2d(base + sl * STAGE, &map_x, kc * 64, arow, &bars->full[sl]);
    tma_load_2d(base + sl * STAGE + CHUNK, bmap, kc * 64, brow, &bars->full[sl]);
  };
  if (threadIdx.x == 0)
    for (int kc = 0; kc < prm.kchunks && kc < ST_STAGES; ++kc) issue(kc);
  __syncwarp();

  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  const uint64_t d0 = make_desc(smem_u32(base), 16, 1024);
  for (int kc = 0; kc < prm.kchunks; ++kc) {
    const uint32_t sl = kc % ST_STAGES, ph = (kc / ST_STAGES) & 1;
    mbar_wait(&bars->full[sl], ph, 510);
    const uint64_t a = d0 + (uint64_t)((sl * STAGE + wg * 64 * 128) >> 4);
    const uint64_t b = d0 + (uint64_t)((sl * STAGE + CHUNK) >> 4);
    reg_fence(acc);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) wgmma_m64n128_ss(acc, a + ks * 2, b + ks * 2, 1u);
    wgmma_commit();
    wgmma_wait_all();
    reg_fence(acc);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&bars->empty[sl]);
    if (threadIdx.x == 0 && kc + ST_STAGES < prm.kchunks) issue(kc + ST_STAGES);
    __syncwarp();
  }
  // accumulator fragment: acc[i] is (row 64 wg + 16 (warp & 3) + lane / 4 + 8 ((i >> 1) & 1),
  //                                   column 8 (i >> 2) + 2 (lane & 3) + (i & 1))
  const int m0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int c0 = 2 * (lane & 3);
  if (!is_g) {
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const int m = m0 + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + c0 + (i & 1);
      prm.S[(size_t)(ni * ST_TILE + col) * ST_T + mi * ST_TILE + m] = acc[i];
    }
  } else {
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const int m = m0 + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + c0;
      *reinterpret_cast<float2*>(prm.G + (size_t)(mi * ST_TILE + m) * ST_T + ni * ST_TILE + col) = make_float2(acc[i], acc[i + 1]);
    }
  }
}

// ------------------------------------------------------------------------------------------
// per-fit / per-epoch preparation
// ------------------------------------------------------------------------------------------
// xnorm[r] = ||x_r||_2 (float64 accumulation), absmax = max |x|
__global__ void sgd_rownorm_kernel(const float* __restrict__ X, int64_t n, int ldx, int d, float* __restrict__ xnorm,
                                   unsigned int* __restrict__ absmax_bits) {
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  double s = 0.0;
  float m = 0.f;
  for (int k = lane; k < d; k += 32) { const float v = X[r * ldx + k]; s += (double)v * (double)v; m = fmaxf(m, fabsf(v)); }
  for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o)); }
  if (lane == 0) {
    xnorm[r] = (float)(sqrt(s) * 1.0000002);       // rounded up: it is used in an error bound
    atomicMax(absmax_bits, __float_as_uint(m));
  }
}

// Xp[i][k] = fp16(X[order[i]][k] * sx) for i < n, zero padding rows / columns
__global__ void sgd_permute_kernel(const float* __restrict__ X, int ldx, int d, const int32_t* __restrict__ order,
                                   int64_t n, int64_t npad, int dpad, float sx, __half* __restrict__ Xp,
                                   const int32_t* __restrict__ ycls, const float* __restrict__ xnorm,
                                   int32_t* __restrict__ ycls_p, float* __restrict__ xnorm_p) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;    // one thread per 8 features
  const int per = dpad >> 3;
  if (idx >= npad * per) return;
  const int64_t i = idx / per;
  const int k0 = (int)(idx - i * per) * 8;
  if (k0 == 0 && i < n) { const int r = order[i]; ycls_p[i] = ycls[r]; xnorm_p[i] = xnorm[r]; }   // sample metadata in walk order
  __align__(16) __half h[8];
  if (i < n) {
    const float* src = X + (size_t)order[i] * ldx + k0;
#pragma unroll
    for (int j = 0; j < 8; ++j) h[j] = __float2half_rn(k0 + j < d ? src[j] * sx : 0.f);
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) h[j] = __float2half_rn(0.f);
  }
  *reinterpret_cast<uint4*>(Xp + (size_t)i * dpad + k0) = *reinterpret_cast<const uint4*>(h);
}

// fp16 image of one column's stored weights: W'[slot] = fp16(w * t), t = 2^(13 - floor(log2 max|w|));
// wmeta[slot] = {1 / (sx * t), ||w||_2 rounded up}
template <int DPL>
__device__ __forceinline__ void sgd_export_row(const float (&w)[DPL], int lane, int d, int dpad, float inv_sx,
                                               __half* __restrict__ Wp_row, float2* __restrict__ meta) {
  float m = 0.f;
  double s = 0.0;
#pragma unroll
  for (int j = 0; j < DPL; ++j) { m = fmaxf(m, fabsf(w[j])); s += (double)w[j] * (double)w[j]; }
  for (int o = 16; o > 0; o >>= 1) { m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o)); s += __shfl_xor_sync(0xffffffffu, s, o); }
  float t = 1.f;
  if (m > 0.f && isfinite(m)) { int e; frexpf(m, &e); t = ldexpf(1.f, 13 - (e - 1)); }
#pragma unroll
  for (int j = 0; j < DPL; ++j) {
    const int k = lane + 32 * j;
    if (k < dpad) Wp_row[k] = __float2half_rn(k < d ? w[j] * t : 0.f);
  }
  if (lane == 0) *meta = make_float2(inv_sx / t, (float)(sqrt(s) * 1.0000002));
}

template <int DPL>
__global__ void __launch_bounds__(128)
sgd_export_kernel(const float* __restrict__ W, int ldw, int d, int dpad, const int32_t* __restrict__ active, int n_active,
                  float inv_sx, __half* __restrict__ Wp, float2* __restrict__ wmeta) {
  const int lane = threadIdx.x & 31;
  const int a = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (a >= n_active) return;
  const int col = active[a];
  float w[DPL];
#pragma unroll
  for (int j = 0; j < DPL; ++j) { const int k = lane + 32 * j; w[j] = k < d ? W[(size_t)col * ldw + k] : 0.f; }
  sgd_export_row<DPL>(w, lane, d, dpad, inv_sx, Wp + (size_t)a * dpad, wmeta + a);
}

// ------------------------------------------------------------------------------------------
// ordered walk over one block of T samples, one warp per label column
// ------------------------------------------------------------------------------------------
struct SgdScanParams {
  const float* X; int ldx, d, dpad;
  const int32_t* ycls; const int32_t* order; const double* eta; const float* cfac;
  const double* ws;          // [n + 1] lazy scale before sample i (identical for every running column)
  const int32_t* ycls_p;     // [n] class id of sample i of the epoch (walk order)
  const float* xnorm_p;      // [n] |x| of sample i of the epoch (walk order)
  int64_t n; int row0, t_len;
  const int32_t* active; int n_active; const int32_t* col_pos;
  float* W; int ldw;
  SgdState* state;
  const float* S; const float* G; const float2* wmeta;
  __half* Wp; float2* wmeta_out;
  float inv_sx, inv_sx2;
  double alpha; int fit_intercept; int last_block;
  double tol; int n_iter_no_change;
  unsigned long long* counters;   // [0] samples screened out, [1] exact evaluations, [2] violators,
                                  // [3] (column, block) scans whose violator log filled up (exact from there on)
};

template <int DPL>
__global__ void __launch_bounds__(128)
sgd_scan_kernel(const SgdScanParams P) {
  constexpr int T = 32;
  const unsigned FULL = 0xffffffffu;
  __shared__ float s_vq[4][ST_VMAX];
  __shared__ int s_vj[4][ST_VMAX];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int a = blockIdx.x * 4 + wib;
  if (a >= P.n_active) return;
  const int col = P.active[a];
  const int pos = P.col_pos[col];
  SgdState st = P.state[col];
  float w[DPL];
#pragma unroll
  for (int j = 0; j < DPL; ++j) {
    const int k = lane + 32 * j;
    w[j] = k < P.d ? P.W[(size_t)col * P.ldw + k] : 0.f;
  }
  double sq_norm = st.sq_norm, intercept = st.intercept, objective_sum = st.objective_sum;
  const float2 wm = P.wmeta[a];
  const float inv_scale = wm.x;
  float nwb = wm.y;                  // bound on |stored weights| (block start + logged updates)
  int nviol = 0;
  bool exact_all = false;            // violator log full: every remaining sample gets the exact dot product
  float* vq = s_vq[wib];
  int* vj = s_vj[wib];
  const float* Srow = P.S + (size_t)a * ST_T;
  unsigned long long n_screen = 0, n_exact = 0, n_viol = 0;
  bool vlog_full = false;

  // per-sample inputs of the window [i0, i0 + 32): coalesced loads in walk order, requested one
  // window ahead (the window normally advances by 32; after an event it is re-read)
  // (only loads here: an instruction that consumes a loaded value would stall the warp for the memory
  // latency and the window would no longer be fetched in the shadow of the previous one)
  constexpr int PV = 4;              // Gram entries of the first PV logged updates travel with the window
  struct Win { double e, ws; float c, nx, s, g[PV]; int yc, nv; };
  auto load_win = [&](int i0w) -> Win {
    Win wv; wv.e = 0.0; wv.ws = 1.0; wv.c = 1.f; wv.nx = 0.f; wv.s = 0.f; wv.yc = -1;
    wv.nv = nviol < PV ? nviol : PV;
#pragma unroll
    for (int v = 0; v < PV; ++v) wv.g[v] = 0.f;
    if (i0w + lane < P.t_len) {
      const int64_t gi = (int64_t)P.row0 + i0w + lane;
      wv.e = P.eta[gi]; wv.ws = P.ws[gi]; wv.c = P.cfac[gi]; wv.nx = P.xnorm_p[gi]; wv.yc = P.ycls_p[gi];
      wv.s = Srow[i0w + lane];
#pragma unroll
      for (int v = 0; v < PV; ++v)
        if (v < nviol) wv.g[v] = P.G[(size_t)vj[v] * ST_T + i0w + lane];
    }
    return wv;
  };
  int i0 = 0;
  Win nxt = load_win(0);
  int nxt_i0 = 0;
  while (i0 < P.t_len) {
    const int Te = (P.t_len - i0) < T ? (P.t_len - i0) : T;
    // lane t < Te owns sample i0 + t of the block
    const Win cw = (nxt_i0 == i0) ? nxt : load_win(i0);
    // Every loaded value of this window is consumed BEFORE the next window is requested: the consumer of a
    // load waits on a scoreboard slot, and a slot re-armed by the new loads would make it wait for them
    // too (ncu, first build: 22 % of the stall samples on the first use of the prefetched S value).
    const double y_l = (cw.yc == pos) ? 1.0 : -1.0, e_l = cw.e + 0.0, ws_l = cw.ws + 0.0;
    const float c_l = cw.c + 0.f, nx_l = cw.nx + 0.f;
    float s_l = cw.s * inv_scale;
#pragma unroll
    for (int v = 0; v < PV; ++v) if (v < cw.nv) s_l = fmaf(vq[v], cw.g[v], s_l);
    if (lane < Te)      // updates logged after the window was requested / beyond the first PV
      for (int v = cw.nv; v < nviol; ++v) s_l = fmaf(vq[v], P.G[(size_t)vj[v] * ST_T + i0 + lane], s_l);
    const double c2_l = (double)__fmul_rn(c_l, c_l);
    asm volatile("" ::: "memory");
    nxt_i0 = i0 + T;
    nxt = load_win(nxt_i0);                       // in flight while this window is processed
    asm volatile("" ::: "memory");
    // A. the norm recurrence sq_norm *= c_t^2 in sample order (lane t keeps the value BEFORE sample t)
    // (lane t multiplies the factors of the samples before it, in order: its own sequential chain; one
    // broadcast and one predicated multiply per step instead of a shared chain with per-lane captures)
    double my_sq = sq_norm;
#pragma unroll
    for (int q = 0; q < T - 1; ++q) {
      const double c2q = __shfl_sync(FULL, c2_l, q);
      if (lane > q) my_sq *= c2q;
    }
    const double my_sq_after = my_sq * c2_l;
    // B. screening: approximate margin against 1 + error bound
    const double pa = (double)(float)((double)s_l * ws_l) + intercept;
    const double za = pa * y_l;
    const double band = (double)ws_l * (double)(ST_KAPPA * nx_l * nwb) + 2.4e-7 * (fabs(pa) + 1.0);
    const bool cand_l = lane < Te && (exact_all || !(za > 1.0 + band));
    // reset_wscale(): the lazy scale falls below 1e-6 after this sample's scale step (same sample for every column)
    const double ws_after_l = ws_l * (double)c_l;
    const bool reset_l = lane < Te && ws_after_l < 1e-6;
    const float normf_l = (float)sqrt(my_sq);
    const double l2_l = __dmul_rn(P.alpha, __dmul_rn(0.5, (double)__fmul_rn(normf_l, normf_l)));
    const unsigned evmask = __ballot_sync(FULL, cand_l || reset_l);
    const int ev = evmask ? __ffs(evmask) - 1 : -1;        // first sample that needs the exact path
    const int nfree = ev >= 0 ? ev : Te;                   // samples 0..nfree-1 are certain non-violators
    // D. their objective terms (loss 0) in order
    // (cur_loss + l2 term with cur_loss = 0.0 is the l2 term itself: the terms are non-negative)
#pragma unroll
    for (int q = 0; q < T; ++q) {
      const double tq = __shfl_sync(FULL, l2_l, q);
      if (q < nfree) objective_sum = __dadd_rn(objective_sum, tq);
    }
    n_screen += nfree;
    if (ev < 0) {
      sq_norm = __shfl_sync(FULL, my_sq_after, Te - 1);
      i0 += Te;
      continue;
    }
    // E. sample ev exactly as _plain_sgd32 does
    {
      const int r = P.order[(int64_t)P.row0 + i0 + ev];
      const double y = __shfl_sync(FULL, y_l, ev);
      const double e = __shfl_sync(FULL, e_l, ev);
      const double wsb = __shfl_sync(FULL, ws_l, ev);
      const double l2t = __shfl_sync(FULL, l2_l, ev);
      const float nxe = __shfl_sync(FULL, nx_l, ev);
      const bool is_cand = __shfl_sync(FULL, (int)cand_l, ev) != 0;
      const bool is_reset = __shfl_sync(FULL, (int)reset_l, ev) != 0;
      const double ws_reset = __shfl_sync(FULL, ws_after_l, ev);
      float x[DPL];
#pragma unroll
      for (int j = 0; j < DPL; ++j) {
        const int k = lane + 32 * j;
        x[j] = k < P.ldx ? __ldg(P.X + (size_t)r * P.ldx + k) : 0.f;
      }
      double acc = 0.0;
#pragma unroll
      for (int j = 0; j < DPL; ++j) acc += (double)__fmul_rn(w[j], x[j]);
      acc = warp_sum(acc);
      const double p = (double)(float)(acc * wsb) + intercept;
      const double z = p * y;
      // (a sample that is only a reset event cleared the margin test: its exact margin is above 1 as well)
      const bool viol = is_cand && z <= 1.0;
      const double cur_loss = viol ? 1.0 - z : 0.0;
      objective_sum = __dadd_rn(objective_sum, __dadd_rn(cur_loss, l2t));
      sq_norm = __shfl_sync(FULL, my_sq_after, ev);          // w.scale(c): sq_norm *= c^2
      n_exact += 1;
      if (is_reset) {
        sgd_reset_wscale<DPL>(w, ws_reset);                   // the host's chain continues from wscale = 1
        exact_all = true;                                      // the block's products were taken with the old weights
      }
      if (viol) {
        const double update = -e * (-y);
        if (update != 0.0) {
          const double wsa = P.ws[(int64_t)P.row0 + i0 + ev + 1];   // wscale after this sample's scale step
          double qd;
          sq_norm = sgd_add<DPL>(w, x, update, wsa, P.fit_intercept, intercept, qd);
          n_viol += 1;
          // log the update for the margins of the samples still to come in this block
          if (nviol < ST_VMAX) {
            if (lane == 0) { vq[nviol] = (float)qd * P.inv_sx2; vj[nviol] = i0 + ev; }
            nviol += 1;
            nwb += fabsf((float)qd) * nxe * 1.0000002f;
            __syncwarp();
          } else {
            exact_all = true;
            vlog_full = true;
          }
        }
      }
    }
    i0 += ev + 1;
  }
  // end of block: weights back, fp16 image for the next block's product
#pragma unroll
  for (int j = 0; j < DPL; ++j) {
    const int k = lane + 32 * j;
    if (k < P.d) P.W[(size_t)col * P.ldw + k] = w[j];
  }
  st.sq_norm = sq_norm; st.intercept = intercept; st.objective_sum = objective_sum;
  if (P.last_block) {
    st.wscale = P.ws[P.n];
    sgd_end_epoch<DPL>(st, w, intercept, objective_sum, P.n, P.tol, P.n_iter_no_change);
  } else {
    sgd_export_row<DPL>(w, lane, P.d, P.dpad, P.inv_sx, P.Wp + (size_t)a * P.dpad, P.wmeta_out + a);
  }
  if (lane == 0) {
    P.state[col] = st;
    if (P.counters) {
      atomicAdd(&P.counters[0], n_screen);
      atomicAdd(&P.counters[1], n_exact);
      atomicAdd(&P.counters[2], n_viol);
      if (vlog_full) atomicAdd(&P.counters[3], 1ull);
    }
  }
}

bool sgd_tc_supported(const Ctx* c, int loss, int shuffle) {
  (void)shuffle;
  if (loss != 0) return false;                         // hinge only: other losses update on every sample
  if (c->d > 1024) return false;
  if (const char* e = getenv("SKDIST_B200_SGD_KERNEL")) {
    if (!strcmp(e, "simt")) return false;
    if (!strcmp(e, "tc")) return true;
  }
  return c->n >= 2 * ST_T;                              // small problems stay on the warp-per-column kernel
}

int SgdTc::init(Ctx* c, const SgdFit& f) {
  const int64_t n = c->n;
  const int d = (int)c->d, ldx = (int)c->ldx;
  dpad = (d + 63) / 64 * 64;
  npad = (n + ST_T - 1) / ST_T * ST_T;
  kpad = (f.B + ST_TILE - 1) / ST_TILE * ST_TILE;
  unsigned int* absmax;
  SKD_CUDA(c, sx.alloc(&dws, (size_t)n + 1));
  SKD_CUDA(c, sx.alloc(&xnorm, (size_t)n));
  SKD_CUDA(c, sx.alloc(&xnorm_p, (size_t)n));
  SKD_CUDA(c, sx.alloc(&ycls_p, (size_t)n));
  SKD_CUDA(c, sx.alloc(&Xp, (size_t)npad * dpad));
  SKD_CUDA(c, sx.alloc(&Wp, (size_t)kpad * dpad));
  SKD_CUDA(c, sx.alloc(&wmeta[0], (size_t)kpad));
  SKD_CUDA(c, sx.alloc(&wmeta[1], (size_t)kpad));
  SKD_CUDA(c, sx.alloc(&S, (size_t)kpad * ST_T));
  SKD_CUDA(c, sx.alloc(&G[0], (size_t)ST_T * ST_T));
  SKD_CUDA(c, sx.alloc(&G[1], (size_t)ST_T * ST_T));
  SKD_CUDA(c, sx.alloc(&absmax, 1));
  SKD_CUDA(c, sx.alloc(&counters, 4));
  const int tiles_t = ST_T / ST_TILE;
  std::vector<int2> hg;
  for (int mi = 0; mi < tiles_t; ++mi) for (int ni = mi; ni < tiles_t; ++ni) hg.push_back(make_int2(mi, ni));
  n_g = (int)hg.size();
  SKD_CUDA(c, sx.alloc(&gtiles, hg.size()));
  SKD_CUDA(c, cudaMemcpyAsync(gtiles, hg.data(), hg.size() * sizeof(int2), cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemsetAsync(absmax, 0, 4, c->stream));
  SKD_CUDA(c, cudaMemsetAsync(counters, 0, 32, c->stream));
  sgd_rownorm_kernel<<<(unsigned)((n + 7) / 8), 256, 0, c->stream>>>(c->X, n, ldx, d, xnorm, absmax);
  c->launches += 1;
  unsigned int hmax_bits = 0;
  SKD_CUDA(c, cudaMemcpyAsync(&hmax_bits, absmax, 4, cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  float hmax; memcpy(&hmax, &hmax_bits, 4);
  if (hmax > 0.f && std::isfinite(hmax)) { int e; frexpf(hmax, &e); sxs = ldexpf(1.f, 13 - (e - 1)); }
  inv_sx = 1.f / sxs;
  inv_sx2 = inv_sx * inv_sx;

  if (tc_make_map_2d(c, &map_x, Xp, (uint64_t)npad, (uint64_t)dpad, ST_TILE)) return 1;
  if (tc_make_map_2d(c, &map_w, Wp, (uint64_t)kpad, (uint64_t)dpad, ST_TILE)) return 1;
  gemm_smem = 1024 + (size_t)ST_STAGES * 2 * ST_TILE * 128 + sizeof(SgdGemmBars) + 64;
  SKD_CUDA(c, cudaFuncSetAttribute(sgd_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gemm_smem));
  for (int i = 0; i < 3; ++i) SKD_CUDA(c, cudaEventCreate(&ev_t[i]));
  SKD_CUDA(c, cudaStreamCreateWithFlags(&sB, cudaStreamNonBlocking));
  SKD_CUDA(c, cudaEventCreateWithFlags(&ev_perm, cudaEventDisableTiming));
  for (int i = 0; i < 2; ++i) {
    SKD_CUDA(c, cudaEventCreateWithFlags(&ev_g[i], cudaEventDisableTiming));
    SKD_CUDA(c, cudaEventCreateWithFlags(&ev_scan[i], cudaEventDisableTiming));
  }
  hcfac.resize(n);
  hws.resize(n + 1);
  return 0;
}

SgdTc::~SgdTc() {
  if (sB) cudaStreamSynchronize(sB);
  for (cudaEvent_t e : {ev_perm, ev_g[0], ev_g[1], ev_scan[0], ev_scan[1], ev_t[0], ev_t[1], ev_t[2]})
    if (e) cudaEventDestroy(e);
  if (sB) cudaStreamDestroy(sB);
}

int SgdTc::epoch(Ctx* c, const SgdFit& f, int epoch, int n_active, bool new_order, bool trace) {
  const int64_t n = c->n;
  const int d = (int)c->d, ldx = (int)c->ldx;
  // the lazy-scale chain wscale *= c_t of the epoch (one float64 multiply per sample, identical for every
  // running column): evaluated once on the host from the device's own c_t
  SKD_CUDA(c, cudaMemcpyAsync(hcfac.data(), f.cfac, (size_t)n * 4, cudaMemcpyDeviceToHost, c->stream));
  if (new_order) {
    const int64_t total = npad * (dpad / 8);
    sgd_permute_kernel<<<(unsigned)((total + 255) / 256), 256, 0, c->stream>>>(c->X, ldx, d, f.order, n, npad, dpad, sxs, Xp,
                                                                             c->ycls, xnorm, ycls_p, xnorm_p);
    c->launches += 1;
  }
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  {
    double wsc = wscale_epoch;
    for (int64_t i = 0; i < n; ++i) {
      hws[i] = wsc;
      wsc *= (double)hcfac[i];
      if (wsc < 1e-6) wsc = 1.0;          // reset_wscale() (the scan kernel rescales the weights at this sample)
    }
    hws[n] = wsc;
    wscale_epoch = wsc;
  }
  SKD_CUDA(c, cudaMemcpyAsync(dws, hws.data(), (size_t)(n + 1) * 8, cudaMemcpyHostToDevice, c->stream));
  c->h2d += n * 8; c->d2h += n * 4;
  const int tiles_t = ST_T / ST_TILE;
  const int kgroups = (n_active + ST_TILE - 1) / ST_TILE;
  SKD_CUDA(c, cudaMemsetAsync(Wp, 0, (size_t)kpad * dpad * sizeof(__half), c->stream));
#define SGD_TC_CASE(D, CALL) case D: CALL(D); break;
#define SGD_EXPORT(D) sgd_export_kernel<D><<<(n_active + 3) / 4, 128, 0, c->stream>>>(f.W, f.ldw, d, dpad, f.active, n_active, inv_sx, Wp, wmeta[0])
  switch (f.dpl) { SGD_TC_CASE(1, SGD_EXPORT) SGD_TC_CASE(2, SGD_EXPORT) SGD_TC_CASE(4, SGD_EXPORT) SGD_TC_CASE(8, SGD_EXPORT)
                   SGD_TC_CASE(16, SGD_EXPORT) SGD_TC_CASE(32, SGD_EXPORT) default: return fail(c, "sgd: bad dpl"); }
  c->launches += 1;
  const int n_blocks = (int)((n + ST_T - 1) / ST_T);
  double t_gemm = 0.0, t_scan = 0.0; int t_cnt = 0;
  // The Gram product of a block does not depend on the weights: it runs one block ahead on a second
  // stream (two G buffers), so only S = X_T W^T sits between two scans.
  SKD_CUDA(c, cudaEventRecord(ev_perm, c->stream));          // Xp of this epoch is complete
  SKD_CUDA(c, cudaStreamWaitEvent(sB, ev_perm, 0));
  auto launch_g = [&](int b) {
    SgdGemmParams gg;
    gg.S = S; gg.G = G[b & 1]; gg.row0 = b * ST_T; gg.n_colgroups = 1; gg.n_s = 0;
    gg.n_g = n_g; gg.gtiles = gtiles; gg.kchunks = dpad / 64;
    sgd_gemm_kernel<<<gg.n_g, ST_THREADS, gemm_smem, sB>>>(map_x, map_w, gg);
    cudaEventRecord(ev_g[b & 1], sB);
  };
  launch_g(0);
  for (int b = 0; b < n_blocks; ++b) {
    if (b + 1 < n_blocks) {
      if (b >= 1) SKD_CUDA(c, cudaStreamWaitEvent(sB, ev_scan[(b + 1) & 1], 0));   // scan(b - 1) is done with that buffer
      launch_g(b + 1);
    }
    SgdGemmParams gp;
    gp.S = S; gp.G = G[b & 1]; gp.row0 = b * ST_T; gp.n_colgroups = kgroups; gp.n_s = tiles_t * kgroups;
    gp.n_g = 0; gp.gtiles = gtiles; gp.kchunks = dpad / 64;
    const bool tb = trace && (epoch == 1 || epoch == 20) && b >= 8 && b < 24;    // kernel split of 16 blocks
    if (tb) cudaEventRecord(ev_t[0], c->stream);
    sgd_gemm_kernel<<<gp.n_s, ST_THREADS, gemm_smem, c->stream>>>(map_x, map_w, gp);
    if (tb) cudaEventRecord(ev_t[1], c->stream);
    SKD_CUDA(c, cudaStreamWaitEvent(c->stream, ev_g[b & 1], 0));
    SgdScanParams sp;
    sp.X = c->X; sp.ldx = ldx; sp.d = d; sp.dpad = dpad; sp.ycls = c->ycls; sp.order = f.order; sp.eta = f.eta;
    sp.cfac = f.cfac; sp.ws = dws; sp.ycls_p = ycls_p; sp.xnorm_p = xnorm_p; sp.n = n; sp.row0 = b * ST_T;
    sp.t_len = (int)std::min<int64_t>(ST_T, n - (int64_t)b * ST_T);
    sp.active = f.active; sp.n_active = n_active; sp.col_pos = f.col_pos; sp.W = f.W; sp.ldw = f.ldw; sp.state = f.state;
    sp.S = S; sp.G = G[b & 1]; sp.wmeta = wmeta[b & 1]; sp.Wp = Wp; sp.wmeta_out = wmeta[(b + 1) & 1];
    sp.inv_sx = inv_sx; sp.inv_sx2 = inv_sx2; sp.alpha = f.alpha; sp.fit_intercept = f.fit_intercept;
    sp.last_block = b == n_blocks - 1; sp.tol = f.tol; sp.n_iter_no_change = f.n_iter_no_change; sp.counters = counters;
#define SGD_SCAN(D) sgd_scan_kernel<D><<<(n_active + 3) / 4, 128, 0, c->stream>>>(sp)
    switch (f.dpl) { SGD_TC_CASE(1, SGD_SCAN) SGD_TC_CASE(2, SGD_SCAN) SGD_TC_CASE(4, SGD_SCAN) SGD_TC_CASE(8, SGD_SCAN)
                     SGD_TC_CASE(16, SGD_SCAN) SGD_TC_CASE(32, SGD_SCAN) default: return fail(c, "sgd: bad dpl"); }
    SKD_CUDA(c, cudaEventRecord(ev_scan[b & 1], c->stream));
    if (tb) {
      cudaEventRecord(ev_t[2], c->stream);
      cudaEventSynchronize(ev_t[2]);
      float m1 = 0.f, m2 = 0.f;
      cudaEventElapsedTime(&m1, ev_t[0], ev_t[1]);
      cudaEventElapsedTime(&m2, ev_t[1], ev_t[2]);
      t_gemm += m1; t_scan += m2; t_cnt += 1;
    }
    c->launches += 3;
  }
#undef SGD_SCAN
#undef SGD_EXPORT
#undef SGD_TC_CASE
  SKD_CUDA(c, cudaGetLastError());
  if (t_cnt > 0)
    fprintf(stderr, "[skd trace] sgd-tc epoch %3d per block (16 blocks, synchronised): S product %.1f us, wait for G + scan %.1f us\n",
            epoch, 1e3 * t_gemm / t_cnt, 1e3 * t_scan / t_cnt);
  return 0;
}

void SgdTc::print_counters() {
  unsigned long long hc[4];
  cudaMemcpy(hc, counters, 32, cudaMemcpyDeviceToHost);
  fprintf(stderr, "[skd trace] sgd-tc samples screened by the tensor-core margins %llu, exact dot products %llu, violators %llu, "
          "violator-log overflows %llu\n", hc[0], hc[1], hc[2], hc[3]);
}

}  // namespace skd
