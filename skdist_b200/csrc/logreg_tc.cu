// logreg_tc.cu -- fused batched logistic loss + gradient on the Hopper tensor cores (sm_90a wgmma).
//
// One launch evaluates f, g of every active (candidate x fold) column, i.e. replaces, for all
// columns at once, the two fp32 sgemv passes + pointwise loop that each reference task runs per
// L-BFGS evaluation (SK/linear_model/_linear_loss.py:291-379; ref search.py:230):
//
//     Z  = W  X^T     (slots x rows)   GEMM1   wgmma, A = W from shared memory, accumulators in registers
//     G  = dloss(Z, y) masked by fold  epilogue on the accumulator registers (CUDA cores)
//     dW = G  X       (slots x d)      GEMM2   wgmma, A operand = G straight from registers
//
// X is read ONCE per tile by TMA into 128B-swizzled shared memory and used by both GEMMs: as
// the K-major B operand of GEMM1 (K = features) and, through a second descriptor over the same
// bytes, as the MN-major B operand of GEMM2 (K = rows).
//
// fp32 fidelity on tensor cores (there is no fp32 MMA): every operand is split into two fp16
// numbers, v = hi + lo (22+ mantissa bits after exact power-of-two pre-scaling per feature /
// per column), and each product is three MMAs hi*hi + hi*lo + lo*hi accumulated in fp32.
//
// Work decomposition: a group = 128 slots, two consumer warpgroups of 64 slots each (wgmma M = 64);
// its rows are cut into TC_NCH chunks; one persistent CTA per run of (group, chunk) items.  Per CTA:
// W_hi and W_lo stationary in shared memory, the gradient accumulators (64 x d fp32 per consumer
// warpgroup) stationary in registers, X streamed in sub-tiles of 32 rows (hi and lo halves) through
// a TMA ring that a producer warpgroup keeps filled.  The accumulator fragment of a 16-row block of Z
// is the register A fragment of one k16 step of GEMM2, so G never leaves the registers.  The two
// consumers take turns on the tensor cores, so that one runs its epilogue while the products of the
// other are in flight.
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "skd_internal.h"
#include "tc_ptx.h"

namespace skd {

constexpr int TC_BC = 128;       // slots per group
constexpr int TC_R = 64;         // rows per tile (the unit of the tile lists and row bit matrices)
constexpr int TC_SUB = 32;       // rows per ring sub-tile (wgmma N of GEMM1, K of GEMM2)
constexpr int TC_NCH = 132;      // fixed row chunks per group (one partial sum per (chunk, slot)); fixing it fixes
                                 // the summation order of every result
constexpr int TC_THREADS = 384;  // producer warpgroup + two consumer warpgroups
// register split of the warpgroups (setmaxnreg): 128 * 24 + 256 * 240 = 64 512 of the SM's 65 536
constexpr uint32_t TC_PRODUCER_REGS = 24;
constexpr uint32_t TC_CONSUMER_REGS = 240;
constexpr uint32_t TC_SMEM_MAX = 232448;   // 227 KB of opt-in shared memory per block
constexpr float XSCALE_TARGET_EXP = 13.f;   // column max scaled into [2^13, 2^14)
constexpr float GSCALE = 16384.f;           // 2^14

// ---------------------------------------------------------------------------------------------
// data preparation kernels
// ---------------------------------------------------------------------------------------------
// per-feature max |x|
__global__ void tc_colmax_kernel(const float* __restrict__ X, int64_t n, int ldx, int d,
                                 unsigned int* __restrict__ colmax_bits) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= d) return;
  int64_t r0 = (int64_t)blockIdx.y * 4096;
  int64_t r1 = r0 + 4096 < n ? r0 + 4096 : n;
  float m = 0.f;
  for (int64_t r = r0; r < r1; ++r) m = fmaxf(m, fabsf(X[r * ldx + k]));
  atomicMax(&colmax_bits[k], __float_as_uint(m));  // non-negative floats order as uints
}

// Exponent of the power-of-two scale that brings a maximum m = f * 2^e (frexpf) into [2^13, 2^14):
// 13 - floor(log2 m).  Capped at 127 so that the scale stays a finite float: a maximum below 2^-114
// then lands below 2^13, and only loses fp16 relative precision on contributions that small.
__device__ __forceinline__ int pow2_scale_exp(int e) { return min((int)XSCALE_TARGET_EXP - (e - 1), 127); }

// scale[k] = 2^(13 - floor(log2(colmax))) ; gscale[k] = 1 / (scale[k] * 2^14)
__global__ void tc_scale_kernel(const unsigned int* __restrict__ colmax_bits, int d, int dpad,
                                float* __restrict__ xscale, double* __restrict__ gscale) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= dpad) return;
  float s = 1.f;
  if (k < d) {
    float m = __uint_as_float(colmax_bits[k]);
    if (m > 0.f && isfinite(m)) {
      int e;
      frexpf(m, &e);  // m = f * 2^e, f in [0.5, 1)  -> floor(log2 m) = e - 1
      s = ldexpf(1.f, pow2_scale_exp(e));
    }
  }
  xscale[k] = s;
  gscale[k] = 1.0 / ((double)s * (double)GSCALE);
}

// Xh, Xl [npad x dpad] fp16 (zero padded), rowmeta[npad] = (fold << 24) | class id (0xFF fold: pad)
__global__ void tc_split_kernel(const float* __restrict__ X, int64_t n, int64_t npad, int ldx, int d,
                                int dpad, const float* __restrict__ xscale,
                                __half* __restrict__ Xh, __half* __restrict__ Xl) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t total = npad * dpad;
  if (idx >= total) return;
  int64_t r = idx / dpad;
  int k = (int)(idx - r * dpad);
  float v = 0.f;
  if (r < n && k < d) v = X[r * ldx + k] * xscale[k];
  __half h = __float2half_rn(v);
  __half l = __float2half_rn(v - __half2float(h));
  Xh[idx] = h;
  Xl[idx] = l;
}

__global__ void tc_rowmeta_kernel(const int32_t* __restrict__ ycls, const int8_t* __restrict__ fold,
                                  int64_t n, int64_t npad, uint32_t* __restrict__ rowmeta) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= npad) return;
  uint32_t m = 0xFF000000u;
  if (r < n) {
    uint32_t f = fold ? (uint32_t)(uint8_t)fold[r] : 0u;
    m = (f << 24) | (ycls ? ((uint32_t)ycls[r] & 0x00FFFFFFu) : 0u);
  }
  rowmeta[r] = m;
}

// rowsg[li][r] = -y * 2^14 for the rows list li trains on (li < n_lists - 1: every row outside
// fold li; last list: every row), 0 for held-out and padding rows.  y = +1 iff class id == pos.
__global__ void tc_rowsg_kernel(const int32_t* __restrict__ ycls, const int8_t* __restrict__ fold,
                                int64_t n, int64_t npad, int n_lists, int pos, float* __restrict__ rowsg) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= npad) return;
  const bool in = r < n;
  const float s = in ? (ycls[r] == pos ? -GSCALE : GSCALE) : 0.f;
  const int f = (in && fold) ? (int)(uint8_t)fold[r] : -1;
  for (int li = 0; li < n_lists; ++li)
    rowsg[(size_t)li * npad + r] = (li < n_lists - 1 && f == li) ? 0.f : s;
}

// Export of the active slots' iterates in tensor-core form (replaces lb_export_kernel):
// w32 = (float)x (SK/_linear_loss.py:216), W' = w32 / xscale * t, t = 2^(13 - floor(log2 max|w32/xscale|)),
// Wh/Wl [slots_pad x dpad] fp16, wmeta[slot] = {1/t, bias, fold, pos}
struct TcSlotParam {
  float inv_t;
  float bias;
  int32_t fold;
  int32_t pos;
  int32_t neg1;   // SlotMeta::pad (0 = one-vs-rest, k + 1 = pair with class k)
  int32_t col;    // column id of the slot in the caller's batch (-1: padding slot); indexes the row bit matrices
};

__global__ void __launch_bounds__(128)
tc_export_kernel(const double* __restrict__ vec, size_t vec_stride, const SlotMeta* __restrict__ slot,
                 const int32_t* __restrict__ n_act, int d, int dpad, const float* __restrict__ xscale,
                 __half* __restrict__ Wh, __half* __restrict__ Wl, TcSlotParam* __restrict__ sp,
                 const double* __restrict__ xin /* optional: explicit points [slots x (d+1)] */,
                 int fit_intercept) {
  __shared__ float red[4];
  const int s = blockIdx.x;
  if (s >= *n_act) return;
  const SlotMeta sm = slot[s];
  if (sm.col < 0) {   // padding slot of the fold-grouped layout: zero weights, keeps its segment's fold
    for (int k = threadIdx.x; k < dpad; k += 128) {
      Wh[(size_t)s * dpad + k] = __float2half_rn(0.f);
      Wl[(size_t)s * dpad + k] = __float2half_rn(0.f);
    }
    if (threadIdx.x == 0) { TcSlotParam p; p.inv_t = 1.f; p.bias = 0.f; p.fold = sm.fold; p.pos = -1; p.neg1 = 0; p.col = -1; sp[s] = p; }
    return;
  }
  const double* x = xin ? xin + (size_t)sm.col * (d + 1) : vec + (size_t)sm.col * vec_stride;
  float m = 0.f;
  for (int k = threadIdx.x; k < d; k += 128) m = fmaxf(m, fabsf((float)x[k] / xscale[k]));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  float t = 1.f;
  if (m > 0.f && isfinite(m)) {
    int e;
    frexpf(m, &e);
    t = ldexpf(1.f, pow2_scale_exp(e));
  }
  for (int k = threadIdx.x; k < dpad; k += 128) {
    float v = 0.f;
    if (k < d) v = ((float)x[k] / xscale[k]) * t;   // power-of-two scalings: exact
    __half h = __float2half_rn(v);
    __half l = __float2half_rn(v - __half2float(h));
    Wh[(size_t)s * dpad + k] = h;
    Wl[(size_t)s * dpad + k] = l;
  }
  if (threadIdx.x == 0) {
    TcSlotParam p;
    p.inv_t = 1.f / t;
    p.bias = fit_intercept ? (float)x[d] : 0.f;
    p.fold = sm.fold;
    p.pos = sm.pos;
    p.neg1 = sm.pad;
    p.col = sm.col;
    sp[s] = p;
  }
}

// ---------------------------------------------------------------------------------------------
// the fused kernel
// ---------------------------------------------------------------------------------------------
struct TcParams {
  const TcSlotParam* sp;     // [slots]
  const uint32_t* rowmeta;   // [npad]
  const float* yreal;        // [npad] regression targets (TC_R2)
  double* lossp;             // [nz x n_act]        (fit)
  double* gsump;             // [nz x n_act]        (fit)
  float* gradp;              // [nz x n_act x ldw]  (fit)
  unsigned long long* correct;  // [n_act]          (score)
  unsigned long long* count;    // [n_act]          (score)
  int n_act;                 // host value: stride of the partial arrays, upper bound of the live slots
  const int32_t* n_act_dev;  // live slot count on the device (nullptr: n_act is exact)
  int groups;
  int n_tiles;               // npad / 64
  int ldw;                   // leading dimension of gradp (== dpad)
  const int32_t* tilelist;   // per-fold lists of tiles with training rows (nullptr: every tile)
  const int32_t* tilecnt;
  int n_lists, n_tiles_ld;
  const float* rowsg;        // TC_FIT_UNI: [n_lists x npad] per-row -y * 2^14 (0 = not a training row of that list)
  long long rowsg_ld;
  const uint32_t* ybits;     // TC_FIT: per-column row label bits (nullptr: class id == pos), see LogregWork
  const uint32_t* mbits;     // TC_FIT: per-column training-row bits (nullptr: every row of the training folds)
  long long rb_words;
  int32_t* deal_log;         // nullptr, or {live groups, groups whose second half is padding, CTAs, CTAs whose
                             // range spans two or more groups} of this launch (the last entry zeroed by the caller)
  const float2* cw;          // TC_FIT_W / TC_FIT_UNI_W: per-column {label-0, label-1} class weights, largest <= 1
};

// TC_FIT_UNI: fit where every slot of a group shares (held-out fold, positive class): the row's
// sign/mask comes from a precomputed per-fold array instead of being decoded per element.
// TC_FIT_W / TC_FIT_UNI_W: the same two fits with class weights (each row's loss and gradient entry
// times its column's weight for the row's label), separate instantiations so that the unweighted
// ones stay as they are.
enum { TC_FIT = 0, TC_SCORE = 1, TC_R2 = 2, TC_FIT_UNI = 3, TC_FIT_W = 4, TC_FIT_UNI_W = 5 };

// shared memory of one CTA: W_hi, W_lo [NCHUNK][128 slots x 64 fp16] + the ring of sub-tiles
template <int NCHUNK>
struct TcSmem {
  static constexpr uint32_t W_CHUNK = TC_BC * 128;
  static constexpr uint32_t X_CHUNK = TC_SUB * 128;
  static constexpr uint32_t W_BYTES = 2 * NCHUNK * W_CHUNK;
  static constexpr uint32_t STAGE = 2 * NCHUNK * X_CHUNK;          // [X_hi chunks | X_lo chunks]
  static constexpr int NS_FIT = (int)((TC_SMEM_MAX - 1024 - 256 - W_BYTES) / STAGE);
  static constexpr int NS = NS_FIT < 8 ? NS_FIT : 8;
  static constexpr size_t BYTES = 1024 + (size_t)W_BYTES + (size_t)NS * STAGE + 256;
  static_assert(NS >= 2, "ring too small");
};

struct __align__(8) TcBarriers {
  uint64_t full[8];    // stage loaded (TMA transaction count)
  uint64_t empty[8];   // stage consumed by both consumer warpgroups
  uint64_t w_full;     // W_hi / W_lo of the current group loaded
  uint64_t w_free;     // both consumers are done with the previous group's W
};

template <int NCHUNK>
__device__ __forceinline__ void wgmma_grad(float (&d)[NCHUNK * 32], const uint32_t (&a)[4], uint64_t b) {
  if constexpr (NCHUNK == 1) wgmma_m64n64_rs_tb(d, a, b);
  else if constexpr (NCHUNK == 2) wgmma_m64n128_rs_tb(d, a, b);
  else if constexpr (NCHUNK == 3) wgmma_m64n192_rs_tb(d, a, b);
  else wgmma_m64n256_rs_tb(d, a, b);
}

__device__ __forceinline__ void two_sum_add(float& hi, float& lo, float v) {
  const float s = hi + v, bb = s - hi;
  lo += (hi - (s - bb)) + (v - bb);
  hi = s;
}

template <int NCHUNK, int MODE>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_eval_kernel(const __grid_constant__ CUtensorMap map_xh, const __grid_constant__ CUtensorMap map_xl,
               const __grid_constant__ CUtensorMap map_wh, const __grid_constant__ CUtensorMap map_wl,
               const TcParams prm) {
  constexpr bool UNI = MODE == TC_FIT_UNI || MODE == TC_FIT_UNI_W;   // row sign from the per-fold arrays
  constexpr bool DECODE = MODE == TC_FIT || MODE == TC_FIT_W;        // row sign decoded per element
  constexpr bool WEIGHTED = MODE == TC_FIT_W || MODE == TC_FIT_UNI_W;
  constexpr bool IS_FIT = UNI || DECODE;
  using SM = TcSmem<NCHUNK>;
  constexpr int NS = SM::NS;
  extern __shared__ uint8_t smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // warpgroup: 0 producer, 1 and 2 consumers (read from lane 0, so the compiler knows it is warp-uniform
  // and keeps the descriptors built from it in uniform registers)
  const int wg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
  const int cw = wg - 1;                           // consumer cw: slots [64 cw, 64 cw + 64) of the group
  const bool wg_leader = (threadIdx.x & 127) == 0;
  uint8_t* base = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* s_wh = base;
  uint8_t* s_wl = base + NCHUNK * SM::W_CHUNK;
  uint8_t* s_ring = base + SM::W_BYTES;
  TcBarriers* bars = reinterpret_cast<TcBarriers*>(s_ring + NS * SM::STAGE);

  if (threadIdx.x == 0) {
    for (int i = 0; i < NS; ++i) { mbar_init(&bars->full[i], 1); mbar_init(&bars->empty[i], 2); }
    mbar_init(&bars->w_full, 1);
    mbar_init(&bars->w_free, 2);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();   // the last block-wide barrier: the roles part here

  // Work split.  A group's tile list (all tiles, or the tiles with training rows of the group's
  // fold) is cut into TC_NCH fixed chunks; a unit = (group, chunk).  A chunk is always accumulated by
  // ONE CTA from a zeroed accumulator and written to partial slot `chunk`, so the partial sums -- and
  // with them every fitted coefficient -- do not depend on the grid, on how many columns share the
  // batch, or on how many GPUs the columns were dealt to.
  // The deal is made here, from the live slot count (the host's count may be a few optimiser rounds
  // old).  The units of the live groups are ordered band-major: bands of band_w consecutive chunks,
  // within a band by group, then by chunk.  That order is cut into gridDim.x equal contiguous ranges,
  // one per CTA.  band_w is one CTA's share, so the CTAs of a band run different groups over the same
  // rows at the same time and X comes from HBM about once per launch.  Every unit weighs the same,
  // also when the group's second consumer warpgroup holds only padding (it then computes nothing, see
  // the consumers): weighing such a unit half made the launches with such groups slower, because the
  // live consumer alone takes much more than half the time of a full group's chunk.
  const int n_live = prm.n_act_dev ? min(prm.n_act, (int)*prm.n_act_dev) : prm.n_act;
  const int n_groups = max(0, min(prm.groups, (n_live + TC_BC - 1) / TC_BC));
  // a fold segment is padded at its end and 128-aligned: slots [64, 128) of a group are all padding
  // exactly when slot 64 is
  auto half_padding = [&](int g) -> bool {
    const int s = g * TC_BC + 64;
    return s >= n_live || prm.sp[s].col < 0;
  };
  struct TcWalk { int g, z, b0, b1, pos; };   // unit (g, chunk z) in band [b0, b1), its position in the order
  const long long total = (long long)TC_NCH * n_groups;
  const int pos_begin = (int)((long long)blockIdx.x * total / gridDim.x);
  const int pos_end = (int)((long long)(blockIdx.x + 1) * total / gridDim.x);
  const int band_w = (int)min((long long)TC_NCH, max(1LL, (total + gridDim.x - 1) / gridDim.x));
  TcWalk start{0, TC_NCH, TC_NCH, TC_NCH, (int)total};
  if (pos_begin < pos_end) {
    start.b0 = pos_begin / (band_w * n_groups) * band_w;   // every earlier band is band_w chunks wide
    start.b1 = min(start.b0 + band_w, TC_NCH);
    const int off = pos_begin - start.b0 * n_groups, width = start.b1 - start.b0;
    start.g = off / width;
    start.z = start.b0 + off % width;
    start.pos = pos_begin;
  }
  auto next_unit = [&](TcWalk& w) {
    ++w.pos;
    if (++w.z < w.b1) return;
    if (++w.g == n_groups) { w.g = 0; w.b0 = w.b1; w.b1 = min(w.b1 + band_w, TC_NCH); }
    w.z = w.b0;
  };
  if (prm.deal_log && threadIdx.x == 0) {
    if (blockIdx.x == 0) {
      int halves = 0;
      for (int g = 0; g < n_groups; ++g) halves += half_padding(g) ? 1 : 0;
      prm.deal_log[0] = n_groups;
      prm.deal_log[1] = halves;
      prm.deal_log[2] = gridDim.x;
    }
    if (pos_begin < pos_end && pos_end > start.pos + (start.b1 - start.z)) atomicAdd(prm.deal_log + 3, 1);
  }
  struct TcItem { int g, z, t0, t1; bool half; const int32_t* tl; };
  auto get_item = [&](const TcWalk& w, TcItem& it) -> bool {
    it.g = w.g;
    it.z = w.z;
    it.half = half_padding(w.g);
    int cnt = prm.n_tiles;
    it.tl = nullptr;
    if (prm.tilelist) {
      const int f = prm.sp[it.g * TC_BC].fold;
      const int li = (f >= 0 && f < prm.n_lists - 1) ? f : prm.n_lists - 1;
      it.tl = prm.tilelist + (size_t)li * prm.n_tiles_ld;
      cnt = prm.tilecnt[li];
    }
    it.t0 = (int)((long long)cnt * it.z / TC_NCH);
    it.t1 = (int)((long long)cnt * (it.z + 1) / TC_NCH);
    return it.t1 > it.t0;       // empty chunks (fewer tiles than chunks) are skipped
  };
  auto sub_row0 = [&](const TcItem& it, int j) -> int {   // first row of sub-tile j of an item
    const int t = it.tl ? it.tl[it.t0 + (j >> 1)] : it.t0 + (j >> 1);
    return t * TC_R + (j & 1) * TC_SUB;
  };

  // Producer: one thread walks the same item sequence as the consumers (same skips, same sub-tile
  // order) and keeps the ring full across item boundaries.  Sub-tile k (running count) goes to stage
  // k % NS once both consumers are done with sub-tile k - NS; a new group's W is loaded once both
  // consumers are done with the previous group's.
  if (wg == 0) {
    setmaxnreg_dec<TC_PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      uint32_t k = 0;
      int w_loads = 0, g_prev = -1;
      for (TcWalk u = start; u.pos < pos_end; next_unit(u)) {
        TcItem it;
        if (!get_item(u, it)) continue;
        if (it.g != g_prev) {
          if (w_loads > 0) mbar_wait(&bars->w_free, (w_loads - 1) & 1, 120);
          mbar_expect_tx(&bars->w_full, SM::W_BYTES);
#pragma unroll
          for (int c = 0; c < NCHUNK; ++c) {
            tma_load_2d(s_wh + c * SM::W_CHUNK, &map_wh, c * 64, it.g * TC_BC, &bars->w_full);
            tma_load_2d(s_wl + c * SM::W_CHUNK, &map_wl, c * 64, it.g * TC_BC, &bars->w_full);
          }
          ++w_loads;
          g_prev = it.g;
        }
        const int nsub = 2 * (it.t1 - it.t0);
        for (int j = 0; j < nsub; ++j, ++k) {
          const uint32_t sl = k % NS;
          if (k >= (uint32_t)NS) mbar_wait(&bars->empty[sl], ((k / NS) - 1) & 1, 100);
          mbar_expect_tx(&bars->full[sl], SM::STAGE);
          const int r0 = sub_row0(it, j);
          uint8_t* dst = s_ring + sl * SM::STAGE;
#pragma unroll
          for (int c = 0; c < NCHUNK; ++c) {
            tma_load_2d(dst + c * SM::X_CHUNK, &map_xh, c * 64, r0, &bars->full[sl]);
            tma_load_2d(dst + (NCHUNK + c) * SM::X_CHUNK, &map_xl, c * 64, r0, &bars->full[sl]);
          }
        }
      }
    }
    return;
  }
  setmaxnreg_inc<TC_CONSUMER_REGS>();

  // Consumers take turns on the tensor cores (named barriers 1 and 2, one per consumer): a turn is
  // the issue of one sub-tile's products (see the sub-tile loop) and hands over to the other consumer,
  // so one consumer's epilogue runs while the other's products are in flight.  Both consumers walk
  // the same sub-tiles, so they take the same number of turns; consumer 0 takes the first.
  const uint32_t bar_mine = 1 + cw, bar_other = 2 - cw;
  auto turn_begin = [&] { named_bar_sync(bar_mine, 256); };
  auto turn_end = [&] { named_bar_arrive(bar_other, 256); };
  if (cw == 1) named_bar_arrive(1, 256);

  // accumulator fragments (wgmma m64nN): register i of a thread holds row 16 (warp & 3) + lane / 4
  // + 8 ((i >> 1) & 1) of its warpgroup's 64 slots and column 8 (i >> 2) + 2 (lane & 3) + (i & 1)
  const int slot_in_wg = (warp & 3) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  constexpr float INV_G = 1.f / GSCALE;
  const uint64_t desc_w = make_desc(smem_u32(s_wh), 16, 1024) + (uint64_t)((cw * 64 * 128) >> 4);
  const uint64_t desc_k = make_desc(smem_u32(s_ring), 16, 1024);              // X as K-major (GEMM1)
  const uint64_t desc_mn = make_desc(smem_u32(s_ring), SM::X_CHUNK, 1024);    // X as MN-major (GEMM2)
  constexpr uint32_t WL_OFF = (NCHUNK * SM::W_CHUNK) >> 4;
  constexpr uint32_t XL_OFF = (NCHUNK * SM::X_CHUNK) >> 4;

  uint32_t h = 0;          // running sub-tile counter (ring position), identical in both consumers
  int w_loads = 0, g_prev = -1;
  for (TcWalk u = start; u.pos < pos_end; next_unit(u)) {
    TcItem it;
    if (!get_item(u, it)) continue;
    const int g = it.g, z_part = it.z;
    const int nsub = 2 * (it.t1 - it.t0);
    if (g != g_prev) {
      // every product of the previous group has completed (each sub-tile ends in wgmma_wait_all):
      // release its W, then wait for this group's
      if (g_prev >= 0 && wg_leader) mbar_arrive(&bars->w_free);
      mbar_wait(&bars->w_full, (w_loads++) & 1, 200);
      g_prev = g;
    }
    if (cw == 1 && it.half) {
      // all 64 slots of this warpgroup are padding: no products, no epilogue, no partials.  It still
      // takes its turns (so the other consumer's hand-overs complete) and releases every stage once
      // the stage is loaded (the ring's phases then stay in step with the producer's).
      for (int j = 0; j < nsub; ++j) {
        const uint32_t hh = h + j, sl = hh % NS;
        mbar_wait(&bars->full[sl], (hh / NS) & 1, 211);
        turn_begin();
        turn_end();
        if (wg_leader) mbar_arrive(&bars->empty[sl]);
      }
      if (IS_FIT) { turn_begin(); turn_end(); }   // the turn of the item's last GEMM2
      h += nsub;
      continue;
    }

    // the two slots of this thread
    TcSlotParam sp[2];
    bool valid[2];
    int slot[2];
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      slot[s] = g * TC_BC + cw * 64 + slot_in_wg + 8 * s;
      valid[s] = slot[s] < n_live;
      sp[s].inv_t = 1.f; sp[s].bias = 0.f; sp[s].fold = -1; sp[s].pos = -1; sp[s].neg1 = 0; sp[s].col = -1;
      if (valid[s]) sp[s] = prm.sp[slot[s]];
    }
    // fit: work on z / 2^14 so that (row sign * 2^14) * z' = +-z and (row sign * 2^14) * sigma is
    // the scaled gradient entry; all power-of-two factors, results identical to the unscaled form
    float zi[2], zb0[2];
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      zi[s] = IS_FIT ? sp[s].inv_t * INV_G : sp[s].inv_t;
      zb0[s] = IS_FIT ? sp[s].bias * INV_G : sp[s].bias;
    }
    float2 cwt[2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};   // class weights of the two slots
    if constexpr (WEIGHTED) {
#pragma unroll
      for (int s = 0; s < 2; ++s)
        if (sp[s].col >= 0) cwt[s] = __ldg(prm.cw + sp[s].col);
    }
    const float* rsg = nullptr;
    if (UNI) {
      const int f = prm.sp[g * TC_BC].fold;
      const int li = (f >= 0 && f < prm.n_lists - 1) ? f : prm.n_lists - 1;
      rsg = prm.rowsg + (size_t)li * prm.rowsg_ld;
    }
    float grad[IS_FIT ? NCHUNK * 32 : 1];
#pragma unroll
    for (int i = 0; i < (IS_FIT ? NCHUNK * 32 : 1); ++i) grad[i] = 0.f;
    // per-item sums as compensated fp32 pairs (TwoSum)
    float ls_hi[2] = {0.f, 0.f}, ls_lo[2] = {0.f, 0.f}, gs_hi[2] = {0.f, 0.f}, gs_lo[2] = {0.f, 0.f};
    unsigned long long n_ok[2] = {0, 0}, n_all[2] = {0, 0};

    // GEMM1 of a sub-tile: Z = W_hi X_hi + W_lo X_hi + W_hi X_lo   [64 slots x 32 rows per warpgroup]
    auto gemm1 = [&](float (&zf)[16], uint32_t stage) {
      const uint64_t bx = desc_k + (uint64_t)((stage * SM::STAGE) >> 4);
#pragma unroll
      for (int ks = 0; ks < NCHUNK * 4; ++ks) {
        const uint32_t aoff = ((ks >> 2) * SM::W_CHUNK + (ks & 3) * 32) >> 4;
        const uint32_t boff = ((ks >> 2) * SM::X_CHUNK + (ks & 3) * 32) >> 4;
        wgmma_m64n32_ss(zf, desc_add(desc_w, aoff), desc_add(bx, boff), ks > 0 ? 1u : 0u);
        wgmma_m64n32_ss(zf, desc_add(desc_w, WL_OFF + aoff), desc_add(bx, boff), 1u);
        wgmma_m64n32_ss(zf, desc_add(desc_w, aoff), desc_add(bx, XL_OFF + boff), 1u);
      }
      wgmma_commit();
    };
    // GEMM2 of a sub-tile: dW += G_hi X_hi + G_lo X_hi + G_hi X_lo   [64 slots x dpad per warpgroup],
    // one batch with every A fragment formed beforehand
    auto gemm2 = [&](const uint32_t (&ahi)[2][4], const uint32_t (&alo)[2][4], uint32_t stage) {
      if constexpr (IS_FIT) {
        const uint64_t bm = desc_mn + (uint64_t)((stage * SM::STAGE) >> 4);
        const uint64_t bh0 = bm, bh1 = bm + (uint64_t)((16 * 128) >> 4);
        wgmma_grad<NCHUNK>(grad, ahi[0], bh0);
        wgmma_grad<NCHUNK>(grad, alo[0], bh0);
        wgmma_grad<NCHUNK>(grad, ahi[0], bh0 + XL_OFF);
        wgmma_grad<NCHUNK>(grad, ahi[1], bh1);
        wgmma_grad<NCHUNK>(grad, alo[1], bh1);
        wgmma_grad<NCHUNK>(grad, ahi[1], bh1 + XL_OFF);
        wgmma_commit();
      }
    };
    // Fit modes keep GEMM2 of sub-tile j - 1 in flight through the epilogue of sub-tile j: one turn
    // issues GEMM1 of j, then GEMM2 of j - 1 (A fragments and stage of j - 1 held in pa / pl / psl);
    // wgmma_wait_one waits for GEMM1 only.  The stage of j - 1 is released after the epilogue of j,
    // and the last GEMM2 of an item is issued in one more turn after the loop.
    uint32_t pa[2][4], pl[2][4], psl = 0;
    for (int j = 0; j < nsub; ++j) {
      const uint32_t hh = h + j, sl = hh % NS, ph = (hh / NS) & 1;
      const int r0 = sub_row0(it, j);
      mbar_wait(&bars->full[sl], ph, 210);

      float zf[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) zf[i] = 0.f;
      const uint32_t slu = __shfl_sync(0xffffffffu, sl, 0);   // warp-uniform copy: uniform-register descriptors
      reg_fence(zf);
      reg_fence(grad);
      turn_begin();
      // straight-line issue in every branch (no control flow between a wgmma_fence and its products,
      // so ptxas needs no warpgroup.arrive between the instructions)
      if (IS_FIT && j > 0) {
        wgmma_fence(); gemm1(zf, slu); gemm2(pa, pl, psl);
      } else {
        wgmma_fence(); gemm1(zf, slu);
      }
      turn_end();
      // per-row data of this thread's 8 rows (columns of the Z fragment), loaded while GEMM1 runs
      uint32_t rm[8];
      float yv[8];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int r = r0 + 8 * q + cq;
        if (UNI) {
          const float2 v = __ldg(reinterpret_cast<const float2*>(rsg + r));
          rm[2 * q] = __float_as_uint(v.x); rm[2 * q + 1] = __float_as_uint(v.y);
        } else {
          const uint2 v = __ldg(reinterpret_cast<const uint2*>(prm.rowmeta + r));
          rm[2 * q] = v.x; rm[2 * q + 1] = v.y;
        }
        if (MODE == TC_R2) {
          const float2 v = __ldg(reinterpret_cast<const float2*>(prm.yreal + r));
          yv[2 * q] = v.x; yv[2 * q + 1] = v.y;
        }
      }
      uint32_t ybw[2] = {0u, 0u}, mbw[2] = {0xFFFFFFFFu, 0xFFFFFFFFu};
      if (DECODE && (prm.ybits || prm.mbits)) {
#pragma unroll
        for (int s = 0; s < 2; ++s) {
          if (sp[s].col < 0) continue;
          const size_t wi = (size_t)sp[s].col * prm.rb_words + (size_t)(r0 / 32);   // one word = the 32 rows of this sub-tile
          if (prm.ybits) ybw[s] = __ldg(prm.ybits + wi);
          if (prm.mbits) mbw[s] = __ldg(prm.mbits + wi);
        }
      }
      if (IS_FIT && j > 0) wgmma_wait_one();
      else wgmma_wait_all();
      reg_fence(zf);

      if constexpr (IS_FIT) {
        float lt[2] = {0.f, 0.f}, gt[2] = {0.f, 0.f};
        float gv[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const int s = (i >> 1) & 1;
          const int rr = 2 * (i >> 2) + (i & 1);        // index into rm: row r0 + 8 (i >> 2) + cq + (i & 1)
          float sg;                       // -y * 2^14 for a training row, 0 otherwise
          if (UNI) {
            sg = __uint_as_float(rm[rr]);
          } else {
            const uint32_t m = rm[rr];
            const int fr = (int)(m >> 24);
            const int cls = (int)(m & 0x00FFFFFFu);
            bool yb = cls == sp[s].pos;
            bool train = (fr != 0xFF) && (fr != sp[s].fold) && (sp[s].neg1 == 0 || yb || cls == sp[s].neg1 - 1);
            {                                 // staged row bit matrices (multilabel targets, sampled negatives)
              const int bit = 8 * (i >> 2) + cq + (i & 1);
              if (prm.ybits) yb = (ybw[s] >> bit) & 1u;
              if (prm.mbits) train = train && ((mbw[s] >> bit) & 1u);
            }
            sg = train ? (yb ? -GSCALE : GSCALE) : 0.f;
          }
          // factor of the row's loss and gradient entry: sg times the class weight of the row's label
          // (label 1 exactly when sg < 0); the margin below keeps the unweighted sg
          const float sgw = WEIGHTED ? sg * (sg < 0.f ? cwt[s].y : cwt[s].x) : sg;
          const float zp = fmaf(zf[i], zi[s], zb0[s]);
          const float uu = sg * zp;       // = -y * z
          const float e = ex2_approx(-fabsf(uu) * 1.4426950408889634f);
          const float s1 = 1.f + e;
          const float loss = fmaf(lg2_approx(s1), 0.6931471805599453f, fmaxf(uu, 0.f));
          const float r = rcp_approx(s1);
          const float sig = (uu >= 0.f) ? r : e * r;
          gv[i] = sgw * sig;              // 2^14 * weight * dloss/dz
          lt[s] = fmaf(fabsf(sgw), loss, lt[s]);   // 2^14 * weight * loss
          gt[s] += gv[i];
        }
#pragma unroll
        for (int s = 0; s < 2; ++s) { two_sum_add(ls_hi[s], ls_lo[s], lt[s]); two_sum_add(gs_hi[s], gs_lo[s], gt[s]); }
        // G as the A operand of GEMM2 (k = the sub-tile's rows): the accumulator fragment of a
        // 16-column block is the A fragment of one k16 step; split into fp16 hi + lo
        uint32_t ahi[2][4], alo[2][4];
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int i = ks * 8 + (q >> 1) * 4 + (q & 1) * 2;
            const uint32_t hi = pack_f16x2(gv[i], gv[i + 1]);
            const float2 hf = unpack_f16x2(hi);
            ahi[ks][q] = hi;
            alo[ks][q] = pack_f16x2(gv[i] - hf.x, gv[i + 1] - hf.y);
          }
        }
        // GEMM2 of j - 1 has completed: release its stage, keep this sub-tile's fragments for the next turn
        if (j > 0) {
          wgmma_wait_all();
          reg_fence(grad);
          reg_hold(pa);
          reg_hold(pl);
          if (wg_leader) mbar_arrive(&bars->empty[psl]);
        }
#pragma unroll
        for (int ks = 0; ks < 2; ++ks)
#pragma unroll
          for (int q = 0; q < 4; ++q) { pa[ks][q] = ahi[ks][q]; pl[ks][q] = alo[ks][q]; }
        psl = slu;
      } else {
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const int s = (i >> 1) & 1;
          const int rr = 2 * (i >> 2) + (i & 1);
          const uint32_t m = rm[rr];
          const float zv = fmaf(zf[i], zi[s], zb0[s]);
          const int fr = (int)(m >> 24);
          const bool in = (fr != 0xFF) && score_code_selects(sp[s].fold, fr);
          if (MODE == TC_R2) {
            const float r = yv[rr] - zv;
            if (in) two_sum_add(ls_hi[s], ls_lo[s], r * r);
          } else {
            const bool yb = (int)(m & 0x00FFFFFFu) == sp[s].pos;
            n_ok[s] += (in && ((zv > 0.f) == yb)) ? 1 : 0;
          }
          n_all[s] += in ? 1 : 0;
        }
        if (wg_leader) mbar_arrive(&bars->empty[sl]);
      }
    }
    h += nsub;
    if constexpr (IS_FIT) {   // the item's last GEMM2 (nsub >= 2: empty chunks are skipped)
      reg_fence(grad);
      turn_begin();
      wgmma_fence(); gemm2(pa, pl, psl);
      turn_end();
      wgmma_wait_all();
      reg_fence(grad);
      reg_hold(pa);
      reg_hold(pl);
      if (wg_leader) mbar_arrive(&bars->empty[psl]);
    }

    // end of item: the four lanes sharing a slot hold partial sums of it; combine them in a fixed
    // order (deterministic) and write this chunk's partial
    if (IS_FIT || MODE == TC_R2) {
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        double ls = (double)ls_hi[s] + (double)ls_lo[s];
        double gs = (double)gs_hi[s] + (double)gs_lo[s];
        ls += __shfl_xor_sync(0xffffffffu, ls, 1);
        gs += __shfl_xor_sync(0xffffffffu, gs, 1);
        ls += __shfl_xor_sync(0xffffffffu, ls, 2);
        gs += __shfl_xor_sync(0xffffffffu, gs, 2);
        if ((lane & 3) == 0 && valid[s]) {
          if (IS_FIT) {   // partial (z_part, slot) has exactly one writer
            prm.lossp[(size_t)z_part * prm.n_act + slot[s]] = ls * (double)INV_G;
            prm.gsump[(size_t)z_part * prm.n_act + slot[s]] = gs * (double)INV_G;
          } else {        // sum of squared residuals of chunk z_part (added in chunk order by tc_r2)
            prm.lossp[(size_t)z_part * prm.n_act + slot[s]] = ls;
          }
        }
      }
    }
    if (IS_FIT) {
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        if (!valid[s]) continue;
        float* dst = prm.gradp + ((size_t)z_part * prm.n_act + slot[s]) * prm.ldw + cq;
#pragma unroll
        for (int b = 0; b < NCHUNK * 8; ++b)
          *reinterpret_cast<float2*>(dst + 8 * b) = make_float2(grad[4 * b + 2 * s], grad[4 * b + 2 * s + 1]);
      }
    }
    if (MODE == TC_R2 || MODE == TC_SCORE) {
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        unsigned long long a = n_all[s], o = n_ok[s];
        a += __shfl_xor_sync(0xffffffffu, a, 1); o += __shfl_xor_sync(0xffffffffu, o, 1);
        a += __shfl_xor_sync(0xffffffffu, a, 2); o += __shfl_xor_sync(0xffffffffu, o, 2);
        if ((lane & 3) == 0 && valid[s] && a > 0) {
          if (MODE == TC_SCORE) atomicAdd(prm.correct + slot[s], o);
          atomicAdd(prm.count + slot[s], a);
        }
      }
    }
  }
  // consumer 1's last hand-over (or its opening one, if there was no work) is still pending on
  // consumer 0's barrier
  if (cw == 0) named_bar_sync(1, 256);
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

// 2-D fp16 row-major [rows x cols] tensor, box = [box_rows x 64 cols], 128B swizzle
int tc_make_map_2d(Ctx* c, CUtensorMap* map, const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return fail(c, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * sizeof(__half)};
  cuuint32_t box[2] = {64, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box,
                  estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char b[128];
    snprintf(b, sizeof(b), "cuTensorMapEncodeTiled failed (%d)", (int)r);
    return fail(c, b);
  }
  return 0;
}

bool tc_supported(const Ctx* c) { return c->d >= 1 && c->d <= 256; }

void tc_free(Ctx* c) {
  TcData& t = c->tc;
  if (t.Xh) cudaFree(t.Xh);
  if (t.Xl) cudaFree(t.Xl);
  if (t.rowmeta) cudaFree(t.rowmeta);
  if (t.yreal_pad) cudaFree(t.yreal_pad);
  if (t.tilelist) cudaFree(t.tilelist);
  if (t.tilecnt) cudaFree(t.tilecnt);
  if (t.rowsg) cudaFree(t.rowsg);
  if (t.xscale) cudaFree(t.xscale);
  if (t.gscale) cudaFree(t.gscale);
  t = TcData();
}

// Build (or refresh) the fp16-split copy of X and the per-row metadata.
int tc_prepare(Ctx* c) {
  TcData& t = c->tc;
  const int64_t n = c->n;
  const int d = (int)c->d, ldx = (int)c->ldx;
  const int dpad = (d + 63) / 64 * 64;
  const int64_t npad = (n + TC_R - 1) / TC_R * TC_R;
  if (!t.x_valid) {
    if (t.Xh && (t.dpad != dpad || t.npad != npad)) tc_free(c);   // same shape restaged: keep the buffers
    if (!t.Xh) {
      t.dpad = dpad;
      t.npad = npad;
      SKD_CUDA(c, cudaMalloc((void**)&t.Xh, (size_t)npad * dpad * sizeof(__half)));
      SKD_CUDA(c, cudaMalloc((void**)&t.Xl, (size_t)npad * dpad * sizeof(__half)));
      SKD_CUDA(c, cudaMalloc((void**)&t.rowmeta, (size_t)npad * sizeof(uint32_t)));
      SKD_CUDA(c, cudaMalloc((void**)&t.xscale, (size_t)dpad * sizeof(float)));
      SKD_CUDA(c, cudaMalloc((void**)&t.gscale, (size_t)dpad * sizeof(double)));
    }
    unsigned int* colmax;
    SKD_CUDA(c, cudaMalloc((void**)&colmax, (size_t)dpad * sizeof(unsigned int)));
    SKD_CUDA(c, cudaMemsetAsync(colmax, 0, (size_t)dpad * sizeof(unsigned int), c->stream));
    dim3 g1((d + 127) / 128, (unsigned)((n + 4095) / 4096));
    tc_colmax_kernel<<<g1, 128, 0, c->stream>>>(c->X, n, ldx, d, colmax);
    tc_scale_kernel<<<(dpad + 127) / 128, 128, 0, c->stream>>>(colmax, d, dpad, t.xscale, t.gscale);
    int64_t total = npad * dpad;
    tc_split_kernel<<<(unsigned)((total + 255) / 256), 256, 0, c->stream>>>(
        c->X, n, npad, ldx, d, dpad, t.xscale, (__half*)t.Xh, (__half*)t.Xl);
    c->launches += 3;
    SKD_CUDA(c, cudaGetLastError());
    SKD_CUDA(c, cudaStreamSynchronize(c->stream));
    cudaFree(colmax);
    if (tc_make_map_2d(c, &t.map_xh, t.Xh, (uint64_t)npad, (uint64_t)dpad, TC_SUB)) return 1;
    if (tc_make_map_2d(c, &t.map_xl, t.Xl, (uint64_t)npad, (uint64_t)dpad, TC_SUB)) return 1;
    t.x_valid = true;
    t.meta_valid = false;
  }
  if (!t.meta_valid) {
    if (!c->ycls && !c->yreal) return fail(c, "tc_prepare: neither labels nor targets staged");
    tc_rowmeta_kernel<<<(unsigned)((npad + 255) / 256), 256, 0, c->stream>>>(c->ycls, c->fold, n, npad,
                                                                            t.rowmeta);
    c->launches += 1;
    {  // per-fold tile lists: list f = tiles holding at least one row NOT in fold f; last list = all
      const int n_tiles = (int)(npad / TC_R);
      const int nf = (c->fold && c->n_folds <= 32 && (int64_t)c->h_fold.size() == n) ? c->n_folds : 0;
      std::vector<int32_t> hl((size_t)(nf + 1) * n_tiles), hc(nf + 1, 0);
      for (int tt = 0; tt < n_tiles; ++tt) {
        uint32_t mask = 0;
        const int64_t r1 = std::min<int64_t>(n, (int64_t)(tt + 1) * TC_R);
        if (nf) for (int64_t r = (int64_t)tt * TC_R; r < r1; ++r) mask |= 1u << c->h_fold[r];
        for (int f = 0; f < nf; ++f)
          if (mask & ~(1u << f)) hl[(size_t)f * n_tiles + hc[f]++] = tt;
        hl[(size_t)nf * n_tiles + hc[nf]++] = tt;
      }
      if (t.tilelist) { cudaFree(t.tilelist); t.tilelist = nullptr; }
      if (t.tilecnt) { cudaFree(t.tilecnt); t.tilecnt = nullptr; }
      SKD_CUDA(c, cudaMalloc((void**)&t.tilelist, hl.size() * 4));
      SKD_CUDA(c, cudaMalloc((void**)&t.tilecnt, hc.size() * 4));
      SKD_CUDA(c, cudaMemcpyAsync(t.tilelist, hl.data(), hl.size() * 4, cudaMemcpyHostToDevice, c->stream));
      SKD_CUDA(c, cudaMemcpyAsync(t.tilecnt, hc.data(), hc.size() * 4, cudaMemcpyHostToDevice, c->stream));
      SKD_CUDA(c, cudaStreamSynchronize(c->stream));
      t.min_list_tiles = n_tiles;
      for (int f = 0; f <= nf; ++f) t.min_list_tiles = std::min(t.min_list_tiles, (int)hc[f]);
      if (t.rowsg && t.n_lists != nf + 1) { cudaFree(t.rowsg); t.rowsg = nullptr; }
      t.n_lists = nf + 1;
      t.rowsg_valid = false;
    }
    if (c->yreal) {
      if (!t.yreal_pad) SKD_CUDA(c, cudaMalloc((void**)&t.yreal_pad, (size_t)npad * sizeof(float)));
      SKD_CUDA(c, cudaMemsetAsync(t.yreal_pad, 0, (size_t)npad * sizeof(float), c->stream));
      SKD_CUDA(c, cudaMemcpyAsync(t.yreal_pad, c->yreal, (size_t)n * sizeof(float), cudaMemcpyDeviceToDevice, c->stream));
    }
    SKD_CUDA(c, cudaGetLastError());
    t.meta_valid = true;
  }
  return 0;
}

int tc_export(Ctx* c, LogregWork& w, int n_act_upper, const double* xin, int fit_intercept) {
  TcData& t = c->tc;
  tc_export_kernel<<<n_act_upper, 128, 0, c->stream>>>(w.lb.vec, w.lb.stride, w.lb.slot, w.lb.n_act, (int)c->d,
                                                       t.dpad, t.xscale, (__half*)w.Wh, (__half*)w.Wl,
                                                       (TcSlotParam*)w.sp, xin, fit_intercept);
  c->launches += 1;
  SKD_CUDA(c, cudaGetLastError());
  return 0;
}

size_t tc_slot_param_bytes() { return sizeof(TcSlotParam); }
int tc_partials_per_slot() { return TC_NCH; }

template <int MODE>
static cudaError_t tc_launch(int nchunk, int grid, cudaStream_t st, const CUtensorMap& xh, const CUtensorMap& xl,
                             const CUtensorMap& wh, const CUtensorMap& wl, const TcParams& prm) {
  switch (nchunk) {
#define TC_CASE(N)                                                                                   \
  case N: {                                                                                          \
    constexpr size_t smem = TcSmem<N>::BYTES;                                                        \
    static bool attr = false;                                                                        \
    if (!attr) {                                                                                     \
      cudaError_t e = cudaFuncSetAttribute(tc_eval_kernel<N, MODE>,                                  \
                                           cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);  \
      if (e != cudaSuccess) return e;                                                                \
      attr = true;                                                                                   \
    }                                                                                                \
    tc_eval_kernel<N, MODE><<<grid, TC_THREADS, smem, st>>>(xh, xl, wh, wl, prm);                    \
    break;                                                                                           \
  }
    TC_CASE(1) TC_CASE(2) TC_CASE(3) TC_CASE(4)
#undef TC_CASE
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

static int tc_run(Ctx* c, LogregWork& w, int n_act, int mode, int* nz_used, unsigned long long* dcorrect,
                  unsigned long long* dcount) {
  TcData& t = c->tc;
  if (nz_used) *nz_used = 0;
  if (n_act <= 0) return 0;
  const int nchunk = t.dpad / 64;
  const int groups = (n_act + TC_BC - 1) / TC_BC;
  const int n_tiles = (int)(t.npad / TC_R);
  // Grid: one CTA per SM (fewer if there are fewer (group, chunk) units); every CTA makes its share
  // of the deal from the live slot count on the device (see the kernel), so the launch shape does not
  // depend on how stale the host's count is.
  const long long units = (long long)groups * TC_NCH;
  const int grid = (int)std::min<long long>(c->sm_count, units);
  const int nz = TC_NCH;
  if (mode == TC_FIT) {
    if ((int64_t)nz * n_act > w.cap_sc) return fail(c, "tc_eval: partial buffer too small");
    // every (chunk, slot) partial has exactly one writer; only chunks without tiles (fewer tiles
    // than chunks in some list) are never written and must read as zero
    if (t.min_list_tiles < TC_NCH) {
      SKD_CUDA(c, cudaMemsetAsync(w.lb.lossp, 0, (size_t)nz * n_act * sizeof(double), c->stream));
      SKD_CUDA(c, cudaMemsetAsync(w.lb.gsump, 0, (size_t)nz * n_act * sizeof(double), c->stream));
      SKD_CUDA(c, cudaMemsetAsync(w.lb.gradp, 0, (size_t)nz * n_act * w.lb.ldw * sizeof(float), c->stream));
    }
  }
  CUtensorMap map_wh, map_wl;
  if (tc_make_map_2d(c, &map_wh, w.Wh, (uint64_t)w.slots_pad_cap, (uint64_t)t.dpad, TC_BC)) return 1;
  if (tc_make_map_2d(c, &map_wl, w.Wl, (uint64_t)w.slots_pad_cap, (uint64_t)t.dpad, TC_BC)) return 1;
  TcParams prm;
  prm.sp = (const TcSlotParam*)w.sp;
  prm.rowmeta = t.rowmeta;
  prm.yreal = t.yreal_pad;
  prm.lossp = w.lb.lossp;
  prm.gsump = w.lb.gsump;
  prm.gradp = w.lb.gradp;
  prm.correct = dcorrect;
  prm.count = dcount;
  prm.n_act = n_act;
  prm.n_act_dev = (mode == TC_FIT) ? w.lb.n_act : nullptr;
  prm.groups = groups;
  prm.n_tiles = n_tiles;
  prm.ldw = w.lb.ldw;
  prm.ybits = mode == TC_FIT ? w.ybits : nullptr;
  prm.mbits = mode == TC_FIT ? w.mbits : nullptr;
  prm.rb_words = w.rb_words;
  prm.deal_log = mode == TC_FIT ? w.deal_log : nullptr;
  // TC_FIT_UNI reads a row's sign from the list of the group's fold, so it needs one list per staged
  // fold (tc_prepare builds them for at most 32 folds); otherwise TC_FIT decodes the fold per element
  const bool uni = mode == TC_FIT && w.lb.grouped && w.uni_pos >= 0 && c->ycls && !w.ybits && !w.mbits &&
                   t.n_lists == c->n_folds + 1;
  if (uni && (!t.rowsg_valid || t.rowsg_pos != w.uni_pos)) {
    if (!t.rowsg) SKD_CUDA(c, cudaMalloc((void**)&t.rowsg, (size_t)t.n_lists * t.npad * sizeof(float)));
    tc_rowsg_kernel<<<(unsigned)((t.npad + 255) / 256), 256, 0, c->stream>>>(c->ycls, c->fold, c->n, t.npad,
                                                                          t.n_lists, w.uni_pos, t.rowsg);
    c->launches += 1;
    SKD_CUDA(c, cudaGetLastError());
    t.rowsg_pos = w.uni_pos;
    t.rowsg_valid = true;
  }
  prm.rowsg = uni ? t.rowsg : nullptr;
  prm.rowsg_ld = t.npad;
  const bool lists = mode == TC_FIT && w.lb.grouped && t.tilelist;
  prm.tilelist = lists ? t.tilelist : nullptr;
  prm.tilecnt = lists ? t.tilecnt : nullptr;
  prm.n_lists = t.n_lists;
  prm.n_tiles_ld = n_tiles;
  if (mode == TC_R2 && !t.yreal_pad) return fail(c, "tc_r2: targets not staged");
  prm.cw = mode == TC_FIT ? w.cw : nullptr;
  const bool weighted = prm.cw != nullptr;
  cudaError_t e = (uni && weighted) ? tc_launch<TC_FIT_UNI_W>(nchunk, grid, c->stream, t.map_xh, t.map_xl, map_wh, map_wl, prm)
                  : uni ? tc_launch<TC_FIT_UNI>(nchunk, grid, c->stream, t.map_xh, t.map_xl, map_wh, map_wl, prm)
                  : (mode == TC_FIT && weighted) ? tc_launch<TC_FIT_W>(nchunk, grid, c->stream, t.map_xh, t.map_xl, map_wh, map_wl, prm)
                  : mode == TC_FIT ? tc_launch<TC_FIT>(nchunk, grid, c->stream, t.map_xh, t.map_xl, map_wh, map_wl, prm)
                  : mode == TC_SCORE ? tc_launch<TC_SCORE>(nchunk, grid, c->stream, t.map_xh, t.map_xl, map_wh, map_wl, prm)
                                     : tc_launch<TC_R2>(nchunk, grid, c->stream, t.map_xh, t.map_xl, map_wh, map_wl, prm);
  c->launches += 1;
  if (e != cudaSuccess) return fail(c, std::string("tc_eval launch: ") + cudaGetErrorString(e));
  if (nz_used) *nz_used = nz;
  return 0;
}

int tc_eval(Ctx* c, LogregWork& w, int n_act, int* nz_used) {
  return tc_run(c, w, n_act, TC_FIT, nz_used, nullptr, nullptr);
}

// Accuracy counts of n_act slots whose weights were exported with tc_export (sp.fold = scoring code).
int tc_score(Ctx* c, LogregWork& w, int n_act, int64_t* dcorrect, int64_t* dcount) {
  return tc_run(c, w, n_act, TC_SCORE, nullptr, (unsigned long long*)dcorrect, (unsigned long long*)dcount);
}

__global__ void tc_chunk_sum_kernel(const double* __restrict__ part, int n_act, double* __restrict__ out) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_act) return;
  double acc = 0.0;
  for (int z = 0; z < TC_NCH; ++z) acc += part[(size_t)z * n_act + s];
  out[s] = acc;
}

// Sum of squared residuals / row counts of n_act regression slots (sp.fold = scoring code).  The kernel
// writes one partial per (chunk, slot) into w.lb.lossp ([TC_NCH x n_act], zeroed by the caller: chunks
// without tiles are not written); they are added here in chunk order, so the sums do not depend on
// which CTA ran which chunk.
int tc_r2(Ctx* c, LogregWork& w, int n_act, double* dsse, int64_t* dcount) {
  if (tc_run(c, w, n_act, TC_R2, nullptr, nullptr, (unsigned long long*)dcount)) return 1;
  tc_chunk_sum_kernel<<<(n_act + 255) / 256, 256, 0, c->stream>>>(w.lb.lossp, n_act, dsse);
  c->launches += 1;
  SKD_CUDA(c, cudaGetLastError());
  return 0;
}

}  // namespace skd
