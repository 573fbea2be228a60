// forest_fast.cu -- the throughput build of the exact depth-first tree builder (classification,
// best splitter): every tree of a forest resident at once, seven 64-thread builders per SM.
//
// Same contract as forest.cu (which stays the general kernel: regression, random splitter, many
// classes): the host draws what the reference's per-tree task `_build_trees` draws
// (ref ensemble.py:68-109), the kernel replays
//   SK/tree/_tree.pyx:139-337      DepthFirstTreeBuilder.build
//   SK/tree/_splitter.pyx:262-504  node_split_best (one xorshift stream per tree, Fisher-Yates
//                                  feature draws, constant-feature bookkeeping, strict '>')
//   SK/tree/_criterion.pyx:605-680 Gini in float64, scikit-learn's operation order
// and the trees are bit-identical to scikit-learn's.
//
// Why a second kernel.  A config-4 tree (2M x 64, 1.26M distinct rows) has 372k nodes; 110k of its
// 184k internal nodes hold <= 32 samples and 58k more hold <= 256; the 1000 nodes above 4096
// samples carry half of all sample visits but none of the time.  The RNG stream makes the nodes of
// one tree strictly sequential, so throughput = (trees in flight) / (latency per node):
//   * 7 builders per SM (64 threads, up to 128 registers, 28 KB shared memory): all 1024 trees of the
//     headline forest run concurrently (the general kernel holds 2 per SM);
//   * a subtree of <= S samples (S = 256 at d = 64) is STAGED: the bin codes of its rows (row-major
//     copy of the binned matrix, 64 B per row) are copied to shared memory once, and the whole
//     subtree -- 9 nodes in 10 -- is then built without touching global memory except for the node
//     records it emits;
//   * staged nodes of <= 32 samples skip the 256-bin histogram: one warp ranks the node's samples of
//     a feature against each other (shuffle all-pairs count: left class weights and sample count of
//     every candidate threshold in one packed integer add per pair);
//   * larger staged nodes build packed 16-bit histograms (sum of <= 256 weights of <= 255 fits);
//   * nodes above S samples gather from the row-major codes (all drawn features of a sample sit in
//     the same 64 bytes) into 32-bit shared-memory histograms and ping-pong between two sample
//     buffers instead of copying the partition back.
// Requirements checked by the host (else forest.cu runs): n_classes <= 4, d <= 255, every feature's
// distinct values more than 1e-7 apart (then "constant" == one present bin and every pair of
// adjacent present bins is a candidate, SK/tree/_partitioner.pyx:210-214), n * 255 < 2^32.
// No tensor cores: integer histogramming and float64 Gini arithmetic.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "forest_common.h"
#include "skd_internal.h"

namespace skd {

// 7 builders x 64 threads per SM.  The register file is split over the four SM sub-partitions (16384
// registers each): 14 warps per SM are at most 4 per sub-partition, i.e. up to 128 registers per thread
// without spilling (96-thread builders are limited to 80 for seven per SM and spilled; 6 per SM means
// two waves for 1024 trees).
constexpr int FF_THREADS = 64;
constexpr int FF_WARPS = FF_THREADS / 32;
constexpr int FF_KB = 8;          // speculative feature draws per batch (unstaged nodes, small staged nodes)
constexpr int FF_KBM = 4;         // ... for staged histogram nodes (packed histograms of four features fit next to the rows)
constexpr int FF_SMAX = 256;      // staged rows at most (local ids are bytes, packed 16-bit sums must hold 256 x 255)
constexpr int FF_SSTK = 64;       // builder-stack entries kept in shared memory
constexpr int FF_SMALL = 32;      // staged nodes up to this size take the ranking path
constexpr double FF_EPSILON = 2.220446049250313e-16;

template <int CM>
struct __align__(8) FfRec {       // builder stack record (SK/tree/_tree.pyx StackRecord) + the node's class sums
  int32_t start, end, depth, parent;
  int32_t flags;                  // n_const [0,16) | is_left bit 16 | sample buffer bit 17
  uint32_t sums[CM];
  int32_t pad_;
  double impurity;
};
struct FfItem {                   // one speculatively drawn feature + the simulation state right after its draw
  int f, fj, nv, nd, fi, ulen;
  uint32_t rs;
  int pad_;
};
template <int CM>
struct __align__(8) FfResult {    // best split of one feature in the current node
  double proxy;                   // scikit-learn's float64 proxy of the split -- valid only if `exact`
  float ptil;                     // its float32 rank value sq_l / w_l + sq_r / w_r (-inf: no valid split)
  int exact;
  int n_left;
  int code;                       // bin_a | bin_b << 8 | is_const << 16
  uint32_t sl[CM];
};

// packed accumulators of the ranking path: class weights in 13-bit fields (32 samples x 255 < 2^13),
// the sample count above them
template <int CM> struct FfAcc { typedef unsigned long long T; static constexpr int CNT = 13 * CM; };
template <> struct FfAcc<2> { typedef unsigned int T; static constexpr int CNT = 26; };

__device__ __forceinline__ uint32_t ff_rand_r(uint32_t* seed) {   // SK/utils/_random.pxd:20-34
  if (*seed == 0) *seed = 1;
  *seed ^= (uint32_t)(*seed << 13);
  *seed ^= (uint32_t)(*seed >> 17);
  *seed ^= (uint32_t)(*seed << 5);
  return *seed % ((uint32_t)2147483647 + 1);
}
__device__ __forceinline__ int ff_rand_int(int low, int high, uint32_t* seed) {
  return low + (int)(ff_rand_r(seed) % (uint32_t)(high - low));
}

// The builder is latency-bound on ONE warp's instruction stream per tree (ncu: 44 % of the stall
// samples are instruction fetch when the kernel is unrolled to 130 KB), so everything below is written
// for a small instruction footprint: one out-of-line copy of the float64 expressions and of the
// histogram scan, rolled loops, shared-memory re-reads instead of unrolled register arrays.

// proxy_impurity_improvement of the Gini criterion for left sums sl, node sums st
// (SK/tree/_criterion.pyx:147-163, 650-680): -w_r * gini_r - w_l * gini_l, no FMA contraction
// (all operands by value: a pointer to a caller's register array would force that array -- and every
// update of it in the caller's loops -- into local memory)
struct FfProxy { double proxy, il, ir; };
__device__ __noinline__ FfProxy ff_proxy4(uint32_t l0, uint32_t l1, uint32_t l2, uint32_t l3,
                                          uint32_t t0, uint32_t t1, uint32_t t2, uint32_t t3, int C, double w_node) {
  const uint32_t l[4] = {l0, l1, l2, l3}, t[4] = {t0, t1, t2, t3};
  double sql = 0.0, sqr = 0.0, wl = 0.0;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    if (c < C) {
      const double a = (double)l[c], b = (double)(t[c] - l[c]);
      wl += a;
      sql = __dadd_rn(sql, __dmul_rn(a, a));
      sqr = __dadd_rn(sqr, __dmul_rn(b, b));
    }
  }
  const double wr = w_node - wl;
  FfProxy r;
  r.il = __dsub_rn(1.0, __ddiv_rn(sql, __dmul_rn(wl, wl)));
  r.ir = __dsub_rn(1.0, __ddiv_rn(sqr, __dmul_rn(wr, wr)));
  r.proxy = __dsub_rn(__dmul_rn(-wr, r.ir), __dmul_rn(wl, r.il));
  return r;
}
// Weighted builds (W): the class weights of the CTA's tree, set before the tree's first node.  Every weighted
// statistic is cw_c * (integer count) in float64.  The float32 rank value works on the weights scaled by the
// power of two ff_cwscale that brings the largest into [1/2, 1) (ranks, bars and w_node all carry the same
// exact factor; the host keeps the fast builder to weights within 2^40 of each other, so no float32
// product or square under- or overflows).
__shared__ double ff_cw[4];
__shared__ float ff_cwf[4];
__shared__ double ff_cwscale;

// ... the same proxy with class weights: sum_left[c] = cw_c * l_c, sum_right[c] = cw_c * t_c - sum_left[c]
// (ClassificationCriterion.update), w_l = sum_c sum_left[c], w_r = w_node - w_l
__device__ __noinline__ FfProxy ff_proxy4w(uint32_t l0, uint32_t l1, uint32_t l2, uint32_t l3,
                                           uint32_t t0, uint32_t t1, uint32_t t2, uint32_t t3, int C, double w_node) {
  const uint32_t l[4] = {l0, l1, l2, l3}, t[4] = {t0, t1, t2, t3};
  double sql = 0.0, sqr = 0.0, wl = 0.0;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    if (c < C) {
      const double a = __dmul_rn(ff_cw[c], (double)l[c]), b = __dsub_rn(__dmul_rn(ff_cw[c], (double)t[c]), a);
      wl = __dadd_rn(wl, a);
      sql = __dadd_rn(sql, __dmul_rn(a, a));
      sqr = __dadd_rn(sqr, __dmul_rn(b, b));
    }
  }
  const double wr = w_node - wl;
  FfProxy r;
  r.il = __dsub_rn(1.0, __ddiv_rn(sql, __dmul_rn(wl, wl)));
  r.ir = __dsub_rn(1.0, __ddiv_rn(sqr, __dmul_rn(wr, wr)));
  r.proxy = __dsub_rn(__dmul_rn(-wr, r.ir), __dmul_rn(wl, r.il));
  return r;
}
template <int CM, bool W>
__device__ __forceinline__ FfProxy ff_proxy(const uint32_t (&sl)[CM], const uint32_t* st, int C, double w_node) {
  if constexpr (W)
    return ff_proxy4w(sl[0], CM > 1 ? sl[1] : 0u, CM > 2 ? sl[2] : 0u, CM > 3 ? sl[3] : 0u,
                      st[0], CM > 1 ? st[1] : 0u, CM > 2 ? st[2] : 0u, CM > 3 ? st[3] : 0u, C, w_node);
  return ff_proxy4(sl[0], CM > 1 ? sl[1] : 0u, CM > 2 ? sl[2] : 0u, CM > 3 ? sl[3] : 0u,
                   st[0], CM > 1 ? st[1] : 0u, CM > 2 ? st[2] : 0u, CM > 3 ? st[3] : 0u, C, w_node);
}

// float32 rank value of a split: sq_l / w_l + sq_r / w_r (= proxy + w_node in exact arithmetic; the
// float32 value is within 2^-20 * w_node of it).  Candidates, features and batches are compared on it;
// scikit-learn's float64 expression is evaluated only for values within FF_BAR * w_node of each other.
// Weighted: a_c = cw_c l_c and b_c = cw_c r_c in float32 (scaled cw_c), w_l = sum a_c, w_r = sum b_c (no
// cancellation against w_node): within 2^-18 * w_node, bar FF_BAR_W (DESIGN.md §4).
constexpr float FF_BAR = 1.9073486328125e-6f;      // 2^-19
constexpr float FF_BAR_W = 7.62939453125e-6f;      // 2^-17
template <int CM, bool W>
__device__ __forceinline__ float ff_rank(const uint32_t* sl, const uint32_t* st, int C, float w_node) {
  float wl = 0.f, sql = 0.f, sqr = 0.f;
  if constexpr (W) {
    float wr = 0.f;
#pragma unroll
    for (int c = 0; c < CM; ++c) if (c < C) {
      const float a = __fmul_rn(ff_cwf[c], (float)sl[c]), b = __fmul_rn(ff_cwf[c], (float)(st[c] - sl[c]));
      wl += a; wr += b; sql = fmaf(a, a, sql); sqr = fmaf(b, b, sqr);
    }
    return __fdividef(sql, wl) + __fdividef(sqr, wr);
  }
#pragma unroll
  for (int c = 0; c < CM; ++c) if (c < C) { const float a = (float)sl[c], b = (float)(st[c] - sl[c]); wl += a; sql = fmaf(a, a, sql); sqr = fmaf(b, b, sqr); }
  return __fdividef(sql, wl) + __fdividef(sqr, w_node - wl);
}
template <int CM, bool W>
__device__ __forceinline__ bool ff_weights_ok(const uint32_t* sl, int C, double w_node, double min_weight_leaf) {
  if (!(min_weight_leaf > 0.0)) return true;
  double wl = 0.0;
#pragma unroll
  for (int c = 0; c < CM; ++c) if (c < C) {
    if constexpr (W) wl = __dadd_rn(wl, __dmul_rn(ff_cw[c], (double)sl[c]));
    else wl += (double)sl[c];
  }
  return !(wl < min_weight_leaf || w_node - wl < min_weight_leaf);
}

// One warp scans the 256 bins of one feature's histogram (8 bins per lane, ascending) and leaves the
// feature's best split in *R.  Two histogram layouts: packed = 0: H[c][256] class weights (32-bit) then
// [256] sample counts; packed = 1: class pairs in 16-bit halves H[c / 2][256], then sample counts, two
// bins per word, from word `hcw`.  st = the node's class sums (shared memory).
template <int CM, bool W>
__device__ __noinline__ void ff_scan(const unsigned int* H, int packed, int hcw, int lane, int C, int n_node,
                                     const uint32_t* st, double w_node, int min_samples_leaf,
                                     double min_weight_leaf, FfResult<CM>* R) {
  auto hn = [&](int b) -> unsigned {
    return packed ? (H[hcw + (b >> 1)] >> ((b & 1) * 16)) & 0xFFFFu : H[C * 256 + b];
  };
  auto hc = [&](int c, int b) -> uint32_t {
    return packed ? (H[(c >> 1) * 256 + b] >> ((c & 1) * 16)) & 0xFFFFu : H[c * 256 + b];
  };
  unsigned ltot = 0, pmask = 0;
  uint32_t sl[CM];       // class weights of this lane's bins, then: left of this lane's first bin
#pragma unroll
  for (int c = 0; c < CM; ++c) sl[c] = 0;
#pragma unroll 2
  for (int j = 0; j < 8; ++j) {
    const unsigned cj = hn(lane * 8 + j);
    ltot += cj;
    if (cj) pmask |= 1u << j;
#pragma unroll
    for (int c = 0; c < CM; ++c) if (c < C) sl[c] += hc(c, lane * 8 + j);
  }
  unsigned pre = ltot;   // exclusive prefix of the sample counts over lanes
#pragma unroll 1
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned v = __shfl_up_sync(0xffffffffu, pre, o);
    if (lane >= o) pre += v;
#pragma unroll
    for (int c = 0; c < CM; ++c) {
      const uint32_t u = __shfl_up_sync(0xffffffffu, sl[c], o);
      if (lane >= o) sl[c] += u;
    }
  }
  pre -= ltot;
#pragma unroll
  for (int c = 0; c < CM; ++c) sl[c] = __shfl_up_sync(0xffffffffu, sl[c], 1);     // inclusive -> exclusive
  if (lane == 0) {
#pragma unroll
    for (int c = 0; c < CM; ++c) sl[c] = 0;
  }
  // first present bin of the lanes above this one
  const int myfirst = pmask ? lane * 8 + __ffs(pmask) - 1 : 1 << 20;
  int run = myfirst;
#pragma unroll 1
  for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_down_sync(0xffffffffu, run, o); if (lane + o < 32) run = min(run, u); }
  const int nx = __shfl_down_sync(0xffffffffu, run, 1);
  const int nxt = lane < 31 ? nx : (1 << 20);
  const int gfirst = __reduce_min_sync(0xffffffffu, myfirst);
  const int mylast = pmask ? lane * 8 + 31 - __clz(pmask) : -1;
  const int glast = __reduce_max_sync(0xffffffffu, mylast);
  const bool is_const = glast <= gfirst;      // distinct values are > 1e-7 apart (host check): one bin == constant
  const float wnf = W ? (float)(w_node * ff_cwscale) : (float)w_node;
  // pass 1: float32 rank value of every candidate of this lane: its best and second best
  float pbest = -INFINITY, psecond = -INFINITY;
  if (!is_const) {
    unsigned run_cnt = pre;
    uint32_t s2[CM];
#pragma unroll
    for (int c = 0; c < CM; ++c) s2[c] = sl[c];
    unsigned pm = pmask;
    while (pm) {                               // this lane's present bins in ascending order
      const int j = __ffs(pm) - 1;
      pm &= pm - 1;
      run_cnt += hn(lane * 8 + j);
#pragma unroll
      for (int c = 0; c < CM; ++c) if (c < C) s2[c] += hc(c, lane * 8 + j);
      if (!pm && nxt >= (1 << 20)) break;       // last present bin of the node: no boundary above it
      const int n_left = (int)run_cnt;
      if (n_left < min_samples_leaf || n_node - n_left < min_samples_leaf) continue;
      if (!ff_weights_ok<CM, W>(s2, C, w_node, min_weight_leaf)) continue;   // exact test: an invalid candidate must not set the bar
      const float pt = ff_rank<CM, W>(s2, st, C, wnf);
      if (pt > pbest) { psecond = pbest; pbest = pt; }
      else if (pt > psecond) psecond = pt;
    }
  }
  float pmax = pbest;
#pragma unroll 1
  for (int o = 16; o > 0; o >>= 1) pmax = fmaxf(pmax, __shfl_xor_sync(0xffffffffu, pmax, o));
  if (!(pmax > -INFINITY)) {
    if (lane == 0) { R->proxy = -INFINITY; R->ptil = -INFINITY; R->exact = 1; R->n_left = 1 << 30; R->code = is_const ? (1 << 16) : 0; }
    return;
  }
  const float pthr = pmax - wnf * (W ? FF_BAR_W : FF_BAR);
  // Is the best candidate alone within the bar?  (a lane's best and second best tell "none", "one" or
  // "several" of its candidates are near)
  const int nnear = (pbest >= pthr ? 1 : 0) + (psecond >= pthr ? 1 : 0);
  const bool single = __reduce_add_sync(0xffffffffu, (unsigned)nnear) == 1u;
  // pass 2 (lanes with a near candidate): the winner's position, bins and left sums; float64 proxies only
  // when several candidates are within the bar (ties then go to the smallest position, as the
  // sequential scan's strict '>' does)
  double bproxy = -INFINITY;
  float bpt = -INFINITY;
  int bnl = 1 << 30, bcode = 0;
  uint32_t bsl[CM];
#pragma unroll
  for (int c = 0; c < CM; ++c) bsl[c] = 0;
  if (nnear > 0) {
    unsigned run_cnt = pre;
    unsigned pm = pmask;
    while (pm) {
      const int j = __ffs(pm) - 1;
      pm &= pm - 1;
      run_cnt += hn(lane * 8 + j);
#pragma unroll
      for (int c = 0; c < CM; ++c) if (c < C) sl[c] += hc(c, lane * 8 + j);
      if (!pm && nxt >= (1 << 20)) break;
      const int n_left = (int)run_cnt;
      if (n_left < min_samples_leaf || n_node - n_left < min_samples_leaf) continue;
      if (!ff_weights_ok<CM, W>(sl, C, w_node, min_weight_leaf)) continue;
      const float pt = ff_rank<CM, W>(sl, st, C, wnf);
      if (!(pt >= pthr)) continue;
      const double proxy = single ? 0.0 : ff_proxy<CM, W>(sl, st, C, w_node).proxy;
      if (single || proxy > bproxy) {
        const int nb2 = pm ? lane * 8 + __ffs(pm) - 1 : nxt;
        bproxy = proxy; bpt = pt; bnl = n_left; bcode = (lane * 8 + j) | (nb2 << 8);
#pragma unroll
        for (int c = 0; c < CM; ++c) bsl[c] = sl[c];
      }
    }
  }
  bool writer = single && nnear > 0;
  if (!single) {
    double wp = bproxy; int wnl = bnl;
#pragma unroll 1
    for (int o = 16; o > 0; o >>= 1) {
      const double op = __shfl_xor_sync(0xffffffffu, wp, o);
      const int onl = __shfl_xor_sync(0xffffffffu, wnl, o);
      if (op > wp || (op == wp && onl < wnl)) { wp = op; wnl = onl; }
    }
    writer = bnl == wnl && bproxy == wp && wp > -INFINITY;   // exactly one lane: positions are unique per bin
  }
  if (writer) {
    R->proxy = bproxy; R->ptil = bpt; R->exact = single ? 0 : 1; R->n_left = bnl; R->code = bcode;
#pragma unroll
    for (int c = 0; c < CM; ++c) R->sl[c] = bsl[c];
  }
}

#define FF_TICK(ph) do { if (P.o_prof && tid == 0) { const long long _t = clock64(); s_prof[ph] += _t - tlast; tlast = _t; } } while (0)

// W: class weights.  The counts, histograms, records and the partition are those of the unweighted build;
// the float64 statistics are cw_c * count (ff_proxy4w) and the float32 rank takes the weighted bar.
template <int CM, bool W>
__global__ void __launch_bounds__(FF_THREADS, 7)
forest_fast_kernel(const FfParams P) {
  typedef typename FfAcc<CM>::T acc_t;
  constexpr int CNT = FfAcc<CM>::CNT;
  constexpr int MP = (FF_SMAX + FF_THREADS - 1) / FF_THREADS;   // passes of the staged partition
  const int slot = blockIdx.x;
  if (slot >= P.n_trees) return;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int C = P.n_classes, d = P.d, dp = P.dp;
  const int64_t n = P.n;

  // ---- shared memory ----
  extern __shared__ __align__(16) unsigned char ff_sm[];
  unsigned int* U = reinterpret_cast<unsigned int*>(ff_sm);                  // FF_UW words, see below
  FfRec<CM>* sstack = reinterpret_cast<FfRec<CM>*>(U + FF_UW);               // [FF_SSTK + 1]; the last one: spill copy
  FfItem* items = reinterpret_cast<FfItem*>(sstack + FF_SSTK + 1);           // [FF_KB]
  FfResult<CM>* results = reinterpret_cast<FfResult<CM>*>(items + FF_KB);    // [FF_KB]
  double* s_dbl = reinterpret_cast<double*>(results + FF_KB);                // [4]
  long long* s_prof = reinterpret_cast<long long*>(s_dbl + 4);               // [16]
  int* s_ctrl = reinterpret_cast<int*>(s_prof + 16);                         // [16]
  int* wsum = s_ctrl + 16;                                                   // [64]
  uint32_t* best_sl = reinterpret_cast<uint32_t*>(wsum + 64);                // [4]
  uint8_t* features = reinterpret_cast<uint8_t*>(best_sl + 4);               // [d]
  uint8_t* constant_features = features + ((d + 3) & ~3);                    // [d]
  uint8_t* undo = constant_features + ((d + 3) & ~3);                        // [2 * (d + 16)] swap log of the draws
  // U, unstaged nodes: hist[k][c][256] class weights (c < C) then [256] sample counts, 32-bit
  const int hstrideA = (C + 1) * 256;
  const int KBA = min(FF_KB, FF_UW / hstrideA);
  // U, staged subtree: rows[S][ws] bin codes | histB[FF_KBM][hbw] packed 16-bit | ord[S] u8 | wcls[S] u16
  const int S = P.stage_rows, ws4 = P.stage_ws * 4;
  const int hcw = 256 * ((C + 1) >> 1);          // packed class-pair words per feature
  const int hbw = hcw + 128;                     // + packed sample counts
  const uint8_t* rowsB = reinterpret_cast<const uint8_t*>(U);
  unsigned int* histB = U + S * P.stage_ws;
  uint8_t* ord = reinterpret_cast<uint8_t*>(histB + FF_KBM * hbw);
  uint16_t* wcls = reinterpret_cast<uint16_t*>(ord + S);
  long long tlast = 0;
  if (tid < 16) s_prof[tid] = 0;

  // ---- initialise the tree: samples with non-zero weight in ascending order (Splitter.init) ----
  for (int i = tid; i < d; i += FF_THREADS) features[i] = (uint8_t)i;
  if (tid < 4) best_sl[tid] = 0;
  // balanced_subsample: 1 until the root's class sums give the weights (only absent classes get 0)
  if constexpr (W) if (tid < 4) ff_cw[tid] = P.cw_bs || tid >= C ? 1.0 : P.cw[tid];
  __syncthreads();
  int n_nz = 0;
  {
    const uint8_t* cnt = P.counts + (size_t)slot * n;
    uint2* dst = P.samp + (size_t)slot * n;
    uint32_t s0 = 0, s1 = 0, s2 = 0, s3 = 0;      // class sums of this thread (CM <= 4)
    int base = 0;
    for (int64_t i0 = 0; i0 < n; i0 += FF_THREADS * 4) {
      unsigned w4[4], y4[4];
      int rk4[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int64_t i = i0 + q * FF_THREADS + tid;
        w4[q] = 0; y4[q] = 0;
        if (i < n) { w4[q] = cnt[i]; y4[q] = (unsigned)P.ycls[i]; }
        if constexpr (W) if (ff_cw[y4[q]] == 0.0) w4[q] = 0;     // rows of weight 0 leave the tree (Splitter.init)
        const unsigned bal = __ballot_sync(0xffffffffu, w4[q] != 0);
        if (lane == 0) wsum[q * FF_WARPS + wid] = __popc(bal);
        rk4[q] = __popc(bal & ((1u << lane) - 1));
      }
      __syncthreads();
      int tot = 0;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
#pragma unroll
        for (int k = 0; k < FF_WARPS; ++k) {
          if (k == wid) rk4[q] += tot;
          tot += wsum[q * FF_WARPS + k];
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (w4[q] != 0) {
          const int64_t i = i0 + q * FF_THREADS + tid;
          dst[base + rk4[q]] = make_uint2((unsigned)i, (w4[q] << 8) | y4[q]);
          s0 += y4[q] == 0 ? w4[q] : 0; s1 += y4[q] == 1 ? w4[q] : 0;
          if (CM > 2) { s2 += y4[q] == 2 ? w4[q] : 0; s3 += y4[q] == 3 ? w4[q] : 0; }
        }
      }
      base += tot;
      __syncthreads();
    }
    n_nz = base;
    for (int o = 16; o > 0; o >>= 1) {
      s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      if (CM > 2) { s2 += __shfl_xor_sync(0xffffffffu, s2, o); s3 += __shfl_xor_sync(0xffffffffu, s3, o); }
    }
    if (lane == 0) {
      atomicAdd(&best_sl[0], s0); atomicAdd(&best_sl[1], s1);
      if (CM > 2) { atomicAdd(&best_sl[2], s2); atomicAdd(&best_sl[3], s3); }
    }
  }
  __syncthreads();
  double w_samples = 0.0;          // weighted_n_samples (integer valued)
  if constexpr (W) {
    if (P.cw_bs) {   // compute_class_weight("balanced") of the bootstrap sample: n / (K_present * N_c)
      if (tid < C) {
        uint32_t nt = 0; int kp = 0;
        for (int c = 0; c < C; ++c) { nt += best_sl[c]; kp += best_sl[c] != 0; }
        ff_cw[tid] = best_sl[tid] ? __ddiv_rn((double)nt, __dmul_rn((double)kp, (double)best_sl[tid])) : 0.0;
      }
      __syncthreads();
    }
    if (tid == 0) {
      double mx = 0.0;
      for (int c = 0; c < C; ++c) mx = fmax(mx, ff_cw[c]);
      int e = 0;
      frexp(mx, &e);
      ff_cwscale = ldexp(1.0, -e);
    }
    __syncthreads();
    if (tid < 4) ff_cwf[tid] = (float)(ff_cw[tid] * ff_cwscale);
#pragma unroll
    for (int c = 0; c < CM; ++c) if (c < C) w_samples = __dadd_rn(w_samples, __dmul_rn(ff_cw[c], (double)best_sl[c]));
  } else {
#pragma unroll
    for (int c = 0; c < CM; ++c) if (c < C) w_samples += (double)best_sl[c];
  }
  // BaseDecisionTree._fit: min_weight_leaf = min_weight_fraction_leaf * sum(sample_weight)
  const double mwl_w = W ? __dmul_rn(P.min_weight_fraction, w_samples) : 0.0;
#define MIN_WEIGHT_LEAF (W ? mwl_w : P.min_weight_leaf)

  uint32_t rstate = P.rand_state[slot];
  int sp = 0, node_count = 0, max_depth_seen = -1, status = 0;
  int st_base = 0, st_end = -1;    // sample range of the staged subtree (empty)
  if (tid == 0) {
    FfRec<CM> r;
    r.start = 0; r.end = n_nz; r.depth = 0; r.parent = -1; r.flags = 0; r.pad_ = 0;
    r.impurity = INFINITY;
#pragma unroll
    for (int c = 0; c < CM; ++c) r.sums[c] = c < C ? best_sl[c] : 0;
    sstack[0] = r;
  }
  sp = 1;
  bool first = true;
  __syncthreads();
  if (P.o_prof) tlast = clock64();

  while (sp > 0 && status == 0) {
    --sp;
    // the popped record is read in place (its stack slot is only overwritten by this node's own push,
    // after the last read); records beyond the shared part of the stack come back through the spill copy
    if (sp >= FF_SSTK) {
      if (tid == 0) sstack[FF_SSTK] = (reinterpret_cast<const FfRec<CM>*>(P.stack) + (size_t)slot * P.stack_cap)[sp];
      __syncthreads();
    }
    const FfRec<CM>* rec = &sstack[sp < FF_SSTK ? sp : FF_SSTK];
    const int start = rec->start, end = rec->end, depth = rec->depth;
    const int n_node = end - start;
    const int n_known = rec->flags & 0xFFFF;
    double w_node = 0.0;
#pragma unroll
    for (int c = 0; c < CM; ++c) if (c < C) {
      if constexpr (W) w_node = __dadd_rn(w_node, __dmul_rn(ff_cw[c], (double)rec->sums[c]));
      else w_node += (double)rec->sums[c];
    }
    double impurity = rec->impurity;
    bool is_leaf = depth >= P.max_depth || n_node < P.min_samples_split || n_node < 2 * P.min_samples_leaf ||
                   w_node < 2.0 * MIN_WEIGHT_LEAF;
    if (first) {   // root: node_impurity()  (SK/tree/_criterion.pyx:620-640)
      double sq = 0.0;
#pragma unroll
      for (int c = 0; c < CM; ++c) if (c < C) {
        const double a = W ? __dmul_rn(ff_cw[c], (double)rec->sums[c]) : (double)rec->sums[c];
        sq = __dadd_rn(sq, __dmul_rn(a, a));
      }
      impurity = __dsub_rn(1.0, __ddiv_rn(sq, __dmul_rn(w_node, w_node)));
      first = false;
    }
    is_leaf = is_leaf || impurity <= FF_EPSILON;
    FF_TICK(0);

    int best_feature = 0, best_nl = -1, best_code = 0, n_total_constants = n_known;
    bool staged = false;
    if (!is_leaf) {
      const int cur = (rec->flags >> 17) & 1;
      // ---------------------------- stage a small subtree ------------------------------------
      staged = start >= st_base && end <= st_end;
      if (!staged && n_node <= S) {
        const uint2* src = (cur ? P.samp_tmp : P.samp) + (size_t)slot * n + start;
        const int cpr = dp >> 4;                       // 16-byte chunks per row
        for (int q = tid; q < n_node * cpr; q += FF_THREADS) {
          const int j = q / cpr, cc = q - j * cpr;
          const uint2 sv = __ldcg(src + j);
          const uint4 v = __ldcg(reinterpret_cast<const uint4*>(P.xrow + (size_t)sv.x * dp) + cc);   // L2 only: L1 is left to the spill slots
          unsigned int* dstw = U + j * P.stage_ws + cc * 4;
          if (cc * 4 + 0 < P.stage_ws) dstw[0] = v.x;
          if (cc * 4 + 1 < P.stage_ws) dstw[1] = v.y;
          if (cc * 4 + 2 < P.stage_ws) dstw[2] = v.z;
          if (cc * 4 + 3 < P.stage_ws) dstw[3] = v.w;
          if (cc == 0) { ord[j] = (uint8_t)j; wcls[j] = (uint16_t)sv.y; }
        }
        st_base = start; st_end = end;
        staged = true;
        __syncthreads();
        FF_TICK(1);
      }
      const int ls = start - st_base;                 // staged: the node is ord[ls, ls + n_node)
      const bool small = staged && n_node <= FF_SMALL;
      const int KB = staged ? (small ? FF_KB : FF_KBM) : KBA;
      if (P.o_prof && tid == 0) s_prof[staged ? (small ? 13 : 12) : 11] += 1;

      // ------------------------------- node_split_best -------------------------------------
      int f_i = d, n_visited = 0, n_found = 0, n_drawn = 0;
      double best_proxy = -INFINITY;
      float best_ptil = -INFINITY;
      bool best_exact = false;
      // Features are drawn from one RNG stream and a draw depends on whether earlier draws of this
      // node turned out constant, so the reference evaluates them one by one.  Thread 0 SPECULATES
      // that none of the next <= KB evaluated features is constant, simulates the draws (logging
      // every swap), the batch is evaluated in parallel, and thread 0 commits the results in draw
      // order; the first constant feature rolls the simulation back to its draw.
      for (;;) {
        if (tid == 0) {
          int nbatch = 0;
          int s_fi = f_i, s_nv = n_visited, s_nd = n_drawn;
          uint32_t s_rs = rstate;
          int ulen = 0;
          while (nbatch < KB && s_fi > n_total_constants &&
                 (s_nv < P.max_features || s_nv <= n_found + s_nd)) {
            s_nv += 1;
            int fj = ff_rand_int(s_nd, s_fi - n_found, &s_rs);
            if (fj < n_known) {   // a known constant: move it to the drawn-constants prefix
              const uint8_t t = features[s_nd]; features[s_nd] = features[fj]; features[fj] = t;
              undo[2 * ulen] = (uint8_t)s_nd; undo[2 * ulen + 1] = (uint8_t)fj; ++ulen;
              s_nd += 1;
              continue;
            }
            fj += n_found;
            FfItem* it = &items[nbatch];
            it->f = features[fj]; it->fj = fj; it->rs = s_rs; it->nv = s_nv; it->nd = s_nd; it->fi = s_fi; it->ulen = ulen;
            s_fi -= 1;          // speculative: not constant
            { const uint8_t t = features[s_fi]; features[s_fi] = features[fj]; features[fj] = t; }
            undo[2 * ulen] = (uint8_t)s_fi; undo[2 * ulen + 1] = (uint8_t)fj; ++ulen;
            nbatch += 1;
          }
          s_ctrl[0] = nbatch;
          s_ctrl[1] = s_fi; s_ctrl[7] = s_nv; s_ctrl[8] = s_nd; s_ctrl[9] = (int)s_rs; s_ctrl[10] = ulen;
          if (nbatch == 0) { f_i = s_fi; n_visited = s_nv; n_drawn = s_nd; rstate = s_rs; }
        } else if (!staged && tid >= 32) {
          for (int i = tid - 32; i < KBA * hstrideA; i += FF_THREADS - 32) U[i] = 0;   // meanwhile: clear the histograms
        }
        __syncthreads();
        FF_TICK(2);
        const int nbatch = s_ctrl[0];
        if (nbatch == 0) break;

        if (!staged) {
          // ---- histograms of all batch features in one pass over the node's samples (global gathers:
          // the drawn features of a sample share one 64-byte row of codes) ----
          const uint2* src = (cur ? P.samp_tmp : P.samp) + (size_t)slot * n;
          int fk[FF_KB];
#pragma unroll
          for (int k = 0; k < FF_KB; ++k) fk[k] = items[k < nbatch ? k : 0].f;
          constexpr int GQ = 4;                        // samples per thread in flight
          for (int i0 = start; i0 < end; i0 += GQ * FF_THREADS) {
            uint2 sv[GQ];
#pragma unroll
            for (int q = 0; q < GQ; ++q) {
              const int i = i0 + q * FF_THREADS + tid;
              sv[q] = i < end ? __ldcg(src + i) : make_uint2(0xFFFFFFFFu, 0u);
            }
            // every code of the round is requested before the first histogram update (a warp issues in
            // order: an atomic that needs a loaded code would hold back the loads behind it)
            unsigned bq[GQ][FF_KB];
#pragma unroll
            for (int q = 0; q < GQ; ++q) {
              const uint8_t* rq = P.xrow + (size_t)(sv[q].x != 0xFFFFFFFFu ? sv[q].x : 0u) * dp;
#pragma unroll
              for (int k = 0; k < FF_KB; ++k) bq[q][k] = (unsigned)__ldg(rq + fk[k]);   // the drawn features of a row share two sectors
            }
#pragma unroll
            for (int q = 0; q < GQ; ++q) {
              if (sv[q].x == 0xFFFFFFFFu) continue;
              const unsigned cq = sv[q].y & 0xFF, wq = sv[q].y >> 8;
#pragma unroll
              for (int k = 0; k < FF_KB; ++k) {
                if (k < nbatch) {
                  unsigned int* H = U + k * hstrideA;
                  atomicAdd(&H[cq * 256 + bq[q][k]], wq);
                  atomicAdd(&H[C * 256 + bq[q][k]], 1u);
                }
              }
            }
          }
          __syncthreads();
          FF_TICK(3);
          for (int k = wid; k < nbatch; k += FF_WARPS) {
            const unsigned int* H = U + k * hstrideA;
            ff_scan<CM, W>(H, 0, 0, lane, C, n_node, rec->sums, w_node, P.min_samples_leaf, MIN_WEIGHT_LEAF, &results[k]);
          }
        } else if (!small) {
          // ---- staged histogram node: warp k builds and scans the packed histogram of item k ----
          for (int k = wid; k < nbatch; k += FF_WARPS) {
            unsigned int* H = histB + k * hbw;
            for (int i = lane; i < hbw; i += 32) H[i] = 0;
            __syncwarp();
            const int f = items[k].f;
            for (int i0 = 0; i0 < n_node; i0 += 4 * 32) {        // four samples per lane and round, loads first
              int lid4[4];
#pragma unroll
              for (int q = 0; q < 4; ++q) { const int i = i0 + q * 32 + lane; lid4[q] = i < n_node ? (int)ord[ls + i] : -1; }
              unsigned b4[4], wc4[4];
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                b4[q] = lid4[q] >= 0 ? (unsigned)rowsB[lid4[q] * ws4 + f] : 0u;
                wc4[q] = lid4[q] >= 0 ? (unsigned)wcls[lid4[q]] : 0u;
              }
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                if (lid4[q] < 0) continue;
                const unsigned cls = wc4[q] & 0xFF, w = wc4[q] >> 8;
                atomicAdd(&H[(cls >> 1) * 256 + b4[q]], w << ((cls & 1) * 16));
                atomicAdd(&H[hcw + (b4[q] >> 1)], 1u << ((b4[q] & 1) * 16));
              }
            }
            __syncwarp();
            ff_scan<CM, W>(H, 1, hcw, lane, C, n_node, rec->sums, w_node, P.min_samples_leaf, MIN_WEIGHT_LEAF, &results[k]);
          }
        } else {
          // ---- staged node of <= 32 samples: lane j holds sample j; every lane counts the samples
          // (and their class weights) whose bin is <= its own: the left side of the candidate
          // threshold just above its value ----
          const bool have = lane < n_node;
          const int lid = have ? ord[ls + lane] : 0;
          const unsigned wc = have ? wcls[lid] : 0u;
          const acc_t pw = have ? (((acc_t)(wc >> 8) << (13 * (wc & 0xFF))) | ((acc_t)1 << CNT)) : (acc_t)0;
          for (int k = wid; k < nbatch; k += FF_WARPS) {
            const int f = items[k].f;
            const unsigned key = have ? (unsigned)rowsB[lid * ws4 + f] : 0xFFFFu;
            acc_t acc = 0;
            unsigned nbn = 0xFFFFu;        // smallest bin above this lane's bin present in the node
#pragma unroll 2
            for (int j = 0; j < n_node; ++j) {
              const unsigned bj = __shfl_sync(0xffffffffu, key, j);
              const acc_t pj = __shfl_sync(0xffffffffu, pw, j);
              if (bj <= key) acc += pj;
              else nbn = min(nbn, bj);
            }
            const bool cand = have && nbn != 0xFFFFu;
            const bool is_const = __ballot_sync(0xffffffffu, cand) == 0u;
            uint32_t sl[CM];
#pragma unroll
            for (int c = 0; c < CM; ++c) sl[c] = (uint32_t)((acc >> (13 * c)) & 0x1FFFu);
            // float32 rank value of this lane's candidate (see ff_scan): the float64 proxy is formed only
            // when two different candidates are within the bar of each other
            float pt = -INFINITY;
            const int n_left = (int)(acc >> CNT);
            if (cand && n_left >= P.min_samples_leaf && n_node - n_left >= P.min_samples_leaf &&
                ff_weights_ok<CM, W>(sl, C, w_node, MIN_WEIGHT_LEAF))
              pt = ff_rank<CM, W>(sl, rec->sums, C, W ? (float)(w_node * ff_cwscale) : (float)w_node);
            float pm = pt;
#pragma unroll 1
            for (int o = 16; o > 0; o >>= 1) pm = fmaxf(pm, __shfl_xor_sync(0xffffffffu, pm, o));
            const bool near = pt > -INFINITY && pt >= pm - (W ? (float)(w_node * ff_cwscale) * FF_BAR_W : (float)w_node * FF_BAR);
            const unsigned nm = __ballot_sync(0xffffffffu, near);
            FfResult<CM>* R = &results[k];
            if (nm == 0u) {
              if (lane == 0) { R->proxy = -INFINITY; R->ptil = -INFINITY; R->exact = 1; R->n_left = 1 << 30; R->code = is_const ? (1 << 16) : 0; }
              continue;
            }
            // lanes with the same bin hold the same candidate
            const unsigned kmin = __reduce_min_sync(0xffffffffu, near ? key : 0xFFFFu);
            const unsigned kmax = __reduce_max_sync(0xffffffffu, near ? key : 0u);
            int wlane = __ffs(nm) - 1;
            double proxy = 0.0;
            if (kmin != kmax) {          // different candidates within the bar: scikit-learn's float64 expression decides
              proxy = -INFINITY;
              if (near) proxy = ff_proxy<CM, W>(sl, rec->sums, C, w_node).proxy;
              double wp = proxy; int wnl = near ? n_left : (1 << 30);
#pragma unroll 1
              for (int o = 16; o > 0; o >>= 1) {
                const double op = __shfl_xor_sync(0xffffffffu, wp, o);
                const int onl = __shfl_xor_sync(0xffffffffu, wnl, o);
                if (op > wp || (op == wp && onl < wnl)) { wp = op; wnl = onl; }
              }
              const unsigned same = __ballot_sync(0xffffffffu, near && n_left == wnl && proxy == wp);
              wlane = __ffs(same) - 1;
            }
            if (lane == wlane) {
              R->proxy = proxy; R->ptil = pt; R->exact = kmin != kmax ? 1 : 0; R->n_left = n_left;
              R->code = (int)(key | (nbn << 8));
#pragma unroll
              for (int c = 0; c < CM; ++c) R->sl[c] = sl[c];
            }
          }
        }
        __syncthreads();
        FF_TICK(staged ? (small ? 6 : 5) : 4);
        // --- thread 0: commit in draw order, roll back at the first constant feature ---
        if (tid == 0) {
          bool rolled = false;
          for (int k = 0; k < nbatch; ++k) {
            const FfResult<CM>& R = results[k];
            if (!(R.code & (1 << 16))) {
              // `proxy > best_proxy` of the reference, decided on the float32 rank values whenever they are
              // more than the bar apart and on scikit-learn's float64 expression otherwise
              if (R.ptil > -INFINITY) {
                const float bar = W ? (float)(w_node * ff_cwscale) * FF_BAR_W : (float)w_node * FF_BAR;
                bool take;
                if (best_nl <= 0 || R.ptil > best_ptil + bar) {          // first valid split / surely larger
                  take = true; best_exact = R.exact != 0; best_proxy = R.proxy;
                } else if (R.ptil < best_ptil - bar) {                   // surely not larger
                  take = false;
                } else {                                                 // within the bar: float64, strict '>'
                  if (!best_exact) {
                    uint32_t bs[CM];
#pragma unroll
                    for (int c = 0; c < CM; ++c) bs[c] = best_sl[c];
                    best_proxy = ff_proxy<CM, W>(bs, rec->sums, C, w_node).proxy;
                    best_exact = true;
                  }
                  double rp = R.proxy;
                  if (!R.exact) {
                    uint32_t rs2[CM];
#pragma unroll
                    for (int c = 0; c < CM; ++c) rs2[c] = R.sl[c];
                    rp = ff_proxy<CM, W>(rs2, rec->sums, C, w_node).proxy;
                  }
                  take = rp > best_proxy;
                  if (take) best_proxy = rp;
                }
                if (take) {
                  best_ptil = R.ptil;
                  best_feature = items[k].f; best_nl = R.n_left; best_code = R.code;
#pragma unroll
                  for (int c = 0; c < CM; ++c) best_sl[c] = R.sl[c];
                }
              }
              continue;
            }
            // undo every swap made after this item's draw, then take the constant branch
            for (int u = s_ctrl[10] - 1; u >= items[k].ulen; --u) {
              const int a = undo[2 * u], b = undo[2 * u + 1];
              const uint8_t t = features[a]; features[a] = features[b]; features[b] = t;
            }
            rstate = items[k].rs; n_visited = items[k].nv; n_drawn = items[k].nd; f_i = items[k].fi;
            { const int fj = items[k].fj;
              const uint8_t t = features[fj]; features[fj] = features[n_total_constants]; features[n_total_constants] = t; }
            n_found += 1;
            n_total_constants += 1;
            rolled = true;
            break;
          }
          if (!rolled) { f_i = s_ctrl[1]; n_visited = s_ctrl[7]; n_drawn = s_ctrl[8]; rstate = (uint32_t)s_ctrl[9]; }
        }
        __syncthreads();
        FF_TICK(7);
      }
      // end of node_split_best: children impurities, improvement, constant-feature invariants
      if (tid == 0) {
        s_ctrl[2] = best_nl; s_ctrl[3] = best_feature; s_ctrl[4] = best_code; s_ctrl[5] = n_total_constants;
        if (best_nl > 0) {
          double wl = 0.0;
#pragma unroll
          for (int c = 0; c < CM; ++c) if (c < C) {
            if constexpr (W) wl = __dadd_rn(wl, __dmul_rn(ff_cw[c], (double)best_sl[c]));
            else wl += (double)best_sl[c];
          }
          const double wr = w_node - wl;
          uint32_t bs[CM];
#pragma unroll
          for (int c = 0; c < CM; ++c) bs[c] = best_sl[c];
          const FfProxy pr = ff_proxy<CM, W>(bs, rec->sums, C, w_node);
          const double il = pr.il, ir = pr.ir;
          // impurity_improvement (SK/tree/_criterion.pyx:163-190)
          const double a = __dmul_rn(__ddiv_rn(wr, w_node), ir);
          const double b = __dmul_rn(__ddiv_rn(wl, w_node), il);
          s_dbl[0] = il; s_dbl[1] = ir;
          s_dbl[2] = __dmul_rn(__ddiv_rn(w_node, w_samples), __dsub_rn(__dsub_rn(impurity, a), b));
        } else {
          s_dbl[0] = 0.0; s_dbl[1] = 0.0; s_dbl[2] = 0.0;
        }
      }
      __syncthreads();
      best_nl = s_ctrl[2]; best_feature = s_ctrl[3]; best_code = s_ctrl[4]; n_total_constants = s_ctrl[5];
      // restore / record the constant-feature prefix (the memcpy pair at the end of node_split_best)
      for (int i = tid; i < n_known; i += FF_THREADS) features[i] = constant_features[i];
      for (int i = n_known + tid; i < n_total_constants; i += FF_THREADS) constant_features[i] = features[i];
      is_leaf = best_nl <= 0 || (s_dbl[2] + FF_EPSILON < P.min_impurity_decrease);
      FF_TICK(8);

      if (best_nl > 0) {
        const unsigned best_bin = (unsigned)(best_code & 0xFF);
        if (staged) {
          // --- stable partition of the node's slice of ord[] ---
          if (n_node <= 32) {
            if (wid == 0) {
              const bool have = lane < n_node;
              const int lid = have ? ord[ls + lane] : 0;
              const bool isl = have && rowsB[lid * ws4 + best_feature] <= best_bin;
              const unsigned bl = __ballot_sync(0xffffffffu, isl);
              const unsigned br = __ballot_sync(0xffffffffu, have && !isl);
              const unsigned lt = (1u << lane) - 1;
              __syncwarp();
              if (have) ord[ls + (isl ? __popc(bl & lt) : best_nl + __popc(br & lt))] = (uint8_t)lid;
            }
          } else {
            // up to S entries, MP per thread, order = (pass, warp, lane)
            int lidp[MP], posp[MP];
#pragma unroll
            for (int q = 0; q < MP; ++q) {
              const int i = q * FF_THREADS + tid;
              const bool have = i < n_node;
              lidp[q] = have ? ord[ls + i] : 0;
              const bool isl = have && rowsB[lidp[q] * ws4 + best_feature] <= best_bin;
              const unsigned bl = __ballot_sync(0xffffffffu, isl);
              const unsigned br = __ballot_sync(0xffffffffu, have && !isl);
              const unsigned lt = (1u << lane) - 1;
              // rank within the warp; bit 30: goes right; -1: no element
              posp[q] = have ? (isl ? __popc(bl & lt) : (__popc(br & lt) | (1 << 30))) : -1;
              if (lane == 0) { wsum[(q * FF_WARPS + wid) * 2] = __popc(bl); wsum[(q * FF_WARPS + wid) * 2 + 1] = __popc(br); }
            }
            __syncthreads();
            int lo = 0, ro = 0;
#pragma unroll
            for (int q = 0; q < MP; ++q) {
#pragma unroll
              for (int k = 0; k < FF_WARPS; ++k) {
                if (k == wid && posp[q] >= 0) posp[q] += (posp[q] & (1 << 30)) ? ro : lo;
                lo += wsum[(q * FF_WARPS + k) * 2]; ro += wsum[(q * FF_WARPS + k) * 2 + 1];
              }
            }
#pragma unroll
            for (int q = 0; q < MP; ++q)
              if (posp[q] >= 0)
                ord[ls + ((posp[q] & (1 << 30)) ? best_nl + (posp[q] & ~(1 << 30)) : posp[q])] = (uint8_t)lidp[q];
          }
        } else {
          // --- partition_samples_final: stable partition into the other sample buffer ---
          const uint2* src = (cur ? P.samp_tmp : P.samp) + (size_t)slot * n;
          uint2* dst = (cur ? P.samp : P.samp_tmp) + (size_t)slot * n;
          int loff = start, roff = start + best_nl;
          constexpr int PQ = 8;                        // samples per thread and round
          for (int i0 = start; i0 < end; i0 += PQ * FF_THREADS) {
            uint2 svq[PQ];
            int posq[PQ];
#pragma unroll
            for (int q = 0; q < PQ; ++q) {
              const int i = i0 + q * FF_THREADS + tid;
              svq[q] = i < end ? __ldcg(src + i) : make_uint2(0xFFFFFFFFu, 0u);
            }
            unsigned codeq[PQ];
#pragma unroll
            for (int q = 0; q < PQ; ++q)
              codeq[q] = svq[q].x != 0xFFFFFFFFu ? (unsigned)__ldcg(P.xrow + (size_t)svq[q].x * dp + best_feature) : 0u;
#pragma unroll
            for (int q = 0; q < PQ; ++q) {
              const bool have = svq[q].x != 0xFFFFFFFFu;
              const bool isl = have && codeq[q] <= best_bin;
              const unsigned bl = __ballot_sync(0xffffffffu, isl);
              const unsigned br = __ballot_sync(0xffffffffu, have && !isl);
              const unsigned lt = (1u << lane) - 1;
              posq[q] = have ? (isl ? __popc(bl & lt) : (__popc(br & lt) | (1 << 30))) : -1;
              if (lane == 0) { wsum[(q * FF_WARPS + wid) * 2] = __popc(bl); wsum[(q * FF_WARPS + wid) * 2 + 1] = __popc(br); }
            }
            __syncthreads();
            int lo = 0, ro = 0;
#pragma unroll
            for (int q = 0; q < PQ; ++q) {
#pragma unroll
              for (int k = 0; k < FF_WARPS; ++k) {
                if (k == wid && posq[q] >= 0) posq[q] += (posq[q] & (1 << 30)) ? ro : lo;
                lo += wsum[(q * FF_WARPS + k) * 2]; ro += wsum[(q * FF_WARPS + k) * 2 + 1];
              }
            }
#pragma unroll
            for (int q = 0; q < PQ; ++q)
              if (posq[q] >= 0) dst[(posq[q] & (1 << 30)) ? roff + (posq[q] & ~(1 << 30)) : loff + posq[q]] = svq[q];
            loff += lo; roff += ro;
            __syncthreads();
          }
        }
      }
      FF_TICK(9);
    } else if (P.o_prof && tid == 0) {
      s_prof[14] += 1;
    }

    // ------------------------------- _add_node + node_value --------------------------------
    const int node_id = node_count;
    if (node_id >= P.node_cap) { status = 1; break; }
    if (tid == 0) {
      // compact node record (32 bytes = one sector): right child | feature + the two bins around the
      // threshold | n_node_samples | depth | class sums.  Left child = id + 1 (depth-first order); the
      // host derives threshold, impurity, weighted_n_node_samples, value and missing_go_to_left.
      uint32_t* nodes = P.o_nodes + (size_t)slot * P.node_cap * 8;
      if (rec->parent >= 0 && !(rec->flags & (1 << 16))) nodes[(size_t)rec->parent * 8] = (uint32_t)node_id;
      const uint32_t code = is_leaf ? 0xFFFFu : ((uint32_t)best_feature | ((uint32_t)(best_code & 0xFFFF) << 16));
      uint4 q0 = make_uint4(0xFFFFFFFFu, code, (uint32_t)n_node, (uint32_t)depth);
      uint4 q1 = make_uint4(rec->sums[0], CM > 1 ? rec->sums[1] : 0u, 0u, 0u);
      if (CM > 2) { q1.z = rec->sums[2]; q1.w = rec->sums[3]; }
      uint4* dstn = reinterpret_cast<uint4*>(nodes + (size_t)node_id * 8);
      dstn[0] = q0;
      dstn[1] = q1;
    }
    node_count += 1;
    if (!is_leaf) {
      if (sp + 2 > P.stack_cap) { status = 2; break; }
      if (tid == 0) {
        FfRec<CM>* gstack = reinterpret_cast<FfRec<CM>*>(P.stack) + (size_t)slot * P.stack_cap;
        const int child_buf = staged ? ((rec->flags >> 17) & 1) : (((rec->flags >> 17) & 1) ^ 1);
        FfRec<CM> rr, rl;
        rr.depth = depth + 1; rr.parent = node_id; rr.pad_ = 0;
        // right child first, then left (popped first)
        rr.start = start + best_nl; rr.end = end; rr.flags = n_total_constants | (child_buf << 17); rr.impurity = s_dbl[1];
        rl = rr;
        rl.start = start; rl.end = start + best_nl; rl.flags = n_total_constants | (1 << 16) | (child_buf << 17); rl.impurity = s_dbl[0];
#pragma unroll
        for (int c = 0; c < CM; ++c) {
          rr.sums[c] = c < C ? rec->sums[c] - best_sl[c] : 0;
          rl.sums[c] = c < C ? best_sl[c] : 0;
        }
        if (sp < FF_SSTK) sstack[sp] = rr; else gstack[sp] = rr;
        if (sp + 1 < FF_SSTK) sstack[sp + 1] = rl; else gstack[sp + 1] = rl;
      }
      sp += 2;
    }
    if (depth > max_depth_seen) max_depth_seen = depth;
    FF_TICK(10);
    __syncthreads();
  }
  if (tid == 0) {
    P.o_count[slot] = node_count;
    P.o_maxdepth[slot] = max_depth_seen;
    P.o_status[slot] = status;
    if (P.o_prof) for (int i = 0; i < 16; ++i) P.o_prof[(size_t)slot * 16 + i] = s_prof[i];
  }
}
#undef FF_TICK
#undef MIN_WEIGHT_LEAF

// ---- host side -----------------------------------------------------------------------------
static size_t ff_smem_bytes(int CM, int d) {
  const size_t rec = CM <= 2 ? sizeof(FfRec<2>) : sizeof(FfRec<4>);
  const size_t res = CM <= 2 ? sizeof(FfResult<2>) : sizeof(FfResult<4>);
  return (size_t)FF_UW * 4 + (FF_SSTK + 1) * rec + FF_KB * sizeof(FfItem) + FF_KB * res + 4 * 8 + 16 * 8 + 16 * 4 + 64 * 4 + 4 * 4 +
         2 * (size_t)((d + 3) & ~3) + 2 * (size_t)(d + 16) + 16;
}

// staged rows per subtree for (d, n_classes), 0 = the fast kernel cannot run this shape
static int ff_stage_rows(int d, int n_classes, int* ws_out) {
  const int ws = ((d + 3) / 4) | 1;                           // odd word stride: conflict-free column reads
  const int hbw = 256 * ((n_classes + 1) / 2) + 128;
  int S = (FF_UW - FF_KBM * hbw) * 4 / (ws * 4 + 3);
  S = std::min(FF_SMAX, S / 32 * 32);
  *ws_out = ws;
  return S >= 64 ? S : 0;
}

bool forest_fast_supported(const Ctx* c, int n_classes, bool reg, int random_split) {
  if (reg || random_split || n_classes > 4 || c->d > 255 || !c->forest.all_coded || !c->forest.well_separated)
    return false;
  if ((double)c->n * 255.0 >= 4294967296.0) return false;
  if (const char* e = getenv("SKDIST_B200_FOREST_KERNEL")) if (!strcmp(e, "general")) return false;
  int ws;
  return ff_stage_rows((int)c->d, n_classes, &ws) > 0;
}

int forest_fast_slots_per_sm() { return 7; }
size_t forest_fast_record_bytes(int n_classes) { return n_classes <= 2 ? sizeof(FfRec<2>) : sizeof(FfRec<4>); }

int forest_fast_launch(Ctx* c, FfParams& P, int nt) {
  int ws = 0;
  P.stage_rows = ff_stage_rows(P.d, P.n_classes, &ws);
  P.stage_ws = ws;
  const int CM = P.n_classes <= 2 ? 2 : 4;
  const size_t smem = ff_smem_bytes(CM, P.d);
  P.n_trees = nt;
  void (*kern)(const FfParams) = CM == 2 ? (P.weighted ? forest_fast_kernel<2, true> : forest_fast_kernel<2, false>)
                                        : (P.weighted ? forest_fast_kernel<4, true> : forest_fast_kernel<4, false>);
  SKD_CUDA(c, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  SKD_CUDA(c, cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  kern<<<nt, FF_THREADS, smem, c->stream>>>(P);
  SKD_CUDA(c, cudaGetLastError());
  c->launches += 1;
  return 0;
}

}  // namespace skd
