// forest.cu -- DistRandomForestClassifier: one persistent CTA per tree, exact depth-first builder.
//
// Replaces the reference's per-tree task `_build_trees` (ref ensemble.py:68-109: bootstrap counts
// as sample_weight, then DecisionTreeClassifier.fit) for the default forest configuration:
//   SK/tree/_tree.pyx:139-337      DepthFirstTreeBuilder.build  (stack order: push right, push left)
//   SK/tree/_splitter.pyx:262-504  node_split_best  (Fisher-Yates feature draws from ONE xorshift
//                                  stream, constant-feature bookkeeping, strict '>' on the proxy)
//   SK/tree/_partitioner.pyx       DensePartitioner (sort node samples by feature value, scan the
//                                  boundaries between values more than 1e-7 apart)
//   SK/tree/_criterion.pyx:605-680 Gini (float64, same operation order; all class sums are integers,
//                                  hence exact and independent of the summation order)
// The sort-and-scan of a node is replaced by a shared-memory histogram over the feature's distinct
// values (<= 256 per feature, precomputed bin codes, feature-major uint8): present bins visited in
// ascending order ARE the sorted distinct values, so every candidate split, its class counts and
// the threshold (v[p-1]/2 + v[p]/2) equal what the sort-based scan sees.  The tree topology, the
// RNG consumption and therefore every later draw are bit-identical to scikit-learn's.
// The random splitter (node_split_random, ExtraTrees) uses the same histograms when every feature has
// codes, and otherwise reads the raw float32 values (min / max pass, drawn threshold, left-side pass),
// so it takes continuous features.
// No tensor cores: the work is integer histogramming, bound by gather bandwidth / latency.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <deque>
#include <mutex>
#include <thread>

#include "forest_common.h"
#include "skd_internal.h"

namespace skd {

constexpr int FO_THREADS = 256;
constexpr int FO_MAXC = 16;      // classes
constexpr int FO_BINS = 256;
constexpr float FEATURE_THRESHOLD = 1e-7f;
constexpr double FO_EPSILON = 2.220446049250313e-16;   // np.finfo('double').eps (SK/tree/_tree.pyx EPSILON)

struct FoRecord {          // builder stack record (SK/tree/_tree.pyx StackRecord) + the node's class sums
  int32_t start, end, depth, parent, is_left, n_const;
  double impurity;
  unsigned long long sums[FO_MAXC];
};

struct FoItem {            // one speculatively drawn feature + the simulation state right after its draw
  int f, fj, nv, nd, fi, ulen;
  uint32_t rs;
  uint32_t rnd;            // random splitter: the rand_r value that rand_uniform turns into the threshold
};
struct FoResult {          // best split of one feature in the current node
  int is_const, pos, bin;
  double proxy, thr, il, ir;
  unsigned long long sl[FO_MAXC];
};
constexpr int FO_KB_MAX = 8;
constexpr int FO_SSTK = 128;     // builder-stack entries kept in shared memory (deeper ones spill to global)
constexpr int FO_HIST_WORDS = 40 * FO_BINS;   // KB * (C + 1) * 256 <= this

struct FoParams {
  const uint8_t* xbin;        // [d][n] bin codes, feature-major (best splitter)
  const float* binval;        // [d][256] distinct values ascending
  const float* xval;          // [d][n] raw values, feature-major: random splitter on features without codes, else nullptr
  const int32_t* ycls;        // [n] class ids (classification)
  const double* yreal;        // [n] float64 targets (regression: MSE criterion), else nullptr
  int64_t n;
  int d, n_classes;
  int max_features, max_depth, min_samples_split, min_samples_leaf;
  int random_split;           // 0: node_split_best (RandomForest), 1: node_split_random (ExtraTrees)
  double min_weight_leaf, min_impurity_decrease;
  // per tree (wave-local index = blockIdx.x)
  const uint8_t* counts;      // [trees_in_wave][n] bootstrap multiplicities (sample_weight)
  const uint32_t* rand_state; // [trees_in_wave]
  int n_trees;
  // per slot work + output buffers
  uint2* samp;                // [slots][n]   (sample index, (weight << 8) | class)
  uint2* samp_tmp;            // [slots][n]
  FoRecord* stack;            // [slots][stack_cap]
  int stack_cap;
  int64_t node_cap;
  int32_t* o_left; int32_t* o_right; int32_t* o_feature; int32_t* o_nsamp; uint8_t* o_mgl;
  double* o_thr; double* o_imp; double* o_wn; double* o_val;   // o_val [node_cap][n_classes]
  int32_t* o_count;           // [slots] node_count
  int32_t* o_maxdepth;        // [slots]
  int32_t* o_status;          // [slots] 0 ok, 1 node capacity, 2 stack capacity
  long long* o_prof;          // [slots][16] cycles per builder phase (SKDIST_B200_FOREST_PROF=1), else nullptr
  // class weights, read only by the weighted instantiation (W): as FfParams
  int cw_bs;
  const double* cw;
  double min_weight_fraction;
};

__device__ __forceinline__ uint32_t fo_rand_r(uint32_t* seed) {   // SK/utils/_random.pxd:20-34
  if (*seed == 0) *seed = 1;
  *seed ^= (uint32_t)(*seed << 13);
  *seed ^= (uint32_t)(*seed >> 17);
  *seed ^= (uint32_t)(*seed << 5);
  return *seed % ((uint32_t)2147483647 + 1);
}
__device__ __forceinline__ int fo_rand_int(int low, int high, uint32_t* seed) {
  return low + (int)(fo_rand_r(seed) % (uint32_t)(high - low));
}

// Gini children impurity, float64 with scikit-learn's operation order (no FMA contraction)
template <int CM>
__device__ __forceinline__ void fo_children_impurity(const unsigned long long* sl, const unsigned long long* st,
                                                     int C, double wl, double wr, double* il, double* ir) {
  double sql = 0.0, sqr = 0.0;
#pragma unroll
  for (int c = 0; c < CM; ++c) {
    if (c < C) {
      const double a = (double)sl[c], b = (double)(st[c] - sl[c]);
      sql = __dadd_rn(sql, __dmul_rn(a, a));
      sqr = __dadd_rn(sqr, __dmul_rn(b, b));
    }
  }
  *il = __dsub_rn(1.0, __ddiv_rn(sql, __dmul_rn(wl, wl)));
  *ir = __dsub_rn(1.0, __ddiv_rn(sqr, __dmul_rn(wr, wr)));
}
// ... with class weights: sum_left[c] = w_c * count, sum_right[c] = sum_total[c] - sum_left[c]
// (ClassificationCriterion.update, SK/tree/_criterion.pyx)
template <int CM>
__device__ __forceinline__ void fo_children_impurity_w(const unsigned long long* sl, const unsigned long long* st,
                                                       const double* cw, int C, double wl, double wr, double* il,
                                                       double* ir) {
  double sql = 0.0, sqr = 0.0;
#pragma unroll
  for (int c = 0; c < CM; ++c) {
    if (c < C) {
      const double a = __dmul_rn(cw[c], (double)sl[c]), b = __dsub_rn(__dmul_rn(cw[c], (double)st[c]), a);
      sql = __dadd_rn(sql, __dmul_rn(a, a));
      sqr = __dadd_rn(sqr, __dmul_rn(b, b));
    }
  }
  *il = __dsub_rn(1.0, __ddiv_rn(sql, __dmul_rn(wl, wl)));
  *ir = __dsub_rn(1.0, __ddiv_rn(sqr, __dmul_rn(wr, wr)));
}

// Node statistics are kept as 64-bit patterns so that the classification path (integer class
// weights) and the regression path (float64 {sum w, sum w*y, sum w*y*y}, MSE criterion
// SK/tree/_criterion.pyx:922-1017) share the stack records, the split records and the scan.
template <bool REG>
__device__ __forceinline__ unsigned long long st_add(unsigned long long a, unsigned long long b) {
  if constexpr (REG) return (unsigned long long)__double_as_longlong(__longlong_as_double((long long)a) + __longlong_as_double((long long)b));
  else return a + b;
}
template <bool REG>
__device__ __forceinline__ unsigned long long st_sub(unsigned long long a, unsigned long long b) {
  if constexpr (REG) return (unsigned long long)__double_as_longlong(__longlong_as_double((long long)a) - __longlong_as_double((long long)b));
  else return a - b;
}
__device__ __forceinline__ double st_d(unsigned long long a) { return __longlong_as_double((long long)a); }
__device__ __forceinline__ unsigned long long d_st(double a) { return (unsigned long long)__double_as_longlong(a); }

// MSE children impurity from the statistics of the left child and of the node
__device__ __forceinline__ void fo_children_mse(const unsigned long long* sl, const unsigned long long* st,
                                                double wl, double wr, double* il, double* ir) {
  const double sum_l = st_d(sl[1]), sq_l = st_d(sl[2]);
  const double sum_r = __dsub_rn(st_d(st[1]), sum_l), sq_r = __dsub_rn(st_d(st[2]), sq_l);
  const double ml = __ddiv_rn(sum_l, wl), mr = __ddiv_rn(sum_r, wr);
  *il = __dsub_rn(__ddiv_rn(sq_l, wl), __dmul_rn(ml, ml));
  *ir = __dsub_rn(__ddiv_rn(sq_r, wr), __dmul_rn(mr, mr));
}

// CM: compile-time bound on the class count (3 statistics when REG), so the per-class arrays of a thread live in registers.
// W: class weights (classification only).  Histograms, records and the partition keep the integer
// counts; the float64 statistics are w_c * count (one rounding), in scikit-learn's operation order.
#define FO_TICK(ph) do { if (P.o_prof && tid == 0) { const long long _t = clock64(); prof[ph] += _t - tlast; tlast = _t; } } while (0)
#define FOR_C(c) _Pragma("unroll") for (int c = 0; c < CM; ++c) if (c < C)
// RAW: random splitter over the raw values (P.xval), a separate instantiation so that the histogram
// instantiations keep their register allocation.
template <int CM, bool REG, bool W, bool RAW>
__global__ void __launch_bounds__(FO_THREADS)
forest_build_kernel(const FoParams P) {
  static_assert(!(REG && W), "class weights are a classification feature");
  const int slot = blockIdx.x;
  if (slot >= P.n_trees) return;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int C = REG ? 3 : P.n_classes, d = P.d;   // REG: the three statistics take the place of the classes
  const int64_t n = P.n;
  uint2* samp = P.samp + (size_t)slot * n;
  uint2* tmp = P.samp_tmp + (size_t)slot * n;
  FoRecord* stack = P.stack + (size_t)slot * P.stack_cap;
  const uint8_t* cnt = P.counts + (size_t)slot * n;
  const int64_t nb = (int64_t)slot * P.node_cap;

  extern __shared__ int fo_sm[];
  int* features = fo_sm;                     // [d]
  int* constant_features = fo_sm + d;        // [d]
  // best splitter, per batch item: [c][bin] class weights (c < C), then [bin] sample counts;
  // random splitter: [item][c][thread] left-side statistics of each thread's samples
  __shared__ __align__(16) unsigned int hist[FO_HIST_WORDS];
  __shared__ float s_mm[2][FO_THREADS / 32][FO_KB_MAX];   // random splitter: per-warp min / max of the batch features
  __shared__ int s_nl[FO_THREADS / 32][FO_KB_MAX];        // random splitter: per-warp left counts
  __shared__ FoItem items[FO_KB_MAX];
  __shared__ FoResult results[FO_KB_MAX];
  __shared__ int s_sim_nd, s_sim_ulen;
  __shared__ uint32_t s_sim_rs;
  __shared__ int wsum[FO_THREADS / 32][2];
  __shared__ int s_ctrl[8];
  __shared__ double s_dbl[4];
  __shared__ FoRecord rec_spill;
  __shared__ unsigned long long best_sl[FO_MAXC];
  __shared__ double s_cw[W ? FO_MAXC : 1];   // W: this tree's class weights
  int2* undo = reinterpret_cast<int2*>(fo_sm + 2 * d);      // [d + 16] swap log of the speculative draws
  float* sbv = reinterpret_cast<float*>(undo + (d + 16));   // [FO_KB_MAX][256] distinct values of the batch features
  FoRecord* sstack = reinterpret_cast<FoRecord*>(sbv + FO_KB_MAX * FO_BINS);   // [FO_SSTK] top of the DFS stack
  // histogram words per feature: classification [C][256] u32 weights + [256] counts; regression
  // [3][256] float64 statistics + [256] counts
  const int hstride = REG ? (3 * 2 + 1) * FO_BINS : (C + 1) * FO_BINS;
  const int KB = min(FO_KB_MAX, FO_HIST_WORDS / hstride);

  // ---- initialise the tree: samples with non-zero weight in ascending order (Splitter.init) ----
  __shared__ int base_s;
  if (tid == 0) base_s = 0;
  for (int i = tid; i < d; i += FO_THREADS) features[i] = i;
  // balanced_subsample: 1 until the root's class sums give the weights (only absent classes get 0)
  if constexpr (W) if (tid < FO_MAXC) s_cw[tid] = P.cw_bs || tid >= C ? 1.0 : P.cw[tid];
  __syncthreads();
  unsigned long long my_sums[CM];
#pragma unroll
  for (int c = 0; c < CM; ++c) my_sums[c] = 0;
  for (int64_t i0 = 0; i0 < n; i0 += FO_THREADS) {
    const int64_t i = i0 + tid;
    unsigned int w = 0, yc = 0;
    if (i < n) { w = cnt[i]; if (!REG) yc = (unsigned)P.ycls[i]; }
    int keep = w != 0;
    if constexpr (W) keep = keep && s_cw[yc] != 0.0;   // rows of weight 0 leave the tree (Splitter.init)
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) wsum[wid][0] = __popc(bal);
    __syncthreads();
    int off = 0, tot = 0;
    for (int k = 0; k < FO_THREADS / 32; ++k) { if (k < wid) off += wsum[k][0]; tot += wsum[k][0]; }
    const int b = base_s;
    if (keep) {
      samp[b + off + __popc(bal & ((1u << lane) - 1))] = make_uint2((unsigned)i, (w << 8) | yc);
      if constexpr (REG) {   // RegressionCriterion.init (SK/tree/_criterion.pyx:  w_y = w*y; sum += w_y; sq += w_y*y)
        const double yv = P.yreal[i], wy = __dmul_rn((double)w, yv);
        my_sums[0] = d_st(st_d(my_sums[0]) + (double)w);
        my_sums[1] = d_st(st_d(my_sums[1]) + wy);
        my_sums[2] = d_st(st_d(my_sums[2]) + __dmul_rn(wy, yv));
      } else {
        FOR_C(c) if ((int)yc == c) my_sums[c] += w;
      }
    }
    __syncthreads();
    if (tid == 0) base_s = b + tot;
    __syncthreads();
  }
  const int n_nz = base_s;
  // reduce the class sums over the block in a fixed order (warps, then the warp totals in warp order):
  // integers are exact anyway, the float64 regression sums are then the same from run to run
  __shared__ unsigned long long red[FO_MAXC];
  unsigned long long* wred = reinterpret_cast<unsigned long long*>(hist);   // [warp][FO_MAXC]
  FOR_C(c) {
    unsigned long long v = my_sums[c];
    for (int o = 16; o > 0; o >>= 1) v = st_add<REG>(v, __shfl_xor_sync(0xffffffffu, v, o));
    if (lane == 0) wred[wid * FO_MAXC + c] = v;
  }
  __syncthreads();
  if (tid < C) {
    unsigned long long v = 0;   // 0 bit pattern == 0.0
    for (int w = 0; w < FO_THREADS / 32; ++w) v = st_add<REG>(v, wred[w * FO_MAXC + tid]);
    red[tid] = v;
  }
  __syncthreads();
  double w_samples = 0.0;
  if constexpr (REG) w_samples = st_d(red[0]);
  else if constexpr (W) {
    if (P.cw_bs) {   // compute_class_weight("balanced") of the bootstrap sample: n / (K_present * N_c)
      if (tid < C) {
        unsigned long long nt = 0; int kp = 0;
        for (int c = 0; c < C; ++c) { nt += red[c]; kp += red[c] != 0; }
        s_cw[tid] = red[tid] ? __ddiv_rn((double)nt, __dmul_rn((double)kp, (double)red[tid])) : 0.0;
      }
      __syncthreads();
    }
    FOR_C(c) w_samples = __dadd_rn(w_samples, __dmul_rn(s_cw[c], (double)red[c]));
  }
  else { FOR_C(c) w_samples += (double)red[c]; }    // weighted_n_samples (integer valued)
  // BaseDecisionTree._fit: min_weight_leaf = min_weight_fraction_leaf * sum(sample_weight)
  const double mwl_w = W ? __dmul_rn(P.min_weight_fraction, w_samples) : 0.0;
#define MIN_WEIGHT_LEAF (W ? mwl_w : P.min_weight_leaf)

  long long prof[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  long long tlast = clock64();
  uint32_t rstate = P.rand_state[slot];
  int sp = 0;           // stack pointer
  int node_count = 0, max_depth_seen = -1, status = 0;
  if (tid == 0) {
    FoRecord r;
    r.start = 0; r.end = n_nz; r.depth = 0; r.parent = -1; r.is_left = 0; r.n_const = 0;
    r.impurity = INFINITY;
    for (int c = 0; c < FO_MAXC; ++c) r.sums[c] = c < C ? red[c] : 0;
    sstack[0] = r;
  }
  sp = 1;
  bool first = true;
  __syncthreads();

  while (sp > 0 && status == 0) {
    --sp;
    FO_TICK(10);
    // the popped record is read in place when it lives in the shared-memory part of the stack (its
    // slot is only overwritten by this node's own push, after the last read)
    if (sp >= FO_SSTK) {
      if (tid == 0) rec_spill = stack[sp];
      __syncthreads();
    }
    const FoRecord& rec = sp < FO_SSTK ? sstack[sp] : rec_spill;
    FO_TICK(0);
    const int start = rec.start, end = rec.end, depth = rec.depth;
    const int n_node = end - start;
    double w_node = 0.0;
    if constexpr (REG) w_node = st_d(rec.sums[0]);
    else if constexpr (W) { FOR_C(c) w_node = __dadd_rn(w_node, __dmul_rn(s_cw[c], (double)rec.sums[c])); }
    else { FOR_C(c) w_node += (double)rec.sums[c]; }
    double impurity = rec.impurity;
    bool is_leaf = depth >= P.max_depth || n_node < P.min_samples_split || n_node < 2 * P.min_samples_leaf ||
                   w_node < 2.0 * MIN_WEIGHT_LEAF;
    if (first) {   // root: node_impurity()  (SK/tree/_criterion.pyx:620-640)
      if constexpr (REG) {   // MSE.node_impurity
        const double mean = __ddiv_rn(st_d(rec.sums[1]), w_node);
        impurity = __dsub_rn(__ddiv_rn(st_d(rec.sums[2]), w_node), __dmul_rn(mean, mean));
      } else if constexpr (W) {
        double sq = 0.0;
        FOR_C(c) { const double a = __dmul_rn(s_cw[c], (double)rec.sums[c]); sq = __dadd_rn(sq, __dmul_rn(a, a)); }
        impurity = __dsub_rn(1.0, __ddiv_rn(sq, __dmul_rn(w_node, w_node)));
      } else {
        double sq = 0.0;
        FOR_C(c) { const double a = (double)rec.sums[c]; sq = __dadd_rn(sq, __dmul_rn(a, a)); }
        impurity = __dsub_rn(1.0, __ddiv_rn(sq, __dmul_rn(w_node, w_node)));
      }
      first = false;
    }
    is_leaf = is_leaf || impurity <= FO_EPSILON;

    // ------------------------------- node_split_best -------------------------------------
    int best_feature = 0, best_pos = end, best_bin = -1, n_total_constants = rec.n_const;
    double best_thr = 0.0, best_il = 0.0, best_ir = 0.0, best_improvement = 0.0;
    int best_mgl = 0;
    if (!is_leaf) {
      const int n_known = rec.n_const;
      int f_i = d, n_visited = 0, n_found = 0, n_drawn = 0;
      n_total_constants = n_known;
      double best_proxy = -INFINITY;
      // Features are drawn from one RNG stream and a draw depends on whether earlier draws of this
      // node turned out constant, so the reference evaluates them one by one.  Here thread 0
      // SPECULATES that none of the next <= KB evaluated features is constant, simulates the
      // draws (logging every swap), all KB histograms are built in one pass over the node's
      // samples, one warp per feature scans its histogram, and thread 0 then commits the results
      // in draw order; the first feature found constant rolls the simulation back to that draw,
      // takes the constant branch and the remaining speculative results are discarded.
      for (;;) {
        if (tid == 0) {
          int nbatch = 0;
          int s_fi = f_i, s_nv = n_visited, s_nd = n_drawn;
          uint32_t s_rs = rstate;
          int ulen = 0;
          while (nbatch < KB && s_fi > n_total_constants &&
                 (s_nv < P.max_features || s_nv <= n_found + s_nd)) {
            s_nv += 1;
            int fj = fo_rand_int(s_nd, s_fi - n_found, &s_rs);
            if (fj < n_known) {   // a known constant: move it to the drawn-constants prefix
              const int t = features[s_nd]; features[s_nd] = features[fj]; features[fj] = t;
              undo[ulen++] = make_int2(s_nd, fj);
              s_nd += 1;
              continue;
            }
            fj += n_found;
            FoItem it;
            it.f = features[fj]; it.fj = fj; it.rs = s_rs; it.nv = s_nv; it.nd = s_nd; it.fi = s_fi; it.ulen = ulen;
            items[nbatch] = it;
            s_fi -= 1;          // speculative: not constant
            { const int t = features[s_fi]; features[s_fi] = features[fj]; features[fj] = t; }
            undo[ulen++] = make_int2(s_fi, fj);
            // node_split_random draws the threshold of a non-constant feature from the same stream
            // right after the feature (SK/tree/_splitter.pyx:633-637)
            if (P.random_split) items[nbatch].rnd = fo_rand_r(&s_rs);
            nbatch += 1;
          }
          s_ctrl[0] = nbatch;
          // keep the simulated end state for the no-rollback case
          s_ctrl[1] = s_fi; s_ctrl[7] = s_nv; s_sim_nd = s_nd; s_sim_rs = s_rs; s_sim_ulen = ulen;
          if (nbatch == 0) { f_i = s_fi; n_visited = s_nv; n_drawn = s_nd; rstate = s_rs; }
        } else if (tid >= 32) {
          // meanwhile the other warps clear the histograms (random splitter: the per-thread left
          // statistics, KB * C * FO_THREADS words, 64-bit when REG, which this covers) of a full batch
          for (int i = tid - 32; i < KB * hstride; i += FO_THREADS - 32) hist[i] = 0;
        }
        __syncthreads();
        FO_TICK(1);
        const int nbatch = s_ctrl[0];
        if (nbatch == 0) break;
        if constexpr (RAW) {
          // ------------------- node_split_random over the raw float32 values -------------------
          // (SK/tree/_splitter.pyx node_split_random, DensePartitioner find_min_max / partition_samples)
          int fk[FO_KB_MAX];   // batch item k reads the column P.xval + fk[k] * n
#pragma unroll
          for (int k = 0; k < FO_KB_MAX; ++k) fk[k] = items[k < nbatch ? k : 0].f;
          // pass A: min and max of every batch feature over the node's samples (exact in any order);
          // all gathers of a sample are issued before the first use
          float mn[FO_KB_MAX], mx[FO_KB_MAX];
#pragma unroll
          for (int k = 0; k < FO_KB_MAX; ++k) { mn[k] = INFINITY; mx[k] = -INFINITY; }
          for (int i = start + tid; i < end; i += FO_THREADS) {
            const unsigned s = samp[i].x;
            float v[FO_KB_MAX];
#pragma unroll
            for (int k = 0; k < FO_KB_MAX; ++k) v[k] = k < nbatch ? __ldg(P.xval + (size_t)fk[k] * n + s) : 0.f;
#pragma unroll
            for (int k = 0; k < FO_KB_MAX; ++k) { mn[k] = fminf(mn[k], v[k]); mx[k] = fmaxf(mx[k], v[k]); }
          }
#pragma unroll
          for (int k = 0; k < FO_KB_MAX; ++k) {
            for (int o = 16; o > 0; o >>= 1) {
              mn[k] = fminf(mn[k], __shfl_xor_sync(0xffffffffu, mn[k], o));
              mx[k] = fmaxf(mx[k], __shfl_xor_sync(0xffffffffu, mx[k], o));
            }
            if (lane == 0) { s_mm[0][wid][k] = mn[k]; s_mm[1][wid][k] = mx[k]; }
          }
          __syncthreads();
          FO_TICK(3);
          // every thread forms the same decisions: constant test in float32, threshold
          // rand_uniform(min, max) in float64 (SK/tree/_utils.pyx), and min if it lands on max
          double thr[FO_KB_MAX];
#pragma unroll
          for (int k = 0; k < FO_KB_MAX; ++k) {
            float lo = s_mm[0][0][k], hi = s_mm[1][0][k];
            for (int w = 1; w < FO_THREADS / 32; ++w) { lo = fminf(lo, s_mm[0][w][k]); hi = fmaxf(hi, s_mm[1][w][k]); }
            thr[k] = -INFINITY;    // constant (or not in the batch): no sample goes left
            if (k < nbatch && !(hi <= lo + FEATURE_THRESHOLD)) {
              const double dlo = (double)lo, dhi = (double)hi;
              double t = __dadd_rn(__ddiv_rn(__dmul_rn(__dsub_rn(dhi, dlo), (double)items[k].rnd), 2147483647.0), dlo);
              if (t == dhi) t = dlo;
              thr[k] = t;
            }
            if (tid == 0 && k < nbatch) { results[k].is_const = thr[k] == -INFINITY; results[k].thr = thr[k]; }
          }
          // pass B: (double)x <= threshold goes left (DensePartitioner.partition_samples); every thread
          // sums its own samples in order into its own column of `hist`, so that the reduction below
          // has a fixed order and the float64 regression sums are the same from run to run
          unsigned nl[FO_KB_MAX];
#pragma unroll
          for (int k = 0; k < FO_KB_MAX; ++k) nl[k] = 0;
          for (int i = start + tid; i < end; i += FO_THREADS) {
            const uint2 sv = samp[i];
            const unsigned cls = sv.y & 0xFF, wgt = sv.y >> 8;
            double yv = 0.0;
            if constexpr (REG) yv = __ldg(P.yreal + sv.x);
            float v[FO_KB_MAX];
#pragma unroll
            for (int k = 0; k < FO_KB_MAX; ++k) v[k] = k < nbatch ? __ldg(P.xval + (size_t)fk[k] * n + sv.x) : 0.f;
            const double wy = __dmul_rn((double)wgt, yv), wyy = __dmul_rn(wy, yv);
#pragma unroll
            for (int k = 0; k < FO_KB_MAX; ++k) {
              if ((double)v[k] <= thr[k]) {
                nl[k] += 1;
                if constexpr (REG) {
                  double* A = reinterpret_cast<double*>(hist) + k * 3 * FO_THREADS + tid;
                  A[0] += (double)wgt;
                  A[FO_THREADS] += wy;
                  A[2 * FO_THREADS] += wyy;
                } else {
                  hist[(k * C + cls) * FO_THREADS + tid] += wgt;
                }
              }
            }
          }
#pragma unroll
          for (int k = 0; k < FO_KB_MAX; ++k) {
            const unsigned t = __reduce_add_sync(0xffffffffu, nl[k]);
            if (lane == 0) s_nl[wid][k] = (int)t;
          }
          __syncthreads();
          FO_TICK(4);
          // one warp per feature: left statistics over the threads (each lane 8 threads in order,
          // then a fixed butterfly), then the split's proxy as node_split_random evaluates it
          for (int k = wid; k < nbatch; k += FO_THREADS / 32) {
            unsigned long long sl[CM];
            FOR_C(c) {
              unsigned long long v = 0;
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const int t = lane * 8 + j;
                if constexpr (REG) v = st_add<REG>(v, d_st(reinterpret_cast<const double*>(hist)[(k * 3 + c) * FO_THREADS + t]));
                else v += hist[(k * C + c) * FO_THREADS + t];
              }
              for (int o = 16; o > 0; o >>= 1) v = st_add<REG>(v, __shfl_xor_sync(0xffffffffu, v, o));
              sl[c] = v;
            }
            if (lane == 0) {
              FoResult* R = &results[k];
              R->proxy = -INFINITY; R->pos = end; R->bin = -1;
              if (!R->is_const) {
                int n_left = 0;
                for (int w = 0; w < FO_THREADS / 32; ++w) n_left += s_nl[w][k];
                const int n_right = n_node - n_left;
                if (n_left >= P.min_samples_leaf && n_right >= P.min_samples_leaf) {
                  double wl = 0.0;
                  if constexpr (REG) wl = st_d(sl[0]);
                  else if constexpr (W) { FOR_C(c) wl = __dadd_rn(wl, __dmul_rn(s_cw[c], (double)sl[c])); }
                  else { FOR_C(c) wl += (double)sl[c]; }
                  const double wr = w_node - wl;
                  if (!(wl < MIN_WEIGHT_LEAF || wr < MIN_WEIGHT_LEAF)) {
                    double il, ir;
                    if constexpr (REG) {
                      fo_children_mse(sl, rec.sums, wl, wr, &il, &ir);
                      const double sum_l = st_d(sl[1]), sum_r = __dsub_rn(st_d(rec.sums[1]), sum_l);
                      R->proxy = __dadd_rn(__ddiv_rn(__dmul_rn(sum_l, sum_l), wl), __ddiv_rn(__dmul_rn(sum_r, sum_r), wr));
                    } else if constexpr (W) {
                      fo_children_impurity_w<CM>(sl, rec.sums, s_cw, C, wl, wr, &il, &ir);
                      R->proxy = __dsub_rn(__dmul_rn(-wr, ir), __dmul_rn(wl, il));
                    } else {
                      fo_children_impurity<CM>(sl, rec.sums, C, wl, wr, &il, &ir);
                      R->proxy = __dsub_rn(__dmul_rn(-wr, ir), __dmul_rn(wl, il));
                    }
                    R->pos = start + n_left; R->il = il; R->ir = ir;
                    FOR_C(c) R->sl[c] = sl[c];
                  }
                }
              }
            }
          }
        } else {
          // --- histograms of all batch features in one pass over the node's samples ---
          // the distinct values of the batch features are staged in the same phase (their loads overlap
          // the gathers below); the scan reads them inside dependent per-candidate loops
          float stage[FO_KB_MAX];   // FO_KB_MAX * 256 values / 256 threads
#pragma unroll
          for (int q = 0; q < FO_KB_MAX; ++q)
            stage[q] = q < nbatch ? __ldg(P.binval + (size_t)items[q].f * FO_BINS + tid) : 0.f;
          FO_TICK(2);
          {
            // all gathers of a sample are issued before the first atomic: one memory round trip per
            // sample instead of one per feature (the dependent load -> atomic chain serialised them)
            const uint8_t* col[FO_KB_MAX];
#pragma unroll
            for (int k = 0; k < FO_KB_MAX; ++k) col[k] = P.xbin + (size_t)items[k < nbatch ? k : 0].f * n;
            for (int i = start + tid; i < end; i += FO_THREADS) {
              const uint2 sv = samp[i];
              const unsigned cls = sv.y & 0xFF, wgt = sv.y >> 8;
              double yv = 0.0;
              if constexpr (REG) yv = __ldg(P.yreal + sv.x);
              unsigned bbs[FO_KB_MAX];
#pragma unroll
              for (int k = 0; k < FO_KB_MAX; ++k) bbs[k] = k < nbatch ? (unsigned)__ldg(col[k] + sv.x) : 0u;
              const double wy = __dmul_rn((double)wgt, yv), wyy = __dmul_rn(wy, yv);
#pragma unroll
              for (int k = 0; k < FO_KB_MAX; ++k) {
                if (k < nbatch) {
                  unsigned int* H = hist + k * hstride;
                  if constexpr (REG) {
                    double* Hd = reinterpret_cast<double*>(H);
                    atomicAdd(&Hd[0 * FO_BINS + bbs[k]], (double)wgt);
                    atomicAdd(&Hd[1 * FO_BINS + bbs[k]], wy);
                    atomicAdd(&Hd[2 * FO_BINS + bbs[k]], wyy);
                    atomicAdd(&H[6 * FO_BINS + bbs[k]], 1u);
                  } else {
                    atomicAdd(&H[cls * FO_BINS + bbs[k]], wgt);
                    atomicAdd(&H[C * FO_BINS + bbs[k]], 1u);
                  }
                }
              }
            }
#pragma unroll
            for (int q = 0; q < FO_KB_MAX; ++q)
              if (q < nbatch) sbv[q * FO_BINS + tid] = stage[q];
          }
          __syncthreads();
          FO_TICK(3);
          // --- one warp per feature: scan the 256 bins (8 per lane) in ascending order ---
          for (int k = wid; k < nbatch; k += FO_THREADS / 32) {
            const unsigned int* H = hist + k * hstride;
            const float* bv = sbv + k * FO_BINS;
            const int cnt_off = REG ? 6 * FO_BINS : C * FO_BINS;
            // statistic c of bin bb as a 64-bit pattern (class weight, or float64 sum for regression)
            auto hbin = [&](int c, int bb) -> unsigned long long {
              if constexpr (REG) return d_st(reinterpret_cast<const double*>(H)[c * FO_BINS + bb]);
              else return (unsigned long long)H[c * FO_BINS + bb];
            };
            unsigned cntb[8];
            unsigned ltot = 0, pmask = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) { cntb[j] = H[cnt_off + lane * 8 + j]; ltot += cntb[j]; if (cntb[j]) pmask |= 1u << j; }
            // exclusive prefix of sample counts over lanes
            unsigned pre = ltot;
            for (int o = 1; o < 32; o <<= 1) { unsigned v = __shfl_up_sync(0xffffffffu, pre, o); if (lane >= o) pre += v; }
            pre -= ltot;
            // class-weight prefixes
            unsigned long long clspre[CM];
            FOR_C(c) {
              unsigned long long t = 0;
#pragma unroll
              for (int j = 0; j < 8; ++j) t = st_add<REG>(t, hbin(c, lane * 8 + j));
              unsigned long long incl = t;
              for (int o = 1; o < 32; o <<= 1) {
                unsigned long long v = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl = st_add<REG>(v, incl);
              }
              const unsigned long long up = __shfl_up_sync(0xffffffffu, incl, 1);   // exclusive prefix
              clspre[c] = lane > 0 ? up : 0ull;
            }
            // first present bin of this lane, then "first present bin in any later lane"
            const int myfirst = pmask ? lane * 8 + __ffs(pmask) - 1 : 1 << 20;
            int nxt = 1 << 20;   // first present bin among lanes > lane
            {
              int v = myfirst;
              // suffix minimum (exclusive)
              int run = v;
              for (int o = 1; o < 32; o <<= 1) { int u = __shfl_down_sync(0xffffffffu, run, o); if (lane + o < 32) run = min(run, u); }
              int nx = __shfl_down_sync(0xffffffffu, run, 1);
              nxt = lane < 31 ? nx : (1 << 20);
            }
            const int gfirst = __reduce_min_sync(0xffffffffu, myfirst);
            const int mylast = pmask ? lane * 8 + 31 - __clz(pmask) : -1;
            const int glast = __reduce_max_sync(0xffffffffu, mylast);
            const bool is_const = bv[glast] <= bv[gfirst] + FEATURE_THRESHOLD;
            if (P.random_split) {   // features on bin codes only
              // one candidate per feature: threshold = rand_uniform(min, max) (SK/tree/_utils.pyx:57-61),
              // samples with (double)value <= threshold go left (DensePartitioner.partition_samples)
              FoResult* R = &results[k];
              double thr = 0.0;
              unsigned nl_lane = 0;
              unsigned long long sl[CM];
              FOR_C(c) sl[c] = 0;
              int nin = 0;
              if (!is_const) {
                const double lo = (double)bv[gfirst], hi = (double)bv[glast];
                thr = __dadd_rn(__ddiv_rn(__dmul_rn(__dsub_rn(hi, lo), (double)items[k].rnd), 2147483647.0), lo);
                if (thr == hi) thr = lo;
  #pragma unroll
                for (int j = 0; j < 8; ++j) {
                  const int bb = lane * 8 + j;
                  if ((double)bv[bb] <= thr) {
                    nin += 1;
                    nl_lane += cntb[j];
                    FOR_C(c) sl[c] = st_add<REG>(sl[c], hbin(c, bb));
                  }
                }
              }
              const unsigned n_left_u = __reduce_add_sync(0xffffffffu, nl_lane);
              const int cutbin = (int)__reduce_add_sync(0xffffffffu, (unsigned)nin) - 1;
              FOR_C(c) {
                // lanes hold consecutive bin ranges: an ordered inclusive scan, read from the last lane
                unsigned long long v = sl[c];
                for (int o = 1; o < 32; o <<= 1) {
                  unsigned long long u = __shfl_up_sync(0xffffffffu, v, o);
                  if (lane >= o) v = st_add<REG>(u, v);
                }
                sl[c] = __shfl_sync(0xffffffffu, v, 31);
              }
              if (lane == 0) {
                R->is_const = is_const; R->proxy = -INFINITY; R->pos = end; R->bin = cutbin; R->thr = thr;
                if (!is_const) {
                  const int n_left = (int)n_left_u, n_right = n_node - n_left;
                  if (n_left >= P.min_samples_leaf && n_right >= P.min_samples_leaf) {
                    double wl = 0.0;
                    if constexpr (REG) wl = st_d(sl[0]);
                    else if constexpr (W) { FOR_C(c) wl = __dadd_rn(wl, __dmul_rn(s_cw[c], (double)sl[c])); }
                    else { FOR_C(c) wl += (double)sl[c]; }
                    const double wr = w_node - wl;
                    if (!(wl < MIN_WEIGHT_LEAF || wr < MIN_WEIGHT_LEAF)) {
                      double il, ir;
                      if constexpr (REG) {
                        fo_children_mse(sl, rec.sums, wl, wr, &il, &ir);
                        const double sum_l = st_d(sl[1]), sum_r = __dsub_rn(st_d(rec.sums[1]), sum_l);
                        R->proxy = __dadd_rn(__ddiv_rn(__dmul_rn(sum_l, sum_l), wl), __ddiv_rn(__dmul_rn(sum_r, sum_r), wr));
                      } else if constexpr (W) {
                        fo_children_impurity_w<CM>(sl, rec.sums, s_cw, C, wl, wr, &il, &ir);
                        R->proxy = __dsub_rn(__dmul_rn(-wr, ir), __dmul_rn(wl, il));
                      } else {
                        fo_children_impurity<CM>(sl, rec.sums, C, wl, wr, &il, &ir);
                        R->proxy = __dsub_rn(__dmul_rn(-wr, ir), __dmul_rn(wl, il));
                      }
                      R->pos = start + n_left; R->il = il; R->ir = ir;
                      FOR_C(c) R->sl[c] = sl[c];
                    }
                  }
                }
              }
              continue;
            }
            // candidates of this lane in ascending bin order
            double bproxy = -INFINITY, bil = 0.0, bir = 0.0;
            int bpos = 1 << 30, bbin = -1, bnext = -1;
            unsigned long long bsl[CM];
            FOR_C(c) bsl[c] = 0;
            if (!is_const) {
              unsigned run_cnt = pre;
              unsigned long long sl[CM];
              FOR_C(c) sl[c] = clspre[c];
              for (int j = 0; j < 8; ++j) {
                if (!cntb[j]) continue;
                const int bb = lane * 8 + j;
                run_cnt += cntb[j];
                FOR_C(c) sl[c] = st_add<REG>(sl[c], hbin(c, bb));
                // next present bin
                const unsigned higher = pmask & ~((2u << j) - 1u);
                const int nb2 = higher ? lane * 8 + __ffs(higher) - 1 : nxt;
                if (nb2 >= (1 << 20)) continue;                              // last present bin
                if (!(bv[nb2] > bv[bb] + FEATURE_THRESHOLD)) continue;       // values within 1e-7: same run
                const int n_left = (int)run_cnt, n_right = n_node - n_left;
                if (n_left < P.min_samples_leaf || n_right < P.min_samples_leaf) continue;
                double wl = 0.0;
                if constexpr (REG) wl = st_d(sl[0]);
                else if constexpr (W) { FOR_C(c) wl = __dadd_rn(wl, __dmul_rn(s_cw[c], (double)sl[c])); }
                else { FOR_C(c) wl += (double)sl[c]; }
                const double wr = w_node - wl;
                if (wl < MIN_WEIGHT_LEAF || wr < MIN_WEIGHT_LEAF) continue;
                double il, ir, proxy;
                if constexpr (REG) {     // MSE.proxy_impurity_improvement: sum_l^2 / w_l + sum_r^2 / w_r
                  fo_children_mse(sl, rec.sums, wl, wr, &il, &ir);
                  const double sum_l = st_d(sl[1]), sum_r = __dsub_rn(st_d(rec.sums[1]), sum_l);
                  proxy = __dadd_rn(__ddiv_rn(__dmul_rn(sum_l, sum_l), wl), __ddiv_rn(__dmul_rn(sum_r, sum_r), wr));
                } else if constexpr (W) {
                  fo_children_impurity_w<CM>(sl, rec.sums, s_cw, C, wl, wr, &il, &ir);
                  proxy = __dsub_rn(__dmul_rn(-wr, ir), __dmul_rn(wl, il));
                } else {
                  fo_children_impurity<CM>(sl, rec.sums, C, wl, wr, &il, &ir);
                  proxy = __dsub_rn(__dmul_rn(-wr, ir), __dmul_rn(wl, il));
                }
                if (proxy > bproxy) {
                  bproxy = proxy; bil = il; bir = ir; bpos = start + n_left; bbin = bb; bnext = nb2;
                  FOR_C(c) bsl[c] = sl[c];
                }
              }
            }
            // warp arg-max; ties keep the smallest position (the sequential scan's strict '>')
            double wp = bproxy; int wpos = bpos;
            for (int o = 16; o > 0; o >>= 1) {
              const double op = __shfl_xor_sync(0xffffffffu, wp, o);
              const int opos = __shfl_xor_sync(0xffffffffu, wpos, o);
              if (op > wp || (op == wp && opos < wpos)) { wp = op; wpos = opos; }
            }
            FoResult* R = &results[k];
            if (lane == 0) { R->is_const = is_const; R->proxy = wp; R->pos = wpos; }
            if (bpos == wpos && bproxy == wp && wp > -INFINITY) {   // unique lane: positions are unique per bin
              R->bin = bbin; R->il = bil; R->ir = bir;
              R->thr = (double)bv[bbin] / 2.0 + (double)bv[bnext] / 2.0;
              FOR_C(c) R->sl[c] = bsl[c];
            }
          }
        }
        __syncthreads();
        FO_TICK(4);
        // --- thread 0: commit in draw order, roll back at the first constant feature ---
        if (tid == 0) {
          bool rolled = false;
          for (int k = 0; k < nbatch; ++k) {
            const FoResult& R = results[k];
            if (!R.is_const) {
              if (R.proxy > best_proxy) {
                best_proxy = R.proxy;
                best_feature = items[k].f; best_pos = R.pos; best_bin = R.bin; best_thr = R.thr;
                best_mgl = (R.pos - start) > (end - R.pos);
                best_il = R.il; best_ir = R.ir;
                FOR_C(c) best_sl[c] = R.sl[c];
              }
              continue;
            }
            // undo every swap made after this item's draw, then take the constant branch
            for (int u = s_sim_ulen - 1; u >= items[k].ulen; --u) {
              const int2 sw = undo[u];
              const int t = features[sw.x]; features[sw.x] = features[sw.y]; features[sw.y] = t;
            }
            rstate = items[k].rs; n_visited = items[k].nv; n_drawn = items[k].nd; f_i = items[k].fi;
            { const int fj = items[k].fj;
              const int t = features[fj]; features[fj] = features[n_total_constants]; features[n_total_constants] = t; }
            n_found += 1;
            n_total_constants += 1;
            rolled = true;
            break;
          }
          if (!rolled) { f_i = s_ctrl[1]; n_visited = s_ctrl[7]; n_drawn = s_sim_nd; rstate = s_sim_rs; }
        }
        __syncthreads();
        FO_TICK(5);
      }
      // restore / record the constant-feature invariants (end of node_split_best)
      if (tid == 0) {
        s_ctrl[2] = best_pos; s_ctrl[3] = best_feature; s_ctrl[4] = best_bin; s_ctrl[5] = n_total_constants;
        s_ctrl[6] = best_mgl;
        s_dbl[0] = best_thr; s_dbl[1] = best_il; s_dbl[2] = best_ir;
        if (best_pos < end) {
          double wl = 0.0;
          if constexpr (REG) wl = st_d(best_sl[0]);
          else if constexpr (W) { FOR_C(c) wl = __dadd_rn(wl, __dmul_rn(s_cw[c], (double)best_sl[c])); }
          else { FOR_C(c) wl += (double)best_sl[c]; }
          const double wr = w_node - wl;
          // impurity_improvement (SK/tree/_criterion.pyx:163-190)
          const double a = __dmul_rn(__ddiv_rn(wr, w_node), best_ir);
          const double b = __dmul_rn(__ddiv_rn(wl, w_node), best_il);
          s_dbl[3] = __dmul_rn(__ddiv_rn(w_node, w_samples), __dsub_rn(__dsub_rn(impurity, a), b));
        } else {
          s_dbl[3] = 0.0;
        }
      }
      __syncthreads();
      FO_TICK(6);
      best_pos = s_ctrl[2]; best_feature = s_ctrl[3]; best_bin = s_ctrl[4]; n_total_constants = s_ctrl[5];
      // restore / record the constant-feature prefix (memcpy pair at the end of node_split_best),
      // spread over the block; the next reader of these arrays is behind later barriers
      for (int i = tid; i < n_known; i += FO_THREADS) features[i] = constant_features[i];
      for (int i = n_known + tid; i < n_total_constants; i += FO_THREADS) constant_features[i] = features[i];
      best_mgl = s_ctrl[6];
      best_thr = s_dbl[0]; best_il = s_dbl[1]; best_ir = s_dbl[2]; best_improvement = s_dbl[3];
      is_leaf = is_leaf || best_pos >= end || (best_improvement + FO_EPSILON < P.min_impurity_decrease);

      if (best_pos < end) {
        // --- partition_samples_final: stable partition (keeps sample indices ascending) ---
        // (random splitter over raw values: the value against the drawn threshold, as partition_samples)
        constexpr bool raw = RAW;
        const uint8_t* xb = raw ? nullptr : P.xbin + (size_t)best_feature * n;
        const float* xv = raw ? P.xval + (size_t)best_feature * n : nullptr;
        __shared__ int loff, roff;
        if (tid == 0) { loff = start; roff = best_pos; }
        __syncthreads();
        for (int i0 = start; i0 < end; i0 += FO_THREADS) {
          const int i = i0 + tid;
          uint2 sv = make_uint2(0, 0);
          int isl = 0, isr = 0;
          if (i < end) {
            sv = samp[i];
            isl = raw ? (double)__ldg(xv + sv.x) <= best_thr : xb[sv.x] <= (unsigned)best_bin;
            isr = !isl;
          }
          const unsigned bl = __ballot_sync(0xffffffffu, isl), br = __ballot_sync(0xffffffffu, isr);
          if (lane == 0) { wsum[wid][0] = __popc(bl); wsum[wid][1] = __popc(br); }
          __syncthreads();
          int lo = 0, ro = 0, lt = 0, rt = 0;
          for (int k = 0; k < FO_THREADS / 32; ++k) {
            if (k < wid) { lo += wsum[k][0]; ro += wsum[k][1]; }
            lt += wsum[k][0]; rt += wsum[k][1];
          }
          const int lb = loff, rb = roff;
          if (isl) tmp[lb + lo + __popc(bl & ((1u << lane) - 1))] = sv;
          if (isr) tmp[rb + ro + __popc(br & ((1u << lane) - 1))] = sv;
          __syncthreads();
          if (tid == 0) { loff = lb + lt; roff = rb + rt; }
          __syncthreads();
        }
        for (int i = start + tid; i < end; i += FO_THREADS) samp[i] = tmp[i];
        __syncthreads();
      }
    }

    FO_TICK(7);
    // ------------------------------- _add_node + node_value --------------------------------
    const int node_id = node_count;
    if (node_id >= P.node_cap) { status = 1; break; }
    if (tid == 0) {
      if (rec.parent >= 0) {
        if (rec.is_left) P.o_left[nb + rec.parent] = node_id; else P.o_right[nb + rec.parent] = node_id;
      }
      P.o_imp[nb + node_id] = impurity;
      P.o_nsamp[nb + node_id] = n_node;
      P.o_wn[nb + node_id] = w_node;
      if (is_leaf) {
        P.o_left[nb + node_id] = -1; P.o_right[nb + node_id] = -1;
        P.o_feature[nb + node_id] = -2; P.o_thr[nb + node_id] = -2.0; P.o_mgl[nb + node_id] = 0;
      } else {
        P.o_feature[nb + node_id] = best_feature; P.o_thr[nb + node_id] = best_thr;
        P.o_mgl[nb + node_id] = (uint8_t)best_mgl;
      }
      if constexpr (REG) {
        P.o_val[nb + node_id] = __ddiv_rn(st_d(rec.sums[1]), w_node);               // node mean (MSE.node_value)
      } else if constexpr (W) {
        FOR_C(c)
          P.o_val[(nb + node_id) * C + c] = __ddiv_rn(__dmul_rn(s_cw[c], (double)rec.sums[c]), w_node);
      } else {
        FOR_C(c)
          P.o_val[(nb + node_id) * C + c] = __ddiv_rn((double)rec.sums[c], w_node);   // class fractions
      }
    }
    node_count += 1;
    if (!is_leaf) {
      if (sp + 2 > P.stack_cap) { status = 2; break; }
      if (tid == 0) {
        FoRecord r;
        r.depth = depth + 1; r.parent = node_id; r.n_const = n_total_constants;
        // right child first, then left (popped first)
        r.start = best_pos; r.end = end; r.is_left = 0; r.impurity = best_ir;
        for (int c = 0; c < FO_MAXC; ++c) r.sums[c] = c < C ? st_sub<REG>(rec.sums[c], best_sl[c]) : 0;
        if (sp < FO_SSTK) sstack[sp] = r; else stack[sp] = r;
        r.start = start; r.end = best_pos; r.is_left = 1; r.impurity = best_il;
        for (int c = 0; c < FO_MAXC; ++c) r.sums[c] = c < C ? best_sl[c] : 0;
        if (sp + 1 < FO_SSTK) sstack[sp + 1] = r; else stack[sp + 1] = r;
      }
      sp += 2;
    }
    if (depth > max_depth_seen) max_depth_seen = depth;
    FO_TICK(8);
    __syncthreads();
  }
  if (tid == 0) {
    P.o_count[slot] = node_count;
    P.o_maxdepth[slot] = max_depth_seen;
    P.o_status[slot] = status;
    if (P.o_prof) for (int i = 0; i < 12; ++i) P.o_prof[(size_t)slot * 16 + i] = prof[i];
  }
}

#undef FOR_C
#undef FO_TICK
#undef MIN_WEIGHT_LEAF

// ------------------------------------ binning ---------------------------------------------
// column f of X -> contiguous buffer
__global__ void fo_extract_col(const float* __restrict__ X, int64_t n, int ldx, int f, float* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = X[i * ldx + f];
}
// mark the first element of each run of equal values in a sorted column
__global__ void fo_mark_unique(const float* __restrict__ sorted, int64_t n, int* __restrict__ n_unique,
                               float* __restrict__ vals /*[256]*/) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (i == 0 || sorted[i] != sorted[i - 1]) {
    int k = atomicAdd(n_unique, 1);
    if (k < FO_BINS) vals[k] = sorted[i];    // unordered; sorted afterwards on the host (<= 256 values)
  }
}
__global__ void fo_bin_col(const float* __restrict__ col, int64_t n, const float* __restrict__ vals, int nv,
                           uint8_t* __restrict__ out) {
  __shared__ float sv[FO_BINS];
  if (threadIdx.x < FO_BINS) sv[threadIdx.x] = threadIdx.x < nv ? vals[threadIdx.x] : INFINITY;
  __syncthreads();
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x = col[i];
  int lo = 0, hi = nv - 1;
  while (lo < hi) { int mid = (lo + hi) >> 1; if (sv[mid] < x) lo = mid + 1; else hi = mid; }
  out[i] = (uint8_t)lo;
}

// feature-major codes -> row-major [n][dp] (padding columns 0)
__global__ void fo_rowmajor_kernel(const uint8_t* __restrict__ xbin, int64_t n, int d, int dp, uint8_t* __restrict__ xrow) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;   // one thread per (row, 4 features)
  const int q = dp >> 2;
  if (idx >= n * q) return;
  const int64_t r = idx / q;
  const int f0 = (int)(idx - r * q) * 4;
  unsigned v = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (f0 + k < d) v |= (unsigned)xbin[(size_t)(f0 + k) * n + r] << (8 * k);
  reinterpret_cast<unsigned*>(xrow)[idx] = v;
}

}  // namespace skd

#include <thrust/device_ptr.h>
#include <thrust/execution_policy.h>
#include <thrust/sort.h>

namespace skd {

void forest_free(Ctx* c) {
  ForestData& f = c->forest;
  if (f.xbin) cudaFree(f.xbin);
  if (f.binval) cudaFree(f.binval);
  if (f.xrow) cudaFree(f.xrow);
  if (f.xval) cudaFree(f.xval);
  f = ForestData();
}

// Bin codes of the staged X (feature-major uint8) + the distinct values per feature, for the best
// splitter.  A feature with more than 256 distinct values gets no codes: only the random splitter,
// which reads raw values, can split it.  values: also keep the raw values feature-major (xval, 4 n d
// bytes) for the random splitter; a later random-splitter fit on the same X adds them to the codes.
int forest_prepare(Ctx* c, bool values) {
  ForestData& fd = c->forest;
  if (fd.valid && (fd.xval || !values)) return 0;
  const int64_t n = c->n;
  const int d = (int)c->d, ldx = (int)c->ldx;
  const unsigned g = (unsigned)((n + 255) / 256);
  if (fd.valid) {
    SKD_CUDA(c, cudaMalloc((void**)&fd.xval, (size_t)d * n * sizeof(float)));
    for (int f = 0; f < d; ++f) fo_extract_col<<<g, 256, 0, c->stream>>>(c->X, n, ldx, f, fd.xval + (size_t)f * n);
    c->launches += d;
    SKD_CUDA(c, cudaGetLastError());
    SKD_CUDA(c, cudaStreamSynchronize(c->stream));
    return 0;
  }
  forest_free(c);
  SKD_CUDA(c, cudaMalloc((void**)&fd.xbin, (size_t)d * n));
  SKD_CUDA(c, cudaMalloc((void**)&fd.binval, (size_t)d * FO_BINS * sizeof(float)));
  if (values) SKD_CUDA(c, cudaMalloc((void**)&fd.xval, (size_t)d * n * sizeof(float)));
  float *col, *srt, *dvals; int* dn;
  Scratch sx(c);
  SKD_CUDA(c, sx.alloc(&col, (size_t)n));
  SKD_CUDA(c, sx.alloc(&srt, (size_t)n));
  SKD_CUDA(c, sx.alloc(&dvals, (size_t)FO_BINS));
  SKD_CUDA(c, sx.alloc(&dn, 1));
  std::vector<float> hv(FO_BINS);
  bool well_separated = true, all_coded = true;
  for (int f = 0; f < d; ++f) {
    float* cf = values ? fd.xval + (size_t)f * n : col;   // the column is the raw-value copy when one is kept
    fo_extract_col<<<g, 256, 0, c->stream>>>(c->X, n, ldx, f, cf);
    SKD_CUDA(c, cudaMemcpyAsync(srt, cf, (size_t)n * 4, cudaMemcpyDeviceToDevice, c->stream));
    thrust::sort(thrust::cuda::par.on(c->stream), thrust::device_pointer_cast(srt), thrust::device_pointer_cast(srt + n));
    SKD_CUDA(c, cudaMemsetAsync(dn, 0, 4, c->stream));
    fo_mark_unique<<<g, 256, 0, c->stream>>>(srt, n, dn, dvals);
    int nu = 0;
    SKD_CUDA(c, cudaMemcpyAsync(&nu, dn, 4, cudaMemcpyDeviceToHost, c->stream));
    SKD_CUDA(c, cudaMemcpyAsync(hv.data(), dvals, FO_BINS * 4, cudaMemcpyDeviceToHost, c->stream));
    SKD_CUDA(c, cudaStreamSynchronize(c->stream));
    c->launches += 2;
    if (nu > FO_BINS) {   // no codes; the distinct values stay +inf
      if (all_coded) { fd.uncoded_feature = f; fd.uncoded_distinct = nu; }
      all_coded = false;
      std::fill(hv.begin(), hv.end(), INFINITY);
      fd.h_binval.insert(fd.h_binval.end(), hv.begin(), hv.end());
      SKD_CUDA(c, cudaMemcpyAsync(fd.binval + (size_t)f * FO_BINS, hv.data(), FO_BINS * 4, cudaMemcpyHostToDevice, c->stream));
      SKD_CUDA(c, cudaStreamSynchronize(c->stream));
      continue;
    }
    for (int i = 0; i < nu; ++i)
      if (hv[i] != hv[i]) return fail(c, "forest: NaN feature values are not supported on the device path");
    std::sort(hv.begin(), hv.begin() + nu);
    for (int i = 0; i + 1 < nu; ++i)      // the splitter's float32 tie test (SK/tree/_partitioner.pyx:210-214)
      if (!(hv[i + 1] > hv[i] + FEATURE_THRESHOLD)) well_separated = false;
    for (int i = nu; i < FO_BINS; ++i) hv[i] = INFINITY;
    fd.h_binval.insert(fd.h_binval.end(), hv.begin(), hv.end());
    SKD_CUDA(c, cudaMemcpyAsync(dvals, hv.data(), FO_BINS * 4, cudaMemcpyHostToDevice, c->stream));
    SKD_CUDA(c, cudaMemcpyAsync(fd.binval + (size_t)f * FO_BINS, hv.data(), FO_BINS * 4, cudaMemcpyHostToDevice, c->stream));
    fo_bin_col<<<g, 256, 0, c->stream>>>(cf, n, dvals, nu, fd.xbin + (size_t)f * n);
    SKD_CUDA(c, cudaStreamSynchronize(c->stream));
    c->launches += 1;
  }
  fd.dp = (d + 15) / 16 * 16;
  if (all_coded) {   // the throughput builder's row-major codes
    SKD_CUDA(c, cudaMalloc((void**)&fd.xrow, (size_t)n * fd.dp));
    const int64_t total = n * (fd.dp / 4);
    fo_rowmajor_kernel<<<(unsigned)((total + 255) / 256), 256, 0, c->stream>>>(fd.xbin, n, d, fd.dp, fd.xrow);
    c->launches += 1;
  }
  fd.all_coded = all_coded;
  fd.well_separated = well_separated && all_coded;
  SKD_CUDA(c, cudaGetLastError());
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  fd.valid = true;
  return 0;
}

// Build `n_trees` trees.  counts: [n_trees][n] uint8 host array of bootstrap multiplicities,
// rand_states: [n_trees] splitter seeds.  Results are delivered tree by tree through `sink`.
// Two builders: forest_fast.cu (classification, best splitter, <= 4 classes: seven trees per SM)
// and the general kernel above (two per SM).  Trees are built in rounds of `slots` concurrent
// trees; the node arrays of a slot hold `node_cap` nodes, sized from the free device memory; a tree
// that outgrows them (status 1) is rebuilt in a later round with the worst-case capacity 2n - 1.
int forest_fit(Ctx* c, int n_trees, const uint8_t* counts, const uint32_t* rand_states, int n_classes,
               int max_features, int max_depth, int min_samples_split, int min_samples_leaf,
               double min_weight_leaf, double min_impurity_decrease, int random_split, const double* h_yreal,
               const ForestClassWeights* cw, ForestSink sink, void* sink_arg) {
  if (forest_prepare(c, false)) return 1;
  // the random splitter reads raw values when a feature has no bin codes; on codes alone its histogram
  // form is faster (config-4 lattice, H100: profiles/README.md)
  const bool raw_values = random_split && !c->forest.all_coded;
  if (raw_values && forest_prepare(c, true)) return 1;
  if (!random_split && !c->forest.all_coded) {
    char b[220];
    snprintf(b, sizeof(b), "forest: feature %d has %d distinct values; the histogram splitter needs <= %d "
             "(continuous features need the sort-based splitter, not built yet)", c->forest.uncoded_feature,
             c->forest.uncoded_distinct, FO_BINS);
    return fail(c, b);
  }
  const bool reg = h_yreal != nullptr;       // regression trees (MSE) on float64 targets
  if (reg) n_classes = 1;
  if (n_classes < 1 || n_classes > FO_MAXC) return fail(c, "forest: device path supports up to 16 classes");
  if (!reg && !c->ycls) return fail(c, "forest: stage labels first");
  const bool weighted = cw != nullptr;
  if (weighted && reg) return fail(c, "forest: class weights are staged but this is a regression fit");
  if (weighted && cw->n_classes != n_classes) return fail(c, "forest: staged class weights do not match n_classes");
  const int64_t n = c->n;
  const int d = (int)c->d;
  if ((size_t)4 * d * sizeof(int) > 6 * 1024) return fail(c, "forest: device path supports up to 384 features (shared-memory feature permutation)");
  bool fast = forest_fast_supported(c, n_classes, reg, random_split);
  if (fast && weighted && !cw->balanced_subsample) {
    // the float32 rank value of the fast builder needs the positive weights within 2^40 of each other
    // (balanced_subsample weights are within n of each other)
    double lo = INFINITY, hi = 0.0;
    for (double w : cw->w) if (w > 0.0) { lo = std::min(lo, w); hi = std::max(hi, w); }
    if (!(hi > 0.0) || hi > 1099511627776.0 * lo) fast = false;
  }
  const int stack_cap = 4096;
  const size_t rec_bytes = fast ? forest_fast_record_bytes(n_classes) : sizeof(FoRecord);
  const size_t node_bytes = fast ? 32 : (size_t)(4 * 4 + 1 + 8 * 3 + 8 * n_classes);   // fast builder: compact records
  const size_t slot_fixed = (size_t)n * 17 + (size_t)stack_cap * rec_bytes + 64;   // two sample buffers + counts + stack
  const int64_t node_cap_max = std::max<int64_t>(2 * n, 16);
  int64_t node_cap = node_cap_max;
  if (const char* e = getenv("SKDIST_B200_FOREST_NODECAP")) {   // experiments / tests: smaller output arrays per tree
    const long long v = atoll(e);
    if (v > 0 && v < node_cap) node_cap = v;
  }
  const bool want_prof = getenv("SKDIST_B200_FOREST_PROF") != nullptr;
  double* dy = nullptr;
  Scratch sy(c);
  if (reg) {
    SKD_CUDA(c, sy.alloc(&dy, (size_t)n));
    SKD_CUDA(c, cudaMemcpyAsync(dy, h_yreal, (size_t)n * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    c->h2d += n * 8;
  }
  double* dcw = nullptr;
  Scratch sw(c);
  if (weighted) {
    std::vector<double> hw(FO_MAXC, 1.0);
    if (!cw->balanced_subsample) std::copy(cw->w.begin(), cw->w.end(), hw.begin());
    SKD_CUDA(c, sw.alloc(&dcw, (size_t)FO_MAXC));
    SKD_CUDA(c, cudaMemcpyAsync(dcw, hw.data(), FO_MAXC * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    c->h2d += FO_MAXC * 8;
  }
  const size_t smem_general = (size_t)2 * d * sizeof(int) + (size_t)(d + 16) * sizeof(int2) +
                              (size_t)FO_KB_MAX * FO_BINS * sizeof(float) + (size_t)FO_SSTK * sizeof(FoRecord);
  // the general builder for this fit (CM: class-count bound; W: class weights)
  void (*general)(const FoParams) = nullptr;
#define FO_PICK(CM, REG, W) (raw_values ? forest_build_kernel<CM, REG, W, true> : forest_build_kernel<CM, REG, W, false>)
  if (reg) general = FO_PICK(4, true, false);
  else if (n_classes <= 2) general = weighted ? FO_PICK(2, false, true) : FO_PICK(2, false, false);
  else if (n_classes <= 4) general = weighted ? FO_PICK(4, false, true) : FO_PICK(4, false, false);
  else if (n_classes <= 8) general = weighted ? FO_PICK(8, false, true) : FO_PICK(8, false, false);
  else general = weighted ? FO_PICK(FO_MAXC, false, true) : FO_PICK(FO_MAXC, false, false);
#undef FO_PICK
  if (!fast) SKD_CUDA(c, cudaFuncSetAttribute(general, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_general));
  std::vector<int> pending(n_trees);
  for (int t = 0; t < n_trees; ++t) pending[t] = t;
  c->forest_kernel_ms = 0.0;
  std::vector<int32_t> hl, hr, hf, hn; std::vector<uint8_t> hm; std::vector<double> ht, hi, hw, hv;
  for (int round = 0; !pending.empty(); ++round) {
    // slots: concurrent trees of this round, bounded by the resident builders and by memory
    size_t free_b = 0, total_b = 0;
    SKD_CUDA(c, cudaMemGetInfo(&free_b, &total_b));
    free_b += c->pool_bytes;                       // idle pooled blocks are reusable
    int slots = (fast ? forest_fast_slots_per_sm() : 2) * c->sm_count;
    if (slots > (int)pending.size()) slots = (int)pending.size();
    const size_t budget = (size_t)((double)free_b * 0.85);
    if (round == 0 && fast && node_cap == node_cap_max) {
      // the node arrays get what the fixed per-tree buffers leave; real trees are far below 2n nodes
      if ((size_t)slots * slot_fixed < budget) {
        const int64_t cap = (int64_t)((budget - (size_t)slots * slot_fixed) / ((size_t)slots * node_bytes));
        node_cap = std::max<int64_t>(4096, std::min<int64_t>(node_cap_max, cap));
      }
    }
    const size_t per_slot = slot_fixed + (size_t)node_cap * node_bytes;
    if ((size_t)slots * per_slot > budget) slots = (int)(budget / per_slot);
    if (slots < 1) return fail(c, "forest: not enough device memory for one tree");
    Scratch sx(c);
    FoParams P;
    memset(&P, 0, sizeof(P));
    uint8_t* dcounts; uint32_t* drs; void* dstack;
    SKD_CUDA(c, sx.alloc(&dcounts, (size_t)slots * n));
    SKD_CUDA(c, sx.alloc(&drs, (size_t)slots));
    SKD_CUDA(c, sx.alloc(&P.samp, (size_t)slots * n));
    SKD_CUDA(c, sx.alloc(&P.samp_tmp, (size_t)slots * n));
    SKD_CUDA(c, sx.alloc((uint8_t**)&dstack, (size_t)slots * stack_cap * rec_bytes));
    uint32_t* d_nodes = nullptr;
    if (fast) {
      SKD_CUDA(c, sx.alloc(&d_nodes, (size_t)slots * node_cap * 8));
    } else {
      SKD_CUDA(c, sx.alloc(&P.o_left, (size_t)slots * node_cap));
      SKD_CUDA(c, sx.alloc(&P.o_right, (size_t)slots * node_cap));
      SKD_CUDA(c, sx.alloc(&P.o_feature, (size_t)slots * node_cap));
      SKD_CUDA(c, sx.alloc(&P.o_nsamp, (size_t)slots * node_cap));
      SKD_CUDA(c, sx.alloc(&P.o_mgl, (size_t)slots * node_cap));
      SKD_CUDA(c, sx.alloc(&P.o_thr, (size_t)slots * node_cap));
      SKD_CUDA(c, sx.alloc(&P.o_imp, (size_t)slots * node_cap));
      SKD_CUDA(c, sx.alloc(&P.o_wn, (size_t)slots * node_cap));
      SKD_CUDA(c, sx.alloc(&P.o_val, (size_t)slots * node_cap * n_classes));
    }
    SKD_CUDA(c, sx.alloc(&P.o_count, (size_t)slots));
    SKD_CUDA(c, sx.alloc(&P.o_maxdepth, (size_t)slots));
    SKD_CUDA(c, sx.alloc(&P.o_status, (size_t)slots));
    long long* d_prof = nullptr;
    if (want_prof) SKD_CUDA(c, sx.alloc(&d_prof, (size_t)slots * 16));
    P.stack = (FoRecord*)dstack;
    P.xbin = c->forest.xbin; P.binval = c->forest.binval; P.xval = raw_values ? c->forest.xval : nullptr; P.ycls = c->ycls; P.yreal = dy;
    P.n = n; P.d = d; P.n_classes = n_classes;
    P.max_features = max_features; P.max_depth = max_depth; P.min_samples_split = min_samples_split;
    P.min_samples_leaf = min_samples_leaf; P.min_weight_leaf = min_weight_leaf;
    P.min_impurity_decrease = min_impurity_decrease;
    P.random_split = random_split ? 1 : 0;
    P.counts = dcounts; P.rand_state = drs; P.stack_cap = stack_cap; P.node_cap = node_cap;
    P.o_prof = d_prof;
    if (weighted) {
      P.cw_bs = cw->balanced_subsample ? 1 : 0; P.cw = dcw; P.min_weight_fraction = cw->min_weight_fraction;
    }
    FfParams F;
    memset(&F, 0, sizeof(F));
    F.xrow = c->forest.xrow; F.ycls = c->ycls; F.n = n; F.d = d; F.dp = c->forest.dp; F.n_classes = n_classes;
    F.max_features = max_features; F.max_depth = max_depth; F.min_samples_split = min_samples_split;
    F.min_samples_leaf = min_samples_leaf; F.min_weight_leaf = min_weight_leaf;
    F.min_impurity_decrease = min_impurity_decrease;
    F.counts = dcounts; F.rand_state = drs; F.samp = P.samp; F.samp_tmp = P.samp_tmp; F.stack = dstack;
    F.stack_cap = stack_cap; F.node_cap = node_cap;
    F.o_nodes = d_nodes;
    F.o_count = P.o_count; F.o_maxdepth = P.o_maxdepth; F.o_status = P.o_status; F.o_prof = d_prof;
    F.weighted = weighted ? 1 : 0; F.cw_bs = P.cw_bs; F.cw = P.cw; F.min_weight_fraction = P.min_weight_fraction;
    std::vector<int32_t> hcount(slots), hdepth(slots), hstatus(slots);
    std::vector<uint32_t> hrs(slots);
    std::vector<int> failed;
    SkdTreeView view;
    for (size_t p0 = 0; p0 < pending.size(); p0 += slots) {
      const int nt = (int)std::min<size_t>(slots, pending.size() - p0);
      const bool contiguous = pending[p0 + nt - 1] - pending[p0] == nt - 1;
      if (!counts) {   // no bootstrap: every row once
        SKD_CUDA(c, cudaMemsetAsync(dcounts, 1, (size_t)nt * n, c->stream));
      } else if (contiguous) {
        SKD_CUDA(c, cudaMemcpyAsync(dcounts, counts + (size_t)pending[p0] * n, (size_t)nt * n, cudaMemcpyHostToDevice, c->stream));
      } else {
        for (int s = 0; s < nt; ++s)
          SKD_CUDA(c, cudaMemcpyAsync(dcounts + (size_t)s * n, counts + (size_t)pending[p0 + s] * n, (size_t)n, cudaMemcpyHostToDevice, c->stream));
      }
      for (int s = 0; s < nt; ++s) hrs[s] = rand_states[pending[p0 + s]];
      SKD_CUDA(c, cudaMemcpyAsync(drs, hrs.data(), (size_t)nt * 4, cudaMemcpyHostToDevice, c->stream));
      c->h2d += (int64_t)nt * n;
      P.n_trees = nt;
      cudaEvent_t k0, k1;
      SKD_CUDA(c, cudaEventCreate(&k0));
      SKD_CUDA(c, cudaEventCreate(&k1));
      SKD_CUDA(c, cudaEventRecord(k0, c->stream));
      if (fast) {
        if (forest_fast_launch(c, F, nt)) return 1;
      } else {
        general<<<nt, FO_THREADS, smem_general, c->stream>>>(P);
        c->launches += 1;
      }
      SKD_CUDA(c, cudaGetLastError());
      SKD_CUDA(c, cudaEventRecord(k1, c->stream));
      SKD_CUDA(c, cudaMemcpyAsync(hcount.data(), P.o_count, nt * 4, cudaMemcpyDeviceToHost, c->stream));
      SKD_CUDA(c, cudaMemcpyAsync(hdepth.data(), P.o_maxdepth, nt * 4, cudaMemcpyDeviceToHost, c->stream));
      SKD_CUDA(c, cudaMemcpyAsync(hstatus.data(), P.o_status, nt * 4, cudaMemcpyDeviceToHost, c->stream));
      SKD_CUDA(c, cudaStreamSynchronize(c->stream));
      { float kms = 0.f; cudaEventElapsedTime(&kms, k0, k1); c->forest_kernel_ms += kms; cudaEventDestroy(k0); cudaEventDestroy(k1); }
      if (want_prof) {
        std::vector<long long> hp((size_t)nt * 16);
        cudaMemcpy(hp.data(), d_prof, hp.size() * 8, cudaMemcpyDeviceToHost);
        static const char* nm_g[12] = {"pop", "speculate", "zero+stage", "histogram", "scan", "commit", "restore+improve", "partition", "add_node+push", "-", "loop barrier", "-"};
        static const char* nm_f[12] = {"pop+header", "stage subtree", "draw", "gather hist", "scan (unstaged)", "hist+scan (staged)", "rank (<=32)", "commit", "finish split", "partition", "add_node+push", "-"};
        const char** nm = fast ? nm_f : nm_g;
        const int np = fast ? 11 : 12;
        double tot = 0; for (int i = 0; i < np; ++i) tot += (double)hp[i];
        for (int i = 0; i < np; ++i) if (hp[i]) fprintf(stderr, "[skd forest prof] tree 0 %-18s %12lld cycles %5.1f%%  (%.0f per node)\n", nm[i], hp[i], 100.0 * hp[i] / tot, (double)hp[i] / hcount[0]);
        if (fast) fprintf(stderr, "[skd forest prof] tree 0 nodes: unstaged %lld, staged histogram %lld, staged rank %lld, leaves %lld; total %.3f Gcycles\n",
                          hp[11], hp[12], hp[13], hp[14], tot * 1e-9);
      }
      if (fast) {
        // compact records: trees come back through a ring of pinned buffers; the copies are issued by
        // this thread, a few host threads wait for them and hand the trees to the consumer (which copies
        // 12 MB per tree out of the pinned buffer: a single thread would be the bottleneck)
        constexpr int NB = 8, NW = 4;
        size_t max_m = 1;
        for (int s = 0; s < nt; ++s) if (hstatus[s] == 0) max_m = std::max(max_m, (size_t)hcount[s]);
        if (c->pin_tree_bytes < max_m * 32) {
          for (void*& pb : c->pin_tree) { if (pb) cudaFreeHost(pb); pb = nullptr; }
          c->pin_tree_bytes = max_m * 32 + (max_m * 32) / 8;
          for (void*& pb : c->pin_tree) SKD_CUDA(c, cudaHostAlloc(&pb, c->pin_tree_bytes, cudaHostAllocDefault));
        }
        std::vector<int> ok;
        for (int s = 0; s < nt; ++s) {
          if (hstatus[s] == 1 && node_cap < node_cap_max) { failed.push_back(pending[p0 + s]); continue; }
          if (hstatus[s] != 0) return fail(c, hstatus[s] == 1 ? "forest: node capacity exceeded" : "forest: builder stack capacity exceeded");
          ok.push_back(s);
        }
        cudaEvent_t evc[NB];
        for (int b = 0; b < NB; ++b) SKD_CUDA(c, cudaEventCreateWithFlags(&evc[b], cudaEventDisableTiming));
        std::mutex mu;
        std::condition_variable cv_job, cv_free;
        std::deque<size_t> ready;
        bool busy[NB] = {false}, finished = false;
        std::atomic<int> cuda_err{0};
        auto worker = [&]() {
          cudaSetDevice(c->device);
          for (;;) {
            size_t k;
            {
              std::unique_lock<std::mutex> lk(mu);
              cv_job.wait(lk, [&] { return !ready.empty() || finished; });
              if (ready.empty()) return;
              k = ready.front(); ready.pop_front();
            }
            const int b = (int)(k % NB), s = ok[k];
            if (cudaEventSynchronize(evc[b]) != cudaSuccess) cuda_err = 1;
            SkdTreeView v;
            v.compact = (const uint32_t*)c->pin_tree[b];
            v.binval = c->forest.h_binval.data();
            v.node_count = hcount[s]; v.max_depth = hdepth[s]; v.n_classes = n_classes;
            v.left = v.right = v.feature = v.n_node_samples = nullptr; v.missing_go_to_left = nullptr;
            v.threshold = v.impurity = v.weighted_n_node_samples = v.value = nullptr;
            sink(sink_arg, pending[p0 + s], &v);
            { std::lock_guard<std::mutex> lk(mu); busy[b] = false; }
            cv_free.notify_all();
          }
        };
        std::vector<std::thread> pool;
        for (int w = 0; w < NW; ++w) pool.emplace_back(worker);
        for (size_t k = 0; k < ok.size(); ++k) {
          const int b = (int)(k % NB), s = ok[k];
          { std::unique_lock<std::mutex> lk(mu); cv_free.wait(lk, [&] { return !busy[b]; }); busy[b] = true; }
          cudaMemcpyAsync(c->pin_tree[b], d_nodes + (size_t)s * node_cap * 8, (size_t)hcount[s] * 32, cudaMemcpyDeviceToHost, c->stream);
          cudaEventRecord(evc[b], c->stream);
          { std::lock_guard<std::mutex> lk(mu); ready.push_back(k); }
          cv_job.notify_one();
          c->d2h += (int64_t)hcount[s] * 32;
        }
        { std::lock_guard<std::mutex> lk(mu); finished = true; }
        cv_job.notify_all();
        for (auto& t : pool) t.join();
        for (int b = 0; b < NB; ++b) cudaEventDestroy(evc[b]);
        if (cuda_err) return fail(c, "forest: copying the trees back failed");
        SKD_CUDA(c, cudaGetLastError());
        continue;
      }
      for (int s = 0; s < nt; ++s) {
        if (hstatus[s] == 1 && node_cap < node_cap_max) { failed.push_back(pending[p0 + s]); continue; }
        if (hstatus[s] != 0) return fail(c, hstatus[s] == 1 ? "forest: node capacity exceeded" : "forest: builder stack capacity exceeded");
        const int m = hcount[s];
        hl.resize(m); hr.resize(m); hf.resize(m); hn.resize(m); hm.resize(m); ht.resize(m); hi.resize(m); hw.resize(m);
        hv.resize((size_t)m * n_classes);
        const size_t o = (size_t)s * node_cap;
        SKD_CUDA(c, cudaMemcpyAsync(hl.data(), P.o_left + o, m * 4, cudaMemcpyDeviceToHost, c->stream));
        SKD_CUDA(c, cudaMemcpyAsync(hr.data(), P.o_right + o, m * 4, cudaMemcpyDeviceToHost, c->stream));
        SKD_CUDA(c, cudaMemcpyAsync(hf.data(), P.o_feature + o, m * 4, cudaMemcpyDeviceToHost, c->stream));
        SKD_CUDA(c, cudaMemcpyAsync(hn.data(), P.o_nsamp + o, m * 4, cudaMemcpyDeviceToHost, c->stream));
        SKD_CUDA(c, cudaMemcpyAsync(hm.data(), P.o_mgl + o, m, cudaMemcpyDeviceToHost, c->stream));
        SKD_CUDA(c, cudaMemcpyAsync(ht.data(), P.o_thr + o, m * 8, cudaMemcpyDeviceToHost, c->stream));
        SKD_CUDA(c, cudaMemcpyAsync(hi.data(), P.o_imp + o, m * 8, cudaMemcpyDeviceToHost, c->stream));
        SKD_CUDA(c, cudaMemcpyAsync(hw.data(), P.o_wn + o, m * 8, cudaMemcpyDeviceToHost, c->stream));
        SKD_CUDA(c, cudaMemcpyAsync(hv.data(), P.o_val + o * n_classes, (size_t)m * n_classes * 8, cudaMemcpyDeviceToHost, c->stream));
        SKD_CUDA(c, cudaStreamSynchronize(c->stream));
        c->d2h += (int64_t)m * (4 * 4 + 1 + 8 * 3 + 8 * n_classes);
        view.node_count = m; view.max_depth = hdepth[s]; view.n_classes = n_classes;
        view.left = hl.data(); view.right = hr.data(); view.feature = hf.data(); view.n_node_samples = hn.data();
        view.missing_go_to_left = hm.data(); view.threshold = ht.data(); view.impurity = hi.data();
        view.weighted_n_node_samples = hw.data(); view.value = hv.data();
        sink(sink_arg, pending[p0 + s], &view);
      }
    }
    pending.swap(failed);
    node_cap = node_cap_max;      // trees that outgrew their arrays: worst-case capacity, fewer at a time
  }
  return 0;
}

}  // namespace skd
