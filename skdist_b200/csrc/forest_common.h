// forest_common.h -- what the two tree builders (forest.cu: general, forest_fast.cu: throughput build for
// classification / best splitter) share: launch parameters, the RNG, the node-record format.
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>

#include <vector>

namespace skd {

struct Ctx;

constexpr int FF_UW = 6144;       // 32-bit words of the fast builder's histogram / staging area (24 KB)
constexpr double FOREST_EPSILON = 2.220446049250313e-16;   // np.finfo('double').eps (SK/tree/_tree.pyx EPSILON)

// Node records, the output of both builders.  Nodes in depth-first order (left child = id + 1); every record
// starts with the same four words:
//   0: right child, patched at the parent when the right child is added; 0xFFFFFFFF for a leaf
//   1: feature in the low 16 bits, 0xFFFF for a leaf
//   2: n_node_samples
//   3: depth
// FOREST_REC_FAST (forest_fast.cu, 32 bytes): word 1 holds the two bins around the threshold in bits 16..31,
//   words 4..7 the uint32 class sums (up to 4 classes).
// FOREST_REC_CLASS / FOREST_REC_REG (forest.cu, 24 + 8 C bytes): the float64 threshold, then the C 64-bit
//   statistics of the node -- integer class sums (C = n_classes), or the float64 bit patterns of
//   {sum w, sum w y, sum w y^2} of a regression tree (C = 3).
// The host forms every float64 field of the tree from them (api.cu: skd_forest_tree_copy).
enum ForestRecordKind : int { FOREST_REC_FAST = 0, FOREST_REC_CLASS = 1, FOREST_REC_REG = 2 };
__host__ __device__ inline int forest_record_stats(int kind, int n_classes) { return kind == FOREST_REC_REG ? 3 : n_classes; }
__host__ __device__ inline size_t forest_record_bytes(int kind, int n_classes) {
  return kind == FOREST_REC_FAST ? 32 : 24 + 8 * (size_t)forest_record_stats(kind, n_classes);
}

// Launch parameters of both builders
struct ForestParams {
  const int32_t* ycls;        // [n] class ids (classification)
  int64_t n;
  int d, n_classes;
  int max_features, max_depth, min_samples_split, min_samples_leaf;
  double min_weight_leaf, min_impurity_decrease;
  // per tree (index = blockIdx.x)
  const uint8_t* counts;      // [trees][n] bootstrap multiplicities (sample_weight)
  const uint32_t* rand_state; // [trees]
  int n_trees;
  // per tree work + output buffers
  uint2* samp;                // [trees][n]   (sample index, (weight << 8) | class)
  uint2* samp_tmp;            // [trees][n]
  void* stack;                // [trees][stack_cap] builder-stack spill (records of the builder's own type)
  int stack_cap;
  int64_t node_cap;
  uint32_t* o_nodes;          // [trees][node_cap] node records (above), forest_record_bytes() each
  int32_t* o_count; int32_t* o_maxdepth; int32_t* o_status;    // [trees]; status 0 ok, 1 node capacity, 2 stack capacity
  long long* o_prof;          // [trees][16] cycles per builder phase / node counts (SKDIST_B200_FOREST_PROF=1), else nullptr
  // class weights (see ForestClassWeights); read only by the weighted instantiations
  int weighted, cw_bs;        // weighted fit; balanced_subsample (weights formed per tree from its root class sums)
  const double* cw;           // [n_classes] weights shared by every tree (cw_bs == 0)
  double min_weight_fraction; // min_weight_leaf of a tree = fraction * its weighted_n_samples
};

struct FfParams : ForestParams {
  const uint8_t* xrow;        // [n][dp] bin codes, row-major (dp = d rounded up to 16)
  int dp;
  int stage_rows, stage_ws;   // staged subtree: max rows, words per staged row (set by forest_fast_launch)
};

// Class weights of a forest classifier fit.  Tree t is fitted with sample_weight count_i * w[y_i]: every
// node statistic is w_c * (integer class count), formed in float64 with one rounding.
struct ForestClassWeights {
  int n_classes = 0;                 // 0: none staged
  std::vector<double> w;             // [n_classes], unused with balanced_subsample
  bool balanced_subsample = false;   // per tree: w_c = n / (K_present * N_c) from the bootstrap class counts N_c
  double min_weight_fraction = 0.0;
};

// balanced_subsample weights from a tree's integer root class sums (compute_class_weight("balanced") of
// the bootstrap sample: n_samples / (n_present_classes * bincount); absent classes 0).  The builders form
// the same two float64 operations on the device.
inline void forest_subsample_weights(const unsigned long long* sums, int C, double* w) {
  uint64_t n = 0; int kp = 0;
  for (int c = 0; c < C; ++c) { n += sums[c]; kp += sums[c] != 0; }
  for (int c = 0; c < C; ++c) {
    const volatile double den = (double)kp * (double)sums[c];
    w[c] = sums[c] ? (double)n / den : 0.0;
  }
}

// scikit-learn's rand_r / rand_int (SK/utils/_random.pxd:20-34): the splitters' xorshift stream
__device__ __forceinline__ uint32_t forest_rand_r(uint32_t* seed) {
  if (*seed == 0) *seed = 1;
  *seed ^= (uint32_t)(*seed << 13);
  *seed ^= (uint32_t)(*seed >> 17);
  *seed ^= (uint32_t)(*seed << 5);
  return *seed % ((uint32_t)2147483647 + 1);
}
__device__ __forceinline__ int forest_rand_int(int low, int high, uint32_t* seed) {
  return low + (int)(forest_rand_r(seed) % (uint32_t)(high - low));
}

bool forest_fast_supported(const Ctx* c, int n_classes, bool reg, int random_split, bool entropy);
int forest_fast_slots_per_sm();
size_t forest_fast_stack_bytes(int n_classes);   // bytes of one builder-stack entry
int forest_fast_launch(Ctx* c, FfParams& P, int nt);

}  // namespace skd
