// forest_common.h -- launch parameters shared by the two tree builders (forest.cu: general,
// forest_fast.cu: throughput build for classification / best splitter).
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>

#include <vector>

namespace skd {

struct Ctx;

constexpr int FF_UW = 6144;       // 32-bit words of the fast builder's histogram / staging area (24 KB)

struct FfParams {
  const uint8_t* xrow;        // [n][dp] bin codes, row-major (dp = d rounded up to 16)
  const int32_t* ycls;        // [n] class ids
  int64_t n;
  int d, dp, n_classes;
  int max_features, max_depth, min_samples_split, min_samples_leaf;
  double min_weight_leaf, min_impurity_decrease;
  int stage_rows, stage_ws;   // staged subtree: max rows, words per staged row (set by forest_fast_launch)
  // per tree (index = blockIdx.x)
  const uint8_t* counts;      // [trees][n] bootstrap multiplicities (sample_weight)
  const uint32_t* rand_state; // [trees]
  int n_trees;
  // per tree work + output buffers
  uint2* samp;                // [trees][n]   (sample index, (weight << 8) | class)
  uint2* samp_tmp;            // [trees][n]
  void* stack;                // [trees][stack_cap] builder-stack spill (records of forest_fast_record_bytes())
  int stack_cap;
  int64_t node_cap;
  uint32_t* o_nodes;          // [trees][node_cap][8] compact node records (see forest_fast.cu: _add_node)
  int32_t* o_count; int32_t* o_maxdepth; int32_t* o_status;    // [trees]; status 0 ok, 1 node capacity, 2 stack capacity
  long long* o_prof;          // [trees][16] cycles per builder phase / node counts (SKDIST_B200_FOREST_PROF=1), else nullptr
  // class weights (see ForestClassWeights); read only by the weighted instantiation
  int weighted, cw_bs;        // weighted fit; balanced_subsample (weights formed per tree from its root class sums)
  const double* cw;           // [n_classes] weights shared by every tree (cw_bs == 0)
  double min_weight_fraction; // min_weight_leaf of a tree = fraction * its weighted_n_samples
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
inline void forest_subsample_weights(const uint32_t* sums, int C, double* w) {
  uint64_t n = 0; int kp = 0;
  for (int c = 0; c < C; ++c) { n += sums[c]; kp += sums[c] != 0; }
  for (int c = 0; c < C; ++c) {
    const volatile double den = (double)kp * (double)sums[c];
    w[c] = sums[c] ? (double)n / den : 0.0;
  }
}

bool forest_fast_supported(const Ctx* c, int n_classes, bool reg, int random_split, bool entropy);
int forest_fast_slots_per_sm();
size_t forest_fast_record_bytes(int n_classes);
int forest_fast_launch(Ctx* c, FfParams& P, int nt);

}  // namespace skd
