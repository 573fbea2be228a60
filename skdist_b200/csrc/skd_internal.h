// skd_internal.h -- context object and helpers shared by the .cu translation units.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <functional>
#include <string>
#include <utility>
#include <vector>

#include "forest_common.h"
#include "lbfgs_core.h"

namespace skd {

struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
};

// Rows per tile of the tensor-core path (logreg_tc.cu): the unit of its tile lists and row bit matrices.  Its
// per-row inputs (rowmeta, rowsg, the staged row bits and sample weights) cover npad = n rounded up to TC_R rows.
constexpr int TC_R = 64;
inline int64_t tc_padded_rows(int64_t n) { return (n + TC_R - 1) / TC_R * TC_R; }

// fp16-split copy of the staged X for the tensor-core path (logreg_tc.cu)
struct TcData {
  void* Xh = nullptr;          // [npad x dpad] fp16, X * xscale rounded to fp16
  void* Xl = nullptr;          // [npad x dpad] fp16, remainder
  uint32_t* rowmeta = nullptr; // [npad] (fold << 24) | class id ; fold 0xFF = padding row
  float* yreal_pad = nullptr;  // [npad] regression targets (zero padded), when staged
  int32_t* tilelist = nullptr; // [(n_lists) x n_tiles] tiles that contain at least one TRAINING row of fold f
  int32_t* tilecnt = nullptr;  // [n_lists]; list index f for fold f, n_lists-1 = every tile (no held-out fold)
  int n_lists = 0;
  int min_list_tiles = 0;      // shortest tile list (chunks without tiles need zeroed partials)
  float* rowsg = nullptr;      // [n_lists x npad] -y * 2^14 per row for positive class rowsg_pos; 0 = not a training row
  int32_t rowsg_pos = -1;
  bool rowsg_valid = false;
  float* xscale = nullptr;     // [dpad] power-of-two per-feature scale
  double* gscale = nullptr;    // [dpad] 1 / (xscale * 2^14): un-scales the gradient partials
  int dpad = 0;
  int64_t npad = 0;
  bool x_valid = false, meta_valid = false;
  CUtensorMap map_xh, map_xl;
};

// binned copy of the staged X for the forest builder (forest.cu)
struct ForestData {
  uint8_t* xbin = nullptr;   // [d][n] bin code of every value, feature-major (features with codes only)
  float* binval = nullptr;   // [d][256] distinct values of each feature, ascending (+inf padded)
  uint8_t* xrow = nullptr;   // [n][dp] the same codes row-major, dp = d rounded up to 16 (forest_fast.cu); only when all_coded
  float* xval = nullptr;     // [d][n] raw values, feature-major: staged by the first random-splitter fit
  int dp = 0;
  bool well_separated = false;   // every feature's adjacent distinct values are more than 1e-7 apart
  bool all_coded = false;        // every feature has <= 256 distinct values (bin codes): the best splitter can run
  int uncoded_feature = -1, uncoded_distinct = 0;   // the first feature without codes and its distinct values
  std::vector<float> h_binval;   // host copy of binval (thresholds of FOREST_REC_FAST records are formed on the host)
  bool valid = false;
};

// host view of one finished tree: node_count node records of `kind` (ForestRecordKind, forest_common.h);
// `binval` ([d][256] distinct feature values) lets the consumer form the thresholds of FOREST_REC_FAST
struct SkdTreeView {
  const uint32_t* records;
  int kind;
  int32_t node_count, max_depth, n_classes;
  const float* binval;
};
typedef void (*ForestSink)(void* arg, int tree_index, const SkdTreeView* view);

// Scoring codes: the per-column col_fold of the scoring entries.  f >= 0 selects the rows of fold f, -2
// every row, -3 - f the rows outside fold f; -1 is not a code.  row_fold is -1 when no folds are staged.
__host__ __device__ __forceinline__ bool score_code_selects(int code, int row_fold) {
  return code == -2 || (code >= 0 && row_fold == code) || (code <= -3 && row_fold != (-3 - code));
}
// the fold a scoring code names (-1: none)
__host__ __device__ __forceinline__ int score_code_fold(int code) {
  return code >= 0 ? code : (code <= -3 ? -3 - code : -1);
}

// One-shot inputs staged for the next call that reads them.  That call takes them off the context
// (std::exchange) before any check, so they never outlive it, whether it succeeds or fails.
struct StagedMasks {          // skd_stage_column_masks: per-column feature masks [cols x d]
  std::vector<uint8_t> mask;
  int32_t cols = 0;
};
struct StagedRowBits {        // skd_stage_row_bits: label of row r in column j / row r trains column j,
  std::vector<uint32_t> y, m; // packed little-endian, `words` 32-bit words per column
  int32_t cols = 0;
  int64_t words = 0;
};
struct StagedClassWeights {   // skd_stage_class_weights: w [cols x k] weight of each class (binary calls:
  std::vector<float> w;       // label 0, label 1), sw_sum [cols] the sum of the column's per-row weights
  std::vector<double> sw_sum; // over its training rows
  int32_t cols = 0, k = 0;
};
struct StagedSampleWeights {  // skd_stage_sample_weights: w [n] per-row weight of every staged row (empty: none)
  std::vector<float> w;
};

struct Ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  std::string err;
  int sm_count = 132;
  int kernel_choice = 0;  // 0 auto, 1 simt, 2 tensor cores (wgmma)
  // staged data
  float* X = nullptr;       // [n x ldx] fp32 row-major
  int64_t n = 0, d = 0, ldx = 0;
  int64_t x_cap_rows = 0;   // allocated rows of X (>= n; the sliced staging pads to a multiple of the world size)
  int64_t pend_n = 0, pend_d = 0;   // shape announced by skd_stage_x_begin, committed by skd_stage_x_commit
  int32_t* ycls = nullptr;  // [n]
  float* yreal = nullptr;   // [n]
  int8_t* fold = nullptr;   // [n]; nullptr = no folds staged (points into fold_store otherwise)
  int8_t* fold_store = nullptr;
  std::vector<int32_t> h_ycls; // host copy of the class ids (training-set sizes of one-vs-one pair columns)
  int32_t ycls_min = 0, ycls_max = -1;  // range of the staged class ids (multinomial entries check it)
  std::vector<int8_t> h_fold;  // host copy of the fold ids (tile lists for fold-aware tile skipping)
  int32_t n_folds = 0;
  std::vector<int64_t> fold_count;  // rows per fold id
  TcData tc;
  ForestData forest;
  int64_t ycls_cap = 0, yreal_cap = 0, fold_cap = 0;   // allocated rows of the staged vectors (reused when large enough)
  int64_t vec_n = 0;        // row count the staged labels / targets / folds belong to (dropped when X changes it)
  // one-shot staged inputs: read by skd_logreg_fit_batch (all four), skd_logreg_loss_grad (class and
  // sample weights), skd_logreg_multinomial_fit_batch (masks, class and sample weights) and skd_forest_fit
  // (forest_cw, n_classes == 0: none; forest_criterion, 0: Gini / MSE, 1: entropy)
  StagedMasks fmask;
  StagedRowBits row_bits;
  StagedClassWeights cw;
  StagedSampleWeights sw;
  float* roww = nullptr;    // device copy of the sample weights a call consumes, [cap] zero padded (reused)
  int64_t roww_cap = 0;
  ForestClassWeights forest_cw;
  int32_t forest_criterion = 0;
  // scratch pool: device blocks released by finished calls, reused by the next ones (Scratch below)
  std::vector<std::pair<void*, size_t>> pool_free;
  size_t pool_bytes = 0;
  // pinned bounce buffers for staging pageable host arrays (api.cu: stage_rows_h2d)
  std::vector<void*> pin_bufs;
  size_t pin_bytes = 0;
  double forest_kernel_ms = 0.0;            // device time of the tree-builder kernels of the last forest_fit (events)
  void* pin_tree[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // pinned ring for finished trees (forest.cu)
  size_t pin_tree_bytes = 0;
  // counters
  int64_t launches = 0, h2d = 0, d2h = 0;
  // optional per-evaluation timing (bench.py roofline): CUDA events on `stream` around every
  // evaluation launch of skd_logreg_fit_batch
  bool prof = false;
  double prof_eval_ms = 0.0;      // summed device time of the evaluation kernels
  double prof_eval_flops = 0.0;   // algorithmic FLOPs of those launches (4 * n_train * d per column)
  int64_t prof_eval_launches = 0; // evaluation launches (one per L-BFGS round)
  int64_t prof_rounds = 0;
  std::vector<cudaEvent_t> prof_events;
  cudaEvent_t timer[2] = {nullptr, nullptr};
};

// error plumbing ---------------------------------------------------------------------
void set_global_error(const std::string& s);
inline int fail(Ctx* c, const std::string& s) {
  if (c) c->err = s;
  set_global_error(s);
  return 1;
}

#define SKD_CUDA(ctx, call)                                                              \
  do {                                                                                   \
    cudaError_t _e = (call);                                                             \
    if (_e != cudaSuccess) {                                                             \
      char _b[512];                                                                      \
      snprintf(_b, sizeof(_b), "%s:%d: %s -> %s", __FILE__, __LINE__, #call,             \
               cudaGetErrorString(_e));                                                  \
      return skd::fail(ctx, _b);                                                         \
    }                                                                                    \
  } while (0)

// Simple RAII device allocation tied to a stream-ordered free at scope exit.
// Scratch device memory of one API call.  Blocks come from (and go back to) a per-context pool so
// that repeated calls (search steps, refits, scoring passes) do not pay cudaMalloc / cudaFree each
// time; every API call synchronises the stream before returning, so a pooled block is idle.
struct Scratch {
  Ctx* ctx;
  std::vector<std::pair<void*, size_t>> blocks;
  explicit Scratch(Ctx* c) : ctx(c) {}
  ~Scratch() {
    for (auto& b : blocks) { ctx->pool_free.push_back(b); ctx->pool_bytes += b.second; }
    // keep the pool bounded: drop the largest idle blocks beyond 6 GB
    while (ctx->pool_bytes > ((size_t)6 << 30) && !ctx->pool_free.empty()) {
      size_t bi = 0;
      for (size_t i = 1; i < ctx->pool_free.size(); ++i)
        if (ctx->pool_free[i].second > ctx->pool_free[bi].second) bi = i;
      cudaFree(ctx->pool_free[bi].first);
      ctx->pool_bytes -= ctx->pool_free[bi].second;
      ctx->pool_free.erase(ctx->pool_free.begin() + bi);
    }
  }
  template <class T>
  cudaError_t alloc(T** out, size_t count) {
    const size_t need = (count * sizeof(T) + 256 + 511) / 512 * 512;
    size_t best = (size_t)-1;
    for (size_t i = 0; i < ctx->pool_free.size(); ++i) {
      const size_t b = ctx->pool_free[i].second;
      if (b >= need && b <= 2 * need + ((size_t)1 << 20) &&
          (best == (size_t)-1 || b < ctx->pool_free[best].second))
        best = i;
    }
    if (best != (size_t)-1) {
      blocks.push_back(ctx->pool_free[best]);
      ctx->pool_bytes -= ctx->pool_free[best].second;
      *out = (T*)ctx->pool_free[best].first;
      ctx->pool_free.erase(ctx->pool_free.begin() + best);
      return cudaSuccess;
    }
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, need);
    if (e != cudaSuccess && !ctx->pool_free.empty()) {   // out of memory: give the idle blocks back and retry
      for (auto& b : ctx->pool_free) cudaFree(b.first);
      ctx->pool_free.clear();
      ctx->pool_bytes = 0;
      cudaGetLastError();
      e = cudaMalloc(&p, need);
    }
    if (e == cudaSuccess) { blocks.push_back({p, need}); *out = (T*)p; }
    return e;
  }
};

// ---- logistic-regression batch solver pieces (logreg_simt.cu / lbfgs_dev.cu) -----------

// Per-slot metadata of the active evaluation batch.
struct SlotMeta {
  int32_t col;     // column id in the caller's batch
  int32_t fold;    // held-out fold id (-1: none)
  int32_t pos;     // positive class id
  int32_t pad;     // neg1: 0 = every other class is a negative (one-vs-rest); k + 1 = only rows of class
                   // `pos` or class k take part (one-vs-one pair)
};

// One batch of device L-BFGS-B problems (lbfgs_dev.cu) and the evaluation partials they read.  Problem b
// (a binary column, or a multinomial candidate) has n = K * (d + 1) variables, variable (k, j) at
// k * (d + 1) + j; the evaluation sees K slots per entry a of the active list (slot a * K + k), K = 1 for
// binary columns.
struct LbfgsBatch {
  int32_t B = 0;               // problems in the batch
  int32_t K = 1;               // classes per problem (1: binary)
  int32_t n = 0;               // variables per problem, K * (d + 1) (intercepts pinned to 0 if !fit_intercept)
  // per problem (indexed by col)
  LbfgsScalars* sc = nullptr;  // [B]
  double* vec = nullptr;       // [B x stride] lbfgs_col_vectors blocks
  size_t stride = 0;           // lbfgs_col_doubles(n, LBFGS_M)
  double* l2 = nullptr;        // [B] l2 strength
  double* inv_n = nullptr;     // [B] 1 / n_train
  int32_t* n_evals = nullptr;  // [B]
  uint8_t* fmask = nullptr;    // [B x d] or nullptr: 1 = feature takes part in the problem's fit
  // active list
  SlotMeta* slot = nullptr;    // [slot_cap] col = problem (-1: padding of the fold-grouped layout)
  int32_t* n_act = nullptr;    // device scalar: entries of the active list
  int32_t* n_run = nullptr;    // device scalar: problems still running, or nullptr (multinomial: n_act)
  // fold-grouped layout (binary tensor-core path): every group of 128 slots holds columns of ONE fold,
  // padded with col = -1 entries, so a group can skip the tiles made only of its held-out rows
  bool grouped = false;
  // evaluation partials of chunk z, indexed by active entry a or slot s = a * K + k
  int32_t nz = 0;              // partials per slot at most
  int32_t ldw = 0;             // row pitch of gradp (ldx, or dpad on the tensor-core path)
  double* lossp = nullptr;     // z * n_act + a
  double* gsump = nullptr;     // z * n_act * K + s
  float* gradp = nullptr;      // (z * n_act * K + s) * ldw + j
  double* gradr = nullptr;     // [slots x ldw] or nullptr: gradp reduced in chunk order (binary tensor-core path)
  const double* gscale = nullptr;  // [d] or nullptr: per-feature un-scaling of gradp (tensor-core path)
  // trial points as fp32 rows [B * K x ldx], then bias [B * K]; nullptr: the tensor-core weights (tc_export)
  float* W = nullptr;
};

// Workspace of one skd_logreg_fit_batch call (device pointers).
struct LogregWork {
  LbfgsBatch lb;        // B columns of d + 1 variables
  int64_t cap_sc = 0;   // capacity of the partial buffers in (chunk, slot) pairs
  int32_t ldg = 0;      // leading dimension of G (columns, padded)
  // per column (indexed by col)
  int32_t* col_fold = nullptr; // [B]
  int32_t* col_pos = nullptr;  // [B]
  int32_t* col_neg1 = nullptr; // [B] or nullptr (see SlotMeta::pad)
  const uint32_t* ybits = nullptr;  // [B x rb_words] or nullptr: bit r of column j = its label of row r (instead of class id == pos)
  const uint32_t* mbits = nullptr;  // [B x rb_words] or nullptr: bit r of column j = row r trains the column
  int64_t rb_words = 0;
  const float2* cw = nullptr;  // [B] or nullptr: {label-0, label-1} weights of column j, largest <= 1
                               // (the power of two that normalised them is folded into inv_n)
  const float* roww = nullptr; // [npad] or nullptr: per-row sample weights, 0 on padding rows (only with cw;
                               // cw is then normalised so that the largest product over a column's training
                               // rows is <= 1)
  float* G = nullptr;          // [n x ldg] pointwise gradients (SIMT path)
  // tensor-core path (logreg_tc.cu)
  bool use_tc = false;
  void* Wh = nullptr;          // [slots_pad_cap x dpad] fp16
  void* Wl = nullptr;          // [slots_pad_cap x dpad] fp16
  void* sp = nullptr;          // [slots_pad_cap] TcSlotParam
  int32_t slots_pad_cap = 0;
  int32_t slot_cap = 0;        // slots incl. padding at the start of the solve
  int32_t uni_pos = -1;        // >= 0: every column of the batch has this positive class (grouped layout only)
  int32_t* deal_log = nullptr; // device [4] or nullptr: the next evaluation's work deal (TcParams::deal_log)
};

// forward (Z = X W^T, pointwise loss / gradient on training rows) + backward (G^T X)
int simt_eval(Ctx* c, LogregWork& w, int n_act, int* nz_used);
// scoring / decision kernels
int simt_score(Ctx* c, int B, const float* dW, const SlotMeta* dslot, int64_t* dcorrect,
               int64_t* dcount);
int simt_decision(Ctx* c, int B, const float* dW, float* dout);
int simt_r2(Ctx* c, int B, const float* dW, const SlotMeta* dslot, double* dsse, int64_t* dcount);
int sgd_fit_batch(Ctx* c, int B, const int32_t* col_pos, int loss, double alpha, int fit_intercept,
                  int max_iter, double tol, int shuffle, uint32_t seed, int lr_type, double eta0,
                  double power_t, double optimal_init, int n_iter_no_change, float* coef_out,
                  double* intercept_out, int32_t* n_iter_out, double* t_out, int32_t* status_out);
// the same fit with per-column alpha / optimal_init and G order groups (rows grows[goff[g] .. goff[g+1]), seed gseed[g])
int sgd_fit_groups(Ctx* c, int B, const int32_t* col_pos, const int32_t* col_group, const double* col_alpha,
                   const double* col_oi, int G, const int64_t* goff, const int32_t* grows, const uint32_t* gseed,
                   int loss, int fit_intercept, int max_iter, double tol, int shuffle, int lr_type, double eta0,
                   double power_t, int n_iter_no_change, float* coef_out, double* intercept_out,
                   int32_t* n_iter_out, double* t_out, int32_t* status_out);
// 2-D fp16 row-major [rows x cols] TMA descriptor, box = [box_rows x 64 cols], 128B swizzle (logreg_tc.cu)
int tc_make_map_2d(Ctx* c, CUtensorMap* map, const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows);
void forest_free(Ctx* c);
int forest_fit(Ctx* c, int n_trees, const uint8_t* counts, const uint32_t* rand_states, int n_classes,
               int max_features, int max_depth, int min_samples_split, int min_samples_leaf,
               double min_weight_leaf, double min_impurity_decrease, bool random_split, bool sort_split,
               bool entropy, const double* h_yreal, const ForestClassWeights* cw, ForestSink sink,
               void* sink_arg);
// weight rows of pitch ldx that predict_device's shared-memory cache holds, at most 8 (0: read from global)
int predict_cache_rows(int64_t ldx);
int predict_device(Ctx* c, const float* dX, int64_t m, int ldx, int d, int B, const float* dW, float* dout);
int forest_predict_device(Ctx* c, const float* dX, int64_t m, int ldx, int n_trees, const int64_t* d_off,
                          const void* d_node, const double* d_thr, const double* d_val, int C, double* d_out);
int ridge_fit_batch(Ctx* c, int B, const double* alpha, const int32_t* hold, int fit_intercept,
                    float* coef_out, int32_t* status_out);
// Caller coefficients [rows x (d+1)] to the kernel layout on the device: weights [rows x ldx], then bias [rows]
int pack_coef(Ctx* c, Scratch& sx, int rows, const float* coef, int64_t d, int64_t ldx, float** dW);

// ---- multinomial logistic regression (logreg_multi.cu) ------------------------------------
// One optimiser problem per candidate with K * (d + 1) variables; active entry a = one candidate
// (slot fold = its held-out fold, -1 none).
struct MultiWork {
  LbfgsBatch lb;                 // B candidates of this solve, K classes, fp32 rows in lb.W
  int64_t rpc = 0;               // rows per chunk (lb.nz chunks, fixed by n alone)
  int32_t ldg = 0;               // leading dimension of G
  float* G = nullptr;            // [n x ldg] raw predictions, overwritten by the pointwise gradients
  const float* cw = nullptr;     // [B x K] or nullptr: weight of each class in the candidate's fit
  const float* roww = nullptr;   // [n] or nullptr (device): sample weight of each row (only with cw)
};
int multi_fit(Ctx* c, int B, int K, const double* l2, const double* inv_n, const int32_t* col_fold, int fit_intercept,
              double tol, int max_iter, const uint8_t* fmask /*[B x d] or nullptr*/,
              const float* cw /*[B x K] or nullptr*/, const float* roww /*device [n] or nullptr*/, float* coef_out,
              int32_t* n_iter_out, int32_t* status_out, double* loss_out, int32_t* n_evals_out);
int multi_loss_grad(Ctx* c, int B, int K, const double* l2, const double* inv_n, const int32_t* col_fold,
                    int fit_intercept, const uint8_t* fmask, const float* cw, const float* roww, const double* w_in,
                    double* loss_out, double* grad_out);
int multi_score(Ctx* c, int B, int K, const float* coef, const int32_t* col_fold, int64_t* conf_out);
int logloss_batch(Ctx* c, int B, int K, const float* coef, const int32_t* col_fold, const int32_t* col_pos,
                  double* loss_sum_out, int64_t* count_out);
// raw predictions / backward product of the fp32 CUDA-core path on arbitrary slot matrices (logreg_simt.cu)
int simt_raw_prediction(Ctx* c, int n_slots, const float* dW, const float* dbias, float* dout, int ldd);
int simt_backward(Ctx* c, const float* G, int ldg, int n_slots, int nz, int64_t rpc, float* gradp);

// Ranked counts of linear classifiers (auc.cu): 2U, n_pos, n_neg and average precision per segment
enum RankScore { RANK_DECISION = 0, RANK_NEG_DECISION = 1, RANK_PROBA = 2 };
int rank_segments(int K, int pairs);
int rank_batch(Ctx* c, int B, int K, const float* coef, const int32_t* col_fold, const int32_t* col_pos, int kind,
               int pairs, int64_t* u2_out, int64_t* n_pos_out, int64_t* n_neg_out, double* ap_out);
// ROC-AUC counts of linear binary classifiers on their decision values: rank_batch with one segment per column
int auc_batch(Ctx* c, int B, const float* coef, const int32_t* col_fold, const int32_t* col_pos, int64_t* u2_out,
              int64_t* n_pos_out, int64_t* n_neg_out);

// tensor-core evaluation (logreg_tc.cu)
bool tc_supported(const Ctx* c);
void tc_free(Ctx* c);
int tc_prepare(Ctx* c);
int tc_export(Ctx* c, LogregWork& w, int n_act_upper, const double* xin, int fit_intercept);
int tc_eval(Ctx* c, LogregWork& w, int n_act, int* nz_used);
int tc_score(Ctx* c, LogregWork& w, int n_act, int64_t* dcorrect, int64_t* dcount);
int tc_r2(Ctx* c, LogregWork& w, int n_act, double* dsse, int64_t* dcount);
size_t tc_slot_param_bytes();
int tc_partials_per_slot();

// device L-BFGS (lbfgs_dev.cu)
// scikit-learn's line-search limit (maxls = 50) and ftol (64 * eps), which every fit passes to scipy
constexpr int LBFGS_MAXLS = 50;
constexpr double LBFGS_FTOL = 64.0 * 2.220446049250313e-16;
constexpr int LBFGS_ROUNDS_PER_SYNC = 4;
// Round cap of a fit (lbfgs_run) and size of its per-round record.  Every round is one evaluation of every
// running problem.  lbfgs_advance consumes at most maxls evaluations per line search: the maxls-th trial
// sets iback = maxls and fails it.  A failed line search with memory restarts once from steepest descent
// (col = 0); a failure without memory ends the fit (LB_ABNORMAL).  So one iteration takes at most
// 2 * maxls evaluations, a fit at most 1 + 2 * maxls * max_iter (the first evaluation consumes no line
// search), and the rounds enqueued after the last problem stopped add fewer than LBFGS_ROUNDS_PER_SYNC.
inline long lbfgs_max_rounds(int max_iter) {
  return 2L * LBFGS_MAXLS * max_iter + 1 + LBFGS_ROUNDS_PER_SYNC;
}
// Allocates the batch's optimiser state and, for slot_cap > 0, its active list and counters (B, K, n set).
int lbfgs_alloc(Ctx* c, Scratch& sx, LbfgsBatch& b, int slot_cap, bool with_n_run);
// State of every problem at w = 0 (SK/linear_model/_logistic.py:443), the dense active list when col_fold is
// given (slot b = problem b, pos col_pos[b] or 0, pad col_neg1[b] or 0), and zero fp32 rows b.W.
int lbfgs_init(Ctx* c, LbfgsBatch& b, const int32_t* col_fold, const int32_t* col_pos, const int32_t* col_neg1,
               double tol, int max_iter, int maxls = LBFGS_MAXLS, double ftol = LBFGS_FTOL);
// One optimiser round on the stream: advance, compact the active list, export the new trial points (into b.W,
// or through tc_export(*tc)).  n_act_in may be a stale upper bound; hist (may be null) receives {slots, running}.
int lbfgs_enqueue(Ctx* c, LbfgsBatch& b, int n_act_in, int nz_used, int fit_intercept, int32_t* hist,
                  LogregWork* tc = nullptr);
// Host round loop of a fit: eval(n_act, round, &nz_used) fills the partials of the active list, then one
// optimiser round; LBFGS_ROUNDS_PER_SYNC rounds per read back of the live counts, until no problem runs.
// hist (may be null) receives {slots, running} of every round.  Returns the rounds enqueued in *rounds.
int lbfgs_run(Ctx* c, LbfgsBatch& b, int n_act, int fit_intercept, int max_iter, int32_t* hist, LogregWork* tc,
              const std::function<int(int n_act, long round, int* nz_used)>& eval, long* rounds);
// caller points dx [rows][K][d+1] (device, float64; row = slot[a].col) as the fp32 rows b.W of n_act_upper entries
int lbfgs_export_points(Ctx* c, LbfgsBatch& b, int n_act_upper, const double* dx);
// f, g of every problem at caller points dx [B][n] from the partials of n_act active entries
int lbfgs_gather(Ctx* c, LbfgsBatch& b, int n_act, int nz_used, int fit_intercept, const double* dx, double* df,
                 double* dg);
// Final coefficients [B][n], iteration counts, statuses, losses and (n_evals_out) evaluation counts copied
// (not yet synchronised) to the host outputs of problems b0 .. b0 + B - 1; loss_out and n_evals_out may be null.
int lbfgs_result(Ctx* c, Scratch& sx, LbfgsBatch& b, int64_t b0, float* coef_out, int32_t* n_iter_out, int32_t* status_out,
                 double* loss_out, int32_t* n_evals_out);

}  // namespace skd
