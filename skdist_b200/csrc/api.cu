// api.cu -- the C-ABI declared in include/skdist_b200.h.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <functional>
#include <memory>
#include <mutex>
#include <thread>
#include <atomic>
#include <chrono>

#include "../../include/skdist_b200.h"
#include "skd_internal.h"

namespace skd {
static std::mutex g_err_mu;
static std::string g_err;
void set_global_error(const std::string& s) {
  std::lock_guard<std::mutex> l(g_err_mu);
  g_err = s;
}
}  // namespace skd

using namespace skd;

struct skd_ctx {
  Ctx c;
};

struct skd_lbfgs {
  LbfgsScalars s;
  LbfgsVectors v;
  std::vector<double> buf;
};

static inline int64_t round_up(int64_t a, int64_t b) { return (a + b - 1) / b * b; }

namespace skd {
int pack_coef(Ctx* c, Scratch& sx, int rows, const float* coef, int64_t d, int64_t ldx, float** dW) {
  std::vector<float> h((size_t)rows * ldx + rows, 0.f);
  for (int j = 0; j < rows; ++j) {
    memcpy(&h[(size_t)j * ldx], coef + (size_t)j * (d + 1), d * sizeof(float));
    h[(size_t)rows * ldx + j] = coef[(size_t)j * (d + 1) + d];
  }
  SKD_CUDA(c, sx.alloc(dW, h.size()));
  SKD_CUDA(c, cudaMemcpyAsync(*dW, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  c->h2d += (int64_t)h.size() * 4;
  return 0;
}
}  // namespace skd

// Copy of n host values into a per-row device vector of the context (buffer reused when it holds n)
template <class T>
static int stage_device_vector(Ctx* c, T*& dst, int64_t& cap, const T* src, int64_t n) {
  if (dst && cap < n) { cudaFree(dst); dst = nullptr; }
  if (!dst) { SKD_CUDA(c, cudaMalloc((void**)&dst, (size_t)n * sizeof(T))); cap = n; }
  SKD_CUDA(c, cudaMemcpyAsync(dst, src, (size_t)n * sizeof(T), cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  c->h2d += n * (int64_t)sizeof(T);
  return 0;
}

// Which evaluation kernel serves this batch: the tensor-core kernel (logreg_tc.cu) or SIMT fp32.
static int eval_dispatch(Ctx* c, LogregWork& w, int n_act, int* nz_used) {
  if (w.use_tc) return tc_eval(c, w, n_act, nz_used);
  return simt_eval(c, w, n_act, nz_used);
}

// 0 = auto: tensor cores whenever the staged shape is supported (d <= 256), else SIMT fp32.
static bool want_tc(const Ctx* c) {
  if (c->kernel_choice == 1) return false;
  if (c->kernel_choice == 2) return true;
  return tc_supported(c) && !getenv("SKDIST_B200_FORCE_SIMT");
}

// want_tc, failing when tensor cores are forced (skd_set_kernel 2) on a shape they do not support
static int use_tensor_cores(Ctx* c, bool* use_tc) {
  if (c->kernel_choice == 2 && !tc_supported(c))
    return fail(c, "tensor-core path requested but the staged shape is unsupported (needs d <= 256)");
  *use_tc = want_tc(c);
  return 0;
}

// Tensor-core weights of `slots` slots: fp16 hi / lo coefficients (zeroed padding) and slot parameters.
static int alloc_tc_weights(Ctx* c, Scratch& sx, LogregWork& w, int slots) {
  w.lb.ldw = c->tc.dpad;
  w.slots_pad_cap = (int)round_up(slots, 128);
  const size_t wbytes = (size_t)w.slots_pad_cap * c->tc.dpad * 2;
  SKD_CUDA(c, sx.alloc((uint8_t**)&w.Wh, wbytes));
  SKD_CUDA(c, sx.alloc((uint8_t**)&w.Wl, wbytes));
  SKD_CUDA(c, sx.alloc((uint8_t**)&w.sp, (size_t)w.slots_pad_cap * tc_slot_param_bytes()));
  SKD_CUDA(c, cudaMemsetAsync(w.Wh, 0, wbytes, c->stream));
  SKD_CUDA(c, cudaMemsetAsync(w.Wl, 0, wbytes, c->stream));
  return 0;
}

// Tensor-core setup of a scoring pass: slot s = column s of coef [B x (d+1)], exported into the weights.
static int tc_scoring_setup(Ctx* c, Scratch& sx, LogregWork& w, int B, const float* coef, SlotMeta* dslot) {
  if (tc_prepare(c)) return 1;
  w.lb.B = B; w.lb.n = (int)c->d + 1; w.use_tc = true;
  w.lb.slot = dslot;
  if (alloc_tc_weights(c, sx, w, B)) return 1;
  SKD_CUDA(c, sx.alloc(&w.lb.n_act, 1));
  std::vector<double> hx((size_t)B * w.lb.n);
  for (size_t i = 0; i < hx.size(); ++i) hx[i] = (double)coef[i];
  double* dx;
  SKD_CUDA(c, sx.alloc(&dx, hx.size()));
  int32_t nb = B;
  SKD_CUDA(c, cudaMemcpyAsync(dx, hx.data(), hx.size() * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(w.lb.n_act, &nb, sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  c->h2d += (int64_t)hx.size() * 8;
  return tc_export(c, w, B, dx, 1);
}

// Decide the evaluation path for a batch and allocate its evaluation buffers.
static int alloc_eval_buffers(Ctx* c, Scratch& sx, LogregWork& w, int B, int slot_cap = 0) {
  const int64_t n = c->n, ldx = c->ldx;
  if (use_tensor_cores(c, &w.use_tc)) return 1;
  if (slot_cap < B) slot_cap = B;
  w.slot_cap = slot_cap;
  // partial sums per slot: row chunks of the SIMT grid, or the fixed chunk count of the tensor-core kernel
  w.cap_sc = w.use_tc ? (int64_t)tc_partials_per_slot() * round_up(slot_cap, 128)
                      : (int64_t)4 * c->sm_count * 64 + slot_cap + 64;
  LbfgsBatch& b = w.lb;
  b.nz = 1024;
  SKD_CUDA(c, sx.alloc(&b.lossp, (size_t)w.cap_sc));
  SKD_CUDA(c, sx.alloc(&b.gsump, (size_t)w.cap_sc));
  if (w.use_tc) {
    if (tc_prepare(c)) return 1;
    b.gscale = c->tc.gscale;
    if (alloc_tc_weights(c, sx, w, slot_cap)) return 1;
    SKD_CUDA(c, sx.alloc(&b.gradp, (size_t)w.cap_sc * b.ldw));
    SKD_CUDA(c, sx.alloc(&b.gradr, (size_t)w.slots_pad_cap * b.ldw));
  } else {
    b.ldw = (int)ldx;
    b.gscale = nullptr;
    w.ldg = (int)round_up(B, 64);
    // the n x B gradient-factor matrix must leave room for X and the solver state: at most 3/4 of the device
    size_t free_b = 0, total_b = 0;
    SKD_CUDA(c, cudaMemGetInfo(&free_b, &total_b));
    if ((double)n * w.ldg * 4.0 > 0.75 * (double)total_b) {
      char b[200];
      snprintf(b, sizeof(b), "skd_logreg_fit_batch: batch too large for one SIMT call (n * B * 4 bytes > %.0f GB, "
               "3/4 of the device); split the batch", 0.75 * (double)total_b / 1e9);
      return fail(c, b);
    }
    SKD_CUDA(c, sx.alloc(&b.W, (size_t)B * ldx + B));
    SKD_CUDA(c, sx.alloc(&w.G, (size_t)n * w.ldg));
    SKD_CUDA(c, sx.alloc(&b.gradp, (size_t)w.cap_sc * ldx));
  }
  return 0;
}

// The fold-grouped slot layout: columns stable-sorted by held-out fold, every fold segment padded with
// col = -1 slots to a multiple of 128 (one MMA group = one fold -> tile skipping).
static int grouped_slot_layout(Ctx* c, int B, const int32_t* col_fold, const int32_t* col_pos, const int32_t* col_neg,
                               std::vector<SlotMeta>& hslots) {
  hslots.clear();
  std::vector<int> order(B);
  for (int j = 0; j < B; ++j) order[j] = j;
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return col_fold[a] < col_fold[b]; });
  for (int i = 0; i < B;) {
    const int f = col_fold[order[i]];
    if (f > 127) return fail(c, "fold id above 127");
    for (; i < B && col_fold[order[i]] == f; ++i) {
      SlotMeta sm; sm.col = order[i]; sm.fold = f < 0 ? -1 : f; sm.pos = col_pos[order[i]];
      sm.pad = (col_neg && col_neg[order[i]] >= 0) ? col_neg[order[i]] + 1 : 0;
      hslots.push_back(sm);
    }
    while (hslots.size() % 128) { SlotMeta sm; sm.col = -1; sm.fold = f < 0 ? -1 : f; sm.pos = -1; sm.pad = 0; hslots.push_back(sm); }
  }
  return 0;
}

// Slot layout of a logistic batch, then its evaluation buffers (alloc_eval_buffers).  The tensor-core
// path runs the fold-grouped layout (grouped_slot_layout), with w.uni_pos set when every column is
// one-vs-rest with the same positive class.  hslots receives that layout; it stays empty for the SIMT
// path, whose slot s is column s.
static int alloc_logreg_slots(Ctx* c, Scratch& sx, LogregWork& w, int B, const int32_t* col_fold,
                              const int32_t* col_pos, const int32_t* col_neg, std::vector<SlotMeta>& hslots) {
  hslots.clear();
  if (want_tc(c) && tc_supported(c) && grouped_slot_layout(c, B, col_fold, col_pos, col_neg, hslots)) return 1;
  if (alloc_eval_buffers(c, sx, w, B, hslots.empty() ? B : (int)hslots.size())) return 1;
  w.lb.grouped = !hslots.empty() && w.use_tc;
  if (!w.lb.grouped) {
    hslots.clear();
    return 0;
  }
  w.uni_pos = col_pos[0];
  for (int j = 1; j < B; ++j)
    if (col_pos[j] != col_pos[0]) { w.uni_pos = -1; break; }
  if (col_neg)
    for (int j = 0; j < B; ++j)
      if (col_neg[j] >= 0) { w.uni_pos = -1; break; }   // pair masks are per column: general epilogue
  return 0;
}

// Non-finite scan of the staged matrix: scikit-learn's estimators reject NaN / infinity in X
// (check_array -> "Input X contains NaN."), so the staging call does too -- at HBM speed, on the
// copy that is already on the device.
__global__ void finite_check_kernel(const float* __restrict__ X, int64_t total, int* __restrict__ flag) {
  int bad = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = X[i];
    bad |= !(fabsf(v) <= 3.402823466e38f);
  }
  if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) atomicOr(flag, 1);
}

// Entropy of one node in bits, as scikit-learn forms it (SK/tree/_criterion.pyx Entropy: e -= p * log(p),
// p = s_c / w in class order, zero sums skipped; SK/tree/_utils.pyx: log(x) = ln(x) / ln(2.0)) with this
// process's libm, the one scikit-learn calls
static double entropy_bits(const double* s, int C, double w) {
  const volatile double ln2 = std::log(2.0);
  volatile double e = 0.0;
  for (int c = 0; c < C; ++c) {
    if (!(s[c] > 0.0)) continue;
    const volatile double p = s[c] / w;
    const volatile double lg = std::log(p) / ln2;
    const volatile double t = p * lg;      // volatile: no contraction of the product into the difference
    e = e - t;
  }
  return e;
}

// Gini of one node, 1 - sum_c s_c^2 / w^2 (SK/tree/_criterion.pyx:650-680)
static double gini(const double* s, int C, double w) {
  volatile double sq = 0.0;
  for (int c = 0; c < C; ++c) {
    const volatile double aa = s[c] * s[c];      // volatile: no contraction of the product into the sum
    sq = sq + aa;
  }
  const volatile double ww = w * w;
  const volatile double q = sq / ww;
  return 1.0 - q;
}

// A node's float64 class sums s_c = cw_c * count_c (one rounding; cw: nullptr when unweighted) and their
// total, weighted_n_node_samples, in class order (SK/tree/_criterion.pyx:483-486)
template <class T>
static double weighted_class_sums(const T* count, int C, const double* cw, double* s) {
  volatile double w = 0.0;
  for (int c = 0; c < C; ++c) {
    const volatile double a = cw ? cw[c] * (double)count[c] : (double)count[c];
    s[c] = a;
    w = w + a;
  }
  return w;
}

// The impurity array of a classification tree (Gini, or entropy in bits) from its integer class sums, as the
// builders and scikit-learn form it.  A node's impurity is the one its parent's children_impurity formed: for
// the root (node_impurity) and a left child from the node's own sums; for a right child from sum_right_c =
// cw_c * t_c - cw_c * l_c and w_right = w_node - w_left.  With non-dyadic class weights those can differ in
// the last bits from the right child's own sums; the tree reports the impurity the builder compared with
// EPSILON and used in the improvement.  Entropy uses this process's libm, the one scikit-learn calls: the
// builder ranks candidates with CUDA's log, which differs from the host's in the last bit on a few inputs.
// sums(i): node i's C class sums; children(i, l, r): node i's children, false for a leaf.
template <class Sums, class Children>
static void forest_class_impurity(int m, int C, const double* cw, bool entropy, Sums sums, Children children,
                                  double* imp) {
  if (m <= 0) return;
  auto impurity = [&](const double* s, double w) { return entropy ? entropy_bits(s, C, w) : gini(s, C, w); };
  std::vector<double> s(C), t(C);
  imp[0] = impurity(s.data(), weighted_class_sums(sums(0), C, cw, s.data()));
  for (int i = 0; i < m; ++i) {
    int l, r;
    if (!children(i, l, r)) continue;
    const double wn = weighted_class_sums(sums(i), C, cw, t.data());
    const double wl = weighted_class_sums(sums(l), C, cw, s.data());
    imp[l] = impurity(s.data(), wl);
    for (int c = 0; c < C; ++c) { const volatile double b = t[c] - s[c]; s[c] = b; }
    const volatile double wr = wn - wl;
    imp[r] = impurity(s.data(), wr);
  }
}

extern "C" {

int skd_version(void) { return 100; }

int skd_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

const char* skd_last_error(skd_ctx* ctx) {
  if (ctx) return ctx->c.err.c_str();
  std::lock_guard<std::mutex> l(g_err_mu);
  static thread_local std::string copy;
  copy = g_err;
  return copy.c_str();
}

int skd_ctx_create(int device, skd_ctx** out) {
  if (!out) return fail(nullptr, "skd_ctx_create: out is NULL");
  *out = nullptr;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return fail(nullptr, std::string("skd_ctx_create: no CUDA device available (") +
                             cudaGetErrorString(e) + "); this library has no CPU fallback");
  }
  if (device < 0 || device >= ndev) return fail(nullptr, "skd_ctx_create: bad device index");
  SKD_CUDA(nullptr, cudaSetDevice(device));
  cudaDeviceProp prop;
  SKD_CUDA(nullptr, cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {   // sm_90a code runs on compute capability 9.0 only
    char b[256];
    snprintf(b, sizeof(b), "skd_ctx_create: device %d is sm_%d%d; this library is built for sm_90a only",
             device, prop.major, prop.minor);
    return fail(nullptr, b);
  }
  skd_ctx* h = new skd_ctx();
  h->c.device = device;
  h->c.sm_count = prop.multiProcessorCount;
  SKD_CUDA(nullptr, cudaStreamCreateWithFlags(&h->c.stream, cudaStreamNonBlocking));
  *out = h;
  return 0;
}

// SKDIST_B200_TRACE=1: host wall-clock per phase of a call (stream synchronised at each mark), to stderr
struct Trace {
  Ctx* c; const char* call; bool on; std::chrono::steady_clock::time_point t;
  Trace(Ctx* c_, const char* call_) : c(c_), call(call_) {
    const char* e = getenv("SKDIST_B200_TRACE");
    on = e && *e && *e != '0';
    t = std::chrono::steady_clock::now();
  }
  void mark(const char* what) {
    if (!on) return;
    cudaStreamSynchronize(c->stream);
    auto n = std::chrono::steady_clock::now();
    fprintf(stderr, "[skd trace] %s %-10s %9.3f ms\n", call, what, std::chrono::duration<double, std::milli>(n - t).count());
    t = n;
  }
};

static void free_staged(Ctx& c) {
  if (c.X) cudaFree(c.X);
  if (c.ycls) cudaFree(c.ycls);
  if (c.yreal) cudaFree(c.yreal);
  if (c.fold_store) cudaFree(c.fold_store);
  if (c.roww) cudaFree(c.roww);
  c.X = nullptr; c.ycls = nullptr; c.yreal = nullptr; c.fold = nullptr; c.fold_store = nullptr;
  c.roww = nullptr; c.roww_cap = 0;
}

int skd_ctx_destroy(skd_ctx* ctx) {
  if (!ctx) return 0;
  cudaSetDevice(ctx->c.device);
  cudaStreamSynchronize(ctx->c.stream);
  free_staged(ctx->c);
  for (void* p : ctx->c.pin_bufs) cudaFreeHost(p);
  ctx->c.pin_bufs.clear();
  for (void* pb : ctx->c.pin_tree) if (pb) cudaFreeHost(pb);
  for (auto& b : ctx->c.pool_free) cudaFree(b.first);
  ctx->c.pool_free.clear();
  tc_free(&ctx->c);
  forest_free(&ctx->c);
  cudaStreamDestroy(ctx->c.stream);
  delete ctx;
  return 0;
}

// Host -> device copy of an [n x d] fp32 matrix (row pitch ldx_src) into dst (row pitch ldx).
// Pinned sources go straight to the copy engine.  Pageable sources (plain numpy arrays) would be
// bounced by the driver through one small internal buffer at a few GB/s; instead T host threads
// each copy their own row blocks into pinned bounce buffers (double-buffered per thread) and
// issue the DMA on their own stream, so memcpy and PCIe transfers of different blocks overlap.
static int stage_rows_h2d(Ctx* c, float* dst, int64_t ldx, const float* src, int64_t n, int64_t d,
                          int64_t ldx_src) {
  cudaPointerAttributes attr;
  bool pinned = cudaPointerGetAttributes(&attr, src) == cudaSuccess && attr.type == cudaMemoryTypeHost;
  cudaGetLastError();
  const size_t total = (size_t)n * d * sizeof(float);
  // rows wider than one bounce block (d * 4 > 8 MiB) cannot go through the threaded bounce: plain copy
  if (pinned || total < ((size_t)8 << 20) || (size_t)d * sizeof(float) > ((size_t)8 << 20)) {
    SKD_CUDA(c, cudaMemcpy2DAsync(dst, ldx * sizeof(float), src, ldx_src * sizeof(float), d * sizeof(float), n,
                                  cudaMemcpyHostToDevice, c->stream));
    SKD_CUDA(c, cudaStreamSynchronize(c->stream));
    return 0;
  }
  const int T = 8, NB = 2;
  const size_t buf_bytes = (size_t)8 << 20;
  if (c->pin_bufs.size() != (size_t)T * NB || c->pin_bytes != buf_bytes) {
    for (void* p : c->pin_bufs) cudaFreeHost(p);
    c->pin_bufs.clear();
    for (int i = 0; i < T * NB; ++i) {
      void* p = nullptr;
      SKD_CUDA(c, cudaHostAlloc(&p, buf_bytes, cudaHostAllocDefault));
      c->pin_bufs.push_back(p);
    }
    c->pin_bytes = buf_bytes;
  }
  const int64_t rows_per_blk = std::max<int64_t>(1, (int64_t)(buf_bytes / ((size_t)d * sizeof(float))));
  const int64_t n_blk = (n + rows_per_blk - 1) / rows_per_blk;
  std::atomic<int> err_code{0};
  std::atomic<int64_t> next_blk{0};
  auto worker = [&](int tid) {
    if (cudaSetDevice(c->device) != cudaSuccess) { err_code = 1; return; }
    cudaStream_t st;
    cudaEvent_t ev[NB];
    if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) { err_code = 1; return; }
    for (int b = 0; b < NB; ++b) cudaEventCreateWithFlags(&ev[b], cudaEventDisableTiming);
    int used = 0;
    for (;;) {
      const int64_t blk = next_blk.fetch_add(1);
      if (blk >= n_blk || err_code) break;
      const int b = used % NB;
      if (used >= NB && cudaEventSynchronize(ev[b]) != cudaSuccess) { err_code = 2; break; }
      float* pb = (float*)c->pin_bufs[(size_t)tid * NB + b];
      const int64_t r0 = blk * rows_per_blk, r1 = std::min(n, r0 + rows_per_blk);
      if (ldx_src == d) {
        memcpy(pb, src + (size_t)r0 * ldx_src, (size_t)(r1 - r0) * d * sizeof(float));
      } else {
        for (int64_t r = r0; r < r1; ++r)
          memcpy(pb + (size_t)(r - r0) * d, src + (size_t)r * ldx_src, (size_t)d * sizeof(float));
      }
      if (cudaMemcpy2DAsync(dst + (size_t)r0 * ldx, ldx * sizeof(float), pb, d * sizeof(float), d * sizeof(float),
                            (size_t)(r1 - r0), cudaMemcpyHostToDevice, st) != cudaSuccess) { err_code = 3; break; }
      cudaEventRecord(ev[b], st);
      ++used;
    }
    if (cudaStreamSynchronize(st) != cudaSuccess) err_code = 4;
    for (int b = 0; b < NB; ++b) cudaEventDestroy(ev[b]);
    cudaStreamDestroy(st);
  };
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));   // the memset of the padding (if any) is ordered before the copies
  std::vector<std::thread> th;
  for (int t = 0; t < T; ++t) th.emplace_back(worker, t);
  for (auto& t : th) t.join();
  if (err_code) {
    char b[128];
    snprintf(b, sizeof(b), "skd_stage_x: threaded host-to-device staging failed (step %d): %s", (int)err_code,
             cudaGetErrorString(cudaGetLastError()));
    return fail(c, b);
  }
  return 0;
}

// device buffer of the staged matrix: kept when the row pitch is unchanged and it is large enough
// (repeated fits on same-sized data); zeroed when the pitch pads the rows
static int ensure_x_buffer(Ctx* c, int64_t n, int64_t d, int64_t n_alloc) {
  const int64_t ldx = round_up(d, 16);
  if (c->X && !(c->ldx == ldx && c->x_cap_rows >= n_alloc && c->x_cap_rows <= n_alloc + n_alloc / 8 + 64)) {
    cudaFree(c->X); c->X = nullptr; c->n = 0; c->x_cap_rows = 0;
  }
  if (!c->X) {
    SKD_CUDA(c, cudaMalloc((void**)&c->X, (size_t)n_alloc * ldx * sizeof(float)));
    c->x_cap_rows = n_alloc;
    c->ldx = ldx;
  }
  if (ldx != d) SKD_CUDA(c, cudaMemsetAsync(c->X, 0, (size_t)c->x_cap_rows * ldx * sizeof(float), c->stream));
  (void)n;
  return 0;
}

// Labels, targets and fold ids describe the rows of one staged X: a matrix with another row count makes them
// stale (a later call must not read n rows out of a vector staged for fewer), so they are dropped with it.
static void drop_stale_row_vectors(Ctx* c, int64_t n_new) {
  if (c->vec_n == n_new) return;
  if (c->ycls) { cudaFree(c->ycls); c->ycls = nullptr; c->ycls_cap = 0; }
  if (c->yreal) { cudaFree(c->yreal); c->yreal = nullptr; c->yreal_cap = 0; }
  if (c->fold_store) { cudaFree(c->fold_store); c->fold_store = nullptr; c->fold_cap = 0; }
  c->fold = nullptr;
  c->n_folds = 0;
  c->fold_count.clear();
  c->h_fold.clear();
  c->h_ycls.clear();
  c->ycls_min = 0; c->ycls_max = -1;
  c->row_bits = {};
  c->tc.meta_valid = false;
  c->vec_n = n_new;
}

static int finite_check_staged(Ctx* c, int64_t n, int64_t ldx) {
  int* dflag;
  Scratch sx(c);
  SKD_CUDA(c, sx.alloc(&dflag, 1));
  SKD_CUDA(c, cudaMemsetAsync(dflag, 0, sizeof(int), c->stream));
  finite_check_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(c->X, n * ldx, dflag);
  c->launches += 1;
  int hflag = 0;
  SKD_CUDA(c, cudaMemcpyAsync(&hflag, dflag, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  if (hflag) {
    cudaFree(c->X); c->X = nullptr; c->n = 0; c->x_cap_rows = 0;
    return fail(c, "Input X contains NaN or infinity.");
  }
  return 0;
}

static int stage_x_common(Ctx* c, const float* src, int64_t n, int64_t d, int64_t ldx_src,
                          cudaMemcpyKind kind) {
  if (!src || n <= 0 || d <= 0 || ldx_src < d) return fail(c, "skd_stage_x: bad arguments");
  SKD_CUDA(c, cudaSetDevice(c->device));
  Trace tr(c, "stage_x");
  int64_t ldx = round_up(d, 16);
  if (ensure_x_buffer(c, n, d, n)) return 1;
  tr.mark("alloc");
  if (kind == cudaMemcpyHostToDevice) {
    if (stage_rows_h2d(c, c->X, ldx, src, n, d, ldx_src)) return 1;
  } else {
    SKD_CUDA(c, cudaMemcpy2DAsync(c->X, ldx * sizeof(float), src, ldx_src * sizeof(float),
                                  d * sizeof(float), n, kind, c->stream));
    SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  }
  tr.mark("copy");
  if (finite_check_staged(c, n, ldx)) return 1;
  tr.mark("check");
  drop_stale_row_vectors(c, n);
  c->n = n; c->d = d; c->ldx = ldx;
  c->tc.x_valid = false;
  c->forest.valid = false;
  if (kind == cudaMemcpyHostToDevice) c->h2d += (int64_t)n * d * sizeof(float);
  return 0;
}

int skd_stage_x(skd_ctx* ctx, const float* X, int64_t n, int64_t d, int64_t ldx) {
  if (!ctx) return fail(nullptr, "skd_stage_x: ctx is NULL");
  return stage_x_common(&ctx->c, X, n, d, ldx, cudaMemcpyHostToDevice);
}

int skd_stage_x_device(skd_ctx* ctx, const float* dX, int64_t n, int64_t d, int64_t ldx) {
  if (!ctx) return fail(nullptr, "skd_stage_x_device: ctx is NULL");
  return stage_x_common(&ctx->c, dX, n, d, ldx, cudaMemcpyDeviceToDevice);
}

// Sliced staging for several ranks that all hold X on the host: every rank copies its own row slice
// (1/N of the matrix through its own PCIe link), the caller all-gathers the slices in place over
// NVLink (the buffer holds n_alloc >= n rows so that the slices can be equal-sized), then commits.
int skd_stage_x_begin(skd_ctx* ctx, int64_t n, int64_t d, int64_t n_alloc, const float** dX, int64_t* ldx_out) {
  if (!ctx) return fail(nullptr, "skd_stage_x_begin: ctx is NULL");
  Ctx* c = &ctx->c;
  if (n <= 0 || d <= 0 || n_alloc < n) return fail(c, "skd_stage_x_begin: bad arguments");
  SKD_CUDA(c, cudaSetDevice(c->device));
  c->n = 0;                              // nothing is staged until the commit
  if (ensure_x_buffer(c, n, d, n_alloc)) return 1;
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  c->pend_n = n; c->pend_d = d;
  if (dX) *dX = c->X;
  if (ldx_out) *ldx_out = c->ldx;
  return 0;
}

int skd_stage_x_rows(skd_ctx* ctx, const float* X_rows, int64_t ld, int64_t row0, int64_t n_rows) {
  if (!ctx) return fail(nullptr, "skd_stage_x_rows: ctx is NULL");
  Ctx* c = &ctx->c;
  if (!c->X || c->pend_n <= 0) return fail(c, "skd_stage_x_rows: call skd_stage_x_begin first");
  if (n_rows == 0) return 0;
  if (!X_rows || row0 < 0 || n_rows < 0 || row0 + n_rows > c->pend_n || ld < c->pend_d)
    return fail(c, "skd_stage_x_rows: bad arguments");
  SKD_CUDA(c, cudaSetDevice(c->device));
  if (stage_rows_h2d(c, c->X + (size_t)row0 * c->ldx, c->ldx, X_rows, n_rows, c->pend_d, ld)) return 1;
  c->h2d += n_rows * c->pend_d * (int64_t)sizeof(float);
  return 0;
}

int skd_stage_x_commit(skd_ctx* ctx) {
  if (!ctx) return fail(nullptr, "skd_stage_x_commit: ctx is NULL");
  Ctx* c = &ctx->c;
  if (!c->X || c->pend_n <= 0) return fail(c, "skd_stage_x_commit: call skd_stage_x_begin first");
  SKD_CUDA(c, cudaSetDevice(c->device));
  const int64_t n = c->pend_n, d = c->pend_d;
  c->pend_n = 0;
  if (finite_check_staged(c, n, c->ldx)) return 1;
  drop_stale_row_vectors(c, n);
  c->n = n; c->d = d;
  c->tc.x_valid = false;
  c->forest.valid = false;
  return 0;
}

int skd_staged_x(skd_ctx* ctx, const float** dX, int64_t* n, int64_t* d, int64_t* ldx) {
  if (!ctx) return fail(nullptr, "skd_staged_x: ctx is NULL");
  Ctx* c = &ctx->c;
  if (!c->X) return fail(c, "skd_staged_x: nothing staged");
  if (dX) *dX = c->X;
  if (n) *n = c->n;
  if (d) *d = c->d;
  if (ldx) *ldx = c->ldx;
  return 0;
}

int skd_stage_labels(skd_ctx* ctx, const int32_t* y, int64_t n) {
  if (!ctx) return fail(nullptr, "skd_stage_labels: ctx is NULL");
  Ctx* c = &ctx->c;
  if (!y || n != c->n) return fail(c, "skd_stage_labels: n does not match the staged X");
  SKD_CUDA(c, cudaSetDevice(c->device));
  if (stage_device_vector(c, c->ycls, c->ycls_cap, y, n)) return 1;
  c->h_ycls.assign(y, y + n);
  const auto mm = std::minmax_element(y, y + n);
  c->ycls_min = *mm.first; c->ycls_max = *mm.second;
  c->tc.meta_valid = false;
  return 0;
}

int skd_stage_targets(skd_ctx* ctx, const float* y, int64_t n) {
  if (!ctx) return fail(nullptr, "skd_stage_targets: ctx is NULL");
  Ctx* c = &ctx->c;
  if (!y || n != c->n) return fail(c, "skd_stage_targets: n does not match the staged X");
  SKD_CUDA(c, cudaSetDevice(c->device));
  if (stage_device_vector(c, c->yreal, c->yreal_cap, y, n)) return 1;
  c->tc.meta_valid = false;
  return 0;
}

int skd_stage_folds(skd_ctx* ctx, const int8_t* fold_id, int64_t n, int32_t n_folds) {
  if (!ctx) return fail(nullptr, "skd_stage_folds: ctx is NULL");
  Ctx* c = &ctx->c;
  SKD_CUDA(c, cudaSetDevice(c->device));
  c->fold = nullptr;
  c->tc.meta_valid = false;
  c->n_folds = 0;
  c->fold_count.clear();
  c->h_fold.clear();
  if (!fold_id) return 0;  // cleared
  if (n != c->n || n_folds <= 0 || n_folds > 127) return fail(c, "skd_stage_folds: bad arguments");
  c->fold_count.assign(n_folds, 0);
  c->h_fold.assign(fold_id, fold_id + n);
  for (int64_t i = 0; i < n; ++i) {
    int f = fold_id[i];
    if (f < 0 || f >= n_folds) return fail(c, "skd_stage_folds: fold id out of range");
    c->fold_count[f] += 1;
  }
  if (stage_device_vector(c, c->fold_store, c->fold_cap, fold_id, n)) return 1;
  c->fold = c->fold_store;
  c->n_folds = n_folds;
  return 0;
}

int skd_stage_column_masks(skd_ctx* ctx, int32_t B, const uint8_t* mask) {
  if (!ctx) return fail(nullptr, "skd_stage_column_masks: ctx is NULL");
  Ctx* c = &ctx->c;
  c->fmask = {};
  if (!mask || B <= 0) return 0;   // cleared
  if (!c->X) return fail(c, "skd_stage_column_masks: stage X first");
  c->fmask.mask.assign(mask, mask + (size_t)B * c->d);
  c->fmask.cols = B;
  return 0;
}

int skd_stage_row_bits(skd_ctx* ctx, int32_t B, const uint8_t* label_bits, const uint8_t* train_bits,
                       int64_t bytes_per_col) {
  if (!ctx) return fail(nullptr, "skd_stage_row_bits: ctx is NULL");
  Ctx* c = &ctx->c;
  c->row_bits = {};
  if (B <= 0 || (!label_bits && !train_bits)) return 0;   // cleared
  if (!c->X) return fail(c, "skd_stage_row_bits: stage X first");
  if (bytes_per_col * 8 < c->n) return fail(c, "skd_stage_row_bits: fewer bits per column than staged rows");
  const int64_t words = tc_padded_rows(c->n) / 32;         // whole tiles of the tensor-core path
  const int64_t use = std::min<int64_t>(bytes_per_col, (c->n + 7) / 8);
  auto pack = [&](const uint8_t* src, std::vector<uint32_t>& dst) {
    dst.assign((size_t)B * words, 0u);
    for (int j = 0; j < B; ++j) {
      memcpy(dst.data() + (size_t)j * words, src + (size_t)j * bytes_per_col, (size_t)use);
      if (c->n & 7) {   // bits beyond the last row must read as 0
        uint8_t* last = reinterpret_cast<uint8_t*>(dst.data() + (size_t)j * words) + (c->n >> 3);
        *last &= (uint8_t)((1u << (c->n & 7)) - 1u);
      }
    }
  };
  if (label_bits) pack(label_bits, c->row_bits.y);
  if (train_bits) pack(train_bits, c->row_bits.m);
  c->row_bits.cols = B;
  c->row_bits.words = words;
  return 0;
}

int skd_stage_class_weights(skd_ctx* ctx, int32_t B, int32_t K, const float* w, const double* sw_sum) {
  if (!ctx) return fail(nullptr, "skd_stage_class_weights: ctx is NULL");
  Ctx* c = &ctx->c;
  c->cw = {};
  if (B <= 0 || !w) return 0;   // cleared
  if (K < 2 || !sw_sum) return fail(c, "skd_stage_class_weights: bad arguments");
  for (int64_t i = 0; i < (int64_t)B * K; ++i)
    if (!(std::isfinite(w[i]) && w[i] >= 0.f)) return fail(c, "skd_stage_class_weights: weights must be finite and >= 0");
  for (int j = 0; j < B; ++j)
    if (!(std::isfinite(sw_sum[j]) && sw_sum[j] > 0.0))
      return fail(c, "skd_stage_class_weights: the sum of a column's weights must be finite and positive");
  c->cw.w.assign(w, w + (size_t)B * K);
  c->cw.sw_sum.assign(sw_sum, sw_sum + B);
  c->cw.cols = B;
  c->cw.k = K;
  return 0;
}

int skd_stage_sample_weights(skd_ctx* ctx, const float* w, int64_t n) {
  if (!ctx) return fail(nullptr, "skd_stage_sample_weights: ctx is NULL");
  Ctx* c = &ctx->c;
  c->sw = {};
  if (!w) return 0;   // cleared
  if (!c->X || n != c->n) return fail(c, "skd_stage_sample_weights: n does not match the staged X");
  for (int64_t i = 0; i < n; ++i)
    if (!(std::isfinite(w[i]) && w[i] >= 0.f)) return fail(c, "skd_stage_sample_weights: weights must be finite and >= 0");
  c->sw.w.assign(w, w + n);
  return 0;
}

int skd_stage_forest_class_weights(skd_ctx* ctx, int32_t n_classes, const double* w, int32_t balanced_subsample,
                                   double min_weight_fraction_leaf) {
  if (!ctx) return fail(nullptr, "skd_stage_forest_class_weights: ctx is NULL");
  Ctx* c = &ctx->c;
  c->forest_cw = {};
  if (n_classes <= 0 || (!w && !balanced_subsample)) return 0;   // cleared
  if (!(std::isfinite(min_weight_fraction_leaf) && min_weight_fraction_leaf >= 0.0 && min_weight_fraction_leaf <= 0.5))
    return fail(c, "skd_stage_forest_class_weights: min_weight_fraction_leaf must be in [0, 0.5]");
  ForestClassWeights cw;
  cw.n_classes = n_classes;
  cw.balanced_subsample = balanced_subsample != 0;
  cw.min_weight_fraction = min_weight_fraction_leaf;
  if (!cw.balanced_subsample) {
    for (int k = 0; k < n_classes; ++k)
      if (!(std::isfinite(w[k]) && w[k] >= 0.0)) return fail(c, "skd_stage_forest_class_weights: weights must be finite and >= 0");
    cw.w.assign(w, w + n_classes);
  }
  c->forest_cw = std::move(cw);
  return 0;
}

int skd_stage_forest_criterion(skd_ctx* ctx, int32_t criterion) {
  if (!ctx) return fail(nullptr, "skd_stage_forest_criterion: ctx is NULL");
  Ctx* c = &ctx->c;
  c->forest_criterion = 0;
  if (criterion != 0 && criterion != 1)
    return fail(c, "skd_stage_forest_criterion: criterion must be 0 (gini / squared error) or 1 (entropy)");
  c->forest_criterion = criterion;
  return 0;
}

// Staged sample weights a call consumes: they need class weights staged for the same call (those carry each
// column's sw_sum) and the staged row count.  They are copied into the context's device buffer, zero padded to
// the whole tiles the tensor-core kernel reads (tc_padded_rows); *droww stays nullptr when none are staged.
static int upload_sample_weights(Ctx* c, const char* who, const StagedSampleWeights& sw, const StagedClassWeights& cw,
                                 const float** droww) {
  *droww = nullptr;
  if (sw.w.empty()) return 0;
  if (cw.cols <= 0)
    return fail(c, std::string(who) + ": sample weights need class weights staged for the same call "
                                      "(all ones without class_weight: they carry each column's sw_sum)");
  if ((int64_t)sw.w.size() != c->n) return fail(c, std::string(who) + ": staged sample weights do not match the staged rows");
  const int64_t npad = tc_padded_rows(c->n);
  std::vector<float> h(sw.w);
  h.resize((size_t)npad, 0.f);
  if (stage_device_vector(c, c->roww, c->roww_cap, h.data(), npad)) return 1;
  *droww = c->roww;
  return 0;
}

// Largest sample weight of the training rows of every binary column, {label 0, label 1}, with the column's rows and
// labels as the kernels form them: rows outside the held-out fold col_fold[j]; label 1 = class col_pos[j]; with
// col_neg (pair columns, col_neg[j] >= 0) only the rows of class col_pos[j] or col_neg[j]; staged row bits
// replace the training rows (bits->m) and the labels (bits->y).
static int column_row_weight_max(Ctx* c, int B, const std::vector<float>& rw, const int32_t* col_fold,
                                 const int32_t* col_pos, const int32_t* col_neg, const StagedRowBits* bits,
                                 std::vector<float2>& mx) {
  const int64_t n = c->n;
  const bool have_bits = bits && bits->cols > 0;
  if ((!have_bits || bits->y.empty()) && (int64_t)c->h_ycls.size() != n)
    return fail(c, "sample weights: labels not staged");
  mx.assign(B, make_float2(0.f, 0.f));
  // largest weight per (fold, class): the folds of a row are 0 without staged folds
  const int nf = c->h_fold.empty() ? 1 : c->n_folds;
  const int lo = c->ycls_min, ncls = std::max(0, c->ycls_max - c->ycls_min + 1);
  std::vector<float> cell;
  if (!have_bits) {
    cell.assign((size_t)nf * ncls, 0.f);
    for (int64_t i = 0; i < n; ++i) {
      const int f = c->h_fold.empty() ? 0 : (int)c->h_fold[i];
      float& m = cell[(size_t)f * ncls + (c->h_ycls[i] - lo)];
      m = std::max(m, rw[i]);
    }
  }
  auto bit = [](const std::vector<uint32_t>& v, int64_t words, int j, int64_t i) {
    return (v[(size_t)j * words + (i >> 5)] >> (i & 31)) & 1u;
  };
  for (int j = 0; j < B; ++j) {
    float m0 = 0.f, m1 = 0.f;
    if (have_bits) {   // row bits: one scan of the rows (the bit matrices exclude folds and pair columns)
      for (int64_t i = 0; i < n; ++i) {
        if (!bits->m.empty() && !bit(bits->m, bits->words, j, i)) continue;
        const bool y1 = bits->y.empty() ? c->h_ycls[i] == col_pos[j] : bit(bits->y, bits->words, j, i) != 0;
        float& m = y1 ? m1 : m0;
        m = std::max(m, rw[i]);
      }
    } else {
      const int neg = col_neg && col_neg[j] >= 0 ? col_neg[j] : INT32_MIN;
      for (int f = 0; f < nf; ++f) {
        if (!c->h_fold.empty() && f == col_fold[j]) continue;
        for (int k = 0; k < ncls; ++k) {
          const int cls = lo + k;
          float& m = cls == col_pos[j] ? m1 : m0;
          if (cls == col_pos[j] || neg == INT32_MIN || cls == neg) m = std::max(m, cell[(size_t)f * ncls + k]);
        }
      }
    }
    mx[j] = make_float2(m0, m1);
  }
  return 0;
}

// Staged class weights of binary columns: weights scaled by the power of two 2^-e that brings the largest row
// factor into (1/2, 1], so that |G| <= 2^14 holds in the fp16 operand of the tensor-core gradient product; 2^e
// goes into inv_n.  Both scalings are exact.  The row factor is the class weight of the row's label, times the
// row's sample weight when those are staged (rw, host copy; the largest product over the column's training rows,
// so that a column whose rows all weigh little does not sink into fp16 subnormals).  l2 = 1 / (C sw_sum),
// inv_n = 2^e / sw_sum (SK/linear_model/_logistic.py:474, 580).
static int binary_class_weights(Ctx* c, const char* who, const StagedClassWeights& cw, int B, const double* C,
                                std::vector<float2>& hcw, std::vector<double>& l2, std::vector<double>& inv_n,
                                const std::vector<float>* rw = nullptr, const int32_t* col_fold = nullptr,
                                const int32_t* col_pos = nullptr, const int32_t* col_neg = nullptr,
                                const StagedRowBits* bits = nullptr) {
  if (cw.cols != B || cw.k != 2) return fail(c, std::string(who) + ": staged class weights do not match this batch (B x 2)");
  std::vector<float2> rmax;
  if (rw && !rw->empty() && column_row_weight_max(c, B, *rw, col_fold, col_pos, col_neg, bits, rmax)) return 1;
  hcw.resize(B);
  for (int j = 0; j < B; ++j) {
    float mx = std::max(cw.w[2 * j], cw.w[2 * j + 1]);
    if (!rmax.empty()) mx = std::max(cw.w[2 * j] * rmax[j].x, cw.w[2 * j + 1] * rmax[j].y);   // float32 products
    if (!(mx > 0.f))
      return fail(c, std::string(who) + (rmax.empty() ? ": every class weight of a column is 0"
                                                       : ": every weight of a column's training rows is 0"));
    int e;
    const float f = frexpf(mx, &e);   // mx = f 2^e, f in [1/2, 1)
    if (f == 0.5f) e -= 1;             // a power of two becomes exactly 1
    hcw[j] = make_float2(ldexpf(cw.w[2 * j], -e), ldexpf(cw.w[2 * j + 1], -e));
    l2[j] = 1.0 / (C[j] * cw.sw_sum[j]);
    inv_n[j] = ldexp(1.0 / cw.sw_sum[j], e);
  }
  return 0;
}

// Training-set size n_train of every logistic column, then l2 = 1 / (C n_train) (SK/linear_model/_logistic.py:580)
// and inv_n = 1 / n_train.  The rows of the column's held-out fold col_fold[j] (< 0: none) do not train;
// with col_neg (pair columns, col_neg[j] >= 0) only the rows of class col_pos[j] or col_neg[j] train; staged
// train bits (bits->m) replace the count.  col_neg and bits may be null.
static int column_train_sizes(Ctx* c, const char* who, int B, const double* C, const int32_t* col_fold,
                              const int32_t* col_pos, const int32_t* col_neg, const StagedRowBits* bits,
                              std::vector<double>& l2, std::vector<double>& inv_n, double* mean_ntrain = nullptr) {
  const int64_t n = c->n;
  l2.resize(B);
  inv_n.resize(B);
  std::vector<int64_t> pair_counts;
  int max_cls = -1;
  double mean = 0.0;
  for (int j = 0; j < B; ++j) {
    int f = col_fold[j];
    int64_t ntrain = n;
    if (f >= 0) {
      if (!c->fold || f >= c->n_folds) return fail(c, std::string(who) + ": col_fold refers to an unstaged fold");
      ntrain = n - c->fold_count[f];
    }
    if (col_neg && col_neg[j] >= 0) {   // pair column: only rows of class col_pos[j] or col_neg[j] train
      if ((int64_t)c->h_ycls.size() != n) return fail(c, std::string(who) + ": labels not staged");
      if (col_neg[j] == col_pos[j]) return fail(c, std::string(who) + ": col_neg equals col_pos");
      if (pair_counts.empty()) {         // rows per (class, fold) once per call
        for (int64_t i = 0; i < n; ++i) if (c->h_ycls[i] > max_cls) max_cls = c->h_ycls[i];
        pair_counts.assign((size_t)(max_cls + 1) * (c->n_folds + 1), 0);
        for (int64_t i = 0; i < n; ++i) {
          const int fi = c->h_fold.empty() ? 0 : (int)c->h_fold[i];
          if (c->h_ycls[i] >= 0) pair_counts[(size_t)c->h_ycls[i] * (c->n_folds + 1) + (c->h_fold.empty() ? 0 : fi)] += 1;
        }
      }
      ntrain = 0;
      for (int cls : {col_pos[j], col_neg[j]}) {
        if (cls < 0 || cls > max_cls) continue;
        for (int ff = 0; ff < (c->h_fold.empty() ? 1 : c->n_folds); ++ff)
          if (ff != f) ntrain += pair_counts[(size_t)cls * (c->n_folds + 1) + ff];
      }
    }
    if (bits && bits->cols > 0 && !bits->m.empty()) {      // training rows of the column = set bits of its mask
      ntrain = 0;
      const uint32_t* mw = bits->m.data() + (size_t)j * bits->words;
      for (int64_t q = 0; q < bits->words; ++q) ntrain += __builtin_popcount(mw[q]);
    }
    if (ntrain <= 0) return fail(c, std::string(who) + ": empty training set");
    if (!(C[j] > 0.0)) return fail(c, std::string(who) + ": C must be positive");
    l2[j] = 1.0 / (C[j] * (double)ntrain);
    inv_n[j] = 1.0 / (double)ntrain;
    mean += (double)ntrain / B;
  }
  if (mean_ntrain) *mean_ntrain = mean;
  return 0;
}

// Device time of a span of one call on the context's stream; the events are freed on every path.
struct DeviceTimer {
  Ctx* c;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  explicit DeviceTimer(Ctx* c_) : c(c_) {}
  ~DeviceTimer() {
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
  }
  int start() {
    SKD_CUDA(c, cudaEventCreate(&e0));
    SKD_CUDA(c, cudaEventCreate(&e1));
    SKD_CUDA(c, cudaEventRecord(e0, c->stream));
    return 0;
  }
  // ends the span, waits for it and writes its length in seconds to *seconds (when not null)
  int stop(double* seconds) {
    SKD_CUDA(c, cudaEventRecord(e1, c->stream));
    SKD_CUDA(c, cudaEventSynchronize(e1));
    float ms = 0.f;
    SKD_CUDA(c, cudaEventElapsedTime(&ms, e0, e1));
    if (seconds) *seconds = ms * 1e-3;
    return 0;
  }
};

int skd_set_kernel(skd_ctx* ctx, int32_t which) {
  if (!ctx) return -1;
  int prev = ctx->c.kernel_choice;
  ctx->c.kernel_choice = which;
  return prev;
}

int skd_profile(skd_ctx* ctx, int32_t enable, double* eval_ms, double* eval_flops,
                int64_t* eval_launches, int64_t* rounds) {
  if (!ctx) return fail(nullptr, "skd_profile: ctx is NULL");
  Ctx* c = &ctx->c;
  if (eval_ms) *eval_ms = c->prof_eval_ms;
  if (eval_flops) *eval_flops = c->prof_eval_flops;
  if (eval_launches) *eval_launches = c->prof_eval_launches;
  if (rounds) *rounds = c->prof_rounds;
  if (enable >= 0) {
    c->prof = enable != 0;
    c->prof_eval_ms = 0.0; c->prof_eval_flops = 0.0; c->prof_eval_launches = 0; c->prof_rounds = 0;
  }
  return 0;
}

int skd_timer_start(skd_ctx* ctx) {
  if (!ctx) return fail(nullptr, "skd_timer_start: ctx is NULL");
  Ctx* c = &ctx->c;
  SKD_CUDA(c, cudaSetDevice(c->device));
  if (!c->timer[0]) {
    SKD_CUDA(c, cudaEventCreate(&c->timer[0]));
    SKD_CUDA(c, cudaEventCreate(&c->timer[1]));
  }
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  SKD_CUDA(c, cudaEventRecord(c->timer[0], c->stream));
  return 0;
}

int skd_timer_stop(skd_ctx* ctx, double* ms_out) {
  if (!ctx) return fail(nullptr, "skd_timer_stop: ctx is NULL");
  Ctx* c = &ctx->c;
  if (!c->timer[0] || !ms_out) return fail(c, "skd_timer_stop: timer not started");
  SKD_CUDA(c, cudaEventRecord(c->timer[1], c->stream));
  SKD_CUDA(c, cudaEventSynchronize(c->timer[1]));
  float ms = 0.f;
  SKD_CUDA(c, cudaEventElapsedTime(&ms, c->timer[0], c->timer[1]));
  *ms_out = ms;
  return 0;
}

int skd_get_counters(skd_ctx* ctx, int64_t* launches, int64_t* h2d, int64_t* d2h) {
  if (!ctx) return fail(nullptr, "skd_get_counters: ctx is NULL");
  if (launches) *launches = ctx->c.launches;
  if (h2d) *h2d = ctx->c.h2d;
  if (d2h) *d2h = ctx->c.d2h;
  return 0;
}

int skd_logreg_fit_batch(skd_ctx* ctx, int32_t B, const double* C, const int32_t* col_fold,
                         const int32_t* col_pos, const int32_t* col_neg, int32_t fit_intercept, double tol,
                         int32_t max_iter, float* coef_out, int32_t* n_iter_out,
                         int32_t* status_out, double* loss_out, int32_t* n_evals_out,
                         double* gpu_seconds_out) {
  if (!ctx) return fail(nullptr, "skd_logreg_fit_batch: ctx is NULL");
  Ctx* c = &ctx->c;
  const StagedClassWeights staged_cw = std::exchange(c->cw, {});
  const StagedSampleWeights staged_sw = std::exchange(c->sw, {});
  const StagedMasks staged_masks = std::exchange(c->fmask, {});
  const StagedRowBits staged_bits = std::exchange(c->row_bits, {});
  if (!c->X || !c->ycls) return fail(c, "skd_logreg_fit_batch: stage X and labels first");
  if (B <= 0 || !C || !col_fold || !col_pos || !coef_out || !n_iter_out || !status_out)
    return fail(c, "skd_logreg_fit_batch: bad arguments");
  if (staged_bits.cols > 0) {
    if (staged_bits.cols != B) return fail(c, "skd_logreg_fit_batch: staged row bit matrices do not match this batch");
    for (int j = 0; j < B; ++j)
      if (col_fold[j] >= 0 || (col_neg && col_neg[j] >= 0))
        return fail(c, "skd_logreg_fit_batch: row bit matrices cannot be combined with folds or pair columns");
  }
  if (max_iter < 1) return fail(c, "skd_logreg_fit_batch: max_iter must be >= 1");
  SKD_CUDA(c, cudaSetDevice(c->device));
  const int64_t d = c->d;
  const int dp = (int)d + 1;

  std::vector<double> l2, inv_n;
  double mean_ntrain = 0.0;
  if (column_train_sizes(c, "skd_logreg_fit_batch", B, C, col_fold, col_pos, col_neg, &staged_bits, l2, inv_n,
                         &mean_ntrain))
    return 1;
  std::vector<float2> hcw;
  const float* droww = nullptr;
  if (upload_sample_weights(c, "skd_logreg_fit_batch", staged_sw, staged_cw, &droww)) return 1;
  if (staged_cw.cols > 0 && binary_class_weights(c, "skd_logreg_fit_batch", staged_cw, B, C, hcw, l2, inv_n, &staged_sw.w,
                                                 col_fold, col_pos, col_neg, &staged_bits))
    return 1;

  Trace tr(c, "logreg_fit");
  Scratch sx(c);
  LogregWork w;
  LbfgsBatch& b = w.lb;
  b.B = B; b.n = dp;
  std::vector<SlotMeta> hslots;
  if (alloc_logreg_slots(c, sx, w, B, col_fold, col_pos, col_neg, hslots)) return 1;
  if (lbfgs_alloc(c, sx, b, w.slot_cap, true)) return 1;
  SKD_CUDA(c, sx.alloc(&w.col_fold, (size_t)B));
  SKD_CUDA(c, sx.alloc(&w.col_pos, (size_t)B));
  std::vector<int32_t> hneg1;
  if (col_neg) {
    hneg1.resize(B);
    for (int j = 0; j < B; ++j) hneg1[j] = col_neg[j] >= 0 ? col_neg[j] + 1 : 0;
    SKD_CUDA(c, sx.alloc(&w.col_neg1, (size_t)B));
  }
  if (!hcw.empty()) {
    float2* dcw;
    SKD_CUDA(c, sx.alloc(&dcw, (size_t)B));
    SKD_CUDA(c, cudaMemcpyAsync(dcw, hcw.data(), B * sizeof(float2), cudaMemcpyHostToDevice, c->stream));
    c->h2d += (int64_t)B * 8;
    w.cw = dcw;
    w.roww = droww;
  }
  const bool use_fmask = staged_masks.cols > 0;
  if (use_fmask) {
    if (staged_masks.cols != B || (int64_t)staged_masks.mask.size() != (int64_t)B * d)
      return fail(c, "skd_logreg_fit_batch: staged column masks do not match this batch (B x d)");
    SKD_CUDA(c, sx.alloc(&b.fmask, (size_t)B * d));
  }
  if (staged_bits.cols > 0) {
    w.rb_words = staged_bits.words;
    if (!staged_bits.y.empty()) {
      uint32_t* dy;
      SKD_CUDA(c, sx.alloc(&dy, staged_bits.y.size()));
      SKD_CUDA(c, cudaMemcpyAsync(dy, staged_bits.y.data(), staged_bits.y.size() * 4, cudaMemcpyHostToDevice, c->stream));
      w.ybits = dy;
      c->h2d += (int64_t)staged_bits.y.size() * 4;
    }
    if (!staged_bits.m.empty()) {
      uint32_t* dm;
      SKD_CUDA(c, sx.alloc(&dm, staged_bits.m.size()));
      SKD_CUDA(c, cudaMemcpyAsync(dm, staged_bits.m.data(), staged_bits.m.size() * 4, cudaMemcpyHostToDevice, c->stream));
      w.mbits = dm;
      c->h2d += (int64_t)staged_bits.m.size() * 4;
    }
    SKD_CUDA(c, cudaStreamSynchronize(c->stream));
    w.uni_pos = -1;
  }

  tr.mark("alloc");
  DeviceTimer timer(c);
  if (timer.start()) return 1;
  SKD_CUDA(c, cudaMemcpyAsync(b.l2, l2.data(), B * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(b.inv_n, inv_n.data(), B * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(w.col_fold, col_fold, B * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(w.col_pos, col_pos, B * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
  if (col_neg) SKD_CUDA(c, cudaMemcpyAsync(w.col_neg1, hneg1.data(), B * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
  if (use_fmask) {
    SKD_CUDA(c, cudaMemcpyAsync(b.fmask, staged_masks.mask.data(), (size_t)B * d, cudaMemcpyHostToDevice, c->stream));
    SKD_CUDA(c, cudaStreamSynchronize(c->stream));
    c->h2d += (int64_t)B * d;
  }
  c->h2d += (int64_t)B * 24;

  if (b.grouped) {
    int32_t ns = (int32_t)hslots.size();
    SKD_CUDA(c, cudaMemcpyAsync(b.slot, hslots.data(), hslots.size() * sizeof(SlotMeta), cudaMemcpyHostToDevice, c->stream));
    SKD_CUDA(c, cudaMemcpyAsync(b.n_act, &ns, sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
  }
  if (lbfgs_init(c, b, b.grouped ? nullptr : w.col_fold, w.col_pos, w.col_neg1, tol, max_iter)) return 1;
  if (w.use_tc && tc_export(c, w, b.grouped ? w.slot_cap : B, nullptr, fit_intercept)) return 1;
  tr.mark("init");
  // Every round records {slots, running} in `hist` so the profile below uses the true counts.
  const long hist_cap = lbfgs_max_rounds(max_iter) + 1;
  int32_t* hist = nullptr;
  SKD_CUDA(c, sx.alloc(&hist, (size_t)2 * hist_cap));
  // SKDIST_B200_TRACE=2 on the tensor-core path: every evaluation also records its work deal
  const bool trace_rounds = tr.on && c->prof && getenv("SKDIST_B200_TRACE")[0] == '2';
  int32_t* deal_hist = nullptr;
  if (trace_rounds && w.use_tc) {
    SKD_CUDA(c, sx.alloc(&deal_hist, (size_t)4 * hist_cap));
    SKD_CUDA(c, cudaMemsetAsync(deal_hist, 0, (size_t)4 * hist_cap * sizeof(int32_t), c->stream));
  }
  size_t ev_used = 0;
  std::vector<int> ev_round;              // round index of every profiled evaluation
  auto eval = [&](int n_act, long round, int* nz_used) -> int {
    if (deal_hist) w.deal_log = round < hist_cap ? deal_hist + 4 * round : nullptr;
    if (c->prof) {
      if (c->prof_events.size() < ev_used + 2) {
        cudaEvent_t e0, e1;
        SKD_CUDA(c, cudaEventCreate(&e0));
        SKD_CUDA(c, cudaEventCreate(&e1));
        c->prof_events.push_back(e0);
        c->prof_events.push_back(e1);
      }
      SKD_CUDA(c, cudaEventRecord(c->prof_events[ev_used], c->stream));
    }
    if (eval_dispatch(c, w, n_act, nz_used)) return 1;
    if (c->prof) {
      SKD_CUDA(c, cudaEventRecord(c->prof_events[ev_used + 1], c->stream));
      ev_used += 2;
      ev_round.push_back((int)round);
    }
    return 0;
  };
  long rounds = 0;
  if (lbfgs_run(c, b, b.grouped ? (int)hslots.size() : B, fit_intercept, max_iter, hist, w.use_tc ? &w : nullptr,
                eval, &rounds))
    return 1;
  // true per-round counts (columns evaluated in round r = running after round r - 1)
  std::vector<double> round_flops;
  std::vector<int> round_act, round_run;
  std::vector<int32_t> hhist((size_t)2 * std::max<long>(rounds, 1), 0);
  if (rounds > 0)
    SKD_CUDA(c, cudaMemcpyAsync(hhist.data(), hist, (size_t)2 * rounds * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
  std::vector<int32_t> hdeal;
  if (deal_hist) {
    hdeal.resize((size_t)4 * std::min<long>(std::max<long>(rounds, 1), hist_cap));
    SKD_CUDA(c, cudaMemcpyAsync(hdeal.data(), deal_hist, hdeal.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
    w.deal_log = nullptr;
  }
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  long live_rounds = 0;
  for (size_t e = 0; e < ev_round.size(); ++e) {
    const int r = ev_round[e];
    const int running = r == 0 ? B : hhist[2 * (r - 1) + 1];
    const int slots = r == 0 ? (b.grouped ? (int)hslots.size() : B) : hhist[2 * (r - 1)];
    round_flops.push_back(4.0 * (double)d * (double)running * mean_ntrain);
    round_act.push_back(slots);
    round_run.push_back(running);
  }
  for (long r = 0; r < rounds; ++r)
    if (r == 0 || hhist[2 * (r - 1) + 1] > 0) ++live_rounds;
  tr.mark("rounds");
  if (c->prof) {
    SKD_CUDA(c, cudaStreamSynchronize(c->stream));
    for (size_t i = 0; i + 1 < ev_used; i += 2) {
      float ms = 0.f;
      SKD_CUDA(c, cudaEventElapsedTime(&ms, c->prof_events[i], c->prof_events[i + 1]));
      const size_t r = i / 2;
      if (trace_rounds && 4 * r + 3 < hdeal.size())   // tensor-core deal: live groups, half-padding groups, CTAs, CTAs over >1 group
        fprintf(stderr, "[skd trace] round %3d slots %5d running %5d groups %4d half %3d ctas %3d cross %3d eval %7.3f ms\n",
                (int)r, round_act[r], round_run[r], hdeal[4 * r], hdeal[4 * r + 1], hdeal[4 * r + 2], hdeal[4 * r + 3], ms);
      else if (trace_rounds)
        fprintf(stderr, "[skd trace] round %3d slots %5d running %5d eval %7.3f ms\n", (int)r, round_act[r],
                round_run[r], ms);
      if (round_run[i / 2] <= 0) continue;      // enqueued past convergence: the kernels returned at once
      c->prof_eval_ms += ms;
      c->prof_eval_flops += round_flops[i / 2];
      c->prof_eval_launches += 1;
    }
    c->prof_rounds += live_rounds;
  }
  if (lbfgs_result(c, sx, b, 0, coef_out, n_iter_out, status_out, loss_out, n_evals_out)) return 1;
  if (timer.stop(gpu_seconds_out)) return 1;
  tr.mark("finish");
  return 0;
}

int skd_logreg_loss_grad(skd_ctx* ctx, int32_t B, const double* w_in, const double* C,
                         const int32_t* col_fold, const int32_t* col_pos, int32_t fit_intercept,
                         double* loss_out, double* grad_out) {
  if (!ctx) return fail(nullptr, "skd_logreg_loss_grad: ctx is NULL");
  Ctx* c = &ctx->c;
  const StagedClassWeights staged_cw = std::exchange(c->cw, {});
  const StagedSampleWeights staged_sw = std::exchange(c->sw, {});
  if (!c->X || !c->ycls) return fail(c, "skd_logreg_loss_grad: stage X and labels first");
  if (B <= 0 || !w_in || !C || !col_fold || !col_pos || !loss_out || !grad_out)
    return fail(c, "skd_logreg_loss_grad: bad arguments");
  SKD_CUDA(c, cudaSetDevice(c->device));
  const int64_t d = c->d, ldx = c->ldx;
  const int dp = (int)d + 1;
  std::vector<double> l2, inv_n;
  if (column_train_sizes(c, "skd_logreg_loss_grad", B, C, col_fold, col_pos, nullptr, nullptr, l2, inv_n)) return 1;
  std::vector<float> hw((size_t)B * ldx + B, 0.f);
  for (int j = 0; j < B; ++j) {
    for (int k = 0; k < d; ++k) hw[(size_t)j * ldx + k] = (float)w_in[(size_t)j * dp + k];
    hw[(size_t)B * ldx + j] = fit_intercept ? (float)w_in[(size_t)j * dp + d] : 0.f;
  }
  std::vector<float2> hcw;
  const float* droww = nullptr;
  if (upload_sample_weights(c, "skd_logreg_loss_grad", staged_sw, staged_cw, &droww)) return 1;
  if (staged_cw.cols > 0 && binary_class_weights(c, "skd_logreg_loss_grad", staged_cw, B, C, hcw, l2, inv_n, &staged_sw.w,
                                                 col_fold, col_pos))
    return 1;
  Scratch sx(c);
  LogregWork w;
  LbfgsBatch& b = w.lb;
  b.B = B; b.n = dp;
  if (!hcw.empty()) {
    float2* dcw;
    SKD_CUDA(c, sx.alloc(&dcw, (size_t)B));
    SKD_CUDA(c, cudaMemcpyAsync(dcw, hcw.data(), B * sizeof(float2), cudaMemcpyHostToDevice, c->stream));
    w.cw = dcw;
    w.roww = droww;
  }
  // the slot layout of skd_logreg_fit_batch: fold-grouped on the tensor cores, slot s = column s on SIMT
  std::vector<SlotMeta> hs;
  if (alloc_logreg_slots(c, sx, w, B, col_fold, col_pos, nullptr, hs)) return 1;
  if (!b.grouped) {
    hs.resize(B);
    for (int j = 0; j < B; ++j) { hs[j].col = j; hs[j].fold = col_fold[j] < 0 ? -1 : col_fold[j]; hs[j].pos = col_pos[j]; hs[j].pad = 0; }
  }
  const int n_slots = (int)hs.size();
  SKD_CUDA(c, sx.alloc(&b.l2, (size_t)B));
  SKD_CUDA(c, sx.alloc(&b.inv_n, (size_t)B));
  SKD_CUDA(c, sx.alloc(&b.slot, (size_t)n_slots));
  SKD_CUDA(c, sx.alloc(&b.n_act, 1));
  double *dx, *df, *dg;
  SKD_CUDA(c, sx.alloc(&dx, (size_t)B * dp));
  SKD_CUDA(c, sx.alloc(&df, (size_t)B));
  SKD_CUDA(c, sx.alloc(&dg, (size_t)B * dp));
  SKD_CUDA(c, cudaMemcpyAsync(b.l2, l2.data(), B * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(b.inv_n, inv_n.data(), B * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(b.slot, hs.data(), n_slots * sizeof(SlotMeta), cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(dx, w_in, (size_t)B * dp * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  if (w.use_tc) {
    SKD_CUDA(c, cudaMemcpyAsync(b.n_act, &n_slots, sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    if (tc_export(c, w, n_slots, dx, fit_intercept)) return 1;
  } else {
    SKD_CUDA(c, cudaMemcpyAsync(b.W, hw.data(), hw.size() * sizeof(float), cudaMemcpyHostToDevice, c->stream));
  }
  int nz_used = 0;
  if (eval_dispatch(c, w, n_slots, &nz_used)) return 1;
  if (lbfgs_gather(c, b, n_slots, nz_used, fit_intercept, dx, df, dg)) return 1;
  SKD_CUDA(c, cudaMemcpyAsync(loss_out, df, B * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(grad_out, dg, (size_t)B * dp * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  return 0;
}

// Scoring codes (score_code_selects) of a scoring entry: -1 is not a code, and a code names a staged fold.
static int check_score_codes(Ctx* c, const char* who, int B, const int32_t* col_fold) {
  for (int j = 0; j < B; ++j) {
    if (col_fold[j] == -1) return fail(c, std::string(who) + ": col_fold -1 is not a scoring code");
    const int f = score_code_fold(col_fold[j]);
    if (f >= 0 && (!c->fold || f >= c->n_folds))
      return fail(c, std::string(who) + ": col_fold refers to an unstaged fold");
  }
  return 0;
}

int skd_linear_score_batch(skd_ctx* ctx, int32_t B, const float* coef, const int32_t* col_fold,
                           const int32_t* col_pos, int64_t* correct_out, int64_t* count_out) {
  if (!ctx) return fail(nullptr, "skd_linear_score_batch: ctx is NULL");
  Ctx* c = &ctx->c;
  if (!c->X || !c->ycls) return fail(c, "skd_linear_score_batch: stage X and labels first");
  if (B <= 0 || !coef || !col_fold || !col_pos || !correct_out || !count_out)
    return fail(c, "skd_linear_score_batch: bad arguments");
  if (check_score_codes(c, "skd_linear_score_batch", B, col_fold)) return 1;
  SKD_CUDA(c, cudaSetDevice(c->device));
  Trace tr(c, "score");
  Scratch sx(c);
  std::vector<SlotMeta> hs(B);
  for (int j = 0; j < B; ++j) { hs[j].col = j; hs[j].fold = col_fold[j]; hs[j].pos = col_pos[j]; hs[j].pad = 0; }
  SlotMeta* dslot; int64_t *dcorrect, *dcount;
  SKD_CUDA(c, sx.alloc(&dslot, (size_t)B));
  SKD_CUDA(c, sx.alloc(&dcorrect, (size_t)B));
  SKD_CUDA(c, sx.alloc(&dcount, (size_t)B));
  SKD_CUDA(c, cudaMemcpyAsync(dslot, hs.data(), B * sizeof(SlotMeta), cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemsetAsync(dcorrect, 0, B * sizeof(int64_t), c->stream));
  SKD_CUDA(c, cudaMemsetAsync(dcount, 0, B * sizeof(int64_t), c->stream));
  bool use_tc;
  if (use_tensor_cores(c, &use_tc)) return 1;
  if (use_tc) {
    // tensor-core GEMM1-only pass with a counting epilogue (logreg_tc.cu, TC_SCORE)
    LogregWork w;
    if (tc_scoring_setup(c, sx, w, B, coef, dslot)) return 1;
    tr.mark("setup");
    if (tc_score(c, w, B, dcorrect, dcount)) return 1;
    tr.mark("kernel");
  } else {
    float* dW;
    if (pack_coef(c, sx, B, coef, c->d, c->ldx, &dW)) return 1;
    if (simt_score(c, B, dW, dslot, dcorrect, dcount)) return 1;
  }
  SKD_CUDA(c, cudaMemcpyAsync(correct_out, dcorrect, B * sizeof(int64_t), cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(count_out, dcount, B * sizeof(int64_t), cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  c->d2h += (int64_t)B * 16;
  return 0;
}

// The entries that take n_classes read class ids 0..n_classes-1.  A row with any other id would still count in
// n_train (so in 1/n_train and l2) while the kernels leave it out of the loss, the gradient and the scores.
static int check_class_ids(Ctx* c, const char* who, int n_classes) {
  if (c->ycls_min < 0 || c->ycls_max >= n_classes)
    return fail(c, std::string(who) + ": staged class ids span " + std::to_string(c->ycls_min) + ".." +
                       std::to_string(c->ycls_max) + ", outside 0..n_classes-1 = 0.." + std::to_string(n_classes - 1));
  return 0;
}

// l2 and inv_n of every multinomial candidate, with the staged masks and class weights checked against the batch:
// the sum of a candidate's per-row weights takes the place of n_train (SK/linear_model/_logistic.py:474).
static int multinomial_constants(Ctx* c, const char* who, int B, int n_classes, const double* C, const int32_t* col_fold,
                                 const StagedMasks& masks, const StagedClassWeights& cw, std::vector<double>& l2,
                                 std::vector<double>& inv_n) {
  if (check_class_ids(c, who, n_classes)) return 1;
  if (column_train_sizes(c, who, B, C, col_fold, nullptr, nullptr, nullptr, l2, inv_n)) return 1;
  if (masks.cols > 0 && (masks.cols != B || (int64_t)masks.mask.size() != (int64_t)B * c->d))
    return fail(c, std::string(who) + ": staged column masks do not match the batch");
  if (cw.cols > 0) {
    if (cw.cols != B || cw.k != n_classes)
      return fail(c, std::string(who) + ": staged class weights do not match this batch (B x n_classes)");
    for (int j = 0; j < B; ++j) {
      l2[j] = 1.0 / (C[j] * cw.sw_sum[j]);
      inv_n[j] = 1.0 / cw.sw_sum[j];
    }
  }
  return 0;
}

int skd_logreg_multinomial_fit_batch(skd_ctx* ctx, int32_t B, int32_t n_classes, const double* C,
                                     const int32_t* col_fold, int32_t fit_intercept, double tol, int32_t max_iter,
                                     float* coef_out, int32_t* n_iter_out, int32_t* status_out, double* loss_out,
                                     int32_t* n_evals_out, double* gpu_seconds_out) {
  if (!ctx) return fail(nullptr, "skd_logreg_multinomial_fit_batch: ctx is NULL");
  Ctx* c = &ctx->c;
  const StagedClassWeights staged_cw = std::exchange(c->cw, {});
  const StagedSampleWeights staged_sw = std::exchange(c->sw, {});
  const StagedMasks staged_masks = std::exchange(c->fmask, {});
  if (!c->X || !c->ycls) return fail(c, "skd_logreg_multinomial_fit_batch: stage X and labels first");
  if (B <= 0 || n_classes < 2 || !C || !col_fold || !coef_out || !n_iter_out || !status_out)
    return fail(c, "skd_logreg_multinomial_fit_batch: bad arguments");
  if (max_iter < 1) return fail(c, "skd_logreg_multinomial_fit_batch: max_iter must be >= 1");
  std::vector<double> l2, inv_n;
  if (multinomial_constants(c, "skd_logreg_multinomial_fit_batch", B, n_classes, C, col_fold, staged_masks, staged_cw,
                            l2, inv_n))
    return 1;
  SKD_CUDA(c, cudaSetDevice(c->device));
  const float* droww = nullptr;
  if (upload_sample_weights(c, "skd_logreg_multinomial_fit_batch", staged_sw, staged_cw, &droww)) return 1;
  Trace tr(c, "multinomial_fit");
  DeviceTimer timer(c);
  if (timer.start()) return 1;
  if (multi_fit(c, B, n_classes, l2.data(), inv_n.data(), col_fold, fit_intercept, tol, max_iter,
                staged_masks.cols > 0 ? staged_masks.mask.data() : nullptr,
                staged_cw.cols > 0 ? staged_cw.w.data() : nullptr, droww, coef_out, n_iter_out, status_out, loss_out,
                n_evals_out))
    return 1;
  return timer.stop(gpu_seconds_out);
}

int skd_logreg_multinomial_loss_grad(skd_ctx* ctx, int32_t B, int32_t n_classes, const double* w_in, const double* C,
                                     const int32_t* col_fold, int32_t fit_intercept, double* loss_out,
                                     double* grad_out) {
  if (!ctx) return fail(nullptr, "skd_logreg_multinomial_loss_grad: ctx is NULL");
  Ctx* c = &ctx->c;
  const StagedClassWeights staged_cw = std::exchange(c->cw, {});
  const StagedSampleWeights staged_sw = std::exchange(c->sw, {});
  const StagedMasks staged_masks = std::exchange(c->fmask, {});
  if (!c->X || !c->ycls) return fail(c, "skd_logreg_multinomial_loss_grad: stage X and labels first");
  if (B <= 0 || n_classes < 2 || !w_in || !C || !col_fold || !loss_out || !grad_out)
    return fail(c, "skd_logreg_multinomial_loss_grad: bad arguments");
  std::vector<double> l2, inv_n;
  if (multinomial_constants(c, "skd_logreg_multinomial_loss_grad", B, n_classes, C, col_fold, staged_masks, staged_cw,
                            l2, inv_n))
    return 1;
  SKD_CUDA(c, cudaSetDevice(c->device));
  const float* droww = nullptr;
  if (upload_sample_weights(c, "skd_logreg_multinomial_loss_grad", staged_sw, staged_cw, &droww)) return 1;
  const int dp = (int)c->d + 1;
  std::vector<double> x(w_in, w_in + (size_t)B * n_classes * dp);
  if (!fit_intercept)   // the fit's intercepts stay at 0 without one
    for (size_t r = 0; r < (size_t)B * n_classes; ++r) x[r * dp + dp - 1] = 0.0;
  Trace tr(c, "multinomial_loss_grad");
  return multi_loss_grad(c, B, n_classes, l2.data(), inv_n.data(), col_fold, fit_intercept,
                         staged_masks.cols > 0 ? staged_masks.mask.data() : nullptr,
                         staged_cw.cols > 0 ? staged_cw.w.data() : nullptr, droww, x.data(), loss_out, grad_out);
}

static int multinomial_check(Ctx* c, const char* who, int32_t B, int32_t n_classes, const float* coef,
                             const int32_t* col_fold) {
  if (!c->X || !c->ycls) return fail(c, std::string(who) + ": stage X and labels first");
  if (B <= 0 || n_classes < 2 || !coef || !col_fold) return fail(c, std::string(who) + ": bad arguments");
  return check_score_codes(c, who, B, col_fold);
}

int skd_multinomial_confusion_batch(skd_ctx* ctx, int32_t B, int32_t n_classes, const float* coef,
                                    const int32_t* col_fold, int64_t* confusion_out) {
  if (!ctx) return fail(nullptr, "skd_multinomial_confusion_batch: ctx is NULL");
  Ctx* c = &ctx->c;
  if (multinomial_check(c, "skd_multinomial_confusion_batch", B, n_classes, coef, col_fold)) return 1;
  if (!confusion_out) return fail(c, "skd_multinomial_confusion_batch: bad arguments");
  if (check_class_ids(c, "skd_multinomial_confusion_batch", n_classes)) return 1;
  SKD_CUDA(c, cudaSetDevice(c->device));
  Trace tr(c, "multinomial_confusion");
  return multi_score(c, B, n_classes, coef, col_fold, confusion_out);
}

int skd_multinomial_score_batch(skd_ctx* ctx, int32_t B, int32_t n_classes, const float* coef,
                                const int32_t* col_fold, int64_t* correct_out, int64_t* count_out) {
  if (!ctx) return fail(nullptr, "skd_multinomial_score_batch: ctx is NULL");
  Ctx* c = &ctx->c;
  if (multinomial_check(c, "skd_multinomial_score_batch", B, n_classes, coef, col_fold)) return 1;
  if (!correct_out || !count_out) return fail(c, "skd_multinomial_score_batch: bad arguments");
  if (check_class_ids(c, "skd_multinomial_score_batch", n_classes)) return 1;
  SKD_CUDA(c, cudaSetDevice(c->device));
  Trace tr(c, "multinomial_score");
  const size_t KK = (size_t)n_classes * n_classes;
  std::vector<int64_t> conf((size_t)B * KK);
  if (multi_score(c, B, n_classes, coef, col_fold, conf.data())) return 1;
  for (int j = 0; j < B; ++j) {
    int64_t tot = 0, diag = 0;
    for (int a = 0; a < n_classes; ++a)
      for (int b = 0; b < n_classes; ++b) {
        const int64_t v = conf[(size_t)j * KK + (size_t)a * n_classes + b];
        tot += v;
        if (a == b) diag += v;
      }
    correct_out[j] = diag;
    count_out[j] = tot;
  }
  return 0;
}

int skd_linear_auc_batch(skd_ctx* ctx, int32_t B, const float* coef, const int32_t* col_fold,
                         const int32_t* col_pos, int64_t* u2_out, int64_t* n_pos_out, int64_t* n_neg_out) {
  if (!ctx) return fail(nullptr, "skd_linear_auc_batch: ctx is NULL");
  Ctx* c = &ctx->c;
  if (!c->X || !c->ycls) return fail(c, "skd_linear_auc_batch: stage X and labels first");
  if (B <= 0 || !coef || !col_fold || !col_pos || !u2_out || !n_pos_out || !n_neg_out)
    return fail(c, "skd_linear_auc_batch: bad arguments");
  if (check_score_codes(c, "skd_linear_auc_batch", B, col_fold)) return 1;
  SKD_CUDA(c, cudaSetDevice(c->device));
  Trace tr(c, "auc");
  return auc_batch(c, B, coef, col_fold, col_pos, u2_out, n_pos_out, n_neg_out);
}

int skd_linear_rank_batch(skd_ctx* ctx, int32_t B, int32_t n_classes, const float* coef, const int32_t* col_fold,
                          const int32_t* col_pos, int32_t score_kind, int32_t pairs, int64_t* u2_out,
                          int64_t* n_pos_out, int64_t* n_neg_out, double* ap_out) {
  if (!ctx) return fail(nullptr, "skd_linear_rank_batch: ctx is NULL");
  Ctx* c = &ctx->c;
  if (n_classes == 2 || n_classes < 1)
    return fail(c, "skd_linear_rank_batch: n_classes is 1 (binary columns) or > 2");
  if (multinomial_check(c, "skd_linear_rank_batch", B, n_classes == 1 ? 2 : n_classes, coef, col_fold)) return 1;
  if (!u2_out || !n_pos_out || !n_neg_out || !ap_out || (n_classes == 1 && !col_pos))
    return fail(c, "skd_linear_rank_batch: bad arguments");
  if (score_kind != RANK_DECISION && score_kind != RANK_NEG_DECISION && score_kind != RANK_PROBA)
    return fail(c, "skd_linear_rank_batch: score_kind is 0 (decision), 1 (negated decision) or 2 (probability)");
  if (pairs != 0 && (pairs != 1 || n_classes == 1))
    return fail(c, "skd_linear_rank_batch: pairs is 0, or 1 with n_classes > 2");
  if (score_kind == RANK_PROBA && n_classes > 128)
    return fail(c, "skd_linear_rank_batch: probabilities of more than 128 classes have no device path");
  if (n_classes > 2 && check_class_ids(c, "skd_linear_rank_batch", n_classes)) return 1;
  if ((int64_t)rank_segments(n_classes, pairs) > 65536)
    return fail(c, "skd_linear_rank_batch: more than 65536 segments per fit");
  SKD_CUDA(c, cudaSetDevice(c->device));
  Trace tr(c, "rank");
  return rank_batch(c, B, n_classes, coef, col_fold, col_pos, score_kind, pairs, u2_out, n_pos_out, n_neg_out, ap_out);
}

int skd_linear_logloss_batch(skd_ctx* ctx, int32_t B, int32_t n_classes, const float* coef, const int32_t* col_fold,
                             const int32_t* col_pos, double* loss_sum_out, int64_t* count_out) {
  if (!ctx) return fail(nullptr, "skd_linear_logloss_batch: ctx is NULL");
  Ctx* c = &ctx->c;
  if (n_classes == 2) return fail(c, "skd_linear_logloss_batch: n_classes is 1 (binary columns) or > 2");
  if (multinomial_check(c, "skd_linear_logloss_batch", B, n_classes == 1 ? 2 : n_classes, coef, col_fold)) return 1;
  if (!loss_sum_out || !count_out || (n_classes == 1 && !col_pos))
    return fail(c, "skd_linear_logloss_batch: bad arguments");
  if (n_classes > 2 && check_class_ids(c, "skd_linear_logloss_batch", n_classes)) return 1;
  SKD_CUDA(c, cudaSetDevice(c->device));
  Trace tr(c, "logloss");
  return logloss_batch(c, B, n_classes, coef, col_fold, col_pos, loss_sum_out, count_out);
}

int skd_ridge_fit_batch(skd_ctx* ctx, int32_t B, const double* alpha, const int32_t* col_fold,
                        int32_t fit_intercept, float* coef_out, int32_t* status_out,
                        double* gpu_seconds_out) {
  if (!ctx) return fail(nullptr, "skd_ridge_fit_batch: ctx is NULL");
  Ctx* c = &ctx->c;
  if (!c->X || !c->yreal) return fail(c, "skd_ridge_fit_batch: stage X and targets first");
  if (B <= 0 || !alpha || !col_fold || !coef_out || !status_out) return fail(c, "skd_ridge_fit_batch: bad arguments");
  SKD_CUDA(c, cudaSetDevice(c->device));
  const int n_folds = c->fold ? c->n_folds : 1;
  std::vector<int32_t> hold(B);
  for (int j = 0; j < B; ++j) {
    if (!(alpha[j] >= 0.0)) return fail(c, "skd_ridge_fit_batch: alpha must be non-negative");
    if (col_fold[j] >= 0) {
      if (!c->fold || col_fold[j] >= c->n_folds) return fail(c, "skd_ridge_fit_batch: col_fold refers to an unstaged fold");
      hold[j] = col_fold[j];
    } else {
      hold[j] = n_folds;   // hold out nothing
    }
  }
  DeviceTimer timer(c);
  if (timer.start()) return 1;
  if (ridge_fit_batch(c, B, alpha, hold.data(), fit_intercept, coef_out, status_out)) return 1;
  return timer.stop(gpu_seconds_out);
}

int skd_linear_r2_batch(skd_ctx* ctx, int32_t B, const float* coef, const int32_t* col_fold,
                        double* sse_out, int64_t* count_out) {
  if (!ctx) return fail(nullptr, "skd_linear_r2_batch: ctx is NULL");
  Ctx* c = &ctx->c;
  if (!c->X || !c->yreal) return fail(c, "skd_linear_r2_batch: stage X and targets first");
  if (B <= 0 || !coef || !col_fold || !sse_out || !count_out) return fail(c, "skd_linear_r2_batch: bad arguments");
  if (check_score_codes(c, "skd_linear_r2_batch", B, col_fold)) return 1;
  SKD_CUDA(c, cudaSetDevice(c->device));
  Scratch sx(c);
  std::vector<SlotMeta> hs(B);
  for (int j = 0; j < B; ++j) { hs[j].col = j; hs[j].fold = col_fold[j]; hs[j].pos = 0; hs[j].pad = 0; }
  SlotMeta* dslot; double* dsse; int64_t* dcount;
  SKD_CUDA(c, sx.alloc(&dslot, (size_t)B));
  SKD_CUDA(c, sx.alloc(&dsse, (size_t)B));
  SKD_CUDA(c, sx.alloc(&dcount, (size_t)B));
  SKD_CUDA(c, cudaMemcpyAsync(dslot, hs.data(), B * sizeof(SlotMeta), cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemsetAsync(dsse, 0, B * sizeof(double), c->stream));
  SKD_CUDA(c, cudaMemsetAsync(dcount, 0, B * sizeof(int64_t), c->stream));
  bool use_tc;
  if (use_tensor_cores(c, &use_tc)) return 1;
  if (use_tc) {
    LogregWork w;
    if (tc_scoring_setup(c, sx, w, B, coef, dslot)) return 1;
    const size_t n_part = (size_t)tc_partials_per_slot() * B;   // per-chunk squared-error sums
    SKD_CUDA(c, sx.alloc(&w.lb.lossp, n_part));
    SKD_CUDA(c, cudaMemsetAsync(w.lb.lossp, 0, n_part * sizeof(double), c->stream));
    if (tc_r2(c, w, B, dsse, dcount)) return 1;
  } else {
    float* dW;
    if (pack_coef(c, sx, B, coef, c->d, c->ldx, &dW)) return 1;
    if (simt_r2(c, B, dW, dslot, dsse, dcount)) return 1;
  }
  SKD_CUDA(c, cudaMemcpyAsync(sse_out, dsse, B * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(count_out, dcount, B * sizeof(int64_t), cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  c->d2h += (int64_t)B * 16;
  return 0;
}

int skd_sgd_fit_batch(skd_ctx* ctx, int32_t B, const int32_t* col_pos, int32_t loss, double alpha,
                      int32_t fit_intercept, int32_t max_iter, double tol, int32_t shuffle,
                      uint32_t seed, int32_t lr_type, double eta0, double power_t, double optimal_init,
                      int32_t n_iter_no_change, float* coef_out, double* intercept_out,
                      int32_t* n_iter_out, double* t_out, int32_t* status_out, double* gpu_seconds_out) {
  if (!ctx) return fail(nullptr, "skd_sgd_fit_batch: ctx is NULL");
  Ctx* c = &ctx->c;
  if (!c->X || !c->ycls) return fail(c, "skd_sgd_fit_batch: stage X and labels first");
  if (B <= 0 || !col_pos || !coef_out || !intercept_out || !n_iter_out || !t_out || !status_out)
    return fail(c, "skd_sgd_fit_batch: bad arguments");
  if (loss < 0 || loss > 1 || lr_type < 0 || lr_type > 2 || !(alpha > 0.0) || max_iter < 1)
    return fail(c, "skd_sgd_fit_batch: unsupported loss / learning rate / alpha / max_iter");
  SKD_CUDA(c, cudaSetDevice(c->device));
  DeviceTimer timer(c);
  if (timer.start()) return 1;
  if (sgd_fit_batch(c, B, col_pos, loss, alpha, fit_intercept, max_iter, tol, shuffle, seed, lr_type, eta0, power_t,
                    optimal_init, n_iter_no_change, coef_out, intercept_out, n_iter_out, t_out, status_out))
    return 1;
  return timer.stop(gpu_seconds_out);
}

int skd_sgd_fit_groups(skd_ctx* ctx, int32_t B, const int32_t* col_pos, const int32_t* col_group,
                       const double* col_alpha, const double* col_optimal_init, int32_t G, const int64_t* group_offsets,
                       const int32_t* group_rows, const uint32_t* group_seeds, int32_t loss, int32_t fit_intercept,
                       int32_t max_iter, double tol, int32_t shuffle, int32_t lr_type, double eta0, double power_t,
                       int32_t n_iter_no_change, float* coef_out, double* intercept_out, int32_t* n_iter_out,
                       double* t_out, int32_t* status_out, double* gpu_seconds_out) {
  if (!ctx) return fail(nullptr, "skd_sgd_fit_groups: ctx is NULL");
  Ctx* c = &ctx->c;
  if (!c->X || !c->ycls) return fail(c, "skd_sgd_fit_groups: stage X and labels first");
  if (B <= 0 || G <= 0 || !col_pos || !col_group || !col_alpha || !col_optimal_init || !group_offsets || !group_rows ||
      !group_seeds || !coef_out || !intercept_out || !n_iter_out || !t_out || !status_out)
    return fail(c, "skd_sgd_fit_groups: bad arguments");
  if (loss < 0 || loss > 1 || lr_type < 0 || lr_type > 2 || max_iter < 1)
    return fail(c, "skd_sgd_fit_groups: unsupported loss / learning rate / max_iter");
  if (c->n >= ((int64_t)1 << 31)) return fail(c, "skd_sgd_fit_groups: row ids are int32, n must be < 2^31");
  for (int32_t j = 0; j < B; ++j) {
    if (col_group[j] < 0 || col_group[j] >= G)
      return fail(c, "skd_sgd_fit_groups: column " + std::to_string(j) + " names group " +
                         std::to_string(col_group[j]) + ", not in [0, G)");
    if (!(col_alpha[j] > 0.0))
      return fail(c, "skd_sgd_fit_groups: column " + std::to_string(j) + " has alpha <= 0");
  }
  if (group_offsets[0] != 0) return fail(c, "skd_sgd_fit_groups: group_offsets[0] must be 0");
  for (int32_t g = 0; g < G; ++g)
    if (group_offsets[g + 1] <= group_offsets[g])
      return fail(c, "skd_sgd_fit_groups: group " + std::to_string(g) + " is empty");
  for (int64_t i = 0; i < group_offsets[G]; ++i)
    if (group_rows[i] < 0 || group_rows[i] >= c->n)
      return fail(c, "skd_sgd_fit_groups: row id " + std::to_string(group_rows[i]) + " at position " +
                         std::to_string(i) + " is outside [0, n)");
  SKD_CUDA(c, cudaSetDevice(c->device));
  DeviceTimer timer(c);
  if (timer.start()) return 1;
  if (sgd_fit_groups(c, B, col_pos, col_group, col_alpha, col_optimal_init, G, group_offsets, group_rows,
                     group_seeds, loss, fit_intercept, max_iter, tol, shuffle, lr_type, eta0, power_t,
                     n_iter_no_change, coef_out, intercept_out, n_iter_out, t_out, status_out))
    return 1;
  return timer.stop(gpu_seconds_out);
}

struct skd_forest {
  struct Tree {
    int32_t max_depth = 0, n_classes = 0, node_count = 0;
    std::vector<int32_t> left, right, feature, nsamp;
    std::vector<uint8_t> mgl;
    std::vector<double> thr, imp, wn, val;
    std::vector<uint32_t> compact;     // 8 words per node (throughput builder); expanded by skd_forest_tree_copy
    std::vector<double> cw;            // class weights the tree was built with (compact records of a weighted fit)
  };
  std::vector<Tree> trees;
  ForestClassWeights cw;               // staged for the fit (n_classes == 0: unweighted)
  int32_t criterion = 0;               // staged for the fit: 0 Gini / MSE, 1 entropy
  std::vector<float> binval;           // [d][256] distinct feature values (thresholds of compact records)
};

static void forest_sink(void* arg, int t, const SkdTreeView* v) {
  skd_forest* f = (skd_forest*)arg;
  skd_forest::Tree& tr = f->trees[t];
  const int m = v->node_count;
  tr.max_depth = v->max_depth; tr.n_classes = v->n_classes; tr.node_count = m;
  // the class weights the tree was built with, for the impurity formed from its class sums
  std::vector<double> cw;
  if (f->cw.n_classes && m > 0 && (v->compact || v->class_sums)) {
    cw = f->cw.w;
    if (f->cw.balanced_subsample) {   // the root's class sums are the bootstrap class counts
      std::vector<uint32_t> root(v->n_classes);
      for (int c = 0; c < v->n_classes; ++c) root[c] = v->compact ? v->compact[4 + c] : (uint32_t)v->class_sums[c];
      cw.resize(v->n_classes);
      forest_subsample_weights(root.data(), v->n_classes, cw.data());
    }
  }
  if (v->compact) {
    tr.compact.assign(v->compact, v->compact + (size_t)m * 8);
    tr.cw = std::move(cw);
    return;
  }
  tr.left.assign(v->left, v->left + m); tr.right.assign(v->right, v->right + m);
  tr.feature.assign(v->feature, v->feature + m); tr.nsamp.assign(v->n_node_samples, v->n_node_samples + m);
  tr.mgl.assign(v->missing_go_to_left, v->missing_go_to_left + m);
  tr.thr.assign(v->threshold, v->threshold + m); tr.imp.assign(v->impurity, v->impurity + m);
  tr.wn.assign(v->weighted_n_node_samples, v->weighted_n_node_samples + m);
  tr.val.assign(v->value, v->value + (size_t)m * v->n_classes);
  if (v->class_sums) {   // entropy trees: the builder's impurity was formed with CUDA's log
    const int C = v->n_classes;
    forest_class_impurity(
        m, C, cw.empty() ? nullptr : cw.data(), true, [&](int i) { return v->class_sums + (size_t)i * C; },
        [&](int i, int& l, int& r) { l = v->left[i]; r = v->right[i]; return l >= 0; }, tr.imp.data());
  }
}

int skd_forest_fit(skd_ctx* ctx, int32_t n_trees, const uint8_t* sample_counts, const uint32_t* rand_states,
                   int32_t n_classes, int32_t max_features, int32_t max_depth, int32_t min_samples_split,
                   int32_t min_samples_leaf, double min_weight_leaf, double min_impurity_decrease,
                   int32_t splitter, const double* y_regression, skd_forest** out, double* gpu_seconds_out) {
  if (!ctx) return fail(nullptr, "skd_forest_fit: ctx is NULL");
  Ctx* c = &ctx->c;
  const ForestClassWeights cw = std::exchange(c->forest_cw, {});
  const int32_t criterion = std::exchange(c->forest_criterion, 0);
  if (!out) return fail(c, "skd_forest_fit: out is NULL");
  *out = nullptr;
  if (!c->X || (!y_regression && !c->ycls)) return fail(c, "skd_forest_fit: stage X and labels first");
  if (n_trees <= 0 || !rand_states || max_features < 1 || min_samples_split < 2 || min_samples_leaf < 1 ||
      splitter < 0 || splitter > 2)
    return fail(c, "skd_forest_fit: bad arguments");
  SKD_CUDA(c, cudaSetDevice(c->device));
  std::unique_ptr<skd_forest> f(new skd_forest());
  f->trees.resize(n_trees);
  f->cw = cw;
  f->criterion = criterion;
  DeviceTimer timer(c);
  if (timer.start()) return 1;
  if (forest_fit(c, n_trees, sample_counts, rand_states, n_classes, max_features, max_depth, min_samples_split,
                 min_samples_leaf, min_weight_leaf, min_impurity_decrease, splitter == 1, splitter == 2,
                 criterion == 1, y_regression, cw.n_classes ? &cw : nullptr, forest_sink, f.get()))
    return 1;
  f->binval = c->forest.h_binval;
  if (timer.stop(gpu_seconds_out)) return 1;
  *out = f.release();
  return 0;
}

int skd_forest_kernel_seconds(skd_ctx* ctx, double* seconds_out) {
  if (!ctx || !seconds_out) return fail(nullptr, "skd_forest_kernel_seconds: bad arguments");
  *seconds_out = ctx->c.forest_kernel_ms * 1e-3;
  return 0;
}

int skd_forest_tree_size(skd_forest* f, int32_t tree, int32_t* node_count, int32_t* max_depth) {
  if (!f || tree < 0 || tree >= (int)f->trees.size()) return fail(nullptr, "skd_forest_tree_size: bad arguments");
  if (node_count) *node_count = f->trees[tree].node_count;
  if (max_depth) *max_depth = f->trees[tree].max_depth;
  return 0;
}

int skd_forest_tree_copy(skd_forest* f, int32_t tree, int32_t* left, int32_t* right, int32_t* feature,
                         double* threshold, double* impurity, int32_t* n_node_samples,
                         double* weighted_n_node_samples, uint8_t* missing_go_to_left, double* value) {
  if (!f || tree < 0 || tree >= (int)f->trees.size()) return fail(nullptr, "skd_forest_tree_copy: bad arguments");
  const skd_forest::Tree& t = f->trees[tree];
  if (!t.compact.empty()) {
    // Compact records of the throughput builder: {right child, feature | bin_a << 16 | bin_b << 24,
    // n_node_samples, depth, class sums[4]}, nodes in depth-first order (left child = id + 1).  The
    // float64 fields are formed here with the builder's (= scikit-learn's) operations:
    //   weighted_n = sum_c s_c;  value_c = s_c / weighted_n                     (weighted_class_sums)
    //   impurity   = Gini, as forest_class_impurity forms it
    //   threshold  = v[a] / 2 + v[b] / 2                                        (SK/tree/_splitter.pyx:459-461)
    const size_t m = (size_t)t.node_count;
    const int C = t.n_classes;
    const uint32_t* r = t.compact.data();
    const float* bv = f->binval.data();
    const double* cw = t.cw.empty() ? nullptr : t.cw.data();
    for (size_t i = 0; i < m; ++i, r += 8) {
      const int32_t rc = (int32_t)r[0];
      const uint32_t code = r[1];
      const bool leaf = (code & 0xFFFFu) == 0xFFFFu;
      if (left) left[i] = leaf ? -1 : (int32_t)i + 1;
      if (right) right[i] = leaf ? -1 : rc;
      if (feature) feature[i] = leaf ? -2 : (int32_t)(code & 0xFFFFu);
      if (threshold) {
        if (leaf) threshold[i] = -2.0;
        else {
          const size_t fo = (size_t)(code & 0xFFFFu) * 256;
          const volatile double ha = (double)bv[fo + ((code >> 16) & 0xFF)] / 2.0;
          const volatile double hb = (double)bv[fo + ((code >> 24) & 0xFF)] / 2.0;
          threshold[i] = ha + hb;
        }
      }
      if (n_node_samples) n_node_samples[i] = (int32_t)r[2];
      if (missing_go_to_left) missing_go_to_left[i] = 0;
      double s[4];
      const double w = weighted_class_sums(r + 4, C, cw, s);
      if (weighted_n_node_samples) weighted_n_node_samples[i] = w;
      if (value) for (int c = 0; c < C; ++c) value[i * C + c] = s[c] / w;
    }
    const uint32_t* rec = t.compact.data();
    auto children = [&](int i, int& l, int& rc) {
      rc = (int32_t)rec[(size_t)i * 8];
      l = i + 1;
      return (rec[(size_t)i * 8 + 1] & 0xFFFFu) != 0xFFFFu && rc > 0;
    };
    if (impurity)
      forest_class_impurity((int)m, C, cw, false, [&](int i) { return rec + (size_t)i * 8 + 4; }, children, impurity);
    if (missing_go_to_left) {      // n_left > n_right (SK/tree/_splitter.pyx: best_split.missing_go_to_left with no missing values)
      int l, rc;
      for (size_t i = 0; i < m; ++i)
        if (children((int)i, l, rc)) missing_go_to_left[i] = rec[(size_t)l * 8 + 2] > rec[(size_t)rc * 8 + 2] ? 1 : 0;
    }
    return 0;
  }
  const size_t m = t.left.size();
  if (left) memcpy(left, t.left.data(), m * 4);
  if (right) memcpy(right, t.right.data(), m * 4);
  if (feature) memcpy(feature, t.feature.data(), m * 4);
  if (threshold) memcpy(threshold, t.thr.data(), m * 8);
  if (impurity) memcpy(impurity, t.imp.data(), m * 8);
  if (n_node_samples) memcpy(n_node_samples, t.nsamp.data(), m * 4);
  if (weighted_n_node_samples) memcpy(weighted_n_node_samples, t.wn.data(), m * 8);
  if (missing_go_to_left) memcpy(missing_go_to_left, t.mgl.data(), m);
  if (value) memcpy(value, t.val.data(), t.val.size() * 8);
  return 0;
}

// The same tree as an array of 64-byte node records {left, right, feature: int64; threshold, impurity:
// float64; n_node_samples: int64; weighted_n_node_samples: float64; missing_go_to_left: uint8 + 7 pad}
// -- scikit-learn's `Node` struct (SK/tree/_tree.pxd:15-25), so that the caller can hand the buffer to
// `Tree.__setstate__` without building it field by field.
int skd_forest_tree_nodes(skd_forest* f, int32_t tree, void* nodes64, double* value) {
  if (!f || tree < 0 || tree >= (int)f->trees.size() || !nodes64) return fail(nullptr, "skd_forest_tree_nodes: bad arguments");
  const skd_forest::Tree& t = f->trees[tree];
  const size_t m = (size_t)t.node_count;
  struct Node64 { int64_t left, right, feature; double threshold, impurity; int64_t n_node_samples; double weighted; uint8_t mgl; uint8_t pad[7]; };
  static_assert(sizeof(Node64) == 64, "node record must be 64 bytes");
  Node64* out = (Node64*)nodes64;
  std::vector<int32_t> l(m), r(m), ft(m), ns(m);
  std::vector<uint8_t> mg(m);
  std::vector<double> th(m), im(m), wn(m);
  if (skd_forest_tree_copy(f, tree, l.data(), r.data(), ft.data(), th.data(), im.data(), ns.data(), wn.data(), mg.data(), value))
    return 1;
  for (size_t i = 0; i < m; ++i) {
    Node64 nd;
    nd.left = l[i]; nd.right = r[i]; nd.feature = ft[i]; nd.threshold = th[i]; nd.impurity = im[i];
    nd.n_node_samples = ns[i]; nd.weighted = wn[i]; nd.mgl = mg[i];
    memset(nd.pad, 0, sizeof(nd.pad));
    out[i] = nd;
  }
  return 0;
}

void skd_forest_free(skd_forest* f) { delete f; }

// Streams m new rows [m x d] (row pitch ld) through `kernel(dX, rows, ldx, dO)` in row chunks whose input
// and output each take <= 256 MiB: threaded pinned-bounce H2D (stage_rows_h2d), one pass of the kernel, D2H
// of the result of out_row_bytes per row into out.  The copy engine is the bottleneck.  *seconds: wall time
// of the chunks.
static int stream_rows(Ctx* c, Scratch& sx, const float* Xnew, int64_t m, int64_t d, int64_t ld, size_t out_row_bytes,
                       void* out, double* seconds,
                       const std::function<int(const float* dX, int64_t rows, int ldx, void* dO)>& kernel) {
  const int64_t ldx = round_up(d, 4);
  const int64_t row_bytes = std::max<int64_t>(ldx * 4, (int64_t)out_row_bytes);
  int64_t rows_per_chunk = std::max<int64_t>(1, ((int64_t)256 << 20) / row_bytes);
  if (rows_per_chunk > m) rows_per_chunk = m;
  float* dX; uint8_t* dO;
  SKD_CUDA(c, sx.alloc(&dX, (size_t)rows_per_chunk * ldx));
  SKD_CUDA(c, sx.alloc(&dO, (size_t)rows_per_chunk * out_row_bytes));
  if (ldx != d) SKD_CUDA(c, cudaMemsetAsync(dX, 0, (size_t)rows_per_chunk * ldx * 4, c->stream));
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  auto w0 = std::chrono::steady_clock::now();
  for (int64_t r0 = 0; r0 < m; r0 += rows_per_chunk) {
    const int64_t mr = std::min(rows_per_chunk, m - r0);
    if (stage_rows_h2d(c, dX, ldx, Xnew + r0 * ld, mr, d, ld)) return 1;
    if (kernel(dX, mr, (int)ldx, dO)) return 1;
    SKD_CUDA(c, cudaMemcpyAsync((uint8_t*)out + r0 * out_row_bytes, dO, (size_t)mr * out_row_bytes,
                                cudaMemcpyDeviceToHost, c->stream));
    SKD_CUDA(c, cudaStreamSynchronize(c->stream));
    c->h2d += mr * d * 4;
    c->d2h += mr * (int64_t)out_row_bytes;
  }
  if (seconds) *seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - w0).count();
  return 0;
}

int skd_predict_linear(skd_ctx* ctx, const float* Xnew, int64_t m, int64_t d, int64_t ld, int32_t B,
                       const float* coef, float* out, double* gpu_seconds_out) {
  if (!ctx) return fail(nullptr, "skd_predict_linear: ctx is NULL");
  Ctx* c = &ctx->c;
  if (!Xnew || m <= 0 || d <= 0 || ld < d || B <= 0 || !coef || !out) return fail(c, "skd_predict_linear: bad arguments");
  SKD_CUDA(c, cudaSetDevice(c->device));
  Scratch sx(c);
  float* dW;
  if (pack_coef(c, sx, B, coef, d, round_up(d, 4), &dW)) return 1;
  return stream_rows(c, sx, Xnew, m, d, ld, (size_t)B * 4, out, gpu_seconds_out,
                     [&](const float* dX, int64_t rows, int ldx, void* dO) {
                       return predict_device(c, dX, rows, ldx, (int)d, B, dW, (float*)dO);
                     });
}

int skd_forest_predict(skd_ctx* ctx, const float* Xnew, int64_t m, int64_t d, int64_t ld,
                       int32_t n_trees, const int64_t* tree_offset, const int32_t* left,
                       const int32_t* right, const int32_t* feature, const double* threshold,
                       const double* value, int32_t n_classes, double* proba_out,
                       double* gpu_seconds_out) {
  if (!ctx) return fail(nullptr, "skd_forest_predict: ctx is NULL");
  Ctx* c = &ctx->c;
  if (!Xnew || m <= 0 || d <= 0 || ld < d || n_trees <= 0 || !tree_offset || !left || !right || !feature ||
      !threshold || !value || n_classes <= 0 || !proba_out)
    return fail(c, "skd_forest_predict: bad arguments");
  SKD_CUDA(c, cudaSetDevice(c->device));
  const int64_t total = tree_offset[n_trees];
  if (tree_offset[0] != 0 || total <= 0) return fail(c, "skd_forest_predict: tree_offset must start at 0 and increase");
  // validate the tree arrays once on the host: a malformed child or feature index must not become
  // an out-of-bounds device read
  std::vector<int32_t> hnode((size_t)total * 4);
  for (int t = 0; t < n_trees; ++t) {
    const int64_t b = tree_offset[t], e = tree_offset[t + 1];
    if (e <= b) return fail(c, "skd_forest_predict: empty tree");
    for (int64_t k = b; k < e; ++k) {
      const int32_t l = left[k], r = right[k], f = feature[k];
      if (l != -1 && (l <= 0 || l >= e - b || r <= 0 || r >= e - b || f < 0 || f >= d))
        return fail(c, "skd_forest_predict: malformed tree arrays");
      hnode[(size_t)k * 4] = l; hnode[(size_t)k * 4 + 1] = r; hnode[(size_t)k * 4 + 2] = l == -1 ? 0 : f;
      hnode[(size_t)k * 4 + 3] = 0;
    }
  }
  Scratch sx(c);
  int64_t* d_off; int32_t* d_node; double *d_thr, *d_val;
  SKD_CUDA(c, sx.alloc(&d_off, (size_t)n_trees + 1));
  SKD_CUDA(c, sx.alloc(&d_node, (size_t)total * 4));
  SKD_CUDA(c, sx.alloc(&d_thr, (size_t)total));
  SKD_CUDA(c, sx.alloc(&d_val, (size_t)total * n_classes));
  SKD_CUDA(c, cudaMemcpyAsync(d_off, tree_offset, ((size_t)n_trees + 1) * 8, cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(d_node, hnode.data(), hnode.size() * 4, cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(d_thr, threshold, (size_t)total * 8, cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(d_val, value, (size_t)total * n_classes * 8, cudaMemcpyHostToDevice, c->stream));
  c->h2d += total * (int64_t)(16 + 8 + 8 * n_classes);
  return stream_rows(c, sx, Xnew, m, d, ld, (size_t)n_classes * 8, proba_out, gpu_seconds_out,
                     [&](const float* dX, int64_t rows, int ldx, void* dO) {
                       return forest_predict_device(c, dX, rows, ldx, n_trees, d_off, d_node, d_thr, d_val, n_classes,
                                                    (double*)dO);
                     });
}

int skd_linear_decision(skd_ctx* ctx, int32_t B, const float* coef, float* out) {
  if (!ctx) return fail(nullptr, "skd_linear_decision: ctx is NULL");
  Ctx* c = &ctx->c;
  if (!c->X) return fail(c, "skd_linear_decision: stage X first");
  if (B <= 0 || !coef || !out) return fail(c, "skd_linear_decision: bad arguments");
  SKD_CUDA(c, cudaSetDevice(c->device));
  Scratch sx(c);
  float *dW, *dout;
  if (pack_coef(c, sx, B, coef, c->d, c->ldx, &dW)) return 1;
  SKD_CUDA(c, sx.alloc(&dout, (size_t)c->n * B));
  // up to 16 models whose rows fit the weight cache 8 at a time run on the row-per-warp kernel; more models
  // or wider rows on the 64 x 64 tiled kernel
  if (B <= 16 && predict_cache_rows(c->ldx) == 8) {
    if (predict_device(c, c->X, c->n, (int)c->ldx, (int)c->d, B, dW, dout)) return 1;
  } else if (simt_decision(c, B, dW, dout)) return 1;
  SKD_CUDA(c, cudaMemcpyAsync(out, dout, (size_t)c->n * B * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  c->d2h += (int64_t)c->n * B * 4;
  return 0;
}

// ---- device optimiser on caller-supplied evaluation partials (tests) ------------------------
}  // extern "C"

struct skd_lbfgs_dev {
  Ctx* c = nullptr;
  std::unique_ptr<Scratch> sx;
  int d = 0, nz = 0, fit_intercept = 1;
  int slot_cap = 0;   // entries of the active list
  size_t rows = 0;    // floats of the exported fp32 rows (0: the grouped layout exports fp16 hi / lo)
  LogregWork w;       // w.lb: the optimiser batch; the rest only for the grouped layout's tensor-core export
  int32_t* hist = nullptr;   // device {slots, running} of the last round
};

static int lbfgs_dev_setup(skd_lbfgs_dev* h, int B, int K, int grouped, const int32_t* col_fold, int use_reduce,
                           int maxiter, int maxls, double pgtol, double ftol, const double* l2, const double* inv_n,
                           const double* gscale, const uint8_t* fmask) {
  Ctx* c = h->c;
  const int d = h->d, dp = d + 1;
  if (!c->X) return fail(c, "skd_lbfgs_dev_create: stage X first (d and the row pitch come from it)");
  if (B <= 0 || K < 1 || d != (int)c->d || h->nz < 1 || !col_fold || !l2 || !inv_n || maxiter < 1 || maxls < 1)
    return fail(c, "skd_lbfgs_dev_create: bad arguments");
  if (K > 1 && (grouped || use_reduce || gscale))
    return fail(c, "skd_lbfgs_dev_create: the multinomial optimiser has the dense layout and the direct gather only");
  SKD_CUDA(c, cudaSetDevice(c->device));
  h->sx.reset(new Scratch(c));
  Scratch& sx = *h->sx;
  LogregWork& w = h->w;
  LbfgsBatch& b = w.lb;
  b.B = B; b.K = K; b.n = K * dp; b.nz = h->nz;
  SKD_CUDA(c, sx.alloc(&h->hist, 2));
  std::vector<int32_t> zeros(B, 0);
  std::vector<SlotMeta> hslots;
  if (grouped) {   // the fit's tensor-core layout; its trial points leave through tc_export
    if (!tc_supported(c)) return fail(c, "skd_lbfgs_dev_create: the grouped layout needs a staged X with d <= 256");
    if (grouped_slot_layout(c, B, col_fold, zeros.data(), nullptr, hslots)) return 1;
    if (tc_prepare(c)) return 1;
    w.use_tc = true;
    b.grouped = true;
    h->slot_cap = (int)hslots.size();
    if (alloc_tc_weights(c, sx, w, h->slot_cap)) return 1;
  } else {
    h->slot_cap = B;
    b.ldw = (int)c->ldx;
    h->rows = (size_t)B * K * c->ldx + (size_t)B * K;
    SKD_CUDA(c, sx.alloc(&b.W, h->rows));
  }
  w.slot_cap = h->slot_cap;
  const size_t cap = (size_t)h->nz * h->slot_cap;
  SKD_CUDA(c, sx.alloc(&b.lossp, cap));
  SKD_CUDA(c, sx.alloc(&b.gsump, cap * K));
  SKD_CUDA(c, sx.alloc(&b.gradp, cap * K * b.ldw));
  if (use_reduce) SKD_CUDA(c, sx.alloc(&b.gradr, (size_t)h->slot_cap * b.ldw));
  if (lbfgs_alloc(c, sx, b, h->slot_cap, K == 1)) return 1;
  if (fmask) {
    SKD_CUDA(c, sx.alloc(&b.fmask, (size_t)B * d));
    SKD_CUDA(c, cudaMemcpyAsync(b.fmask, fmask, (size_t)B * d, cudaMemcpyHostToDevice, c->stream));
  }
  if (gscale) {
    double* dgs;
    SKD_CUDA(c, sx.alloc(&dgs, (size_t)d));
    SKD_CUDA(c, cudaMemcpyAsync(dgs, gscale, d * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    b.gscale = dgs;
  }
  int32_t* dfold;
  SKD_CUDA(c, sx.alloc(&dfold, (size_t)B));
  SKD_CUDA(c, cudaMemcpyAsync(dfold, col_fold, B * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(b.l2, l2, B * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(b.inv_n, inv_n, B * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  if (b.n_run) SKD_CUDA(c, cudaMemcpyAsync(b.n_run, &B, sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
  if (b.grouped) {
    const int32_t ns = h->slot_cap;
    SKD_CUDA(c, cudaMemcpyAsync(b.slot, hslots.data(), hslots.size() * sizeof(SlotMeta), cudaMemcpyHostToDevice, c->stream));
    SKD_CUDA(c, cudaMemcpyAsync(b.n_act, &ns, sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
  }
  if (lbfgs_init(c, b, b.grouped ? nullptr : dfold, nullptr, nullptr, pgtol, maxiter, maxls, ftol)) return 1;
  if (w.use_tc && tc_export(c, w, h->slot_cap, nullptr, h->fit_intercept)) return 1;
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  return 0;
}

// One round: the caller's per-column parts scattered into the partial buffers by the current slot list with
// stride n_act_in (NaN in every slot that holds no live column), then the fit's optimiser round itself.
static int lbfgs_dev_round(skd_lbfgs_dev* h, int n_act_in, const double* loss_parts, const double* gsum_parts,
                           const float* grad_parts, double* x_out, void* state_out, int32_t* slot_out,
                           int32_t* counts_out, float* rows_out) {
  Ctx* c = h->c;
  LbfgsBatch& b = h->w.lb;
  const int B = b.B, K = b.K, d = h->d, nz = h->nz, ldw = b.ldw;
  std::vector<SlotMeta> hs(h->slot_cap);
  int32_t live = 0;
  SKD_CUDA(c, cudaMemcpyAsync(hs.data(), b.slot, hs.size() * sizeof(SlotMeta), cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(&live, b.n_act, sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  if (n_act_in < live || n_act_in > h->slot_cap)
    return fail(c, "skd_lbfgs_dev_step: n_act_in must lie between the live slot count and the slot capacity");
  const double nan = std::nan("");
  const size_t ns = (size_t)n_act_in * K;   // partial rows per chunk
  std::vector<double> lp((size_t)nz * n_act_in, nan), gs((size_t)nz * ns, nan);
  std::vector<float> gp((size_t)nz * ns * ldw, std::nanf(""));
  for (int s = 0; s < live; ++s) {
    const int col = hs[s].col;
    if (col < 0) continue;
    for (int z = 0; z < nz; ++z) {
      lp[(size_t)z * n_act_in + s] = loss_parts[(size_t)col * nz + z];
      for (int k = 0; k < K; ++k) {
        const size_t row = (size_t)z * ns + (size_t)s * K + k, src = ((size_t)col * K + k) * nz + z;
        gs[row] = gsum_parts[src];
        memcpy(&gp[row * ldw], grad_parts + src * d, d * sizeof(float));
      }
    }
  }
  SKD_CUDA(c, cudaMemcpyAsync(b.lossp, lp.data(), lp.size() * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(b.gsump, gs.data(), gs.size() * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(b.gradp, gp.data(), gp.size() * sizeof(float), cudaMemcpyHostToDevice, c->stream));
  if (lbfgs_enqueue(c, b, n_act_in, nz, h->fit_intercept, h->hist, b.grouped ? &h->w : nullptr)) return 1;
  SKD_CUDA(c, cudaMemcpy2DAsync(x_out, b.n * sizeof(double), b.vec, b.stride * sizeof(double), b.n * sizeof(double), B,
                                cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(state_out, b.sc, B * sizeof(LbfgsScalars), cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(slot_out, b.slot, h->slot_cap * sizeof(SlotMeta), cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(counts_out, b.n_act, sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(counts_out + 1, b.n_run ? b.n_run : b.n_act, sizeof(int32_t), cudaMemcpyDeviceToHost,
                              c->stream));
  SKD_CUDA(c, cudaMemcpyAsync(counts_out + 2, h->hist, 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
  if (rows_out && h->rows)
    SKD_CUDA(c, cudaMemcpyAsync(rows_out, b.W, h->rows * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  SKD_CUDA(c, cudaStreamSynchronize(c->stream));
  return 0;
}

static int lbfgs_dev_result(skd_lbfgs_dev* h, float* coef_out, int32_t* n_iter_out, int32_t* status_out,
                            double* loss_out) {
  Scratch sx(h->c);
  if (lbfgs_result(h->c, sx, h->w.lb, 0, coef_out, n_iter_out, status_out, loss_out, nullptr)) return 1;
  SKD_CUDA(h->c, cudaStreamSynchronize(h->c->stream));
  return 0;
}

extern "C" {

skd_lbfgs_dev* skd_lbfgs_dev_create(skd_ctx* ctx, int32_t B, int32_t K, int32_t d, int32_t fit_intercept,
                                    int32_t grouped, const int32_t* col_fold, int32_t nz, int32_t use_reduce,
                                    int32_t maxiter, int32_t maxls, double pgtol, double ftol, const double* l2,
                                    const double* inv_n, const double* gscale, const uint8_t* fmask,
                                    int32_t* dims_out) {
  if (!ctx) { fail(nullptr, "skd_lbfgs_dev_create: ctx is NULL"); return nullptr; }
  std::unique_ptr<skd_lbfgs_dev> h(new skd_lbfgs_dev());
  h->c = &ctx->c; h->d = d; h->nz = nz; h->fit_intercept = fit_intercept ? 1 : 0;
  if (lbfgs_dev_setup(h.get(), B, K, grouped, col_fold, use_reduce, maxiter, maxls, pgtol, ftol, l2, inv_n, gscale,
                      fmask))
    return nullptr;
  if (dims_out) {
    dims_out[0] = h->w.lb.n; dims_out[1] = h->slot_cap; dims_out[2] = h->w.lb.ldw; dims_out[3] = (int32_t)h->rows;
  }
  return h.release();
}

int skd_lbfgs_dev_step(skd_lbfgs_dev* h, int32_t n_act_in, const double* loss_parts, const double* gsum_parts,
                       const float* grad_parts, double* x_out, void* state_out, int32_t* slot_out,
                       int32_t* counts_out, float* rows_out) {
  if (!h) return fail(nullptr, "skd_lbfgs_dev_step: handle is NULL");
  if (!loss_parts || !gsum_parts || !grad_parts || !x_out || !state_out || !slot_out || !counts_out)
    return fail(h->c, "skd_lbfgs_dev_step: bad arguments");
  return lbfgs_dev_round(h, n_act_in, loss_parts, gsum_parts, grad_parts, x_out, state_out, slot_out, counts_out,
                         rows_out);
}

int skd_lbfgs_dev_finish(skd_lbfgs_dev* h, float* coef_out, int32_t* n_iter_out, int32_t* status_out,
                         double* loss_out) {
  if (!h) return fail(nullptr, "skd_lbfgs_dev_finish: handle is NULL");
  if (!coef_out || !n_iter_out || !status_out || !loss_out) return fail(h->c, "skd_lbfgs_dev_finish: bad arguments");
  return lbfgs_dev_result(h, coef_out, n_iter_out, status_out, loss_out);
}

void skd_lbfgs_dev_free(skd_lbfgs_dev* h) { delete h; }

// ---- host-side L-BFGS object (tests) ----------------------------------------------------
skd_lbfgs* skd_lbfgs_create(int32_t n, int32_t m, int32_t maxiter, int32_t maxls, double pgtol,
                            double ftol) {
  skd_lbfgs* h = new skd_lbfgs();
  lbfgs_init(h->s, n, m, maxiter, maxls, pgtol, ftol);
  h->buf.assign(lbfgs_col_doubles(n, m), 0.0);
  h->v = lbfgs_col_vectors(h->buf.data(), n, m);
  return h;
}
double* skd_lbfgs_x(skd_lbfgs* h) { return h->v.x; }
double* skd_lbfgs_g(skd_lbfgs* h) { return h->v.g; }
int skd_lbfgs_advance(skd_lbfgs* h, double f) {
  SeqPar P;
  lbfgs_advance(P, h->s, h->v, f);
  return h->s.status;
}
int skd_lbfgs_nit(skd_lbfgs* h) { return h->s.nit; }
int skd_lbfgs_nfev(skd_lbfgs* h) { return h->s.nfev; }
void skd_lbfgs_state(skd_lbfgs* h, void* out) { memcpy(out, &h->s, sizeof(LbfgsScalars)); }
void skd_lbfgs_set_state(skd_lbfgs* h, const void* in) { memcpy(&h->s, in, sizeof(LbfgsScalars)); }
int skd_lbfgs_state_bytes(void) { return (int)sizeof(LbfgsScalars); }
void skd_lbfgs_free(skd_lbfgs* h) { delete h; }

}  // extern "C"
