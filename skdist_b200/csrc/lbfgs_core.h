// lbfgs_core.h -- per-column L-BFGS-B (unconstrained specialisation) state machine.
//
// Replaces, for the batched device solver, the optimiser that the reference's
// per-task fit runs on the CPU:
//   skdist/distribute/search.py:230 (estimator_.fit)
//     -> sklearn/linear_model/_logistic.py:584-598  scipy.optimize.minimize(method="L-BFGS-B",
//        options maxiter=max_iter, maxls=50, gtol=tol, ftol=64*eps)
//     -> scipy/optimize/_lbfgsb_py.py:393-437 (reverse-communication loop around setulb)
//     -> L-BFGS-B 3.0 (Byrd, Lu, Nocedal, Zhu; Morales & Nocedal 2011): mainlb / lnsrlb /
//        dcsrch / dcstep / matupd.
//
// With no bounds (nbd == 0 for every variable, which is what sklearn passes) L-BFGS-B
// reduces to: direction d = -H g with H the limited-memory BFGS inverse Hessian built
// from the last `m` (s, y) pairs and H0 = (1/theta) I, theta = y'y / s'y; More'-Thuente
// line search (dcsrch: ftol=1e-3, gtol=0.9, xtol=0.1, stpmin=0, stpmax=1e10); first step
// 1/||d||, later steps 1; pair skipped when s'y <= eps * (-g_old'd * stp); memory dropped
// and the iteration restarted from steepest descent when the line search fails; stop on
// max|g| <= pgtol, on (f_old - f) <= factr*eps*max(|f_old|,|f|,1), or when the iteration
// count reaches maxiter (checked, as in scipy's wrapper, before the convergence tests).
// The direction is evaluated with the two-loop recursion, which is algebraically the
// compact-representation product that subsm() forms (difference: rounding, ~1e-16 rel).
//
// The same code is compiled for the host (sequential `SeqPar` policy; used by the CPU-side
// tests that pin it against scipy's setulb trajectories) and for the device (lbfgs_dev.cu:
// one warp per binary column, `WarpPar`; one CTA per multinomial candidate, `CtaPar`).  All
// threads of a column's warp or CTA execute the scalar logic redundantly; dot products are
// reductions that return the same value to every thread, so control flow stays uniform.
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define SKD_HD __host__ __device__ __forceinline__
#else
#define SKD_HD inline
#endif

namespace skd {

enum LbfgsStatus : int32_t {
  LB_RUNNING = 0,       // wants f,g at x
  LB_CONV_PGTOL = 1,    // CONVERGENCE: NORM_OF_PROJECTED_GRADIENT_<=_PGTOL
  LB_CONV_FTOL = 2,     // CONVERGENCE: REL_REDUCTION_OF_F_<=_FACTR*EPSMCH
  LB_MAXITER = 3,       // STOP: TOTAL NO. of ITERATIONS REACHED LIMIT
  LB_ABNORMAL = 4,      // ABNORMAL_TERMINATION_IN_LNSRCH
  LB_NONFINITE = 5      // f or g not finite (maps to error_score handling on the host)
};

// line-search internal task
enum { LS_START = 0, LS_FG = 1, LS_CONV = 2, LS_WARN = 3, LS_ERROR = 4 };

struct LbfgsScalars {
  // problem / options
  int32_t n;        // number of variables (d + fit_intercept)
  int32_t m;        // memory (10)
  int32_t maxiter;
  int32_t maxls;
  double pgtol;
  double ftol_abs;  // factr * epsmch  (== sklearn's ftol = 64*eps)
  // optimiser state
  int32_t status;
  int32_t started;  // 0 until the first f,g has been consumed
  int32_t iter;     // L-BFGS-B internal iteration counter
  int32_t nit;      // scipy wrapper's n_iterations
  int32_t nfev;
  int32_t col;      // number of stored pairs
  int32_t head;     // ring index of the oldest pair
  int32_t ifun, iback;
  double theta;
  double f, fold;
  double gd, gdold, stp, dnorm, dtd, sbgnrm;
  // dcsrch state
  int32_t ls_brackt, ls_stage;
  double ginit, gtest, gx, gy, finit, fx, fy, stx, sty, stmin, stmax, width, width1;
};

// Vector storage for one column.  All arrays have length n except S,Y (m*n) and rho/alpha (m).
struct LbfgsVectors {
  double* x;   // current point (the point at which f,g are requested / were evaluated)
  double* g;   // gradient at x (filled by the caller before advance())
  double* t;   // x at the start of the line search
  double* r;   // g at the start of the line search
  double* d;   // search direction
  double* S;   // m x n, ring buffer
  double* Y;   // m x n
  double* rho; // m : 1 / (s_i' y_i)
  double* alpha; // m scratch
};

// Memory of every device fit: scikit-learn leaves scipy's default, m = 10.
constexpr int LBFGS_M = 10;

// Doubles of one column's vector storage: x, g, t, r, d, then S, Y, then rho, alpha.
SKD_HD size_t lbfgs_col_doubles(int n, int m) { return (size_t)(5 + 2 * m) * n + 2 * m; }

// The column's vectors in the block of lbfgs_col_doubles(n, m) doubles at base.
SKD_HD LbfgsVectors lbfgs_col_vectors(double* base, int n, int m) {
  LbfgsVectors v;
  double* p = base;
  v.x = p; p += n;
  v.g = p; p += n;
  v.t = p; p += n;
  v.r = p; p += n;
  v.d = p; p += n;
  v.S = p; p += (size_t)m * n;
  v.Y = p; p += (size_t)m * n;
  v.rho = p; p += m;
  v.alpha = p;
  return v;
}

// --- MINPACK-2 dcstep -------------------------------------------------------------------
SKD_HD void dcstep(double& stx, double& fx, double& dx, double& sty, double& fy, double& dy,
                   double& stp, double fp, double dp, int32_t& brackt, double stpmin,
                   double stpmax) {
  double sgnd = dp * (dx / fabs(dx));
  double stpf, stpc, stpq, theta, s, gamma, p, q, r;
  if (fp > fx) {
    theta = 3.0 * (fx - fp) / (stp - stx) + dx + dp;
    s = fmax(fabs(theta), fmax(fabs(dx), fabs(dp)));
    gamma = s * sqrt((theta / s) * (theta / s) - (dx / s) * (dp / s));
    if (stp < stx) gamma = -gamma;
    p = (gamma - dx) + theta;
    q = ((gamma - dx) + gamma) + dp;
    r = p / q;
    stpc = stx + r * (stp - stx);
    stpq = stx + ((dx / ((fx - fp) / (stp - stx) + dx)) / 2.0) * (stp - stx);
    if (fabs(stpc - stx) < fabs(stpq - stx)) stpf = stpc;
    else stpf = stpc + (stpq - stpc) / 2.0;
    brackt = 1;
  } else if (sgnd < 0.0) {
    theta = 3.0 * (fx - fp) / (stp - stx) + dx + dp;
    s = fmax(fabs(theta), fmax(fabs(dx), fabs(dp)));
    gamma = s * sqrt((theta / s) * (theta / s) - (dx / s) * (dp / s));
    if (stp > stx) gamma = -gamma;
    p = (gamma - dp) + theta;
    q = ((gamma - dp) + gamma) + dx;
    r = p / q;
    stpc = stp + r * (stx - stp);
    stpq = stp + (dp / (dp - dx)) * (stx - stp);
    if (fabs(stpc - stp) > fabs(stpq - stp)) stpf = stpc;
    else stpf = stpq;
    brackt = 1;
  } else if (fabs(dp) < fabs(dx)) {
    theta = 3.0 * (fx - fp) / (stp - stx) + dx + dp;
    s = fmax(fabs(theta), fmax(fabs(dx), fabs(dp)));
    gamma = s * sqrt(fmax(0.0, (theta / s) * (theta / s) - (dx / s) * (dp / s)));
    if (stp > stx) gamma = -gamma;
    p = (gamma - dp) + theta;
    q = (gamma + (dx - dp)) + gamma;
    r = p / q;
    if (r < 0.0 && gamma != 0.0) stpc = stp + r * (stx - stp);
    else if (stp > stx) stpc = stpmax;
    else stpc = stpmin;
    stpq = stp + (dp / (dp - dx)) * (stx - stp);
    if (brackt) {
      if (fabs(stpc - stp) < fabs(stpq - stp)) stpf = stpc;
      else stpf = stpq;
      if (stp > stx) stpf = fmin(stp + 0.66 * (sty - stp), stpf);
      else stpf = fmax(stp + 0.66 * (sty - stp), stpf);
    } else {
      if (fabs(stpc - stp) > fabs(stpq - stp)) stpf = stpc;
      else stpf = stpq;
      stpf = fmin(stpmax, stpf);
      stpf = fmax(stpmin, stpf);
    }
  } else {
    if (brackt) {
      theta = 3.0 * (fp - fy) / (sty - stp) + dy + dp;
      s = fmax(fabs(theta), fmax(fabs(dy), fabs(dp)));
      gamma = s * sqrt((theta / s) * (theta / s) - (dy / s) * (dp / s));
      if (stp > sty) gamma = -gamma;
      p = (gamma - dp) + theta;
      q = ((gamma - dp) + gamma) + dy;
      r = p / q;
      stpc = stp + r * (sty - stp);
      stpf = stpc;
    } else if (stp > stx) {
      stpf = stpmax;
    } else {
      stpf = stpmin;
    }
  }
  if (fp > fx) {
    sty = stp; fy = fp; dy = dp;
  } else {
    if (sgnd < 0.0) { sty = stx; fy = fx; dy = dx; }
    stx = stp; fx = fp; dx = dp;
  }
  stp = stpf;
}

// --- MINPACK-2 dcsrch (ftol=1e-3, gtol=0.9, xtol=0.1 as lnsrlb passes them) -------------
// Returns LS_FG / LS_CONV / LS_WARN / LS_ERROR.  `task_in` is LS_START on the first call.
SKD_HD int dcsrch(LbfgsScalars& s, double f, double g, double& stp, int task_in,
                  double stpmin, double stpmax) {
  const double ftol = 1e-3, gtol = 0.9, xtol = 0.1;
  const double p5 = 0.5, p66 = 0.66, xtrapl = 1.1, xtrapu = 4.0;
  if (task_in == LS_START) {
    if (stp < stpmin || stp > stpmax || g >= 0.0) return LS_ERROR;
    s.ls_brackt = 0;
    s.ls_stage = 1;
    s.finit = f;
    s.ginit = g;
    s.gtest = ftol * s.ginit;
    s.width = stpmax - stpmin;
    s.width1 = s.width / p5;
    s.stx = 0.0; s.fx = s.finit; s.gx = s.ginit;
    s.sty = 0.0; s.fy = s.finit; s.gy = s.ginit;
    s.stmin = 0.0;
    s.stmax = stp + xtrapu * stp;
    return LS_FG;
  }
  double ftest = s.finit + stp * s.gtest;
  if (s.ls_stage == 1 && f <= ftest && g >= 0.0) s.ls_stage = 2;
  int task = LS_FG;
  if (s.ls_brackt && (stp <= s.stmin || stp >= s.stmax)) task = LS_WARN;
  if (s.ls_brackt && s.stmax - s.stmin <= xtol * s.stmax) task = LS_WARN;
  if (stp == stpmax && f <= ftest && g <= s.gtest) task = LS_WARN;
  if (stp == stpmin && (f > ftest || g >= s.gtest)) task = LS_WARN;
  if (f <= ftest && fabs(g) <= gtol * (-s.ginit)) task = LS_CONV;
  if (task != LS_FG) return task;

  if (s.ls_stage == 1 && f <= s.fx && f > ftest) {
    double fm = f - stp * s.gtest;
    double fxm = s.fx - s.stx * s.gtest;
    double fym = s.fy - s.sty * s.gtest;
    double gm = g - s.gtest;
    double gxm = s.gx - s.gtest;
    double gym = s.gy - s.gtest;
    dcstep(s.stx, fxm, gxm, s.sty, fym, gym, stp, fm, gm, s.ls_brackt, s.stmin, s.stmax);
    s.fx = fxm + s.stx * s.gtest;
    s.fy = fym + s.sty * s.gtest;
    s.gx = gxm + s.gtest;
    s.gy = gym + s.gtest;
  } else {
    dcstep(s.stx, s.fx, s.gx, s.sty, s.fy, s.gy, stp, f, g, s.ls_brackt, s.stmin, s.stmax);
  }
  if (s.ls_brackt) {
    if (fabs(s.sty - s.stx) >= p66 * s.width1) stp = s.stx + p5 * (s.sty - s.stx);
    s.width1 = s.width;
    s.width = fabs(s.sty - s.stx);
  }
  if (s.ls_brackt) {
    s.stmin = fmin(s.stx, s.sty);
    s.stmax = fmax(s.stx, s.sty);
  } else {
    s.stmin = stp + xtrapl * (stp - s.stx);
    s.stmax = stp + xtrapu * (stp - s.stx);
  }
  stp = fmax(stp, stpmin);
  stp = fmin(stp, stpmax);
  if ((s.ls_brackt && (stp <= s.stmin || stp >= s.stmax)) ||
      (s.ls_brackt && s.stmax - s.stmin <= xtol * s.stmax))
    stp = s.stx;
  return LS_FG;
}

SKD_HD void lbfgs_init(LbfgsScalars& s, int n, int m, int maxiter, int maxls, double pgtol,
                       double ftol_abs) {
  s.n = n; s.m = m; s.maxiter = maxiter; s.maxls = maxls; s.pgtol = pgtol;
  s.ftol_abs = ftol_abs;
  s.status = LB_RUNNING; s.started = 0; s.iter = 0; s.nit = 0; s.nfev = 0;
  s.col = 0; s.head = 0; s.ifun = 0; s.iback = 0; s.theta = 1.0;
  s.f = 0.0; s.fold = 0.0; s.gd = 0.0; s.gdold = 0.0; s.stp = 0.0; s.dnorm = 0.0;
  s.dtd = 0.0; s.sbgnrm = 0.0;
  s.ls_brackt = 0; s.ls_stage = 1;
  s.ginit = s.gtest = s.gx = s.gy = s.finit = s.fx = s.fy = 0.0;
  s.stx = s.sty = s.stmin = s.stmax = s.width = s.width1 = 0.0;
}

// Par policy interface:
//   int  tid(), nthr();   void sync();
//   double dot(const double* a, const double* b, int n);     // same value in all threads
//   double amax(const double* a, int n);                     // max |a_i|, same in all threads
template <class Par>
SKD_HD void lbfgs_direction(Par& P, LbfgsScalars& s, LbfgsVectors& v) {
  const int n = s.n, m = s.m;
  // d = -g
  for (int i = P.tid(); i < n; i += P.nthr()) v.d[i] = -v.g[i];
  P.sync();
  if (s.col == 0) return;
  // two-loop recursion, newest pair first
  for (int k = s.col - 1; k >= 0; --k) {
    int j = (s.head + k) % m;
    const double* sj = v.S + (size_t)j * n;
    const double* yj = v.Y + (size_t)j * n;
    double a = v.rho[j] * P.dot(sj, v.d, n);
    if (P.tid() == 0) v.alpha[j] = a;
    for (int i = P.tid(); i < n; i += P.nthr()) v.d[i] -= a * yj[i];
    P.sync();
  }
  double inv_theta = 1.0 / s.theta;
  for (int i = P.tid(); i < n; i += P.nthr()) v.d[i] *= inv_theta;
  P.sync();
  for (int k = 0; k < s.col; ++k) {
    int j = (s.head + k) % m;
    const double* sj = v.S + (size_t)j * n;
    const double* yj = v.Y + (size_t)j * n;
    double b = v.rho[j] * P.dot(yj, v.d, n);
    double a = v.alpha[j];
    for (int i = P.tid(); i < n; i += P.nthr()) v.d[i] += (a - b) * sj[i];
    P.sync();
  }
}

// Begin a line search along v.d from (x, f, g); moves x to the first trial point.
// Returns false if the line search could not be started (ascent direction).
template <class Par>
SKD_HD bool lbfgs_begin_linesearch(Par& P, LbfgsScalars& s, LbfgsVectors& v) {
  const int n = s.n;
  s.dtd = P.dot(v.d, v.d, n);
  s.dnorm = sqrt(s.dtd);
  const double stpmx = 1e10;
  if (s.iter == 0) s.stp = fmin(1.0 / s.dnorm, stpmx);
  else s.stp = 1.0;
  for (int i = P.tid(); i < n; i += P.nthr()) { v.t[i] = v.x[i]; v.r[i] = v.g[i]; }
  s.fold = s.f;
  s.ifun = 0;
  s.iback = 0;
  P.sync();
  s.gd = P.dot(v.g, v.d, n);
  s.gdold = s.gd;
  if (!(s.gd < 0.0)) return false;  // info = -4
  int task = dcsrch(s, s.f, s.gd, s.stp, LS_START, 0.0, stpmx);
  if (task == LS_ERROR) return false;
  s.ifun = 1;
  s.nfev += 1;
  s.iback = 0;
  double stp = s.stp;
  for (int i = P.tid(); i < n; i += P.nthr()) v.x[i] = stp * v.d[i] + v.t[i];
  P.sync();
  return true;
}

// Drop the memory and restart from steepest descent at the restored point.
// Returns false if even that fails (abnormal termination).
template <class Par>
SKD_HD void lbfgs_new_direction_or_fail(Par& P, LbfgsScalars& s, LbfgsVectors& v) {
  // loop: try direction; on line-search start failure with memory, drop memory and retry
  for (;;) {
    lbfgs_direction(P, s, v);
    if (lbfgs_begin_linesearch(P, s, v)) return;
    // failed to start (info != 0): restore is a no-op (x,g,f untouched)
    if (s.col == 0) { s.status = LB_ABNORMAL; return; }
    s.col = 0; s.head = 0; s.theta = 1.0;
  }
}

// Consume f (already including any penalty) and g at x; advance until the next
// evaluation request or termination.  On return with status == LB_RUNNING the caller must
// evaluate f,g at v.x and call again.  On termination v.x holds the result.
template <class Par>
SKD_HD void lbfgs_advance(Par& P, LbfgsScalars& s, LbfgsVectors& v, double f_new) {
  const int n = s.n;
  if (s.status != LB_RUNNING) return;
  if (!(fabs(f_new) <= 1.79e308)) {  // NaN or Inf
    s.status = LB_NONFINITE;
    return;
  }
  if (!s.started) {
    s.started = 1;
    s.f = f_new;
    s.nfev = 1;
    s.sbgnrm = P.amax(v.g, n);
    if (s.sbgnrm <= s.pgtol) { s.status = LB_CONV_PGTOL; return; }
    lbfgs_new_direction_or_fail(P, s, v);
    return;
  }
  // ---- inside a line search: lnsrlb label 556 ----
  s.f = f_new;
  s.gd = P.dot(v.g, v.d, n);
  const double stpmx = 1e10;
  int task = dcsrch(s, s.f, s.gd, s.stp, LS_FG, 0.0, stpmx);
  if (task == LS_FG) {
    s.ifun += 1;
    s.iback = s.ifun - 1;
    if (s.iback >= s.maxls) {
      // line search failed: restore the previous iterate
      for (int i = P.tid(); i < n; i += P.nthr()) { v.x[i] = v.t[i]; v.g[i] = v.r[i]; }
      s.f = s.fold;
      P.sync();
      if (s.col == 0) { s.status = LB_ABNORMAL; return; }
      s.col = 0; s.head = 0; s.theta = 1.0;
      lbfgs_new_direction_or_fail(P, s, v);
      return;
    }
    // counted here, not above: a line search that has run out of maxls requests no evaluation
    s.nfev += 1;
    double stp = s.stp;
    for (int i = P.tid(); i < n; i += P.nthr()) v.x[i] = stp * v.d[i] + v.t[i];
    P.sync();
    return;
  }
  if (task == LS_ERROR) {
    for (int i = P.tid(); i < n; i += P.nthr()) { v.x[i] = v.t[i]; v.g[i] = v.r[i]; }
    s.f = s.fold;
    P.sync();
    if (s.col == 0) { s.status = LB_ABNORMAL; return; }
    s.col = 0; s.head = 0; s.theta = 1.0;
    lbfgs_new_direction_or_fail(P, s, v);
    return;
  }
  // ---- line search finished (CONV or WARN): new iterate ----
  s.iter += 1;
  s.sbgnrm = P.amax(v.g, n);
  // scipy wrapper (task NEW_X): count the iteration, stop on maxiter before testing convergence
  s.nit += 1;
  if (s.nit >= s.maxiter) { s.status = LB_MAXITER; return; }
  if (s.sbgnrm <= s.pgtol) { s.status = LB_CONV_PGTOL; return; }
  double ddum = fmax(fabs(s.fold), fmax(fabs(s.f), 1.0));
  if ((s.fold - s.f) <= s.ftol_abs * ddum) { s.status = LB_CONV_FTOL; return; }
  // r = g - r ; s = stp * d
  for (int i = P.tid(); i < n; i += P.nthr()) v.r[i] = v.g[i] - v.r[i];
  P.sync();
  double rr = P.dot(v.r, v.r, n);
  double dr, dd;
  double stp = s.stp;
  if (stp == 1.0) {
    dr = s.gd - s.gdold;
    dd = -s.gdold;
  } else {
    dr = (s.gd - s.gdold) * stp;
    dd = -s.gdold * stp;
  }
  const double epsmch = 2.220446049250313e-16;
  if (dr <= epsmch * dd) {
    // skip the update
  } else {
    int m = s.m, slot;
    if (s.col < m) { slot = (s.head + s.col) % m; s.col += 1; }
    else { slot = s.head; s.head = (s.head + 1) % m; }
    double* sj = v.S + (size_t)slot * n;
    double* yj = v.Y + (size_t)slot * n;
    for (int i = P.tid(); i < n; i += P.nthr()) { sj[i] = stp * v.d[i]; yj[i] = v.r[i]; }
    if (P.tid() == 0) v.rho[slot] = 1.0 / dr;
    s.theta = rr / dr;
    P.sync();
  }
  lbfgs_new_direction_or_fail(P, s, v);
}

// Sequential policy (host tests; also usable on device by a single thread).
struct SeqPar {
  SKD_HD int tid() const { return 0; }
  SKD_HD int nthr() const { return 1; }
  SKD_HD void sync() const {}
  SKD_HD double dot(const double* a, const double* b, int n) const {
    double acc = 0.0;
    for (int i = 0; i < n; ++i) acc += a[i] * b[i];
    return acc;
  }
  SKD_HD double amax(const double* a, int n) const {
    double mx = 0.0;
    for (int i = 0; i < n; ++i) mx = fmax(mx, fabs(a[i]));
    return mx;
  }
};

}  // namespace skd
