// MAP fit of the fitted-hyperparameter GP baseline: one CTA per (dataset, prefix length t) problem runs the whole
// L-BFGS fit -- objective, gradient, two-loop recursion, More-Thuente line search, the noise bound and the stopping
// tests -- and then forms the predictive of row t.  No host loop, no per-iteration launch, no device-to-host sync.
// Restates the maths of reference priors/fast_gp_mix.py:24-55,156-169 (botorch SingleTaskGP with Gamma priors,
// fit_gpytorch_model = scipy L-BFGS-B on ExactMarginalLogLikelihood), see include/pfn_b200.h for the contract.
//
// Per objective evaluation, everything in fp64 shared memory (A is t x t with an odd leading dimension):
//   build K (lower)  ->  Cholesky in place (lower, pivots in dg)  ->  L^-1 into the upper triangle (stored transposed)
//   ->  K^-1 = L^-T L^-1 into the strict lower triangle + dg  ->  alpha = K^-1 (y - mean)
//   ->  df = -(1/t) [ 1/2 sum_ij (alpha alpha^T - K^-1)_ij dK_ij + dlog-priors ],  dK recomputed from x (not stored).
// Every reduction has a fixed order, so a problem's result depends on its own inputs only (bitwise repeatable).
// The factorisation and the trace terms live in gp_posterior.cuh, shared with the NUTS sampler (gp_mcmc.cu); this file
// adds the softplus / raw-noise parameterisation, the 1/t scaling and the optimiser.
#include <math_constants.h>

#include "gp_posterior.cuh"

namespace pfn {
namespace {

using gp::FT;
using gp::FW;
using gp::LOG_2PI;
using gp::Problem;
using gp::log_gamma_pdf;
constexpr int FM = 10;                         // L-BFGS memory (scipy's maxcor default)
constexpr int FN = PFN_GP_FIT_MAX_F + 3;       // parameters: rho_1..F, rho_s, noise, mean
constexpr int LS_MAX = 20;                     // evaluations per line search (scipy's maxls)
constexpr double LS_FTOL = 1e-3, LS_GTOL = 0.9, LS_XTOL = 0.1;   // L-BFGS-B's dcsrch constants
constexpr double XTRAPL = 1.1, XTRAPU = 4.0, STP_BIG = 1e10;
constexpr double EPSMCH = 2.220446049250313e-16;

struct LineSearch {                            // More-Thuente (MINPACK-2 dcsrch) state
  double stp, stpmin, stpmax, finit, ginit, gtest, width, width1;
  double stx, fx, gx, sty, fy, gy, stmin, stmax;
  int brackt, stage, nfev;
};

struct FitState {
  double x[FN], g[FN], x0[FN], g0[FN], d[FN], trial[FN], alpha[FM];
  double S[FM][FN], Y[FM][FN];
  double f, dg0;
  int head, count, iter, nfev, status, mode, more;
  LineSearch ls;
};

struct Eval {                                  // derived parameters and results of one evaluation
  double inv_ls[PFN_GP_FIT_MAX_F], dls[PFN_GP_FIT_MAX_F], ls[PFN_GP_FIT_MAX_F];
  double s, ds, noise, c;
  double red[FW * 8];
  double f, g[FN];
  int pd;
};

enum { LS_FG = 0, LS_CONV = 1, LS_WARN = 2 };

__device__ __forceinline__ double softplus(double r) { return r > 20.0 ? r : log1p(exp(r)); }       // torch threshold 20
__device__ __forceinline__ double softplus_grad(double r) { return r > 20.0 ? 1.0 : 1.0 / (1.0 + exp(-r)); }

// f and grad at th (all threads).  Leaves alpha in al and K^-1 in (strict lower of A, dg) when the matrix is PD.
__device__ void evaluate(const Problem& P, const double* th, double* A, double* dg, double* yc, double* al, Eval& E) {
  const int tid = threadIdx.x;
  const int t = P.t, F = P.F;
  for (int d = tid; d < F; d += FT) {
    const double l = softplus(th[d]);
    E.ls[d] = l;
    E.inv_ls[d] = 1.0 / l;
    E.dls[d] = softplus_grad(th[d]);
  }
  if (tid == 0) {
    E.s = softplus(th[F]);
    E.ds = softplus_grad(th[F]);
    E.noise = th[F + 1];
    E.c = th[F + 2];
  }
  __syncthreads();
  const double s = E.s, noise = E.noise;
  double sums[6];                              // logdet/2, quad, sum alpha, sum W k, sum W_ii, -
  const int pd = gp::lml_terms(P, E.inv_ls, s, noise, E.c, A, dg, yc, al, E.red, sums, [&](int d, double v) {
    if (tid == 0) {
      const double il = E.inv_ls[d];
      const double dlogn = 0.5 * s * il * il * il * v;
      const double dprior = (P.ls_a - 1.0) * il - P.ls_b;
      E.g[d] = -(dlogn + dprior) * E.dls[d] / t;
    }
  });
  if (!pd) {
    if (tid == 0) { E.f = CUDART_INF; E.pd = 0; }
    __syncthreads();
    return;
  }
  if (tid == 0) {
    double logn = -0.5 * sums[1] - sums[0] - 0.5 * t * LOG_2PI;
    double prior = log_gamma_pdf(s, P.os_a, P.os_b) + log_gamma_pdf(noise, P.nz_a, P.nz_b);
    for (int d = 0; d < F; ++d) prior += log_gamma_pdf(E.ls[d], P.ls_a, P.ls_b);
    E.f = -(logn + prior) / t;
    E.g[F] = -(0.5 * sums[3] + (P.os_a - 1.0) / s - P.os_b) * E.ds / t;
    E.g[F + 1] = -(0.5 * sums[4] + (P.nz_a - 1.0) / noise - P.nz_b) / t;
    E.g[F + 2] = -sums[2] / t;
    E.pd = 1;
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------ line search
__device__ void dcstep(double& stx, double& fx, double& dx, double& sty, double& fy, double& dy, double& stp, double fp,
                       double dp, int& brackt, double stpmin, double stpmax) {
  const double sgnd = dp * (dx / fabs(dx));
  double stpf;
  if (fp > fx) {
    const double theta = 3.0 * (fx - fp) / (stp - stx) + dx + dp;
    const double s = fmax(fabs(theta), fmax(fabs(dx), fabs(dp)));
    double gamma = s * sqrt((theta / s) * (theta / s) - (dx / s) * (dp / s));
    if (stp < stx) gamma = -gamma;
    const double p = (gamma - dx) + theta, q = ((gamma - dx) + gamma) + dp, r = p / q;
    const double stpc = stx + r * (stp - stx);
    const double stpq = stx + ((dx / ((fx - fp) / (stp - stx) + dx)) / 2.0) * (stp - stx);
    stpf = fabs(stpc - stx) < fabs(stpq - stx) ? stpc : stpc + (stpq - stpc) / 2.0;
    brackt = 1;
  } else if (sgnd < 0.0) {
    const double theta = 3.0 * (fx - fp) / (stp - stx) + dx + dp;
    const double s = fmax(fabs(theta), fmax(fabs(dx), fabs(dp)));
    double gamma = s * sqrt((theta / s) * (theta / s) - (dx / s) * (dp / s));
    if (stp > stx) gamma = -gamma;
    const double p = (gamma - dp) + theta, q = ((gamma - dp) + gamma) + dx, r = p / q;
    const double stpc = stp + r * (stx - stp);
    const double stpq = stp + (dp / (dp - dx)) * (stx - stp);
    stpf = fabs(stpc - stp) > fabs(stpq - stp) ? stpc : stpq;
    brackt = 1;
  } else if (fabs(dp) < fabs(dx)) {
    const double theta = 3.0 * (fx - fp) / (stp - stx) + dx + dp;
    const double s = fmax(fabs(theta), fmax(fabs(dx), fabs(dp)));
    double gamma = s * sqrt(fmax(0.0, (theta / s) * (theta / s) - (dx / s) * (dp / s)));
    if (stp > stx) gamma = -gamma;
    const double p = (gamma - dp) + theta, q = (gamma + (dx - dp)) + gamma, r = p / q;
    double stpc;
    if (r < 0.0 && gamma != 0.0) stpc = stp + r * (stx - stp);
    else if (stp > stx) stpc = stpmax;
    else stpc = stpmin;
    const double stpq = stp + (dp / (dp - dx)) * (stx - stp);
    if (brackt) {
      stpf = fabs(stpc - stp) < fabs(stpq - stp) ? stpc : stpq;
      stpf = stp > stx ? fmin(stp + 0.66 * (sty - stp), stpf) : fmax(stp + 0.66 * (sty - stp), stpf);
    } else {
      stpf = fabs(stpc - stp) > fabs(stpq - stp) ? stpc : stpq;
      stpf = fmax(stpmin, fmin(stpmax, stpf));
    }
  } else {
    if (brackt) {
      const double theta = 3.0 * (fp - fy) / (sty - stp) + dy + dp;
      const double s = fmax(fabs(theta), fmax(fabs(dy), fabs(dp)));
      double gamma = s * sqrt((theta / s) * (theta / s) - (dy / s) * (dp / s));
      if (stp > sty) gamma = -gamma;
      const double p = (gamma - dp) + theta, q = ((gamma - dp) + gamma) + dy, r = p / q;
      stpf = stp + r * (sty - stp);
    } else {
      stpf = stp > stx ? stpmax : stpmin;
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

__device__ void ls_start(LineSearch& L, double f, double g, double stp, double stpmax) {
  L.stp = stp; L.stpmin = 0.0; L.stpmax = stpmax;
  L.brackt = 0; L.stage = 1; L.finit = f; L.ginit = g; L.gtest = LS_FTOL * g;
  L.width = stpmax; L.width1 = 2.0 * stpmax;
  L.stx = 0.0; L.fx = f; L.gx = g; L.sty = 0.0; L.fy = f; L.gy = g;
  L.stmin = 0.0; L.stmax = stp + XTRAPU * stp;
  L.nfev = 0;
}

// One dcsrch step after evaluating (f, g = f'(stp)): LS_FG with a new L.stp, or the step is accepted.
__device__ int ls_step(LineSearch& L, double f, double g) {
  const double ftest = L.finit + L.stp * L.gtest;
  if (L.stage == 1 && f <= ftest && g >= 0.0) L.stage = 2;
  if (L.brackt && (L.stp <= L.stmin || L.stp >= L.stmax)) return LS_WARN;
  if (L.brackt && L.stmax - L.stmin <= LS_XTOL * L.stmax) return LS_WARN;
  if (L.stp == L.stpmax && f <= ftest && g <= L.gtest) return LS_WARN;
  if (L.stp == L.stpmin && (f > ftest || g >= L.gtest)) return LS_WARN;
  if (f <= ftest && fabs(g) <= LS_GTOL * (-L.ginit)) return LS_CONV;
  if (L.stage == 1 && f <= L.fx && f > ftest) {
    const double fm = f - L.stp * L.gtest, gm = g - L.gtest;
    double fxm = L.fx - L.stx * L.gtest, fym = L.fy - L.sty * L.gtest;
    double gxm = L.gx - L.gtest, gym = L.gy - L.gtest;
    dcstep(L.stx, fxm, gxm, L.sty, fym, gym, L.stp, fm, gm, L.brackt, L.stmin, L.stmax);
    L.fx = fxm + L.stx * L.gtest; L.fy = fym + L.sty * L.gtest;
    L.gx = gxm + L.gtest; L.gy = gym + L.gtest;
  } else {
    dcstep(L.stx, L.fx, L.gx, L.sty, L.fy, L.gy, L.stp, f, g, L.brackt, L.stmin, L.stmax);
  }
  if (L.brackt) {
    if (fabs(L.sty - L.stx) >= 0.66 * L.width1) L.stp = L.stx + 0.5 * (L.sty - L.stx);
    L.width1 = L.width;
    L.width = fabs(L.sty - L.stx);
    L.stmin = fmin(L.stx, L.sty);
    L.stmax = fmax(L.stx, L.sty);
  } else {
    L.stmin = L.stp + XTRAPL * (L.stp - L.stx);
    L.stmax = L.stp + XTRAPU * (L.stp - L.stx);
  }
  L.stp = fmin(fmax(L.stp, L.stpmin), L.stpmax);
  if (L.brackt && (L.stp <= L.stmin || L.stp >= L.stmax || L.stmax - L.stmin <= LS_XTOL * L.stmax)) L.stp = L.stx;
  return LS_FG;
}

// ------------------------------------------------------------------------------------------------ L-BFGS (thread 0)
struct Opt {
  int n, ks;                                   // parameter count, index of the noise
  double lb, ftol, gtol;
  int max_iter, max_eval;
};

__device__ double proj_grad_norm(const Opt& O, const double* x, const double* g) {
  double m = 0.0;
  for (int i = 0; i < O.n; ++i) {
    double gi = g[i];
    if (i == O.ks && gi > 0.0) gi = fmin(x[i] - O.lb, gi);
    m = fmax(m, fabs(gi));
  }
  return m;
}

__device__ __forceinline__ double dotm(const double* a, const double* b, int n, int skip) {
  double v = 0.0;
  for (int i = 0; i < n; ++i)
    if (i != skip) v = fma(a[i], b[i], v);
  return v;
}

// Search direction from the current point (two-loop recursion over the free coordinates; the noise is fixed while it
// sits on its bound with a gradient pushing it down), step bounds, first trial point.  Returns 0 when no descent is left.
__device__ int start_iteration(const Opt& O, FitState& S) {
  const int n = O.n, ks = O.ks;
  const int fix = (S.x[ks] <= O.lb && S.g[ks] > 0.0) ? ks : -1;
  for (int attempt = 0; attempt < 2; ++attempt) {
    for (int i = 0; i < n; ++i) S.d[i] = (i == fix) ? 0.0 : S.g[i];
    double gamma = 1.0;
    for (int k = 0; k < S.count; ++k) {
      const int idx = (S.head - 1 - k + FM) % FM;
      const double sy = dotm(S.S[idx], S.Y[idx], n, fix);
      S.alpha[idx] = 0.0;
      if (!(sy > 0.0)) continue;
      const double a = dotm(S.S[idx], S.d, n, fix) / sy;
      S.alpha[idx] = a;
      for (int i = 0; i < n; ++i)
        if (i != fix) S.d[i] = fma(-a, S.Y[idx][i], S.d[i]);
      if (k == 0) gamma = sy / dotm(S.Y[idx], S.Y[idx], n, fix);
    }
    for (int i = 0; i < n; ++i) S.d[i] *= gamma;
    for (int k = S.count - 1; k >= 0; --k) {
      const int idx = (S.head - 1 - k + FM) % FM;
      const double sy = dotm(S.S[idx], S.Y[idx], n, fix);
      if (!(sy > 0.0)) continue;
      const double b = dotm(S.Y[idx], S.d, n, fix) / sy;
      for (int i = 0; i < n; ++i)
        if (i != fix) S.d[i] = fma(S.alpha[idx] - b, S.S[idx][i], S.d[i]);
    }
    for (int i = 0; i < n; ++i) S.d[i] = -S.d[i];
    if (S.x[ks] <= O.lb && S.d[ks] < 0.0) S.d[ks] = 0.0;
    S.dg0 = dotm(S.g, S.d, n, -1);
    if (S.dg0 < 0.0) break;
    if (S.count == 0) return 0;
    S.count = 0;                               // not a descent direction: drop the memory, steepest descent
  }
  if (!(S.dg0 < 0.0)) return 0;
  double dnorm = sqrt(dotm(S.d, S.d, n, -1));
  double stpmax = S.iter == 0 ? 1.0 : STP_BIG;
  if (S.d[ks] < 0.0) stpmax = fmin(stpmax, (S.x[ks] - O.lb) / (-S.d[ks]));
  const double stp = S.iter == 0 ? fmin(1.0 / dnorm, stpmax) : fmin(1.0, stpmax);
  if (!(stp > 0.0)) return 0;
  for (int i = 0; i < n; ++i) { S.x0[i] = S.x[i]; S.g0[i] = S.g[i]; }
  ls_start(S.ls, S.f, S.dg0, stp, stpmax);
  for (int i = 0; i < n; ++i) S.trial[i] = fma(stp, S.d[i], S.x0[i]);
  S.trial[ks] = fmax(S.trial[ks], O.lb);
  return 1;
}

// After an evaluation at S.trial: returns 1 when S.trial holds the next point to evaluate, 0 when the fit is over.
__device__ int opt_step(const Opt& O, FitState& S, const Eval& E) {
  const int n = O.n;
  S.nfev++;
  if (S.mode == 0) {                           // the starting point
    for (int i = 0; i < n; ++i) { S.x[i] = S.trial[i]; S.g[i] = E.g[i]; }
    S.f = E.f;
    if (!E.pd || !isfinite(E.f)) { S.status = PFN_GP_FIT_NOT_PD; return 0; }
    if (proj_grad_norm(O, S.x, S.g) <= O.gtol) { S.status = PFN_GP_FIT_CONVERGED; return 0; }
    if (S.iter >= O.max_iter || S.nfev >= O.max_eval) { S.status = PFN_GP_FIT_MAX_ITER; return 0; }
    S.mode = 1;
    if (!start_iteration(O, S)) { S.status = PFN_GP_FIT_CONVERGED; return 0; }
    return 1;
  }
  S.ls.nfev++;
  int task;
  if (!E.pd || !isfinite(E.f)) {
    // a trial point whose matrix is not PD counts as f = +inf: step back toward the best point of the search
    const double bad = S.ls.stp;
    S.ls.stpmax = bad;
    S.ls.stmax = fmin(S.ls.stmax, bad);
    S.ls.stp = S.ls.stx + 0.5 * (bad - S.ls.stx);
    task = LS_FG;
  } else {
    task = ls_step(S.ls, E.f, dotm(E.g, S.d, n, -1));
  }
  if (task == LS_FG) {
    if (S.nfev >= O.max_eval) { S.status = PFN_GP_FIT_MAX_ITER; return 0; }
    if (S.ls.nfev >= LS_MAX || !(S.ls.stp > 0.0)) {           // line-search failure: S.x is still the last iterate
      if (S.count == 0) { S.status = PFN_GP_FIT_LINE_SEARCH; return 0; }
      S.count = 0;
      if (!start_iteration(O, S)) { S.status = PFN_GP_FIT_LINE_SEARCH; return 0; }
      return 1;
    }
    for (int i = 0; i < n; ++i) S.trial[i] = fma(S.ls.stp, S.d[i], S.x0[i]);
    S.trial[O.ks] = fmax(S.trial[O.ks], O.lb);
    return 1;
  }
  // accepted (dcsrch convergence or warning, as in L-BFGS-B)
  S.iter++;
  const double f_old = S.f;
  for (int i = 0; i < n; ++i) {
    S.x0[i] = S.trial[i] - S.x0[i];            // s
    S.g0[i] = E.g[i] - S.g0[i];                // y
    S.x[i] = S.trial[i];
    S.g[i] = E.g[i];
  }
  S.f = E.f;
  if (proj_grad_norm(O, S.x, S.g) <= O.gtol) { S.status = PFN_GP_FIT_CONVERGED; return 0; }
  if (f_old - S.f <= O.ftol * fmax(fmax(fabs(f_old), fabs(S.f)), 1.0)) { S.status = PFN_GP_FIT_CONVERGED; return 0; }
  const double sy = dotm(S.x0, S.g0, n, -1);
  if (sy > EPSMCH * S.ls.stp * (-S.dg0)) {
    for (int i = 0; i < n; ++i) { S.S[S.head][i] = S.x0[i]; S.Y[S.head][i] = S.g0[i]; }
    S.head = (S.head + 1) % FM;
    S.count = min(S.count + 1, FM);
  }
  if (S.iter >= O.max_iter || S.nfev >= O.max_eval) { S.status = PFN_GP_FIT_MAX_ITER; return 0; }
  if (!start_iteration(O, S)) { S.status = PFN_GP_FIT_CONVERGED; return 0; }
  return 1;
}

__global__ void __launch_bounds__(FT, 1) gp_fit_kernel(const gp::PrefixArgs<pfn_gp_fit_desc> args) {
  const pfn_gp_fit_desc& D = args.d;
  extern __shared__ __align__(16) double fit_dyn[];
  __shared__ FitState S;
  __shared__ Eval E;
  const int tid = threadIdx.x;
  const int slot = blockIdx.x / D.B, b = blockIdx.x % D.B;
  const int t = args.slot_t[slot], ti = args.slot_i[slot];
  const long long p = static_cast<long long>(ti) * D.B + b;
  const int F = D.F, n = F + 3;
  const int ld = t | 1;                        // odd: the column walks of the sweeps hit distinct banks
  const int tmax = args.slot_t[0];
  double* A = fit_dyn;                                   // [t, ld]
  double* xs = A + static_cast<size_t>(tmax) * (tmax | 1);   // [t, F]
  double* ys = xs + static_cast<size_t>(tmax) * F;       // [t]
  double* dg = ys + tmax;
  double* yc = dg + tmax;
  double* al = yc + tmax;
  double* ks = al + tmax;                                // [t] and x* [F]
  double* xstar = ks + tmax;

  const float* xb = D.x + static_cast<size_t>(b) * D.T * F;
  const float* yb = D.y + static_cast<size_t>(b) * D.T;
  for (int i = tid; i < t * F; i += FT) xs[i] = static_cast<double>(xb[i]);
  for (int i = tid; i < t; i += FT) ys[i] = static_cast<double>(yb[i]);
  const bool predict_row = t < D.T;
  if (predict_row)
    for (int i = tid; i < F; i += FT) xstar[i] = static_cast<double>(xb[static_cast<size_t>(t) * F + i]);
  if (tid == 0) {
    for (int i = 0; i < n; ++i) {
      double v;
      if (D.theta0) v = D.theta0[p * n + i];
      else v = i == F + 1 ? D.noise_init : 0.0;
      S.trial[i] = v;
    }
    S.head = S.count = S.iter = S.nfev = S.mode = 0;
    S.status = PFN_GP_FIT_CONVERGED;
  }
  __syncthreads();

  const Problem P{xs, ys, t, F, ld, D.kernel_type, D.ls_conc, D.ls_rate, D.os_conc, D.os_rate, D.noise_conc, D.noise_rate};
  const Opt O{n, F + 1, D.noise_lb, D.ftol, D.gtol, D.max_iter, D.max_eval};
  for (;;) {
    evaluate(P, S.trial, A, dg, yc, al, E);
    if (D.max_iter <= 0) break;
    if (tid == 0) S.more = opt_step(O, S, E);
    __syncthreads();
    if (!S.more) break;
  }
  if (D.max_iter <= 0) {
    if (tid == 0) {
      for (int i = 0; i < n; ++i) S.x[i] = S.trial[i];
      S.status = E.pd ? PFN_GP_FIT_CONVERGED : PFN_GP_FIT_NOT_PD;
      S.nfev = 1;
    }
    __syncthreads();
  } else if (S.status != PFN_GP_FIT_NOT_PD) {
    evaluate(P, S.x, A, dg, yc, al, E);       // alpha and K^-1 of the returned point (also its f and gradient)
  }
  double mean = CUDART_NAN, var = CUDART_NAN;
  if (predict_row && E.pd) gp::predict(P, E.inv_ls, E.s, E.c, xstar, A, dg, al, ks, E.red, mean, var);
  if (tid == 0) {
    for (int i = 0; i < n; ++i) {
      D.theta[p * n + i] = S.x[i];
      if (D.grad) D.grad[p * n + i] = E.pd ? E.g[i] : CUDART_NAN;
    }
    D.f[p] = E.pd ? E.f : CUDART_INF;
    if (D.mean) D.mean[p] = mean;
    if (D.var) D.var[p] = var;
    D.iters[p] = S.iter;
    D.nevals[p] = S.nfev;
    D.status[p] = S.status;
  }
}

}  // namespace
}  // namespace pfn

using namespace pfn;

extern "C" int pfn_gp_fit(const pfn_gp_fit_desc* d, void* stream) {
  gp::PrefixArgs<pfn_gp_fit_desc> a;
  if (const int rc = gp::check_prefix_problems(d, "gp_fit", a)) return rc;
  PFN_CHECK_ARG(d->x && d->y && d->theta && d->f && d->iters && d->nevals && d->status, "gp_fit: null input or output pointer");
  PFN_CHECK_ARG(d->noise_lb > 0.0, "gp_fit: noise_lb must be positive");
  PFN_CHECK_ARG(d->theta0 != nullptr || d->noise_init >= d->noise_lb, "gp_fit: noise_init %g below the bound %g",
                d->noise_init, d->noise_lb);
  const size_t smem = gp::problem_smem(a.slot_t[0], d->F);
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set))
    PFN_CUDA_OK(cudaFuncSetAttribute(gp_fit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     static_cast<int>(gp::problem_smem(PFN_GP_FIT_MAX_T, PFN_GP_FIT_MAX_F))));
  gp_fit_kernel<<<d->B * d->n_ts, FT, smem, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  PFN_LAUNCH_OK();
  return 0;
}
