// Fully Bayesian GP baseline: one CTA per (prefix t, dataset) problem runs a whole NUTS chain over the hyperparameters
// u = log(ls_1..F, s, noise) of the Gamma-prior Matern-ARD GP, then forms the predictive of row t under every kept
// sample.  No host loop, no per-iteration launch.  Restates reference priors/fast_gp_mix.py:171-268 (pyro NUTS with
// adapt_step_size=True, everything else at pyro 1.7's defaults) targeting the posterior p(u | y[:t]); see
// include/pfn_b200.h for the contract and oracle/gp_mcmc_oracle.py (nuts_chain) for the sampler written out on the CPU.
//
// Every potential evaluation is the fit's fp64 shared-memory factorisation (gp_posterior.cuh), run by all threads; the
// tree logic (leapfrog updates, multinomial selection, U-turn tests, adaptation) runs on thread 0 between evaluations.
// The tree is built iteratively: the complete subtrees of the doubling in progress sit on a stack indexed by level and
// merge like a binary counter, so a subtree stops at its first turning or divergent node exactly as pyro's recursion does.
// This file is compiled with -fmad=false: the sampler's arithmetic is then the plain IEEE sequence the CPU restatement
// performs (the potential itself uses explicit fma() and is unaffected).
#include <math_constants.h>

#include "counter_rng.cuh"
#include "gp_posterior.cuh"

namespace pfn {
namespace {

using gp::FT;
using gp::FW;
using gp::Problem;

constexpr int MAXF = PFN_GP_FIT_MAX_F;
constexpr int DM = PFN_GP_FIT_MAX_F + 2;       // sampled coordinates: log ls_1..F, log s, log noise
constexpr int MAXD = PFN_GP_MCMC_MAX_DEPTH;
constexpr int MAX_WINDOWS = 40;
constexpr double TARGET_ACCEPT = 0.8;          // dual averaging (pyro.ops.dual_averaging, Stan's constants)
constexpr double DA_GAMMA = 0.05, DA_T0 = 10.0, DA_KAPPA = 0.75;
constexpr double MAX_ENERGY_ERROR = 1000.0;    // pyro NUTS _max_sliced_energy
constexpr double LOG_ACCEPT_THRESHOLD = -0.2231435513142097;    // log(0.8), the step-size search's direction threshold
constexpr int SEARCH_MAX = 100;                // doublings / halvings per step-size search (pyro has no cap)
constexpr int INIT_TRIES = 100;                // uniform initial points tried until the potential is finite (pyro's)
constexpr double TWO_PI = 6.283185307179586;

struct Node {                                  // a complete subtree of the doubling in progress
  double w_first[DM], w_last[DM], w_sum[DM];   // whitened momenta M^-1/2 r of its first / last leaf, and their sum
  double z[DM], g[DM], pe;                     // its multinomial proposal
  double weight;                               // log sum of exp(-energy error) over its leaves
};

struct Nuts {
  double z[DM], g[DM], pe;                     // the chain's state with its potential and gradient
  double inv_m[DM], sqrt_im[DM], rsqrt_im[DM];
  double ez[2][DM], er[2][DM], eg[2][DM], ew[2][DM];   // trajectory ends: 0 = left, 1 = right
  double w_sum[DM], weight, energy0;
  double trial[DM], rhalf[DM];                 // the point being evaluated and its half-step momentum
  Node stack[MAXD + 1];
  Node cur;
  double acc_sum, sub_acc, acc_sampling;
  int n_prop, sub_n;
  double eps, da_center, da_x, da_xavg, da_gavg;
  int da_t;
  double wf_mean[DM], wf_m2[DM];
  int wf_n;
  int win_end[MAX_WINDOWS], nwin, cw;
  double s_energy0, s_scale;
  int s_dir, s_count, s_first;
  int d, it, depth, dir, leaf;
  uint32_t seed, key_b, key_t, key_it, ctr;
  int diag[PFN_GP_MCMC_NDIAG];
};

struct MEval {
  double ls[MAXF], inv_ls[MAXF];
  double s, noise;
  double red[FW * 8];
  double U, g[DM];
  int pd;
};

// ------------------------------------------------------------------------------------------------ random numbers (thread 0)
// Draw k of iteration key `it` is uniform_double(hash5(seed, b, t, it, 2k), hash5(.., 2k + 1)).
__device__ double uniform(Nuts& N) {
  const uint32_t hi = hash5(N.seed, N.key_b, N.key_t, N.key_it, 2u * N.ctr);
  const uint32_t lo = hash5(N.seed, N.key_b, N.key_t, N.key_it, 2u * N.ctr + 1u);
  N.ctr++;
  return uniform_double(hi, lo);
}
// Box-Muller, cosine branch; 1 - U is in (0, 1]
__device__ double normal(Nuts& N) {
  const double u1 = 1.0 - uniform(N);
  const double u2 = uniform(N);
  return sqrt(-2.0 * log(u1)) * cos(TWO_PI * u2);
}

// ------------------------------------------------------------------------------------------------ potential (all threads)
__device__ __forceinline__ double log_gamma_u(double u, double theta, double a, double b) {
  return a * log(b) - lgamma(a) + a * u - b * theta;    // log Gamma(e^u; a, b) + u
}

__device__ void potential(const Problem& P, const double* u, double* A, double* dg, double* yc, double* al, MEval& E,
                          int* diag) {
  const int tid = threadIdx.x, t = P.t, F = P.F;
  for (int d = tid; d < F; d += FT) {
    const double l = exp(u[d]);
    E.ls[d] = l;
    E.inv_ls[d] = 1.0 / l;
  }
  if (tid == 0) {
    E.s = exp(u[F]);
    E.noise = exp(u[F + 1]);
  }
  __syncthreads();
  const double s = E.s, noise = E.noise;
  double sums[6];
  const int pd = gp::lml_terms(P, E.inv_ls, s, noise, 0.0, A, dg, yc, al, E.red, sums, [&](int d, double v) {
    if (tid == 0) {
      const double il = E.inv_ls[d];
      E.g[d] = -(0.5 * s * il * il * v) - P.ls_a + P.ls_b * E.ls[d];
    }
  });
  if (tid == 0) {
    diag[PFN_GP_MCMC_EVALS]++;
    if (pd) {
      const double logn = -0.5 * sums[1] - sums[0] - 0.5 * t * gp::LOG_2PI;
      double lp = log_gamma_u(u[F], s, P.os_a, P.os_b) + log_gamma_u(u[F + 1], noise, P.nz_a, P.nz_b);
      for (int d = 0; d < F; ++d) lp += log_gamma_u(u[d], E.ls[d], P.ls_a, P.ls_b);
      const double U = -(logn + lp);
      E.U = U < CUDART_INF ? U : CUDART_INF;   // NaN counts as +inf
      E.g[F] = -(0.5 * s * sums[3]) - P.os_a + P.os_b * s;
      E.g[F + 1] = -(0.5 * noise * sums[4]) - P.nz_a + P.nz_b * noise;
    } else {
      E.U = CUDART_INF;
      for (int k = 0; k < F + 2; ++k) E.g[k] = 0.0;
      diag[PFN_GP_MCMC_NOT_PD]++;
    }
    E.pd = pd;
  }
  __syncthreads();
}

// Parameters and factorisation only, for the predictive (all threads): 1 when K is PD.
__device__ int factor_at(const Problem& P, const double* u, double* A, double* dg, double* yc, double* al, MEval& E,
                         int* diag) {
  const int tid = threadIdx.x, F = P.F;
  for (int d = tid; d < F; d += FT) {
    const double l = exp(u[d]);
    E.ls[d] = l;
    E.inv_ls[d] = 1.0 / l;
  }
  if (tid == 0) {
    E.s = exp(u[F]);
    E.noise = exp(u[F + 1]);
    diag[PFN_GP_MCMC_EVALS]++;
  }
  __syncthreads();
  double log_dg;
  return gp::factor(P, E.inv_ls, E.s, E.noise, 0.0, A, dg, yc, al, log_dg);
}

// ------------------------------------------------------------------------------------------------ NUTS (thread 0)
__device__ double logaddexp(double x, double y) {                 // pyro's _logaddexp
  const double mn = x < y ? x : y, mx = x < y ? y : x;
  return log1p(exp(mn - mx)) + mx;
}

__device__ double kinetic(const double* w, int d) {
  double e = 0.0;
  for (int i = 0; i < d; ++i) e = e + w[i] * w[i];
  return 0.5 * e;
}

// generalised no-U-turn criterion in whitened momenta (pyro NUTS._is_turning)
__device__ int is_turning(const double* wl, const double* wr, const double* wsum, int d) {
  double left = 0.0, right = 0.0;
  for (int i = 0; i < d; ++i) {
    const double rho = wsum[i] - (wl[i] + wr[i]) / 2.0;
    left = left + wl[i] * rho;
    right = right + wr[i] * rho;
  }
  return left <= 0.0 || right <= 0.0;
}

__device__ void set_inv_mass(Nuts& N, int i, double v) {
  N.inv_m[i] = v;
  N.sqrt_im[i] = sqrt(v);
  N.rsqrt_im[i] = 1.0 / sqrt(v);
}

// momentum draw: whitened w ~ N(0, I) into wout, r = M^1/2 w into rout; returns the kinetic energy
__device__ double draw_momentum(Nuts& N, double* rout, double* wout) {
  for (int i = 0; i < N.d; ++i) {
    const double w = normal(N);
    wout[i] = w;
    rout[i] = w * N.rsqrt_im[i];
  }
  return kinetic(wout, N.d);
}

// first half of a leapfrog step from (z, r, g) with signed step e: rhalf and the trial position
__device__ void leapfrog_begin(Nuts& N, const double* z, const double* r, const double* g, double e) {
  const double h = 0.5 * e;
  for (int i = 0; i < N.d; ++i) {
    N.rhalf[i] = r[i] + h * (-g[i]);
    N.trial[i] = z[i] + e * (N.inv_m[i] * N.rhalf[i]);
  }
}

// second half at the evaluated trial point: momentum r and whitened w; returns the total energy (+inf for NaN)
__device__ double leapfrog_end(Nuts& N, const MEval& E, double e, double* r, double* w) {
  const double h = 0.5 * e;
  for (int i = 0; i < N.d; ++i) {
    r[i] = N.rhalf[i] + h * (-E.g[i]);
    w[i] = r[i] * N.sqrt_im[i];
  }
  const double en = E.U + kinetic(w, N.d);
  return en == en ? en : CUDART_INF;
}

__device__ void copy(double* dst, const double* src, int d) {
  for (int i = 0; i < d; ++i) dst[i] = src[i];
}

__device__ void da_reset(Nuts& N) {
  N.da_center = log(10.0 * N.eps);
  N.da_xavg = 0.0;
  N.da_gavg = 0.0;
  N.da_t = 0;
}

__device__ void da_step(Nuts& N, double g) {
  N.da_t++;
  const double tt = N.da_t + DA_T0;
  N.da_gavg = (1.0 - 1.0 / tt) * N.da_gavg + g / tt;
  N.da_x = N.da_center - sqrt(static_cast<double>(N.da_t)) / DA_GAMMA * N.da_gavg;
  const double wt = pow(static_cast<double>(N.da_t), -DA_KAPPA);
  N.da_xavg = (1.0 - wt) * N.da_xavg + wt * N.da_x;
}

// Stan's windows as pyro builds them (adaptation.WarmupAdapter._build_adaptation_schedule): end index of every window
__device__ void build_schedule(Nuts& N, int W) {
  N.nwin = 0;
  N.cw = 0;
  if (W < 20) {
    N.win_end[N.nwin++] = W - 1;
    return;
  }
  int start_buf = 75, end_buf = 50, init_win = 25;
  if (start_buf + end_buf + init_win > W) {
    start_buf = static_cast<int>(0.15 * W);
    end_buf = static_cast<int>(0.1 * W);
    init_win = W - start_buf - end_buf;
  }
  N.win_end[N.nwin++] = start_buf - 1;
  const int end_start = W - end_buf;
  int next_size = init_win, next_start = start_buf;
  while (next_start < end_start && N.nwin < MAX_WINDOWS - 1) {
    const int cur_start = next_start;
    int cur_size = next_size;
    if (3 * cur_size <= end_start - cur_start) next_size = 2 * cur_size;
    else cur_size = end_start - cur_start;
    next_start = cur_start + cur_size;
    N.win_end[N.nwin++] = next_start - 1;
  }
  N.win_end[N.nwin++] = W - 1;
}

// ---- step-size search (pyro HMC._find_reasonable_step_size) from the current state
__device__ void search_trial_begin(Nuts& N) {
  if (!N.s_first) N.eps = N.s_scale * N.eps;
  double* r = N.er[0];                         // scratch: the trajectory ends are free between iterations
  double* w = N.ew[0];
  N.s_energy0 = draw_momentum(N, r, w) + N.pe;
  leapfrog_begin(N, N.z, r, N.g, N.eps);
}

__device__ int search_trial_end(Nuts& N, const MEval& E) {
  const double en = leapfrog_end(N, E, N.eps, N.er[1], N.ew[1]);
  const double delta = en - N.s_energy0;
  const int dir = LOG_ACCEPT_THRESHOLD < -delta ? 1 : -1;
  if (N.s_first) {
    N.s_first = 0;
    N.s_dir = dir;
    N.s_scale = dir == 1 ? 2.0 : 0.5;
    return 1;
  }
  if (dir != N.s_dir) return 0;
  return ++N.s_count < SEARCH_MAX;
}

// ---- one NUTS iteration
__device__ void iteration_begin(Nuts& N) {
  N.key_it = static_cast<uint32_t>(N.it) + 1u;
  N.ctr = 0;
  N.energy0 = draw_momentum(N, N.er[0], N.ew[0]) + N.pe;
  copy(N.er[1], N.er[0], N.d);
  copy(N.ew[1], N.ew[0], N.d);
  for (int s = 0; s < 2; ++s) {
    copy(N.ez[s], N.z, N.d);
    copy(N.eg[s], N.g, N.d);
  }
  copy(N.w_sum, N.ew[0], N.d);
  N.weight = 0.0;
  N.acc_sum = 0.0;
  N.n_prop = 0;
  N.depth = 0;
}

__device__ void subtree_begin(Nuts& N) {
  N.dir = uniform(N) < 0.5 ? 1 : 0;
  N.leaf = 0;
  N.sub_acc = 0.0;
  N.sub_n = 0;
  const int s = N.dir;
  leapfrog_begin(N, N.ez[s], N.er[s], N.eg[s], s ? N.eps : -N.eps);
}

// After the evaluation of a leaf: 0 = next leaf prepared, 1 = subtree complete, 2 = turning, 3 = divergent.
__device__ int leaf_end(Nuts& N, const MEval& E) {
  const int s = N.dir, d = N.d;
  const double e = s ? N.eps : -N.eps;
  N.diag[PFN_GP_MCMC_LEAPFROG]++;
  const double en = leapfrog_end(N, E, e, N.er[s], N.ew[s]);
  copy(N.ez[s], N.trial, d);
  copy(N.eg[s], E.g, d);
  const double sliced = en + (-N.energy0);
  const double delta = en - N.energy0;
  const double acc = exp(-delta);
  N.sub_acc = N.sub_acc + (acc < 1.0 ? acc : 1.0);
  N.sub_n++;
  if (sliced > MAX_ENERGY_ERROR) return 3;
  Node& C = N.cur;
  copy(C.w_first, N.ew[s], d);
  copy(C.w_last, N.ew[s], d);
  copy(C.w_sum, N.ew[s], d);
  copy(C.z, N.trial, d);
  copy(C.g, E.g, d);
  C.pe = E.U;
  C.weight = -sliced;
  int lvl = 0;
  for (; (N.leaf >> lvl) & 1; ++lvl) {         // merge with the earlier subtree of the same size (first half)
    const Node& H = N.stack[lvl];
    const double w = logaddexp(H.weight, C.weight);
    const double p_other = exp(C.weight - w);
    if (!(uniform(N) < p_other)) {
      copy(C.z, H.z, d);
      copy(C.g, H.g, d);
      C.pe = H.pe;
    }
    C.weight = w;
    for (int i = 0; i < d; ++i) C.w_sum[i] = H.w_sum[i] + C.w_sum[i];
    copy(C.w_first, H.w_first, d);
    if (is_turning(C.w_first, C.w_last, C.w_sum, d)) return 2;
  }
  if (++N.leaf == (1 << N.depth)) return 1;
  N.stack[lvl] = C;
  leapfrog_begin(N, N.ez[s], N.er[s], N.eg[s], e);
  return 0;
}

// After a subtree: 1 when the iteration's trajectory is complete.
__device__ int subtree_end(Nuts& N, int status, int max_depth, int W) {
  const int d = N.d;
  N.acc_sum = N.acc_sum + N.sub_acc;
  N.n_prop += N.sub_n;
  if (status == 3) {
    N.diag[N.it < W ? PFN_GP_MCMC_DIV_WARMUP : PFN_GP_MCMC_DIV_SAMPLING]++;
    return 1;
  }
  if (status == 2) return 1;
  N.depth++;
  const Node& C = N.cur;
  const double p_new = exp(C.weight - N.weight);
  if (uniform(N) < p_new) {                    // biased progressive sampling
    copy(N.z, C.z, d);
    copy(N.g, C.g, d);
    N.pe = C.pe;
  }
  for (int i = 0; i < d; ++i) N.w_sum[i] = N.w_sum[i] + C.w_sum[i];
  if (is_turning(N.ew[0], N.ew[1], N.w_sum, d)) return 1;
  N.weight = logaddexp(N.weight, C.weight);
  if (N.depth >= max_depth) {
    N.diag[PFN_GP_MCMC_MAX_DEPTH_HITS]++;
    return 1;
  }
  return 0;
}

// Warmup adaptation after iteration it (pyro WarmupAdapter.step at t = it + 1).  Returns 1 when a step-size search follows.
__device__ int adapt(Nuts& N, double accept_prob, int W) {
  const int t = N.it + 1;
  if (t >= W) return 0;
  const int mm = N.cw > 0 && N.cw < N.nwin - 1;
  da_step(N, TARGET_ACCEPT - accept_prob);
  N.eps = exp(N.da_x);
  if (mm) {
    N.wf_n++;
    for (int i = 0; i < N.d; ++i) {
      const double pre = N.z[i] - N.wf_mean[i];
      N.wf_mean[i] = N.wf_mean[i] + pre / N.wf_n;
      const double post = N.z[i] - N.wf_mean[i];
      N.wf_m2[i] = N.wf_m2[i] + pre * post;
    }
  }
  if (t != N.win_end[N.cw]) return 0;
  if (N.cw == N.nwin - 1) {
    N.cw++;
    N.eps = exp(N.da_xavg);
    return 0;
  }
  if (N.cw == 0) {
    N.cw++;
    return 0;
  }
  const double n = N.wf_n;
  for (int i = 0; i < N.d; ++i) {
    const double cov = N.wf_m2[i] / (n - 1.0);
    set_inv_mass(N, i, (n / (n + 5.0)) * cov + 1e-3 * (5.0 / (n + 5.0)));
    N.wf_mean[i] = 0.0;
    N.wf_m2[i] = 0.0;
  }
  N.wf_n = 0;
  N.cw++;
  return 1;
}

// rows of x a problem keeps in shared memory: its t rows and the predictive rows after them
__host__ __device__ __forceinline__ int mcmc_x_rows(int t, int T, int n_pred) { return min(T, t + n_pred); }

// A [tmax, tmax|1], x [rows, F], y, dg, yc, al, ks [tmax]; never above gp::problem_smem(T, F) since rows <= T
inline size_t mcmc_smem(int tmax, int T, int F, int n_pred) {
  return (static_cast<size_t>(tmax) * (tmax | 1) + static_cast<size_t>(mcmc_x_rows(tmax, T, n_pred)) * F + 5 * tmax) *
         sizeof(double);
}

struct McmcArgs {
  pfn_gp_mcmc_desc d;
  int slot_t[PFN_GP_FIT_MAX_T];                // prefix lengths, largest first
  int slot_i[PFN_GP_FIT_MAX_T];                // their index in d.ts
};

// Step-size search from the chain's state (all threads), then a fresh dual-averaging centre.  Thread 0's decisions reach
// the other threads through __syncthreads_or, never through shared memory that thread 0 may rewrite before they read it.
__device__ void step_size_search(const Problem& P, Nuts& N, MEval& E, double* A, double* dg, double* yc, double* al) {
  const int tid = threadIdx.x;
  if (tid == 0) {
    N.s_first = 1;
    N.s_count = 0;
    search_trial_begin(N);
  }
  __syncthreads();
  for (;;) {
    potential(P, N.trial, A, dg, yc, al, E, N.diag);
    int more = 0;
    if (tid == 0) {
      more = search_trial_end(N, E);
      if (more) search_trial_begin(N);
      else da_reset(N);
    }
    if (!__syncthreads_or(more)) break;
  }
}

__global__ void __launch_bounds__(FT, 1) gp_mcmc_kernel(const McmcArgs args) {
  const pfn_gp_mcmc_desc& D = args.d;
  extern __shared__ __align__(16) double mcmc_dyn[];
  __shared__ Nuts N;
  __shared__ MEval E;
  const int tid = threadIdx.x;
  const int slot = blockIdx.x / D.B, b = blockIdx.x % D.B;
  const int t = args.slot_t[slot], ti = args.slot_i[slot];
  const long long p = static_cast<long long>(ti) * D.B + b;
  const int F = D.F, d = F + 2;
  const int W = D.warmup_steps, S = D.num_samples, So = S > 0 ? S : 1;
  const int ld = t | 1;
  const int tmax = args.slot_t[0];
  double* A = mcmc_dyn;
  double* xs = A + static_cast<size_t>(tmax) * (tmax | 1);   // rows 0 .. min(T, t + n_pred) - 1: the data, then x*
  double* ys = xs + static_cast<size_t>(mcmc_x_rows(tmax, D.T, D.n_pred)) * F;
  double* dg = ys + tmax;
  double* yc = dg + tmax;
  double* al = yc + tmax;
  double* ks = al + tmax;

  const float* xb = D.x + static_cast<size_t>(b) * D.T * F;
  const float* yb = D.y + static_cast<size_t>(b) * D.T;
  for (int i = tid; i < mcmc_x_rows(t, D.T, D.n_pred) * F; i += FT) xs[i] = static_cast<double>(xb[i]);
  for (int i = tid; i < t; i += FT) ys[i] = static_cast<double>(yb[i]);
  const bool predict_row = t < D.T;
  if (tid == 0) {
    N.d = d;
    N.seed = D.seed;
    N.key_b = static_cast<uint32_t>(b);
    N.key_t = static_cast<uint32_t>(t);
    N.key_it = 0;
    N.ctr = 0;
    for (int k = 0; k < PFN_GP_MCMC_NDIAG; ++k) N.diag[k] = 0;
    for (int i = 0; i < d; ++i) {
      set_inv_mass(N, i, 1.0);
      N.wf_mean[i] = N.wf_m2[i] = 0.0;
    }
    N.wf_n = 0;
    N.eps = 1.0;
    N.acc_sampling = 0.0;
    build_schedule(N, W);
  }
  __syncthreads();
  const Problem P{xs, ys, t, F, ld, D.kernel_type, D.ls_conc, D.ls_rate, D.os_conc, D.os_rate, D.noise_conc, D.noise_rate};
  double* out_u = D.samples + p * So * d;      // u of every kept sample; turned into theta at the end

  // ---- initial point: the caller's, or u ~ U(-2, 2) until the potential is finite
  int finite = 0;
  for (int attempt = 0;; ++attempt) {
    if (tid == 0)
      for (int i = 0; i < d; ++i) N.trial[i] = D.init ? D.init[p * d + i] : -2.0 + 4.0 * uniform(N);
    __syncthreads();
    potential(P, N.trial, A, dg, yc, al, E, N.diag);
    int stop = 0;
    if (tid == 0) {
      copy(N.z, N.trial, d);
      copy(N.g, E.g, d);
      N.pe = E.U;
      finite = E.U < CUDART_INF;
      stop = D.init != nullptr || finite || attempt + 1 >= INIT_TRIES;
    }
    if (__syncthreads_or(stop)) break;
  }
  if (!__syncthreads_or(finite) && (D.init == nullptr || W + S > 0)) {
    // no finite starting point (the caller's, or none among INIT_TRIES uniform draws): the chain is not run and says so
    // with NaN results
    if (tid == 0) {
      for (int k = 0; k < So; ++k) {
        for (int i = 0; i < d; ++i) {
          out_u[static_cast<size_t>(k) * d + i] = CUDART_NAN;
          if (D.log_samples) D.log_samples[(p * So + k) * d + i] = CUDART_NAN;
        }
        for (int j = 0; j < D.n_pred; ++j) {
          if (D.mean) D.mean[(p * So + k) * D.n_pred + j] = CUDART_NAN;
          if (D.var) D.var[(p * So + k) * D.n_pred + j] = CUDART_NAN;
        }
      }
      if (D.potential) D.potential[p] = CUDART_INF;
      if (D.grad)
        for (int i = 0; i < d; ++i) D.grad[p * d + i] = CUDART_NAN;
      D.step_size[p] = CUDART_NAN;
      D.accept[p] = CUDART_NAN;
      if (D.trace)
        for (long long i = 0; i < static_cast<long long>(W + S) * (d + 2); ++i) D.trace[p * (W + S) * (d + 2) + i] = CUDART_NAN;
      for (int k = 0; k < PFN_GP_MCMC_NDIAG; ++k) D.diag[p * PFN_GP_MCMC_NDIAG + k] = N.diag[k];
    }
    return;
  }

  if (W == 0 && S == 0) {                      // evaluate-only: U, grad and the predictive at init
    if (tid == 0) copy(out_u, N.z, d);
  } else {
    step_size_search(P, N, E, A, dg, yc, al);
    for (int it = 0; it < W + S; ++it) {
      if (tid == 0) {
        N.it = it;
        iteration_begin(N);
        subtree_begin(N);
      }
      __syncthreads();
      for (;;) {                               // doubling
        int leaf_status = 0;                   // thread 0's leaf_end result; the others only learn whether it is 0
        for (;;) {                             // leaves of the new subtree
          potential(P, N.trial, A, dg, yc, al, E, N.diag);
          if (tid == 0) leaf_status = leaf_end(N, E);
          if (__syncthreads_or(leaf_status)) break;
        }
        int tree_done = 0;
        if (tid == 0) {
          tree_done = subtree_end(N, leaf_status, D.max_tree_depth, W);
          if (!tree_done) subtree_begin(N);
        }
        if (__syncthreads_or(tree_done)) break;
      }
      int search = 0;
      if (tid == 0) {
        const double accept_prob = N.acc_sum / N.n_prop;
        if (D.trace) {
          double* row = D.trace + (p * (W + S) + it) * (d + 2);
          copy(row, N.z, d);
          row[d] = N.eps;
          row[d + 1] = N.depth;
        }
        if (it >= W) {
          copy(out_u + static_cast<size_t>(it - W) * d, N.z, d);
          N.acc_sampling = N.acc_sampling + accept_prob;
        } else {
          search = adapt(N, accept_prob, W);
        }
      }
      if (__syncthreads_or(search)) step_size_search(P, N, E, A, dg, yc, al);
    }
  }
  if (tid == 0) {
    if (D.potential) D.potential[p] = N.pe;
    if (D.grad)
      for (int i = 0; i < d; ++i) D.grad[p * d + i] = N.g[i];
    D.step_size[p] = (W == 0 && S == 0) ? 0.0 : N.eps;
    D.accept[p] = S > 0 ? N.acc_sampling / S : CUDART_NAN;
  }
  // ---- predictive of rows t .. t + n_pred - 1 under every kept sample: one factorisation per sample, no gradient
  // (evaluate-only: at init, whose factorisation is still in A)
  const int want = predict_row && D.mean != nullptr;
  for (int k = 0; k < So; ++k) {
    int have = E.pd;
    if (S > 0 && want) {
      if (tid == 0) copy(N.trial, out_u + static_cast<size_t>(k) * d, d);
      __syncthreads();
      have = factor_at(P, N.trial, A, dg, yc, al, E, N.diag);
    }
    for (int j = 0; j < D.n_pred; ++j) {
      double mean = CUDART_NAN, var = CUDART_NAN;
      if (want && have && t + j < D.T)
        gp::predict(P, E.inv_ls, E.s, 0.0, xs + static_cast<size_t>(t + j) * F, A, dg, al, ks, E.red, mean, var);
      if (tid == 0) {
        if (D.mean) D.mean[(p * So + k) * D.n_pred + j] = mean;
        if (D.var) D.var[(p * So + k) * D.n_pred + j] = var;
      }
    }
    if (tid == 0) {
      double* uk = out_u + static_cast<size_t>(k) * d;
      if (D.log_samples)
        for (int i = 0; i < d; ++i) D.log_samples[(p * So + k) * d + i] = uk[i];
      for (int i = 0; i < d; ++i) uk[i] = exp(uk[i]);
    }
    __syncthreads();
  }
  if (tid == 0)
    for (int k = 0; k < PFN_GP_MCMC_NDIAG; ++k) D.diag[p * PFN_GP_MCMC_NDIAG + k] = N.diag[k];
}

}  // namespace
}  // namespace pfn

using namespace pfn;

extern "C" int pfn_gp_mcmc(const pfn_gp_mcmc_desc* d, void* stream) {
  PFN_CHECK_ARG(d != nullptr, "gp_mcmc: null descriptor");
  PFN_CHECK_ARG(d->B > 0 && d->T > 0 && d->F > 0 && d->n_ts > 0, "gp_mcmc: empty problem B=%d T=%d F=%d n_ts=%d", d->B,
                d->T, d->F, d->n_ts);
  PFN_CHECK_ARG(d->T <= PFN_GP_FIT_MAX_T, "gp_mcmc: T=%d exceeds %d (the t x t fp64 matrix lives in shared memory)", d->T,
                PFN_GP_FIT_MAX_T);
  PFN_CHECK_ARG(d->F <= PFN_GP_FIT_MAX_F, "gp_mcmc: F=%d exceeds %d", d->F, PFN_GP_FIT_MAX_F);
  PFN_CHECK_ARG(d->n_ts <= PFN_GP_FIT_MAX_T, "gp_mcmc: n_ts=%d exceeds %d", d->n_ts, PFN_GP_FIT_MAX_T);
  PFN_CHECK_ARG(d->ts != nullptr, "gp_mcmc: ts is null");
  PFN_CHECK_ARG(d->kernel_type >= PFN_KERNEL_MATERN12 && d->kernel_type <= PFN_KERNEL_MATERN52,
                "gp_mcmc: kernel type %d is not a Matern kernel", d->kernel_type);
  PFN_CHECK_ARG(d->x && d->y && d->samples && d->step_size && d->accept && d->diag,
                "gp_mcmc: null input or output pointer");
  PFN_CHECK_ARG(d->ls_rate > 0.0 && d->os_rate > 0.0 && d->noise_rate > 0.0 && d->ls_conc > 0.0 && d->os_conc > 0.0 &&
                d->noise_conc > 0.0, "gp_mcmc: Gamma prior parameters must be positive");
  PFN_CHECK_ARG(d->num_samples >= 0 && d->warmup_steps >= 0, "gp_mcmc: negative num_samples=%d or warmup_steps=%d",
                d->num_samples, d->warmup_steps);
  PFN_CHECK_ARG(static_cast<long long>(d->num_samples) + d->warmup_steps <= 0x7fffffffLL, "gp_mcmc: too many iterations");
  PFN_CHECK_ARG(d->num_samples + d->warmup_steps > 0 || d->init != nullptr,
                "gp_mcmc: warmup_steps = num_samples = 0 evaluates at init, which is null");
  PFN_CHECK_ARG(d->n_pred >= 1 && d->n_pred <= PFN_GP_FIT_MAX_T, "gp_mcmc: n_pred=%d outside [1, %d]", d->n_pred,
                PFN_GP_FIT_MAX_T);
  PFN_CHECK_ARG(d->max_tree_depth >= 1 && d->max_tree_depth <= PFN_GP_MCMC_MAX_DEPTH,
                "gp_mcmc: max_tree_depth=%d outside [1, %d]", d->max_tree_depth, PFN_GP_MCMC_MAX_DEPTH);
  PFN_CHECK_ARG(static_cast<long long>(d->B) * d->n_ts <= 0x7fffffffLL, "gp_mcmc: too many problems");
  McmcArgs a;
  a.d = *d;
  for (int i = 0; i < d->n_ts; ++i) {
    PFN_CHECK_ARG(d->ts[i] >= 1 && d->ts[i] <= d->T, "gp_mcmc: ts[%d]=%d outside [1, T=%d]", i, d->ts[i], d->T);
    a.slot_t[i] = d->ts[i];
    a.slot_i[i] = i;
  }
  for (int i = 1; i < d->n_ts; ++i)            // largest t first
    for (int j = i; j > 0 && a.slot_t[j] > a.slot_t[j - 1]; --j) {
      const int tt = a.slot_t[j]; a.slot_t[j] = a.slot_t[j - 1]; a.slot_t[j - 1] = tt;
      const int ii = a.slot_i[j]; a.slot_i[j] = a.slot_i[j - 1]; a.slot_i[j - 1] = ii;
    }
  const size_t smem = mcmc_smem(a.slot_t[0], d->T, d->F, d->n_pred);
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set))
    PFN_CUDA_OK(cudaFuncSetAttribute(gp_mcmc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     static_cast<int>(gp::problem_smem(PFN_GP_FIT_MAX_T, PFN_GP_FIT_MAX_F))));
  gp_mcmc_kernel<<<d->B * d->n_ts, FT, smem, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  PFN_LAUNCH_OK();
  return 0;
}
