// Fully Bayesian GP baseline: one CTA per (prefix t, dataset) problem runs a whole NUTS chain over the hyperparameters
// u = log(ls_1..F, s, noise) of the Gamma-prior Matern-ARD GP, then forms the predictive of row t under every kept
// sample.  No host loop, no per-iteration launch.  Restates reference priors/fast_gp_mix.py:171-268 (pyro NUTS with
// adapt_step_size=True, everything else at pyro 1.7's defaults) targeting the posterior p(u | y[:t]); see
// include/pfn_b200.h for the contract and oracle/gp_mcmc_oracle.py (nuts_chain) for the sampler written out on the CPU.
//
// The chain is nuts.cuh's, shared with bnn_mcmc.cu, with its vector pool in static shared memory.  Its sums run in
// element order (ElementSum: d <= PFN_GP_FIT_MAX_F + 2 < 256, so thread i owns element i alone), the order nuts_chain
// adds in.  Every potential evaluation is the fit's fp64 shared-memory factorisation (gp_posterior.cuh), run by all
// threads; thread i forms dU/du_i.  This file is compiled with -fmad=false: the sampler's arithmetic is then the plain
// IEEE sequence the CPU restatement performs (the potential itself uses explicit fma() and is unaffected).
#include "gp_posterior.cuh"
#include "nuts.cuh"

namespace pfn {
namespace {

using gp::FT;
using gp::FW;
using gp::Problem;

constexpr int MAXF = PFN_GP_FIT_MAX_F;
constexpr int DM = PFN_GP_FIT_MAX_F + 2;       // sampled coordinates: log ls_1..F, log s, log noise
using Sum = nuts::ElementSum<DM>;
using Chain = nuts::Chain<Sum>;
static_assert(FT == nuts::NT, "one CTA runs the factorisation and the chain");

struct Params {                                // lengthscales at the point last evaluated or factorised
  double ls[MAXF], inv_ls[MAXF];
  double red[FW * 8];
};

__device__ __forceinline__ double log_gamma_u(double u, double theta, double a, double b) {
  return a * log(b) - lgamma(a) + a * u - b * theta;    // log Gamma(e^u; a, b) + u
}

struct Model {
  Problem P;
  double *A, *dg, *yc, *al;
  Params* E;
  double s, noise;                             // outputscale and noise at the point last evaluated or factorised
  int pd;                                      // whether its K was positive definite

  __device__ void set_params(const double* u) {
    for (int k = threadIdx.x; k < P.F; k += FT) {
      const double l = exp(u[k]);
      E->ls[k] = l;
      E->inv_ls[k] = 1.0 / l;
    }
    s = exp(u[P.F]);
    noise = exp(u[P.F + 1]);
    __syncthreads();
  }

  // nuts.cuh's model hook; NOT_PD counts the evaluations whose K was not positive definite (U = +inf, gradient 0)
  template <class Fn>
  __device__ double evaluate(Chain& c, double& third, Fn per_elem) {
    const int tid = threadIdx.x, t = P.t, F = P.F;
    const double* u = c.trial;
    double* ge = c.vec(nuts::V_GE);
    set_params(u);
    double v[1] = {0.0}, sums[6];
    pd = gp::lml_terms(P, E->inv_ls, s, noise, 0.0, A, dg, yc, al, E->red, sums, [&](int k, double val) {
      if (tid == k) {
        const double il = E->inv_ls[k];
        ge[k] = -(0.5 * s * il * il * val) - P.ls_a + P.ls_b * E->ls[k];
        v[0] = v[0] + per_elem(k, ge[k]);
      }
    });
    double U = CUDART_INF;
    if (pd) {
      const double logn = -0.5 * sums[1] - sums[0] - 0.5 * t * gp::LOG_2PI;
      double lp = log_gamma_u(u[F], s, P.os_a, P.os_b) + log_gamma_u(u[F + 1], noise, P.nz_a, P.nz_b);
      for (int k = 0; k < F; ++k) lp += log_gamma_u(u[k], E->ls[k], P.ls_a, P.ls_b);
      const double Uf = -(logn + lp);
      U = Uf < CUDART_INF ? Uf : CUDART_INF;   // NaN counts as +inf
      if (tid == F) ge[F] = -(0.5 * s * sums[3]) - P.os_a + P.os_b * s;
      if (tid == F + 1) ge[F + 1] = -(0.5 * noise * sums[4]) - P.nz_a + P.nz_b * noise;
      if (tid == F || tid == F + 1) v[0] = v[0] + per_elem(tid, ge[tid]);
    } else {
      for (int i = tid; i < c.d; i += FT) {
        ge[i] = 0.0;
        v[0] = v[0] + per_elem(i, 0.0);
      }
      c.diag[PFN_GP_MCMC_NOT_PD]++;
    }
    c.diag[PFN_GP_MCMC_EVALS]++;
    c.sum(v);
    third = v[0];
    return U;
  }
};

// rows of x a problem keeps in shared memory: its t rows and the predictive rows after them
__host__ __device__ __forceinline__ int mcmc_x_rows(int t, int T, int n_pred) { return min(T, t + n_pred); }

// A [tmax, tmax|1], x [rows, F], y, dg, yc, al, ks [tmax]; never above gp::problem_smem(T, F) since rows <= T
inline size_t mcmc_smem(int tmax, int T, int F, int n_pred) {
  return (static_cast<size_t>(tmax) * (tmax | 1) + static_cast<size_t>(mcmc_x_rows(tmax, T, n_pred)) * F + 5 * tmax) *
         sizeof(double);
}

__global__ void __launch_bounds__(FT, 1) gp_mcmc_kernel(const gp::PrefixArgs<pfn_gp_mcmc_desc> args) {
  const pfn_gp_mcmc_desc& D = args.d;
  extern __shared__ __align__(16) double mcmc_dyn[];
  __shared__ nuts::Shared<Sum> sh;
  __shared__ double trial[DM], pool[nuts::POOL_VECS * DM];
  __shared__ Params E;
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
  Chain c;
  nuts::start(c, &sh, trial, pool, d, D.seed, static_cast<uint32_t>(b), static_cast<uint32_t>(t), W);
  const Problem P{xs, ys, t, F, ld, D.kernel_type, D.ls_conc, D.ls_rate, D.os_conc, D.os_rate, D.noise_conc, D.noise_rate};
  Model m{P, A, dg, yc, al, &E, 0.0, 0.0, 0};
  double* out_u = D.samples + p * So * d;      // u of every kept sample; turned into theta at the end
  double* trace = D.trace ? D.trace + p * (W + S) * (d + 2) : nullptr;
  const bool finite = nuts::run(c, m, D.init ? D.init + p * d : nullptr, W, S, D.max_tree_depth, out_u, trace);
  const bool ran = W + S > 0;                  // otherwise evaluate-only: U, grad and the predictive at init
  nuts::store_outputs(c, finite, W, S, p, out_u, D.potential, D.grad, D.step_size, D.accept);
  if (!finite && !ran) {
    // evaluate-only at an init whose U is not finite: step size 0 and the gradient found there, as for a finite U
    if (tid == 0) D.step_size[p] = 0.0;
    if (D.grad) nuts::copy(D.grad + p * d, c.vec(nuts::V_G), d);
  }
  if (!finite && ran) {
    // no finite starting point (the caller's, or none among INIT_TRIES uniform draws): the chain is not run and its
    // predictive is NaN
    if (tid == 0)
      for (int k = 0; k < So; ++k) {
        for (int i = 0; i < d; ++i)
          if (D.log_samples) D.log_samples[(p * So + k) * d + i] = CUDART_NAN;
        for (int j = 0; j < D.n_pred; ++j) {
          if (D.mean) D.mean[(p * So + k) * D.n_pred + j] = CUDART_NAN;
          if (D.var) D.var[(p * So + k) * D.n_pred + j] = CUDART_NAN;
        }
      }
    nuts::store_diag(c, D.diag + p * PFN_GP_MCMC_NDIAG);
    return;
  }
  // ---- predictive of rows t .. t + n_pred - 1 under every kept sample (warmup only: the state the warmup ended in): one
  // factorisation per sample, no gradient (evaluate-only: at init, whose factorisation is still in A)
  const int want = t < D.T && D.mean != nullptr;
  for (int k = 0; k < So; ++k) {
    double* uk = out_u + static_cast<size_t>(k) * d;
    if (ran && want) {
      nuts::copy(trial, uk, d);
      __syncthreads();
      m.set_params(trial);
      c.diag[PFN_GP_MCMC_EVALS]++;
      double log_dg;
      m.pd = gp::factor(P, E.inv_ls, m.s, m.noise, 0.0, A, dg, yc, al, log_dg);
    }
    for (int j = 0; j < D.n_pred; ++j) {
      double mean = CUDART_NAN, var = CUDART_NAN;
      if (want && m.pd && t + j < D.T)
        gp::predict(P, E.inv_ls, m.s, 0.0, xs + static_cast<size_t>(t + j) * F, A, dg, al, ks, E.red, mean, var);
      if (tid == 0) {
        if (D.mean) D.mean[(p * So + k) * D.n_pred + j] = mean;
        if (D.var) D.var[(p * So + k) * D.n_pred + j] = var;
      }
    }
    for (int i = tid; i < d; i += FT) {
      if (D.log_samples) D.log_samples[(p * So + k) * d + i] = uk[i];
      uk[i] = exp(uk[i]);
    }
    __syncthreads();
  }
  nuts::store_diag(c, D.diag + p * PFN_GP_MCMC_NDIAG);
}

}  // namespace
}  // namespace pfn

using namespace pfn;

extern "C" int pfn_gp_mcmc(const pfn_gp_mcmc_desc* d, void* stream) {
  gp::PrefixArgs<pfn_gp_mcmc_desc> a;
  if (const int rc = gp::check_prefix_problems(d, "gp_mcmc", a)) return rc;
  if (const int rc = nuts::check_chain(d, "gp_mcmc", d->x && d->y)) return rc;
  PFN_CHECK_ARG(d->n_pred >= 1 && d->n_pred <= PFN_GP_FIT_MAX_T, "gp_mcmc: n_pred=%d outside [1, %d]", d->n_pred,
                PFN_GP_FIT_MAX_T);
  const size_t smem = mcmc_smem(a.slot_t[0], d->T, d->F, d->n_pred);
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set))
    PFN_CUDA_OK(cudaFuncSetAttribute(gp_mcmc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     static_cast<int>(gp::problem_smem(PFN_GP_FIT_MAX_T, PFN_GP_FIT_MAX_F))));
  gp_mcmc_kernel<<<d->B * d->n_ts, FT, smem, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  PFN_LAUNCH_OK();
  return 0;
}
