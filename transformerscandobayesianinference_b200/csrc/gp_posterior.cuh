// fp64 pieces of the Gamma-prior Matern-ARD GP shared by the MAP fit (gp_fit.cu) and the NUTS sampler (gp_mcmc.cu).
// One CTA of GP_FT threads owns one problem; the t x t matrix A (odd leading dimension) lives in shared memory.
//   build K (lower)  ->  Cholesky in place (lower, pivots in dg)  ->  L^-1 into the upper triangle (stored transposed)
//   ->  K^-1 = L^-T L^-1 into the strict lower triangle + dg  ->  alpha = K^-1 (y - c)
//   ->  the trace terms of d log N / d theta (W = alpha alpha^T - K^-1), with dK recomputed from x (not stored).
// Each kernel composes its own parameterisation and priors from these terms.  Every reduction has a fixed order, so a
// problem's result depends on its own inputs only (bitwise repeatable).  On the host: the launch arguments of both
// kernels and the check of the descriptor fields they share.
#pragma once
#include <math_constants.h>

#include "common.cuh"
#include "../../include/pfn_b200.h"

namespace pfn {
namespace gp {

constexpr int FT = 256;                        // threads per CTA: a 16 x 16 grid for the triangular sweeps
constexpr int FW = FT / 32;
constexpr double LOG_2PI = 1.8378770664093453;

// k(r) and g(r) = -k'(r) / r of the Matern kernels, from r^2 (g is the factor of dk/dls_d = g Delta_d^2 / ls_d^3)
__device__ __forceinline__ void matern(double r2, int kt, double& k, double& g) {
  const double r = sqrt(r2);
  if (kt == PFN_KERNEL_MATERN12) {
    const double e = exp(-r);
    k = e;
    g = r > 0.0 ? e / r : 0.0;                 // r -> 0 pairs (duplicate rows): the derivative term vanishes
  } else if (kt == PFN_KERNEL_MATERN32) {
    const double a = 1.7320508075688772 * r, e = exp(-a);
    k = (1.0 + a) * e;
    g = 3.0 * e;
  } else {
    const double a = 2.23606797749979 * r, e = exp(-a);
    k = (1.0 + a + (5.0 / 3.0) * r2) * e;
    g = (5.0 / 3.0) * (1.0 + a) * e;
  }
}

// Fixed-order block sum of K values (every thread receives the same sums).
template <int K>
__device__ __forceinline__ void block_sum(double (&v)[K], double* red) {
#pragma unroll
  for (int q = 0; q < K; ++q)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[q] += __shfl_xor_sync(0xffffffffu, v[q], o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int q = 0; q < K; ++q) red[q * FW + (threadIdx.x >> 5)] = v[q];
  __syncthreads();
#pragma unroll
  for (int q = 0; q < K; ++q) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < FW; ++w) s += red[q * FW + w];
    v[q] = s;
  }
}

__device__ __forceinline__ double log_gamma_pdf(double v, double a, double b) {
  return a * log(b) - lgamma(a) + (a - 1.0) * log(v) - b * v;
}

// Cholesky of the t x t lower triangle of A in place (all threads), right-looking, one barrier per column: phase j
// updates the trailing block with the unscaled column j and scales column j-1 (nobody reads it in phase j).  On success
// returns t, with L's strict lower triangle in A and its diagonal in dg.  Otherwise returns the first pivot j that is not
// positive: columns < j - 1 of L and dg[0 .. j-1] are then final, column j - 1 below the diagonal still awaits its
// division by dg[j-1], and the rest of A is unspecified.
__device__ __forceinline__ int cholesky_lower(double* A, double* dg, int t, int ld) {
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  for (int j = 0; j < t; ++j) {
    const double dj = A[j * ld + j];
    if (!(dj > 0.0) || !isfinite(dj)) return j;                  // uniform: every thread read the same pivot
    const double inv_d = 1.0 / dj;
    if (tid == 0) dg[j] = sqrt(dj);
    if (j > 0)
      for (int r = j + tid; r < t; r += FT) A[r * ld + j - 1] /= dg[j - 1];
    for (int r = j + 1 + ty; r < t; r += 16) {
      const double arj = A[r * ld + j] * inv_d;
      for (int q = j + 1 + tx; q <= r; q += 16) A[r * ld + q] = fma(-arj, A[q * ld + j], A[r * ld + q]);
    }
    __syncthreads();
  }
  return t;
}

struct Problem {
  const double* xs;                            // [t, F] rows of the dataset
  const double* ys;                            // [t]
  int t, F, ld, kt;
  double ls_a, ls_b, os_a, os_b, nz_a, nz_b;   // Gamma(concentration, rate) priors
};

// Factorisation of K = s k(x, x; ls) + noise I (all threads; inv_ls [F] in shared memory, visible to all): returns 0
// when K is not positive definite.  Otherwise alpha = K^-1 (y - c) is left in al, y - c in yc, K^-1 in (strict lower of A,
// dg), and every thread's log_dg holds log L_ii of its row tid (0 for tid >= t).
__device__ __forceinline__ int factor(const Problem& P, const double* inv_ls, double s, double noise, double c, double* A,
                                      double* dg, double* yc, double* al, double& log_dg) {
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int t = P.t, F = P.F, ld = P.ld;
  // ---- K, lower triangle
  for (int r = ty; r < t; r += 16)
    for (int q = tx; q <= r; q += 16) {
      double v = s + noise;                    // k(x, x) = 1
      if (q != r) {
        double r2 = 0.0;
        for (int d = 0; d < F; ++d) {
          const double df = (P.xs[r * F + d] - P.xs[q * F + d]) * inv_ls[d];
          r2 = fma(df, df, r2);
        }
        double k, g;
        matern(r2, P.kt, k, g);
        v = s * k;
      }
      A[r * ld + q] = v;
    }
  for (int i = tid; i < t; i += FT) yc[i] = P.ys[i] - c;
  __syncthreads();
  if (cholesky_lower(A, dg, t, ld) < t) return 0;
  log_dg = tid < t ? log(dg[tid]) : 0.0;       // t <= FT
  // ---- L^-1 into the upper triangle, transposed: U[j][i] = X[i][j] (i >= j), row k of X final after phase k-1.
  for (int j = ty; j < t; j += 16)
    for (int i = j + tx; i < t; i += 16) A[j * ld + i] = (i == j) ? 1.0 : 0.0;
  __syncthreads();
  for (int k = 0; k < t; ++k) {
    const double inv_lkk = 1.0 / dg[k];
    if (k > 0) {
      const double inv_prev = 1.0 / dg[k - 1];
      for (int j = tid; j < k; j += FT) A[j * ld + k - 1] *= inv_prev;
    }
    for (int i = k + 1 + tx; i < t; i += 16) {
      const double lik = A[i * ld + k] * inv_lkk;
      for (int j = ty; j <= k; j += 16) A[j * ld + i] = fma(-lik, A[j * ld + k], A[j * ld + i]);
    }
    __syncthreads();
  }
  {
    const double inv_last = 1.0 / dg[t - 1];
    for (int j = tid; j < t; j += FT) A[j * ld + t - 1] *= inv_last;
  }
  __syncthreads();
  // ---- K^-1 = X^T X: (r, q), q <= r, = sum_{k >= r} U[r][k] U[q][k]; strict lower -> A, diagonal -> dg
  for (int r = ty; r < t; r += 16)
    for (int q = tx; q <= r; q += 16) {
      double v = 0.0;
      for (int k = r; k < t; ++k) v = fma(A[r * ld + k], A[q * ld + k], v);
      if (q == r) dg[r] = v; else A[r * ld + q] = v;
    }
  __syncthreads();
  // ---- alpha = K^-1 (y - c)
  for (int i = tid; i < t; i += FT) {
    double v = 0.0;
    for (int j = 0; j < t; ++j) {
      const double kij = j < i ? A[i * ld + j] : (j > i ? A[j * ld + i] : dg[i]);
      v = fma(kij, yc[j], v);
    }
    al[i] = v;
  }
  __syncthreads();
  return 1;
}

// log N(y | c, K) terms (all threads, arguments as for factor).  Returns 0 when K is not positive definite.  Otherwise
// every thread holds
//   sums = {1/2 log det K, (y-c)^T alpha, sum alpha, sum_ij W_ij k_ij, sum_i W_ii, -}
// and per_dim(d, v) is called by every thread with v = sum_{i>j} P_ij Delta_d^2, P = 2 W g, for d = 0..F-1 in order.
// alpha is left in al and K^-1 in (strict lower of A, dg).
template <typename PerDim>
__device__ __forceinline__ int lml_terms(const Problem& P, const double* inv_ls, double s, double noise, double c,
                                         double* A, double* dg, double* yc, double* al, double* red, double (&sums)[6],
                                         PerDim per_dim) {
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int t = P.t, F = P.F, ld = P.ld;
  double log_dg;
  if (!factor(P, inv_ls, s, noise, c, A, dg, yc, al, log_dg)) return 0;
  // ---- pass 1: W = alpha alpha^T - K^-1; sum W k (outputscale), sum_i W_ii (noise); P = 2 W g -> upper triangle
  sums[0] = log_dg;
  sums[1] = sums[2] = sums[3] = sums[4] = sums[5] = 0.0;
  for (int i = tid; i < t; i += FT) {
    sums[1] = fma(yc[i], al[i], sums[1]);
    sums[2] += al[i];
    const double wii = fma(al[i], al[i], -dg[i]);
    sums[3] += wii;
    sums[4] += wii;
  }
  for (int r = ty; r < t; r += 16)
    for (int q = tx; q < r; q += 16) {
      double r2 = 0.0;
      for (int d = 0; d < F; ++d) {
        const double df = (P.xs[r * F + d] - P.xs[q * F + d]) * inv_ls[d];
        r2 = fma(df, df, r2);
      }
      double k, g;
      matern(r2, P.kt, k, g);
      const double w = fma(al[r], al[q], -A[r * ld + q]);
      sums[3] = fma(2.0 * w, k, sums[3]);
      A[q * ld + r] = 2.0 * w * g;
    }
  block_sum(sums, red);
  // ---- pass 2: per input dimension, sum P Delta_d^2
  for (int d = 0; d < F; ++d) {
    double v[1] = {0.0};
    for (int r = ty; r < t; r += 16)
      for (int q = tx; q < r; q += 16) {
        const double df = P.xs[r * F + d] - P.xs[q * F + d];
        v[0] = fma(A[q * ld + r], df * df, v[0]);
      }
    block_sum(v, red);
    per_dim(d, v[0]);
  }
  return 1;
}

// Latent predictive at xstar after lml_terms (all threads): mean = c + k*^T alpha, var = s - k*^T K^-1 k*.
__device__ __forceinline__ void predict(const Problem& P, const double* inv_ls, double s, double c, const double* xstar,
                                        const double* A, const double* dg, const double* al, double* ks, double* red,
                                        double& mean, double& var) {
  const int tid = threadIdx.x, t = P.t, F = P.F, ld = P.ld;
  for (int i = tid; i < t; i += FT) {
    double r2 = 0.0;
    for (int d = 0; d < F; ++d) {
      const double df = (P.xs[i * F + d] - xstar[d]) * inv_ls[d];
      r2 = fma(df, df, r2);
    }
    double k, g;
    matern(r2, P.kt, k, g);
    ks[i] = s * k;
  }
  __syncthreads();
  double v[2] = {0.0, 0.0};
  for (int i = tid; i < t; i += FT) {
    double u = 0.0;
    for (int j = 0; j < t; ++j) {
      const double kij = j < i ? A[i * ld + j] : (j > i ? A[j * ld + i] : dg[i]);
      u = fma(kij, ks[j], u);
    }
    v[0] = fma(ks[i], al[i], v[0]);
    v[1] = fma(ks[i], u, v[1]);
  }
  block_sum(v, red);
  mean = c + v[0];
  var = s - v[1];
}

// Dynamic shared memory of one problem at the largest prefix tmax: A [tmax, tmax|1], x [tmax, F], y, dg, yc, al, ks [tmax],
// x* [F].
inline size_t problem_smem(int tmax, int F) {
  return (static_cast<size_t>(tmax) * (tmax | 1) + static_cast<size_t>(tmax) * F + 6 * tmax + F) * sizeof(double);
}

// ------------------------------------------------------------------------------------------------ host
// Launch arguments of a kernel over the (prefix, dataset) problems of a descriptor (pfn_gp_fit_desc, pfn_gp_mcmc_desc):
// CTA slot * B + b solves prefix slot_t[slot] of dataset b.
template <class Desc>
struct PrefixArgs {
  Desc d;
  int slot_t[PFN_GP_FIT_MAX_T];                // prefix lengths, largest first
  int slot_i[PFN_GP_FIT_MAX_T];                // their index in d.ts
};

// Checks the fields the two descriptors share, with `who` (the entry point's name) heading every message, and fills a.
// Returns 0 on success.
template <class Desc>
inline int check_prefix_problems(const Desc* d, const char* who, PrefixArgs<Desc>& a) {
  PFN_CHECK_ARG(d != nullptr, "%s: null descriptor", who);
  PFN_CHECK_ARG(d->B > 0 && d->T > 0 && d->F > 0 && d->n_ts > 0, "%s: empty problem B=%d T=%d F=%d n_ts=%d", who, d->B,
                d->T, d->F, d->n_ts);
  PFN_CHECK_ARG(d->T <= PFN_GP_FIT_MAX_T, "%s: T=%d exceeds %d (the t x t fp64 matrix lives in shared memory)", who, d->T,
                PFN_GP_FIT_MAX_T);
  PFN_CHECK_ARG(d->F <= PFN_GP_FIT_MAX_F, "%s: F=%d exceeds %d", who, d->F, PFN_GP_FIT_MAX_F);
  PFN_CHECK_ARG(d->n_ts <= PFN_GP_FIT_MAX_T, "%s: n_ts=%d exceeds %d", who, d->n_ts, PFN_GP_FIT_MAX_T);
  PFN_CHECK_ARG(d->ts != nullptr, "%s: ts is null", who);
  PFN_CHECK_ARG(d->kernel_type >= PFN_KERNEL_MATERN12 && d->kernel_type <= PFN_KERNEL_MATERN52,
                "%s: kernel type %d is not a Matern kernel", who, d->kernel_type);
  PFN_CHECK_ARG(d->ls_rate > 0.0 && d->os_rate > 0.0 && d->noise_rate > 0.0 && d->ls_conc > 0.0 && d->os_conc > 0.0 &&
                d->noise_conc > 0.0, "%s: Gamma prior parameters must be positive", who);
  PFN_CHECK_ARG(static_cast<long long>(d->B) * d->n_ts <= 0x7fffffffLL, "%s: too many problems", who);
  a.d = *d;
  for (int i = 0; i < d->n_ts; ++i) {
    PFN_CHECK_ARG(d->ts[i] >= 1 && d->ts[i] <= d->T, "%s: ts[%d]=%d outside [1, T=%d]", who, i, d->ts[i], d->T);
    a.slot_t[i] = d->ts[i];
    a.slot_i[i] = i;
  }
  // largest t first, so the longest CTAs start in the first wave instead of forming its tail
  for (int i = 1; i < d->n_ts; ++i)
    for (int j = i; j > 0 && a.slot_t[j] > a.slot_t[j - 1]; --j) {
      const int tt = a.slot_t[j]; a.slot_t[j] = a.slot_t[j - 1]; a.slot_t[j - 1] = tt;
      const int ii = a.slot_i[j]; a.slot_i[j] = a.slot_i[j - 1]; a.slot_i[j - 1] = ii;
    }
  return 0;
}

}  // namespace gp
}  // namespace pfn
