// Baselines of the sklearn-backed priors, every prefix of every dataset in one launch, fp64:
//   pfn_ridge_prefix : priors/ridge.py:23-34, Ridge(alpha).fit(x[:t], y[:t]).predict(x[t]) for t = 1 .. T-1
//   pfn_exact_gp     : priors/gp.py, the fixed-length-scale RBF GaussianProcessRegressor: its per-prefix predictive
//                      (evaluate, :41-62) and its prior draw (sample_y of the unfitted model, :19-34)
// One CTA per dataset.  Every reduction has a fixed order, so a dataset's results depend on its own inputs only.
#include <float.h>

#include "gp_posterior.cuh"

namespace pfn {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxSweeps = 60;              // one-sided Jacobi sweeps per prefix (a handful suffice)

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------------ ridge
// Shared state: R [F, F+1] = [R | Q^T yc] with R^T R = Xc^T Xc over the rows folded in so far (exactly zero rows beyond
// their count: a rotation against an empty row is a swap), W its copy that the Jacobi sweeps rotate, mu [F+1] the running
// means (y last), a [F+1] the row being folded in, coef [F] per row of W.
inline size_t ridge_smem(int F) { return (static_cast<size_t>(2) * F * (F + 1) + 2 * (F + 1) + F) * sizeof(double); }

// Folds the row a into R by Givens rotations (all threads).  Rows of R are in shared memory with leading dimension F + 1.
__device__ __forceinline__ void givens_fold(double* R, double* a, int F) {
  const int ld = F + 1;
  for (int k = 0; k < F; ++k) {
    const double ak = a[k];
    if (ak == 0.0) continue;                  // uniform: every thread read the same value after the last barrier
    const double rk = R[k * ld + k];
    const double h = hypot(rk, ak), c = rk / h, s = ak / h;
    __syncthreads();                          // R[k][k] and a[k] read by everyone before they change
    for (int j = k + threadIdx.x; j <= F; j += kThreads) {
      const double r = R[k * ld + j], v = a[j];
      R[k * ld + j] = fma(c, r, s * v);
      a[j] = fma(-s, r, c * v);
    }
    __syncthreads();
  }
}

// One-sided Jacobi on the rows of W (their first F columns), the last column rotated along: on return the rows are
// orthogonal, W_i = s_i v_i^T with (U^T Q^T yc)_i in column F.  Pairs follow a round-robin schedule, one warp per pair.
__device__ __forceinline__ void jacobi_rows(double* W, int F, int* rotated) {
  const int ld = F + 1, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = F + (F & 1);                  // players; an odd F adds an idle one
  for (int sweep = 0; sweep < kMaxSweeps; ++sweep) {
    if (threadIdx.x == 0) *rotated = 0;
    __syncthreads();
    for (int r = 0; r < n - 1; ++r) {
      for (int m = warp; m < n / 2; m += kWarps) {
        const int p = m == 0 ? n - 1 : (r + m) % (n - 1);
        const int q = (r - m + n - 1) % (n - 1);
        if (p >= F || q >= F) continue;
        double* wp = W + p * ld;
        double* wq = W + q * ld;
        double app = 0.0, aqq = 0.0, apq = 0.0;
        for (int c = lane; c < F; c += 32) {
          const double vp = wp[c], vq = wq[c];
          app = fma(vp, vp, app);
          aqq = fma(vq, vq, aqq);
          apq = fma(vp, vq, apq);
        }
        app = warp_sum_d(app);
        aqq = warp_sum_d(aqq);
        apq = warp_sum_d(apq);
        if (fabs(apq) > DBL_EPSILON * sqrt(app * aqq)) {        // false for an empty row and for NaN
          const double zeta = (aqq - app) / (2.0 * apq);
          // tan of the rotation angle, the root of t^2 + 2 zeta t - 1 of smaller magnitude; 1 / (2 zeta) where zeta^2
          // would overflow (badly scaled rows), so that every flagged rotation changes the rows
          const double t = fabs(zeta) > 1e150 ? 0.5 / zeta
                                              : copysign(1.0, zeta) / (fabs(zeta) + sqrt(fma(zeta, zeta, 1.0)));
          const double c = 1.0 / sqrt(fma(t, t, 1.0)), s = c * t;
          for (int j = lane; j <= F; j += 32) {
            const double vp = wp[j], vq = wq[j];
            wp[j] = fma(c, vp, -s * vq);
            wq[j] = fma(s, vp, c * vq);
          }
          if (lane == 0) *rotated = 1;
        }
      }
      __syncthreads();
    }
    const int any = *rotated;
    __syncthreads();
    if (!any) break;
  }
}

__global__ void __launch_bounds__(kThreads) ridge_prefix_kernel(pfn_ridge_prefix_desc D) {
  extern __shared__ double sm[];
  __shared__ double red[kWarps];
  __shared__ int rotated;
  const int F = D.F, T = D.T, ld = F + 1, b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double* R = sm;
  double* W = R + F * ld;
  double* mu = W + F * ld;
  double* a = mu + ld;
  double* coef = a + ld;
  const float* xb = D.x + static_cast<size_t>(b) * T * F;
  const size_t o = static_cast<size_t>(b) * T;

  for (int i = tid; i < F * ld; i += kThreads) R[i] = 0.0;
  if (tid == 0) { D.pred[o] = NAN; D.sq_err[o] = NAN; }
  __syncthreads();
  for (int i = 0; i < T; ++i) {
    if (i > 0) {
      // ---- prefix t = i: w from the SVD of the factor, then the prediction of row i
      const int t = i;
      for (int q = tid; q < F * ld; q += kThreads) W[q] = R[q];
      __syncthreads();
      jacobi_rows(W, F, &rotated);
      for (int r = warp; r < F; r += kWarps) {
        double s2 = 0.0;
        for (int c = lane; c < F; c += 32) s2 = fma(W[r * ld + c], W[r * ld + c], s2);
        s2 = warp_sum_d(s2);
        if (lane == 0) coef[r] = s2;
      }
      __syncthreads();
      double s2max = 0.0;
      for (int r = 0; r < F; ++r) s2max = fmax(s2max, coef[r]);
      const double cut = static_cast<double>(t > F ? t : F) * DBL_EPSILON;
      const double cut2 = cut * cut * s2max;
      __syncthreads();                        // coef read by everyone before it is overwritten
      for (int r = tid; r < F; r += kThreads) {
        const double s2 = coef[r];
        const bool keep = D.alpha > 0.0 ? s2 > 0.0 : s2 > cut2;
        coef[r] = keep ? W[r * ld + F] / (s2 + D.alpha) : 0.0;
      }
      __syncthreads();
      double v = 0.0;
      for (int f = tid; f < F; f += kThreads) {
        double w = 0.0;
        for (int r = 0; r < F; ++r) w = fma(W[r * ld + f], coef[r], w);
        v = fma(static_cast<double>(xb[static_cast<size_t>(t) * F + f]) - mu[f], w, v);
      }
      v = warp_sum_d(v);
      if (lane == 0) red[warp] = v;
      __syncthreads();
      if (tid == 0) {
        double p = 0.0;
        for (int w = 0; w < kWarps; ++w) p += red[w];
        p += mu[F];
        const double e = static_cast<double>(D.target[o + t]) - p;
        D.pred[o + t] = p;
        D.sq_err[o + t] = e * e;
      }
      __syncthreads();
    }
    if (i == T - 1) break;
    // ---- fold row i in: a = sqrt(i / (i + 1)) (row - mean of the rows before it), then the running means
    const double inv_n = 1.0 / static_cast<double>(i + 1), scale = sqrt(static_cast<double>(i) * inv_n);
    for (int f = tid; f <= F; f += kThreads) {
      const double v = f < F ? static_cast<double>(xb[static_cast<size_t>(i) * F + f]) : static_cast<double>(D.y[o + i]);
      const double delta = i == 0 ? 0.0 : v - mu[f];
      a[f] = scale * delta;
      mu[f] = i == 0 ? v : fma(delta, inv_n, mu[f]);
    }
    __syncthreads();
    if (i > 0) givens_fold(R, a, F);
  }
}

// ------------------------------------------------------------------------------------------------ exact GP
// exp(-|x_r / ls - x_q / ls|^2 / 2), the quotients formed in fp64 before the differences, as sklearn's RBF forms them
__device__ __forceinline__ double rbf(const float* __restrict__ xr, const float* __restrict__ xq, int F, double ls) {
  double s = 0.0;
  for (int f = 0; f < F; ++f) {
    const double d = static_cast<double>(xr[f]) / ls - static_cast<double>(xq[f]) / ls;
    s = fma(d, d, s);
  }
  return exp(-0.5 * s);
}

inline size_t exact_gp_smem(int T) { return (static_cast<size_t>(T) * (T | 1) + 2 * T) * sizeof(double); }

__global__ void __launch_bounds__(gp::FT) exact_gp_evaluate_kernel(pfn_exact_gp_desc D) {
  extern __shared__ double sm[];
  const int T = D.T, F = D.F, ld = T | 1, b = blockIdx.x, tid = threadIdx.x;
  double* A = sm;
  double* dg = A + T * ld;
  double* zs = dg + T;
  const float* xb = D.x + static_cast<size_t>(b) * T * F;
  const size_t o = static_cast<size_t>(b) * T;
  const double ls = D.length_scale;

  // the lower triangle as one flat loop: the nested 16 x 16 form spills a register around the fp64 divisions of rbf
  for (int e = tid; e < T * T; e += gp::FT) {
    const int r = e / T, q = e - r * T;
    if (q <= r) A[r * ld + q] = q == r ? 1.0 + D.alpha : rbf(xb + r * F, xb + q * F, F, ls);
  }
  __syncthreads();
  const int n = gp::cholesky_lower(A, dg, T, ld);
  if (n < T && n > 0) {                       // finish column n - 1, so that rows <= n of L are usable (row n lacks its pivot)
    for (int r = n + tid; r < T; r += gp::FT) A[r * ld + n - 1] /= dg[n - 1];
    __syncthreads();
  }
  // z = L^-1 y over the rows < n, one thread per row (T <= FT)
  double r = tid < n ? static_cast<double>(D.y[o + tid]) : 0.0;
  for (int k = 0; k < n; ++k) {
    if (tid == k) zs[k] = r / dg[k];
    __syncthreads();
    if (tid > k && tid < n) r = fma(-A[tid * ld + k], zs[k], r);
  }
  // prefix t predicts row t from row t of L: mean = L_t,<t z_<t, var = 1 - |L_t,<t|^2 (= pivot t - alpha)
  for (int t = 1 + tid; t < T; t += gp::FT) {
    double mean = NAN, var = NAN;
    if (t <= n) {
      double m = 0.0, s = 0.0;
      for (int k = 0; k < t; ++k) {
        const double l = A[t * ld + k];
        m = fma(l, zs[k], m);
        s = fma(l, l, s);
      }
      mean = m;
      var = fmax(1.0 - s, 0.0);
    }
    D.mean[o + t] = mean;
    D.var[o + t] = var;
  }
  if (tid == 0) {
    D.mean[o] = NAN;
    D.var[o] = NAN;
    D.status[b] = n + 1 < T ? n + 1 : 0;    // pivot n belongs to prefix n + 1, which is fitted only when n + 1 <= T - 1
  }
}

// Diagonal-pivoted Cholesky of K (unit diagonal, no noise), left-looking: column k of P L is formed from K's column of
// pivot k, computed from x, minus the earlier columns.  Thread i owns row i (its residual diagonal and chosen flag).
__global__ void __launch_bounds__(gp::FT) exact_gp_sample_kernel(pfn_exact_gp_desc D) {
  extern __shared__ double sm[];
  __shared__ double red_v[gp::FW];
  __shared__ int red_i[gp::FW];
  __shared__ int order[PFN_GP_FIT_MAX_T];
  __shared__ int taken[PFN_GP_FIT_MAX_T];
  const int T = D.T, F = D.F, ld = T | 1, b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double* G = sm;                             // G[k * ld + i] = (P L)[i][k]
  const float* xb = D.x + static_cast<size_t>(b) * T * F;
  const size_t o = static_cast<size_t>(b) * T;
  const double ls = D.length_scale;
  const double tol = static_cast<double>(T) * DBL_EPSILON;

  double dres = 1.0;                          // residual diagonal of row tid
  bool chosen = tid >= T;
  int rank = 0;
  for (int k = 0; k < T; ++k) {
    // the largest residual diagonal among the rows not chosen, ties to the smallest row
    double v = chosen ? -1.0 : dres;
    int idx = chosen ? T : tid;
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
      const double ov = __shfl_xor_sync(0xffffffffu, v, s);
      const int oi = __shfl_xor_sync(0xffffffffu, idx, s);
      if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; }
    }
    if (lane == 0) { red_v[warp] = v; red_i[warp] = idx; }
    __syncthreads();
    double dmax = red_v[0];
    int p = red_i[0];
    for (int w = 1; w < gp::FW; ++w)
      if (red_v[w] > dmax || (red_v[w] == dmax && red_i[w] < p)) { dmax = red_v[w]; p = red_i[w]; }
    if (!(dmax > tol)) break;                 // uniform; also stops on NaN
    const double piv = sqrt(dmax);
    if (tid < T) {
      double g = 0.0;
      if (tid == p) {
        g = piv;
        chosen = true;
      } else if (!chosen) {
        double s = rbf(xb + tid * F, xb + p * F, F, ls);
        for (int m = 0; m < k; ++m) s = fma(-G[m * ld + tid], G[m * ld + p], s);
        g = s / piv;
        dres = fma(-g, g, dres);
      }
      G[k * ld + tid] = g;
    }
    if (tid == 0) order[k] = p;
    rank = k + 1;
    __syncthreads();
  }
  if (tid < T) {
    double y = 0.0;
    for (int k = 0; k < rank; ++k) y = fma(G[k * ld + tid], static_cast<double>(D.z[o + k]), y);
    D.sample[o + tid] = static_cast<float>(y);
    taken[tid] = chosen ? 1 : 0;
  }
  if (tid == 0) D.rank[b] = rank;
  if (D.factor != nullptr) {
    double* fb = D.factor + static_cast<size_t>(b) * T * T;
    for (int e = tid; e < T * T; e += gp::FT) {
      const int i = e / T, k = e % T;
      fb[e] = k < rank ? G[k * ld + i] : 0.0;
    }
  }
  if (D.perm != nullptr) {
    __syncthreads();
    if (tid == 0) {
      int* pb = D.perm + o;
      for (int k = 0; k < rank; ++k) pb[k] = order[k];
      int k = rank;
      for (int i = 0; i < T; ++i)
        if (!taken[i]) pb[k++] = i;
    }
  }
}

}  // namespace
}  // namespace pfn

extern "C" int pfn_ridge_prefix(const pfn_ridge_prefix_desc* d, void* stream) {
  using namespace pfn;
  PFN_CHECK_ARG(d != nullptr, "ridge_prefix: null descriptor");
  PFN_CHECK_ARG(d->B > 0 && d->T > 0 && d->F > 0, "ridge_prefix: empty problem B=%d T=%d F=%d", d->B, d->T, d->F);
  PFN_CHECK_ARG(d->F <= PFN_RIDGE_MAX_F, "ridge_prefix: F=%d exceeds %d", d->F, PFN_RIDGE_MAX_F);
  PFN_CHECK_ARG(d->alpha >= 0.0 && d->alpha < INFINITY, "ridge_prefix: alpha=%g must be finite and >= 0", d->alpha);
  PFN_CHECK_ARG(d->x && d->y && d->target && d->pred && d->sq_err, "ridge_prefix: null pointer in the descriptor");
  static bool attr_set[64];
  if (first_use_on_device(attr_set))
    PFN_CUDA_OK(cudaFuncSetAttribute(ridge_prefix_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     static_cast<int>(ridge_smem(PFN_RIDGE_MAX_F))));
  ridge_prefix_kernel<<<d->B, kThreads, ridge_smem(d->F), reinterpret_cast<cudaStream_t>(stream)>>>(*d);
  PFN_LAUNCH_OK();
  return 0;
}

extern "C" int pfn_exact_gp(const pfn_exact_gp_desc* d, void* stream) {
  using namespace pfn;
  PFN_CHECK_ARG(d != nullptr, "exact_gp: null descriptor");
  PFN_CHECK_ARG(d->B > 0 && d->T > 0 && d->F > 0, "exact_gp: empty problem B=%d T=%d F=%d", d->B, d->T, d->F);
  PFN_CHECK_ARG(d->T <= PFN_GP_FIT_MAX_T, "exact_gp: T=%d exceeds %d (the T x T fp64 matrix lives in shared memory)", d->T,
                PFN_GP_FIT_MAX_T);
  PFN_CHECK_ARG(d->length_scale > 0.0 && d->length_scale < INFINITY, "exact_gp: length_scale=%g must be finite and > 0",
                d->length_scale);
  PFN_CHECK_ARG(d->mode == PFN_EXACT_GP_EVALUATE || d->mode == PFN_EXACT_GP_SAMPLE, "exact_gp: unknown mode %d", d->mode);
  PFN_CHECK_ARG(d->x != nullptr, "exact_gp: x is null");
  const bool evaluate = d->mode == PFN_EXACT_GP_EVALUATE;
  if (evaluate) {
    PFN_CHECK_ARG(d->alpha >= 0.0 && d->alpha < INFINITY, "exact_gp: alpha=%g must be finite and >= 0", d->alpha);
    PFN_CHECK_ARG(d->y && d->mean && d->var && d->status, "exact_gp: evaluate needs y, mean, var and status");
  } else {
    PFN_CHECK_ARG(d->z && d->sample && d->rank, "exact_gp: sample needs z, sample and rank");
  }
  const size_t smem = exact_gp_smem(d->T);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  static bool attr_set[64];
  if (first_use_on_device(attr_set)) {
    const int mx = static_cast<int>(exact_gp_smem(PFN_GP_FIT_MAX_T));
    PFN_CUDA_OK(cudaFuncSetAttribute(exact_gp_evaluate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, mx));
    PFN_CUDA_OK(cudaFuncSetAttribute(exact_gp_sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, mx));
  }
  if (evaluate)
    exact_gp_evaluate_kernel<<<d->B, gp::FT, smem, st>>>(*d);
  else
    exact_gp_sample_kernel<<<d->B, gp::FT, smem, st>>>(*d);
  PFN_LAUNCH_OK();
  return 0;
}
