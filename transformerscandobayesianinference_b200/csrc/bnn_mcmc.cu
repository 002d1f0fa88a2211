// NUTS baseline of the Bayesian NN (reference mcmc_svi_transformer_on_bayesian.py:249-267 eval_mcmc, model :28-67): one CTA
// per dataset runs a whole NUTS chain over theta = (W1 [E, F], b1 [E], W2 [2, E], b2 [2]), d = E F + 3 E + 2 coordinates,
// then forms the class-1 probability of every test row under every kept sample.  No host loop, no per-iteration launch.
// The chain is nuts.cuh's, shared with gp_mcmc.cu, with its tree-ordered reduction (TreeSum); its contract on the CPU is
// oracle/gp_mcmc_oracle.py (nuts_chain), which adds sequentially, so the two differ in the last bits of every sum.  See
// include/pfn_b200.h.
//
// The vector pool (PFN_BNN_MCMC_VECTORS - 1 vectors of d doubles) sits in dynamic shared memory after the data when it
// fits and in a caller-allocated global workspace otherwise; the trial point is always in shared memory.
//
// The potential: thread r forms row r's hidden vector, logits and softmax (dl = p - onehot, nll) from the data in shared
// memory; then thread i % NT accumulates dU/dtheta_i over the rows in order (dW1 = (W2^T dl) x^T, dW2 = dl h^T with h
// recomputed).  Compiled with -fmad=false: the sampler's arithmetic is the plain IEEE sequence the CPU restatement performs.
#include "common.cuh"
#include "nuts.cuh"

namespace pfn {
namespace {

using nuts::NT;
using Chain = nuts::Chain<nuts::TreeSum>;

constexpr double HALF_LOG_2PI = 0.9189385332046727;
constexpr size_t kMaxSmem = 200 * 1024;
static_assert(nuts::POOL_VECS + 1 == PFN_BNN_MCMC_VECTORS, "the trial point (always in shared memory) plus the pool");

// ------------------------------------------------------------------------------------------------ potential
// the two logits of a row under the parameters th
__device__ void row_logits(const double* th, int F, int E, const double* x, double& l0, double& l1) {
  const double *W1 = th, *b1 = th + E * F, *W2 = b1 + E, *b2 = W2 + 2 * E;
  l0 = b2[0];
  l1 = b2[1];
  for (int e = 0; e < E; ++e) {
    double h = b1[e];
    for (int f = 0; f < F; ++f) h = h + W1[e * F + f] * x[f];
    l0 = l0 + W2[e] * h;
    l1 = l1 + W2[E + e] * h;
  }
}

__device__ double logsumexp2(double l0, double l1) {
  const double m = l0 < l1 ? l1 : l0;
  return m + log(exp(l0 - m) + exp(l1 - m));
}

struct Model {
  const double* xs;                            // training rows [n, F]
  const int* ys;                               // their classes
  double *dl, *nll;                            // per row: p - onehot [n, 2] and -log p[y]
  int n, F, E;

  // d(sum_r nll_r)/d theta_i at th from the rows' dl, accumulated over the rows in order
  __device__ double grad_nll(const double* th, int i) const {
    const int EF = E * F;
    const double *W1 = th, *b1 = th + EF, *W2 = b1 + E;
    double acc = 0.0;
    if (i < EF + E) {                          // W1[e, f] (x_f) or b1[e] (1): dh_e = W2[0, e] dl_0 + W2[1, e] dl_1
      const int e = i < EF ? i / F : i - EF, f = i < EF ? i - e * F : -1;
      const double a0 = W2[e], a1 = W2[E + e];
      for (int r = 0; r < n; ++r) {
        const double dh = a0 * dl[2 * r] + a1 * dl[2 * r + 1];
        acc = acc + (f >= 0 ? dh * xs[r * F + f] : dh);
      }
    } else if (i < EF + 3 * E) {               // W2[k, e]: dl_k h_e
      const int k = (i - EF - E) / E, e = (i - EF - E) - k * E;
      for (int r = 0; r < n; ++r) {
        double h = b1[e];
        for (int f = 0; f < F; ++f) h = h + W1[e * F + f] * xs[r * F + f];
        acc = acc + dl[2 * r + k] * h;
      }
    } else {                                   // b2[k]
      const int k = i - EF - 3 * E;
      for (int r = 0; r < n; ++r) acc = acc + dl[2 * r + k];
    }
    return acc;
  }

  // nuts.cuh's model hook; NOT_PD counts the evaluations whose U is not finite
  template <class Fn>
  __device__ double evaluate(Chain& c, double& third, Fn per_elem) const {
    const int tid = threadIdx.x;
    for (int r = tid; r < n; r += NT) {
      double l0, l1;
      row_logits(c.trial, F, E, xs + r * F, l0, l1);
      const double lse = logsumexp2(l0, l1);
      const int y = ys[r];
      dl[2 * r] = exp(l0 - lse) - (y == 0 ? 1.0 : 0.0);
      dl[2 * r + 1] = exp(l1 - lse) - (y == 1 ? 1.0 : 0.0);
      nll[r] = lse - (y ? l1 : l0);
    }
    __syncthreads();
    double v[3] = {0.0, 0.0, 0.0};
    double* ge = c.vec(nuts::V_GE);
    for (int i = tid; i < c.d; i += NT) {
      const double th = c.trial[i];
      const double g = th + grad_nll(c.trial, i);
      ge[i] = g;
      v[0] = v[0] + th * th;
      v[2] = v[2] + per_elem(i, g);
    }
    for (int r = tid; r < n; r += NT) v[1] = v[1] + nll[r];
    c.sum(v);
    third = v[2];
    const double U = (0.5 * v[0] + c.d * HALF_LOG_2PI) + v[1];
    c.diag[PFN_GP_MCMC_EVALS]++;
    if (U < CUDART_INF) return U;
    c.diag[PFN_GP_MCMC_NOT_PD]++;
    return CUDART_INF;                         // NaN counts as +inf
  }
};

__host__ __device__ inline int bnn_dim(int F, int E) { return E * F + 3 * E + 2; }

// trial [d], x [n, F], dl [n, 2], nll [n] doubles, then the classes [n] as ints (padded to a double)
inline size_t data_smem(int d, int n, int F) {
  return (static_cast<size_t>(d) + static_cast<size_t>(n) * F + 3 * static_cast<size_t>(n) + (n + 1) / 2) * sizeof(double);
}
inline size_t pool_bytes(int d) { return static_cast<size_t>(nuts::POOL_VECS) * d * sizeof(double); }

__global__ void __launch_bounds__(NT, 1) bnn_mcmc_kernel(const pfn_bnn_mcmc_desc D, int pool_in_smem) {
  extern __shared__ __align__(16) double bnn_dyn[];
  __shared__ nuts::Shared<nuts::TreeSum> sh;
  const int tid = threadIdx.x, b = blockIdx.x;
  const int F = D.F, E = D.E, n = D.n, d = bnn_dim(F, E);
  const int W = D.warmup_steps, S = D.num_samples, So = S > 0 ? S : 1;
  double* trial = bnn_dyn;
  double* xs = trial + d;
  double* dl = xs + static_cast<size_t>(n) * F;
  double* nll = dl + 2 * n;
  int* ys = reinterpret_cast<int*>(nll + n);
  double* pool = pool_in_smem ? nll + n + (n + 1) / 2 : D.workspace + static_cast<size_t>(b) * nuts::POOL_VECS * d;
  Chain c;
  nuts::start(c, &sh, trial, pool, d, D.seed, static_cast<uint32_t>(b), static_cast<uint32_t>(n), W);
  for (int i = tid; i < n * F; i += NT) xs[i] = static_cast<double>(D.x_train[static_cast<size_t>(b) * n * F + i]);
  for (int i = tid; i < n; i += NT) ys[i] = D.y_train[static_cast<size_t>(b) * n + i] > 0.5f ? 1 : 0;
  const Model m{xs, ys, dl, nll, n, F, E};
  double* out = D.samples + static_cast<size_t>(b) * So * d;
  double* trace = D.trace ? D.trace + static_cast<size_t>(b) * (W + S) * (d + 2) : nullptr;
  const bool finite = nuts::run(c, m, D.init ? D.init + static_cast<size_t>(b) * d : nullptr, W, S, D.max_tree_depth, out,
                                trace);
  nuts::store_outputs(c, finite, W, S, b, out, D.potential, D.grad, D.step_size, D.accept);
  // ---- class-1 probability of every test row under every kept sample
  if (D.probs || D.obs) {
    c.key_it = static_cast<uint32_t>(W + S) + 1u;
    for (int k = 0; k < So; ++k) {
      __syncthreads();
      nuts::copy(trial, out + static_cast<size_t>(k) * d, d);
      __syncthreads();
      for (int j = tid; j < D.n_test; j += NT) {
        const float* xr = D.x_test + (static_cast<size_t>(b) * D.n_test + j) * F;
        double l0 = trial[d - 2], l1 = trial[d - 1];
        const double *W1 = trial, *b1 = W1 + E * F, *W2 = b1 + E;
        for (int e = 0; e < E; ++e) {
          double h = b1[e];
          for (int f = 0; f < F; ++f) h = h + W1[e * F + f] * static_cast<double>(xr[f]);
          l0 = l0 + W2[e] * h;
          l1 = l1 + W2[E + e] * h;
        }
        const double p1 = exp(l1 - logsumexp2(l0, l1));
        const size_t o = (static_cast<size_t>(b) * So + k) * D.n_test + j;
        if (D.probs) D.probs[o] = p1;
        if (D.obs) D.obs[o] = nuts::uniform_at(c, static_cast<uint32_t>(k) * D.n_test + j) < p1 ? 1.0f : 0.0f;
      }
    }
  }
  nuts::store_diag(c, D.diag + b * PFN_GP_MCMC_NDIAG);
}

// 0 on success with *in_smem set; the descriptor's sizes only (no pointers)
int check_sizes(const pfn_bnn_mcmc_desc* d, const char* who, int* in_smem) {
  PFN_CHECK_ARG(d != nullptr, "%s: null descriptor", who);
  PFN_CHECK_ARG(d->N > 0 && d->n > 0 && d->F > 0 && d->E > 0 && d->n_test >= 0,
                "%s: empty problem N=%d n=%d F=%d E=%d n_test=%d", who, d->N, d->n, d->F, d->E, d->n_test);
  const long long dim = static_cast<long long>(d->E) * d->F + 3LL * d->E + 2;
  PFN_CHECK_ARG(dim <= PFN_BNN_MAX_D, "%s: d = E F + 3 E + 2 = %lld exceeds %d", who, dim, PFN_BNN_MAX_D);
  PFN_CHECK_ARG(d->n <= PFN_BNN_MAX_N, "%s: n=%d training rows exceed %d", who, d->n, PFN_BNN_MAX_N);
  const size_t data = data_smem(static_cast<int>(dim), d->n, d->F);
  PFN_CHECK_ARG(data <= kMaxSmem, "%s: n=%d rows of F=%d features need %zu bytes of shared memory (limit %zu)", who, d->n,
                d->F, data, kMaxSmem);
  *in_smem = data + pool_bytes(static_cast<int>(dim)) <= kMaxSmem;
  return 0;
}

}  // namespace
}  // namespace pfn

using namespace pfn;

extern "C" int pfn_bnn_mcmc_workspace(const pfn_bnn_mcmc_desc* d) {
  int in_smem = 0;
  if (check_sizes(d, "bnn_mcmc_workspace", &in_smem) != 0) return -1;
  return in_smem ? 0 : nuts::POOL_VECS * bnn_dim(d->F, d->E);
}

extern "C" int pfn_bnn_mcmc(const pfn_bnn_mcmc_desc* d, void* stream) {
  int in_smem = 0;
  if (const int rc = check_sizes(d, "bnn_mcmc", &in_smem)) return rc;
  if (const int rc = nuts::check_chain(d, "bnn_mcmc", d->x_train && d->y_train)) return rc;
  PFN_CHECK_ARG(d->n_test == 0 || (d->probs == nullptr && d->obs == nullptr) || d->x_test != nullptr,
                "bnn_mcmc: probs or obs wanted but x_test is null");
  PFN_CHECK_ARG(in_smem || d->workspace != nullptr,
                "bnn_mcmc: the sampler state of d=%d does not fit in shared memory and workspace is null", bnn_dim(d->F, d->E));
  const int dim = bnn_dim(d->F, d->E);
  const size_t smem = data_smem(dim, d->n, d->F) + (in_smem ? pool_bytes(dim) : 0);
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set))
    PFN_CUDA_OK(cudaFuncSetAttribute(bnn_mcmc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     static_cast<int>(kMaxSmem)));
  bnn_mcmc_kernel<<<d->N, NT, smem, reinterpret_cast<cudaStream_t>(stream)>>>(*d, in_smem);
  PFN_LAUNCH_OK();
  return 0;
}
