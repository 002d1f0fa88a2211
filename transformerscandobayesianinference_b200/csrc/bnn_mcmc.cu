// NUTS baseline of the Bayesian NN (reference mcmc_svi_transformer_on_bayesian.py:249-267 eval_mcmc, model :28-67): one CTA
// per dataset runs a whole NUTS chain over theta = (W1 [E, F], b1 [E], W2 [2, E], b2 [2]), d = E F + 3 E + 2 coordinates,
// then forms the class-1 probability of every test row under every kept sample.  No host loop, no per-iteration launch.
// The algorithm, constants and random-number keys are those of gp_mcmc.cu and of oracle/gp_mcmc_oracle.py (nuts_chain),
// which is its contract on the CPU; see include/pfn_b200.h.
//
// Where gp_mcmc.cu keeps its <= 7-coordinate state in one struct and does the vector work on thread 0, the state here is a
// pool of d-vectors (chain state, trajectory ends, the per-level stack of complete subtrees, Welford accumulators) in
// dynamic shared memory when it fits and in a caller-allocated global workspace otherwise.  Element i of every vector is
// always touched by thread i % NT, so chains of elementwise updates (leapfrog halves, copies, subtree merges, Welford)
// need no barrier; barriers separate them only from the potential, which reads the whole trial point, and from the
// reductions (kinetic energy, U-turn dot products, |theta|^2, the summed log-likelihood).  A reduction adds per-thread
// partials in a fixed order (butterfly within a warp, then the warps in sequence) and hands every thread the same bits,
// so the chain's scalars (energies, weights, step size, dual averaging, counters, the counter-based random draws) are
// kept redundantly in registers by all threads and every branch is uniform without a broadcast.  Nothing depends on
// which other chains share the launch.
//
// The potential: thread r forms row r's hidden vector, logits and softmax (dl = p - onehot, nll) from the data in shared
// memory; then thread i % NT accumulates dU/dtheta_i over the rows in order (dW1 = (W2^T dl) x^T, dW2 = dl h^T with h
// recomputed).  Compiled with -fmad=false: the sampler's arithmetic is the plain IEEE sequence the CPU restatement performs.
#include <math_constants.h>

#include "common.cuh"
#include "counter_rng.cuh"
#include "../../include/pfn_b200.h"

namespace pfn {
namespace {

constexpr int NT = 256, NW = NT / 32;
constexpr int MAXD = PFN_GP_MCMC_MAX_DEPTH;
constexpr int MAX_WINDOWS = 40;
constexpr double TARGET_ACCEPT = 0.8;          // dual averaging (pyro.ops.dual_averaging, Stan's constants)
constexpr double DA_GAMMA = 0.05, DA_T0 = 10.0, DA_KAPPA = 0.75;
constexpr double MAX_ENERGY_ERROR = 1000.0;    // pyro NUTS _max_sliced_energy
constexpr double LOG_ACCEPT_THRESHOLD = -0.2231435513142097;    // log(0.8), the step-size search's direction threshold
constexpr int SEARCH_MAX = 100;                // doublings / halvings per step-size search (pyro has no cap)
constexpr int INIT_TRIES = 100;                // uniform initial points tried until the potential is finite (pyro's)
constexpr double TWO_PI = 6.283185307179586;
constexpr double HALF_LOG_2PI = 0.9189385332046727;
constexpr size_t kMaxSmem = 200 * 1024;

// the vector pool; a node (a complete subtree of the doubling in progress) is five vectors: the whitened momenta of its
// first / last leaf, their sum over its leaves, and its multinomial proposal (z, g)
enum { V_Z, V_G, V_INV_M, V_SQRT_IM, V_RSQRT_IM, V_EZ, V_ER = V_EZ + 2, V_EG = V_ER + 2, V_EW = V_EG + 2, V_WSUM = V_EW + 2,
       V_RHALF, V_WF_MEAN, V_WF_M2, V_GE, V_NODES };
enum { N_WFIRST, N_WLAST, N_WSUM, N_Z, N_G, NODE_VECS };
constexpr int CUR = MAXD + 1;                  // node index of the subtree being built; 0 .. MAXD are the stack levels
constexpr int POOL_VECS = V_NODES + (MAXD + 2) * NODE_VECS;
static_assert(POOL_VECS + 1 == PFN_BNN_MCMC_VECTORS, "the trial point (always in shared memory) plus the pool");

struct Shared {                                // written by thread 0 only, read by all after a barrier
  double node_pe[MAXD + 1], node_weight[MAXD + 1];
  int win_end[MAX_WINDOWS];
  double red[2][NW][3];
};

struct Ctx {                                   // per-thread view of the chain; the scalars are identical on all threads
  Shared* sh;
  double *trial, *pool;                        // the point being evaluated [d] (shared) and the vector pool
  const double* xs;                            // training rows [n, F]
  const int* ys;                               // their classes
  double *dl, *nll;                            // per row: p - onehot [n, 2] and -log p[y]
  int d, n, F, E, parity;
  uint32_t seed, key_b, key_t, key_it, ctr;
  double pe, eps;
  double da_center, da_x, da_xavg, da_gavg;
  int da_t, wf_n, nwin, cw;
  int diag[PFN_GP_MCMC_NDIAG];
  __device__ double* vec(int slot) const { return pool + static_cast<size_t>(slot) * d; }
  __device__ double* node(int k, int which) const { return vec(V_NODES + k * NODE_VECS + which); }
};

// Sums v[0..K) over the CTA in a fixed order; every thread returns with the same bits.  The two buffers alternate, so a
// call's partials are never overwritten before every thread has read them.
template <int K>
__device__ void block_sum(Ctx& c, double (&v)[K]) {
  const int tid = threadIdx.x;
#pragma unroll
  for (int k = 0; k < K; ++k)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] = v[k] + __shfl_xor_sync(0xffffffffu, v[k], o);
  double(*red)[3] = c.sh->red[c.parity];
  c.parity ^= 1;
  if ((tid & 31) == 0)
#pragma unroll
    for (int k = 0; k < K; ++k) red[tid >> 5][k] = v[k];
  __syncthreads();
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double s = red[0][k];
    for (int w = 1; w < NW; ++w) s = s + red[w][k];
    v[k] = s;
  }
}

// ------------------------------------------------------------------------------------------------ random numbers
// Draw k of iteration key `it` is uniform_double(hash5(seed, b, n, it, 2k), hash5(.., 2k + 1)).
__device__ double uniform_at(const Ctx& c, uint32_t k) {
  return uniform_double(hash5(c.seed, c.key_b, c.key_t, c.key_it, 2u * k), hash5(c.seed, c.key_b, c.key_t, c.key_it, 2u * k + 1u));
}
__device__ double uniform(Ctx& c) { return uniform_at(c, c.ctr++); }
// Box-Muller, cosine branch, from draws k and k + 1; 1 - U is in (0, 1]
__device__ double normal_at(const Ctx& c, uint32_t k) {
  const double u1 = 1.0 - uniform_at(c, k);
  const double u2 = uniform_at(c, k + 1u);
  return sqrt(-2.0 * log(u1)) * cos(TWO_PI * u2);
}

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

// d(sum_r nll_r)/d theta_i from the rows' dl, accumulated over the rows in order
__device__ double grad_nll(const Ctx& c, int i) {
  const int F = c.F, E = c.E, n = c.n, EF = E * F;
  const double *th = c.trial, *W1 = th, *b1 = th + EF, *W2 = b1 + E;
  double acc = 0.0;
  if (i < EF + E) {                            // W1[e, f] (x_f) or b1[e] (1): dh_e = W2[0, e] dl_0 + W2[1, e] dl_1
    const int e = i < EF ? i / F : i - EF, f = i < EF ? i - e * F : -1;
    const double a0 = W2[e], a1 = W2[E + e];
    for (int r = 0; r < n; ++r) {
      const double dh = a0 * c.dl[2 * r] + a1 * c.dl[2 * r + 1];
      acc = acc + (f >= 0 ? dh * c.xs[r * F + f] : dh);
    }
  } else if (i < EF + 3 * E) {                 // W2[k, e]: dl_k h_e
    const int k = (i - EF - E) / E, e = (i - EF - E) - k * E;
    for (int r = 0; r < n; ++r) {
      double h = b1[e];
      for (int f = 0; f < F; ++f) h = h + W1[e * F + f] * c.xs[r * F + f];
      acc = acc + c.dl[2 * r + k] * h;
    }
  } else {                                     // b2[k]
    const int k = i - EF - 3 * E;
    for (int r = 0; r < n; ++r) acc = acc + c.dl[2 * r + k];
  }
  return acc;
}

// U and its gradient (into V_GE) at the trial point, which every thread may read on entry.  per_elem(i, g_i) runs on the
// owner of element i right after g_i is known and returns a term of a third sum (the fused second leapfrog half returns
// w_i^2); its total comes back in `third`.  Returns U, +inf when it is not finite (the gradient is then not used: the
// trajectory ends as a divergence).
template <class Fn>
__device__ double evaluate(Ctx& c, double& third, Fn per_elem) {
  const int tid = threadIdx.x;
  for (int r = tid; r < c.n; r += NT) {
    double l0, l1;
    row_logits(c.trial, c.F, c.E, c.xs + r * c.F, l0, l1);
    const double lse = logsumexp2(l0, l1);
    const int y = c.ys[r];
    c.dl[2 * r] = exp(l0 - lse) - (y == 0 ? 1.0 : 0.0);
    c.dl[2 * r + 1] = exp(l1 - lse) - (y == 1 ? 1.0 : 0.0);
    c.nll[r] = lse - (y ? l1 : l0);
  }
  __syncthreads();
  double v[3] = {0.0, 0.0, 0.0};
  double* ge = c.vec(V_GE);
  for (int i = tid; i < c.d; i += NT) {
    const double th = c.trial[i];
    const double g = th + grad_nll(c, i);
    ge[i] = g;
    v[0] = v[0] + th * th;
    v[2] = v[2] + per_elem(i, g);
  }
  for (int r = tid; r < c.n; r += NT) v[1] = v[1] + c.nll[r];
  block_sum(c, v);
  third = v[2];
  const double U = (0.5 * v[0] + c.d * HALF_LOG_2PI) + v[1];
  c.diag[PFN_GP_MCMC_EVALS]++;
  if (U < CUDART_INF) return U;
  c.diag[PFN_GP_MCMC_NOT_PD]++;
  return CUDART_INF;                           // NaN counts as +inf
}

// ------------------------------------------------------------------------------------------------ NUTS
__device__ double logaddexp(double x, double y) {                 // pyro's _logaddexp
  const double mn = x < y ? x : y, mx = x < y ? y : x;
  return log1p(exp(mn - mx)) + mx;
}

// momentum draw: whitened w ~ N(0, I) into slot wv, r = M^1/2 w into slot rv; returns the kinetic energy
__device__ double draw_momentum(Ctx& c, int rv, int wv) {
  double *r = c.vec(rv), *w = c.vec(wv);
  const double* rsqrt_im = c.vec(V_RSQRT_IM);
  double v[1] = {0.0};
  for (int i = threadIdx.x; i < c.d; i += NT) {
    const double wi = normal_at(c, c.ctr + 2u * i);
    w[i] = wi;
    r[i] = wi * rsqrt_im[i];
    v[0] = v[0] + wi * wi;
  }
  c.ctr += 2u * c.d;
  block_sum(c, v);
  return 0.5 * v[0];
}

// first half of a leapfrog step from (z, r, g) with signed step e: rhalf and the trial point
__device__ void leapfrog_begin(Ctx& c, int zv, int rv, int gv, double e) {
  const double h = 0.5 * e;
  const double *z = c.vec(zv), *r = c.vec(rv), *g = c.vec(gv), *inv_m = c.vec(V_INV_M);
  double* rhalf = c.vec(V_RHALF);
  for (int i = threadIdx.x; i < c.d; i += NT) {
    rhalf[i] = r[i] + h * (-g[i]);
    c.trial[i] = z[i] + e * (inv_m[i] * rhalf[i]);
  }
  __syncthreads();
}

// generalised no-U-turn criterion in whitened momenta (pyro NUTS._is_turning)
__device__ int is_turning(Ctx& c, const double* wl, const double* wr, const double* wsum) {
  double v[2] = {0.0, 0.0};
  for (int i = threadIdx.x; i < c.d; i += NT) {
    const double rho = wsum[i] - (wl[i] + wr[i]) / 2.0;
    v[0] = v[0] + wl[i] * rho;
    v[1] = v[1] + wr[i] * rho;
  }
  block_sum(c, v);
  return v[0] <= 0.0 || v[1] <= 0.0;
}

__device__ void copy(double* dst, const double* src, int d) {
  for (int i = threadIdx.x; i < d; i += NT) dst[i] = src[i];
}

// Stan's windows as pyro builds them (adaptation.WarmupAdapter._build_adaptation_schedule): end index of every window
__device__ int build_schedule(int* win_end, int W, bool store) {
  int nwin = 0;
  auto push = [&](int v) {
    if (store) win_end[nwin] = v;
    nwin++;
  };
  if (W < 20) {
    push(W - 1);
    return nwin;
  }
  int start_buf = 75, end_buf = 50, init_win = 25;
  if (start_buf + end_buf + init_win > W) {
    start_buf = static_cast<int>(0.15 * W);
    end_buf = static_cast<int>(0.1 * W);
    init_win = W - start_buf - end_buf;
  }
  push(start_buf - 1);
  const int end_start = W - end_buf;
  int next_size = init_win, next_start = start_buf;
  while (next_start < end_start && nwin < MAX_WINDOWS - 1) {
    const int cur_start = next_start;
    int cur_size = next_size;
    if (3 * cur_size <= end_start - cur_start) next_size = 2 * cur_size;
    else cur_size = end_start - cur_start;
    next_start = cur_start + cur_size;
    push(next_start - 1);
  }
  push(W - 1);
  return nwin;
}

// step-size search from the chain's state (pyro HMC._find_reasonable_step_size), then a fresh dual-averaging centre
__device__ void step_size_search(Ctx& c) {
  bool first = true;
  int count = 0, s_dir = 0;
  double scale = 1.0;
  const double *rhalf = c.vec(V_RHALF), *sqrt_im = c.vec(V_SQRT_IM);
  for (;;) {
    if (!first) c.eps = scale * c.eps;
    const double e0 = draw_momentum(c, V_ER, V_EW) + c.pe;   // scratch: the trajectory ends are free between iterations
    leapfrog_begin(c, V_Z, V_ER, V_G, c.eps);
    const double h = 0.5 * c.eps;
    double ww;
    const double U = evaluate(c, ww, [&](int i, double g) {
      const double w = (rhalf[i] + h * (-g)) * sqrt_im[i];
      return w * w;
    });
    double en = U + 0.5 * ww;
    if (!(en == en)) en = CUDART_INF;
    const double delta = en - e0;
    const int dir = LOG_ACCEPT_THRESHOLD < -delta ? 1 : -1;
    if (first) {
      first = false;
      s_dir = dir;
      scale = dir == 1 ? 2.0 : 0.5;
      continue;
    }
    if (dir != s_dir) break;
    if (!(++count < SEARCH_MAX)) break;
  }
  c.da_center = log(10.0 * c.eps);
  c.da_xavg = 0.0;
  c.da_gavg = 0.0;
  c.da_t = 0;
}

// One NUTS iteration from the chain's state; returns the mean acceptance statistic and the tree depth.
__device__ double iteration(Ctx& c, int it, int W, int max_depth, int& depth_out) {
  const int tid = threadIdx.x, d = c.d;
  Shared& sh = *c.sh;
  c.key_it = static_cast<uint32_t>(it) + 1u;
  c.ctr = 0;
  const double energy0 = draw_momentum(c, V_ER, V_EW) + c.pe;
  {
    const double *z = c.vec(V_Z), *g = c.vec(V_G), *r0 = c.vec(V_ER), *w0 = c.vec(V_EW);
    double *ez0 = c.vec(V_EZ), *ez1 = c.vec(V_EZ + 1), *eg0 = c.vec(V_EG), *eg1 = c.vec(V_EG + 1);
    double *r1 = c.vec(V_ER + 1), *w1 = c.vec(V_EW + 1), *wsum = c.vec(V_WSUM);
    for (int i = tid; i < d; i += NT) {
      r1[i] = r0[i];
      w1[i] = w0[i];
      ez0[i] = ez1[i] = z[i];
      eg0[i] = eg1[i] = g[i];
      wsum[i] = w0[i];
    }
  }
  double weight = 0.0, acc_sum = 0.0;
  int n_prop = 0, depth = 0;
  const double *rhalf = c.vec(V_RHALF), *sqrt_im = c.vec(V_SQRT_IM), *ge = c.vec(V_GE);
  double *Cwf = c.node(CUR, N_WFIRST), *Cwl = c.node(CUR, N_WLAST), *Cws = c.node(CUR, N_WSUM);
  double *Cz = c.node(CUR, N_Z), *Cg = c.node(CUR, N_G);
  for (;;) {                                   // doubling
    const int s = uniform(c) < 0.5 ? 1 : 0;
    const double e = s ? c.eps : -c.eps, h = 0.5 * e;
    double *ez = c.vec(V_EZ + s), *er = c.vec(V_ER + s), *eg = c.vec(V_EG + s), *ew = c.vec(V_EW + s);
    double sub_acc = 0.0, Cpe = 0.0, Cweight = 0.0;
    int sub_n = 0, status = 1;                 // 1 = subtree complete, 2 = turning, 3 = divergent
    for (int leaf = 0; leaf < (1 << depth); ++leaf) {
      leapfrog_begin(c, V_EZ + s, V_ER + s, V_EG + s, e);
      double ww;
      const double U = evaluate(c, ww, [&](int i, double g) {   // second half: the end of the trajectory moves on
        const double r = rhalf[i] + h * (-g);
        const double w = r * sqrt_im[i];
        er[i] = r;
        ew[i] = w;
        ez[i] = c.trial[i];
        eg[i] = g;
        return w * w;
      });
      c.diag[PFN_GP_MCMC_LEAPFROG]++;
      double en = U + 0.5 * ww;
      if (!(en == en)) en = CUDART_INF;
      const double sliced = en + (-energy0);
      const double acc = exp(-(en - energy0));
      sub_acc = sub_acc + (acc < 1.0 ? acc : 1.0);
      sub_n++;
      if (sliced > MAX_ENERGY_ERROR) {
        status = 3;
        break;
      }
      for (int i = tid; i < d; i += NT) {
        Cwf[i] = Cwl[i] = Cws[i] = ew[i];
        Cz[i] = c.trial[i];
        Cg[i] = ge[i];
      }
      Cpe = U;
      Cweight = -sliced;
      int lvl = 0;
      for (; (leaf >> lvl) & 1; ++lvl) {       // merge with the earlier subtree of the same size (first half)
        const double w = logaddexp(sh.node_weight[lvl], Cweight);
        const double p_other = exp(Cweight - w);
        const bool keep_first = !(uniform(c) < p_other);
        if (keep_first) Cpe = sh.node_pe[lvl];
        Cweight = w;
        const double *Hwf = c.node(lvl, N_WFIRST), *Hws = c.node(lvl, N_WSUM), *Hz = c.node(lvl, N_Z), *Hg = c.node(lvl, N_G);
        for (int i = tid; i < d; i += NT) {
          if (keep_first) {
            Cz[i] = Hz[i];
            Cg[i] = Hg[i];
          }
          Cws[i] = Hws[i] + Cws[i];
          Cwf[i] = Hwf[i];
        }
        if (is_turning(c, Cwf, Cwl, Cws)) {
          status = 2;
          break;
        }
      }
      if (status == 2) break;
      if (leaf + 1 < (1 << depth)) {
        for (int k = 0; k < NODE_VECS; ++k) copy(c.node(lvl, k), c.node(CUR, k), d);
        if (tid == 0) {
          sh.node_pe[lvl] = Cpe;
          sh.node_weight[lvl] = Cweight;
        }
      }
    }
    acc_sum = acc_sum + sub_acc;
    n_prop += sub_n;
    if (status == 3) {
      if (it < W) c.diag[PFN_GP_MCMC_DIV_WARMUP]++;
      else c.diag[PFN_GP_MCMC_DIV_SAMPLING]++;
      break;
    }
    if (status == 2) break;
    depth++;
    const double p_new = exp(Cweight - weight);
    const bool take = uniform(c) < p_new;      // biased progressive sampling
    double *z = c.vec(V_Z), *g = c.vec(V_G), *wsum = c.vec(V_WSUM);
    for (int i = tid; i < d; i += NT) {
      if (take) {
        z[i] = Cz[i];
        g[i] = Cg[i];
      }
      wsum[i] = wsum[i] + Cws[i];
    }
    if (take) c.pe = Cpe;
    if (is_turning(c, c.vec(V_EW), c.vec(V_EW + 1), wsum)) break;
    weight = logaddexp(weight, Cweight);
    if (depth >= max_depth) {
      c.diag[PFN_GP_MCMC_MAX_DEPTH_HITS]++;
      break;
    }
  }
  depth_out = depth;
  return acc_sum / n_prop;
}

// Warmup adaptation after iteration it (pyro WarmupAdapter.step at t = it + 1).  Returns 1 when a step-size search follows.
__device__ int adapt(Ctx& c, int it, double accept_prob, int W) {
  const int t = it + 1, tid = threadIdx.x;
  if (t >= W) return 0;
  const int mm = c.cw > 0 && c.cw < c.nwin - 1;
  c.da_t++;
  const double tt = c.da_t + DA_T0;
  c.da_gavg = (1.0 - 1.0 / tt) * c.da_gavg + (TARGET_ACCEPT - accept_prob) / tt;
  c.da_x = c.da_center - sqrt(static_cast<double>(c.da_t)) / DA_GAMMA * c.da_gavg;
  const double wt = pow(static_cast<double>(c.da_t), -DA_KAPPA);
  c.da_xavg = (1.0 - wt) * c.da_xavg + wt * c.da_x;
  c.eps = exp(c.da_x);
  const double* z = c.vec(V_Z);
  double *wf_mean = c.vec(V_WF_MEAN), *wf_m2 = c.vec(V_WF_M2);
  if (mm) {
    c.wf_n++;
    for (int i = tid; i < c.d; i += NT) {
      const double pre = z[i] - wf_mean[i];
      wf_mean[i] = wf_mean[i] + pre / c.wf_n;
      const double post = z[i] - wf_mean[i];
      wf_m2[i] = wf_m2[i] + pre * post;
    }
  }
  if (t != c.sh->win_end[c.cw]) return 0;
  if (c.cw == c.nwin - 1) {
    c.cw++;
    c.eps = exp(c.da_xavg);
    return 0;
  }
  if (c.cw == 0) {
    c.cw++;
    return 0;
  }
  const double n = c.wf_n;
  double *inv_m = c.vec(V_INV_M), *sqrt_im = c.vec(V_SQRT_IM), *rsqrt_im = c.vec(V_RSQRT_IM);
  for (int i = tid; i < c.d; i += NT) {
    const double cov = wf_m2[i] / (n - 1.0);
    const double v = (n / (n + 5.0)) * cov + 1e-3 * (5.0 / (n + 5.0));
    inv_m[i] = v;
    sqrt_im[i] = sqrt(v);
    rsqrt_im[i] = 1.0 / sqrt(v);
    wf_mean[i] = 0.0;
    wf_m2[i] = 0.0;
  }
  c.wf_n = 0;
  c.cw++;
  return 1;
}

inline int bnn_dim(int F, int E) { return E * F + 3 * E + 2; }

// trial [d], x [n, F], dl [n, 2], nll [n] doubles, then the classes [n] as ints (padded to a double)
inline size_t data_smem(int d, int n, int F) {
  return (static_cast<size_t>(d) + static_cast<size_t>(n) * F + 3 * static_cast<size_t>(n) + (n + 1) / 2) * sizeof(double);
}
inline size_t pool_bytes(int d) { return static_cast<size_t>(POOL_VECS) * d * sizeof(double); }

__global__ void __launch_bounds__(NT, 1) bnn_mcmc_kernel(const pfn_bnn_mcmc_desc D, int pool_in_smem) {
  extern __shared__ __align__(16) double bnn_dyn[];
  __shared__ Shared sh;
  const int tid = threadIdx.x, b = blockIdx.x;
  const int F = D.F, E = D.E, n = D.n, d = E * F + 3 * E + 2;
  const int W = D.warmup_steps, S = D.num_samples, So = S > 0 ? S : 1;
  Ctx c;
  c.sh = &sh;
  c.trial = bnn_dyn;
  double* xs = c.trial + d;
  c.dl = xs + static_cast<size_t>(n) * F;
  c.nll = c.dl + 2 * n;
  int* ys = reinterpret_cast<int*>(c.nll + n);
  c.pool = pool_in_smem ? c.nll + n + (n + 1) / 2 : D.workspace + static_cast<size_t>(b) * POOL_VECS * d;
  c.xs = xs;
  c.ys = ys;
  c.d = d; c.n = n; c.F = F; c.E = E; c.parity = 0;
  c.seed = D.seed;
  c.key_b = static_cast<uint32_t>(b);
  c.key_t = static_cast<uint32_t>(n);
  c.key_it = 0;
  c.ctr = 0;
  c.pe = 0.0;
  c.eps = 1.0;
  c.da_center = c.da_x = c.da_xavg = c.da_gavg = 0.0;
  c.da_t = 0; c.wf_n = 0; c.cw = 0;
  for (int k = 0; k < PFN_GP_MCMC_NDIAG; ++k) c.diag[k] = 0;
  c.nwin = build_schedule(sh.win_end, W, tid == 0);

  for (int i = tid; i < n * F; i += NT) xs[i] = static_cast<double>(D.x_train[static_cast<size_t>(b) * n * F + i]);
  for (int i = tid; i < n; i += NT) ys[i] = D.y_train[static_cast<size_t>(b) * n + i] > 0.5f ? 1 : 0;
  {
    double *inv_m = c.vec(V_INV_M), *sqrt_im = c.vec(V_SQRT_IM), *rsqrt_im = c.vec(V_RSQRT_IM);
    double *wf_mean = c.vec(V_WF_MEAN), *wf_m2 = c.vec(V_WF_M2);
    for (int i = tid; i < d; i += NT) {
      inv_m[i] = sqrt_im[i] = rsqrt_im[i] = 1.0;
      wf_mean[i] = wf_m2[i] = 0.0;
    }
  }
  double* out = D.samples + static_cast<size_t>(b) * So * d;
  auto none = [](int, double) { return 0.0; };

  // ---- initial point: the caller's, or theta ~ U(-2, 2) until the potential is finite
  bool finite = false;
  for (int attempt = 0;; ++attempt) {
    for (int i = tid; i < d; i += NT)
      c.trial[i] = D.init ? D.init[static_cast<size_t>(b) * d + i] : -2.0 + 4.0 * uniform_at(c, c.ctr + i);
    c.ctr += d;
    __syncthreads();
    double unused;
    c.pe = evaluate(c, unused, none);
    finite = c.pe < CUDART_INF;
    if (D.init != nullptr || finite || attempt + 1 >= INIT_TRIES) break;
  }
  copy(c.vec(V_Z), c.trial, d);
  copy(c.vec(V_G), c.vec(V_GE), d);
  const bool run = finite && W + S > 0;
  if (run) {
    step_size_search(c);
    double acc_sampling = 0.0;
    for (int it = 0; it < W + S; ++it) {
      const double eps_used = c.eps;
      int depth;
      const double accept_prob = iteration(c, it, W, D.max_tree_depth, depth);
      const double* z = c.vec(V_Z);
      if (D.trace) {
        double* row = D.trace + (static_cast<size_t>(b) * (W + S) + it) * (d + 2);
        copy(row, z, d);
        if (tid == 0) {
          row[d] = eps_used;
          row[d + 1] = depth;
        }
      }
      if (it >= W) {
        copy(out + static_cast<size_t>(it - W) * d, z, d);
        acc_sampling = acc_sampling + accept_prob;
      } else if (adapt(c, it, accept_prob, W)) {
        step_size_search(c);
      }
    }
    if (S == 0) copy(out, c.vec(V_Z), d);      // warmup only: the one output row is the state the warmup ended in
    if (tid == 0) {
      D.step_size[b] = c.eps;
      D.accept[b] = S > 0 ? acc_sampling / S : CUDART_NAN;
    }
  } else {
    // evaluate-only (W = S = 0): the point itself; no finite starting point: the chain is not run and says so with NaN
    const double* z = c.vec(V_Z);
    for (int k = 0; k < So; ++k)
      for (int i = tid; i < d; i += NT) out[static_cast<size_t>(k) * d + i] = finite || W + S == 0 ? z[i] : CUDART_NAN;
    if (D.trace)
      for (size_t i = tid; i < static_cast<size_t>(W + S) * (d + 2); i += NT)
        D.trace[static_cast<size_t>(b) * (W + S) * (d + 2) + i] = CUDART_NAN;
    if (tid == 0) {
      D.step_size[b] = finite ? 0.0 : CUDART_NAN;
      D.accept[b] = CUDART_NAN;
    }
  }
  if (D.potential && tid == 0) D.potential[b] = c.pe;
  if (D.grad) {
    const double* g = c.vec(V_G);
    for (int i = tid; i < d; i += NT) D.grad[static_cast<size_t>(b) * d + i] = finite ? g[i] : CUDART_NAN;
  }
  // ---- class-1 probability of every test row under every kept sample
  if (D.probs || D.obs) {
    c.key_it = static_cast<uint32_t>(W + S) + 1u;
    for (int k = 0; k < So; ++k) {
      __syncthreads();
      copy(c.trial, out + static_cast<size_t>(k) * d, d);
      __syncthreads();
      for (int j = tid; j < D.n_test; j += NT) {
        const float* xr = D.x_test + (static_cast<size_t>(b) * D.n_test + j) * F;
        double l0 = c.trial[d - 2], l1 = c.trial[d - 1];
        const double *W1 = c.trial, *b1 = W1 + E * F, *W2 = b1 + E;
        for (int e = 0; e < E; ++e) {
          double h = b1[e];
          for (int f = 0; f < F; ++f) h = h + W1[e * F + f] * static_cast<double>(xr[f]);
          l0 = l0 + W2[e] * h;
          l1 = l1 + W2[E + e] * h;
        }
        const double p1 = exp(l1 - logsumexp2(l0, l1));
        const size_t o = (static_cast<size_t>(b) * So + k) * D.n_test + j;
        if (D.probs) D.probs[o] = p1;
        if (D.obs) D.obs[o] = uniform_at(c, static_cast<uint32_t>(k) * D.n_test + j) < p1 ? 1.0f : 0.0f;
      }
    }
  }
  if (tid == 0)
    for (int k = 0; k < PFN_GP_MCMC_NDIAG; ++k) D.diag[b * PFN_GP_MCMC_NDIAG + k] = c.diag[k];
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
  return in_smem ? 0 : POOL_VECS * bnn_dim(d->F, d->E);
}

extern "C" int pfn_bnn_mcmc(const pfn_bnn_mcmc_desc* d, void* stream) {
  int in_smem = 0;
  if (const int rc = check_sizes(d, "bnn_mcmc", &in_smem)) return rc;
  PFN_CHECK_ARG(d->x_train && d->y_train && d->samples && d->step_size && d->accept && d->diag,
                "bnn_mcmc: null input or output pointer");
  PFN_CHECK_ARG(d->n_test == 0 || (d->probs == nullptr && d->obs == nullptr) || d->x_test != nullptr,
                "bnn_mcmc: probs or obs wanted but x_test is null");
  PFN_CHECK_ARG(d->num_samples >= 0 && d->warmup_steps >= 0, "bnn_mcmc: negative num_samples=%d or warmup_steps=%d",
                d->num_samples, d->warmup_steps);
  PFN_CHECK_ARG(static_cast<long long>(d->num_samples) + d->warmup_steps <= 0x7fffffffLL, "bnn_mcmc: too many iterations");
  PFN_CHECK_ARG(d->num_samples + d->warmup_steps > 0 || d->init != nullptr,
                "bnn_mcmc: warmup_steps = num_samples = 0 evaluates at init, which is null");
  PFN_CHECK_ARG(d->max_tree_depth >= 1 && d->max_tree_depth <= PFN_GP_MCMC_MAX_DEPTH,
                "bnn_mcmc: max_tree_depth=%d outside [1, %d]", d->max_tree_depth, PFN_GP_MCMC_MAX_DEPTH);
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
