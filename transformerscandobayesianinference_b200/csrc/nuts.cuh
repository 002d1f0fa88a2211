// The NUTS chain of the two MCMC baselines (gp_mcmc.cu, bnn_mcmc.cu): pyro 1.7's NUTS at its defaults (multinomial
// sampling, generalised no-U-turn criterion, divergence at an energy error above 1000, step size found by doubling /
// halving and adapted by dual averaging to acceptance 0.8, diagonal mass matrix adapted in Stan's windows), written out on
// the CPU by oracle/gp_mcmc_oracle.py (nuts_chain), which is its contract.
//
// One CTA of NT threads runs one chain.  Its state is a pool of d-vectors (chain state, trajectory ends, the per-level
// stack of complete subtrees, Welford accumulators) wherever the kernel puts it.  Element i of every vector is always
// touched by thread i % NT, so chains of elementwise updates (leapfrog halves, copies, subtree merges, Welford) need no
// barrier; barriers separate them only from the potential, which reads the whole trial point, and from the reductions
// (kinetic energy, U-turn dot products).  A reduction hands every thread the same bits, so the chain's scalars (energies,
// weights, step size, dual averaging, counters, the counter-based random draws) are kept redundantly in registers by all
// threads and every branch is uniform without a broadcast.  The tree is built iteratively: the complete subtrees of the
// doubling in progress sit on a stack indexed by level and merge like a binary counter, so a subtree stops at its first
// turning or divergent node exactly as pyro's recursion does.  Nothing depends on which other chains share the launch.
//
// The kernel supplies the pool, the trial point, the reduction order Sum (TreeSum or ElementSum below) and a model with
//   template <class Fn> double evaluate(Chain<Sum>& c, double& third, Fn per_elem)
// which evaluates U at c.trial (every thread may read it on entry; +inf when U is not finite), writes dU/dtheta into
// vector V_GE, calls per_elem(i, g_i) on the owner of element i once g_i is known and returns the c.sum of its results in
// `third` (the fused second leapfrog half returns w_i^2), and counts PFN_GP_MCMC_EVALS and PFN_GP_MCMC_NOT_PD itself.
// After run, store_outputs and store_diag write the outputs every chain has; check_chain checks their descriptor fields.
//
// Random draw k of iteration key `it` is uniform_double(hash5(seed, key_b, key_t, it, 2k), hash5(.., 2k + 1)); the initial
// point and the first step-size search use key 0, iteration it and the searches after it key it + 1.  Compile with
// -fmad=false: the sampler's arithmetic is then the plain IEEE sequence nuts_chain performs.
#pragma once
#include <math_constants.h>

#include "common.cuh"
#include "counter_rng.cuh"
#include "../../include/pfn_b200.h"

namespace pfn {
namespace nuts {

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

// the vector pool; a node (a complete subtree of the doubling in progress) is five vectors: the whitened momenta of its
// first / last leaf, their sum over its leaves, and its multinomial proposal (z, g)
enum { V_Z, V_G, V_INV_M, V_SQRT_IM, V_RSQRT_IM, V_EZ, V_ER = V_EZ + 2, V_EG = V_ER + 2, V_EW = V_EG + 2, V_WSUM = V_EW + 2,
       V_RHALF, V_WF_MEAN, V_WF_M2, V_GE, V_NODES };
enum { N_WFIRST, N_WLAST, N_WSUM, N_Z, N_G, NODE_VECS };
constexpr int CUR = MAXD + 1;                  // node index of the subtree being built; 0 .. MAXD are the stack levels
constexpr int POOL_VECS = V_NODES + (MAXD + 2) * NODE_VECS;

// The reduction orders: sum every thread's partials v[0..K), K <= 3, into the same bits on every thread.
// TreeSum: butterfly within a warp, then the warps in sequence.
struct TreeSum {
  static constexpr int SLOTS = NW;
  template <int K>
  static __device__ void sum(double (*red)[3], int, double (&v)[K]) {
    const int tid = threadIdx.x;
#pragma unroll
    for (int k = 0; k < K; ++k)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v[k] = v[k] + __shfl_xor_sync(0xffffffffu, v[k], o);
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
};

// ElementSum: element order from 0.0, the order of a serial loop over the elements (and of nuts_chain).  Needs d <= NT,
// so that thread i's partial is element i's term alone.
template <int MAX_DIM>
struct ElementSum {
  static_assert(MAX_DIM <= NT, "one owner thread per element");
  static constexpr int SLOTS = MAX_DIM;
  template <int K>
  static __device__ void sum(double (*red)[3], int d, double (&v)[K]) {
    const int tid = threadIdx.x;
    if (tid < d)
#pragma unroll
      for (int k = 0; k < K; ++k) red[tid][k] = v[k];
    __syncthreads();
#pragma unroll
    for (int k = 0; k < K; ++k) {
      double s = 0.0;
      for (int i = 0; i < d; ++i) s = s + red[i][k];
      v[k] = s;
    }
  }
};

template <class Sum>
struct Shared {                                // written by thread 0 (red: by the reducing threads), read by all after a barrier
  double node_pe[MAXD + 1], node_weight[MAXD + 1];
  int win_end[MAX_WINDOWS];
  double red[2][Sum::SLOTS][3];
};

template <class Sum>
struct Chain {                                 // per-thread view of the chain; the scalars are identical on all threads
  Shared<Sum>* sh;
  double *trial, *pool;                        // the point being evaluated [d] and the vector pool
  int d, parity;
  uint32_t seed, key_b, key_t, key_it, ctr;
  double pe, eps, accept;
  double da_center, da_x, da_xavg, da_gavg;
  int da_t, wf_n, nwin, cw;
  int diag[PFN_GP_MCMC_NDIAG];
  __device__ double* vec(int slot) const { return pool + static_cast<size_t>(slot) * d; }
  __device__ double* node(int k, int which) const { return vec(V_NODES + k * NODE_VECS + which); }
  // The two buffers alternate, so a call's partials are never overwritten before every thread has read them.
  template <int K>
  __device__ void sum(double (&v)[K]) {
    Sum::sum(sh->red[parity], d, v);
    parity ^= 1;
  }
};

// ------------------------------------------------------------------------------------------------ random numbers
template <class C>
__device__ double uniform_at(const C& c, uint32_t k) {
  return uniform_double(hash5(c.seed, c.key_b, c.key_t, c.key_it, 2u * k), hash5(c.seed, c.key_b, c.key_t, c.key_it, 2u * k + 1u));
}
template <class C>
__device__ double uniform(C& c) { return uniform_at(c, c.ctr++); }
// Box-Muller, cosine branch, from draws k and k + 1; 1 - U is in (0, 1]
template <class C>
__device__ double normal_at(const C& c, uint32_t k) {
  const double u1 = 1.0 - uniform_at(c, k);
  const double u2 = uniform_at(c, k + 1u);
  return sqrt(-2.0 * log(u1)) * cos(TWO_PI * u2);
}

// ------------------------------------------------------------------------------------------------ NUTS
__device__ inline double logaddexp(double x, double y) {          // pyro's _logaddexp
  const double mn = x < y ? x : y, mx = x < y ? y : x;
  return log1p(exp(mn - mx)) + mx;
}

__device__ inline void copy(double* dst, const double* src, int d) {
  for (int i = threadIdx.x; i < d; i += NT) dst[i] = src[i];
}

// Stan's windows as pyro builds them (adaptation.WarmupAdapter._build_adaptation_schedule): end index of every window
__device__ inline int build_schedule(int* win_end, int W, bool store) {
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

// A fresh chain of W warmup iterations with the keys (seed, key_b, key_t): unit mass matrix, step size 1
template <class Sum>
__device__ void start(Chain<Sum>& c, Shared<Sum>* sh, double* trial, double* pool, int d, uint32_t seed, uint32_t key_b,
                      uint32_t key_t, int W) {
  c.sh = sh;
  c.trial = trial;
  c.pool = pool;
  c.d = d;
  c.parity = 0;
  c.seed = seed;
  c.key_b = key_b;
  c.key_t = key_t;
  c.key_it = 0;
  c.ctr = 0;
  c.pe = 0.0;
  c.eps = 1.0;
  c.accept = CUDART_NAN;
  c.da_center = c.da_x = c.da_xavg = c.da_gavg = 0.0;
  c.da_t = 0; c.wf_n = 0; c.cw = 0;
  for (int k = 0; k < PFN_GP_MCMC_NDIAG; ++k) c.diag[k] = 0;
  c.nwin = build_schedule(sh->win_end, W, threadIdx.x == 0);
  double *inv_m = c.vec(V_INV_M), *sqrt_im = c.vec(V_SQRT_IM), *rsqrt_im = c.vec(V_RSQRT_IM);
  double *wf_mean = c.vec(V_WF_MEAN), *wf_m2 = c.vec(V_WF_M2);
  for (int i = threadIdx.x; i < d; i += NT) {
    inv_m[i] = sqrt_im[i] = rsqrt_im[i] = 1.0;
    wf_mean[i] = wf_m2[i] = 0.0;
  }
}

// momentum draw: whitened w ~ N(0, I) into slot wv, r = M^1/2 w into slot rv; returns the kinetic energy
template <class Sum>
__device__ double draw_momentum(Chain<Sum>& c, int rv, int wv) {
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
  c.sum(v);
  return 0.5 * v[0];
}

// first half of a leapfrog step from (z, r, g) with signed step e: rhalf and the trial point
template <class Sum>
__device__ void leapfrog_begin(Chain<Sum>& c, int zv, int rv, int gv, double e) {
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
template <class Sum>
__device__ int is_turning(Chain<Sum>& c, const double* wl, const double* wr, const double* wsum) {
  double v[2] = {0.0, 0.0};
  for (int i = threadIdx.x; i < c.d; i += NT) {
    const double rho = wsum[i] - (wl[i] + wr[i]) / 2.0;
    v[0] = v[0] + wl[i] * rho;
    v[1] = v[1] + wr[i] * rho;
  }
  c.sum(v);
  return v[0] <= 0.0 || v[1] <= 0.0;
}

// step-size search from the chain's state (pyro HMC._find_reasonable_step_size), then a fresh dual-averaging centre
template <class Sum, class Model>
__device__ void step_size_search(Chain<Sum>& c, Model& m) {
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
    const double U = m.evaluate(c, ww, [&](int i, double g) {
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
template <class Sum, class Model>
__device__ double iteration(Chain<Sum>& c, Model& m, int it, int W, int max_depth, int& depth_out) {
  const int tid = threadIdx.x, d = c.d;
  Shared<Sum>& sh = *c.sh;
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
      const double U = m.evaluate(c, ww, [&](int i, double g) {   // second half: the end of the trajectory moves on
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
template <class Sum>
__device__ int adapt(Chain<Sum>& c, int it, double accept_prob, int W) {
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

// The chain: its initial point, from init [d] or (init null) theta ~ U(-2, 2) until U is finite, at most INIT_TRIES
// draws; then W warmup and S kept iterations.  Returns whether the initial point's U is finite.  The iterations run when
// it is and W + S > 0: out [max(S, 1), d] receives the kept states (S = 0: the state the warmup ended in), trace [W + S,
// d + 2] (optional) per iteration the state after it, the step size it used and its tree depth, c.accept the mean
// acceptance statistic of the sampling phase (NaN without one).  Without a finite initial point the trace is NaN and out
// is not written; with W = S = 0 neither is.  On return vectors V_Z, V_G and c.pe are the chain's last state.
template <class Sum, class Model>
__device__ bool run(Chain<Sum>& c, Model& m, const double* init, int W, int S, int max_depth, double* out, double* trace) {
  const int tid = threadIdx.x, d = c.d;
  bool finite = false;
  for (int attempt = 0;; ++attempt) {
    for (int i = tid; i < d; i += NT) c.trial[i] = init ? init[i] : -2.0 + 4.0 * uniform_at(c, c.ctr + i);
    if (!init) c.ctr += d;
    __syncthreads();
    double unused;
    c.pe = m.evaluate(c, unused, [](int, double) { return 0.0; });
    finite = c.pe < CUDART_INF;
    if (init != nullptr || finite || attempt + 1 >= INIT_TRIES) break;
  }
  copy(c.vec(V_Z), c.trial, d);
  copy(c.vec(V_G), c.vec(V_GE), d);
  if (!finite) {
    if (trace)
      for (size_t i = tid; i < static_cast<size_t>(W + S) * (d + 2); i += NT) trace[i] = CUDART_NAN;
    return false;
  }
  if (W + S == 0) return true;
  step_size_search(c, m);
  double acc_sampling = 0.0;
  for (int it = 0; it < W + S; ++it) {
    const double eps_used = c.eps;
    int depth;
    const double accept_prob = iteration(c, m, it, W, max_depth, depth);
    const double* z = c.vec(V_Z);
    if (trace) {
      double* row = trace + static_cast<size_t>(it) * (d + 2);
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
      step_size_search(c, m);
    }
  }
  if (S == 0) copy(out, c.vec(V_Z), d);        // warmup only: the one output row is the state the warmup ended in
  else c.accept = acc_sampling / S;
  return true;
}

// The outputs of chain p after run (finite: what it returned; W, S and out as passed to it): step_size, accept and the
// optional potential [p] and grad [p, d].  An evaluate-only call (W = S = 0) stores its point as the one row of out.  A
// chain without a finite starting point is not run: out, its step size and gradient are NaN, its potential +inf (c.pe)
// and its acceptance NaN (c.accept).  The counters follow with store_diag once the kernel's own work is counted.
template <class Sum>
__device__ void store_outputs(const Chain<Sum>& c, bool finite, int W, int S, size_t p, double* out, double* potential,
                              double* grad, double* step_size, double* accept) {
  const int tid = threadIdx.x, d = c.d;
  const bool ran = finite && W + S > 0;
  if (!ran) {
    const double* z = c.vec(V_Z);
    for (int k = 0; k < (S > 0 ? S : 1); ++k)
      for (int i = tid; i < d; i += NT) out[static_cast<size_t>(k) * d + i] = finite || W + S == 0 ? z[i] : CUDART_NAN;
  }
  if (tid == 0) {
    step_size[p] = ran ? c.eps : finite ? 0.0 : CUDART_NAN;
    accept[p] = c.accept;
    if (potential) potential[p] = c.pe;
  }
  if (grad) {
    const double* g = c.vec(V_G);
    for (int i = tid; i < d; i += NT) grad[p * d + i] = finite ? g[i] : CUDART_NAN;
  }
}

// diag [PFN_GP_MCMC_NDIAG]: the chain's counters
template <class Sum>
__device__ void store_diag(const Chain<Sum>& c, int* diag) {
  if (threadIdx.x == 0)
    for (int k = 0; k < PFN_GP_MCMC_NDIAG; ++k) diag[k] = c.diag[k];
}

// ------------------------------------------------------------------------------------------------ host
// The chain fields of a sampler's descriptor (pfn_gp_mcmc_desc, pfn_bnn_mcmc_desc), with `who` (the entry point's name)
// heading every message; inputs: whether the caller's input pointers are set.  Returns 0 on success.
template <class Desc>
inline int check_chain(const Desc* d, const char* who, bool inputs) {
  PFN_CHECK_ARG(inputs && d->samples && d->step_size && d->accept && d->diag, "%s: null input or output pointer", who);
  PFN_CHECK_ARG(d->num_samples >= 0 && d->warmup_steps >= 0, "%s: negative num_samples=%d or warmup_steps=%d", who,
                d->num_samples, d->warmup_steps);
  PFN_CHECK_ARG(static_cast<long long>(d->num_samples) + d->warmup_steps <= 0x7fffffffLL, "%s: too many iterations", who);
  PFN_CHECK_ARG(d->num_samples + d->warmup_steps > 0 || d->init != nullptr,
                "%s: warmup_steps = num_samples = 0 evaluates at init, which is null", who);
  PFN_CHECK_ARG(d->max_tree_depth >= 1 && d->max_tree_depth <= PFN_GP_MCMC_MAX_DEPTH,
                "%s: max_tree_depth=%d outside [1, %d]", who, d->max_tree_depth, PFN_GP_MCMC_MAX_DEPTH);
  return 0;
}

}  // namespace nuts
}  // namespace pfn
