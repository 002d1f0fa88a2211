// Bayesian-NN prior (reference priors/pyro.py:10-34 calling mcmc_svi_transformer_on_bayesian.py:28-67 once per dataset).
//
// One CTA per dataset: the d network weights and the T x F inputs are drawn into shared memory (fp32 values, as the
// reference's), every row's two logits W2 (W1 x + b1) + b2, its softmax and its class draw are formed from them in fp64 by
// one thread per row, and x is written standardised over the sequence axis ((x - mean) / (unbiased std + 1e-6), statistics
// in fp64, one warp per feature).  Random numbers are counter-based hashes of (seed, tag, dataset, counter).
#include "common.cuh"
#include "counter_rng.cuh"
#include "../../include/pfn_b200.h"

namespace pfn {
namespace {

enum : uint32_t { TAG_WEIGHT = 201, TAG_X, TAG_CLASS };
constexpr int kThreads = 256;
constexpr double TWO_PI = 6.283185307179586;
constexpr size_t kMaxSmem = 200 * 1024;

__device__ __forceinline__ double uniform(uint32_t seed, uint32_t tag, uint32_t b, uint32_t i, uint32_t k) {
  return uniform_double(hash5(seed, tag, b, i, 2u * k), hash5(seed, tag, b, i, 2u * k + 1u));
}
// Box-Muller, cosine branch; 1 - U is in (0, 1]
__device__ __forceinline__ float normal(uint32_t seed, uint32_t tag, uint32_t b, uint32_t i) {
  const double u1 = 1.0 - uniform(seed, tag, b, i, 0), u2 = uniform(seed, tag, b, i, 1);
  return static_cast<float>(sqrt(-2.0 * log(u1)) * cos(TWO_PI * u2));
}

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(kThreads)
bnn_prior_kernel(uint32_t seed, int dataset_offset, int B, int T, int F, int E, float* __restrict__ x, float* __restrict__ y,
                 float* __restrict__ weights, float* __restrict__ x_raw, double* __restrict__ u_out) {
  extern __shared__ __align__(16) unsigned char prior_dyn[];
  const int d = E * F + 3 * E + 2;
  double* mean = reinterpret_cast<double*>(prior_dyn);       // [F]
  double* scale = mean + F;                                  // [F]: unbiased std + 1e-6
  float* th = reinterpret_cast<float*>(scale + F);           // [d]
  float* xs = th + d;                                        // [T, F]
  const int tid = threadIdx.x, b = blockIdx.x;
  const uint32_t key = static_cast<uint32_t>(dataset_offset + b);

  for (int i = tid; i < d; i += kThreads) {
    th[i] = normal(seed, TAG_WEIGHT, key, i);
    if (weights) weights[static_cast<size_t>(b) * d + i] = th[i];
  }
  for (int i = tid; i < T * F; i += kThreads) {
    xs[i] = normal(seed, TAG_X, key, i);
    if (x_raw) x_raw[(static_cast<size_t>(i / F) * B + b) * F + i % F] = xs[i];
  }
  __syncthreads();

  const float *W1 = th, *b1 = th + E * F, *W2 = b1 + E, *b2 = W2 + 2 * E;
  for (int t = tid; t < T; t += kThreads) {
    double l0 = b2[0], l1 = b2[1];
    for (int e = 0; e < E; ++e) {
      double h = b1[e];
      for (int f = 0; f < F; ++f) h = fma(static_cast<double>(W1[e * F + f]), static_cast<double>(xs[t * F + f]), h);
      l0 = fma(static_cast<double>(W2[e]), h, l0);
      l1 = fma(static_cast<double>(W2[E + e]), h, l1);
    }
    const double p0 = 1.0 / (1.0 + exp(l1 - l0));            // softmax(l)[0]
    const double u = uniform(seed, TAG_CLASS, key, t, 0);
    y[static_cast<size_t>(t) * B + b] = u < p0 ? 0.0f : 1.0f;
    if (u_out) u_out[static_cast<size_t>(t) * B + b] = u;
  }

  const int warp = tid >> 5, lane = tid & 31;
  for (int f = warp; f < F; f += kThreads / 32) {
    double s = 0.0;
    for (int t = lane; t < T; t += 32) s += xs[t * F + f];
    const double m = warp_sum_f64(s) / T;
    double q = 0.0;
    for (int t = lane; t < T; t += 32) {
      const double c = xs[t * F + f] - m;
      q = fma(c, c, q);
    }
    q = warp_sum_f64(q);
    if (lane == 0) {
      mean[f] = m;
      scale[f] = sqrt(q / (T - 1)) + 1e-6;                   // T = 1: NaN, as torch.std gives
    }
  }
  __syncthreads();
  for (int i = tid; i < T * F; i += kThreads) {
    const int f = i % F;
    x[(static_cast<size_t>(i / F) * B + b) * F + f] = static_cast<float>((xs[i] - mean[f]) / scale[f]);
  }
}

}  // namespace
}  // namespace pfn

using namespace pfn;

extern "C" int pfn_bnn_prior(uint32_t seed, int dataset_offset, int B, int T, int F, int E, float* x, float* y,
                             float* weights, float* x_raw, double* u, void* stream) {
  PFN_CHECK_ARG(B > 0 && T > 0 && F > 0 && E > 0, "bnn_prior: empty problem B=%d T=%d F=%d E=%d", B, T, F, E);
  PFN_CHECK_ARG(dataset_offset >= 0, "bnn_prior: negative dataset_offset=%d", dataset_offset);
  const long long d = static_cast<long long>(E) * F + 3LL * E + 2;
  PFN_CHECK_ARG(d <= PFN_BNN_MAX_D, "bnn_prior: d = E F + 3 E + 2 = %lld exceeds %d", d, PFN_BNN_MAX_D);
  const size_t smem = 2 * F * sizeof(double) + (static_cast<size_t>(d) + static_cast<size_t>(T) * F) * sizeof(float);
  PFN_CHECK_ARG(smem <= kMaxSmem, "bnn_prior: T=%d rows of F=%d features need %zu bytes of shared memory (limit %zu)", T, F,
                smem, kMaxSmem);
  PFN_CHECK_ARG(x != nullptr && y != nullptr, "bnn_prior: null output pointer");
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set))
    PFN_CUDA_OK(cudaFuncSetAttribute(bnn_prior_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     static_cast<int>(kMaxSmem)));
  bnn_prior_kernel<<<B, kThreads, smem, reinterpret_cast<cudaStream_t>(stream)>>>(seed, dataset_offset, B, T, F, E, x, y,
                                                                                  weights, x_raw, u);
  PFN_LAUNCH_OK();
  return 0;
}
