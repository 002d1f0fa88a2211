// Shared helpers for the PFN sm_90a kernels (error reporting, dtype traits, warp reductions).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

namespace pfn {

// ---------------------------------------------------------------------------------------------
// Error plumbing: every C-ABI entry returns 0 on success, non-zero on failure and stores a
// message readable through pfn_last_error(). No C++ exception ever crosses the ABI.
// ---------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
const char* get_error();

#define PFN_CHECK_ARG(cond, ...)                                   \
  do {                                                             \
    if (!(cond)) {                                                 \
      ::pfn::set_error(__VA_ARGS__);                               \
      return 1;                                                    \
    }                                                              \
  } while (0)

#define PFN_CUDA_OK(expr)                                                              \
  do {                                                                                 \
    cudaError_t _e = (expr);                                                           \
    if (_e != cudaSuccess) {                                                           \
      ::pfn::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return 2;                                                                        \
    }                                                                                  \
  } while (0)

#define PFN_LAUNCH_OK()                                                                \
  do {                                                                                 \
    cudaError_t _e = cudaGetLastError();                                               \
    if (_e != cudaSuccess) {                                                           \
      ::pfn::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
      return 3;                                                                        \
    }                                                                                  \
  } while (0)

enum DType : int { kF32 = 0, kBF16 = 1 };

__host__ __device__ inline size_t dtype_size(int dt) { return dt == kF32 ? 4 : 2; }

// ---------------------------------------------------------------------------------------------
// Device-side scalar conversion
// ---------------------------------------------------------------------------------------------
template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// exact-erf GELU (the reference uses activation='gelu' => erf form, transformer.py:17)
__device__ __forceinline__ float gelu_erf(float u) { return 0.5f * u * (1.0f + erff(u * 0.70710678118654752f)); }
__device__ __forceinline__ float gelu_erf_grad(float u) {
  const float cdf = 0.5f * (1.0f + erff(u * 0.70710678118654752f));
  const float pdf = 0.39894228040143268f * __expf(-0.5f * u * u);
  return cdf + u * pdf;
}

// Fast erf-GELU for the bf16 tensor-core epilogues.  Phi(u) = 0.5 (1 + erf(u / sqrt 2)) is replaced by
//   Phi(u) ~= 0.5 (1 + tanh(u q(u^2))),   q(t) = c0 + c1 t + c2 t^2   (minimax fit against erf, tools/fit_gelu.py):
//   max |dPhi| 6.7e-5, max |dGELU| 3.7e-5, max |dGELU'| 9.3e-5 over the real line for the exact formula; the hardware
//   tanh.approx (relative error 2^-11) adds <= 2.4e-4 |u| -- all below the bf16 resolution of the stored activations.
//   u^2 is clamped at 80 (|u| ~ 8.9, Phi already 0 / 1 to 1e-18): c2 < 0 would turn q negative
//   beyond |u| ~ 10.5.  The fp32 parity engine (SIMT kernels) keeps erff.
__device__ __forceinline__ float fast_rcp(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fast_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fast_tanh(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
constexpr float kGeluC0 = 0.7974228190582262f, kGeluC1 = 0.0370038563083048f, kGeluC2 = -0.0003475408844912201f;
// GELU uses the exp/rcp form of the sigmoid, GELU' the tanh form (both the same approximant).
constexpr float kGeluK = -2.8853900817779268f;   // -2 log2(e)
__device__ __forceinline__ float gelu_fast(float u) {
  // u Phi(u), Phi = 1 / (1 + 2^(K u q(u^2)))  (identical to 0.5 (1 + tanh(u q)); relative accuracy kept in the tails)
  const float u2 = fminf(u * u, 80.0f);
  const float q = fmaf(u2, fmaf(u2, kGeluC2 * kGeluK, kGeluC1 * kGeluK), kGeluC0 * kGeluK);
  return u * fast_rcp(1.0f + fast_ex2(u * q));
}
// derivative of the approximant itself: Phi + 0.5 u (1 - t^2) p'(u), p(u) = u q(u^2), t = tanh(p)
__device__ __forceinline__ float gelu_grad_fast(float u) {
  const float u2 = fminf(u * u, 80.0f);
  const float t = fast_tanh(u * fmaf(u2, fmaf(u2, kGeluC2, kGeluC1), kGeluC0));
  const float hdp = fmaf(u2, fmaf(u2, 2.5f * kGeluC2, 1.5f * kGeluC1), 0.5f * kGeluC0);   // 0.5 p'(u)
  return fmaf(u * hdp, fmaf(-t, t, 1.0f), fmaf(0.5f, t, 0.5f));
}

// gelu and its derivative from ONE evaluation of the sigmoid: Phi = 1 / (1 + 2^(K u q(u^2))) = sigma(2 p(u)), so
// d/du [u Phi] = Phi + u * 2 p'(u) * Phi (1 - Phi)   (the same approximant gelu_grad_fast differentiates: 1 - tanh^2 = 4 Phi (1 - Phi))
__device__ __forceinline__ void gelu_and_grad_fast(float u, float& g, float& gp) {
  const float u2 = fminf(u * u, 80.0f);
  const float q = fmaf(u2, fmaf(u2, kGeluC2 * kGeluK, kGeluC1 * kGeluK), kGeluC0 * kGeluK);
  const float phi = fast_rcp(1.0f + fast_ex2(u * q));
  const float dp2 = fmaf(u2, fmaf(u2, 10.0f * kGeluC2, 6.0f * kGeluC1), 2.0f * kGeluC0);     // 2 p'(u)
  g = u * phi;
  gp = fmaf(u * dp2, fmaf(-phi, phi, phi), phi);
}

int num_sms();

// Per-device one-time setup guard (function attributes such as the dynamic shared-memory limit are per device).
inline bool first_use_on_device(bool (&done)[64]) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return true;
  if (done[dev]) return false;
  done[dev] = true;
  return true;
}

}  // namespace pfn
