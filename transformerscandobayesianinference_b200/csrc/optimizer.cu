// Optimizer step glue of the training inner loop (reference train.py:94-97: clip_grad_norm_(1.) then Adam.step()) as two
// launches over ALL parameter tensors: (1) sum of squared gradients, (2) clip coefficient + Adam update + bf16 copy of the
// updated weight (the operand the next step's wgmma GEMMs read, so no per-step cast pass).  HBM-bound: per element one
// read of g for the norm, then reads of p, g, m, v and writes of p, m, v (+ 2 bytes of shadow).
// Work is cut into chunks of ADAM_CHUNK elements; `chunk_start[t]` is the first chunk of tensor t (prefix sums), so CTA b
// finds its tensor by a short binary search -- no per-tensor launches, no host loop.
#include "common.cuh"
#include "../../include/pfn_b200.h"

namespace pfn {

constexpr int ADAM_CHUNK = 8192;           // elements per CTA (256 threads x 8 float4)

__device__ __forceinline__ int adam_find_tensor(const int* __restrict__ chunk_start, int n_tensors, int chunk) {
  int lo = 0, hi = n_tensors - 1;          // largest t with chunk_start[t] <= chunk
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (chunk_start[mid] <= chunk) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(256)
adam_gradnorm_kernel(const pfn_adam_tensor* __restrict__ table, const int* __restrict__ chunk_start, int n_tensors,
                     float* __restrict__ norm_sq) {
  const int t = adam_find_tensor(chunk_start, n_tensors, blockIdx.x);
  const pfn_adam_tensor e = table[t];
  const long long base = static_cast<long long>(blockIdx.x - chunk_start[t]) * ADAM_CHUNK;
  const long long end = base + ADAM_CHUNK < e.n ? base + ADAM_CHUNK : e.n;
  float acc = 0.f;
  const bool vec = (reinterpret_cast<uintptr_t>(e.g) & 15) == 0;
  if (vec) {
    for (long long i = base + threadIdx.x * 4LL; i < end; i += 1024) {
      if (i + 4 <= end) {
        const float4 g = *reinterpret_cast<const float4*>(e.g + i);
        acc += g.x * g.x + g.y * g.y + g.z * g.z + g.w * g.w;
      } else {
        for (long long k = i; k < end; ++k) acc += e.g[k] * e.g[k];
      }
    }
  } else {
    for (long long i = base + threadIdx.x; i < end; i += 256) acc += e.g[i] * e.g[i];
  }
  __shared__ float red[8];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 8) {
    float v = red[threadIdx.x];
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) v += __shfl_xor_sync(0xffu, v, o);
    if (threadIdx.x == 0) atomicAdd(norm_sq, v);
  }
}

struct AdamHyper {
  float lr, beta1, beta2, eps, weight_decay, max_grad_norm;
  float bias_corr1, bias_corr2_sqrt;
};

__device__ __forceinline__ void adam_one(float& p, float g, float& m, float& v, const AdamHyper& h, float clip) {
  g *= clip;
  if (h.weight_decay != 0.f) g = fmaf(h.weight_decay, p, g);            // torch.optim.Adam: L2 term added to the gradient
  m = fmaf(h.beta1, m, (1.f - h.beta1) * g);
  v = fmaf(h.beta2, v, (1.f - h.beta2) * g * g);
  const float denom = sqrtf(v) / h.bias_corr2_sqrt + h.eps;
  p -= (h.lr / h.bias_corr1) * (m / denom);
}

__global__ void __launch_bounds__(256)
adam_update_kernel(const pfn_adam_tensor* __restrict__ table, const int* __restrict__ chunk_start, int n_tensors,
                   const float* __restrict__ norm_sq, AdamHyper h) {
  const int t = adam_find_tensor(chunk_start, n_tensors, blockIdx.x);
  const pfn_adam_tensor e = table[t];
  const long long base = static_cast<long long>(blockIdx.x - chunk_start[t]) * ADAM_CHUNK;
  const long long end = base + ADAM_CHUNK < e.n ? base + ADAM_CHUNK : e.n;
  float clip = 1.f;
  if (h.max_grad_norm > 0.f) {              // torch.nn.utils.clip_grad_norm_: coef = max_norm / (total_norm + 1e-6), clamped to 1
    clip = h.max_grad_norm / (sqrtf(*norm_sq) + 1e-6f);
    clip = clip < 1.f ? clip : 1.f;
  }
  __nv_bfloat16* sh = reinterpret_cast<__nv_bfloat16*>(e.p_bf16);
  const bool vec = ((reinterpret_cast<uintptr_t>(e.p) | reinterpret_cast<uintptr_t>(e.g) | reinterpret_cast<uintptr_t>(e.m) |
                     reinterpret_cast<uintptr_t>(e.v)) & 15) == 0 && (reinterpret_cast<uintptr_t>(sh) & 7) == 0;
  if (vec) {
    for (long long i = base + threadIdx.x * 4LL; i < end; i += 1024) {
      if (i + 4 <= end) {
        float4 p = *reinterpret_cast<float4*>(e.p + i);
        const float4 g = *reinterpret_cast<const float4*>(e.g + i);
        float4 m = *reinterpret_cast<float4*>(e.m + i);
        float4 v = *reinterpret_cast<float4*>(e.v + i);
        adam_one(p.x, g.x, m.x, v.x, h, clip); adam_one(p.y, g.y, m.y, v.y, h, clip);
        adam_one(p.z, g.z, m.z, v.z, h, clip); adam_one(p.w, g.w, m.w, v.w, h, clip);
        *reinterpret_cast<float4*>(e.p + i) = p;
        *reinterpret_cast<float4*>(e.m + i) = m;
        *reinterpret_cast<float4*>(e.v + i) = v;
        if (sh != nullptr) {
          __nv_bfloat162 lo = __floats2bfloat162_rn(p.x, p.y), hi = __floats2bfloat162_rn(p.z, p.w);
          uint2 pk;
          pk.x = *reinterpret_cast<uint32_t*>(&lo); pk.y = *reinterpret_cast<uint32_t*>(&hi);
          *reinterpret_cast<uint2*>(sh + i) = pk;
        }
      } else {
        for (long long k = i; k < end; ++k) {
          float p = e.p[k], m = e.m[k], v = e.v[k];
          adam_one(p, e.g[k], m, v, h, clip);
          e.p[k] = p; e.m[k] = m; e.v[k] = v;
          if (sh != nullptr) sh[k] = __float2bfloat16_rn(p);
        }
      }
    }
  } else {
    for (long long i = base + threadIdx.x; i < end; i += 256) {
      float p = e.p[i], m = e.m[i], v = e.v[i];
      adam_one(p, e.g[i], m, v, h, clip);
      e.p[i] = p; e.m[i] = m; e.v[i] = v;
      if (sh != nullptr) sh[i] = __float2bfloat16_rn(p);
    }
  }
}

}  // namespace pfn

using namespace pfn;

extern "C" int pfn_adam_chunk_elems(void) { return ADAM_CHUNK; }

extern "C" int pfn_adam_step(const pfn_adam_tensor* table_dev, const int* chunk_start_dev, int n_tensors, int n_chunks,
                             float lr, float beta1, float beta2, float eps, float weight_decay, float max_grad_norm,
                             int step, float* norm_sq_dev, void* stream) {
  PFN_CHECK_ARG(table_dev != nullptr && chunk_start_dev != nullptr && norm_sq_dev != nullptr, "adam_step: null table");
  PFN_CHECK_ARG(n_tensors > 0 && n_chunks > 0 && step >= 1, "adam_step: bad sizes n_tensors=%d n_chunks=%d step=%d", n_tensors,
                n_chunks, step);
  PFN_CHECK_ARG(beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f && eps >= 0.f, "adam_step: bad hyper-parameters");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  AdamHyper h;
  h.lr = lr; h.beta1 = beta1; h.beta2 = beta2; h.eps = eps; h.weight_decay = weight_decay; h.max_grad_norm = max_grad_norm;
  h.bias_corr1 = 1.f - powf(beta1, static_cast<float>(step));
  h.bias_corr2_sqrt = sqrtf(1.f - powf(beta2, static_cast<float>(step)));
  if (max_grad_norm > 0.f) {
    PFN_CUDA_OK(cudaMemsetAsync(norm_sq_dev, 0, sizeof(float), s));
    adam_gradnorm_kernel<<<n_chunks, 256, 0, s>>>(table_dev, chunk_start_dev, n_tensors, norm_sq_dev);
    PFN_LAUNCH_OK();
  }
  adam_update_kernel<<<n_chunks, 256, 0, s>>>(table_dev, chunk_start_dev, n_tensors, norm_sq_dev, h);
  PFN_LAUNCH_OK();
  return 0;
}
