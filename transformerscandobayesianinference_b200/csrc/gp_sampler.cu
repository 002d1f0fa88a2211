// GP prior sampler: one CTA per dataset builds the kernel matrix on the fly, factors it with a blocked
// left-looking Cholesky in true fp32 (FFMA) and applies the factor to z in the same pass:
//     K = os * k(x, x; ls) + (noise + jitter) I ,   L = chol(K) ,   y = L z
// Restates the sampling maths the reference obtains from gpytorch (priors/fast_gp.py:13-32,48-56:
// ScaleKernel(RBFKernel) + GaussianLikelihood noise, MultivariateNormal.sample -> cholesky root times randn)
// and, with per-dataset hyperparameters and Matern-nu kernels, priors/fast_gp_mix.py:24-55,88-99.
//
// Left-looking, panel width 32:  for panel p (columns c0..c0+31)
//     U[r, :]  = K[r, c0:c0+32] - L[r, 0:c0] L[c0:c0+32, 0:c0]^T          (128x32 tiles, 4x4 register micro-tiles)
//     L11      = chol(U[c0:c0+32, :])                                     (one warp, rows in registers, shuffles)
//     L[r, c0:c0+32] = U[r, :] L11^-T  for r > c0+31                      (one thread per row, L11 broadcast from smem)
//     y[r]    += L[r, c0:c0+32] . z[c0:c0+32]
// K is never materialised; the only HBM traffic is writing the factor once and re-reading finished panels.
// The factor is kept TRANSPOSED in `work` (work[b][c][r] = L[r][c]): panel re-reads become contiguous rows that stream
// through a 3-stage cp.async ring straight into the k-major smem tiles, and the panel write-back is coalesced.
#include "common.cuh"
#include "../../include/pfn_b200.h"

namespace pfn {

constexpr int NB = 32;        // panel width
constexpr int GP_MAX_F = 128;
constexpr int GP_STAGES = 3;

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, bool valid) {
  const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
  const int bytes = valid ? 16 : 0;   // src-size 0 => zero fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ float gp_kernel_value(float d2, float os, int kernel_type) {
  if (kernel_type == PFN_KERNEL_RBF) return os * expf(-0.5f * d2);
  const float r = sqrtf(d2);
  if (kernel_type == PFN_KERNEL_MATERN12) return os * expf(-r);
  if (kernel_type == PFN_KERNEL_MATERN32) {
    const float a = 1.7320508075688772f * r;
    return os * (1.0f + a) * expf(-a);
  }
  const float a = 2.23606797749979f * r;
  return os * (1.0f + a + (5.0f / 3.0f) * d2) * expf(-a);
}

// TR = rows per update tile; the CTA has 2 TR threads.  TR = 64 (128 threads, 49 KB of shared memory, 4 CTAs per SM) keeps four
// independent datasets on an SM, so that the serial phases of one (32x32 diagonal block in one warp, row solves, ring
// fill) overlap the products of the others, and 512 datasets fit in ONE wave of 592 slots (TR = 128: 2 CTAs per SM, 296
// slots, two waves).
template <int TR>
__global__ void __launch_bounds__(2 * TR, TR == 64 ? 4 : 2)
gp_sample_kernel(const float* __restrict__ x, const float* __restrict__ z, const float* __restrict__ ls,
                 const float* __restrict__ os_arr, const float* __restrict__ noise_arr, float jitter, int kernel_type,
                 float* __restrict__ y, float* work, int* __restrict__ info, int T, int F, int ldw) {
  extern __shared__ __align__(16) float gp_dyn[];         // the cp.async ring lives in dynamic shared memory (60 KB)
  constexpr int NT = 2 * TR;                                                                      // threads per CTA
  float (*sR)[NB][TR] = reinterpret_cast<float (*)[NB][TR]>(gp_dyn);                              // sR[s][k][r] = L[r0 + r, j0 + k]
  float (*sC)[NB][NB] = reinterpret_cast<float (*)[NB][NB]>(gp_dyn + GP_STAGES * NB * TR);        // sC[s][k][c] = L[c0 + c, j0 + k]
  __shared__ float sU[TR][NB + 1];                  // updated tile, row-major (padded)
  __shared__ __align__(16) float sL[NB][NB];        // L11 (row-major), unit rows past the matrix edge
  __shared__ float sLinv[NB];
  __shared__ float sz[NB];
  __shared__ float s_inv_ls[GP_MAX_F];
  __shared__ int s_info;

  const int b = blockIdx.x;
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const float* xb = x + static_cast<size_t>(b) * T * F;
  const float* zb = z + static_cast<size_t>(b) * T;
  float* yb = y + static_cast<size_t>(b) * T;
  float* Lt = work + static_cast<size_t>(b) * T * ldw;   // Lt[c * ldw + r] = L[r][c]
  const float os = os_arr[b];
  const float diag_add = noise_arr[b] + jitter;

  for (int f = tid; f < F; f += NT) s_inv_ls[f] = 1.0f / ls[static_cast<size_t>(b) * F + f];
  if (tid == 0) s_info = 0;
  for (int r = tid; r < T; r += NT) yb[r] = 0.f;
  __syncthreads();

  const int ty = tid >> 3;   // 0..TR/4-1 -> rows ty*4 .. ty*4+3 of the tile
  const int tx = tid & 7;    // 0..7  -> cols tx*4 .. tx*4+3 of the panel

  for (int c0 = 0; c0 < T; c0 += NB) {
    const int nb = min(NB, T - c0);
    if (tid < NB) sz[tid] = (c0 + tid < T) ? zb[c0 + tid] : 0.f;
    for (int r0 = c0; r0 < T; r0 += TR) {
      // ---------------------------------------------------------------- update: acc = L[r,0:c0] L[c,0:c0]^T
      float acc[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
      // 3-stage cp.async ring over the 32-column chunks of the finished panels (rows of Lt are contiguous in r)
      const int nch = c0 / NB;
      auto issue = [&](int ch) {
        const int st = ch % GP_STAGES;
        const int j0 = ch * NB;
        // sR: 32 k-rows x TR floats = 8 TR 16-byte pieces (4 per thread); sC: 32 x 32 floats = 256 pieces
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int piece = tid + q * NT;
          const int k = piece / (TR / 4), r4 = (piece % (TR / 4)) * 4;
          const int r = r0 + r4;
          cp_async16(&sR[st][k][r4], Lt + static_cast<size_t>(j0 + k) * ldw + r, r < ldw);
        }
#pragma unroll
        for (int piece = tid; piece < 256; piece += NT) {
          const int k = piece >> 3, c4 = (piece & 7) * 4;
          const int c = c0 + c4;
          cp_async16(&sC[st][k][c4], Lt + static_cast<size_t>(j0 + k) * ldw + c, c < ldw);
        }
      };
#pragma unroll
      for (int sidx = 0; sidx < GP_STAGES - 1; ++sidx) {
        if (sidx < nch) issue(sidx);
        cp_async_commit();
      }
      for (int ch = 0; ch < nch; ++ch) {
        cp_async_wait<GP_STAGES - 2>();
        __syncthreads();
        if (ch + GP_STAGES - 1 < nch) issue(ch + GP_STAGES - 1);
        cp_async_commit();
        const int st = ch % GP_STAGES;
#pragma unroll
        for (int k = 0; k < NB; ++k) {
          const float4 a = *reinterpret_cast<const float4*>(&sR[st][k][ty * 4]);
          const float4 bb = *reinterpret_cast<const float4*>(&sC[st][k][tx * 4]);
          const float av[4] = {a.x, a.y, a.z, a.w};
          const float bv[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
      }
      cp_async_wait<0>();
      __syncthreads();     // every thread is done with the ring before the next tile refills it
      // ---------------------------------------------------------------- U = K - acc   (kernel built on the fly)
      {
        float d2[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) d2[i][j] = 0.f;
        for (int f = 0; f < F; ++f) {
          const float il = s_inv_ls[f];
          float xr[4], xc[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int r = r0 + ty * 4 + i;
            xr[i] = r < T ? xb[static_cast<size_t>(r) * F + f] * il : 0.f;
            const int c = c0 + tx * 4 + i;
            xc[i] = c < T ? xb[static_cast<size_t>(c) * F + f] * il : 0.f;
          }
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) { const float df = xr[i] - xc[j]; d2[i][j] = fmaf(df, df, d2[i][j]); }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int r = r0 + ty * 4 + i;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int c = c0 + tx * 4 + j;
            float u = 0.f;
            if (r < T && c < T) {
              u = gp_kernel_value(d2[i][j], os, kernel_type);
              if (r == c) u = os + diag_add;   // k(x,x) = 1 for every supported kernel
              u -= acc[i][j];
            }
            sU[ty * 4 + i][tx * 4 + j] = u;
          }
        }
      }
      __syncthreads();
      // ---------------------------------------------------------------- diagonal block: chol in registers (warp 0)
      if (r0 == c0) {
        if (tid < 32) {
          float row[NB];
#pragma unroll
          for (int c = 0; c < NB; ++c) row[c] = sU[lane][c];
          if (lane >= nb) {
#pragma unroll
            for (int c = 0; c < NB; ++c) row[c] = (c == lane) ? 1.0f : 0.f;
          }
#pragma unroll
          for (int j = 0; j < NB; ++j) {
            float djj = __shfl_sync(0xffffffffu, row[j], j);
            if (!(djj > 0.f)) {
              if (lane == 0 && s_info == 0) s_info = c0 + j + 1;
              djj = 1.0f;
            }
            const float ljj = sqrtf(djj);
            const float lij = (lane > j) ? row[j] / ljj : (lane == j ? ljj : 0.f);
            row[j] = lij;
#pragma unroll
            for (int c = j + 1; c < NB; ++c) {
              const float lcj = __shfl_sync(0xffffffffu, lij, c);
              if (lane >= c) row[c] = fmaf(-lij, lcj, row[c]);
            }
          }
#pragma unroll
          for (int c = 0; c < NB; ++c) sL[lane][c] = (c <= lane) ? row[c] : 0.f;
          float dg = 1.0f;
#pragma unroll
          for (int c = 0; c < NB; ++c) dg = (c == lane) ? row[c] : dg;
          sLinv[lane] = 1.0f / dg;
        }
        __syncthreads();
      }
      // ---------------------------------------------------------------- write the diagonal block / solve the rows below
      if (tid < TR) {
        const int r = r0 + tid;
        if (r < T) {
          float v[NB];
          if (r0 == c0 && tid < NB) {
#pragma unroll
            for (int c = 0; c < NB; ++c) v[c] = sL[tid][c];
          } else {
#pragma unroll
            for (int c = 0; c < NB; ++c) {
              float a = sU[tid][c];
#pragma unroll
              for (int p = 0; p < c; ++p) a = fmaf(-v[p], sL[c][p], a);
              v[c] = a * sLinv[c];
            }
          }
          float dot = 0.f;
#pragma unroll
          for (int c = 0; c < NB; ++c) dot = fmaf(v[c], sz[c], dot);
          yb[r] += dot;
#pragma unroll
          for (int c = 0; c < NB; ++c) {
            if (c0 + c < T) Lt[static_cast<size_t>(c0 + c) * ldw + r] = v[c];     // lanes = consecutive r: coalesced
          }
        }
      }
      __syncthreads();
    }
  }
  if (tid == 0) info[b] = s_info;
}

constexpr int gp_dyn_smem(int tr) { return GP_STAGES * (NB * tr + NB * NB) * static_cast<int>(sizeof(float)); }

}  // namespace pfn

using namespace pfn;

extern "C" int pfn_gp_sample(const float* x, const float* z, const float* ls, const float* os, const float* noise,
                             float jitter, int kernel_type, float* y, float* work, int* info, int Bn, int T, int F,
                             void* stream) {
  PFN_CHECK_ARG(Bn > 0 && T > 0 && F > 0, "gp_sample: bad shape Bn=%d T=%d F=%d", Bn, T, F);
  PFN_CHECK_ARG(F <= GP_MAX_F, "gp_sample: F=%d exceeds %d", F, GP_MAX_F);
  PFN_CHECK_ARG(kernel_type >= PFN_KERNEL_RBF && kernel_type <= PFN_KERNEL_MATERN52, "gp_sample: bad kernel type %d", kernel_type);
  PFN_CHECK_ARG((reinterpret_cast<uintptr_t>(work) & 15) == 0, "gp_sample: work buffer must be 16-byte aligned");
  const int ldw = (T + 3) & ~3;
  // the small tile only once the batch no longer fills the GPU with the large one
#ifdef PFN_GP_TR
  const bool small_tile = PFN_GP_TR == 64;
#else
  const bool small_tile = Bn > 2 * num_sms();
#endif
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set)) {
    PFN_CUDA_OK(cudaFuncSetAttribute(gp_sample_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, gp_dyn_smem(64)));
    PFN_CUDA_OK(cudaFuncSetAttribute(gp_sample_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, gp_dyn_smem(128)));
  }
  if (small_tile)
    gp_sample_kernel<64><<<Bn, 128, gp_dyn_smem(64), s>>>(x, z, ls, os, noise, jitter, kernel_type, y, work, info, T, F, ldw);
  else
    gp_sample_kernel<128><<<Bn, 256, gp_dyn_smem(128), s>>>(x, z, ls, os, noise, jitter, kernel_type, y, work, info, T, F, ldw);
  PFN_LAUNCH_OK();
  return 0;
}
