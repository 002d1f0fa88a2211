// fp32-FMA GEMM with the same contract as the tensor-core path (pfn_gemm_desc): used for the fp32 parity
// mode and for shapes/alignments the tensor-core kernel does not accept.  64x64x16 tiles, 4x4 micro-tiles.
#include "common.cuh"
#include "../../include/pfn_b200.h"

namespace pfn {

template <typename T>
__global__ void __launch_bounds__(256)
gemm_simt_kernel(const pfn_gemm_desc d, int kb_per_split) {
  constexpr int BM = 64, BN = 64, BK = 16;
  __shared__ float sA[BK][BM + 4];
  __shared__ float sB[BK][BN + 4];
  const T* A = reinterpret_cast<const T*>(d.A);
  const T* Bm = reinterpret_cast<const T*>(d.B);
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int num_kb = (d.K + BK - 1) / BK;
  const int kb0 = blockIdx.z * kb_per_split;
  const int kb1 = min(kb0 + kb_per_split, num_kb);
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int kb = kb0; kb < kb1; ++kb) {
    const int k0 = kb * BK;
    // ---- load A tile into sA[k][m]
    if (!d.a_mn_major) {
      const int r = tid >> 2, kq = (tid & 3) * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int m = m0 + r, k = k0 + kq + j;
        sA[kq + j][r] = (m < d.M && k < d.K) ? to_f32<T>(A[static_cast<size_t>(m) * d.lda + k]) : 0.f;
      }
    } else {
      const int kk = tid >> 4, c = (tid & 15) * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int m = m0 + c + j, k = k0 + kk;
        sA[kk][c + j] = (m < d.M && k < d.K) ? to_f32<T>(A[static_cast<size_t>(k) * d.lda + m]) : 0.f;
      }
    }
    if (!d.b_mn_major) {
      const int r = tid >> 2, kq = (tid & 3) * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int n = n0 + r, k = k0 + kq + j;
        sB[kq + j][r] = (n < d.N && k < d.K) ? to_f32<T>(Bm[static_cast<size_t>(n) * d.ldb + k]) : 0.f;
      }
    } else {
      const int kk = tid >> 4, c = (tid & 15) * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int n = n0 + c + j, k = k0 + kk;
        sB[kk][c + j] = (n < d.N && k < d.K) ? to_f32<T>(Bm[static_cast<size_t>(k) * d.ldb + n]) : 0.f;
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = sA[k][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = sB[k][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }

  const bool first_split = blockIdx.z == 0;
  const T* aux = reinterpret_cast<const T*>(d.aux);
  T* C2 = reinterpret_cast<T*>(d.C2);
  const bool atomic = d.accumulate || gridDim.z > 1;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= d.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= d.N) continue;
      float v = acc[i][j];
      if (d.bias != nullptr && first_split) v += d.bias[n];
      if (d.epilogue == PFN_EPI_GELU) {
        if (C2 != nullptr) C2[static_cast<size_t>(m) * d.ldc2 + n] = from_f32<T>(v);
        v = gelu_erf(v);
      }
      if (aux != nullptr) {
        const float a = to_f32<T>(aux[static_cast<size_t>(m) * d.ld_aux + n]);
        if (d.epilogue == PFN_EPI_GELU_BWD) v *= gelu_erf_grad(a);
        else if (first_split) v += a;
      }
      if (d.c_dtype == PFN_F32) {
        float* dst = reinterpret_cast<float*>(d.C) + static_cast<size_t>(m) * d.ldc + n;
        if (atomic) atomicAdd(dst, v);
        else *dst = v;
      } else {
        reinterpret_cast<__nv_bfloat16*>(d.C)[static_cast<size_t>(m) * d.ldc + n] = __float2bfloat16_rn(v);
      }
    }
  }
}

}  // namespace pfn

extern "C" int pfn_gemm_simt(const pfn_gemm_desc* d, void* stream) {
  using namespace pfn;
  PFN_CHECK_ARG(d != nullptr, "gemm_simt: null descriptor");
  PFN_CHECK_ARG(d->M > 0 && d->N > 0 && d->K > 0, "gemm_simt: empty problem %d x %d x %d", d->M, d->N, d->K);
  PFN_CHECK_ARG(d->ab_dtype == PFN_F32 || d->ab_dtype == PFN_BF16, "gemm_simt: bad ab_dtype %d", d->ab_dtype);
  PFN_CHECK_ARG(d->epilogue >= 0 && d->epilogue <= PFN_EPI_GELU_BWD, "gemm_simt: bad epilogue %d", d->epilogue);
  PFN_CHECK_ARG(d->c2_gelu_grad == 0, "gemm_simt: c2_gelu_grad is a tensor-core-path option");
  PFN_CHECK_ARG(d->epilogue != PFN_EPI_GELU_BWD || d->aux != nullptr, "gemm_simt: GELU' epilogue needs aux");
  const int num_kb = (d->K + 15) / 16;
  int splits = d->k_splits <= 0 ? 1 : d->k_splits;
  if (splits > num_kb) splits = num_kb;
  const int per = (num_kb + splits - 1) / splits;
  splits = (num_kb + per - 1) / per;
  PFN_CHECK_ARG(!(d->accumulate || splits > 1) || d->c_dtype == PFN_F32, "gemm_simt: accumulate needs fp32 C");
  PFN_CHECK_ARG(d->epilogue == PFN_EPI_NONE || splits == 1, "gemm_simt: split-K cannot be combined with an activation");
  dim3 grid((d->N + 63) / 64, (d->M + 63) / 64, splits);
  PFN_CHECK_ARG(grid.y <= 65535, "gemm_simt: M too large for this path (%d)", d->M);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (d->ab_dtype == PFN_F32) gemm_simt_kernel<float><<<grid, 256, 0, s>>>(*d, per);
  else gemm_simt_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(*d, per);
  PFN_LAUNCH_OK();
  return 0;
}
