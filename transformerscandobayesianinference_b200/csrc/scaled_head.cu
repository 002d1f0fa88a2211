// Row work of the reference's learned-temperature decoder heads (reference decoders.py:6-30), between the head's second
// GEMM and the loss.  One warp per row, lanes strided over the columns (coalesced), fp32 throughout.  Every sum runs in a
// fixed order (per-lane sequential, then the xor butterfly, then fixed shared-memory trees): no atomics, so two runs give
// the same bits, and the depth of every sum is stated in include/pfn_b200.h for the error bounds of oracle/decoders_oracle.py.
#include "common.cuh"
#include "../../include/pfn_b200.h"

namespace pfn {

// reference decoders.py:17, torch.tensor([...]) in float32: 1.4 and 1.7 are their fp32 roundings
__constant__ float kHeadTemps[PFN_HEAD_TEMPS] = {1.f, 1.4f, 1.7f, 2.f, 5.f, 10.f, 20.f, 40.f, 80.f, 160.f};

// p_k = softmax(zt)_k in lane k < 10 (0 elsewhere); returns temp = sum_k p_k c_k in every lane
__device__ __forceinline__ float head_temp(const float* __restrict__ zt, int lane, float& p) {
  const float v = lane < PFN_HEAD_TEMPS ? zt[lane] : -INFINITY;
  const float m = warp_max(v);
  const float e = lane < PFN_HEAD_TEMPS ? expf(v - m) : 0.f;
  p = e / warp_sum(e);
  return warp_sum(lane < PFN_HEAD_TEMPS ? p * kHeadTemps[lane] : 0.f);
}

__global__ void __launch_bounds__(256)
scaled_head_fwd_kernel(const float* __restrict__ zz, int ldz, int n_out, float* __restrict__ out, int ldo,
                       float* __restrict__ temp_out, int rows) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int row = warp; row < rows; row += nwarps) {
    const float* z = zz + static_cast<size_t>(row) * ldz;
    float p;
    const float t = head_temp(z + n_out, lane, p);
    float* o = out + static_cast<size_t>(row) * ldo;
    for (int c = lane; c < n_out; c += 32) o[c] = z[c] / t;
    if (lane == 0) temp_out[row] = t;
  }
}

// dzz[:, :n_out] = g / temp;  dzz[:, n_out + k] = p_k (c_k - temp) dtemp,  dtemp = -(sum_j g_j z_j) / temp^2;  zero padding
template <typename TD>
__global__ void __launch_bounds__(256)
scaled_head_bwd_kernel(const float* __restrict__ g, int ldg, const float* __restrict__ zz, int ldz,
                       const float* __restrict__ temp, int n_out, TD* __restrict__ dzz, int ldd, int n_cols_pad, int rows) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int row = warp; row < rows; row += nwarps) {
    const float* z = zz + static_cast<size_t>(row) * ldz;
    const float* gr = g + static_cast<size_t>(row) * ldg;
    TD* d = dzz + static_cast<size_t>(row) * ldd;
    float p;
    head_temp(z + n_out, lane, p);             // p only: the forward's temp is read back (same bits)
    const float t = temp[row];
    float s = 0.f;
    for (int c = lane; c < n_out; c += 32) {
      const float gc = gr[c];
      s = fmaf(gc, z[c], s);
      d[c] = from_f32<TD>(gc / t);
    }
    const float dtemp = -warp_sum(s) / (t * t);
    if (lane < PFN_HEAD_TEMPS) d[n_out + lane] = from_f32<TD>(p * (kHeadTemps[lane] - t) * dtemp);
    for (int c = n_out + PFN_HEAD_TEMPS + lane; c < n_cols_pad; c += 32) d[c] = from_f32<TD>(0.f);
  }
}

// Sum of v[0, n) by the 256 threads of a CTA: thread i adds v[i], v[i + 256], ... in turn, then a fixed tree over the
// threads.  Depth ceil(n / 256) + 8; every CTA that calls it gets the same bits.
__device__ __forceinline__ float cta_sum_256(const float* __restrict__ v, int n, float* red) {
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += 256) s += v[i];
  red[threadIdx.x] = s;
  __syncthreads();
#pragma unroll
  for (int w = 128; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  const float r = red[0];
  __syncthreads();
  return r;
}

// out = z / S, S = sum(T_param) formed by every CTA from the parameter itself (40 KB out of L2 at the reference's 10000
// entries), so that no launch or host sync separates the sum from its use; CTA 0 stores S for the backward
__global__ void __launch_bounds__(256)
fixed_head_fwd_kernel(const float* __restrict__ z, int ldz, int n_out, const float* __restrict__ Tp, int n_t,
                      float* __restrict__ out, int ldo, float* __restrict__ S_out, int rows) {
  __shared__ float red[256];
  const float S = cta_sum_256(Tp, n_t, red);
  if (blockIdx.x == 0 && threadIdx.x == 0) *S_out = S;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int row = warp; row < rows; row += nwarps) {
    const float* zr = z + static_cast<size_t>(row) * ldz;
    float* o = out + static_cast<size_t>(row) * ldo;
    for (int c = lane; c < n_out; c += 32) o[c] = zr[c] / S;
  }
}

// dz = g / S with zero padding; row_dot[row] = sum_j g_j z_j (lanes sequential, then the butterfly)
template <typename TD>
__global__ void __launch_bounds__(256)
fixed_head_bwd_rows_kernel(const float* __restrict__ g, int ldg, const float* __restrict__ z, int ldz,
                           const float* __restrict__ S_in, int n_out, TD* __restrict__ dz, int ldd, int n_cols_pad,
                           float* __restrict__ row_dot, int rows) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const float S = *S_in;
  for (int row = warp; row < rows; row += nwarps) {
    const float* zr = z + static_cast<size_t>(row) * ldz;
    const float* gr = g + static_cast<size_t>(row) * ldg;
    TD* d = dz + static_cast<size_t>(row) * ldd;
    float s = 0.f;
    for (int c = lane; c < n_out; c += 32) {
      const float gc = gr[c];
      s = fmaf(gc, zr[c], s);
      d[c] = from_f32<TD>(gc / S);
    }
    for (int c = n_out + lane; c < n_cols_pad; c += 32) d[c] = from_f32<TD>(0.f);
    s = warp_sum(s);
    if (lane == 0) row_dot[row] = s;
  }
}

// One CTA of 1024 threads: D = sum of row_dot (thread i adds rows i, i + 1024, ... in turn, then a fixed 10-level tree);
// every dT_i = -D / S^2
__global__ void __launch_bounds__(1024)
fixed_head_bwd_fill_kernel(const float* __restrict__ row_dot, int rows, const float* __restrict__ S_in,
                           float* __restrict__ dT, int n_t) {
  __shared__ float red[1024];
  float s = 0.f;
  for (int i = threadIdx.x; i < rows; i += 1024) s += row_dot[i];
  red[threadIdx.x] = s;
  __syncthreads();
#pragma unroll
  for (int w = 512; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  const float S = *S_in;
  const float v = -red[0] / (S * S);
  for (int i = threadIdx.x; i < n_t; i += 1024) dT[i] = v;
}

int row_grid(int rows) {
  int grid = (rows + 7) / 8;
  const int max_grid = num_sms() * 8;
  if (grid > max_grid) grid = max_grid;
  return grid > 0 ? grid : 1;
}

}  // namespace pfn

using namespace pfn;

extern "C" int pfn_scaled_head_fwd(const float* zz, int ldz, int n_out, float* out, int ldo, float* temp, int rows,
                                   void* stream) {
  PFN_CHECK_ARG(n_out >= 1 && ldz >= n_out + PFN_HEAD_TEMPS && ldo >= n_out && rows >= 0,
                "scaled_head_fwd: n_out=%d ldz=%d ldo=%d rows=%d", n_out, ldz, ldo, rows);
  if (rows == 0) return 0;
  scaled_head_fwd_kernel<<<row_grid(rows), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(zz, ldz, n_out, out, ldo,
                                                                                             temp, rows);
  PFN_LAUNCH_OK();
  return 0;
}

extern "C" int pfn_scaled_head_bwd(const float* g, int ldg, const float* zz, int ldz, const float* temp, int n_out,
                                   void* dzz, int ldd, int d_dtype, int n_cols_pad, int rows, void* stream) {
  PFN_CHECK_ARG(n_out >= 1 && ldg >= n_out && ldz >= n_out + PFN_HEAD_TEMPS && n_cols_pad >= n_out + PFN_HEAD_TEMPS &&
                ldd >= n_cols_pad && rows >= 0 && (d_dtype == PFN_F32 || d_dtype == PFN_BF16),
                "scaled_head_bwd: n_out=%d ldg=%d ldz=%d pad=%d ldd=%d rows=%d dtype=%d", n_out, ldg, ldz, n_cols_pad,
                ldd, rows, d_dtype);
  if (rows == 0) return 0;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (d_dtype == PFN_F32)
    scaled_head_bwd_kernel<float><<<row_grid(rows), 256, 0, s>>>(g, ldg, zz, ldz, temp, n_out,
                                                                reinterpret_cast<float*>(dzz), ldd, n_cols_pad, rows);
  else
    scaled_head_bwd_kernel<__nv_bfloat16><<<row_grid(rows), 256, 0, s>>>(
        g, ldg, zz, ldz, temp, n_out, reinterpret_cast<__nv_bfloat16*>(dzz), ldd, n_cols_pad, rows);
  PFN_LAUNCH_OK();
  return 0;
}

extern "C" int pfn_fixed_scaled_head_fwd(const float* z, int ldz, int n_out, const float* T, int n_t, float* out,
                                         int ldo, float* S, int rows, void* stream) {
  PFN_CHECK_ARG(n_out >= 1 && ldz >= n_out && ldo >= n_out && n_t >= 1 && rows >= 0,
                "fixed_scaled_head_fwd: n_out=%d ldz=%d ldo=%d n_t=%d rows=%d", n_out, ldz, ldo, n_t, rows);
  fixed_head_fwd_kernel<<<row_grid(rows), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(z, ldz, n_out, T, n_t, out,
                                                                                            ldo, S, rows);
  PFN_LAUNCH_OK();
  return 0;
}

extern "C" int pfn_fixed_scaled_head_bwd(const float* g, int ldg, const float* z, int ldz, const float* S, int n_out,
                                         void* dz, int ldd, int d_dtype, int n_cols_pad, float* row_dot, float* dT,
                                         int n_t, int rows, void* stream) {
  PFN_CHECK_ARG(n_out >= 1 && ldg >= n_out && ldz >= n_out && n_cols_pad >= n_out && ldd >= n_cols_pad && n_t >= 1 &&
                rows >= 0 && (d_dtype == PFN_F32 || d_dtype == PFN_BF16),
                "fixed_scaled_head_bwd: n_out=%d ldg=%d ldz=%d pad=%d ldd=%d n_t=%d rows=%d dtype=%d", n_out, ldg, ldz,
                n_cols_pad, ldd, n_t, rows, d_dtype);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (rows > 0) {
    if (d_dtype == PFN_F32)
      fixed_head_bwd_rows_kernel<float><<<row_grid(rows), 256, 0, s>>>(g, ldg, z, ldz, S, n_out,
                                                                       reinterpret_cast<float*>(dz), ldd, n_cols_pad,
                                                                       row_dot, rows);
    else
      fixed_head_bwd_rows_kernel<__nv_bfloat16><<<row_grid(rows), 256, 0, s>>>(
          g, ldg, z, ldz, S, n_out, reinterpret_cast<__nv_bfloat16*>(dz), ldd, n_cols_pad, row_dot, rows);
    PFN_LAUNCH_OK();
  }
  fixed_head_bwd_fill_kernel<<<1, 1024, 0, s>>>(row_dot, rows, S, dT, n_t);
  PFN_LAUNCH_OK();
  return 0;
}
