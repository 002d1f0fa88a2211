// HBM-bound row kernels of the transformer step: embedding, LayerNorm fwd/bwd, column sums.
// One warp per token row, 16-byte vector accesses, fp32 statistics; column reductions (dgamma, dbeta, bias
// gradients) are accumulated per lane across the rows a warp owns, combined per CTA in shared memory and
// flushed with one atomicAdd per column per CTA.
#include "common.cuh"
#include "../../include/pfn_b200.h"

namespace pfn {

// --------------------------------------------------------------------------------------------
// 8-element vector load/store helpers (bf16: one 16 B access, fp32: two 16 B accesses)
// --------------------------------------------------------------------------------------------
template <typename T> __device__ __forceinline__ void load8(const T* p, float (&v)[8]);
template <> __device__ __forceinline__ void load8<float>(const float* p, float (&v)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p);
  const float4 b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
template <> __device__ __forceinline__ void load8<__nv_bfloat16>(const __nv_bfloat16* p, float (&v)[8]) {
  const uint4 pk = *reinterpret_cast<const uint4*>(p);
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&pk);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 t = __bfloat1622float2(h[j]);
    v[2 * j] = t.x; v[2 * j + 1] = t.y;
  }
}
template <typename T> __device__ __forceinline__ void store8(T* p, const float (&v)[8]);
template <> __device__ __forceinline__ void store8<float>(float* p, const float (&v)[8]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
}
template <> __device__ __forceinline__ void store8<__nv_bfloat16>(__nv_bfloat16* p, const float (&v)[8]) {
  uint4 pk;
  __nv_bfloat162 t0 = __floats2bfloat162_rn(v[0], v[1]);
  __nv_bfloat162 t1 = __floats2bfloat162_rn(v[2], v[3]);
  __nv_bfloat162 t2 = __floats2bfloat162_rn(v[4], v[5]);
  __nv_bfloat162 t3 = __floats2bfloat162_rn(v[6], v[7]);
  pk.x = *reinterpret_cast<uint32_t*>(&t0); pk.y = *reinterpret_cast<uint32_t*>(&t1);
  pk.z = *reinterpret_cast<uint32_t*>(&t2); pk.w = *reinterpret_cast<uint32_t*>(&t3);
  *reinterpret_cast<uint4*>(p) = pk;
}

// --------------------------------------------------------------------------------------------
// Embedding forward: out[row,:] = x[row,:] Wx^T + bx + (t < sep ? y[row] wy + by : 0)
// --------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
embed_fwd_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ Wx,
                 const float* __restrict__ bx, const float* __restrict__ wy, const float* __restrict__ by,
                 T* __restrict__ out, int rows, int train_rows, int F, int E) {
  constexpr int ROWS = 8;
  extern __shared__ float sx[];  // [ROWS][F] + [ROWS] y
  float* sy = sx + ROWS * F;
  const int r0 = blockIdx.x * ROWS;
  for (int i = threadIdx.x; i < ROWS * F; i += blockDim.x) {
    const int r = r0 + i / F;
    sx[i] = r < rows ? x[static_cast<size_t>(r0) * F + i] : 0.f;
  }
  if (threadIdx.x < ROWS) {
    const int r = r0 + threadIdx.x;
    sy[threadIdx.x] = (r < rows && r < train_rows) ? y[r] : 0.f;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    const float bxe = bx[e], wye = wy[e], bye = by[e];
    float acc[ROWS];
#pragma unroll
    for (int r = 0; r < ROWS; ++r) acc[r] = bxe;
    for (int f = 0; f < F; ++f) {
      const float w = Wx[static_cast<size_t>(e) * F + f];
#pragma unroll
      for (int r = 0; r < ROWS; ++r) acc[r] = fmaf(sx[r * F + f], w, acc[r]);
    }
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      const int row = r0 + r;
      if (row < rows) {
        float v = acc[r];
        if (row < train_rows) v += fmaf(sy[r], wye, bye);
        out[static_cast<size_t>(row) * E + e] = from_f32<T>(v);
      }
    }
  }
}

// Embedding backward: thread owns column e, loops over a chunk of rows.
template <typename T, int FMAX>
__global__ void __launch_bounds__(128)
embed_bwd_kernel(const T* __restrict__ dout, const float* __restrict__ x, const float* __restrict__ y,
                 float* __restrict__ dWx, float* __restrict__ dbx, float* __restrict__ dwy, float* __restrict__ dby,
                 int rows, int train_rows, int F, int E, int rows_per_cta, int f0) {
  const int e = blockIdx.y * blockDim.x + threadIdx.x;
  const int r_begin = blockIdx.x * rows_per_cta;
  const int r_end = min(r_begin + rows_per_cta, rows);
  float accw[FMAX];
#pragma unroll
  for (int f = 0; f < FMAX; ++f) accw[f] = 0.f;
  float sd = 0.f, sdt = 0.f, sdy = 0.f;
  if (e < E) {
    for (int r = r_begin; r < r_end; ++r) {
      const float d = to_f32<T>(dout[static_cast<size_t>(r) * E + e]);
      sd += d;
      if (r < train_rows) { sdt += d; sdy = fmaf(d, y[r], sdy); }
#pragma unroll
      for (int f = 0; f < FMAX; ++f)
        if (f0 + f < F) accw[f] = fmaf(d, x[static_cast<size_t>(r) * F + f0 + f], accw[f]);
    }
#pragma unroll
    for (int f = 0; f < FMAX; ++f)
      if (f0 + f < F) atomicAdd(&dWx[static_cast<size_t>(e) * F + f0 + f], accw[f]);
    if (f0 == 0) {
      atomicAdd(&dbx[e], sd);
      atomicAdd(&dwy[e], sdy);
      atomicAdd(&dby[e], sdt);
    }
  }
}

// --------------------------------------------------------------------------------------------
// LayerNorm forward / backward.  One warp per row, NCH = 8-element chunks per lane (E <= 256*NCH).  Each warp stages its
// input rows through a private cp.async ring in shared memory and reduces one row while the next DEPTH - 1 are in flight,
// so the bytes in flight take no registers.  That matters most in the backward, whose three per-lane column accumulators
// need twice the registers of the forward: it runs half the forward's 8-warp CTAs per SM.  A ring slot holds columns
// [0, ROW) of one row as they lie in memory, so a lane's chunk sits at the same column offset in the slot as in the row.
// --------------------------------------------------------------------------------------------
template <typename T, int NCH>
struct LnRing {
  static constexpr int ROW = NCH * 256;                         // elements of one staged row
  static constexpr int ROW_BYTES = ROW * sizeof(T);
  // Two forward CTAs and one backward CTA per SM; rows of at most 512 B run twice as many, because with so little work
  // per row the warps of one or two CTAs cannot hide each row's shuffle reductions, and no ring depth makes up for it
  // (measured at bf16 E = 128 on an H100).
  static constexpr int FWD_CTAS = ROW_BYTES <= 512 ? 4 : 2, BWD_CTAS = FWD_CTAS / 2;
  // 128 KB of ring per SM in either direction (8 rows at bf16 E = 512), but at least 3 rows, so that two stay in flight
  // beyond the one being reduced.
  static constexpr int DEPTH = 8192 / (BWD_CTAS * ROW_BYTES) > 3 ? 8192 / (BWD_CTAS * ROW_BYTES) : 3;
  static constexpr size_t WARP_BYTES = static_cast<size_t>(DEPTH) * ROW_BYTES;  // one tensor's ring of one warp
};

// One lane's 8-element chunk, global -> shared: one 16-byte cp.async for bf16, two for fp32.
template <typename T>
__device__ __forceinline__ void ln_cp_async8(T* smem_dst, const T* gsrc) {
#pragma unroll
  for (int k = 0; k < 8; k += 16 / static_cast<int>(sizeof(T)))
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;"
                 ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst + k))), "l"(gsrc + k) : "memory");
}

template <typename T, int NCH>
__global__ void __launch_bounds__(256, LnRing<T, NCH>::FWD_CTAS)
layernorm_fwd_kernel(const T* __restrict__ z, int ldz, const float* __restrict__ gamma, const float* __restrict__ beta,
                     T* __restrict__ h, int ldh, float* __restrict__ mean_out, float* __restrict__ rstd_out, int rows,
                     int E, float eps) {
  using R = LnRing<T, NCH>;
  extern __shared__ __align__(16) uint8_t ln_smem[];
  const int lane = threadIdx.x & 31;
  const int warp_in_cta = threadIdx.x >> 5;
  const int warps_per_cta = blockDim.x >> 5;
  T* ring = reinterpret_cast<T*>(ln_smem) + static_cast<size_t>(warp_in_cta) * R::DEPTH * R::ROW;
  const int warp = blockIdx.x * warps_per_cta + warp_in_cta;
  const int nwarps = gridDim.x * warps_per_cta;
  const float inv_e = 1.0f / static_cast<float>(E);
  float gm[NCH][8], bt[NCH][8];
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
#pragma unroll
    for (int i = 0; i < 8; ++i) { gm[c][i] = 0.f; bt[c][i] = 0.f; }
    const int col = (c * 32 + lane) * 8;
    if (col < E) { load8<float>(gamma + col, gm[c]); load8<float>(beta + col, bt[c]); }
  }
  auto issue = [&](int r, int slot) {
    if (r < rows) {
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        const int col = (c * 32 + lane) * 8;
        if (col < E) ln_cp_async8(ring + slot * R::ROW + col, z + static_cast<size_t>(r) * ldz + col);
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
#pragma unroll
  for (int k = 0; k < R::DEPTH - 1; ++k) issue(warp + k * nwarps, k);
  int it = 0;
  for (int row = warp; row < rows; row += nwarps, ++it) {
    asm volatile("cp.async.wait_group %0;" ::"n"(R::DEPTH - 2) : "memory");
    __syncwarp();                       // this row has landed for every lane; every lane is done with the slot refilled next
    const T* zr = ring + (it % R::DEPTH) * R::ROW;
    issue(row + (R::DEPTH - 1) * nwarps, (it + R::DEPTH - 1) % R::DEPTH);
    float v[NCH][8];
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int col = (c * 32 + lane) * 8;
      if (col < E) {
        load8<T>(zr + col, v[c]);
#pragma unroll
        for (int i = 0; i < 8; ++i) s += v[c][i];
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) v[c][i] = 0.f;
      }
    }
    const float mean = warp_sum(s) * inv_e;
    float ss = 0.f;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int col = (c * 32 + lane) * 8;
      if (col < E) {
#pragma unroll
        for (int i = 0; i < 8; ++i) { const float dlt = v[c][i] - mean; ss = fmaf(dlt, dlt, ss); }
      }
    }
    const float rstd = rsqrtf(warp_sum(ss) * inv_e + eps);
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int col = (c * 32 + lane) * 8;
      if (col < E) {
        float o[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] = fmaf((v[c][i] - mean) * rstd, gm[c][i], bt[c][i]);
        store8<T>(h + static_cast<size_t>(row) * ldh + col, o);
      }
    }
    if (lane == 0) { mean_out[row] = mean; rstd_out[row] = rstd; }
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
}

// Shared memory: sred [3][E] for the CTA's column sums, then each warp's ring, whose slot k holds dh in half 2k and z in
// half 2k + 1.
template <typename T, int NCH>
__global__ void __launch_bounds__(256, LnRing<T, NCH>::BWD_CTAS)
layernorm_bwd_kernel(const T* __restrict__ dh, int lddh, const T* __restrict__ z, int ldz,
                     const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
                     const float* __restrict__ gamma, T* __restrict__ dz, int lddz, float* __restrict__ dgamma,
                     float* __restrict__ dbeta, float* __restrict__ colsum_out, int rows, int E) {
  using R = LnRing<T, NCH>;
  extern __shared__ __align__(16) uint8_t ln_smem[];
  float* sred = reinterpret_cast<float*>(ln_smem);
  const int lane = threadIdx.x & 31;
  const int warp_in_cta = threadIdx.x >> 5;
  const int warps_per_cta = blockDim.x >> 5;
  T* ring = reinterpret_cast<T*>(ln_smem + ((3 * E * 4 + 15) & ~15)) + static_cast<size_t>(warp_in_cta) * R::DEPTH * 2 * R::ROW;
  const int warp = blockIdx.x * warps_per_cta + warp_in_cta;
  const int nwarps = gridDim.x * warps_per_cta;
  const float inv_e = 1.0f / static_cast<float>(E);
  for (int i = threadIdx.x; i < 3 * E; i += blockDim.x) sred[i] = 0.f;
  __syncthreads();

  float ag[NCH][8], ab[NCH][8], ac[NCH][8], gm[NCH][8];
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
#pragma unroll
    for (int i = 0; i < 8; ++i) { ag[c][i] = 0.f; ab[c][i] = 0.f; ac[c][i] = 0.f; gm[c][i] = 0.f; }
    const int col = (c * 32 + lane) * 8;
    if (col < E) load8<float>(gamma + col, gm[c]);
  }
  auto issue = [&](int r, int slot) {
    if (r < rows) {
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        const int col = (c * 32 + lane) * 8;
        if (col < E) {
          ln_cp_async8(ring + (slot * 2 + 0) * R::ROW + col, dh + static_cast<size_t>(r) * lddh + col);
          ln_cp_async8(ring + (slot * 2 + 1) * R::ROW + col, z + static_cast<size_t>(r) * ldz + col);
        }
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
#pragma unroll
  for (int k = 0; k < R::DEPTH - 1; ++k) issue(warp + k * nwarps, k);
  float m_l = 0.f, s_l = 0.f;         // statistics of rows it .. it + 31 of this warp, one per lane
  int it = 0;
  for (int row = warp; row < rows; row += nwarps, ++it) {
    if ((it & 31) == 0) {
      const long long r = static_cast<long long>(row) + static_cast<long long>(lane) * nwarps;
      m_l = r < rows ? __ldg(mean_in + r) : 0.f;
      s_l = r < rows ? __ldg(rstd_in + r) : 0.f;
    }
    const float mean = __shfl_sync(0xffffffffu, m_l, it & 31), rstd = __shfl_sync(0xffffffffu, s_l, it & 31);
    asm volatile("cp.async.wait_group %0;" ::"n"(R::DEPTH - 2) : "memory");
    __syncwarp();                       // this row has landed for every lane; every lane is done with the slot refilled next
    const T* dr = ring + (it % R::DEPTH) * 2 * R::ROW;
    const T* zr = dr + R::ROW;
    float xh[NCH][8], g[NCH][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int col = (c * 32 + lane) * 8;
      if (col < E) {
        float d[8], zz[8];
        load8<T>(dr + col, d);
        load8<T>(zr + col, zz);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          xh[c][i] = (zz[i] - mean) * rstd;
          g[c][i] = d[i] * gm[c][i];
          s1 += g[c][i];
          s2 = fmaf(g[c][i], xh[c][i], s2);
          ag[c][i] = fmaf(d[i], xh[c][i], ag[c][i]);
          ab[c][i] += d[i];
        }
      }
    }
    issue(row + (R::DEPTH - 1) * nwarps, (it + R::DEPTH - 1) % R::DEPTH);   // after the reads of this row's slot
    s1 = warp_sum(s1) * inv_e;
    s2 = warp_sum(s2) * inv_e;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int col = (c * 32 + lane) * 8;
      if (col < E) {
        float o[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          o[i] = rstd * (g[c][i] - s1 - xh[c][i] * s2);
          ac[c][i] += o[i];
        }
        store8<T>(dz + static_cast<size_t>(row) * lddz + col, o);
      }
    }
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  // CTA-level combine, then one atomic per column per CTA
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    const int col = (c * 32 + lane) * 8;
    if (col < E) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        atomicAdd(&sred[col + i], ag[c][i]);
        atomicAdd(&sred[E + col + i], ab[c][i]);
        atomicAdd(&sred[2 * E + col + i], ac[c][i]);
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < E; i += blockDim.x) {
    if (dgamma != nullptr) atomicAdd(&dgamma[i], sred[i]);
    if (dbeta != nullptr) atomicAdd(&dbeta[i], sred[E + i]);
    if (colsum_out != nullptr) atomicAdd(&colsum_out[i], sred[2 * E + i]);
  }
}

// Generic (any E) fallbacks: one warp per row, scalar accesses, re-reading the row from cache.
template <typename T>
__global__ void layernorm_fwd_generic(const T* z, int ldz, const float* gamma, const float* beta, T* h, int ldh,
                                      float* mean_out, float* rstd_out, int rows, int E, float eps) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int row = warp; row < rows; row += nwarps) {
    const T* zr = z + static_cast<size_t>(row) * ldz;
    float s = 0.f;
    for (int i = lane; i < E; i += 32) s += to_f32<T>(zr[i]);
    const float mean = warp_sum(s) / E;
    float ss = 0.f;
    for (int i = lane; i < E; i += 32) { const float d = to_f32<T>(zr[i]) - mean; ss = fmaf(d, d, ss); }
    const float rstd = rsqrtf(warp_sum(ss) / E + eps);
    for (int i = lane; i < E; i += 32)
      h[static_cast<size_t>(row) * ldh + i] = from_f32<T>(fmaf((to_f32<T>(zr[i]) - mean) * rstd, gamma[i], beta[i]));
    if (lane == 0) { mean_out[row] = mean; rstd_out[row] = rstd; }
  }
}

template <typename T>
__global__ void layernorm_bwd_generic(const T* dh, int lddh, const T* z, int ldz, const float* mean_in,
                                      const float* rstd_in, const float* gamma, T* dz, int lddz, float* dgamma,
                                      float* dbeta, float* colsum_out, int rows, int E) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int row = warp; row < rows; row += nwarps) {
    const float mean = mean_in[row], rstd = rstd_in[row];
    const T* zr = z + static_cast<size_t>(row) * ldz;
    const T* dr = dh + static_cast<size_t>(row) * lddh;
    float s1 = 0.f, s2 = 0.f;
    for (int i = lane; i < E; i += 32) {
      const float xh = (to_f32<T>(zr[i]) - mean) * rstd;
      const float g = to_f32<T>(dr[i]) * gamma[i];
      s1 += g; s2 = fmaf(g, xh, s2);
    }
    s1 = warp_sum(s1) / E; s2 = warp_sum(s2) / E;
    for (int i = lane; i < E; i += 32) {
      const float xh = (to_f32<T>(zr[i]) - mean) * rstd;
      const float d = to_f32<T>(dr[i]);
      const float o = rstd * (d * gamma[i] - s1 - xh * s2);
      dz[static_cast<size_t>(row) * lddz + i] = from_f32<T>(o);
      if (dgamma != nullptr) atomicAdd(&dgamma[i], d * xh);
      if (dbeta != nullptr) atomicAdd(&dbeta[i], d);
      if (colsum_out != nullptr) atomicAdd(&colsum_out[i], o);
    }
  }
}

// --------------------------------------------------------------------------------------------
// Column sums.  Vector path: one warp streams whole rows with 16 B loads (lane owns 8 consecutive columns per
// 256-column group), accumulates in registers over the rows it owns, CTA combines in shared memory, one atomicAdd
// per column per CTA.  Generic path: one thread per column.
// --------------------------------------------------------------------------------------------
template <typename T, int NV>
__global__ void __launch_bounds__(256)
colsum_vec_kernel(const T* __restrict__ X0, int ld, float* __restrict__ out0, int rows, int N0) {
  extern __shared__ float sred[];   // [N]
  // blockIdx.y selects a group of NV*256 columns
  const int col_base = blockIdx.y * NV * 256;
  const T* X = X0 + col_base;
  float* out = out0 + col_base;
  const int N = min(N0 - col_base, NV * 256);
  const int lane = threadIdx.x & 31;
  const int warps_per_cta = blockDim.x >> 5;
  const int warp = blockIdx.x * warps_per_cta + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * warps_per_cta;
  for (int i = threadIdx.x; i < N; i += blockDim.x) sred[i] = 0.f;
  __syncthreads();
  float acc[NV][8];
#pragma unroll
  for (int v = 0; v < NV; ++v)
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[v][i] = 0.f;
  for (int row = warp; row < rows; row += nwarps) {
    const T* xr = X + static_cast<size_t>(row) * ld;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      const int col = (v * 32 + lane) * 8;
      if (col < N) {
        float x[8];
        load8<T>(xr + col, x);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[v][i] += x[i];
      }
    }
  }
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    const int col = (v * 32 + lane) * 8;
    if (col < N) {
#pragma unroll
      for (int i = 0; i < 8; ++i) atomicAdd(&sred[col + i], acc[v][i]);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < N; i += blockDim.x) atomicAdd(&out[i], sred[i]);
}

template <typename T>
__global__ void __launch_bounds__(256)
colsum_kernel(const T* __restrict__ X, int ld, float* __restrict__ out, int rows, int N, int rows_per_cta) {
  const int col = blockIdx.y * blockDim.x + threadIdx.x;
  const int r_begin = blockIdx.x * rows_per_cta;
  const int r_end = min(r_begin + rows_per_cta, rows);
  if (col >= N) return;
  float s = 0.f;
  for (int r = r_begin; r < r_end; ++r) s += to_f32<T>(X[static_cast<size_t>(r) * ld + col]);
  atomicAdd(&out[col], s);
}

}  // namespace pfn

using namespace pfn;

extern "C" int pfn_embed_fwd(const float* x, const float* y, const float* Wx, const float* bx, const float* wy,
                             const float* by, void* out, int out_dtype, int T, int B, int F, int E, int sep,
                             void* stream) {
  PFN_CHECK_ARG(T > 0 && B > 0 && F > 0 && E > 0, "embed_fwd: bad shape T=%d B=%d F=%d E=%d", T, B, F, E);
  PFN_CHECK_ARG(sep >= 0 && sep <= T, "embed_fwd: sep %d outside [0,%d]", sep, T);
  PFN_CHECK_ARG(F <= 1024, "embed_fwd: F=%d too large for the fused kernel (route through the GEMM)", F);
  const int rows = T * B, train_rows = sep * B;
  const int grid = (rows + 7) / 8;
  const size_t smem = (8 * F + 8) * sizeof(float);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (out_dtype == PFN_F32)
    embed_fwd_kernel<float><<<grid, 256, smem, s>>>(x, y, Wx, bx, wy, by, reinterpret_cast<float*>(out), rows,
                                                    train_rows, F, E);
  else
    embed_fwd_kernel<__nv_bfloat16><<<grid, 256, smem, s>>>(x, y, Wx, bx, wy, by,
                                                            reinterpret_cast<__nv_bfloat16*>(out), rows, train_rows, F, E);
  PFN_LAUNCH_OK();
  return 0;
}

extern "C" int pfn_embed_bwd(const void* dout, int dtype, const float* x, const float* y, float* dWx, float* dbx,
                             float* dwy, float* dby, int T, int B, int F, int E, int sep, void* stream) {
  PFN_CHECK_ARG(T > 0 && B > 0 && F > 0 && E > 0, "embed_bwd: bad shape");
  PFN_CHECK_ARG(sep >= 0 && sep <= T, "embed_bwd: sep %d outside [0,%d]", sep, T);
  const int rows = T * B, train_rows = sep * B;
  const int rows_per_cta = 512;
  dim3 grid((rows + rows_per_cta - 1) / rows_per_cta, (E + 127) / 128);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  constexpr int FMAX = 8;
  for (int f0 = 0; f0 < F; f0 += FMAX) {
    if (dtype == PFN_F32)
      embed_bwd_kernel<float, FMAX><<<grid, 128, 0, s>>>(reinterpret_cast<const float*>(dout), x, y, dWx, dbx, dwy, dby,
                                                         rows, train_rows, F, E, rows_per_cta, f0);
    else
      embed_bwd_kernel<__nv_bfloat16, FMAX><<<grid, 128, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(dout), x, y, dWx,
                                                                 dbx, dwy, dby, rows, train_rows, F, E, rows_per_cta, f0);
    PFN_LAUNCH_OK();
  }
  return 0;
}

// Vector-path launches: LnRing's CTAs per SM, no more than the rows need.  An SM has 228 KB of shared memory, of which
// 1 KB is reserved per CTA.
template <typename T, int NCH>
static int layernorm_fwd_vec(const T* z, int ldz, const float* gamma, const float* beta, T* h, int ldh, float* mean,
                             float* rstd, int rows, int E, float eps, cudaStream_t s) {
  using R = LnRing<T, NCH>;
  constexpr size_t smem = 8 * R::WARP_BYTES;
  static_assert(R::FWD_CTAS * (smem + 1024) <= 228 * 1024, "the forward CTAs must fit on an SM");
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set))
    PFN_CUDA_OK(cudaFuncSetAttribute(layernorm_fwd_kernel<T, NCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  int grid = R::FWD_CTAS * num_sms();
  if (grid > (rows + 7) / 8) grid = (rows + 7) / 8;
  layernorm_fwd_kernel<T, NCH><<<grid, 256, smem, s>>>(z, ldz, gamma, beta, h, ldh, mean, rstd, rows, E, eps);
  PFN_LAUNCH_OK();
  return 0;
}

template <typename T, int NCH>
static int layernorm_bwd_vec(const T* dh, int lddh, const T* z, int ldz, const float* mean, const float* rstd,
                             const float* gamma, T* dz, int lddz, float* dgamma, float* dbeta, float* colsum_out, int rows,
                             int E, cudaStream_t s) {
  using R = LnRing<T, NCH>;
  constexpr size_t rings = 8 * 2 * R::WARP_BYTES;
  constexpr size_t max_smem = 3 * R::ROW * sizeof(float) + rings;
  static_assert(R::BWD_CTAS * (max_smem + 1024) <= 228 * 1024, "the backward CTAs must fit on an SM");
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set))
    PFN_CUDA_OK(cudaFuncSetAttribute(layernorm_bwd_kernel<T, NCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(max_smem)));
  const size_t smem = ((3 * static_cast<size_t>(E) * 4 + 15) & ~size_t(15)) + rings;
  int grid = R::BWD_CTAS * num_sms();
  if (grid > (rows + 7) / 8) grid = (rows + 7) / 8;
  layernorm_bwd_kernel<T, NCH><<<grid, 256, smem, s>>>(dh, lddh, z, ldz, mean, rstd, gamma, dz, lddz, dgamma, dbeta, colsum_out, rows, E);
  PFN_LAUNCH_OK();
  return 0;
}

template <typename T>
static int layernorm_fwd_dispatch(const void* z, int ldz, const float* gamma, const float* beta, void* h, int ldh,
                                  float* mean, float* rstd, int rows, int E, float eps, cudaStream_t s) {
  const T* zp = reinterpret_cast<const T*>(z);
  T* hp = reinterpret_cast<T*>(h);
  const bool vec = (E % 8 == 0) && (ldz % 8 == 0) && (ldh % 8 == 0) && E <= 1024 &&
                   ((reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(h) |
                     reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(beta)) & 15) == 0;
  if (vec) {
    if (E <= 256) return layernorm_fwd_vec<T, 1>(zp, ldz, gamma, beta, hp, ldh, mean, rstd, rows, E, eps, s);
    if (E <= 512) return layernorm_fwd_vec<T, 2>(zp, ldz, gamma, beta, hp, ldh, mean, rstd, rows, E, eps, s);
    return layernorm_fwd_vec<T, 4>(zp, ldz, gamma, beta, hp, ldh, mean, rstd, rows, E, eps, s);
  }
  int grid = (rows + 7) / 8;
  if (grid > num_sms() * 8) grid = num_sms() * 8;
  layernorm_fwd_generic<T><<<grid, 256, 0, s>>>(zp, ldz, gamma, beta, hp, ldh, mean, rstd, rows, E, eps);
  PFN_LAUNCH_OK();
  return 0;
}

extern "C" int pfn_layernorm_fwd(const void* z, int ldz, const float* gamma, const float* beta, void* h, int ldh,
                                 float* mean, float* rstd, int rows, int E, float eps, int dtype, void* stream) {
  PFN_CHECK_ARG(rows > 0 && E > 0, "layernorm_fwd: bad shape rows=%d E=%d", rows, E);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == PFN_F32) return layernorm_fwd_dispatch<float>(z, ldz, gamma, beta, h, ldh, mean, rstd, rows, E, eps, s);
  return layernorm_fwd_dispatch<__nv_bfloat16>(z, ldz, gamma, beta, h, ldh, mean, rstd, rows, E, eps, s);
}

template <typename T>
static int layernorm_bwd_dispatch(const void* dh, int lddh, const void* z, int ldz, const float* mean,
                                  const float* rstd, const float* gamma, void* dz, int lddz, float* dgamma, float* dbeta,
                                  float* colsum_out, int rows, int E, cudaStream_t s) {
  const T* dhp = reinterpret_cast<const T*>(dh);
  const T* zp = reinterpret_cast<const T*>(z);
  T* dzp = reinterpret_cast<T*>(dz);
  const bool vec = (E % 8 == 0) && (ldz % 8 == 0) && (lddh % 8 == 0) && (lddz % 8 == 0) && E <= 1024 &&
                   ((reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(dh) | reinterpret_cast<uintptr_t>(dz) |
                     reinterpret_cast<uintptr_t>(gamma)) & 15) == 0;
  if (vec) {
    if (E <= 256) return layernorm_bwd_vec<T, 1>(dhp, lddh, zp, ldz, mean, rstd, gamma, dzp, lddz, dgamma, dbeta, colsum_out, rows, E, s);
    if (E <= 512) return layernorm_bwd_vec<T, 2>(dhp, lddh, zp, ldz, mean, rstd, gamma, dzp, lddz, dgamma, dbeta, colsum_out, rows, E, s);
    return layernorm_bwd_vec<T, 4>(dhp, lddh, zp, ldz, mean, rstd, gamma, dzp, lddz, dgamma, dbeta, colsum_out, rows, E, s);
  }
  int grid = (rows + 7) / 8;
  if (grid > num_sms() * 4) grid = num_sms() * 4;
  layernorm_bwd_generic<T><<<grid, 256, 0, s>>>(dhp, lddh, zp, ldz, mean, rstd, gamma, dzp, lddz, dgamma, dbeta, colsum_out, rows, E);
  PFN_LAUNCH_OK();
  return 0;
}

extern "C" int pfn_layernorm_bwd(const void* dh, int lddh, const void* z, int ldz, const float* mean, const float* rstd,
                                 const float* gamma, void* dz, int lddz, float* dgamma, float* dbeta, float* colsum_out,
                                 int rows, int E, int dtype, void* stream) {
  PFN_CHECK_ARG(rows > 0 && E > 0, "layernorm_bwd: bad shape rows=%d E=%d", rows, E);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == PFN_F32)
    return layernorm_bwd_dispatch<float>(dh, lddh, z, ldz, mean, rstd, gamma, dz, lddz, dgamma, dbeta, colsum_out, rows, E, s);
  return layernorm_bwd_dispatch<__nv_bfloat16>(dh, lddh, z, ldz, mean, rstd, gamma, dz, lddz, dgamma, dbeta, colsum_out, rows, E, s);
}

template <typename T>
static int colsum_dispatch(const void* X, int ld, float* out, int rows, int N, cudaStream_t s) {
  const T* xp = reinterpret_cast<const T*>(X);
  const bool vec = (N % 8 == 0) && (ld % 8 == 0) && (reinterpret_cast<uintptr_t>(X) & 15) == 0;
  if (vec) {
    int gx = num_sms() * 4;
    const int max_grid = (rows + 7) / 8;
    if (gx > max_grid) gx = max_grid;
    if (N <= 256) colsum_vec_kernel<T, 1><<<gx, 256, 256 * sizeof(float), s>>>(xp, ld, out, rows, N);
    else if (N <= 512) colsum_vec_kernel<T, 2><<<gx, 256, 512 * sizeof(float), s>>>(xp, ld, out, rows, N);
    else {
      const int groups = (N + 1023) / 1024;            // 1024 columns (NV = 4) per blockIdx.y
      int gxx = gx / groups > 0 ? (gx * 2) / groups : 1;
      if (gxx > max_grid) gxx = max_grid;
      colsum_vec_kernel<T, 4><<<dim3(gxx, groups), 256, 1024 * sizeof(float), s>>>(xp, ld, out, rows, N);
    }
  } else {
    int rows_per_cta = (rows + num_sms() * 2 - 1) / (num_sms() * 2);
    if (rows_per_cta < 64) rows_per_cta = 64;
    dim3 grid((rows + rows_per_cta - 1) / rows_per_cta, (N + 255) / 256);
    colsum_kernel<T><<<grid, 256, 0, s>>>(xp, ld, out, rows, N, rows_per_cta);
  }
  PFN_LAUNCH_OK();
  return 0;
}

extern "C" int pfn_colsum(const void* X, int ld, int dtype, float* out, int rows, int N, void* stream) {
  PFN_CHECK_ARG(rows > 0 && N > 0, "colsum: bad shape rows=%d N=%d", rows, N);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == PFN_F32) return colsum_dispatch<float>(X, ld, out, rows, N, s);
  return colsum_dispatch<__nv_bfloat16>(X, ld, out, rows, N, s);
}
