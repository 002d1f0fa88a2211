// Convolutional image encoder (encoders.Conv): valid 3x3 convolutions + ReLU on NHWC activations of 64 channels, their
// data and weight gradients, and the spatial mean that ends the stack.
//
//   conv64_tc_kernel<false>   64 -> 64 forward, bf16: implicit GEMM on wgmma m64n64k16, M = 128 consecutive output pixels
//                             (flattened over images, so that a tile of a small image spans several images and a tile of a
//                             large one a few rows), N = 64, K = 9 taps x 64 channels.  The input pixels the tile reads (its
//                             rows plus the 2-row halo) are staged by cp.async, double-buffered, in 128-byte rows whose
//                             16-byte chunks are XOR-swizzled by the pixel index; ldmatrix gathers the A fragments of every
//                             tap from per-row addresses (the tap is a pixel offset).  The 576 x 64 weight block stays in
//                             shared memory (K-major, 128-byte swizzle) for the persistent CTA's lifetime.  Epilogue: bias,
//                             ReLU, bf16 NHWC store.
//   conv64_tc_kernel<true>    64 -> 64 data gradient, bf16: the same kernel on the zero-padded output gradient with the
//                             flipped weights; the epilogue applies the ReLU mask of the layer below and writes that
//                             layer's padded gradient, its zero border included.
//   conv64_wgrad_tc_kernel    64 -> 64 weight gradient, bf16: per (pixel chunk, tap) a 64 x 64 block of
//                             dW[co, ci] = sum_p g[p, co] x[p + tap, ci] on mma.m16n8k16 (both operands MN-major, read by
//                             ldmatrix.trans), fp32 partials per chunk; the tap-0 CTAs also sum g for the bias.
//   conv_direct_*             fp32-FMA direct convolutions: the input conv (C_in = 1) in both precisions, and the fp32
//                             parity path of the 64 -> 64 layers.
//   conv_wgrad_reduce_kernel  sums the per-chunk partials in chunk order into dw / db (no floating-point atomics).
#include "common.cuh"
#include "tc_common.cuh"
#include "../../include/pfn_b200.h"

namespace pfn {
namespace {

constexpr int kCh = PFN_CONV_CH;
constexpr int kTile = 128;              // output pixels per wgmma tile: two consumer warpgroups x 64 rows
constexpr int kTcThreads = 256;
constexpr int kWBytes = 9 * kCh * kCh * 2;
constexpr int kBlockPx = 64;            // pixels per k-block of a weight gradient
// most pixel chunks a weight gradient is split into: the input conv's direct kernel has one thread per weight (640), so
// it takes its parallelism from many chunks; the 64 -> 64 gradients have 37 k outputs per chunk
constexpr int kWgradChunks = 128, kWgradChunksIn = 1024;
constexpr int kDirectThreads = 256;

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, bool valid) {
  const uint32_t d = tc::smem_u32(smem_dst);
  const int bytes = valid ? 16 : 0;     // 0: zero-fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldmatrix_x4(uint32_t* r, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t* r, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16_16816(float* d, const uint32_t* a, const uint32_t* b) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
               "{%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// output pixel m of the side-so grids (flattened over images) -> the input pixel of its tap (0, 0) on side-si grids
__host__ __device__ __forceinline__ int in_pixel(int m, int si, int so) {
  const int po = so * so;
  const int n = m / po, rem = m - n * po;
  const int r = rem / so, c = rem - r * so;
  return (n * si + r) * si + c;
}
// output pixel m of the side-so grids -> its pixel in buffers of side so + 2 pad that hold the grids `pad` pixels in
__device__ __forceinline__ int padded_pixel(int m, int so, int pad) { return in_pixel(m, so + 2 * pad, so) + pad * (so + 2 * pad) + pad; }

// The 2-pixel zero border of a padded gradient (side so + 4) is written by the kernels that fill its interior: border
// pixel (R, C) belongs to the interior pixel (clamp(R), clamp(C)), so each is written once, by an edge pixel.
// `fn(offset)` stores zero at the border pixel `offset` pixels away from interior pixel (r, c).
template <typename F>
__device__ __forceinline__ void for_owned_border(int so, int r, int c, F&& fn) {
  if (r > 0 && r < so - 1 && c > 0 && c < so - 1) return;
  const int ps = so + 4;
  const int r0 = r == 0 ? -2 : 0, r1 = r == so - 1 ? 2 : 0, c0 = c == 0 ? -2 : 0, c1 = c == so - 1 ? 2 : 0;
  for (int dr = r0; dr <= r1; ++dr)
    for (int dc = c0; dc <= c1; ++dc)
      if (dr != 0 || dc != 0) fn(dr * ps + dc);
}

// input pixels (rows of 128 B) a tile of kTile consecutive output pixels can read: kTile - 1 steps between its output
// pixels, each +1, +3 at a row end and +2 si + 3 at an image end, then the last pixel's 3 x 3 window
int tc_span(int si) {
  const int so = si - 2;
  return (kTile - 1) + 2 * ((kTile - 1) / so + 1) + 2 * si * ((kTile - 1) / (so * so) + 1) + 2 * si + 3;
}
size_t tc_smem(int si) { return 1024 + kWBytes + 2 * static_cast<size_t>(tc_span(si)) * kCh * 2; }

template <bool DGRAD>
__global__ void __launch_bounds__(kTcThreads, 1)
conv64_tc_kernel(const __nv_bfloat16* __restrict__ in, int si, int M, const __nv_bfloat16* __restrict__ wB,
                 const float* __restrict__ bias, const __nv_bfloat16* __restrict__ mask, __nv_bfloat16* __restrict__ out,
                 int span) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* w_s = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  auto stage = [&](int b) { return w_s + kWBytes + b * span * kCh * 2; };
  const int so = si - 2;
  const int pad = DGRAD ? 2 : 0;
  const int n_tiles = (M + kTile - 1) / kTile;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wg = warp >> 2, wq = warp & 3;

  for (int i = tid; i < 9 * kCh * 8; i += kTcThreads) {
    const int t = i >> 9, co = (i >> 3) & 63, ch = i & 7;
    cp_async16(w_s + t * 8192 + co * 128 + ((ch ^ (co & 7)) << 4), wB + static_cast<size_t>(co) * 9 * kCh + t * kCh + ch * 8, true);
  }
  auto stage_tile = [&](int tile, uint8_t* buf) {
    const int m0 = tile * kTile, m1 = min(m0 + kTile, M) - 1;
    const int base = in_pixel(m0, si, so);
    const int cnt = in_pixel(m1, si, so) + 2 * si + 3 - base;
    for (int i = tid; i < cnt * 8; i += kTcThreads) {
      const int q = i >> 3, ch = i & 7;
      cp_async16(buf + q * 128 + ((ch ^ (q & 7)) << 4), in + static_cast<size_t>(base + q) * kCh + ch * 8, true);
    }
  };

  int tile = blockIdx.x;
  if (tile < n_tiles) stage_tile(tile, stage(0));
  cp_async_commit();
  const uint32_t w_u = tc::smem_u32(w_s);
  for (int it = 0; tile < n_tiles; tile += gridDim.x, ++it) {
    if (tile + static_cast<int>(gridDim.x) < n_tiles) stage_tile(tile + gridDim.x, stage((it + 1) & 1));
    cp_async_commit();
    cp_async_wait<1>();
    tc::fence_proxy_async_smem();       // the weights, written through cp.async, are read by wgmma (async proxy)
    __syncthreads();

    const int m0 = tile * kTile, mlast = min(m0 + kTile, M) - 1;
    const int base = in_pixel(m0, si, so);
    // ldmatrix row of this lane: A row (lane & 15) of the warp's 16, 16-byte chunk 2 kk + (lane >> 4) of K
    const int q0 = in_pixel(min(m0 + wg * 64 + wq * 16 + (lane & 15), mlast), si, so) - base;
    const uint32_t buf_u = tc::smem_u32(stage(it & 1));
    const int half = lane >> 4;
    auto load_tap = [&](uint32_t* a, int t) {
      const int q = q0 + (t / 3) * si + (t % 3);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) ldmatrix_x4(a + 4 * kk, buf_u + q * 128 + (((2 * kk + half) ^ (q & 7)) << 4));
    };
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    uint32_t a[2][16];
    load_tap(a[0], 0);
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      tc::wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        tc::wgmma_m64n64k16_rs(acc, &a[t & 1][4 * kk], tc::wgmma_smem_desc(w_u + t * 8192 + kk * 32, 16, 1024), 1);
      tc::wgmma_commit();
      if (t + 1 < 9) {
        tc::wgmma_wait<1>();            // tap t - 1's MMAs, which read a[(t + 1) & 1], are done
        load_tap(a[(t + 1) & 1], t + 1);
      }
    }
    tc::wgmma_wait<0>();

    const int ps = so + 2 * pad;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = m0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
      if (m > mlast) continue;
      const int n = m / (so * so), rem = m - n * so * so, r = rem / so, c = rem - r * so;
      __nv_bfloat16* o = out + static_cast<size_t>((n * ps + r + pad) * ps + c + pad) * kCh;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int col = 8 * j + 2 * (lane & 3);
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if constexpr (DGRAD) {
          const __nv_bfloat162 mk = *reinterpret_cast<const __nv_bfloat162*>(mask + static_cast<size_t>(m) * kCh + col);
          v0 = __bfloat162float(mk.x) > 0.f ? v0 : 0.f;
          v1 = __bfloat162float(mk.y) > 0.f ? v1 : 0.f;
        } else {
          v0 = fmaxf(v0 + bias[col], 0.f);
          v1 = fmaxf(v1 + bias[col + 1], 0.f);
        }
        *reinterpret_cast<__nv_bfloat162*>(o + col) = __floats2bfloat162_rn(v0, v1);
      }
      if constexpr (DGRAD) {
        const int lane_col = 2 * (lane & 3);
        for_owned_border(so, r, c, [&](int off) {
#pragma unroll
          for (int j = 0; j < 8; ++j)
            *reinterpret_cast<__nv_bfloat162*>(o + static_cast<ptrdiff_t>(off) * kCh + 8 * j + lane_col) =
                __floats2bfloat162_rn(0.f, 0.f);
        });
      }
    }
    __syncthreads();                    // every warp is done with stage(it & 1) before it is refilled
  }
  cp_async_wait<0>();
}

__global__ void __launch_bounds__(128)
conv64_wgrad_tc_kernel(const __nv_bfloat16* __restrict__ g, const __nv_bfloat16* __restrict__ x, int si, int M,
                       int chunk_px, float* __restrict__ ws) {
  __shared__ __align__(128) uint8_t gs[2][kBlockPx * 128];
  __shared__ __align__(128) uint8_t xs[2][kBlockPx * 128];
  const int so = si - 2;
  const int chunk = blockIdx.x, tap = blockIdx.y;
  const int toff = (tap / 3) * si + tap % 3;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp >> 1, wn = warp & 1;
  const int c0 = chunk * chunk_px, c1 = min(c0 + chunk_px, M);
  const int nkb = (c1 - c0 + kBlockPx - 1) / kBlockPx;

  auto stage = [&](int kb, int b) {
    for (int i = tid; i < kBlockPx * 8; i += 128) {
      const int q = i >> 3, ch = i & 7;
      const int m = c0 + kb * kBlockPx + q;
      const bool valid = m < c1;
      const int mm = valid ? m : c0;
      const int sw = ((ch ^ (q & 7)) << 4);
      cp_async16(gs[b] + q * 128 + sw, g + static_cast<size_t>(padded_pixel(mm, so, 2)) * kCh + ch * 8, valid);
      cp_async16(xs[b] + q * 128 + sw, x + static_cast<size_t>(in_pixel(mm, si, so) + toff) * kCh + ch * 8, valid);
    }
  };

  float acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int k = 0; k < 4; ++k) acc[i][j][k] = 0.f;
  float bsum = 0.f;

  stage(0, 0);
  cp_async_commit();
  for (int kb = 0; kb < nkb; ++kb) {
    if (kb + 1 < nkb) stage(kb + 1, (kb + 1) & 1);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const uint32_t g_u = tc::smem_u32(gs[kb & 1]), x_u = tc::smem_u32(xs[kb & 1]);
#pragma unroll
    for (int k16 = 0; k16 < 4; ++k16) {
      uint32_t a[2][4], b[4][2];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const int k = k16 * 16 + (lane & 7) + ((lane >> 4) << 3);
        const int col = wm * 32 + mt * 16 + (((lane >> 3) & 1) << 3);
        ldmatrix_x4_trans(a[mt], g_u + k * 128 + (((col >> 3) ^ (k & 7)) << 4));
      }
#pragma unroll
      for (int np = 0; np < 2; ++np) {
        const int k = k16 * 16 + (lane & 7) + (((lane >> 3) & 1) << 3);
        const int col = wn * 32 + np * 16 + ((lane >> 4) << 3);
        uint32_t r[4];
        ldmatrix_x4_trans(r, x_u + k * 128 + (((col >> 3) ^ (k & 7)) << 4));
        b[2 * np][0] = r[0]; b[2 * np][1] = r[1]; b[2 * np + 1][0] = r[2]; b[2 * np + 1][1] = r[3];
      }
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) mma_bf16_16816(acc[mt][nt], a[mt], b[nt]);
    }
    if (tap == 0 && tid < kCh) {
      const __nv_bfloat16* gb = reinterpret_cast<const __nv_bfloat16*>(gs[kb & 1]);
      for (int q = 0; q < kBlockPx; ++q) bsum += __bfloat162float(gb[q * 64 + (((tid >> 3) ^ (q & 7)) << 3) + (tid & 7)]);
    }
    __syncthreads();
  }
  cp_async_wait<0>();

  constexpr int J = kCh * 9 + 1;
  float* wsc = ws + static_cast<size_t>(chunk) * kCh * J;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int co = wm * 32 + mt * 16 + (lane >> 2) + ((e >> 1) << 3);
        const int ci = wn * 32 + nt * 8 + 2 * (lane & 3) + (e & 1);
        wsc[co * J + ci * 9 + tap] = acc[mt][nt][e];
      }
  if (tap == 0 && tid < kCh) wsc[tid * J + kCh * 9] = bsum;
}

// ---------------------------------------------------------------------------------------------
// direct fp32-FMA kernels: one thread per (output pixel, channel), 4 pixels x 64 channels per block
// ---------------------------------------------------------------------------------------------
template <int CIN, typename Tout>
__global__ void __launch_bounds__(kDirectThreads)
conv_direct_fwd_kernel(const float* __restrict__ x, int si, int M, const float* __restrict__ w,
                       const float* __restrict__ bias, Tout* __restrict__ y) {
  const int co = threadIdx.x, m = blockIdx.x * 4 + threadIdx.y;
  if (m >= M) return;
  const int base = in_pixel(m, si, si - 2);
  float acc = bias[co];
  for (int ci = 0; ci < CIN; ++ci)
#pragma unroll
    for (int t = 0; t < 9; ++t)
      acc = fmaf(x[static_cast<size_t>(base + (t / 3) * si + t % 3) * CIN + ci], w[(co * CIN + ci) * 9 + t], acc);
  y[static_cast<size_t>(m) * kCh + co] = from_f32<Tout>(fmaxf(acc, 0.f));
}

// dx[i, j, ci] = sum_{co, tap} gpad[i + dr, j + dc, co] w[co, ci, 2 - dr, 2 - dc], times [x > 0]; S = side of x
__global__ void __launch_bounds__(kDirectThreads)
conv_direct_dgrad_kernel(const float* __restrict__ g, int S, int M, const float* __restrict__ w,
                         const float* __restrict__ mask, float* __restrict__ out) {
  const int ci = threadIdx.x, m = blockIdx.x * 4 + threadIdx.y;
  if (m >= M) return;
  const int base = in_pixel(m, S + 2, S);
  float acc = 0.f;
  for (int co = 0; co < kCh; ++co)
#pragma unroll
    for (int t = 0; t < 9; ++t)
      acc = fmaf(g[static_cast<size_t>(base + (t / 3) * (S + 2) + t % 3) * kCh + co], w[(co * kCh + ci) * 9 + 8 - t], acc);
  float* o = out + static_cast<size_t>(padded_pixel(m, S, 2)) * kCh + ci;
  *o = mask[static_cast<size_t>(m) * kCh + ci] > 0.f ? acc : 0.f;
  const int r = (m % (S * S)) / S, c = m % S;
  for_owned_border(S, r, c, [&](int off) { o[static_cast<ptrdiff_t>(off) * kCh] = 0.f; });
}

// per (pixel chunk, output j): j = co (9 C_in + 1) + k, k = ci 9 + tap, or k = 9 C_in for the bias
template <int CIN, typename Tg>
__global__ void __launch_bounds__(kDirectThreads)
conv_direct_wgrad_kernel(const Tg* __restrict__ g, const float* __restrict__ x, int si, int M, int chunk_px,
                         float* __restrict__ ws) {
  constexpr int J1 = CIN * 9 + 1;
  const int j = blockIdx.y * kDirectThreads + threadIdx.x;
  if (j >= kCh * J1) return;
  const int so = si - 2, ps = so + 4;
  const int co = j / J1, k = j - co * J1;
  const bool is_bias = k == CIN * 9;
  const int ci = is_bias ? 0 : k / 9, tap = is_bias ? 0 : k % 9;
  const int toff = (tap / 3) * si + tap % 3;
  const int c0 = blockIdx.x * chunk_px, c1 = min(c0 + chunk_px, M);
  const int po = so * so;
  int n = c0 / po, r = (c0 - n * po) / so, c = c0 - n * po - r * so;
  int gp = (n * ps + r + 2) * ps + c + 2, xp = (n * si + r) * si + c;
  float acc = 0.f;
  for (int m = c0; m < c1; ++m) {
    const float gv = to_f32<Tg>(g[static_cast<size_t>(gp) * kCh + co]);
    acc = is_bias ? acc + gv : fmaf(gv, x[static_cast<size_t>(xp + toff) * CIN + ci], acc);
    ++gp; ++xp;
    if (++c == so) {
      c = 0; gp += 4; xp += 2;
      if (++r == so) { r = 0; gp += 4 * ps; xp += 2 * si; }
    }
  }
  ws[static_cast<size_t>(blockIdx.x) * kCh * J1 + j] = acc;
}

__global__ void conv_wgrad_reduce_kernel(const float* __restrict__ ws, int n_chunks, int J1, float* __restrict__ dw,
                                         float* __restrict__ db) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= kCh * J1) return;
  float s = 0.f;
  for (int c = 0; c < n_chunks; ++c) s += ws[static_cast<size_t>(c) * kCh * J1 + j];
  const int co = j / J1, k = j - co * J1;
  if (k == J1 - 1) db[co] = s;
  else dw[co * (J1 - 1) + k] = s;
}

template <typename T>
__global__ void __launch_bounds__(256) conv_mean_fwd_kernel(const T* __restrict__ y, int P, T* __restrict__ feat) {
  __shared__ float part[4][kCh];
  const int co = threadIdx.x & 63, grp = threadIdx.x >> 6, n = blockIdx.x;
  const T* yi = y + static_cast<size_t>(n) * P * kCh;
  float s = 0.f;
  for (int p = grp; p < P; p += 4) s += to_f32<T>(yi[static_cast<size_t>(p) * kCh + co]);
  part[grp][co] = s;
  __syncthreads();
  if (grp == 0) feat[n * kCh + co] = from_f32<T>((((part[0][co] + part[1][co]) + part[2][co]) + part[3][co]) / P);
}

template <typename T>
__global__ void conv_mean_bwd_kernel(const T* __restrict__ dfeat, const T* __restrict__ y, int N, int s, T* __restrict__ g) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int P = s * s;
  if (i >= static_cast<size_t>(N) * P * kCh) return;
  const int m = static_cast<int>(i / kCh), co = static_cast<int>(i % kCh), n = m / P;
  const float v = to_f32<T>(dfeat[n * kCh + co]) / static_cast<float>(P);
  T* o = g + static_cast<size_t>(padded_pixel(m, s, 2)) * kCh + co;
  *o = from_f32<T>(to_f32<T>(y[i]) > 0.f ? v : 0.f);
  const int r = (m % P) / s, c = m % s;
  for_owned_border(s, r, c, [&](int off) { o[static_cast<ptrdiff_t>(off) * kCh] = from_f32<T>(0.f); });
}

int wgrad_chunks(int M, int C_in, int* chunk_px) {
  const int nb = (M + kBlockPx - 1) / kBlockPx;
  const int most = C_in == 1 ? kWgradChunksIn : kWgradChunks;
  const int per = (nb + most - 1) / most;
  *chunk_px = per * kBlockPx;
  return (M + *chunk_px - 1) / *chunk_px;
}

int check_desc(const pfn_conv_desc* d, const char* what) {
  PFN_CHECK_ARG(d != nullptr, "%s: null descriptor", what);
  PFN_CHECK_ARG(d->N > 0, "%s: N=%d images", what, d->N);
  PFN_CHECK_ARG(d->S >= 4 && d->S <= PFN_CONV_MAX_SIDE, "%s: side S=%d outside [4, %d]", what, d->S, PFN_CONV_MAX_SIDE);
  PFN_CHECK_ARG(d->C_in == 1 || d->C_in == kCh, "%s: C_in=%d (1 or %d)", what, d->C_in, kCh);
  PFN_CHECK_ARG(d->dtype == PFN_F32 || d->dtype == PFN_BF16, "%s: dtype %d", what, d->dtype);
  PFN_CHECK_ARG(static_cast<long long>(d->N) * (d->S + 4) * (d->S + 4) * kCh < (1ll << 31),
                "%s: N=%d images of side %d exceed the 32-bit pixel index", what, d->N, d->S);
  return 0;
}

bool g_tc_attr_done[2][64];

template <bool DGRAD>
int launch_tc(const __nv_bfloat16* in, int si, int M, const void* wB, const float* bias, const void* mask, void* out,
              cudaStream_t st) {
  const size_t smem = tc_smem(si);
  if (first_use_on_device(g_tc_attr_done[DGRAD]))
    PFN_CUDA_OK(cudaFuncSetAttribute(conv64_tc_kernel<DGRAD>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     static_cast<int>(tc_smem(PFN_CONV_MAX_SIDE + 2))));
  const int n_tiles = (M + kTile - 1) / kTile;
  conv64_tc_kernel<DGRAD><<<min(n_tiles, num_sms()), kTcThreads, smem, st>>>(
      in, si, M, static_cast<const __nv_bfloat16*>(wB), bias, static_cast<const __nv_bfloat16*>(mask),
      static_cast<__nv_bfloat16*>(out), tc_span(si));
  PFN_LAUNCH_OK();
  return 0;
}

}  // namespace
}  // namespace pfn

extern "C" int pfn_conv_fwd(const pfn_conv_desc* d, void* stream) {
  using namespace pfn;
  if (int rc = check_desc(d, "conv_fwd")) return rc;
  PFN_CHECK_ARG(d->x && d->w && d->bias && d->y, "conv_fwd: null pointer in the descriptor");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int so = d->S - 2, M = d->N * so * so;
  if (d->C_in == kCh && d->dtype == PFN_BF16)
    return launch_tc<false>(static_cast<const __nv_bfloat16*>(d->x), d->S, M, d->w, d->bias, nullptr, d->y, st);
  const dim3 block(kCh, 4), grid((M + 3) / 4);
  const float* x = static_cast<const float*>(d->x);
  const float* w = static_cast<const float*>(d->w);
  if (d->C_in == 1 && d->dtype == PFN_BF16)
    conv_direct_fwd_kernel<1, __nv_bfloat16><<<grid, block, 0, st>>>(x, d->S, M, w, d->bias, static_cast<__nv_bfloat16*>(d->y));
  else if (d->C_in == 1)
    conv_direct_fwd_kernel<1, float><<<grid, block, 0, st>>>(x, d->S, M, w, d->bias, static_cast<float*>(d->y));
  else
    conv_direct_fwd_kernel<kCh, float><<<grid, block, 0, st>>>(x, d->S, M, w, d->bias, static_cast<float*>(d->y));
  PFN_LAUNCH_OK();
  return 0;
}

extern "C" int pfn_conv_dgrad(const pfn_conv_desc* d, void* stream) {
  using namespace pfn;
  if (int rc = check_desc(d, "conv_dgrad")) return rc;
  PFN_CHECK_ARG(d->C_in == kCh, "conv_dgrad: C_in=%d (the input conv has no data gradient)", d->C_in);
  PFN_CHECK_ARG(d->x && d->w && d->g && d->y, "conv_dgrad: null pointer in the descriptor");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int M = d->N * d->S * d->S;
  if (d->dtype == PFN_BF16)
    return launch_tc<true>(static_cast<const __nv_bfloat16*>(d->g), d->S + 2, M, d->w, nullptr, d->x, d->y, st);
  conv_direct_dgrad_kernel<<<(M + 3) / 4, dim3(kCh, 4), 0, st>>>(static_cast<const float*>(d->g), d->S, M,
                                                                   static_cast<const float*>(d->w),
                                                                   static_cast<const float*>(d->x), static_cast<float*>(d->y));
  PFN_LAUNCH_OK();
  return 0;
}

extern "C" int pfn_conv_wgrad_workspace(const pfn_conv_desc* d) {
  using namespace pfn;
  if (check_desc(d, "conv_wgrad_workspace")) return -1;
  int chunk_px;
  const int so = d->S - 2;
  return wgrad_chunks(d->N * so * so, d->C_in, &chunk_px) * kCh * (9 * d->C_in + 1);
}

extern "C" int pfn_conv_wgrad(const pfn_conv_desc* d, void* stream) {
  using namespace pfn;
  if (int rc = check_desc(d, "conv_wgrad")) return rc;
  PFN_CHECK_ARG(d->x && d->g && d->dw && d->db && d->workspace, "conv_wgrad: null pointer in the descriptor");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int so = d->S - 2, M = d->N * so * so;
  int chunk_px;
  const int n_chunks = wgrad_chunks(M, d->C_in, &chunk_px);
  const int J1 = 9 * d->C_in + 1;
  const dim3 dgrid(n_chunks, (kCh * J1 + kDirectThreads - 1) / kDirectThreads);
  const float* x = static_cast<const float*>(d->x);
  if (d->C_in == kCh && d->dtype == PFN_BF16)
    conv64_wgrad_tc_kernel<<<dim3(n_chunks, 9), 128, 0, st>>>(static_cast<const __nv_bfloat16*>(d->g),
                                                              static_cast<const __nv_bfloat16*>(d->x), d->S, M, chunk_px,
                                                              d->workspace);
  else if (d->C_in == 1 && d->dtype == PFN_BF16)
    conv_direct_wgrad_kernel<1, __nv_bfloat16><<<dgrid, kDirectThreads, 0, st>>>(
        static_cast<const __nv_bfloat16*>(d->g), x, d->S, M, chunk_px, d->workspace);
  else if (d->C_in == 1)
    conv_direct_wgrad_kernel<1, float><<<dgrid, kDirectThreads, 0, st>>>(static_cast<const float*>(d->g), x, d->S, M,
                                                                         chunk_px, d->workspace);
  else
    conv_direct_wgrad_kernel<kCh, float><<<dgrid, kDirectThreads, 0, st>>>(static_cast<const float*>(d->g), x, d->S, M,
                                                                           chunk_px, d->workspace);
  PFN_LAUNCH_OK();
  conv_wgrad_reduce_kernel<<<(kCh * J1 + 255) / 256, 256, 0, st>>>(d->workspace, n_chunks, J1, d->dw, d->db);
  PFN_LAUNCH_OK();
  return 0;
}

extern "C" int pfn_conv_mean_fwd(const void* y, int N, int s, int dtype, void* feat, void* stream) {
  using namespace pfn;
  PFN_CHECK_ARG(y && feat, "conv_mean_fwd: null pointer");
  PFN_CHECK_ARG(N > 0 && s > 0 && s <= PFN_CONV_MAX_SIDE, "conv_mean_fwd: N=%d, side %d", N, s);
  PFN_CHECK_ARG(dtype == PFN_F32 || dtype == PFN_BF16, "conv_mean_fwd: dtype %d", dtype);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == PFN_BF16)
    conv_mean_fwd_kernel<<<N, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(y), s * s, static_cast<__nv_bfloat16*>(feat));
  else
    conv_mean_fwd_kernel<<<N, 256, 0, st>>>(static_cast<const float*>(y), s * s, static_cast<float*>(feat));
  PFN_LAUNCH_OK();
  return 0;
}

extern "C" int pfn_conv_mean_bwd(const void* dfeat, const void* y, int N, int s, int dtype, void* g, void* stream) {
  using namespace pfn;
  PFN_CHECK_ARG(dfeat && y && g, "conv_mean_bwd: null pointer");
  PFN_CHECK_ARG(N > 0 && s > 0 && s <= PFN_CONV_MAX_SIDE, "conv_mean_bwd: N=%d, side %d", N, s);
  PFN_CHECK_ARG(static_cast<long long>(N) * (s + 4) * (s + 4) * kCh < (1ll << 31), "conv_mean_bwd: N=%d too large", N);
  PFN_CHECK_ARG(dtype == PFN_F32 || dtype == PFN_BF16, "conv_mean_bwd: dtype %d", dtype);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t total = static_cast<size_t>(N) * s * s * kCh;
  const unsigned blocks = static_cast<unsigned>((total + 255) / 256);
  if (dtype == PFN_BF16)
    conv_mean_bwd_kernel<<<blocks, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(dfeat), static_cast<const __nv_bfloat16*>(y),
                                                 N, s, static_cast<__nv_bfloat16*>(g));
  else
    conv_mean_bwd_kernel<<<blocks, 256, 0, st>>>(static_cast<const float*>(dfeat), static_cast<const float*>(y), N, s,
                                                 static_cast<float*>(g));
  PFN_LAUNCH_OK();
  return 0;
}
