// Bar-distribution ("Riemann") negative log density, forward and backward, one warp per query row.
// Restates reference bar_distribution.py:19-33 (BarDistribution) and :83-108 (FullSupportBarDistribution):
// bucket lookup (bit-exact integer result), log-softmax over the bars, gather, width scaling and the
// half-normal tails — fused into a single pass over the logits (read once fwd, read once + write once bwd).
#include "common.cuh"
#include "../../include/pfn_b200.h"

namespace pfn {

// torch.searchsorted(borders, y) (right=False): first i with borders[i] >= y; then the reference's fix-ups
//   idx = i - 1 ; y == borders[0] -> 0 ; y == borders[-1] -> n_bars - 1          (bar_distribution.py:19-23)
__device__ __forceinline__ long long bucket_index(const float* __restrict__ borders, int n_bars, float y) {
  int lo = 0, hi = n_bars + 1;  // search in [0, n_bars+1)
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (borders[mid] < y) lo = mid + 1;
    else hi = mid;
  }
  long long idx = static_cast<long long>(lo) - 1;
  if (y == borders[0]) idx = 0;
  if (y == borders[n_bars]) idx = n_bars - 1;
  return idx;
}

__global__ void bucket_idx_kernel(const float* __restrict__ y, const float* __restrict__ borders, int n_bars,
                                  long long* __restrict__ idx, int rows) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < rows) idx[r] = bucket_index(borders, n_bars, y[r]);
}

template <typename T>
__global__ void __launch_bounds__(256)
bar_nll_fwd_kernel(const T* __restrict__ logits, int ld, const float* __restrict__ y,
                   const float* __restrict__ borders, int n_bars, int full_support, float* __restrict__ nll,
                   long long* __restrict__ idx_out, float* __restrict__ lse_out, int* __restrict__ oob_count, int rows) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int row = warp; row < rows; row += nwarps) {
    const T* z = logits + static_cast<size_t>(row) * ld;
    // online log-sum-exp, lanes strided over the bars (coalesced).  A -inf logit adds nothing (as in log_softmax); it is
    // skipped so that a lane whose running max is still -inf does not form expf(-inf - -inf) = NaN.  A row of -inf only
    // gives lse = -inf and a NaN nll, as torch does; a NaN logit still propagates.
    float m = -INFINITY, s = 0.f;
    for (int c = lane; c < n_bars; c += 32) {
      const float v = to_f32<T>(z[c]);
      if (v > m) { s = s * expf(m - v) + 1.0f; m = v; }
      else if (v != -INFINITY) s += expf(v - m);
    }
    const float mall = warp_max(m);
    s = (m == -INFINITY) ? 0.f : s * expf(m - mall);
    const float lse = mall + logf(warp_sum(s));

    const float yv = y[row];
    long long idx = bucket_index(borders, n_bars, yv);
    bool oob = (idx < 0) || (idx >= n_bars);
    if (full_support) {
      idx = idx < 0 ? 0 : (idx >= n_bars ? n_bars - 1 : idx);
      oob = false;
    }
    float out;
    if (oob) {
      out = __int_as_float(0x7fc00000);  // NaN; the host raises like the reference assert (bar_distribution.py:27)
      if (lane == 0) atomicAdd(oob_count, 1);
    } else {
      const int k = static_cast<int>(idx);
      const float w = borders[k + 1] - borders[k];
      const float zk = to_f32<T>(z[k]);
      // log_prob = (z_k - lse) - log(w)
      float log_prob = (zk - lse) - logf(w);
      if (full_support) {
        // HalfNormal(s).log_prob(v) = log(2) - log(s) - 0.5 log(2 pi) - v^2 / (2 s^2),  s = w / icdf_{HN(1)}(0.5)
        constexpr float kIcdfHalf = 0.6744897501960817f;
        constexpr float kLog2 = 0.6931471805599453f;
        constexpr float kHalfLog2Pi = 0.9189385332046727f;
        if (k == 0) {
          const float sc = w / kIcdfHalf;
          const float v = fmaxf(borders[1] - yv, 1e-8f);
          log_prob += (kLog2 - logf(sc) - kHalfLog2Pi - (v * v) / (2.0f * sc * sc)) + logf(w);
        }
        if (k == n_bars - 1) {
          const float sc = w / kIcdfHalf;
          const float v = yv - borders[n_bars - 1];
          log_prob += (kLog2 - logf(sc) - kHalfLog2Pi - (v * v) / (2.0f * sc * sc)) + logf(w);
        }
      }
      out = -log_prob;
    }
    if (lane == 0) {
      nll[row] = out;
      idx_out[row] = idx;
      lse_out[row] = lse;
    }
  }
}

template <typename T, typename TD>
__global__ void __launch_bounds__(256)
bar_nll_bwd_kernel(const T* __restrict__ logits, int ld, const long long* __restrict__ idx,
                   const float* __restrict__ lse, const float* __restrict__ g, TD* __restrict__ dlogits, int ld_d,
                   int n_bars, int n_cols_pad, int rows) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int row = warp; row < rows; row += nwarps) {
    const T* z = logits + static_cast<size_t>(row) * ld;
    TD* dz = dlogits + static_cast<size_t>(row) * ld_d;
    const float l = lse[row];
    const float gr = g[row];
    const int k = static_cast<int>(idx[row]);
    for (int c = lane; c < n_cols_pad; c += 32) {
      float v = 0.f;
      if (c < n_bars) {
        v = expf(to_f32<T>(z[c]) - l);
        if (c == k) v -= 1.0f;
        v *= gr;
      }
      dz[c] = from_f32<TD>(v);
    }
  }
}

}  // namespace pfn

using namespace pfn;

extern "C" int pfn_bar_bucket_idx(const float* y, const float* borders, int n_bars, int64_t* idx, int rows,
                                  void* stream) {
  PFN_CHECK_ARG(n_bars >= 1, "bar_bucket_idx: n_bars=%d", n_bars);
  if (rows <= 0) return 0;
  bucket_idx_kernel<<<(rows + 255) / 256, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      y, borders, n_bars, reinterpret_cast<long long*>(idx), rows);
  PFN_LAUNCH_OK();
  return 0;
}

extern "C" int pfn_bar_nll_fwd(const void* logits, int ld, int dtype, const float* y, const float* borders, int n_bars,
                               int full_support, float* nll, int64_t* idx, float* lse, int* oob_count, int rows,
                               void* stream) {
  PFN_CHECK_ARG(n_bars >= 1 && ld >= n_bars, "bar_nll_fwd: n_bars=%d ld=%d", n_bars, ld);
  PFN_CHECK_ARG(!full_support || n_bars > 1, "bar_nll_fwd: FullSupport needs more than one bar (bar_distribution.py:90)");
  if (rows <= 0) return 0;
  int grid = (rows + 7) / 8;
  const int max_grid = num_sms() * 8;
  if (grid > max_grid) grid = max_grid;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == PFN_F32)
    bar_nll_fwd_kernel<float><<<grid, 256, 0, s>>>(reinterpret_cast<const float*>(logits), ld, y, borders, n_bars,
                                                   full_support, nll, reinterpret_cast<long long*>(idx), lse, oob_count, rows);
  else
    bar_nll_fwd_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(logits), ld, y, borders,
                                                           n_bars, full_support, nll, reinterpret_cast<long long*>(idx),
                                                           lse, oob_count, rows);
  PFN_LAUNCH_OK();
  return 0;
}

extern "C" int pfn_bar_nll_bwd(const void* logits, int ld, int dtype, const int64_t* idx, const float* lse,
                               const float* g, void* dlogits, int ld_d, int d_dtype, int n_bars, int n_cols_pad,
                               int rows, void* stream) {
  PFN_CHECK_ARG(n_bars >= 1 && ld >= n_bars && n_cols_pad >= n_bars && ld_d >= n_cols_pad,
                "bar_nll_bwd: n_bars=%d ld=%d pad=%d ld_d=%d", n_bars, ld, n_cols_pad, ld_d);
  if (rows <= 0) return 0;
  int grid = (rows + 7) / 8;
  const int max_grid = num_sms() * 8;
  if (grid > max_grid) grid = max_grid;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const long long* ix = reinterpret_cast<const long long*>(idx);
  if (dtype == PFN_F32 && d_dtype == PFN_F32)
    bar_nll_bwd_kernel<float, float><<<grid, 256, 0, s>>>(reinterpret_cast<const float*>(logits), ld, ix, lse, g,
                                                          reinterpret_cast<float*>(dlogits), ld_d, n_bars, n_cols_pad, rows);
  else if (dtype == PFN_F32 && d_dtype == PFN_BF16)
    bar_nll_bwd_kernel<float, __nv_bfloat16><<<grid, 256, 0, s>>>(reinterpret_cast<const float*>(logits), ld, ix, lse, g,
                                                                  reinterpret_cast<__nv_bfloat16*>(dlogits), ld_d, n_bars, n_cols_pad, rows);
  else if (dtype == PFN_BF16 && d_dtype == PFN_F32)
    bar_nll_bwd_kernel<__nv_bfloat16, float><<<grid, 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(logits), ld, ix, lse, g,
                                                                  reinterpret_cast<float*>(dlogits), ld_d, n_bars, n_cols_pad, rows);
  else
    bar_nll_bwd_kernel<__nv_bfloat16, __nv_bfloat16><<<grid, 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(logits), ld, ix, lse, g,
                                                                          reinterpret_cast<__nv_bfloat16*>(dlogits), ld_d, n_bars, n_cols_pad, rows);
  PFN_LAUNCH_OK();
  return 0;
}
