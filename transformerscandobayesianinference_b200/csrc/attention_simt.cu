// fp32-FMA masked attention (forward, dQ, dK/dV) for the fp32 parity mode and for head sizes / dtypes the
// tensor-core kernels do not take.  One warp per (batch, head, row); the head dimension is spread over the
// lanes, scores are reduced with warp shuffles, softmax is computed online.  The single_eval_pos mask of
// reference transformer.py:35-41 is implicit:  keys(i) = [0, sep)  U  {i if i >= sep}.
#include "common.cuh"
#include "dropout.cuh"
#include "../../include/pfn_b200.h"

namespace pfn {

template <typename T, int DPL>
__device__ __forceinline__ void load_head(const T* base, int dh, int lane, float (&v)[DPL]) {
#pragma unroll
  for (int c = 0; c < DPL; ++c) {
    const int d = lane + 32 * c;
    v[c] = d < dh ? to_f32<T>(base[d]) : 0.f;
  }
}
template <typename T, int DPL>
__device__ __forceinline__ void store_head(T* base, int dh, int lane, const float (&v)[DPL]) {
#pragma unroll
  for (int c = 0; c < DPL; ++c) {
    const int d = lane + 32 * c;
    if (d < dh) base[d] = from_f32<T>(v[c]);
  }
}

template <typename T, int DPL>
__global__ void __launch_bounds__(256)
attn_fwd_simt_kernel(const pfn_attn_desc d) {
  const int E = d.H * d.dh;
  const long long total = static_cast<long long>(d.B) * d.H * d.T;
  const int lane = threadIdx.x & 31;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const T* qkv = reinterpret_cast<const T*>(d.qkv);
  T* out = reinterpret_cast<T*>(d.out);
  for (long long task = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; task < total; task += nwarps) {
    // task order: i fastest within (b,h) so neighbouring warps share K/V rows in cache
    const int i = static_cast<int>(task % d.T);
    const int bh = static_cast<int>(task / d.T);
    const int h = bh % d.H, b = bh / d.H;
    float q[DPL], o[DPL];
    load_head<T, DPL>(qkv + (static_cast<size_t>(i) * d.B + b) * d.ld_qkv + h * d.dh, d.dh, lane, q);
#pragma unroll
    for (int c = 0; c < DPL; ++c) { q[c] *= d.scale; o[c] = 0.f; }
    float m = -INFINITY, l = 0.f;
    const int nkeys = d.sep + (i >= d.sep ? 1 : 0);
    for (int jj = 0; jj < nkeys; ++jj) {
      const int j = jj < d.sep ? jj : i;
      const T* krow = qkv + (static_cast<size_t>(j) * d.B + b) * d.ld_qkv + E + h * d.dh;
      float k[DPL], v[DPL];
      load_head<T, DPL>(krow, d.dh, lane, k);
      load_head<T, DPL>(krow + E, d.dh, lane, v);
      float s = 0.f;
#pragma unroll
      for (int c = 0; c < DPL; ++c) s = fmaf(q[c], k[c], s);
      s = warp_sum(s);
      const float m_new = fmaxf(m, s);
      const float corr = expf(m - m_new);
      const float p = expf(s - m_new);
      l = l * corr + p;                 // the softmax normaliser is over ALL visible keys; dropout acts on the probabilities
      const float pd = (d.drop_thr > 0 && !drop_keep(d.drop_seed, static_cast<uint32_t>(bh) * d.T + i, j, d.drop_thr)) ? 0.f : p;
#pragma unroll
      for (int c = 0; c < DPL; ++c) o[c] = fmaf(pd, v[c], o[c] * corr);
      m = m_new;
    }
    const float inv_l = (d.drop_thr > 0 ? drop_scale(d.drop_thr) : 1.0f) / l;
#pragma unroll
    for (int c = 0; c < DPL; ++c) o[c] *= inv_l;
    store_head<T, DPL>(out + (static_cast<size_t>(i) * d.B + b) * d.ld_out + h * d.dh, d.dh, lane, o);
    if (lane == 0) d.lse[static_cast<size_t>(bh) * d.T + i] = m + logf(l);
  }
}

// dQ (+ delta, + the diagonal-key contributions that are the ONLY gradient of k_i, v_i for query rows)
template <typename T, int DPL>
__global__ void __launch_bounds__(256)
attn_bwd_dq_simt_kernel(const pfn_attn_desc d, float* __restrict__ delta) {
  const int E = d.H * d.dh;
  const long long total = static_cast<long long>(d.B) * d.H * d.T;
  const int lane = threadIdx.x & 31;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const T* qkv = reinterpret_cast<const T*>(d.qkv);
  const T* outp = reinterpret_cast<const T*>(d.out);
  const T* dout = reinterpret_cast<const T*>(d.dout);
  T* dqkv = reinterpret_cast<T*>(d.dqkv);
  for (long long task = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; task < total; task += nwarps) {
    const int i = static_cast<int>(task % d.T);
    const int bh = static_cast<int>(task / d.T);
    const int h = bh % d.H, b = bh / d.H;
    const size_t tok = static_cast<size_t>(i) * d.B + b;
    float q[DPL], dO[DPL], O[DPL], dq[DPL];
    load_head<T, DPL>(qkv + tok * d.ld_qkv + h * d.dh, d.dh, lane, q);
    load_head<T, DPL>(dout + tok * d.ld_dout + h * d.dh, d.dh, lane, dO);
    load_head<T, DPL>(outp + tok * d.ld_out + h * d.dh, d.dh, lane, O);
    float dl = 0.f;
#pragma unroll
    for (int c = 0; c < DPL; ++c) { dl = fmaf(dO[c], O[c], dl); dq[c] = 0.f; }
    dl = warp_sum(dl);
    if (lane == 0) delta[static_cast<size_t>(bh) * d.T + i] = dl;
    const float lse = d.lse[static_cast<size_t>(bh) * d.T + i];
    const int nkeys = d.sep + (i >= d.sep ? 1 : 0);
    for (int jj = 0; jj < nkeys; ++jj) {
      const int j = jj < d.sep ? jj : i;
      const T* krow = qkv + (static_cast<size_t>(j) * d.B + b) * d.ld_qkv + E + h * d.dh;
      float k[DPL], v[DPL];
      load_head<T, DPL>(krow, d.dh, lane, k);
      load_head<T, DPL>(krow + E, d.dh, lane, v);
      float s = 0.f, dp = 0.f;
#pragma unroll
      for (int c = 0; c < DPL; ++c) { s = fmaf(q[c], k[c], s); dp = fmaf(dO[c], v[c], dp); }
      s = warp_sum(s) * d.scale;
      dp = warp_sum(dp);
      const float p = expf(s - lse);
      // dropout on the probabilities: Pd = P m / (1 - p_drop);  dP = m dPd / (1 - p_drop);  dS = P (dP - delta)
      const float mk = d.drop_thr > 0 ? (drop_keep(d.drop_seed, static_cast<uint32_t>(bh) * d.T + i, j, d.drop_thr) ? drop_scale(d.drop_thr) : 0.f) : 1.f;
      const float ds = p * (mk * dp - dl) * d.scale;
#pragma unroll
      for (int c = 0; c < DPL; ++c) dq[c] = fmaf(ds, k[c], dq[c]);
      if (jj >= d.sep) {
        float dk[DPL], dv[DPL];
#pragma unroll
        for (int c = 0; c < DPL; ++c) { dk[c] = ds * q[c]; dv[c] = p * mk * dO[c]; }
        store_head<T, DPL>(dqkv + tok * d.ld_dqkv + E + h * d.dh, d.dh, lane, dk);
        store_head<T, DPL>(dqkv + tok * d.ld_dqkv + 2 * E + h * d.dh, d.dh, lane, dv);
      }
    }
    store_head<T, DPL>(dqkv + tok * d.ld_dqkv + h * d.dh, d.dh, lane, dq);
  }
}

// dK, dV of the train keys j < sep: every row i attends to them.
template <typename T, int DPL>
__global__ void __launch_bounds__(256)
attn_bwd_dkv_simt_kernel(const pfn_attn_desc d, const float* __restrict__ delta) {
  const int E = d.H * d.dh;
  const long long total = static_cast<long long>(d.B) * d.H * d.sep;
  const int lane = threadIdx.x & 31;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const T* qkv = reinterpret_cast<const T*>(d.qkv);
  const T* dout = reinterpret_cast<const T*>(d.dout);
  T* dqkv = reinterpret_cast<T*>(d.dqkv);
  for (long long task = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; task < total; task += nwarps) {
    const int j = static_cast<int>(task % d.sep);
    const int bh = static_cast<int>(task / d.sep);
    const int h = bh % d.H, b = bh / d.H;
    const size_t tokj = static_cast<size_t>(j) * d.B + b;
    float k[DPL], v[DPL], dk[DPL], dv[DPL];
    load_head<T, DPL>(qkv + tokj * d.ld_qkv + E + h * d.dh, d.dh, lane, k);
    load_head<T, DPL>(qkv + tokj * d.ld_qkv + 2 * E + h * d.dh, d.dh, lane, v);
#pragma unroll
    for (int c = 0; c < DPL; ++c) { dk[c] = 0.f; dv[c] = 0.f; }
    for (int i = 0; i < d.T; ++i) {
      const size_t tok = static_cast<size_t>(i) * d.B + b;
      float q[DPL], dO[DPL];
      load_head<T, DPL>(qkv + tok * d.ld_qkv + h * d.dh, d.dh, lane, q);
      load_head<T, DPL>(dout + tok * d.ld_dout + h * d.dh, d.dh, lane, dO);
      float s = 0.f, dp = 0.f;
#pragma unroll
      for (int c = 0; c < DPL; ++c) { s = fmaf(q[c], k[c], s); dp = fmaf(dO[c], v[c], dp); }
      s = warp_sum(s) * d.scale;
      dp = warp_sum(dp);
      const float p = expf(s - d.lse[static_cast<size_t>(bh) * d.T + i]);
      const float mk = d.drop_thr > 0 ? (drop_keep(d.drop_seed, static_cast<uint32_t>(bh) * d.T + i, j, d.drop_thr) ? drop_scale(d.drop_thr) : 0.f) : 1.f;
      const float ds = p * (mk * dp - delta[static_cast<size_t>(bh) * d.T + i]) * d.scale;
#pragma unroll
      for (int c = 0; c < DPL; ++c) { dv[c] = fmaf(p * mk, dO[c], dv[c]); dk[c] = fmaf(ds, q[c], dk[c]); }
    }
    store_head<T, DPL>(dqkv + tokj * d.ld_dqkv + E + h * d.dh, d.dh, lane, dk);
    store_head<T, DPL>(dqkv + tokj * d.ld_dqkv + 2 * E + h * d.dh, d.dh, lane, dv);
  }
}

static int check_attn_desc(const pfn_attn_desc* d, bool bwd, const char* who) {
  PFN_CHECK_ARG(d != nullptr, "%s: null descriptor", who);
  PFN_CHECK_ARG(d->T > 0 && d->B > 0 && d->H > 0 && d->dh > 0, "%s: bad shape T=%d B=%d H=%d dh=%d", who, d->T, d->B,
                d->H, d->dh);
  PFN_CHECK_ARG(d->sep >= 0 && d->sep <= d->T, "%s: sep %d outside [0,%d]", who, d->sep, d->T);
  PFN_CHECK_ARG(d->dtype == PFN_F32 || d->dtype == PFN_BF16, "%s: bad dtype %d", who, d->dtype);
  PFN_CHECK_ARG(d->qkv && d->out && d->lse, "%s: null qkv/out/lse", who);
  PFN_CHECK_ARG(d->batch_major == 0 || d->batch_major == 1, "%s: bad batch_major %d", who, d->batch_major);
  PFN_CHECK_ARG(d->drop_thr >= 0 && d->drop_thr <= 255, "%s: dropout threshold %d outside [0,255]", who, d->drop_thr);
  PFN_CHECK_ARG(d->ld_qkv >= 3 * d->H * d->dh && d->ld_out >= d->H * d->dh, "%s: leading dims too small", who);
  if (bwd) {
    PFN_CHECK_ARG(d->dout && d->dqkv && d->delta, "%s: null dout/dqkv/delta", who);
    PFN_CHECK_ARG(d->ld_dqkv >= 3 * d->H * d->dh && d->ld_dout >= d->H * d->dh, "%s: leading dims too small", who);
  }
  return 0;
}

template <typename T, int DPL>
static int launch_attn_simt(const pfn_attn_desc* d, bool bwd, cudaStream_t s) {
  const long long tasks = static_cast<long long>(d->B) * d->H * d->T;
  long long grid = (tasks + 7) / 8;
  const long long max_grid = static_cast<long long>(num_sms()) * 16;
  if (grid > max_grid) grid = max_grid;
  if (!bwd) {
    attn_fwd_simt_kernel<T, DPL><<<static_cast<int>(grid), 256, 0, s>>>(*d);
    PFN_LAUNCH_OK();
    return 0;
  }
  attn_bwd_dq_simt_kernel<T, DPL><<<static_cast<int>(grid), 256, 0, s>>>(*d, d->delta);
  PFN_LAUNCH_OK();
  if (d->sep > 0) {
    const long long tasks2 = static_cast<long long>(d->B) * d->H * d->sep;
    long long grid2 = (tasks2 + 7) / 8;
    if (grid2 > max_grid) grid2 = max_grid;
    attn_bwd_dkv_simt_kernel<T, DPL><<<static_cast<int>(grid2), 256, 0, s>>>(*d, d->delta);
    PFN_LAUNCH_OK();
  }
  return 0;
}

template <typename T>
static int dispatch_attn_simt(const pfn_attn_desc* d, bool bwd, cudaStream_t s) {
  if (d->dh <= 32) return launch_attn_simt<T, 1>(d, bwd, s);
  if (d->dh <= 64) return launch_attn_simt<T, 2>(d, bwd, s);
  if (d->dh <= 128) return launch_attn_simt<T, 4>(d, bwd, s);
  PFN_CHECK_ARG(d->dh <= 256, "attention_simt: head dim %d > 256 unsupported", d->dh);
  return launch_attn_simt<T, 8>(d, bwd, s);
}

int check_attn_desc_public(const pfn_attn_desc* d, bool bwd, const char* who) { return check_attn_desc(d, bwd, who); }

}  // namespace pfn

using namespace pfn;

extern "C" int pfn_attention_fwd_simt(const pfn_attn_desc* d, void* stream) {
  if (int rc = check_attn_desc(d, false, "attention_fwd_simt")) return rc;
  PFN_CHECK_ARG(d->batch_major == 0, "attention_fwd_simt: batch-major token order is only implemented by the tensor-core kernels");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  return d->dtype == PFN_F32 ? dispatch_attn_simt<float>(d, false, s) : dispatch_attn_simt<__nv_bfloat16>(d, false, s);
}

extern "C" int pfn_attention_bwd_simt(const pfn_attn_desc* d, void* stream) {
  if (int rc = check_attn_desc(d, true, "attention_bwd_simt")) return rc;
  PFN_CHECK_ARG(d->batch_major == 0, "attention_bwd_simt: batch-major token order is only implemented by the tensor-core kernels");
  PFN_CHECK_ARG(d->delta_token_major == 0, "attention_bwd_simt: a precomputed token-major delta is only consumed by the tensor-core kernels");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  return d->dtype == PFN_F32 ? dispatch_attn_simt<float>(d, true, s) : dispatch_attn_simt<__nv_bfloat16>(d, true, s);
}
