// fp32-FMA masked attention (forward, dQ, dK/dV) for the fp32 parity mode and for head sizes / dtypes the
// tensor-core kernels do not take.  One warp per (batch, head, row); the head dimension is spread over the
// lanes, scores are reduced with warp shuffles, softmax is computed online.  The single_eval_pos mask of
// reference transformer.py:35-41 is implicit:  keys(i) = [0, sep)  U  {i if i >= sep}.  The forward also serves the
// context attention (pfn_attention_ctx_fwd_simt): there the sep keys come from the K/V cache and every row has its own key.
// In the ragged entry points (pfn_attention_ragged_fwd_simt, pfn_attention_ctx_ragged_fwd_simt and the training pair
// pfn_attention_ragged_train_{fwd,bwd}_simt) dataset b has n_keys[b] keys in place of sep.  The context attention also
// has a backward (pfn_attention_ctx_bwd_simt): the dQ kernel on the cached keys, whose gradient is not formed.
#include "common.cuh"
#include "dropout.cuh"
#include "../../include/pfn_b200_ragged.h"
#include "../../include/pfn_b200_ragged_train.h"
#include "../../include/pfn_b200_input_grad.h"

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

// The keys shared by all rows of batch b: its first sep_b keys, K of key j at kv + (j*B + b)*ld + h*dh, V at + v_off (the
// packed qkv itself for the masked attention, the K/V cache for the context attention).  sep_b is sep, or in the ragged
// kernel n_keys[b] clamped to [0, sep].  Rows i >= min(diag_from, sep_b) also attend to their own key; the key order is the
// same in all uses, so a query row gets the same bits from any entry point.
struct SharedKeys {
  const void* kv; int ld; int v_off; int diag_from;
  const int* n_keys;
};

template <typename T, int DPL, bool kRagged>
__global__ void __launch_bounds__(256)
attn_fwd_simt_kernel(const pfn_attn_desc d, const SharedKeys sk) {
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
    const int sep = kRagged ? min(max(__ldg(sk.n_keys + b), 0), d.sep) : d.sep;
    const int nkeys = sep + (i >= (kRagged ? min(sk.diag_from, sep) : sk.diag_from) ? 1 : 0);
    for (int jj = 0; jj < nkeys; ++jj) {
      const int j = jj < sep ? jj : i;
      const T* krow = jj < sep ? reinterpret_cast<const T*>(sk.kv) + (static_cast<size_t>(j) * d.B + b) * sk.ld + h * d.dh
                               : qkv + (static_cast<size_t>(i) * d.B + b) * d.ld_qkv + E + h * d.dh;
      const int v_off = jj < sep ? sk.v_off : E;
      float k[DPL], v[DPL];
      load_head<T, DPL>(krow, d.dh, lane, k);
      load_head<T, DPL>(krow + v_off, d.dh, lane, v);
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
    if (lane == 0 && d.lse) d.lse[static_cast<size_t>(bh) * d.T + i] = m + logf(l);
  }
}

// the key count of dataset b: sep, or n_keys[b] clamped to [0, sep] in the ragged kernels
template <bool kRagged>
__device__ __forceinline__ int simt_sep(const pfn_attn_desc& d, const int* n_keys, int b) {
  return kRagged ? min(max(__ldg(n_keys + b), 0), d.sep) : d.sep;
}

// dQ (+ delta, + the diagonal-key contributions that are the ONLY gradient of k_i, v_i for query rows), over the keys sk
// in the order of the forward
template <typename T, int DPL, bool kRagged>
__global__ void __launch_bounds__(256)
attn_bwd_dq_simt_kernel(const pfn_attn_desc d, float* __restrict__ delta, const SharedKeys sk) {
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
    const int sep = simt_sep<kRagged>(d, sk.n_keys, b);
    const int nkeys = sep + (i >= (kRagged ? min(sk.diag_from, sep) : sk.diag_from) ? 1 : 0);
    for (int jj = 0; jj < nkeys; ++jj) {
      const int j = jj < sep ? jj : i;
      const T* krow = jj < sep ? reinterpret_cast<const T*>(sk.kv) + (static_cast<size_t>(j) * d.B + b) * sk.ld + h * d.dh
                               : qkv + tok * d.ld_qkv + E + h * d.dh;
      float k[DPL], v[DPL];
      load_head<T, DPL>(krow, d.dh, lane, k);
      load_head<T, DPL>(krow + (jj < sep ? sk.v_off : E), d.dh, lane, v);
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
      if (jj >= sep) {
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

// dK, dV of the train keys j < sep (j < n_keys[b] when ragged): every row i attends to them.
template <typename T, int DPL, bool kRagged>
__global__ void __launch_bounds__(256)
attn_bwd_dkv_simt_kernel(const pfn_attn_desc d, const float* __restrict__ delta, const int* __restrict__ n_keys) {
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
    if (kRagged && j >= simt_sep<true>(d, n_keys, b)) continue;     // a row of b's own: the dQ kernel wrote its dK, dV
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
static int launch_attn_simt(const pfn_attn_desc* d, bool bwd, cudaStream_t s, const SharedKeys& sk) {
  const long long tasks = static_cast<long long>(d->B) * d->H * d->T;
  long long grid = (tasks + 7) / 8;
  const long long max_grid = static_cast<long long>(num_sms()) * 16;
  if (grid > max_grid) grid = max_grid;
  if (!bwd) {
    if (sk.n_keys) attn_fwd_simt_kernel<T, DPL, true><<<static_cast<int>(grid), 256, 0, s>>>(*d, sk);
    else attn_fwd_simt_kernel<T, DPL, false><<<static_cast<int>(grid), 256, 0, s>>>(*d, sk);
    PFN_LAUNCH_OK();
    return 0;
  }
  if (sk.n_keys) attn_bwd_dq_simt_kernel<T, DPL, true><<<static_cast<int>(grid), 256, 0, s>>>(*d, d->delta, sk);
  else attn_bwd_dq_simt_kernel<T, DPL, false><<<static_cast<int>(grid), 256, 0, s>>>(*d, d->delta, sk);
  PFN_LAUNCH_OK();
  // the shared keys are rows of qkv, which get dK / dV, when rows below diag_from exist: the masked attention with sep > 0
  // (the context attention's cached keys have diag_from 0 and are constants)
  if (sk.diag_from > 0) {
    const long long tasks2 = static_cast<long long>(d->B) * d->H * d->sep;
    long long grid2 = (tasks2 + 7) / 8;
    if (grid2 > max_grid) grid2 = max_grid;
    if (sk.n_keys) attn_bwd_dkv_simt_kernel<T, DPL, true><<<static_cast<int>(grid2), 256, 0, s>>>(*d, d->delta, sk.n_keys);
    else attn_bwd_dkv_simt_kernel<T, DPL, false><<<static_cast<int>(grid2), 256, 0, s>>>(*d, d->delta, nullptr);
    PFN_LAUNCH_OK();
  }
  return 0;
}

template <typename T>
static int dispatch_attn_simt(const pfn_attn_desc* d, bool bwd, cudaStream_t s, const SharedKeys& sk) {
  if (d->dh <= 32) return launch_attn_simt<T, 1>(d, bwd, s, sk);
  if (d->dh <= 64) return launch_attn_simt<T, 2>(d, bwd, s, sk);
  if (d->dh <= 128) return launch_attn_simt<T, 4>(d, bwd, s, sk);
  PFN_CHECK_ARG(d->dh <= 256, "attention_simt: head dim %d > 256 unsupported", d->dh);
  return launch_attn_simt<T, 8>(d, bwd, s, sk);
}

// the keys of the masked attention: [0, sep) (or [0, n_keys[b])) of the packed qkv, and row i's own key for i >= sep
static SharedKeys masked_keys(const pfn_attn_desc* d, const int* n_keys = nullptr) {
  const size_t esz = d->dtype == PFN_F32 ? 4 : 2;
  return {static_cast<const char*>(d->qkv) + esz * d->H * d->dh, d->ld_qkv, d->H * d->dh, d->sep, n_keys};
}

// the keys of the context attention: [0, n) (or [0, n_keys[b])) of the cache, and every row's own key
static SharedKeys cached_keys(const pfn_attn_ctx_desc* d, const int* n_keys = nullptr) {
  return {d->kv, d->ld_kv, d->H * d->dh, 0, n_keys};
}

// rows of the masked-attention forward with T = m query rows and sep = n shared keys taken from the cache
static pfn_attn_desc ctx_as_masked(const pfn_attn_ctx_desc* d) {
  pfn_attn_desc a = {};
  a.T = d->m; a.B = d->B; a.H = d->H; a.dh = d->dh; a.sep = d->n;
  a.dtype = d->dtype; a.scale = d->scale;
  a.qkv = d->qkv; a.ld_qkv = d->ld_qkv;
  a.out = d->out; a.ld_out = d->ld_out;
  return a;
}

static int dispatch_attn_simt(const pfn_attn_desc* d, bool bwd, cudaStream_t s, const SharedKeys& sk) {
  return d->dtype == PFN_F32 ? dispatch_attn_simt<float>(d, bwd, s, sk) : dispatch_attn_simt<__nv_bfloat16>(d, bwd, s, sk);
}

int check_attn_desc_public(const pfn_attn_desc* d, bool bwd, const char* who) { return check_attn_desc(d, bwd, who); }

int check_attn_ctx_desc(const pfn_attn_ctx_desc* d, const char* who) {
  PFN_CHECK_ARG(d != nullptr, "%s: null descriptor", who);
  PFN_CHECK_ARG(d->m > 0 && d->n >= 0 && d->B > 0 && d->H > 0 && d->dh > 0, "%s: bad shape m=%d n=%d B=%d H=%d dh=%d", who,
                d->m, d->n, d->B, d->H, d->dh);
  PFN_CHECK_ARG(d->dtype == PFN_F32 || d->dtype == PFN_BF16, "%s: bad dtype %d", who, d->dtype);
  PFN_CHECK_ARG(d->qkv && d->out && (d->kv || d->n == 0), "%s: null qkv/kv/out", who);
  PFN_CHECK_ARG(d->ld_qkv >= 3 * d->H * d->dh && d->ld_out >= d->H * d->dh && (d->n == 0 || d->ld_kv >= 2 * d->H * d->dh),
                "%s: leading dims too small", who);
  PFN_CHECK_ARG(static_cast<long long>(d->m + d->n) * d->B * d->H < (1LL << 31), "%s: too many rows", who);
  return 0;
}

int attn_ragged_as_masked(const pfn_attn_ragged_desc* d, pfn_attn_desc* a, const char* who) {
  PFN_CHECK_ARG(d != nullptr, "%s: null descriptor", who);
  PFN_CHECK_ARG(d->n_keys != nullptr, "%s: null n_keys", who);
  *a = pfn_attn_desc{};
  a->T = d->T; a->B = d->B; a->H = d->H; a->dh = d->dh; a->sep = d->T;
  a->dtype = d->dtype; a->scale = d->scale;
  a->qkv = d->qkv; a->ld_qkv = d->ld_qkv;
  a->out = d->out; a->ld_out = d->ld_out;
  PFN_CHECK_ARG(d->T > 0 && d->B > 0 && d->H > 0 && d->dh > 0, "%s: bad shape T=%d B=%d H=%d dh=%d", who, d->T, d->B, d->H,
                d->dh);
  PFN_CHECK_ARG(d->dtype == PFN_F32 || d->dtype == PFN_BF16, "%s: bad dtype %d", who, d->dtype);
  PFN_CHECK_ARG(d->qkv && d->out, "%s: null qkv/out", who);
  PFN_CHECK_ARG(d->ld_qkv >= 3 * d->H * d->dh && d->ld_out >= d->H * d->dh, "%s: leading dims too small", who);
  return 0;
}

int check_attn_ctx_grad_desc(const pfn_attn_ctx_grad_desc* d, bool bwd, const char* who) {
  PFN_CHECK_ARG(d != nullptr, "%s: null descriptor", who);
  if (int rc = check_attn_ctx_desc(&d->c, who)) return rc;
  PFN_CHECK_ARG(d->lse != nullptr, "%s: null lse", who);
  if (bwd) {
    PFN_CHECK_ARG(d->dout && d->dqkv && d->delta, "%s: null dout/dqkv/delta", who);
    PFN_CHECK_ARG(d->ld_dqkv >= 3 * d->c.H * d->c.dh && d->ld_dout >= d->c.H * d->c.dh, "%s: leading dims too small", who);
  }
  return 0;
}

int attn_ctx_ragged_as_ctx(const pfn_attn_ctx_ragged_desc* d, pfn_attn_ctx_desc* c, const char* who) {
  PFN_CHECK_ARG(d != nullptr, "%s: null descriptor", who);
  PFN_CHECK_ARG(d->n_keys != nullptr, "%s: null n_keys", who);
  c->m = d->m; c->n = d->n; c->B = d->B; c->H = d->H; c->dh = d->dh;
  c->dtype = d->dtype; c->scale = d->scale;
  c->qkv = d->qkv; c->ld_qkv = d->ld_qkv;
  c->kv = d->kv; c->ld_kv = d->ld_kv;
  c->out = d->out; c->ld_out = d->ld_out;
  return check_attn_ctx_desc(c, who);
}

}  // namespace pfn

using namespace pfn;

extern "C" int pfn_attention_fwd_simt(const pfn_attn_desc* d, void* stream) {
  if (int rc = check_attn_desc(d, false, "attention_fwd_simt")) return rc;
  PFN_CHECK_ARG(d->batch_major == 0, "attention_fwd_simt: batch-major token order is only implemented by the tensor-core kernels");
  return dispatch_attn_simt(d, false, reinterpret_cast<cudaStream_t>(stream), masked_keys(d));
}

extern "C" int pfn_attention_bwd_simt(const pfn_attn_desc* d, void* stream) {
  if (int rc = check_attn_desc(d, true, "attention_bwd_simt")) return rc;
  PFN_CHECK_ARG(d->batch_major == 0, "attention_bwd_simt: batch-major token order is only implemented by the tensor-core kernels");
  PFN_CHECK_ARG(d->delta_token_major == 0, "attention_bwd_simt: a precomputed token-major delta is only consumed by the tensor-core kernels");
  return dispatch_attn_simt(d, true, reinterpret_cast<cudaStream_t>(stream), masked_keys(d));
}

extern "C" int pfn_attention_ctx_fwd_simt(const pfn_attn_ctx_desc* d, void* stream) {
  if (int rc = check_attn_ctx_desc(d, "attention_ctx_fwd_simt")) return rc;
  const pfn_attn_desc a = ctx_as_masked(d);
  return dispatch_attn_simt(&a, false, reinterpret_cast<cudaStream_t>(stream), cached_keys(d));
}

extern "C" int pfn_attention_ragged_fwd_simt(const pfn_attn_ragged_desc* d, void* stream) {
  pfn_attn_desc a;
  if (int rc = attn_ragged_as_masked(d, &a, "attention_ragged_fwd_simt")) return rc;
  return dispatch_attn_simt(&a, false, reinterpret_cast<cudaStream_t>(stream), masked_keys(&a, d->n_keys));
}

extern "C" int pfn_attention_ctx_ragged_fwd_simt(const pfn_attn_ctx_ragged_desc* d, void* stream) {
  pfn_attn_ctx_desc c;
  if (int rc = attn_ctx_ragged_as_ctx(d, &c, "attention_ctx_ragged_fwd_simt")) return rc;
  const pfn_attn_desc a = ctx_as_masked(&c);
  return dispatch_attn_simt(&a, false, reinterpret_cast<cudaStream_t>(stream), cached_keys(&c, d->n_keys));
}

// the ragged training descriptor checked as the scalar one (its sep the bound of the key counts)
static int check_ragged_train_simt(const pfn_attn_ragged_train_desc* d, bool bwd, const char* who) {
  PFN_CHECK_ARG(d != nullptr && d->n_keys != nullptr, "%s: null descriptor / n_keys", who);
  if (int rc = check_attn_desc(&d->a, bwd, who)) return rc;
  PFN_CHECK_ARG(d->a.batch_major == 0, "%s: batch-major token order is only implemented by the tensor-core kernels", who);
  PFN_CHECK_ARG(d->a.delta_token_major == 0, "%s: a precomputed token-major delta is only consumed by the tensor-core kernels",
                who);
  return 0;
}

extern "C" int pfn_attention_ragged_train_fwd_simt(const pfn_attn_ragged_train_desc* d, void* stream) {
  if (int rc = check_ragged_train_simt(d, false, "attention_ragged_train_fwd_simt")) return rc;
  return dispatch_attn_simt(&d->a, false, reinterpret_cast<cudaStream_t>(stream), masked_keys(&d->a, d->n_keys));
}

extern "C" int pfn_attention_ragged_train_bwd_simt(const pfn_attn_ragged_train_desc* d, void* stream) {
  if (int rc = check_ragged_train_simt(d, true, "attention_ragged_train_bwd_simt")) return rc;
  return dispatch_attn_simt(&d->a, true, reinterpret_cast<cudaStream_t>(stream), masked_keys(&d->a, d->n_keys));
}

// the context attention with lse, as the masked attention with T = m, sep = n over the cached keys
static pfn_attn_desc ctx_grad_as_masked(const pfn_attn_ctx_grad_desc* d) {
  pfn_attn_desc a = ctx_as_masked(&d->c);
  a.lse = d->lse;
  a.dout = d->dout; a.ld_dout = d->ld_dout;
  a.dqkv = d->dqkv; a.ld_dqkv = d->ld_dqkv;
  a.delta = d->delta;
  return a;
}

extern "C" int pfn_attention_ctx_grad_fwd_simt(const pfn_attn_ctx_grad_desc* d, void* stream) {
  if (int rc = check_attn_ctx_grad_desc(d, false, "attention_ctx_grad_fwd_simt")) return rc;
  const pfn_attn_desc a = ctx_grad_as_masked(d);
  return dispatch_attn_simt(&a, false, reinterpret_cast<cudaStream_t>(stream), cached_keys(&d->c, d->n_keys));
}

extern "C" int pfn_attention_ctx_bwd_simt(const pfn_attn_ctx_grad_desc* d, void* stream) {
  if (int rc = check_attn_ctx_grad_desc(d, true, "attention_ctx_bwd_simt")) return rc;
  const pfn_attn_desc a = ctx_grad_as_masked(d);
  return dispatch_attn_simt(&a, true, reinterpret_cast<cudaStream_t>(stream), cached_keys(&d->c, d->n_keys));
}
