// Tensor-core masked attention for the single_eval_pos mask (reference transformer.py:35-41), head dim 128, bf16.
//
//   keys(i) = [0, sep)  U  {i if i >= sep}        o_i = softmax_j(q_i.k_j / sqrt(dh)) v_j
//
// The [T,T] mask is never built: the dense part (keys < sep) runs on the tensor cores in 64-key blocks and the single
// diagonal key of a query row is a 128-wide dot product done by the four lanes that own the row.  Q/K/V rows are read
// straight out of the packed [T*B, 3E] in-projection output, so there is no head-split / transpose kernel.
//
// One CTA (4 warps) per (batch, head, 64-row query tile); warp w owns query rows [16 w, 16 w + 16).  K and V blocks are
// double-buffered with cp.async so the loads of block j+1 overlap the MMAs and softmax of block j:
//   S_j = Q K_j^T (mma.sync, fp32)  ->  online softmax in the log2 domain  ->  P_j as bf16 A fragments  ->  O += P_j V_j
// P_j never leaves the registers: the S accumulator layout of two n-tiles is the A fragment layout of one k-step.
#include "attention_common.cuh"

namespace pfn {

constexpr int ATT_BM = 64;                                // query rows per CTA
constexpr int ATT_BN = 64;                                // keys per block
constexpr int ATT_TILE_BYTES = ATT_BM * ATT_ROW_BYTES;    // 16 KB
constexpr int ATT_FWD_SMEM = 5 * ATT_TILE_BYTES;          // Q + 2 x K + 2 x V

struct AttnFwdParams {
  int T, B, H, sep;
  float scale_log2;   // scale * log2(e)
  const __nv_bfloat16* qkv; int ld_qkv;
  __nv_bfloat16* out; int ld_out;
  float* lse;
  int n_qtiles;
  int batch_major;
  uint32_t drop_seed; int drop_thr;   // dropout on the probabilities (thr 0 = off), csrc/dropout.cuh
};

__global__ void __launch_bounds__(128, 2)
attn_fwd_tc_kernel(const AttnFwdParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* sQ = smem;
  uint8_t* sK = smem + ATT_TILE_BYTES;                    // buffer s at + s * 16 KB
  uint8_t* sV = smem + 3 * ATT_TILE_BYTES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qt = static_cast<int>(blockIdx.x) % p.n_qtiles;
  const int bh = static_cast<int>(blockIdx.x) / p.n_qtiles;
  const int h = bh % p.H, b = bh / p.H;
  const int E = p.H * ATT_DH;
  const int i0 = qt * ATT_BM;
  const int nblk = (p.sep + ATT_BN - 1) / ATT_BN;

  att_load_tile<ATT_BM>(sQ, p.qkv, p.ld_qkv, h * ATT_DH, i0, p.T, b, p.T, p.B, p.batch_major);
  if (nblk > 0) {
    att_load_tile<ATT_BN>(sK, p.qkv, p.ld_qkv, E + h * ATT_DH, 0, p.sep, b, p.T, p.B, p.batch_major);
    att_load_tile<ATT_BN>(sV, p.qkv, p.ld_qkv, 2 * E + h * ATT_DH, 0, p.sep, b, p.T, p.B, p.batch_major);
  }
  tc::cp_async_commit();

  float o[16][4];
#pragma unroll
  for (int j = 0; j < 16; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const int r0 = 16 * warp;
  const uint32_t drow0 = static_cast<uint32_t>(bh) * p.T + i0 + r0 + (lane >> 2);   // dropout row of this lane's first row
  const uint32_t q_s = tc::smem_u32(sQ);

  for (int kb = 0; kb < nblk; ++kb) {
    if (kb + 1 < nblk) {
      const int nb = (kb + 1) & 1;
      att_load_tile<ATT_BN>(sK + nb * ATT_TILE_BYTES, p.qkv, p.ld_qkv, E + h * ATT_DH, (kb + 1) * ATT_BN, p.sep, b, p.T, p.B, p.batch_major);
      att_load_tile<ATT_BN>(sV + nb * ATT_TILE_BYTES, p.qkv, p.ld_qkv, 2 * E + h * ATT_DH, (kb + 1) * ATT_BN, p.sep, b, p.T, p.B, p.batch_major);
      tc::cp_async_commit();
      tc::cp_async_wait<1>();
    } else {
      tc::cp_async_wait<0>();
    }
    __syncthreads();
    const uint32_t k_s = tc::smem_u32(sK + (kb & 1) * ATT_TILE_BYTES);
    const uint32_t v_s = tc::smem_u32(sV + (kb & 1) * ATT_TILE_BYTES);

    float s[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      uint32_t a[4];
      att_frag_a(a, q_s, r0, kk * 16, lane);
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t bb[4];
        att_frag_b(bb, k_s, np * 16, kk * 16, lane);
        tc::mma_bf16_16816(s[2 * np], a, bb[0], bb[1]);
        tc::mma_bf16_16816(s[2 * np + 1], a, bb[2], bb[3]);
      }
    }
    // online softmax (log2 domain); keys >= sep of the last block are masked
    const int key0 = kb * ATT_BN + 2 * (lane & 3);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const bool ok = key0 + 8 * j + (e & 1) < p.sep;
        s[j][e] = ok ? s[j][e] * p.scale_log2 : -INFINITY;
        mx[e >> 1] = fmaxf(mx[e >> 1], s[j][e]);
      }
    float corr[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float mn = fmaxf(m[r], quad_max(mx[r]));
      corr[r] = fast_ex2(m[r] - mn);
      m[r] = mn;
      l[r] *= corr[r];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float pr = fast_ex2(s[j][e] - m[e >> 1]);
        l[e >> 1] += pr;
        if (p.drop_thr > 0 && !drop_keep(p.drop_seed, drow0 + 8 * (e >> 1), key0 + 8 * j + (e & 1), p.drop_thr)) s[j][e] = 0.f;
        else s[j][e] = pr;
      }
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      o[j][0] *= corr[0]; o[j][1] *= corr[0];
      o[j][2] *= corr[1]; o[j][3] *= corr[1];
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t a[4];
      a[0] = tc::pack_bf16x2(s[2 * kk][0], s[2 * kk][1]);
      a[1] = tc::pack_bf16x2(s[2 * kk][2], s[2 * kk][3]);
      a[2] = tc::pack_bf16x2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      a[3] = tc::pack_bf16x2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
      for (int dp = 0; dp < 8; ++dp) {
        uint32_t bb[4];
        att_frag_bt(bb, v_s, kk * 16, dp * 16, lane);
        tc::mma_bf16_16816(o[2 * dp], a, bb[0], bb[1]);
        tc::mma_bf16_16816(o[2 * dp + 1], a, bb[2], bb[3]);
      }
    }
    __syncthreads();     // this buffer is refilled by the next iteration's loads
  }

  // diagonal key of the query rows (i >= sep), normalisation, stores
  const float dscale = p.drop_thr > 0 ? drop_scale(p.drop_thr) : 1.0f;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = i0 + r0 + (lane >> 2) + 8 * r;
    float lr = quad_sum(l[r]);
    const bool valid = i < p.T;
    const bool diag = valid && i >= p.sep;
    const __nv_bfloat16* qrow = p.qkv + att_tok(valid ? i : 0, b, p.T, p.B, p.batch_major) * p.ld_qkv + h * ATT_DH;
    float sd = 0.f;
    if (diag) {
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float2 q = att_ld2(qrow, j, lane), k = att_ld2(qrow + E, j, lane);
        sd = fmaf(q.x, k.x, fmaf(q.y, k.y, sd));
      }
    }
    sd = quad_sum(sd) * p.scale_log2;
    if (diag) {
      const float mn = fmaxf(m[r], sd);
      const float c = fast_ex2(m[r] - mn);
      const float pr = fast_ex2(sd - mn);
      lr = lr * c + pr;
      m[r] = mn;
      const float pd = (p.drop_thr > 0 && !drop_keep(p.drop_seed, drow0 + 8 * r, i, p.drop_thr)) ? 0.f : pr;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float2 v = att_ld2(qrow + 2 * E, j, lane);
        o[j][2 * r] = fmaf(pd, v.x, o[j][2 * r] * c);
        o[j][2 * r + 1] = fmaf(pd, v.y, o[j][2 * r + 1] * c);
      }
    }
    if (valid) {
      const float inv = dscale / lr;
      __nv_bfloat16* orow = p.out + att_tok(i, b, p.T, p.B, p.batch_major) * p.ld_out + h * ATT_DH;
#pragma unroll
      for (int j = 0; j < 16; ++j) att_st2(orow, j, lane, o[j][2 * r] * inv, o[j][2 * r + 1] * inv);
      if ((lane & 3) == 0) p.lse[static_cast<size_t>(bh) * p.T + i] = (m[r] + __log2f(lr)) * 0.69314718055994531f;
    }
  }
}

}  // namespace pfn

using namespace pfn;

extern "C" int pfn_attention_fwd_tc(const pfn_attn_desc* d, void* stream) {
  if (int rc = check_tc_attn(d, false, "attention_fwd_tc")) return rc;
  AttnFwdParams p;
  p.T = d->T; p.B = d->B; p.H = d->H; p.sep = d->sep;
  p.scale_log2 = d->scale * 1.4426950408889634f;
  p.qkv = reinterpret_cast<const __nv_bfloat16*>(d->qkv); p.ld_qkv = d->ld_qkv;
  p.out = reinterpret_cast<__nv_bfloat16*>(d->out); p.ld_out = d->ld_out;
  p.lse = d->lse;
  p.n_qtiles = (d->T + ATT_BM - 1) / ATT_BM;
  p.batch_major = d->batch_major;
  p.drop_seed = d->drop_seed; p.drop_thr = d->drop_thr;
  const long long grid = static_cast<long long>(p.n_qtiles) * d->B * d->H;
  PFN_CHECK_ARG(grid < (1LL << 31), "attention_fwd_tc: too many tiles");
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set)) {
    PFN_CUDA_OK(cudaFuncSetAttribute(attn_fwd_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_FWD_SMEM));
  }
  attn_fwd_tc_kernel<<<static_cast<unsigned>(grid), 128, ATT_FWD_SMEM, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  PFN_LAUNCH_OK();
  return 0;
}
