// Tensor-core backward of the single_eval_pos-masked attention (head dim 128, bf16), three kernels:
//
//  (0) attn_bwd_delta_kernel  delta[b,h,i] = dO_i . O_i   (one warp per token row, HBM-bound, 16 B vectors); skipped when
//      the caller passes the token-major delta the out-projection dgrad's ROWDOT epilogue already produced
//
//  (1) attn_bwd_dq_kernel     one CTA (4 warps) per (batch, head, 64-row query tile); loop over 64-key blocks of the train keys:
//          S_j  = Q K_j^T      dP_j = dO V_j^T                                 (mma.sync, fp32)
//          dS_j = exp2(S_j c - lse2) * (dP_j - delta) * scale  -> bf16 A fragments (registers)
//          dQ  += dS_j K_j
//      For a query row (i >= sep) the diagonal key is attended by that row only, so dK_i = dS_ii q_i and dV_i = P_ii dO_i are
//      complete: the four lanes that own the row compute and store them, and add dS_ii k_i to dQ.
//
//  (2) attn_bwd_dkv_kernel    one CTA (4 warps) per (batch, head, 64-key tile of the train keys), loop over 32-row query blocks:
//          S^T = K Q_i^T       dP^T = V dO_i^T     (row = key, column = query row)
//          dV += (P^T . mask) dO_i ;   dK += dS^T Q_i
//
// Q/K/V/dO rows come straight out of the packed [T*B, 3E] qkv / [T*B, E] dO buffers; no transposes, no atomics on dQKV.
#include "attention_common.cuh"

namespace pfn {

constexpr int AB_BM = 64;                                 // dQ kernel: query rows per CTA; key block size
constexpr int AB_TILE = AB_BM * ATT_ROW_BYTES;            // 16 KB
constexpr int AB_DQ_SMEM = 6 * AB_TILE;                   // Q + dO + 2 x K + 2 x V
constexpr int AB_QB = 32;                                 // dK/dV kernel: query rows per block
constexpr int AB_QTILE = AB_QB * ATT_ROW_BYTES;           // 8 KB
constexpr int AB_DKV_SMEM = 2 * AB_TILE + 4 * AB_QTILE + 2 * 2 * AB_QB * 4;   // K + V + 2 x (Q, dO) + 2 x (lse2, delta)

struct AttnBwdParams {
  int T, B, H, sep;
  float scale, scale_log2;
  const __nv_bfloat16* qkv; int ld_qkv;
  const __nv_bfloat16* dout; int ld_dout;
  __nv_bfloat16* dqkv; int ld_dqkv;
  const float* lse;
  const float* delta;
  int delta_tm;          // 1: delta is token-major [T*B, H] (GEMM ROWDOT epilogue); 0: [B*H, T]
  float* dq_colsum;      // optional [H*dh]: += column sums of dQ
  uint32_t drop_seed; int drop_thr;   // dropout on the attention probabilities (thr 0 = off), csrc/dropout.cuh
  int n_tiles;
  int batch_major;
};

__device__ __forceinline__ float ab_delta(const AttnBwdParams& p, int b, int h, int i) {
  return p.delta_tm ? p.delta[att_tok(i, b, p.T, p.B, 0) * p.H + h] : p.delta[(static_cast<size_t>(b) * p.H + h) * p.T + i];
}

// =====================================================================================================================
// Kernel 0: delta = rowsum(dO * O) per (batch, head, row)
// =====================================================================================================================
__global__ void __launch_bounds__(256)
attn_bwd_delta_kernel(const __nv_bfloat16* __restrict__ out, int ld_out, const __nv_bfloat16* __restrict__ dout,
                      int ld_dout, float* __restrict__ delta, int T, int B, int H, int batch_major) {
  // one warp per token; a 128-wide head = 16 lanes x 8 elements, so a warp covers two heads per pass
  const int lane = threadIdx.x & 31;
  const long long warp = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const long long rows = static_cast<long long>(T) * B;
  for (long long tok = warp; tok < rows; tok += nwarps) {
    const int t = batch_major ? static_cast<int>(tok % T) : static_cast<int>(tok / B);
    const int b = batch_major ? static_cast<int>(tok / T) : static_cast<int>(tok % B);
    for (int h0 = 0; h0 < H; h0 += 2) {
      const int h = h0 + (lane >> 4);
      float acc = 0.f;
      if (h < H) {
        const int col = h * ATT_DH + (lane & 15) * 8;
        const uint4 pa = *reinterpret_cast<const uint4*>(out + tok * ld_out + col);
        const uint4 pb = *reinterpret_cast<const uint4*>(dout + tok * ld_dout + col);
        const __nv_bfloat162* ha = reinterpret_cast<const __nv_bfloat162*>(&pa);
        const __nv_bfloat162* hb = reinterpret_cast<const __nv_bfloat162*>(&pb);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 x = __bfloat1622float2(ha[j]);
          const float2 y = __bfloat1622float2(hb[j]);
          acc = fmaf(x.x, y.x, acc);
          acc = fmaf(x.y, y.y, acc);
        }
      }
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if ((lane & 15) == 0 && h < H) delta[(static_cast<size_t>(b) * H + h) * T + t] = acc;
    }
  }
}

// =====================================================================================================================
// Kernel 1: dQ (+ dK, dV of the query rows' own keys)
// =====================================================================================================================
__global__ void __launch_bounds__(128, 2)
attn_bwd_dq_kernel(const AttnBwdParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* sQ = smem;
  uint8_t* sD = smem + AB_TILE;
  uint8_t* sK = smem + 2 * AB_TILE;                       // buffer s at + s * 16 KB
  uint8_t* sV = smem + 4 * AB_TILE;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qt = static_cast<int>(blockIdx.x) % p.n_tiles;
  const int bh = static_cast<int>(blockIdx.x) / p.n_tiles;
  const int h = bh % p.H, b = bh / p.H;
  const int E = p.H * ATT_DH;
  const int i0 = qt * AB_BM;
  const int nblk = (p.sep + AB_BM - 1) / AB_BM;
  const int r0 = 16 * warp;

  att_load_tile<AB_BM>(sQ, p.qkv, p.ld_qkv, h * ATT_DH, i0, p.T, b, p.T, p.B, p.batch_major);
  att_load_tile<AB_BM>(sD, p.dout, p.ld_dout, h * ATT_DH, i0, p.T, b, p.T, p.B, p.batch_major);
  if (nblk > 0) {
    att_load_tile<AB_BM>(sK, p.qkv, p.ld_qkv, E + h * ATT_DH, 0, p.sep, b, p.T, p.B, p.batch_major);
    att_load_tile<AB_BM>(sV, p.qkv, p.ld_qkv, 2 * E + h * ATT_DH, 0, p.sep, b, p.T, p.B, p.batch_major);
  }
  tc::cp_async_commit();

  // per-row statistics of this lane's two rows
  float lse2[2], dl[2];
  uint32_t drow[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = i0 + r0 + (lane >> 2) + 8 * r;
    const bool valid = i < p.T;
    lse2[r] = valid ? p.lse[static_cast<size_t>(bh) * p.T + i] * 1.4426950408889634f : INFINITY;
    dl[r] = valid ? ab_delta(p, b, h, i) : 0.f;
    drow[r] = static_cast<uint32_t>(bh) * p.T + i;
  }
  const float dscale = p.drop_thr > 0 ? drop_scale(p.drop_thr) : 1.0f;

  float dq[16][4];
#pragma unroll
  for (int j = 0; j < 16; ++j) dq[j][0] = dq[j][1] = dq[j][2] = dq[j][3] = 0.f;
  const uint32_t q_s = tc::smem_u32(sQ), d_s = tc::smem_u32(sD);

  for (int kb = 0; kb < nblk; ++kb) {
    if (kb + 1 < nblk) {
      const int nb = (kb + 1) & 1;
      att_load_tile<AB_BM>(sK + nb * AB_TILE, p.qkv, p.ld_qkv, E + h * ATT_DH, (kb + 1) * AB_BM, p.sep, b, p.T, p.B, p.batch_major);
      att_load_tile<AB_BM>(sV + nb * AB_TILE, p.qkv, p.ld_qkv, 2 * E + h * ATT_DH, (kb + 1) * AB_BM, p.sep, b, p.T, p.B, p.batch_major);
      tc::cp_async_commit();
      tc::cp_async_wait<1>();
    } else {
      tc::cp_async_wait<0>();
    }
    __syncthreads();
    const uint32_t k_s = tc::smem_u32(sK + (kb & 1) * AB_TILE);
    const uint32_t v_s = tc::smem_u32(sV + (kb & 1) * AB_TILE);

    float s[8][4], dp[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = dp[j][0] = dp[j][1] = dp[j][2] = dp[j][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      uint32_t aq[4], ad[4];
      att_frag_a(aq, q_s, r0, kk * 16, lane);
      att_frag_a(ad, d_s, r0, kk * 16, lane);
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t bk[4], bv[4];
        att_frag_b(bk, k_s, np * 16, kk * 16, lane);
        att_frag_b(bv, v_s, np * 16, kk * 16, lane);
        tc::mma_bf16_16816(s[2 * np], aq, bk[0], bk[1]);
        tc::mma_bf16_16816(s[2 * np + 1], aq, bk[2], bk[3]);
        tc::mma_bf16_16816(dp[2 * np], ad, bv[0], bv[1]);
        tc::mma_bf16_16816(dp[2 * np + 1], ad, bv[2], bv[3]);
      }
    }
    // dS = P (mask dP - delta) scale  (keys >= sep of the last block get P = 0)
    const int key0 = kb * AB_BM + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = key0 + 8 * j + (e & 1);
        const float pr = key < p.sep ? fast_ex2(fmaf(s[j][e], p.scale_log2, -lse2[e >> 1])) : 0.f;
        const float mk = p.drop_thr > 0 ? (drop_keep(p.drop_seed, drow[e >> 1], key, p.drop_thr) ? dscale : 0.f) : 1.f;
        s[j][e] = pr * fmaf(mk, dp[j][e], -dl[e >> 1]) * p.scale;
      }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t a[4];
      a[0] = tc::pack_bf16x2(s[2 * kk][0], s[2 * kk][1]);
      a[1] = tc::pack_bf16x2(s[2 * kk][2], s[2 * kk][3]);
      a[2] = tc::pack_bf16x2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      a[3] = tc::pack_bf16x2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
      for (int dd = 0; dd < 8; ++dd) {
        uint32_t bb[4];
        att_frag_bt(bb, k_s, kk * 16, dd * 16, lane);
        tc::mma_bf16_16816(dq[2 * dd], a, bb[0], bb[1]);
        tc::mma_bf16_16816(dq[2 * dd + 1], a, bb[2], bb[3]);
      }
    }
    __syncthreads();     // this buffer is refilled by the next iteration's loads
  }
  tc::cp_async_wait<0>();

  // diagonal keys of the query rows, dQ stores, column sums
  float cs[16][2];
#pragma unroll
  for (int j = 0; j < 16; ++j) cs[j][0] = cs[j][1] = 0.f;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = i0 + r0 + (lane >> 2) + 8 * r;
    const bool valid = i < p.T;
    const bool diag = valid && i >= p.sep;
    const size_t tok = att_tok(valid ? i : 0, b, p.T, p.B, p.batch_major);
    const __nv_bfloat16* qrow = p.qkv + tok * p.ld_qkv + h * ATT_DH;
    const __nv_bfloat16* drw = p.dout + tok * p.ld_dout + h * ATT_DH;
    __nv_bfloat16* grow = p.dqkv + tok * p.ld_dqkv + h * ATT_DH;
    float sd = 0.f, dpd = 0.f;
    if (diag) {
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float2 q = att_ld2(qrow, j, lane), k = att_ld2(qrow + E, j, lane);
        const float2 g = att_ld2(drw, j, lane), v = att_ld2(qrow + 2 * E, j, lane);
        sd = fmaf(q.x, k.x, fmaf(q.y, k.y, sd));
        dpd = fmaf(g.x, v.x, fmaf(g.y, v.y, dpd));
      }
    }
    sd = quad_sum(sd);
    dpd = quad_sum(dpd);
    if (diag) {
      const float pr = fast_ex2(fmaf(sd, p.scale_log2, -lse2[r]));
      const float mk = p.drop_thr > 0 ? (drop_keep(p.drop_seed, drow[r], i, p.drop_thr) ? dscale : 0.f) : 1.f;
      const float ds = pr * fmaf(mk, dpd, -dl[r]) * p.scale;
      const float pm = pr * mk;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float2 q = att_ld2(qrow, j, lane), k = att_ld2(qrow + E, j, lane), g = att_ld2(drw, j, lane);
        dq[j][2 * r] = fmaf(ds, k.x, dq[j][2 * r]);
        dq[j][2 * r + 1] = fmaf(ds, k.y, dq[j][2 * r + 1]);
        att_st2(grow + E, j, lane, ds * q.x, ds * q.y);
        att_st2(grow + 2 * E, j, lane, pm * g.x, pm * g.y);
      }
    }
    if (valid) {
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        att_st2(grow, j, lane, dq[j][2 * r], dq[j][2 * r + 1]);
        cs[j][0] += __bfloat162float(__float2bfloat16_rn(dq[j][2 * r]));
        cs[j][1] += __bfloat162float(__float2bfloat16_rn(dq[j][2 * r + 1]));
      }
    }
  }
  if (p.dq_colsum != nullptr) {
    // reduce over the eight row groups of the warp (lanes with equal lane & 3), then one atomic per column and warp
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float v = cs[j][e];
        v += __shfl_xor_sync(0xffffffffu, v, 4);
        v += __shfl_xor_sync(0xffffffffu, v, 8);
        v += __shfl_xor_sync(0xffffffffu, v, 16);
        if (lane < 4) atomicAdd(p.dq_colsum + h * ATT_DH + 8 * j + 2 * lane + e, v);
      }
  }
}

// =====================================================================================================================
// Kernel 2: dK, dV of the train keys
// =====================================================================================================================
__global__ void __launch_bounds__(128, 2)
attn_bwd_dkv_kernel(const AttnBwdParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* sK = smem;
  uint8_t* sV = smem + AB_TILE;
  uint8_t* sQ = smem + 2 * AB_TILE;                       // buffer s at + s * 8 KB
  uint8_t* sD = sQ + 2 * AB_QTILE;
  float* sStat = reinterpret_cast<float*>(sD + 2 * AB_QTILE);   // [2][2][AB_QB]: lse2, delta
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kt = static_cast<int>(blockIdx.x) % p.n_tiles;
  const int bh = static_cast<int>(blockIdx.x) / p.n_tiles;
  const int h = bh % p.H, b = bh / p.H;
  const int E = p.H * ATT_DH;
  const int j0 = kt * AB_BM;
  const int r0 = 16 * warp;                               // this warp's keys: j0 + r0 .. + 15
  const int nqb = (p.T + AB_QB - 1) / AB_QB;

  auto load_block = [&](int qb, int buf) {
    att_load_tile<AB_QB>(sQ + buf * AB_QTILE, p.qkv, p.ld_qkv, h * ATT_DH, qb * AB_QB, p.T, b, p.T, p.B, p.batch_major);
    att_load_tile<AB_QB>(sD + buf * AB_QTILE, p.dout, p.ld_dout, h * ATT_DH, qb * AB_QB, p.T, b, p.T, p.B, p.batch_major);
    if (threadIdx.x < AB_QB) {
      const int i = qb * AB_QB + threadIdx.x;
      const bool valid = i < p.T;
      sStat[buf * 2 * AB_QB + threadIdx.x] = valid ? p.lse[static_cast<size_t>(bh) * p.T + i] * 1.4426950408889634f : INFINITY;
      sStat[buf * 2 * AB_QB + AB_QB + threadIdx.x] = valid ? ab_delta(p, b, h, i) : 0.f;
    }
  };
  att_load_tile<AB_BM>(sK, p.qkv, p.ld_qkv, E + h * ATT_DH, j0, p.sep, b, p.T, p.B, p.batch_major);
  att_load_tile<AB_BM>(sV, p.qkv, p.ld_qkv, 2 * E + h * ATT_DH, j0, p.sep, b, p.T, p.B, p.batch_major);
  load_block(0, 0);
  tc::cp_async_commit();

  const float dscale = p.drop_thr > 0 ? drop_scale(p.drop_thr) : 1.0f;
  float dk[16][4], dv[16][4];
#pragma unroll
  for (int j = 0; j < 16; ++j) dk[j][0] = dk[j][1] = dk[j][2] = dk[j][3] = dv[j][0] = dv[j][1] = dv[j][2] = dv[j][3] = 0.f;
  const uint32_t k_s = tc::smem_u32(sK), v_s = tc::smem_u32(sV);
  const int key_a = j0 + r0 + (lane >> 2);                // this lane's keys: key_a, key_a + 8
  const uint32_t drow_base = static_cast<uint32_t>(bh) * p.T;

  for (int qb = 0; qb < nqb; ++qb) {
    const int buf = qb & 1;
    if (qb + 1 < nqb) {
      load_block(qb + 1, buf ^ 1);
      tc::cp_async_commit();
      tc::cp_async_wait<1>();
    } else {
      tc::cp_async_wait<0>();
    }
    __syncthreads();
    const uint32_t q_s = tc::smem_u32(sQ + buf * AB_QTILE), d_s = tc::smem_u32(sD + buf * AB_QTILE);
    const float* st_lse = sStat + buf * 2 * AB_QB;
    const float* st_dl = st_lse + AB_QB;

    float s[4][4], dp[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = dp[j][0] = dp[j][1] = dp[j][2] = dp[j][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      uint32_t ak[4], av[4];
      att_frag_a(ak, k_s, r0, kk * 16, lane);
      att_frag_a(av, v_s, r0, kk * 16, lane);
#pragma unroll
      for (int np = 0; np < 2; ++np) {
        uint32_t bq[4], bd[4];
        att_frag_b(bq, q_s, np * 16, kk * 16, lane);
        att_frag_b(bd, d_s, np * 16, kk * 16, lane);
        tc::mma_bf16_16816(s[2 * np], ak, bq[0], bq[1]);
        tc::mma_bf16_16816(s[2 * np + 1], ak, bq[2], bq[3]);
        tc::mma_bf16_16816(dp[2 * np], av, bd[0], bd[1]);
        tc::mma_bf16_16816(dp[2 * np + 1], av, bd[2], bd[3]);
      }
    }
    // element (key, query i): P^T = exp2(S^T c - lse2_i), P^T mask -> s, dS^T -> dp
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int ci = 8 * j + 2 * (lane & 3) + (e & 1);
        const int i = qb * AB_QB + ci;
        const float pr = fast_ex2(fmaf(s[j][e], p.scale_log2, -st_lse[ci]));
        const float mk = p.drop_thr > 0 ? (drop_keep(p.drop_seed, drow_base + i, key_a + 8 * (e >> 1), p.drop_thr) ? dscale : 0.f) : 1.f;
        dp[j][e] = pr * fmaf(mk, dp[j][e], -st_dl[ci]) * p.scale;
        s[j][e] = pr * mk;
      }
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) {
      uint32_t ap[4], as[4];
      ap[0] = tc::pack_bf16x2(s[2 * kk][0], s[2 * kk][1]);
      ap[1] = tc::pack_bf16x2(s[2 * kk][2], s[2 * kk][3]);
      ap[2] = tc::pack_bf16x2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      ap[3] = tc::pack_bf16x2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
      as[0] = tc::pack_bf16x2(dp[2 * kk][0], dp[2 * kk][1]);
      as[1] = tc::pack_bf16x2(dp[2 * kk][2], dp[2 * kk][3]);
      as[2] = tc::pack_bf16x2(dp[2 * kk + 1][0], dp[2 * kk + 1][1]);
      as[3] = tc::pack_bf16x2(dp[2 * kk + 1][2], dp[2 * kk + 1][3]);
#pragma unroll
      for (int dd = 0; dd < 8; ++dd) {
        uint32_t bd[4], bq[4];
        att_frag_bt(bd, d_s, kk * 16, dd * 16, lane);
        att_frag_bt(bq, q_s, kk * 16, dd * 16, lane);
        tc::mma_bf16_16816(dv[2 * dd], ap, bd[0], bd[1]);
        tc::mma_bf16_16816(dv[2 * dd + 1], ap, bd[2], bd[3]);
        tc::mma_bf16_16816(dk[2 * dd], as, bq[0], bq[1]);
        tc::mma_bf16_16816(dk[2 * dd + 1], as, bq[2], bq[3]);
      }
    }
    __syncthreads();     // this buffer is refilled by the next iteration's loads
  }

#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int key = key_a + 8 * r;
    if (key < p.sep) {
      __nv_bfloat16* grow = p.dqkv + att_tok(key, b, p.T, p.B, p.batch_major) * p.ld_dqkv + h * ATT_DH;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        att_st2(grow + E, j, lane, dk[j][2 * r], dk[j][2 * r + 1]);
        att_st2(grow + 2 * E, j, lane, dv[j][2 * r], dv[j][2 * r + 1]);
      }
    }
  }
}

}  // namespace pfn

using namespace pfn;

extern "C" int pfn_attention_bwd_tc(const pfn_attn_desc* d, void* stream) {
  if (int rc = check_tc_attn(d, true, "attention_bwd_tc")) return rc;
  PFN_CHECK_ARG(!(d->delta_token_major && d->batch_major), "attention_bwd_tc: a token-major delta implies the reference token order");
  AttnBwdParams p;
  p.T = d->T; p.B = d->B; p.H = d->H; p.sep = d->sep;
  p.scale = d->scale; p.scale_log2 = d->scale * 1.4426950408889634f;
  p.qkv = reinterpret_cast<const __nv_bfloat16*>(d->qkv); p.ld_qkv = d->ld_qkv;
  p.dout = reinterpret_cast<const __nv_bfloat16*>(d->dout); p.ld_dout = d->ld_dout;
  p.dqkv = reinterpret_cast<__nv_bfloat16*>(d->dqkv); p.ld_dqkv = d->ld_dqkv;
  p.lse = d->lse; p.delta = d->delta; p.dq_colsum = d->dq_colsum; p.delta_tm = d->delta_token_major;
  p.drop_seed = d->drop_seed; p.drop_thr = d->drop_thr;
  p.batch_major = d->batch_major;
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set)) {
    PFN_CUDA_OK(cudaFuncSetAttribute(attn_bwd_dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AB_DQ_SMEM));
    PFN_CUDA_OK(cudaFuncSetAttribute(attn_bwd_dkv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AB_DKV_SMEM));
  }
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (!d->delta_token_major) {
    const long long rows = static_cast<long long>(d->T) * d->B;
    long long grid = (rows + 7) / 8;
    if (grid > 8LL * num_sms()) grid = 8LL * num_sms();
    attn_bwd_delta_kernel<<<static_cast<int>(grid), 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(d->out), d->ld_out,
                                                                 p.dout, p.ld_dout, d->delta, d->T, d->B, d->H, d->batch_major);
    PFN_LAUNCH_OK();
  }
  p.n_tiles = (d->T + AB_BM - 1) / AB_BM;
  long long grid = static_cast<long long>(p.n_tiles) * d->B * d->H;
  PFN_CHECK_ARG(grid < (1LL << 31), "attention_bwd_tc: too many tiles");
  attn_bwd_dq_kernel<<<static_cast<unsigned>(grid), 128, AB_DQ_SMEM, s>>>(p);
  PFN_LAUNCH_OK();
  if (d->sep > 0) {
    p.n_tiles = (d->sep + AB_BM - 1) / AB_BM;
    grid = static_cast<long long>(p.n_tiles) * d->B * d->H;
    attn_bwd_dkv_kernel<<<static_cast<unsigned>(grid), 128, AB_DKV_SMEM, s>>>(p);
    PFN_LAUNCH_OK();
  }
  return 0;
}
