// Tensor-core backward of the single_eval_pos-masked attention (head dim 128, bf16), three kernels:
//
//  (0) attn_bwd_delta_kernel  delta[b,h,i] = dO_i . O_i   (one warp per token row, HBM-bound, 16 B vectors); skipped when
//      the caller passes the token-major delta the out-projection dgrad's ROWDOT epilogue already produced
//
//  (1) attn_bwd_dq_kernel     persistent: one CTA per SM walks the (batch, head, 128-row query tile) list; per tile, loop
//      over 64-key blocks of the train keys:
//          S_j  = Q K_j^T      dP_j = dO V_j^T                                 (wgmma m64n64k16, fp32)
//          dS_j = exp2(S_j c - lse2) * (dP_j - delta) * scale  -> bf16 A fragments (registers)
//          dQ  += dS_j K_j                                                      (wgmma m64n128k16, A from registers)
//      software-pipelined like the forward: S_j / dP_j and dQ += dS_{j-1} K_{j-1} are issued together and dS_j is computed
//      while the dQ MMAs of block j-1 run.  For a query row (i >= sep) the diagonal key is attended by that row only, so
//      dK_i = dS_ii q_i and dV_i = P_ii dO_i are complete: producer warps 9-11 compute them one tile ahead, together with
//      every row's lse2 and delta, and hand lse2, delta and dS_ii to the consumers through a double-buffered array in
//      shared memory; the consumers add dS_ii k_i to dQ.
//
//  (2) attn_bwd_dkv_kernel    one CTA per (batch, head, 128-key tile of the train keys), K and V resident, loop over 64-row
//      Q/dO blocks:
//          S^T = K Q_i^T       dP^T = V dO_i^T     (row = key, column = query row; m64n64k16)
//          dV += (P^T . mask) dO_i ;   dK += dS^T Q_i                           (m64n128k16, A from registers)
//
// Both are warp-specialised: warpgroup 2 (producer; 64 registers in (1), 40 in (2)) issues the TMA loads into a ring of
// stages, warpgroups 0 and 1 (consumers; 208 registers in (1), 232 in (2)) each own 64 rows of the tile (query rows in
// (1), keys in (2)).  The fp32 S / dP
// accumulators are packed to bf16 in place as the A operand of the second pair of MMAs, so P and dS never touch shared
// memory.  Q/K/V/dO rows come straight out of the packed [T*B, 3E] qkv / [T*B, E] dO buffers through 3-D tensor maps
// (columns, batch, time) whose two row strides encode the token order; the TMA zero-fills rows past T (Q, dO) and keys
// past sep (K, V).  One 128-byte-swizzled tile serves as a K-major operand (S = Q K^T) and as an MN-major one
// (dQ += dS K), so nothing is transposed.  No atomics on dQKV: every element is written exactly once.
#include "attention_common.cuh"

namespace pfn {

constexpr int AB_ROWS = ATT_TILE_ROWS;                    // rows of one consumer warpgroup; key / query block size
constexpr int AB_TILE = ATT_TILE;                         // 16 KB: 64 rows x 128 bf16 = two 8 KB boxes of 64 columns
constexpr int AB_THREADS = 3 * 128;
constexpr int AB_DQ_STAGES = 4;                           // K/V blocks in flight (dQ kernel)
constexpr int AB_DKV_STAGES = 3;                          // Q/dO blocks in flight (dK/dV kernel)
constexpr int AB_DQ_STAT_WARPS = 3;                       // producer warps 9-11: per-row statistics of the next tile
// dQ kernel: Q, dO of the tile (2 x 2 x 16 KB), ring of (K, V), two buffers of per-row (lse2, delta, ds_ii), barriers
constexpr int AB_DQ_OFF_RING = 4 * AB_TILE;
constexpr int AB_DQ_OFF_STAT = AB_DQ_OFF_RING + AB_DQ_STAGES * 2 * AB_TILE;
constexpr int AB_DQ_OFF_BAR = AB_DQ_OFF_STAT + 2 * 3 * 128 * 4;
constexpr int AB_DQ_SMEM = AB_DQ_OFF_BAR + (2 * AB_DQ_STAGES + 2 + 4) * 8 + 1024;   // + 1 KB alignment slack
// dK/dV kernel: K, V of the tile (2 x 2 x 16 KB), ring of (Q, dO), ring of (lse2, delta), barriers
constexpr int AB_DKV_OFF_RING = 4 * AB_TILE;
constexpr int AB_DKV_OFF_STAT = AB_DKV_OFF_RING + AB_DKV_STAGES * 2 * AB_TILE;
constexpr int AB_DKV_OFF_BAR = AB_DKV_OFF_STAT + AB_DKV_STAGES * 2 * AB_ROWS * 4;
constexpr int AB_DKV_SMEM = AB_DKV_OFF_BAR + (2 * AB_DKV_STAGES + 1) * 8 + 1024;
static_assert(AB_DQ_SMEM <= 232448 && AB_DKV_SMEM <= 232448, "the tiles and rings must fit the 227 KB of shared memory");

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
  int n_tiles;           // 128-row tiles per (batch, head): query rows (dQ kernel) or train keys (dK/dV kernel)
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
__global__ void __launch_bounds__(AB_THREADS, 1)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV,
                   const __grid_constant__ CUtensorMap tmDO, const AttnBwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = att_smem_base(smem_raw);
  uint8_t* sQ = smem;                                     // warpgroup g's 64 rows at + g * 16 KB
  uint8_t* sD = smem + 2 * AB_TILE;
  const AttPipe<AB_DQ_STAGES> pp(smem + AB_DQ_OFF_RING, reinterpret_cast<uint64_t*>(smem + AB_DQ_OFF_BAR));
  // tile it's statistics are in buffer it & 1: [0, 128) lse2, [128, 256) delta, [256, 384) ds_ii of the tile's rows
  float* sStat = reinterpret_cast<float*>(smem + AB_DQ_OFF_STAT);
  uint64_t* st_full = pp.q_empty + 1;                     // [2] written by the statistics warps
  uint64_t* st_empty = st_full + 2;                       // [2] read by every consumer thread
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int E = p.H * ATT_DH;
  const int nblk = (p.sep + AB_ROWS - 1) / AB_ROWS;
  const int n_units = p.n_tiles * p.B * p.H;
  const float dscale = p.drop_thr > 0 ? drop_scale(p.drop_thr) : 1.0f;
  if (threadIdx.x == 0) {
    pp.init();
    for (int s = 0; s < 2; ++s) {
      tc::mbar_init(&st_full[s], 32 * AB_DQ_STAT_WARPS);
      tc::mbar_init(&st_empty[s], 256);
    }
    tc::mbar_fence_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // ------------------------------------------------------------------ producer: TMA (thread 256), statistics (warps 9-11)
    // 64 registers: the statistics warps keep two rows in flight (with 40 or 48 they spill), so the consumers get 208:
    // 2 x 128 x 208 + 128 x 64 <= 64 K
    tc::setmaxnreg_dec<64>();
    if (warp > 8) {
      // Per tile: lse2 and delta of its 128 rows, and for each row i >= sep its diagonal key: s_ii = q_i.k_i,
      // dp_ii = dO_i.v_i, ds_ii = P_ii (mask dp_ii - delta_i) scale, which completes dK_i = ds_ii q_i and dV_i = P_ii mask
      // dO_i (stored here) and leaves ds_ii k_i for the consumers' dQ.  Warp pw owns the rows r = pw (mod 3).  A row is
      // read by the whole warp with 16-byte loads: lanes 0-15 take q_i and k_i, lanes 16-31 dO_i and v_i, eight columns
      // each; the two halves then store dK_i and dV_i.  Two rows are in flight at a time.
      const int pw = warp - 9;
      for (int u = blockIdx.x, it = 0; u < n_units; u += gridDim.x, ++it) {
        const AttUnit unit = att_unit(u, p.n_tiles, p.H);
        const int sb = it & 1;
        float* st = sStat + sb * 3 * 128;
        tc::mbar_wait_suspend(&st_empty[sb], ((it >> 1) & 1) ^ 1);
#pragma unroll 1
        for (int r = pw + AB_DQ_STAT_WARPS * lane; r < 128; r += 32 * AB_DQ_STAT_WARPS) {
          const int i = unit.tile * 128 + r;
          const bool valid = i < p.T;
          st[r] = valid ? p.lse[static_cast<size_t>(unit.bh) * p.T + i] * 1.4426950408889634f : INFINITY;
          st[128 + r] = valid ? ab_delta(p, unit.b, unit.h, i) : 0.f;
        }
        __syncwarp();
        // the lane's half and columns come from an opaque lane index in every row, so that the address arithmetic built on
        // them is formed next to its loads instead of being hoisted out of the loops and held in registers throughout
        auto tok_of = [&](int r) { return att_tok(unit.tile * 128 + r, unit.b, p.T, p.B, p.batch_major); };
        auto load_row = [&](int r, uint4& xv, uint4& yv) {
          const int l = static_cast<int>(att_opaque(lane)), half = l >> 4, c8 = (l & 15) * 8;
          const size_t tok = tok_of(r);
          const __nv_bfloat16* qrow = p.qkv + tok * p.ld_qkv + unit.h * ATT_DH + c8;
          xv = *reinterpret_cast<const uint4*>(half ? p.dout + tok * p.ld_dout + unit.h * ATT_DH + c8 : qrow);   // q_i | dO_i
          yv = *reinterpret_cast<const uint4*>(qrow + (1 + half) * E);                                      // k_i | v_i
        };
        auto finish_row = [&](int r, uint4 xv, uint4 yv) {
          const int l = static_cast<int>(att_opaque(lane)), half = l >> 4, c8 = (l & 15) * 8;
          const __nv_bfloat162* x2 = reinterpret_cast<const __nv_bfloat162*>(&xv);
          const __nv_bfloat162* y2 = reinterpret_cast<const __nv_bfloat162*>(&yv);
          float dot = 0.f;
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const float2 a = __bfloat1622float2(x2[c]), bb = __bfloat1622float2(y2[c]);
            dot = fmaf(a.x, bb.x, fmaf(a.y, bb.y, dot));
          }
#pragma unroll
          for (int o = 8; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
          const float sd = __shfl_sync(0xffffffffu, dot, 0), dpd = __shfl_sync(0xffffffffu, dot, 16);
          const int i = unit.tile * 128 + r;
          const float pr = fast_ex2(fmaf(sd, p.scale_log2, -st[r]));
          const float mk = p.drop_thr > 0 ? (drop_keep(p.drop_seed, static_cast<uint32_t>(unit.bh) * p.T + i, i, p.drop_thr) ? dscale : 0.f) : 1.f;
          const float ds = pr * fmaf(mk, dpd, -st[128 + r]) * p.scale;
          const float f = half ? pr * mk : ds;
          uint4 o;
          uint32_t* o32 = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const float2 a = __bfloat1622float2(x2[c]);
            o32[c] = tc::pack_bf16x2(f * a.x, f * a.y);
          }
          *reinterpret_cast<uint4*>(p.dqkv + tok_of(r) * p.ld_dqkv + unit.h * ATT_DH + (1 + half) * E + c8) = o;   // dK_i | dV_i
          if (lane == 0) st[256 + r] = ds;
        };
        const int r_lo = max(0, p.sep - unit.tile * 128), r_hi = min(128, p.T - unit.tile * 128);
        for (int r = r_lo + (pw - r_lo % AB_DQ_STAT_WARPS + AB_DQ_STAT_WARPS) % AB_DQ_STAT_WARPS; r < r_hi;
             r += 2 * AB_DQ_STAT_WARPS) {
          const int r2 = r + AB_DQ_STAT_WARPS < r_hi ? r + AB_DQ_STAT_WARPS : r;
          uint4 xa, ya, xb, yb;
          load_row(r, xa, ya);
          load_row(r2, xb, yb);
          finish_row(r, xa, ya);
          if (r2 != r) finish_row(r2, xb, yb);
        }
        tc::mbar_arrive(&st_full[sb]);
      }
    } else if (threadIdx.x == 256) {
      tc::tma_prefetch_desc(&tmQ);
      tc::tma_prefetch_desc(&tmKV);
      tc::tma_prefetch_desc(&tmDO);
      att_kv_producer(pp, &tmKV, n_units, p.n_tiles, p.H, nblk, 4 * AB_TILE, [&](const AttUnit& unit) {
        for (int g = 0; g < 2; ++g) {
          const int t0 = unit.tile * 128 + 64 * g;
          att_load_tile(sQ + g * AB_TILE, &tmQ, pp.q_full, unit.h * ATT_DH, unit.b, t0);
          att_load_tile(sD + g * AB_TILE, &tmDO, pp.q_full, unit.h * ATT_DH, unit.b, t0);
        }
      });
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroups
  tc::setmaxnreg_inc<208>();
  const int g = warp >> 2, wq = warp & 3;
  const uint32_t q_tile = tc::smem_u32(sQ + g * AB_TILE), d_tile = tc::smem_u32(sD + g * AB_TILE);
  AttRing<AB_DQ_STAGES> ring;
  bool timed_out = false;
  for (int u = blockIdx.x, it = 0; u < n_units && !timed_out; u += gridDim.x, ++it) {
    const AttUnit unit = att_unit(u, p.n_tiles, p.H);
    const int i0 = unit.tile * 128 + 64 * g + 16 * wq + (lane >> 2);    // this lane's rows: i0, i0 + 8

    // per-row statistics of this lane's two rows (and ds_ii of its diagonal keys), prepared by the statistics warps
    const int sb = it & 1;
    if (!tc::mbar_wait_bounded(&st_full[sb], (it >> 1) & 1)) { timed_out = true; break; }
    float lse2[2], dl[2], dsd[2];
    uint32_t drow[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int rr = i0 + 8 * r - unit.tile * 128;
      lse2[r] = sStat[sb * 3 * 128 + rr];
      dl[r] = sStat[sb * 3 * 128 + 128 + rr];
      dsd[r] = sStat[sb * 3 * 128 + 256 + rr];
      drow[r] = static_cast<uint32_t>(unit.bh) * p.T + i0 + 8 * r;
    }
    tc::mbar_arrive(&st_empty[sb]);

    // Key loop (att_key_loop): S_kb = Q K_kb^T and dP_kb = dO V_kb^T as the first MMA group, dS_kb computed while
    // dQ += dS_{kb-1} K_{kb-1} runs, then packed into the A fragments.  The first dQ MMA of the tile writes dq
    // (scale-d = 0), so nothing but wgmma defines it until then.
    float dq[64], s[32], dp[32];
    uint32_t ads[16];
    auto issue_sdp = [&](int st) {
      const uint32_t k_s = tc::smem_u32(pp.ring + st * 2 * AB_TILE);
      const uint32_t v_s = k_s + AB_TILE;
      const uint32_t q_s = att_opaque(q_tile), d_s = att_opaque(d_tile);
      tc::wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) att_mma_n64(s, att_desc_k(q_s, kk), att_desc_k(k_s, kk), kk);
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) att_mma_n64(dp, att_desc_k(d_s, kk), att_desc_k(v_s, kk), kk);
      tc::wgmma_commit();
    };
    auto issue_dq = [&](int st, bool accumulate) {
      const uint32_t k_s = tc::smem_u32(pp.ring + st * 2 * AB_TILE);
      tc::wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) tc::wgmma_m64n128k16_rs(dq, ads + 4 * kk, att_desc_mn(k_s, kk), accumulate || kk > 0);
      tc::wgmma_commit();
    };
    // dS = P (mask dP - delta) scale into s (keys >= sep of the last block get P = 0); element 4 j + e is row
    // i0 + 8 (e >> 1), key kb * 64 + 8 j + 2 (lane & 3) + (e & 1)
    auto compute_ds = [&](int kb) {
      const int key0 = kb * AB_ROWS + 2 * (lane & 3);
#pragma unroll
      for (int e = 0; e < 32; ++e) {
        const int r = (e >> 1) & 1;
        const int key = key0 + 8 * (e >> 2) + (e & 1);
        const float pr = key < p.sep ? fast_ex2(fmaf(s[e], p.scale_log2, -lse2[r])) : 0.f;
        const float mk = p.drop_thr > 0 ? (drop_keep(p.drop_seed, drow[r], key, p.drop_thr) ? dscale : 0.f) : 1.f;
        s[e] = pr * fmaf(mk, dp[e], -dl[r]) * p.scale;
      }
    };
    auto pack_ds = [&]() {
#pragma unroll
      for (int e = 0; e < 16; ++e) ads[e] = tc::pack_bf16x2(s[2 * e], s[2 * e + 1]);
    };
    // k_i of this lane's diagonal keys (rows i >= sep), loaded while the tile's last dQ MMAs run; dq[4 j + 2 r + c] is
    // row i0 + 8 r, column 8 j + 2 (lane & 3) + c
    uint32_t kd[2][16];
    auto load_kd = [&]() {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int i = i0 + 8 * r;
        const bool diag = i < p.T && i >= p.sep;
        const __nv_bfloat16* krow = p.qkv + att_tok(diag ? i : 0, unit.b, p.T, p.B, p.batch_major) * p.ld_qkv + E + unit.h * ATT_DH;
#pragma unroll
        for (int j = 0; j < 16; ++j)
          kd[r][j] = diag ? *reinterpret_cast<const uint32_t*>(krow + 8 * j + 2 * (lane & 3)) : 0u;
      }
    };
    if (att_key_loop(pp, ring, it, nblk, issue_sdp, issue_dq, [&] { tc::wgmma_fence_regs(s); tc::wgmma_fence_regs(dp); },
                     [&] { tc::wgmma_fence_regs(dq); }, compute_ds, pack_ds, load_kd)) {
      timed_out = true;
      break;
    }

    // dQ = dq + ds_ii k_i, stores, column sums over the bf16-rounded values
    float cs[16][2];
#pragma unroll
    for (int j = 0; j < 16; ++j) cs[j][0] = cs[j][1] = 0.f;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int i = i0 + 8 * r;
      if (i < p.T) {
        const bool diag = i >= p.sep;
        __nv_bfloat16* grow = p.dqkv + att_tok(i, unit.b, p.T, p.B, p.batch_major) * p.ld_dqkv + unit.h * ATT_DH;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          float x = nblk > 0 ? dq[4 * j + 2 * r] : 0.f, y = nblk > 0 ? dq[4 * j + 2 * r + 1] : 0.f;
          if (diag) {
            const float2 k = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&kd[r][j]));
            x = fmaf(dsd[r], k.x, x);
            y = fmaf(dsd[r], k.y, y);
          }
          att_st2(grow, j, lane, x, y);
          cs[j][0] += __bfloat162float(__float2bfloat16_rn(x));
          cs[j][1] += __bfloat162float(__float2bfloat16_rn(y));
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
          if (lane < 4) atomicAdd(p.dq_colsum + unit.h * ATT_DH + 8 * j + 2 * lane + e, v);
        }
    }
  }
  if (timed_out) asm volatile("trap;");
}

// =====================================================================================================================
// Kernel 2: dK, dV of the train keys
// =====================================================================================================================
__global__ void __launch_bounds__(AB_THREADS, 1)
attn_bwd_dkv_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV,
                    const __grid_constant__ CUtensorMap tmDO, const AttnBwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = att_smem_base(smem_raw);
  uint8_t* sK = smem;                                     // warpgroup g's 64 keys at + g * 16 KB
  uint8_t* sV = smem + 2 * AB_TILE;
  uint8_t* sRing = smem + AB_DKV_OFF_RING;                // stage s: Q at + 2 s * 16 KB, dO at + (2 s + 1) * 16 KB
  float* sStat = reinterpret_cast<float*>(smem + AB_DKV_OFF_STAT);   // stage s: lse2 at [128 s], delta at [128 s + 64]
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + AB_DKV_OFF_BAR);
  uint64_t* empty = full + AB_DKV_STAGES;
  uint64_t* kv_bar = empty + AB_DKV_STAGES;               // K, V of the tile have landed
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const AttUnit unit = att_unit(blockIdx.x, p.n_tiles, p.H);
  const int E = p.H * ATT_DH;
  const int nqb = (p.T + AB_ROWS - 1) / AB_ROWS;
  if (threadIdx.x == 0) {
    for (int s = 0; s < AB_DKV_STAGES; ++s) {
      tc::mbar_init(&full[s], 1 + AB_ROWS);              // the TMA thread's expect_tx + one arrival per statistics row
      tc::mbar_init(&empty[s], 2);
    }
    tc::mbar_init(kv_bar, 1);
    tc::mbar_fence_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // ------------------------------------------------------------------ producer: TMA (warp 8), lse2 / delta (warps 10, 11)
    tc::setmaxnreg_dec<40>();
    const int pt = threadIdx.x - 256;
    AttRing<AB_DKV_STAGES> ring;
    if (pt == 0) {
      tc::tma_prefetch_desc(&tmQ);
      tc::tma_prefetch_desc(&tmKV);
      tc::tma_prefetch_desc(&tmDO);
      tc::mbar_expect_tx(kv_bar, 4 * AB_TILE);
      for (int g = 0; g < 2; ++g) {
        const int j0 = unit.tile * 128 + 64 * g;
        att_load_tile(sK + g * AB_TILE, &tmKV, kv_bar, E + unit.h * ATT_DH, unit.b, j0);
        att_load_tile(sV + g * AB_TILE, &tmKV, kv_bar, 2 * E + unit.h * ATT_DH, unit.b, j0);
      }
      for (int qb = 0; qb < nqb; ++qb) {
        tc::mbar_wait_suspend(&empty[ring.stage], ring.phase ^ 1);
        uint8_t* dst = sRing + ring.stage * 2 * AB_TILE;
        tc::mbar_expect_tx(&full[ring.stage], 2 * AB_TILE);
        att_load_tile(dst, &tmQ, &full[ring.stage], unit.h * ATT_DH, unit.b, qb * AB_ROWS);
        att_load_tile(dst + AB_TILE, &tmDO, &full[ring.stage], unit.h * ATT_DH, unit.b, qb * AB_ROWS);
        ring.advance();
      }
    } else if (pt >= 64) {
      const int r = pt - 64;
      for (int qb = 0; qb < nqb; ++qb) {
        const int i = qb * AB_ROWS + r;
        const bool valid = i < p.T;
        const float l2 = valid ? p.lse[static_cast<size_t>(unit.bh) * p.T + i] * 1.4426950408889634f : INFINITY;
        const float dl = valid ? ab_delta(p, unit.b, unit.h, i) : 0.f;
        tc::mbar_wait_suspend(&empty[ring.stage], ring.phase ^ 1);
        sStat[ring.stage * 2 * AB_ROWS + r] = l2;
        sStat[ring.stage * 2 * AB_ROWS + AB_ROWS + r] = dl;
        tc::mbar_arrive(&full[ring.stage]);
        ring.advance();
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroups
  tc::setmaxnreg_inc<232>();
  const int g = warp >> 2, wq = warp & 3;
  const int tid = threadIdx.x & 127;
  const uint32_t k_tile = tc::smem_u32(sK + g * AB_TILE), v_tile = tc::smem_u32(sV + g * AB_TILE);
  const float dscale = p.drop_thr > 0 ? drop_scale(p.drop_thr) : 1.0f;
  const int key_a = unit.tile * 128 + 64 * g + 16 * wq + (lane >> 2);   // this lane's keys: key_a, key_a + 8
  const uint32_t drow_base = static_cast<uint32_t>(unit.bh) * p.T;
  tc::mbar_wait(kv_bar, 0);

  // The first MMAs write dk / dv (scale-d = 0), so nothing but wgmma defines them until the loop has drained.
  float dk[64], dv[64];
  AttRing<AB_DKV_STAGES> ring;
  bool timed_out = false;
  for (int qb = 0; qb < nqb; ++qb) {
    if (!tc::mbar_wait_bounded(&full[ring.stage], ring.phase)) { timed_out = true; break; }
    const uint32_t q_s = tc::smem_u32(sRing + ring.stage * 2 * AB_TILE);
    const uint32_t d_s = q_s + AB_TILE;
    const uint32_t k_s = att_opaque(k_tile), v_s = att_opaque(v_tile);
    const float* st_lse = sStat + ring.stage * 2 * AB_ROWS;
    const float* st_dl = st_lse + AB_ROWS;
    float s[32], dp[32];
    tc::wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) att_mma_n64(s, att_desc_k(k_s, kk), att_desc_k(q_s, kk), kk);
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) att_mma_n64(dp, att_desc_k(v_s, kk), att_desc_k(d_s, kk), kk);
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    tc::wgmma_fence_regs(s);
    tc::wgmma_fence_regs(dp);

    // element 4 j + e is (key key_a + 8 (e >> 1), query row qb * 64 + 8 j + 2 (lane & 3) + (e & 1)).  Per 16 query rows
    // kk: P^T . mask -> ap, dS^T -> as, then dV += ap dO and dK += as Q for those rows, so the MMAs of one slice run while
    // the next is computed and the A fragments take the registers that S^T and dP^T free.
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t ap[4], as[4];
#pragma unroll
      for (int jj = 0; jj < 2; ++jj)
#pragma unroll
        for (int e = 0; e < 4; e += 2) {
          const int j = 2 * kk + jj;
          float pm[2], ds[2];
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int ci = 8 * j + 2 * (lane & 3) + c;
            const int i = qb * AB_ROWS + ci;
            const float pr = fast_ex2(fmaf(s[4 * j + e + c], p.scale_log2, -st_lse[ci]));
            const float mk = p.drop_thr > 0 ? (drop_keep(p.drop_seed, drow_base + i, key_a + 8 * (e >> 1), p.drop_thr) ? dscale : 0.f) : 1.f;
            ds[c] = pr * fmaf(mk, dp[4 * j + e + c], -st_dl[ci]) * p.scale;
            pm[c] = pr * mk;
          }
          ap[2 * jj + (e >> 1)] = tc::pack_bf16x2(pm[0], pm[1]);
          as[2 * jj + (e >> 1)] = tc::pack_bf16x2(ds[0], ds[1]);
        }
      tc::wgmma_fence();
      tc::wgmma_m64n128k16_rs(dv, ap, att_desc_mn(d_s, kk), qb > 0 || kk > 0);
      tc::wgmma_m64n128k16_rs(dk, as, att_desc_mn(q_s, kk), qb > 0 || kk > 0);
    }
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    if (tid == 0) tc::mbar_arrive(&empty[ring.stage]);
    ring.advance();
  }
  tc::wgmma_fence_regs(dk);
  tc::wgmma_fence_regs(dv);

  // dk[4 j + 2 r + c] is key key_a + 8 r, column 8 j + 2 (lane & 3) + c
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int key = key_a + 8 * r;
    if (key < p.sep) {
      __nv_bfloat16* grow = p.dqkv + att_tok(key, unit.b, p.T, p.B, p.batch_major) * p.ld_dqkv + unit.h * ATT_DH;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        att_st2(grow + E, j, lane, dk[4 * j + 2 * r], dk[4 * j + 2 * r + 1]);
        att_st2(grow + 2 * E, j, lane, dv[4 * j + 2 * r], dv[4 * j + 2 * r + 1]);
      }
    }
  }
  if (timed_out) asm volatile("trap;");
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
  const int E = d->H * ATT_DH;
  CUtensorMap tmQ, tmKV, tmDO;
  if (int rc = att_qkv_maps(d, &tmQ, &tmKV)) return rc;
  if (int rc = att_tensor_map(&tmDO, d->dout, E, d->ld_dout, d->T, d->B, d->T, d->batch_major)) return rc;
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set))
    PFN_CUDA_OK(cudaFuncSetAttribute(attn_bwd_dkv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AB_DKV_SMEM));
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (!d->delta_token_major) {
    const long long rows = static_cast<long long>(d->T) * d->B;
    long long grid = (rows + 7) / 8;
    if (grid > 8LL * num_sms()) grid = 8LL * num_sms();
    attn_bwd_delta_kernel<<<static_cast<int>(grid), 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(d->out), d->ld_out,
                                                                 p.dout, p.ld_dout, d->delta, d->T, d->B, d->H, d->batch_major);
    PFN_LAUNCH_OK();
  }
  p.n_tiles = (d->T + 127) / 128;
  if (int rc = att_launch_persistent<attn_bwd_dq_kernel>("attention_bwd_tc", static_cast<long long>(p.n_tiles) * d->B * d->H,
                                                         AB_THREADS, AB_DQ_SMEM, s, tmQ, tmKV, tmDO, p))
    return rc;
  if (d->sep > 0) {
    p.n_tiles = (d->sep + 127) / 128;
    const long long grid = static_cast<long long>(p.n_tiles) * d->B * d->H;
    attn_bwd_dkv_kernel<<<static_cast<unsigned>(grid), AB_THREADS, AB_DKV_SMEM, s>>>(tmQ, tmKV, tmDO, p);
    PFN_LAUNCH_OK();
  }
  return 0;
}
