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
//      shared memory; the consumers add dS_ii k_i to dQ, which leaves through a staging tile and TMA stores.
//
//  (2) attn_bwd_dkv_kernel    persistent: one CTA per SM walks the (batch, head, 128-key tile of the train keys) list,
//      key tile fastest; per tile K and V resident, loop over 64-row Q/dO blocks:
//          S^T = K Q_i^T       dP^T = V dO_i^T     (row = key, column = query row; m64n64k16)
//          dV += (P^T . mask) dO_i ;   dK += dS^T Q_i                           (m64n128k16, A from registers)
//      K/V are double-buffered across tiles, so the next tile's land while the current one runs; dK and dV are staged in
//      the tile's own K/V buffer once its last MMAs are done and leave by TMA stores clipped at sep.
//
// Both are warp-specialised: warpgroup 2 (producer; 64 registers in (1), 40 in (2)) issues the TMA loads into a ring of
// stages, warpgroups 0 and 1 (consumers; 208 registers in (1), 232 in (2)) each own 64 rows of the tile (query rows in
// (1), keys in (2)).  The fp32 S / dP
// accumulators are packed to bf16 in place as the A operand of the second pair of MMAs, so P and dS never touch shared
// memory.  Q/K/V/dO rows come straight out of the packed [T*B, 3E] qkv / [T*B, E] dO buffers through 3-D tensor maps
// (columns, batch, time) whose two row strides encode the token order; the TMA zero-fills rows past T (Q, dO) and keys
// past sep (K, V).  One 128-byte-swizzled tile serves as a K-major operand (S = Q K^T) and as an MN-major one
// (dQ += dS K), so nothing is transposed.  No atomics on dQKV: every element is written exactly once.
//
// Ragged datasets (kRagged, pfn_attention_ragged_train_bwd_tc): dataset b has its own separator s_b = n_keys[b] <= sep.
// In the dQ kernel a unit runs ceil(s_b / 64) key blocks, masks keys >= s_b in its last one, and rows i >= s_b have their
// diagonal key.  In the dK/dV kernel the key tiles at or past s_b have no work and are skipped by every role of the CTA
// alike; a warpgroup whose 64 keys straddle s_b stores its rows < s_b directly instead of by the TMA, whose map clips
// at sep only.  The keys [s_b, sep) are real rows of qkv, loaded and masked like the keys past sep.
//
// Context attention (kCtx, pfn_attention_ctx_bwd_tc): the dQ kernel alone, on the operands of the context forward.  Q and
// dO are the query rows' [m*B, 3E] qkv and [m*B, E] dO (T = m), the key blocks come from the [n*B, 2E] K/V cache through
// its own map (sep = n, or n_keys[b] when ragged), and every row has its diagonal key.  The cached keys are constants, so
// no dK/dV kernel runs: dqkv receives dQ and the dK_i, dV_i of each row's own key.
#include "attention_common.cuh"

namespace pfn {

constexpr int AB_ROWS = ATT_TILE_ROWS;                    // rows of one consumer warpgroup; key / query block size
constexpr int AB_TILE = ATT_TILE;                         // 16 KB: 64 rows x 128 bf16 = two 8 KB boxes of 64 columns
constexpr int AB_THREADS = 3 * 128;
constexpr int AB_DQ_STAGES = 3;                           // K/V blocks in flight (dQ kernel)
constexpr int AB_DKV_STAGES = 3;                          // Q/dO blocks in flight (dK/dV kernel)
constexpr int AB_DQ_STAT_WARPS = 3;                       // producer warps 9-11: per-row statistics of the next tile
constexpr int AB_DQ_ROW_SLOTS = 8;                        // diagonal rows in flight per statistics warp
constexpr int AB_DQ_ROW_SLOT = 1024;                      // one row's q_i | dO_i (512 B), then k_i | v_i (512 B)
// dQ kernel: Q, dO of the tile (2 x 2 x 16 KB), ring of (K, V), the dQ staging tile (2 x 16 KB), two buffers of
// per-row (lse2, delta, ds_ii), the statistics warps' rings of diagonal rows, barriers
constexpr int AB_DQ_OFF_RING = 4 * AB_TILE;
constexpr int AB_DQ_OFF_OUT = AB_DQ_OFF_RING + AB_DQ_STAGES * 2 * AB_TILE;
constexpr int AB_DQ_OFF_STAT = AB_DQ_OFF_OUT + 2 * AB_TILE;
constexpr int AB_DQ_OFF_ROWS = AB_DQ_OFF_STAT + 2 * 3 * 128 * 4;
constexpr int AB_DQ_OFF_BAR = AB_DQ_OFF_ROWS + AB_DQ_STAT_WARPS * AB_DQ_ROW_SLOTS * AB_DQ_ROW_SLOT;
constexpr int AB_DQ_SMEM = AB_DQ_OFF_BAR + (2 * AB_DQ_STAGES + 2 + 4) * 8 + 1024;   // + 1 KB alignment slack
// dK/dV kernel: two buffers of the tile's K, V (2 x 2 x 2 x 16 KB), ring of (Q, dO), ring of (lse2, delta), barriers
constexpr int AB_DKV_KV = 4 * AB_TILE;
constexpr int AB_DKV_OFF_RING = 2 * AB_DKV_KV;
constexpr int AB_DKV_OFF_STAT = AB_DKV_OFF_RING + AB_DKV_STAGES * 2 * AB_TILE;
constexpr int AB_DKV_OFF_BAR = AB_DKV_OFF_STAT + AB_DKV_STAGES * 2 * AB_ROWS * 4;
constexpr int AB_DKV_SMEM = AB_DKV_OFF_BAR + (2 * AB_DKV_STAGES + 4) * 8 + 1024;
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
  const int* n_keys;     // [B] per-dataset separators (kRagged only)
};

// the separator of dataset b: sep, or n_keys[b] clamped to [0, sep] in the ragged kernels
template <bool kRagged>
__device__ __forceinline__ int ab_sep(const AttnBwdParams& p, int b) {
  return kRagged ? min(max(__ldg(p.n_keys + b), 0), p.sep) : p.sep;
}

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
template <bool kCtx, bool kRagged>
__global__ void __launch_bounds__(AB_THREADS, 1)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV,
                   const __grid_constant__ CUtensorMap tmDO, const __grid_constant__ CUtensorMap tmDQ,
                   const AttnBwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = att_smem_base(smem_raw);
  uint8_t* sQ = smem;                                     // warpgroup g's 64 rows at + g * 16 KB
  uint8_t* sD = smem + 2 * AB_TILE;
  uint8_t* sOut = smem + AB_DQ_OFF_OUT;                   // warpgroup g's 64 rows of dQ at + g * 16 KB
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
    // 64 registers for the statistics warps' row arithmetic, so the consumers get 208: 2 x 128 x 208 + 128 x 64 <= 64 K
    tc::setmaxnreg_dec<64>();
    if (warp > 8) {
      // Per tile: lse2 and delta of its 128 rows, and for each row i >= sep its diagonal key: s_ii = q_i.k_i,
      // dp_ii = dO_i.v_i, ds_ii = P_ii (mask dp_ii - delta_i) scale, which completes dK_i = ds_ii q_i and dV_i = P_ii mask
      // dO_i (stored here) and leaves ds_ii k_i for the consumers' dQ.  Warp pw owns the rows r = pw (mod 3).  A row is
      // read by the whole warp in 16-byte pieces: lanes 0-15 take q_i and k_i, lanes 16-31 dO_i and v_i, eight columns
      // each; the two halves then store dK_i and dV_i.  The pieces come through the warp's ring of AB_DQ_ROW_SLOTS rows
      // in shared memory (cp.async, one commit group per row), so that many rows are in flight while one is finished.
      // A lane reads back only the bytes its own copies wrote, so its cp.async wait is all the synchronisation needed.
      const int pw = warp - 9;
      uint8_t* lane_rows = smem + AB_DQ_OFF_ROWS + pw * AB_DQ_ROW_SLOTS * AB_DQ_ROW_SLOT + 16 * lane;
      for (int u = blockIdx.x, it = 0; u < n_units; u += gridDim.x, ++it) {
        const AttUnit unit = att_unit(u, p.n_tiles, p.H);
        const int sb = it & 1;
        float* st = sStat + sb * 3 * 128;
        // the warp's diagonal rows of the tile: row k is r0 + 3 k, k < n_rows, in slot k % AB_DQ_ROW_SLOTS
        const int r_lo = kCtx ? 0 : max(0, ab_sep<kRagged>(p, unit.b) - unit.tile * 128), r_hi = min(128, p.T - unit.tile * 128);
        const int r0 = r_lo + (pw - r_lo % AB_DQ_STAT_WARPS + AB_DQ_STAT_WARPS) % AB_DQ_STAT_WARPS;
        const int n_rows = r0 < r_hi ? (r_hi - r0 + AB_DQ_STAT_WARPS - 1) / AB_DQ_STAT_WARPS : 0;
        // the lane's half and columns come from an opaque lane index in every row, so that the address arithmetic built on
        // them is formed next to its copies instead of being hoisted out of the loops and held in registers throughout
        auto tok_of = [&](int r) { return att_tok(unit.tile * 128 + r, unit.b, p.T, p.B, p.batch_major); };
        // one commit group per row, empty past the last, so that the wait before row k is always for row k
        auto issue_row = [&](int k) {
          if (k < n_rows) {
            const int l = static_cast<int>(att_opaque(lane)), half = l >> 4, c8 = (l & 15) * 8;
            const size_t tok = tok_of(r0 + AB_DQ_STAT_WARPS * k);
            const __nv_bfloat16* qrow = p.qkv + tok * p.ld_qkv + unit.h * ATT_DH + c8;
            uint8_t* slot = lane_rows + (k % AB_DQ_ROW_SLOTS) * AB_DQ_ROW_SLOT;
            tc::cp_async16(slot, half ? p.dout + tok * p.ld_dout + unit.h * ATT_DH + c8 : qrow);   // q_i | dO_i
            tc::cp_async16(slot + AB_DQ_ROW_SLOT / 2, qrow + (1 + half) * E);                      // k_i | v_i
          }
          tc::cp_async_commit();
        };
        // the first rows are in flight while the consumers free the statistics buffer and lse2 / delta are read
        for (int k = 0; k < AB_DQ_ROW_SLOTS; ++k) issue_row(k);
        tc::mbar_wait_suspend(&st_empty[sb], ((it >> 1) & 1) ^ 1);
#pragma unroll 1
        for (int r = pw + AB_DQ_STAT_WARPS * lane; r < 128; r += 32 * AB_DQ_STAT_WARPS) {
          const int i = unit.tile * 128 + r;
          const bool valid = i < p.T;
          st[r] = valid ? p.lse[static_cast<size_t>(unit.bh) * p.T + i] * 1.4426950408889634f : INFINITY;
          st[128 + r] = valid ? ab_delta(p, unit.b, unit.h, i) : 0.f;
        }
        __syncwarp();
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
#pragma unroll 1
        for (int k = 0; k < n_rows; ++k) {
          tc::cp_async_wait<AB_DQ_ROW_SLOTS - 1>();
          const uint8_t* slot = lane_rows + (k % AB_DQ_ROW_SLOTS) * AB_DQ_ROW_SLOT;
          const uint4 xv = *reinterpret_cast<const uint4*>(slot), yv = *reinterpret_cast<const uint4*>(slot + AB_DQ_ROW_SLOT / 2);
          finish_row(r0 + AB_DQ_STAT_WARPS * k, xv, yv);
          issue_row(k + AB_DQ_ROW_SLOTS);       // refills the slot just read: finish_row has consumed its values
        }
        tc::mbar_arrive(&st_full[sb]);
      }
    } else if (threadIdx.x == 256) {
      tc::tma_prefetch_desc(&tmQ);
      tc::tma_prefetch_desc(&tmKV);
      tc::tma_prefetch_desc(&tmDO);
      tc::tma_prefetch_desc(&tmDQ);
      auto nblk_of = [&](const AttUnit& unit) { return kRagged ? (ab_sep<true>(p, unit.b) + AB_ROWS - 1) / AB_ROWS : nblk; };
      att_kv_producer(pp, &tmKV, n_units, p.n_tiles, p.H, nblk_of, kCtx ? 0 : E, kCtx ? E : 2 * E, 4 * AB_TILE,
                      [&](const AttUnit& unit) {
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
  const int tid = threadIdx.x & 127;
  const uint32_t q_tile = tc::smem_u32(sQ + g * AB_TILE), d_tile = tc::smem_u32(sD + g * AB_TILE);
  uint8_t* out_tile = sOut + g * AB_TILE;
  AttRing<AB_DQ_STAGES> ring;
  bool timed_out = false;
  for (int u = blockIdx.x, it = 0; u < n_units && !timed_out; u += gridDim.x, ++it) {
    const AttUnit unit = att_unit(u, p.n_tiles, p.H);
    const int i0 = unit.tile * 128 + 64 * g + 16 * wq + (lane >> 2);    // this lane's rows: i0, i0 + 8
    const int sep = ab_sep<kRagged>(p, unit.b);
    const int unit_nblk = kRagged ? (sep + AB_ROWS - 1) / AB_ROWS : nblk;

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
        const float pr = key < sep ? fast_ex2(fmaf(s[e], p.scale_log2, -lse2[r])) : 0.f;
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
        const bool diag = i < p.T && (kCtx || i >= sep);
        const __nv_bfloat16* krow = p.qkv + att_tok(diag ? i : 0, unit.b, p.T, p.B, p.batch_major) * p.ld_qkv + E + unit.h * ATT_DH;
#pragma unroll
        for (int j = 0; j < 16; ++j)
          kd[r][j] = diag ? *reinterpret_cast<const uint32_t*>(krow + 8 * j + 2 * (lane & 3)) : 0u;
      }
    };
    if (att_key_loop(pp, ring, it, unit_nblk, issue_sdp, issue_dq, [&] { tc::wgmma_fence_regs(s); tc::wgmma_fence_regs(dp); },
                     [&] { tc::wgmma_fence_regs(dq); }, compute_ds, pack_ds, load_kd)) {
      timed_out = true;
      break;
    }

    // dQ = dq + ds_ii k_i, staged in the warpgroup's dQ tile (once the TMA has read the previous tile's out of it) and
    // stored by the TMA, which drops the rows >= T; the column sums are read back from the staged tile
    if (tid == 0) tc::bulk_wait_read<0>();
    tc::named_bar_sync(1 + g, 128);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int i = i0 + 8 * r;
      if (i < p.T) {
        const bool diag = kCtx || i >= sep;
        const int lr = 16 * wq + (lane >> 2) + 8 * r;              // row i in the warpgroup's 64
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          float x = unit_nblk > 0 ? dq[4 * j + 2 * r] : 0.f, y = unit_nblk > 0 ? dq[4 * j + 2 * r + 1] : 0.f;
          if (diag) {
            const float2 k = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&kd[r][j]));
            x = fmaf(dsd[r], k.x, x);
            y = fmaf(dsd[r], k.y, y);
          }
          *reinterpret_cast<uint32_t*>(out_tile + att_tile_off2(lr, j, lane)) = tc::pack_bf16x2(x, y);
        }
      }
    }
    tc::fence_proxy_async_smem();
    tc::named_bar_sync(1 + g, 128);
    if (tid == 0 && unit.tile * 128 + 64 * g < p.T) {
      att_store_tile(&tmDQ, out_tile, unit.h * ATT_DH, unit.b, unit.tile * 128 + 64 * g);
      tc::bulk_commit();
    }
    const int rows = min(64, p.T - (unit.tile * 128 + 64 * g));
    if (p.dq_colsum != nullptr && rows > 0) {
      // thread tid sums column tid of the warpgroup's staged rows < T (the bf16 values as stored): one atomic per column
      const uint8_t* col = out_tile + (tid >> 6) * 8192 + 2 * (tid & 7);
      float v = 0.f;
#pragma unroll 8
      for (int r = 0; r < rows; ++r)
        v += __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(col + r * 128 + ((((tid & 63) >> 3) ^ (r & 7)) << 4)));
      atomicAdd(p.dq_colsum + unit.h * ATT_DH + tid, v);
    }
  }
  if (tid == 0) tc::bulk_wait<0>();
  if (timed_out) asm volatile("trap;");
}

// =====================================================================================================================
// Kernel 2: dK, dV of the train keys
// =====================================================================================================================
template <bool kRagged>
__global__ void __launch_bounds__(AB_THREADS, 1)
attn_bwd_dkv_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV,
                    const __grid_constant__ CUtensorMap tmDO, const __grid_constant__ CUtensorMap tmDKV,
                    const AttnBwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = att_smem_base(smem_raw);
  // the CTA's it-th tile uses K/V buffer it & 1: warpgroup g's 64 keys of K at + g * 16 KB, of V at + (2 + g) * 16 KB
  uint8_t* sRing = smem + AB_DKV_OFF_RING;                // stage s: Q at + 2 s * 16 KB, dO at + (2 s + 1) * 16 KB
  float* sStat = reinterpret_cast<float*>(smem + AB_DKV_OFF_STAT);   // stage s: lse2 at [128 s], delta at [128 s + 64]
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + AB_DKV_OFF_BAR);
  uint64_t* empty = full + AB_DKV_STAGES;
  uint64_t* kv_full = empty + AB_DKV_STAGES;              // [2] K, V of the buffer's tile have landed
  uint64_t* kv_empty = kv_full + 2;                       // [2] both warpgroups' dK/dV stores have read the buffer
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int E = p.H * ATT_DH;
  const int nqb = (p.T + AB_ROWS - 1) / AB_ROWS;
  const int n_units = p.n_tiles * p.B * p.H;
  // Ragged: a live unit costs the same nqb query blocks whatever its dataset, so what balances the CTAs is how many live
  // units each meets.  With the key tile fastest, a CTA's stride through the list meets only the tiles u % n_tiles takes
  // on its residues, and the high tiles are the ones most often dead.  The tiles of every odd (batch, head) therefore run
  // in reverse order, so that a CTA meets tile t and tile n_tiles - 1 - t alike; the tiles of one (batch, head) stay
  // neighbours, so the CTAs that run them at the same time still share its Q and dO in L2.
  auto unit_of = [&](int u) {
    AttUnit unit = att_unit(u, p.n_tiles, p.H);
    if (kRagged && (unit.bh & 1)) unit.tile = p.n_tiles - 1 - unit.tile;
    return unit;
  };
  // the CTA's first unit at or after u that has keys below its dataset's separator (every unit when uniform)
  auto live = [&](int u) {
    if (kRagged)
      for (; u < n_units; u += gridDim.x) {
        const AttUnit unit = unit_of(u);
        if (unit.tile * 128 < ab_sep<true>(p, unit.b)) break;
      }
    return u;
  };
  if (threadIdx.x == 0) {
    for (int s = 0; s < AB_DKV_STAGES; ++s) {
      tc::mbar_init(&full[s], 1 + AB_ROWS);              // the TMA thread's expect_tx + one arrival per statistics row
      tc::mbar_init(&empty[s], 2);
    }
    for (int s = 0; s < 2; ++s) {
      tc::mbar_init(&kv_full[s], 1);
      tc::mbar_init(&kv_empty[s], 2);
    }
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
      tc::tma_prefetch_desc(&tmDKV);
      // K and V of unit u, the CTA's j-th, into buffer j & 1 once the stores of tile j - 2 have read it
      auto load_kv = [&](int u, int j) {
        const AttUnit unit = unit_of(u);
        uint8_t* kv = smem + (j & 1) * AB_DKV_KV;
        tc::mbar_wait_suspend(&kv_empty[j & 1], ((j >> 1) & 1) ^ 1);
        tc::mbar_expect_tx(&kv_full[j & 1], 4 * AB_TILE);
        for (int g = 0; g < 2; ++g) {
          const int j0 = unit.tile * 128 + 64 * g;
          att_load_tile(kv + g * AB_TILE, &tmKV, &kv_full[j & 1], E + unit.h * ATT_DH, unit.b, j0);
          att_load_tile(kv + (2 + g) * AB_TILE, &tmKV, &kv_full[j & 1], 2 * E + unit.h * ATT_DH, unit.b, j0);
        }
      };
      const int first = live(blockIdx.x);
      if (!kRagged || first < n_units) load_kv(first, 0);     // a uniform grid has a unit for every CTA
      // the next tile's K/V go in after the Q/dO of block claim_at, so that the wait for the buffer (released under the
      // current tile's first block) leaves the consumers a block in hand; never before block 0, whose MMAs release it
      const int claim_at = min(1, nqb - 1);
      for (int u = first, it = 0; u < n_units; ++it) {
        const AttUnit unit = unit_of(u);
        const int next = live(u + gridDim.x);
        for (int qb = 0; qb < nqb; ++qb) {
          tc::mbar_wait_suspend(&empty[ring.stage], ring.phase ^ 1);
          uint8_t* dst = sRing + ring.stage * 2 * AB_TILE;
          tc::mbar_expect_tx(&full[ring.stage], 2 * AB_TILE);
          att_load_tile(dst, &tmQ, &full[ring.stage], unit.h * ATT_DH, unit.b, qb * AB_ROWS);
          att_load_tile(dst + AB_TILE, &tmDO, &full[ring.stage], unit.h * ATT_DH, unit.b, qb * AB_ROWS);
          ring.advance();
          if (qb == claim_at && next < n_units) load_kv(next, it + 1);
        }
        u = next;
      }
    } else if (pt >= 64) {
      const int r = pt - 64;
      for (int u = live(blockIdx.x); u < n_units; u = live(u + gridDim.x)) {
        const AttUnit unit = unit_of(u);
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
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroups
  tc::setmaxnreg_inc<232>();
  const int g = warp >> 2, wq = warp & 3;
  const int tid = threadIdx.x & 127;
  const float dscale = p.drop_thr > 0 ? drop_scale(p.drop_thr) : 1.0f;

  // The first MMAs of a tile write dk / dv (scale-d = 0), so nothing but wgmma defines them until its loop has drained.
  float dk[64], dv[64];
  AttRing<AB_DKV_STAGES> ring;
  bool timed_out = false;
  for (int u = live(blockIdx.x), it = 0; u < n_units && !timed_out; u = live(u + gridDim.x), ++it) {
    const AttUnit unit = unit_of(u);
    uint8_t* k_buf = smem + (it & 1) * AB_DKV_KV + g * AB_TILE;
    uint8_t* v_buf = k_buf + 2 * AB_TILE;
    const uint32_t k_tile = tc::smem_u32(k_buf), v_tile = tc::smem_u32(v_buf);
    const int key_a = unit.tile * 128 + 64 * g + 16 * wq + (lane >> 2);   // this lane's keys: key_a, key_a + 8
    const uint32_t drow_base = static_cast<uint32_t>(unit.bh) * p.T;
    if (!tc::mbar_wait_bounded(&kv_full[it & 1], (it >> 1) & 1)) { timed_out = true; break; }
    // ragged: a warpgroup whose 64 keys all lie at or past the separator has nothing to store; it only passes the
    // query blocks on (its arrivals keep the barrier counts of the uniform kernel)
    const bool idle = kRagged && unit.tile * 128 + 64 * g >= ab_sep<kRagged>(p, unit.b);

    for (int qb = 0; qb < nqb; ++qb) {
      if (!tc::mbar_wait_bounded(&full[ring.stage], ring.phase)) { timed_out = true; break; }
      if (idle) {
        if (qb == 0 && it > 0 && tid == 0) {
          tc::bulk_wait_read<0>();
          tc::mbar_arrive(&kv_empty[(it - 1) & 1]);
        }
        if (tid == 0) tc::mbar_arrive(&empty[ring.stage]);
        ring.advance();
        continue;
      }
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
      // the previous tile's dK/dV stores have read its buffer by now (or shortly): release it to the producer
      if (qb == 0 && it > 0 && tid == 0) {
        tc::bulk_wait_read<0>();
        tc::mbar_arrive(&kv_empty[(it - 1) & 1]);
      }

      // element 4 j + e is (key key_a + 8 (e >> 1), query row qb * 64 + 8 j + 2 (lane & 3) + (e & 1)).  Per 16 query
      // rows kk: P^T . mask -> ap, dS^T -> as, then dV += ap dO and dK += as Q for those rows, so the MMAs of one slice
      // run while the next is computed and the A fragments take the registers that S^T and dP^T free.
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
    if (timed_out) break;

    // The warpgroup's K and V tiles are free (its last MMAs that read them have completed): dK and dV go there in the
    // layout the TMA reads (128-byte swizzle: the 16-byte chunk index of a 128-byte row is XORed with row & 7), then
    // leave by TMA stores that drop the keys >= sep.  dk[4 j + 2 r + c] is key row 16 wq + (lane >> 2) + 8 r of the
    // warpgroup's 64, column 8 j + 2 (lane & 3) + c.
    const int j0 = unit.tile * 128 + 64 * g;
    if (kRagged) {
      const int sep = ab_sep<true>(p, unit.b);
      if (j0 + AB_ROWS > sep) {
        // the keys >= sep of this dataset are its own rows (their dK, dV came from the dQ kernel): only the keys < sep
        // are stored, one accumulator pair at a time
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int key = j0 + 16 * wq + (lane >> 2) + 8 * r;
          if (key < sep) {
            __nv_bfloat16* row = p.dqkv + att_tok(key, unit.b, p.T, p.B, p.batch_major) * p.ld_dqkv + E + unit.h * ATT_DH +
                                 2 * (lane & 3);
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              *reinterpret_cast<uint32_t*>(row + 8 * j) = tc::pack_bf16x2(dk[4 * j + 2 * r], dk[4 * j + 2 * r + 1]);
              *reinterpret_cast<uint32_t*>(row + E + 8 * j) = tc::pack_bf16x2(dv[4 * j + 2 * r], dv[4 * j + 2 * r + 1]);
            }
          }
        }
        continue;
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int lr = 16 * wq + (lane >> 2) + 8 * r;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int off = att_tile_off2(lr, j, lane);
        *reinterpret_cast<uint32_t*>(k_buf + off) = tc::pack_bf16x2(dk[4 * j + 2 * r], dk[4 * j + 2 * r + 1]);
        *reinterpret_cast<uint32_t*>(v_buf + off) = tc::pack_bf16x2(dv[4 * j + 2 * r], dv[4 * j + 2 * r + 1]);
      }
    }
    tc::fence_proxy_async_smem();
    tc::named_bar_sync(1 + g, 128);
    if (tid == 0 && j0 < p.sep) {
      att_store_tile(&tmDKV, k_buf, E + unit.h * ATT_DH, unit.b, j0);
      att_store_tile(&tmDKV, v_buf, 2 * E + unit.h * ATT_DH, unit.b, j0);
      tc::bulk_commit();
    }
  }
  if (tid == 0) tc::bulk_wait<0>();
  if (timed_out) asm volatile("trap;");
}

// The backward over d with separator n_keys[b] for dataset b when kRagged
template <bool kRagged>
static int launch_attn_bwd_tc(const pfn_attn_desc* d, const int* n_keys, cudaStream_t s, const char* who) {
  if (int rc = check_tc_attn(d, true, who)) return rc;
  PFN_CHECK_ARG(!(d->delta_token_major && d->batch_major), "%s: a token-major delta implies the reference token order", who);
  AttnBwdParams p;
  p.T = d->T; p.B = d->B; p.H = d->H; p.sep = d->sep;
  p.scale = d->scale; p.scale_log2 = d->scale * 1.4426950408889634f;
  p.qkv = reinterpret_cast<const __nv_bfloat16*>(d->qkv); p.ld_qkv = d->ld_qkv;
  p.dout = reinterpret_cast<const __nv_bfloat16*>(d->dout); p.ld_dout = d->ld_dout;
  p.dqkv = reinterpret_cast<__nv_bfloat16*>(d->dqkv); p.ld_dqkv = d->ld_dqkv;
  p.lse = d->lse; p.delta = d->delta; p.dq_colsum = d->dq_colsum; p.delta_tm = d->delta_token_major;
  p.drop_seed = d->drop_seed; p.drop_thr = d->drop_thr;
  p.batch_major = d->batch_major;
  p.n_keys = n_keys;
  const int E = d->H * ATT_DH;
  CUtensorMap tmQ, tmKV, tmDO, tmDQ;
  if (int rc = att_qkv_maps(d, &tmQ, &tmKV)) return rc;
  if (int rc = att_tensor_map(&tmDO, d->dout, E, d->ld_dout, d->T, d->B, d->T, d->batch_major)) return rc;
  if (int rc = att_tensor_map(&tmDQ, d->dqkv, 3 * E, d->ld_dqkv, d->T, d->B, d->T, d->batch_major)) return rc;
  if (!d->delta_token_major) {
    const long long rows = static_cast<long long>(d->T) * d->B;
    long long grid = (rows + 7) / 8;
    if (grid > 8LL * num_sms()) grid = 8LL * num_sms();
    attn_bwd_delta_kernel<<<static_cast<int>(grid), 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(d->out), d->ld_out,
                                                                 p.dout, p.ld_dout, d->delta, d->T, d->B, d->H, d->batch_major);
    PFN_LAUNCH_OK();
  }
  p.n_tiles = (d->T + 127) / 128;
  if (int rc = att_launch_persistent<attn_bwd_dq_kernel<false, kRagged>>(who, static_cast<long long>(p.n_tiles) * d->B * d->H,
                                                                         AB_THREADS, AB_DQ_SMEM, s, tmQ, tmKV, tmDO, tmDQ, p))
    return rc;
  if (d->sep > 0) {
    // dK/dV of the train keys, stored through a map whose t extent of sep drops the keys >= sep of the last tile
    CUtensorMap tmDKV;
    if (int rc = att_tensor_map(&tmDKV, d->dqkv, 3 * E, d->ld_dqkv, d->T, d->B, d->sep, d->batch_major)) return rc;
    p.n_tiles = (d->sep + 127) / 128;
    if (int rc = att_launch_persistent<attn_bwd_dkv_kernel<kRagged>>(who, static_cast<long long>(p.n_tiles) * d->B * d->H,
                                                                     AB_THREADS, AB_DKV_SMEM, s, tmQ, tmKV, tmDO, tmDKV, p))
      return rc;
  }
  return 0;
}

// The context backward over d (dQ kernel only) with n_keys[b] cached keys for dataset b when kRagged
template <bool kRagged>
static int launch_attn_ctx_bwd_tc(const pfn_attn_ctx_grad_desc* d, cudaStream_t s, const char* who) {
  if (int rc = check_attn_ctx_grad_desc(d, true, who)) return rc;
  const pfn_attn_ctx_desc& c = d->c;
  PFN_CHECK_ARG(c.dtype == PFN_BF16, "%s: bf16 only", who);
  PFN_CHECK_ARG(c.dh == ATT_DH, "%s: head dim %d unsupported (built for 128)", who, c.dh);
  PFN_CHECK_ARG(c.ld_qkv % 8 == 0 && c.ld_kv % 8 == 0 && c.ld_out % 8 == 0 && d->ld_dout % 8 == 0 && d->ld_dqkv % 8 == 0,
                "%s: leading dims must be multiples of 8", who);
  // with n == 0 no key block is loaded; the key map then only needs a valid base
  const void* kv = c.n > 0 ? c.kv : c.qkv;
  PFN_CHECK_ARG(((reinterpret_cast<uintptr_t>(c.qkv) | reinterpret_cast<uintptr_t>(kv) | reinterpret_cast<uintptr_t>(c.out) |
                  reinterpret_cast<uintptr_t>(d->dout) | reinterpret_cast<uintptr_t>(d->dqkv)) & 15) == 0,
                "%s: qkv/kv/out/dout/dqkv must be 16-byte aligned", who);
  AttnBwdParams p;
  p.T = c.m; p.B = c.B; p.H = c.H; p.sep = c.n;
  p.scale = c.scale; p.scale_log2 = c.scale * 1.4426950408889634f;
  p.qkv = reinterpret_cast<const __nv_bfloat16*>(c.qkv); p.ld_qkv = c.ld_qkv;
  p.dout = reinterpret_cast<const __nv_bfloat16*>(d->dout); p.ld_dout = d->ld_dout;
  p.dqkv = reinterpret_cast<__nv_bfloat16*>(d->dqkv); p.ld_dqkv = d->ld_dqkv;
  p.lse = d->lse; p.delta = d->delta; p.dq_colsum = nullptr; p.delta_tm = 0;
  p.drop_seed = 0; p.drop_thr = 0;
  p.batch_major = 0;
  p.n_keys = d->n_keys;
  const int E = c.H * ATT_DH;
  CUtensorMap tmQ, tmKV, tmDO, tmDQ;
  if (int rc = att_tensor_map(&tmQ, c.qkv, 3 * E, c.ld_qkv, c.m, c.B, c.m, 0)) return rc;
  if (int rc = att_tensor_map(&tmKV, kv, c.n > 0 ? 2 * E : 3 * E, c.n > 0 ? c.ld_kv : c.ld_qkv, c.n, c.B, c.n > 0 ? c.n : 1, 0))
    return rc;
  if (int rc = att_tensor_map(&tmDO, d->dout, E, d->ld_dout, c.m, c.B, c.m, 0)) return rc;
  if (int rc = att_tensor_map(&tmDQ, d->dqkv, 3 * E, d->ld_dqkv, c.m, c.B, c.m, 0)) return rc;
  const long long rows = static_cast<long long>(c.m) * c.B;
  long long grid = (rows + 7) / 8;
  if (grid > 8LL * num_sms()) grid = 8LL * num_sms();
  attn_bwd_delta_kernel<<<static_cast<int>(grid), 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(c.out), c.ld_out,
                                                               p.dout, p.ld_dout, d->delta, c.m, c.B, c.H, 0);
  PFN_LAUNCH_OK();
  p.n_tiles = (c.m + 127) / 128;
  return att_launch_persistent<attn_bwd_dq_kernel<true, kRagged>>(who, static_cast<long long>(p.n_tiles) * c.B * c.H,
                                                                   AB_THREADS, AB_DQ_SMEM, s, tmQ, tmKV, tmDO, tmDQ, p);
}

}  // namespace pfn

using namespace pfn;

extern "C" int pfn_attention_bwd_tc(const pfn_attn_desc* d, void* stream) {
  return launch_attn_bwd_tc<false>(d, nullptr, reinterpret_cast<cudaStream_t>(stream), "attention_bwd_tc");
}

extern "C" int pfn_attention_ragged_train_bwd_tc(const pfn_attn_ragged_train_desc* d, void* stream) {
  PFN_CHECK_ARG(d != nullptr && d->n_keys != nullptr, "attention_ragged_train_bwd_tc: null descriptor / n_keys");
  return launch_attn_bwd_tc<true>(&d->a, d->n_keys, reinterpret_cast<cudaStream_t>(stream), "attention_ragged_train_bwd_tc");
}

extern "C" int pfn_attention_ctx_bwd_tc(const pfn_attn_ctx_grad_desc* d, void* stream) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const char* who = "attention_ctx_bwd_tc";
  PFN_CHECK_ARG(d != nullptr, "%s: null descriptor", who);
  return d->n_keys ? launch_attn_ctx_bwd_tc<true>(d, s, who) : launch_attn_ctx_bwd_tc<false>(d, s, who);
}
