// Tensor-core masked attention for the single_eval_pos mask (reference transformer.py:35-41), head dim 128, bf16.
//
//   keys(i) = [0, sep)  U  {i if i >= sep}        o_i = softmax_j(q_i.k_j / sqrt(dh)) v_j
//
// The [T,T] mask is never built: the dense part (keys < sep) runs on the tensor cores in 64-key blocks and the single
// diagonal key of a query row is a 128-wide dot product done by the four lanes that own the row.  Q/K/V rows are read
// straight out of the packed [T*B, 3E] in-projection output, so there is no head-split / transpose kernel.
//
// attn_fwd_kernel is persistent: one CTA per SM walks the (batch, head, 128-row query tile) units on the K/V pipeline it
// shares with the dQ backward kernel (AttPipe, attention_common.cuh).  Warpgroup 2 (producer, 40 registers) TMA-loads
// the tile's Q and a 4-stage ring of (K, V) 64-key blocks; warpgroups 0 and 1 (consumers, 232 registers) each own 64
// query rows and run, per key block j,
//   S_j = Q K_j^T (wgmma m64n64k16, fp32)  ->  online softmax in the log2 domain  ->  P_j as bf16 A fragments (registers)
//   ->  O += P_j V_j (wgmma m64n128k16, A from registers, V read MN-major)
// with S_j and the PV MMAs of block j-1 issued together, so the softmax of block j runs under the previous P V.  A row's
// diagonal key is folded in before the loop: m = s_ii, l = 1, O = keep_ii v_i (rows < sep start from -inf, 0, 0).
// O / l is packed to bf16 into a 128-byte-swizzled staging tile per warpgroup and written with TMA tile stores, which
// clip rows past T.
#include "attention_common.cuh"

namespace pfn {

constexpr int AF_THREADS = 3 * 128;
constexpr int AF_STAGES = 4;                              // (K, V) blocks in flight
// Q of the tile (2 x 16 KB), output staging (2 x 16 KB), ring of (K, V), barriers
constexpr int AF_OFF_STG = 2 * ATT_TILE;
constexpr int AF_OFF_RING = 4 * ATT_TILE;
constexpr int AF_OFF_BAR = AF_OFF_RING + AF_STAGES * 2 * ATT_TILE;
constexpr int AF_SMEM = AF_OFF_BAR + (2 * AF_STAGES + 2) * 8 + 1024;   // + 1 KB alignment slack
static_assert(AF_SMEM <= 232448, "the tiles and the ring must fit the 227 KB of shared memory");

struct AttnFwdParams {
  int T, B, H, sep;
  float scale_log2;   // scale * log2(e)
  const __nv_bfloat16* qkv; int ld_qkv;
  float* lse;
  int n_tiles;        // 128-row query tiles per (batch, head)
  int batch_major;
  uint32_t drop_seed; int drop_thr;   // dropout on the probabilities (thr 0 = off), csrc/dropout.cuh
};

__global__ void __launch_bounds__(AF_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV,
                const __grid_constant__ CUtensorMap tmO, const AttnFwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = att_smem_base(smem_raw);
  uint8_t* sQ = smem;                                     // warpgroup g's 64 rows at + g * 16 KB
  uint8_t* sStg = smem + AF_OFF_STG;                      // warpgroup g's output staging at + g * 16 KB
  const AttPipe<AF_STAGES> pp(smem + AF_OFF_RING, reinterpret_cast<uint64_t*>(smem + AF_OFF_BAR));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int E = p.H * ATT_DH;
  const int nblk = (p.sep + ATT_TILE_ROWS - 1) / ATT_TILE_ROWS;
  const int n_units = p.n_tiles * p.B * p.H;
  if (threadIdx.x == 0) {
    pp.init();
    tc::mbar_fence_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // ------------------------------------------------------------------ TMA producer
    tc::setmaxnreg_dec<40>();
    if (threadIdx.x == 256) {
      tc::tma_prefetch_desc(&tmQ);
      tc::tma_prefetch_desc(&tmKV);
      att_kv_producer(pp, &tmKV, n_units, p.n_tiles, p.H, nblk, 2 * ATT_TILE, [&](const AttUnit& unit) {
        for (int g = 0; g < 2; ++g)
          att_load_tile(sQ + g * ATT_TILE, &tmQ, pp.q_full, unit.h * ATT_DH, unit.b, unit.tile * 128 + 64 * g);
      });
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroups
  tc::setmaxnreg_inc<232>();
  const int g = warp >> 2, wq = warp & 3;
  const int tid = threadIdx.x & 127;
  const uint32_t q_tile = tc::smem_u32(sQ + g * ATT_TILE);
  uint8_t* stg = sStg + g * ATT_TILE;
  const float dscale = p.drop_thr > 0 ? drop_scale(p.drop_thr) : 1.0f;
  AttRing<AF_STAGES> ring;
  bool timed_out = false;
  for (int u = blockIdx.x, it = 0; u < n_units && !timed_out; u += gridDim.x, ++it) {
    const AttUnit unit = att_unit(u, p.n_tiles, p.H);
    const int t0 = unit.tile * 128 + 64 * g;
    const int i0 = t0 + 16 * wq + (lane >> 2);            // this lane's rows: i0, i0 + 8

    // Diagonal key first: o[4 j + 2 r + c] is row i0 + 8 r, column 8 j + 2 (lane & 3) + c.  A row i >= sep starts from
    // m = s_ii, l = 1 (this lane's share of l: 1 in lane 0 of the quad) and O = keep_ii v_i; the loads are in flight
    // while the first TMA waits run.
    float o[64], m[2], l[2];
    uint32_t drow[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int i = i0 + 8 * r;
      const bool diag = i < p.T && i >= p.sep;
      drow[r] = static_cast<uint32_t>(unit.bh) * p.T + i;
      const __nv_bfloat16* qrow = p.qkv + att_tok(diag ? i : 0, unit.b, p.T, p.B, p.batch_major) * p.ld_qkv + unit.h * ATT_DH;
      float sd = 0.f;
      if (diag) {
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float2 q = att_ld2(qrow, j, lane), k = att_ld2(qrow + E, j, lane);
          sd = fmaf(q.x, k.x, fmaf(q.y, k.y, sd));
        }
      }
      sd = quad_sum(sd) * p.scale_log2;
      m[r] = diag ? sd : -INFINITY;
      l[r] = diag && (lane & 3) == 0 ? 1.f : 0.f;
      const bool keep = diag && (p.drop_thr == 0 || drop_keep(p.drop_seed, drow[r], i, p.drop_thr));
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float2 v = keep ? att_ld2(qrow + 2 * E, j, lane) : make_float2(0.f, 0.f);
        o[4 * j + 2 * r] = v.x;
        o[4 * j + 2 * r + 1] = v.y;
      }
    }

    // Key loop (att_key_loop): S_kb = Q K_kb^T, its online softmax while PV_{kb-1} (O += P_{kb-1} V_{kb-1}) runs, then
    // O rescaled and P_kb packed.
    float s[32];
    uint32_t ap[16];
    float corr[2];
    auto issue_s = [&](int st) {
      const uint32_t k_s = tc::smem_u32(pp.ring + st * 2 * ATT_TILE);
      const uint32_t q_s = att_opaque(q_tile);
      tc::wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) att_mma_n64(s, att_desc_k(q_s, kk), att_desc_k(k_s, kk), kk);
      tc::wgmma_commit();
    };
    auto issue_pv = [&](int st, bool) {                  // always accumulates: O starts from the diagonal key
      const uint32_t v_s = tc::smem_u32(pp.ring + st * 2 * ATT_TILE) + ATT_TILE;
      tc::wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) tc::wgmma_m64n128k16_rs(o, ap + 4 * kk, att_desc_mn(v_s, kk), 1);
      tc::wgmma_commit();
    };
    // Online softmax of block kb in s.  Element 4 j + e of S is row i0 + 8 (e >> 1), key kb * 64 + 8 j + 2 (lane & 3) +
    // (e & 1); keys >= sep (only in the last block) are masked.  The running max m is in the scaled log2 domain; the
    // scale > 0 is applied to the block max and inside the exp2 argument, p = 2^(s c - m).  l sums the probabilities
    // before dropout; s is left holding them after dropout.
    auto softmax = [&](int kb) {
      const int key0 = kb * ATT_TILE_ROWS + 2 * (lane & 3);
      if (kb * ATT_TILE_ROWS + ATT_TILE_ROWS > p.sep) {
#pragma unroll
        for (int e = 0; e < 32; ++e)
          if (key0 + 8 * (e >> 2) + (e & 1) >= p.sep) s[e] = -INFINITY;
      }
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int e = 0; e < 32; ++e) mx[(e >> 1) & 1] = fmaxf(mx[(e >> 1) & 1], s[e]);
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const float mn = fmaxf(m[r], quad_max(mx[r]) * p.scale_log2);
        corr[r] = fast_ex2(m[r] - mn);
        m[r] = mn;
        l[r] *= corr[r];
      }
#pragma unroll
      for (int e = 0; e < 32; ++e) {
        const int r = (e >> 1) & 1;
        const float pr = fast_ex2(fmaf(s[e], p.scale_log2, -m[r]));
        l[r] += pr;
        s[e] = p.drop_thr > 0 && !drop_keep(p.drop_seed, drow[r], key0 + 8 * (e >> 2) + (e & 1), p.drop_thr) ? 0.f : pr;
      }
    };
    auto rescale_pack = [&]() {
#pragma unroll
      for (int e = 0; e < 64; ++e) o[e] *= corr[(e >> 1) & 1];
#pragma unroll
      for (int e = 0; e < 16; ++e) ap[e] = tc::pack_bf16x2(s[2 * e], s[2 * e + 1]);
    };
    if (att_key_loop(pp, ring, it, nblk, issue_s, issue_pv, [&] { tc::wgmma_fence_regs(s); },
                     [&] { tc::wgmma_fence_regs(o); }, softmax, rescale_pack, [] {})) {
      timed_out = true;
      break;
    }

    // epilogue: O / l -> bf16 into the staging tile (two 64-column boxes, 128-byte swizzle: 16-byte chunk c of row rr at
    // c ^ (rr & 7)), then one thread stores it with the TMA; lse = ln(sum_j exp(s_ij)) from one lane per row
    if (tid == 0) tc::bulk_wait_read<0>();                // the previous tile's store has read the staging tile
    tc::named_bar_sync(1 + g, 128);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int i = i0 + 8 * r;
      const float lr = quad_sum(l[r]);
      const float inv = dscale / lr;
      const int rr = 16 * wq + (lane >> 2) + 8 * r;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const uint32_t off = (j >> 3) * 8192 + rr * 128 + (((j & 7) ^ (rr & 7)) << 4) + (lane & 3) * 4;
        *reinterpret_cast<uint32_t*>(stg + off) = tc::pack_bf16x2(o[4 * j + 2 * r] * inv, o[4 * j + 2 * r + 1] * inv);
      }
      if (i < p.T && (lane & 3) == 0) p.lse[static_cast<size_t>(unit.bh) * p.T + i] = (m[r] + __log2f(lr)) * 0.69314718055994531f;
    }
    tc::fence_proxy_async_smem();
    tc::named_bar_sync(1 + g, 128);
    if (tid == 0 && t0 < p.T) {
      tc::tma_store_3d(&tmO, stg, unit.h * ATT_DH, unit.b, t0);
      tc::tma_store_3d(&tmO, stg + 8192, unit.h * ATT_DH + 64, unit.b, t0);
      tc::bulk_commit();
    }
  }
  if (tid == 0) tc::bulk_wait<0>();
  if (timed_out) asm volatile("trap;");
}

}  // namespace pfn

using namespace pfn;

extern "C" int pfn_attention_fwd_tc(const pfn_attn_desc* d, void* stream) {
  if (int rc = check_tc_attn(d, false, "attention_fwd_tc")) return rc;
  AttnFwdParams p;
  p.T = d->T; p.B = d->B; p.H = d->H; p.sep = d->sep;
  p.scale_log2 = d->scale * 1.4426950408889634f;
  p.qkv = reinterpret_cast<const __nv_bfloat16*>(d->qkv); p.ld_qkv = d->ld_qkv;
  p.lse = d->lse;
  p.n_tiles = (d->T + 127) / 128;
  p.batch_major = d->batch_major;
  p.drop_seed = d->drop_seed; p.drop_thr = d->drop_thr;
  const int E = d->H * ATT_DH;
  CUtensorMap tmQ, tmKV, tmO;
  if (int rc = att_qkv_maps(d, &tmQ, &tmKV)) return rc;
  // out: rows past T are not written
  if (int rc = att_tensor_map(&tmO, d->out, E, d->ld_out, d->T, d->B, d->T, d->batch_major)) return rc;
  return att_launch_persistent<attn_fwd_kernel>("attention_fwd_tc", static_cast<long long>(p.n_tiles) * d->B * d->H,
                                                AF_THREADS, AF_SMEM, reinterpret_cast<cudaStream_t>(stream), tmQ, tmKV, tmO, p);
}
