// Shared pieces of the tensor-core attention kernels (attention_tc.cu: forward; attention_bwd_tc.cu: backward), head dim 128,
// bf16, warpgroup MMA (wgmma) with fp32 accumulation and TMA-fed operands.
//
// An operand tile is 64 rows of one head: two 8 KB boxes of 64 columns (128 B per row) in the 128-byte swizzle, loaded
// by the TMA straight out of the packed [T*B, 3E] qkv buffer through a 3-D tensor map (columns, batch, time).  The same
// tile is a K-major wgmma operand (S = Q K^T) and an MN-major one (O += P V, dQ += dS K), so nothing is transposed.
#pragma once
#include "common.cuh"
#include "dropout.cuh"
#include "tc_common.cuh"
#include "../../include/pfn_b200_ragged.h"
#include "../../include/pfn_b200_ragged_train.h"
#include "../../include/pfn_b200_input_grad.h"

namespace pfn {

constexpr int ATT_DH = 128;
constexpr int ATT_ROW_BYTES = ATT_DH * 2;
constexpr int ATT_TILE_ROWS = 64;                             // rows of one TMA box / one wgmma M or key block
constexpr int ATT_TILE = ATT_TILE_ROWS * ATT_ROW_BYTES;       // 16 KB

int check_attn_desc_public(const pfn_attn_desc* d, bool bwd, const char* who);
int check_attn_ctx_desc(const pfn_attn_ctx_desc* d, const char* who);
// the descriptor of the same forward with sep = T and no lse / over the cache of n rows, checked; the key counts stay in d
int attn_ragged_as_masked(const pfn_attn_ragged_desc* d, pfn_attn_desc* a, const char* who);
int attn_ctx_ragged_as_ctx(const pfn_attn_ctx_ragged_desc* d, pfn_attn_ctx_desc* c, const char* who);
// the context-attention descriptor with lse (and, for the backward, dout / dqkv / delta), checked
int check_attn_ctx_grad_desc(const pfn_attn_ctx_grad_desc* d, bool bwd, const char* who);

// token row of (time t, batch b) in the [T*B, cols] activations
__device__ __forceinline__ size_t att_tok(int t, int b, int T, int B, int batch_major) {
  return batch_major ? static_cast<size_t>(b) * T + t : static_cast<size_t>(t) * B + b;
}

// wgmma descriptors of a 64-row tile (two 64-column boxes 8 KB apart, 128-byte swizzle), k16 step kk:
// K-major (the tile's columns are the k index, kk < 8) and MN-major (its rows are the k index, kk < 4)
__device__ __forceinline__ uint64_t att_desc_k(uint32_t tile, int kk) {
  return tc::wgmma_smem_desc(tile + (kk >> 2) * 8192 + (kk & 3) * 32, 16, 1024);
}
__device__ __forceinline__ uint64_t att_desc_mn(uint32_t tile, int kk) {
  return tc::wgmma_smem_desc(tile + kk * 2048, 8192, 1024);
}
// The address of a tile that stays resident across a loop, made opaque in every iteration so that the descriptors of its
// k16 steps are formed next to their MMAs instead of being hoisted out of the loop and held in registers throughout.
__device__ __forceinline__ uint32_t att_opaque(uint32_t addr) {
  asm volatile("" : "+r"(addr));
  return addr;
}
// k16 step kk of a 64 x 64 score block; the first step writes the accumulator
__device__ __forceinline__ void att_mma_n64(float (&d)[32], uint64_t a_desc, uint64_t b_desc, int kk) {
  if (kk == 0) tc::wgmma_m64n64k16<0>(d, a_desc, b_desc);
  else tc::wgmma_m64n64k16<1>(d, a_desc, b_desc);
}

// TMA of rows [t0, t0 + 64) of one head (columns col0 .. col0 + 127) into a 16 KB tile
__device__ __forceinline__ void att_load_tile(uint8_t* dst, const CUtensorMap* m, uint64_t* bar, int col0, int b, int t0) {
  tc::tma_load_3d(dst, m, bar, col0, b, t0);
  tc::tma_load_3d(dst + 8192, m, bar, col0 + 64, b, t0);
}

// TMA store of a 16 KB tile to rows [t0, t0 + 64) of one head (columns col0 .. col0 + 127); rows at t >= the map's t
// extent are not written.  The caller commits the bulk group.
__device__ __forceinline__ void att_store_tile(const CUtensorMap* m, const uint8_t* src, int col0, int b, int t0) {
  tc::tma_store_3d(m, src, col0, b, t0);
  tc::tma_store_3d(m, src + 8192, col0 + 64, b, t0);
}
// Byte offset in a 16 KB tile of the columns 8 j + 2 (lane & 3) + {0, 1} of row `row` (an m16n8 accumulator pair): the
// 128-byte swizzle XORs the 16-byte chunk index within a 128-byte row with row & 7
__device__ __forceinline__ int att_tile_off2(int row, int j, int lane) {
  return (j >> 3) * 8192 + row * 128 + (((j & 7) ^ (row & 7)) << 4) + 4 * (lane & 3);
}

// A work unit: one 128-row tile of one (batch, head).  Unit u is tile u % n_tiles of (batch, head) bh = u / n_tiles, so
// the tiles of one (batch, head) are neighbours and the CTAs that run them at the same time share its K/V in L2.
struct AttUnit {
  int tile;   // 128-row tile: of the query rows, or of the train keys in the dK/dV kernel
  int bh, h, b;
};
__device__ __forceinline__ AttUnit att_unit(int u, int n_tiles, int H) {
  const int bh = u / n_tiles;
  return {u % n_tiles, bh, bh % H, bh / H};
}

// Position in a ring of STAGES buffers: the stage and the parity of the barrier phase that completes it
template <int STAGES>
struct AttRing {
  int stage = 0;
  uint32_t phase = 0;
  __device__ __forceinline__ void advance() { if (++stage == STAGES) { stage = 0; phase ^= 1; } }
};

// the dynamic shared memory from its first 1 KB boundary, as the 128-byte swizzle needs (the sizes include the slack)
__device__ __forceinline__ uint8_t* att_smem_base(uint8_t* raw) {
  return raw + ((1024u - (tc::smem_u32(raw) & 1023u)) & 1023u);
}

// The K/V pipeline of the persistent kernels (forward, dQ backward): one TMA thread streams the 64-key blocks of the
// train keys through a ring of STAGES (K, V) stages to two consumer warpgroups, and hands them the query operands of the
// CTA's current tile (Q, and dO in the backward) through q_full / q_empty.  Its barriers are 2 STAGES + 2 words.
template <int STAGES>
struct AttPipe {
  uint8_t* ring;        // stage s: K at + 2 s * 16 KB, V at + (2 s + 1) * 16 KB
  uint64_t* kv_full;    // [STAGES] the stage's K and V have landed
  uint64_t* kv_empty;   // [STAGES] both warpgroups' MMAs that read the stage have completed
  uint64_t* q_full;     // the query operands of the CTA's current tile have landed
  uint64_t* q_empty;    // both warpgroups' last MMAs that read them have completed
  __device__ __forceinline__ AttPipe(uint8_t* ring_smem, uint64_t* bars)
      : ring(ring_smem), kv_full(bars), kv_empty(bars + STAGES), q_full(bars + 2 * STAGES), q_empty(bars + 2 * STAGES + 1) {}
  // by one thread, before tc::mbar_fence_init() and the block barrier
  __device__ __forceinline__ void init() const {
    for (int s = 0; s < STAGES; ++s) {
      tc::mbar_init(&kv_full[s], 1);
      tc::mbar_init(&kv_empty[s], 2);
    }
    tc::mbar_init(q_full, 1);
    tc::mbar_init(q_empty, 2);
  }
};

// The producer of the pipeline (one thread): for each of the CTA's units, the nblk_of(unit) key blocks of its (batch,
// head).  The next tile's query operands go in once the consumers are done with the current ones, which is before its
// last key block is (so the first key blocks of the next tile are already in flight by then): load_q(unit) issues
// q_bytes of TMA loads on q_full.  k_col / v_col: the first column of head 0's K and V in the map tmKV.
template <int STAGES, class NBlk, class LoadQ>
__device__ __forceinline__ void att_kv_producer(const AttPipe<STAGES>& pp, const CUtensorMap* tmKV, int n_units, int n_tiles,
                                                int H, NBlk&& nblk_of, int k_col, int v_col, uint32_t q_bytes,
                                                LoadQ&& load_q) {
  AttRing<STAGES> ring;
  for (int u = blockIdx.x, it = 0; u < n_units; u += gridDim.x, ++it) {
    const AttUnit unit = att_unit(u, n_tiles, H);
    const int nblk = nblk_of(unit);
    auto claim_q = [&]() {
      if (it > 0) tc::mbar_wait_suspend(pp.q_empty, (it - 1) & 1);
      tc::mbar_expect_tx(pp.q_full, q_bytes);
      load_q(unit);
    };
    const int claim_at = min(STAGES - 1, nblk - 1);
    if (nblk == 0) claim_q();
    for (int kb = 0; kb < nblk; ++kb) {
      if (kb == claim_at) claim_q();
      tc::mbar_wait_suspend(&pp.kv_empty[ring.stage], ring.phase ^ 1);
      uint8_t* dst = pp.ring + ring.stage * 2 * ATT_TILE;
      tc::mbar_expect_tx(&pp.kv_full[ring.stage], 2 * ATT_TILE);
      att_load_tile(dst, tmKV, &pp.kv_full[ring.stage], k_col + unit.h * ATT_DH, unit.b, kb * ATT_TILE_ROWS);
      att_load_tile(dst + ATT_TILE, tmKV, &pp.kv_full[ring.stage], v_col + unit.h * ATT_DH, unit.b, kb * ATT_TILE_ROWS);
      ring.advance();
    }
  }
}

// One consumer warpgroup's key loop over the nblk key blocks of the CTA's it-th tile.  Block kb issues its first MMA
// group (issue_a: S, or S and dP) and the second group of block kb - 1 (issue_b: O += P V, or dQ += dS K; the flag is
// false for the tile's first) back to back, waits for the first only and runs math(kb) (softmax, or dS) under the
// second, then waits for it, releases its stage and runs pack() (the next A fragments).  before_tail() is issued under
// the tile's last MMAs, or at once when there are none; fence_a / fence_b fence the two groups' accumulators.
// The accumulators are written only when no MMA that owns them is in flight: otherwise ptxas serialises the whole wgmma
// pipeline.  For the same reason a timed-out wait inside the loop is recorded and the block runs on; the tile is
// abandoned once the pipeline has drained.  Returns true when a wait timed out: the caller leaves its tile loop and
// traps after it, so that ptxas keeps the register budget setmaxnreg raised (tc::mbar_wait_bounded).
template <int STAGES, class IssueA, class IssueB, class FenceA, class FenceB, class Math, class Pack, class BeforeTail>
__device__ __forceinline__ bool att_key_loop(const AttPipe<STAGES>& pp, AttRing<STAGES>& ring, int it, int nblk,
                                             IssueA&& issue_a, IssueB&& issue_b, FenceA&& fence_a, FenceB&& fence_b,
                                             Math&& math, Pack&& pack, BeforeTail&& before_tail) {
  const bool leader = (threadIdx.x & 127) == 0;
  if (!tc::mbar_wait_bounded(pp.q_full, it & 1)) return true;
  if (nblk > 0) {
    if (!tc::mbar_wait_bounded(&pp.kv_full[ring.stage], ring.phase)) return true;
    issue_a(ring.stage);
    tc::wgmma_wait<0>();
    fence_a();
    if (nblk == 1 && leader) tc::mbar_arrive(pp.q_empty);
    math(0);
    pack();
    int cur = ring.stage;                   // ring stage of the block whose second group is next
    ring.advance();
    bool timed_out = false;
    for (int kb = 1; kb < nblk; ++kb) {
      if (!timed_out && !tc::mbar_wait_bounded(&pp.kv_full[ring.stage], ring.phase)) timed_out = true;
      issue_a(ring.stage);
      issue_b(cur, kb > 1);
      tc::wgmma_wait<1>();
      fence_a();
      if (kb == nblk - 1 && leader) tc::mbar_arrive(pp.q_empty);
      math(kb);
      tc::wgmma_wait<0>();
      fence_b();
      if (leader) tc::mbar_arrive(&pp.kv_empty[cur]);
      cur = ring.stage;
      ring.advance();
      pack();
    }
    issue_b(cur, nblk > 1);
    before_tail();
    tc::wgmma_wait<0>();
    fence_b();
    if (timed_out) return true;
    if (leader) tc::mbar_arrive(&pp.kv_empty[cur]);
  } else {
    if (leader) tc::mbar_arrive(pp.q_empty);
    before_tail();
  }
  return false;
}

// the 32 columns of a 128-wide head row that lane `lane` owns in an m16n8 accumulator row: 8 j + 2 (lane & 3) + {0, 1}
__device__ __forceinline__ float2 att_ld2(const __nv_bfloat16* row, int j, int lane) {
  return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(row + 8 * j + 2 * (lane & 3)));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}

// what the tensor-core kernels need of a checked descriptor's forward operands
static inline int check_tc_operands(const pfn_attn_desc* d, const char* who) {
  PFN_CHECK_ARG(d->dtype == PFN_BF16, "%s: bf16 only", who);
  PFN_CHECK_ARG(d->dh == ATT_DH, "%s: head dim %d unsupported (built for 128)", who, d->dh);
  PFN_CHECK_ARG(d->ld_qkv % 8 == 0 && d->ld_out % 8 == 0, "%s: leading dims must be multiples of 8", who);
  PFN_CHECK_ARG(((reinterpret_cast<uintptr_t>(d->qkv) | reinterpret_cast<uintptr_t>(d->out)) & 15) == 0,
                "%s: qkv/out must be 16-byte aligned", who);
  return 0;
}

static inline int check_tc_attn(const pfn_attn_desc* d, bool bwd, const char* who) {
  if (int rc = check_attn_desc_public(d, bwd, who)) return rc;
  if (int rc = check_tc_operands(d, who)) return rc;
  if (bwd) {
    PFN_CHECK_ARG(d->ld_dout % 8 == 0 && d->ld_dqkv % 8 == 0, "%s: leading dims must be multiples of 8", who);
    PFN_CHECK_ARG(((reinterpret_cast<uintptr_t>(d->dout) | reinterpret_cast<uintptr_t>(d->dqkv)) & 15) == 0,
                  "%s: dout/dqkv must be 16-byte aligned", who);
  }
  return 0;
}

// Launch of a persistent kernel over `units` work units: one CTA per SM, or one per unit when there are fewer.  The
// kernel's dynamic shared-memory limit is raised on its first launch on each device.
template <auto Kernel, class... Args>
static inline int att_launch_persistent(const char* who, long long units, int threads, int smem, cudaStream_t s,
                                        const Args&... args) {
  PFN_CHECK_ARG(units < (1LL << 31), "%s: too many tiles", who);
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set)) PFN_CUDA_OK(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const int grid = units < num_sms() ? static_cast<int>(units) : num_sms();
  Kernel<<<static_cast<unsigned>(grid), threads, smem, s>>>(args...);
  PFN_LAUNCH_OK();
  return 0;
}

// 3-D tensor map (columns, batch, time) over a [T*B, ld] bf16 activation, token row t*B + b (or b*T + t when batch-major),
// with a box of 64 columns x 1 x 64 rows and the 128-byte swizzle; rows at t >= t_extent read as zeros (and are not
// written by a store)
static inline int att_tensor_map(CUtensorMap* m, const void* base, int cols, int ld, int T, int B, int t_extent,
                                 int batch_major) {
  const uint64_t row = static_cast<uint64_t>(ld) * 2;
  const uint64_t dims[3] = {static_cast<uint64_t>(cols), static_cast<uint64_t>(B), static_cast<uint64_t>(t_extent)};
  const uint64_t strides[3] = {0, batch_major ? row * T : row, batch_major ? row : row * B};
  const uint32_t box[3] = {64, 1, ATT_TILE_ROWS};
  return make_tensor_map(m, base, false, 3, dims, strides, box, true);
}

// The two maps over the packed qkv: Q rows up to T, and K / V with keys past sep reading as zeros (the map needs a
// non-empty extent; with sep = 0 no key block is loaded)
static inline int att_qkv_maps(const pfn_attn_desc* d, CUtensorMap* tmQ, CUtensorMap* tmKV) {
  const int E = d->H * ATT_DH;
  if (int rc = att_tensor_map(tmQ, d->qkv, 3 * E, d->ld_qkv, d->T, d->B, d->T, d->batch_major)) return rc;
  return att_tensor_map(tmKV, d->qkv, 3 * E, d->ld_qkv, d->T, d->B, d->sep > 0 ? d->sep : 1, d->batch_major);
}

}  // namespace pfn
