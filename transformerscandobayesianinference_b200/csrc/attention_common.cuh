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
#include "../../include/pfn_b200.h"

namespace pfn {

constexpr int ATT_DH = 128;
constexpr int ATT_ROW_BYTES = ATT_DH * 2;
constexpr int ATT_TILE_ROWS = 64;                             // rows of one TMA box / one wgmma M or key block
constexpr int ATT_TILE = ATT_TILE_ROWS * ATT_ROW_BYTES;       // 16 KB

int check_attn_desc_public(const pfn_attn_desc* d, bool bwd, const char* who);

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

// the 32 columns of a 128-wide head row that lane `lane` owns in an m16n8 accumulator row: 8 j + 2 (lane & 3) + {0, 1}
__device__ __forceinline__ float2 att_ld2(const __nv_bfloat16* row, int j, int lane) {
  return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(row + 8 * j + 2 * (lane & 3)));
}
__device__ __forceinline__ void att_st2(__nv_bfloat16* row, int j, int lane, float x, float y) {
  *reinterpret_cast<uint32_t*>(row + 8 * j + 2 * (lane & 3)) = tc::pack_bf16x2(x, y);
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}

static inline int check_tc_attn(const pfn_attn_desc* d, bool bwd, const char* who) {
  if (int rc = check_attn_desc_public(d, bwd, who)) return rc;
  PFN_CHECK_ARG(d->dtype == PFN_BF16, "%s: bf16 only", who);
  PFN_CHECK_ARG(d->dh == ATT_DH, "%s: head dim %d unsupported (built for 128)", who, d->dh);
  PFN_CHECK_ARG(d->ld_qkv % 8 == 0 && d->ld_out % 8 == 0, "%s: leading dims must be multiples of 8", who);
  PFN_CHECK_ARG(((reinterpret_cast<uintptr_t>(d->qkv) | reinterpret_cast<uintptr_t>(d->out)) & 15) == 0,
                "%s: qkv/out must be 16-byte aligned", who);
  if (bwd) {
    PFN_CHECK_ARG(d->ld_dout % 8 == 0 && d->ld_dqkv % 8 == 0, "%s: leading dims must be multiples of 8", who);
    PFN_CHECK_ARG(((reinterpret_cast<uintptr_t>(d->dout) | reinterpret_cast<uintptr_t>(d->dqkv)) & 15) == 0,
                  "%s: dout/dqkv must be 16-byte aligned", who);
  }
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
