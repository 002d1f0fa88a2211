// Shared pieces of the tensor-core attention kernels (attention_tc.cu: forward; attention_bwd_tc.cu: backward), head dim 128,
// bf16, warp-level mma.sync m16n8k16 with fp32 accumulation.
//
// Operand tiles live in shared memory as [rows][128] bf16 (256 B per row).  The sixteen 16-byte chunks of a row are
// XOR-swizzled with the row index (chunk c of row r sits at c ^ (r & 7)), so the eight rows one ldmatrix reads hit eight
// different bank groups.
#pragma once
#include "common.cuh"
#include "dropout.cuh"
#include "tc_common.cuh"
#include "../../include/pfn_b200.h"

namespace pfn {

constexpr int ATT_DH = 128;
constexpr int ATT_ROW_BYTES = ATT_DH * 2;

int check_attn_desc_public(const pfn_attn_desc* d, bool bwd, const char* who);

// byte offset of element (r, c) in a swizzled [rows][128] bf16 tile
__device__ __forceinline__ uint32_t att_sw(int r, int c) {
  return static_cast<uint32_t>(r * ATT_ROW_BYTES + ((((c >> 3) ^ (r & 7))) << 4) + (c & 7) * 2);
}

// token row of (time t, batch b) in the [T*B, cols] activations
__device__ __forceinline__ size_t att_tok(int t, int b, int T, int B, int batch_major) {
  return batch_major ? static_cast<size_t>(b) * T + t : static_cast<size_t>(t) * B + b;
}

// cp.async of NROWS rows [t0, t0 + NROWS) of one head (columns col0 .. col0 + 127 of a [T*B, ld] bf16 matrix) into a
// swizzled tile; rows outside [t0, t_end) are zero-filled.  All 128 threads of the CTA take part.
template <int NROWS>
__device__ __forceinline__ void att_load_tile(uint8_t* tile, const __nv_bfloat16* base, int ld, int col0, int t0, int t_end,
                                              int b, int T, int B, int batch_major) {
  const uint32_t s = tc::smem_u32(tile);
#pragma unroll
  for (int k = 0; k < NROWS * 16 / 128; ++k) {
    const int idx = static_cast<int>(threadIdx.x) + 128 * k;
    const int r = idx >> 4, c = idx & 15;
    const int t = t0 + r;
    const bool ok = t < t_end;
    const __nv_bfloat16* src = ok ? base + att_tok(t, b, T, B, batch_major) * ld + col0 + c * 8 : base;
    tc::cp_async16(s + att_sw(r, c * 8), src, ok ? 16u : 0u);
  }
}

// A fragment (16 rows x 16 columns at (r0, c0)) of a swizzled tile
__device__ __forceinline__ void att_frag_a(uint32_t (&a)[4], uint32_t tile, int r0, int c0, int lane) {
  tc::ldmatrix_x4(a, tile + att_sw(r0 + (lane & 15), c0 + ((lane >> 4) << 3)));
}
// B fragments of two n-tiles (rows n0 .. n0 + 15 of the tile are the n index, columns k0 .. k0 + 15 the k index):
// b[0], b[1] for n-tile n0, b[2], b[3] for n-tile n0 + 8
__device__ __forceinline__ void att_frag_b(uint32_t (&b)[4], uint32_t tile, int n0, int k0, int lane) {
  tc::ldmatrix_x4(b, tile + att_sw(n0 + (lane & 7) + ((lane >> 4) << 3), k0 + (((lane >> 3) & 1) << 3)));
}
// B fragments of two n-tiles where the tile's rows are the k index (k0 .. k0 + 15) and its columns the n index
// (n0 .. n0 + 15): b[0], b[1] for n-tile n0, b[2], b[3] for n-tile n0 + 8
__device__ __forceinline__ void att_frag_bt(uint32_t (&b)[4], uint32_t tile, int k0, int n0, int lane) {
  tc::ldmatrix_x4_trans(b, tile + att_sw(k0 + (lane & 7) + (((lane >> 3) & 1) << 3), n0 + ((lane >> 4) << 3)));
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

}  // namespace pfn
