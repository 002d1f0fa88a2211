// Warp-specialised TMA + wgmma GEMM for sm_90a.
//
//   C[M,N] (+)= epilogue( sum_k A(m,k) * B(n,k) )      bf16 operands, fp32 accumulation in registers
//
// Replaces the cuBLASLt addmm calls the reference reaches through nn.Linear / in_proj / out_proj
// (reference transformer.py:17-18,23,84-85; torch nn/functional.py:6478 `_in_projection_packed`).
//
// Operand storage ("major"):
//   K-major  : element (i,k) at base + i*ld + k        (activations x, weights W[N,K] for y = x W^T)
//   MN-major : element (i,k) at base + k*ld + i        (W used for dgrad, dY / X used for wgrad)
// so forward, dgrad and wgrad all run on the same kernel without any transposed copies in HBM: wgmma reads either
// layout straight from the 128-byte-swizzled tiles the TMA writes.
//
// Structure (one CTA per 128 x 128 output tile and k-split, two CTAs per SM so one CTA's epilogue overlaps the other's
// main loop):
//   warps 0..3, 4..7 : two consumer warpgroups; warpgroup g issues wgmma m64n128k16 for rows [64g, 64g + 64) of the tile
//                      and runs the epilogue (bias / GELU / residual / GELU' / product / row dot) from its registers
//   warp 8           : TMA producer (cp.async.bulk.tensor, 128B swizzle, mbarrier complete_tx) over a kStages ring
#include "common.cuh"
#include "tc_common.cuh"
#include "../../include/pfn_b200.h"

namespace pfn {

struct GemmTcParams {
  int M, N, K;
  const float* bias;             // [N] fp32 or null
  const __nv_bfloat16* aux;      // residual / pre-activation (GELU') / factor (MUL) / row-dot partner : [M, ld_aux] bf16, or null
  int ld_aux;
  void* C;                       // bf16 or fp32 [M, ldc]
  int ldc;
  int c_f32;                     // 1 => C is fp32
  __nv_bfloat16* C2;             // optional second output of the GELU epilogue
  int ldc2;
  int act;                       // PFN_EPI_*
  int accumulate;                // 1 => atomically add into fp32 C (split-K / grad accumulation)
  int kb_per_split;              // k-blocks (of 64) per split
  int tiles_m, tiles_n;
  float* rowdot_out;             // PFN_EPI_ROWDOT: [M, rowdot_groups] fp32, += sum over a column group of C * aux
  int rowdot_width, rowdot_groups;
  int c2_grad;                   // GELU with C2: C2 = gelu'(pre) instead of pre
};

constexpr int kBlockM = 128;
constexpr int kBlockN = 128;
constexpr int kBlockK = 64;
constexpr int kStages = 3;
constexpr int kABytes = kBlockM * kBlockK * 2;        // 16 KB
constexpr int kBBytes = kBlockN * kBlockK * 2;        // 16 KB
constexpr int kNumThreads = 2 * 128 + 32;
constexpr int kSmemBytes = kStages * (kABytes + kBBytes) + 64 + 1024;   // ring + barriers + 1 KB alignment slack
static_assert(2 * kSmemBytes <= 232448, "two CTAs per SM must fit the 227 KB of shared memory");

template <bool A_MN, bool B_MN>
__global__ void __launch_bounds__(kNumThreads, 2)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  // 1 KB alignment (128-byte swizzle atoms) by an offset on the __shared__ symbol
  uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sA = smem;
  uint8_t* sB = smem + kStages * kABytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kStages * (kABytes + kBBytes));
  uint64_t* empty_bar = full_bar + kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      tc::mbar_init(&full_bar[s], 1);
      tc::mbar_init(&empty_bar[s], 2);          // one arrival per consumer warpgroup
    }
    tc::mbar_fence_init();
  }
  __syncthreads();

  const int tiles = p.tiles_m * p.tiles_n;
  const int split = static_cast<int>(blockIdx.x) / tiles;
  const int tile = static_cast<int>(blockIdx.x) - split * tiles;
  const int m0 = (tile / p.tiles_n) * kBlockM;
  const int n0 = (tile % p.tiles_n) * kBlockN;
  const int num_kb_total = (p.K + kBlockK - 1) / kBlockK;
  const int kb0 = split * p.kb_per_split;
  const int kb1 = min(kb0 + p.kb_per_split, num_kb_total);

  if (warp == 8) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0) {
      tc::tma_prefetch_desc(&tmA);
      tc::tma_prefetch_desc(&tmB);
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        tc::mbar_wait_suspend(&empty_bar[stage], phase ^ 1);
        uint8_t* a_dst = sA + stage * kABytes;
        uint8_t* b_dst = sB + stage * kBBytes;
        const int k0 = kb * kBlockK;
        tc::mbar_expect_tx(&full_bar[stage], kABytes + kBBytes);
        if constexpr (!A_MN) {
          tc::tma_load_2d(a_dst, &tmA, &full_bar[stage], k0, m0);
        } else {
          tc::tma_load_2d(a_dst, &tmA, &full_bar[stage], m0, k0);
          tc::tma_load_2d(a_dst + 8192, &tmA, &full_bar[stage], m0 + 64, k0);
        }
        if constexpr (!B_MN) {
          tc::tma_load_2d(b_dst, &tmB, &full_bar[stage], k0, n0);
        } else {
          tc::tma_load_2d(b_dst, &tmB, &full_bar[stage], n0, k0);
          tc::tma_load_2d(b_dst + 8192, &tmB, &full_bar[stage], n0 + 64, k0);
        }
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroups: main loop
  const int g = warp >> 2;                 // warpgroup: rows [64 g, 64 g + 64) of the tile
  // The first MMA of the tile writes the accumulator (scale-d = 0), so nothing but wgmma defines `acc` until the pipeline
  // has drained: any other definition inside it makes ptxas serialise the wgmma instructions.
  float acc[64];
  {
    int stage = 0, prev = 0;
    uint32_t phase = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      tc::mbar_wait(&full_bar[stage], phase);
      const uint32_t a_addr = tc::smem_u32(sA + stage * kABytes) + g * 8192;   // K-major: 64 rows x 128 B; MN-major: chunk g
      const uint32_t b_addr = tc::smem_u32(sB + stage * kBBytes);
      tc::wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBlockK / 16; ++k) {
        // K-major: advance 16 elements (32 B) inside the 128 B swizzle row.
        // MN-major: advance 16 k-rows (16 * 128 B); LBO = stride between 64-wide M/N chunks.
        const uint64_t a_desc = A_MN ? tc::wgmma_smem_desc(a_addr + k * 2048, 8192, 1024)
                                     : tc::wgmma_smem_desc(a_addr + k * 32, 16, 1024);
        const uint64_t b_desc = B_MN ? tc::wgmma_smem_desc(b_addr + k * 2048, 8192, 1024)
                                     : tc::wgmma_smem_desc(b_addr + k * 32, 16, 1024);
        tc::wgmma_m64n128k16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, a_desc, b_desc, (kb > kb0 || k > 0) ? 1u : 0u);
      }
      tc::wgmma_commit();
      tc::wgmma_wait<1>();                 // the previous k-block's MMAs are done: its stage can be refilled
      if (kb > kb0 && (threadIdx.x & 127) == 0) tc::mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    tc::wgmma_wait<0>();
    tc::wgmma_fence_regs(acc);
    if ((threadIdx.x & 127) == 0) tc::mbar_arrive(&empty_bar[prev]);
  }

  // -------------------------------------------------------------------- epilogue from the accumulator fragments
  // acc[4 j + e]: row 64 g + 16 (warp & 3) + lane / 4 + 8 (e >> 1), column 8 j + 2 (lane & 3) + (e & 1)
  const bool add_bias = p.bias != nullptr && split == 0;
  const bool use_aux = p.aux != nullptr && (p.act == PFN_EPI_GELU_BWD || split == 0);
  const int cq = 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = m0 + 64 * g + 16 * (warp & 3) + (lane >> 2) + 8 * h;
    const bool row_ok = row < p.M;
    float rowdot = 0.f;
    if (row_ok) {
#pragma unroll
      for (int j = 0; j < kBlockN / 8; ++j) {
        const int col = n0 + 8 * j + cq;
        if (col >= p.N) continue;
        const bool pair = col + 1 < p.N;
        float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
        if (add_bias) { f0 += __ldg(p.bias + col); if (pair) f1 += __ldg(p.bias + col + 1); }
        if (p.act == PFN_EPI_GELU) {
          if (p.C2 != nullptr) {
            __nv_bfloat16* c2 = p.C2 + static_cast<size_t>(row) * p.ldc2 + col;
            float s0 = f0, s1 = f1;
            if (p.c2_grad) { gelu_and_grad_fast(f0, f0, s0); gelu_and_grad_fast(f1, f1, s1); }
            else { f0 = gelu_fast(f0); f1 = gelu_fast(f1); }
            if (pair) *reinterpret_cast<uint32_t*>(c2) = tc::pack_bf16x2(s0, s1);
            else c2[0] = __float2bfloat16_rn(s0);
          } else {
            f0 = gelu_fast(f0); f1 = gelu_fast(f1);
          }
        }
        if (use_aux) {
          const __nv_bfloat16* ap = p.aux + static_cast<size_t>(row) * p.ld_aux + col;
          float a0, a1 = 0.f;
          if (pair) {
            const float2 t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(ap));
            a0 = t.x; a1 = t.y;
          } else {
            a0 = __bfloat162float(ap[0]);
          }
          if (p.act == PFN_EPI_GELU_BWD) {
            f0 *= gelu_grad_fast(a0); f1 *= gelu_grad_fast(a1);
          } else if (p.act == PFN_EPI_MUL) {
            f0 *= a0; f1 *= a1;
          } else if (p.act == PFN_EPI_ROWDOT) {
            // the products use the bf16-ROUNDED outputs (what the consumer of C will read), so that the row sum is
            // exactly the dot product of the stored C with aux
            rowdot = fmaf(__bfloat162float(__float2bfloat16_rn(f0)), a0, rowdot);
            if (pair) rowdot = fmaf(__bfloat162float(__float2bfloat16_rn(f1)), a1, rowdot);
          } else {
            f0 += a0; f1 += a1;
          }
        }
        if (p.c_f32) {
          float* dst = reinterpret_cast<float*>(p.C) + static_cast<size_t>(row) * p.ldc + col;
          if (p.accumulate) { atomicAdd(dst, f0); if (pair) atomicAdd(dst + 1, f1); }
          else if (pair) *reinterpret_cast<float2*>(dst) = make_float2(f0, f1);
          else dst[0] = f0;
        } else {
          __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(p.C) + static_cast<size_t>(row) * p.ldc + col;
          if (pair) *reinterpret_cast<uint32_t*>(dst) = tc::pack_bf16x2(f0, f1);
          else dst[0] = __float2bfloat16_rn(f0);
        }
      }
    }
    if (p.act == PFN_EPI_ROWDOT) {
      // the four lanes of a quad hold the same row; the tile's 128 columns lie in one group (width % 128 == 0)
      rowdot += __shfl_xor_sync(0xffffffffu, rowdot, 1);
      rowdot += __shfl_xor_sync(0xffffffffu, rowdot, 2);
      if ((lane & 3) == 0 && row_ok)
        atomicAdd(p.rowdot_out + static_cast<size_t>(row) * p.rowdot_groups + n0 / p.rowdot_width, rowdot);
    }
  }
}

template <bool A_MN, bool B_MN>
static int launch_gemm_tc(const pfn_gemm_desc* d, cudaStream_t stream) {
  CUtensorMap tmA, tmB;
  {
    uint64_t dims[2], strides[2];
    uint32_t box[2];
    if (!A_MN) { dims[0] = d->K; dims[1] = d->M; box[0] = 64; box[1] = kBlockM; }
    else       { dims[0] = d->M; dims[1] = d->K; box[0] = 64; box[1] = 64; }
    strides[0] = 0; strides[1] = static_cast<uint64_t>(d->lda) * 2;
    if (int rc = make_tensor_map_bf16(&tmA, d->A, 2, dims, strides, box, true)) return rc;
    if (!B_MN) { dims[0] = d->K; dims[1] = d->N; box[0] = 64; box[1] = kBlockN; }
    else       { dims[0] = d->N; dims[1] = d->K; box[0] = 64; box[1] = 64; }
    strides[1] = static_cast<uint64_t>(d->ldb) * 2;
    if (int rc = make_tensor_map_bf16(&tmB, d->B, 2, dims, strides, box, true)) return rc;
  }
  GemmTcParams p;
  p.M = d->M; p.N = d->N; p.K = d->K;
  p.bias = d->bias;
  p.aux = reinterpret_cast<const __nv_bfloat16*>(d->aux);
  p.ld_aux = d->ld_aux;
  p.C = d->C; p.ldc = d->ldc; p.c_f32 = d->c_dtype == PFN_F32;
  p.C2 = reinterpret_cast<__nv_bfloat16*>(d->C2); p.ldc2 = d->ldc2;
  p.act = d->epilogue;
  p.c2_grad = d->c2_gelu_grad;
  p.rowdot_out = d->rowdot_out; p.rowdot_width = d->rowdot_width > 0 ? d->rowdot_width : 1;
  p.rowdot_groups = (d->N + p.rowdot_width - 1) / p.rowdot_width;
  p.tiles_m = (d->M + kBlockM - 1) / kBlockM;
  p.tiles_n = (d->N + kBlockN - 1) / kBlockN;
  const int num_kb = (d->K + kBlockK - 1) / kBlockK;
  int splits = d->k_splits <= 0 ? 1 : d->k_splits;
  if (splits > num_kb) splits = num_kb;
  const int per = (num_kb + splits - 1) / splits;
  splits = (num_kb + per - 1) / per;
  p.kb_per_split = per;
  p.accumulate = (d->accumulate || splits > 1) ? 1 : 0;
  PFN_CHECK_ARG(!p.accumulate || p.c_f32, "gemm_tc: accumulate / split-K requires an fp32 output");
  const long long total = static_cast<long long>(p.tiles_m) * p.tiles_n * splits;
  PFN_CHECK_ARG(total < (1LL << 31), "gemm_tc: too many tiles");
  auto kern = gemm_tc_kernel<A_MN, B_MN>;
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set)) {
    PFN_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
  }
  kern<<<static_cast<unsigned>(total), kNumThreads, kSmemBytes, stream>>>(tmA, tmB, p);
  PFN_LAUNCH_OK();
  return 0;
}

}  // namespace pfn

extern "C" int pfn_gemm_bf16_tc(const pfn_gemm_desc* d, void* stream) {
  using namespace pfn;
  PFN_CHECK_ARG(d != nullptr, "gemm_tc: null descriptor");
  PFN_CHECK_ARG(d->M > 0 && d->N > 0 && d->K > 0, "gemm_tc: empty problem %d x %d x %d", d->M, d->N, d->K);
  PFN_CHECK_ARG(d->lda % 8 == 0 && d->ldb % 8 == 0, "gemm_tc: lda/ldb must be multiples of 8 elements (got %d, %d)",
                d->lda, d->ldb);
  PFN_CHECK_ARG(d->epilogue >= 0 && d->epilogue <= PFN_EPI_MUL, "gemm_tc: bad epilogue %d", d->epilogue);
  PFN_CHECK_ARG(d->epilogue != PFN_EPI_MUL || (d->aux != nullptr && d->k_splits <= 1 && !d->accumulate), "gemm_tc: MUL epilogue needs aux and no split-K");
  PFN_CHECK_ARG(!d->c2_gelu_grad || (d->epilogue == PFN_EPI_GELU && d->C2 != nullptr), "gemm_tc: c2_gelu_grad needs the GELU epilogue with C2");
  PFN_CHECK_ARG(d->epilogue != PFN_EPI_ROWDOT || (d->aux != nullptr && d->rowdot_out != nullptr && d->rowdot_width >= 128 &&
                                                  d->rowdot_width % 128 == 0 && d->k_splits <= 1 && !d->accumulate),
                "gemm_tc: ROWDOT epilogue needs aux, rowdot_out, a group width that is a multiple of 128 and no split-K");
  PFN_CHECK_ARG(d->epilogue != PFN_EPI_GELU_BWD || d->aux != nullptr, "gemm_tc: GELU' epilogue needs aux = pre-activation");
  const bool vec_ok = (d->c_dtype == PFN_F32 ? d->ldc % 4 == 0 : d->ldc % 8 == 0) &&
                      (reinterpret_cast<uintptr_t>(d->C) & 15) == 0;
  PFN_CHECK_ARG(vec_ok, "gemm_tc: C must be 16-byte aligned with ldc multiple of 16 bytes");
  PFN_CHECK_ARG(d->aux == nullptr || (d->ld_aux % 8 == 0 && (reinterpret_cast<uintptr_t>(d->aux) & 15) == 0),
                "gemm_tc: aux must be 16-byte aligned with ld multiple of 8");
  PFN_CHECK_ARG(d->C2 == nullptr || (d->ldc2 % 8 == 0 && (reinterpret_cast<uintptr_t>(d->C2) & 15) == 0),
                "gemm_tc: C2 must be 16-byte aligned with ld multiple of 8");
  PFN_CHECK_ARG(d->bias == nullptr || (reinterpret_cast<uintptr_t>(d->bias) & 15) == 0, "gemm_tc: bias must be 16-byte aligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  switch ((d->a_mn_major ? 2 : 0) | (d->b_mn_major ? 1 : 0)) {
    case 0: return launch_gemm_tc<false, false>(d, s);
    case 1: return launch_gemm_tc<false, true>(d, s);
    case 2: return launch_gemm_tc<true, false>(d, s);
    default: return launch_gemm_tc<true, true>(d, s);
  }
}
