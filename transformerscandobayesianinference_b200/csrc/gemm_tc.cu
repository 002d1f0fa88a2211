// Persistent ping-pong TMA + wgmma GEMM for sm_90a.
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
// Structure: one CTA per SM walks a static schedule of work units (128 x 128 output tile, k-split), unit += gridDim.
// Units are numbered split-major and, inside a split, row-major over the tiles (n fastest), so the CTAs working at the
// same time read the same A row blocks and the same k range: A comes from HBM about once.
//   warpgroup 2 (producer, 40 registers) : one thread issues the TMA loads of every unit of the CTA into a kStages ring,
//                                          running ahead across unit boundaries, plus each unit's aux block into the
//                                          staging buffer of the warpgroup that will run its epilogue
//   warpgroups 0, 1 (consumers, 232 registers) : the CTA's units alternate between them (ping-pong).  A consumer runs the
//                                          whole 128 x 128 tile (2 x wgmma m64n128k16 per k16 step, 128 fp32 accumulators
//                                          per thread) and then its epilogue, while the other warpgroup runs the next
//                                          unit's main loop.  A pair of named barriers hands the tensor pipe over, so the
//                                          two main loops never interleave.
// Epilogue (bias / GELU / residual / GELU' / product / row dot) per warp on its 32 rows: aux is read from the staging
// buffer the TMA filled during the main loop, bias from shared memory, and the results (C2, then C) are written back to
// the same staging buffer and leave with TMA tile stores (bf16, fp32) or TMA fp32 reduce-adds (split-K / accumulate).
// The TMA clips the ragged M / N edges, so nothing outside [M, N] is written.
#include "common.cuh"
#include "tc_common.cuh"
#include "../../include/pfn_b200.h"

namespace pfn {

struct GemmTcParams {
  int M, N;
  const float* bias;             // [N] fp32 or null (added in split 0)
  int has_aux;                   // aux tensor map is valid
  int aux_all_splits;            // GELU': every split scales by gelu'(aux); otherwise aux enters split 0 only
  int c_f32;                     // 1 => C is fp32
  int accumulate;                // 1 => fp32 reduce-add into C (split-K / grad accumulation)
  int num_kb;                    // k-blocks (of 64) in K
  int kb_per_split;              // k-blocks per split
  int tiles_n, tiles;            // output tiles along N, in total
  int units;                     // tiles * splits
  float* rowdot_out;             // PFN_EPI_ROWDOT: [M, rowdot_groups] fp32, += sum over a column group of C * aux
  int rowdot_width, rowdot_groups;
};

// Epilogue kinds, one kernel instantiation each (two where aux is an optional residual: with and without it): the
// epilogue is unrolled over the 128 accumulators of a thread, and keeping only the active variant keeps the kernel's
// code inside the instruction cache.
enum EpiKind : int { kEpiNone, kEpiGelu, kEpiGeluPre, kEpiGeluGrad, kEpiGeluBwd, kEpiRowdot, kEpiMul };

constexpr int kBlockM = 128;
constexpr int kBlockN = 128;
constexpr int kBlockK = 64;
constexpr int kStages = 5;
constexpr int kABytes = kBlockM * kBlockK * 2;        // 16 KB
constexpr int kBBytes = kBlockN * kBlockK * 2;        // 16 KB
constexpr int kOutBytes = kBlockM * kBlockN * 2;      // 32 KB staging per consumer warpgroup (a bf16 tile)
constexpr int kNumThreads = 3 * 128;
constexpr int kOffB = kStages * kABytes;
constexpr int kOffOut = kStages * (kABytes + kBBytes);
constexpr int kOffBias = kOffOut + 2 * kOutBytes;
constexpr int kOffBar = kOffBias + 2 * kBlockN * 4;
constexpr int kNumBars = 2 * kStages + 4;
constexpr int kSmemBytes = kOffBar + kNumBars * 8 + 1024;   // + 1 KB alignment slack (128-byte swizzle atoms)
static_assert(kSmemBytes <= 232448, "the ring, two staging buffers and the barriers must fit the 227 KB of shared memory");

struct Unit {
  int m0, n0, kb0, nkb, split;
};
__device__ __forceinline__ Unit unit_at(const GemmTcParams& p, int u) {
  Unit w;
  w.split = u / p.tiles;
  const int tile = u - w.split * p.tiles;
  w.m0 = (tile / p.tiles_n) * kBlockM;
  w.n0 = (tile % p.tiles_n) * kBlockN;
  w.kb0 = w.split * p.kb_per_split;
  w.nkb = min(p.kb_per_split, p.num_kb - w.kb0);
  return w;
}

// The epilogue math of one accumulator pair (columns col, col + 1 of one row), in the order of the reference formula.
// `ep` is the pair's slot in the staging buffer: it holds aux on entry and receives C2.  The code is branch-free, so that
// the compiler can issue the staging-buffer loads of many pairs ahead of their use:
//   - the bias is always added: sBias holds -0.0f where no bias applies, and x + (-0.0f) == x for every x, -0.0f
//     included;
//   - with AUX the aux pair is always loaded (the slot lies inside the staging buffer whatever its contents) and then
//     selected: where it does not apply (past N, or a split-K unit other than the first) it is -0.0f, again an exact
//     identity for the residual add.  The other aux kinds (GELU', MUL, ROWDOT) use aux in every unit, and their columns
//     past N are neither stored (the TMA clips them) nor summed (ROWDOT checks col).
template <int EPI, bool AUX>
__device__ __forceinline__ void epi_pair(const GemmTcParams& p, float& f0, float& f1, float2 b, bool use_aux,
                                         uint8_t* ep, int col, float& rowdot) {
  float a0 = -0.f, a1 = -0.f;
  if constexpr (AUX) {
    const float2 t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(ep));
    a0 = use_aux ? t.x : -0.f;
    a1 = use_aux ? t.y : -0.f;
  }
  f0 += b.x; f1 += b.y;
  if constexpr (EPI == kEpiGeluPre || EPI == kEpiGeluGrad) {
    float s0 = f0, s1 = f1;
    if constexpr (EPI == kEpiGeluGrad) { gelu_and_grad_fast(f0, f0, s0); gelu_and_grad_fast(f1, f1, s1); }
    else { f0 = gelu_fast(f0); f1 = gelu_fast(f1); }
    *reinterpret_cast<uint32_t*>(ep) = tc::pack_bf16x2(s0, s1);
  } else if constexpr (EPI == kEpiGelu) {
    f0 = gelu_fast(f0); f1 = gelu_fast(f1);
  }
  if constexpr (AUX) {
    if constexpr (EPI == kEpiGeluBwd) {
      f0 *= gelu_grad_fast(a0); f1 *= gelu_grad_fast(a1);
    } else if constexpr (EPI == kEpiMul) {
      f0 *= a0; f1 *= a1;
    } else if constexpr (EPI == kEpiRowdot) {
      // the products use the bf16-ROUNDED outputs (what the consumer of C will read), so that the row sum is exactly
      // the dot product of the stored C with aux; columns past N may hold a previous tile's staging data
      if (col < p.N) rowdot = fmaf(__bfloat162float(__float2bfloat16_rn(f0)), a0, rowdot);
      if (col + 1 < p.N) rowdot = fmaf(__bfloat162float(__float2bfloat16_rn(f1)), a1, rowdot);
    } else {
      // __fadd_rn: never contracted into an FMA with the GELU's last multiply, so C rounds as a separate add
      f0 = __fadd_rn(f0, a0); f1 = __fadd_rn(f1, a1);
    }
  }
}

template <bool A_MN, bool B_MN, int EPI, bool AUX>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmAux, const __grid_constant__ CUtensorMap tmC,
               const __grid_constant__ CUtensorMap tmC2, const GemmTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  // 1 KB alignment (128-byte swizzle atoms) by an offset on the __shared__ symbol
  uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sA = smem;
  uint8_t* sB = smem + kOffB;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kOffBar);
  uint64_t* empty_bar = full_bar + kStages;
  uint64_t* aux_bar = empty_bar + kStages;      // [2] aux block of the warpgroup's current unit has landed
  uint64_t* free_bar = aux_bar + 2;             // [2] the warpgroup's staging buffer is free again (one arrival per warp)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      tc::mbar_init(&full_bar[s], 1);
      tc::mbar_init(&empty_bar[s], 1);
    }
    for (int g = 0; g < 2; ++g) {
      tc::mbar_init(&aux_bar[g], 1);
      tc::mbar_init(&free_bar[g], 4);
    }
    tc::mbar_fence_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // ------------------------------------------------------------------ TMA producer
    tc::setmaxnreg_dec<40>();
    if (threadIdx.x == 256) {
      tc::tma_prefetch_desc(&tmA);
      tc::tma_prefetch_desc(&tmB);
      if (p.has_aux) tc::tma_prefetch_desc(&tmAux);
      int stage = 0;
      uint32_t phase = 0;
      for (int u = blockIdx.x, i = 0; u < p.units; u += gridDim.x, ++i) {
        const int g = i & 1;
        const Unit w = unit_at(p, u);
        // The staging buffer is claimed before the unit's last k-block is issued: the warpgroup cannot finish this unit (and
        // free the buffer once more) before that, so the parity below never refers to a phase two completions old.  The
        // warpgroup's previous unit is the CTA's unit i - 2, its (i / 2 - 1)-th.
        const int claim_at = min(kStages, w.nkb) - 1;
        for (int kb = 0; kb < w.nkb; ++kb) {
          if (kb == claim_at) {
            if (i >= 2) tc::mbar_wait_suspend(&free_bar[g], ((i >> 1) - 1) & 1);
            if (p.has_aux && (p.aux_all_splits || w.split == 0)) {
              uint8_t* dst = smem + kOffOut + g * kOutBytes;
              const int halves = w.n0 + 64 < p.N ? 2 : 1;
              tc::mbar_expect_tx(&aux_bar[g], halves * (kOutBytes / 2));
              for (int h = 0; h < halves; ++h)
                tc::tma_load_2d(dst + h * (kOutBytes / 2), &tmAux, &aux_bar[g], w.n0 + 64 * h, w.m0);
            }
          }
          tc::mbar_wait_suspend(&empty_bar[stage], phase ^ 1);
          uint8_t* a_dst = sA + stage * kABytes;
          uint8_t* b_dst = sB + stage * kBBytes;
          const int k0 = (w.kb0 + kb) * kBlockK;
          tc::mbar_expect_tx(&full_bar[stage], kABytes + kBBytes);
          if constexpr (!A_MN) {
            tc::tma_load_2d(a_dst, &tmA, &full_bar[stage], k0, w.m0);
          } else {
            tc::tma_load_2d(a_dst, &tmA, &full_bar[stage], w.m0, k0);
            tc::tma_load_2d(a_dst + 8192, &tmA, &full_bar[stage], w.m0 + 64, k0);
          }
          if constexpr (!B_MN) {
            tc::tma_load_2d(b_dst, &tmB, &full_bar[stage], k0, w.n0);
          } else {
            tc::tma_load_2d(b_dst, &tmB, &full_bar[stage], w.n0, k0);
            tc::tma_load_2d(b_dst + 8192, &tmB, &full_bar[stage], w.n0 + 64, k0);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroups
  tc::setmaxnreg_inc<232>();
  const int g = warp >> 2;                 // consumer warpgroup: runs the CTA's units i with i % 2 == g
  const int wq = warp & 3;                 // warp inside the warpgroup: tile rows 16 wq + [0, 16) and 64 + 16 wq + [0, 16)
  const int tid = threadIdx.x & 127;
  uint8_t* sOut = smem + kOffOut + g * kOutBytes;
  float* sBias = reinterpret_cast<float*>(smem + kOffBias) + g * kBlockN;
  const int rl = lane >> 2, q = lane & 3;
  // Staging layout (the TMA's 128-byte swizzle): column half hc (64 bf16 = 128 B per row) at hc * 16 KB, rows at 128 B,
  // 16-byte chunk c of row r at chunk c ^ (r & 7).  The warp's 16-row slab of m-half mh starts at (4 mh + wq) * 2 KB, so
  // each warp stores its own boxes of 16 rows.  Accumulator acc_mh[4 j + e] is tile row 64 mh + 16 wq + rl + 8 (e >> 1),
  // column 8 j + 2 q + (e & 1); rl == r & 7, so the eight rows of one store hit eight different chunks (no bank conflict).
  uint8_t* wslab = sOut + wq * 2048 + rl * 128;
  int kb_count = 0, aux_count = 0;
  float acc0[64], acc1[64];
  for (int u = blockIdx.x, i = 0; u < p.units; u += gridDim.x, ++i) {
    const Unit w = unit_at(p, u);
    if ((i & 1) != g) { kb_count += w.nkb; continue; }
    const bool add_bias = p.bias != nullptr && w.split == 0;
    const float bias_v = add_bias && w.n0 + tid < p.N ? __ldg(p.bias + w.n0 + tid) : -0.f;   // -0: see epi_pair
    // the other warpgroup has drained its main loop (and this warpgroup has left its previous epilogue: all 128 threads
    // take part in the barrier, so sBias is free)
    if (i > 0) tc::named_bar_sync(1 + g, 256);
    sBias[tid] = bias_v;

    // ------------------------------------------------------------------ main loop
    // The first MMA of the tile writes the accumulator (scale-d = 0), so nothing but wgmma defines `acc` until the pipeline
    // has drained: any other definition inside it makes ptxas serialise the wgmma instructions.
    {
      int stage = kb_count % kStages, prev = 0;
      uint32_t phase = (kb_count / kStages) & 1;
      for (int kb = 0; kb < w.nkb; ++kb) {
        tc::mbar_wait(&full_bar[stage], phase);
        const uint32_t a_addr = tc::smem_u32(sA + stage * kABytes);     // K-major: rows 64 mh.. at +8 KB; MN-major: chunk mh
        const uint32_t b_addr = tc::smem_u32(sB + stage * kBBytes);
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k) {
          // K-major: advance 16 elements (32 B) inside the 128 B swizzle row.
          // MN-major: advance 16 k-rows (16 * 128 B); LBO = stride between 64-wide M/N chunks.
          const uint32_t a_off = A_MN ? k * 2048 : k * 32;
          const uint64_t a_desc0 = A_MN ? tc::wgmma_smem_desc(a_addr + a_off, 8192, 1024) : tc::wgmma_smem_desc(a_addr + a_off, 16, 1024);
          const uint64_t a_desc1 = A_MN ? tc::wgmma_smem_desc(a_addr + 8192 + a_off, 8192, 1024)
                                        : tc::wgmma_smem_desc(a_addr + 8192 + a_off, 16, 1024);
          const uint64_t b_desc = B_MN ? tc::wgmma_smem_desc(b_addr + k * 2048, 8192, 1024)
                                       : tc::wgmma_smem_desc(b_addr + k * 32, 16, 1024);
          const uint32_t accum = (kb > 0 || k > 0) ? 1u : 0u;
          tc::wgmma_m64n128k16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc0, a_desc0, b_desc, accum);
          tc::wgmma_m64n128k16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc1, a_desc1, b_desc, accum);
        }
        tc::wgmma_commit();
        tc::wgmma_wait<1>();               // the previous k-block's MMAs are done: its stage can be refilled
        if (kb > 0 && tid == 0) tc::mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      tc::wgmma_wait<0>();
      tc::wgmma_fence_regs(acc0);
      tc::wgmma_fence_regs(acc1);
      if (tid == 0) tc::mbar_arrive(&empty_bar[prev]);
      kb_count += w.nkb;
    }
    // hand the tensor pipe to the other warpgroup (if the CTA has a next unit), then the epilogue
    if (u + static_cast<int>(gridDim.x) < p.units) tc::named_bar_arrive(2 - g, 256);
    tc::named_bar_sync(3 + g, 128);        // sBias written by the whole warpgroup

    // ------------------------------------------------------------------ epilogue, per warp
    const bool use_aux = p.has_aux && (p.aux_all_splits || w.split == 0);
    if (use_aux) { tc::mbar_wait(&aux_bar[g], aux_count & 1); ++aux_count; }
    float rowdot[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
    for (int j = 0; j < kBlockN / 8; ++j) {
      const int col = w.n0 + 8 * j + 2 * q;
      const float2 b = *reinterpret_cast<const float2*>(sBias + 8 * j + 2 * q);
      // aux past N is zero (TMA fill) or, for a column half the producer skipped, stale: read it only inside N
      const bool aux_j = use_aux && col < p.N;
#pragma unroll
      for (int mh = 0; mh < 2; ++mh) {
        float* acc = mh ? acc1 : acc0;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          uint8_t* ep = wslab + (j >> 3) * 16384 + mh * 8192 + h * 1024 + (((j & 7) ^ rl) << 4) + 4 * q;
          epi_pair<EPI, AUX>(p, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], b, aux_j, ep, col, rowdot[mh][h]);
        }
      }
    }
    if constexpr (EPI == kEpiRowdot) {
      // the four lanes of a quad hold the same row; the tile's 128 columns lie in one group (width % 128 == 0)
#pragma unroll
      for (int mh = 0; mh < 2; ++mh) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float r = rowdot[mh][h];
          r += __shfl_xor_sync(0xffffffffu, r, 1);
          r += __shfl_xor_sync(0xffffffffu, r, 2);
          const int row = w.m0 + 64 * mh + 16 * wq + rl + 8 * h;
          if (q == 0 && row < p.M)
            atomicAdd(p.rowdot_out + static_cast<size_t>(row) * p.rowdot_groups + w.n0 / p.rowdot_width, r);
        }
      }
    }
    // the warp's four boxes of 16 rows x 64 bf16 (C2 and bf16 C) or 16 rows x 32 fp32 (one half of fp32 C)
    auto store_boxes = [&](const CUtensorMap* map, int col0, int box_cols, bool reduce) {
      tc::fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) {
#pragma unroll
        for (int mh = 0; mh < 2; ++mh) {
          const int r0 = w.m0 + 64 * mh + 16 * wq;
#pragma unroll
          for (int hc = 0; hc < 2; ++hc) {
            const int c0 = w.n0 + col0 + hc * box_cols;
            if (r0 >= p.M || c0 >= p.N) continue;
            const uint8_t* src = sOut + hc * 16384 + (4 * mh + wq) * 2048;
            if (reduce) tc::tma_reduce_add_2d(map, src, c0, r0);
            else tc::tma_store_2d(map, src, c0, r0);
          }
        }
        tc::bulk_commit();
        tc::bulk_wait_read<0>();
      }
      __syncwarp();
    };
    if constexpr (EPI == kEpiGeluPre || EPI == kEpiGeluGrad) store_boxes(&tmC2, 0, 64, false);
    if (!p.c_f32) {
#pragma unroll
      for (int j = 0; j < kBlockN / 8; ++j) {
#pragma unroll
        for (int mh = 0; mh < 2; ++mh) {
          const float* acc = mh ? acc1 : acc0;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            uint8_t* ep = wslab + (j >> 3) * 16384 + mh * 8192 + h * 1024 + (((j & 7) ^ rl) << 4) + 4 * q;
            *reinterpret_cast<uint32_t*>(ep) = tc::pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
          }
        }
      }
      store_boxes(&tmC, 0, 64, false);
    } else {
      // fp32: two passes of 64 columns; a box row is 32 fp32 (128 B), column quarter hc of the pass at hc * 16 KB
      __syncwarp();                        // every lane has read its aux before the fp32 layout overwrites the slab
#pragma unroll
      for (int pass = 0; pass < 2; ++pass) {
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int j = 8 * pass + jj;
          const int chunk = 2 * (jj & 3) + (q >> 1);
#pragma unroll
          for (int mh = 0; mh < 2; ++mh) {
            const float* acc = mh ? acc1 : acc0;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              uint8_t* ep = wslab + (jj >> 2) * 16384 + mh * 8192 + h * 1024 + ((chunk ^ rl) << 4) + 8 * (q & 1);
              *reinterpret_cast<float2*>(ep) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
          }
        }
        store_boxes(&tmC, 64 * pass, 32, p.accumulate != 0);
      }
    }
    // the staging buffer may take the next aux block
    if (lane == 0) tc::mbar_arrive(&free_bar[g]);
  }
  if (lane == 0) tc::bulk_wait<0>();
}

template <bool A_MN, bool B_MN, int EPI, bool AUX>
static int launch_gemm_tc(const pfn_gemm_desc* d, cudaStream_t stream) {
  CUtensorMap tmA, tmB, tmAux, tmC, tmC2;
  memset(&tmAux, 0, sizeof(tmAux));
  memset(&tmC2, 0, sizeof(tmC2));
  const bool c_f32 = d->c_dtype == PFN_F32;
  {
    uint64_t dims[2], strides[2];
    uint32_t box[2];
    if (!A_MN) { dims[0] = d->K; dims[1] = d->M; box[0] = 64; box[1] = kBlockM; }
    else       { dims[0] = d->M; dims[1] = d->K; box[0] = 64; box[1] = 64; }
    strides[0] = 0; strides[1] = static_cast<uint64_t>(d->lda) * 2;
    if (int rc = make_tensor_map(&tmA, d->A, false, 2, dims, strides, box, true)) return rc;
    if (!B_MN) { dims[0] = d->K; dims[1] = d->N; box[0] = 64; box[1] = kBlockN; }
    else       { dims[0] = d->N; dims[1] = d->K; box[0] = 64; box[1] = 64; }
    strides[1] = static_cast<uint64_t>(d->ldb) * 2;
    if (int rc = make_tensor_map(&tmB, d->B, false, 2, dims, strides, box, true)) return rc;
    // epilogue tensors: [M, N] row-major with a leading dimension
    dims[0] = d->N; dims[1] = d->M;
    box[0] = c_f32 ? 32 : 64; box[1] = 16;
    strides[1] = static_cast<uint64_t>(d->ldc) * (c_f32 ? 4 : 2);
    if (int rc = make_tensor_map(&tmC, d->C, c_f32, 2, dims, strides, box, true)) return rc;
    box[0] = 64;
    if (d->C2 != nullptr) {
      strides[1] = static_cast<uint64_t>(d->ldc2) * 2;
      if (int rc = make_tensor_map(&tmC2, d->C2, false, 2, dims, strides, box, true)) return rc;
    }
    if (d->aux != nullptr) {
      box[1] = kBlockM;
      strides[1] = static_cast<uint64_t>(d->ld_aux) * 2;
      if (int rc = make_tensor_map(&tmAux, d->aux, false, 2, dims, strides, box, true)) return rc;
    }
  }
  GemmTcParams p;
  p.M = d->M; p.N = d->N;
  p.bias = d->bias;
  p.has_aux = d->aux != nullptr;
  p.aux_all_splits = d->epilogue == PFN_EPI_GELU_BWD;
  p.c_f32 = c_f32;
  p.rowdot_out = d->rowdot_out; p.rowdot_width = d->rowdot_width > 0 ? d->rowdot_width : 1;
  p.rowdot_groups = (d->N + p.rowdot_width - 1) / p.rowdot_width;
  const int tiles_m = (d->M + kBlockM - 1) / kBlockM;
  p.tiles_n = (d->N + kBlockN - 1) / kBlockN;
  const int num_kb = (d->K + kBlockK - 1) / kBlockK;
  int splits = d->k_splits <= 0 ? 1 : d->k_splits;
  if (splits > num_kb) splits = num_kb;
  const int per = (num_kb + splits - 1) / splits;
  splits = (num_kb + per - 1) / per;
  p.num_kb = num_kb;
  p.kb_per_split = per;
  p.accumulate = (d->accumulate || splits > 1) ? 1 : 0;
  PFN_CHECK_ARG(!p.accumulate || p.c_f32, "gemm_tc: accumulate / split-K requires an fp32 output");
  const long long tiles = static_cast<long long>(tiles_m) * p.tiles_n;
  const long long total = tiles * splits;
  PFN_CHECK_ARG(total < (1LL << 31), "gemm_tc: too many tiles");
  p.tiles = static_cast<int>(tiles);
  p.units = static_cast<int>(total);
  auto kern = gemm_tc_kernel<A_MN, B_MN, EPI, AUX>;
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set)) {
    PFN_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
  }
  const int grid = p.units < num_sms() ? p.units : num_sms();
  kern<<<static_cast<unsigned>(grid), kNumThreads, kSmemBytes, stream>>>(tmA, tmB, tmAux, tmC, tmC2, p);
  PFN_LAUNCH_OK();
  return 0;
}

template <int EPI, bool AUX>
static int launch_layout(const pfn_gemm_desc* d, cudaStream_t s) {
  switch ((d->a_mn_major ? 2 : 0) | (d->b_mn_major ? 1 : 0)) {
    case 0: return launch_gemm_tc<false, false, EPI, AUX>(d, s);
    case 1: return launch_gemm_tc<false, true, EPI, AUX>(d, s);
    case 2: return launch_gemm_tc<true, false, EPI, AUX>(d, s);
    default: return launch_gemm_tc<true, true, EPI, AUX>(d, s);
  }
}

// the epilogue kinds whose aux is optional (a residual added last) have one instantiation without it and one with it
template <int EPI>
static int launch_aux(const pfn_gemm_desc* d, cudaStream_t s) {
  return d->aux != nullptr ? launch_layout<EPI, true>(d, s) : launch_layout<EPI, false>(d, s);
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
  int epi = kEpiNone;
  switch (d->epilogue) {
    case PFN_EPI_GELU: epi = d->C2 == nullptr ? kEpiGelu : d->c2_gelu_grad ? kEpiGeluGrad : kEpiGeluPre; break;
    case PFN_EPI_GELU_BWD: epi = kEpiGeluBwd; break;
    case PFN_EPI_ROWDOT: epi = kEpiRowdot; break;
    case PFN_EPI_MUL: epi = kEpiMul; break;
    default: break;
  }
  switch (epi) {
    case kEpiGelu: return launch_aux<kEpiGelu>(d, s);
    case kEpiGeluPre: return launch_aux<kEpiGeluPre>(d, s);
    case kEpiGeluGrad: return launch_aux<kEpiGeluGrad>(d, s);
    case kEpiGeluBwd: return launch_layout<kEpiGeluBwd, true>(d, s);      // aux is required (checked above)
    case kEpiRowdot: return launch_layout<kEpiRowdot, true>(d, s);
    case kEpiMul: return launch_layout<kEpiMul, true>(d, s);
    default: return launch_aux<kEpiNone>(d, s);
  }
}
