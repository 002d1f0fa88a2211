// Library runtime: error string, device query cache, TMA tensor-map encoding.
#include <stdarg.h>
#include <mutex>

#include "common.cuh"
#include "tc_common.cuh"
#include "../../include/pfn_b200.h"

namespace pfn {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* get_error() { return g_err; }

int num_sms() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<EncodeTiledFn>(p);
    }
  });
  return fn;
}

int make_tensor_map(CUtensorMap* out, const void* base, bool f32, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes, const uint32_t* box, bool swizzle128) {
  EncodeTiledFn fn = get_encode_fn();
  PFN_CHECK_ARG(fn != nullptr, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  PFN_CHECK_ARG((reinterpret_cast<uintptr_t>(base) & 15) == 0, "TMA base pointer %p not 16-byte aligned", base);
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bx[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    estr[i] = 1;
    if (i > 0) {
      PFN_CHECK_ARG((strides_bytes[i] & 15) == 0, "TMA stride %llu (dim %d) not a multiple of 16 bytes",
                    (unsigned long long)strides_bytes[i], i);
      gstr[i - 1] = strides_bytes[i];
    }
  }
  CUresult r = fn(out, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16,
                  static_cast<cuuint32_t>(rank), const_cast<void*>(base), gdim,
                  gstr, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  PFN_CHECK_ARG(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims %llu,%llu box %u,%u)",
                (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0), box[0],
                rank > 1 ? box[1] : 0);
  return 0;
}

}  // namespace pfn

extern "C" {
const char* pfn_last_error(void) { return pfn::get_error(); }
int pfn_version(void) { return PFN_B200_VERSION; }
int pfn_num_sms(void) { return pfn::num_sms(); }
}
