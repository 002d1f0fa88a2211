// Stroke prior (reference priors/stroke.py:9-116): synthetic handwriting classes drawn and blurred on the device.
//
//   geometry : one thread per (dataset, class, stroke) runs the reference's rejection loop for that stroke (:24-37) --
//              length and start redrawn on iterations 0, 3, 6, ..., a direction on every iteration, accepted when the
//              unrounded end point lies in [0, S-1]^2 -- capped at `max_iters` iterations; a capped stroke raises *cap_flag
//              and keeps its last draw.
//   render   : one warp per image (t, b) of class cls[t, b] (:45-60): width, offset and per-stroke jitter, end points
//              rounded half to even, the strokes rasterised like Pillow's ImageDraw.line into shared memory, ink pixels
//              filled with U{200..254}, GaussianBlur(0.2), then x[t, b, :] = k / 255 (ToTensor) and optionally
//              (x - mean) / (std + 1e-6) per image.  Written straight into the sequence-first [T, B, S*S] layout.
//
// Random numbers are counter-based hashes of (seed, dataset, class, stroke, iteration) and (seed, position, dataset,
// stroke or pixel), so a batch is a pure function of its seed and the draw order of threads does not matter.
#include "common.cuh"
#include "counter_rng.cuh"
#include "stroke_raster.cuh"
#include "../../include/pfn_b200.h"

namespace pfn {
namespace {

enum : uint32_t { TAG_NSTROKES = 1, TAG_LEN, TAG_SX, TAG_SY, TAG_RAD_HI, TAG_RAD_LO, TAG_WIDTH, TAG_OFFX, TAG_OFFY,
                  TAG_JITX, TAG_JITY, TAG_FILL };

constexpr int kWarpsPerBlock = 8;
constexpr int kSegBytes = PFN_STROKE_MAX_STROKES * 16;     // per warp: staged segments, then the image and its blur scratch

__host__ __device__ __forceinline__ int warp_smem(int S) { return kSegBytes + ((2 * S * S + 15) & ~15); }

__global__ void __launch_bounds__(128)
stroke_geometry_kernel(pfn_stroke_desc d, uint32_t seed, int B, int* __restrict__ geom, double* __restrict__ turns,
                       int* __restrict__ cap_flag) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int smax = d.strokes_max;
  if (idx >= B * d.C * smax) return;
  const int s = idx % smax, bc = idx / smax;
  const uint32_t b = static_cast<uint32_t>(bc / d.C), c = static_cast<uint32_t>(bc % d.C);
  const int n = uniform_int(hash5(seed, TAG_NSTROKES, b, c, 0), d.strokes_min, d.strokes_max);
  int* g = geom + static_cast<size_t>(idx) * 4;
  if (s >= n) {
    g[0] = g[1] = g[2] = g[3] = 0;
    turns[idx] = 0.0;
    return;
  }
  const uint32_t cs = c * 64u + static_cast<uint32_t>(s);
  const double lim = static_cast<double>(d.S - 1);
  int len = 0, sx = 0, sy = 0;
  double turn = 0.0;
  bool ok = false;
  for (int it = 0; it < d.max_iters && !ok; ++it) {
    const uint32_t u = static_cast<uint32_t>(it);
    if (it % 3 == 0) {
      len = uniform_int(hash5(seed, TAG_LEN, b, cs, u), d.len_min, d.len_max);
      sx = uniform_int(hash5(seed, TAG_SX, b, cs, u), d.start_min, d.start_max);
      sy = uniform_int(hash5(seed, TAG_SY, b, cs, u), d.start_min, d.start_max);
    }
    // radians = 2 pi turn; sincospi needs no large-argument reduction (no local-memory table)
    turn = uniform_double(hash5(seed, TAG_RAD_HI, b, cs, u), hash5(seed, TAG_RAD_LO, b, cs, u));
    double sn, cn;
    sincospi(2.0 * turn, &sn, &cn);
    const double ex = sx + cn * len, ey = sy + sn * len;
    ok = ex >= 0.0 && ex <= lim && ey >= 0.0 && ey <= lim;
  }
  if (!ok) atomicOr(cap_flag, 1);
  g[0] = sx; g[1] = sy; g[2] = len; g[3] = 1;
  turns[idx] = turn;
}

// Draw the strokes (bit s of `valid` set) of one image into img (0 / 1 mask; the caller zeroed it).  Stroke s starts its
// rows at lane s, so the serial thin lines of different strokes run on different lanes.
__device__ __forceinline__ void raster_warp(uint8_t* img, int S, const int4* seg, uint32_t valid, int width, int lane) {
  for (int s = 0; s < PFN_STROKE_MAX_STROKES; ++s)
    if ((valid >> s) & 1u)
      stroke::draw_line(img, S, seg[s].x, seg[s].y, seg[s].z, seg[s].w, width, 1, (lane + 32 - s) & 31, 32);
}

// Blur a (uint8, S x S) in place with b as scratch: three passes along rows, three along columns.
__device__ __forceinline__ void blur_warp(uint8_t* a, uint8_t* b, int S, int lane) {
  const int n = S * S;
  uint8_t* src = a;
  uint8_t* dst = b;
  for (int pass = 0; pass < 2 * stroke::kBlurPasses; ++pass) {
    const bool rows = pass < stroke::kBlurPasses;
    for (int p = lane; p < n; p += 32) {
      const int r = p / S, col = p - r * S;
      dst[p] = rows ? stroke::blur_tap(src + r * S, col, S, 1) : stroke::blur_tap(src + col, r, S, S);
    }
    __syncwarp();
    uint8_t* t = src; src = dst; dst = t;
  }
  static_assert(stroke::kBlurPasses % 2 == 1, "an even total number of passes leaves the result in a");
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32)
stroke_render_kernel(pfn_stroke_desc d, uint32_t seed, const int* __restrict__ cls, const int* __restrict__ geom,
                     const double* __restrict__ turns, float* __restrict__ x, int T, int B, int normalize) {
  extern __shared__ uint8_t smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int S = d.S, n = S * S;
  int4* seg = reinterpret_cast<int4*>(smem + warp * warp_smem(S));
  uint8_t* img = reinterpret_cast<uint8_t*>(seg + PFN_STROKE_MAX_STROKES);
  uint8_t* tmp = img + n;
  const int image = blockIdx.x * kWarpsPerBlock + warp;
  if (image >= T * B) return;
  const uint32_t t = static_cast<uint32_t>(image / B), b = static_cast<uint32_t>(image % B);
  const int c = cls[image];

  for (int p = lane; p < n; p += 32) img[p] = 0;
  const int width = uniform_int(hash5(seed, TAG_WIDTH, t, b, 0), d.width_min, d.width_max);
  const int ox = uniform_int(hash5(seed, TAG_OFFX, t, b, 0), d.offset_min, d.offset_max);
  const int oy = uniform_int(hash5(seed, TAG_OFFY, t, b, 0), d.offset_min, d.offset_max);
  const int base = (static_cast<int>(b) * d.C + c) * d.strokes_max;
  bool have = false;
  if (lane < d.strokes_max) {                 // lane s: end points of stroke s
    const int s = lane;
    const int* g = geom + static_cast<size_t>(base + s) * 4;
    have = g[3] != 0;
    if (have) {
      double sn, cn;
      sincospi(2.0 * turns[base + s], &sn, &cn);
      const int jx = uniform_int(hash5(seed, TAG_JITX, t, b, s), d.jitter_min, d.jitter_max);
      const int jy = uniform_int(hash5(seed, TAG_JITY, t, b, s), d.jitter_min, d.jitter_max);
      const int x0 = g[0] + ox, y0 = g[1] + oy;
      // Python round(): half to even
      seg[s] = make_int4(x0, y0, static_cast<int>(rint(x0 + (cn * g[2] + jx))), static_cast<int>(rint(y0 + (sn * g[2] + jy))));
    }
  }
  const uint32_t valid = __ballot_sync(0xffffffffu, have);
  __syncwarp();
  raster_warp(img, S, seg, valid, width, lane);
  __syncwarp();
  for (int p = lane; p < n; p += 32)
    if (img[p]) img[p] = static_cast<uint8_t>(uniform_int(hash5(seed, TAG_FILL, t, b, p), 200, 254));
  __syncwarp();
  blur_warp(img, tmp, S, lane);

  float* out = x + static_cast<size_t>(image) * n;
  if (!normalize) {
    for (int p = lane; p < n; p += 32) out[p] = __fdiv_rn(static_cast<float>(img[p]), 255.f);
    return;
  }
  float sum = 0.f;
  for (int p = lane; p < n; p += 32) sum += __fdiv_rn(static_cast<float>(img[p]), 255.f);
  const float mean = warp_sum(sum) / n;
  float ssd = 0.f;
  for (int p = lane; p < n; p += 32) {
    const float v = __fdiv_rn(static_cast<float>(img[p]), 255.f) - mean;
    ssd += v * v;
  }
  const float inv = 1.f / (sqrtf(warp_sum(ssd) / (n - 1)) + 1e-6f);
  for (int p = lane; p < n; p += 32) out[p] = (__fdiv_rn(static_cast<float>(img[p]), 255.f) - mean) * inv;
}

// Oracle hook: rasterise and blur caller-supplied segment sets with the sampler's own device functions.
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
stroke_raster_kernel(const int* __restrict__ segs, const int* __restrict__ nseg, const int* __restrict__ widths,
                     const uint8_t* __restrict__ fill, uint8_t* __restrict__ mask, uint8_t* __restrict__ blurred, int N, int K,
                     int S) {
  extern __shared__ uint8_t smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = S * S;
  int4* seg = reinterpret_cast<int4*>(smem + warp * warp_smem(S));
  uint8_t* img = reinterpret_cast<uint8_t*>(seg + PFN_STROKE_MAX_STROKES);
  uint8_t* tmp = img + n;
  const int i = blockIdx.x * kWarpsPerBlock + warp;
  if (i >= N) return;
  for (int p = lane; p < n; p += 32) img[p] = 0;
  const int ns = min(max(nseg[i], 0), K);
  if (lane < ns) {
    const int* q = segs + (static_cast<size_t>(i) * K + lane) * 4;
    seg[lane] = make_int4(q[0], q[1], q[2], q[3]);
  }
  const uint32_t valid = __ballot_sync(0xffffffffu, lane < ns);
  __syncwarp();
  raster_warp(img, S, seg, valid, widths[i], lane);
  __syncwarp();
  const size_t off = static_cast<size_t>(i) * n;
  for (int p = lane; p < n; p += 32) {
    mask[off + p] = img[p];
    if (img[p]) img[p] = fill != nullptr ? fill[off + p] : 128;
  }
  __syncwarp();
  blur_warp(img, tmp, S, lane);
  for (int p = lane; p < n; p += 32) blurred[off + p] = img[p];
}

int image_smem(int S) { return kWarpsPerBlock * warp_smem(S); }

int prepare_smem(const void* kernel, int bytes) {
  if (bytes > 48 * 1024) PFN_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  return 0;
}

int check_desc(const pfn_stroke_desc* d) {
  PFN_CHECK_ARG(d != nullptr, "stroke prior: null descriptor");
  PFN_CHECK_ARG(d->S >= 1 && d->S <= PFN_STROKE_MAX_SIDE, "stroke prior: image side %d outside [1, %d]", d->S, PFN_STROKE_MAX_SIDE);
  PFN_CHECK_ARG(d->C >= 1, "stroke prior: %d classes", d->C);
  PFN_CHECK_ARG(d->strokes_min >= 0 && d->strokes_min <= d->strokes_max && d->strokes_max <= PFN_STROKE_MAX_STROKES,
                "stroke prior: strokes per class [%d, %d] outside [0, %d]", d->strokes_min, d->strokes_max, PFN_STROKE_MAX_STROKES);
  PFN_CHECK_ARG(d->len_min <= d->len_max && d->start_min <= d->start_max && d->width_min <= d->width_max &&
                    d->offset_min <= d->offset_max && d->jitter_min <= d->jitter_max,
                "stroke prior: an empty integer range (random.randint(a, b) needs a <= b)");
  PFN_CHECK_ARG(d->max_iters >= 1, "stroke prior: max_iters %d", d->max_iters);
  return 0;
}

}  // namespace
}  // namespace pfn

using namespace pfn;

extern "C" int pfn_stroke_geometry(const pfn_stroke_desc* d, uint32_t seed, int B, int* geom, double* turns, int* cap_flag,
                                   void* stream) {
  if (int rc = check_desc(d)) return rc;
  PFN_CHECK_ARG(B >= 1 && geom != nullptr && turns != nullptr && cap_flag != nullptr, "stroke_geometry: bad arguments");
  const int total = B * d->C * d->strokes_max;
  if (total == 0) return 0;
  stroke_geometry_kernel<<<(total + 127) / 128, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(*d, seed, B, geom,
                                                                                                  turns, cap_flag);
  PFN_LAUNCH_OK();
  return 0;
}

extern "C" int pfn_stroke_render(const pfn_stroke_desc* d, uint32_t seed, const int* cls, const int* geom,
                                 const double* turns, float* x, int T, int B, int normalize, void* stream) {
  if (int rc = check_desc(d)) return rc;
  PFN_CHECK_ARG(T >= 1 && B >= 1 && cls != nullptr && geom != nullptr && turns != nullptr && x != nullptr,
                "stroke_render: bad arguments");
  const int smem = image_smem(d->S);
  if (int rc = prepare_smem(reinterpret_cast<const void*>(stroke_render_kernel), smem)) return rc;
  const long long images = static_cast<long long>(T) * B;
  PFN_CHECK_ARG(images < (1ll << 31), "stroke_render: %lld images", images);
  stroke_render_kernel<<<static_cast<int>((images + kWarpsPerBlock - 1) / kWarpsPerBlock), kWarpsPerBlock * 32, smem,
                         reinterpret_cast<cudaStream_t>(stream)>>>(*d, seed, cls, geom, turns, x, T, B, normalize);
  PFN_LAUNCH_OK();
  return 0;
}

extern "C" int pfn_stroke_raster(const int* segs, const int* nseg, const int* widths, const uint8_t* fill, uint8_t* mask,
                                 uint8_t* blurred, int N, int K, int S, void* stream) {
  PFN_CHECK_ARG(segs != nullptr && nseg != nullptr && widths != nullptr && mask != nullptr && blurred != nullptr && N >= 1,
                "stroke_raster: bad arguments");
  PFN_CHECK_ARG(K >= 1 && K <= PFN_STROKE_MAX_STROKES, "stroke_raster: %d segments per image outside [1, %d]", K, PFN_STROKE_MAX_STROKES);
  PFN_CHECK_ARG(S >= 1 && S <= PFN_STROKE_MAX_SIDE, "stroke_raster: image side %d outside [1, %d]", S, PFN_STROKE_MAX_SIDE);
  const int smem = image_smem(S);
  if (int rc = prepare_smem(reinterpret_cast<const void*>(stroke_raster_kernel), smem)) return rc;
  stroke_raster_kernel<<<(N + kWarpsPerBlock - 1) / kWarpsPerBlock, kWarpsPerBlock * 32, smem,
                         reinterpret_cast<cudaStream_t>(stream)>>>(segs, nseg, widths, fill, mask, blurred, N, K, S);
  PFN_LAUNCH_OK();
  return 0;
}
