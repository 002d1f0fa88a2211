// Omniglot few-shot episodes (reference priors/omniglot.py:36-72 over datasets/omniglotNshot.py:16-77 and :172-230).
//
// One CTA per episode b.  Thread 0 makes the episode-level draws into shared memory: the classes (Floyd's algorithm over the
// pool, then a Fisher-Yates shuffle, since Floyd's output order is not uniform; in Jonas mode an alphabet and a shuffle
// of its first n_way characters), the support order and the query class.  Thread j < n_way draws class j's images
// (a partial Fisher-Yates over the 20, the last drawn one being the query image) and its rot90 turn.  Then one warp
// per output row t reads the bank image through the rot90 index map, finds its ink bounding box with warp min / max
// reductions, draws the shift that keeps the ink inside the image, and writes the S*S floats of x[t, b, :] (16-byte
// stores when S*S is a multiple of 4).
//
// Random numbers are counter-based hashes of (seed, tag, episode, counters): a batch is a pure function of its seed.
#include "common.cuh"
#include "counter_rng.cuh"
#include "../../include/pfn_b200.h"

namespace pfn {
namespace {

enum : uint32_t { TAG_CLASS = 101, TAG_CLASS_PERM, TAG_ALPHABET, TAG_IMAGE, TAG_ROT, TAG_ORDER, TAG_QUERY, TAG_QUERY_IMAGE,
                  TAG_TX, TAG_TY };

constexpr int kWarps = 8;
constexpr int kMaxT = PFN_OMNIGLOT_MAX_WAY * (PFN_OMNIGLOT_IMAGES - 1) + 1;

// index into the source image of pixel (i, j) of np.rot90(src, k, axes=(-2, -1))
__device__ __forceinline__ int rot_index(int i, int j, int k, int S) {
  switch (k) {
    case 1: return j * S + (S - 1 - i);
    case 2: return (S - 1 - i) * S + (S - 1 - j);
    case 3: return (S - 1 - j) * S + i;
    default: return i * S + j;
  }
}

__global__ void __launch_bounds__(kWarps * 32)
omniglot_episode_kernel(pfn_omniglot_desc d, uint32_t seed, const uint8_t* __restrict__ bank, const int* __restrict__ alpha_start,
                        float* __restrict__ x, int64_t* __restrict__ y, int64_t* __restrict__ target_y) {
  __shared__ float lut[256];
  __shared__ int cls[PFN_OMNIGLOT_MAX_WAY];
  __shared__ int8_t rot[PFN_OMNIGLOT_MAX_WAY];
  __shared__ int8_t img[PFN_OMNIGLOT_MAX_WAY][PFN_OMNIGLOT_IMAGES];
  __shared__ int16_t slot[kMaxT];                // row t -> label * 32 + index into img[label]
  const int tid = threadIdx.x;
  const uint32_t b = blockIdx.x;
  const int S = d.S, n = S * S, nw = d.n_way, ks = d.k_shot, T = d.T;

  // (1.0 - v / 255.0) in fp64, rounded to fp32: the reference's x / 255., 1 - x, astype(np.float32)
  for (int v = tid; v < 256; v += blockDim.x) lut[v] = __double2float_rn(__dsub_rn(1.0, __ddiv_rn(static_cast<double>(v), 255.0)));

  if (tid == 0) {
    if (d.jonas) {
      const int a = uniform_int(hash5(seed, TAG_ALPHABET, b, 0, 0), 0, d.n_alpha - 1);
      const int first = alpha_start[a];
      for (int j = 0; j < nw; ++j) cls[j] = first + j;
    } else {
      // Floyd: a uniform n_way-subset of the pool ...
      int m = 0;
      for (int i = d.pool_n - nw; i < d.pool_n; ++i) {
        const int r = uniform_int(hash5(seed, TAG_CLASS, b, static_cast<uint32_t>(i), 0), 0, i);
        bool seen = false;
        for (int q = 0; q < m; ++q) seen |= cls[q] == r;
        cls[m++] = seen ? i : r;
      }
      for (int j = 0; j < nw; ++j) cls[j] += d.pool_lo;
    }
    // ... in a uniformly random order (np.random.choice / np.random.permutation)
    for (int i = nw - 1; i > 0; --i) {
      const int r = uniform_int(hash5(seed, TAG_CLASS_PERM, b, static_cast<uint32_t>(i), 0), 0, i);
      const int c = cls[i]; cls[i] = cls[r]; cls[r] = c;
    }
    const int ns = nw * ks;
    for (int t = 0; t < ns; ++t) slot[t] = static_cast<int16_t>((t / ks) * 32 + t % ks);     // class-major
    if (!d.jonas)
      for (int i = ns - 1; i > 0; --i) {
        const int r = uniform_int(hash5(seed, TAG_ORDER, b, static_cast<uint32_t>(i), 0), 0, i);
        const int16_t s = slot[i]; slot[i] = slot[r]; slot[r] = s;
      }
    const int jq = uniform_int(hash5(seed, TAG_QUERY, b, 0, 0), 0, nw - 1);
    slot[T - 1] = static_cast<int16_t>(jq * 32 + ks);
  }
  if (tid < nw) {
    const int j = tid;
    int8_t perm[PFN_OMNIGLOT_IMAGES];
    if (d.jonas && !d.train) {
      // support: images 0..k_shot-1 in a random order; query: uniform on k_shot..19
      for (int i = 0; i < ks; ++i) perm[i] = static_cast<int8_t>(i);
      for (int i = ks - 1; i > 0; --i) {
        const int r = uniform_int(hash5(seed, TAG_IMAGE, b, j, i), 0, i);
        const int8_t s = perm[i]; perm[i] = perm[r]; perm[r] = s;
      }
      perm[ks] = static_cast<int8_t>(uniform_int(hash5(seed, TAG_QUERY_IMAGE, b, j, 0), ks, PFN_OMNIGLOT_IMAGES - 1));
    } else {
      // k_shot + 1 distinct images in a uniformly random order: partial Fisher-Yates
      for (int i = 0; i < PFN_OMNIGLOT_IMAGES; ++i) perm[i] = static_cast<int8_t>(i);
      for (int i = 0; i <= ks; ++i) {
        const int r = uniform_int(hash5(seed, TAG_IMAGE, b, j, i), i, PFN_OMNIGLOT_IMAGES - 1);
        const int8_t s = perm[i]; perm[i] = perm[r]; perm[r] = s;
      }
    }
    for (int i = 0; i <= ks; ++i) img[j][i] = perm[i];
    rot[j] = d.jonas ? 0 : static_cast<int8_t>(uniform_int(hash5(seed, TAG_ROT, b, j, 0), 0, 3));
  }
  __syncthreads();

  const size_t B = static_cast<size_t>(d.B);
  for (int t = tid; t < T; t += blockDim.x) {
    const int64_t label = slot[t] >> 5;
    y[t * B + b] = label;
    target_y[t * B + b] = t == T - 1 ? label : -100;
  }

  const int warp = tid >> 5, lane = tid & 31;
  for (int t = warp; t < T; t += kWarps) {
    const int j = slot[t] >> 5, k = rot[j];
    const uint8_t* src = bank + (static_cast<size_t>(cls[j]) * PFN_OMNIGLOT_IMAGES + img[j][slot[t] & 31]) * n;
    int tx = 0, ty = 0;
    if (d.translate) {
      // ink bounding box of the source image, then mapped through the turn
      unsigned r0 = 0xFFFFu, r1 = 0, c0 = 0xFFFFu, c1 = 0;
      for (int p = lane; p < n; p += 32)
        if (__ldg(src + p) != 255) {
          const unsigned r = p / S, c = p - r * S;
          r0 = min(r0, r); r1 = max(r1, r); c0 = min(c0, c); c1 = max(c1, c);
        }
      r0 = __reduce_min_sync(0xffffffffu, r0); r1 = __reduce_max_sync(0xffffffffu, r1);
      c0 = __reduce_min_sync(0xffffffffu, c0); c1 = __reduce_max_sync(0xffffffffu, c1);
      if (r0 != 0xFFFFu) {
        const int a0 = r0, a1 = r1, b0 = c0, b1 = c1, m = S - 1;
        int R0 = a0, R1 = a1, C0 = b0, C1 = b1;
        if (k == 1) { R0 = m - b1; R1 = m - b0; C0 = a0; C1 = a1; }
        else if (k == 2) { R0 = m - a1; R1 = m - a0; C0 = m - b1; C1 = m - b0; }
        else if (k == 3) { R0 = b0; R1 = b1; C0 = m - a1; C1 = m - a0; }
        tx = uniform_int(hash5(seed, TAG_TX, b, t, 0), -C0, m - C1);
        ty = uniform_int(hash5(seed, TAG_TY, b, t, 0), -R0, m - R1);
      }
    }
    float* out = x + (static_cast<size_t>(t) * B + b) * n;
    auto pixel = [&](int p) -> float {
      const int r = p / S, c = p - r * S, i = r - ty, jj = c - tx;
      return (i >= 0 && i < S && jj >= 0 && jj < S) ? lut[__ldg(src + rot_index(i, jj, k, S))] : 0.f;
    };
    if ((n & 3) == 0) {
      float4* out4 = reinterpret_cast<float4*>(out);
      for (int q = lane; q < n / 4; q += 32) out4[q] = make_float4(pixel(4 * q), pixel(4 * q + 1), pixel(4 * q + 2), pixel(4 * q + 3));
    } else {
      for (int p = lane; p < n; p += 32) out[p] = pixel(p);
    }
  }
}

}  // namespace
}  // namespace pfn

using namespace pfn;

extern "C" int pfn_omniglot_episodes(const pfn_omniglot_desc* d, uint32_t seed, const uint8_t* bank, const int* alpha_start,
                                     float* x, int64_t* y, int64_t* target_y, void* stream) {
  PFN_CHECK_ARG(d != nullptr, "omniglot: null descriptor");
  PFN_CHECK_ARG(d->S >= 1 && d->S <= PFN_OMNIGLOT_MAX_SIDE, "omniglot: image side %d outside [1, %d]", d->S, PFN_OMNIGLOT_MAX_SIDE);
  PFN_CHECK_ARG(d->n_way >= 1 && d->n_way <= PFN_OMNIGLOT_MAX_WAY, "omniglot: n_way %d outside [1, %d]", d->n_way,
                PFN_OMNIGLOT_MAX_WAY);
  PFN_CHECK_ARG(d->k_shot >= 0 && d->k_shot + 1 <= PFN_OMNIGLOT_IMAGES, "omniglot: k_shot %d: k_shot + 1 images of %d per class",
                d->k_shot, PFN_OMNIGLOT_IMAGES);
  PFN_CHECK_ARG(d->T == d->n_way * d->k_shot + 1, "omniglot: T = %d, n_way * k_shot + 1 = %d", d->T, d->n_way * d->k_shot + 1);
  PFN_CHECK_ARG(d->B >= 1 && static_cast<long long>(d->B) * d->T < (1ll << 31), "omniglot: %d episodes of %d rows", d->B, d->T);
  PFN_CHECK_ARG(d->n_classes >= 1, "omniglot: %d classes in the bank", d->n_classes);
  if (d->jonas) {
    PFN_CHECK_ARG(alpha_start != nullptr && d->n_alpha >= 1, "omniglot: Jonas mode needs the split's alphabets");
    PFN_CHECK_ARG(d->n_way <= d->alpha_min, "omniglot: n_way %d exceeds the smallest alphabet of the split (%d characters)",
                  d->n_way, d->alpha_min);
  } else {
    PFN_CHECK_ARG(d->pool_lo >= 0 && d->pool_n >= 0 && d->pool_lo + d->pool_n <= d->n_classes,
                  "omniglot: class pool [%d, %d) outside the bank's %d classes", d->pool_lo, d->pool_lo + d->pool_n, d->n_classes);
    PFN_CHECK_ARG(d->n_way <= d->pool_n, "omniglot: n_way %d exceeds the pool of %d classes", d->n_way, d->pool_n);
  }
  PFN_CHECK_ARG(bank != nullptr && x != nullptr && y != nullptr && target_y != nullptr, "omniglot: null buffer");
  omniglot_episode_kernel<<<d->B, kWarps * 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(*d, seed, bank, alpha_start, x, y,
                                                                                          target_y);
  PFN_LAUNCH_OK();
  return 0;
}
