// Pillow-exact rasterisation and blur of the stroke prior's images (reference priors/stroke.py:47-60):
//   ImageDraw.line([x0, y0, x1, y1], fill=128, width=w) on an S x S "L" canvas, then ImageFilter.GaussianBlur(0.2).
//
// Integer end points only (the reference rounds them before drawing).  x is the column, y the row.  Pixels off the canvas
// are clipped one by one, exactly as Pillow's point / hline writers do.
//   width <= 1 : Bresenham from (x0, y0) towards (x1, y1) without the end pixel, then the end pixel as a point.
//   width  > 1 : a quadrilateral offset by round-half-up / round-half-down multiples of the unit normal, filled by a
//                scanline pass over its four edges (float32 intersections, horizontal edges drawn as spans, an edge's
//                lower end point counted twice unless it lies on the last scanline).
//   blur       : Pillow's extended box blur for radius 0.2 with 3 passes: box radius 0, so every pass is
//                out[i] = (in[i] * W + (in[i-1] + in[i+1]) * F + 2^23) >> 24 with clamped (replicated) edges, three
//                passes along rows, then three along columns, rounding to uint8 after every pass.
// Every function takes (lane, lanes): the work of one image is split over the lanes of a warp on the device; the host
// build of the same code (lanes = 1) is what the rasteriser was checked with.
#pragma once
#include <stdint.h>
#include <math.h>

#ifndef __CUDACC__
#define __host__
#define __device__
#define __forceinline__ inline
#endif

namespace pfn {
namespace stroke {

// Box-blur weights of GaussianBlur(0.2): W = (uint32)(2^24 / (2 r + 1)), F = (2^24 - W) / 2 with the extended box radius
// r = 0.00675676 of three passes (Gwosdek et al., SSVM 2011).  A lone 255 on black becomes 237 with 4-neighbours 6.
constexpr uint32_t kBlurW = 16553519u;
constexpr uint32_t kBlurF = (16777216u - kBlurW) / 2u;
constexpr int kBlurPasses = 3;

// float32 arithmetic without contraction to FMA (Pillow's scanline intersections are a separate multiply and add)
__host__ __device__ __forceinline__ float mul_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ __forceinline__ float add_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ __forceinline__ float div_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}

// round half up / half down of a float, in float arithmetic (x + 0.5f is rounded to float before floor / ceil)
__host__ __device__ __forceinline__ int round_up_f(float f) {
  return f >= 0.f ? static_cast<int>(floorf(add_rn(f, 0.5f))) : -static_cast<int>(floorf(add_rn(fabsf(f), 0.5f)));
}
__host__ __device__ __forceinline__ int round_down_f(float f) {
  return f >= 0.f ? static_cast<int>(ceilf(add_rn(f, -0.5f))) : -static_cast<int>(ceilf(add_rn(fabsf(f), -0.5f)));
}
__host__ __device__ __forceinline__ int round_up_d(double f) {
  return f >= 0.0 ? static_cast<int>(floor(f + 0.5)) : -static_cast<int>(floor(fabs(f) + 0.5));
}
__host__ __device__ __forceinline__ int round_down_d(double f) {
  return f >= 0.0 ? static_cast<int>(ceil(f - 0.5)) : -static_cast<int>(ceil(fabs(f) - 0.5));
}

__host__ __device__ __forceinline__ void put(uint8_t* img, int S, int x, int y, uint8_t v) {
  if (x >= 0 && x < S && y >= 0 && y < S) img[y * S + x] = v;
}

__host__ __device__ __forceinline__ void hline(uint8_t* img, int S, int x0, int y, int x1, uint8_t v) {
  if (y < 0 || y >= S) return;
  if (x0 < 0) x0 = 0;
  else if (x0 >= S) return;
  if (x1 < 0) return;
  else if (x1 >= S) x1 = S - 1;
  for (int x = x0; x <= x1; ++x) img[y * S + x] = v;
}

// width <= 1: Bresenham; the start pixel is drawn, the end pixel is drawn once more as a point.  Serial: one lane.
__host__ __device__ inline void thin_line(uint8_t* img, int S, int x0, int y0, int x1, int y1, uint8_t v) {
  int dx = x1 - x0, dy = y1 - y0;
  const int xs = dx < 0 ? -1 : 1, ys = dy < 0 ? -1 : 1;
  dx = dx < 0 ? -dx : dx;
  dy = dy < 0 ? -dy : dy;
  int x = x0, y = y0;
  if (dx == 0) {
    for (int i = 0; i < dy; ++i, y += ys) put(img, S, x, y, v);
  } else if (dy == 0) {
    for (int i = 0; i < dx; ++i, x += xs) put(img, S, x, y, v);
  } else if (dx > dy) {
    const int n = dx, ddy = 2 * dy, ddx = 2 * dx;
    int e = ddy - dx;
    for (int i = 0; i < n; ++i) {
      put(img, S, x, y, v);
      if (e >= 0) { y += ys; e -= ddx; }
      e += ddy;
      x += xs;
    }
  } else {
    const int n = dy, ddx = 2 * dx, ddy = 2 * dy;
    int e = ddx - dy;
    for (int i = 0; i < n; ++i) {
      put(img, S, x, y, v);
      if (e >= 0) { x += xs; e -= ddy; }
      e += ddx;
      y += ys;
    }
  }
  put(img, S, x1, y1, v);
}

struct Edge {
  int xmin, xmax, ymin, ymax, x0, y0;
  float dx;
};

__host__ __device__ __forceinline__ Edge make_edge(int x0, int y0, int x1, int y1) {
  Edge e;
  e.xmin = x0 <= x1 ? x0 : x1;
  e.xmax = x0 <= x1 ? x1 : x0;
  e.ymin = y0 <= y1 ? y0 : y1;
  e.ymax = y0 <= y1 ? y1 : y0;
  e.dx = y0 == y1 ? 0.f : div_rn(static_cast<float>(x1 - x0), static_cast<float>(y1 - y0));
  e.x0 = x0;
  e.y0 = y0;
  return e;
}

__host__ __device__ __forceinline__ float edge_x(const Edge& e, int y) {
  return add_rn(mul_rn(static_cast<float>(y - e.y0), e.dx), static_cast<float>(e.x0));
}

// width > 1: the quadrilateral of Pillow's wide line, filled scanline by scanline; lanes split the scanlines.
__host__ __device__ inline void wide_line(uint8_t* img, int S, int x0, int y0, int x1, int y1, int width, uint8_t v,
                                          int lane, int lanes) {
  const int dx = x1 - x0, dy = y1 - y0;
  if (dx == 0 && dy == 0) {
    if (lane == 0) put(img, S, x0, y0, v);
    return;
  }
  const double big = sqrt(static_cast<double>(dx * dx + dy * dy));
  const double small = (width - 1) / 2.0;
  const double rmax = round_up_d(small) / big, rmin = round_down_d(small) / big;
  const int dxmin = round_down_d(rmin * dy), dxmax = round_down_d(rmax * dy);
  const int dymin = round_down_d(rmin * dx), dymax = round_down_d(rmax * dx);
  const int vx[4] = {x0 - dxmin, x1 - dxmin, x1 + dxmax, x0 + dxmax};
  const int vy[4] = {y0 + dymax, y1 + dymax, y1 - dymin, y0 - dymin};
  // Every array below is indexed by unrolled loop counters only, so it lives in registers (no local memory).
  Edge e[4];
  int ymin = S - 1, ymax = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    e[i] = make_edge(vx[i], vy[i], vx[(i + 1) & 3], vy[(i + 1) & 3]);
    ymin = e[i].ymin < ymin ? e[i].ymin : ymin;
    ymax = e[i].ymax > ymax ? e[i].ymax : ymax;
    if (e[i].ymin == e[i].ymax && lane == 0) hline(img, S, e[i].xmin, e[i].ymin, e[i].xmax, v);   // horizontal edge: a span
  }
  if (ymin < 0) ymin = 0;
  if (ymax > S) ymax = S;
  for (int y = ymin + lane; y <= ymax; y += lanes) {
    // scanline intersections; an edge's lower end point counts twice unless it is on the polygon's last scanline
    float xx[8];
    int j = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) xx[k] = INFINITY;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (e[i].ymin != e[i].ymax && y >= e[i].ymin && y <= e[i].ymax) {
        const float xi = edge_x(e[i], y);
        const int reps = (y == e[i].ymax && y < ymax) ? 2 : 1;
#pragma unroll
        for (int k = 0; k < 8; ++k)
          if (k >= j && k < j + reps) xx[k] = xi;
        j += reps;
      }
    }
#pragma unroll
    for (int a = 0; a < 8; ++a)                         // sort (odd-even transposition network, unused slots are +inf)
#pragma unroll
      for (int k = a & 1; k < 7; k += 2) {
        const float lo = fminf(xx[k], xx[k + 1]), hi = fmaxf(xx[k], xx[k + 1]);
        xx[k] = lo;
        xx[k + 1] = hi;
      }
#pragma unroll
    for (int i = 1; i < 8; i += 2) {
      if (i < j) {
        const int xa = round_up_f(xx[i - 1]), xb = round_down_f(xx[i]);
        if (xb >= xa) hline(img, S, xa, y, xb, v);
      }
    }
  }
}

__host__ __device__ __forceinline__ void draw_line(uint8_t* img, int S, int x0, int y0, int x1, int y1, int width,
                                                   uint8_t v, int lane, int lanes) {
  if (width <= 1) {
    if (lane == 0) thin_line(img, S, x0, y0, x1, y1, v);
  } else {
    wide_line(img, S, x0, y0, x1, y1, width, v, lane, lanes);
  }
}

// One 1-D box pass of the blur over the line starting at src[0] with element stride `step` (n elements).
__host__ __device__ __forceinline__ uint8_t blur_tap(const uint8_t* src, int i, int n, int step) {
  const uint32_t l = src[(i > 0 ? i - 1 : 0) * step], c = src[i * step], r = src[(i < n - 1 ? i + 1 : n - 1) * step];
  return static_cast<uint8_t>((c * kBlurW + (l + r) * kBlurF + (1u << 23)) >> 24);
}

}  // namespace stroke
}  // namespace pfn
