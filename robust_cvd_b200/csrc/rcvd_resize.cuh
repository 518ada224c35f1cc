// rcvd_resize.cuh -- downscaled colour frames on the GPU (the reference's Video.downscale_frames, video.py:154-182, which loads each
// frame as np.float32(img) / 255.0 and runs cv2.resize(img, (w, h), interpolation=cv2.INTER_AREA), utils/image_io.py:26-97).
//
// Bit-equal to OpenCV 4.13's INTER_AREA on float32 images (imgproc/src/resize.cpp), restated in tests/resize_ref.py.  The scale of an
// axis is s = 1 / (dst / src) in double: src / dst differs in the last bit, and at 98 -> 20 that moves a tap.  Three paths:
//   integer  both factors integers >= 1 (|s - round(s)| < DBL_EPSILON): acc = 0 plus the cell's values in row-major order, four at a
//            time as acc += ((v0 + v1) + v2) + v3 (resizeAreaFast_'s unrolled loop), then one at a time; the result
//            acc * float32(1 / (ix iy)).
//   area     other factors, both >= 1: per-axis tables of computeResizeAreaTab (weights in double, rounded to float32); a source row
//            is buf = buf + v alpha over the x entries in order, the output sum = sum + beta buf over the y entries in order.
//   linear   either axis upscales (the align rounding can round a side up past the source): per axis the two taps
//            (i, 1 - f), (min(i + 1, n - 1), f) of resize's area mode, horizontal first.  v0 a0 + v1 a1 is the area path's
//            accumulation (0 + v0 a0) + v1 a1 for the non-negative values of an image, so both run the same loop.
// The tables are built on the host (resize_axis_taps); each thread owns one output pixel and its three channels and recomputes the
// source-row sums it needs, so the order of every sum is the reference's whatever the launch shape.  Every float op is an explicit _rn
// intrinsic: nvcc contracts a * b + c into an FMA by default, and OpenCV's build does not.
#pragma once
#include <cuda_runtime.h>
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <vector>

namespace rcvd {

constexpr int kRsThreads = 256;   // also the size of the u8 -> float table every block fills

// Per output index d of one axis: the taps [off[d], off[d + 1]) of (source index, weight).
struct ResizeAxis {
  const int* off;
  const int* src;
  const float* wt;
};

struct ResizeArgs {
  int W, H;                    // source size
  int w, h;                    // output size
  int frame0;                  // first frame of this launch (blockIdx.y is relative to it)
  const uint8_t* src;          // [frames][H][W][3]
  int ix, iy;                  // integer path's factors (0: the tables)
  float inv_area;              // float32(1 / (ix iy))
  ResizeAxis x, y;
  int png;                     // 0: float32 [frames][h][w][3] in the source's channel order; 1: u8 in reversed channel order
  void* out;
};

// Per-axis tables for n source samples -> m outputs (host, double as OpenCV computes them).  linear: the upscale path's two taps.
// The host code is built with FMA contraction off (NVCC_FLAGS): (d + 1) - (i + 1) inv and d s + s must round twice.
inline void resize_axis_taps(int n, int m, bool linear, std::vector<int>& off, std::vector<int>& src, std::vector<float>& wt) {
  const double s = 1.0 / ((double)m / n), inv = (double)m / n;
  off.assign(1, 0); src.clear(); wt.clear();
  auto tap = [&](int k, float a) { src.push_back(k); wt.push_back(a); };
  for (int d = 0; d < m; ++d) {
    if (linear) {
      int i = (int)std::floor(d * s);
      float f = (float)((d + 1) - (i + 1) * inv);
      f = f <= 0 ? 0.f : f - (float)(int)std::floor(f);
      if (i >= n - 1) { f = 0.f; i = n - 1; }
      tap(i, 1.f - f);
      tap(std::min(i + 1, n - 1), f);
    } else {   // computeResizeAreaTab
      const double f1 = d * s, f2 = f1 + s, cw = std::min(s, n - f1);
      int i1 = (int)std::ceil(f1), i2 = (int)std::floor(f2);
      i2 = std::min(i2, n - 1);
      i1 = std::min(i1, i2);
      if (i1 - f1 > 1e-3) tap(i1 - 1, (float)((i1 - f1) / cw));
      for (int k = i1; k < i2; ++k) tap(k, (float)(1.0 / cw));
      if (f2 - i2 > 1e-3) tap(i2, (float)(std::min(std::min(f2 - i2, 1.0), cw) / cw));
    }
    off.push_back((int)src.size());
  }
}

// grid (ceil(h*w / kRsThreads), frames of this launch)
__global__ void __launch_bounds__(kRsThreads) k_resize_area(ResizeArgs a) {
  __shared__ float lut[256];   // np.float32(u) / 255.0: one float32 division
  lut[threadIdx.x] = __fdiv_rn((float)threadIdx.x, 255.f);
  __syncthreads();
  const int pix = blockIdx.x * kRsThreads + threadIdx.x;
  if (pix >= a.w * a.h) return;
  const int x = pix % a.w, y = pix / a.w;
  const size_t f = (size_t)a.frame0 + blockIdx.y;
  const uint8_t* img = a.src + f * a.H * a.W * 3;
  float v[3] = {0.f, 0.f, 0.f};
  if (a.ix > 0) {
    const int n = a.ix * a.iy;
    const uint8_t* cell = img + ((size_t)y * a.iy * a.W + (size_t)x * a.ix) * 3;
    auto at = [&](int k, int c) { return lut[cell[((size_t)(k / a.ix) * a.W + k % a.ix) * 3 + c]]; };
    int k = 0;
    for (; k + 4 <= n; k += 4)
#pragma unroll
      for (int c = 0; c < 3; ++c)
        v[c] = __fadd_rn(v[c], __fadd_rn(__fadd_rn(__fadd_rn(at(k, c), at(k + 1, c)), at(k + 2, c)), at(k + 3, c)));
    for (; k < n; ++k)
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c] = __fadd_rn(v[c], at(k, c));
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = __fmul_rn(v[c], a.inv_area);
  } else {
    const int x0 = a.x.off[x], x1 = a.x.off[x + 1];
    for (int j = a.y.off[y]; j < a.y.off[y + 1]; ++j) {
      const uint8_t* row = img + (size_t)a.y.src[j] * a.W * 3;
      float buf[3] = {0.f, 0.f, 0.f};
      for (int k = x0; k < x1; ++k) {
        const uint8_t* p = row + (size_t)a.x.src[k] * 3;
        const float al = a.x.wt[k];
#pragma unroll
        for (int c = 0; c < 3; ++c) buf[c] = __fadd_rn(buf[c], __fmul_rn(lut[p[c]], al));
      }
      const float be = a.y.wt[j];
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c] = __fadd_rn(v[c], __fmul_rn(be, buf[c]));
    }
  }
  const size_t o = (f * a.h * a.w + pix) * 3;
  if (a.png) {   // cv2.imwrite(fn, img * 255): float32 x * 255, rounded half to even, saturated; PNG stores the BGR array as R, G, B
    uint8_t* out = (uint8_t*)a.out + o;
#pragma unroll
    for (int c = 0; c < 3; ++c) out[2 - c] = (uint8_t)min(max(__float2int_rn(__fmul_rn(v[c], 255.f)), 0), 255);
  } else {
    float* out = (float*)a.out + o;
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c] = v[c];
  }
}

}  // namespace rcvd
