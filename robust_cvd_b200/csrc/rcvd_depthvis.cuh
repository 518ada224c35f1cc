// rcvd_depthvis.cuh -- depth visualisations on the GPU (the reference's visualization.visualize_depth_dir / visualize_depth,
// utils/visualization.py:53-134).
//
// Two passes, each over a batch of frames of one size:
//   range   one CTA per frame (k_depth_range): the count n of finite values and, for each of two quantiles, the order statistics at
//           numpy's linear-method neighbours floor(v) and floor(v) + 1 of the virtual index v = (n - 1) q (both n - 1 when
//           v >= n - 1).  A radix select over order-preserving keys (a float's sign-flipped bits, a u8 value itself), eight bits
//           per pass, all four ranks at once; q = 0 and q = 1 select the minimum and the maximum.  The host interpolates them as
//           np.percentile does.
//   colour  one thread per pixel (k_depth_color): index = np.uint8(((d - offset) / scale) ** 0.5 * 255), then a 256-entry table.
// Two input kinds, as the reference reads them:
//   F32   a .raw disparity [h][w] float32; float32 arithmetic (the bounds enter as float32, numpy's NEP 50 weak-scalar rule), and
//         v = float32(n - 1) * float32(q) in float32, as np.percentile computes it for a float32 array.
//   U8C3  an image read by cv2.imread, [h][w][3] u8 (B, G, R); float64 arithmetic on each channel, then cv2.applyColorMap's
//         conversion to gray of the three indices, (3735 B + 19235 G + 9798 R + 2^14) >> 15; the percentiles are over all 3 h w values.
// np.uint8 of a float on x86-64 truncates through a 32-bit integer: NaN, +-inf and |x| >= 2^31 give 0, other values wrap modulo 256
// (-1 gives 255, 300.5 gives 44).  Every float op is an explicit _rn intrinsic: nvcc contracts a * b + c into an FMA by default.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace rcvd {

constexpr int kDvSelThreads = 512;   // range pass: one CTA per frame
constexpr int kDvThreads = 256;      // colour pass: one thread per pixel
constexpr int kDvRanks = 4;          // (floor, next) for each of two quantiles

struct DepthVisArgs {
  int w, h;
  int u8;                 // 0: F32, 1: U8C3
  const void* src;        // [frames][h][w] float32 or [frames][h][w][3] u8
  int frame0;             // colour pass: first frame of this launch (blockIdx.y is relative to it)
  double q[2];            // range pass: the quantiles (float32 values for F32)
  long long* counts;      // [frames]
  double* stats;          // [frames][kDvRanks]
  double offset, scale;   // colour pass (float32 values for F32)
  const uint8_t* lut;     // [256][3], copied out as it stands
  uint8_t* index;         // [frames][h][w] or null
  uint8_t* rgb;           // [frames][h][w][3] or null
};

// x86-64's float -> uint8 conversion (cvttss2si / cvttsd2si to int32, low byte)
__device__ __forceinline__ uint8_t dv_u8(float x) { return fabsf(x) < 2147483648.f ? (uint8_t)__float2int_rz(x) : 0; }
__device__ __forceinline__ uint8_t dv_u8(double x) { return fabs(x) < 2147483648.0 ? (uint8_t)__double2int_rz(x) : 0; }

// order-preserving key of a finite float (-0 sorts before +0; the two are equal as values)
__device__ __forceinline__ uint32_t dv_key(float x) {
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float dv_unkey(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// grid (frames), block kDvSelThreads
__global__ void __launch_bounds__(kDvSelThreads) k_depth_range(DepthVisArgs a) {
  __shared__ unsigned hist[kDvRanks][256];
  __shared__ unsigned long long s_n;
  __shared__ long long rank[kDvRanks];
  __shared__ uint32_t prefix[kDvRanks];
  const size_t f = blockIdx.x;
  const long long m = (long long)a.w * a.h * (a.u8 ? 3 : 1);
  const float* src32 = (const float*)a.src + f * m;
  const uint8_t* src8 = (const uint8_t*)a.src + f * m;
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  long long n;
  if (a.u8) {
    n = m;
  } else {
    unsigned long long c = 0;
    for (long long i = threadIdx.x; i < m; i += kDvSelThreads) c += isfinite(src32[i]);
    atomicAdd(&s_n, c);
    __syncthreads();
    n = (long long)s_n;
  }
  if (threadIdx.x == 0) a.counts[f] = n;
  if (n == 0) return;
  if (threadIdx.x < 2) {   // numpy's _get_indexes for the linear method
    const int j = threadIdx.x;
    double v, last = (double)(n - 1);
    if (a.u8) {
      v = __dmul_rn(last, a.q[j]);
    } else {
      const float v32 = __fmul_rn(__ll2float_rn(n - 1), (float)a.q[j]);
      v = v32; last = __ll2float_rn(n - 1);   // the comparison v >= n - 1 is in float32
    }
    long long p = (long long)floor(v), nx = p + 1;
    if (v >= last) p = nx = n - 1;
    rank[2 * j] = p; rank[2 * j + 1] = nx;
    prefix[2 * j] = prefix[2 * j + 1] = 0;
  }
  __syncthreads();
  // a u8 value is its own key, in the top eight bits, so one pass selects it
  const int last_shift = a.u8 ? 24 : 0;
  uint32_t himask = 0;
  for (int shift = 24; shift >= last_shift; shift -= 8) {
    for (int i = threadIdx.x; i < kDvRanks * 256; i += kDvSelThreads) (&hist[0][0])[i] = 0;
    __syncthreads();
    uint32_t pre[kDvRanks];
#pragma unroll
    for (int r = 0; r < kDvRanks; ++r) pre[r] = prefix[r];
    for (long long i = threadIdx.x; i < m; i += kDvSelThreads) {
      uint32_t k;
      if (a.u8) k = (uint32_t)src8[i] << 24;
      else { const float x = src32[i]; if (!isfinite(x)) continue; k = dv_key(x); }
#pragma unroll
      for (int r = 0; r < kDvRanks; ++r)
        if (((k ^ pre[r]) & himask) == 0) atomicAdd(&hist[r][(k >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (threadIdx.x < kDvRanks) {   // the bin holding rank r among the keys that share its prefix so far
      const int r = threadIdx.x;
      long long k = rank[r];
      int b = 0;
      for (; b < 255 && k >= (long long)hist[r][b]; ++b) k -= hist[r][b];
      rank[r] = k;
      prefix[r] |= (uint32_t)b << shift;
    }
    himask |= 0xffu << shift;
    __syncthreads();
  }
  if (threadIdx.x < kDvRanks) {
    const uint32_t k = prefix[threadIdx.x];
    a.stats[f * kDvRanks + threadIdx.x] = a.u8 ? (double)(k >> 24) : (double)dv_unkey(k);
  }
}

// grid (ceil(h*w / kDvThreads), frames of this launch), block kDvThreads
__global__ void __launch_bounds__(kDvThreads) k_depth_color(DepthVisArgs a) {
  __shared__ uint8_t lut[256 * 3];
  for (int i = threadIdx.x; i < 256 * 3; i += kDvThreads) lut[i] = a.lut ? a.lut[i] : 0;
  __syncthreads();
  const long long wh = (long long)a.w * a.h;
  const long long pix = (long long)blockIdx.x * kDvThreads + threadIdx.x;
  if (pix >= wh) return;
  const size_t p = ((size_t)a.frame0 + blockIdx.y) * wh + pix;
  int idx;
  if (a.u8) {
    const uint8_t* s = (const uint8_t*)a.src + p * 3;
    int c3[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double t = __dsqrt_rn(__ddiv_rn(__dsub_rn((double)s[c], a.offset), a.scale));
      c3[c] = dv_u8(__dmul_rn(t, 255.0));
    }
    idx = (c3[0] * 3735 + c3[1] * 19235 + c3[2] * 9798 + (1 << 14)) >> 15;   // cv::cvtColor(BGR2GRAY), 8-bit
  } else {
    const float d = ((const float*)a.src)[p];
    const float t = __fsqrt_rn(__fdiv_rn(__fsub_rn(d, (float)a.offset), (float)a.scale));
    idx = dv_u8(__fmul_rn(t, 255.f));
  }
  if (a.index) a.index[p] = (uint8_t)idx;
  if (a.rgb) {
#pragma unroll
    for (int c = 0; c < 3; ++c) a.rgb[p * 3 + c] = lut[idx * 3 + c];
  }
}

}  // namespace rcvd
