// rcvd_bilateral.cuh -- joint depth / colour bilateral depth filter (DESIGN.md section 1 row 8f-5).
//
// Restates DepthVideoProcessor::bilateralFilter (reference lib/Processor.cpp:183-313).  For output pixel (x, y) of frame f the
// samples are the depths of frames max(0, f - fr) .. min(F - 1, f + fr) at [x - r, x + r] x [y - r, y + r] clamped to the image,
// visited in the order frame -> row -> column.  Each sample's weight is
//   e = 0;  e += -(d - dref)^2 / depthSigma^2  (depthSigma > 0);  e += -|c - cref|^2 / colorSigma^2  (colorSigma > 0);
//   weight = e != 0 ? expf(e) : 1
// and the output is the weighted mean sum(d w) / sum(w) (0 if sum(w) <= 0) or the weighted median: the samples sorted as
// std::pair<float, float> (depth, then weight) and the first one whose running weight reaches sum(w) / 2 (0 if none does).
// All arithmetic is float32 in that order with explicit round-to-nearest intrinsics (no FMA contraction).
//
// Layout: depth [F][h][w] f32, colour [F][h][w][3] f32 (BGR; only read when colorSigma > 0), out_frames [num_out] local frame
// indices, out [num_out][h][w] f32.
//
// Mean: one thread per output pixel, a CTA owns a 32 x 8 tile.  Per window frame the tile plus an r-pixel halo of depth (and colour)
// is staged in shared memory with cp.async, double-buffered across frames.  Halos too large for shared memory read global memory.
// Median: one warp per output pixel.  The warp writes the S samples as 64-bit keys (orderable depth bits | orderable weight bits) to
// its shared-memory slice, lane 0 sums the weights in window order, the warp sorts the keys (bitonic) and lane 0 walks the running
// weight in sorted order.  S is at most kBilateralMaxSamples.
#pragma once
#include "rcvd_ptx.cuh"

namespace rcvd {

constexpr int kBfTx = 32, kBfTy = 8;              // mean: output tile of one CTA (one thread per pixel)
constexpr int kBfMedianWarps = 4;                 // median: warps (= pixels in flight) per CTA
constexpr int kBilateralMaxSamples = 4096;        // median: largest window (keys per warp: 32 KB of shared memory)

struct BilateralArgs {
  const float* depth; const float* color; const int* out_frames; float* out;
  int F, w, h, frame_radius, radius;
  int out_base;                                   // output index of blockIdx.z == 0
  int use_depth;                                  // depthSigma > 0
  float depth_sigma, color_sigma;
  int sw, sh;                                     // mean: staged tile incl. halo (kBfTx + 2r) x (kBfTy + 2r)
  int P;                                          // median: keys per warp (power of two >= the largest window)
};

// lib/Processor.cpp:264-280
template <bool COLOR>
__device__ __forceinline__ float bf_weight(float d, float dref, bool use_depth, float ds2, float c0, float c1, float c2,
                                           float r0, float r1, float r2, float cs2) {
  float e = 0.f;
  if (use_depth) { const float t = __fsub_rn(d, dref); e = __fadd_rn(e, __fdiv_rn(-__fmul_rn(t, t), ds2)); }
  if (COLOR) {
    const float t0 = __fsub_rn(c0, r0), t1 = __fsub_rn(c1, r1), t2 = __fsub_rn(c2, r2);
    const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(t0, t0), __fmul_rn(t1, t1)), __fmul_rn(t2, t2));
    e = __fadd_rn(e, __fdiv_rn(-d2, cs2));
  }
  return e != 0.f ? expf(e) : 1.f;
}

template <bool COLOR, bool STAGED>
__global__ void __launch_bounds__(kBfTx * kBfTy) k_bilateral_mean(BilateralArgs a) {
  extern __shared__ float bf_smem[];
  const int tx0 = blockIdx.x * kBfTx, ty0 = blockIdx.y * kBfTy;
  const int x = tx0 + (threadIdx.x % kBfTx), y = ty0 + (threadIdx.x / kBfTx);
  const int o = a.out_base + blockIdx.z, frame = a.out_frames[o];
  const int f0 = max(0, frame - a.frame_radius), f1 = min(a.F - 1, frame + a.frame_radius);
  const size_t plane = (size_t)a.w * a.h;
  const bool inside = x < a.w && y < a.h;
  const int r = a.radius;
  const int sx0 = tx0 - r, sy0 = ty0 - r, tile = a.sw * a.sh, buf = COLOR ? 4 * tile : tile;
  // the staged rectangle clipped to the image: the clamped windows never reach outside it
  const int cx0 = max(sx0, 0), cx1 = min(sx0 + a.sw, a.w), cy0 = max(sy0, 0), cy1 = min(sy0 + a.sh, a.h);
  const int nx = cx1 - cx0, ny = cy1 - cy0;
  auto stage = [&](int f, int b) {
    float* sd = bf_smem + b * buf;
    const float* gd = a.depth + (size_t)f * plane;
    for (int i = threadIdx.x; i < nx * ny; i += kBfTx * kBfTy) {
      const int yy = cy0 + i / nx, xx = cx0 + i % nx;
      cp_async4_ca(sd + (yy - sy0) * a.sw + (xx - sx0), gd + (size_t)yy * a.w + xx);
    }
    if (COLOR) {
      float* sc = sd + tile;
      const float* gc = a.color + (size_t)f * plane * 3;
      for (int i = threadIdx.x; i < 3 * nx * ny; i += kBfTx * kBfTy) {
        const int yy = cy0 + i / (3 * nx), xc = i % (3 * nx);
        cp_async4_ca(sc + (yy - sy0) * 3 * a.sw + 3 * (cx0 - sx0) + xc, gc + ((size_t)yy * a.w + cx0) * 3 + xc);
      }
    }
    cp_async_commit();
  };
  float dref = 0.f, r0 = 0.f, r1 = 0.f, r2 = 0.f;
  if (inside) {
    const size_t p = (size_t)frame * plane + (size_t)y * a.w + x;
    dref = a.depth[p];
    if (COLOR) { r0 = a.color[3 * p]; r1 = a.color[3 * p + 1]; r2 = a.color[3 * p + 2]; }
  }
  const bool use_depth = a.use_depth != 0;
  const float ds2 = __fmul_rn(a.depth_sigma, a.depth_sigma), cs2 = __fmul_rn(a.color_sigma, a.color_sigma);
  const int x0 = max(0, x - r), x1 = min(a.w - 1, x + r), y0 = max(0, y - r), y1 = min(a.h - 1, y + r);
  float sum_d = 0.f, sum_w = 0.f;
  if (STAGED) stage(f0, 0);
  for (int f = f0; f <= f1; ++f) {
    const float* sd = bf_smem + ((f - f0) & 1) * buf;
    if (STAGED) {
      if (f < f1) { stage(f + 1, (f - f0 + 1) & 1); cp_async_wait<1>(); } else cp_async_wait<0>();
      __syncthreads();
    }
    if (inside) {
      for (int wy = y0; wy <= y1; ++wy)
        for (int wx = x0; wx <= x1; ++wx) {
          float d, c0 = 0.f, c1 = 0.f, c2 = 0.f;
          if (STAGED) {
            const int s = (wy - sy0) * a.sw + (wx - sx0);
            d = sd[s];
            if (COLOR) { const float* c = sd + tile + (wy - sy0) * 3 * a.sw + 3 * (wx - sx0); c0 = c[0]; c1 = c[1]; c2 = c[2]; }
          } else {
            const size_t p = (size_t)f * plane + (size_t)wy * a.w + wx;
            d = __ldg(a.depth + p);
            if (COLOR) { c0 = __ldg(a.color + 3 * p); c1 = __ldg(a.color + 3 * p + 1); c2 = __ldg(a.color + 3 * p + 2); }
          }
          const float wgt = bf_weight<COLOR>(d, dref, use_depth, ds2, c0, c1, c2, r0, r1, r2, cs2);
          sum_d = __fadd_rn(sum_d, __fmul_rn(d, wgt)); sum_w = __fadd_rn(sum_w, wgt);
        }
    }
    if (STAGED) __syncthreads();   // the next iteration stages into the buffer just read
  }
  if (inside) a.out[(size_t)blockIdx.z * plane + (size_t)y * a.w + x] = sum_w > 0.f ? __fdiv_rn(sum_d, sum_w) : 0.f;
}

// float -> unsigned with the same order (non-NaN); -0 is mapped like +0 so that equal depths compare equal, as in std::pair
__device__ __forceinline__ uint32_t bf_ord(float v) {
  const uint32_t u = __float_as_uint(v == 0.f ? 0.f : v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float bf_unord(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

template <bool COLOR>
__global__ void __launch_bounds__(32 * kBfMedianWarps) k_bilateral_median(BilateralArgs a) {
  extern __shared__ unsigned long long bf_keys[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long pix = (long long)blockIdx.x * kBfMedianWarps + warp;
  if (pix >= (long long)a.w * a.h) return;      // whole warps leave; the kernel has no block-wide barrier
  unsigned long long* key = bf_keys + (size_t)warp * a.P;
  const int x = (int)(pix % a.w), y = (int)(pix / a.w);
  const int o = a.out_base + blockIdx.z, frame = a.out_frames[o];
  const int f0 = max(0, frame - a.frame_radius), f1 = min(a.F - 1, frame + a.frame_radius);
  const size_t plane = (size_t)a.w * a.h;
  const int r = a.radius;
  const int x0 = max(0, x - r), x1 = min(a.w - 1, x + r), y0 = max(0, y - r), y1 = min(a.h - 1, y + r);
  const int nx = x1 - x0 + 1, nxy = nx * (y1 - y0 + 1), S = nxy * (f1 - f0 + 1);
  const size_t pref = (size_t)frame * plane + (size_t)y * a.w + x;
  const float dref = __ldg(a.depth + pref);
  float r0 = 0.f, r1 = 0.f, r2 = 0.f;
  if (COLOR) { r0 = __ldg(a.color + 3 * pref); r1 = __ldg(a.color + 3 * pref + 1); r2 = __ldg(a.color + 3 * pref + 2); }
  const bool use_depth = a.use_depth != 0;
  const float ds2 = __fmul_rn(a.depth_sigma, a.depth_sigma), cs2 = __fmul_rn(a.color_sigma, a.color_sigma);
  for (int i = lane; i < a.P; i += 32) {   // key i = sample i in window order; the padding sorts last
    unsigned long long k = ~0ull;
    if (i < S) {
      const int wf = i / nxy, rem = i - wf * nxy, wy = y0 + rem / nx, wx = x0 + rem % nx;
      const size_t p = (size_t)(f0 + wf) * plane + (size_t)wy * a.w + wx;
      const float d = __ldg(a.depth + p);
      float c0 = 0.f, c1 = 0.f, c2 = 0.f;
      if (COLOR) { c0 = __ldg(a.color + 3 * p); c1 = __ldg(a.color + 3 * p + 1); c2 = __ldg(a.color + 3 * p + 2); }
      const float wgt = bf_weight<COLOR>(d, dref, use_depth, ds2, c0, c1, c2, r0, r1, r2, cs2);
      k = ((unsigned long long)bf_ord(d) << 32) | bf_ord(wgt);
    }
    key[i] = k;
  }
  __syncwarp();
  float half = 0.f;
  if (lane == 0) {                               // sumWeight in window order (lib/Processor.cpp:287)
    float s = 0.f;
    for (int i = 0; i < S; ++i) s = __fadd_rn(s, bf_unord((uint32_t)key[i]));
    half = __fdiv_rn(s, 2.f);
  }
  half = __shfl_sync(0xffffffffu, half, 0);
  for (int k = 2; k <= a.P; k <<= 1)             // bitonic sort, ascending; each lane owns P / 64 disjoint pairs per stage
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = lane; t < (a.P >> 1); t += 32) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1)), l = i + j;
        const unsigned long long u = key[i], v = key[l];
        if ((u > v) == ((i & k) == 0)) { key[i] = v; key[l] = u; }
      }
      __syncwarp();
    }
  if (lane == 0) {                               // lib/Processor.cpp:292-304
    float cum = 0.f, res = 0.f;
    for (int i = 0; i < S; ++i) {
      const unsigned long long k = key[i];
      cum = __fadd_rn(cum, bf_unord((uint32_t)k));
      if (cum >= half) { res = bf_unord((uint32_t)(k >> 32)); break; }
    }
    a.out[(size_t)blockIdx.z * plane + (size_t)y * a.w + x] = res;
  }
}

}  // namespace rcvd
