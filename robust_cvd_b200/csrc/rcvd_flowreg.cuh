// rcvd_flowreg.cuh -- the per-pixel geometry of the homography-registered optical flows on the GPU (the reference's
// optical_flow_homography.getimage / infer / resize_flow, optical_flow_homography.py:139-242, run by Flow.compute_flow, flow.py:84-126).
//
// k_homography_warp: img2_registered = cv2.warpPerspective(frame2, H_BA, (W, H)) of an 8-bit BGR frame, INTER_LINEAR, BORDER_CONSTANT 0,
// bit-equal to OpenCV 4.13's fixed-point path (imgproc/src/imgwarp.cpp), restated in tests/flow_register_ref.py:
//   - the map is cv::invert(H_BA) (its closed form; computed by the caller); coordinates are in double without FMA, in OpenCV's
//     order: per block of bw columns (bw = min(1024 / min(16, H), W)) X0 = (M0 x0 + M1 y) + M2 at the block's first column x0, then
//     X0 + M0 (x - x0).  The block width is part of the arithmetic: another x0 changes the last bit of some coordinates;
//   - w = W0 + M6 (x - x0) becomes 32 / w, or 0 when w == 0 (every such pixel then samples source (0, 0));
//   - X = clamp((X0 + M0 (x - x0)) w, INT_MIN, INT_MAX) rounded half to even (a NaN clamps to INT_MAX, as the scalar loop does), then
//     sx = X >> 5 saturated to int16, fx = X & 31, likewise y;
//   - the weights of fraction (fx, fy) are the host table's (warp_weight_table: initInterTab2D's exact products times 2^15);
//   - per channel (sum of weight * tap + 2^14) >> 15, a tap outside the image read as 0.
// k_flow_unregister: the .raw values of flow_i_j from the model's flow (u, v) of the pair, without the float64 full-size flow:
//   - at each source tap (x, y): fxx = float32(x) + u and fyy = float32(y) + v in float32;
//   - np.linalg.inv(H_BA).dot([fxx; fyy; 1]) per row as OpenBLAS' dgemm computes it on x86-64: fma(h2, 1, fma(h1, fyy, h0 fxx)), the
//     first product rounded (the plain sum (h0 x + h1 y) + h2 differs in about 15 % of the pixels);
//   - x / z - fx and y / z - fy in double;
//   - cv2.resize(INTER_CUBIC) to (w, h) as resize.cpp computes it for float64: float32 Keys coefficients and first taps from the host
//     tables (resize_cubic_taps), taps clamped to the image, the horizontal pass ((p0 + p1) + p2) + p3 in double -- at border columns
//     from 0 + p0, which turns a -0 sum into +0 -- then the vertical pass over the four clamped rows likewise; an unchanged size is
//     a copy (the cubic pass would turn an inf into a NaN);
//   - times (w / W, h / H) in double, then rounded to float32 as the .raw writer casts.
// One thread per output pixel; each recomputes what it reads, so no result depends on the launch shape.  Every float op is an explicit
// _rn intrinsic: nvcc contracts a * b + c into an FMA by default, and OpenCV's build does not.
#pragma once
#include <cuda_runtime.h>
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <vector>

namespace rcvd {

constexpr int kFrThreads = 256;
constexpr int kWarpTab = 32;   // INTER_TAB_SIZE

struct HomographyWarpArgs {
  int W, H;                    // frame size (the output has it too)
  int bw;                      // warpPerspective's block width
  int pair0;                   // first pair of this launch (blockIdx.y is relative to it)
  const uint8_t* frames;       // [frames][H][W][3]
  const int* pair_frame;       // [pairs] local id of the frame to warp
  const double* minv;          // [pairs][9] cv::invert(H_BA)
  const int* wtab;             // [32 * 32][4] weights of taps (0,0), (1,0), (0,1), (1,1)
  uint8_t* out;                // [pairs][H][W][3]
};

struct FlowUnregisterArgs {
  int W, H;                    // the model's flow
  int w, h;                    // the output (color_down)
  int copy;                    // w == W and h == H: cv2.resize copies
  int pair0;
  const float* flow;           // [pairs][H][W][2]
  const double* hinv;          // [pairs][9] np.linalg.inv(H_BA)
  const int* xs;               // [w] first source column of the cubic taps (before clamping: floor(f) - 1)
  const float* xc;             // [w][4] coefficients
  const uint8_t* xin;          // [w] all four taps inside (resize.cpp's interior columns)
  const int* ys;               // [h]
  const float* yc;             // [h][4]
  double sx, sy;               // w / W, h / H
  float* out;                  // [pairs][h][w][2]
};

// initInterTab2D(INTER_LINEAR, fixpt): per fraction (fy, fx) the float products (1 - fx/32 or fx/32)(1 - fy/32 or fy/32) times 2^15.
// The products are multiples of 2^-10, so every weight is exact and the four sum to 2^15: OpenCV's sum fix-up never changes one.  The
// single weight 2^15 of fraction (0, 0) does not fit OpenCV's int16 table, but 32767 and 32768 both map every u8 value v to itself
// ((32767 v + 2^14) >> 15 = v for v < 2^14), so the exact value is used.
inline std::vector<int> warp_weight_table() {
  std::vector<int> t(kWarpTab * kWarpTab * 4);
  for (int fy = 0; fy < kWarpTab; ++fy)
    for (int fx = 0; fx < kWarpTab; ++fx) {
      const int ax[2] = {kWarpTab - fx, fx}, ay[2] = {kWarpTab - fy, fy};
      for (int k = 0; k < 4; ++k) t[(fy * kWarpTab + fx) * 4 + k] = ay[k >> 1] * ax[k & 1] * ((1 << 15) / (kWarpTab * kWarpTab));
    }
  return t;
}

// interpolateCubic(f) in float32, A = -0.75, every product rounded (the host code is built with FMA contraction off).
inline void cubic_coeffs(float x, float c[4]) {
  const float A = -0.75f;
  c[0] = ((A * (x + 1) - 5 * A) * (x + 1) + 8 * A) * (x + 1) - 4 * A;
  c[1] = ((A + 2) * x - (A + 3)) * x * x + 1;
  c[2] = ((A + 2) * (1 - x) - (A + 3)) * (1 - x) * (1 - x) + 1;
  c[3] = 1.f - c[0] - c[1] - c[2];
}

// resize.cpp's INTER_CUBIC table of one axis, n source samples -> m outputs: s = 1 / (m / n) in double, f = float((d + 0.5) s - 0.5),
// s0 = floor(f), f -= s0 in float32; first tap s0 - 1; interior when s0 - 1 >= 0 and s0 + 2 <= n - 1.
inline void resize_cubic_taps(int n, int m, std::vector<int>& first, std::vector<float>& coef, std::vector<uint8_t>& inside) {
  const double s = 1.0 / ((double)m / n);
  first.resize(m); coef.resize((size_t)m * 4); inside.resize(m);
  for (int d = 0; d < m; ++d) {
    float f = (float)((d + 0.5) * s - 0.5);
    const int s0 = (int)std::floor(f);
    f -= (float)s0;
    cubic_coeffs(f, &coef[(size_t)d * 4]);
    first[d] = s0 - 1;
    inside[d] = s0 >= 1 && s0 + 2 <= n - 1;
  }
}

// grid (ceil(H*W / kFrThreads), pairs of this launch)
__global__ void __launch_bounds__(kFrThreads) k_homography_warp(HomographyWarpArgs a) {
  const int pix = blockIdx.x * kFrThreads + threadIdx.x;
  if (pix >= a.W * a.H) return;
  const int x = pix % a.W, y = pix / a.W;
  const int p = a.pair0 + blockIdx.y;
  const double* M = a.minv + (size_t)p * 9;
  const int x1 = x % a.bw;
  const double x0 = (double)(x - x1), yd = (double)y, x1d = (double)x1;
  const double X0 = __dadd_rn(__dadd_rn(__dmul_rn(M[0], x0), __dmul_rn(M[1], yd)), M[2]);
  const double Y0 = __dadd_rn(__dadd_rn(__dmul_rn(M[3], x0), __dmul_rn(M[4], yd)), M[5]);
  const double W0 = __dadd_rn(__dadd_rn(__dmul_rn(M[6], x0), __dmul_rn(M[7], yd)), M[8]);
  double w = __dadd_rn(W0, __dmul_rn(M[6], x1d));
  w = w != 0.0 ? __ddiv_rn((double)kWarpTab, w) : 0.0;
  // fmin(INT_MAX, NaN) is INT_MAX, as std::min(INT_MAX, NaN) in the scalar loop
  const double Xd = fmax((double)INT_MIN, fmin((double)INT_MAX, __dmul_rn(__dadd_rn(X0, __dmul_rn(M[0], x1d)), w)));
  const double Yd = fmax((double)INT_MIN, fmin((double)INT_MAX, __dmul_rn(__dadd_rn(Y0, __dmul_rn(M[3], x1d)), w)));
  const int X = __double2int_rn(Xd), Y = __double2int_rn(Yd);
  const int sx = min(max(X >> 5, -32768), 32767), sy = min(max(Y >> 5, -32768), 32767);
  const int* wt = a.wtab + ((Y & (kWarpTab - 1)) * kWarpTab + (X & (kWarpTab - 1))) * 4;
  const uint8_t* img = a.frames + (size_t)a.pair_frame[p] * a.H * a.W * 3;
  int acc[3] = {1 << 14, 1 << 14, 1 << 14};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int tx = sx + (k & 1), ty = sy + (k >> 1);
    if (tx < 0 || tx >= a.W || ty < 0 || ty >= a.H) continue;   // BORDER_CONSTANT 0
    const uint8_t* s = img + ((size_t)ty * a.W + tx) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) acc[c] += wt[k] * s[c];
  }
  uint8_t* o = a.out + ((size_t)p * a.H * a.W + pix) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c] = (uint8_t)min(max(acc[c] >> 15, 0), 255);
}

// The un-registered flow of source pixel (x, y): (x / z - x, y / z - y) of inv(H_BA) (x + u, y + v, 1), as infer computes it.
__device__ __forceinline__ void unregistered_at(const FlowUnregisterArgs& a, const float* flow, const double* h, int x, int y, double& fu, double& fv) {
  const float2 uv = *reinterpret_cast<const float2*>(flow + ((size_t)y * a.W + x) * 2);
  const double X = (double)__fadd_rn((float)x, uv.x), Y = (double)__fadd_rn((float)y, uv.y);
  const double r0 = __dadd_rn(__fma_rn(h[1], Y, __dmul_rn(h[0], X)), h[2]);   // fma(h2, 1, t) is t + h2
  const double r1 = __dadd_rn(__fma_rn(h[4], Y, __dmul_rn(h[3], X)), h[5]);
  const double r2 = __dadd_rn(__fma_rn(h[7], Y, __dmul_rn(h[6], X)), h[8]);
  fu = __dsub_rn(__ddiv_rn(r0, r2), (double)x);
  fv = __dsub_rn(__ddiv_rn(r1, r2), (double)y);
}

// grid (ceil(h*w / kFrThreads), pairs of this launch)
__global__ void __launch_bounds__(kFrThreads) k_flow_unregister(FlowUnregisterArgs a) {
  const int pix = blockIdx.x * kFrThreads + threadIdx.x;
  if (pix >= a.w * a.h) return;
  const int dx = pix % a.w, dy = pix / a.w;
  const size_t p = (size_t)a.pair0 + blockIdx.y;
  const float* flow = a.flow + p * a.H * a.W * 2;
  double hm[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) hm[k] = a.hinv[p * 9 + k];
  double ru, rv;
  if (a.copy) {
    unregistered_at(a, flow, hm, dx, dy, ru, rv);
  } else {
    const float* cx = a.xc + (size_t)dx * 4;
    const float* cy = a.yc + (size_t)dy * 4;
    const bool inside = a.xin[dx];
    ru = 0.0; rv = 0.0;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int sy = min(max(a.ys[dy] + r, 0), a.H - 1);
      double hu = 0.0, hv = 0.0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int sx = min(max(a.xs[dx] + k, 0), a.W - 1);
        double fu, fv;
        unregistered_at(a, flow, hm, sx, sy, fu, fv);
        const double c = (double)cx[k];
        const double pu = __dmul_rn(fu, c), pv = __dmul_rn(fv, c);
        if (k == 0 && inside) { hu = pu; hv = pv; }            // the interior sum starts at p0, a border sum at 0 + p0
        else { hu = __dadd_rn(hu, pu); hv = __dadd_rn(hv, pv); }
      }
      const double c = (double)cy[r];
      const double pu = __dmul_rn(hu, c), pv = __dmul_rn(hv, c);
      if (r == 0) { ru = pu; rv = pv; }
      else { ru = __dadd_rn(ru, pu); rv = __dadd_rn(rv, pv); }
    }
  }
  float2 o;
  o.x = __double2float_rn(__dmul_rn(ru, a.sx));
  o.y = __double2float_rn(__dmul_rn(rv, a.sy));
  *reinterpret_cast<float2*>(a.out + (p * a.h * a.w + pix) * 2) = o;
}

}  // namespace rcvd
