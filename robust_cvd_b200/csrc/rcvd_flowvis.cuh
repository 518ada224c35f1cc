// rcvd_flowvis.cuh -- flow visualisations on the GPU (the reference's Flow.visualize_flow, flow.py:128-178: utils/flowlib.py's
// Middlebury colouring, utils/visualization.py's apply_mask and flow.py's warp_by_flow, numpy plus torch, one pair at a time).
//
// Pass 1 (k_flow_vis_stats), one thread per pixel and flow of a pair: rad = sqrt(u^2 + v^2) in float32 with unknown pixels (|u| or
// |v| > 1e7) zeroed, reduced to the flow's maximum over the non-NaN pixels (float bits of a non-negative float order as unsigned ints,
// so atomicMax is exact) and a NaN flag.  Max and OR do not depend on the order, so every run gives the same result.
//
// Pass 2 (k_flow_vis), one thread per pixel position of a pair.  The thread owns that position in each of the composite's eight tiles
// and in both warps, so each flow's colour is computed once.  Everything the reference computes in float64 is computed here in
// float64 with explicit _rn intrinsics, so nvcc's FMA contraction cannot change a rounding.  The quirks kept, each where it happens:
// max(-1, nan), the float64 normalisation, the wheel wrap, the float32 colour tiles, cv2's conversion to 8 bits, the BGR channel order
// and the warp's mixed grid conventions.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cfloat>

namespace rcvd {

constexpr int kFvThreads = 256;
constexpr int kFvWheel = 55;

struct FlowVisArgs {
  int w, h;
  int pair0;                         // first pair of this launch (blockIdx.y is relative to it)
  const int* pair_frames;            // [P][2] local colour ids
  const float* flow_ij, *flow_ji;    // [P][h][w][2]
  const uint8_t* mask_ij, *mask_ji;  // [P][h][w]
  const float* colors;               // [F][h][w][3], the raw files' channel order
  unsigned* stats;                   // [P][2][2]: float bits of the flow's max rad, NaN flag (flow 0: i -> j)
  uint8_t* vis;                      // [P][2h][4w][3] in PNG (RGB) byte order
  uint8_t* warp_ij, *warp_ji;        // [P][h][w][3] in PNG byte order, or nullptr (no warp)
  float* warp_values;                // [P][2][h][w][3] array order, or nullptr
};

// grid (ceil(h*w / kFvThreads), pairs of this launch, 2 flows)
__global__ void __launch_bounds__(kFvThreads) k_flow_vis_stats(FlowVisArgs a) {
  const int dir = blockIdx.z;
  const size_t p = (size_t)a.pair0 + blockIdx.y, plane = (size_t)a.w * a.h;
  const int pix = blockIdx.x * kFvThreads + threadIdx.x;
  unsigned bits = 0;
  bool nan = false;
  if (pix < (int)plane) {
    float2 uv = __ldg(reinterpret_cast<const float2*>((dir == 0 ? a.flow_ij : a.flow_ji) + p * plane * 2) + pix);
    if (fabsf(uv.x) > 1e7f || fabsf(uv.y) > 1e7f) uv = make_float2(0.f, 0.f);     // flowlib's UNKNOWN_FLOW_THRESH
    const float rad = __fsqrt_rn(__fadd_rn(__fmul_rn(uv.x, uv.x), __fmul_rn(uv.y, uv.y)));
    nan = isnan(rad);
    bits = nan ? 0u : __float_as_uint(rad);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) bits = max(bits, __shfl_xor_sync(0xffffffffu, bits, o));
  __shared__ unsigned s_max[kFvThreads / 32];
  if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = bits;
  const int any_nan = __syncthreads_or(nan);
  if (threadIdx.x == 0) {
    for (int k = 1; k < kFvThreads / 32; ++k) bits = max(bits, s_max[k]);
    unsigned* st = a.stats + (p * 2 + dir) * 2;
    if (bits) atomicMax(st, bits);
    if (any_nan) atomicOr(st + 1, 1u);
  }
}

// cv2.imwrite's convertTo(CV_8U): cvRound (round half to even), then saturate; x86's conversion returns INT_MIN for NaN and for values
// outside the int32 range, which saturates to 0.
__device__ __forceinline__ uint8_t fv_to_u8(double x) {
  const double r = rint(x);
  if (!(r >= -2147483648.0 && r <= 2147483647.0)) return 0;
  return (uint8_t)fmin(fmax(r, 0.0), 255.0);
}

// flowlib.compute_color at one pixel, RGB in out.  u, v are the float32 flow with unknown pixels zeroed; d = maxrad + eps in float64.
__device__ __forceinline__ void fv_flow_color(float u, float v, double d, const double (*wheel)[3], double out[3]) {
  // u / (maxrad + eps): np.finfo(float).eps is a numpy float64, so under numpy 2's promotion the normalised flow is float64
  double un = __ddiv_rn((double)u, d), vn = __ddiv_rn((double)v, d);
  const bool nan = isnan(un) || isnan(vn);
  if (nan) un = vn = 0.0;                        // zeroed before the wheel; black below
  const double rad = __dsqrt_rn(__dadd_rn(__dmul_rn(un, un), __dmul_rn(vn, vn)));
  const double ang = __ddiv_rn(atan2(-vn, -un), 3.141592653589793);
  const double fk = __dadd_rn(__dmul_rn(__ddiv_rn(__dadd_rn(ang, 1.0), 2.0), (double)(kFvWheel - 1)), 1.0);
  // k0 in [1, 55]; the clamp only guards against an atan2 a rounding past pi.  k1 = 56 wraps to 1.
  const int k0 = min(max((int)floor(fk), 1), kFvWheel), k1 = k0 == kFvWheel ? 1 : k0 + 1;
  const double f = __dsub_rn(fk, (double)k0), g = __dsub_rn(1.0, f);   // fk - k0 is float64 (k0 is int64 in numpy)
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    double col = __dadd_rn(__dmul_rn(g, wheel[k0 - 1][c]), __dmul_rn(f, wheel[k1 - 1][c]));
    col = rad <= 1.0 ? __dsub_rn(1.0, __dmul_rn(rad, __dsub_rn(1.0, col))) : __dmul_rn(col, 0.75);
    out[c] = nan ? 0.0 : floor(__dmul_rn(255.0, col));
  }
}

// One coordinate of the warp's sample position.  geometry.sample builds grid = 2 uv / (W-1) - 1 (align_corners=True's convention) and
// grid_sample unnormalises with align_corners=False, ((g + 1) W - 1) / 2: the two conventions mix, so a pixel reads at x W / (W-1) - 1/2.
// uv and the grid are torch tensor ops in float32; the unnormalisation is torch's CUDA kernel, whose nvcc build contracts it to an FMA.
// Border padding clamps to [0, W-1]; fmaxf returns 0 for NaN, as torch's CUDA clip does.
__device__ __forceinline__ float fv_source(int pix, float flow, int size) {
  const float uv = __fadd_rn((float)pix, flow);
  const float g = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, uv), (float)(size - 1)), 1.f);
  const float s = __fmul_rn(__fmaf_rn(__fadd_rn(g, 1.f), (float)size, -1.f), 0.5f);
  return fminf(fmaxf(s, 0.f), (float)(size - 1));
}

// grid_sample(bilinear) of 255 * img [h][w][3] at (px, py) as torch's CUDA kernel sums it: taps outside the image are skipped.
__device__ __forceinline__ void fv_warp_sample(const float* __restrict__ img, int w, int h, float px, float py, float out[3]) {
  const float x0 = floorf(px), y0 = floorf(py), x1 = __fadd_rn(x0, 1.f), y1 = __fadd_rn(y0, 1.f);
  const int ix = (int)x0, iy = (int)y0;
  const float wx0 = __fsub_rn(x1, px), wx1 = __fsub_rn(px, x0), wy0 = __fsub_rn(y1, py), wy1 = __fsub_rn(py, y0);
  const float wt[4] = {__fmul_rn(wx0, wy0), __fmul_rn(wx1, wy0), __fmul_rn(wx0, wy1), __fmul_rn(wx1, wy1)};
  const int tx[4] = {ix, ix + 1, ix, ix + 1}, ty[4] = {iy, iy, iy + 1, iy + 1};
  out[0] = out[1] = out[2] = 0.f;
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    if (tx[t] >= w || ty[t] >= h) continue;
    const float* q = img + ((size_t)ty[t] * w + tx[t]) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c] = __fmaf_rn(__fmul_rn(__ldg(q + c), 255.f), wt[t], out[c]);   // the tensor holds 255 * colour
  }
}

// grid (ceil(h*w / kFvThreads), pairs of this launch)
__global__ void __launch_bounds__(kFvThreads) k_flow_vis(FlowVisArgs a) {
  // the Middlebury wheel / 255 (flowlib's tmp[k] / 255): six hue segments; in each one channel stays at 255 while another ramps up
  // or down by floor(255 k / n)
  __shared__ double s_wheel[kFvWheel][3];
  for (int t = threadIdx.x; t < kFvWheel * 3; t += kFvThreads) {
    constexpr int len[6] = {15, 6, 4, 11, 13, 6}, full[6] = {0, 1, 1, 2, 2, 0}, ramp[6] = {1, 0, 2, 1, 0, 2};
    constexpr bool up[6] = {true, false, true, false, true, false};
    const int k = t / 3, c = t % 3;
    int s = 0, start = 0;
    while (k >= start + len[s]) start += len[s++];
    const double r = floor(__ddiv_rn(255.0 * (k - start), (double)len[s]));
    const double val = c == full[s] ? 255.0 : c == ramp[s] ? (up[s] ? r : 255.0 - r) : 0.0;
    s_wheel[k][c] = __ddiv_rn(val, 255.0);
  }
  __syncthreads();
  const size_t p = (size_t)a.pair0 + blockIdx.y, plane = (size_t)a.w * a.h;
  const int pix = blockIdx.x * kFvThreads + threadIdx.x;
  if (pix >= (int)plane) return;
  const int x = pix % a.w, y = pix / a.w;
  const float* col[2] = {a.colors + (size_t)a.pair_frames[2 * p] * plane * 3, a.colors + (size_t)a.pair_frames[2 * p + 1] * plane * 3};
  const float* flo[2] = {a.flow_ij + p * plane * 2, a.flow_ji + p * plane * 2};
  const uint8_t msk[2] = {a.mask_ij[p * plane + pix], a.mask_ji[p * plane + pix]};
  double img[2][3];
  float2 fl[2];
  for (int d = 0; d < 2; ++d) {
    fl[d] = __ldg(reinterpret_cast<const float2*>(flo[d]) + pix);
    const unsigned* st = a.stats + (p * 2 + d) * 2;
    // maxrad = max(-1, np.max(rad)) is Python's max: with a NaN rad, NaN > -1 is False and it yields -1, so the flow is divided by
    // -1 + eps (negated, not normalised); an all-zero flow is divided by eps
    const double d_norm = __dadd_rn(st[1] ? -1.0 : (double)__uint_as_float(st[0]), DBL_EPSILON);
    const bool unknown = fabsf(fl[d].x) > 1e7f || fabsf(fl[d].y) > 1e7f;
    fv_flow_color(unknown ? 0.f : fl[d].x, unknown ? 0.f : fl[d].y, d_norm, s_wheel, img[d]);
    if (unknown) img[d][0] = img[d][1] = img[d][2] = 0.0;     // unknown pixels are black
  }
  // composite [255 c_i, 255 c_j, img_ij, img_ji] over the same tiles through apply_mask (mask_ij on the i tiles, mask_ji on the j
  // tiles).  The top row is float32 (hstack of float32 colours and u8 images); apply_mask is 0.7 im + 0.3 (1 - (mask > 0)) [0, 255, 0],
  // where 0.7 * a float32 colour stays float32 and 0.7 * a u8 image is float64; the vstack is float64 and cv2.imwrite rounds it.
  uint8_t* row0 = a.vis + ((p * 2 * a.h + y) * 4 * a.w + x) * 3;
  uint8_t* row1 = row0 + (size_t)a.h * 4 * a.w * 3;
  for (int d = 0; d < 2; ++d) {
    const float* c = col[d] + (size_t)pix * 3;
    const double green = msk[d] > 0 ? 0.0 : 76.5;             // 0.3 * 255
    uint8_t* t0 = row0 + (size_t)d * a.w * 3, *t1 = row1 + (size_t)d * a.w * 3;
    uint8_t* f0 = row0 + (size_t)(2 + d) * a.w * 3, *f1 = row1 + (size_t)(2 + d) * a.w * 3;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      // cv2.imwrite reads every tile as BGR: array channel ch is PNG byte 2 - ch.  The flow images are RGB, so they land with red and
      // blue swapped, as in the reference.
      const float c255 = __fmul_rn(__ldg(c + ch), 255.f);
      const double g = ch == 1 ? green : 0.0;
      t0[2 - ch] = fv_to_u8((double)c255);
      t1[2 - ch] = fv_to_u8(__dadd_rn((double)__fmul_rn(0.7f, c255), g));
      f0[2 - ch] = (uint8_t)img[d][ch];
      f1[2 - ch] = fv_to_u8(__dadd_rn(__dmul_rn(0.7, img[d][ch]), g));
    }
  }
  if (!a.warp_ij) return;
  // warps: frame_i_j_warped is colour j at p + flow_ij, frame_j_i_warped colour i at p + flow_ji
  for (int d = 0; d < 2; ++d) {
    float v[3];
    fv_warp_sample(col[1 - d], a.w, a.h, fv_source(x, fl[d].x, a.w), fv_source(y, fl[d].y, a.h), v);
    uint8_t* o = (d == 0 ? a.warp_ij : a.warp_ji) + (p * plane + pix) * 3;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) o[2 - ch] = fv_to_u8((double)v[ch]);
    if (a.warp_values) {
      float* wv = a.warp_values + ((p * 2 + d) * plane + pix) * 3;
      wv[0] = v[0]; wv[1] = v[1]; wv[2] = v[2];
    }
  }
}

}  // namespace rcvd
