// rcvd_flowmask.cuh -- forward-backward flow-consistency masks on the GPU (the reference's Flow.compute_flow_masks, flow.py:180-209,
// which runs utils/consistency.py: numpy plus torch.nn.functional.grid_sample on CPU tensors).
//
// One thread per pixel and direction of a pair (i, j).  Direction 0 takes ref = i, tgt = j and the flow i -> j; direction 1 the
// reverse.  At pixel (x, y) with ref flow (u, v):
//   1. target position X = x + u, Y = y + v in float64 (exact), in-image test 0 <= X <= W-1, 0 <= Y <= H-1 (NaN fails);
//   2. grid coordinate g = float32(2 X / W - 1) in float64, as the reference builds grid_sample's grid;
//   3. grid_sample(bilinear, border, align_corners=False) in float32, as torch's vectorised CPU kernel computes it:
//      p = fma(g + 1, W / 2, -0.5), clamped to [0, W-1]; weights from floor(p); the four taps summed as
//      fma(se, w_se, fma(sw, w_sw, fma(ne, w_ne, nw * w_nw))), a tap past the last row / column reading 0;
//   4. flow check: sse(flow_ref, sample(-flow_tgt)) < flow_thresh_sq; photometric check: sse(color_ref, sample(color_tgt)) <
//      color_thresh_sq.  sse = d0^2 + d1^2 (+ d2^2) in that order, no contraction (numpy's order); NaN fails.
// The mask is the AND of the three tests, written as 0 / 255.  Every float op is an explicit _rn intrinsic so that nvcc's FMA
// contraction cannot change a rounding.  Sampling -flow_tgt is the negated sample of flow_tgt exactly (every step is odd in the data).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace rcvd {

constexpr int kFmThreads = 256;

struct FlowMaskArgs {
  int w, h;
  int pair0;                         // first pair of this launch (blockIdx.y is relative to it)
  const int* pair_frames;            // [P][2] local colour ids
  const float* flow_ij, *flow_ji;    // [P][h][w][2]
  const float* colors;               // [F][h][w][3] BGR
  float flow_thresh_sq, color_thresh_sq;
  uint8_t* mask_ij, *mask_ji;        // [P][h][w]
  unsigned long long* counts;        // [P][2] or nullptr
  float* sse_flow, *sse_color;       // [P][2][h][w] or nullptr
};

// float32 source coordinate of grid_sample (align_corners = False, border padding) from the float64 target position
__device__ __forceinline__ float fm_source_coord(double pos, int size) {
  const float g = __double2float_rn(__dadd_rn(__ddiv_rn(__dmul_rn(2.0, pos), (double)size), -1.0));
  const float p = __fmaf_rn(__fadd_rn(g, 1.f), (float)size * 0.5f, -0.5f);
  return fminf(fmaxf(p, 0.f), (float)(size - 1));
}

// bilinear sample of C channels of img [h][w][C] at the clamped source position (px, py)
template <int C>
__device__ __forceinline__ void fm_sample(const float* __restrict__ img, int w, int h, float px, float py, float out[C]) {
  const float xw = floorf(px), yn = floorf(py);
  const float fw = __fsub_rn(px, xw), fe = __fsub_rn(1.f, fw), fn = __fsub_rn(py, yn), fs = __fsub_rn(1.f, fn);
  const float wnw = __fmul_rn(fs, fe), wne = __fmul_rn(fs, fw), wsw = __fmul_rn(fn, fe), wse = __fmul_rn(fn, fw);
  const int ix = (int)xw, iy = (int)yn;
  const bool e = ix + 1 < w, s = iy + 1 < h;
  const float* r0 = img + ((size_t)iy * w + ix) * C;
  const float* r1 = r0 + (size_t)w * C;
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const float nw = __ldg(r0 + c), ne = e ? __ldg(r0 + C + c) : 0.f;
    const float sw = s ? __ldg(r1 + c) : 0.f, se = (e && s) ? __ldg(r1 + C + c) : 0.f;
    out[c] = __fmaf_rn(se, wse, __fmaf_rn(sw, wsw, __fmaf_rn(ne, wne, __fmul_rn(nw, wnw))));
  }
}

// grid (ceil(h*w / kFmThreads), pairs of this launch, 2 directions)
__global__ void __launch_bounds__(kFmThreads) k_flow_masks(FlowMaskArgs a) {
  const int dir = blockIdx.z;
  const size_t p = (size_t)a.pair0 + blockIdx.y, plane = (size_t)a.w * a.h;
  const int pix = blockIdx.x * kFmThreads + threadIdx.x;
  bool ok = false;
  if (pix < (int)plane) {
    const int x = pix % a.w, y = pix / a.w;
    const float* fref = (dir == 0 ? a.flow_ij : a.flow_ji) + p * plane * 2;
    const float* ftgt = (dir == 0 ? a.flow_ji : a.flow_ij) + p * plane * 2;
    const float* cref = a.colors + (size_t)a.pair_frames[2 * p + dir] * plane * 3;
    const float* ctgt = a.colors + (size_t)a.pair_frames[2 * p + 1 - dir] * plane * 3;
    const float2 uv = __ldg(reinterpret_cast<const float2*>(fref) + pix);
    const double X = __dadd_rn((double)x, (double)uv.x), Y = __dadd_rn((double)y, (double)uv.y);
    const bool inside = X >= 0.0 && X <= (double)(a.w - 1) && Y >= 0.0 && Y <= (double)(a.h - 1);
    float sf = __int_as_float(0x7fc00000), sc = sf;   // NaN where the target position is NaN (grid_sample's value there is unspecified)
    if (!isnan(X) && !isnan(Y)) {
      const float px = fm_source_coord(X, a.w), py = fm_source_coord(Y, a.h);
      float fs[2], cs[3];
      fm_sample<2>(ftgt, a.w, a.h, px, py, fs);
      fm_sample<3>(ctgt, a.w, a.h, px, py, cs);
      const float d0 = __fadd_rn(uv.x, fs[0]), d1 = __fadd_rn(uv.y, fs[1]);   // flow_ref - sample(-flow_tgt)
      sf = __fadd_rn(__fmul_rn(d0, d0), __fmul_rn(d1, d1));
      const float* c0 = cref + (size_t)pix * 3;
      const float e0 = __fsub_rn(__ldg(c0), cs[0]), e1 = __fsub_rn(__ldg(c0 + 1), cs[1]), e2 = __fsub_rn(__ldg(c0 + 2), cs[2]);
      sc = __fadd_rn(__fadd_rn(__fmul_rn(e0, e0), __fmul_rn(e1, e1)), __fmul_rn(e2, e2));
    }
    ok = inside && sf < a.flow_thresh_sq && sc < a.color_thresh_sq;
    (dir == 0 ? a.mask_ij : a.mask_ji)[p * plane + pix] = ok ? 255 : 0;
    if (a.sse_flow) a.sse_flow[(p * 2 + dir) * plane + pix] = sf;
    if (a.sse_color) a.sse_color[(p * 2 + dir) * plane + pix] = sc;
  }
  // per-direction count: one block-wide reduction, one atomic per block (an integer sum: the same on every run)
  const int n = __syncthreads_count(ok);
  if (a.counts && threadIdx.x == 0 && n) atomicAdd(a.counts + 2 * p + dir, (unsigned long long)n);
}

}  // namespace rcvd
