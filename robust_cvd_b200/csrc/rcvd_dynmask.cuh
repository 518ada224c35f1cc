// rcvd_dynmask.cuh -- dynamic-object masks on the GPU (the per-pixel work of the reference's dynamic_mask_generation,
// dynamic_mask_generation.py:107-182, around its Mask R-CNN predictor).
//
// For a batch of frames of one size, each with its own run of (already selected) instance masks:
//   union   k_dm_union: u[f][p] = OR over the frame's instances of (instances[k][p] != 0); with frames, also the anonymised frame
//           anon[f][p] = u ? (255, 255, 255) : (R, G, B) of the B, G, R frame (cv2.imwrite stores the B, G, R copy as R, G, B).
//   rows    k_dm_rows: one warp per row, the horizontal half of cv2.dilate(u, ones(d, d)).
//   columns k_dm_col_ends + k_dm_cols: one thread per column segment of seg rows, the vertical half, then cv2.bitwise_not:
//           mask = dilated ? 0 : 255.
// cv2.dilate's window at output x is [x - a, x + b] with a = d / 2 (its default anchor) and b = d - 1 - a, so it is asymmetric for
// even d; pixels outside the image never contribute, and d = 0 (an empty kernel) is 3 x 3, as OpenCV substitutes.  Each half is
// binary: x is set iff the nearest set pixel at or before x is within a, or the nearest one at or after x is within b.  Both
// distances come from running scans, a forward and a backward sweep, so the cost per pixel does not depend on d.  The host clamps a
// and b to max(w, h) (a longer reach covers the same pixels), so every distance fits an int.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace rcvd {

constexpr int kDmThreads = 256;

struct DynMaskArgs {
  int w, h;
  int a, b;                     // the window [x - a, x + b] on both axes
  int frame0;                   // union / columns: first frame of this launch (blockIdx.y is relative to it)
  int F;                        // rows: frames of the call
  int seg;                      // columns: rows per column segment
  const long long* offsets;     // [frames + 1] instance runs
  const uint8_t* instances;     // [total][h][w], non-zero = inside
  const uint8_t* frames;        // [frames][h][w][3] B, G, R, or null
  uint8_t* u;                   // [frames][h][w] union (0 / 1), then the horizontal dilation
  uint8_t* mask;                // [frames][h][w] out
  int2* ends;                   // [frames][ceil(h / seg)][w] first and last set row of each column segment (-1: none)
  uint8_t* anon;                // [frames][h][w][3] R, G, B out, or null
};

// grid (ceil(plane / (kDmThreads * V)), frames of this launch), block kDmThreads; V = 16 reads 16-byte vectors and needs plane % 16 == 0
template <int V>
__global__ void __launch_bounds__(kDmThreads) k_dm_union(DynMaskArgs a) {
  const size_t plane = (size_t)a.w * a.h;
  const size_t f = (size_t)a.frame0 + blockIdx.y;
  const size_t p0 = ((size_t)blockIdx.x * kDmThreads + threadIdx.x) * V;
  if (p0 >= plane) return;
  const long long k0 = a.offsets[f], k1 = a.offsets[f + 1];
  uint8_t in[V];
  if constexpr (V == 16) {
    uint4 acc = make_uint4(0, 0, 0, 0);
    for (long long k = k0; k < k1; ++k) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(a.instances + (size_t)k * plane + p0));
      acc.x |= v.x; acc.y |= v.y; acc.z |= v.z; acc.w |= v.w;
    }
    const uint32_t wd[4] = {acc.x, acc.y, acc.z, acc.w};
#pragma unroll
    for (int i = 0; i < 16; ++i) in[i] = ((wd[i >> 2] >> (8 * (i & 3))) & 0xffu) != 0;
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) ow[j] = in[4 * j] | (in[4 * j + 1] << 8) | (in[4 * j + 2] << 16) | ((uint32_t)in[4 * j + 3] << 24);
    *reinterpret_cast<uint4*>(a.u + f * plane + p0) = o;
  } else {
    uint8_t acc = 0;
    for (long long k = k0; k < k1; ++k) acc |= __ldg(a.instances + (size_t)k * plane + p0);
    in[0] = acc != 0;
    a.u[f * plane + p0] = in[0];
  }
  if (a.anon) {
#pragma unroll
    for (int i = 0; i < V; ++i) {
      const size_t p = f * plane + p0 + i;
      const uint8_t* s = a.frames + p * 3;
      uint8_t* d = a.anon + p * 3;
      d[0] = in[i] ? 255 : s[2]; d[1] = in[i] ? 255 : s[1]; d[2] = in[i] ? 255 : s[0];
    }
  }
}

// grid (ceil(F * h / warps per block)), block kDmThreads: one warp per row, in place on u.  The forward sweep carries the last set
// column (a warp max scan plus the previous chunk's carry) and writes whether it is within a; the backward sweep carries the next
// set column (a min scan) and ORs in whether it is within b.  Each lane reads and writes only its own pixel.
__global__ void __launch_bounds__(kDmThreads) k_dm_rows(DynMaskArgs a) {
  const long long row = ((long long)blockIdx.x * kDmThreads + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= (long long)a.F * a.h) return;
  uint8_t* r = a.u + (size_t)row * a.w;
  // "no set pixel": with a, b <= max(w, h) < 2^30, x + 2^30 and 2^31 - 1 - x exceed any reach and cannot overflow
  const int none_before = -(1 << 30), none_after = 0x7fffffff;
  int carry = none_before;
  for (int x0 = 0; x0 < a.w; x0 += 32) {
    const int x = x0 + lane;
    const bool in = x < a.w;
    const uint8_t v = in ? r[x] : 0;
    int last = v ? x : none_before;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
      const int o = __shfl_up_sync(0xffffffffu, last, s);
      if (lane >= s) last = max(last, o);
    }
    last = max(last, carry);
    carry = __shfl_sync(0xffffffffu, last, 31);
    if (in) r[x] = (v ? 2 : 0) | ((x - last <= a.a) ? 1 : 0);   // bit 1 keeps the union pixel for the backward sweep
  }
  carry = none_after;
  const int nchunks = (a.w + 31) / 32;
  for (int c = nchunks - 1; c >= 0; --c) {
    const int x = c * 32 + lane;
    const bool in = x < a.w;
    const uint8_t v = in ? r[x] : 0;
    int next = (v & 2) ? x : none_after;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
      const int o = __shfl_down_sync(0xffffffffu, next, s);
      if (lane + s < 32) next = min(next, o);
    }
    next = min(next, carry);
    carry = __shfl_sync(0xffffffffu, next, 0);
    if (in) r[x] = ((v & 1) || next - x <= a.b) ? 1 : 0;
  }
}

// grid (ceil(w / kDmThreads), ceil(h / seg), frames of this launch), block kDmThreads: the first and last set row of each column
// segment of the horizontally dilated u, for k_dm_cols' carries between segments.
__global__ void __launch_bounds__(kDmThreads) k_dm_col_ends(DynMaskArgs a) {
  const int x = blockIdx.x * kDmThreads + threadIdx.x;
  if (x >= a.w) return;
  const size_t plane = (size_t)a.w * a.h, f = (size_t)a.frame0 + blockIdx.z;
  const int y0 = blockIdx.y * a.seg, y1 = min(a.h, y0 + a.seg);
  const uint8_t* src = a.u + f * plane + x;
  int first = -1, last = -1;
  for (int y = y0; y < y1; ++y)
    if (src[(size_t)y * a.w]) { if (first < 0) first = y; last = y; }
  a.ends[(f * gridDim.y + blockIdx.y) * a.w + x] = make_int2(first, last);
}

// grid as k_dm_col_ends, block kDmThreads: one thread per column segment, coalesced across the warp.  The carry into the segment (the
// last set row above it, the first set row below it) is that of the nearest segment holding one, from k_dm_col_ends' table; the
// lookup stops where no row of a farther segment can be within reach.  The forward sweep writes whether the last set row is within a
// into mask (as 1 / 0); the backward sweep ORs in whether the next set row is within b and writes the inverted result.
__global__ void __launch_bounds__(kDmThreads) k_dm_cols(DynMaskArgs a) {
  const int x = blockIdx.x * kDmThreads + threadIdx.x;
  if (x >= a.w) return;
  const size_t plane = (size_t)a.w * a.h, f = (size_t)a.frame0 + blockIdx.z;
  const int seg = blockIdx.y, nseg = gridDim.y;
  const int y0 = seg * a.seg, y1 = min(a.h, y0 + a.seg);
  const int2* ends = a.ends + f * nseg * a.w + x;
  const int none_before = -(1 << 30), none_after = 0x7fffffff;   // as in k_dm_rows
  int last = none_before, next = none_after;
  for (int s = seg - 1; s >= 0 && y0 - ((s + 1) * a.seg - 1) <= a.a; --s) {   // (s + 1) seg - 1: the closest row segment s holds
    const int l = ends[(size_t)s * a.w].y;
    if (l >= 0) { last = l; break; }
  }
  for (int s = seg + 1; s < nseg && s * a.seg - (y1 - 1) <= a.b; ++s) {
    const int n = ends[(size_t)s * a.w].x;
    if (n >= 0) { next = n; break; }
  }
  const uint8_t* src = a.u + f * plane + x;
  uint8_t* dst = a.mask + f * plane + x;
  for (int y = y0; y < y1; ++y) {
    if (src[(size_t)y * a.w]) last = y;
    dst[(size_t)y * a.w] = (y - last <= a.a) ? 1 : 0;
  }
  for (int y = y1 - 1; y >= y0; --y) {
    if (src[(size_t)y * a.w]) next = y;
    const bool set = dst[(size_t)y * a.w] || next - y <= a.b;
    dst[(size_t)y * a.w] = set ? 0 : 255;
  }
}

}  // namespace rcvd
