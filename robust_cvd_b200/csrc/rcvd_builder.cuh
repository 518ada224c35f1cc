// rcvd_builder.cuh -- GPU flow-constraint builder (SURVEY.md section 8f-2).
//
// Restates FlowConstraintsCollection::compute for pairs and triplets (reference lib/FlowConstraints.cpp:401-550) and the
// greedy disc sampler sampleConstraints (:352-397) for a whole batch of frame pairs / triplets at once:
//   1. k_gray / k_sobel_products / k_box_h / k_box_v_eig : cv::cvtColor(BGR2GRAY) + cv::cornerMinEigenVal(blockSize 3,
//      ksize 3, BORDER_REFLECT_101) per source frame in the exact operation order of OpenCV 4.13's AVX2 code paths
//      (found by search against cv2, tests/test_host.py): fused multiply-adds where OpenCV's universal intrinsics use
//      v_fma / v_muladd, the box sum in double like cv::boxFilter's CV_64F accumulator, everything else unfused float
//      (explicit _rn intrinsics) -- np.array_equal with cv2.cornerMinEigenVal and with robust_cvd_b200/host/constraints.cpp;
//   2. k_pair_candidates / k_triplet_candidates : the per-pixel admission tests (:427-457, :497-541), writing a per-item
//      priority plane (corner score) and state plane (0 candidate, 2 not a candidate);
//   3. k_select_round : the sequential sampler "sort by score, accept a pixel unless an accepted one lies within the disc"
//      is the lexicographically-first maximal independent set of the conflict graph (pixels <= separation apart) under the
//      priority (score descending, scan index ascending -- std::sort leaves ties unspecified in the reference).  It is
//      computed by monotone rounds: a candidate is accepted once every higher-priority candidate in its disc is rejected,
//      rejected as soon as one of them is accepted.  Identical result to the sequential loop, any number of rounds;
//   4. k_emit : survivors with their scaled locations (:330-342) and priority keys; the host part of the C ABI call orders
//      each item's survivors by priority (they are few: ~600 per pair at separation 10).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace rcvd {

__device__ __forceinline__ int reflect101(int p, int n) {
  if (n == 1) return 0;
  while (p < 0 || p >= n) p = p < 0 ? -p : 2 * n - 2 - p;
  return p;
}

// cv::cvtColor(BGR2GRAY), CV_32F: fma(r, 0.299f, fma(b, 0.114f, g * 0.587f))  (RGB2Gray<float> SIMD body)
__global__ void __launch_bounds__(256) k_gray(const float* __restrict__ bgr, float* __restrict__ gray, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float b = bgr[3 * i], g = bgr[3 * i + 1], r = bgr[3 * i + 2];
  gray[i] = __fmaf_rn(r, 0.299f, __fmaf_rn(b, 0.114f, __fmul_rn(g, 0.587f)));
}

// Sobel derivatives (scale 1/12 folded into the smoothing kernel, cv::Sobel) and their products; planes[0..2] = dx*dx, dx*dy, dy*dy.
//   dx: row [-1 0 1] unscaled, column [s 2s s]:  fma(rd[y-1] + rd[y+1], s, rd[y] * 2s)         (SymmColumnSmallVec_32f)
//   dy: row [s 2s s]: fma(M, 2s, (L + R) * s) in the vector body, fma(L + R, s, M * 2s) in the scalar tail x >= 4 floor(w / 4)
//       (SymmRowSmallVec_32f / the compiler-contracted scalar loop), column [-1 0 1]: rs[y+1] - rs[y-1]
__global__ void __launch_bounds__(256) k_sobel_products(const float* __restrict__ gray, float* __restrict__ planes, int F, int h, int w) {
  const size_t plane = (size_t)w * h, i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= plane * F) return;
  const int f = (int)(i / plane), p = (int)(i % plane), y = p / w, x = p % w;
  const float* G = gray + (size_t)f * plane;
  const float scale = 1.f / 12.f, scale2 = __fmul_rn(2.f, scale);
  const bool tail = x >= (w & ~3);
  float rd[3], rs[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int yy = reflect101(y + k - 1, h);
    const float a = G[(size_t)yy * w + reflect101(x - 1, w)], b = G[(size_t)yy * w + x], c = G[(size_t)yy * w + reflect101(x + 1, w)];
    rd[k] = __fsub_rn(c, a);
    const float lr = __fadd_rn(a, c);
    rs[k] = tail ? __fmaf_rn(lr, scale, __fmul_rn(b, scale2)) : __fmaf_rn(b, scale2, __fmul_rn(lr, scale));
  }
  const float dx = __fmaf_rn(__fadd_rn(rd[0], rd[2]), scale, __fmul_rn(rd[1], scale2));
  const float dy = __fsub_rn(rs[2], rs[0]);
  const size_t FP = plane * F;
  planes[i] = __fmul_rn(dx, dx); planes[FP + i] = __fmul_rn(dx, dy); planes[2 * FP + i] = __fmul_rn(dy, dy);
}
// 3x3 box sum of the three product planes (normalize = false): cv::boxFilter accumulates CV_32F input in double and rounds once --
// horizontal pass (RowSum, ksize 3: (a + b) + c in double), then the sliding vertical pass + min eigenvalue
__global__ void __launch_bounds__(256) k_box_h(const float* __restrict__ in, double* __restrict__ out, size_t rows, int w) {   // rows = 3*F*h
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * w) return;
  const size_t r = i / w; const int x = (int)(i % w);
  const float* R = in + r * w;
  out[i] = ((double)R[reflect101(x - 1, w)] + (double)R[x]) + (double)R[reflect101(x + 1, w)];
}
// Vertical pass exactly like cv::boxFilter's ColumnSum<double, float>: a running column sum SUM = rows[y-1] + rows[y] slides down the
// image (s0 = SUM + rows[y+1]; out = float(s0); SUM = s0 - rows[y-1]).  The double additions are almost always exact, but when the nine
// products sum to an exact float tie the last bit of the running double decides the rounding, so the recurrence is kept: one thread per
// (frame, column) walks the rows (loads coalesced across columns), three planes at once, and finishes with the min-eigenvalue formula.
__global__ void __launch_bounds__(128) k_box_v_eig(const double* __restrict__ tmp, float* __restrict__ score, int F, int h, int w) {
  const size_t plane = (size_t)w * h;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= F * w) return;
  const int f = i / w, x = i % w;
  const size_t FP = plane * F;
  const double* T0 = tmp + (size_t)f * plane + x; const double* T1 = T0 + FP; const double* T2 = T1 + FP;
  const size_t rm = (size_t)reflect101(-1, h) * w;
  double s[3] = {T0[rm] + T0[0], T1[rm] + T1[0], T2[rm] + T2[0]};
  for (int y = 0; y < h; ++y) {
    const size_t rn = (size_t)reflect101(y + 1, h) * w, ro = (size_t)reflect101(y - 1, h) * w;
    const double a0 = s[0] + T0[rn], a1 = s[1] + T1[rn], a2 = s[2] + T2[rn];
    s[0] = a0 - T0[ro]; s[1] = a1 - T1[ro]; s[2] = a2 - T2[ro];
    const float a = __fmul_rn((float)a0, 0.5f), b = (float)a1, c = __fmul_rn((float)a2, 0.5f);
    const float d = __fsub_rn(a, c);
    score[(size_t)f * plane + (size_t)y * w + x] = __fsub_rn(__fadd_rn(a, c), __fsqrt_rn(__fadd_rn(__fmul_rn(d, d), __fmul_rn(b, b))));
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// Static flags (reference FlowConstraintsCollection::setStaticFlagFromDynamicMask, lib/FlowConstraints.cpp:573-660, and
// dynamicDistance, :257-286): cv::distanceTransform(mask >= 127, DIST_L2, 5) per frame, then every constraint end looks its
// distance up.  OpenCV's 5x5 chamfer is a sequential two-pass scan in 16.16 fixed point; its in-row recurrence
//     d[x] = min(c[x], d[x-1] + 1.0)      (c[x]: candidates from the two rows above, already final)
// is a prefix minimum of c[k] - k * 1.0 (integers: associative, so the parallel scan is bit-identical to the sequential loop);
// rows stay sequential.  One CTA per frame, 256 columns per scan step, the forward values kept in a global scratch plane.
// ---------------------------------------------------------------------------------------------------------------------------
constexpr unsigned kChamHV = 65536u;
constexpr int kChamThreads = 256;

// inclusive prefix minimum over the block (thread order), combined with `carry` (minimum of everything before this chunk);
// returns the prefix value of this thread; carry is updated to include the whole chunk.  warp_sm: >= 8 ints of shared memory.
__device__ __forceinline__ int block_prefix_min(int v, int* warp_sm, int& carry) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v = min(v, t); }
  if (lane == 31) warp_sm[wid] = v;
  __syncthreads();
  int before = carry;
  for (int q = 0; q < wid; ++q) before = min(before, warp_sm[q]);
  int total = carry;
  for (int q = 0; q < kChamThreads / 32; ++q) total = min(total, warp_sm[q]);
  __syncthreads();
  carry = total;
  return min(v, before);
}

__global__ void __launch_bounds__(kChamThreads) k_chamfer5(const uint8_t* __restrict__ masks, unsigned* __restrict__ scratch, float* __restrict__ dist, int h, int w) {
  __shared__ int warp_sm[kChamThreads / 32];
  const unsigned DIAG = (unsigned)(1.4f * 65536.f + 0.5f), LONGW = (unsigned)(2.1969f * 65536.f + 0.5f);
  const unsigned INIT = 0x7fffffffu >> 2, DMAX = 0x7fffffffu - (1u << 16);
  const size_t plane = (size_t)w * h;
  const uint8_t* M = masks + blockIdx.x * plane;
  unsigned* T = scratch + blockIdx.x * plane;
  float* D = dist + blockIdx.x * plane;
  auto at = [&](int y, int x) -> unsigned { return (y < 0 || y >= h || x < 0 || x >= w) ? INIT : T[(size_t)y * w + x]; };
  // forward pass (top-left to bottom-right)
  for (int y = 0; y < h; ++y) {
    int carry = (int)(INIT + kChamHV);                 // d[-1] = INIT in the shifted domain: INIT - (-1) * HV
    for (int c0 = 0; c0 < w; c0 += kChamThreads) {
      const int x = c0 + threadIdx.x;
      int v = 0x7fffffff;
      if (x < w) {
        unsigned c = 0;
        if (M[(size_t)y * w + x] >= 127) {               // dynamicDistance binarises the mask: < 127 -> 0 (dynamic), else 255
          c = at(y - 2, x - 1) + LONGW;
          c = min(c, at(y - 2, x + 1) + LONGW); c = min(c, at(y - 1, x - 2) + LONGW); c = min(c, at(y - 1, x - 1) + DIAG);
          c = min(c, at(y - 1, x) + kChamHV); c = min(c, at(y - 1, x + 1) + DIAG); c = min(c, at(y - 1, x + 2) + LONGW);
        }
        v = (int)c - x * (int)kChamHV;
      }
      const int pm = block_prefix_min(v, warp_sm, carry);
      if (x < w) T[(size_t)y * w + x] = (unsigned)(pm + x * (int)kChamHV);
    }
    __syncthreads();                                     // row y visible to the whole block before row y + 1 reads it
  }
  // backward pass (bottom-right to top-left), mirrored column index j = w - 1 - x
  const float scale = 1.f / 65536.f;
  for (int y = h - 1; y >= 0; --y) {
    int carry = (int)(INIT + kChamHV);
    for (int c0 = 0; c0 < w; c0 += kChamThreads) {
      const int j = c0 + threadIdx.x, x = w - 1 - j;
      int v = 0x7fffffff;
      if (j < w) {
        unsigned c = T[(size_t)y * w + x];
        c = min(c, at(y + 2, x + 1) + LONGW); c = min(c, at(y + 2, x - 1) + LONGW); c = min(c, at(y + 1, x + 2) + LONGW);
        c = min(c, at(y + 1, x + 1) + DIAG); c = min(c, at(y + 1, x) + kChamHV); c = min(c, at(y + 1, x - 1) + DIAG);
        c = min(c, at(y + 1, x - 2) + LONGW);
        v = (int)c - j * (int)kChamHV;
      }
      const int pm = block_prefix_min(v, warp_sm, carry);
      if (j < w) {
        const unsigned d = (unsigned)(pm + j * (int)kChamHV);
        T[(size_t)y * w + x] = d;
        D[(size_t)y * w + x] = __fmul_rn(__uint2float_rn(min(d, DMAX)), scale);
      }
    }
    __syncthreads();
  }
}

// The pixel a constraint end is looked up at: (int(loc.x * w), int(loc.y * w)) -- the reference scales y by the image WIDTH as
// well (:618-621, :725-744) -- clamped to the image, where the reference indexes unchecked.
__device__ __forceinline__ int2 end_pixel(const float* loc, int h, int w) {
  const int ix = (int)__fmul_rn(loc[0], (float)w), iy = (int)__fmul_rn(loc[1], (float)w);
  return make_int2(min(max(ix, 0), w - 1), min(max(iy, 0), h - 1));
}

// isStatic of every pair / triplet constraint: dist > distance at all ends (end_pixel).  items: [n][3] frames (-1 = unused end),
// locs: [total][2 * ends] float32.
__global__ void __launch_bounds__(256) k_static_flags(const float* __restrict__ dist, int h, int w, float distance, int ends, const int* __restrict__ item_frames,
                                                       const long long* __restrict__ offsets, int nitems, const float* __restrict__ locs, uint8_t* __restrict__ flags) {
  const int item = blockIdx.y;
  if (item >= nitems) return;
  const long long b = offsets[item], n = offsets[item + 1] - b;
  const size_t plane = (size_t)w * h;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float* L = locs + (size_t)(b + i) * 2 * ends;
    bool st = true;
    for (int e = 0; e < ends; ++e) {
      const int f = item_frames[item * 3 + e];
      const int2 p = end_pixel(L + 2 * e, h, w);
      st = st && (dist[(size_t)f * plane + (size_t)p.y * w + p.x] > distance);
    }
    flags[b + i] = st ? 1 : 0;
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// Static-flag pruning (reference FlowConstraintsCollection::pruneStaticFlag, lib/FlowConstraints.cpp:662-748): every non-static pair
// constraint stamps a disc of radius `distance` around its end in each of its two frames; then every pair / triplet constraint with an
// end on a stamped pixel becomes non-static.  The per-frame byte masks of the reference are bit planes here, [F][h][words] u32 with
// words = ceil(w / 32), zeroed before the stamps; a disc row is one span of set bits, so it is stamped with a few word-wide atomicOr.
// ---------------------------------------------------------------------------------------------------------------------------
// One warp per non-static pair constraint, its lanes over the rows of each end's disc.  The centre is not clamped: the reference's
// loop bounds clip the disc to the image, so a centre at or beyond row h stamps only the disc rows that fall inside.  A pair whose two
// frames are equal stamps end 0 only (key.first == frame picks c[0]).  flags are the input flags, not yet pruned.
__global__ void __launch_bounds__(256) k_prune_stamp(unsigned* __restrict__ bits, int h, int w, int words, int distance, const int* __restrict__ pair_frames,
                                                      const long long* __restrict__ offsets, int npairs, const float* __restrict__ locs, const uint8_t* __restrict__ flags) {
  const int item = blockIdx.y;
  if (item >= npairs) return;
  const long long b = offsets[item], n = offsets[item + 1] - b;
  const int lane = threadIdx.x & 31, f0 = pair_frames[item * 3], f1 = pair_frames[item * 3 + 1];
  const long long d = distance, d2 = d * d;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long i = warp0; i < n; i += nwarps) {
    if (flags[b + i]) continue;
    const float* L = locs + (size_t)(b + i) * 4;
    for (int e = 0; e < (f0 == f1 ? 1 : 2); ++e) {
      const long long cx = (int)__fmul_rn(L[2 * e], (float)w), cy = (int)__fmul_rn(L[2 * e + 1], (float)w);
      unsigned* plane = bits + (size_t)(e ? f1 : f0) * h * words;
      for (long long y = max(0ll, cy - d) + lane; y <= min((long long)h - 1, cy + d); y += 32) {
        // half-width of the disc row: the largest k with k^2 + dy^2 <= d^2 (integer square root, corrected in 64-bit)
        const long long dy = y - cy, r2 = d2 - dy * dy;
        long long k = (long long)sqrt((double)r2);
        while (k * k > r2) --k;
        while ((k + 1) * (k + 1) <= r2) ++k;
        const long long x0 = max(0ll, cx - k), x1 = min((long long)w - 1, cx + k);
        if (x0 > x1) continue;
        unsigned* row = plane + (size_t)y * words;
        for (int wd = (int)(x0 >> 5); wd <= (int)(x1 >> 5); ++wd) {
          const int lo = max((int)x0 - 32 * wd, 0), hi = min((int)x1 - 32 * wd, 31);
          atomicOr(row + wd, (0xffffffffu >> (31 - hi)) & (0xffffffffu << lo));
        }
      }
    }
  }
}
// Shaped like k_static_flags: a static constraint with any end (end_pixel) on a stamped pixel becomes non-static; others keep their flag.
__global__ void __launch_bounds__(256) k_prune_lookup(const unsigned* __restrict__ bits, int h, int w, int words, int ends, const int* __restrict__ item_frames,
                                                       const long long* __restrict__ offsets, int nitems, const float* __restrict__ locs, uint8_t* __restrict__ flags) {
  const int item = blockIdx.y;
  if (item >= nitems) return;
  const long long b = offsets[item], n = offsets[item + 1] - b;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (!flags[b + i]) continue;
    const float* L = locs + (size_t)(b + i) * 2 * ends;
    bool hit = false;
    for (int e = 0; e < ends; ++e) {
      const int2 p = end_pixel(L + 2 * e, h, w);
      hit = hit || ((bits[((size_t)item_frames[item * 3 + e] * h + p.y) * words + (p.x >> 5)] >> (p.x & 31)) & 1u);
    }
    if (hit) flags[b + i] = 0;
  }
}

struct BuilderArgs {
  const float* corner;      // [F][h][w]
  const float* dyn;         // [F][dh][dw] or nullptr (no dynamic mask stream: distance = FLT_MAX everywhere)
  const int* pair_frames;   // [P][2]
  const float* pair_flow; const uint8_t* pair_mask;          // [P][h][w][2], [P][h][w]
  const int* trip_frames;   // [T] centre frame
  const float* trip_flow; const uint8_t* trip_mask;          // [T][2][h][w][2], [T][2][h][w]  (0: t -> t-1, 1: t -> t+1)
  float* prio; uint8_t* state;                               // [P+T][h][w]
  int P, T, h, w, dh, dw, sep;
  float min_dyn, dsx, dsy, sx, sy;
};

__device__ __forceinline__ float dyn_at(const BuilderArgs& a, int frame, int ys, int xs) {
  if (!a.dyn) return 3.402823466e+38f;
  ys = min(max(ys, 0), a.dh - 1); xs = min(max(xs, 0), a.dw - 1);   // the reference indexes without a bounds check
  return a.dyn[((size_t)frame * a.dh + ys) * a.dw + xs];
}

// pair admission (:427-457)
__global__ void __launch_bounds__(256) k_pair_candidates(BuilderArgs a) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x, item = blockIdx.y;
  const int plane = a.w * a.h;
  if (p >= plane) return;
  const int iy0 = p / a.w, ix0 = p % a.w;
  const int f0 = a.pair_frames[2 * item], f1 = a.pair_frames[2 * item + 1];
  const size_t q = (size_t)item * plane + p;
  bool ok = false;
  const int iy0s = (int)__fadd_rn(__fmul_rn((float)iy0, a.dsy), 0.5f), ix0s = (int)__fadd_rn(__fmul_rn((float)ix0, a.dsx), 0.5f);
  if (a.pair_mask[q] && dyn_at(a, f0, iy0s, ix0s) > a.min_dyn) {
    const float fx1 = __fadd_rn((float)ix0, a.pair_flow[2 * q]), fy1 = __fadd_rn((float)iy0, a.pair_flow[2 * q + 1]);
    const int ix1 = (int)__fadd_rn(fx1, 0.5f), iy1 = (int)__fadd_rn(fy1, 0.5f);
    if (ix1 >= 0 && ix1 < a.w && iy1 >= 0 && iy1 < a.h) {
      const int ix1s = (int)__fadd_rn(__fmul_rn(fx1, a.dsx), 0.5f), iy1s = (int)__fadd_rn(__fmul_rn(fy1, a.dsy), 0.5f);
      ok = dyn_at(a, f1, iy1s, ix1s) > a.min_dyn;
    }
  }
  a.state[q] = ok ? 0 : 2;
  a.prio[q] = a.corner[(size_t)f0 * plane + p];
}
// triplet admission (:497-541), quirks kept: the score is read at column ix0 (the flowed x of frame t-1) of row iy1, and the
// third dynamic test uses the distance image of the centre frame
__global__ void __launch_bounds__(256) k_triplet_candidates(BuilderArgs a) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x, t = blockIdx.y;
  const int plane = a.w * a.h;
  if (p >= plane) return;
  const int iy1 = p / a.w, ix1 = p % a.w;
  const int fc = a.trip_frames[t];
  const size_t q0 = ((size_t)t * 2) * plane + p, q2 = ((size_t)t * 2 + 1) * plane + p, o = (size_t)(a.P + t) * plane + p;
  bool ok = false; float score = 0.f;
  const int iy1s = (int)__fadd_rn(__fmul_rn((float)iy1, a.dsy), 0.5f), ix1s = (int)__fadd_rn(__fmul_rn((float)ix1, a.dsx), 0.5f);
  if (a.trip_mask[q0] && a.trip_mask[q2] && dyn_at(a, fc, iy1s, ix1s) > a.min_dyn) {
    const float fx0 = __fadd_rn((float)ix1, a.trip_flow[2 * q0]), fy0 = __fadd_rn((float)iy1, a.trip_flow[2 * q0 + 1]);
    const int ix0 = (int)__fadd_rn(fx0, 0.5f), iy0 = (int)__fadd_rn(fy0, 0.5f);
    const float fx2 = __fadd_rn((float)ix1, a.trip_flow[2 * q2]), fy2 = __fadd_rn((float)iy1, a.trip_flow[2 * q2 + 1]);
    const int ix2 = (int)__fadd_rn(fx2, 0.5f), iy2 = (int)__fadd_rn(fy2, 0.5f);
    if (ix0 >= 0 && ix0 < a.w && iy0 >= 0 && iy0 < a.h && ix2 >= 0 && ix2 < a.w && iy2 >= 0 && iy2 < a.h) {
      const int ix0s = (int)__fadd_rn(__fmul_rn(fx0, a.dsx), 0.5f), iy0s = (int)__fadd_rn(__fmul_rn(fy0, a.dsy), 0.5f);
      const int ix2s = (int)__fadd_rn(__fmul_rn(fx2, a.dsx), 0.5f), iy2s = (int)__fadd_rn(__fmul_rn(fy2, a.dsy), 0.5f);
      if (dyn_at(a, fc - 1, iy0s, ix0s) > a.min_dyn && dyn_at(a, fc, iy2s, ix2s) > a.min_dyn) {
        ok = true; score = a.corner[(size_t)fc * plane + (size_t)iy1 * a.w + ix0];
      }
    }
  }
  a.state[o] = ok ? 0 : 2;
  a.prio[o] = score;
}

// One monotone round of the greedy-equivalent selection.  state: 0 undecided candidate, 1 accepted, 2 rejected / not a candidate.
__global__ void __launch_bounds__(256) k_select_round(BuilderArgs a, unsigned long long* __restrict__ undecided) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x, item = blockIdx.y;
  const int plane = a.w * a.h;
  if (p >= plane) return;
  uint8_t* st = a.state + (size_t)item * plane;
  if (st[p] != 0) return;
  const float* pr = a.prio + (size_t)item * plane;
  const float s = pr[p];
  const int y = p / a.w, x = p % a.w, sep = a.sep, sep2 = sep * sep;
  const int y0 = max(0, y - sep), y1 = min(a.h - 1, y + sep), x0 = max(0, x - sep), x1 = min(a.w - 1, x + sep);
  bool blocked = false;
  for (int yy = y0; yy <= y1; ++yy) {
    const int dy = yy - y;
    for (int xx = x0; xx <= x1; ++xx) {
      const int dx = xx - x;
      if (dx * dx + dy * dy > sep2) continue;
      const int q = yy * a.w + xx;
      if (q == p) continue;
      const uint8_t sq = reinterpret_cast<volatile uint8_t*>(st)[q];
      if (sq == 2) continue;
      const float t = pr[q];
      if (!(t > s || (t == s && q < p))) continue;      // q sorts after p: it cannot stop p
      if (sq == 1) { st[p] = 2; return; }                // inside the disc of an accepted, earlier pixel
      blocked = true;                                    // an earlier pixel is still undecided
    }
  }
  if (blocked) atomicAdd(undecided, 1ull); else st[p] = 1;
}

__global__ void __launch_bounds__(256) k_count_accepted(BuilderArgs a, unsigned long long* __restrict__ counts) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x, item = blockIdx.y;
  const int plane = a.w * a.h;
  const bool acc = p < plane && a.state[(size_t)item * plane + p] == 1;
  const unsigned m = __ballot_sync(0xffffffffu, acc);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(&counts[item], (unsigned long long)__popc(m));
}
// survivors -> (pixel index, score, scaled locations); order within an item is arbitrary here
__global__ void __launch_bounds__(256) k_emit(BuilderArgs a, const unsigned long long* __restrict__ offsets, unsigned long long* __restrict__ cursor,
                                              int* __restrict__ out_idx, float* __restrict__ out_score, float* __restrict__ pair_out, float* __restrict__ trip_out,
                                              unsigned long long pair_total) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x, item = blockIdx.y;
  const int plane = a.w * a.h;
  if (p >= plane || a.state[(size_t)item * plane + p] != 1) return;
  const unsigned long long slot = offsets[item] + atomicAdd(&cursor[item], 1ull);
  out_idx[slot] = p; out_score[slot] = a.prio[(size_t)item * plane + p];
  const int y = p / a.w, x = p % a.w;
  if (item < a.P) {
    const size_t q = (size_t)item * plane + p;
    const float fx1 = __fadd_rn((float)x, a.pair_flow[2 * q]), fy1 = __fadd_rn((float)y, a.pair_flow[2 * q + 1]);
    float* o = pair_out + slot * 4;
    o[0] = __fmul_rn((float)x, a.sx); o[1] = __fmul_rn((float)y, a.sy); o[2] = __fmul_rn(fx1, a.sx); o[3] = __fmul_rn(fy1, a.sy);
  } else {
    const int t = item - a.P;
    const size_t q0 = ((size_t)t * 2) * plane + p, q2 = ((size_t)t * 2 + 1) * plane + p;
    const float fx0 = __fadd_rn((float)x, a.trip_flow[2 * q0]), fy0 = __fadd_rn((float)y, a.trip_flow[2 * q0 + 1]);
    const float fx2 = __fadd_rn((float)x, a.trip_flow[2 * q2]), fy2 = __fadd_rn((float)y, a.trip_flow[2 * q2 + 1]);
    float* o = trip_out + (slot - pair_total) * 6;
    o[0] = __fmul_rn(fx0, a.sx); o[1] = __fmul_rn(fy0, a.sy); o[2] = __fmul_rn((float)x, a.sx); o[3] = __fmul_rn((float)y, a.sy);
    o[4] = __fmul_rn(fx2, a.sx); o[5] = __fmul_rn(fy2, a.sy);
  }
}

}  // namespace rcvd
