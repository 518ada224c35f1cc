// rcvd_tracks.cuh -- long point tracks on the GPU (DepthVideoProcessor::computeTracks, reference lib/Processor.cpp:646-886).
//
// The reference walks the frames in order.  In frame f it first continues the tracks of frame f-1 along the flow f-1 -> f, in
// ascending track id, dropping a track that lands inside the prune disc of one continued before it, then spawns new tracks at
// corner-like pixels (score descending) that no spawn disc covers yet.  Both greedy passes are lexicographically-first maximal
// independent sets and are computed by monotone rounds, as k_select_round does for the constraint builder:
//   1. k_tr_continue : one thread per track of f-1: flow-mask test, flow step, in-image and dynamic-distance tests (>=);
//   2. k_tr_prune_round : conflict = landing pixels within the prune radius, priority = track order.  Several tracks can land on one
//      pixel, so a round reads two pixel planes: the smallest accepted candidate index per pixel (monotone, read live) and the
//      smallest index still undecided after the previous round (rebuilt every round in a ring of three planes);
//   3. k_tr_stamp : spawn discs of the continued tracks;
//   4. k_tr_spawn_init / k_tr_spawn_round : the spawn greedy on the pixel plane.  The reference checks and stamps a candidate at the
//      re-derived pixel m(x, y) (pixel -> normalised location -> pixel, not the identity: some rows / columns map to y-1 / x-1), so
//      conflicts are tested between mapped positions; m moves a pixel by at most one, so a window of radius r+1 finds them all;
//   5. k_tr_emit : one CTA writes the frame's track list: continued tracks in id order, then the spawned ones in (score desc, scan
//      index asc) order, which the pixels were radix-sorted into (k_tr_sort_keys), with consecutive new ids.
// Float arithmetic is float32 with explicit _rn intrinsics in the reference's operation order (its build has no FMA contraction).
// Where the reference reads outside an image (a dynamic-distance lookup at -1, a track row rounded to h) the nearest pixel is read.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cub/block/block_scan.cuh>

namespace rcvd {

constexpr unsigned kTrNone = 0xffffffffu;
constexpr int kTrEmitThreads = 1024;

struct TrackArgs {
  int w, h, dw, dh;          // colour size; dynamic-distance size (= colour size without a dynamic mask)
  int spawn_r, prune_r;
  float min_dyn, ia, dsx, dsy;
  const float* dist;         // this frame's distance image [dh][dw], nullptr: FLT_MAX everywhere
};

__device__ __forceinline__ float tr_dist(const TrackArgs& a, int ys, int xs) {
  if (!a.dist) return 3.402823466e+38f;
  ys = min(max(ys, 0), a.dh - 1); xs = min(max(xs, 0), a.dw - 1);
  return a.dist[(size_t)ys * a.dw + xs];
}

// continuation tests of the tracks of frame f-1 (:772-803); state 0 = candidate, 2 = dropped.  und0[pixel] = smallest candidate index.
__global__ void __launch_bounds__(256) k_tr_continue(TrackArgs a, int n, const float* __restrict__ prev_loc, const float* __restrict__ flow,
                                                      const uint8_t* __restrict__ fmask, int* __restrict__ pix, float* __restrict__ loc,
                                                      uint8_t* __restrict__ state, unsigned* __restrict__ und0) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float fx0 = __fmul_rn(prev_loc[2 * i], (float)a.w), fy0 = __fmul_rn(__fdiv_rn(prev_loc[2 * i + 1], a.ia), (float)a.h);
  const int ix0 = min(max((int)__fadd_rn(fx0, 0.5f), 0), a.w - 1), iy0 = min(max((int)__fadd_rn(fy0, 0.5f), 0), a.h - 1);
  uint8_t st = 2;
  const size_t q = (size_t)iy0 * a.w + ix0;
  if (fmask[q]) {
    const float fx1 = __fadd_rn(fx0, flow[2 * q]), fy1 = __fadd_rn(fy0, flow[2 * q + 1]);
    const int ix1 = (int)__fadd_rn(fx1, 0.5f), iy1 = (int)__fadd_rn(fy1, 0.5f);   // truncation: fx1 in (-1.5, -0.5] gives 0
    if (ix1 >= 0 && ix1 < a.w && iy1 >= 0 && iy1 < a.h &&
        tr_dist(a, (int)__fmul_rn(fy1, a.dsy), (int)__fmul_rn(fx1, a.dsx)) >= a.min_dyn) {
      st = 0;
      const int p = iy1 * a.w + ix1;
      pix[i] = p;
      loc[2 * i] = __fdiv_rn(fx1, (float)a.w); loc[2 * i + 1] = __fmul_rn(__fdiv_rn(fy1, (float)a.h), a.ia);
      atomicMin(&und0[p], (unsigned)i);
    }
  }
  state[i] = st;
}

// One monotone round of the prune selection.  cnt[k] counts the candidates still undecided after round k; a round after a round that
// left none returns at once, so the host can enqueue more rounds than needed.  und_cur: undecided after round k-1 (read), und_next:
// undecided after round k (written), und_clear: reset for round k+1.  Threads cover max(n, w*h).
__global__ void __launch_bounds__(256) k_tr_prune_round(TrackArgs a, int n, int k, const int* __restrict__ pix, uint8_t* __restrict__ state,
                                                         unsigned* __restrict__ acc, const unsigned* __restrict__ und_cur,
                                                         unsigned* __restrict__ und_next, unsigned* __restrict__ und_clear, unsigned* __restrict__ cnt) {
  if (k > 0 && cnt[k - 1] == 0) return;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < a.w * a.h) und_clear[t] = kTrNone;
  if (t >= n || state[t] != 0) return;
  const int p = pix[t], y = p / a.w, x = p % a.w, r = a.prune_r, r2 = r * r;
  bool blocked = false;
  for (int yy = max(0, y - r); yy <= min(a.h - 1, y + r); ++yy) {
    const int dy = yy - y;
    for (int xx = max(0, x - r); xx <= min(a.w - 1, x + r); ++xx) {
      const int dx = xx - x;
      if (dx * dx + dy * dy > r2) continue;
      const int q = yy * a.w + xx;
      if (reinterpret_cast<volatile unsigned*>(acc)[q] < (unsigned)t) { state[t] = 2; return; }   // an earlier track was kept here
      if (und_cur[q] < (unsigned)t) blocked = true;
    }
  }
  if (blocked) { atomicAdd(&cnt[k], 1u); atomicMin(&und_next[p], (unsigned)t); }
  else { state[t] = 1; atomicMin(&acc[p], (unsigned)t); }
}

// spawn disc (createDiskKernel / splatKernel: rx^2 + ry^2 <= r^2, clipped to the image) of every continued track: one CTA per track
__global__ void __launch_bounds__(256) k_tr_stamp(TrackArgs a, const int* __restrict__ pix, const uint8_t* __restrict__ state, uint8_t* __restrict__ spawn_mask) {
  const int t = blockIdx.x;
  if (state[t] != 1) return;
  const int p = pix[t], y = p / a.w, x = p % a.w, r = a.spawn_r, d = 2 * r + 1;
  for (int k = threadIdx.x; k < d * d; k += blockDim.x) {
    const int dy = k / d - r, dx = k % d - r, yy = y + dy, xx = x + dx;
    if (yy >= 0 && yy < a.h && xx >= 0 && xx < a.w && dx * dx + dy * dy <= r * r) spawn_mask[yy * a.w + xx] = 1;
  }
}

// spawn candidates (:816-833): flow mask of f-1 -> f (if any), dynamic distance > min (strict), mapped pixel not yet covered
__global__ void __launch_bounds__(256) k_tr_spawn_init(TrackArgs a, const uint8_t* __restrict__ fmask, const uint8_t* __restrict__ spawn_mask,
                                                        const int* __restrict__ mx, const int* __restrict__ my, uint8_t* __restrict__ state) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.w * a.h) return;
  const int y = p / a.w, x = p % a.w;
  const bool cand = (!fmask || fmask[p]) && tr_dist(a, (int)__fmul_rn((float)y, a.dsy), (int)__fmul_rn((float)x, a.dsx)) > a.min_dyn;
  state[p] = (cand && !spawn_mask[my[y] * a.w + mx[x]]) ? 0 : 2;
}

// One monotone round of the spawn selection on mapped positions; priority (score desc, scan index asc).  Same early exit as the prune.
__global__ void __launch_bounds__(256) k_tr_spawn_round(TrackArgs a, int k, const float* __restrict__ score, const int* __restrict__ mx,
                                                         const int* __restrict__ my, uint8_t* __restrict__ state, unsigned* __restrict__ cnt) {
  if (k > 0 && cnt[k - 1] == 0) return;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.w * a.h || state[p] != 0) return;
  const float s = score[p];
  const int y = p / a.w, x = p % a.w, mxp = mx[x], myp = my[y], r = a.spawn_r, r2 = r * r, R = r + 1;
  bool blocked = false;
  for (int yy = max(0, y - R); yy <= min(a.h - 1, y + R); ++yy) {
    const int dy = my[yy] - myp;
    for (int xx = max(0, x - R); xx <= min(a.w - 1, x + R); ++xx) {
      const int q = yy * a.w + xx;
      if (q == p) continue;
      const uint8_t sq = reinterpret_cast<volatile uint8_t*>(state)[q];
      if (sq == 2) continue;
      const int dx = mx[xx] - mxp;
      if (dx * dx + dy * dy > r2) continue;
      const float t = score[q];
      if (!(t > s || (t == s && q < p))) continue;
      if (sq == 1) { state[p] = 2; return; }
      blocked = true;
    }
  }
  if (blocked) atomicAdd(&cnt[k], 1u); else state[p] = 1;
}

// sort keys: ascending key = score descending (-0 read as +0, as the comparison does), then pixel index ascending
__global__ void __launch_bounds__(256) k_tr_sort_keys(const float* __restrict__ score, int n, unsigned long long* __restrict__ keys) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const float s = score[p];
  unsigned u = s == 0.f ? 0u : __float_as_uint(s);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);   // order-preserving
  keys[p] = ((unsigned long long)(~u) << 32) | (unsigned)p;
}

// The frame's track list: continued tracks (candidate order = id order), then the spawned ones in sorted order with ids
// next_id, next_id + 1, ...  counts = {continued, spawned}.  One CTA.
__global__ void __launch_bounds__(kTrEmitThreads) k_tr_emit(TrackArgs a, int n_prev, const int* __restrict__ prev_id, const uint8_t* __restrict__ cstate,
                                                            const float* __restrict__ cloc, int spawn, const unsigned long long* __restrict__ sorted,
                                                            const uint8_t* __restrict__ sstate, int next_id, int* __restrict__ cur_id,
                                                            float* __restrict__ cur_loc, int* __restrict__ counts) {
  using Scan = cub::BlockScan<int, kTrEmitThreads>;
  __shared__ typename Scan::TempStorage tmp;
  int base = 0;
  for (int c0 = 0; c0 < n_prev; c0 += kTrEmitThreads) {
    const int i = c0 + threadIdx.x;
    const int f = (i < n_prev && cstate[i] == 1) ? 1 : 0;
    int r, tot;
    Scan(tmp).ExclusiveSum(f, r, tot);
    if (f) { cur_id[base + r] = prev_id[i]; cur_loc[2 * (base + r)] = cloc[2 * i]; cur_loc[2 * (base + r) + 1] = cloc[2 * i + 1]; }
    base += tot;
    __syncthreads();
  }
  const int n_cont = base;
  const int plane = a.w * a.h;
  if (spawn) {
    for (int c0 = 0; c0 < plane; c0 += kTrEmitThreads) {
      const int k = c0 + threadIdx.x;
      const int p = k < plane ? (int)(unsigned)sorted[k] : 0;
      const int f = (k < plane && sstate[p] == 1) ? 1 : 0;
      int r, tot;
      Scan(tmp).ExclusiveSum(f, r, tot);
      if (f) {
        const int o = base + r, y = p / a.w, x = p % a.w;
        cur_id[o] = next_id + (o - n_cont);
        cur_loc[2 * o] = __fdiv_rn((float)x, (float)a.w); cur_loc[2 * o + 1] = __fmul_rn(__fdiv_rn((float)y, (float)a.h), a.ia);
      }
      base += tot;
      __syncthreads();
    }
  }
  if (threadIdx.x == 0) { counts[0] = n_cont; counts[1] = base - n_cont; }
}

}  // namespace rcvd
