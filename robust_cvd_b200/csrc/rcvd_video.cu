// rcvd_video.cu -- C ABI (include/rcvd.h) of the video-processing entry points: dense depth / spatial transforms, the flow-guided
// and bilateral depth filters, the flow-constraint builder, static flags and their pruning, long point tracks, the flow-consistency masks, the flow visualisations, the downscaled colour frames, the depth visualisations, the homography-registered flows and the dynamic-object masks.  Like the solver (rcvd_api.cu) they
// have NO CPU fallback: without a usable CUDA device every one of them fails with RCVD_ERR_NO_DEVICE.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <optional>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include "rcvd_host.h"
#include "rcvd_dense.cuh"
#include "rcvd_filter.cuh"
#include "rcvd_bilateral.cuh"
#include "rcvd_builder.cuh"
#include "rcvd_tracks.cuh"
#include "rcvd_flowmask.cuh"
#include "rcvd_flowvis.cuh"
#include "rcvd_resize.cuh"
#include "rcvd_depthvis.cuh"
#include "rcvd_flowreg.cuh"
#include "rcvd_dynmask.cuh"

using namespace rcvd;

// The device side of one video entry point: the device made current, a stream of its own and every buffer allocated on it.
// The destructor frees the buffers, waits for the stream and destroys it, and only then makes the caller's device current again.
struct VideoCall {
  std::optional<DevGuard> guard;
  cudaStream_t st = nullptr;
  std::vector<void*> bufs;
  bool ok = true;
  int64_t* launches = nullptr;
  VideoCall() = default;
  VideoCall(const VideoCall&) = delete;
  VideoCall& operator=(const VideoCall&) = delete;
  int open(int device, int64_t& launch_count) {   // launch() adds to the entry point's rcvd_*_launch_count counter
    if (int rc = check_device(device)) return rc;
    guard.emplace(device);
    if (guard->err != cudaSuccess) return set_err(RCVD_ERR_CUDA, "cudaSetDevice(%d) failed: %s", device, cudaGetErrorString(guard->err));
    cudaStream_t s;
    CK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    st = s;
    launches = &launch_count;
    return RCVD_OK;
  }
  template <class... Params, class... Args>
  int launch(void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, Args... args) {
    if (int rc = launch_kernel(kernel, grid, block, smem, st, false, args...)) return rc;
    ++*launches;
    return RCVD_OK;
  }
  // at least 16 bytes; a failure is remembered for allocated() and cleared from the runtime's last error
  void* alloc(size_t bytes) {
    void* ptr = nullptr;
    if (cudaMallocAsync(&ptr, std::max<size_t>(bytes, 16), st) != cudaSuccess) { ok = false; cudaGetLastError(); return nullptr; }
    bufs.push_back(ptr);
    return ptr;
  }
  void* upload(const void* src, size_t bytes) {
    void* d = alloc(bytes);
    if (d && src && bytes) cudaMemcpyAsync(d, src, bytes, cudaMemcpyHostToDevice, st);
    return d;
  }
  // checked before the first launch: a kernel on a null buffer faults with an illegal address, a sticky error of the whole
  // context, and PyTorch shares this context
  bool allocated() const { return ok; }
  // errors of the unchecked copies, memsets and sort, then the stream's; both always run, so no copy into host memory is pending after
  int sync(const char* what) {
    const cudaError_t enq = cudaGetLastError();
    const cudaError_t e = cudaStreamSynchronize(st);
    if (enq != cudaSuccess || e != cudaSuccess) return set_err(RCVD_ERR_CUDA, "%s failed: %s", what, cudaGetErrorString(enq != cudaSuccess ? enq : e));
    return RCVD_OK;
  }
  ~VideoCall() {
    if (!st) return;
    for (void* b : bufs) cudaFreeAsync(b, st);
    cudaStreamSynchronize(st); cudaStreamDestroy(st);
  }
};

// ---- dense transform application (next-row kernels) ----
template <int MODE>
static int dense_run(const rcvd_config* cfg, int device, const double* params_in, int nparams, int param_off, const float* src, void* out, size_t out_bytes, int h, int w) {
  Layout L;
  if (!cfg || !make_layout(*cfg, L)) return set_err(RCVD_ERR_INVALID, "unsupported transform configuration");
  if (int rc = check_device(device)) return rc;
  SET_DEVICE(device);
  std::vector<double> pv(L.nf, 0.0);
  for (int i = 0; i < nparams; ++i) pv[param_off + i] = params_in[i];
  double* d_p = nullptr; float* d_src = nullptr; void* d_out = nullptr;
  const size_t n = (size_t)w * h;
  // per-frame calls (DepthFrame::depth(), paramMap, warp for every frame of a video): stream-ordered pool allocations and one
  // synchronisation instead of three cudaMalloc/cudaFree pairs per call
  static thread_local cudaStream_t st = nullptr; static thread_local int st_dev = -1;
  if (!st || st_dev != device) {
    if (st) cudaStreamDestroy(st);
    CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking)); st_dev = device;
    cudaMemPool_t pool; unsigned long long keep = ~0ull;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
  }
  CK(cudaMallocAsync((void**)&d_p, pv.size() * 8, st)); CK(cudaMallocAsync(&d_out, out_bytes, st));
  CK(cudaMemcpyAsync(d_p, pv.data(), pv.size() * 8, cudaMemcpyHostToDevice, st));
  if (src) { CK(cudaMallocAsync((void**)&d_src, n * 4, st)); CK(cudaMemcpyAsync(d_src, src, n * 4, cudaMemcpyHostToDevice, st)); }
  const int rc = launch_kernel(k_dense<MODE>, nblk(n), 256, 0, st, false, *cfg, L, d_p, d_src, d_out, h, w);
  cudaError_t e = rc ? cudaSuccess : cudaMemcpyAsync(out, d_out, out_bytes, cudaMemcpyDeviceToHost, st);
  cudaFreeAsync(d_p, st); cudaFreeAsync(d_out, st); if (d_src) cudaFreeAsync(d_src, st);
  if (rc) return rc;
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return set_err(RCVD_ERR_CUDA, "dense kernel failed: %s", cudaGetErrorString(e));
  return RCVD_OK;
}
RCVD_API int32_t rcvd_depth_apply(const rcvd_config* cfg, int32_t device, const double* dp, const float* src, float* dst, int32_t h, int32_t w) {
  Layout L; if (!cfg || !make_layout(*cfg, L)) return set_err(RCVD_ERR_INVALID, "unsupported transform configuration");
  return dense_run<0>(cfg, device, dp, L.nd, L.offD, src, dst, (size_t)w * h * 4, h, w);
}
RCVD_API int32_t rcvd_depth_param_map(const rcvd_config* cfg, int32_t device, const double* dp, double* out, int32_t h, int32_t w) {
  Layout L; if (!cfg || !make_layout(*cfg, L)) return set_err(RCVD_ERR_INVALID, "unsupported transform configuration");
  if (cfg->depth_type != RCVD_DEPTH_GRID) return set_err(RCVD_ERR_INVALID, "Parameter map not implemented for this transform type.");
  return dense_run<1>(cfg, device, dp, L.nd, L.offD, nullptr, out, (size_t)w * h * L.k * 8, h, w);
}
RCVD_API int32_t rcvd_spatial_warp(const rcvd_config* cfg, int32_t device, const double* sp, float* out, int32_t h, int32_t w) {
  Layout L; if (!cfg || !make_layout(*cfg, L)) return set_err(RCVD_ERR_INVALID, "unsupported transform configuration");
  return dense_run<2>(cfg, device, sp, L.ns, L.offS, nullptr, out, (size_t)w * h * 8, h, w);
}

RCVD_API int32_t rcvd_trim_device_memory(int32_t device) {
  if (int rc = check_device(device)) return rc;
  SET_DEVICE(device);
  CK(cudaDeviceSynchronize());
  cudaMemPool_t pool;
  CK(cudaDeviceGetDefaultMemPool(&pool, device));
  CK(cudaMemPoolTrimTo(pool, 0));
  unsigned long long none = 0;                       // rcvd_problem_create raises the threshold again for the next solve
  cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &none);
  return RCVD_OK;
}
// The device the host layer should work on: RCVD_DEVICE if set, else the caller's current CUDA device (so that a process launched
// per GPU -- torchrun LOCAL_RANK + torch.cuda.set_device -- lands on its own GPU); -1 without a usable device.
RCVD_API int32_t rcvd_current_device(void) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { cudaGetLastError(); return -1; }
  if (const char* e = getenv("RCVD_DEVICE")) { const int d = atoi(e); return (d >= 0 && d < ndev) ? d : -1; }
  int d = 0;
  if (cudaGetDevice(&d) != cudaSuccess) { cudaGetLastError(); return -1; }
  return d;
}

// ---------------------------------------------------------------------------
// Flow-guided temporal depth filter (rcvd_filter.cuh)
// ---------------------------------------------------------------------------
static int64_t g_filter_launches = 0;
RCVD_API int32_t rcvd_flow_guided_filter(const rcvd_filter_params* prm, int32_t device, const float* depth, const float* cams,
                                         const float* fwd_flow, const uint8_t* fwd_mask, const float* bwd_flow, const uint8_t* bwd_mask,
                                         const int32_t* far_pairs, const float* far_flow, const uint8_t* far_mask, float* out) {
  if (!prm || !depth || !cams || !out) return set_err(RCVD_ERR_INVALID, "null argument");
  const rcvd_filter_params& q = *prm;
  if (q.num_frames <= 0 || q.num_out <= 0 || q.first_out < 0 || q.first_out + q.num_out > q.num_frames || q.width <= 0 || q.height <= 0 ||
      q.depth_width <= 0 || q.depth_height <= 0 || q.frame_radius < 0 || q.spatial_radius < 0 || q.num_far < 0 || !(q.inv_aspect > 0.f))
    return set_err(RCVD_ERR_INVALID, "bad filter parameters");
  if (q.frame_radius > 0 && q.num_frames > 1 && (!fwd_flow || !fwd_mask || !bwd_flow || !bwd_mask)) return set_err(RCVD_ERR_INVALID, "flow stacks missing");
  if (q.num_far > 0 && (!far_pairs || !far_flow || !far_mask)) return set_err(RCVD_ERR_INVALID, "far-connection arrays missing");
  VideoCall call;
  if (int rc = call.open(device, g_filter_launches)) return rc;
  const int F = q.num_frames; const size_t plane = (size_t)q.width * q.height, dplane = (size_t)q.depth_width * q.depth_height;
  // cameras: tan(fov / 2) in float on the host, like DepthVideo::project (lib/DepthVideo.cpp:640-641)
  std::vector<float> hc((size_t)F * 12, 0.f);
  for (int f = 0; f < F; ++f) {
    for (int i = 0; i < 7; ++i) hc[(size_t)f * 12 + i] = cams[(size_t)f * 9 + i];
    hc[(size_t)f * 12 + 7] = std::tan(cams[(size_t)f * 9 + 7] / 2.f);
    hc[(size_t)f * 12 + 8] = std::tan(cams[(size_t)f * 9 + 8] / 2.f);
  }
  // far connections grouped by source frame (stable: the caller's order within a frame is kept)
  std::vector<int> far_begin(F + 1, 0), order(q.num_far), pairs_sorted((size_t)2 * q.num_far);
  int maxfar = 0;
  for (int k = 0; k < q.num_far; ++k) {
    const int s = far_pairs[2 * k], d = far_pairs[2 * k + 1];
    if (s < 0 || s >= F || d < 0 || d >= F) return set_err(RCVD_ERR_INVALID, "far connection %d out of range", k);
    far_begin[s + 1]++;
  }
  for (int f = 0; f < F; ++f) { maxfar = std::max(maxfar, far_begin[f + 1]); far_begin[f + 1] += far_begin[f]; }
  { std::vector<int> cur(far_begin.begin(), far_begin.end() - 1); for (int k = 0; k < q.num_far; ++k) order[cur[far_pairs[2 * k]]++] = k; }
  FilterArgs a{};
  a.depth = (const float*)call.upload(depth, (size_t)F * dplane * 4);
  a.cams = (const float*)call.upload(hc.data(), hc.size() * 4);
  const bool chains = q.frame_radius > 0 && F > 1;
  a.fwd_flow = (const float*)call.upload(chains ? fwd_flow : nullptr, chains ? (size_t)F * plane * 8 : 0); a.fwd_mask = (const uint8_t*)call.upload(chains ? fwd_mask : nullptr, chains ? (size_t)F * plane : 0);
  a.bwd_flow = (const float*)call.upload(chains ? bwd_flow : nullptr, chains ? (size_t)F * plane * 8 : 0); a.bwd_mask = (const uint8_t*)call.upload(chains ? bwd_mask : nullptr, chains ? (size_t)F * plane : 0);
  if (q.num_far > 0) {
    float* ff = (float*)call.alloc((size_t)q.num_far * plane * 8); uint8_t* fm = (uint8_t*)call.alloc((size_t)q.num_far * plane);
    if (ff && fm)
      for (int k = 0; k < q.num_far; ++k) {   // sorted order on the device
        cudaMemcpyAsync(ff + (size_t)k * plane * 2, far_flow + (size_t)order[k] * plane * 2, plane * 8, cudaMemcpyHostToDevice, call.st);
        cudaMemcpyAsync(fm + (size_t)k * plane, far_mask + (size_t)order[k] * plane, plane, cudaMemcpyHostToDevice, call.st);
        pairs_sorted[2 * k] = far_pairs[2 * order[k]]; pairs_sorted[2 * k + 1] = far_pairs[2 * order[k] + 1];
      }
    a.far_flow = ff; a.far_mask = fm;
    a.far_pairs = (const int*)call.upload(pairs_sorted.data(), pairs_sorted.size() * 4);
    a.far_begin = (const int*)call.upload(far_begin.data(), far_begin.size() * 4);
  }
  float* const out_dev = (float*)call.alloc((size_t)q.num_out * plane * 4);
  const int win = 2 * q.spatial_radius + 1;
  a.max_samples = win * win * (1 + 2 * q.frame_radius + maxfar);
  // the weighted median sorts a per-pixel sample row: the scratch is bounded to ~1 GiB by filtering the range in frame chunks
  const size_t per_frame_scratch = plane * (size_t)a.max_samples * sizeof(float2);
  const int chunk = q.median ? (int)std::max<size_t>(1, std::min<size_t>((size_t)q.num_out, ((size_t)1 << 30) / std::max<size_t>(per_frame_scratch, 1))) : q.num_out;
  if (q.median) a.scratch = (float2*)call.alloc((size_t)chunk * per_frame_scratch);
  if (!call.allocated()) return set_err(RCVD_ERR_CUDA, "device allocation failed in rcvd_flow_guided_filter");
  cudaMemsetAsync(out_dev, 0, (size_t)q.num_out * plane * 4, call.st);
  a.F = F; a.last_frame = q.first_out + q.num_out - 1;
  a.w = q.width; a.h = q.height; a.wd = q.depth_width; a.hd = q.depth_height;
  a.frame_radius = q.frame_radius; a.spatial_radius = q.spatial_radius; a.median = q.median; a.inv_aspect = q.inv_aspect;
  for (int c0 = 0; c0 < q.num_out; c0 += chunk) {
    a.first_out = q.first_out + c0; a.num_out = std::min(chunk, q.num_out - c0); a.out = out_dev + (size_t)c0 * plane;
    const dim3 grid((q.width + 31) / 32, (q.height + 3) / 4, a.num_out);
    if (int rc = call.launch(q.median ? k_flow_guided_filter<true> : k_flow_guided_filter<false>, grid, 128, 0, a)) return rc;
  }
  cudaMemcpyAsync(out, out_dev, (size_t)q.num_out * plane * 4, cudaMemcpyDeviceToHost, call.st);
  return call.sync("flow-guided filter");
}
RCVD_API int64_t rcvd_filter_launch_count() { return g_filter_launches; }

// ---------------------------------------------------------------------------
// Joint depth / colour bilateral filter (rcvd_bilateral.cuh)
// ---------------------------------------------------------------------------
RCVD_API int32_t rcvd_bilateral_filter(const rcvd_bilateral_params* prm, int32_t device, const float* depth, const float* color_bgr,
                                       const int32_t* out_frames, const rcvd_config* xform_cfg, const double* xform_params, float* out) {
  if (!prm || !depth || !out_frames || !out) return set_err(RCVD_ERR_INVALID, "null argument");
  const rcvd_bilateral_params& q = *prm;
  const int F = q.num_frames;
  if (F <= 0 || q.width <= 0 || q.height <= 0 || q.num_out <= 0 || q.frame_radius < 0 || q.spatial_radius < 0 || (q.median != 0 && q.median != 1))
    return set_err(RCVD_ERR_INVALID, "bad bilateral filter parameters");
  for (int i = 0; i < q.num_out; ++i)
    if (out_frames[i] < 0 || out_frames[i] >= F || (i > 0 && out_frames[i] <= out_frames[i - 1]))
      return set_err(RCVD_ERR_INVALID, "output frames must be ascending local indices in [0, num_frames)");
  const bool color = q.color_sigma > 0.f;
  if (color && !color_bgr) return set_err(RCVD_ERR_INVALID, "color_sigma > 0 needs the colour stack");
  // in place, a later output frame reads xform(filtered) of the frames before it (the reference writes into the stream it reads)
  const bool recur = q.in_place != 0 && q.frame_radius > 0;
  Layout L{};
  if (recur) {
    if (!xform_cfg || !make_layout(*xform_cfg, L)) return set_err(RCVD_ERR_INVALID, "in-place filtering needs a supported depth-transform configuration");
    if (L.nd > 0 && !xform_params) return set_err(RCVD_ERR_INVALID, "in-place filtering needs the per-frame depth-transform parameters");
  }
  const long long r = q.spatial_radius, fr = q.frame_radius;
  const long long max_samples = std::min<long long>(2 * r + 1, q.width) * std::min<long long>(2 * r + 1, q.height) * std::min<long long>(2 * fr + 1, F);
  if (q.median && max_samples > kBilateralMaxSamples)
    return set_err(RCVD_ERR_INVALID, "the weighted median supports at most %d samples per pixel; this window has %lld", kBilateralMaxSamples, max_samples);
  VideoCall call;
  if (int rc = call.open(device, g_filter_launches)) return rc;
  const size_t plane = (size_t)q.width * q.height;
  // launch geometry and shared memory
  BilateralArgs a{};
  a.F = F; a.w = q.width; a.h = q.height; a.frame_radius = q.frame_radius; a.radius = q.spatial_radius;
  a.use_depth = q.depth_sigma > 0.f; a.depth_sigma = q.depth_sigma; a.color_sigma = q.color_sigma;
  size_t smem = 0; bool staged = false;
  if (q.median) {
    a.P = 32; while (a.P < max_samples) a.P <<= 1;
    smem = (size_t)kBfMedianWarps * a.P * sizeof(unsigned long long);
  } else {
    a.sw = kBfTx + 2 * q.spatial_radius; a.sh = kBfTy + 2 * q.spatial_radius;
    const size_t bytes = 2 * (size_t)a.sw * a.sh * (color ? 4 : 1) * sizeof(float);   // two frame buffers
    staged = bytes <= 200 * 1024;
    smem = staged ? bytes : 0;
  }
  void (*const filter)(BilateralArgs) = q.median ? (color ? k_bilateral_median<true> : k_bilateral_median<false>)
                                      : color    ? (staged ? k_bilateral_mean<true, true> : k_bilateral_mean<true, false>)
                                                 : (staged ? k_bilateral_mean<false, true> : k_bilateral_mean<false, false>);
  auto launch_filter = [&](int base, int n) {
    a.out_base = base;
    const dim3 grid = q.median ? dim3((unsigned)((plane + kBfMedianWarps - 1) / kBfMedianWarps), 1, n)
                               : dim3((q.width + kBfTx - 1) / kBfTx, (q.height + kBfTy - 1) / kBfTy, n);
    return call.launch(filter, grid, q.median ? 32 * kBfMedianWarps : kBfTx * kBfTy, smem, a);
  };
  if (smem > 48 * 1024) CK(cudaFuncSetAttribute((const void*)filter, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // per-frame transform vectors in the dense kernel's frame layout (depth parameters at offD)
  std::vector<double> pv;
  if (recur) {
    pv.assign((size_t)F * L.nf, 0.0);
    for (int f = 0; f < F; ++f) for (int i = 0; i < L.nd; ++i) pv[(size_t)f * L.nf + L.offD + i] = xform_params[(size_t)f * L.nd + i];
  }
  float* d_depth = (float*)call.upload(depth, (size_t)F * plane * 4);
  a.depth = d_depth;
  a.color = color ? (const float*)call.upload(color_bgr, (size_t)F * plane * 12) : nullptr;
  a.out_frames = (const int*)call.upload(out_frames, (size_t)q.num_out * 4);
  float* const out_dev = (float*)call.alloc((size_t)q.num_out * plane * 4);
  const double* d_pv = recur ? (const double*)call.upload(pv.data(), pv.size() * 8) : nullptr;
  if (!call.allocated()) return set_err(RCVD_ERR_CUDA, "device allocation failed in rcvd_bilateral_filter");
  if (recur) {
    // frame-sequential: filter output o, then rewrite its slot of the depth stack with xform_o(filtered) for the frames after it
    for (int o = 0; o < q.num_out; ++o) {
      a.out = out_dev + (size_t)o * plane;
      if (int rc = launch_filter(o, 1)) return rc;
      const int f = out_frames[o];
      if (int rc = call.launch(k_dense<0>, nblk(plane), 256, 0, *xform_cfg, L, d_pv + (size_t)f * L.nf, a.out, d_depth + (size_t)f * plane, q.height, q.width)) return rc;
    }
  } else {
    for (int o = 0; o < q.num_out; o += 65535) {   // grid.z limit
      a.out = out_dev + (size_t)o * plane;
      if (int rc = launch_filter(o, std::min(65535, q.num_out - o))) return rc;
    }
  }
  cudaMemcpyAsync(out, out_dev, (size_t)q.num_out * plane * 4, cudaMemcpyDeviceToHost, call.st);
  return call.sync("bilateral filter");
}

// ---------------------------------------------------------------------------
// Corner scores, shared by the constraint builder and the tracks (rcvd_builder.cuh)
// ---------------------------------------------------------------------------
// cv::cornerMinEigenVal(cv::cvtColor(BGR2GRAY), 3) of F colour frames [F][H][W][3] f32 in one batched pass into the [F][H][W] scores
// `corner`.  Nothing is launched once an allocation of the call has failed; the caller reports that through call.allocated().
static int enqueue_corner_scores(VideoCall& call, const float* color_bgr, int F, int H, int W, const float*& corner) {
  const size_t FP = (size_t)F * H * W;
  float* d_bgr = (float*)call.upload(color_bgr, FP * 12);
  float* d_gray = (float*)call.alloc(FP * 4), *d_pl = (float*)call.alloc(FP * 12), *d_corner = (float*)call.alloc(FP * 4); double* d_tmp = (double*)call.alloc(FP * 24);
  corner = d_corner;
  if (!call.allocated()) return RCVD_OK;
  if (int rc = call.launch(k_gray, (unsigned)((FP + 255) / 256), 256, 0, d_bgr, d_gray, FP)) return rc;
  if (int rc = call.launch(k_sobel_products, (unsigned)((FP + 255) / 256), 256, 0, d_gray, d_pl, F, H, W)) return rc;
  if (int rc = call.launch(k_box_h, (unsigned)((FP * 3 + 255) / 256), 256, 0, d_pl, d_tmp, (size_t)3 * F * H, W)) return rc;
  return call.launch(k_box_v_eig, (unsigned)(((size_t)F * W + 127) / 128), 128, 0, d_tmp, d_corner, F, H, W);
}

// ---------------------------------------------------------------------------
// GPU flow-constraint builder (rcvd_builder.cuh)
// ---------------------------------------------------------------------------
static int64_t g_builder_launches = 0, g_builder_rounds = 0;
RCVD_API int64_t rcvd_builder_launch_count() { return g_builder_launches; }
RCVD_API int64_t rcvd_builder_last_rounds() { return g_builder_rounds; }
RCVD_API int32_t rcvd_build_constraints(const rcvd_builder_params* prm, int32_t device, const float* color_bgr, const float* dyn_dist,
                                        const int32_t* pair_frames, const float* pair_flow, const uint8_t* pair_mask,
                                        const int32_t* trip_frames, const float* trip_flow, const uint8_t* trip_mask,
                                        int64_t* pair_offsets, float* pair_out, int64_t pair_capacity,
                                        int64_t* trip_offsets, float* trip_out, int64_t trip_capacity) {
  if (!prm || !color_bgr) return set_err(RCVD_ERR_INVALID, "null argument");
  const rcvd_builder_params& q = *prm;
  const int P = q.num_pairs, T = q.num_triplets, F = q.num_frames, I = P + T;
  if (F <= 0 || q.width <= 0 || q.height <= 0 || P < 0 || T < 0 || q.match_separation < 0 || !(q.inv_aspect > 0.f)) return set_err(RCVD_ERR_INVALID, "bad builder parameters");
  if ((P > 0 && (!pair_frames || !pair_flow || !pair_mask || !pair_offsets)) || (T > 0 && (!trip_frames || !trip_flow || !trip_mask || !trip_offsets)))
    return set_err(RCVD_ERR_INVALID, "null argument");
  if (dyn_dist && (q.dyn_width <= 0 || q.dyn_height <= 0)) return set_err(RCVD_ERR_INVALID, "bad dynamic-distance size");
  for (int i = 0; i < P; ++i) if (pair_frames[2 * i] < 0 || pair_frames[2 * i] >= F || pair_frames[2 * i + 1] < 0 || pair_frames[2 * i + 1] >= F) return set_err(RCVD_ERR_INVALID, "pair %d out of range", i);
  for (int i = 0; i < T; ++i) if (trip_frames[i] < 1 || trip_frames[i] >= F) return set_err(RCVD_ERR_INVALID, "triplet %d out of range", i);
  if (pair_offsets) pair_offsets[0] = 0;
  if (trip_offsets) trip_offsets[0] = 0;
  if (I == 0) return RCVD_OK;
  VideoCall call;
  if (int rc = call.open(device, g_builder_launches)) return rc;
  const int W = q.width, H = q.height;
  const size_t plane = (size_t)W * H;
  BuilderArgs a{};
  if (int rc = enqueue_corner_scores(call, color_bgr, F, H, W, a.corner)) return rc;
  a.dyn = dyn_dist ? (const float*)call.upload(dyn_dist, (size_t)F * q.dyn_width * q.dyn_height * 4) : nullptr;
  a.pair_frames = (const int*)call.upload(pair_frames, (size_t)P * 8); a.pair_flow = (const float*)call.upload(pair_flow, (size_t)P * plane * 8); a.pair_mask = (const uint8_t*)call.upload(pair_mask, (size_t)P * plane);
  a.trip_frames = (const int*)call.upload(trip_frames, (size_t)T * 4); a.trip_flow = (const float*)call.upload(trip_flow, (size_t)T * 2 * plane * 8); a.trip_mask = (const uint8_t*)call.upload(trip_mask, (size_t)T * 2 * plane);
  a.prio = (float*)call.alloc((size_t)I * plane * 4); a.state = (uint8_t*)call.alloc((size_t)I * plane);
  unsigned long long* d_cnt = (unsigned long long*)call.alloc((size_t)(2 * I + 2) * 8);   // [0] undecided, [1..I] counts / offsets, [I+1..2I] cursors
  if (!call.allocated()) return set_err(RCVD_ERR_CUDA, "device allocation failed in rcvd_build_constraints");
  a.P = P; a.T = T; a.h = H; a.w = W; a.dh = q.dyn_height; a.dw = q.dyn_width; a.sep = q.match_separation; a.min_dyn = q.min_dynamic_distance;
  // dynamic-mask scale (lib/FlowConstraints.cpp:415-417); without a dynamic mask the distance image has the colour size (:277-285)
  a.dsx = dyn_dist ? q.dyn_width / float(W) : 1.f; a.dsy = dyn_dist ? q.dyn_height / float(H) : 1.f;
  a.sx = 1.f / W; a.sy = q.inv_aspect / H;
  const unsigned gx = (unsigned)((plane + 255) / 256);
  if (P > 0) { if (int rc = call.launch(k_pair_candidates, dim3(gx, P), 256, 0, a)) return rc; }
  if (T > 0) { if (int rc = call.launch(k_triplet_candidates, dim3(gx, T), 256, 0, a)) return rc; }
  // ---- selection rounds until nothing is undecided ----
  int rounds = 0;
  for (;;) {
    cudaMemsetAsync(d_cnt, 0, 8, call.st);
    if (int rc = call.launch(k_select_round, dim3(gx, I), 256, 0, a, d_cnt)) return rc;
    ++rounds;
    unsigned long long und = 0;
    cudaMemcpyAsync(&und, d_cnt, 8, cudaMemcpyDeviceToHost, call.st);
    if (int rc = call.sync("constraint selection")) return rc;
    if (und == 0) break;
    if (rounds > 4 * (W + H) + 16) return set_err(RCVD_ERR_CUDA, "constraint selection did not converge");
  }
  g_builder_rounds = rounds;
  // ---- counts, offsets, emission ----
  cudaMemsetAsync(d_cnt, 0, (size_t)(2 * I + 2) * 8, call.st);
  if (int rc = call.launch(k_count_accepted, dim3(gx, I), 256, 0, a, d_cnt + 1)) return rc;
  std::vector<unsigned long long> cnt(I), off(I + 1, 0);
  cudaMemcpyAsync(cnt.data(), d_cnt + 1, (size_t)I * 8, cudaMemcpyDeviceToHost, call.st);
  if (int rc = call.sync("constraint count read-back")) return rc;
  for (int i = 0; i < I; ++i) off[i + 1] = off[i] + cnt[i];
  const unsigned long long pair_total = off[P], total = off[I];
  for (int i = 0; i < P; ++i) pair_offsets[i + 1] = (int64_t)off[i + 1];
  for (int i = 0; i < T; ++i) trip_offsets[i + 1] = (int64_t)(off[P + i + 1] - pair_total);
  if ((int64_t)pair_total > pair_capacity || (int64_t)(total - pair_total) > trip_capacity || (pair_total > 0 && !pair_out) || (total > pair_total && !trip_out))
    return set_err(RCVD_ERR_INVALID, "output capacity too small: %llu pair and %llu triplet constraints", pair_total, total - pair_total);
  if (total == 0) return RCVD_OK;
  unsigned long long* d_off = (unsigned long long*)call.upload(off.data(), (size_t)(I + 1) * 8);
  int* d_idx = (int*)call.alloc(total * 4); float* d_score = (float*)call.alloc(total * 4);
  float* d_po = (float*)call.alloc(std::max<size_t>(pair_total, 1) * 16); float* d_to = (float*)call.alloc(std::max<size_t>(total - pair_total, 1) * 24);
  if (!call.allocated()) return set_err(RCVD_ERR_CUDA, "device allocation failed in rcvd_build_constraints");
  if (int rc = call.launch(k_emit, dim3(gx, I), 256, 0, a, d_off, d_cnt + 1 + I, d_idx, d_score, d_po, d_to, pair_total)) return rc;
  std::vector<int> idx(total); std::vector<float> score(total), po(pair_total * 4), to((total - pair_total) * 6);
  cudaMemcpyAsync(idx.data(), d_idx, total * 4, cudaMemcpyDeviceToHost, call.st); cudaMemcpyAsync(score.data(), d_score, total * 4, cudaMemcpyDeviceToHost, call.st);
  if (pair_total) cudaMemcpyAsync(po.data(), d_po, pair_total * 16, cudaMemcpyDeviceToHost, call.st);
  if (total > pair_total) cudaMemcpyAsync(to.data(), d_to, (total - pair_total) * 24, cudaMemcpyDeviceToHost, call.st);
  if (int rc = call.sync("constraint emission")) return rc;
  // order each item's survivors by priority (host: a few hundred entries per item)
  std::vector<unsigned long long> perm;
  for (int i = 0; i < I; ++i) {
    const unsigned long long b = off[i], n = cnt[i];
    perm.resize(n); for (unsigned long long k = 0; k < n; ++k) perm[k] = b + k;
    std::sort(perm.begin(), perm.end(), [&](unsigned long long x, unsigned long long y) { return score[x] > score[y] || (score[x] == score[y] && idx[x] < idx[y]); });
    for (unsigned long long k = 0; k < n; ++k) {
      if (i < P) std::memcpy(pair_out + (b + k) * 4, po.data() + perm[k] * 4, 16);
      else std::memcpy(trip_out + (b - pair_total + k) * 6, to.data() + (perm[k] - pair_total) * 6, 24);
    }
  }
  return RCVD_OK;
}

// ---------------------------------------------------------------------------
// Dynamic-mask distance transform + static flags, and their pruning, on the device (rcvd_builder.cuh)
// ---------------------------------------------------------------------------
// One constraint family of rcvd_static_flags / rcvd_prune_static_flags as the caller gives it: n groups, each with its frames (a pair's
// two, or the centre t of the triplet t-1, t, t+1), offsets [n+1], then per constraint the locations of its `ends` ends and a flag.
struct FlagList {
  const char* what; int ends; int32_t n; const int32_t* frames; const int64_t* offsets; const float* locs; uint8_t* flags;
  int64_t total() const { return n > 0 ? offsets[n] : 0; }
  // The list rules of include/rcvd.h, checked on the host before the call opens its device: a refused call needs no device and leaves
  // the caller's flags as they were, and the kernels only index inside the lists.
  int check(int F) const {
    if (n < 0) return set_err(RCVD_ERR_INVALID, "negative %s count", what);
    if (n > 0 && (!frames || !offsets)) return set_err(RCVD_ERR_INVALID, "null argument");
    if (n > 0 && offsets[0] != 0) return set_err(RCVD_ERR_INVALID, "%s offsets must start at 0", what);
    for (int i = 0; i < n; ++i) {
      const bool ok = ends == 2 ? frames[2 * i] >= 0 && frames[2 * i] < F && frames[2 * i + 1] >= 0 && frames[2 * i + 1] < F : frames[i] >= 1 && frames[i] + 1 < F;
      if (!ok || offsets[i + 1] < offsets[i]) return set_err(RCVD_ERR_INVALID, "bad %s %d", what, i);
    }
    if (total() > 0 && (!locs || !flags)) return set_err(RCVD_ERR_INVALID, "null argument");
    return RCVD_OK;
  }
};
// A family on the device as k_static_flags, k_prune_stamp and k_prune_lookup read it: the frame of each end [n][3] (-1 past a pair's
// two ends), offsets, locations and flags (a copy of the caller's with `with_flags`, else unset for the kernel to write).
struct DevFlagList { int n, ends; int64_t total; const int* frames; const long long* offsets; const float* locs; uint8_t* flags; };
static DevFlagList upload_flag_list(VideoCall& call, const FlagList& l, bool with_flags) {
  std::vector<int32_t> f3((size_t)l.n * 3, -1);
  for (int i = 0; i < l.n; ++i)
    for (int e = 0; e < l.ends; ++e) f3[3 * i + e] = l.ends == 2 ? l.frames[2 * i + e] : l.frames[i] - 1 + e;
  const int64_t total = l.total();
  return {l.n, l.ends, total, (const int*)call.upload(f3.data(), f3.size() * 4),
          (const long long*)call.upload(l.offsets, l.n > 0 ? (size_t)(l.n + 1) * 8 : 0), (const float*)call.upload(l.locs, (size_t)total * 8 * l.ends),
          (uint8_t*)(with_flags ? call.upload(l.flags, (size_t)total) : call.alloc((size_t)total))};
}

static int64_t g_flag_launches = 0;
RCVD_API int64_t rcvd_static_flag_launch_count() { return g_flag_launches; }
// dist_out (optional): [F][h][w] float32 = cv::distanceTransform(mask >= 127 ? 255 : 0, DIST_L2, 5) of every frame (fixed-point chamfer).
RCVD_API int32_t rcvd_static_flags(int32_t device, const uint8_t* masks, int32_t F, int32_t h, int32_t w, float distance,
                                   int32_t num_pairs, const int32_t* pair_frames, const int64_t* pair_offsets, const float* pair_locs, uint8_t* pair_static,
                                   int32_t num_triplets, const int32_t* trip_frames, const int64_t* trip_offsets, const float* trip_locs, uint8_t* trip_static,
                                   float* dist_out) {
  if (!masks || F <= 0 || h <= 0 || w <= 0) return set_err(RCVD_ERR_INVALID, "bad static-flag arguments");
  const FlagList pairs{"pair", 2, num_pairs, pair_frames, pair_offsets, pair_locs, pair_static}, trips{"triplet", 3, num_triplets, trip_frames, trip_offsets, trip_locs, trip_static};
  if (int rc = pairs.check(F)) return rc;
  if (int rc = trips.check(F)) return rc;
  VideoCall call;
  if (int rc = call.open(device, g_flag_launches)) return rc;
  const size_t plane = (size_t)w * h;
  const uint8_t* d_masks = (const uint8_t*)call.upload(masks, (size_t)F * plane);
  unsigned* d_scratch = (unsigned*)call.alloc((size_t)F * plane * 4); float* d_dist = (float*)call.alloc((size_t)F * plane * 4);
  const DevFlagList dp = upload_flag_list(call, pairs, false), dt = upload_flag_list(call, trips, false);
  if (!call.allocated()) return set_err(RCVD_ERR_CUDA, "device allocation failed in rcvd_static_flags");
  if (int rc = call.launch(k_chamfer5, F, kChamThreads, 0, d_masks, d_scratch, d_dist, h, w)) return rc;
  for (const DevFlagList* d : {&dp, &dt})
    if (d->total > 0)
      if (int rc = call.launch(k_static_flags, dim3(8, d->n), 256, 0, d_dist, h, w, distance, d->ends, d->frames, d->offsets, d->n, d->locs, d->flags)) return rc;
  if (dp.total > 0) cudaMemcpyAsync(pair_static, dp.flags, (size_t)dp.total, cudaMemcpyDeviceToHost, call.st);
  if (dt.total > 0) cudaMemcpyAsync(trip_static, dt.flags, (size_t)dt.total, cudaMemcpyDeviceToHost, call.st);
  if (dist_out) cudaMemcpyAsync(dist_out, d_dist, (size_t)F * plane * 4, cudaMemcpyDeviceToHost, call.st);
  return call.sync("static-flag kernels");
}

// pair_static / trip_static are read and updated in place (flags only go from static to non-static).  Nothing is launched when no
// pair constraint is non-static or the distance is negative: the flags cannot change then.
RCVD_API int32_t rcvd_prune_static_flags(int32_t device, int32_t F, int32_t h, int32_t w, int32_t distance,
                                         int32_t num_pairs, const int32_t* pair_frames, const int64_t* pair_offsets, const float* pair_locs, uint8_t* pair_static,
                                         int32_t num_triplets, const int32_t* trip_centres, const int64_t* trip_offsets, const float* trip_locs, uint8_t* trip_static) {
  if (F <= 0 || h <= 0 || w <= 0) return set_err(RCVD_ERR_INVALID, "bad static-flag pruning arguments");
  const FlagList pairs{"pair", 2, num_pairs, pair_frames, pair_offsets, pair_locs, pair_static}, trips{"triplet", 3, num_triplets, trip_centres, trip_offsets, trip_locs, trip_static};
  if (int rc = pairs.check(F)) return rc;
  if (int rc = trips.check(F)) return rc;
  bool stamps = false;
  for (int64_t i = 0; i < pairs.total() && !stamps; ++i) stamps = pair_static[i] == 0;
  if (!stamps || distance < 0) return RCVD_OK;
  VideoCall call;
  if (int rc = call.open(device, g_flag_launches)) return rc;
  const int words = (w + 31) / 32;
  const size_t bits_bytes = (size_t)F * h * words * 4;
  unsigned* d_bits = (unsigned*)call.alloc(bits_bytes);
  const DevFlagList dp = upload_flag_list(call, pairs, true), dt = upload_flag_list(call, trips, true);
  if (!call.allocated()) return set_err(RCVD_ERR_CUDA, "device allocation failed in rcvd_prune_static_flags");
  cudaMemsetAsync(d_bits, 0, bits_bytes, call.st);
  if (int rc = call.launch(k_prune_stamp, dim3(8, dp.n), 256, 0, d_bits, h, w, words, distance, dp.frames, dp.offsets, dp.n, dp.locs, dp.flags)) return rc;
  for (const DevFlagList* d : {&dp, &dt})
    if (d->total > 0)
      if (int rc = call.launch(k_prune_lookup, dim3(8, d->n), 256, 0, d_bits, h, w, words, d->ends, d->frames, d->offsets, d->n, d->locs, d->flags)) return rc;
  cudaMemcpyAsync(pair_static, dp.flags, (size_t)dp.total, cudaMemcpyDeviceToHost, call.st);
  if (dt.total > 0) cudaMemcpyAsync(trip_static, dt.flags, (size_t)dt.total, cudaMemcpyDeviceToHost, call.st);
  return call.sync("static-flag pruning kernels");
}

// ---------------------------------------------------------------------------
// Long point tracks (rcvd_tracks.cuh)
// ---------------------------------------------------------------------------
static int64_t g_track_launches = 0;
RCVD_API int64_t rcvd_tracks_launch_count() { return g_track_launches; }
RCVD_API int32_t rcvd_compute_tracks(const rcvd_track_params* prm, int32_t device, const float* color_bgr, const uint8_t* dyn_masks,
                                     const float* flow, const uint8_t* flow_mask, const uint8_t* frame_flags,
                                     int64_t* frame_offsets, int32_t* obs_track, float* obs_loc, int64_t capacity, int64_t* num_tracks) {
  if (!prm || !color_bgr || !frame_flags || !frame_offsets || !num_tracks) return set_err(RCVD_ERR_INVALID, "null argument");
  const rcvd_track_params& q = *prm;
  const int F = q.num_frames, W = q.width, H = q.height;
  if (F <= 0 || W <= 0 || H <= 0 || q.spawn_distance < 0 || q.prune_distance < 0 || !(q.inv_aspect > 0.f) || (size_t)W * H >= (1u << 31))
    return set_err(RCVD_ERR_INVALID, "bad track parameters");
  if (dyn_masks && (q.dyn_width <= 0 || q.dyn_height <= 0)) return set_err(RCVD_ERR_INVALID, "bad dynamic-mask size");
  bool need_flow = false, need_mask = false;
  for (int f = 0; f < F; ++f) { need_flow |= (frame_flags[f] & RCVD_TRACK_FLOW) != 0; need_mask |= (frame_flags[f] & RCVD_TRACK_MASK) != 0; }
  if ((need_flow && !flow) || (need_mask && !flow_mask)) return set_err(RCVD_ERR_INVALID, "null argument");
  for (int f = 0; f <= F; ++f) frame_offsets[f] = 0;
  *num_tracks = 0;
  VideoCall call;
  if (int rc = call.open(device, g_track_launches)) return rc;
  const int plane = W * H;
  const size_t FP = (size_t)F * plane, dplane = dyn_masks ? (size_t)q.dyn_width * q.dyn_height : 0;
  const int max_rounds = 4 * (W + H) + 16, max_live = 2 * plane;   // at most one continued and one spawned track per pixel
  // the re-derived pixel of a spawn candidate (:844-845): x -> int(float(x / float(w)) * w), y -> int(float(float(y / float(h)) * ia) / ia * h)
  std::vector<int> mxv(W), myv(H);
  for (int x = 0; x < W; ++x) { volatile float u = x / float(W); volatile float v = u * W; mxv[x] = (int)v; }
  for (int y = 0; y < H; ++y) { volatile float u = y / float(H); volatile float v = u * q.inv_aspect; volatile float t = v / q.inv_aspect; volatile float z = t * H; myv[y] = (int)z; }
  // ---- corner scores and distance images of every frame, batched ----
  const float* d_corner = nullptr;
  if (int rc = enqueue_corner_scores(call, color_bgr, F, H, W, d_corner)) return rc;
  uint8_t* d_dmask = dyn_masks ? (uint8_t*)call.upload(dyn_masks, (size_t)F * dplane) : nullptr;
  unsigned* d_cscratch = dyn_masks ? (unsigned*)call.alloc((size_t)F * dplane * 4) : nullptr;
  float* d_dist = dyn_masks ? (float*)call.alloc((size_t)F * dplane * 4) : nullptr;
  const float* d_flow = need_flow ? (const float*)call.upload(flow, FP * 8) : nullptr;
  const uint8_t* d_fmask = need_mask ? (const uint8_t*)call.upload(flow_mask, FP) : nullptr;
  const int* d_mx = (const int*)call.upload(mxv.data(), (size_t)W * 4), *d_my = (const int*)call.upload(myv.data(), (size_t)H * 4);
  // ---- per-frame working set ----
  int* d_id[2] = {(int*)call.alloc((size_t)max_live * 4), (int*)call.alloc((size_t)max_live * 4)};
  float* d_loc[2] = {(float*)call.alloc((size_t)max_live * 8), (float*)call.alloc((size_t)max_live * 8)};
  int* d_pix = (int*)call.alloc((size_t)max_live * 4); float* d_cloc = (float*)call.alloc((size_t)max_live * 8); uint8_t* d_cstate = (uint8_t*)call.alloc(max_live);
  unsigned* d_acc = (unsigned*)call.alloc((size_t)plane * 4);
  unsigned* d_und[3] = {(unsigned*)call.alloc((size_t)plane * 4), (unsigned*)call.alloc((size_t)plane * 4), (unsigned*)call.alloc((size_t)plane * 4)};
  uint8_t* d_smask = (uint8_t*)call.alloc(plane); uint8_t* d_sstate = (uint8_t*)call.alloc(plane);
  unsigned long long* d_keys = (unsigned long long*)call.alloc((size_t)plane * 8), *d_sorted = (unsigned long long*)call.alloc((size_t)plane * 8);
  unsigned* d_cnt = (unsigned*)call.alloc((size_t)2 * max_rounds * 4);   // [0, max_rounds) prune rounds, then spawn rounds
  int* d_counts = (int*)call.alloc(8);
  size_t sort_bytes = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, sort_bytes, d_keys, d_sorted, plane, 0, 64, call.st);
  void* d_sort_tmp = call.alloc(sort_bytes);
  if (!call.allocated()) return set_err(RCVD_ERR_CUDA, "device allocation failed in rcvd_compute_tracks");
  if (dyn_masks) { if (int rc = call.launch(k_chamfer5, F, kChamThreads, 0, d_dmask, d_cscratch, d_dist, q.dyn_height, q.dyn_width)) return rc; }
  TrackArgs a{};
  a.w = W; a.h = H; a.dw = dyn_masks ? q.dyn_width : W; a.dh = dyn_masks ? q.dyn_height : H;
  a.spawn_r = q.spawn_distance; a.prune_r = q.prune_distance; a.min_dyn = q.min_dynamic_distance; a.ia = q.inv_aspect;
  // dynamic-mask scale (:657-663); without a mask the distance is FLT_MAX at colour size
  a.dsx = dyn_masks ? q.dyn_width / float(W) : 1.f; a.dsy = dyn_masks ? q.dyn_height / float(H) : 1.f;
  // ---- the frame loop: one host round trip per frame (round convergence + list sizes) ----
  std::vector<int32_t> ids; std::vector<float> locs;
  int cur = 0, n_prev = 0, next_id = 0, rp = 4, rs = 16;
  std::vector<unsigned> cnt_h((size_t)2 * max_rounds);
  int counts_h[2] = {0, 0};
  // enqueues the copy of the finished list of local frame g (n entries, buffer slot b) into the outputs
  auto flush = [&](int g, int b, int n) {
    frame_offsets[g + 1] = frame_offsets[g] + n;
    if (n == 0) return;
    ids.resize((size_t)frame_offsets[g + 1]); locs.resize((size_t)frame_offsets[g + 1] * 2);
    cudaMemcpyAsync(ids.data() + frame_offsets[g], d_id[b], (size_t)n * 4, cudaMemcpyDeviceToHost, call.st);
    cudaMemcpyAsync(locs.data() + 2 * frame_offsets[g], d_loc[b], (size_t)n * 8, cudaMemcpyDeviceToHost, call.st);
  };
  for (int f = 0; f < F; ++f) {
    const uint8_t fl = frame_flags[f];
    const int prev = cur, nxt = cur ^ 1;
    if (!(fl & RCVD_TRACK_IN_RANGE) || !(fl & RCVD_TRACK_HAS_COLOR)) {   // the frame gets no tracks (:714-727)
      if (f > 0) { flush(f - 1, prev, n_prev); if (int rc = call.sync("track read-back")) return rc; }
      n_prev = 0; cur = nxt;
      continue;
    }
    a.dist = dyn_masks ? d_dist + (size_t)f * dplane : nullptr;
    const bool cont = f > 0 && n_prev > 0 && (fl & RCVD_TRACK_FLOW) && (fl & RCVD_TRACK_MASK);
    const bool spawn = f < F - 1;
    const float* score = d_corner + (size_t)f * plane;
    if (spawn) {
      if (int rc = call.launch(k_tr_sort_keys, nblk(plane), 256, 0, score, plane, d_keys)) return rc;
      cub::DeviceRadixSort::SortKeys(d_sort_tmp, sort_bytes, d_keys, d_sorted, plane, 0, 64, call.st);
    }
    for (;;) {   // rounds enqueued blind (they stop early on the device); a frame whose rounds did not all finish is run again with more
      cudaMemsetAsync(d_cnt, 0, (size_t)2 * max_rounds * 4, call.st);
      cudaMemsetAsync(d_smask, 0, plane, call.st);
      if (cont) {
        cudaMemsetAsync(d_acc, 0xff, (size_t)plane * 4, call.st); cudaMemsetAsync(d_und[0], 0xff, (size_t)plane * 4, call.st); cudaMemsetAsync(d_und[1], 0xff, (size_t)plane * 4, call.st);
        if (int rc = call.launch(k_tr_continue, nblk(n_prev), 256, 0, a, n_prev, d_loc[prev], d_flow + (size_t)f * plane * 2, d_fmask + (size_t)f * plane, d_pix, d_cloc, d_cstate, d_und[0])) return rc;
        for (int k = 0; k < rp; ++k)
          if (int rc = call.launch(k_tr_prune_round, nblk(std::max(n_prev, plane)), 256, 0, a, n_prev, k, d_pix, d_cstate, d_acc, d_und[k % 3], d_und[(k + 1) % 3], d_und[(k + 2) % 3], d_cnt)) return rc;
        if (int rc = call.launch(k_tr_stamp, n_prev, 256, 0, a, d_pix, d_cstate, d_smask)) return rc;
      }
      if (spawn) {
        const uint8_t* sm = (fl & RCVD_TRACK_MASK) ? d_fmask + (size_t)f * plane : nullptr;
        if (int rc = call.launch(k_tr_spawn_init, nblk(plane), 256, 0, a, sm, d_smask, d_mx, d_my, d_sstate)) return rc;
        for (int k = 0; k < rs; ++k)
          if (int rc = call.launch(k_tr_spawn_round, nblk(plane), 256, 0, a, k, score, d_mx, d_my, d_sstate, d_cnt + max_rounds)) return rc;
      }
      if (int rc = call.launch(k_tr_emit, 1, kTrEmitThreads, 0, a, cont ? n_prev : 0, d_id[prev], d_cstate, d_cloc, spawn ? 1 : 0, d_sorted, d_sstate, next_id, d_id[nxt], d_loc[nxt], d_counts))
        return rc;
      if (f > 0) flush(f - 1, prev, n_prev);
      cudaMemcpyAsync(cnt_h.data(), d_cnt, (size_t)2 * max_rounds * 4, cudaMemcpyDeviceToHost, call.st);
      cudaMemcpyAsync(counts_h, d_counts, 8, cudaMemcpyDeviceToHost, call.st);
      if (int rc = call.sync("track computation")) return rc;
      const bool p_done = !cont || cnt_h[rp - 1] == 0, s_done = !spawn || cnt_h[max_rounds + rs - 1] == 0;
      if (p_done && s_done) {
        // next frame: a few rounds more than this one needed
        if (cont) { int used = 1; while (used < rp && cnt_h[used - 1] != 0) ++used; rp = std::max(2, used + 1); }
        if (spawn) { int used = 1; while (used < rs && cnt_h[max_rounds + used - 1] != 0) ++used; rs = std::max(2, used + 2); }
        break;
      }
      if ((!p_done && rp >= max_rounds) || (!s_done && rs >= max_rounds)) return set_err(RCVD_ERR_CUDA, "track selection did not converge");
      if (!p_done) rp = std::min(max_rounds, 2 * rp);
      if (!s_done) rs = std::min(max_rounds, 2 * rs);
      if (f > 0) frame_offsets[f] = frame_offsets[f - 1];   // the previous list is copied again
    }
    n_prev = counts_h[0] + counts_h[1];
    next_id += counts_h[1];
    cur = nxt;
  }
  flush(F - 1, cur, n_prev);
  if (int rc = call.sync("track read-back")) return rc;
  *num_tracks = next_id;
  const int64_t total = frame_offsets[F];
  if (total > capacity || (total > 0 && (!obs_track || !obs_loc))) return set_err(RCVD_ERR_INVALID, "output capacity too small: %lld observations", (long long)total);
  if (total > 0) { std::memcpy(obs_track, ids.data(), (size_t)total * 4); std::memcpy(obs_loc, locs.data(), (size_t)total * 8); }
  return RCVD_OK;
}

// ---------------------------------------------------------------------------
// Flow-consistency masks (rcvd_flowmask.cuh)
// ---------------------------------------------------------------------------
static int64_t g_flowmask_launches = 0;
RCVD_API int64_t rcvd_flow_mask_launch_count() { return g_flowmask_launches; }
// The argument rules of rcvd_flow_masks, checked on the host before any device is needed.
static int check_flow_mask_args(const rcvd_flow_mask_params* prm, const int32_t* pair_frames, const float* flow_ij, const float* flow_ji, const float* colors) {
  if (!prm) return set_err(RCVD_ERR_INVALID, "null argument");
  const rcvd_flow_mask_params& q = *prm;
  if (q.width <= 0 || q.height <= 0 || q.num_frames <= 0 || q.num_pairs < 0 || (int64_t)q.width * q.height >= (int64_t(1) << 31) ||
      std::isnan(q.flow_thresh_sq) || std::isnan(q.color_thresh_sq))
    return set_err(RCVD_ERR_INVALID, "bad flow-mask parameters");
  if (q.num_pairs > 0 && (!pair_frames || !flow_ij || !flow_ji || !colors)) return set_err(RCVD_ERR_INVALID, "null argument");
  for (int i = 0; i < 2 * q.num_pairs; ++i)
    if (pair_frames[i] < 0 || pair_frames[i] >= q.num_frames) return set_err(RCVD_ERR_INVALID, "pair %d out of range", i / 2);
  return RCVD_OK;
}
// Uploads the inputs of rcvd_flow_masks and allocates its outputs on the call's device; a.pair0 is left for the launches.
static FlowMaskArgs upload_flow_mask_inputs(VideoCall& call, const rcvd_flow_mask_params& q, const int32_t* pair_frames, const float* flow_ij,
                                            const float* flow_ji, const float* colors, bool counts, bool sse_flow, bool sse_color) {
  const size_t P = q.num_pairs, plane = (size_t)q.width * q.height;
  FlowMaskArgs a{};
  a.w = q.width; a.h = q.height; a.flow_thresh_sq = q.flow_thresh_sq; a.color_thresh_sq = q.color_thresh_sq;
  a.pair_frames = (const int*)call.upload(pair_frames, P * 8);
  a.flow_ij = (const float*)call.upload(flow_ij, P * plane * 8); a.flow_ji = (const float*)call.upload(flow_ji, P * plane * 8);
  a.colors = (const float*)call.upload(colors, (size_t)q.num_frames * plane * 12);
  a.mask_ij = (uint8_t*)call.alloc(P * plane); a.mask_ji = (uint8_t*)call.alloc(P * plane);
  a.counts = counts ? (unsigned long long*)call.alloc(P * 16) : nullptr;
  a.sse_flow = sse_flow ? (float*)call.alloc(P * plane * 8) : nullptr;
  a.sse_color = sse_color ? (float*)call.alloc(P * plane * 8) : nullptr;
  return a;
}
// every pair in launches of at most 65535 (grid.y) pairs
static int launch_flow_masks(VideoCall& call, FlowMaskArgs a, int P) {
  if (a.counts) cudaMemsetAsync(a.counts, 0, (size_t)P * 16, call.st);
  const unsigned gx = (unsigned)nblk((size_t)a.w * a.h, kFmThreads);
  for (int p0 = 0; p0 < P; p0 += 65535) {
    a.pair0 = p0;
    if (int rc = call.launch(k_flow_masks, dim3(gx, std::min(65535, P - p0), 2), kFmThreads, 0, a)) return rc;
  }
  return RCVD_OK;
}
RCVD_API int32_t rcvd_flow_masks(const rcvd_flow_mask_params* prm, int32_t device, const int32_t* pair_frames, const float* flow_ij, const float* flow_ji,
                                 const float* colors, uint8_t* mask_ij, uint8_t* mask_ji, int64_t* counts, float* sse_flow, float* sse_color) {
  if (int rc = check_flow_mask_args(prm, pair_frames, flow_ij, flow_ji, colors)) return rc;
  const rcvd_flow_mask_params& q = *prm;
  if (q.num_pairs > 0 && (!mask_ij || !mask_ji)) return set_err(RCVD_ERR_INVALID, "null argument");
  if (q.num_pairs == 0) return RCVD_OK;
  VideoCall call;
  if (int rc = call.open(device, g_flowmask_launches)) return rc;
  const size_t P = q.num_pairs, plane = (size_t)q.width * q.height;
  const FlowMaskArgs a = upload_flow_mask_inputs(call, q, pair_frames, flow_ij, flow_ji, colors, counts != nullptr, sse_flow != nullptr, sse_color != nullptr);
  if (!call.allocated()) return set_err(RCVD_ERR_CUDA, "device allocation failed in rcvd_flow_masks");
  if (int rc = launch_flow_masks(call, a, q.num_pairs)) return rc;
  cudaMemcpyAsync(mask_ij, a.mask_ij, P * plane, cudaMemcpyDeviceToHost, call.st);
  cudaMemcpyAsync(mask_ji, a.mask_ji, P * plane, cudaMemcpyDeviceToHost, call.st);
  if (counts) cudaMemcpyAsync(counts, a.counts, P * 16, cudaMemcpyDeviceToHost, call.st);   // unsigned long long -> int64_t: counts < 2^31
  if (sse_flow) cudaMemcpyAsync(sse_flow, a.sse_flow, P * plane * 8, cudaMemcpyDeviceToHost, call.st);
  if (sse_color) cudaMemcpyAsync(sse_color, a.sse_color, P * plane * 8, cudaMemcpyDeviceToHost, call.st);
  return call.sync("flow-mask kernel");
}
RCVD_API int32_t rcvd_debug_time_flow_masks(const rcvd_flow_mask_params* prm, int32_t device, const int32_t* pair_frames, const float* flow_ij,
                                            const float* flow_ji, const float* colors, int32_t reps, double* ms) {
  if (int rc = check_flow_mask_args(prm, pair_frames, flow_ij, flow_ji, colors)) return rc;
  if (reps < 1 || !ms || prm->num_pairs == 0) return set_err(RCVD_ERR_INVALID, "bad timing arguments");
  VideoCall call;
  if (int rc = call.open(device, g_flowmask_launches)) return rc;
  const FlowMaskArgs a = upload_flow_mask_inputs(call, *prm, pair_frames, flow_ij, flow_ji, colors, true, false, false);
  if (!call.allocated()) return set_err(RCVD_ERR_CUDA, "device allocation failed in rcvd_debug_time_flow_masks");
  if (int rc = launch_flow_masks(call, a, prm->num_pairs)) return rc;   // warm-up
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  cudaEventRecord(e0, call.st);
  int rc = RCVD_OK;
  for (int r = 0; r < reps && rc == RCVD_OK; ++r) rc = launch_flow_masks(call, a, prm->num_pairs);
  cudaEventRecord(e1, call.st);
  if (rc == RCVD_OK) rc = call.sync("flow-mask timing");
  float t = 0.f;
  if (rc == RCVD_OK) cudaEventElapsedTime(&t, e0, e1);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  *ms = (double)t / reps;
  return rc;
}

// ---------------------------------------------------------------------------
// Flow visualisations (rcvd_flowvis.cuh)
// ---------------------------------------------------------------------------
static int64_t g_flowvis_launches = 0;
RCVD_API int64_t rcvd_flow_vis_launch_count() { return g_flowvis_launches; }
RCVD_API int32_t rcvd_flow_visualize(const rcvd_flow_vis_params* prm, int32_t device, const int32_t* pair_frames, const float* flow_ij,
                                     const float* flow_ji, const uint8_t* mask_ij, const uint8_t* mask_ji, const float* colors, uint8_t* vis,
                                     uint8_t* warp_ij, uint8_t* warp_ji, float* warp_values, float* maxrad, uint8_t* has_nan) {
  if (!prm) return set_err(RCVD_ERR_INVALID, "null argument");
  const rcvd_flow_vis_params& q = *prm;
  if (q.width < 2 || q.height < 2 || q.num_frames <= 0 || q.num_pairs < 0 || 8 * (int64_t)q.width * q.height >= (int64_t(1) << 31))
    return set_err(RCVD_ERR_INVALID, "bad flow-visualisation parameters");
  if (q.num_pairs == 0) return RCVD_OK;
  if (!pair_frames || !flow_ij || !flow_ji || !mask_ij || !mask_ji || !colors || !vis || (q.warp && (!warp_ij || !warp_ji)))
    return set_err(RCVD_ERR_INVALID, "null argument");
  for (int i = 0; i < 2 * q.num_pairs; ++i)
    if (pair_frames[i] < 0 || pair_frames[i] >= q.num_frames) return set_err(RCVD_ERR_INVALID, "pair %d out of range", i / 2);
  VideoCall call;
  if (int rc = call.open(device, g_flowvis_launches)) return rc;
  const size_t P = q.num_pairs, plane = (size_t)q.width * q.height;
  FlowVisArgs a{};
  a.w = q.width; a.h = q.height;
  a.pair_frames = (const int*)call.upload(pair_frames, P * 8);
  a.flow_ij = (const float*)call.upload(flow_ij, P * plane * 8); a.flow_ji = (const float*)call.upload(flow_ji, P * plane * 8);
  a.mask_ij = (const uint8_t*)call.upload(mask_ij, P * plane); a.mask_ji = (const uint8_t*)call.upload(mask_ji, P * plane);
  a.colors = (const float*)call.upload(colors, (size_t)q.num_frames * plane * 12);
  a.stats = (unsigned*)call.alloc(P * 16);
  a.vis = (uint8_t*)call.alloc(P * plane * 24);
  if (q.warp) {
    a.warp_ij = (uint8_t*)call.alloc(P * plane * 3); a.warp_ji = (uint8_t*)call.alloc(P * plane * 3);
    if (warp_values) a.warp_values = (float*)call.alloc(P * plane * 24);
  }
  if (!call.allocated()) return set_err(RCVD_ERR_CUDA, "device allocation failed in rcvd_flow_visualize");
  cudaMemsetAsync(a.stats, 0, P * 16, call.st);
  const unsigned gx = (unsigned)nblk(plane, kFvThreads);
  for (int p0 = 0; p0 < q.num_pairs; p0 += 65535) {     // grid.y <= 65535 pairs per launch
    a.pair0 = p0;
    const unsigned np = (unsigned)std::min(65535, q.num_pairs - p0);
    if (int rc = call.launch(k_flow_vis_stats, dim3(gx, np, 2), kFvThreads, 0, a)) return rc;
    if (int rc = call.launch(k_flow_vis, dim3(gx, np), kFvThreads, 0, a)) return rc;
  }
  cudaMemcpyAsync(vis, a.vis, P * plane * 24, cudaMemcpyDeviceToHost, call.st);
  if (q.warp) {
    cudaMemcpyAsync(warp_ij, a.warp_ij, P * plane * 3, cudaMemcpyDeviceToHost, call.st);
    cudaMemcpyAsync(warp_ji, a.warp_ji, P * plane * 3, cudaMemcpyDeviceToHost, call.st);
    if (warp_values) cudaMemcpyAsync(warp_values, a.warp_values, P * plane * 24, cudaMemcpyDeviceToHost, call.st);
  }
  std::vector<unsigned> st;
  if (maxrad || has_nan) {
    st.resize(P * 4);
    cudaMemcpyAsync(st.data(), a.stats, P * 16, cudaMemcpyDeviceToHost, call.st);
  }
  if (int rc = call.sync("flow-visualisation kernels")) return rc;
  for (size_t k = 0; k < 2 * P && !st.empty(); ++k) {
    if (maxrad) std::memcpy(maxrad + k, &st[2 * k], 4);
    if (has_nan) has_nan[k] = st[2 * k + 1] ? 1 : 0;
  }
  return RCVD_OK;
}

// ---------------------------------------------------------------------------
// Downscaled colour frames (rcvd_resize.cuh)
// ---------------------------------------------------------------------------
static int64_t g_resize_launches = 0;
RCVD_API int64_t rcvd_resize_launch_count() { return g_resize_launches; }
// The argument rules of rcvd_resize_area, checked on the host before any device is needed (outputs: checked when non-null).
static int check_resize_args(const rcvd_resize_params* prm, const uint8_t* frames, void* const* outputs, bool need_outputs) {
  if (!prm) return set_err(RCVD_ERR_INVALID, "null argument");
  const rcvd_resize_params& q = *prm;
  auto bad_size = [](int w, int h) { return w <= 0 || h <= 0 || (int64_t)w * h >= (int64_t(1) << 31); };
  if (bad_size(q.width, q.height) || q.num_frames < 0) return set_err(RCVD_ERR_INVALID, "bad resize source: %d x %d, %d frames", q.width, q.height, q.num_frames);
  if (q.num_outputs < 1 || q.num_outputs > RCVD_RESIZE_MAX_OUTPUTS) return set_err(RCVD_ERR_INVALID, "%d resize outputs (1 .. %d)", q.num_outputs, RCVD_RESIZE_MAX_OUTPUTS);
  for (int k = 0; k < q.num_outputs; ++k) {
    const rcvd_resize_output& o = q.outputs[k];
    if (bad_size(o.width, o.height) || (o.kind != RCVD_RESIZE_RAW && o.kind != RCVD_RESIZE_PNG))
      return set_err(RCVD_ERR_INVALID, "bad resize output %d: %d x %d, kind %d", k, o.width, o.height, o.kind);
  }
  if (q.num_frames > 0 && !frames) return set_err(RCVD_ERR_INVALID, "null argument");
  if (need_outputs && q.num_frames > 0) {
    if (!outputs) return set_err(RCVD_ERR_INVALID, "null argument");
    for (int k = 0; k < q.num_outputs; ++k)
      if (!outputs[k]) return set_err(RCVD_ERR_INVALID, "null buffer for resize output %d", k);
  }
  return RCVD_OK;
}
// Uploads the frames once and every output's tables; allocates the outputs (a.frame0 is left for the launches).
static std::vector<ResizeArgs> upload_resize_inputs(VideoCall& call, const rcvd_resize_params& q, const uint8_t* frames) {
  const size_t F = q.num_frames;
  const uint8_t* d_src = (const uint8_t*)call.upload(frames, F * q.width * q.height * 3);
  std::vector<ResizeArgs> out;
  for (int k = 0; k < q.num_outputs; ++k) {
    const rcvd_resize_output& o = q.outputs[k];
    ResizeArgs a{};
    a.W = q.width; a.H = q.height; a.w = o.width; a.h = o.height; a.src = d_src; a.png = o.kind == RCVD_RESIZE_PNG;
    const double sx = 1.0 / ((double)o.width / q.width), sy = 1.0 / ((double)o.height / q.height);
    const int isx = (int)std::nearbyint(sx), isy = (int)std::nearbyint(sy);
    if (sx >= 1 && sy >= 1 && std::abs(sx - isx) < DBL_EPSILON && std::abs(sy - isy) < DBL_EPSILON) {
      a.ix = isx; a.iy = isy; a.inv_area = 1.f / (float)(isx * isy);
    } else {
      const bool linear = sx < 1 || sy < 1;
      // reused for the y tables: a copy from pageable memory has read its source when cudaMemcpyAsync returns
      std::vector<int> off, src; std::vector<float> wt;
      resize_axis_taps(q.width, o.width, linear, off, src, wt);
      a.x = {(const int*)call.upload(off.data(), off.size() * 4), (const int*)call.upload(src.data(), src.size() * 4), (const float*)call.upload(wt.data(), wt.size() * 4)};
      resize_axis_taps(q.height, o.height, linear, off, src, wt);
      a.y = {(const int*)call.upload(off.data(), off.size() * 4), (const int*)call.upload(src.data(), src.size() * 4), (const float*)call.upload(wt.data(), wt.size() * 4)};
    }
    a.out = call.alloc(F * o.width * o.height * 3 * (a.png ? 1 : 4));
    out.push_back(a);
  }
  return out;
}
// every output, every frame in launches of at most 65535 (grid.y) frames
static int launch_resize(VideoCall& call, std::vector<ResizeArgs> outs, int F) {
  for (ResizeArgs& a : outs)
    for (int f0 = 0; f0 < F; f0 += 65535) {
      a.frame0 = f0;
      if (int rc = call.launch(k_resize_area, dim3(nblk((size_t)a.w * a.h, kRsThreads), std::min(65535, F - f0)), kRsThreads, 0, a)) return rc;
    }
  return RCVD_OK;
}
RCVD_API int32_t rcvd_resize_area(const rcvd_resize_params* prm, int32_t device, const uint8_t* frames, void* const* outputs) {
  if (int rc = check_resize_args(prm, frames, outputs, true)) return rc;
  const rcvd_resize_params& q = *prm;
  if (q.num_frames == 0) return RCVD_OK;
  VideoCall call;
  if (int rc = call.open(device, g_resize_launches)) return rc;
  const std::vector<ResizeArgs> outs = upload_resize_inputs(call, q, frames);
  if (!call.allocated()) return set_err(RCVD_ERR_CUDA, "device allocation failed in rcvd_resize_area");
  if (int rc = launch_resize(call, outs, q.num_frames)) return rc;
  for (int k = 0; k < q.num_outputs; ++k)
    cudaMemcpyAsync(outputs[k], outs[k].out, (size_t)q.num_frames * outs[k].w * outs[k].h * 3 * (outs[k].png ? 1 : 4), cudaMemcpyDeviceToHost, call.st);
  return call.sync("resize kernel");
}
RCVD_API int32_t rcvd_debug_time_resize_area(const rcvd_resize_params* prm, int32_t device, const uint8_t* frames, int32_t reps, double* ms) {
  if (int rc = check_resize_args(prm, frames, nullptr, false)) return rc;
  if (reps < 1 || !ms || prm->num_frames == 0) return set_err(RCVD_ERR_INVALID, "bad timing arguments");
  VideoCall call;
  if (int rc = call.open(device, g_resize_launches)) return rc;
  const std::vector<ResizeArgs> outs = upload_resize_inputs(call, *prm, frames);
  if (!call.allocated()) return set_err(RCVD_ERR_CUDA, "device allocation failed in rcvd_debug_time_resize_area");
  if (int rc = launch_resize(call, outs, prm->num_frames)) return rc;   // warm-up
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  cudaEventRecord(e0, call.st);
  int rc = RCVD_OK;
  for (int r = 0; r < reps && rc == RCVD_OK; ++r) rc = launch_resize(call, outs, prm->num_frames);
  cudaEventRecord(e1, call.st);
  if (rc == RCVD_OK) rc = call.sync("resize timing");
  float t = 0.f;
  if (rc == RCVD_OK) cudaEventElapsedTime(&t, e0, e1);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  *ms = (double)t / reps;
  return rc;
}

// ---------------------------------------------------------------------------
// Depth visualisations (rcvd_depthvis.cuh)
// ---------------------------------------------------------------------------
static int64_t g_depth_vis_launches = 0;
RCVD_API int64_t rcvd_depth_vis_launch_count() { return g_depth_vis_launches; }
// The argument rules of rcvd_depth_visualize, checked on the host before any device is needed.
static int check_depth_vis_args(const rcvd_depth_vis_params* prm, const void* frames, const uint8_t* colormap, bool range, const int64_t* counts,
                                const double* stats, const uint8_t* rgb) {
  if (!prm) return set_err(RCVD_ERR_INVALID, "null argument");
  const rcvd_depth_vis_params& q = *prm;
  if (q.width <= 0 || q.height <= 0 || (int64_t)q.width * q.height * 3 >= (int64_t(1) << 31) || q.num_frames < 0)
    return set_err(RCVD_ERR_INVALID, "bad depth visualisation frames: %d x %d, %d frames", q.width, q.height, q.num_frames);
  if (q.kind != RCVD_DEPTH_VIS_F32 && q.kind != RCVD_DEPTH_VIS_U8C3) return set_err(RCVD_ERR_INVALID, "unknown depth visualisation kind %d", q.kind);
  if (!counts != !stats) return set_err(RCVD_ERR_INVALID, "the range pass needs both counts and stats");
  if (range && !(q.q[0] >= 0 && q.q[0] <= 1 && q.q[1] >= 0 && q.q[1] <= 1)) return set_err(RCVD_ERR_INVALID, "quantiles %g, %g outside [0, 1]", q.q[0], q.q[1]);
  if (q.num_frames > 0 && !frames) return set_err(RCVD_ERR_INVALID, "null argument");
  if (rgb && !colormap) return set_err(RCVD_ERR_INVALID, "rgb output without a colormap");
  return RCVD_OK;
}
static DepthVisArgs depth_vis_args(VideoCall& call, const rcvd_depth_vis_params& q, const void* frames, const uint8_t* colormap) {
  DepthVisArgs a{};
  a.w = q.width; a.h = q.height; a.u8 = q.kind == RCVD_DEPTH_VIS_U8C3;
  a.src = call.upload(frames, (size_t)q.num_frames * q.width * q.height * (a.u8 ? 3 : 4));
  a.q[0] = q.q[0]; a.q[1] = q.q[1]; a.offset = q.offset; a.scale = q.scale;
  a.lut = colormap ? (const uint8_t*)call.upload(colormap, 256 * 3) : nullptr;
  return a;
}
static int launch_depth_range(VideoCall& call, const DepthVisArgs& a, int F) {
  return call.launch(k_depth_range, dim3(F), kDvSelThreads, 0, a);
}
// every frame in launches of at most 65535 (grid.y) frames
static int launch_depth_color(VideoCall& call, DepthVisArgs a, int F) {
  for (int f0 = 0; f0 < F; f0 += 65535) {
    a.frame0 = f0;
    if (int rc = call.launch(k_depth_color, dim3(nblk((size_t)a.w * a.h, kDvThreads), std::min(65535, F - f0)), kDvThreads, 0, a)) return rc;
  }
  return RCVD_OK;
}
RCVD_API int32_t rcvd_depth_visualize(const rcvd_depth_vis_params* prm, int32_t device, const void* frames, const uint8_t* colormap,
                                      int64_t* counts, double* stats, uint8_t* index, uint8_t* rgb) {
  if (int rc = check_depth_vis_args(prm, frames, colormap, counts != nullptr, counts, stats, rgb)) return rc;
  const rcvd_depth_vis_params& q = *prm;
  const size_t F = q.num_frames, px = F * q.width * q.height;
  if (F == 0) return RCVD_OK;
  VideoCall call;
  if (int rc = call.open(device, g_depth_vis_launches)) return rc;
  DepthVisArgs a = depth_vis_args(call, q, frames, colormap);
  if (counts) { a.counts = (long long*)call.alloc(F * 8); a.stats = (double*)call.alloc(F * kDvRanks * 8); }
  if (index) a.index = (uint8_t*)call.alloc(px);
  if (rgb) a.rgb = (uint8_t*)call.alloc(px * 3);
  if (!call.allocated()) return set_err(RCVD_ERR_CUDA, "device allocation failed in rcvd_depth_visualize");
  if (counts) {
    if (int rc = launch_depth_range(call, a, q.num_frames)) return rc;
    cudaMemcpyAsync(counts, a.counts, F * 8, cudaMemcpyDeviceToHost, call.st);
    cudaMemcpyAsync(stats, a.stats, F * kDvRanks * 8, cudaMemcpyDeviceToHost, call.st);
  }
  if (index || rgb) {
    if (int rc = launch_depth_color(call, a, q.num_frames)) return rc;
    if (index) cudaMemcpyAsync(index, a.index, px, cudaMemcpyDeviceToHost, call.st);
    if (rgb) cudaMemcpyAsync(rgb, a.rgb, px * 3, cudaMemcpyDeviceToHost, call.st);
  }
  return call.sync("depth visualisation kernels");
}
RCVD_API int32_t rcvd_debug_time_depth_visualize(const rcvd_depth_vis_params* prm, int32_t device, const void* frames, const uint8_t* colormap,
                                                 int32_t reps, double* ms_range, double* ms_color) {
  if (int rc = check_depth_vis_args(prm, frames, colormap, true, nullptr, nullptr, nullptr)) return rc;
  if (reps < 1 || !ms_range || !ms_color || !colormap || prm->num_frames == 0) return set_err(RCVD_ERR_INVALID, "bad timing arguments");
  const size_t F = prm->num_frames;
  VideoCall call;
  if (int rc = call.open(device, g_depth_vis_launches)) return rc;
  DepthVisArgs a = depth_vis_args(call, *prm, frames, colormap);
  a.counts = (long long*)call.alloc(F * 8); a.stats = (double*)call.alloc(F * kDvRanks * 8);
  a.rgb = (uint8_t*)call.alloc(F * prm->width * prm->height * 3);
  if (!call.allocated()) return set_err(RCVD_ERR_CUDA, "device allocation failed in rcvd_debug_time_depth_visualize");
  cudaEvent_t e[3];
  for (cudaEvent_t& ev : e) CK(cudaEventCreate(&ev));
  int rc = launch_depth_range(call, a, prm->num_frames);   // warm-up
  if (rc == RCVD_OK) rc = launch_depth_color(call, a, prm->num_frames);
  cudaEventRecord(e[0], call.st);
  for (int r = 0; r < reps && rc == RCVD_OK; ++r) rc = launch_depth_range(call, a, prm->num_frames);
  cudaEventRecord(e[1], call.st);
  for (int r = 0; r < reps && rc == RCVD_OK; ++r) rc = launch_depth_color(call, a, prm->num_frames);
  cudaEventRecord(e[2], call.st);
  if (rc == RCVD_OK) rc = call.sync("depth visualisation timing");
  float t0 = 0.f, t1 = 0.f;
  if (rc == RCVD_OK) { cudaEventElapsedTime(&t0, e[0], e[1]); cudaEventElapsedTime(&t1, e[1], e[2]); }
  for (cudaEvent_t ev : e) cudaEventDestroy(ev);
  *ms_range = (double)t0 / reps; *ms_color = (double)t1 / reps;
  return rc;
}

// ---------------------------------------------------------------------------
// Homography-registered optical flows (rcvd_flowreg.cuh)
// ---------------------------------------------------------------------------
static int64_t g_flowreg_launches = 0;
RCVD_API int64_t rcvd_flow_register_launch_count() { return g_flowreg_launches; }
// mean device ms of one launch(call) over reps runs after a warm-up run, between two CUDA events
template <class Launch>
static int time_launches(VideoCall& call, int reps, double* ms, const char* what, Launch launch) {
  if (int rc = launch()) return rc;   // warm-up
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  cudaEventRecord(e0, call.st);
  int rc = RCVD_OK;
  for (int r = 0; r < reps && rc == RCVD_OK; ++r) rc = launch();
  cudaEventRecord(e1, call.st);
  if (rc == RCVD_OK) rc = call.sync(what);
  float t = 0.f;
  if (rc == RCVD_OK) cudaEventElapsedTime(&t, e0, e1);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  *ms = (double)t / reps;
  return rc;
}

// The argument rules of rcvd_homography_warp, checked on the host before any device is needed.
static int check_homography_warp_args(const rcvd_homography_warp_params* prm, const uint8_t* frames, const int32_t* pair_frames, const double* inverse) {
  if (!prm) return set_err(RCVD_ERR_INVALID, "null argument");
  const rcvd_homography_warp_params& q = *prm;
  if (q.width <= 0 || q.height <= 0 || 3 * (int64_t)q.width * q.height >= (int64_t(1) << 31) || q.num_pairs < 0 || q.num_frames < 0 ||
      (q.num_pairs > 0 && q.num_frames == 0))
    return set_err(RCVD_ERR_INVALID, "bad homography-warp parameters: %d x %d, %d pairs, %d frames", q.width, q.height, q.num_pairs, q.num_frames);
  if (q.num_pairs > 0 && (!frames || !pair_frames || !inverse)) return set_err(RCVD_ERR_INVALID, "null argument");
  for (int i = 0; i < q.num_pairs; ++i)
    if (pair_frames[i] < 0 || pair_frames[i] >= q.num_frames) return set_err(RCVD_ERR_INVALID, "pair %d: frame %d out of range", i, pair_frames[i]);
  return RCVD_OK;
}
static HomographyWarpArgs upload_homography_warp_inputs(VideoCall& call, const rcvd_homography_warp_params& q, const uint8_t* frames,
                                                        const int32_t* pair_frames, const double* inverse) {
  const size_t P = q.num_pairs, img = (size_t)q.width * q.height * 3;
  HomographyWarpArgs a{};
  a.W = q.width; a.H = q.height;
  a.bw = std::min(1024 / std::min(16, q.height), q.width);
  a.frames = (const uint8_t*)call.upload(frames, (size_t)q.num_frames * img);
  a.pair_frame = (const int*)call.upload(pair_frames, P * 4);
  a.minv = (const double*)call.upload(inverse, P * 72);
  const std::vector<int> tab = warp_weight_table();   // read by the copy before cudaMemcpyAsync returns (pageable source)
  a.wtab = (const int*)call.upload(tab.data(), tab.size() * 4);
  a.out = (uint8_t*)call.alloc(P * img);
  return a;
}
// every pair in launches of at most 65535 (grid.y) pairs
static int launch_homography_warp(VideoCall& call, HomographyWarpArgs a, int P) {
  const unsigned gx = (unsigned)nblk((size_t)a.W * a.H, kFrThreads);
  for (int p0 = 0; p0 < P; p0 += 65535) {
    a.pair0 = p0;
    if (int rc = call.launch(k_homography_warp, dim3(gx, std::min(65535, P - p0)), kFrThreads, 0, a)) return rc;
  }
  return RCVD_OK;
}
RCVD_API int32_t rcvd_homography_warp(const rcvd_homography_warp_params* prm, int32_t device, const uint8_t* frames, const int32_t* pair_frames,
                                      const double* inverse, uint8_t* registered) {
  if (int rc = check_homography_warp_args(prm, frames, pair_frames, inverse)) return rc;
  const rcvd_homography_warp_params& q = *prm;
  if (q.num_pairs == 0) return RCVD_OK;
  if (!registered) return set_err(RCVD_ERR_INVALID, "null argument");
  VideoCall call;
  if (int rc = call.open(device, g_flowreg_launches)) return rc;
  const HomographyWarpArgs a = upload_homography_warp_inputs(call, q, frames, pair_frames, inverse);
  if (!call.allocated()) return set_err(RCVD_ERR_CUDA, "device allocation failed in rcvd_homography_warp");
  if (int rc = launch_homography_warp(call, a, q.num_pairs)) return rc;
  cudaMemcpyAsync(registered, a.out, (size_t)q.num_pairs * q.width * q.height * 3, cudaMemcpyDeviceToHost, call.st);
  return call.sync("homography-warp kernel");
}
RCVD_API int32_t rcvd_debug_time_homography_warp(const rcvd_homography_warp_params* prm, int32_t device, const uint8_t* frames,
                                                 const int32_t* pair_frames, const double* inverse, int32_t reps, double* ms) {
  if (int rc = check_homography_warp_args(prm, frames, pair_frames, inverse)) return rc;
  if (reps < 1 || !ms || prm->num_pairs == 0) return set_err(RCVD_ERR_INVALID, "bad timing arguments");
  VideoCall call;
  if (int rc = call.open(device, g_flowreg_launches)) return rc;
  const HomographyWarpArgs a = upload_homography_warp_inputs(call, *prm, frames, pair_frames, inverse);
  if (!call.allocated()) return set_err(RCVD_ERR_CUDA, "device allocation failed in rcvd_debug_time_homography_warp");
  return time_launches(call, reps, ms, "homography-warp timing", [&] { return launch_homography_warp(call, a, prm->num_pairs); });
}

// The argument rules of rcvd_flow_unregister, checked on the host before any device is needed.
static int check_flow_unregister_args(const rcvd_flow_unregister_params* prm, const float* flow, const double* h_inv) {
  if (!prm) return set_err(RCVD_ERR_INVALID, "null argument");
  const rcvd_flow_unregister_params& q = *prm;
  auto bad_size = [](int w, int h) { return w <= 0 || h <= 0 || 2 * (int64_t)w * h >= (int64_t(1) << 31); };
  if (bad_size(q.width, q.height) || bad_size(q.out_width, q.out_height) || q.num_pairs < 0)
    return set_err(RCVD_ERR_INVALID, "bad flow-unregister parameters: %d x %d -> %d x %d, %d pairs", q.width, q.height, q.out_width, q.out_height, q.num_pairs);
  if (q.num_pairs > 0 && (!flow || !h_inv)) return set_err(RCVD_ERR_INVALID, "null argument");
  return RCVD_OK;
}
// Uploads the flows, the inverses and the cubic tables, and allocates the output (a.pair0 is left for the launches).
static FlowUnregisterArgs upload_flow_unregister_inputs(VideoCall& call, const rcvd_flow_unregister_params& q, const float* flow, const double* h_inv) {
  const size_t P = q.num_pairs;
  FlowUnregisterArgs a{};
  a.W = q.width; a.H = q.height; a.w = q.out_width; a.h = q.out_height;
  a.copy = q.out_width == q.width && q.out_height == q.height;
  a.sx = q.out_width / (double)q.width; a.sy = q.out_height / (double)q.height;
  a.flow = (const float*)call.upload(flow, P * q.width * q.height * 8);
  a.hinv = (const double*)call.upload(h_inv, P * 72);
  // reused for the y tables: a copy from pageable memory has read its source when cudaMemcpyAsync returns
  std::vector<int> first; std::vector<float> coef; std::vector<uint8_t> inside;
  resize_cubic_taps(q.width, q.out_width, first, coef, inside);
  a.xs = (const int*)call.upload(first.data(), first.size() * 4);
  a.xc = (const float*)call.upload(coef.data(), coef.size() * 4);
  a.xin = (const uint8_t*)call.upload(inside.data(), inside.size());
  resize_cubic_taps(q.height, q.out_height, first, coef, inside);
  a.ys = (const int*)call.upload(first.data(), first.size() * 4);
  a.yc = (const float*)call.upload(coef.data(), coef.size() * 4);
  a.out = (float*)call.alloc(P * q.out_width * q.out_height * 8);
  return a;
}
static int launch_flow_unregister(VideoCall& call, FlowUnregisterArgs a, int P) {
  const unsigned gx = (unsigned)nblk((size_t)a.w * a.h, kFrThreads);
  for (int p0 = 0; p0 < P; p0 += 65535) {
    a.pair0 = p0;
    if (int rc = call.launch(k_flow_unregister, dim3(gx, std::min(65535, P - p0)), kFrThreads, 0, a)) return rc;
  }
  return RCVD_OK;
}
RCVD_API int32_t rcvd_flow_unregister(const rcvd_flow_unregister_params* prm, int32_t device, const float* flow, const double* h_inv, float* out) {
  if (int rc = check_flow_unregister_args(prm, flow, h_inv)) return rc;
  const rcvd_flow_unregister_params& q = *prm;
  if (q.num_pairs == 0) return RCVD_OK;
  if (!out) return set_err(RCVD_ERR_INVALID, "null argument");
  VideoCall call;
  if (int rc = call.open(device, g_flowreg_launches)) return rc;
  const FlowUnregisterArgs a = upload_flow_unregister_inputs(call, q, flow, h_inv);
  if (!call.allocated()) return set_err(RCVD_ERR_CUDA, "device allocation failed in rcvd_flow_unregister");
  if (int rc = launch_flow_unregister(call, a, q.num_pairs)) return rc;
  cudaMemcpyAsync(out, a.out, (size_t)q.num_pairs * q.out_width * q.out_height * 8, cudaMemcpyDeviceToHost, call.st);
  return call.sync("flow-unregister kernel");
}
RCVD_API int32_t rcvd_debug_time_flow_unregister(const rcvd_flow_unregister_params* prm, int32_t device, const float* flow, const double* h_inv,
                                                 int32_t reps, double* ms) {
  if (int rc = check_flow_unregister_args(prm, flow, h_inv)) return rc;
  if (reps < 1 || !ms || prm->num_pairs == 0) return set_err(RCVD_ERR_INVALID, "bad timing arguments");
  VideoCall call;
  if (int rc = call.open(device, g_flowreg_launches)) return rc;
  const FlowUnregisterArgs a = upload_flow_unregister_inputs(call, *prm, flow, h_inv);
  if (!call.allocated()) return set_err(RCVD_ERR_CUDA, "device allocation failed in rcvd_debug_time_flow_unregister");
  return time_launches(call, reps, ms, "flow-unregister timing", [&] { return launch_flow_unregister(call, a, prm->num_pairs); });
}

// ---------------------------------------------------------------------------
// Dynamic-object masks (rcvd_dynmask.cuh)
// ---------------------------------------------------------------------------
static int64_t g_dynmask_launches = 0;
RCVD_API int64_t rcvd_dynamic_mask_launch_count() { return g_dynmask_launches; }
// The argument rules of rcvd_dynamic_masks, checked on the host before any device is needed.
static int check_dynamic_mask_args(const rcvd_dynamic_mask_params* prm, const int64_t* offsets, const uint8_t* instances, const uint8_t* frames,
                                   bool anon) {
  if (!prm) return set_err(RCVD_ERR_INVALID, "null argument");
  const rcvd_dynamic_mask_params& q = *prm;
  if (q.width <= 0 || q.height <= 0 || 3 * (int64_t)q.width * q.height >= (int64_t(1) << 31) || q.num_frames < 0 || q.dilation < 0)
    return set_err(RCVD_ERR_INVALID, "bad dynamic-mask parameters: %d x %d, %d frames, dilation %d", q.width, q.height, q.num_frames, q.dilation);
  if (anon && !frames) return set_err(RCVD_ERR_INVALID, "the anonymised frames need the frames");
  if (q.num_frames == 0) return RCVD_OK;
  if (!offsets) return set_err(RCVD_ERR_INVALID, "null argument");
  if (offsets[0] != 0) return set_err(RCVD_ERR_INVALID, "instance offsets must start at 0");
  for (int f = 0; f < q.num_frames; ++f)
    if (offsets[f + 1] < offsets[f]) return set_err(RCVD_ERR_INVALID, "instance offsets decrease at frame %d", f);
  if (offsets[q.num_frames] > 0 && !instances) return set_err(RCVD_ERR_INVALID, "null argument");
  return RCVD_OK;
}
static DynMaskArgs upload_dynamic_mask_inputs(VideoCall& call, const rcvd_dynamic_mask_params& q, const int64_t* offsets, const uint8_t* instances,
                                              const uint8_t* frames, bool anon) {
  const size_t F = q.num_frames, plane = (size_t)q.width * q.height;
  DynMaskArgs a{};
  a.w = q.width; a.h = q.height; a.F = q.num_frames;
  const int d = q.dilation == 0 ? 3 : q.dilation;   // cv::dilate replaces an empty kernel by 3 x 3
  const int reach = std::max(q.width, q.height);     // a longer reach covers the same pixels
  a.a = std::min(d / 2, reach); a.b = std::min(d - 1 - d / 2, reach);   // its default anchor (d / 2, d / 2)
  a.seg = std::max(64, (q.height + 65534) / 65535);  // at most 65535 (grid.y) segments per column
  a.offsets = (const long long*)call.upload(offsets, (F + 1) * 8);
  a.instances = (const uint8_t*)call.upload(instances, (size_t)offsets[F] * plane);
  a.frames = anon ? (const uint8_t*)call.upload(frames, F * plane * 3) : nullptr;
  a.u = (uint8_t*)call.alloc(F * plane);
  a.mask = (uint8_t*)call.alloc(F * plane);
  a.ends = (int2*)call.alloc(F * ((q.height + a.seg - 1) / a.seg) * q.width * sizeof(int2));
  a.anon = anon ? (uint8_t*)call.alloc(F * plane * 3) : nullptr;
  return a;
}
// the three kernels over every frame, in launches of at most 65535 (grid.y) frames
static int launch_dynamic_masks(VideoCall& call, DynMaskArgs a) {
  const size_t plane = (size_t)a.w * a.h;
  const bool vec = plane % 16 == 0;   // every frame's and instance's plane then starts 16-byte aligned
  for (int f0 = 0; f0 < a.F; f0 += 65535) {
    a.frame0 = f0;
    const unsigned n = (unsigned)std::min(65535, a.F - f0);
    if (int rc = vec ? call.launch(k_dm_union<16>, dim3(nblk(plane, kDmThreads * 16), n), kDmThreads, 0, a)
                     : call.launch(k_dm_union<1>, dim3(nblk(plane, kDmThreads), n), kDmThreads, 0, a)) return rc;
  }
  if (int rc = call.launch(k_dm_rows, dim3(nblk((size_t)a.F * a.h * 32, kDmThreads)), kDmThreads, 0, a)) return rc;
  const unsigned nseg = (unsigned)((a.h + a.seg - 1) / a.seg);
  for (int f0 = 0; f0 < a.F; f0 += 65535) {
    a.frame0 = f0;
    const dim3 grid(nblk(a.w, kDmThreads), nseg, std::min(65535, a.F - f0));
    if (int rc = call.launch(k_dm_col_ends, grid, kDmThreads, 0, a)) return rc;
    if (int rc = call.launch(k_dm_cols, grid, kDmThreads, 0, a)) return rc;
  }
  return RCVD_OK;
}
RCVD_API int32_t rcvd_dynamic_masks(const rcvd_dynamic_mask_params* prm, int32_t device, const int64_t* instance_offsets, const uint8_t* instances,
                                    const uint8_t* frames, uint8_t* masks, uint8_t* anon) {
  if (int rc = check_dynamic_mask_args(prm, instance_offsets, instances, frames, anon != nullptr)) return rc;
  const rcvd_dynamic_mask_params& q = *prm;
  if (q.num_frames == 0) return RCVD_OK;
  if (!masks) return set_err(RCVD_ERR_INVALID, "null argument");
  VideoCall call;
  if (int rc = call.open(device, g_dynmask_launches)) return rc;
  const DynMaskArgs a = upload_dynamic_mask_inputs(call, q, instance_offsets, instances, frames, anon != nullptr);
  if (!call.allocated()) return set_err(RCVD_ERR_CUDA, "device allocation failed in rcvd_dynamic_masks");
  if (int rc = launch_dynamic_masks(call, a)) return rc;
  const size_t px = (size_t)q.num_frames * q.width * q.height;
  cudaMemcpyAsync(masks, a.mask, px, cudaMemcpyDeviceToHost, call.st);
  if (anon) cudaMemcpyAsync(anon, a.anon, px * 3, cudaMemcpyDeviceToHost, call.st);
  return call.sync("dynamic-mask kernels");
}
RCVD_API int32_t rcvd_debug_time_dynamic_masks(const rcvd_dynamic_mask_params* prm, int32_t device, const int64_t* instance_offsets,
                                               const uint8_t* instances, const uint8_t* frames, int32_t reps, double* ms) {
  if (int rc = check_dynamic_mask_args(prm, instance_offsets, instances, frames, false)) return rc;
  if (reps < 1 || !ms || prm->num_frames == 0) return set_err(RCVD_ERR_INVALID, "bad timing arguments");
  VideoCall call;
  if (int rc = call.open(device, g_dynmask_launches)) return rc;
  const DynMaskArgs a = upload_dynamic_mask_inputs(call, *prm, instance_offsets, instances, frames, frames != nullptr);
  if (!call.allocated()) return set_err(RCVD_ERR_CUDA, "device allocation failed in rcvd_debug_time_dynamic_masks");
  return time_launches(call, reps, ms, "dynamic-mask timing", [&] { return launch_dynamic_masks(call, a); });
}
