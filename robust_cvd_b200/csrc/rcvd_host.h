// rcvd_host.h -- host helpers of the C ABI shared by the solver (rcvd_api.cu) and the video-processing entry points (rcvd_video.cu).
#pragma once
#include <cstddef>
#include <cuda_runtime.h>
#include "../../include/rcvd.h"

#define RCVD_API extern "C" __attribute__((visibility("default")))

// Sets this thread's rcvd_last_error() text (printf format) and returns `code`.  Defined in rcvd_api.cu: one error string per thread.
int set_err(int code, const char* fmt, ...);
#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return set_err(RCVD_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); } while (0)

// Every entry point works on the device it is given and puts the caller's current device back on exit (the caller may be a PyTorch
// process working on another GPU of the node).
struct DevGuard {
  int prev = -1; cudaError_t err = cudaSuccess;
  explicit DevGuard(int d) { if (cudaGetDevice(&prev) != cudaSuccess) prev = -1; err = cudaSetDevice(d); }
  ~DevGuard() { if (prev >= 0) cudaSetDevice(prev); }
};
#define SET_DEVICE(d) DevGuard dev_guard_(d); if (dev_guard_.err != cudaSuccess) return set_err(RCVD_ERR_CUDA, "cudaSetDevice(%d) failed: %s", (int)(d), cudaGetErrorString(dev_guard_.err))

static inline int nblk(size_t n, int b = 256) { return (int)((n + b - 1) / b); }

// Every kernel of the library is launched here.  A refused launch is reported at once, and its error is cleared from the runtime's
// last error, so that it is not reported a second time by a later check of the same thread.
// pdl: a programmatic dependent launch, which may start before its predecessor on the stream ends (it waits with griddepcontrol.wait).
template <class... Params, class... Args>
static int launch_kernel(void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, bool pdl, Args... args) {
  cudaLaunchAttribute attr = {};
  attr.id = cudaLaunchAttributeProgrammaticStreamSerialization; attr.val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t lc = {};
  lc.gridDim = grid; lc.blockDim = block; lc.dynamicSmemBytes = smem; lc.stream = s; lc.attrs = &attr; lc.numAttrs = pdl ? 1 : 0;
  const cudaError_t e = cudaLaunchKernelEx(&lc, kernel, args...);
  if (e != cudaSuccess) { cudaGetLastError(); return set_err(RCVD_ERR_CUDA, "launch failed: %s", cudaGetErrorString(e)); }
  return RCVD_OK;
}

// RCVD_OK when `device` is a usable CUDA device, else RCVD_ERR_NO_DEVICE: there is no CPU fallback behind any entry point.
static inline int check_device(int device) {
  int ndev = 0;
  const cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || device < 0 || device >= ndev)
    return set_err(RCVD_ERR_NO_DEVICE, "no usable CUDA device (%s); this library has no CPU fallback", e != cudaSuccess ? cudaGetErrorString(e) : "device ordinal out of range");
  return RCVD_OK;
}
