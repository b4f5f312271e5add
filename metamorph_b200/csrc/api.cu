// metamorph_b200 — C-ABI plumbing shared by all kernels: thread-local error text, device queries.
#include "common.cuh"
#include <stdlib.h>
#include <stdarg.h>
#include <map>
#include <mutex>
#include <tuple>

static thread_local char g_err[1024] = "";

void mm_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

MM_API const char* mm_last_error() { return g_err; }

int mm_pdl_enabled() {
  static const int on = [] {
    const char* e = getenv("MM_PDL");
    return (e && e[0] == '0') ? 0 : 1;
  }();
  return on;
}

int mm_pdl_mode() {
  static const int mode = [] {
    if (!mm_pdl_enabled()) return 0;
    const char* e = getenv("MM_PDL_MODE");
    return e ? atoi(e) : 3;
  }();
  return mode;
}

int mm_num_sms() {
  static int sms = 0;
  static std::once_flag once;
  std::call_once(once, [] {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0)
      sms = 132;  // H100 SXM
  });
  return sms;
}

void* mm_stream_scratch(int tag, size_t bytes, cudaStream_t stream) {
  static std::mutex mu;
  static std::map<std::tuple<int, uintptr_t, int>, std::pair<void*, size_t>> bufs;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    mm_set_error("mm_stream_scratch: no current device");
    return nullptr;
  }
  std::lock_guard<std::mutex> lock(mu);
  auto& b = bufs[std::make_tuple(dev, (uintptr_t)stream, tag)];
  if (b.second < bytes) {
    if (b.first != nullptr) {
      cudaStreamSynchronize(stream);   // earlier work on this stream may still use the old buffer
      cudaFree(b.first);
    }
    b = {nullptr, 0};
    void* p = nullptr;
    if (cudaMalloc(&p, bytes) != cudaSuccess || cudaMemsetAsync(p, 0, bytes, stream) != cudaSuccess) {
      if (p != nullptr) cudaFree(p);
      mm_set_error("mm_stream_scratch: could not allocate %zu bytes", bytes);
      return nullptr;
    }
    b = {p, bytes};
  }
  return b.first;
}

MM_API int mm_abi_version() { return 1; }

// Returns 0 when the current device is sm_90 (H100); a negative code (+ message) otherwise: the library holds sm_90a
// code only, which no other architecture can load.
MM_API int mm_check_device() {
  int dev = 0, major = 0, minor = 0;
  MM_CHECK_CUDA(cudaGetDevice(&dev));
  MM_CHECK_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  MM_CHECK_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  if (major != 9 || minor != 0) {
    mm_set_error("metamorph_b200 kernels are built for sm_90a only; device is sm_%d%d", major, minor);
    return MM_ERR_ARCH;
  }
  return MM_OK;
}
