// Library-level entry points of the C ABI: version, error string, device query.
#include "dtb_common.cuh"
#include <atomic>
#include <cstring>
#include <cstdlib>

namespace dtb {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;   // H100 SXM
    cached[dev] = n;
  }
  return cached[dev];
}

}  // namespace dtb

extern "C" {

int dtb_version(void) { return 200; }

long long dtb_launch_count(void) { return dtb::g_launches.load(); }

// a replayed CUDA graph launches the kernels that were counted once at capture time: the host adds them per replay
void dtb_launch_count_add(long long n) { dtb::g_launches.fetch_add(n, std::memory_order_relaxed); }

const char* dtb_last_error(void) { return dtb::g_err; }

// debug aid: capture status of a stream -- 0 not capturing, 1 capturing, 2 capture invalidated, negative = CUDA error
int dtb_capture_status(void* stream) {
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  const cudaError_t e = cudaStreamIsCapturing((cudaStream_t)stream, &st);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return -(int)e;
  }
  return (int)st;
}

int dtb_device_sm_count(int* out_host) {
  DTB_CHECK_ARG(out_host != nullptr, "out_host is NULL");
  int dev = 0;
  DTB_CUDA_OK(cudaGetDevice(&dev));
  DTB_CUDA_OK(cudaDeviceGetAttribute(out_host, cudaDevAttrMultiProcessorCount, dev));
  return DTB_OK;
}

}  // extern "C"
