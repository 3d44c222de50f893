// capi.cu -- ABI housekeeping for include/mrx.h: version, last-error string, device props; and
// the host helpers the other sources share (device info, shared-memory opt-in, offsets scan).
#include <stdarg.h>
#include <string.h>

#include <mutex>

#include "common.cuh"

namespace mrx {

static thread_local char g_last_error[512] = "";

void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
  va_end(ap);
}

// ---- per-device launch constants, queried once (not on every launch)
static std::mutex g_dev_mutex;
static DevInfo g_dev_info[kMaxDevices];
static bool g_dev_known[kMaxDevices];

int current_device_info(DevInfo *out) {
  int dev = 0;
  MRX_CUDA(cudaGetDevice(&dev));
  MRX_CHECK_SUPPORTED(dev >= 0 && dev < kMaxDevices, "device ordinal %d not supported", dev);
  std::lock_guard<std::mutex> lock(g_dev_mutex);
  if (!g_dev_known[dev]) {
    DevInfo d;
    d.device = dev;
    MRX_CUDA(cudaDeviceGetAttribute(&d.sms, cudaDevAttrMultiProcessorCount, dev));
    MRX_CUDA(cudaDeviceGetAttribute(&d.max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    g_dev_info[dev] = d;
    g_dev_known[dev] = true;
  }
  *out = g_dev_info[dev];
  return MRX_OK;
}

int ensure_dynamic_smem(const void *func, SmemCache *cache, int device, int bytes) {
  std::lock_guard<std::mutex> lock(g_dev_mutex);
  if (cache->set[device] >= bytes) return MRX_OK;
  const cudaError_t e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) {
    cudaFuncAttributes fa;
    memset(&fa, 0, sizeof(fa));
    cudaGetLastError();   // do not leave the error pending for the caller's next CUDA call
    cudaFuncGetAttributes(&fa, func);
    cudaGetLastError();
    set_error("cannot opt a kernel into %d B of dynamic shared memory on device %d: %s "
              "(static %zu B, current max dynamic %d B)",
              bytes, device, cudaGetErrorString(e), fa.sharedSizeBytes, fa.maxDynamicSharedSizeBytes);
    return MRX_E_CUDA;
  }
  cache->set[device] = bytes;
  return MRX_OK;
}

// ---- the second half of every count-then-write pair (RLE, contours): counts -> offsets
constexpr int kOffsetsScanThreads = 1024;

__global__ void __launch_bounds__(kOffsetsScanThreads)
offsets_scan_kernel(long long *v, int n) {
  const long long total = block_scan_range<kOffsetsScanThreads>(v, 0, n);
  if (threadIdx.x == 0) v[n] = total;
}

int launch_offsets_scan(long long *d_v, int n, cudaStream_t st) {
  offsets_scan_kernel<<<1, kOffsetsScanThreads, 0, st>>>(d_v, n);
  MRX_LAUNCH_CHECK("offsets_scan_kernel");
  return MRX_OK;
}

}  // namespace mrx

extern "C" int mrx_abi_version(void) { return MRX_ABI_VERSION; }

extern "C" const char *mrx_last_error(void) { return mrx::g_last_error; }

extern "C" int mrx_device_props(int device, int *sm_count, int *cc_major, int *cc_minor,
                                int *max_smem_optin) {
  MRX_CHECK_ARG(sm_count && cc_major && cc_minor && max_smem_optin,
                "mrx_device_props: null pointer");
  MRX_CUDA(cudaDeviceGetAttribute(sm_count, cudaDevAttrMultiProcessorCount, device));
  MRX_CUDA(cudaDeviceGetAttribute(cc_major, cudaDevAttrComputeCapabilityMajor, device));
  MRX_CUDA(cudaDeviceGetAttribute(cc_minor, cudaDevAttrComputeCapabilityMinor, device));
  MRX_CUDA(cudaDeviceGetAttribute(max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin,
                                  device));
  return MRX_OK;
}
