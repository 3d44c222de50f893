// alloc.cu -- device memory for the mask canvas, compressible where the GPU offers it.
//
// The canvas [H,W,N] of 0/1 bytes is mostly zeros (a kept mask covers a few percent of its
// image), and the expand kernel's time is the time HBM takes to absorb it.  Hopper's compute data
// compression shrinks such lines in L2 on their way to DRAM and expands them on the way back, so
// the same logical bytes cost fewer physical ones; no reader or writer changes.  It is a property
// of the allocation, requested through the driver's virtual-memory calls (cuMemCreate with
// CU_MEM_ALLOCATION_COMP_GENERIC), which cudaMalloc cannot ask for.
//
// The driver calls are reached through cudaGetDriverEntryPointByVersion, so the library still
// links the shared CUDA runtime only (no -lcuda).
#include <cuda.h>
#include <cudaTypedefs.h>

#include <mutex>

#include "common.cuh"

namespace mrx {
namespace {

struct Vmm {
  PFN_cuDeviceGetAttribute_v2000 device_get_attribute;
  PFN_cuMemGetAllocationGranularity_v10020 granularity;
  PFN_cuMemCreate_v10020 create;
  PFN_cuMemGetAllocationPropertiesFromHandle_v10020 properties;
  PFN_cuMemRelease_v10020 release;
  PFN_cuMemAddressReserve_v10020 reserve;
  PFN_cuMemAddressFree_v10020 address_free;
  PFN_cuMemMap_v10020 map;
  PFN_cuMemUnmap_v10020 unmap;
  PFN_cuMemSetAccess_v10020 set_access;
};

std::once_flag g_vmm_once;
Vmm g_vmm;
bool g_vmm_ok = false;

template <class F>
bool entry_point(const char *name, F *fn) {
  cudaDriverEntryPointQueryResult q;
  const cudaError_t e = cudaGetDriverEntryPointByVersion(name, reinterpret_cast<void **>(fn), 12000,
                                                         cudaEnableDefault, &q);
  return e == cudaSuccess && q == cudaDriverEntryPointSuccess && *fn != nullptr;
}

const Vmm *vmm() {
  std::call_once(g_vmm_once, [] {
    Vmm v;
    g_vmm_ok = entry_point("cuDeviceGetAttribute", &v.device_get_attribute) &&
               entry_point("cuMemGetAllocationGranularity", &v.granularity) &&
               entry_point("cuMemCreate", &v.create) &&
               entry_point("cuMemGetAllocationPropertiesFromHandle", &v.properties) &&
               entry_point("cuMemRelease", &v.release) &&
               entry_point("cuMemAddressReserve", &v.reserve) &&
               entry_point("cuMemAddressFree", &v.address_free) &&
               entry_point("cuMemMap", &v.map) && entry_point("cuMemUnmap", &v.unmap) &&
               entry_point("cuMemSetAccess", &v.set_access);
    g_vmm = v;
  });
  return g_vmm_ok ? &g_vmm : nullptr;
}

CUmemAllocationProp device_prop(int dev, bool compressed) {
  CUmemAllocationProp p = {};
  p.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  p.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  p.location.id = dev;
  p.allocFlags.compressionType = compressed ? CU_MEM_ALLOCATION_COMP_GENERIC : CU_MEM_ALLOCATION_COMP_NONE;
  return p;
}

// The size an allocation of `bytes` maps: rounded up to the larger of the compressible and the
// plain granularity, so that free computes the same size whichever of the two was granted.
CUresult mapped_size(const Vmm *v, int dev, unsigned long long bytes, size_t *size) {
  size_t g = 1;
  for (bool compressed : {false, true}) {
    const CUmemAllocationProp p = device_prop(dev, compressed);
    size_t gi = 0;
    const CUresult r = v->granularity(&gi, &p, CU_MEM_ALLOC_GRANULARITY_MINIMUM);
    if (r != CUDA_SUCCESS) {
      if (compressed) continue;   // no compressible granularity: plain memory only
      return r;
    }
    if (gi > g) g = gi;
  }
  *size = (static_cast<size_t>(bytes) + g - 1) / g * g;
  return CUDA_SUCCESS;
}

}  // namespace
}  // namespace mrx

using namespace mrx;

#define MRX_CU(call)                                                                   \
  do {                                                                                 \
    const CUresult r_ = (call);                                                        \
    if (r_ != CUDA_SUCCESS) {                                                          \
      ::mrx::set_error("%s failed: CUresult %d (%s:%d)", #call, static_cast<int>(r_), \
                       __FILE__, __LINE__);                                            \
      return MRX_E_CUDA;                                                               \
    }                                                                                  \
  } while (0)

extern "C" int mrx_device_alloc(unsigned long long bytes, void **d_ptr, int *compressed) {
  MRX_CHECK_ARG(d_ptr != nullptr && compressed != nullptr && bytes > 0,
                "mrx_device_alloc: bad arguments");
  *d_ptr = nullptr;
  *compressed = 0;
  const Vmm *v = vmm();
  MRX_CHECK_SUPPORTED(v != nullptr, "mrx_device_alloc: the driver does not provide the "
                                    "virtual-memory entry points");
  int dev = 0;
  MRX_CUDA(cudaGetDevice(&dev));
  MRX_CUDA(cudaSetDevice(dev));   // makes the primary context current on this thread
  int supported = 0;
  MRX_CU(v->device_get_attribute(&supported, CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED,
                                 static_cast<CUdevice>(dev)));
  size_t size = 0;
  MRX_CU(mapped_size(v, dev, bytes, &size));

  CUmemGenericAllocationHandle h = 0;
  CUmemAllocationProp p = device_prop(dev, supported != 0);
  if (!supported || v->create(&h, size, &p, 0) != CUDA_SUCCESS) {
    p = device_prop(dev, false);
    MRX_CU(v->create(&h, size, &p, 0));
  }
  CUmemAllocationProp granted = {};
  CUdeviceptr base = 0;
  CUresult r = v->properties(&granted, h);
  if (r == CUDA_SUCCESS) r = v->reserve(&base, size, 0, 0, 0);
  if (r == CUDA_SUCCESS) {
    r = v->map(base, size, 0, h, 0);
    if (r == CUDA_SUCCESS) {
      CUmemAccessDesc access = {};
      access.location = p.location;
      access.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
      r = v->set_access(base, size, &access, 1);
      if (r != CUDA_SUCCESS) v->unmap(base, size);
    }
    if (r != CUDA_SUCCESS) v->address_free(base, size);
  }
  // the mapping keeps the memory alive: the handle is not needed past this point
  v->release(h);
  if (r != CUDA_SUCCESS) {
    set_error("mrx_device_alloc: mapping %zu bytes failed: CUresult %d", size, static_cast<int>(r));
    return MRX_E_CUDA;
  }
  *d_ptr = reinterpret_cast<void *>(base);
  *compressed = granted.allocFlags.compressionType == CU_MEM_ALLOCATION_COMP_GENERIC;
  return MRX_OK;
}

extern "C" int mrx_device_free(void *d_ptr, unsigned long long bytes) {
  if (d_ptr == nullptr) return MRX_OK;
  const Vmm *v = vmm();
  MRX_CHECK_SUPPORTED(v != nullptr, "mrx_device_free: the driver does not provide the "
                                    "virtual-memory entry points");
  int dev = 0;
  MRX_CUDA(cudaGetDevice(&dev));
  size_t size = 0;
  MRX_CU(mapped_size(v, dev, bytes, &size));
  MRX_CUDA(cudaDeviceSynchronize());   // as cudaFree: no kernel may still be using the range
  const CUdeviceptr base = reinterpret_cast<CUdeviceptr>(d_ptr);
  MRX_CU(v->unmap(base, size));
  MRX_CU(v->address_free(base, size));
  return MRX_OK;
}
