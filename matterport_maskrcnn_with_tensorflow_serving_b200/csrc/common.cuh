// common.cuh -- shared helpers for the sm_90a kernels behind include/mrx.h.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/mrx.h"

namespace mrx {

// ---------------------------------------------------------------- host-side errors
void set_error(const char *fmt, ...);

#define MRX_CHECK_ARG(cond, ...)                 \
  do {                                           \
    if (!(cond)) {                               \
      ::mrx::set_error(__VA_ARGS__);             \
      return MRX_E_INVALID;                      \
    }                                            \
  } while (0)

#define MRX_CHECK_SUPPORTED(cond, ...)           \
  do {                                           \
    if (!(cond)) {                               \
      ::mrx::set_error(__VA_ARGS__);             \
      return MRX_E_UNSUPPORTED;                  \
    }                                            \
  } while (0)

#define MRX_CUDA(call)                                                         \
  do {                                                                         \
    cudaError_t e_ = (call);                                                   \
    if (e_ != cudaSuccess) {                                                   \
      ::mrx::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), \
                       __FILE__, __LINE__);                                    \
      return MRX_E_CUDA;                                                       \
    }                                                                          \
  } while (0)

#define MRX_LAUNCH_CHECK(name)                                                 \
  do {                                                                         \
    cudaError_t e_ = cudaGetLastError();                                       \
    if (e_ != cudaSuccess) {                                                   \
      ::mrx::set_error("launch of %s failed: %s", name, cudaGetErrorString(e_)); \
      return MRX_E_CUDA;                                                       \
    }                                                                          \
  } while (0)

// ---------------------------------------------------------------- host-side launch constants
constexpr int kMaxDevices = 64;

struct DevInfo {
  int device, sms, max_smem_optin;
};
// SM count / opt-in shared memory of the current device, queried once per device.
int current_device_info(DevInfo *out);

// Remembers, per device, the dynamic shared-memory size a kernel has been opted into, so that
// cudaFuncSetAttribute runs when the requirement grows, not on every launch.
struct SmemCache {
  int set[kMaxDevices];
};
int ensure_dynamic_smem(const void *func, SmemCache *cache, int device, int bytes);

// Exclusive scan of d_v[0, n) in place on `st`, with their sum stored at d_v[n] (one CTA).
int launch_offsets_scan(long long *d_v, int n, cudaStream_t st);

// ---------------------------------------------------------------- output slots
// The byte canvas or the packed planes of a planned batch (mrx.h, "Output slots"): image b's
// slot starts at base + off[b].  T is const for the kernels that only read the slots.  (Pointers
// in a struct do not carry __restrict__ into a kernel: a kernel that relied on restrict-qualified
// pointer parameters reads off[] with __ldg, or keeps those parameters.)
template <typename T>
struct Slots {
  T *base;
  const long long *off;   // [B] int64 byte offsets
};

// The one host check of a batch's output slots (unmold.cu): null pointers, then B and R.
// Returns MRX_OK or MRX_E_INVALID, with mrx_last_error() naming `fn`.
int check_slots(const char *fn, const void *base, const long long *off, const int *counts,
                const int *geom, int B, int R);

// ---------------------------------------------------------------- device: PTX wrappers
#if defined(__CUDACC__)

__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)
               : "memory");
}

__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

// arrive (count 1) and add `bytes` to the transaction count the phase waits for
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}

// add `bytes` to the transaction count of the current phase without arriving
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}

// plain arrive (count 1), release semantics at CTA scope
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// named barrier among `nthreads` threads (id 1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  } while (!done);
}

// ---- variants taking 32-bit shared-window addresses (no generic->shared conversion per call)
__device__ __forceinline__ void mbar_arrive_a(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}

__device__ __forceinline__ void mbar_expect_tx_a(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}

// try_wait with a suspend-time hint: the thread sleeps in hardware until the phase
// completes (or the hint elapses) instead of spinning through the issue slots
__device__ __forceinline__ void mbar_wait_a(uint32_t bar, uint32_t parity) {
  uint32_t done;
#pragma unroll 1
  do {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}"
        : "=r"(done)
        : "r"(bar), "r"(parity), "r"(20000u)
        : "memory");
  } while (!done);
}

// one try_wait with an explicit suspend-time hint (ns); returns whether the phase completed
__device__ __forceinline__ bool mbar_try_wait_a(uint32_t bar, uint32_t parity, uint32_t hint_ns) {
  uint32_t done;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(done)
      : "r"(bar), "r"(parity), "r"(hint_ns)
      : "memory");
  return done != 0;
}

__device__ __forceinline__ void bulk_g2s_a(uint32_t smem_dst, const void *gmem_src, uint32_t bytes,
                                           uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_dst),
      "l"(gmem_src), "r"(bytes), "r"(bar)
      : "memory");
}

// 1-D TMA: global -> shared, completion reported to an mbarrier (SASS: UBLKCP).
// dst/src 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gmem_src, uint32_t bytes,
                                         uint64_t *bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_u32(smem_dst)),
      "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// 1-D TMA: shared -> global, tracked by the bulk async-group of the issuing thread.
__device__ __forceinline__ void bulk_s2g(void *gmem_dst, const void *smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst),
               "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}

__device__ __forceinline__ void bulk_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}

// wait until the sources of all but the newest N committed bulk groups have been read
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}

template <int N>
__device__ __forceinline__ void bulk_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// make generic-proxy writes to shared memory visible to the async proxy (TMA)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---------------------------------------------------------------- device: scans
// inclusive scan of v over the lanes of a full warp
template <typename T>
__device__ __forceinline__ T warp_inclusive_scan(T v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += u;
  }
  return v;
}

// sum of v over a full warp, in every lane
template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Exclusive scan of v over the CTA (every thread calls it); total = the CTA's sum.
template <typename T, int kThreads>
__device__ __forceinline__ T block_exclusive_scan(T v, T *s_warp, T &total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const T incl = warp_inclusive_scan(v, lane);
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  T before = 0, sum = 0;
#pragma unroll 4
  for (int w = 0; w < kThreads / 32; ++w) {
    const T x = s_warp[w];
    if (w < warp) before += x;
    sum += x;
  }
  __syncthreads();   // s_warp may be reused
  total = sum;
  return before + incl - v;
}

// Exclusive scan of a[lo, hi) in place by one CTA of kThreads (every thread calls it), kThreads
// elements per pass in T with a 64-bit carry between passes; returns the sum of the range.
template <int kThreads, typename T>
__device__ __forceinline__ long long block_scan_range(T *a, int lo, int hi) {
  __shared__ T s_warp[kThreads / 32];
  long long carry = 0;
  for (int base = lo; base < hi; base += kThreads) {
    const int i = base + threadIdx.x;
    const T v = i < hi ? a[i] : T(0);
    T tot;
    const T ex = block_exclusive_scan<T, kThreads>(v, s_warp, tot);
    if (i < hi) a[i] = static_cast<T>(carry + ex);
    carry += tot;
  }
  return carry;
}

#endif  // __CUDACC__

}  // namespace mrx
