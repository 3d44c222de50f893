// store_ceiling.cu -- developer microbenchmark (not part of the product): how fast can the GPU
// be WRITTEN with the store pattern of mask_expand (shared memory -> HBM bulk copies), without
// any of the kernel's box work?  Gives the practical ceiling for the kernel's roofline and
// compares job geometries (one contiguous chunk vs. k row segments of a 2-D tile).
//
//   mkdir -p build && nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o build/store_ceiling tools/store_ceiling.cu
//   build/store_ceiling        (prints one line per pattern)
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#define CK(x)                                                                      \
  do {                                                                             \
    cudaError_t e = (x);                                                           \
    if (e != cudaSuccess) {                                                        \
      printf("%s failed: %s\n", #x, cudaGetErrorString(e));                        \
      exit(1);                                                                     \
    }                                                                              \
  } while (0)

__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// rows x seg bytes per job; row r of job j goes to base + job_off(j) + r * row_stride
struct P {
  unsigned char *dst;
  long long total;      // canvas bytes
  int seg;              // bytes per row segment (multiple of 16)
  int rows;             // row segments per job
  long long row_stride; // distance between the rows of a job
  int segs_per_row;     // jobs side by side in a row band
  long long band_bytes; // rows * row_stride
  int jobs;
  int nb;               // chunk buffers per warp
  int zero;             // re-zero the buffer after each store
  int delay;            // clocks of pretend compute per job (spin) before the store
  int order;            // 0: atomic ticket, 1: static round robin (job = worker + k * workers)
  int jitter;           // delay varies per job: uniform in [delay - jitter, delay + jitter] (hash of the job)
  int victim;           // 1: the CTA's last warp stores nothing; lane 0 times a shared-memory load, a global
                        // load and a global atomic, back to back, until the other warps are done
  unsigned long long *vstats;   // [4]: sum of LDS / LDG / ATOMG cycles, samples
  unsigned int *counter;
};

template <int kWarps>
__global__ void __launch_bounds__(kWarps * 32, 1) store_kernel(const P p) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int job_bytes = p.seg * p.rows;
  unsigned char *mine = smem + static_cast<size_t>(warp) * p.nb * job_bytes;
  for (int i = lane; i < (p.nb * job_bytes) / 16; i += 32)
    reinterpret_cast<uint4 *>(mine)[i] = make_uint4(0, 0, 0, 0);
  __syncwarp();
  int k = 0;
  __shared__ int s_done;
  __shared__ int s_word[32];
  if (threadIdx.x == 0) s_done = 0;
  if (threadIdx.x < 32) s_word[threadIdx.x] = threadIdx.x;
  __syncthreads();
  const int store_warps = p.victim ? kWarps - 1 : kWarps;
  if (p.victim && warp == kWarps - 1) {
    // ---- the victim: what do ordinary memory instructions cost while the others store?
    if (lane == 0) {
      unsigned long long lds = 0, ldg = 0, atm = 0, n = 0;
      int idx = 0;
      while (*reinterpret_cast<volatile int *>(&s_done) < store_warps) {
        long long t0 = clock64();
        idx = *reinterpret_cast<volatile int *>(&s_word[idx & 31]);
        long long t1 = clock64();
        const unsigned g = *reinterpret_cast<volatile unsigned *>(p.counter + 1 + (idx & 1));
        long long t2 = clock64();
        const unsigned a = atomicAdd(p.counter + 4, g & 0u) ;
        long long t3 = clock64() + (a & 0u);
        lds += t1 - t0; ldg += t2 - t1; atm += t3 - t2; ++n;
        __nanosleep(200);
      }
      atomicAdd(p.vstats + 0, lds); atomicAdd(p.vstats + 1, ldg); atomicAdd(p.vstats + 2, atm); atomicAdd(p.vstats + 3, n);
    }
    return;
  }
  const int worker = blockIdx.x * store_warps + warp, workers = gridDim.x * store_warps;
  while (true) {
    int j = 0;
    if (p.order == 1) {
      j = worker + k * workers;
    } else {
      if (lane == 0) j = static_cast<int>(atomicAdd(p.counter, 1u));
      j = __shfl_sync(0xffffffffu, j, 0);
    }
    if (j >= p.jobs) break;
    unsigned char *buf = mine + static_cast<size_t>(k % p.nb) * job_bytes;
    // the store issued nb jobs ago from this buffer must have been read out
    if (lane == 0) {
      if (p.nb == 1) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
      else if (p.nb == 2) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
      else if (p.nb == 3) asm volatile("cp.async.bulk.wait_group.read 2;" ::: "memory");
      else asm volatile("cp.async.bulk.wait_group.read 3;" ::: "memory");
    }
    __syncwarp();
    if (p.zero) {
      for (int i = lane; i < job_bytes / 16; i += 32)
        reinterpret_cast<uint4 *>(buf)[i] = make_uint4(0, 0, 0, 0);
    }
    __syncwarp();
    if (p.delay) {
      long long d = p.delay;
      if (p.jitter) {
        unsigned h = static_cast<unsigned>(j) * 2654435761u;
        h ^= h >> 15; h *= 2246822519u; h ^= h >> 13;
        d += static_cast<long long>(h % static_cast<unsigned>(2 * p.jitter + 1)) - p.jitter;
      }
      const long long t0 = clock64();
      while (clock64() - t0 < d) {}
      __syncwarp();
    }
    if (lane == 0) {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      const int band = j / p.segs_per_row, sg = j % p.segs_per_row;
      unsigned char *d = p.dst + band * p.band_bytes + static_cast<long long>(sg) * p.seg;
      for (int r = 0; r < p.rows; ++r)
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(
                         d + r * p.row_stride),
                     "r"(smem_u32(buf + r * p.seg)), "r"(p.seg)
                     : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    ++k;
  }
  if (lane == 0) {
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    atomicAdd(&s_done, 1);
  }
}

__global__ void plain_fill(uint4 *dst, long long n16) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n16; i += stride)
    dst[i] = make_uint4(0, 0, 0, 0);
}

template <int kWarps>
static float run(P p, int sms, int iters) {
  const size_t smem = static_cast<size_t>(kWarps) * p.nb * p.seg * p.rows;
  if (smem > 227 * 1024) return -1.f;
  CK(cudaFuncSetAttribute(store_kernel<kWarps>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                          static_cast<int>(smem)));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  float best = 1e9f;
  for (int it = 0; it < iters + 2; ++it) {
    CK(cudaMemsetAsync(p.counter, 0, 4));
    CK(cudaEventRecord(e0));
    store_kernel<kWarps><<<sms, kWarps * 32, smem>>>(p);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    if (it >= 2 && ms < best) best = ms;
  }
  CK(cudaGetLastError());
  return best;
}

template <int kWarps>
static void grid_row(P p, int sms, const char *tag) {
  const float t = run<kWarps>(p, sms, 5);
  printf("  %d warps %.4f ms (%.0f GB/s)", kWarps, t, t > 0 ? p.total / t / 1e6 : 0.f);
}

// focused grid for the team kernel's pattern: 3200-byte row segments, zero-fill per job, one
// buffer per stream; streams per SM x rows per job x pretend-compute x claim order
static int team_grid(unsigned char *dst, unsigned int *counter, int sms, long long total, long long RW) {
  const int rows_list[] = {8, 10, 12, 16, 20};
  const int delays[] = {0, 3000, 8000};
  for (int order = 0; order <= 1; ++order)
    for (int delay : delays)
      for (int rows : rows_list) {
        P p;
        p.dst = dst; p.total = total; p.seg = 3200; p.rows = rows; p.row_stride = RW;
        p.segs_per_row = static_cast<int>(RW / 3200);
        p.band_bytes = rows * RW;
        p.jobs = static_cast<int>((1024 / rows) * 32 * (RW / 3200));   // whole bands only
        p.total = static_cast<long long>(p.jobs) * 3200 * rows;
        p.nb = 1; p.zero = 1; p.delay = delay; p.order = order; p.jitter = 0; p.victim = 0; p.vstats = nullptr; p.counter = counter;
        // bands of one image follow each other; images are 1024 rows apart
        printf("order %d delay %5d rows %2d :", order, delay, rows);
        grid_row<2>(p, sms, ""); grid_row<3>(p, sms, ""); grid_row<4>(p, sms, "");
        grid_row<5>(p, sms, ""); grid_row<6>(p, sms, ""); grid_row<8>(p, sms, "");
        printf("\n");
      }
  return 0;
}

static int jitter_grid(unsigned char *dst, unsigned int *counter, int sms, long long total, long long RW) {
  const int delays[] = {3000, 4000, 5000, 5800, 6500};
  const int jitters[] = {0, 1, 2};   // 0: none, 1: +-50 %, 2: +-90 %
  for (int delay : delays)
    for (int jm : jitters) {
      P p;
      p.dst = dst; p.seg = 3200; p.rows = 10; p.row_stride = RW;
      p.segs_per_row = static_cast<int>(RW / 3200);
      p.band_bytes = p.rows * RW;
      p.jobs = static_cast<int>((1024 / p.rows) * 32 * (RW / 3200));
      p.total = static_cast<long long>(p.jobs) * 3200 * p.rows;
      p.nb = 1; p.zero = 1; p.delay = delay; p.order = 0; p.victim = 0; p.vstats = nullptr; p.counter = counter;
      p.jitter = jm == 0 ? 0 : (jm == 1 ? delay / 2 : delay * 9 / 10);
      printf("delay %5d jitter %5d rows 10 :", delay, p.jitter);
      grid_row<5>(p, sms, ""); grid_row<6>(p, sms, "");
      printf("\n");
    }
  return 0;
}

// mode `v`: 6 storing warps + 1 victim warp per SM; 32000-byte jobs as 10 x 3200 B row segments (the team
// kernel's tile), as 1 x 32000 B and as 2 x 16000 B; pretend compute 0 / 4000 clocks
static int victim_grid(unsigned char *dst, unsigned int *counter, int sms, long long RW) {
  unsigned long long *vs;
  CK(cudaMalloc(&vs, 32));
  struct G { int seg, rows; long long stride; };
  const G gs[] = {{3200, 10, RW}, {32000, 1, 32000}, {16000, 2, 16000}, {6400, 5, 6400}};
  for (const G &g : gs)
    for (int delay : {0, 4000, 5800}) {
      P p;
      p.dst = dst; p.seg = g.seg; p.rows = g.rows; p.row_stride = g.stride;
      if (g.rows == 10) {
        p.segs_per_row = static_cast<int>(RW / 3200);
        p.band_bytes = 10 * RW;
        p.jobs = (1024 / 10) * 32 * p.segs_per_row;
      } else {   // contiguous jobs
        p.segs_per_row = 1;
        p.band_bytes = 32000;
        p.jobs = 104000;
      }
      p.total = static_cast<long long>(p.jobs) * 32000;
      p.nb = 1; p.zero = 1; p.delay = delay; p.order = 0; p.jitter = 0; p.victim = 1; p.vstats = vs; p.counter = counter;
      CK(cudaMemset(vs, 0, 32));
      CK(cudaMemset(counter, 0, 32));
      const float t = run<7>(p, sms, 3);
      unsigned long long h[4];
      CK(cudaMemcpy(h, vs, 32, cudaMemcpyDeviceToHost));
      const double n = h[3] ? static_cast<double>(h[3]) : 1.0;
      printf("seg %5d x %2d delay %5d : %.4f ms (%.0f GB/s)   victim LDS %.0f  LDG %.0f  ATOMG %.0f clocks (n=%llu)\n", g.seg,
             g.rows, delay, t, p.total / t / 1e6, h[0] / n, h[1] / n, h[2] / n, h[3]);
    }
  return 0;
}

int main(int argc, char **argv) {
  const long long H = 1024, W = 1024, N = 100, B = 32;
  const long long RW = W * N;
  const long long total = H * RW * B;   // 3.36 GB
  unsigned char *dst;
  unsigned int *counter;
  CK(cudaMalloc(&dst, total));
  CK(cudaMalloc(&counter, 64));
  CK(cudaMemset(counter, 0, 64));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  const int sms = prop.multiProcessorCount;
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  float ms;
  if (argc > 1 && argv[1][0] == 't') return team_grid(dst, counter, sms, total, RW);
  if (argc > 1 && argv[1][0] == 'j') return jitter_grid(dst, counter, sms, total, RW);
  if (argc > 1 && argv[1][0] == 'v') return victim_grid(dst, counter, sms, RW);
  // 1. cudaMemset
  for (int it = 0; it < 3; ++it) {
    CK(cudaEventRecord(e0));
    CK(cudaMemsetAsync(dst, 0, total));
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    CK(cudaEventElapsedTime(&ms, e0, e1));
  }
  printf("cudaMemset            : %.4f ms  %.0f GB/s\n", ms, total / ms / 1e6);
  // 2. plain st.global.v4 grid-stride
  for (int it = 0; it < 3; ++it) {
    CK(cudaEventRecord(e0));
    plain_fill<<<sms * 8, 256>>>(reinterpret_cast<uint4 *>(dst), total / 16);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    CK(cudaEventElapsedTime(&ms, e0, e1));
  }
  printf("plain st.v4 fill      : %.4f ms  %.0f GB/s\n", ms, total / ms / 1e6);

  struct Geo { int seg, rows; };
  const Geo geos[] = {{25600, 1}, {3200, 8}, {6400, 4}, {1600, 16}, {12800, 2}, {51200, 1}, {6400, 8}, {3200, 16}, {12800, 1}, {1600, 8}};
  for (const Geo &g : geos) {
    for (int zero = 0; zero <= 1; ++zero) {
      for (int nb = 1; nb <= 4; nb *= 2) {
        P p;
        p.dst = dst;
        p.total = total;
        p.seg = g.seg;
        p.rows = g.rows;
        p.row_stride = RW;
        p.segs_per_row = static_cast<int>(RW / g.seg);
        p.band_bytes = g.rows * RW;
        p.jobs = static_cast<int>(total / (static_cast<long long>(g.seg) * g.rows));
        p.nb = nb;
        p.zero = zero;
        p.delay = 0;
        p.order = 0;
        p.jitter = 0;
        p.victim = 0;
        p.vstats = nullptr;
        p.counter = counter;
        const float t2 = run<2>(p, sms, 5);
        const float t4 = run<4>(p, sms, 5);
        const float t8 = run<8>(p, sms, 5);
        printf("seg %6d x rows %2d zero %d nb %d : 2 warps %.4f ms (%.0f GB/s) | 4 warps %.4f ms (%.0f GB/s) | 8 warps %.4f ms (%.0f GB/s)\n",
               g.seg, g.rows, zero, nb, t2, t2 > 0 ? total / t2 / 1e6 : 0.f, t4,
               t4 > 0 ? total / t4 / 1e6 : 0.f, t8, t8 > 0 ? total / t8 / 1e6 : 0.f);
      }
    }
  }
  return 0;
}
