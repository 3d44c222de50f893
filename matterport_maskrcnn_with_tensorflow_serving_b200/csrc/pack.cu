// pack.cu -- bit-pack an existing [H,W,N] byte canvas (SURVEY.md 8f rank 4: compact mask transport).
// An EXTENSION, not the reference layout: unmold_detections returns bool [H,W,N] (1 byte per
// element, 105 MB per 1024x1024x100 image) and this is what mrx_mask_expand writes.  Callers
// that can take packed masks get   packed[n][y][xb] = np.packbits(masks[:, :, n], axis=1)
// (8 pixels per byte, most significant bit first, rows padded to whole bytes): 8x less
// device -> host traffic; np.unpackbits(packed, axis=-1, count=W).transpose(1, 2, 0) restores
// the reference array exactly.  (mrx_mask_expand_packed, expand_bits.cu, produces the same
// bytes without ever writing the byte canvas; this kernel serves callers that hold one.)
//
// HBM-read bound: N bytes per pixel in, N/8 out.  Two kernels, each image goes to one of them:
//
// pack_quads_kernel (N % 4 == 0, e.g. the full 100 instances).  A thread owns 32 consecutive
// pixels x 4 consecutive instances: thirty-two 4-byte loads (the 0/1 bytes of its four instances
// at each pixel), folded with
//     acc[b] |= (word & 0x01010101) << (7 - k)        pixel 8*b + k of the thread's 32
// into one output byte per (8 pixels, instance), transposed with eight byte permutes into one
// 32-bit word per instance plane and stored.  Two forms, chosen per image:
//   staged (up to ~220 instance slots): the CTA's 256 pixels arrive as eight 1-D bulk copies
//     (TMA) and the loads are conflict-free shared-memory loads (the kernel reads 8 bytes for
//     each it writes, so it can beat a copy's rate);
//   direct (more slots than that): the loads go to global memory, lanes laid out 4 pixel runs x
//     8 quads so that every load instruction reads four fully used 32-byte sectors -- slower
//     (latency of many small loads).
// (Staging with ordinary loads and stores costs 2 x 25.6 KB of shared-memory traffic per
// 25.6 KB of canvas and runs at the shared-memory bandwidth, well below the HBM roofline.)
//
// pack_bytes_kernel (any N, any alignment; ragged instance counts): 256 consecutive pixels of a
// row staged in shared memory at their global address mod 16 (one bulk copy), then one instance
// per lane slot.
#include "common.cuh"

namespace mrx {

constexpr int kPackThreads = 256;
constexpr int kPackPixels = 256;
constexpr int kPackRuns = kPackPixels / 32;   // runs of 32 pixels per CTA (staged form)

// Bytes between two staged runs of 32 pixels x N instances: 16 mod 128, so that consecutive
// runs start four banks apart, and room for the run at its offset a = address mod 16 -- N % 4
// == 0: a <= 12 and aligned words only, 32*N + 16 is enough; other N: the highest word touched
// ends at a + 32*N + 6.
__host__ __device__ inline int pack_run_pitch(int N) {
  return (N & 3) == 0 ? 32 * N + 16 : ((32 * N + 22 - 16 + 127) & ~127) + 16;
}
// ... and the largest such pitch over 1..R instances (the pitch is not monotonic in N)
inline int pack_max_run_pitch(int R) {
  int m = 0;
  for (int n = R > 3 ? R - 3 : 1; n <= R; ++n) m = pack_run_pitch(n) > m ? pack_run_pitch(n) : m;
  return m;
}


__global__ void __launch_bounds__(kPackThreads)
pack_quads_kernel(const unsigned char *__restrict__ canvas, const long long *__restrict__ canvas_off,
                  const int *__restrict__ counts, const int *__restrict__ geom,
                  unsigned char *__restrict__ packed, const long long *__restrict__ packed_off,
                  int stage_bytes) {
  extern __shared__ __align__(128) unsigned char stage[];
  const int b = blockIdx.z;
  const int H = geom[b * MRX_GEOM_INTS + 0], W = geom[b * MRX_GEOM_INTS + 1];
  const int y = blockIdx.y;
  const int N = counts[b];
  if (y >= H || N <= 0) return;
  const int nquads = (N + 3) >> 2;                   // the last quad may hold 1-3 instances
  const int wb = (W + 7) >> 3;
  const long long plane = static_cast<long long>(H) * wb;

  // acc[bq] byte j = packed byte bq of instance 4q + j  ->  word of instance j = bytes 0..3,
  // stored to the four planes
  auto emit = [&](const uint32_t (&acc)[4], int q, int x0) {
    const int nv = min(4, N - 4 * q);                // instances of this quad
    const uint32_t t0 = __byte_perm(acc[0], acc[1], 0x5140), t1 = __byte_perm(acc[2], acc[3], 0x5140);
    const uint32_t t2 = __byte_perm(acc[0], acc[1], 0x7362), t3 = __byte_perm(acc[2], acc[3], 0x7362);
    const uint32_t out[4] = {__byte_perm(t0, t1, 0x5410), __byte_perm(t0, t1, 0x7632),
                             __byte_perm(t2, t3, 0x5410), __byte_perm(t2, t3, 0x7632)};
    unsigned char *dst = packed + packed_off[b] + (static_cast<long long>(4 * q) * H + y) * wb + (x0 >> 3);
    const int nb = min(4, wb - (x0 >> 3));           // bytes of this run inside the packed row
    const bool word_ok = nb == 4 && ((reinterpret_cast<uintptr_t>(dst) | static_cast<uintptr_t>(plane)) & 3u) == 0u;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (j >= nv) break;
      unsigned char *o = dst + j * plane;
      if (word_ok) {
        *reinterpret_cast<uint32_t *>(o) = out[j];
      } else {
        for (int t = 0; t < nb; ++t) o[t] = static_cast<unsigned char>(out[j] >> (8 * t));
      }
    }
  };

  // ---- staged form (whenever eight runs of 32 pixels fit the shared memory given): the CTA's
  // 256 pixels come in as eight 1-D bulk copies (TMA), one per run, each from the run's address
  // rounded down to 16 bytes (the offset `a` is the same for all eight: 32*N is a multiple of
  // 16) and each run 32*N + 16 bytes further than the last, so that the eight runs of one
  // instance quad sit in eight different banks.  Thread u owns (run u % 8, quad u / 8):
  // conflict-free 4-byte shared loads, and the eight lanes of a quad store 32 contiguous bytes
  // of each of its four planes.
  const int run_pitch = pack_run_pitch(N);
  if (kPackRuns * run_pitch <= stage_bytes) {
    const int x_block = blockIdx.x * kPackPixels;
    if (x_block >= W) return;
    __shared__ __align__(8) uint64_t s_bar;
    const int npx_block = min(kPackPixels, W - x_block);
    const unsigned char *src = canvas + canvas_off[b] + (static_cast<long long>(y) * W + x_block) * N;
    const int a = static_cast<int>(reinterpret_cast<uintptr_t>(src) & 15u);   // multiple of 4
    if (threadIdx.x < 32) {
      if (threadIdx.x == 0) {
        mbar_init(&s_bar, 1);
        fence_mbar_init();
      }
      __syncwarp();
      const int r = threadIdx.x;
      const int npx_r = r < kPackRuns ? max(0, min(32, npx_block - 32 * r)) : 0;
      // whole 16-byte words: a run may take up to 15 bytes of its neighbours or of the slot's
      // padding (every slot starts 16-byte aligned and holds whole words, see mrx.h), never
      // unmapped memory
      const unsigned bytes = npx_r ? (static_cast<unsigned>(a + npx_r * N) + 15u) & ~15u : 0u;
      const unsigned total = warp_sum(bytes);
      if (r == 0) mbar_arrive_expect_tx(&s_bar, total);
      __syncwarp();
      if (bytes)
        bulk_g2s(stage + r * run_pitch, src + static_cast<long long>(32 * r) * N - a, bytes, &s_bar);
    }
    __syncthreads();   // the barrier is initialised
    mbar_wait(&s_bar, 0);
    for (int u = threadIdx.x; u < kPackRuns * nquads; u += kPackThreads) {
      const int r = u & (kPackRuns - 1), q = u / kPackRuns;
      const int npx = min(32, npx_block - 32 * r);
      if (npx <= 0) continue;
      const unsigned o0 = static_cast<unsigned>(r * run_pitch + a + 4 * q);
      uint32_t acc[4];
      if (((a | N) & 3) == 0) {
        // every (pixel, quad) word is 4-byte aligned
        const unsigned char *sp = stage + o0;
#pragma unroll
        for (int bq = 0; bq < 4; ++bq) {
          uint32_t v = 0u;
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const int px = 8 * bq + k;
            const uint32_t w = (npx == 32 || px < npx)
                                   ? *reinterpret_cast<const uint32_t *>(sp + px * N) : 0u;
            v |= (w & 0x01010101u) << (7 - k);
          }
          acc[bq] = v;
        }
      } else {
        // any N, any alignment: the quad's four bytes straddle two words
#pragma unroll
        for (int bq = 0; bq < 4; ++bq) {
          uint32_t v = 0u;
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const int px = 8 * bq + k;
            uint32_t w = 0u;
            if (npx == 32 || px < npx) {
              const unsigned o = o0 + static_cast<unsigned>(px * N);
              const uint32_t *wp = reinterpret_cast<const uint32_t *>(stage + (o & ~3u));
              w = __funnelshift_r(wp[0], wp[1], o << 3);   // (shift taken mod 32)
            }
            v |= (w & 0x01010101u) << (7 - k);
          }
          acc[bq] = v;
        }
      }
      emit(acc, q, x_block + 32 * r);
    }
    return;
  }

  // ---- direct form (very many instances: the runs do not fit): no shared memory, N % 4 == 0
  // only (other N: pack_bytes_kernel)
  if ((N & 3) != 0) return;
  const int lane = threadIdx.x & 31;
  const int qblocks = (nquads + 7) >> 3;             // 8 instance quads per warp
  const int pblocks = (W + 127) >> 7;                // 4 runs of 32 pixels per warp
  const int wid = blockIdx.x * (kPackThreads / 32) + (threadIdx.x >> 5);
  if (wid >= pblocks * qblocks) return;
  const int pb = wid / qblocks, qb = wid - pb * qblocks;
  const int run = pb * 4 + (lane >> 3);              // which run of 32 pixels of the row
  const int q = qb * 8 + (lane & 7);
  const int x0 = run << 5;
  if (x0 >= W || q >= nquads) return;
  const int npx = min(32, W - x0);
  // N % 4 == 0 and 16-byte aligned slots: every (pixel, quad) word is 4-byte aligned
  const uint32_t *src = reinterpret_cast<const uint32_t *>(
                            canvas + canvas_off[b] + (static_cast<long long>(y) * W + x0) * N) + q;
  uint32_t acc[4];
  const unsigned stride = static_cast<unsigned>(nquads);   // words per pixel (32-bit index math)
  const unsigned stride_bytes = static_cast<unsigned>(N);
  const unsigned char *srcb = reinterpret_cast<const unsigned char *>(src);
  if (npx == 32) {
    // whole run inside the row (always, when W % 32 == 0): 32 unpredicated loads
#pragma unroll
    for (int bq = 0; bq < 4; ++bq) {
      uint32_t w[8];
#pragma unroll
      for (int k = 0; k < 8; ++k)   // one 32x32+64 multiply-add per address
        w[k] = __ldg(reinterpret_cast<const uint32_t *>(
            srcb + static_cast<unsigned long long>(8 * bq + k) * static_cast<unsigned long long>(stride_bytes)));
      uint32_t a = 0u;
#pragma unroll
      for (int k = 0; k < 8; ++k) a |= (w[k] & 0x01010101u) << (7 - k);
      acc[bq] = a;
    }
  } else {
#pragma unroll
    for (int bq = 0; bq < 4; ++bq) {
      uint32_t a = 0u;
      for (int k = 0; k < 8; ++k) {
        const int px = 8 * bq + k;
        const uint32_t w = px < npx ? __ldg(src + static_cast<unsigned>(px) * stride) : 0u;
        a |= (w & 0x01010101u) << (7 - k);
      }
      acc[bq] = a;
    }
  }
  emit(acc, q, x0);
}

// A fixed number of CTAs walks every image: an image packed by pack_quads_kernel (N % 4 == 0)
// costs each CTA one test, not one empty CTA per 256 pixels.
__global__ void __launch_bounds__(kPackThreads)
pack_bytes_kernel(const unsigned char *__restrict__ canvas, const long long *__restrict__ canvas_off,
                  const int *__restrict__ counts, const int *__restrict__ geom,
                  unsigned char *__restrict__ packed, const long long *__restrict__ packed_off,
                  int B, int stage_bytes) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ __align__(8) uint64_t s_bar;
  const int t = threadIdx.x;
  if (t == 0) {
    mbar_init(&s_bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  unsigned phase = 0u;
  // jobs (256 pixels of one row) are numbered across all the images this kernel packs and dealt
  // round robin to the CTAs: no per-image tail
  int base = 0;
  int job = blockIdx.x;
  for (int b = 0; b < B; ++b) {
  const int N = counts[b];
  // pack_quads_kernel has taken every image whose runs fit its staging buffer or N % 4 == 0
  if (N <= 0 || (N & 3) == 0 || kPackRuns * pack_run_pitch(N) <= stage_bytes) continue;
  const int H = geom[b * MRX_GEOM_INTS + 0], W = geom[b * MRX_GEOM_INTS + 1];
  const int xblocks = (W + kPackPixels - 1) / kPackPixels;
  const int njobs = H * xblocks;
  for (; job < base + njobs; job += gridDim.x) {
  const int local = job - base;
  const int y = local / xblocks;
  const int x0 = (local - y * xblocks) * kPackPixels;
  const int npx = min(kPackPixels, W - x0);
  __syncthreads();   // the previous job's readers are done with the staging buffer

  // ---- stage the npx * N bytes of these pixels at their global address mod 16: one 1-D bulk
  // copy (TMA) of whole 16-byte words
  const unsigned char *src = canvas + canvas_off[b] + (static_cast<long long>(y) * W + x0) * N;
  const int nbytes = npx * N;
  const int a = static_cast<int>(reinterpret_cast<uintptr_t>(src) & 15u);
  if (t == 0) {
    // every canvas slot starts 16-byte aligned and holds whole 16-byte words (see mrx.h): the
    // first and last word of the run may include neighbouring pixels' bytes, never unmapped memory
    const unsigned n16 = static_cast<unsigned>(a + nbytes + 15) >> 4;
    mbar_arrive_expect_tx(&s_bar, n16 * 16u);
    bulk_g2s(smem, src - a, n16 * 16u, &s_bar);
  }
  mbar_wait(&s_bar, phase);
  phase ^= 1u;
  const unsigned char *px0 = smem + a;   // byte of (pixel x0, instance 0)

  const int wb = (W + 7) >> 3;                        // bytes per packed row
  const long long plane = static_cast<long long>(H) * wb;
  unsigned char *dst = packed + packed_off[b] + static_cast<long long>(y) * wb + (x0 >> 3);
  const int ngroups = (npx + 7) >> 3;                 // 8-pixel groups = output bytes per plane
  const int lane = t & 31, warp = t >> 5;
  const int gs = lane >> 3, qs = lane & 7;            // 4 pixel groups x 8 instances per warp step
  const int nblocks = (N + 7) >> 3;
  const int gblocks = (ngroups + 3) >> 2;
  for (int step = warp; step < gblocks * nblocks; step += kPackThreads / 32) {
    const int gb = step / nblocks, nb = step - gb * nblocks;
    const int g = gb * 4 + gs, n = nb * 8 + qs;
    if (g >= ngroups || n >= N) continue;
    const unsigned char *bp = px0 + static_cast<size_t>(8 * g) * N + n;
    const int live = min(8, npx - 8 * g);
    unsigned acc = 0u;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const unsigned v = (k < live) ? bp[k * N] : 0u;
      acc |= (v & 1u) << (7 - k);
    }
    dst[g + static_cast<long long>(n) * plane] = static_cast<unsigned char>(acc);
  }
  }   // jobs of image b
  base += njobs;
  }   // images
}

}  // namespace mrx

extern "C" int mrx_pack_masks(const unsigned char *d_canvas, const long long *d_canvas_off,
                              const int *d_counts, const int *d_geom, unsigned char *d_packed,
                              const long long *d_packed_off, int B, int R, int max_h, int max_w,
                              void *stream) {
  using namespace mrx;
  const char *fn = "mrx_pack_masks";
  if (int rc = check_slots(fn, d_canvas, d_canvas_off, d_counts, d_geom, B, R)) return rc;
  MRX_CHECK_ARG(d_packed && d_packed_off, "%s: null pointer", fn);
  MRX_CHECK_ARG(max_h >= 0 && max_w >= 0, "%s: bad max_h %d / max_w %d", fn, max_h, max_w);
  if (B == 0 || max_h == 0 || max_w == 0) return MRX_OK;
  MRX_CHECK_SUPPORTED(max_h <= 65535, "%s: image taller than 65535 rows", fn);
  DevInfo dev;
  if (int rc = current_device_info(&dev)) return rc;
  // Everything is decided before the first launch, so that a batch either kernel cannot take
  // leaves the packed output untouched.  pack_quads_kernel's staged form takes every image while
  // eight runs of R instance slots fit the shared memory of a quarter of an SM (four or more CTAs
  // resident); beyond that, its direct form packs the images with N % 4 == 0 and
  // pack_bytes_kernel the others.
  int stage_bytes = kPackRuns * pack_max_run_pitch(R);
  if (stage_bytes + 1024 > dev.max_smem_optin / 4) stage_bytes = 0;
  const size_t bytes_smem = stage_bytes ? 0 : static_cast<size_t>(kPackPixels) * R + 32;
  MRX_CHECK_SUPPORTED(bytes_smem <= static_cast<size_t>(dev.max_smem_optin),
                      "%s: R=%d needs %zu B of shared memory (limit %d)", fn, R, bytes_smem,
                      dev.max_smem_optin);
  static SmemCache quads_cache, bytes_cache;
  if (int rc = ensure_dynamic_smem(reinterpret_cast<const void *>(pack_quads_kernel), &quads_cache,
                                   dev.device, stage_bytes))
    return rc;
  int bytes_occ = 0;
  if (bytes_smem) {
    if (int rc = ensure_dynamic_smem(reinterpret_cast<const void *>(pack_bytes_kernel), &bytes_cache,
                                     dev.device, static_cast<int>(bytes_smem)))
      return rc;
    MRX_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bytes_occ, pack_bytes_kernel,
                                                           kPackThreads, bytes_smem));
  }

  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int max_quads = (R + 3) >> 2;
  const int warps_per_row = ((max_w + 127) >> 7) * ((max_quads + 7) >> 3);
  // the grid covers both forms: one CTA per 256 pixels (staged) / per eight warps' worth of
  // (pixel run, quad) blocks (direct)
  const int direct_ctas = (warps_per_row + kPackThreads / 32 - 1) / (kPackThreads / 32);
  const int staged_ctas = (max_w + kPackPixels - 1) / kPackPixels;
  dim3 grid(stage_bytes ? staged_ctas : direct_ctas, max_h, B);
  pack_quads_kernel<<<grid, kPackThreads, stage_bytes, st>>>(
      d_canvas, d_canvas_off, d_counts, d_geom, d_packed, d_packed_off, stage_bytes);
  MRX_LAUNCH_CHECK("pack_quads_kernel");
  if (bytes_smem) {
    pack_bytes_kernel<<<dev.sms * max(bytes_occ, 1), kPackThreads, bytes_smem, st>>>(
        d_canvas, d_canvas_off, d_counts, d_geom, d_packed, d_packed_off, B, stage_bytes);
    MRX_LAUNCH_CHECK("pack_bytes_kernel");
  }
  return MRX_OK;
}
