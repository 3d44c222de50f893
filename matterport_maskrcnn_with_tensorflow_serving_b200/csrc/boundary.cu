// boundary.cu -- the boundary of every packed plane, as boundary_iou_api's mask_to_boundary
// computes it: mask AND NOT the mask eroded by a (2d+1) x (2d+1) square, where everything outside
// the plane's region counts as 0 (cv2.erode of the mask padded with one pixel of zeros, d
// iterations of a 3 x 3 kernel: a pixel stays iff the whole square around it lies inside the
// image and is set).  A prediction is zero outside its box, so its region is the box; ground
// truth takes the whole image.  One rule serves both.
//
//   mask_boundary_kernel  CTA per plane, both steps of the separable erosion:
//     vertical    a thread per byte column walks down the region's rows: van Herk / Gil-Werman
//                 suffix ANDs over blocks of 2d+1 rows (stored d rows down, in the output plane),
//                 then prefix ANDs, so each row costs three ANDs for any d;
//     horizontal  a warp per row: the vertically eroded row in shared memory as 32-pixel words,
//                 ANDed with itself shifted by 1, 2, 4, ... pixels (funnel shifts across words)
//                 up to the largest power of two p <= 2d+1, then two shifted reads of that cover
//                 the window; the row's bytes are rewritten as mask AND NOT eroded.
#include "planes.cuh"

namespace mrx {

namespace boundary {

using overlaps::plane_of;

constexpr int kWarps = 8;

// bits [lo, hi) of a 32-pixel word (bit 31 = pixel 0), 0 <= lo, hi <= 32
__device__ __forceinline__ uint32_t span_mask(int lo, int hi) {
  if (hi <= lo) return 0u;
  const uint32_t m = hi - lo == 32 ? 0xFFFFFFFFu : ((1u << (hi - lo)) - 1u);
  return m << (32 - hi);
}

// bytes 4k .. 4k + 3 (those below nb) of p as a word, byte 4k in bits 31-24: pixel order
__device__ __forceinline__ uint32_t load_word(const unsigned char *p, int k, int nb) {
  uint32_t v = 0u;
#pragma unroll
  for (int t = 0; t < 4; ++t) v = (v << 8) | (4 * k + t < nb ? p[4 * k + t] : 0u);
  return v;
}

__device__ __forceinline__ void store_word(unsigned char *p, int k, int nb, uint32_t v) {
#pragma unroll
  for (int t = 0; t < 4; ++t)
    if (4 * k + t < nb) p[4 * k + t] = static_cast<unsigned char>(v >> (24 - 8 * t));
}

// the 32 pixels of row[] from position P on (bit 31 = pixel P), 0 outside [0, 32 * nw)
__device__ __forceinline__ uint32_t bits_at(const uint32_t *row, int nw, int P) {
  const int q = P >> 5;
  const uint32_t hi = q >= 0 && q < nw ? row[q] : 0u;
  const uint32_t lo = q + 1 >= 0 && q + 1 < nw ? row[q + 1] : 0u;
  return __funnelshift_l(lo, hi, P & 31);
}

// s_rows: kWarps x 2 x nw_max words of dynamic shared memory
__global__ void __launch_bounds__(kWarps * 32)
mask_boundary_kernel(Slots<const unsigned char> in, Slots<unsigned char> out,
                     const int *__restrict__ counts, const int *__restrict__ geom,
                     const int4 *__restrict__ regions, const int *__restrict__ dilation, int R,
                     int nw_max) {
  extern __shared__ uint32_t s_rows[];
  const int k = blockIdx.x, b = blockIdx.y;
  if (k >= counts[b]) return;
  const int H = geom[b * MRX_GEOM_INTS + 0], W = geom[b * MRX_GEOM_INTS + 1];
  const int wb = (W + 7) >> 3;
  const int4 r4 = regions[static_cast<size_t>(b) * R + k];
  const int y1 = max(r4.x, 0), x1 = max(r4.y, 0), y2 = min(r4.z, H), x2 = min(r4.w, W);
  if (y2 <= y1 || x2 <= x1) return;
  const int h = y2 - y1, cb0 = x1 >> 3, nb = ((x2 - 1) >> 3) - cb0 + 1, nw = (nb + 3) >> 2;
  // the region's first row and byte column in both planes
  const unsigned char *src = plane_of(in, b, k, H, wb) + static_cast<long long>(y1) * wb + cb0;
  unsigned char *dst = out.base + out.off[b] + static_cast<long long>(k) * H * wb +
                       static_cast<long long>(y1) * wb + cb0;
  const int d = max(dilation[b], 1);
  // the square fits the region at all (d < 2^30 then, so L and every position below fit int)
  const bool erode = 2LL * d + 1 <= h && 2LL * d + 1 <= x2 - x1;
  const int L = erode ? 2 * d + 1 : 0;

  if (erode) {
    // vertical: V(r) = AND of rows r - d .. r + d = s(r - d) & g(r + d) for d <= r < h - d, with
    // s the suffix and g the prefix ANDs within blocks of L rows.  s(a) for a <= h - L goes to
    // dst row a + d, where the forward walk reads it back just before it writes V(a + d) there.
    for (int c = threadIdx.x; c < nb; c += blockDim.x) {
      for (int k0 = 0; k0 <= h - L; k0 += L) {
        unsigned s = 0xFFu;
        for (int r = k0 + L - 1; r >= k0; --r) {
          s &= src[static_cast<long long>(r) * wb + c];
          if (r <= h - L) dst[static_cast<long long>(r + d) * wb + c] = static_cast<unsigned char>(s);
        }
      }
      unsigned g = 0u;
      for (int q = 0, in_block = 0; q < h; ++q) {
        const unsigned m = src[static_cast<long long>(q) * wb + c];
        g = in_block ? g & m : m;
        in_block = in_block + 1 == L ? 0 : in_block + 1;
        if (q >= 2 * d) {
          unsigned char *v = dst + static_cast<long long>(q - d) * wb + c;
          *v = static_cast<unsigned char>(*v & g);
        }
      }
    }
    __syncthreads();   // the vertically eroded rows, written by other threads, are read below
  }

  // horizontal, a warp per row; pixel P of the row's words is x = 8 * cb0 + P
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int P0 = x1 - 8 * cb0, P1 = x2 - 8 * cb0;
  uint32_t *A = s_rows + warp * 2 * nw_max, *T = A + nw_max;
  for (int r = warp; r < h; r += kWarps) {
    const long long ro = static_cast<long long>(r) * wb;
    const bool row_eroded = erode && r >= d && r < h - d;
    int p = 0;
    __syncwarp();      // the previous row's reads of A are done
    if (row_eroded) {
      for (int w = lane; w < nw; w += 32)
        A[w] = load_word(dst + ro, w, nb) & span_mask(max(P0 - 32 * w, 0), min(P1 - 32 * w, 32));
      __syncwarp();
      // A_2s(P) = A_s(P) & A_s(P + s): the AND of pixels P .. P + 2s - 1
      for (p = 1; 2 * p <= L; p <<= 1) {
        for (int w = lane; w < nw; w += 32) T[w] = A[w] & bits_at(A, nw, 32 * w + p);
        __syncwarp();
        uint32_t *t = A;
        A = T;
        T = t;
      }
    }
    for (int w = lane; w < nw; w += 32) {
      // eroded(P) = A_p(P - d) & A_p(P - d + L - p): the two cover P - d .. P + d (2p > L)
      const uint32_t e =
          row_eroded ? bits_at(A, nw, 32 * w - d) & bits_at(A, nw, 32 * w - d + L - p) : 0u;
      const uint32_t m = load_word(src + ro, w, nb) &
                         span_mask(max(P0 - 32 * w, 0), min(P1 - 32 * w, 32));
      store_word(dst + ro, w, nb, m & ~e);
    }
  }
}

}  // namespace boundary

}  // namespace mrx

using namespace mrx;

extern "C" int mrx_mask_boundary(const unsigned char *d_packed, const long long *d_packed_off,
                                 const int *d_counts, const int *d_geom, const int *d_regions,
                                 const int *d_dilation, unsigned char *d_boundary, int B, int R,
                                 int max_w, void *stream) {
  const char *fn = "mrx_mask_boundary";
  if (int rc = check_slots(fn, d_packed, d_packed_off, d_counts, d_geom, B, R)) return rc;
  MRX_CHECK_ARG(d_regions, "%s: the region argument d_regions is required", fn);
  MRX_CHECK_ARG(d_dilation && d_boundary, "%s: null pointer", fn);
  MRX_CHECK_ARG(max_w >= 1, "%s: bad max_w %d (need max_w>=1)", fn, max_w);
  if (B == 0) return MRX_OK;
  const int nw_max = ((max_w + 7) / 8 + 3) / 4;
  const long long smem = 4LL * boundary::kWarps * 2 * nw_max;
  DevInfo dev;
  if (int rc = current_device_info(&dev)) return rc;
  MRX_CHECK_SUPPORTED(smem <= dev.max_smem_optin,
                      "%s: max_w %d needs %lld bytes of shared memory (the device has %d)", fn,
                      max_w, smem, dev.max_smem_optin);
  static SmemCache cache;
  if (int rc = ensure_dynamic_smem(reinterpret_cast<const void *>(boundary::mask_boundary_kernel),
                                   &cache, dev.device, static_cast<int>(smem)))
    return rc;
  boundary::mask_boundary_kernel<<<dim3(R, B), boundary::kWarps * 32, static_cast<size_t>(smem),
                                   static_cast<cudaStream_t>(stream)>>>(
      {d_packed, d_packed_off}, {d_boundary, d_packed_off}, d_counts, d_geom,
      reinterpret_cast<const int4 *>(d_regions), d_dilation, R, nw_max);
  MRX_LAUNCH_CHECK("mask_boundary_kernel");
  return MRX_OK;
}
