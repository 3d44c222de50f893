// planes.cuh -- reading two bit-packed plane sets of one batch together, shared by the mask scorers
// mask_overlaps_kernel (overlaps.cu), coco_iou_kernel and coco_boundary_iou_kernel (cocoeval.cu):
// the side description (Planes) and its argument check, the culled walk over the pairs of one
// prediction with the AND-popcount of their intersection rectangle (and its variant that counts
// the boundary planes of the pair too), and the scores of the rank kernels.
//
// Planes are uint8 [N, H, ceil(W/8)], most significant bit first, as mrx_pack_masks /
// mrx_mask_expand_packed write them.  Pixel x of a row is bit 7 - (x & 7) of byte x >> 3 in every
// plane of an image, so the bytes of two planes line up column for column; only their addresses
// differ in alignment (a plane is H * ceil(W/8) bytes).
#pragma once

#include "common.cuh"

namespace mrx {

// The store of a CTA of kWarps warps that writes one band of 32 rows x 32 * kWarps columns of a
// packed plane (rle_planes_kernel, poly_planes_kernel): lane l of warp w holds in `word` the
// column word of column x0 + 32w + (l ^ 7), bit r for row y0 + r.  A 5-step __shfl_xor_sync
// transpose turns the 32 column words into 32 row words (assigning the columns as lane ^ 7 puts
// every row word in np.packbits byte order); the band goes through shared memory and leaves as
// rows of 32 contiguous bytes, byte columns cb0 .. cb0 + 31.  Every byte of the band inside the
// plane (rows < H, byte columns < wb) is written.  Called by every thread of the CTA.
template <int kWarps>
__device__ __forceinline__ void store_band(uint32_t word, uint32_t (&s_band)[32][kWarps],
                                           unsigned char *plane, int y0, int cb0, int H, int wb) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // 32 x 32 bit transpose: lane l's bit r is (row r, column l ^ 7); afterwards lane r's bit l is
#pragma unroll
  for (int sh = 16; sh > 0; sh >>= 1) {
    const uint32_t lo_mask = sh == 16 ? 0x0000FFFFu : sh == 8 ? 0x00FF00FFu : sh == 4 ? 0x0F0F0F0Fu
                             : sh == 2 ? 0x33333333u : 0x55555555u;
    const uint32_t v = __shfl_xor_sync(0xffffffffu, word, sh);
    word = (lane & sh) ? (word & ~lo_mask) | ((v >> sh) & lo_mask)
                       : (word & lo_mask) | ((v << sh) & ~lo_mask);
  }
  s_band[lane][warp] = word;   // little endian: byte q holds columns 8q .. 8q + 7, MSB first
  __syncthreads();
  const unsigned char *band = reinterpret_cast<const unsigned char *>(s_band);
  const int cb = cb0 + lane;
#pragma unroll
  for (int pass = 0; pass < 32 / kWarps; ++pass) {
    const int r = pass * kWarps + warp, y = y0 + r;
    if (y < H && cb < wb) plane[static_cast<long long>(y) * wb + cb] = band[r * 32 + lane];
  }
}

namespace overlaps {

struct Planes {
  Slots<const unsigned char> packed;   // image b: uint8 [R, H_b, wb_b]
  const int *counts;                   // [B]
  const long long *areas;              // [B, R]
  const int4 *extents;                 // [B, R] (y1, x1, y2, x2), exclusive ends
  int R;
};

// The checks of mrx_mask_overlaps and mrx_coco_ious on their two plane sets, in the order mrx.h
// states: "Output slots" for each set, null areas or extents, `outputs` (false when one of the
// caller's own pointers is null), then 4-byte-aligned bases; every message starts with fn.  On
// MRX_OK, p1 and p2 describe the two sets.
inline int check_plane_pair(const char *fn, const unsigned char *packed1, const long long *off1,
                            const int *counts1, const long long *areas1, const int *extents1,
                            int R1, const unsigned char *packed2, const long long *off2,
                            const int *counts2, const long long *areas2, const int *extents2,
                            int R2, const int *geom, int B, bool outputs, Planes &p1, Planes &p2) {
  if (int rc = check_slots(fn, packed1, off1, counts1, geom, B, R1)) return rc;
  if (int rc = check_slots(fn, packed2, off2, counts2, geom, B, R2)) return rc;
  MRX_CHECK_ARG(areas1 && extents1 && areas2 && extents2, "%s: null areas or extents", fn);
  MRX_CHECK_ARG(outputs, "%s: null pointer", fn);
  MRX_CHECK_ARG(((reinterpret_cast<uintptr_t>(packed1) | reinterpret_cast<uintptr_t>(packed2)) &
                 3u) == 0u,
                "%s: packed bases must be 4-byte aligned", fn);
  p1 = {{packed1, off1}, counts1, areas1, reinterpret_cast<const int4 *>(extents1), R1};
  p2 = {{packed2, off2}, counts2, areas2, reinterpret_cast<const int4 *>(extents2), R2};
  return MRX_OK;
}

__device__ __forceinline__ const unsigned char *plane_of(const Slots<const unsigned char> &s,
                                                         int b, int k, int H, int wb) {
  return s.base + s.off[b] + static_cast<long long>(k) * H * wb;
}

// The n (1..4) bytes at p as a little-endian word (byte p in bits 0-7), the rest zero, from the
// aligned words that hold them (only those: never a word past the last byte wanted).
__device__ __forceinline__ uint32_t load_bytes(const unsigned char *p, int n) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint32_t *w = reinterpret_cast<const uint32_t *>(a & ~static_cast<uintptr_t>(3));
  const int s = static_cast<int>(a & 3u);
  const uint32_t lo = __ldg(w);
  const uint32_t hi = s + n > 4 ? __ldg(w + 1) : 0u;
  const uint32_t v = __funnelshift_r(lo, hi, 8 * s);
  return n >= 4 ? v : v & ((1u << (8 * n)) - 1u);
}

// pixels of rows [y1, y2) x columns [x1, x2) set in both planes, summed over the warp
__device__ __forceinline__ long long and_count(const unsigned char *p1, const unsigned char *p2,
                                               int wb, int y1, int x1, int y2, int x2, int lane) {
  const int jb0 = x1 >> 3, nbytes = ((x2 - 1) >> 3) - jb0 + 1;
  const int nw = (nbytes + 3) >> 2;
  // edge bytes: pixels from x1 in the first byte, up to x2 - 1 in the last
  const uint32_t first = 0xFFu >> (x1 & 7), last = (0xFFu << (7 - ((x2 - 1) & 7))) & 0xFFu;
  const int total = (y2 - y1) * nw;
  long long n = 0;
  for (int e = lane; e < total; e += 32) {
    const int r = e / nw, c = e - r * nw;
    const long long o = static_cast<long long>(y1 + r) * wb + jb0 + 4 * c;
    const int nv = min(4, nbytes - 4 * c);
    uint32_t m = load_bytes(p1 + o, nv) & load_bytes(p2 + o, nv);
    if (c == 0) m &= first | 0xFFFFFF00u;
    if (c == nw - 1) {
      const int q = 8 * (nv - 1);
      m &= ~(0xFFu << q) | (last << q);
    }
    n += __popc(m);
  }
  return warp_sum(n);
}

// Plane i of p1 against every plane j < M_b of p2 with keep(j), in image b: one CTA of kWarps
// warps, a warp per j.  A pair whose extents do not meet (or with an empty mask) gets inter = 0
// without a read; the others AND and popcount the intersection rectangle, four bytes of a row per
// lane, each realigned from aligned words with a funnel shift.  Lane 0 then calls
// emit(j, inter, a1, a2) with the exact counts.
template <int kWarps, class Keep, class Emit>
__device__ __forceinline__ void walk_pairs(const Planes &p1, const Planes &p2,
                                           const int *__restrict__ geom, int b, int i, Keep keep,
                                           Emit emit) {
  const int M = p2.counts[b];
  const int H = geom[b * MRX_GEOM_INTS + 0], W = geom[b * MRX_GEOM_INTS + 1];
  const int wb = (W + 7) >> 3;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t i1 = static_cast<size_t>(b) * p1.R + i;
  const long long a1 = p1.areas[i1];
  const int4 e1 = p1.extents[i1];
  const unsigned char *plane1 = plane_of(p1.packed, b, i, H, wb);
  for (int j = warp; j < M; j += kWarps) {
    if (!keep(j)) continue;
    const size_t i2 = static_cast<size_t>(b) * p2.R + j;
    const long long a2 = p2.areas[i2];
    const int4 e2 = p2.extents[i2];
    const int y1 = max(e1.x, e2.x), x1 = max(e1.y, e2.y), y2 = min(e1.z, e2.z), x2 = min(e1.w, e2.w);
    long long inter = 0;
    if (a1 && a2 && y2 > y1 && x2 > x1)
      inter = and_count(plane1, plane_of(p2.packed, b, j, H, wb), wb, y1, x1, y2, x2, lane);
    if (lane == 0) emit(j, inter, a1, a2);
  }
}

// walk_pairs over the masks p1, p2 and their boundary planes q1, q2 at once (coco_boundary_iou_kernel):
// q1, q2 hold the boundaries in the slots of p1, p2 (same offsets, counts and R) with their own
// areas.  A boundary has its mask's tight extents, so the masks' cull and intersection rectangle
// serve both counts.  Lane 0 calls emit(j, inter, a1, a2, binter, ba1, ba2).
template <int kWarps, class Keep, class Emit>
__device__ __forceinline__ void walk_boundary_pairs(const Planes &p1, const Planes &p2,
                                                    const Planes &q1, const Planes &q2,
                                                    const int *__restrict__ geom, int b, int i,
                                                    Keep keep, Emit emit) {
  const int M = p2.counts[b];
  const int H = geom[b * MRX_GEOM_INTS + 0], W = geom[b * MRX_GEOM_INTS + 1];
  const int wb = (W + 7) >> 3;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t i1 = static_cast<size_t>(b) * p1.R + i;
  const long long a1 = p1.areas[i1], ba1 = q1.areas[i1];
  const int4 e1 = p1.extents[i1];
  const unsigned char *plane1 = plane_of(p1.packed, b, i, H, wb);
  const unsigned char *bplane1 = plane_of(q1.packed, b, i, H, wb);
  for (int j = warp; j < M; j += kWarps) {
    if (!keep(j)) continue;
    const size_t i2 = static_cast<size_t>(b) * p2.R + j;
    const long long a2 = p2.areas[i2], ba2 = q2.areas[i2];
    const int4 e2 = p2.extents[i2];
    const int y1 = max(e1.x, e2.x), x1 = max(e1.y, e2.y), y2 = min(e1.z, e2.z), x2 = min(e1.w, e2.w);
    long long inter = 0, binter = 0;
    if (a1 && a2 && y2 > y1 && x2 > x1) {
      inter = and_count(plane1, plane_of(p2.packed, b, j, H, wb), wb, y1, x1, y2, x2, lane);
      binter = and_count(bplane1, plane_of(q2.packed, b, j, H, wb), wb, y1, x1, y2, x2, lane);
    }
    if (lane == 0) emit(j, inter, a1, a2, binter, ba1, ba2);
  }
}

// score i of a rank kernel's [B, R] scores, float32 or (f64) float64
__device__ __forceinline__ double score_at(const void *scores, int f64, size_t i) {
  return f64 ? static_cast<const double *>(scores)[i]
             : static_cast<double>(static_cast<const float *>(scores)[i]);
}

}  // namespace overlaps

}  // namespace mrx
