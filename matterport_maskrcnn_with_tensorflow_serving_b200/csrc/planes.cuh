// planes.cuh -- reading two bit-packed plane sets of one batch together: the side description
// (Planes) and the AND-popcount of an intersection rectangle, shared by mask_overlaps_kernel
// (overlaps.cu) and coco_iou_kernel (cocoeval.cu).
//
// Planes are uint8 [N, H, ceil(W/8)], most significant bit first, as mrx_pack_masks /
// mrx_mask_expand_packed write them.  Pixel x of a row is bit 7 - (x & 7) of byte x >> 3 in every
// plane of an image, so the bytes of two planes line up column for column; only their addresses
// differ in alignment (a plane is H * ceil(W/8) bytes).
#pragma once

#include "common.cuh"

namespace mrx {

namespace overlaps {

struct Planes {
  Slots<const unsigned char> packed;   // image b: uint8 [R, H_b, wb_b]
  const int *counts;                   // [B]
  const long long *areas;              // [B, R]
  const int4 *extents;                 // [B, R] (y1, x1, y2, x2), exclusive ends
  int R;
};

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

}  // namespace overlaps

}  // namespace mrx
