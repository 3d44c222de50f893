// contours.cu -- mask outlines as polygons, the contour part of visualize.display_instances
// (serve.py:160-169): per instance, skimage.measure.find_contours(padded_mask, 0.5) on the mask
// padded with one row / column of zeros on every side, vertices as (x, y) = fliplr(v) - 1.
//
// Input: the bit-packed planes of mrx_pack_masks / mrx_mask_expand_packed (uint8 [N, H, ceil(W/8)],
// most significant bit first), so the outlines describe exactly the masks unmold_detections
// returns.  Each instance is traced inside a caller-given region (y1, x1, y2, x2) of pixels;
// pixels outside it count as 0.  With the one-pixel pad ring that is (y2-y1+1) x (x2-x1+1)
// marching-squares cells, cell (r, c) having the pixels (r-1, c-1), (r-1, c), (r, c-1), (r, c) as
// its corners (image coordinates; pixels outside the region or the image are 0).
//
// find_contours emits its segments cell by cell in raster order (the saddles 6 and 9 give two, in
// the order of the table below) and _assemble_contours joins them.  For a 0/1 image that join has
// a closed form, which is what the kernels compute:
//   - every vertex is an edge midpoint with exactly one segment leaving and one arriving, so each
//     segment has one successor and the segments form disjoint cycles (at least 4 long);
//   - contours are ordered by the smallest segment number of their cycle;
//   - a contour starts at the to-point of the LARGEST segment number of its cycle, follows the
//     successors and repeats its first vertex at the end (L + 1 vertices for L segments).
//
//   contour_count_kernel  warp per (instance, cell row): 34 cells per lane from two pixel rows with
//                         bit operations, segments per row
//   contour_row_scan_kernel / offsets_scan_kernel (capi.cu)   row offsets per instance, instance
//                         offsets
//   --- one host read of the total S and of the longest instance ---
//   contour_link_kernel   the same walk over three cell rows: each segment's raster number, its
//                         to-vertex, and its successor's number (row offset + popcount prefix)
//   contour_jump_kernel   ceil(log2(max S_i)) rounds of pointer jumping: each segment learns the
//                         smallest and largest number of its cycle and its distance to the largest
//   contour_head / scan / write kernels   contour lengths, an exclusive scan over the segments
//                         (contours and vertices before each cycle head; the tile sums by
//                         offsets_scan_kernel), the vertex stores
//
// Pointer jumping reads one 16-byte record per segment and round at a random address: the cost is
// about ceil(log2(max S_i)) x 48 bytes of traffic per segment, far above the counting walk.
#include "common.cuh"

namespace mrx {

namespace contours {

constexpr int kRowWarps = 8;            // warps (cell rows) per CTA of the count / link kernels
constexpr int kScanThreads = 1024;
constexpr int kScanItems = 4;           // consecutive segments per thread of the segment scan
constexpr int kScanTile = kScanThreads * kScanItems;

// cell edges
constexpr int kTop = 0, kBottom = 1, kLeft = 2, kRight = 3;

constexpr uint32_t pack_edges(const int (&e)[16]) {
  uint32_t v = 0;
  for (int q = 0; q < 16; ++q) v |= static_cast<uint32_t>(e[q]) << (2 * q);
  return v;
}
// find_contours' segment table (vertex_connect_high = False), case = ul + 2 ur + 4 ll + 8 lr,
// (from, to) of the first segment:
//   1 (T,L)  2 (R,T)  3 (R,L)  4 (L,B)  5 (T,B)  6 (R,T)  7 (R,B)
//   8 (B,R)  9 (T,L) 10 (B,T) 11 (B,L) 12 (L,R) 13 (T,R) 14 (L,T)
// and the saddles' second segment: case 6 (L,B), case 9 (B,R).  A segment's successor is the
// segment of the neighbour across its to-edge that leaves through the same edge, so only the
// to-edges are stored; the one neighbour with two candidates is a saddle, whose second segment
// leaves through the left edge (case 6) or the bottom edge (case 9).
constexpr int kFirstTo[16] = {0, kLeft, kTop, kLeft, kBottom, kBottom, kTop, kBottom,
                              kRight, kLeft, kTop, kLeft, kRight, kRight, kTop, 0};
constexpr uint32_t kToTab = pack_edges(kFirstTo);

// window of one lane: cells c0 - 1 + j, j in [0, 34); its own cells are j in [1, 33)
constexpr uint64_t kWindow = (1ull << 34) - 1;
constexpr uint64_t kOwn = kWindow & ~1ull & ~(1ull << 33);

struct Params {
  Slots<const unsigned char> packed;   // image b: uint8 [R, H_b, wb_b] (mrx.h, "Output slots")
  const int *counts;             // [B]
  const int *geom;               // [B, 8]
  const int4 *regions;           // [B, R] (y1, x1, y2, x2) pixels
  int *row_off;                  // [B*R, row_pitch]: segments per cell row -> exclusive offsets
  long long *inst_off;           // [B*R + 1]
  int R, row_pitch;
  // link pass
  int *succ;                     // [S]
  float2 *to;                    // [S]
  int4 *jump;                    // [S] (jump pointer, min, max, distance to max)
};

struct Region {
  int y1, x1, y2, x2;            // pixels; empty: y2 == y1
};

struct Inst {
  const unsigned char *plane;
  int wb, nrows, nwords;
  Region g;
};

// instance k of image b, its region clamped to the image; nrows = 0 when there is nothing to trace
__device__ __forceinline__ Inst inst_of(const Params &p, int b, int k) {
  Inst in;
  const int H = p.geom[b * MRX_GEOM_INTS + 0], W = p.geom[b * MRX_GEOM_INTS + 1];
  in.wb = (W + 7) >> 3;
  in.plane = p.packed.base + p.packed.off[b] +static_cast<long long>(k) * H * in.wb;
  const int4 r = p.regions[static_cast<size_t>(b) * p.R + k];
  in.g = {max(r.x, 0), max(r.y, 0), min(r.z, H), min(r.w, W)};
  const bool empty = k >= p.counts[b] || in.g.y2 <= in.g.y1 || in.g.x2 <= in.g.x1;
  in.nrows = empty ? 0 : min(in.g.y2 - in.g.y1 + 1, p.row_pitch);
  in.nwords = empty ? 0 : (in.g.x2 - in.g.x1 + 1 + 31) >> 5;
  if (empty) in.g = {0, 0, 0, 0};
  return in;
}

// bits [a, b) of a 64-bit word (clipped to [0, 64))
__device__ __forceinline__ uint64_t span_mask(int a, int b) {
  a = max(a, 0);
  b = min(b, 64);
  if (b <= a) return 0ull;
  const uint64_t hi = b == 64 ? ~0ull : (1ull << b) - 1ull;
  return hi & ~((1ull << a) - 1ull);
}

// bit t = pixel (y, x + t) for t < 41; zero outside the region.  Rows are byte-aligned only, so
// the bytes are loaded one by one.
__device__ __forceinline__ uint64_t pixel_bits(const Inst &in, int y, int x) {
  if (y < in.g.y1 || y >= in.g.y2) return 0ull;
  const unsigned char *row = in.plane + static_cast<size_t>(y) * in.wb;
  const int jb = x >> 3;   // floor
  uint64_t v = 0ull;
#pragma unroll
  for (int t = 0; t < 6; ++t) {
    const int j = jb + t;
    const uint64_t byte = (j >= 0 && j < in.wb) ? __ldg(row + j) : 0u;
    v |= byte << (56 - 8 * t);
  }
  v = __brevll(v << (x & 7));
  return v & span_mask(in.g.x1 - x, in.g.x2 - x);
}

// the cases of the 34 cells c0 - 1 + j of cell row r, as corner bit masks over j
struct CellRow {
  uint64_t ul, ur, ll, lr, ne, s6, s9;
  __device__ __forceinline__ uint64_t saddle() const { return s6 | s9; }
  __device__ __forceinline__ int own_count() const {
    return __popcll(ne & kOwn) + __popcll((s6 | s9) & kOwn);
  }
  // segments of the own cells before window cell j (j in [1, 33])
  __device__ __forceinline__ int before(int j) const {
    const uint64_t lo = kOwn & ((1ull << j) - 1ull);
    return __popcll(ne & lo) + __popcll((s6 | s9) & lo);
  }
};

__device__ __forceinline__ CellRow cell_row(const Inst &in, int r, int c0) {
  const uint64_t t = pixel_bits(in, r - 1, c0 - 2), u = pixel_bits(in, r, c0 - 2);
  CellRow cr;
  cr.ul = t;
  cr.ur = t >> 1;
  cr.ll = u;
  cr.lr = u >> 1;
  const uint64_t any = cr.ul | cr.ur | cr.ll | cr.lr, all = cr.ul & cr.ur & cr.ll & cr.lr;
  cr.ne = any & ~all & kWindow;
  cr.s6 = ~cr.ul & cr.ur & cr.ll & ~cr.lr & kWindow;
  cr.s9 = cr.ul & ~cr.ur & ~cr.ll & cr.lr & kWindow;
  return cr;
}

// One warp per (instance, cell row): segments of the row, lanes on 32-cell words.
__global__ void __launch_bounds__(kRowWarps * 32)
contour_count_kernel(const Params p) {
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * kRowWarps + (threadIdx.x >> 5);
  const int k = blockIdx.y, b = blockIdx.z;
  const Inst in = inst_of(p, b, k);
  if (j >= in.nrows) return;
  const int r = in.g.y1 + j;
  int n = 0;
  for (int w = lane; w < in.nwords; w += 32) n += cell_row(in, r, in.g.x1 + 32 * w).own_count();
  n = warp_sum(n);
  if (lane == 0) p.row_off[(static_cast<size_t>(b) * p.R + k) * p.row_pitch + j] = n;
}

// One CTA per instance: exclusive scan of its cell rows' counts (in place), instance total out.
__global__ void __launch_bounds__(256)
contour_row_scan_kernel(const Params p) {
  const int k = blockIdx.x, b = blockIdx.y;
  const size_t inst = static_cast<size_t>(b) * p.R + k;
  const long long total = block_scan_range<256>(p.row_off + inst * p.row_pitch, 0, inst_of(p, b, k).nrows);
  if (threadIdx.x == 0) p.inst_off[inst] = total;
}

// The count walk again over the rows above, at and below: every segment of the row gets its
// number, its to-vertex and its successor's number.
__global__ void __launch_bounds__(kRowWarps * 32)
contour_link_kernel(const Params p) {
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * kRowWarps + (threadIdx.x >> 5);
  const int k = blockIdx.y, b = blockIdx.z;
  const Inst in = inst_of(p, b, k);
  if (j >= in.nrows) return;
  const size_t inst = static_cast<size_t>(b) * p.R + k;
  const int r = in.g.y1 + j;
  const int *ro = p.row_off + inst * p.row_pitch;
  const int ib = static_cast<int>(p.inst_off[inst]);
  // first segment number of the rows above / at / below (advanced word chunk by word chunk)
  int base_u = ib + (j > 0 ? ro[j - 1] : 0);
  int base_c = ib + ro[j];
  int base_d = ib + (j + 1 < in.nrows ? ro[j + 1] : 0);
  for (int w0 = 0; w0 < in.nwords; w0 += 32) {
    const int w = w0 + lane;
    const bool valid = w < in.nwords;
    const int c0 = in.g.x1 + 32 * w;
    CellRow up{}, cr{}, dn{};
    if (valid) {
      up = cell_row(in, r - 1, c0);
      cr = cell_row(in, r, c0);
      dn = cell_row(in, r + 1, c0);
    }
    const int nu = up.own_count(), nc = cr.own_count(), nd = dn.own_count();
    const int iu = warp_inclusive_scan(nu, lane), ic = warp_inclusive_scan(nc, lane),
              id = warp_inclusive_scan(nd, lane);
    // first segment number of this word's own cells in each row
    const int wu = base_u + iu - nu, wc = base_c + ic - nc, wd = base_d + id - nd;
    base_u += __shfl_sync(0xffffffffu, iu, 31);
    base_c += __shfl_sync(0xffffffffu, ic, 31);
    base_d += __shfl_sync(0xffffffffu, id, 31);
    if (!valid) continue;
    const uint64_t sad_c = cr.saddle();
    for (uint64_t m = cr.ne & kOwn; m; m &= m - 1ull) {
      const int jj = __ffsll(static_cast<long long>(m)) - 1;
      const int q = static_cast<int>((cr.ul >> jj) & 1ull) | static_cast<int>((cr.ur >> jj) & 1ull) << 1 |
                    static_cast<int>((cr.ll >> jj) & 1ull) << 2 | static_cast<int>((cr.lr >> jj) & 1ull) << 3;
      const int c = c0 - 1 + jj;
      const int first = wc + cr.before(jj);
      const int nseg = 1 + static_cast<int>((sad_c >> jj) & 1ull);
#pragma unroll 1
      for (int t = 0; t < nseg; ++t) {
        const int to = t == 0 ? static_cast<int>((kToTab >> (2 * q)) & 3u) : (q == 6 ? kBottom : kRight);
        int next;
        float2 v;
        switch (to) {
          case kTop:      // enters the cell above through its bottom edge (case 9's second segment)
            next = wu + up.before(jj) + static_cast<int>((up.s9 >> jj) & 1ull);
            v = make_float2(c - 0.5f, static_cast<float>(r - 1));
            break;
          case kBottom:   // enters the cell below through its top edge
            next = wd + dn.before(jj);
            v = make_float2(c - 0.5f, static_cast<float>(r));
            break;
          case kLeft: {   // enters the cell to the left through its right edge
            const int jl = jj - 1;
            next = jl == 0 ? wc - 1 - static_cast<int>((sad_c & 1ull) != 0) : wc + cr.before(jl);
            v = make_float2(static_cast<float>(c - 1), r - 0.5f);
            break;
          }
          default: {      // right: enters the cell to the right through its left edge
            const int jr = jj + 1;   // (case 6's second segment)
            next = wc + cr.before(jr) + static_cast<int>((cr.s6 >> jr) & 1ull);
            v = make_float2(static_cast<float>(c), r - 0.5f);
            break;
          }
        }
        const int s = first + t;
        p.succ[s] = next;
        p.to[s] = v;
        p.jump[s] = make_int4(next, s, s, 0);
      }
    }
  }
}

// One round of pointer jumping.  Record of s over the 2^k segments s, succ(s), ...:
//   x = the segment 2^k steps on, y = smallest number, z = largest number, w = steps to the first
// occurrence of z.  Once 2^k >= the cycle length, y and z are the cycle's and w = the distance
// from s to the cycle's largest segment.
__global__ void __launch_bounds__(256)
contour_jump_kernel(const int4 *__restrict__ in, int4 *__restrict__ out, int S, int span) {
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < S; s += gridDim.x * blockDim.x) {
    const int4 a = in[s];
    const int4 t = in[a.x];
    int4 o;
    o.x = t.x;
    o.y = min(a.y, t.y);
    if (t.z > a.z) {
      o.z = t.z;
      o.w = span + t.w;
    } else {
      o.z = a.z;
      o.w = a.w;
    }
    out[s] = o;
  }
}

// Cycle heads (the smallest segment of each cycle): contour length L, and the scan input
// (1 contour, L + 1 vertices) packed as (count << 32) | vertices.
__global__ void __launch_bounds__(256)
contour_head_kernel(const int4 *__restrict__ f, const int *__restrict__ succ,
                    unsigned long long *__restrict__ scan, int *__restrict__ len, int S) {
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < S; s += gridDim.x * blockDim.x) {
    const int4 r = f[s];
    unsigned long long v = 0ull;
    if (r.y == s) {
      const int L = f[succ[r.z]].w + 1;   // the largest segment's successor is L - 1 steps from it
      len[s] = L;
      v = (1ull << 32) | static_cast<unsigned>(L + 1);
    }
    scan[s] = v;
  }
}

// exclusive scan of the packed (contours, vertices) pairs: tile sums, scan of the tile sums (total
// at bsum[ntiles], launch_offsets_scan), tile scans
__global__ void __launch_bounds__(kScanThreads)
contour_scan_reduce_kernel(const unsigned long long *__restrict__ v, unsigned long long *bsum, int S) {
  __shared__ unsigned long long s_warp[kScanThreads / 32];
  const long long i0 = static_cast<long long>(blockIdx.x) * kScanTile + threadIdx.x * kScanItems;
  unsigned long long x = 0ull;
#pragma unroll
  for (int t = 0; t < kScanItems; ++t)
    if (i0 + t < S) x += v[i0 + t];
  unsigned long long tot;
  block_exclusive_scan<unsigned long long, kScanThreads>(x, s_warp, tot);
  if (threadIdx.x == 0) bsum[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(kScanThreads)
contour_scan_apply_kernel(unsigned long long *v, const unsigned long long *__restrict__ bsum, int S) {
  __shared__ unsigned long long s_warp[kScanThreads / 32];
  const long long i0 = static_cast<long long>(blockIdx.x) * kScanTile + threadIdx.x * kScanItems;
  unsigned long long x[kScanItems], sum = 0ull;
#pragma unroll
  for (int t = 0; t < kScanItems; ++t) {
    x[t] = i0 + t < S ? v[i0 + t] : 0ull;
    sum += x[t];
  }
  unsigned long long tot;
  unsigned long long run = bsum[blockIdx.x] +
                           block_exclusive_scan<unsigned long long, kScanThreads>(sum, s_warp, tot);
#pragma unroll
  for (int t = 0; t < kScanItems; ++t) {
    if (i0 + t < S) v[i0 + t] = run;
    run += x[t];
  }
}

// Vertex j (1..L) of a contour is the to-point of the segment j steps after its largest one; the
// largest segment also stores vertex 0.  Cycle heads store their contour's vertex offset.
__global__ void __launch_bounds__(256)
contour_write_kernel(const int4 *__restrict__ f, const int *__restrict__ len,
                     const unsigned long long *__restrict__ pre, const float2 *__restrict__ to,
                     float2 *__restrict__ verts, long long *__restrict__ contour_off, int S) {
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < S; s += gridDim.x * blockDim.x) {
    const int4 r = f[s];
    const int m = r.y;
    const unsigned long long pm = pre[m];
    const unsigned base = static_cast<unsigned>(pm);
    const int L = len[m];
    const float2 v = to[s];
    verts[base + static_cast<unsigned>(L - r.w)] = v;
    if (r.w == 0) verts[base] = v;
    if (m == s) contour_off[pm >> 32] = static_cast<long long>(base);
  }
}

// contours before every instance, and the closing vertex offset
__global__ void __launch_bounds__(256)
contour_finish_kernel(const long long *__restrict__ inst_off, const unsigned long long *pre,
                      const unsigned long long *total, long long *contour_off,
                      long long *inst_contour_off, int n, int S) {
  const unsigned long long t = S > 0 ? *total : 0ull;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += gridDim.x * blockDim.x) {
    const long long o = inst_off[i];
    inst_contour_off[i] = static_cast<long long>((o < S ? pre[o] : t) >> 32);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) contour_off[t >> 32] = static_cast<long long>(t & 0xffffffffull);
}

}  // namespace contours

}  // namespace mrx

using namespace mrx;

static int fill_contour_params(contours::Params &prm, const char *fn, const unsigned char *d_packed,
                               const long long *d_packed_off, const int *d_counts,
                               const int *d_geom, const int *d_regions, const int *d_row_off,
                               const long long *d_inst_off, int B, int R, int max_h) {
  if (int rc = check_slots(fn, d_packed, d_packed_off, d_counts, d_geom, B, R)) return rc;
  MRX_CHECK_ARG(d_row_off && d_inst_off, "%s: null pointer", fn);
  MRX_CHECK_ARG(d_regions, "%s: the region argument d_regions is required", fn);
  MRX_CHECK_ARG(max_h >= 1 && max_h < (1 << 30), "%s: bad max_h %d (need 1<=max_h<2^30)", fn,
                max_h);
  prm = {};
  prm.packed = {d_packed, d_packed_off};
  prm.counts = d_counts;
  prm.geom = d_geom;
  prm.regions = reinterpret_cast<const int4 *>(d_regions);
  prm.row_off = const_cast<int *>(d_row_off);
  prm.inst_off = const_cast<long long *>(d_inst_off);
  prm.R = R;
  prm.row_pitch = max_h + 1;
  return MRX_OK;
}

static dim3 row_grid(int B, int R, int max_h) {
  return dim3((max_h + 1 + contours::kRowWarps - 1) / contours::kRowWarps, R, B);
}

extern "C" int mrx_contours_count(const unsigned char *d_packed, const long long *d_packed_off,
                                  const int *d_counts, const int *d_geom, const int *d_regions,
                                  int *d_row_off, long long *d_inst_off, int B, int R, int max_h,
                                  void *stream) {
  contours::Params prm;
  if (int rc = fill_contour_params(prm, "mrx_contours_count", d_packed, d_packed_off, d_counts,
                                   d_geom, d_regions, d_row_off, d_inst_off, B, R, max_h))
    return rc;
  if (B == 0) return MRX_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  contours::contour_count_kernel<<<row_grid(B, R, max_h), contours::kRowWarps * 32, 0, st>>>(prm);
  MRX_LAUNCH_CHECK("contour_count_kernel");
  contours::contour_row_scan_kernel<<<dim3(R, B), 256, 0, st>>>(prm);
  MRX_LAUNCH_CHECK("contour_row_scan_kernel");
  return launch_offsets_scan(d_inst_off, B * R, st);
}

extern "C" int mrx_contours_write(const unsigned char *d_packed, const long long *d_packed_off,
                                  const int *d_counts, const int *d_geom, const int *d_regions,
                                  const int *d_row_off, const long long *d_inst_off,
                                  long long total_segments, long long max_inst_segments,
                                  void *d_scratch, float *d_vertices, long long *d_contour_off,
                                  long long *d_inst_contour_off, int B, int R, int max_h,
                                  void *stream) {
  using namespace contours;
  Params prm;
  if (int rc = fill_contour_params(prm, "mrx_contours_write", d_packed, d_packed_off, d_counts,
                                   d_geom, d_regions, d_row_off, d_inst_off, B, R, max_h))
    return rc;
  MRX_CHECK_ARG(d_contour_off && d_inst_contour_off, "mrx_contours_write: null pointer");
  MRX_CHECK_ARG(total_segments >= 0 && max_inst_segments >= 0 &&
                    max_inst_segments <= total_segments,
                "mrx_contours_write: bad segment counts S=%lld max=%lld", total_segments,
                max_inst_segments);
  MRX_CHECK_SUPPORTED(total_segments <= MRX_MAX_CONTOUR_SEGMENTS,
                      "mrx_contours_write: %lld segments (limit %d per call)", total_segments,
                      MRX_MAX_CONTOUR_SEGMENTS);
  MRX_CHECK_ARG(total_segments == 0 || (d_scratch && d_vertices),
                "mrx_contours_write: null scratch or vertex pointer");
  if (B == 0) return MRX_OK;
  const int S = static_cast<int>(total_segments);
  DevInfo dev;
  if (int rc = current_device_info(&dev)) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int ntiles = (S + kScanTile - 1) / kScanTile;
  // scratch: two jump records, to-points and successors per segment, then the tile sums
  unsigned char *base = static_cast<unsigned char *>(d_scratch);
  int4 *jump[2] = {reinterpret_cast<int4 *>(base), reinterpret_cast<int4 *>(base + 16ll * S)};
  prm.to = reinterpret_cast<float2 *>(base + 32ll * S);
  prm.succ = reinterpret_cast<int *>(base + 40ll * S);
  unsigned long long *bsum = reinterpret_cast<unsigned long long *>(base + ((44ll * S + 15) & ~15ll));
  prm.jump = jump[0];
  const int grid = S > 0 ? min((S + 255) / 256, dev.sms * 8) : 1;
  if (S > 0) {
    contour_link_kernel<<<row_grid(B, R, max_h), kRowWarps * 32, 0, st>>>(prm);
    MRX_LAUNCH_CHECK("contour_link_kernel");
    int cur = 0;
    for (long long span = 1; span < max_inst_segments; span <<= 1) {
      contour_jump_kernel<<<grid, 256, 0, st>>>(jump[cur], jump[cur ^ 1], S, static_cast<int>(span));
      MRX_LAUNCH_CHECK("contour_jump_kernel");
      cur ^= 1;
    }
    // the other record buffer now holds the scan values (8 B) and the contour lengths (4 B)
    unsigned long long *scan = reinterpret_cast<unsigned long long *>(jump[cur ^ 1]);
    int *len = reinterpret_cast<int *>(reinterpret_cast<unsigned char *>(jump[cur ^ 1]) + 8ll * S);
    contour_head_kernel<<<grid, 256, 0, st>>>(jump[cur], prm.succ, scan, len, S);
    MRX_LAUNCH_CHECK("contour_head_kernel");
    contour_scan_reduce_kernel<<<ntiles, kScanThreads, 0, st>>>(scan, bsum, S);
    MRX_LAUNCH_CHECK("contour_scan_reduce_kernel");
    // The tile sums are (contours << 32) | vertices pairs.  Every partial sum stays below 2^61 and
    // the low half never carries (V = S + C < 2^32 at MRX_MAX_CONTOUR_SEGMENTS), so the signed
    // 64-bit scan gives the same bits as an unsigned one.
    if (int rc = launch_offsets_scan(reinterpret_cast<long long *>(bsum), ntiles, st)) return rc;
    contour_scan_apply_kernel<<<ntiles, kScanThreads, 0, st>>>(scan, bsum, S);
    MRX_LAUNCH_CHECK("contour_scan_apply_kernel");
    contour_write_kernel<<<grid, 256, 0, st>>>(jump[cur], len, scan, prm.to,
                                               reinterpret_cast<float2 *>(d_vertices),
                                               d_contour_off, S);
    MRX_LAUNCH_CHECK("contour_write_kernel");
    contour_finish_kernel<<<(B * R + 256) / 256, 256, 0, st>>>(d_inst_off, scan, bsum + ntiles,
                                                               d_contour_off, d_inst_contour_off,
                                                               B * R, S);
  } else {
    contour_finish_kernel<<<(B * R + 256) / 256, 256, 0, st>>>(d_inst_off, nullptr, nullptr,
                                                               d_contour_off, d_inst_contour_off,
                                                               B * R, 0);
  }
  MRX_LAUNCH_CHECK("contour_finish_kernel");
  return MRX_OK;
}
