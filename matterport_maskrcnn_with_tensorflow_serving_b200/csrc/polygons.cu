// polygons.cu -- COCO polygon ground truth to packed planes, bit for bit as pycocotools'
// rleFrPoly (maskApi.c) + rleMerge(intersect = 0) + rleDecode would give them.
//
// rleFrPoly walks every edge of the x5 upsampled polygon densely, keeps the points where the
// walk changes column in the original resolution as "toggles" at column-major positions
// xd*H + yd, and sorts them into runs: pixel p is set iff an odd number of toggles lie at
// positions <= p.  Sort-free, pixel (y, x) is the parity of every toggle in columns < x XOR the
// parity of the toggles of column x at rows <= y (a toggle at row H of column x counts only for
// columns > x).  The parts of an instance are ORed.
//
//   poly_toggles_kernel  CTA per part, thread per column: the thread finds the column's toggles
//                        edge by edge (<= 1 per edge inside it, <= 1 where two edges meet), in
//                        closed form for an x-major edge and by a binary search over the walk
//                        for a y-major one, so the work per edge does not grow with how far it
//                        runs outside the image; a block scan of the counts places each column's
//                        rows in the part's bucket and gives the parity of the columns before it
//   poly_planes_kernel   CTA per band of 32 rows x 256 columns of one plane, warp per 32 x 32
//                        block, lane per column: per part, the carry bit XOR a suffix mask per
//                        toggle of the column, ORed over the parts; store_band (planes.cuh)
//                        transposes and stores the band as rle_planes_kernel does
//
// Exactness: the minor coordinate of a walked point is (int)(a + s*t + .5) evaluated as
// pycocotools' x86-64 builds do, one rounding per operation (__dmul_rn / __dadd_rn, no FMA
// contraction) and truncation toward zero.  The downsampling tests, `(xd + .5) / 5 - .5` is an
// integer in [0, W-1] and `ceil(clamp((yd + .5) / 5 - .5, 0, H))`, are exact in integers: a
// quotient that is not an integer lies at least 0.2 from one, far beyond the double's error
// for |yd| < 2^32.
#include <climits>

#include "planes.cuh"

namespace mrx {

namespace polygons {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

// (int)(a + s*t + .5) as maskApi.c computes it
__device__ __forceinline__ long long minor_at(long long a, double s, long long t) {
  return __double2ll_rz(__dadd_rn(__dadd_rn(static_cast<double>(a),
                                            __dmul_rn(s, static_cast<double>(t))), 0.5));
}

// One edge of rleFrPoly's walk, from vertex (xa, ya) to (xb, yb) (scaled and rounded): the
// endpoints swapped when walking "backwards", points t = 0 .. n, emitted in the original
// direction (t = n .. 0 when flipped).
struct Edge {
  long long xs, ys, xe, ye, n;
  double s;
  bool xmaj, flip;

  __device__ __forceinline__ Edge(int2 a, int2 b) {
    const long long dx = llabs(static_cast<long long>(b.x) - a.x);
    const long long dy = llabs(static_cast<long long>(b.y) - a.y);
    xmaj = dx >= dy;
    flip = xmaj ? a.x > b.x : a.y > b.y;
    xs = flip ? b.x : a.x;
    ys = flip ? b.y : a.y;
    xe = flip ? a.x : b.x;
    ye = flip ? a.y : b.y;
    n = xmaj ? dx : dy;
    // a zero-length edge divides 0 by 0 in pycocotools; its one point never decides a toggle
    // (its column equals both neighbours' wherever that column is inside the image)
    s = n == 0 ? 0.0 : __ddiv_rn(static_cast<double>(xmaj ? ye - ys : xe - xs),
                                 static_cast<double>(n));
  }
  __device__ __forceinline__ long long u(long long t) const {
    return xmaj ? xs + t : minor_at(xs, s, t);
  }
  __device__ __forceinline__ long long v(long long t) const {
    return xmaj ? minor_at(ys, s, t) : ys + t;
  }
};

// the toggle row of a point pair whose lower row (scaled) is vmin
__device__ __forceinline__ int toggle_row(long long vmin, int H) {
  return vmin <= 2 ? 0 : static_cast<int>(min(static_cast<long long>(H), (vmin + 2) / 5));
}

// emit(row) for every toggle of part `v` (nv >= 1 vertices, closed) in column X
template <class Emit>
__device__ __forceinline__ void column_toggles(const int2 *__restrict__ v, int nv, int X, int H,
                                               Emit emit) {
  const long long c = 5LL * X + 2;   // a pair toggles column X iff its xd is c
  for (int j = 0; j < nv; ++j) {
    const int2 a = v[j], b = v[j + 1 < nv ? j + 1 : 0];
    // every walked point of the edge has u within 1 of [min x, max x], so the pair (c, c + 1)
    // inside it, or the pair where it meets the previous edge at a (xd within 2 of a.x), needs c
    // within 3 of that range: most edges of a part are culled here, in integers
    if (c + 1 < static_cast<long long>(min(a.x, b.x)) - 3 ||
        c > static_cast<long long>(max(a.x, b.x)) + 3)
      continue;
    const Edge e(a, b);
    const long long tf = e.flip ? e.n : 0, tl = e.flip ? 0 : e.n;
    const long long fu = e.u(tf);
    if (j > 0) {
      // the pair of the previous edge's last point and this edge's first
      const Edge p(v[j - 1], a);
      const long long pl = p.flip ? 0 : p.n, pu = p.u(pl);
      if (fu != pu && (fu < pu ? fu : fu - 1) == c) emit(toggle_row(min(e.v(tf), p.v(pl)), H));
    }
    const long long lu = e.u(tl);
    if (e.xmaj) {
      // u runs through xs .. xe one by one: the pair (c, c + 1)
      if (c >= e.xs && c + 1 <= e.xe) emit(toggle_row(min(e.v(c - e.xs), e.v(c + 1 - e.xs)), H));
    } else if (min(fu, lu) <= c && max(fu, lu) > c) {
      // u is monotone in t: the first t1 past c (u > c rising, u <= c falling) ends the one pair
      // that can give xd = c, (t1 - 1, t1) in t.  The pair's xd is its second emitted point's u
      // when u falls along the walk, that u - 1 when it rises: the point at t1 unless flipped
      const bool rising = e.s >= 0.0;
      long long lo = 0, hi = e.n;   // pred(lo) false, pred(hi) true
      while (hi - lo > 1) {
        const long long mid = lo + ((hi - lo) >> 1);
        if ((e.u(mid) > c) == rising)
          hi = mid;
        else
          lo = mid;
      }
      const long long want = rising != e.flip ? c + 1 : c;
      if (e.u(e.flip ? lo : hi) == want) emit(toggle_row(e.ys + lo, H));
    }
  }
}

__global__ void __launch_bounds__(kThreads)
poly_toggles_kernel(const int2 *__restrict__ vert, const long long *__restrict__ part_vert,
                    const int *__restrict__ part_inst, const long long *__restrict__ part_col,
                    const long long *__restrict__ part_tog, const int *__restrict__ geom, int R,
                    int *__restrict__ tog, long long *__restrict__ col_start,
                    unsigned char *__restrict__ carry) {
  __shared__ long long s_ll[kWarps];
  const int p = blockIdx.x;
  const int b = part_inst[p] / R;
  const int H = geom[b * MRX_GEOM_INTS + 0], W = geom[b * MRX_GEOM_INTS + 1];
  const int2 *v = vert + part_vert[p];
  const int nv = static_cast<int>(part_vert[p + 1] - part_vert[p]);
  long long *cs = col_start + part_col[p];
  unsigned char *cy = carry + part_col[p];
  const long long t0 = part_tog[p], t1 = part_tog[p + 1];
  long long done = 0;   // toggles of the columns before this pass
  for (int base = 0; base < W; base += kThreads) {
    const int X = base + threadIdx.x;
    long long n = 0;
    if (X < W) column_toggles(v, nv, X, H, [&](int) { ++n; });
    long long pass;
    const long long ex = done + block_exclusive_scan<long long, kThreads>(n, s_ll, pass);
    if (X < W) {
      // the host sizes the bucket from a bound on every edge; the clamp keeps every store (and
      // every later read) inside it whatever the bound
      long long q = t0 + ex;
      cs[X] = min(q, t1);
      cy[X] = static_cast<unsigned char>(ex & 1);
      column_toggles(v, nv, X, H, [&](int y) {
        if (q < t1) tog[q] = y;
        ++q;
      });
    }
    done += pass;
  }
  if (threadIdx.x == 0) cs[W] = min(t0 + done, t1);
}

__global__ void __launch_bounds__(kThreads)
poly_planes_kernel(Slots<unsigned char> packed, const int *__restrict__ inst_part,
                   const long long *__restrict__ part_col, const long long *__restrict__ col_start,
                   const unsigned char *__restrict__ carry, const int *__restrict__ tog,
                   const int *__restrict__ counts, const int *__restrict__ geom, int R,
                   int bands_x) {
  __shared__ uint32_t s_band[32][kWarps];   // row r: the band's 32 bytes, warp w's at [4w, 4w+4)
  const int k = blockIdx.y, b = blockIdx.z;
  if (k >= counts[b]) return;
  const size_t i = static_cast<size_t>(b) * R + k;
  const int p0 = inst_part[i], p1 = inst_part[i + 1];
  if (p0 >= p1) return;   // not a polygon instance: its plane is another path's
  const int H = geom[b * MRX_GEOM_INTS + 0], W = geom[b * MRX_GEOM_INTS + 1];
  const int wb = (W + 7) >> 3;
  const int y0 = (blockIdx.x / bands_x) * 32, cb0 = (blockIdx.x % bands_x) * 32;
  if (y0 >= H || cb0 >= wb) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int x = cb0 * 8 + warp * 32 + (lane ^ 7);
  uint32_t word = 0;   // pad columns (x >= W) stay zero
  if (x < W) {
    for (int p = p0; p < p1; ++p) {
      const long long o = part_col[p] + x;
      uint32_t w = carry[o] ? 0xFFFFFFFFu : 0u;
      for (long long q = col_start[o], qe = col_start[o + 1]; q < qe; ++q) {
        const int y = tog[q];
        if (y < y0)
          w = ~w;
        else if (y < y0 + 32)
          w ^= 0xFFFFFFFFu << (y - y0);
      }
      word |= w;
    }
  }
  store_band<kWarps>(word, s_band,
                     packed.base + packed.off[b] + static_cast<long long>(k) * H * wb, y0, cb0, H,
                     wb);
}

}  // namespace polygons

}  // namespace mrx

using namespace mrx;

extern "C" int mrx_poly_decode(const int *d_vert, const long long *d_part_vert,
                               const int *d_part_inst, const long long *d_part_col,
                               const long long *d_part_tog, int P, const int *d_inst_part,
                               int *d_tog, long long *d_col_start, unsigned char *d_carry,
                               const int *d_counts, const int *d_geom,
                               const long long *d_packed_off, unsigned char *d_packed, int B, int R,
                               int max_h, int max_w, void *stream) {
  const char *fn = "mrx_poly_decode";
  if (int rc = check_slots(fn, d_packed, d_packed_off, d_counts, d_geom, B, R)) return rc;
  MRX_CHECK_ARG(d_vert && d_part_vert && d_part_inst && d_part_col && d_part_tog && d_inst_part &&
                    d_tog && d_col_start && d_carry,
                "%s: null pointer", fn);
  MRX_CHECK_ARG(P >= 0, "%s: bad part count P=%d (need >= 0)", fn, P);
  MRX_CHECK_ARG(max_h >= 1 && max_w >= 1, "%s: bad extents max_h=%d max_w=%d (need >= 1)", fn,
                max_h, max_w);
  const long long bands_y = (max_h + 31LL) / 32, bands_x = ((max_w + 7LL) / 8 + 31) / 32;
  MRX_CHECK_SUPPORTED(bands_y * bands_x <= INT_MAX, "%s: image of %d x %d too large", fn, max_h,
                      max_w);
  if (B == 0 || P == 0) return MRX_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  polygons::poly_toggles_kernel<<<P, polygons::kThreads, 0, st>>>(
      reinterpret_cast<const int2 *>(d_vert), d_part_vert, d_part_inst, d_part_col, d_part_tog,
      d_geom, R, d_tog, d_col_start, d_carry);
  MRX_LAUNCH_CHECK("poly_toggles_kernel");
  polygons::poly_planes_kernel<<<dim3(static_cast<unsigned>(bands_y * bands_x), R, B),
                                 polygons::kThreads, 0, st>>>(
      {d_packed, d_packed_off}, d_inst_part, d_part_col, d_col_start, d_carry, d_tog, d_counts,
      d_geom, R, static_cast<int>(bands_x));
  MRX_LAUNCH_CHECK("poly_planes_kernel");
  return MRX_OK;
}
