// rle.cu -- COCO run-length masks straight from the 28x28 tiles (SURVEY.md 8f rank 4: the second
// compact format it names; the output of serve.py:147 re-encoded).
//
// EXTENSION, not the reference layout.  For every kept instance the result is the
// "uncompressed RLE" of pycocotools, {'size': [H, W], 'counts': [...]}: the [H, W] mask read in
// COLUMN-major order as alternating runs of zeros and ones, starting with zeros (a leading 0
// when the first pixel is set).  The mask itself is never materialised: the kernels evaluate the
// same samples as mrx_mask_expand (same exact integer source coordinates, same fp32 weights,
// same two fused multiply-adds -- horizontal then vertical), but with lanes on 32 adjacent
// COLUMNS walking DOWN the box, so each lane meets the pixels of its column in run-length
// order and only has to note where the value changes.
//
//   rle_walk_kernel<false>   per (instance, 32-column block): number of transitions per column
//   rle_scan_kernel          per instance: exclusive scan over its columns, instance total
//   offsets_scan_kernel      exclusive scan of the instance totals (capi.cu, one CTA)
//   rle_walk_kernel<true>    the same walk again, now writing each transition's flat position
//                            x*H + y at (instance base + column offset + running index)
//   rle_counts_kernel        positions -> run lengths (differences, closing run to H*W)
//
// mrx_rle_strings turns those run lengths into pycocotools' compressed RLE ("counts" string of
// mask.encode, its rleToString) on the device:
//   rle_string_count_kernel  per instance: characters of its string
//   offsets_scan_kernel      exclusive scan of the instance lengths (capi.cu, one CTA)
//   rle_string_write_kernel  per instance: the characters, a CTA-wide scan per chunk of runs
//
// Column seams: column x continues at (x+1, 0) after (x, H-1).  Outside its box an instance is
// zero, so a column starts after a zero unless the box spans the full height (then it starts
// after the previous column's last pixel), and a run still open at the last box row is closed
// by a transition at the first pixel below the box (or at the top of the next column).
//
// Instruction-bound on the in-box samples like the packed expand kernel; the output is a few
// bytes per run (a few MB per batch of real masks).
#include "expand.cuh"

namespace mrx {

namespace rle {

constexpr int kWalkWarps = 8;

struct RleParams {
  TileBatch t;
  int *col_count;             // [B,R,max_w]: transitions per column -> exclusive offsets (scan)
  long long *inst_off;        // [B*R + 1]: totals -> exclusive offsets of the instances
  unsigned int *positions;    // [total] flat positions of the transitions (write pass)
  int max_w;
};

// One warp: instance k of image b, columns [32*cb, 32*cb + 32).
template <bool kWrite>
__global__ void __launch_bounds__(kWalkWarps * 32)
rle_walk_kernel(const RleParams p) {
  const int lane = threadIdx.x & 31;
  const int cb = blockIdx.x * kWalkWarps + (threadIdx.x >> 5);
  const int k = blockIdx.y, b = blockIdx.z;
  if (k >= p.t.counts[b]) return;
  const int H = p.t.geom[b * MRX_GEOM_INTS + 0], W = p.t.geom[b * MRX_GEOM_INTS + 1];
  const int4 bx = __ldg(p.t.boxes + static_cast<size_t>(b) * p.t.R + k);   // (y1, x1, y2, x2)
  if (!box_in_canvas(bx, H, W) || (cb << 5) >= bx.w || (cb << 5) + 32 <= bx.y) return;
  const int mh = p.t.mh, mw = p.t.mw;
  const int bh = bx.z - bx.x, bw = bx.w - bx.y;
  const int D = 2 * bw, Dy = 2 * bh;
  const float invD = __fdiv_rn(1.0f, static_cast<float>(D));
  const float invDy = __fdiv_rn(1.0f, static_cast<float>(Dy));
  const int tile = __ldg(p.t.tile_index + static_cast<size_t>(b) * p.t.R + k);
  const bool lanecol = lane >= 1 && lane <= mw;      // lane l holds tile column l - 1
  const int lcol = min(max(lane - 1, 0), mw - 1);
  const LaneRows raw{p.t.tiles + (static_cast<size_t>(b) * p.t.R + tile) * mh * mw + lcol, mh, mw, lanecol};
  // horizontal source coordinate of column x: taps idx, idx + 1 of the zero-padded tile row
  auto hcoord = [&](int x, int &idx, float &wx) {
    const SrcPos s = src_floor(src_num(mw, x, bx.y, bw), D, invD);
    idx = min(max(s.i + 1, 0), 30);
    wx = src_weight(s.rem, invD);
  };
  const int x = (cb << 5) + lane;
  const bool colvalid = x >= bx.y && x < bx.w;
  int idx;
  float wx;
  hcoord(x, idx, wx);
  const float thr = colvalid ? 0.5f : __int_as_float(0x7f800000);

  const SrcPos first = src_floor(src_num(mh, bx.x, bx.x, bh), Dy, invDy);   // first box row
  int jcur = first.i, remy = first.rem;
  const SrcStep ystep = src_step(2 * mh, Dy);   // source-row advance per canvas row

  const bool full = bx.x == 0 && bx.z == H;          // column seams carry the previous column's bit
  unsigned int *out = nullptr;
  if (kWrite) {
    const size_t inst = static_cast<size_t>(b) * p.t.R + k;
    out = p.positions + p.inst_off[inst] + (colvalid ? p.col_count[inst * p.max_w + x] : 0);
  }
  const unsigned base = static_cast<unsigned>(x) * static_cast<unsigned>(H);
  int n = 0;
  bool prev = false;
  // With a full-height box the first row's predecessor is the previous column's LAST pixel:
  // one extra sample (column x - 1, row H - 1), evaluated exactly as that column's own walk
  // evaluates it.
  bool prev_top = false;
  if (full) {
    // last row's vertical coordinate (same exact arithmetic, from the row index)
    const SrcPos last = src_floor(src_num(mh, bx.z - 1, bx.x, bh), Dy, invDy);
    int idp;
    float wxp;
    hcoord(x - 1, idp, wxp);
    const float rt = raw(last.i), rbv = raw(last.i + 1);
    const float vl = lerp(src_weight(last.rem, invDy), hrow(rt, idp, wxp), hrow(rbv, idp, wxp));
    prev_top = colvalid && x - 1 >= bx.y && vl >= 0.5f;
  }
  prev = prev_top;

  int j0 = jcur;
  float ht = hrow(raw(jcur), idx, wx), hb = hrow(raw(jcur + 1), idx, wx);
  float rawn = raw(jcur + 2);
  float dh = hb - ht;
  bool cur = false;
  for (int r = bx.x; r < bx.z; ++r) {
    if (j0 != jcur) {   // warp-uniform
      if (j0 == jcur + 1) {
        ht = hb;
        hb = hrow(rawn, idx, wx);
      } else {
        ht = hrow(raw(j0), idx, wx);
        hb = hrow(raw(j0 + 1), idx, wx);
      }
      jcur = j0;
      rawn = raw(jcur + 2);
      dh = hb - ht;
    }
    const float v = fmaf(src_weight(remy, invDy), dh, ht);
    cur = v >= thr;
    if (cur != prev) {
      if (kWrite) out[n] = base + static_cast<unsigned>(r);
      ++n;
    }
    prev = cur;
    src_advance(j0, remy, ystep, Dy);
  }
  // a run still open at the last box row ends at the next pixel in column-major order -- below
  // the box, or the top of the next column -- unless that pixel is the next column of a
  // full-height box (its own top comparison sees it) or lies past the end of the image
  if (cur) {
    const bool next_is_box = full && x + 1 < bx.w;
    const unsigned long long pend = bx.z < H ? static_cast<unsigned long long>(base) + bx.z
                                             : static_cast<unsigned long long>(base) + H;
    if (!next_is_box && pend < static_cast<unsigned long long>(H) * W) {
      if (kWrite) out[n] = static_cast<unsigned>(pend);
      ++n;
    }
  }
  if (!kWrite && colvalid) p.col_count[(static_cast<size_t>(b) * p.t.R + k) * p.max_w + x] = n;
}

// One CTA per instance: exclusive scan of its box columns' transition counts (in place), total out.
__global__ void __launch_bounds__(256)
rle_scan_kernel(const RleParams p) {
  const int k = blockIdx.x, b = blockIdx.y;
  const size_t inst = static_cast<size_t>(b) * p.t.R + k;
  int x1 = 0, x2 = 0;   // no columns: not a kept instance, or its box is outside the canvas
  if (k < p.t.counts[b]) {
    const int H = p.t.geom[b * MRX_GEOM_INTS + 0], W = p.t.geom[b * MRX_GEOM_INTS + 1];
    const int4 bx = p.t.boxes[inst];
    if (box_in_canvas(bx, H, W)) {
      x1 = bx.y;
      x2 = bx.w;
    }
  }
  const long long total = block_scan_range<256>(p.col_count + inst * p.max_w, x1, x2);
  if (threadIdx.x == 0) p.inst_off[inst] = total;
}

// positions -> run lengths.  Instance i has T = inst_off[i+1] - inst_off[i] transitions and
// T + 1 runs; its runs start at counts + inst_off[i] + i.
__global__ void __launch_bounds__(256)
rle_counts_kernel(const unsigned int *__restrict__ positions, const long long *__restrict__ inst_off,
                  const int *__restrict__ counts_per_image, const int *__restrict__ geom, int R,
                  unsigned int *__restrict__ counts) {
  const int k = blockIdx.x, b = blockIdx.y;
  if (k >= counts_per_image[b]) return;
  const size_t inst = static_cast<size_t>(b) * R + k;
  const long long lo = inst_off[inst], hi = inst_off[inst + 1];
  const unsigned total = static_cast<unsigned>(geom[b * MRX_GEOM_INTS + 0]) *
                         static_cast<unsigned>(geom[b * MRX_GEOM_INTS + 1]);
  unsigned int *o = counts + lo + inst;
  const long long T = hi - lo;
  for (long long j = threadIdx.x; j <= T; j += 256) {
    const unsigned a = j == 0 ? 0u : positions[lo + j - 1];
    const unsigned e = j == T ? total : positions[lo + j];
    o[j] = e - a;
  }
}

// ---- compressed strings.  Run j of an instance is stored as the signed delta
// x = cnts[j] - cnts[j-2] (cnts[j] itself for j <= 2) in little-endian 5-bit groups, each written
// as the character '0' + group, with 0x20 added to every group but the last; the last group's bit
// 0x10 is the sign.  x needs bits(x ^ (x >> 63)) + 1 bits in two's complement, so
// (bits + 5) / 5 characters: 1 to 7 for run lengths below 2^32.
constexpr int kStrThreads = 256;

__device__ __forceinline__ long long run_delta(const unsigned int *cnts, long long j) {
  long long x = cnts[j];
  if (j > 2) x -= cnts[j - 2];
  return x;
}

__device__ __forceinline__ int delta_chars(long long x) {
  return (64 - __clzll(x ^ (x >> 63)) + 5) / 5;
}

// kept instance k of image b: its runs (cnts, m of them), as rle_counts_kernel wrote them
struct InstRuns {
  const unsigned int *cnts;
  long long m;
};

__device__ __forceinline__ InstRuns inst_runs(const unsigned int *runs, const long long *inst_off,
                                              size_t inst) {
  const long long lo = inst_off[inst];
  return {runs + lo + inst, inst_off[inst + 1] - lo + 1};
}

// One CTA per instance: length of its string (0 for k >= counts[b]).
__global__ void __launch_bounds__(kStrThreads)
rle_string_count_kernel(const unsigned int *__restrict__ runs,
                        const long long *__restrict__ inst_off,
                        const int *__restrict__ counts_per_image, int R,
                        long long *__restrict__ str_len) {
  __shared__ long long s_warp[kStrThreads / 32];
  const int k = blockIdx.x, b = blockIdx.y;
  const size_t inst = static_cast<size_t>(b) * R + k;
  if (k >= counts_per_image[b]) {
    if (threadIdx.x == 0) str_len[inst] = 0;
    return;
  }
  const InstRuns r = inst_runs(runs, inst_off, inst);
  long long n = 0;
  for (long long j = threadIdx.x; j < r.m; j += kStrThreads) n += delta_chars(run_delta(r.cnts, j));
  long long total;
  block_exclusive_scan<long long, kStrThreads>(n, s_warp, total);
  if (threadIdx.x == 0) str_len[inst] = total;
}

// One CTA per instance, kStrThreads runs per pass: a scan of the pass's character counts places
// every run's characters after those of the runs before it.
__global__ void __launch_bounds__(kStrThreads)
rle_string_write_kernel(const unsigned int *__restrict__ runs,
                        const long long *__restrict__ inst_off,
                        const int *__restrict__ counts_per_image, int R,
                        const long long *__restrict__ str_off, unsigned char *__restrict__ str) {
  __shared__ int s_warp[kStrThreads / 32];
  const int k = blockIdx.x, b = blockIdx.y;
  if (k >= counts_per_image[b]) return;
  const size_t inst = static_cast<size_t>(b) * R + k;
  const InstRuns r = inst_runs(runs, inst_off, inst);
  unsigned char *o = str + str_off[inst];
  for (long long base = 0; base < r.m; base += kStrThreads) {
    const long long j = base + threadIdx.x;
    long long x = 0;
    int n = 0;
    if (j < r.m) {
      x = run_delta(r.cnts, j);
      n = delta_chars(x);
    }
    int pass;
    const int at = block_exclusive_scan<int, kStrThreads>(n, s_warp, pass);
    for (int c = 0; c < n; ++c) {
      const int g = static_cast<int>(x & 0x1f);
      x >>= 5;
      o[at + c] = static_cast<unsigned char>('0' + (c + 1 < n ? g | 0x20 : g));
    }
    o += pass;
  }
}

}  // namespace rle

}  // namespace mrx

using namespace mrx;

extern "C" int mrx_rle_count(const float *d_tiles, const int *d_tile_index, const int *d_boxes,
                             const int *d_counts, const int *d_geom, int *d_col_count,
                             long long *d_inst_off, int B, int R, int mh, int mw, int max_w,
                             void *stream) {
  const TileBatch t{d_tiles, d_tile_index, reinterpret_cast<const int4 *>(d_boxes), d_counts,
                    d_geom, B, R, mh, mw};
  if (int rc = check_tile_batch("mrx_rle_count", t, MRX_MAX_LANE_MASK_W)) return rc;
  MRX_CHECK_ARG(d_col_count && d_inst_off && max_w >= 1,
                "mrx_rle_count: null pointer or max_w %d < 1", max_w);
  if (B == 0) return MRX_OK;
  const rle::RleParams prm{t, d_col_count, d_inst_off, nullptr, max_w};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int cblocks = (max_w + 31) >> 5;
  dim3 grid((cblocks + rle::kWalkWarps - 1) / rle::kWalkWarps, R, B);
  rle::rle_walk_kernel<false><<<grid, rle::kWalkWarps * 32, 0, st>>>(prm);
  MRX_LAUNCH_CHECK("rle_walk_kernel<count>");
  rle::rle_scan_kernel<<<dim3(R, B), 256, 0, st>>>(prm);
  MRX_LAUNCH_CHECK("rle_scan_kernel");
  return launch_offsets_scan(d_inst_off, B * R, st);
}

extern "C" int mrx_rle_write(const float *d_tiles, const int *d_tile_index, const int *d_boxes,
                             const int *d_counts, const int *d_geom, int *d_col_count,
                             long long *d_inst_off, unsigned int *d_positions,
                             unsigned int *d_run_lengths, int B, int R, int mh, int mw, int max_w,
                             void *stream) {
  const TileBatch t{d_tiles, d_tile_index, reinterpret_cast<const int4 *>(d_boxes), d_counts,
                    d_geom, B, R, mh, mw};
  if (int rc = check_tile_batch("mrx_rle_write", t, MRX_MAX_LANE_MASK_W)) return rc;
  MRX_CHECK_ARG(d_col_count && d_inst_off && d_positions && d_run_lengths && max_w >= 1,
                "mrx_rle_write: null pointer or max_w %d < 1", max_w);
  if (B == 0) return MRX_OK;
  const rle::RleParams prm{t, d_col_count, d_inst_off, d_positions, max_w};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int cblocks = (max_w + 31) >> 5;
  dim3 grid((cblocks + rle::kWalkWarps - 1) / rle::kWalkWarps, R, B);
  rle::rle_walk_kernel<true><<<grid, rle::kWalkWarps * 32, 0, st>>>(prm);
  MRX_LAUNCH_CHECK("rle_walk_kernel<write>");
  rle::rle_counts_kernel<<<dim3(R, B), 256, 0, st>>>(d_positions, d_inst_off, d_counts, d_geom, R,
                                                     d_run_lengths);
  MRX_LAUNCH_CHECK("rle_counts_kernel");
  return MRX_OK;
}

extern "C" int mrx_rle_strings(const unsigned int *d_run_lengths, const long long *d_inst_off,
                               const int *d_counts, int B, int R, long long *d_str_off,
                               unsigned char *d_str, void *stream) {
  MRX_CHECK_ARG(d_run_lengths && d_inst_off && d_counts && d_str_off && d_str,
                "mrx_rle_strings: null pointer");
  MRX_CHECK_ARG(B >= 0 && B <= MRX_MAX_BATCH && R >= 1 && R <= 65534,
                "mrx_rle_strings: bad sizes B=%d R=%d (need 0<=B<=%d, 1<=R<=65534)", B, R,
                MRX_MAX_BATCH);
  if (B == 0) return MRX_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  rle::rle_string_count_kernel<<<dim3(R, B), rle::kStrThreads, 0, st>>>(
      d_run_lengths, d_inst_off, d_counts, R, d_str_off);
  MRX_LAUNCH_CHECK("rle_string_count_kernel");
  if (int rc = launch_offsets_scan(d_str_off, B * R, st)) return rc;
  rle::rle_string_write_kernel<<<dim3(R, B), rle::kStrThreads, 0, st>>>(
      d_run_lengths, d_inst_off, d_counts, R, d_str_off, d_str);
  MRX_LAUNCH_CHECK("rle_string_write_kernel");
  return MRX_OK;
}
