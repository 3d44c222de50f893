// overlaps.cu -- scoring predicted masks against ground truth on the packed planes: upstream's
// compute_overlaps_masks (mask IoU) and the matching loop of compute_matches (mrcnn/utils.py).
//
// Input: bit-packed planes as mrx_pack_masks / mrx_mask_expand_packed write them (planes.cuh).
//
//   mask_extents_kernel  CTA per plane: popcount area and tight extent inside a region, warps on
//                        rows, lanes on bytes
//   mask_overlaps_kernel CTA per (image, prediction), warp per ground-truth instance: every pair
//                        through walk_pairs (planes.cuh), so a pair whose extents do not meet (or
//                        with an empty mask) gets its IoU without a read
//   mask_rank_kernel     CTA per image: rank of every prediction by score (descending, NaN first,
//                        ties larger index first), by counting
//   mask_match_kernel    warp per (image, threshold): predictions in rank order, each takes the
//                        best unmatched candidate of its class (an argmax over the warp)
//
// IoU arithmetic is NumPy's float32 order: i = f32(inter), u = (f32(a1) + f32(a2)) - i, i / u,
// each rounded once (exact counts; bit-equal to NumPy while H*W <= 2^24).
#include <climits>

#include "planes.cuh"

namespace mrx {

namespace overlaps {

constexpr int kWarps = 8;

// ---------------------------------------------------------------- extents
__global__ void __launch_bounds__(kWarps * 32)
mask_extents_kernel(Slots<const unsigned char> packed, const int *__restrict__ counts,
                    const int *__restrict__ geom, const int4 *__restrict__ regions,
                    long long *__restrict__ areas, int4 *__restrict__ extents, int R) {
  const int k = blockIdx.x, b = blockIdx.y;
  if (k >= counts[b]) return;
  const int H = geom[b * MRX_GEOM_INTS + 0], W = geom[b * MRX_GEOM_INTS + 1];
  const int wb = (W + 7) >> 3;
  const int4 r = regions[static_cast<size_t>(b) * R + k];
  const int y1 = max(r.x, 0), x1 = max(r.y, 0), y2 = min(r.z, H), x2 = min(r.w, W);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long area = 0;
  int ymin = INT_MAX, xmin = INT_MAX, ymax = -1, xmax = -1;
  if (y2 > y1 && x2 > x1) {
    const unsigned char *plane = plane_of(packed, b, k, H, wb);
    const int jb0 = x1 >> 3, jb1 = (x2 - 1) >> 3;
    for (int y = y1 + warp; y < y2; y += kWarps) {
      const unsigned char *row = plane + static_cast<long long>(y) * wb;
      for (int j = jb0 + lane; j <= jb1; j += 32) {
        // pixels [x1, x2) of byte j: bit 7 - t is pixel 8j + t
        const int lo = max(x1 - 8 * j, 0), hi = min(x2 - 8 * j, 8);
        const unsigned v = __ldg(row + j) & (0xFFu >> lo) & (0xFFu << (8 - hi));
        if (v) {
          area += __popc(v);
          ymin = min(ymin, y);
          ymax = max(ymax, y);
          xmin = min(xmin, 8 * j + __clz(v) - 24);
          xmax = max(xmax, 8 * j + 8 - __ffs(v));
        }
      }
    }
  }
  area = warp_sum(area);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ymin = min(ymin, __shfl_xor_sync(0xffffffffu, ymin, o));
    xmin = min(xmin, __shfl_xor_sync(0xffffffffu, xmin, o));
    ymax = max(ymax, __shfl_xor_sync(0xffffffffu, ymax, o));
    xmax = max(xmax, __shfl_xor_sync(0xffffffffu, xmax, o));
  }
  __shared__ long long s_area[kWarps];
  __shared__ int4 s_ext[kWarps];
  if (lane == 0) {
    s_area[warp] = area;
    s_ext[warp] = make_int4(ymin, xmin, ymax, xmax);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    long long a = 0;
    int4 e = make_int4(INT_MAX, INT_MAX, -1, -1);
    for (int w = 0; w < kWarps; ++w) {
      a += s_area[w];
      e = make_int4(min(e.x, s_ext[w].x), min(e.y, s_ext[w].y), max(e.z, s_ext[w].z),
                    max(e.w, s_ext[w].w));
    }
    const size_t i = static_cast<size_t>(b) * R + k;
    areas[i] = a;
    extents[i] = a ? make_int4(e.x, e.y, e.z + 1, e.w + 1) : make_int4(0, 0, 0, 0);
  }
}

// ---------------------------------------------------------------- overlaps
__global__ void __launch_bounds__(kWarps * 32)
mask_overlaps_kernel(const Planes p1, const Planes p2, const int *__restrict__ geom,
                     float *__restrict__ out) {
  const int i = blockIdx.x, b = blockIdx.y;
  if (i >= p1.counts[b]) return;
  float *row = out + (static_cast<size_t>(b) * p1.R + i) * p2.R;
  walk_pairs<kWarps>(
      p1, p2, geom, b, i, [](int) { return true; },
      [&](int j, long long inter, long long a1, long long a2) {
        const float fi = __ll2float_rn(inter);
        const float u = __fsub_rn(__fadd_rn(__ll2float_rn(a1), __ll2float_rn(a2)), fi);
        row[j] = __fdiv_rn(fi, u);   // 0 / 0 = NaN: both masks empty
      });
}

// ---------------------------------------------------------------- ranks and matches
struct MatchParams {
  const float *overlaps;      // [B, R1, R2]
  const int *pred_counts;     // [B]
  const int *pred_class;      // [B, R1]
  const void *scores;         // [B, R1] f32 / f64
  const int *gt_counts;       // [B]
  const int *gt_class;        // [B, R2]
  int *order;                 // [B, R1]
  int *pred_match;            // [T, B, R1]
  int *gt_match;              // [T, B, R2]
  int B, R1, R2, score_f64;
  double score_threshold;
  double thresholds[MRX_MAX_IOU_THRESHOLDS];
};

// rank of prediction i = the predictions before it: higher score, NaN above every number, equal
// scores by larger index (np.argsort(kind="stable")[::-1])
__global__ void __launch_bounds__(256) mask_rank_kernel(const MatchParams p) {
  const int b = blockIdx.x;
  const int N = p.pred_counts[b];
  const size_t base = static_cast<size_t>(b) * p.R1;
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    const double si = score_at(p.scores, p.score_f64, base + i);
    const bool ni = isnan(si);
    int rank = 0;
    for (int k = 0; k < N; ++k) {
      const double sk = score_at(p.scores, p.score_f64, base + k);
      const bool nk = isnan(sk);
      const bool tie = (nk && ni) || sk == si;
      rank += (nk && !ni) || (!nk && !ni && sk > si) || (tie && k > i);
    }
    p.order[base + rank] = i;
  }
}

// Prediction i (rank order) matches the first ground-truth instance j of np.argsort(overlaps[i])
// reversed (stable: NaN first, ties larger j first) that is unmatched, of i's class, and whose IoU
// is NaN or at least both thresholds.  Lane j % 32 owns gt_match[j].
__global__ void __launch_bounds__(32) mask_match_kernel(const MatchParams p) {
  const int b = blockIdx.x, t = blockIdx.y, lane = threadIdx.x;
  const int N = p.pred_counts[b], M = p.gt_counts[b];
  const double thr = p.thresholds[t], sthr = p.score_threshold;
  int *gm = p.gt_match + (static_cast<size_t>(t) * p.B + b) * p.R2;
  int *pm = p.pred_match + (static_cast<size_t>(t) * p.B + b) * p.R1;
  const int *gcls = p.gt_class + static_cast<size_t>(b) * p.R2;
  for (int j = lane; j < M; j += 32) gm[j] = -1;
  for (int r = 0; r < N; ++r) {
    const int i = p.order[static_cast<size_t>(b) * p.R1 + r];
    const int ci = p.pred_class[static_cast<size_t>(b) * p.R1 + i];
    const float *row = p.overlaps + (static_cast<size_t>(b) * p.R1 + i) * p.R2;
    // key: 2 = NaN above 1 = a number (its bits order like its value, IoU >= +0), then j
    unsigned long long best = 0ull;
    for (int j = lane; j < M; j += 32) {
      if (gm[j] != -1 || gcls[j] != ci) continue;
      const float v = row[j];
      unsigned long long key = 0ull;
      if (isnan(v))
        key = (2ull << 62) | static_cast<unsigned>(j);
      else if (static_cast<double>(v) >= thr && static_cast<double>(v) >= sthr)
        key = (1ull << 62) | (static_cast<unsigned long long>(__float_as_uint(v)) << 16) |
              static_cast<unsigned>(j);
      best = key > best ? key : best;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long x = __shfl_xor_sync(0xffffffffu, best, o);
      best = x > best ? x : best;
    }
    const int j = best ? static_cast<int>(best & 0xFFFFu) : -1;
    if (j >= 0 && lane == (j & 31)) gm[j] = r;
    if (lane == 0) pm[r] = j;
  }
}

}  // namespace overlaps

}  // namespace mrx

using namespace mrx;

extern "C" int mrx_mask_extents(const unsigned char *d_packed, const long long *d_packed_off,
                                const int *d_counts, const int *d_geom, const int *d_regions,
                                long long *d_areas, int *d_extents, int B, int R, void *stream) {
  const char *fn = "mrx_mask_extents";
  if (int rc = check_slots(fn, d_packed, d_packed_off, d_counts, d_geom, B, R)) return rc;
  MRX_CHECK_ARG(d_regions, "%s: the region argument d_regions is required", fn);
  MRX_CHECK_ARG(d_areas && d_extents, "%s: null pointer", fn);
  if (B == 0) return MRX_OK;
  overlaps::mask_extents_kernel<<<dim3(R, B), overlaps::kWarps * 32, 0,
                                  static_cast<cudaStream_t>(stream)>>>(
      {d_packed, d_packed_off}, d_counts, d_geom, reinterpret_cast<const int4 *>(d_regions),
      d_areas, reinterpret_cast<int4 *>(d_extents), R);
  MRX_LAUNCH_CHECK("mask_extents_kernel");
  return MRX_OK;
}

extern "C" int mrx_mask_overlaps(const unsigned char *d_packed1, const long long *d_packed_off1,
                                 const int *d_counts1, const long long *d_areas1,
                                 const int *d_extents1, int R1,
                                 const unsigned char *d_packed2, const long long *d_packed_off2,
                                 const int *d_counts2, const long long *d_areas2,
                                 const int *d_extents2, int R2, const int *d_geom,
                                 float *d_overlaps, int B, void *stream) {
  overlaps::Planes p1, p2;
  if (int rc = overlaps::check_plane_pair("mrx_mask_overlaps", d_packed1, d_packed_off1, d_counts1,
                                          d_areas1, d_extents1, R1, d_packed2, d_packed_off2,
                                          d_counts2, d_areas2, d_extents2, R2, d_geom, B,
                                          d_overlaps != nullptr, p1, p2))
    return rc;
  if (B == 0) return MRX_OK;
  overlaps::mask_overlaps_kernel<<<dim3(R1, B), overlaps::kWarps * 32, 0,
                                   static_cast<cudaStream_t>(stream)>>>(p1, p2, d_geom, d_overlaps);
  MRX_LAUNCH_CHECK("mask_overlaps_kernel");
  return MRX_OK;
}

extern "C" int mrx_mask_matches(const float *d_overlaps, const int *d_pred_counts,
                                const int *d_pred_class_ids, const void *d_scores, int score_dtype,
                                const int *d_gt_counts, const int *d_gt_class_ids,
                                const double *thresholds, int T, double score_threshold,
                                int *d_order, int *d_pred_match, int *d_gt_match, int B, int R1,
                                int R2, void *stream) {
  const char *fn = "mrx_mask_matches";
  MRX_CHECK_ARG(d_overlaps && d_pred_counts && d_pred_class_ids && d_scores && d_gt_counts &&
                    d_gt_class_ids && thresholds && d_order && d_pred_match && d_gt_match,
                "%s: null pointer", fn);
  MRX_CHECK_ARG(B >= 0 && B <= MRX_MAX_BATCH, "%s: bad B %d (need 0<=B<=%d)", fn, B, MRX_MAX_BATCH);
  MRX_CHECK_ARG(R1 >= 1 && R1 <= 65534 && R2 >= 1 && R2 <= 65534,
                "%s: bad R1 %d / R2 %d (need 1<=R<=65534)", fn, R1, R2);
  MRX_CHECK_ARG(T >= 1 && T <= MRX_MAX_IOU_THRESHOLDS, "%s: bad T %d (need 1<=T<=%d)", fn, T,
                MRX_MAX_IOU_THRESHOLDS);
  MRX_CHECK_ARG(score_dtype == MRX_F32 || score_dtype == MRX_F64, "%s: bad score dtype %d", fn,
                score_dtype);
  if (B == 0) return MRX_OK;
  overlaps::MatchParams p{};
  p.overlaps = d_overlaps;
  p.pred_counts = d_pred_counts;
  p.pred_class = d_pred_class_ids;
  p.scores = d_scores;
  p.gt_counts = d_gt_counts;
  p.gt_class = d_gt_class_ids;
  p.order = d_order;
  p.pred_match = d_pred_match;
  p.gt_match = d_gt_match;
  p.B = B;
  p.R1 = R1;
  p.R2 = R2;
  p.score_f64 = score_dtype == MRX_F64;
  p.score_threshold = score_threshold;
  for (int t = 0; t < T; ++t) p.thresholds[t] = thresholds[t];
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  overlaps::mask_rank_kernel<<<B, 256, 0, st>>>(p);
  MRX_LAUNCH_CHECK("mask_rank_kernel");
  overlaps::mask_match_kernel<<<dim3(B, T), 32, 0, st>>>(p);
  MRX_LAUNCH_CHECK("mask_match_kernel");
  return MRX_OK;
}
