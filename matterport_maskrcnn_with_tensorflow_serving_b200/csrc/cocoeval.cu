// cocoeval.cu -- the per-image half of pycocotools' COCOeval: computeIoU for iouType "segm" on the
// packed planes (maskApi.c rleIou), for "boundary" (boundary_iou_api) on the packed planes and
// their boundary planes (boundary.cu), and for "bbox" on [x, y, w, h] boxes (bbIou), and the
// matching loop of evaluateImg, which does not care where its IoUs come from.  The host keeps what
// accumulate needs: per detection its category, rank, score, area and match / ignore bits.
//
//   coco_rank_kernel   CTA per image: each prediction's dense category (through a class map),
//                      its rank within (image, category) in np.argsort(-score, kind="mergesort")
//                      order (descending, ties smaller index first, NaN last), whether that rank
//                      is below maxDets[-1], and the image's walk order (the same order across
//                      categories), by counting
//   lvis_rank_kernel   the same counting loop (rank_image, one template over the keep rule) for
//                      lvis-api's LVISEval: cat, rank and walk as above, but kept is whether the
//                      walk position is below max_dets (LVISResults' per-image cut over every
//                      result) and the category is positive or negative for the image (the
//                      federated filter of LVISEval._prepare, a [B, K] status table)
//   coco_iou_kernel    CTA per (image, prediction), warp per ground-truth instance: the pair walk
//                      of mask_overlaps_kernel (walk_pairs, planes.cuh) over the pairs of one
//                      category whose prediction is kept; a pair whose extents do not meet gets 0
//                      without a read
//   coco_boundary_iou_kernel the same grid and walk counting each pair's masks and boundaries
//                      together (walk_boundary_pairs), writing the smaller of the two IoUs
//   coco_box_iou_kernel CTA per (image, prediction), thread per ground-truth instance: bbIou of
//                      the pairs of one category whose prediction is kept, and the prediction's
//                      area w*h (loadRes' area of a bbox result)
//   coco_match_kernel  warp per (image, threshold, area range): predictions in walk order, each
//                      takes the argmax of (not ignored, IoU, position) over its candidates; one
//                      template over the detection area's type (mask pixels, or box w*h)
//
// Mask IoU arithmetic is rleIou's: (double)i / (double)u of exact counts, 0 when i = 0, u = the
// detection's area for a crowd instance and a_dt + a_gt - i otherwise.  Box IoU arithmetic is
// bbIou's, operation for operation and unfused (see coco_box_iou_kernel).
#include "planes.cuh"

namespace mrx {

namespace cocoeval {

using overlaps::Planes;
using overlaps::score_at;
using overlaps::walk_boundary_pairs;
using overlaps::walk_pairs;

constexpr int kWarps = 8;

// ---------------------------------------------------------------- ranks
struct RankParams {
  const int *class_ids;       // [B, R]
  const void *scores;         // [B, R] f32 / f64
  const int *counts;          // [B]
  const int *class_map;       // [C]
  int *cat;                   // [B, R]
  int *rank;                  // [B, R]
  unsigned char *keep;        // [B, R]
  int *walk;                  // [B, R]
  int R, C, score_f64, max_det;
};

// k comes before i in np.argsort(-score, kind="mergesort"): numbers before NaN, higher scores
// first, equal scores (and NaN among NaN) by index
__device__ __forceinline__ bool before(double sk, int k, double si, int i) {
  const bool nk = isnan(sk), ni = isnan(si);
  if (nk != ni) return ni;
  if (!nk && sk != si) return sk > si;
  return k < i;
}

// COCOeval's maxDets cut: the first maxDets[-1] of each (image, category)
struct CocoKeep {
  __device__ __forceinline__ bool operator()(const RankParams &p, int, int ci, int rank,
                                             int) const {
    return ci >= 0 && rank < p.max_det;
  }
};

// LVISEval's: the first max_dets of the image across every category (walk counts them all,
// categories that are not evaluated included), then only categories positive or negative for it
struct LvisKeep {
  const unsigned char *status;  // [B, K]
  int K;
  __device__ __forceinline__ bool operator()(const RankParams &p, int b, int ci, int,
                                             int walk) const {
    return ci >= 0 && ci < K && walk < p.max_det &&
           (status[static_cast<size_t>(b) * K + ci] & MRX_LVIS_EVALUATED);
  }
};

// one CTA's image b: every prediction's dense category, then its rank within (image, category)
// and its walk position by counting the predictions before it
template <typename Keep>
__device__ __forceinline__ void rank_image(const RankParams &p, const Keep keep) {
  const int b = blockIdx.x;
  const int N = p.counts[b];
  const size_t base = static_cast<size_t>(b) * p.R;
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    const int c = p.class_ids[base + i];
    const int k = c >= 0 && c < p.C ? p.class_map[c] : -1;
    p.cat[base + i] = k < 0 ? -1 : k;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    const double si = score_at(p.scores, p.score_f64, base + i);
    const int ci = p.cat[base + i];
    int rank = 0, walk = 0;
    for (int k = 0; k < N; ++k) {
      const bool bf = before(score_at(p.scores, p.score_f64, base + k), k, si, i);
      walk += bf;
      rank += bf && p.cat[base + k] == ci;
    }
    p.rank[base + i] = rank;
    p.keep[base + i] = keep(p, b, ci, rank, walk);
    p.walk[base + walk] = i;
  }
}

__global__ void __launch_bounds__(256) coco_rank_kernel(const RankParams p) {
  rank_image(p, CocoKeep{});
}

__global__ void __launch_bounds__(256) lvis_rank_kernel(const RankParams p,
                                                        const unsigned char *__restrict__ status,
                                                        int K) {
  rank_image(p, LvisKeep{status, K});
}

// ---------------------------------------------------------------- IoUs
// rleIou of one pair from exact counts: 0 when inter = 0, else inter / u rounded once, u the
// detection's area a1 for a crowd instance and a1 + a2 - inter otherwise
__device__ __forceinline__ double rle_iou(long long inter, long long a1, long long a2, bool crowd) {
  const long long u = crowd ? a1 : a1 + a2 - inter;
  return inter ? __ddiv_rn(static_cast<double>(inter), static_cast<double>(u)) : 0.0;
}

__global__ void __launch_bounds__(kWarps * 32)
coco_iou_kernel(const Planes p1, const Planes p2, const int *__restrict__ geom,
                const int *__restrict__ pred_cat, const unsigned char *__restrict__ pred_keep,
                const int *__restrict__ gt_cat, const unsigned char *__restrict__ gt_crowd,
                double *__restrict__ out) {
  const int i = blockIdx.x, b = blockIdx.y;
  if (i >= p1.counts[b]) return;
  const size_t i1 = static_cast<size_t>(b) * p1.R + i;
  if (!pred_keep[i1]) return;
  const int ci = pred_cat[i1];
  const size_t gb = static_cast<size_t>(b) * p2.R;
  double *row = out + i1 * p2.R;
  walk_pairs<kWarps>(
      p1, p2, geom, b, i, [&](int j) { return gt_cat[gb + j] == ci; },
      [&](int j, long long inter, long long a1, long long a2) {
        row[j] = rle_iou(inter, a1, a2, gt_crowd[gb + j]);
      });
}

// computeIoU for "boundary": np.minimum of rleIou on the masks and rleIou on the boundaries, both
// with the crowd rule, from one walk over both pairs (q1, q2: the boundary planes of p1, p2)
__global__ void __launch_bounds__(kWarps * 32)
coco_boundary_iou_kernel(const Planes p1, const Planes p2, const Planes q1, const Planes q2,
                         const int *__restrict__ geom, const int *__restrict__ pred_cat,
                         const unsigned char *__restrict__ pred_keep,
                         const int *__restrict__ gt_cat, const unsigned char *__restrict__ gt_crowd,
                         double *__restrict__ out) {
  const int i = blockIdx.x, b = blockIdx.y;
  if (i >= p1.counts[b]) return;
  const size_t i1 = static_cast<size_t>(b) * p1.R + i;
  if (!pred_keep[i1]) return;
  const int ci = pred_cat[i1];
  const size_t gb = static_cast<size_t>(b) * p2.R;
  double *row = out + i1 * p2.R;
  walk_boundary_pairs<kWarps>(
      p1, p2, q1, q2, geom, b, i, [&](int j) { return gt_cat[gb + j] == ci; },
      [&](int j, long long inter, long long a1, long long a2, long long binter, long long ba1,
          long long ba2) {
        const bool crowd = gt_crowd[gb + j];
        row[j] = fmin(rle_iou(inter, a1, a2, crowd), rle_iou(binter, ba1, ba2, crowd));
      });
}

constexpr int kBoxThreads = 128;

struct BoxIouParams {
  const void *pred_boxes;     // [B, R1, 4] int32 (y1, x1, y2, x2) or float64 (x, y, w, h)
  const int *pred_counts;     // [B]
  const int *pred_cat;        // [B, R1]
  const unsigned char *pred_keep;
  const double *gt_boxes;     // [B, R2, 4] (x, y, w, h)
  const int *gt_counts;       // [B]
  const int *gt_cat;          // [B, R2]
  const unsigned char *gt_crowd;
  double *pred_area;          // [B, R1]
  double *iou;                // [B, R1, R2]
  int R1, R2, pred_xywh;
};

// maskApi.c bbIou for one prediction against every instance of its category.  pycocotools' x86-64
// build rounds every operation; nvcc would contract w*h into da + ga - w*h (an FMA), so each one is
// an explicit _rn intrinsic.  An engine box becomes [x1, y1, x2 - x1, y2 - y1] exactly (int32
// differences are exact in double), the `bbox` of build_coco_results.
__global__ void __launch_bounds__(kBoxThreads) coco_box_iou_kernel(const BoxIouParams p) {
  const int i = blockIdx.x, b = blockIdx.y;
  if (i >= p.pred_counts[b]) return;
  const size_t i1 = static_cast<size_t>(b) * p.R1 + i;
  if (!p.pred_keep[i1]) return;
  double d[4];
  if (p.pred_xywh) {
    const double *q = static_cast<const double *>(p.pred_boxes) + 4 * i1;
    for (int k = 0; k < 4; ++k) d[k] = q[k];
  } else {
    const int *q = static_cast<const int *>(p.pred_boxes) + 4 * i1;
    d[0] = q[1];
    d[1] = q[0];
    d[2] = __dsub_rn(q[3], q[1]);
    d[3] = __dsub_rn(q[2], q[0]);
  }
  const double da = __dmul_rn(d[2], d[3]);
  if (threadIdx.x == 0) p.pred_area[i1] = da;
  const int ci = p.pred_cat[i1];
  const int M = p.gt_counts[b];
  const size_t gb = static_cast<size_t>(b) * p.R2;
  double *row = p.iou + i1 * p.R2;
  for (int j = threadIdx.x; j < M; j += blockDim.x) {
    if (p.gt_cat[gb + j] != ci) continue;
    const double *g = p.gt_boxes + 4 * (gb + j);
    double o = 0.0;
    const double w = __dsub_rn(fmin(__dadd_rn(d[2], d[0]), __dadd_rn(g[2], g[0])), fmax(d[0], g[0]));
    if (!(w <= 0)) {
      const double h =
          __dsub_rn(fmin(__dadd_rn(d[3], d[1]), __dadd_rn(g[3], g[1])), fmax(d[1], g[1]));
      if (!(h <= 0)) {
        const double inter = __dmul_rn(w, h);
        const double u =
            p.gt_crowd[gb + j] ? da : __dsub_rn(__dadd_rn(da, __dmul_rn(g[2], g[3])), inter);
        o = __ddiv_rn(inter, u);
      }
    }
    row[j] = o;
  }
}

// ---------------------------------------------------------------- matches
template <typename Area>
struct MatchParams {
  const double *iou;          // [B, R1, R2]
  const int *pred_counts;     // [B]
  const int *pred_cat;        // [B, R1]
  const unsigned char *pred_keep;
  const int *walk;            // [B, R1]
  const Area *pred_area;      // [B, R1]: mask pixels (int64) or box w*h (float64)
  const int *gt_counts;       // [B]
  const int *gt_cat;          // [B, R2]
  const unsigned char *gt_crowd;
  const double *gt_area;      // [B, R2]
  int *dt_match;              // [A, T, B, R1]
  unsigned char *dt_ignore;   // [A, T, B, R1]
  int B, R1, R2, T;
  double thresholds[MRX_MAX_IOU_THRESHOLDS];
  double area_rng[2 * MRX_MAX_AREA_RANGES];
};

// evaluateImg's loop in closed form: the candidates of a prediction are the instances of its
// category that are unmatched (or crowd) with IoU >= the threshold; it takes the non-ignored one
// with the largest IoU, else the ignored one with the largest IoU, ties going to the later one of
// the ground truth stable-sorted with the non-ignored first -- within each of the two groups that
// order is the index order, so the key is (not ignored, IoU bits, then j).  Lane j % 32 scans
// instance j; the matched set is a bitmask in shared memory, written by the one winning lane.
template <typename Area>
__global__ void __launch_bounds__(32) coco_match_kernel(const MatchParams<Area> p) {
  __shared__ unsigned s_matched[(65534 + 31) / 32];
  const int b = blockIdx.x, t = blockIdx.y, a = blockIdx.z, lane = threadIdx.x;
  const int N = p.pred_counts[b], M = p.gt_counts[b];
  const double thr = p.thresholds[t], lo = p.area_rng[2 * a], hi = p.area_rng[2 * a + 1];
  const size_t pb = static_cast<size_t>(b) * p.R1, gb = static_cast<size_t>(b) * p.R2;
  const size_t ob = (static_cast<size_t>(a) * p.T + t) * p.B * p.R1 + pb;
  for (int w = lane; w < (M + 31) / 32; w += 32) s_matched[w] = 0u;
  __syncwarp();
  for (int r = 0; r < N; ++r) {
    const int i = p.walk[pb + r];
    if (!p.pred_keep[pb + i]) continue;
    const int ci = p.pred_cat[pb + i];
    const double *row = p.iou + (pb + i) * p.R2;
    unsigned long long best = 0ull;
    int bj = -1;
    for (int j = lane; j < M; j += 32) {
      if (p.gt_cat[gb + j] != ci) continue;
      const bool crowd = p.gt_crowd[gb + j];
      if (!crowd && (s_matched[j >> 5] >> (j & 31) & 1u)) continue;
      const double v = row[j];
      if (!(v >= thr)) continue;
      const double ga = p.gt_area[gb + j];
      const bool ig = crowd || ga < lo || ga > hi;
      const unsigned long long key =
          (ig ? 0ull : 1ull << 62) | static_cast<unsigned long long>(__double_as_longlong(v));
      if (key >= best || bj < 0) {
        best = key;
        bj = j;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long ok = __shfl_xor_sync(0xffffffffu, best, o);
      const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
      if (oj >= 0 && (bj < 0 || ok > best || (ok == best && oj > bj))) {
        best = ok;
        bj = oj;
      }
    }
    if (bj >= 0 && lane == (bj & 31)) s_matched[bj >> 5] |= 1u << (bj & 31);
    if (lane == 0) {
      bool ig;
      if (bj >= 0) {
        ig = !(best >> 62);
      } else {
        const double da = static_cast<double>(p.pred_area[pb + i]);
        ig = da < lo || da > hi;
      }
      p.dt_match[ob + i] = bj;
      p.dt_ignore[ob + i] = ig;
    }
    __syncwarp();
  }
}

}  // namespace cocoeval

}  // namespace mrx

using namespace mrx;

extern "C" int mrx_coco_ranks(const int *d_class_ids, const void *d_scores, int score_dtype,
                              const int *d_counts, const int *d_class_map, int C, int max_det,
                              int *d_cat, int *d_rank, unsigned char *d_keep, int *d_walk, int B,
                              int R, void *stream) {
  const char *fn = "mrx_coco_ranks";
  MRX_CHECK_ARG(d_class_ids && d_scores && d_counts && d_class_map && d_cat && d_rank && d_keep &&
                    d_walk,
                "%s: null pointer", fn);
  MRX_CHECK_ARG(B >= 0 && B <= MRX_MAX_BATCH, "%s: bad B %d (need 0<=B<=%d)", fn, B, MRX_MAX_BATCH);
  MRX_CHECK_ARG(R >= 1 && R <= 65534, "%s: bad R %d (need 1<=R<=65534)", fn, R);
  MRX_CHECK_ARG(C >= 1, "%s: bad C %d (need C>=1)", fn, C);
  MRX_CHECK_ARG(max_det >= 1, "%s: bad max_det %d (need max_det>=1)", fn, max_det);
  MRX_CHECK_ARG(score_dtype == MRX_F32 || score_dtype == MRX_F64, "%s: bad score dtype %d", fn,
                score_dtype);
  if (B == 0) return MRX_OK;
  const cocoeval::RankParams p{d_class_ids, d_scores, d_counts, d_class_map, d_cat, d_rank,
                               d_keep,      d_walk,   R,        C,           score_dtype == MRX_F64,
                               max_det};
  cocoeval::coco_rank_kernel<<<B, 256, 0, static_cast<cudaStream_t>(stream)>>>(p);
  MRX_LAUNCH_CHECK("coco_rank_kernel");
  return MRX_OK;
}

extern "C" int mrx_lvis_ranks(const int *d_class_ids, const void *d_scores, int score_dtype,
                              const int *d_counts, const int *d_class_map, int C,
                              const unsigned char *d_status, int K, int max_det, int *d_cat,
                              int *d_rank, unsigned char *d_keep, int *d_walk, int B, int R,
                              void *stream) {
  const char *fn = "mrx_lvis_ranks";
  MRX_CHECK_ARG(d_class_ids && d_scores && d_counts && d_class_map && d_status && d_cat && d_rank &&
                    d_keep && d_walk,
                "%s: null pointer", fn);
  MRX_CHECK_ARG(B >= 0 && B <= MRX_MAX_BATCH, "%s: bad B %d (need 0<=B<=%d)", fn, B, MRX_MAX_BATCH);
  MRX_CHECK_ARG(R >= 1 && R <= 65534, "%s: bad R %d (need 1<=R<=65534)", fn, R);
  MRX_CHECK_ARG(C >= 1, "%s: bad C %d (need C>=1)", fn, C);
  MRX_CHECK_ARG(K >= 1, "%s: bad K %d (need K>=1)", fn, K);
  MRX_CHECK_ARG(max_det >= 1, "%s: bad max_det %d (need max_det>=1)", fn, max_det);
  MRX_CHECK_ARG(score_dtype == MRX_F32 || score_dtype == MRX_F64, "%s: bad score dtype %d", fn,
                score_dtype);
  if (B == 0) return MRX_OK;
  const cocoeval::RankParams p{d_class_ids, d_scores, d_counts, d_class_map, d_cat, d_rank,
                               d_keep,      d_walk,   R,        C,           score_dtype == MRX_F64,
                               max_det};
  cocoeval::lvis_rank_kernel<<<B, 256, 0, static_cast<cudaStream_t>(stream)>>>(p, d_status, K);
  MRX_LAUNCH_CHECK("lvis_rank_kernel");
  return MRX_OK;
}

extern "C" int mrx_coco_ious(const unsigned char *d_packed1, const long long *d_packed_off1,
                             const int *d_counts1, const long long *d_areas1,
                             const int *d_extents1, const int *d_pred_cat,
                             const unsigned char *d_pred_keep, int R1,
                             const unsigned char *d_packed2, const long long *d_packed_off2,
                             const int *d_counts2, const long long *d_areas2,
                             const int *d_extents2, const int *d_gt_cat,
                             const unsigned char *d_gt_crowd, int R2, const int *d_geom,
                             double *d_iou, int B, void *stream) {
  overlaps::Planes p1, p2;
  if (int rc = overlaps::check_plane_pair(
          "mrx_coco_ious", d_packed1, d_packed_off1, d_counts1, d_areas1, d_extents1, R1,
          d_packed2, d_packed_off2, d_counts2, d_areas2, d_extents2, R2, d_geom, B,
          d_pred_cat && d_pred_keep && d_gt_cat && d_gt_crowd && d_iou, p1, p2))
    return rc;
  if (B == 0) return MRX_OK;
  cocoeval::coco_iou_kernel<<<dim3(R1, B), cocoeval::kWarps * 32, 0,
                              static_cast<cudaStream_t>(stream)>>>(
      p1, p2, d_geom, d_pred_cat, d_pred_keep, d_gt_cat, d_gt_crowd, d_iou);
  MRX_LAUNCH_CHECK("coco_iou_kernel");
  return MRX_OK;
}

extern "C" int mrx_coco_boundary_ious(
    const unsigned char *d_packed1, const long long *d_packed_off1, const int *d_counts1,
    const long long *d_areas1, const int *d_extents1, const unsigned char *d_boundary1,
    const long long *d_boundary_areas1, const int *d_pred_cat, const unsigned char *d_pred_keep,
    int R1, const unsigned char *d_packed2, const long long *d_packed_off2, const int *d_counts2,
    const long long *d_areas2, const int *d_extents2, const unsigned char *d_boundary2,
    const long long *d_boundary_areas2, const int *d_gt_cat, const unsigned char *d_gt_crowd,
    int R2, const int *d_geom, double *d_iou, int B, void *stream) {
  const char *fn = "mrx_coco_boundary_ious";
  overlaps::Planes p1, p2;
  if (int rc = overlaps::check_plane_pair(
          fn, d_packed1, d_packed_off1, d_counts1, d_areas1, d_extents1, R1, d_packed2,
          d_packed_off2, d_counts2, d_areas2, d_extents2, R2, d_geom, B,
          d_boundary1 && d_boundary_areas1 && d_boundary2 && d_boundary_areas2 && d_pred_cat &&
              d_pred_keep && d_gt_cat && d_gt_crowd && d_iou,
          p1, p2))
    return rc;
  MRX_CHECK_ARG(((reinterpret_cast<uintptr_t>(d_boundary1) |
                  reinterpret_cast<uintptr_t>(d_boundary2)) & 3u) == 0u,
                "%s: boundary bases must be 4-byte aligned", fn);
  if (B == 0) return MRX_OK;
  overlaps::Planes q1 = p1, q2 = p2;
  q1.packed.base = d_boundary1;
  q1.areas = d_boundary_areas1;
  q2.packed.base = d_boundary2;
  q2.areas = d_boundary_areas2;
  cocoeval::coco_boundary_iou_kernel<<<dim3(R1, B), cocoeval::kWarps * 32, 0,
                                       static_cast<cudaStream_t>(stream)>>>(
      p1, p2, q1, q2, d_geom, d_pred_cat, d_pred_keep, d_gt_cat, d_gt_crowd, d_iou);
  MRX_LAUNCH_CHECK("coco_boundary_iou_kernel");
  return MRX_OK;
}

namespace {

template <typename Area>
int coco_match(const char *fn, const double *d_iou, const int *d_pred_counts, const int *d_pred_cat,
               const unsigned char *d_pred_keep, const int *d_walk, const Area *d_pred_area,
               const int *d_gt_counts, const int *d_gt_cat, const unsigned char *d_gt_crowd,
               const double *d_gt_area, const double *thresholds, int T, const double *area_rng,
               int A, int *d_dt_match, unsigned char *d_dt_ignore, int B, int R1, int R2,
               void *stream) {
  MRX_CHECK_ARG(d_iou && d_pred_counts && d_pred_cat && d_pred_keep && d_walk && d_pred_area &&
                    d_gt_counts && d_gt_cat && d_gt_crowd && d_gt_area && thresholds && area_rng &&
                    d_dt_match && d_dt_ignore,
                "%s: null pointer", fn);
  MRX_CHECK_ARG(B >= 0 && B <= MRX_MAX_BATCH, "%s: bad B %d (need 0<=B<=%d)", fn, B, MRX_MAX_BATCH);
  MRX_CHECK_ARG(R1 >= 1 && R1 <= 65534 && R2 >= 1 && R2 <= 65534,
                "%s: bad R1 %d / R2 %d (need 1<=R<=65534)", fn, R1, R2);
  MRX_CHECK_ARG(T >= 1 && T <= MRX_MAX_IOU_THRESHOLDS, "%s: bad T %d (need 1<=T<=%d)", fn, T,
                MRX_MAX_IOU_THRESHOLDS);
  MRX_CHECK_ARG(A >= 1 && A <= MRX_MAX_AREA_RANGES, "%s: bad A %d (need 1<=A<=%d)", fn, A,
                MRX_MAX_AREA_RANGES);
  if (B == 0) return MRX_OK;
  cocoeval::MatchParams<Area> p{};
  p.iou = d_iou;
  p.pred_counts = d_pred_counts;
  p.pred_cat = d_pred_cat;
  p.pred_keep = d_pred_keep;
  p.walk = d_walk;
  p.pred_area = d_pred_area;
  p.gt_counts = d_gt_counts;
  p.gt_cat = d_gt_cat;
  p.gt_crowd = d_gt_crowd;
  p.gt_area = d_gt_area;
  p.dt_match = d_dt_match;
  p.dt_ignore = d_dt_ignore;
  p.B = B;
  p.R1 = R1;
  p.R2 = R2;
  p.T = T;
  for (int t = 0; t < T; ++t) p.thresholds[t] = thresholds[t];
  for (int a = 0; a < 2 * A; ++a) p.area_rng[a] = area_rng[a];
  cocoeval::coco_match_kernel<Area>
      <<<dim3(B, T, A), 32, 0, static_cast<cudaStream_t>(stream)>>>(p);
  MRX_LAUNCH_CHECK("coco_match_kernel");
  return MRX_OK;
}

}  // namespace

extern "C" int mrx_coco_match(const double *d_iou, const int *d_pred_counts, const int *d_pred_cat,
                              const unsigned char *d_pred_keep, const int *d_walk,
                              const long long *d_pred_area, const int *d_gt_counts,
                              const int *d_gt_cat, const unsigned char *d_gt_crowd,
                              const double *d_gt_area, const double *thresholds, int T,
                              const double *area_rng, int A, int *d_dt_match,
                              unsigned char *d_dt_ignore, int B, int R1, int R2, void *stream) {
  return coco_match("mrx_coco_match", d_iou, d_pred_counts, d_pred_cat, d_pred_keep, d_walk,
                    d_pred_area, d_gt_counts, d_gt_cat, d_gt_crowd, d_gt_area, thresholds, T,
                    area_rng, A, d_dt_match, d_dt_ignore, B, R1, R2, stream);
}

extern "C" int mrx_coco_match_f64area(const double *d_iou, const int *d_pred_counts,
                                      const int *d_pred_cat, const unsigned char *d_pred_keep,
                                      const int *d_walk, const double *d_pred_area,
                                      const int *d_gt_counts, const int *d_gt_cat,
                                      const unsigned char *d_gt_crowd, const double *d_gt_area,
                                      const double *thresholds, int T, const double *area_rng,
                                      int A, int *d_dt_match, unsigned char *d_dt_ignore, int B,
                                      int R1, int R2, void *stream) {
  return coco_match("mrx_coco_match_f64area", d_iou, d_pred_counts, d_pred_cat, d_pred_keep,
                    d_walk, d_pred_area, d_gt_counts, d_gt_cat, d_gt_crowd, d_gt_area, thresholds,
                    T, area_rng, A, d_dt_match, d_dt_ignore, B, R1, R2, stream);
}

extern "C" int mrx_coco_box_ious(const void *d_pred_boxes, int box_form, const int *d_pred_counts,
                                 const int *d_pred_cat, const unsigned char *d_pred_keep, int R1,
                                 const double *d_gt_boxes, const int *d_gt_counts,
                                 const int *d_gt_cat, const unsigned char *d_gt_crowd, int R2,
                                 double *d_pred_area, double *d_iou, int B, void *stream) {
  const char *fn = "mrx_coco_box_ious";
  MRX_CHECK_ARG(d_pred_boxes && d_pred_counts && d_pred_cat && d_pred_keep && d_gt_boxes &&
                    d_gt_counts && d_gt_cat && d_gt_crowd && d_pred_area && d_iou,
                "%s: null pointer", fn);
  MRX_CHECK_ARG(B >= 0 && B <= MRX_MAX_BATCH, "%s: bad B %d (need 0<=B<=%d)", fn, B, MRX_MAX_BATCH);
  MRX_CHECK_ARG(R1 >= 1 && R1 <= 65534 && R2 >= 1 && R2 <= 65534,
                "%s: bad R1 %d / R2 %d (need 1<=R<=65534)", fn, R1, R2);
  MRX_CHECK_ARG(box_form == MRX_BOX_YXYX_I32 || box_form == MRX_BOX_XYWH_F64,
                "%s: bad box form %d", fn, box_form);
  if (B == 0) return MRX_OK;
  const cocoeval::BoxIouParams p{d_pred_boxes, d_pred_counts, d_pred_cat,  d_pred_keep,
                                 d_gt_boxes,   d_gt_counts,   d_gt_cat,    d_gt_crowd,
                                 d_pred_area,  d_iou,         R1,          R2,
                                 box_form == MRX_BOX_XYWH_F64};
  cocoeval::coco_box_iou_kernel<<<dim3(R1, B), cocoeval::kBoxThreads, 0,
                                  static_cast<cudaStream_t>(stream)>>>(p);
  MRX_LAUNCH_CHECK("coco_box_iou_kernel");
  return MRX_OK;
}
