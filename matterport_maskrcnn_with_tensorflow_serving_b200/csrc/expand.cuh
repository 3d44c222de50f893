// expand.cuh -- shared declarations of the mask-expand kernels (csrc/unmold.cu: generic
// kernel + C ABI; csrc/expand_team.cu: the default team kernel; csrc/expand_bits.cu: the
// bit-packed output; csrc/rle.cu: run-length output) and the one definition of the sample
// they all compute.
#pragma once

#include "common.cuh"

namespace mrx {

#if defined(__CUDACC__)
// ---- the sample (DESIGN.md 3.1).  Canvas pixel d of a box [lo, hi) samples the zero-padded
// tile (`in` wide on that axis) at the half-pixel-centre source coordinate
//   (d - lo + 0.5) * in / ext - 0.5 = A / D,   A = in * (2 (d - lo) + 1) - ext,  D = 2 ext,
// with ext = hi - lo.  A / D is split exactly into floor i (in [-1, in-1]) and remainder rem
// (in [0, D)) with integers; the weight rem * (1/D) is the one fp32 rounding.  The sample is
// lerp(wy, lerp(wx, ...row j...), lerp(wx, ...row j+1...)): two fp32 FMAs, horizontal first.
// All integer quantities are < 2^24, so their float conversions are exact.

// numerator A of the source coordinate of canvas pixel d in the box [lo, lo + ext)
__device__ __forceinline__ int src_num(int in, int d, int lo, int ext) {
  return in * (2 * (d - lo) + 1) - ext;
}

struct SrcPos {
  int i;     // floor(A / D)
  int rem;   // A - i * D, in [0, D)
};

// floor and remainder of A / D (D > 0), given inv_d = __fdiv_rn(1, D): the fp32 estimate is
// off by at most one and is corrected with integers
__device__ __forceinline__ SrcPos src_floor(int A, int D, float inv_d) {
  int i = __float2int_rd(static_cast<float>(A) * inv_d);
  int rem = A - i * D;
  if (rem < 0) {
    --i;
    rem += D;
  } else if (rem >= D) {
    ++i;
    rem -= D;
  }
  return {i, rem};
}

__device__ __forceinline__ float src_weight(int rem, float inv_d) {
  return static_cast<float>(rem) * inv_d;
}

// Advance of the source coordinate per `num / 2` canvas pixels of `in` (num = 2 * in * steps):
// quotient and remainder of num / D.  Applied with src_advance.
struct SrcStep {
  int q, r;
};

__device__ __forceinline__ SrcStep src_step(int num, int D) {
  int q = 0;
  if (D <= num) q = num / D;
  return {q, num - q * D};
}

__device__ __forceinline__ void src_advance(int &i, int &rem, SrcStep s, int D) {
  rem += s.r;
  i += s.q;
  if (rem >= D) {
    rem -= D;
    ++i;
  }
}

__device__ __forceinline__ float lerp(float w, float lo, float hi) { return fmaf(w, hi - lo, lo); }

// box (y1, x1, y2, x2) non-empty and inside an H x W canvas
__device__ __forceinline__ bool box_in_canvas(int4 bx, int H, int W) {
  return bx.x >= 0 && bx.y >= 0 && bx.z <= H && bx.w <= W && bx.z > bx.x && bx.w > bx.y;
}

// Tile row j in lane-column layout: lane l holds column l - 1 (lanecol: 1 <= l <= mw), the
// other lanes and rows outside the tile hold the zero padding.  col = the lane's column of row 0.
struct LaneRows {
  const float *col;
  int mh, mw;
  bool lanecol;
  __device__ __forceinline__ float operator()(int j) const {
    const float v = __ldg(col + static_cast<unsigned>(min(max(j, 0), mh - 1) * mw));
    return (lanecol && j >= 0 && j < mh) ? v : 0.f;
  }
};

// horizontal interpolation of a row in lane-column layout: taps idx = i + 1 and idx + 1
__device__ __forceinline__ float hrow(float rv, int idx, float wx) {
  const float lo = __shfl_sync(0xffffffffu, rv, idx);
  const float hi = __shfl_sync(0xffffffffu, rv, idx + 1);
  return lerp(wx, lo, hi);
}

// ---- the scheduler of the persistent kernels.  Workers draw tickets 0, 1, ... from words[0]
// of their scheduler pair; ticket j names the j-th work item of the batch, image by image.
// Work table, on warp 0: s_prefix[b] = the work items of the images before b (b in [0, B]),
// *s_total = all of them; work_of_b(b) = the items of image b.  The caller synchronises.
// (Callers capture by value: a lambda holding a reference to the kernel's parameter struct
// changes how the rest of the kernel is optimised.)
template <typename WorkOf>
__device__ __forceinline__ void image_work_table(int B, WorkOf work_of_b, int *s_prefix, int *s_total) {
  const int lane = threadIdx.x & 31;
  int carry = 0;
  for (int base = 0; base < B; base += 32) {
    const int b = base + lane;
    const int incl = warp_inclusive_scan(b < B ? work_of_b(b) : 0, lane);
    if (b < B) s_prefix[b + 1] = carry + incl;
    carry += __shfl_sync(0xffffffffu, incl, 31);
  }
  if (lane == 0) {
    s_prefix[0] = 0;
    *s_total = carry;
  }
}

// One thread of a worker that is done: counts it in words[1], and the last of the grid's
// gridDim.x * workers_per_cta workers (CTAs, teams or warps) leaves both words at zero for the
// next launch (no memset between launches).
__device__ __forceinline__ void retire_worker(unsigned int *words, unsigned workers_per_cta) {
  __threadfence();
  if (atomicAdd(words + 1, 1u) == gridDim.x * workers_per_cta - 1u) {
    words[0] = 0u;
    words[1] = 0u;
  }
}
#endif  // __CUDACC__

// The batch mrx_unmold_prepare leaves on the device, as every kernel that reads the class tiles
// takes it (mrx.h, "Tile batch").
struct TileBatch {
  const float *tiles;           // [B,R,mh,mw]
  const int *tile_index;        // [B,R] tile of kept instance k = tiles[b][tile_index[b][k]]
  const int4 *boxes;            // [B,R] (y1,x1,y2,x2)
  const int *counts;            // [B]
  const int *geom;              // [B,8]
  int B, R, mh, mw;
};

// The one host check of a tile batch (unmold.cu): pointers, sizes, then the tile shape against
// max_mw (MRX_MAX_MASK_DIM, or MRX_MAX_LANE_MASK_W for the kernels that keep a tile row in one
// warp's lanes).  Returns MRX_OK or the error code, with mrx_last_error() naming `fn`.
int check_tile_batch(const char *fn, const TileBatch &t, int max_mw);

struct ExpandParams {
  TileBatch t;
  Slots<unsigned char> canvas;  // image b: bytes [H_b, W_b, N_b] (mrx.h, "Output slots")
  unsigned int *job_counter;    // [0] tile ticket, [1] teams / CTAs retired; zero between launches
  float *values;                // test instantiation only: pre-threshold samples, indexed like canvas
  int chunk_bytes;
  int flags;                    // team kernel development switches (MRX_EXPAND_FLAGS; -DMRX_DEV only)
};

// The default kernel: teams of warps build 2-D tiles (one persistent CTA per SM).  want_buf =
// upper bound of a team's tile buffer in bytes (0 = as large as fits).  Returns MRX_OK, an
// error code with mrx_last_error() set, or MRX_E_UNSUPPORTED when R does not fit a buffer or
// mw > MRX_MAX_LANE_MASK_W (the caller then takes the generic kernel).
int launch_expand_team(const ExpandParams &prm, const DevInfo &dev, int want_buf, cudaStream_t st);

}  // namespace mrx
