// rle_decode.cu -- COCO run-length encodings to packed planes: the inverse of rle.cu, for ground
// truth that arrives as pycocotools' compressed strings or uncompressed count lists.
//
//   rle_parse_kernel   CTA per instance, one character per thread and pass: a block scan of the
//                      "ends a value" flags gives each value its index, its thread assembles it
//                      from the (at most 7) groups before it, and two scans, over odd and over
//                      even indices from 2, undo the deltas
//   rle_ends_kernel    CTA per instance: inclusive scan of the runs as int64 run ends (positions
//                      pass 2^31 when H*W does) and the check that they sum to H*W
//   rle_planes_kernel  CTA per band of 32 rows x 256 columns of one plane, warp per 32 x 32 block,
//                      lane per column: the lane finds the run covering its first pixel by binary
//                      search over the run ends and ORs the ones-runs into a 32-bit column word;
//                      store_band (planes.cuh) transposes the 32 column words of each warp and
//                      stores the band as rows of 32 contiguous bytes
//
// Runs are column-major (Fortran order, pixel (y, x) at x*H + y), starting with zeros.
#include <climits>

#include "planes.cuh"

namespace mrx {

namespace rle_decode {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxGroups = 7;   // a count below 2^32 has a delta of at most 7 groups

__device__ __forceinline__ bool continues(unsigned char c) {
  return ((static_cast<int>(c) - '0') & 0x20) != 0;
}

// ---------------------------------------------------------------- strings -> runs
__global__ void __launch_bounds__(kThreads)
rle_parse_kernel(const unsigned char *__restrict__ str, const long long *__restrict__ str_off,
                 const int *__restrict__ counts, int R, unsigned int *__restrict__ runs,
                 int *__restrict__ run_count, int *__restrict__ status) {
  __shared__ int s_int[kWarps];
  __shared__ long long s_ll[kWarps];
  __shared__ int s_status;
  const int k = blockIdx.x, b = blockIdx.y;
  if (k >= counts[b]) return;
  const size_t i = static_cast<size_t>(b) * R + k;
  const long long s0 = str_off[i], L = str_off[i + 1] - s0;
  if (L <= 0) return;   // left to the caller (an uncompressed instance, or nothing)
  if (L > INT_MAX) {
    if (threadIdx.x == 0) {
      run_count[i] = 0;
      status[i] = MRX_RLE_ST_RANGE;
    }
    return;
  }
  if (threadIdx.x == 0) s_status = 0;
  const unsigned char *s = str + s0;
  unsigned int *out = runs + s0;
  int st = 0;
  long long nval = 0, odd = 0, even = 0;   // values before this pass, the two chains' sums
  for (long long base = 0; base < L; base += kThreads) {
    const long long p = base + threadIdx.x;
    bool end = false;
    long long x = 0;
    if (p < L) {
      const int g = static_cast<int>(s[p]) - '0';
      if (g < 0 || g > 63) st |= MRX_RLE_ST_CHAR;
      end = (g & 0x20) == 0;
      if (!end && p == L - 1) st |= MRX_RLE_ST_TRUNC;
      if (end) {
        // the value's groups: the continuation characters right before p, then p
        int n = 1;
        while (n <= kMaxGroups && p - n >= 0 && continues(s[p - n])) ++n;
        if (n > kMaxGroups) {
          st |= MRX_RLE_ST_RANGE;
        } else {
          for (int t = 0; t < n; ++t)
            x |= static_cast<long long>((static_cast<int>(s[p - n + 1 + t]) - '0') & 0x1f) << (5 * t);
          if (g & 0x10) x |= -1LL << (5 * n);
        }
      }
    }
    int pass_vals;
    const long long j = nval + block_exclusive_scan<int, kThreads>(end ? 1 : 0, s_int, pass_vals);
    // cnts[j] = x_j + cnts[j-2] for j > 2: odd j sum the odd values, even j >= 2 the even ones
    // from index 2 (cnts[0] and cnts[2] take no delta)
    const long long xo = end && (j & 1) ? x : 0, xe = end && !(j & 1) && j >= 2 ? x : 0;
    long long pass_odd, pass_even;
    const long long co = odd + block_exclusive_scan<long long, kThreads>(xo, s_ll, pass_odd) + xo;
    const long long ce = even + block_exclusive_scan<long long, kThreads>(xe, s_ll, pass_even) + xe;
    if (end) {
      // the first value out of range is exact: every earlier count of its chain was in range
      const long long c = j == 0 ? x : (j & 1) ? co : ce;
      if (c < 0 || c > 0xFFFFFFFFLL) st |= MRX_RLE_ST_RANGE;
      out[j] = static_cast<unsigned int>(c);
    }
    nval += pass_vals;
    odd += pass_odd;
    even += pass_even;
  }
  if (st) atomicOr(&s_status, st);
  __syncthreads();
  if (threadIdx.x == 0) {
    run_count[i] = static_cast<int>(nval);
    status[i] = s_status;
  }
}

// ---------------------------------------------------------------- runs -> run ends
__global__ void __launch_bounds__(kThreads)
rle_ends_kernel(const unsigned int *__restrict__ runs, const long long *__restrict__ run_off,
                const int *__restrict__ run_count, const int *__restrict__ counts,
                const int *__restrict__ geom, int R, long long *__restrict__ ends,
                int *__restrict__ status) {
  __shared__ long long s_ll[kWarps];
  const int k = blockIdx.x, b = blockIdx.y;
  if (k >= counts[b]) return;
  const size_t i = static_cast<size_t>(b) * R + k;
  const long long o = run_off[i];
  const int m = run_count[i];
  long long carry = 0;
  for (int base = 0; base < m; base += kThreads) {
    const int j = base + threadIdx.x;
    const long long v = j < m ? runs[o + j] : 0;
    long long pass;
    const long long ex = block_exclusive_scan<long long, kThreads>(v, s_ll, pass);
    if (j < m) ends[o + j] = carry + ex + v;
    carry += pass;
  }
  const long long hw = static_cast<long long>(geom[b * MRX_GEOM_INTS + 0]) *
                       geom[b * MRX_GEOM_INTS + 1];
  if (threadIdx.x == 0 && carry != hw) status[i] |= MRX_RLE_ST_SUM;
}

// ---------------------------------------------------------------- run ends -> packed planes
// the first run j in [lo, hi) whose end passes position p (hi when none does)
__device__ __forceinline__ int first_end_after(const long long *e, int lo, int hi, long long p) {
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (e[mid] > p)
      hi = mid;
    else
      lo = mid + 1;
  }
  return lo;
}

__global__ void __launch_bounds__(kThreads)
rle_planes_kernel(Slots<unsigned char> packed, const long long *__restrict__ run_off,
                  const int *__restrict__ run_count, const long long *__restrict__ ends,
                  const int *__restrict__ counts, const int *__restrict__ geom,
                  const int *__restrict__ status, int R, int bands_x) {
  __shared__ uint32_t s_band[32][kWarps];   // row r: the band's 32 bytes, warp w's at [4w, 4w+4)
  const int k = blockIdx.y, b = blockIdx.z;
  if (k >= counts[b]) return;
  const size_t i = static_cast<size_t>(b) * R + k;
  if (status[i]) return;   // a flagged instance's plane is unspecified: nothing is written
  const int H = geom[b * MRX_GEOM_INTS + 0], W = geom[b * MRX_GEOM_INTS + 1];
  const int wb = (W + 7) >> 3;
  const int y0 = (blockIdx.x / bands_x) * 32, cb0 = (blockIdx.x % bands_x) * 32;
  if (y0 >= H || cb0 >= wb) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int x0 = cb0 * 8 + warp * 32;
  uint32_t word = 0;
  if (x0 < W) {
    const long long *e = ends + run_off[i];
    const int m = run_count[i];
    const int rows = min(32, H - y0);
    const int last = min(W - 1 - x0, 31);   // the warp's columns are x0 .. x0 + last
    // the warp's runs: from the one covering its first pixel to the one covering its last
    int j = 0;
    if (lane < 2)
      j = first_end_after(e, 0, m, lane ? static_cast<long long>(x0 + last) * H + y0 + rows - 1
                                        : static_cast<long long>(x0) * H + y0);
    const int jlo = __shfl_sync(0xffffffffu, j, 0), jhi = __shfl_sync(0xffffffffu, j, 1);
    const int c = lane ^ 7;
    if (c <= last) {
      const long long p0 = static_cast<long long>(x0 + c) * H + y0, p1 = p0 + rows;
      j = first_end_after(e, jlo, jhi, p0);
      long long s = j ? e[j - 1] : 0;
      for (; j <= jhi && s < p1; ++j) {
        const long long en = e[j];
        if ((j & 1) && en > s) {
          const int lo = static_cast<int>(max(s, p0) - p0), hi = static_cast<int>(min(en, p1) - p0);
          word |= (hi - lo == 32 ? 0xFFFFFFFFu : ((1u << (hi - lo)) - 1u)) << lo;
        }
        s = en;
      }
    }
  }
  store_band<kWarps>(word, s_band,
                     packed.base + packed.off[b] + static_cast<long long>(k) * H * wb, y0, cb0, H,
                     wb);
}

}  // namespace rle_decode

}  // namespace mrx

using namespace mrx;

extern "C" int mrx_rle_parse(const unsigned char *d_str, const long long *d_str_off,
                             const int *d_counts, unsigned int *d_runs, int *d_run_count,
                             int *d_status, int B, int R, void *stream) {
  const char *fn = "mrx_rle_parse";
  MRX_CHECK_ARG(d_str && d_str_off && d_counts && d_runs && d_run_count && d_status,
                "%s: null pointer", fn);
  MRX_CHECK_ARG(B >= 0 && B <= MRX_MAX_BATCH && R >= 1 && R <= 65534,
                "%s: bad sizes B=%d R=%d (need 0<=B<=%d, 1<=R<=65534)", fn, B, R, MRX_MAX_BATCH);
  if (B == 0) return MRX_OK;
  rle_decode::rle_parse_kernel<<<dim3(R, B), rle_decode::kThreads, 0,
                                 static_cast<cudaStream_t>(stream)>>>(
      d_str, d_str_off, d_counts, R, d_runs, d_run_count, d_status);
  MRX_LAUNCH_CHECK("rle_parse_kernel");
  return MRX_OK;
}

extern "C" int mrx_rle_decode(const unsigned int *d_runs, const long long *d_run_off,
                              const int *d_run_count, long long *d_run_end, int *d_status,
                              const int *d_counts, const int *d_geom,
                              const long long *d_packed_off, unsigned char *d_packed, int B, int R,
                              int max_h, int max_w, void *stream) {
  const char *fn = "mrx_rle_decode";
  if (int rc = check_slots(fn, d_packed, d_packed_off, d_counts, d_geom, B, R)) return rc;
  MRX_CHECK_ARG(d_runs && d_run_off && d_run_count && d_run_end && d_status, "%s: null pointer",
                fn);
  MRX_CHECK_ARG(max_h >= 1 && max_w >= 1, "%s: bad extents max_h=%d max_w=%d (need >= 1)", fn,
                max_h, max_w);
  const long long bands_y = (max_h + 31LL) / 32, bands_x = ((max_w + 7LL) / 8 + 31) / 32;
  MRX_CHECK_SUPPORTED(bands_y * bands_x <= INT_MAX, "%s: image of %d x %d too large", fn, max_h,
                      max_w);
  if (B == 0) return MRX_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  rle_decode::rle_ends_kernel<<<dim3(R, B), rle_decode::kThreads, 0, st>>>(
      d_runs, d_run_off, d_run_count, d_counts, d_geom, R, d_run_end, d_status);
  MRX_LAUNCH_CHECK("rle_ends_kernel");
  rle_decode::rle_planes_kernel<<<dim3(static_cast<unsigned>(bands_y * bands_x), R, B),
                                  rle_decode::kThreads, 0, st>>>(
      {d_packed, d_packed_off}, d_run_off, d_run_count, d_run_end, d_counts, d_geom, d_status, R,
      static_cast<int>(bands_x));
  MRX_LAUNCH_CHECK("rle_planes_kernel");
  return MRX_OK;
}
