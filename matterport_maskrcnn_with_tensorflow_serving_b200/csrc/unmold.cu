// unmold.cu -- the serving post-processing path of the reference,
// api_utils.unmold_detections (serve.py:147-154), as sm_90a kernels.
//
//   unmold_prepare_kernel    steps 1-6 of the upstream body (trim, class ids, window
//                            normalisation, box affine + denorm, zero-area compaction) and
//                            masks = mrcnn_mask[src_index, :, :, class_ids] -> fp32 tiles
//   mask_expand_kernel       per-instance resize + threshold + paste + np.stack(axis=-1),
//                            fused: one bulk (TMA) store per chunk of the [H,W,N] canvas
//                            (the generic kernel; expand_team.cu holds the default one)
//
// Data layout in HBM (all row-major, caller-owned):
//   detections [B,R,6] f32|f64        mrcnn_mask [B,R,mh,mw,C] f32|f64
//   boxes [B,R,4] i32   class_ids/src_index [B,R] i32   scores [B,R]   counts/status [B]
//   tiles [B,R,mh,mw] f32 (selected class only, 3136 B per instance at 28x28)
//   canvas: image b at canvas + canvas_off[b], bytes [H_b, W_b, N_b] (N innermost)
#include <stdlib.h>

#include "expand.cuh"

namespace mrx {

// =====================================================================================
// prologue (steps 1-6) and class-tile gather: one launch, grid (R + 1, B)
// =====================================================================================
constexpr int kPrepareThreads = 256;

template <typename T>
struct BoxAffine;

// detections arrive as float64 (serve.py:131-136 builds them from Python floats):
//   boxes(float64) - shift(float32 array) -> float64 ; / scale(float32 array) -> float64
template <>
struct BoxAffine<double> {
  __device__ static double apply(double v, float shift, float scale) {
    return __ddiv_rn(__dsub_rn(v, static_cast<double>(shift)), static_cast<double>(scale));
  }
};
// float32 detections: numpy keeps the affine in float32, widening only in denorm_boxes
template <>
struct BoxAffine<float> {
  __device__ static double apply(float v, float shift, float scale) {
    return static_cast<double>(__fdiv_rn(__fsub_rn(v, shift), scale));
  }
};

__device__ __forceinline__ float norm_coord_f32(int v, int shift, int extent_minus_1) {
  // utils.norm_boxes: (int - int) / int in float64, then astype(float32)
  return __double2float_rn(
      __ddiv_rn(static_cast<double>(v - shift), static_cast<double>(extent_minus_1)));
}

__device__ __forceinline__ int denorm_coord(double v, int extent_minus_1, int shift) {
  // utils.denorm_boxes: around(v * (extent-1) + shift).astype(int32); around = half-to-even
  const double t = __dadd_rn(__dmul_rn(v, static_cast<double>(extent_minus_1)),
                             static_cast<double>(shift));
  return __double2int_rn(t);
}

// One CTA does image b (every thread of the CTA must call it).
template <typename T>
__device__ __forceinline__ void prologue_body(const int b, const T *__restrict__ det, int R, int C,
                                              const int *__restrict__ geom, int *__restrict__ boxes,
                                              int *__restrict__ class_ids, T *__restrict__ scores,
                                              int *__restrict__ src_index, int *__restrict__ counts,
                                              int *__restrict__ status,
                                              unsigned int *__restrict__ job_counter) {
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int warp = tid >> 5;
  constexpr int kWarps = kPrepareThreads / 32;

  __shared__ int s_first_zero;
  __shared__ int s_status;
  __shared__ int s_wcnt[kWarps];

  if (tid == 0) {
    s_first_zero = R;
    s_status = 0;
    if (b == 0 && job_counter != nullptr) {   // scheduler words of mrx_mask_expand*: ticket, retired
      job_counter[0] = 0u;
      job_counter[1] = 0u;
    }
  }
  __syncthreads();

  const T *d = det + static_cast<size_t>(b) * R * 6;
  // step 1: N = index of the first row whose class_id == 0 (zero padding), else R
  for (int t = tid; t < R; t += kPrepareThreads) {
    if (d[t * 6 + 4] == T(0)) atomicMin(&s_first_zero, t);
  }
  __syncthreads();
  const int n_trim = s_first_zero;

  // step 3: window = norm_boxes(window, image_shape[:2]) -> float32
  const int *g = geom + b * MRX_GEOM_INTS;
  const int orig_h = g[0], orig_w = g[1], img_h = g[2], img_w = g[3];
  const float wy1 = norm_coord_f32(g[4], 0, img_h - 1);
  const float wx1 = norm_coord_f32(g[5], 0, img_w - 1);
  const float wy2 = norm_coord_f32(g[6], 1, img_h - 1);
  const float wx2 = norm_coord_f32(g[7], 1, img_w - 1);
  const float wh = __fsub_rn(wy2, wy1);  // np.float32 scalar arithmetic
  const float ww = __fsub_rn(wx2, wx1);

  int running = 0;
  int my_status = 0;
  for (int base = 0; base < n_trim; base += kPrepareThreads) {
    const int t = base + tid;
    bool keep = false, in_canvas = true;
    int y1 = 0, x1 = 0, y2 = 0, x2 = 0, cls = 0;
    T score = T(0);
    if (t < n_trim) {
      const T *row = d + t * 6;
      // steps 4-5: affine into the window, then pixels of the original image
      y1 = denorm_coord(BoxAffine<T>::apply(row[0], wy1, wh), orig_h - 1, 0);
      x1 = denorm_coord(BoxAffine<T>::apply(row[1], wx1, ww), orig_w - 1, 0);
      y2 = denorm_coord(BoxAffine<T>::apply(row[2], wy1, wh), orig_h - 1, 1);
      x2 = denorm_coord(BoxAffine<T>::apply(row[3], wx1, ww), orig_w - 1, 1);
      cls = static_cast<int>(row[4]);  // astype(int32): truncation
      score = row[5];
      // step 6: drop rows with (y2 - y1) * (x2 - x1) <= 0   (int32 arithmetic)
      keep = ((y2 - y1) * (x2 - x1)) > 0;
      // numpy fancy indexing accepts class ids in [-C, C); astype(int32) turns NaN into
      // INT_MIN on the host, where the device conversion gives 0
      if (cls < -C || cls >= C || isnan(row[4])) my_status |= MRX_ST_CLASS_RANGE;
      in_canvas = !(y1 < 0 || x1 < 0 || y2 > orig_h || x2 > orig_w || y2 <= y1 || x2 <= x1);
      if (keep && !in_canvas) my_status |= MRX_ST_BOX_RANGE;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_wcnt[warp] = __popc(bal);
    __syncthreads();
    int before = running, total = 0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) {
      const int c = s_wcnt[w];
      if (w < warp) before += c;
      total += c;
    }
    if (keep) {
      const int pos = before + __popc(bal & ((1u << lane) - 1u));
      const size_t o = static_cast<size_t>(b) * R + pos;
      reinterpret_cast<int4 *>(boxes)[o] = make_int4(y1, x1, y2, x2);
      class_ids[o] = cls;
      scores[o] = score;
      src_index[o] = t;
    }
    running += total;
    __syncthreads();
  }
  if (my_status) atomicOr(&s_status, my_status);
  __syncthreads();
  if (tid == 0) {
    counts[b] = running;
    status[b] = s_status;
  }
}

// One wanted element per 128-byte line (the class stride C*4 B exceeds a line): ask L2 for the
// smallest fill it offers (64 B) instead of the default 128 B -- the DRAM traffic of this
// kernel is pure over-fetch (ncu: 321 MB for 10 MB of wanted elements with the default).
__device__ __forceinline__ float ld_strided(const float *p) {
  float v;
  asm volatile("ld.global.nc.L2::64B.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ double ld_strided(const double *p) {
  double v;
  asm volatile("ld.global.nc.L2::64B.f64 %0, [%1];" : "=d"(v) : "l"(p));
  return v;
}

// copy the `tile_elems` elements in[0], in[C], in[2C], ... to out[0 .. tile_elems) as float32
template <typename T>
__device__ __forceinline__ void gather_strided(const T *__restrict__ in, int tile_elems, int C,
                                               float *__restrict__ out) {  // every element is its own 32-byte sector (stride C): keep four loads in flight per thread
  for (int p0 = threadIdx.x; p0 < tile_elems; p0 += 4 * kPrepareThreads) {
    T v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int p = p0 + k * kPrepareThreads;
      v[k] = (p < tile_elems) ? ld_strided(in + static_cast<size_t>(p) * C) : T(0);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int p = p0 + k * kPrepareThreads;
      if (p < tile_elems) out[p] = static_cast<float>(v[k]);
    }
  }
}

// One launch for steps 1-6 AND the class-tile gather (the two do not depend on each other when
// the tiles are stored by ORIGINAL detection row): grid (R + 1, B); CTA (t < R, b) copies the
// tile of row t's own class -- rows whose class_id is exactly 0 can never be kept (the first of
// them ends the list) and are skipped; a class_id such as 0.5 truncates to class 0 but does not
// end the list, so its tile is gathered -- and CTA (R, b) runs the prologue of image b.  The
// expand kernels then find instance k's tile through src_index[b][k].
template <typename TD, typename TM>
__global__ void __launch_bounds__(kPrepareThreads)
unmold_prepare_kernel(const TD *__restrict__ det, const TM *__restrict__ mask, int R, int C,
                      int tile_elems, const int *__restrict__ geom, int *__restrict__ boxes,
                      int *__restrict__ class_ids, TD *__restrict__ scores,
                      int *__restrict__ src_index, int *__restrict__ counts,
                      int *__restrict__ status, unsigned int *__restrict__ job_counter,
                      float *__restrict__ tiles) {
  const int b = blockIdx.y;
  if (static_cast<int>(blockIdx.x) == R) {
    prologue_body<TD>(b, det, R, C, geom, boxes, class_ids, scores, src_index, counts,
                                      status, job_counter);
    return;
  }
  const int t = blockIdx.x;
  const TD class_id = det[(static_cast<size_t>(b) * R + t) * 6 + 4];
  if (class_id == TD(0)) return;       // the trim's test, on the raw value
  int cls = static_cast<int>(class_id);   // astype(int32)
  if (cls < 0) cls += C;
  if (cls < 0 || cls >= C) cls = 0;    // flagged by the prologue (NaN too); stay in bounds
  gather_strided(mask + (static_cast<size_t>(b) * R + t) * tile_elems * C + cls, tile_elems, C,
                 tiles + (static_cast<size_t>(b) * R + t) * tile_elems);
}

// =====================================================================================
// mask expand: persistent CTAs, each builds one chunk of a canvas in shared memory
// =====================================================================================
//
// A job is `chunk_bytes` consecutive bytes of one image's [H,W,N] canvas (flat byte
// stream; N innermost so a pixel is N consecutive bytes).  Per job the CTA
//   1. lists the (box, row) pairs that intersect the chunk            -> entries
//      (lane-parallel: one thread per pair does all per-entry scalar math once)
//   2. stages the two tile rows each entry interpolates between with a 1-D TMA bulk
//      copy (224 B at mw = 28)
//   3. walks each entry's x-span: exact integer source coordinate (incremental along
//      the span), the sample of expand.cuh (both staged rows interpolated horizontally,
//      then vertically), >= 0.5, byte store into the shared chunk
//   4. hands the chunk to the TMA with one bulk store (HBM sees one write per byte)
// Zero fill is the memset of the shared chunk, skipped for the part already known zero.
// Job descriptors are computed by one thread a job ahead (double-buffered in smem) so
// the 32-bit divisions are off the critical path of the other warps.
constexpr int kExpandThreads = 256;
constexpr int kEMax = 64;  // entries per pass == pairs tested per pass

struct __align__(16) Entry {
  int obase;    // byte offset of (row, x=0, n) relative to the chunk start
  int xa, xb;   // span [xa, xb) of canvas columns inside the chunk and the box
  int x1;       // box left
  int D;        // 2 * box width
  float invD;   // 1 / D
  SrcStep step; // source-column advance per 32 canvas columns: (64*mw) / D and remainder
  float wy;     // vertical weight of the lower source row
  int otop;     // float offset of the upper source row inside the staging slot, -1 = outside
  int obot;     // same for the lower source row
};

struct __align__(16) JobInfo {
  const float *tiles_b;
  const int4 *boxes_b;
  unsigned char *dst;
  int valid;
  int H, W, N;
  int len, len16;
  int g0, g1, r0, n_pairs, sub;
  int pad_;
};


__device__ __forceinline__ void make_job(const ExpandParams &p, const int *s_jobs, int total_jobs,
                                         int job, int &cur_b, JobInfo *out) {
  if (job >= total_jobs) {
    out->valid = 0;
    return;
  }
  while (job >= s_jobs[cur_b + 1]) ++cur_b;
  const int b = cur_b;
  const int H = p.t.geom[b * MRX_GEOM_INTS + 0];
  const int W = p.t.geom[b * MRX_GEOM_INTS + 1];
  const int N = p.t.counts[b];
  const unsigned L = static_cast<unsigned>(H) * W * N;         // host guarantees < 2^31
  const unsigned c0 = static_cast<unsigned>(job - s_jobs[b]) * p.chunk_bytes;
  const int len = static_cast<int>(min(static_cast<unsigned>(p.chunk_bytes), L - c0));
  const int g0 = static_cast<int>(c0 / N);               // first pixel touched
  const int g1 = static_cast<int>((c0 + len - 1) / N);   // last pixel touched
  const int r0 = g0 / W;
  const int r1 = g1 / W;
  out->tiles_b = p.t.tiles + static_cast<size_t>(b) * p.t.R * p.t.mh * p.t.mw;
  out->boxes_b = p.t.boxes + static_cast<size_t>(b) * p.t.R;
  out->dst = p.canvas.base + p.canvas.off[b] + c0;
  out->H = H;
  out->W = W;
  out->N = N;
  out->len = len;
  out->len16 = (len + 15) & ~15;
  out->g0 = g0;
  out->g1 = g1;
  out->r0 = r0;
  out->n_pairs = (r1 - r0 + 1) * N;
  out->sub = static_cast<int>(c0 - static_cast<unsigned>(g0) * N);   // bytes of pixel g0 before c0
  out->valid = 1;
}

__global__ void __launch_bounds__(kExpandThreads)
mask_expand_kernel(const ExpandParams p) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int warp = tid >> 5;
  const int mh = p.t.mh, mw = p.t.mw;
  const int slot_floats = 2 * mw;             // two tile rows
  const uint32_t slot_bytes = slot_floats * 4;

  // ---- carve shared memory
  unsigned char *s_out = smem;                                        // chunk_bytes
  float *s_stage = reinterpret_cast<float *>(smem + p.chunk_bytes);   // kEMax slots
  Entry *s_entry = reinterpret_cast<Entry *>(s_stage + kEMax * slot_floats);
  int *s_jobs = reinterpret_cast<int *>(s_entry + kEMax);             // B + 1 prefix
  __shared__ JobInfo s_job[2];
  __shared__ uint64_t s_bar;
  __shared__ int s_count[2];
  __shared__ int s_next;
  __shared__ int s_total;

  // ---- job table: jobs_b = ceil(H*W*N_b / chunk); exclusive prefix in s_jobs
  if (warp == 0) {
    image_work_table(p.t.B, [=](int b) {
      const long long bytes = static_cast<long long>(p.t.geom[b * MRX_GEOM_INTS + 0]) *
                              p.t.geom[b * MRX_GEOM_INTS + 1] * p.t.counts[b];
      return static_cast<int>((bytes + p.chunk_bytes - 1) / p.chunk_bytes);
    }, s_jobs, &s_total);
  }
  if (tid == 0) {
    mbar_init(&s_bar, 1);
    fence_mbar_init();
    s_count[0] = 0;
    s_count[1] = 0;
  }
  __syncthreads();
  const int total_jobs = s_total;

  const uint32_t s_out_addr = smem_u32(s_out);
  uint32_t bar_parity = 0;
  int pass_parity = 0;
  int cur_b = 0;       // thread 0 only: image of the most recently described job
  int next_job = 0;    // thread 0 only
  int clean = 0;       // bytes [0, clean) of s_out known to be zero
  if (tid == 0) {
    const int j = static_cast<int>(atomicAdd(p.job_counter, 1u));
    make_job(p, s_jobs, total_jobs, j, cur_b, &s_job[0]);
    next_job = static_cast<int>(atomicAdd(p.job_counter, 1u));
  }

  for (int k = 0;; ++k) {
    if (tid == 0) bulk_wait_read<0>();   // the previous chunk has left shared memory
    __syncthreads();   // (S1) job descriptor visible, s_out and staging reusable
    const JobInfo J = s_job[k & 1];
    if (!J.valid) break;

    // ---- zero fill (memset of the part of the shared chunk not known to be zero)
    if (clean < J.len16) {
      uint4 *o4 = reinterpret_cast<uint4 *>(s_out);
      const int n16 = J.len16 >> 4;
      for (int i = (clean >> 4) + tid; i < n16; i += kExpandThreads)
        o4[i] = make_uint4(0u, 0u, 0u, 0u);
      clean = J.len16;
    }
    bool wrote = false;

    for (int p0 = 0; p0 < J.n_pairs; p0 += kEMax) {
      if (p0 > 0) {
        fence_proxy_async_smem();   // generic accesses to staging before the next TMA fill
        __syncthreads();
      }
      // ---- 1. entries: thread t tests pair p0 + t and does the per-entry scalar math
      if (tid < kEMax) {
        const int pr = p0 + tid;
        bool valid = false;
        Entry e;
        int jc = 0, n = 0, tile = 0;
        if (pr < J.n_pairs) {
          const int dr = pr / J.N;
          n = pr - dr * J.N;
          const int row = J.r0 + dr;
          const int4 bx = __ldg(J.boxes_b + n);   // (y1, x1, y2, x2)
          tile = __ldg(p.t.tile_index + (J.boxes_b - p.t.boxes) + n);
          const int xlo = max(0, J.g0 - row * J.W);
          const int xhi = min(J.W, J.g1 + 1 - row * J.W);
          const int xa = max(xlo, bx.y);
          const int xb = min(xhi, bx.w);
          valid = box_in_canvas(bx, J.H, J.W) && row >= bx.x && row < bx.z && xa < xb;
          if (valid) {
            const int bh = bx.z - bx.x;
            const int Dy = 2 * bh;
            const float invDy = __fdiv_rn(1.0f, static_cast<float>(Dy));
            const SrcPos sy = src_floor(src_num(mh, row, bx.x, bh), Dy, invDy);   // sy.i in [-1, mh-1]
            jc = min(max(sy.i, 0), mh - 2);       // staged rows: jc, jc+1
            e.obase = (row * J.W - J.g0) * J.N + n - J.sub;
            e.xa = xa;
            e.xb = xb;
            e.x1 = bx.y;
            e.D = 2 * (bx.w - bx.y);
            e.invD = __fdiv_rn(1.0f, static_cast<float>(e.D));
            e.step = src_step(64 * mw, e.D);
            e.wy = src_weight(sy.rem, invDy);
            e.otop = (sy.i < 0) ? -1 : (sy.i - jc) * mw;
            e.obot = (sy.i + 1 > mh - 1) ? -1 : (sy.i + 1 - jc) * mw;
          }
        }
        const unsigned bal = __ballot_sync(0xffffffffu, valid);
        int base = 0;
        if (lane == 0 && bal) base = atomicAdd(&s_count[pass_parity], __popc(bal));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (valid) {
          const int slot = base + __popc(bal & ((1u << lane) - 1u));
          s_entry[slot] = e;
          // ---- 2a. stage tile rows jc, jc+1
          bulk_g2s(s_stage + slot * slot_floats,
                   J.tiles_b + (static_cast<size_t>(tile) * mh + jc) * mw, slot_bytes, &s_bar);
        }
      }
      if (tid == 0) s_next = 0;
      __syncthreads();   // (S2) entries + count visible; zero fill complete
      const int E = s_count[pass_parity];
      if (tid == 0) {
        s_count[pass_parity ^ 1] = 0;
        if (E > 0) mbar_arrive_expect_tx(&s_bar, E * slot_bytes);
        if (p0 == 0) {
          // describe the next job while the tile rows are in flight
          make_job(p, s_jobs, total_jobs, next_job, cur_b, &s_job[(k + 1) & 1]);
          next_job = static_cast<int>(atomicAdd(p.job_counter, 1u));
        }
      }
      pass_parity ^= 1;
      if (E == 0) continue;
      wrote = true;
      mbar_wait(&s_bar, bar_parity);
      bar_parity ^= 1;

      // ---- 3. warps grab entries and walk their x-spans
      while (true) {
        int ei = 0;
        if (lane == 0) ei = atomicAdd(&s_next, 1);
        ei = __shfl_sync(0xffffffffu, ei, 0);
        if (ei >= E) break;
        const Entry e = s_entry[ei];
        const float *slot = s_stage + ei * slot_floats;
        // column c of the staged row at offset o (-1: the row is outside the tile), zero
        // outside the tile
        auto tap = [&](int o, int c) { return (o >= 0 && c >= 0 && c < mw) ? slot[o + c] : 0.f; };
        int x = e.xa + lane;
        if (x < e.xb) {
          // exact start coordinate for this lane, then advance by 32 columns per step
          SrcPos sx = src_floor(src_num(mw, x, e.x1, e.D >> 1), e.D, e.invD);
          unsigned off = static_cast<unsigned>(e.obase + x * J.N);
          const unsigned ulen = static_cast<unsigned>(J.len);
          const unsigned ostep = 32u * J.N;
          while (true) {
            const float wx = src_weight(sx.rem, e.invD);
            const float ht = lerp(wx, tap(e.otop, sx.i), tap(e.otop, sx.i + 1));
            const float hb = lerp(wx, tap(e.obot, sx.i), tap(e.obot, sx.i + 1));
            if (lerp(e.wy, ht, hb) >= 0.5f && off < ulen)
              asm volatile("st.shared.u8 [%0], %1;" ::"r"(s_out_addr + off), "r"(1u) : "memory");
            x += 32;
            if (x >= e.xb) break;
            off += ostep;
            src_advance(sx.i, sx.rem, e.step, e.D);
          }
        }
      }
    }

    // ---- 4. hand the chunk to the TMA
    fence_proxy_async_smem();
    __syncthreads();   // (S3)
    if (tid == 0) {
      bulk_s2g(J.dst, s_out, static_cast<uint32_t>(J.len16));
      bulk_commit();
    }
    if (wrote) clean = 0;
  }
  if (tid == 0) {
    bulk_wait_all<0>();
    retire_worker(p.job_counter, 1u);   // the workers are the CTAs
  }
}

}  // namespace mrx

// =====================================================================================
// C ABI
// =====================================================================================
using namespace mrx;

// the batch size limits shared by the tile batch and the output slots
static int check_batch_sizes(const char *fn, int B, int R) {
  MRX_CHECK_ARG(B >= 0 && B <= MRX_MAX_BATCH && R >= 1 && R <= 65534,
                "%s: bad sizes B=%d R=%d (need 0<=B<=%d, 1<=R<=65534)", fn, B, R, MRX_MAX_BATCH);
  return MRX_OK;
}

int mrx::check_slots(const char *fn, const void *base, const long long *off, const int *counts,
                     const int *geom, int B, int R) {
  MRX_CHECK_ARG(base && off && counts && geom, "%s: null pointer", fn);
  return check_batch_sizes(fn, B, R);
}

int mrx::check_tile_batch(const char *fn, const TileBatch &t, int max_mw) {
  MRX_CHECK_ARG(t.tiles && t.boxes && t.counts && t.geom, "%s: null pointer", fn);
  if (int rc = check_batch_sizes(fn, t.B, t.R)) return rc;
  MRX_CHECK_SUPPORTED(t.mh >= 2 && t.mh <= MRX_MAX_MASK_DIM && t.mw >= 4 && t.mw <= max_mw &&
                          (t.mw % 4) == 0,
                      "%s: mask tile %dx%d unsupported (need 2<=mh<=%d, 4<=mw<=%d, mw%%4==0)", fn,
                      t.mh, t.mw, MRX_MAX_MASK_DIM, max_mw);
  // (after the shape checks: a shape no kernel takes is reported as such)
  MRX_CHECK_ARG(t.tile_index, "%s: null tile index", fn);
  return MRX_OK;
}

extern "C" int mrx_unmold_prepare(const void *d_detections, int det_dtype, const void *d_mrcnn_mask,
                                  int mask_dtype, int B, int R, int mh, int mw, int C,
                                  const int *d_geom, int *d_boxes, int *d_class_ids, void *d_scores,
                                  int *d_src_index, int *d_counts, int *d_status,
                                  float *d_tiles, unsigned int *d_sched, void *stream) {
  MRX_CHECK_ARG(d_detections && d_mrcnn_mask && d_geom && d_boxes && d_class_ids && d_scores &&
                    d_src_index && d_counts && d_status && d_tiles,
                "mrx_unmold_prepare: null pointer");
  MRX_CHECK_ARG(B >= 0 && B <= 65535 && R >= 1 && R <= 65534 && C >= 1 && mh >= 1 && mw >= 1 &&
                    mw <= MRX_MAX_MASK_DIM,
                "mrx_unmold_prepare: bad sizes B=%d R=%d C=%d tile %dx%d", B, R, C, mh, mw);
  MRX_CHECK_ARG((det_dtype == MRX_F32 || det_dtype == MRX_F64) &&
                    (mask_dtype == MRX_F32 || mask_dtype == MRX_F64),
                "mrx_unmold_prepare: dtypes %d / %d", det_dtype, mask_dtype);
  if (B == 0) return MRX_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  dim3 grid(R + 1, B);
#define MRX_PREPARE(TD, TM)                                                                      \
  unmold_prepare_kernel<TD, TM><<<grid, kPrepareThreads, 0, st>>>(                                \
      static_cast<const TD *>(d_detections), static_cast<const TM *>(d_mrcnn_mask), R, C, mh * mw, \
      d_geom, d_boxes, d_class_ids, static_cast<TD *>(d_scores), d_src_index, d_counts, d_status,   \
      d_sched, d_tiles)
  if (det_dtype == MRX_F64 && mask_dtype == MRX_F64) MRX_PREPARE(double, double);
  else if (det_dtype == MRX_F64) MRX_PREPARE(double, float);
  else if (mask_dtype == MRX_F64) MRX_PREPARE(float, double);
  else MRX_PREPARE(float, float);
#undef MRX_PREPARE
  MRX_LAUNCH_CHECK("unmold_prepare_kernel");
  return MRX_OK;
}

// mrx_mask_expand and mrx_mask_expand_values (`fn`), after check_tile_batch and check_slots
static int mask_expand_impl(const char *fn, const TileBatch &t, Slots<unsigned char> canvas,
                            float *d_values, int chunk_bytes, int ctas_per_sm,
                            unsigned int *d_sched, void *stream) {
  MRX_CHECK_ARG(d_sched, "%s: null pointer", fn);
  const int want_buf = chunk_bytes;   // team kernel: upper bound of a team's tile buffer, 0 = auto
  if (chunk_bytes == 0) chunk_bytes = 25600;
  MRX_CHECK_ARG(chunk_bytes >= 1024 && (chunk_bytes % 16) == 0,
                "%s: chunk_bytes %d must be a multiple of 16, >= 1024", fn, chunk_bytes);
  if (t.B == 0) return MRX_OK;

  DevInfo dev;
  if (int rc = current_device_info(&dev)) return rc;

  ExpandParams prm{t, canvas, d_sched, d_values, chunk_bytes, 0};
#ifdef MRX_DEV
  if (const char *f = getenv("MRX_EXPAND_FLAGS")) prm.flags = atoi(f);
#endif
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // the team kernel refuses tiles wider than MRX_MAX_LANE_MASK_W and R too large for its tile
  // buffers: those take the generic kernel
  const int rc = launch_expand_team(prm, dev, want_buf, st);
  if (rc != MRX_E_UNSUPPORTED) return rc;
  MRX_CHECK_SUPPORTED(d_values == nullptr,
                      "mrx_mask_expand_values: shape outside the team kernel (R=%d, mw=%d)", t.R,
                      t.mw);
  const size_t smem = static_cast<size_t>(chunk_bytes) +
                      static_cast<size_t>(kEMax) * 2 * t.mw * sizeof(float) +
                      static_cast<size_t>(kEMax) * sizeof(Entry) +
                      static_cast<size_t>(t.B + 1) * sizeof(int);
  MRX_CHECK_SUPPORTED(smem <= static_cast<size_t>(dev.max_smem_optin),
                      "mrx_mask_expand: %zu B shared memory > device limit %d (chunk_bytes too "
                      "large)",
                      smem, dev.max_smem_optin);
  static SmemCache cache;
  if (int rc = ensure_dynamic_smem(reinterpret_cast<const void *>(mask_expand_kernel), &cache,
                                   dev.device, static_cast<int>(smem)))
    return rc;
  int occ = 0;
  MRX_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, mask_expand_kernel,
                                                         kExpandThreads, smem));
  MRX_CHECK_SUPPORTED(occ >= 1, "mrx_mask_expand: kernel does not fit on an SM");
  if (ctas_per_sm > 0 && ctas_per_sm < occ) occ = ctas_per_sm;
  mask_expand_kernel<<<dev.sms * occ, kExpandThreads, smem, st>>>(prm);
  MRX_LAUNCH_CHECK("mask_expand_kernel");
  return MRX_OK;
}

extern "C" int mrx_mask_expand(const float *d_tiles, const int *d_tile_index, const int *d_boxes,
                               const int *d_counts, const int *d_geom,
                               const long long *d_canvas_off, unsigned char *d_canvas, int B,
                               int R, int mh, int mw, int chunk_bytes, int ctas_per_sm,
                               unsigned int *d_sched, void *stream) {
  const TileBatch t{d_tiles, d_tile_index, reinterpret_cast<const int4 *>(d_boxes), d_counts,
                    d_geom, B, R, mh, mw};
  const char *fn = "mrx_mask_expand";
  if (int rc = check_tile_batch(fn, t, MRX_MAX_MASK_DIM)) return rc;
  if (int rc = check_slots(fn, d_canvas, d_canvas_off, d_counts, d_geom, B, R)) return rc;
  return mask_expand_impl(fn, t, {d_canvas, d_canvas_off}, nullptr, chunk_bytes, ctas_per_sm,
                          d_sched, stream);
}

extern "C" int mrx_mask_expand_values(const float *d_tiles, const int *d_tile_index,
                                      const int *d_boxes, const int *d_counts,
                                      const int *d_geom, const long long *d_canvas_off,
                                      unsigned char *d_canvas, float *d_values, int B, int R,
                                      int mh, int mw, unsigned int *d_sched, void *stream) {
  const TileBatch t{d_tiles, d_tile_index, reinterpret_cast<const int4 *>(d_boxes), d_counts,
                    d_geom, B, R, mh, mw};
  const char *fn = "mrx_mask_expand_values";
  if (int rc = check_tile_batch(fn, t, MRX_MAX_LANE_MASK_W)) return rc;
  if (int rc = check_slots(fn, d_canvas, d_canvas_off, d_counts, d_geom, B, R)) return rc;
  MRX_CHECK_ARG(d_values != nullptr, "%s: null pointer", fn);
  return mask_expand_impl(fn, t, {d_canvas, d_canvas_off}, d_values, 0, 0, d_sched, stream);
}
