// expand_bits.cu -- mask expand with BIT-PACKED output (SURVEY.md 8f rank 4: compact masks).
//
// EXTENSION, not the reference layout: unmold_detections (serve.py:147-154)
// returns bool [H,W,N], one byte per element, and that is what mrx_mask_expand writes and what
// the headline benchmark measures.  This kernel computes the SAME samples (same exact integer
// source coordinates, same fp32 weights, same two fused multiply-adds in the same order as
// expand_team.cu, so the bits equal np.packbits of that kernel's bytes exactly) but writes
//     packed[n][y][:] = np.packbits(masks[y, :, n])         uint8 [N, H, ceil(W/8)]
// -- 8x fewer bytes to HBM, to the host, or over NVLink to the gathering rank, and no zero fill
// of bytes that carry no information: outside its box an instance's plane is stored from one
// shared page of zeros.
//
// Work decomposition: a UNIT is `rb` consecutive rows of one instance's plane = rb * WB
// contiguous bytes (WB = ceil(W/8)).  Warps work alone (no block-level barrier after the
// prologue): a warp claims one unit at a time from a global counter and, per unit,
//   - outside the box rows: one bulk copy (shared -> global, TMA) from the CTA's zero page;
//   - else: zero its own buffer, then per group of four 32-column blocks of the box: horizontal
//     source coordinate of the lane's column in each block once, then walk the unit's rows --
//     the vertical source coordinate advances by exact integer arithmetic once per row for the
//     whole group, each block adds one FFMA + compare + ballot and one 4-byte (or <= 4
//     one-byte) shared-memory store of the ballot (four independent chains hide each other's
//     latency); lanes are assigned to columns in packbits order (lane ^ 7) so the ballot IS
//     the output word; then one bulk copy.
// Each warp has two buffers so that the store of unit k overlaps the computation of unit k+1.
// Planes whose row pitch is not a multiple of 16 bytes (W = 1333: WB = 167) keep each unit in
// shared memory at its global address mod 16; the aligned body goes out as a bulk copy and the
// <= 15 head / tail bytes as byte stores.  HBM sees every output byte written exactly once.
//
// Bound: instruction issue over the in-box samples (~6 warp instructions per row of 32
// columns) plus 1/8 of the canvas bytes to HBM; see DESIGN.md 3.9 for the measured figures.
#include <stdlib.h>

#include <type_traits>

#include "expand.cuh"

#ifndef MRX_BITS_WARPS_DEFAULT
#define MRX_BITS_WARPS_DEFAULT 16
#endif

namespace mrx {

namespace bits {

constexpr int kGroup = 4;   // column blocks a warp walks side by side (independent chains)

struct BitsParams {
  TileBatch t;
  Slots<unsigned char> packed;   // image b: uint8 [N_b, H_b, ceil(W_b/8)] (mrx.h, "Output slots")
  unsigned int *sched;           // [2] unit ticket, [3] warps retired (MRX_SCHED_WORDS)
  int ubuf;                      // bytes of one unit buffer (multiple of 16, incl. 16 B of slack)
};

// rows per unit for a plane with WB bytes per row
__device__ __forceinline__ int unit_rows(int WB, int ubuf) { return max(1, (ubuf - 16) / WB); }

// Store `len` bytes held in shared memory at `s` (placed so that s and g are congruent mod 16)
// to global `g`: the 16-byte aligned body as one bulk copy issued by lane 0, the head / tail
// bytes by the first lanes.  Returns after the copies are issued (not completed).
__device__ __forceinline__ void store_unit(unsigned char *g, const unsigned char *s, int len, int lane) {
  const int a = static_cast<int>(reinterpret_cast<uintptr_t>(g) & 15u);
  const int head = min((16 - a) & 15, len);
  const int body = (len - head) & ~15;
  const int tail = len - head - body;
  if (lane == 0) {
    if (body > 0) bulk_s2g(g + head, s + head, static_cast<uint32_t>(body));
    bulk_commit();
  }
  if (lane < head + tail) {
    const int o = lane < head ? lane : body + lane;   // head + body + (lane - head)
    g[o] = s[o];
  }
}

template <int kWarps>
__global__ void __launch_bounds__(kWarps * 32, 1)
mask_expand_bits_kernel(const BitsParams p) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int warp = tid >> 5;
  const int mh = p.t.mh, mw = p.t.mw;
  const int ubuf = p.ubuf;

  // ---- shared memory: [zero page][2 buffers per warp][unit prefix per image]
  unsigned char *s_zero = smem;
  unsigned char *s_mine = smem + static_cast<size_t>(ubuf) * (1 + 2 * warp);
  int *s_prefix = reinterpret_cast<int *>(smem + static_cast<size_t>(ubuf) * (1 + 2 * kWarps));
  __shared__ int s_total;

  for (int i = tid; i < (ubuf >> 4); i += kWarps * 32)
    reinterpret_cast<uint4 *>(s_zero)[i] = make_uint4(0u, 0u, 0u, 0u);
  if (warp == 0) {
    image_work_table(p.t.B, [=](int b) {
      const int H = p.t.geom[b * MRX_GEOM_INTS + 0], W = p.t.geom[b * MRX_GEOM_INTS + 1];
      const int rb = unit_rows((W + 7) >> 3, ubuf);
      return p.t.counts[b] * ((H + rb - 1) / rb);
    }, s_prefix, &s_total);
  }
  fence_proxy_async_smem();   // the zero page is read by bulk copies only
  __syncthreads();
  const int total = s_total;

  const bool lanecol = lane >= 1 && lane <= mw;      // lane l holds tile column l - 1
  const int lcol = min(max(lane - 1, 0), mw - 1);
  int cur_b = 0;          // image of the current unit (search cursor, units are claimed in order)
  int cached_b = -1;      // image whose constants are cached below
  int H = 0, W = 0, WB = 0, rb = 1, nbands = 1;
  const float *tiles_b = nullptr;
  const int *tidx_b = nullptr;
  const int4 *boxes_b = nullptr;
  unsigned char *out_b = nullptr;
  int which = 0;          // buffer the next computed unit uses

  while (true) {
    // one unit per claim: a unit costs anything from one bulk copy (rows outside the box) to
    // ~50 rows x 16 column blocks of samples, so coarser claims leave a tail of busy warps
    int u0 = 0;
    if (lane == 0) u0 = static_cast<int>(atomicAdd(p.sched + 2, 1u));
    u0 = __shfl_sync(0xffffffffu, u0, 0);
    if (u0 >= total) break;
    {
      const int u = u0;
      while (u >= s_prefix[cur_b + 1]) ++cur_b;
      if (cur_b != cached_b) {
        cached_b = cur_b;
        H = p.t.geom[cur_b * MRX_GEOM_INTS + 0];
        W = p.t.geom[cur_b * MRX_GEOM_INTS + 1];
        WB = (W + 7) >> 3;
        rb = unit_rows(WB, ubuf);
        nbands = (H + rb - 1) / rb;
        tiles_b = p.t.tiles + static_cast<size_t>(cur_b) * p.t.R * mh * mw;
        boxes_b = p.t.boxes + static_cast<size_t>(cur_b) * p.t.R;
        tidx_b = p.t.tile_index + static_cast<size_t>(cur_b) * p.t.R;
        out_b = p.packed.base + p.packed.off[cur_b];
      }
      const int local = u - s_prefix[cur_b];
      const int n = local / nbands;
      const int band = local - n * nbands;
      const int r0 = band * rb;
      const int rows = min(rb, H - r0);
      const int len = rows * WB;
      unsigned char *g = out_b + (static_cast<size_t>(n) * H + r0) * WB;
      const int a = static_cast<int>(reinterpret_cast<uintptr_t>(g) & 15u);

      const int4 bx = __ldg(boxes_b + n);   // (y1, x1, y2, x2)
      const int ya = max(bx.x, r0), yb = min(bx.z, r0 + rows);
      if (!box_in_canvas(bx, H, W) || ya >= yb) {
        store_unit(g, s_zero + a, len, lane);   // nothing of the box in these rows
        continue;
      }

      // ---- this warp's buffer: wait until its previous bulk copy has read it, then clear it
      unsigned char *buf = s_mine + which * ubuf;
      which ^= 1;
      if (lane == 0) bulk_wait_read<1>();   // all but the newest group (the other buffer / zeros)
      __syncwarp();
      for (int i = lane; i < ((a + len + 15) >> 4); i += 32)
        reinterpret_cast<uint4 *>(buf)[i] = make_uint4(0u, 0u, 0u, 0u);
      __syncwarp();

      // ---- per-box constants
      const int bh = bx.z - bx.x, bw = bx.w - bx.y;
      const int D = 2 * bw, Dy = 2 * bh;
      const float invD = __fdiv_rn(1.0f, static_cast<float>(D));
      const float invDy = __fdiv_rn(1.0f, static_cast<float>(Dy));
      const SrcPos first = src_floor(src_num(mh, ya, bx.x, bh), Dy, invDy);   // row ya
      const SrcStep ystep = src_step(2 * mh, Dy);   // source-row advance per canvas row
      const int tile = __ldg(tidx_b + n);
      const LaneRows raw{tiles_b + static_cast<unsigned>(tile * mh * mw + lcol), mh, mw, lanecol};
      const bool word_ok = ((a | WB) & 3) == 0;   // every ballot word lands 4-byte aligned
      const uint32_t row0_addr = smem_u32(buf) + static_cast<uint32_t>(a + (ya - r0) * WB);

      // kGroup column blocks side by side: the vertical walk (integer coordinate, weight, source
      // row advance) and the tile row fetches are shared, the per-block chains are independent
      const int cb_last = (bx.w - 1) >> 5;
      for (int cb0 = bx.y >> 5; cb0 <= cb_last; cb0 += kGroup) {
        int idx[kGroup];
        float wx[kGroup], thr[kGroup], ht[kGroup], hb[kGroup], dh[kGroup];
        bool store[kGroup];    // this lane stores (a byte of) block c's ballot
#pragma unroll
        for (int c = 0; c < kGroup; ++c) {
          const int cb = cb0 + c;
          // lane -> column in packbits order: bit l of the ballot is pixel 8*(l/8) + 7 - l%8
          const int x = (cb << 5) + (lane ^ 7);
          const bool colvalid = cb <= cb_last && x >= bx.y && x < bx.w;
          const SrcPos sx = src_floor(src_num(mw, x, bx.y, bw), D, invD);
          // columns outside the box still run the shuffles: keep their lane index in range
          idx[c] = min(max(sx.i + 1, 0), 30);
          wx[c] = src_weight(sx.rem, invD);
          thr[c] = colvalid ? 0.5f : __int_as_float(0x7f800000);
          // bytes of the block inside the row: lane 0 stores the word when rows are 4-byte
          // aligned (then all four are inside), else lane t < nbytes stores byte t
          const int nbytes = cb <= cb_last ? min(4, WB - (cb << 2)) : 0;
          store[c] = word_ok ? (lane == 0 && nbytes > 0) : (lane < nbytes);
        }
        int jcur = first.i, j0 = first.i, remy = first.rem;
        {
          const float ra = raw(jcur), rbv = raw(jcur + 1);
#pragma unroll
          for (int c = 0; c < kGroup; ++c) {
            ht[c] = hrow(ra, idx[c], wx[c]);
            hb[c] = hrow(rbv, idx[c], wx[c]);
            dh[c] = hb[c] - ht[c];
          }
        }
        float rawn = raw(jcur + 2);   // fetched one advance ahead
        uint32_t addr = row0_addr + static_cast<uint32_t>(cb0 << 2);
        // the row loop, once per store form so that the form is not re-decided per row
        auto rows = [&](auto word_tag) {
          constexpr bool kWord = decltype(word_tag)::value;
          const uint32_t sh = kWord ? 0u : 8u * lane;          // byte t of the ballot for lane t
          for (int r = ya; r < yb; ++r) {
            if (j0 != jcur) {   // warp-uniform
              if (j0 == jcur + 1) {
#pragma unroll
                for (int c = 0; c < kGroup; ++c) {
                  ht[c] = hb[c];
                  hb[c] = hrow(rawn, idx[c], wx[c]);
                }
              } else {
                const float ra = raw(j0), rbv = raw(j0 + 1);
#pragma unroll
                for (int c = 0; c < kGroup; ++c) {
                  ht[c] = hrow(ra, idx[c], wx[c]);
                  hb[c] = hrow(rbv, idx[c], wx[c]);
                }
              }
              jcur = j0;
              rawn = raw(jcur + 2);
#pragma unroll
              for (int c = 0; c < kGroup; ++c) dh[c] = hb[c] - ht[c];
            }
            const float wy = src_weight(remy, invDy);
#pragma unroll
            for (int c = 0; c < kGroup; ++c) {
              const float v = fmaf(wy, dh[c], ht[c]);
              const unsigned bal = __ballot_sync(0xffffffffu, v >= thr[c]);
              if (store[c]) {
                if (kWord) asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr + 4u * c), "r"(bal));
                else asm volatile("st.shared.u8 [%0], %1;" ::"r"(addr + 4u * c + lane), "r"(bal >> sh));
              }
            }
            addr += static_cast<uint32_t>(WB);
            src_advance(j0, remy, ystep, Dy);
          }
        };
        if (word_ok) rows(std::true_type{});
        else rows(std::false_type{});
      }
      fence_proxy_async_smem();   // this lane's bytes -> visible to the bulk copy
      __syncwarp();
      store_unit(g, buf + a, len, lane);
    }
  }
  // ---- drain this warp's copies, then retire (the workers are the warps)
  if (lane == 0) {
    bulk_wait_all<0>();
    retire_worker(p.sched + 2, kWarps);
  }
}

}  // namespace bits

}  // namespace mrx

using namespace mrx;

template <int kWarps>
static int launch_bits(mrx::bits::BitsParams prm, const DevInfo &dev, int max_w, cudaStream_t st) {
  using namespace mrx::bits;
  const size_t fixed = static_cast<size_t>(prm.t.B + 1) * sizeof(int) + 1024;   // prefix + static + slack
  int ubuf = static_cast<int>((static_cast<size_t>(dev.max_smem_optin) - fixed) / (1 + 2 * kWarps)) & ~127;
  if (ubuf > 8192) ubuf = 8192;
  const int wb = (max_w + 7) >> 3;
  MRX_CHECK_SUPPORTED(wb + 16 <= ubuf, "mrx_mask_expand_packed: image %d pixels wide does not fit a "
                      "unit buffer of %d bytes", max_w, ubuf);
  prm.ubuf = ubuf;
  const size_t smem = static_cast<size_t>(ubuf) * (1 + 2 * kWarps) + static_cast<size_t>(prm.t.B + 1) * sizeof(int);
  static SmemCache cache;
  if (int rc = ensure_dynamic_smem(reinterpret_cast<const void *>(mask_expand_bits_kernel<kWarps>), &cache,
                                   dev.device, static_cast<int>(smem)))
    return rc;
  mask_expand_bits_kernel<kWarps><<<dev.sms, kWarps * 32, smem, st>>>(prm);
  MRX_LAUNCH_CHECK("mask_expand_bits_kernel");
  return MRX_OK;
}

extern "C" int mrx_mask_expand_packed(const float *d_tiles, const int *d_tile_index,
                                      const int *d_boxes, const int *d_counts,
                                      const int *d_geom, const long long *d_packed_off,
                                      unsigned char *d_packed, int B, int R, int mh, int mw,
                                      int max_w, unsigned int *d_sched, void *stream) {
  using namespace mrx::bits;
  const TileBatch t{d_tiles, d_tile_index, reinterpret_cast<const int4 *>(d_boxes), d_counts,
                    d_geom, B, R, mh, mw};
  const char *fn = "mrx_mask_expand_packed";
  if (int rc = check_tile_batch(fn, t, MRX_MAX_LANE_MASK_W)) return rc;
  if (int rc = check_slots(fn, d_packed, d_packed_off, d_counts, d_geom, B, R)) return rc;
  MRX_CHECK_ARG(d_sched, "%s: null pointer", fn);
  MRX_CHECK_ARG(max_w >= 1, "%s: bad max_w %d", fn, max_w);
  if (B == 0) return MRX_OK;
  DevInfo dev;
  if (int rc = current_device_info(&dev)) return rc;
  const BitsParams prm{t, {d_packed, d_packed_off}, d_sched, 0};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#ifdef MRX_DEV
  if (const char *e = getenv("MRX_BITS_WARPS")) {
    const int w = atoi(e);
    if (w == 8) return launch_bits<8>(prm, dev, max_w, st);
    if (w == 16) return launch_bits<16>(prm, dev, max_w, st);
    if (w == 24) return launch_bits<24>(prm, dev, max_w, st);
    if (w == 32) return launch_bits<32>(prm, dev, max_w, st);
  }
#endif
  return launch_bits<MRX_BITS_WARPS_DEFAULT>(prm, dev, max_w, st);
}
