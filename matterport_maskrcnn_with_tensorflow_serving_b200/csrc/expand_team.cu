// expand_team.cu -- the mask-expand kernel (the hot kernel of the path): 2-D canvas tiles built by
// TEAMS of warps, one role per warp and three named barriers per tile.
//
// Why: the store pattern alone (shared memory -> HBM bulk copies of k x 3200 B, no box work)
// runs at the HBM write rate (tools/store_ceiling.cu); a warp-specialised producer / consumer /
// store-warp design over mbarrier rings (an earlier version, removed) fell well short: its producer warps
// -- one dependent instruction stream listing (box,row) entries and issuing a TMA load per
// entry -- were the critical path.  Here a tile is kTileRows canvas rows high, so a
// box meets a tile once (not once per row); the horizontal source coordinate of a 32-column
// block is computed once and reused for every row; the bilinear sample is evaluated as
//   v = ht + wy * (hb - ht),   ht / hb = horizontal interpolation of source rows j / j+1
// so that consecutive canvas rows share ht, hb until the source row advances; and the tile rows
// come straight from L2 (the packed tiles of an image are 3136 B each).
//
//   CTA  = kTeams teams x kTeamWarps warps, one persistent CTA per SM
//   team = owns ONE tile buffer in shared memory and loops over tiles handed out by a global
//          counter (box density varies over the canvas: a static assignment leaves a tail):
//            B1 | warp 0   : bulk-store the finished tile, one row per lane
//               |            (cp.async.bulk.global.shared::cta), wait until the buffer is read
//               | last warp: fetch + decode the tile after next
//               | others   : cull the boxes of the next tile into the team's entry list
//            B2 | all      : zero the buffer  (this IS the canvas zero fill)
//            B3 | all      : items = (entry, 32-column block), dealt round robin to the warps:
//               |            fetch four (or six) tile rows, interpolate them horizontally with two
//               |            warp shuffles each, then walk the canvas rows: one FFMA, one
//               |            compare, one st.shared.u8 per row, the (ht, hb) pair advancing
//               |            through a register queue by predicate -- straight-line code
//          While one team waits for its buffer to drain, the other teams compute.
//
// A tile is P pixels x kTileRows rows of one image: row r is P*N contiguous canvas bytes
// (N innermost).  When W*N is a multiple of 16 every row segment is 16-byte aligned and is
// stored by one bulk copy.  Otherwise ("flat" shapes, e.g. W = 1333 with ragged N) each row is
// placed in shared memory at the same offset mod 16 as its global address, the 16-byte
// aligned body goes out as a bulk copy and the <= 15 head / tail bytes as byte stores.
// HBM sees every canvas byte written exactly once either way.
//
// The same kernel template is instantiated a second time with kValues = true
// (mrx_mask_expand_values): identical cull / hrow / walk code, plus a float store of every
// pre-threshold sample -- the parity tests check the 1e-6 value contract on THIS code.
//
// Development builds only (-DMRX_DEV via MRX_NVCC_FLAGS; never in the shipped library):
// MRX_EXPAND_FLAGS 0x100 no items, 0x200 no zero fill, 0x400 no store;
// MRX_EXPAND_TEAMS=<teams>x<warps>x<rows> picks another compiled shape; -DMRX_TEAM_PROFILE adds
// per-phase cycle counts (tools/team_profile.py).
#include <stdlib.h>
#include <string.h>

#include <type_traits>

#include "expand.cuh"

namespace mrx {

namespace team {

constexpr int kMaxP = 2048;   // tile width limit in pixels (64 column blocks; small N only)
constexpr int kCand = 128;   // boxes tested per cull pass == capacity of the entry list

// One box that meets the tile, with everything about it that is the same for all of its
// column blocks (written once by the culling lane).
struct __align__(16) TEntry {
  int x1, x2;    // box columns
  int npk;       // n | tile << 8 | ra << 16 | rb << 22 : instance, its tile's index, first and
                 // one-past-last tile row in the box
  float invD;    // 1 / (2 * box width)
  int Dy;        // 2 * box height
  float invDy;   // 1 / Dy
  int j0a;       // floor of the vertical source coordinate of tile row ra, in [-1, mh-1]
  int remya;     // its remainder: (coordinate - j0a) * Dy
};

struct __align__(16) TJob {
  const float *tiles_b;
  const int4 *boxes_b;
  unsigned char *g0;   // global address of (row y0, pixel x0, instance 0)
  int valid;
  int N, H, W;
  int x0, pw;          // first pixel and width in pixels
  int y0, kk;          // first row and number of rows
  int pitch;           // shared-memory distance between tile rows (multiple of 16)
  unsigned RW;         // canvas row bytes W * N
  int ident;           // instance k's tile is tile k (no row was dropped): skip the index lookup
  int pad1_;
};

// Tile geometry of an image: tile width in pixels and the shared-memory row pitch.
// `rowcap` = buffer bytes / tile rows (a multiple of 16).
// A warp draws 32 columns at a time, so a tile is a whole number of 32-column blocks -- plus a
// last partial block when that adds at least half a block: at N = 55 a row holds 62 pixels, and
// 32 + 30 columns fill the buffer (and amortise the per-tile costs) twice as well as 32 alone.
__device__ __forceinline__ int whole_blocks(int p) {
  if (p < 32) return p;
  return (p & 31) >= 16 ? p : (p & ~31);
}

__device__ __forceinline__ void tile_geom(int W, int N, int rowcap, int &P, int &pitch) {
  const unsigned RW = static_cast<unsigned>(W) * N;
  if ((RW & 15u) == 0u) {
    // pixel granularity that keeps P*N a multiple of 16: 16 / gcd(N, 16)
    const int m = 16 / (((N | 16) & -(N | 16)));   // lowest set bit of N|16 == gcd(N,16)
    int p = (rowcap / N) / m * m;
    if (p > kMaxP) p = kMaxP;   // a multiple of 16, hence of m
    p = whole_blocks(p);        // (stays a multiple of m: m divides 16 and 32)
    if (p < m) p = m;           // the host checks 16 * R * kTileRows <= buffer
    if (p >= W) p = W;
    P = p;
    pitch = p * N;              // multiple of 16 (p multiple of m, or p = W with RW % 16 == 0)
  } else {
    int p = (rowcap - 32) / N;
    if (p > kMaxP) p = kMaxP;
    p = whole_blocks(p);
    if (p < 1) p = 1;
    if (p >= W) p = W;
    P = p;
    pitch = ((p * N + 15) & ~15) + 16;   // room for the alignment shift (<= 15) of a row
  }
}

__device__ __forceinline__ int tiles_of(int H, int W, int N, int rowcap, int tile_rows) {
  if (N <= 0 || H <= 0 || W <= 0) return 0;
  int P, pitch;
  tile_geom(W, N, rowcap, P, pitch);
  return ((W + P - 1) / P) * ((H + tile_rows - 1) / tile_rows);
}

// ---- phase profile (build with -DMRX_TEAM_PROFILE): per-warp cycle totals of the six phases
// of a team's tile loop, read back with mrx_debug_team_profile()
#ifdef MRX_TEAM_PROFILE
constexpr int kProfCtas = 256;   // CTAs (= SMs) the profile has room for
__device__ long long g_team_prof[kProfCtas * 32 * 12];
#define PROF_DECL long long prof_t = clock64(), prof_acc[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
#define PROF_ADD(k, v) prof_acc[k] += (v);
#define PROF_NOW clock64()
#define PROF_MARK(k)                         \
  {                                          \
    const long long now_ = clock64();        \
    prof_acc[k] += now_ - prof_t;            \
    prof_t = now_;                           \
  }
#define PROF_FLUSH                                                                   \
  if (lane == 0 && blockIdx.x < kProfCtas && warp < 32) {                            \
    for (int k_ = 0; k_ < 12; ++k_)                                                  \
      g_team_prof[(blockIdx.x * 32 + warp) * 12 + k_] = prof_acc[k_];                \
  }
#else
#define PROF_DECL
#define PROF_MARK(k)
#define PROF_FLUSH
#define PROF_ADD(k, v)
#define PROF_NOW 0
#endif

#ifdef MRX_DEV
#define MRX_FLAG(p, bit) ((p).flags & (bit))
#else
#define MRX_FLAG(p, bit) 0
#endif

// The next tile ticket, drawn a tile before it is used.  The counter is kept as a FLOAT while
// the launch has fewer than 2^24 tiles (tickets are exact): ptxas turns an integer atomic add of
// a constant into its warp-aggregated form (vote, popc, shuffle), and the shuffle reads the
// returned value at once, which puts the counter's round trip through a store-saturated L2 on
// the team's path.  It leaves a float add alone.  Zero is zero in both formats (the reset at the
// end of every launch, the memset).  Returns raw bits; ticket_value() converts where the ticket
// is used (a conversion next to the atomic would wait for it).
__device__ __forceinline__ unsigned draw_ticket(unsigned int *counter, bool as_float) {
  unsigned v;
  if (as_float)
    asm volatile("atom.global.add.f32 %0, [%1], 0f3F800000;" : "=r"(v) : "l"(counter) : "memory");
  else
    v = atomicAdd(counter, 1u);
  return v;
}
__device__ __forceinline__ int ticket_value(unsigned raw, bool as_float) {
  return as_float ? static_cast<int>(__uint_as_float(raw)) : static_cast<int>(raw);
}

__device__ __forceinline__ void team_bar(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// kValues: also store every pre-threshold sample as float (test instantiation, see the header).
template <int kTeams, int kTeamWarps, int kTileRows, bool kValues>
__global__ void __launch_bounds__(kTeams * kTeamWarps * 32, 1)
mask_expand_team_kernel(const ExpandParams p, const int buf_bytes) {
  static_assert(kTileRows <= 32 && kTeamWarps >= 3, "one store lane per tile row; cull + decode warps");
  static_assert(2 * kTeams + 1 <= 16, "two named barriers per team");
  extern __shared__ __align__(128) unsigned char smem[];
  constexpr int kTeamThreads = kTeamWarps * 32;
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int warp = tid >> 5;
  const int tm = warp / kTeamWarps;            // team
  const int wt = warp - tm * kTeamWarps;       // warp within the team
  const int tt = tid - tm * kTeamThreads;      // thread within the team
  const int mh = p.t.mh, mw = p.t.mw;
  const int rowcap = (buf_bytes / kTileRows) & ~15;

  // ---- carve shared memory: [team buffers][team entry lists][team job descriptors][prefix]
  unsigned char *s_buf = smem + static_cast<size_t>(tm) * buf_bytes;
  TEntry *s_ent = reinterpret_cast<TEntry *>(smem + static_cast<size_t>(kTeams) * buf_bytes) + tm * kCand;
  TJob *s_job = reinterpret_cast<TJob *>(smem + static_cast<size_t>(kTeams) * buf_bytes +
                                         static_cast<size_t>(kTeams) * kCand * sizeof(TEntry)) + tm * 2;
  int *s_prefix = reinterpret_cast<int *>(smem + static_cast<size_t>(kTeams) * buf_bytes +
                                          static_cast<size_t>(kTeams) * kCand * sizeof(TEntry) +
                                          static_cast<size_t>(kTeams) * 2 * sizeof(TJob));
  __shared__ int s_total;
  __shared__ int s_ecount[kTeams][2];
  __shared__ unsigned char s_hit[kTeams][kCand];   // box index - cbase of every hit of a cull pass

  // ---- tiles per image -> prefix sums (first warp)
  if (warp == 0) {
    image_work_table(p.t.B, [=](int b) {
      return tiles_of(p.t.geom[b * MRX_GEOM_INTS + 0], p.t.geom[b * MRX_GEOM_INTS + 1], p.t.counts[b], rowcap, kTileRows);
    }, s_prefix, &s_total);
  }
  __syncthreads();
  const int total = s_total;
  const int bar_id = 1 + tm;
  const uint32_t buf_addr = smem_u32(s_buf);

  // decode tile `j` into *out (one thread); cur_b is the caller's search cursor
  // (per-image constants live in shared memory: registers would cost every thread)
  struct DecodeCache {
    unsigned char *canvas;
    int b, H, W, N, P, pitch, tx, ident;
  };
  __shared__ DecodeCache s_dc[kTeams];
  DecodeCache &dc = s_dc[tm];
  auto decode = [&](int j, int &cur_b, TJob *out) {
    if (j >= total) {
      out->valid = 0;
      return;
    }
    while (j >= s_prefix[cur_b + 1]) ++cur_b;
    const int b = cur_b;
    if (b != dc.b) {   // per-image constants (divisions), kept by the decoding thread
      dc.b = b;
      dc.H = p.t.geom[b * MRX_GEOM_INTS + 0];
      dc.W = p.t.geom[b * MRX_GEOM_INTS + 1];
      dc.N = p.t.counts[b];
      int P_, pitch_;
      tile_geom(dc.W, dc.N, rowcap, P_, pitch_);
      dc.P = P_;
      dc.pitch = pitch_;
      dc.tx = (dc.W + P_ - 1) / P_;
      dc.canvas = p.canvas.base + p.canvas.off[b];
      // kept rows are in increasing order: no row was dropped iff the last one kept its index
      dc.ident = dc.N == 0 || p.t.tile_index[static_cast<size_t>(b) * p.t.R + dc.N - 1] == dc.N - 1;
    }
    const int H = dc.H, W = dc.W, N = dc.N, P = dc.P, pitch = dc.pitch, tiles_x = dc.tx;
    const int local = j - s_prefix[b];
    const int band = local / tiles_x;
    const int tx = local - band * tiles_x;
    const unsigned RW = static_cast<unsigned>(W) * N;
    out->tiles_b = p.t.tiles + static_cast<size_t>(b) * p.t.R * mh * mw;
    out->boxes_b = p.t.boxes + static_cast<size_t>(b) * p.t.R;
    out->x0 = tx * P;
    out->pw = min(P, W - tx * P);
    out->y0 = band * kTileRows;
    out->kk = min(kTileRows, H - band * kTileRows);
    out->g0 = dc.canvas + static_cast<size_t>(band * kTileRows) * RW +
              static_cast<size_t>(tx * P) * N;
    out->N = N;
    out->H = H;
    out->W = W;
    out->pitch = pitch;
    out->RW = RW;
    out->ident = dc.ident;
    out->valid = 1;
  };

  // cull the boxes [cbase, cbase + kCand) of tile `jb` into the team's entry list, by the warps
  // w0 = 0 .. wstep-1 of the team.  Two steps: every warp tests 32 boxes per trip and appends the
  // hits to a byte list; after a barrier among the culling warps the per-entry arithmetic (two
  // divisions, the exact vertical source coordinate) runs once per 32 hits instead of once per
  // trip that happened to contain a hit.
  auto cull = [&](const TJob &jb, int cslot, int cbase, int w0, int wstep) {
    for (int c = w0 * 32; c < kCand; c += wstep * 32) {
      const int n = cbase + c + lane;
      bool hit = false;
      if (n < jb.N) {
        const int4 bx = __ldg(jb.boxes_b + n);
        // box_in_canvas() spelled out: the call changes this kernel's code generation
        const bool sane = bx.x >= 0 && bx.y >= 0 && bx.z <= jb.H && bx.w <= jb.W && bx.z > bx.x &&
                          bx.w > bx.y;
        hit = sane && bx.y < jb.x0 + jb.pw && bx.w > jb.x0 && bx.x < jb.y0 + jb.kk && bx.z > jb.y0;
      }
      const unsigned bal = __ballot_sync(0xffffffffu, hit);
      if (bal != 0u) {
        int slot = 0;
        if (lane == 0) slot = atomicAdd(&s_ecount[tm][cslot], __popc(bal));
        slot = __shfl_sync(0xffffffffu, slot, 0) + __popc(bal & ((1u << lane) - 1u));
        if (hit) s_hit[tm][slot] = static_cast<unsigned char>(c + lane);
      }
    }
    team_bar(1 + kTeams + tm, wstep * 32);   // the culling warps only
    const int E = s_ecount[tm][cslot];
    for (int h = w0 * 32 + lane; h < E; h += wstep * 32) {
      const int n = cbase + s_hit[tm][h];
      const int4 bx = __ldg(jb.boxes_b + n);
      const int bh = bx.z - bx.x;
      const int ra = max(bx.x, jb.y0) - jb.y0, rb = min(bx.z, jb.y0 + jb.kk) - jb.y0;
      TEntry e;
      e.x1 = bx.y;
      e.x2 = bx.w;
      const int tile = jb.ident ? n : __ldg(p.t.tile_index + (jb.boxes_b - p.t.boxes) + n);
      e.npk = n | (tile << 8) | (ra << 16) | (rb << 22);
      e.invD = __fdiv_rn(1.0f, static_cast<float>(2 * (bx.w - bx.y)));
      e.Dy = 2 * bh;
      e.invDy = __fdiv_rn(1.0f, static_cast<float>(2 * bh));
      const SrcPos sy = src_floor(src_num(mh, jb.y0 + ra, bx.x, bh), e.Dy, e.invDy);   // tile row ra
      e.j0a = sy.i;
      e.remya = sy.rem;
      s_ent[h] = e;
    }
  };

  // ---- prologue of the pipeline: decode the first two tiles, cull the first
  // (the team's last warp decodes, its first warp stores, the ones between cull)
  int cur_b = 0;   // search cursor of decode(); meaningful in the decoding thread only
  // The decoding lane holds one ticket ahead of the descriptor it fills: the counter's round trip
  // through an L2 that is saturated with stores takes thousands of cycles (the decode warp used
  // to reach the tile barrier after the storing warp); drawn a tile early, it is off the path.
  unsigned ticket = 0u;   // raw bits, see draw_ticket()
  const bool float_tickets = total < (1 << 24) - 4 * static_cast<int>(gridDim.x) * kTeams;   // (+ the draws past the end)
  if (wt == kTeamWarps - 1 && lane == 0) {
    // tiles are handed out by a global counter (reset by mrx_unmold_prepare): box density
    // varies across the canvas, a static assignment leaves a tail of late teams
    const int t0 = ticket_value(draw_ticket(p.job_counter, float_tickets), float_tickets);
    const int t1 = ticket_value(draw_ticket(p.job_counter, float_tickets), float_tickets);
    ticket = draw_ticket(p.job_counter, float_tickets);
    dc.b = -1;
    decode(t0, cur_b, &s_job[0]);
    decode(t1, cur_b, &s_job[1]);
    s_ecount[tm][0] = 0;
    s_ecount[tm][1] = 0;
    if (ticket == 0xffffffffu) p.job_counter[0] = 0u;   // (never true) all three tickets are drawn: see the end
  }
  team_bar(bar_id, kTeamThreads);
  // the workers are the teams
  if (!s_job[0].valid) {   // fewer tiles than teams: nothing for this team
    if (tt == 0) retire_worker(p.job_counter, kTeams);
    return;
  }
  cull(s_job[0], 0, 0, wt, kTeamWarps);

  int slot = 0;      // s_job[slot] / s_ecount[tm][slot] belong to the tile being drawn
  PROF_DECL
  while (true) {
    // ================= B2: entry list of this tile complete, buffer drained
    PROF_MARK(5)
    team_bar(bar_id, kTeamThreads);
    PROF_MARK(0)
    const TJob *jp = &s_job[slot];
    const int N = jp->N, x0 = jp->x0, pw = jp->pw, y0 = jp->y0, kk = jp->kk, pitch = jp->pitch;
    const unsigned RW = jp->RW;
    unsigned char *const g0 = jp->g0;
    const float *const tiles_b = jp->tiles_b;
    if (tt == 0) s_ecount[tm][slot ^ 1] = 0;   // the next tile's counter (idle since tile j-1)
    // canvas zero fill (fixed trip count: predicated stores, no loop bookkeeping)
    if (!MRX_FLAG(p, 0x200)) {
      uint4 *o4 = reinterpret_cast<uint4 *>(s_buf);
      const int rem = ((kk * pitch) >> 4) - tt;   // 16-byte words from this thread's first one on
      // the largest tile buffer a team can get (232 448 B of shared memory per CTA)
      constexpr int kMaxBuf = (232448 - kTeams * (kCand * static_cast<int>(sizeof(TEntry)) +
                                                  2 * static_cast<int>(sizeof(TJob)))) / kTeams;
      constexpr int kMaxZero = (kMaxBuf / 16 + kTeamThreads - 1) / kTeamThreads;
#pragma unroll
      for (int k = 0; k < kMaxZero; ++k)
        if (k * kTeamThreads < rem) o4[tt + k * kTeamThreads] = make_uint4(0u, 0u, 0u, 0u);
    }
    int cbase = 0;
    PROF_MARK(1)
    while (true) {
      // ================= B3: buffer zeroed / entry list of this pass complete
      team_bar(bar_id, kTeamThreads);
      PROF_MARK(2)
      const int E = MRX_FLAG(p, 0x100) ? 0 : s_ecount[tm][slot];
      // ---- items: (entry, 32-column block) pairs, item i = entry * nblk + block, dealt round
      // robin to the team's warps (at N = 100 a tile is one block wide and an item is an entry)
      const int nblk = (pw + 31) >> 5;
      const bool lanecol = lane >= 1 && lane <= mw;
      const int lcol = min(max(lane - 1, 0), mw - 1);
      const int a0 = static_cast<int>(reinterpret_cast<uintptr_t>(g0) & 15u);
      const int rw15 = static_cast<int>(RW & 15u);
      const bool aligned = (a0 | rw15) == 0;   // every tile row starts 16-byte aligned
      int ei = 0, c = wt;                      // this warp's next item
      if (nblk == 1) {
        ei = wt;
        c = 0;
      }
      while (true) {
        if (nblk == 1) {
          if (c != 0) {   // c was advanced by kTeamWarps
            ei += kTeamWarps;
            c = 0;
          }
        } else {
          while (c >= nblk) {
            c -= nblk;
            ++ei;
          }
        }
        if (ei >= E) break;
        const long long it_t0 = PROF_NOW;
        const int4 ea = *reinterpret_cast<const int4 *>(&s_ent[ei]);          // x1, x2, npk, invD
        const int xa = max(ea.x, x0), xb = min(ea.y, x0 + pw);
        const int xc = x0 + (c << 5);
        c += kTeamWarps;
        if (xc + 32 <= xa || xc >= xb) continue;                              // block outside the box
        const int4 eb = *(reinterpret_cast<const int4 *>(&s_ent[ei]) + 1);    // Dy, invDy, j0a, remya
        const float invD = __int_as_float(ea.w), invDy = __int_as_float(eb.y);
        const int Dy = eb.x;
        const int n = ea.z & 0xff, tile = (ea.z >> 8) & 0xff, ra = (ea.z >> 16) & 63,
                  rb = (ea.z >> 22) & 63;
        const int x = xc + lane;
        const bool colvalid = x >= xa && x < xb;
        // exact horizontal source coordinate of this lane's column: taps idx, idx + 1 of the
        // zero-padded tile row in lane-column layout, weight wx
        const int D = 2 * (ea.y - ea.x);
        const SrcPos sx = src_floor(src_num(mw, x, ea.x, ea.y - ea.x), D, invD);
        const int idx = sx.i + 1;
        const float wx = src_weight(sx.rem, invD);
        const float *tp = tiles_b + static_cast<unsigned>(tile * mh * mw + lcol);
        const LaneRows raw{tp, mh, mw, lanecol};
        // the bilinear sample is  ht + wy * (hb - ht)  with ht, hb the horizontal interpolations
        // of source rows jcur, jcur + 1; consecutive canvas rows share them until the source row
        // advances
        int jcur = eb.z, remy = eb.w;
        uint32_t addr = buf_addr + static_cast<uint32_t>(ra * pitch + (x - x0) * N + n);
        const int cnt = rb - ra;
        // kValues: where the sample of (tile row ra, this lane's column, instance n) goes
        [[maybe_unused]] float *vout = nullptr;
        if (kValues)
          vout = p.values + (g0 - p.canvas.base) + static_cast<size_t>(ra) * RW +
                 static_cast<size_t>(x - x0) * N + n;
        int step = 2 * mh;
        // the byte every set sample stores: 1, derived from a value ptxas cannot fold (the sign
        // bit of a pitch), or it re-materialises the constant (and a byte merge) in front of
        // every one of the row stores
        unsigned one = 1u ^ (static_cast<unsigned>(pitch) >> 31);
        asm volatile("" : "+r"(step));   // one register, not a constant-bank read per row
        if (Dy > step && remy + (cnt - 1) * step < 5 * Dy) {
          // ---- the common case: a box tall enough that the tile meets at most 6 of its source
          // rows (jcur .. jcur+5).  Straight-line, branch-free: the rows are fetched and
          // interpolated horizontally up front (four of them, six when more than two advances
          // are possible inside the tile); the canvas rows then walk a register queue
          // (ht, hb, q2, q3 [, q4, q5]) that shifts by predicate when the source row advances.
          // Rows past the box (i >= cnt) are predicated off.
          // rows jcur .. jcur+5 of the tile in lane-column layout; row k is real when
          // 0 <= jcur + k < mh (only k = 0 can be the zero row above the tile: jcur >= -1)
          const int lim = lanecol ? mh - jcur : 0;   // row k is inside the tile iff k < lim
          const float *pr = tp + static_cast<unsigned>(max(jcur, 0) * mw);
          // most boxes are tall enough that the tile meets only jcur .. jcur+3 (at most two
          // advances): fetch and interpolate rows 4 and 5 only when they can be reached
          const bool deep = remy + (cnt - 1) * step >= 3 * Dy;   // warp-uniform
          float r0 = 0.f, r1 = 0.f, r2 = 0.f, r3 = 0.f, r4 = 0.f, r5 = 0.f;
          if (jcur >= 0) {
            if (0 < lim) r0 = __ldg(pr);
            pr += mw;
          }
          if (1 < lim) r1 = __ldg(pr);
          if (2 < lim) r2 = __ldg(pr + mw);
          if (3 < lim) r3 = __ldg(pr + 2 * mw);
          if (deep && 4 < lim) r4 = __ldg(pr + 3 * mw);
          if (deep && 5 < lim) r5 = __ldg(pr + 4 * mw);
          const float thr = colvalid ? 0.5f : __int_as_float(0x7f800000);
          float ht = hrow(r0, idx, wx), hb = hrow(r1, idx, wx), q2 = hrow(r2, idx, wx),
                q3 = hrow(r3, idx, wx);
          float dh = hb - ht;
          const long long it_t1 = PROF_NOW;
          PROF_ADD(8, it_t1 - it_t0)
          PROF_ADD(10, 1)
          PROF_ADD(11, cnt)
          // The vertical weight of a tile row is the same for all 32 columns, so lane i computes
          // it for row i (and how many source rows lie before it) once per item; the rows then
          // take it with a shuffle instead of each lane redoing the integer walk (9 % fewer
          // instructions per launch; the time did not move: the kernel is not issue-bound).
          // Rows past the box get a NaN weight: their sample compares false.
          float wl;
          unsigned advmask;
          {
            const SrcPos s = src_floor(remy + lane * step, Dy, invDy);   // rows past jcur
            wl = lane < cnt ? src_weight(s.rem, invDy) : __int_as_float(0x7fc00000);
            // bit i: the source row advances between tile rows i and i + 1 (Dy > step: by one)
            advmask = __ballot_sync(0xffffffffu, __shfl_down_sync(0xffffffffu, s.i, 1) != s.i);
          }
          auto walk = [&](auto aligned_tag, auto deep_tag) {
            constexpr bool kAligned = decltype(aligned_tag)::value;
            constexpr bool kDeep = decltype(deep_tag)::value;
            float q4 = 0.f, q5 = 0.f;
            if (kDeep) {
              q4 = hrow(r4, idx, wx);
              q5 = hrow(r5, idx, wx);
            }
            int sh = kAligned ? 0 : ((a0 + ra * rw15) & 15);   // row address mod 16 in HBM
#pragma unroll
            for (int i = 0; i < kTileRows; ++i) {
              const float v = fmaf(__shfl_sync(0xffffffffu, wl, i), dh, ht);
              if (v >= thr)
                asm volatile("st.shared.u8 [%0], %1;" ::"r"(addr + static_cast<uint32_t>(sh)), "r"(one));
              const bool adv = (advmask >> i) & 1u;      // warp-uniform, applied as a predicate
              if (kValues) {
                if (colvalid && i < cnt) vout[static_cast<size_t>(i) * RW] = v;
              }
              addr += static_cast<uint32_t>(pitch);
              if (!kAligned) sh = (sh + rw15) & 15;
              ht = adv ? hb : ht;
              hb = adv ? q2 : hb;
              q2 = adv ? q3 : q2;
              if (kDeep) {
                q3 = adv ? q4 : q3;
                q4 = adv ? q5 : q4;
              }
              dh = hb - ht;
            }
          };
          if (aligned) {
            if (deep) walk(std::true_type{}, std::true_type{});
            else walk(std::true_type{}, std::false_type{});
          } else {
            if (deep) walk(std::false_type{}, std::true_type{});
            else walk(std::false_type{}, std::false_type{});
          }
          PROF_ADD(9, PROF_NOW - it_t1)
          continue;
        }
        float rawn = raw(jcur + 2);
        float ht = hrow(raw(jcur), idx, wx), hb = hrow(raw(jcur + 1), idx, wx);
        float dh = hb - ht;
        // ---- general case: any box height, any alignment
        const SrcStep ystep = src_step(2 * mh, Dy);   // source-row advance per canvas row
        int j0 = jcur;
        int sh = (a0 + ra * rw15) & 15;
        for (int r = ra; r < rb; ++r) {
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
          if (v >= 0.5f && colvalid)
            asm volatile("st.shared.u8 [%0], %1;" ::"r"(addr + static_cast<uint32_t>(sh)), "r"(1u));
          if (kValues) {
            if (colvalid) vout[static_cast<size_t>(r - ra) * RW] = v;
          }
          addr += static_cast<uint32_t>(pitch);
          sh = (sh + rw15) & 15;
          // src_advance() spelled out: the call changes this kernel's code generation
          remy += ystep.r;
          j0 += ystep.q;
          if (remy >= Dy) {
            remy -= Dy;
            ++j0;
          }
        }
      }
      cbase += kCand;
      if (cbase >= N) break;
      // more boxes than one pass holds (N > kCand): another pass over the same tile
      team_bar(bar_id, kTeamThreads);   // everyone is done with the entry list
      if (tt == 0) s_ecount[tm][slot] = 0;
      team_bar(bar_id, kTeamThreads);
      cull(*jp, slot, cbase, wt, kTeamWarps);
    }
    PROF_MARK(3)
    fence_proxy_async_smem();   // this thread's tile bytes -> visible to the bulk copies

    // ================= B1: tile complete
    team_bar(bar_id, kTeamThreads);
    PROF_MARK(4)
    const int nslot = slot ^ 1;
    const bool more = s_job[nslot].valid != 0;
    if (wt == 0) {
      // ---- store the tile: lane r owns the bulk copy of row r (its 16-byte aligned body)
      const bool mine = lane < kk;
      const int len = pw * N;
      if (mine && !MRX_FLAG(p, 0x400)) {
        unsigned char *g = g0 + static_cast<size_t>(lane) * RW;
        const int a = static_cast<int>(reinterpret_cast<uintptr_t>(g) & 15u);
        unsigned char *s = s_buf + lane * pitch + a;
        const int head = min((16 - a) & 15, len);
        const int body = (len - head) & ~15;
        if (body > 0) {
          fence_proxy_async_smem();
          bulk_s2g(g + head, s + head, static_cast<uint32_t>(body));
          bulk_commit();
        }
      }
      // ---- unaligned shapes: the <= 15 head and <= 15 tail bytes of every row, one byte per
      // lane (generic-proxy copies; the bulk copies above only read the buffer)
      if (((reinterpret_cast<uintptr_t>(g0) | RW | static_cast<unsigned>(len)) & 15u) != 0u &&
          !MRX_FLAG(p, 0x400)) {
        for (int r = 0; r < kk; ++r) {
          unsigned char *g = g0 + static_cast<size_t>(r) * RW;
          const int a = static_cast<int>(reinterpret_cast<uintptr_t>(g) & 15u);
          const unsigned char *s = s_buf + r * pitch + a;
          const int head = min((16 - a) & 15, len);
          const int body = (len - head) & ~15;
          const int tail = len - head - body;
          if (lane < head + tail) {
            const int o = lane < head ? lane : body + lane;   // head + body + (lane - head)
            g[o] = s[o];
          }
        }
      }
      __syncwarp();
      PROF_MARK(6)
      // ---- the buffer may be re-zeroed once the bulk copies have read it
      if (mine) {
        if (more) bulk_wait_read<0>();
        else bulk_wait_all<0>();
      }
    } else if (more) {
      if (wt == kTeamWarps - 1) {
        // ---- the descriptor of this tile retires: decode the tile after next into it
        if (lane == 0) {
          const int mine = ticket_value(ticket, float_tickets);
          ticket = draw_ticket(p.job_counter, float_tickets);   // used one tile from now
          decode(mine, cur_b, &s_job[slot]);
        }
        __syncwarp();
        PROF_MARK(7)
      } else {
        cull(s_job[nslot], nslot, 0, wt - 1, kTeamWarps - 2);
      }
    }
    if (!more) break;
    slot = nslot;
  }
  // the decoding lane's last ticket must have been drawn before the team retires (the last team
  // of the grid zeroes the counter): reading its value waits for it
  if (ticket == 0xffffffffu) p.job_counter[0] = 0u;   // (never true: not a ticket in either format)
  team_bar(bar_id, kTeamThreads);
  if (tt == 0) retire_worker(p.job_counter, kTeams);
  PROF_MARK(5)
  PROF_FLUSH
}

}  // namespace team

template <int kTeams, int kTeamWarps, int kTileRows, bool kValues>
static int launch_team_cfg(const ExpandParams &prm, const DevInfo &dev, int want_buf, cudaStream_t st) {
  using namespace team;
  const int max_optin = dev.max_smem_optin;
  constexpr size_t kStatic = 256 + static_cast<size_t>(kTeams) * (kCand + 48);   // static __shared__ of the kernel
  const size_t fixed = static_cast<size_t>(kTeams) * kCand * sizeof(TEntry) +
                       static_cast<size_t>(kTeams) * 2 * sizeof(TJob) +
                       static_cast<size_t>(prm.t.B + 1) * sizeof(int) + kStatic;
  MRX_CHECK_SUPPORTED(fixed + static_cast<size_t>(kTeams) * 2048 <= static_cast<size_t>(max_optin),
                      "mrx_mask_expand: batch of %d images does not fit the scheduler table", prm.t.B);
  // (the kernel's zero fill is unrolled for tile buffers of up to this size)
  constexpr int kMaxBuf = (232448 - kTeams * (kCand * static_cast<int>(sizeof(TEntry)) +
                                              2 * static_cast<int>(sizeof(TJob)))) / kTeams;
  const int avail = min(static_cast<int>((static_cast<size_t>(max_optin) - fixed) / kTeams), kMaxBuf) & ~127;
  // a tile row must hold 16 pixels of R instances (aligned shapes) / one pixel + alignment shift
  const int need = (max(16 * prm.t.R, prm.t.R + 48) * kTileRows + 127) & ~127;
  // (an entry packs the instance and its tile index into 8 bits each)
  if (need > avail || prm.t.R > 256) return MRX_E_UNSUPPORTED;   // caller falls back to the generic kernel
  int buf = avail;
  if (want_buf > 0 && want_buf < buf) buf = want_buf & ~127;
  if (buf < need) buf = need;
  const size_t smem = static_cast<size_t>(kTeams) * buf + fixed - kStatic;
  auto kern = mask_expand_team_kernel<kTeams, kTeamWarps, kTileRows, kValues>;
  static SmemCache cache;
  if (int rc = ensure_dynamic_smem(reinterpret_cast<const void *>(kern), &cache, dev.device,
                                   static_cast<int>(smem)))
    return rc;
  // the two scheduler words are zero here: the caller zeroed them once and every launch
  // (and mrx_unmold_prepare) leaves them zeroed
  kern<<<dev.sms, kTeams * kTeamWarps * 32, smem, st>>>(prm, buf);
  MRX_LAUNCH_CHECK("mask_expand_team_kernel");
  return MRX_OK;
}

#ifdef MRX_TEAM_PROFILE
extern "C" int mrx_debug_team_profile(long long *host_dst, int count) {
  MRX_CUDA(cudaDeviceSynchronize());
  MRX_CUDA(cudaMemcpyFromSymbol(host_dst, team::g_team_prof, sizeof(long long) * count));
  return MRX_OK;
}
#endif

// The shipped shape: 6 teams x 5 warps, 10-row tiles (tools/kernel_sweep.py compares the others).
int launch_expand_team(const ExpandParams &prm, const DevInfo &dev, int want_buf, cudaStream_t st) {
  if (prm.t.mw > MRX_MAX_LANE_MASK_W) return MRX_E_UNSUPPORTED;   // caller falls back to the generic kernel
  if (prm.values != nullptr) return launch_team_cfg<6, 5, 10, true>(prm, dev, want_buf, st);
#ifdef MRX_DEV
  // development sweep: MRX_EXPAND_TEAMS="<teams>x<warps>x<rows>"
  int teams = 6, warps = 5, rows = 10;
  if (const char *e = getenv("MRX_EXPAND_TEAMS")) {
    int a = 0, b = 0, c = 0;
    if (sscanf(e, "%dx%dx%d", &a, &b, &c) == 3) {
      teams = a;
      warps = b;
      rows = c;
    }
  }
#define MRX_TEAM_CASE(T, W, R) \
  if (teams == T && warps == W && rows == R) return launch_team_cfg<T, W, R, false>(prm, dev, want_buf, st)
  MRX_TEAM_CASE(4, 7, 16);
  MRX_TEAM_CASE(5, 5, 12);
  MRX_TEAM_CASE(5, 6, 12);
  MRX_TEAM_CASE(6, 4, 10);
  MRX_TEAM_CASE(6, 5, 10);
  MRX_TEAM_CASE(6, 5, 11);
  MRX_TEAM_CASE(7, 4, 9);
#undef MRX_TEAM_CASE
  set_error("mrx_mask_expand: MRX_EXPAND_TEAMS=%dx%dx%d is not a compiled shape", teams, warps, rows);
  return MRX_E_INVALID;
#else
  return launch_team_cfg<6, 5, 10, false>(prm, dev, want_buf, st);
#endif
}

}  // namespace mrx
