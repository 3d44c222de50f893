// jpeg.cu -- baseline JPEG decode on the device, bit for bit as cv2.imdecode (libjpeg-turbo,
// JDCT_ISLOW, fancy upsampling): mrx_jpeg_coefficients (unstuff, self-synchronising Huffman decode,
// DC prediction) and mrx_jpeg_pixels (islow IDCT, upsampling, colour, EXIF orientation).
//
// The host (jpeg.py) parses the headers and lays out the batch: a descriptor of int64 words per
// image (the D_* indices below mirror jpeg.py) and per image a table blob of 3 components x
// (quant int32[64] in natural order, DC table, AC table).  Every read is bounded by the sizes the
// descriptor gives; an image whose status word has a bit is skipped by the later kernels.
//
// Huffman decode (Weissenberger & Schmidt, ICPP 2018): each restart unit is cut into subsequences
// of S bits.  A decoder state at a codeword boundary is (bit position, block in MCU, zig-zag index).
// Every subsequence is decoded from a guessed start; inside a CTA each thread re-decodes from its
// predecessor's exit until nothing changes (subsequence 0 of a unit is exact, and every round fixes
// one more).  A per-image walk then fixes the first subsequences of the CTAs in order, re-decoding
// only until the stored exit state is met again.  No host loop, no inter-CTA waits.
#include "common.cuh"

namespace mrx {
namespace {

enum {
  D_FILE_OFF, D_FILE_LEN, D_SCAN_OFF, D_H, D_W, D_NCOMP, D_COLOR, D_ORIENT,
  D_HMAX, D_VMAX, D_MCUX, D_MCUY, D_BPM, D_RI, D_NUNITS,
  D_UNST_OFF, D_UNIT_BIT, D_UNIT_SUB, D_SUB_OFF, D_SUB_CAP, D_COEF_OFF, D_NBLOCKS,
  D_PLANE_OFF = 22, D_COMP_H = 25, D_COMP_V = 28, D_PLANE_BW = 31, D_PLANE_BH = 34, D_DW = 37,
  D_DH = 40, D_BLK_COMP = 43, D_BLK_DX = 53, D_BLK_DY = 63, D_UNIT_BASE = 73, DESC_WORDS = 80
};

constexpr int kFastBits = 9;
constexpr int kHuffBytes = 2 * (1 << kFastBits) + 4 * 18 + 4 * 18 + 256;
constexpr int kCompTabBytes = 4 * 64 + 2 * kHuffBytes;
constexpr int kTabBytes = 3 * kCompTabBytes;
constexpr int kThreads = 256;
constexpr int kSentinel = 0xFF00;        // exit state after an invalid code: block 255
constexpr int kFatal = MRX_JPEG_ST_RST | MRX_JPEG_ST_MARKER;

__constant__ unsigned char c_zigzag[80] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33,
    40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36,
    29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54,
    47, 55, 62, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63};

struct Huff {
  const unsigned short *lookup;
  const int *maxcode, *valptr;
  const unsigned char *vals;
};

__device__ __forceinline__ Huff huff_at(const unsigned char *p) {
  Huff h;
  h.lookup = reinterpret_cast<const unsigned short *>(p);
  h.maxcode = reinterpret_cast<const int *>(p + 2 * (1 << kFastBits));
  h.valptr = h.maxcode + 18;
  h.vals = p + 2 * (1 << kFastBits) + 4 * 36;
  return h;
}

// the 32 bits starting at bit p of the unstuffed stream (reads 5 bytes: the buffer is padded)
__device__ __forceinline__ uint32_t peek32(const unsigned char *u, uint32_t p) {
  const unsigned char *q = u + (p >> 3);
  const uint64_t v = (uint64_t(q[0]) << 32) | (uint64_t(q[1]) << 24) | (uint64_t(q[2]) << 16) |
                     (uint64_t(q[3]) << 8) | uint64_t(q[4]);
  return uint32_t(v >> (8 - (p & 7)));
}

// one codeword at the top of w: symbol and code length, or length 0 for a bad code
__device__ __forceinline__ int huff_decode(const Huff &h, uint32_t w, int &len) {
  const int f = h.lookup[w >> (32 - kFastBits)];
  if (f) {
    len = f >> 8;
    return f & 255;
  }
  const int code16 = int(w >> 16);
#pragma unroll 1
  for (int l = kFastBits + 1; l <= 16; ++l) {
    const int code = code16 >> (16 - l);
    if (code <= h.maxcode[l]) {
      len = l;
      return h.vals[h.valptr[l] + code];
    }
  }
  len = 0;
  return 0;
}

__device__ __forceinline__ int huff_extend(uint32_t r, int s) {
  return int(r) < (1 << (s - 1)) ? int(r) - (1 << s) + 1 : int(r);
}

// The per-image context the decode loops need, loaded once per thread.
struct Ctx {
  const unsigned char *u;          // image's unstuffed stream
  const unsigned char *tabs;       // image's table blob
  unsigned char comp[10];          // component of each block of the MCU
  int bpm;
};

__device__ __forceinline__ void load_ctx(Ctx &c, const long long *D, const unsigned char *unst,
                                         const unsigned char *tabs, int b) {
  c.u = unst + D[D_UNST_OFF];
  c.tabs = tabs + size_t(b) * kTabBytes;
  c.bpm = int(D[D_BPM]);
  for (int i = 0; i < 10; ++i) c.comp[i] = i < c.bpm ? (unsigned char)D[D_BLK_COMP + i] : 0;
}

// Decode from state (p, cz = block << 8 | zig-zag) while p < end.  Counts the blocks started.
// kWrite: also write the coefficients of blocks [next_blk - (z > 0), limit) and flag codes that
// run past unit_end.  Returns a status bit (0, MRX_JPEG_ST_CODE, MRX_JPEG_ST_TRUNC).
template <bool kWrite>
__device__ int decode_span(const Ctx &c, uint32_t &p, int &cz, uint32_t end, uint32_t unit_end,
                           int &blocks, int &next_blk, int limit, short *coef) {
  int blk = cz >> 8, z = cz & 255;
  int cur = next_blk - 1;
#pragma unroll 1
  while (p < end) {
    if (kWrite && (z == 0 ? next_blk : cur) >= limit) break;   // past the unit's last block
    const unsigned char *ct = c.tabs + c.comp[blk] * kCompTabBytes + 256;
    const uint32_t w = peek32(c.u, p);
    int len, s, r = 0;
    if (z == 0) {
      s = huff_decode(huff_at(ct), w, len);
    } else {
      const int rs = huff_decode(huff_at(ct + kHuffBytes), w, len);
      r = rs >> 4;
      s = rs & 15;
    }
    if (len == 0) {
      cz = kSentinel;
      p = end;
      return MRX_JPEG_ST_CODE;
    }
    const uint32_t np = p + len + s;
    if (kWrite && np > unit_end) return MRX_JPEG_ST_TRUNC;
    const int v = s ? huff_extend((w << len) >> (32 - s), s) : 0;
    p = np;
    if (z == 0) {
      ++blocks;
      cur = next_blk++;
      if (kWrite) coef[size_t(cur) * 64] = short(v);
      z = 1;
    } else if (s) {
      z += r;
      if (kWrite) coef[size_t(cur) * 64 + c_zigzag[z]] = short(v);
      ++z;
    } else if (r == 15) {
      z += 16;
    } else {
      z = 64;
    }
    if (z >= 64) {
      z = 0;
      blk = blk + 1 == c.bpm ? 0 : blk + 1;
    }
    cz = (blk << 8) | z;
  }
  return 0;
}

// ------------------------------------------------------------------ 1. unstuff
// One CTA per image: drops the 0x00 after each 0xFF, ends the scan at the first marker that is not
// RSTn, splits it into restart units (start bits), checks the RST count and sequence, and lays out
// the subsequences of every unit.
constexpr int kUnstuffPer = 16;

__global__ void __launch_bounds__(kThreads) jpeg_unstuff_kernel(
    const unsigned char *__restrict__ files, const long long *__restrict__ desc, int S,
    unsigned char *__restrict__ unst, int *__restrict__ work, int *__restrict__ status) {
  const int b = blockIdx.x;
  const long long *D = desc + size_t(b) * DESC_WORDS;
  const unsigned char *f = files + D[D_FILE_OFF];
  const long long len = D[D_FILE_LEN], s0 = D[D_SCAN_OFF];
  const int n_units = int(D[D_NUNITS]);
  unsigned char *u = unst + D[D_UNST_OFF];
  int *unit_bit = work + D[D_UNIT_BIT], *unit_sub = work + D[D_UNIT_SUB];
  int *sub_unit = work + D[D_SUB_OFF];
  const long long cap = D[D_SUB_CAP];
  __shared__ unsigned long long s_warp[kThreads / 32];
  __shared__ long long s_end;
  __shared__ int s_bad, s_fatal;
  if (threadIdx.x == 0) {
    s_end = len;
    s_bad = 0;
  }
  __syncthreads();
  unsigned long long carry = 0;   // rst count << 32 | kept bytes
  // `end` is every thread's copy of s_end taken after the same barrier, so the loop bound is
  // uniform across the CTA: s_end itself shrinks while a pass looks for the end marker.
  long long end = len;
  for (long long base = s0; base < end; base += kThreads * kUnstuffPer) {
    const long long lo = base + threadIdx.x * kUnstuffPer;
    // the first marker that ends the scan in this thread's bytes
    for (long long i = lo; i < lo + kUnstuffPer && i < len; ++i) {
      if (f[i] == 0xFF && (i == s0 || f[i - 1] != 0xFF)) {
        const int nx = i + 1 < len ? f[i + 1] : 0xD9;
        if (nx != 0x00 && (nx < 0xD0 || nx > 0xD7)) {
          atomicMin(reinterpret_cast<unsigned long long *>(&s_end),
                    (unsigned long long)i);
          break;
        }
      }
    }
    __syncthreads();
    end = s_end;
    unsigned int keep = 0, rst = 0;
    for (long long i = lo; i < lo + kUnstuffPer && i < end; ++i) {
      const bool second = i > s0 && f[i - 1] == 0xFF;
      if (second) continue;
      if (f[i] == 0xFF && i + 1 < len && f[i + 1] != 0x00) ++rst;
      else ++keep;
    }
    unsigned long long tot;
    const unsigned long long ex = block_exclusive_scan<unsigned long long, kThreads>(
        (unsigned long long)rst << 32 | keep, s_warp, tot);
    unsigned long long at = carry + ex;
    for (long long i = lo; i < lo + kUnstuffPer && i < end; ++i) {
      const bool second = i > s0 && f[i - 1] == 0xFF;
      if (second) continue;
      if (f[i] == 0xFF && i + 1 < len && f[i + 1] != 0x00) {
        const int k = int(at >> 32) + 1;        // the unit this RST starts
        if (k >= n_units || f[i + 1] != 0xD0 + ((k - 1) & 7)) {
          s_bad = 1;
        } else {
          unit_bit[k] = int(uint32_t(at) * 8u);
        }
        at += 1ull << 32;
      } else {
        u[uint32_t(at)] = f[i];
        at += 1;
      }
    }
    carry += tot;
    __syncthreads();
  }
  const uint32_t kept = uint32_t(carry);
  if (threadIdx.x == 0) {
    int st = 0;
    if (s_bad || int(carry >> 32) != n_units - 1) st |= MRX_JPEG_ST_RST;
    if (end < len) {   // the scan's end marker, after any fill bytes, must be EOI
      long long i = end;
      while (i < len && f[i] == 0xFF) ++i;
      if (i < len && f[i] != 0xD9) st |= MRX_JPEG_ST_MARKER;
    }
    if (st) atomicOr(status + b, st);
    s_fatal = st;
    unit_bit[0] = 0;
    unit_bit[n_units] = int(kept * 8u);
    sub_unit[4 * cap] = 0;        // no subsequences unless the layout below is made
    sub_unit[4 * cap + 1] = 0;    // sync rounds (largest over the image's CTAs)
    sub_unit[4 * cap + 2] = 0;    // subsequences the walk re-decoded
  }
  if (threadIdx.x < 8) u[kept + threadIdx.x] = 0;
  __syncthreads();
  // A wrong or missing RSTn leaves unit starts unwritten: no layout is made from them (the later
  // kernels skip the image).  Otherwise the units are in order and their subsequences fit the cap.
  if (s_fatal) return;
  // subsequences: at least one per unit (a unit without data is caught as truncated)
  for (int k = threadIdx.x; k < n_units; k += kThreads) {
    const int bits = unit_bit[k + 1] - unit_bit[k];
    unit_sub[k] = bits > 0 ? (bits + S - 1) / S : 1;
  }
  __syncthreads();
  const long long n_sub = block_scan_range<kThreads, int>(unit_sub, 0, n_units);
  __syncthreads();
  if (threadIdx.x == 0) {
    unit_sub[n_units] = int(n_sub);
    sub_unit[4 * cap] = int(n_sub);
  }
  for (int k = threadIdx.x; k < n_units; k += kThreads) {
    const int hi = k + 1 < n_units ? unit_sub[k + 1] : int(n_sub);
    for (int j = unit_sub[k]; j < hi; ++j) sub_unit[j] = k;
  }
}

// State of subsequence j of an image: its unit, bit range and whether its start is known.
struct Sub {
  int unit, first;
  uint32_t start, end, unit_end;
};

__device__ __forceinline__ Sub sub_at(const int *unit_bit, const int *unit_sub,
                                      const int *sub_unit, int j, int S) {
  Sub s;
  s.unit = sub_unit[j];
  s.first = unit_sub[s.unit];
  const uint32_t us = uint32_t(unit_bit[s.unit]);
  s.unit_end = uint32_t(unit_bit[s.unit + 1]);
  s.start = us + uint32_t(j - s.first) * uint32_t(S);
  s.end = min(s.start + uint32_t(S), s.unit_end);
  return s;
}

// ------------------------------------------------------------------ 2. sync within a CTA
// kSyncThreads subsequences per CTA.  A round re-decodes the subsequences whose entry changed;
// the rounds end when a change no longer alters an exit, so their number is the longest run of
// guesses that are out of step with their predecessor (the block of the MCU matters as much as
// the bit position).  The walk below fixes one CTA boundary at a time.
constexpr int kSyncThreads = 256;

__global__ void __launch_bounds__(kSyncThreads) jpeg_sync_kernel(
    const long long *__restrict__ desc, const unsigned char *__restrict__ tabs,
    const unsigned char *__restrict__ unst, int S, int *__restrict__ work,
    const int *__restrict__ status) {
  const int b = blockIdx.y;
  const long long *D = desc + size_t(b) * DESC_WORDS;
  if (status[b] & kFatal) return;
  const long long cap = D[D_SUB_CAP];
  const int *unit_bit = work + D[D_UNIT_BIT], *unit_sub = work + D[D_UNIT_SUB];
  int *sub = work + D[D_SUB_OFF];
  const int n_sub = sub[4 * cap];
  const int j0 = blockIdx.x * kSyncThreads;
  if (j0 >= n_sub) return;
  Ctx c;
  load_ctx(c, D, unst, tabs, b);
  const int j = j0 + threadIdx.x;
  const bool active = j < n_sub;
  Sub s{};
  bool known = true;
  uint32_t in_p = 0, p = 0;
  int in_cz = 0, cz = 0, blocks = 0, nb = 0;
  if (active) {
    s = sub_at(unit_bit, unit_sub, sub, j, S);
    known = j == s.first;
    in_p = p = s.start;
    decode_span<false>(c, p, cz, s.end, s.unit_end, blocks, nb, 0, nullptr);
  }
  __shared__ uint32_t s_p[kSyncThreads];
  __shared__ int s_cz[kSyncThreads];
  int changed = 1, rounds = 0;
#pragma unroll 1
  while (true) {
    s_p[threadIdx.x] = p;
    s_cz[threadIdx.x] = cz;
    __syncthreads();
    changed = 0;
    if (active && !known && threadIdx.x > 0) {
      const uint32_t pp = s_p[threadIdx.x - 1];
      const int pcz = s_cz[threadIdx.x - 1];
      if (pp != in_p || pcz != in_cz) {
        in_p = pp;
        in_cz = pcz;
        uint32_t np = pp;
        int ncz = pcz, nbk = 0;
        nb = 0;
        if (ncz != kSentinel) decode_span<false>(c, np, ncz, s.end, s.unit_end, nbk, nb, 0, nullptr);
        else np = max(np, s.end);
        changed = np != p || ncz != cz;
        p = np;
        cz = ncz;
        blocks = nbk;
      }
    }
    if (!__syncthreads_or(changed)) break;
    ++rounds;
  }
  if (active) {
    sub[cap + j] = int(p);
    sub[2 * cap + j] = cz;
    sub[3 * cap + j] = blocks;
  }
  if (threadIdx.x == 0) atomicMax(sub + 4 * cap + 1, rounds);
}

// ------------------------------------------------------------------ 3. walk across CTAs
__global__ void jpeg_walk_kernel(const long long *__restrict__ desc,
                                 const unsigned char *__restrict__ tabs,
                                 const unsigned char *__restrict__ unst, int B, int S,
                                 int *__restrict__ work, const int *__restrict__ status) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const long long *D = desc + size_t(b) * DESC_WORDS;
  if (status[b] & kFatal) return;
  const long long cap = D[D_SUB_CAP];
  const int *unit_bit = work + D[D_UNIT_BIT], *unit_sub = work + D[D_UNIT_SUB];
  int *sub = work + D[D_SUB_OFF];
  const int n_sub = sub[4 * cap];
  Ctx c;
  load_ctx(c, D, unst, tabs, b);
  int j = kSyncThreads, redone = 0;
#pragma unroll 1
  while (j < n_sub) {
    Sub s = sub_at(unit_bit, unit_sub, sub, j, S);
    uint32_t p = uint32_t(sub[cap + j - 1]);
    int cz = sub[2 * cap + j - 1];
#pragma unroll 1
    while (j != s.first) {
      int blocks = 0, nb = 0;
      if (cz != kSentinel) decode_span<false>(c, p, cz, s.end, s.unit_end, blocks, nb, 0, nullptr);
      else p = max(p, s.end);
      ++redone;
      const bool same = int(p) == sub[cap + j] && cz == sub[2 * cap + j];
      sub[cap + j] = int(p);
      sub[2 * cap + j] = cz;
      sub[3 * cap + j] = blocks;
      if (same || ++j >= n_sub) break;
      s = sub_at(unit_bit, unit_sub, sub, j, S);
    }
    j = (j / kSyncThreads + 1) * kSyncThreads;
  }
  sub[4 * cap + 2] = redone;
}

// ------------------------------------------------------------------ 4. blocks before each subsequence
__global__ void __launch_bounds__(kThreads) jpeg_block_scan_kernel(
    const long long *__restrict__ desc, int *__restrict__ work, const int *__restrict__ status) {
  const int b = blockIdx.x;
  const long long *D = desc + size_t(b) * DESC_WORDS;
  if (status[b] & kFatal) return;
  const long long cap = D[D_SUB_CAP];
  int *sub = work + D[D_SUB_OFF];
  block_scan_range<kThreads, int>(sub + 3 * cap, 0, sub[4 * cap]);
}

// ------------------------------------------------------------------ 5. coefficients
__global__ void __launch_bounds__(kThreads) jpeg_write_kernel(
    const long long *__restrict__ desc, const unsigned char *__restrict__ tabs,
    const unsigned char *__restrict__ unst, int S, const int *__restrict__ work,
    short *__restrict__ coef, int *__restrict__ status) {
  const int b = blockIdx.y;
  const long long *D = desc + size_t(b) * DESC_WORDS;
  if (status[b] & kFatal) return;
  const long long cap = D[D_SUB_CAP];
  const int *unit_bit = work + D[D_UNIT_BIT], *unit_sub = work + D[D_UNIT_SUB];
  const int *sub = work + D[D_SUB_OFF];
  const int n_sub = sub[4 * cap];
  const int j = blockIdx.x * kThreads + threadIdx.x;
  if (j >= n_sub) return;
  Ctx c;
  load_ctx(c, D, unst, tabs, b);
  const Sub s = sub_at(unit_bit, unit_sub, sub, j, S);
  uint32_t p = s.start;
  int cz = 0;
  if (j != s.first) {
    p = uint32_t(sub[cap + j - 1]);
    cz = sub[2 * cap + j - 1];
    if (cz == kSentinel) return;      // the code before it was bad: flagged there if it mattered
  }
  const int ri = int(D[D_RI]), bpm = c.bpm;
  const long long mcus = D[D_MCUX] * D[D_MCUY];
  const int ubase = s.unit * ri * bpm;
  const int limit = ubase + int(min((long long)ri, mcus - (long long)s.unit * ri)) * bpm;
  const int *scanned = sub + 3 * cap;
  int next_blk = ubase + scanned[j] - scanned[s.first];
  int blocks = 0;
  int st = decode_span<true>(c, p, cz, s.end, s.unit_end, blocks, next_blk, limit,
                             coef + D[D_COEF_OFF] * 64);
  if (!st && s.end == s.unit_end) {   // the unit's last subsequence: every block must be complete
    if (next_blk < limit || ((cz & 255) != 0 && next_blk - 1 < limit)) st = MRX_JPEG_ST_TRUNC;
  }
  if (st) atomicOr(status + b, st);
}

// ------------------------------------------------------------------ 6. DC prediction
// One CTA per restart unit: per component, the prefix sums of the DC differences in MCU order,
// kept in int32 (a sum outside it is an error, as in libjpeg-turbo) and stored truncated to int16.
__global__ void __launch_bounds__(kThreads) jpeg_dc_kernel(
    const long long *__restrict__ desc, const int *__restrict__ unit_img,
    short *__restrict__ coef, int *__restrict__ status) {
  const int g = blockIdx.x;
  const int b = unit_img[g];
  const long long *D = desc + size_t(b) * DESC_WORDS;
  if (status[b]) return;
  const int u = g - int(D[D_UNIT_BASE]);
  const int ri = int(D[D_RI]), bpm = int(D[D_BPM]);
  const long long mcus = D[D_MCUX] * D[D_MCUY];
  const long long m0 = (long long)u * ri, m1 = min(m0 + ri, mcus);
  short *cf = coef + D[D_COEF_OFF] * 64;
  int comp[10];
  for (int i = 0; i < 10; ++i) comp[i] = i < bpm ? int(D[D_BLK_COMP + i]) : 0;
  __shared__ long long s_warp[kThreads / 32];
  long long carry[3] = {0, 0, 0};
  bool bad = false;
  for (long long base = m0; base < m1; base += kThreads) {
    const long long m = base + threadIdx.x;
    long long sum[3] = {0, 0, 0};
    if (m < m1)
      for (int i = 0; i < bpm; ++i) sum[comp[i]] += cf[(m * bpm + i) * 64];
    long long ex[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      long long tot;
      ex[k] = block_exclusive_scan<long long, kThreads>(sum[k], s_warp, tot) + carry[k];
      carry[k] += tot;
    }
    if (m < m1) {
      for (int i = 0; i < bpm; ++i) {
        short *q = cf + (m * bpm + i) * 64;
        const long long v = ex[comp[i]] + *q;
        ex[comp[i]] = v;
        if (v < -2147483648LL || v > 2147483647LL) bad = true;
        *q = short(int(v));
      }
    }
  }
  if (bad) atomicOr(status + b, MRX_JPEG_ST_DC);
}

// ------------------------------------------------------------------ 7. islow IDCT
constexpr int FIX_0_298631336 = 2446, FIX_0_390180644 = 3196, FIX_0_541196100 = 4433,
              FIX_0_765366865 = 6270, FIX_0_899976223 = 7373, FIX_1_175875602 = 9633,
              FIX_1_501321110 = 12299, FIX_1_847759065 = 15137, FIX_1_961570560 = 16069,
              FIX_2_053119869 = 16819, FIX_2_562915447 = 20995, FIX_3_072711026 = 25172;
constexpr int CONST_BITS = 13, PASS1_BITS = 2;

// jidctint.c's 1-D butterfly on x[0..8) (int64, as JLONG); out: the 8 undescaled results
__device__ __forceinline__ void idct_1d(const long long *x, long long *o) {
  long long z2 = x[2], z3 = x[6];
  long long z1 = (z2 + z3) * FIX_0_541196100;
  const long long tmp2 = z1 + z3 * -FIX_1_847759065;
  const long long tmp3 = z1 + z2 * FIX_0_765366865;
  const long long tmp0 = (x[0] + x[4]) * (1LL << CONST_BITS);
  const long long tmp1 = (x[0] - x[4]) * (1LL << CONST_BITS);
  const long long t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  long long t0 = x[7], t1 = x[5], t2 = x[3], t3 = x[1];
  z1 = t0 + t3;
  z2 = t1 + t2;
  z3 = t0 + t2;
  long long z4 = t1 + t3;
  const long long z5 = (z3 + z4) * FIX_1_175875602;
  t0 *= FIX_0_298631336;
  t1 *= FIX_2_053119869;
  t2 *= FIX_3_072711026;
  t3 *= FIX_1_501321110;
  z1 *= -FIX_0_899976223;
  z2 *= -FIX_2_562915447;
  z3 = z3 * -FIX_1_961570560 + z5;
  z4 = z4 * -FIX_0_390180644 + z5;
  t0 += z1 + z3;
  t1 += z2 + z4;
  t2 += z2 + z3;
  t3 += z1 + z4;
  o[0] = t10 + t3; o[7] = t10 - t3;
  o[1] = t11 + t2; o[6] = t11 - t2;
  o[2] = t12 + t1; o[5] = t12 - t1;
  o[3] = t13 + t0; o[4] = t13 - t0;
}

// jdmaster.c's post-IDCT range-limit table, indexed by x & 1023 (not a clamp)
__device__ __forceinline__ unsigned char range_limit(long long x) {
  const int v = int(x & 1023);
  return v < 128 ? v + 128 : v < 512 ? 255 : v < 896 ? 0 : v - 896;
}

// 8 threads per block: thread r runs column r, then row r, through shared memory.
__global__ void __launch_bounds__(kThreads) jpeg_idct_kernel(
    const long long *__restrict__ desc, const unsigned char *__restrict__ tabs,
    const short *__restrict__ coef, unsigned char *__restrict__ planes,
    const int *__restrict__ status) {
  const int b = blockIdx.y;
  const long long *D = desc + size_t(b) * DESC_WORDS;
  if (status[b]) return;
  const long long nblocks = D[D_NBLOCKS];
  const long long blk = (long long)blockIdx.x * (kThreads / 8) + (threadIdx.x >> 3);
  if ((long long)blockIdx.x * (kThreads / 8) >= nblocks) return;
  const int r = threadIdx.x & 7;
  __shared__ int ws[kThreads / 8][64];
  int *w = ws[threadIdx.x >> 3];
  const bool active = blk < nblocks;
  const int bpm = int(D[D_BPM]);
  int ci = 0;
  long long bx = 0, by = 0;
  if (active) {
    const long long m = blk / bpm;
    const int c = int(blk - m * bpm);
    ci = int(D[D_BLK_COMP + c]);
    const long long mx = m % D[D_MCUX], my = m / D[D_MCUX];
    bx = mx * D[D_COMP_H + ci] + D[D_BLK_DX + c];
    by = my * D[D_COMP_V + ci] + D[D_BLK_DY + c];
    const int *q = reinterpret_cast<const int *>(tabs + size_t(b) * kTabBytes +
                                                 ci * kCompTabBytes);
    const short *in = coef + (D[D_COEF_OFF] + blk) * 64;
    long long x[8], o[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) x[k] = (long long)in[k * 8 + r] * q[k * 8 + r];
    idct_1d(x, o);
    const long long half = 1LL << (CONST_BITS - PASS1_BITS - 1);
#pragma unroll
    for (int k = 0; k < 8; ++k) w[k * 8 + r] = int((o[k] + half) >> (CONST_BITS - PASS1_BITS));
  }
  __syncwarp();
  if (active) {
    long long x[8], o[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) x[k] = w[r * 8 + k];
    idct_1d(x, o);
    const int sh = CONST_BITS + PASS1_BITS + 3;
    unsigned char px[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) px[k] = range_limit((o[k] + (1LL << (sh - 1))) >> sh);
    const long long pw = D[D_PLANE_BW + ci] * 8;
    unsigned char *dst = planes + D[D_PLANE_OFF + ci] + (by * 8 + r) * pw + bx * 8;
    uint2 v;
    v.x = px[0] | px[1] << 8 | px[2] << 16 | uint32_t(px[3]) << 24;
    v.y = px[4] | px[5] << 8 | px[6] << 16 | uint32_t(px[7]) << 24;
    *reinterpret_cast<uint2 *>(dst) = v;
  }
}

// ------------------------------------------------------------------ 8. upsample, colour, orient
// jdsample.c: the method jinit_upsampler picks for (h_expand, v_expand); rows above the first and
// below the last real row are duplicates of those rows (jdmainct.c's context rows).
__device__ __forceinline__ int upsample(const unsigned char *p, long long pw, int he, int ve,
                                        int dw, int dh, int y, int x) {
  if (he == 1 && ve == 1) return p[(long long)y * pw + x];
  if (he == 1 && ve == 2) {
    const int i = y >> 1;
    const int n = (y & 1) ? min(i + 1, dh - 1) : max(i - 1, 0);
    return (3 * p[(long long)i * pw + x] + p[(long long)n * pw + x] + 1 + (y & 1)) >> 2;
  }
  if (he == 2 && dw > 2 && (ve == 1 || ve == 2)) {
    const int j = x >> 1, odd = x & 1;
    const int jn = odd ? j + 1 : j - 1;
    const bool edge = odd ? j == dw - 1 : j == 0;
    if (ve == 1) {
      const unsigned char *row = p + (long long)y * pw;
      if (edge) return row[j];
      return (3 * row[j] + row[jn] + 1 + odd) >> 2;
    }
    const int i = y >> 1;
    const int n = (y & 1) ? min(i + 1, dh - 1) : max(i - 1, 0);
    const unsigned char *r0 = p + (long long)i * pw, *r1 = p + (long long)n * pw;
    const int cs = 3 * r0[j] + r1[j];
    if (edge) return (4 * cs + 8 - odd) >> 4;
    const int cn = 3 * r0[jn] + r1[jn];
    return (3 * cs + cn + 8 - odd) >> 4;
  }
  return p[(long long)(y / ve) * pw + x / he];   // replication (int_upsample, narrow h2v1/h2v2)
}

__device__ __forceinline__ unsigned char clamp255(int v) {
  return (unsigned char)min(max(v, 0), 255);
}

__global__ void __launch_bounds__(kThreads) jpeg_pixels_kernel(
    const long long *__restrict__ desc, const unsigned char *__restrict__ planes,
    unsigned char *__restrict__ out, const long long *__restrict__ out_off,
    const int *__restrict__ status) {
  const int b = blockIdx.y;
  const long long *D = desc + size_t(b) * DESC_WORDS;
  if (status[b]) return;
  const int H = int(D[D_H]), W = int(D[D_W]);
  const long long idx = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (idx >= (long long)H * W) return;
  const int y = int(idx / W), x = int(idx - (long long)y * W);
  const int nc = int(D[D_NCOMP]);
  int v[3];
  for (int ci = 0; ci < nc; ++ci) {
    const int he = int(D[D_HMAX] / D[D_COMP_H + ci]), ve = int(D[D_VMAX] / D[D_COMP_V + ci]);
    v[ci] = upsample(planes + D[D_PLANE_OFF + ci], D[D_PLANE_BW + ci] * 8, he, ve,
                     int(D[D_DW + ci]), int(D[D_DH + ci]), y, x);
  }
  unsigned char rgb[3];
  const int color = int(D[D_COLOR]);
  if (color == 0) {
    rgb[0] = rgb[1] = rgb[2] = (unsigned char)v[0];
  } else if (color == 2) {
    rgb[0] = v[0]; rgb[1] = v[1]; rgb[2] = v[2];
  } else {   // jdcolor.c ycc_rgb_convert: FIX(x) = (int)(x * 65536 + 0.5)
    const int cb = v[1] - 128, cr = v[2] - 128;
    const int half = 1 << 15;
    rgb[0] = clamp255(v[0] + ((91881 * cr + half) >> 16));
    rgb[1] = clamp255(v[0] + ((-46802 * cr + (-22554 * cb + half)) >> 16));
    rgb[2] = clamp255(v[0] + ((116130 * cb + half) >> 16));
  }
  // OpenCV's EXIF orientation as an index map on the store
  const int o = int(D[D_ORIENT]);
  int oy = y, ox = x, ow = W;
  switch (o) {
    case 2: ox = W - 1 - x; break;
    case 3: oy = H - 1 - y; ox = W - 1 - x; break;
    case 4: oy = H - 1 - y; break;
    case 5: oy = x; ox = y; ow = H; break;
    case 6: oy = x; ox = H - 1 - y; ow = H; break;
    case 7: oy = W - 1 - x; ox = H - 1 - y; ow = H; break;
    case 8: oy = W - 1 - x; ox = y; ow = H; break;
    default: break;
  }
  unsigned char *dst = out + out_off[b] + ((long long)oy * ow + ox) * 3;
  dst[0] = rgb[0];
  dst[1] = rgb[1];
  dst[2] = rgb[2];
}

int check_batch(const char *fn, int B, int max_items) {
  MRX_CHECK_ARG(B >= 0 && B <= MRX_MAX_BATCH, "%s: B=%d outside [0, %d]", fn, B, MRX_MAX_BATCH);
  MRX_CHECK_ARG(max_items >= 1, "%s: a max extent below 1", fn);
  return MRX_OK;
}

}  // namespace
}  // namespace mrx

using namespace mrx;

extern "C" int mrx_jpeg_coefficients(const unsigned char *d_files, const long long *d_desc,
                                     const unsigned char *d_tabs, const int *d_unit_img, int B,
                                     int U, int S, int max_subs, unsigned char *d_unst,
                                     int *d_work, short *d_coef, long long coef_blocks,
                                     int *d_status, void *stream) {
  MRX_CHECK_ARG(d_files && d_desc && d_tabs && d_unit_img && d_unst && d_work && d_coef &&
                    d_status,
                "mrx_jpeg_coefficients: null pointer");
  if (int rc = check_batch("mrx_jpeg_coefficients", B, max_subs)) return rc;
  MRX_CHECK_ARG(S >= 32 && S <= 65536 && S % 32 == 0,
                "mrx_jpeg_coefficients: S=%d is not a multiple of 32 in [32, 65536]", S);
  MRX_CHECK_ARG(U >= B && coef_blocks >= 1, "mrx_jpeg_coefficients: U=%d, coef_blocks=%lld", U,
                coef_blocks);
  if (B == 0) return MRX_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MRX_CUDA(cudaMemsetAsync(d_status, 0, sizeof(int) * B, st));
  MRX_CUDA(cudaMemsetAsync(d_coef, 0, sizeof(short) * 64 * size_t(coef_blocks), st));
  jpeg_unstuff_kernel<<<B, kThreads, 0, st>>>(d_files, d_desc, S, d_unst, d_work, d_status);
  MRX_LAUNCH_CHECK("jpeg_unstuff_kernel");
  const dim3 gs((max_subs + kSyncThreads - 1) / kSyncThreads, B);
  jpeg_sync_kernel<<<gs, kSyncThreads, 0, st>>>(d_desc, d_tabs, d_unst, S, d_work, d_status);
  MRX_LAUNCH_CHECK("jpeg_sync_kernel");
  jpeg_walk_kernel<<<(B + 63) / 64, 64, 0, st>>>(d_desc, d_tabs, d_unst, B, S, d_work, d_status);
  MRX_LAUNCH_CHECK("jpeg_walk_kernel");
  jpeg_block_scan_kernel<<<B, kThreads, 0, st>>>(d_desc, d_work, d_status);
  MRX_LAUNCH_CHECK("jpeg_block_scan_kernel");
  const dim3 grid((max_subs + kThreads - 1) / kThreads, B);
  jpeg_write_kernel<<<grid, kThreads, 0, st>>>(d_desc, d_tabs, d_unst, S, d_work, d_coef,
                                               d_status);
  MRX_LAUNCH_CHECK("jpeg_write_kernel");
  jpeg_dc_kernel<<<U, kThreads, 0, st>>>(d_desc, d_unit_img, d_coef, d_status);
  MRX_LAUNCH_CHECK("jpeg_dc_kernel");
  return MRX_OK;
}

extern "C" int mrx_jpeg_pixels(const long long *d_desc, const unsigned char *d_tabs,
                               const short *d_coef, const int *d_status, int B, int max_blocks,
                               long long max_pixels, unsigned char *d_planes,
                               unsigned char *d_out, const long long *d_out_off, void *stream) {
  MRX_CHECK_ARG(d_desc && d_tabs && d_coef && d_status && d_planes && d_out && d_out_off,
                "mrx_jpeg_pixels: null pointer");
  if (int rc = check_batch("mrx_jpeg_pixels", B, max_blocks)) return rc;
  MRX_CHECK_ARG(max_pixels >= 1 && max_pixels <= (1LL << 32),
                "mrx_jpeg_pixels: max_pixels=%lld", max_pixels);
  if (B == 0) return MRX_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 gi((max_blocks + kThreads / 8 - 1) / (kThreads / 8), B);
  jpeg_idct_kernel<<<gi, kThreads, 0, st>>>(d_desc, d_tabs, d_coef, d_planes, d_status);
  MRX_LAUNCH_CHECK("jpeg_idct_kernel");
  const dim3 gp(unsigned((max_pixels + kThreads - 1) / kThreads), B);
  jpeg_pixels_kernel<<<gp, kThreads, 0, st>>>(d_desc, d_planes, d_out, d_out_off, d_status);
  MRX_LAUNCH_CHECK("jpeg_pixels_kernel");
  return MRX_OK;
}
