// png_decode.cu -- PNG files decoded bit for bit as cv2.imdecode(buf, IMREAD_COLOR) then BGR2RGB
// (libpng: strip_16, expand gray 1/2/4 by bit replication, palette to RGB, gray to RGB, strip
// alpha; Adam7; EXIF orientation).  The host (png.DecodePlan) has parsed every chunk but the
// image data; one stream-ordered batch (mrx.h, "PNG decode"):
//   gather    one warp per IDAT chunk: the payload into the image's contiguous zlib stream, and
//             the chunk's CRC-32 (partial CRCs per lane, combined as the encoder combines them)
//   find      one thread per byte of the zlib stream: the bit positions where a dynamic block
//             header starts that zlib's inflate would accept, into K slots per tile of
//             MRX_PNG_DEC_TILE_BITS bits
//   measure   one warp per candidate: its block decoded to the end-of-block code without
//             writing (end bit, bytes, how far a distance reaches before the block, BFINAL)
//   chain     one warp per image walks from the first bit: a valid measured candidate where one
//             starts, else the block measured there; the image's true block list, its errors
//   expand    one warp per chained block writes its bytes as cells at their absolute offsets: a
//             value, or a reference to a byte before the block
//   resolve   one CTA per image, blocks in order: each reference reads the byte it points at
//   adler     per tile of kTile bytes: Adler-32 partial sums of the filtered stream, only where
//             libpng would check the trailer (the stream ends exactly with the image's rows)
//   unfilter  one CTA per image, a wavefront over rows: thread t owns row g * kThreads + t and
//             takes pixel column s - t at step s, so the pixel above is one step old
//   pixels    one thread per output pixel: sample extraction, bit depth to 8, palette, gray to
//             RGB, alpha dropped, the Adam7 pass it lives in, EXIF orientation on the store
#include "common.cuh"
#include "deflate.cuh"

namespace mrx {
namespace {

constexpr int kThreads = 256;
constexpr int kTile = 2048;
constexpr int kLutBits = 10;                 // first-level Huffman lookup
constexpr int kGatherWarps = 4;

// desc words per image (png.py DD_*)
enum {
  DD_Z_OFF = 0, DD_Z_LEN, DD_FILT_OFF, DD_N, DD_H, DD_W, DD_CT, DD_DEPTH, DD_INTERLACE, DD_ORIENT,
  DD_PLTE_N, DD_BLK_OFF, DD_BLK_CAP, DD_WSIZE, DD_TILE_OFF, DD_NTILES, DD_WORDS = 16
};
// chunk words (png.py CK_*)
enum { CK_IMG = 0, CK_SRC, CK_LEN, CK_DST, CK_WORDS };

__constant__ unsigned char c_adam7[7][4] = {{0, 0, 8, 8}, {4, 0, 8, 8}, {0, 4, 4, 8},
                                            {2, 0, 4, 4}, {0, 2, 2, 4}, {1, 0, 2, 2},
                                            {0, 1, 1, 2}};   // x0, y0, dx, dy

__device__ __forceinline__ int channels_of(int ct) {
  return ct == 2 ? 3 : ct == 4 ? 2 : ct == 6 ? 4 : 1;
}

// pass p's width and height (the whole image when not interlaced, p = 0)
__device__ __forceinline__ void pass_size(int p, bool il, int H, int W, int &pw, int &ph) {
  if (!il) {
    pw = W, ph = H;
    return;
  }
  const int x0 = c_adam7[p][0], y0 = c_adam7[p][1], dx = c_adam7[p][2], dy = c_adam7[p][3];
  pw = W > x0 ? (W - x0 + dx - 1) / dx : 0;
  ph = H > y0 ? (H - y0 + dy - 1) / dy : 0;
}

__device__ __forceinline__ long long row_bytes(int pw, int bits_pp) {
  return ((long long)pw * bits_pp + 7) >> 3;
}

// ------------------------------------------------------------------ gather + IDAT CRC-32
__global__ void __launch_bounds__(32 * kGatherWarps) png_gather_kernel(
    const unsigned char *__restrict__ files, const long long *__restrict__ desc,
    const long long *__restrict__ chunks, long long n_chunks, unsigned char *__restrict__ z,
    int *__restrict__ status) {
  __shared__ unsigned table[256];
  __shared__ unsigned x2n[32];
  crc_tables(table, x2n);
  __syncthreads();
  const long long c = (long long)blockIdx.x * kGatherWarps + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (c >= n_chunks) return;
  const long long *C = chunks + c * CK_WORDS;
  const int b = int(C[CK_IMG]);
  const long long len = C[CK_LEN];
  const unsigned char *src = files + C[CK_SRC];       // the chunk type; its data follows
  unsigned char *dst = z + desc[size_t(b) * DD_WORDS + DD_Z_OFF] + C[CK_DST];
  const long long total = len + 4, seg = (total + 31) / 32;
  const long long lo = min(lane * seg, total), hi = min((lane + 1) * seg, total);
  unsigned crc = 0xFFFFFFFFu;
  for (long long j = lo; j < hi; ++j) {
    const unsigned char v = src[j];
    crc = crc_byte(table, crc, v);
    if (j >= 4) dst[j - 4] = v;
  }
  crc ^= 0xFFFFFFFFu;
  unsigned all = crc;
  for (int l = 1; l < 32; ++l) {
    const unsigned cl = __shfl_sync(0xFFFFFFFFu, crc, l);
    const long long ll = min((l + 1) * seg, total) - min(l * seg, total);
    if (lane == 0 && ll > 0) all = crc_combine(x2n, all, cl, ll);
  }
  if (lane == 0) {
    const unsigned char *t = src + total;
    const unsigned want = (unsigned(t[0]) << 24) | (unsigned(t[1]) << 16) | (unsigned(t[2]) << 8) | t[3];
    if (want != all) atomicOr(status + b, MRX_PNG_ST_CRC);
  }
}

// ------------------------------------------------------------------ inflate
struct Bits {
  const unsigned char *z;
  long long len, pos;        // pos: the next byte to load
  unsigned long long buf;
  int cnt;
  __device__ void fill() {
    while (cnt <= 56) {
      buf |= (unsigned long long)(pos < len ? __ldg(z + pos) : 0) << cnt;
      ++pos;
      cnt += 8;
    }
  }
  __device__ unsigned get(int n) {   // n <= 32
    fill();
    const unsigned v = unsigned(buf & ((1ull << n) - 1));
    buf >>= n;
    cnt -= n;
    return v;
  }
  __device__ long long bit() const { return pos * 8 - cnt; }   // bits consumed
  __device__ bool over() const { return bit() > len * 8; }     // read past the stream
};

// one canonical code: counts per length, symbols by (length, value), a kLutBits first level
struct Huff {
  unsigned short count[16];
  unsigned short sym[320];
  unsigned short lut[1 << kLutBits];   // length << 9 | symbol; 0 = longer than kLutBits or none
};

// inftrees.c's acceptance: -1 over-subscribed, -2 incomplete (allowed only for a single code of
// length 1 in the literal/length and distance codes; never for the code-length code), else the
// number of codes.  Lane 0 has set count[]; the warp builds sym[] and lut[].
__device__ int huff_build(Huff &h, const unsigned char *len, int n, bool codes) {
  const int lane = threadIdx.x & 31;
  int left = 1, ncodes = 0, maxlen = 0;
  for (int l = 1; l < 16; ++l) {
    left = (left << 1) - h.count[l];
    if (left < 0) return -1;
    ncodes += h.count[l];
    if (h.count[l]) maxlen = l;
  }
  if (left > 0 && (codes || maxlen != 1) && ncodes > 0) return -2;
  if (codes && ncodes == 0) return -2;
  for (int i = lane; i < (1 << kLutBits); i += 32) h.lut[i] = 0;
  __syncwarp();
  if (lane == 0) {
    unsigned short offs[16];
    offs[1] = 0;
    for (int l = 1; l < 15; ++l) offs[l + 1] = offs[l] + h.count[l];
    for (int s = 0; s < n; ++s)
      if (len[s]) h.sym[offs[len[s]]++] = (unsigned short)s;
  }
  __syncwarp();
  // first level: the k-th code of length l (canonical order) fills every index whose low l bits
  // are its bit-reversed value
  int code = 0, k = 0;
  for (int l = 1; l <= kLutBits; ++l) {
    for (int j = 0; j < h.count[l]; ++j, ++k, ++code) {
      const unsigned rev = __brev(unsigned(code)) >> (32 - l);
      const unsigned short e = (unsigned short)((l << 9) | h.sym[k]);
      for (int i = lane; i < (1 << (kLutBits - l)); i += 32) h.lut[rev | (unsigned(i) << l)] = e;
    }
    code <<= 1;
  }
  __syncwarp();
  return ncodes;
}

// the next symbol, or -1 for a code no symbol has
__device__ __forceinline__ int huff_decode(const Huff &h, Bits &br) {
  br.fill();
  const unsigned short e = h.lut[br.buf & ((1u << kLutBits) - 1)];
  if (e) {
    const int l = e >> 9;
    br.buf >>= l;
    br.cnt -= l;
    return e & 511;
  }
  int code = 0, first = 0, index = 0;   // puff.c's canonical walk for the longer codes
  for (int l = 1; l < 16; ++l) {
    code |= int(br.buf & 1);
    br.buf >>= 1;
    br.cnt -= 1;
    const int count = h.count[l];
    if (code - count < first) return h.sym[index + (code - first)];
    index += count;
    first = (first + count) << 1;
    code <<= 1;
  }
  return -1;
}

struct InflateSmem {
  Huff lit, dist, cl;
  unsigned char lens[320];
  int err, nlen, ndist;
};

// one decoded deflate block: its end bit, the bytes it describes, how far its farthest distance
// reaches before the block's first byte, BFINAL, and an error with the bytes described before it
struct BlockOut {
  long long end, len, need, err_at;
  int final, err;
};

// Decode the block whose header starts at bit `start` of an image's zlib stream z (warp-
// collective; lane 0 decodes).  pos: the block's first output position when `absolute` (then a
// distance past the stream start is an error), else 0 (the measure of a candidate: distances may
// reach before the block, `need` records how far).  With cells, every byte below n is written
// as a cell: the literal value (< 256), 256 + the position of a byte before ref_base (resolved
// later, in block order), or, for a source at or past ref_base, that source's cell.
__device__ BlockOut run_block(InflateSmem &S, const unsigned char *z, long long zlen,
                              long long start, long long pos, bool absolute, long long wsize,
                              int *cells, long long ref_base, long long n) {
  const int lane = threadIdx.x & 31;
  Bits br{z, zlen, start >> 3, 0, 0};
  br.get(int(start & 7));
  long long p = pos, need = 0;
  int err = 0, final = 0, typ = 0;
  if (lane == 0) {
    final = int(br.get(1));
    typ = int(br.get(2));
  }
  final = __shfl_sync(0xFFFFFFFFu, final, 0);
  typ = __shfl_sync(0xFFFFFFFFu, typ, 0);
  do {
    if (typ == 3) {
      err = MRX_PNG_ST_CODE;
      break;
    }
    if (typ == 0) {   // stored
      long long L = 0, at = 0;
      if (lane == 0) {
        br.get(br.cnt & 7);
        const unsigned len = br.get(16), nlen = br.get(16);
        if (br.over()) err = MRX_PNG_ST_TRUNC;
        else if (len != (~nlen & 0xFFFFu)) err = MRX_PNG_ST_CODE;
        L = len;
        at = br.bit() >> 3;   // whole bytes are buffered: the block's bytes start here
      }
      err = __shfl_sync(0xFFFFFFFFu, err, 0);
      L = __shfl_sync(0xFFFFFFFFu, L, 0);
      at = __shfl_sync(0xFFFFFFFFu, at, 0);
      if (err) break;
      const long long avail = zlen - at;
      if (cells) {
        const long long put = max(0LL, min(min(L, avail), n - p));
        for (long long k = lane; k < put; k += 32) cells[p + k] = __ldg(z + at + k);
      }
      if (L > avail) {
        err = MRX_PNG_ST_TRUNC;
        break;
      }
      p += L;
      if (lane == 0) {
        br.pos = at + L;
        br.buf = 0;
        br.cnt = 0;
      }
      break;
    }
    // Huffman block: the codes into shared memory
    if (lane == 0) {
      int nlen = 288, ndist = 32;
      if (typ == 1) {
        for (int s = 0; s < 288; ++s) S.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
        for (int s = 0; s < 32; ++s) S.lens[288 + s] = 5;
      } else {
        nlen = int(br.get(5)) + 257;
        ndist = int(br.get(5)) + 1;
        const int ncl = int(br.get(4)) + 4;
        if (nlen > 286 || ndist > 30) err = MRX_PNG_ST_CODE;
        for (int k = 0; k < 19; ++k) S.lens[k] = 0;
        for (int k = 0; k < ncl; ++k) S.lens[c_bl_order[k]] = (unsigned char)br.get(3);
      }
      S.err = err;
      S.nlen = nlen;
      S.ndist = ndist;
    }
    __syncwarp();
    err = S.err;
    if (err) break;
    const int nlen = S.nlen, ndist = S.ndist;
    if (typ == 2) {
      if (lane == 0) {
        for (int l = 0; l < 16; ++l) S.cl.count[l] = 0;
        for (int k = 0; k < 19; ++k) S.cl.count[S.lens[k]]++;
        S.cl.count[0] = 0;
      }
      __syncwarp();
      unsigned char cl[19];
      for (int k = 0; k < 19; ++k) cl[k] = S.lens[k];
      if (huff_build(S.cl, cl, 19, true) < 0) {
        err = MRX_PNG_ST_CODE;
        break;
      }
      if (lane == 0) {
        int have = 0;
        while (have < nlen + ndist && !err) {
          const int s = huff_decode(S.cl, br);
          if (s < 0) {
            err = MRX_PNG_ST_CODE;
          } else if (s < 16) {
            S.lens[have < nlen ? have : 288 + have - nlen] = (unsigned char)s;
            ++have;
          } else {
            int rep, v = 0;
            if (s == 16) {
              if (have == 0) {
                err = MRX_PNG_ST_CODE;
                break;
              }
              const int prev = have - 1;
              v = S.lens[prev < nlen ? prev : 288 + prev - nlen];
              rep = 3 + int(br.get(2));
            } else {
              rep = s == 17 ? 3 + int(br.get(3)) : 11 + int(br.get(7));
            }
            if (have + rep > nlen + ndist) {
              err = MRX_PNG_ST_CODE;
              break;
            }
            for (; rep; --rep, ++have) S.lens[have < nlen ? have : 288 + have - nlen] = (unsigned char)v;
          }
        }
        if (!err && br.over()) err = MRX_PNG_ST_TRUNC;
        if (!err && S.lens[kEndBlock] == 0) err = MRX_PNG_ST_CODE;
        for (int s = nlen; s < 288; ++s) S.lens[s] = 0;
        for (int s = ndist; s < 32; ++s) S.lens[288 + s] = 0;
        S.err = err;
      }
      __syncwarp();
      err = S.err;
      if (err) break;
    }
    if (lane == 0) {
      for (int l = 0; l < 16; ++l) S.lit.count[l] = S.dist.count[l] = 0;
      for (int s = 0; s < 288; ++s) S.lit.count[S.lens[s]]++;
      for (int s = 0; s < 32; ++s) S.dist.count[S.lens[288 + s]]++;
      S.lit.count[0] = S.dist.count[0] = 0;
    }
    __syncwarp();
    const int lb = huff_build(S.lit, S.lens, 288, false);
    const int db = huff_build(S.dist, S.lens + 288, 32, false);
    if (lb < 0 || db < 0) {
      err = MRX_PNG_ST_CODE;
      break;
    }
    // the symbols; fixed codes 286, 287 and distances 30, 31 are invalid as in zlib.  Lane 0
    // writes a run of literals alone; the warp meets at each match and at the end of the block
    while (true) {
      int sym = 0, len = 0, dist = 0, e = 0;
      if (lane == 0) {
        while (true) {
          sym = huff_decode(S.lit, br);
          if (sym < 0 || sym > 285) {
            e = MRX_PNG_ST_CODE;
          } else if (sym > kEndBlock) {
            const int c = sym - 257;
            len = c_base_length[c] + 3 + int(br.get(c_extra_lbits[c]));
            const int d = huff_decode(S.dist, br);
            if (d < 0 || d > 29) e = MRX_PNG_ST_CODE;
            else dist = c_base_dist[d] + int(br.get(c_extra_dbits[d]));
          }
          if (!e && br.over()) e = MRX_PNG_ST_TRUNC;
          if (e || sym >= kEndBlock) break;
          if (cells && p < n) cells[p] = sym;
          ++p;
        }
      }
      e = __shfl_sync(0xFFFFFFFFu, e, 0);
      sym = __shfl_sync(0xFFFFFFFFu, sym, 0);
      p = __shfl_sync(0xFFFFFFFFu, p, 0);
      if (e) {
        err = e;
        break;
      }
      if (sym == kEndBlock) break;
      len = __shfl_sync(0xFFFFFFFFu, len, 0);
      dist = __shfl_sync(0xFFFFFFFFu, dist, 0);
      if (dist > wsize || (absolute && dist > p)) {
        err = MRX_PNG_ST_DIST;
        break;
      }
      need = max(need, dist - (p - pos));
      if (cells) {
        __syncwarp();
        const long long put = max(0LL, min((long long)len, n - p));
        for (long long k = lane; k < put; k += 32) {
          const long long src = p - dist + k % dist;
          cells[p + k] = src < ref_base ? int(256 + src) : cells[src];
        }
        __syncwarp();
      }
      p += len;
    }
  } while (false);
  long long end = 0;
  if (lane == 0) end = br.bit();
  end = __shfl_sync(0xFFFFFFFFu, end, 0);
  BlockOut r;
  r.end = end;
  r.len = p - pos;
  r.need = need;
  r.err_at = p;
  r.final = final;
  r.err = err;
  return r;
}

// ------------------------------------------------------------------ find: candidate block starts
// A dynamic block header zlib's inflate would accept starting at `bit`: HLIT <= 29, HDIST <= 29, a
// complete code-length code, code lengths that decode (no repeat of nothing, no overrun), a
// nonzero end-of-block length, and literal/length and distance codes inftrees.c builds.
__device__ bool header_ok(const unsigned char *z, long long zlen, long long bit) {
  Bits br{z, zlen, bit >> 3, 0, 0};
  br.get(int(bit & 7));
  br.get(1);
  if (br.get(2) != 2) return false;
  const int nlen = int(br.get(5)) + 257, ndist = int(br.get(5)) + 1, ncl = int(br.get(4)) + 4;
  if (nlen > 286 || ndist > 30) return false;
  unsigned char cl[19];
  for (int k = 0; k < 19; ++k) cl[k] = 0;
  for (int k = 0; k < ncl; ++k) cl[c_bl_order[k]] = (unsigned char)br.get(3);
  int cnt[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int k = 0; k < 19; ++k) cnt[cl[k]]++;
  int left = 1;
  for (int l = 1; l < 8; ++l) {
    left = 2 * left - cnt[l];
    if (left < 0) return false;
  }
  if (left != 0) return false;   // incomplete or empty
  unsigned char sym[19];
  int offs[8];
  offs[1] = 0;
  for (int l = 1; l < 7; ++l) offs[l + 1] = offs[l] + cnt[l];
  for (int k = 0; k < 19; ++k)
    if (cl[k]) sym[offs[cl[k]]++] = (unsigned char)k;
  int lc[16], dc[16];
  for (int l = 0; l < 16; ++l) lc[l] = dc[l] = 0;
  int have = 0, prev = 0, eob = 0;
  while (have < nlen + ndist) {
    br.fill();
    int code = 0, first = 0, index = 0, s = -1;
    for (int l = 1; l < 8; ++l) {
      code |= int(br.buf & 1);
      br.buf >>= 1;
      br.cnt -= 1;
      if (code - cnt[l] < first) {
        s = sym[index + code - first];
        break;
      }
      index += cnt[l];
      first = (first + cnt[l]) << 1;
      code <<= 1;
    }
    int rep = 1, v = s;
    if (s == 16) {
      if (have == 0) return false;
      v = prev;
      rep = 3 + int(br.get(2));
    } else if (s == 17) {
      v = 0;
      rep = 3 + int(br.get(3));
    } else if (s == 18) {
      v = 0;
      rep = 11 + int(br.get(7));
    }
    if (have + rep > nlen + ndist) return false;
    for (; rep; --rep, ++have) {
      if (have < nlen) {
        lc[v]++;
        if (have == kEndBlock) eob = v;
      } else {
        dc[v]++;
      }
    }
    prev = v;
  }
  if (br.over() || eob == 0) return false;
  for (int which = 0; which < 2; ++which) {
    const int *c = which ? dc : lc;
    int lf = 1, nc = 0, maxl = 0;
    for (int l = 1; l < 16; ++l) {
      lf = 2 * lf - c[l];
      if (lf < 0) return false;
      nc += c[l];
      if (c[l]) maxl = l;
    }
    if (lf > 0 && nc > 0 && maxl != 1) return false;
  }
  return true;
}

// one thread per byte of an image's zlib stream: the 8 bit positions starting in it
__global__ void __launch_bounds__(kThreads) png_find_kernel(
    const long long *__restrict__ desc, const unsigned char *__restrict__ z, int K,
    long long *__restrict__ cand, int *__restrict__ tile_cnt, long long *__restrict__ info,
    const int *__restrict__ status) {
  const int b = blockIdx.y;
  const long long *D = desc + size_t(b) * DD_WORDS;
  const long long zlen = D[DD_Z_LEN];
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x + 2;   // after the header
  if (i >= zlen || status[b]) return;
  const unsigned char *zi = z + D[DD_Z_OFF];
  unsigned long long w = 0;
  for (int k = 0; k < 8; ++k)
    w |= (unsigned long long)(i + k < zlen ? __ldg(zi + i + k) : 0) << (8 * k);
  int found = 0;
  for (int s = 0; s < 8; ++s) {
    const unsigned long long v = w >> s;
    if (((v >> 1) & 3) != 2 || ((v >> 3) & 31) > 29 || ((v >> 8) & 31) > 29) continue;
    const long long bit = 8 * i + s;
    if (!header_ok(zi, zlen, bit)) continue;
    ++found;
    const long long t = D[DD_TILE_OFF] + bit / MRX_PNG_DEC_TILE_BITS;
    const int slot = atomicAdd(tile_cnt + t, 1);
    if (slot < K) cand[t * K + slot] = bit;
  }
  if (found)
    atomicAdd(reinterpret_cast<unsigned long long *>(info + size_t(b) * MRX_PNG_DEC_INFO_WORDS +
                                                     MRX_PNG_DEC_CAND), (unsigned long long)found);
}

constexpr int kWarps = 4;   // warps per CTA of the measure and expand kernels

// ------------------------------------------------------------------ measure: one warp per slot
__global__ void __launch_bounds__(32 * kWarps) png_measure_kernel(
    const long long *__restrict__ desc, const unsigned char *__restrict__ z, int K,
    const long long *__restrict__ cand, const int *__restrict__ tile_cnt,
    long long *__restrict__ meas, const int *__restrict__ status) {
  __shared__ InflateSmem S[kWarps];
  const int b = blockIdx.y, w = threadIdx.x >> 5;
  const long long *D = desc + size_t(b) * DD_WORDS;
  const long long slot = (long long)blockIdx.x * kWarps + w;
  if (slot >= D[DD_NTILES] * K || status[b]) return;
  const long long t = D[DD_TILE_OFF] + slot / K;
  const long long g = t * K + slot % K;
  if (slot % K >= tile_cnt[t]) return;
  const BlockOut r = run_block(S[w], z + D[DD_Z_OFF], D[DD_Z_LEN], cand[g], 0, false,
                               D[DD_WSIZE], nullptr, 0, 0);
  if ((threadIdx.x & 31) == 0) {
    long long *m = meas + 4 * g;
    m[0] = r.end;
    m[1] = r.len;
    m[2] = r.need;
    m[3] = r.err ? 0 : 1 | (r.final << 1);
  }
}

// ------------------------------------------------------------------ chain: one warp per image
// The image's true block list from its first bit: a measured candidate where one starts at the
// current bit, else the block measured here.  Errors are placed by the bytes described before
// them: one at or before the image's last byte (a distance too far back: before it) is refused,
// as libpng refuses it; past it libpng has every row and only warns, so the chain ends there.
__global__ void __launch_bounds__(32) png_chain_kernel(
    const long long *__restrict__ desc, const unsigned char *__restrict__ z, int K,
    const long long *__restrict__ cand, const int *__restrict__ tile_cnt,
    const long long *__restrict__ meas, long long *__restrict__ blocks, int *__restrict__ cells,
    long long *__restrict__ info, int *__restrict__ status) {
  __shared__ InflateSmem S;
  const int b = blockIdx.x, lane = threadIdx.x;
  const long long *D = desc + size_t(b) * DD_WORDS;
  long long *I = info + size_t(b) * MRX_PNG_DEC_INFO_WORDS;
  if (status[b]) return;
  const long long n = D[DD_N], zlen = D[DD_Z_LEN], wsize = D[DD_WSIZE], cap = D[DD_BLK_CAP];
  const unsigned char *zi = z + D[DD_Z_OFF];
  long long *blk = blocks + 2 * D[DD_BLK_OFF];
  long long bit = 16, p = 0, nblk = 0, seq = 0;   // the 2-byte zlib header was checked on the host
  int err = 0;
  bool final = false, past = false;
  while (!err && !final && !past) {
    const long long t = D[DD_TILE_OFF] + bit / MRX_PNG_DEC_TILE_BITS;
    const long long g = t * K + lane;
    const bool hit = t < D[DD_TILE_OFF] + D[DD_NTILES] && lane < K && lane < tile_cnt[t] &&
                     cand[g] == bit && (meas[4 * g + 3] & 1);
    const unsigned ballot = __ballot_sync(0xFFFFFFFFu, hit);
    BlockOut r;
    bool redo = !ballot;
    if (ballot) {
      const long long *m = meas + 4 * (t * K + (__ffs(ballot) - 1));
      r.end = m[0];
      r.len = m[1];
      r.need = m[2];
      r.final = int(m[3] >> 1);
      r.err = 0;
      redo = r.need > p;   // reaches before the stream start: find where
    }
    if (redo) {
      r = run_block(S, zi, zlen, bit, p, true, wsize, nullptr, 0, n);
      r.err_at -= p;
      ++seq;
    }
    if (lane == 0 && nblk < cap) {
      blk[2 * nblk] = bit;
      blk[2 * nblk + 1] = p;
    }
    ++nblk;
    if (r.err) {
      const long long at = p + r.err_at;
      if (r.err != MRX_PNG_ST_TRUNC && (at > n || (r.err == MRX_PNG_ST_DIST && at >= n))) {
        past = true;
      } else {
        err = r.err;
      }
      p = at;
    } else {
      p += r.len;
      bit = r.end;
      final = r.final;
    }
  }
  // the trailer is checked when the stream holds exactly the image's rows; with more, libpng
  // has every row before it reaches the trailer and only warns
  long long adler = -1;
  if (!err && !past) {
    if (p < n) {
      err = MRX_PNG_ST_TRUNC;
    } else if (lane == 0) {
      Bits br{zi, zlen, (bit + 7) >> 3, 0, 0};   // byte-aligned, big-endian
      adler = 0;
      for (int k = 0; k < 4; ++k) adler = adler << 8 | br.get(8);
      if (br.over()) err = MRX_PNG_ST_TRUNC;
      if (p > n) adler = -1;
    }
    err = __shfl_sync(0xFFFFFFFFu, err, 0);
  }
  if (!err && p < n) err = MRX_PNG_ST_TRUNC;
  // more blocks than the list holds: this warp expands the image itself, in order
  if (!err && nblk > cap) {
    long long q = 0, at = 16;
    for (long long k = 0; k < nblk; ++k) {
      const BlockOut r = run_block(S, zi, zlen, at, q, true, wsize, cells + D[DD_FILT_OFF], 0, n);
      if (r.err) break;
      q += r.len;
      at = r.end;
    }
  }
  if (lane == 0) {
    if (err) atomicOr(status + b, err);
    I[MRX_PNG_DEC_NBLK] = nblk;
    I[MRX_PNG_DEC_SEQ] = seq;
    I[MRX_PNG_DEC_OUT] = p;
    I[MRX_PNG_DEC_ADLER] = err ? -1 : adler;
  }
}

// ------------------------------------------------------------------ expand: one warp per block
__global__ void __launch_bounds__(32 * kWarps) png_expand_kernel(
    const long long *__restrict__ desc, const unsigned char *__restrict__ z,
    const long long *__restrict__ blocks, const long long *__restrict__ info,
    int *__restrict__ cells, const int *__restrict__ status) {
  __shared__ InflateSmem S[kWarps];
  const int b = blockIdx.y, w = threadIdx.x >> 5;
  const long long *D = desc + size_t(b) * DD_WORDS;
  const long long k = (long long)blockIdx.x * kWarps + w;
  const long long nblk = info[size_t(b) * MRX_PNG_DEC_INFO_WORDS + MRX_PNG_DEC_NBLK];
  if (status[b] || k >= nblk || nblk > D[DD_BLK_CAP]) return;
  const long long *e = blocks + 2 * (D[DD_BLK_OFF] + k);
  const long long n = D[DD_N];
  if (e[1] >= n) return;
  // a block of the chain decodes as it did there, up to its error if the chain ended on one
  run_block(S[w], z + D[DD_Z_OFF], D[DD_Z_LEN], e[0], e[1], true, D[DD_WSIZE],
            cells + D[DD_FILT_OFF], e[1], n);
}

// ------------------------------------------------------------------ resolve: blocks in order
// A reference points before its block, so once the earlier blocks hold bytes it reads a byte.
__global__ void __launch_bounds__(kThreads) png_resolve_kernel(
    const long long *__restrict__ desc, const long long *__restrict__ blocks,
    const long long *__restrict__ info, const int *__restrict__ cells,
    unsigned char *__restrict__ filt, const int *__restrict__ status) {
  const int b = blockIdx.x;
  const long long *D = desc + size_t(b) * DD_WORDS;
  if (status[b]) return;
  const long long *I = info + size_t(b) * MRX_PNG_DEC_INFO_WORDS;
  const long long n = D[DD_N], nblk = I[MRX_PNG_DEC_NBLK];
  const bool listed = nblk <= D[DD_BLK_CAP];
  const long long *blk = blocks + 2 * D[DD_BLK_OFF];
  const int *c = cells + D[DD_FILT_OFF];
  unsigned char *out = filt + D[DD_FILT_OFF];
  for (long long k = 0; k < (listed ? nblk : 1); ++k) {
    const long long lo = listed ? blk[2 * k + 1] : 0;
    if (lo >= n) break;
    const long long hi = listed && k + 1 < nblk ? min(blk[2 * k + 3], n) : n;
    for (long long q = lo + threadIdx.x; q < hi; q += kThreads) {
      const int v = c[q];
      out[q] = v < 256 ? (unsigned char)v : out[v - 256];
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------ Adler-32 partial sums
__global__ void __launch_bounds__(kThreads) png_adler_kernel(const long long *__restrict__ desc,
                                                             const unsigned char *__restrict__ filt,
                                                             long long *__restrict__ info,
                                                             const int *__restrict__ status) {
  const int b = blockIdx.y;
  const long long *D = desc + size_t(b) * DD_WORDS;
  long long *I = info + size_t(b) * MRX_PNG_DEC_INFO_WORDS;
  const long long n = D[DD_N];
  if (status[b] || I[MRX_PNG_DEC_ADLER] < 0 || (long long)blockIdx.x * kTile >= n) return;
  const unsigned char *s = filt + D[DD_FILT_OFF];
  unsigned long long a = 0, bs = 0;
  for (long long i = (long long)blockIdx.x * kTile + threadIdx.x;
       i < min(n, (long long)(blockIdx.x + 1) * kTile); i += kThreads) {
    const unsigned v = s[i];
    a += v;
    bs += (unsigned long long)((n - i) % kMod) * v;
  }
  a = warp_sum(a);
  bs = warp_sum(bs);
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(reinterpret_cast<unsigned long long *>(I + MRX_PNG_DEC_ADLER_A), a % kMod);
    atomicAdd(reinterpret_cast<unsigned long long *>(I + MRX_PNG_DEC_ADLER_B), bs % kMod);
  }
}

// ------------------------------------------------------------------ unfilter (wavefront)
__device__ __forceinline__ int paeth(int a, int b, int c) {
  const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
  return pa <= pb && pa <= pc ? a : pb <= pc ? b : c;
}

__global__ void __launch_bounds__(kThreads) png_unfilter_kernel(const long long *__restrict__ desc,
                                                                unsigned char *__restrict__ filt,
                                                                const long long *__restrict__ info,
                                                                int *__restrict__ status) {
  __shared__ int s_skip;
  const int b = blockIdx.x, t = threadIdx.x;
  const long long *D = desc + size_t(b) * DD_WORDS;
  const long long *I = info + size_t(b) * MRX_PNG_DEC_INFO_WORDS;
  if (t == 0) {
    int st = status[b];
    const long long want = I[MRX_PNG_DEC_ADLER];
    if (!st && want >= 0) {
      const long long n = D[DD_N];
      const unsigned a = unsigned((1 + I[MRX_PNG_DEC_ADLER_A]) % kMod);
      const unsigned bb = unsigned((n % kMod + I[MRX_PNG_DEC_ADLER_B]) % kMod);
      if ((((unsigned long long)bb << 16) | a) != (unsigned long long)want) {
        st |= MRX_PNG_ST_ADLER;
        atomicOr(status + b, MRX_PNG_ST_ADLER);
      }
    }
    s_skip = st;
  }
  __syncthreads();
  if (s_skip) return;
  const int H = int(D[DD_H]), W = int(D[DD_W]), ct = int(D[DD_CT]), depth = int(D[DD_DEPTH]);
  const bool il = D[DD_INTERLACE] != 0;
  const int bits_pp = channels_of(ct) * depth, bpp = max(1, bits_pp >> 3);
  unsigned char *base = filt + D[DD_FILT_OFF];
  int bad = 0;
  for (int pass = 0; pass < (il ? 7 : 1); ++pass) {
    int pw, ph;
    pass_size(pass, il, H, W, pw, ph);
    if (pw == 0 || ph == 0) continue;
    const long long rb = row_bytes(pw, bits_pp), stride = rb + 1;
    const long long cols = (rb + bpp - 1) / bpp;
    for (long long g = 0; g < ph; g += kThreads) {
      const long long r = g + t;
      unsigned char *row = base + r * stride;
      const bool live = r < ph;
      const int f = live ? row[0] : 0;
      if (f > 4) bad = 1;
      int left[8] = {0, 0, 0, 0, 0, 0, 0, 0}, upleft[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      for (long long s = 0; s < cols + kThreads - 1; ++s) {
        const long long c = s - t;
        if (live && c >= 0 && c < cols && f <= 4) {
          for (int j = 0; j < bpp; ++j) {
            const long long i = c * bpp + j;
            if (i >= rb) break;
            const int up = r > 0 ? row[i + 1 - stride] : 0;
            int x = row[i + 1];
            switch (f) {
              case 1: x += left[j]; break;
              case 2: x += up; break;
              case 3: x += (left[j] + up) >> 1; break;
              case 4: x += paeth(left[j], up, upleft[j]); break;
              default: break;
            }
            x &= 255;
            row[i + 1] = (unsigned char)x;
            left[j] = x;
            upleft[j] = up;
          }
        }
        __syncthreads();
      }
    }
    base += ph * stride;
  }
  if (bad) atomicOr(status + b, MRX_PNG_ST_FILTER);
}

// ------------------------------------------------------------------ pixels
__global__ void __launch_bounds__(kThreads) png_pixels_kernel(
    const long long *__restrict__ desc, const unsigned char *__restrict__ filt,
    const unsigned char *__restrict__ plte, const int *__restrict__ status,
    unsigned char *__restrict__ out, const long long *__restrict__ out_off) {
  const int b = blockIdx.y;
  const long long *D = desc + size_t(b) * DD_WORDS;
  const int H = int(D[DD_H]), W = int(D[DD_W]);
  const long long q = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (q >= (long long)H * W || status[b]) return;
  const int y = int(q / W), x = int(q - (long long)y * W);
  const int ct = int(D[DD_CT]), depth = int(D[DD_DEPTH]);
  const bool il = D[DD_INTERLACE] != 0;
  const int nc = channels_of(ct), bits_pp = nc * depth;
  // the pass holding (x, y) and the pass's rows before it
  int pass = 0, px = x, py = y;
  long long at = D[DD_FILT_OFF];
  if (il) {
    for (pass = 0; pass < 7; ++pass) {
      const int x0 = c_adam7[pass][0], y0 = c_adam7[pass][1];
      const int dx = c_adam7[pass][2], dy = c_adam7[pass][3];
      if (x % dx == x0 && y % dy == y0) break;
      int pw, ph;
      pass_size(pass, true, H, W, pw, ph);
      if (pw && ph) at += ph * (row_bytes(pw, bits_pp) + 1);
    }
    px = x / c_adam7[pass][2];
    py = y / c_adam7[pass][3];
  }
  int pw, ph;
  pass_size(pass, il, H, W, pw, ph);
  const unsigned char *row = filt + at + py * (row_bytes(pw, bits_pp) + 1) + 1;
  int v[4];
  if (depth == 8 || depth == 16) {
    const int step = depth >> 3;
    for (int k = 0; k < nc; ++k) v[k] = row[((long long)px * nc + k) * step];   // high byte
  } else {
    const long long bit = (long long)px * depth;
    const int s = row[bit >> 3] >> (8 - depth - int(bit & 7)) & ((1 << depth) - 1);
    v[0] = ct == 3 ? s : s * (255 / ((1 << depth) - 1));
  }
  unsigned char rgb[3];
  if (ct == 3) {
    const unsigned char *pe = plte + size_t(b) * 768 + 3 * v[0];
    const bool in = v[0] < int(D[DD_PLTE_N]);
    for (int k = 0; k < 3; ++k) rgb[k] = in ? pe[k] : 0;
  } else if (ct == 2 || ct == 6) {
    for (int k = 0; k < 3; ++k) rgb[k] = (unsigned char)v[k];
  } else {
    rgb[0] = rgb[1] = rgb[2] = (unsigned char)v[0];
  }
  // OpenCV's EXIF orientation as an index map on the store (as mrx_jpeg_pixels)
  int oy = y, ox = x, ow = W;
  switch (int(D[DD_ORIENT])) {
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

}  // namespace
}  // namespace mrx

using namespace mrx;

extern "C" int mrx_png_decode(const unsigned char *d_files, const long long *d_desc,
                              const long long *d_chunks, const unsigned char *d_plte, int B,
                              long long n_chunks, long long max_n, long long max_pixels,
                              long long max_zlen, long long max_tiles, long long total_tiles,
                              long long max_blocks, int K, unsigned char *d_z, long long *d_cand,
                              int *d_tile_cnt, long long *d_meas, int *d_cells,
                              unsigned char *d_filt, long long *d_blocks, long long *d_info,
                              int *d_status, unsigned char *d_out, const long long *d_out_off,
                              void *stream) {
  MRX_CHECK_ARG(d_files && d_desc && d_chunks && d_plte && d_z && d_cand && d_tile_cnt &&
                    d_meas && d_cells && d_filt && d_blocks && d_info && d_status && d_out &&
                    d_out_off,
                "mrx_png_decode: null pointer");
  MRX_CHECK_ARG(B >= 0 && B <= MRX_MAX_BATCH, "mrx_png_decode: B=%d outside [0, %d]", B,
                MRX_MAX_BATCH);
  MRX_CHECK_ARG(n_chunks >= B && n_chunks <= (1LL << 31),
                "mrx_png_decode: n_chunks=%lld outside [B, 2^31]", n_chunks);
  MRX_CHECK_ARG(max_n >= 2 && max_n <= MRX_PNG_DEC_MAX_FILTERED,
                "mrx_png_decode: max_n=%lld outside [2, %lld]", max_n,
                (long long)MRX_PNG_DEC_MAX_FILTERED);
  MRX_CHECK_ARG(max_pixels >= 1 && max_pixels <= (1LL << 30),
                "mrx_png_decode: max_pixels=%lld outside [1, 2^30]", max_pixels);
  MRX_CHECK_ARG(max_zlen >= 2 && max_zlen <= MRX_PNG_DEC_MAX_FILE && max_tiles >= 1 &&
                    total_tiles >= max_tiles && max_blocks >= 1,
                "mrx_png_decode: max_zlen=%lld, max_tiles=%lld, total_tiles=%lld, "
                "max_blocks=%lld",
                max_zlen, max_tiles, total_tiles, max_blocks);
  MRX_CHECK_ARG(K >= 0 && K <= MRX_PNG_DEC_MAX_SLOTS, "mrx_png_decode: K=%d outside [0, %d]", K,
                MRX_PNG_DEC_MAX_SLOTS);
  if (B == 0) return MRX_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MRX_CUDA(cudaMemsetAsync(d_status, 0, sizeof(int) * size_t(B), st));
  MRX_CUDA(cudaMemsetAsync(d_info, 0, sizeof(long long) * MRX_PNG_DEC_INFO_WORDS * size_t(B), st));
  MRX_CUDA(cudaMemsetAsync(d_tile_cnt, 0, sizeof(int) * size_t(total_tiles), st));
  png_gather_kernel<<<unsigned((n_chunks + kGatherWarps - 1) / kGatherWarps), 32 * kGatherWarps, 0,
                      st>>>(d_files, d_desc, d_chunks, n_chunks, d_z, d_status);
  MRX_LAUNCH_CHECK("png_gather_kernel");
  if (K > 0) {
    const dim3 gf(unsigned((max_zlen + kThreads - 1) / kThreads), B);
    png_find_kernel<<<gf, kThreads, 0, st>>>(d_desc, d_z, K, d_cand, d_tile_cnt, d_info, d_status);
    MRX_LAUNCH_CHECK("png_find_kernel");
    const dim3 gm(unsigned((max_tiles * K + kWarps - 1) / kWarps), B);
    png_measure_kernel<<<gm, 32 * kWarps, 0, st>>>(d_desc, d_z, K, d_cand, d_tile_cnt, d_meas,
                                                   d_status);
    MRX_LAUNCH_CHECK("png_measure_kernel");
  }
  png_chain_kernel<<<B, 32, 0, st>>>(d_desc, d_z, K, d_cand, d_tile_cnt, d_meas, d_blocks,
                                     d_cells, d_info, d_status);
  MRX_LAUNCH_CHECK("png_chain_kernel");
  const dim3 ge(unsigned((max_blocks + kWarps - 1) / kWarps), B);
  png_expand_kernel<<<ge, 32 * kWarps, 0, st>>>(d_desc, d_z, d_blocks, d_info, d_cells, d_status);
  MRX_LAUNCH_CHECK("png_expand_kernel");
  png_resolve_kernel<<<B, kThreads, 0, st>>>(d_desc, d_blocks, d_info, d_cells, d_filt, d_status);
  MRX_LAUNCH_CHECK("png_resolve_kernel");
  const dim3 ga(unsigned((max_n + kTile - 1) / kTile), B);
  png_adler_kernel<<<ga, kThreads, 0, st>>>(d_desc, d_filt, d_info, d_status);
  MRX_LAUNCH_CHECK("png_adler_kernel");
  png_unfilter_kernel<<<B, kThreads, 0, st>>>(d_desc, d_filt, d_info, d_status);
  MRX_LAUNCH_CHECK("png_unfilter_kernel");
  const dim3 gp(unsigned((max_pixels + kThreads - 1) / kThreads), B);
  png_pixels_kernel<<<gp, kThreads, 0, st>>>(d_desc, d_filt, d_plte, d_status, d_out, d_out_off);
  MRX_LAUNCH_CHECK("png_pixels_kernel");
  return MRX_OK;
}
