// png.cu -- PNG files byte for byte as cv2.imwrite(path, rgb[..., ::-1]) writes them: Sub-filtered
// rows (unfiltered when the width is 1), zlib level 1 / Z_RLE / memLevel 8, 8192-byte IDAT chunks.
//
// One stream-ordered batch (mrx.h, "PNG encode"; tests/png_oracle.py restates every step):
//   filter   the filtered rows into the stream buffer
//   starts   per tile of kTile positions: the stretches (bytes equal to their predecessor) that
//            start in it, and the Adler-32 partial sums                 -> scan over tiles
//   stretch  each stretch's first and one-past-last position
//   symbols  each position's symbol code (zlib's deflate_rle parse), symbols per tile -> scan
//   symidx   each block's first position (a block is 16383 symbols)
//   hist     one CTA per block: literal/length frequencies and the match count
//   trees    one thread per block: trees.c's trees, the block type, the dynamic header bits
//   layout   one thread per image: each block's first bit, the stream and file sizes
//   weights  per tile: the code bits of its symbols                      -> scan over tiles
//   emit     every symbol's code at its bit, stored blocks' bytes
//   frame    one warp per block: block header, tree description, end-of-block code, LEN/NLEN
//   file     one warp per IDAT chunk: chunk bytes and CRC-32; signature, IHDR and IEND
#include "common.cuh"

namespace mrx {
namespace {

constexpr int kThreads = 256;
constexpr int kItems = 8;
constexpr int kTile = kThreads * kItems;   // png.TILE
constexpr int kSyms = 16383;               // symbols per block (zlib's lit_bufsize - 1)
constexpr int kMaxMatch = 258;
constexpr int kLCodes = 286, kDCodes = 30, kBLCodes = 19;
constexpr int kHeap = 2 * kLCodes + 1;
constexpr int kEndBlock = 256;
constexpr int kTabWords = 654;             // per block: freq[287], code[287], header bits[80]
constexpr int kFreq = 0, kCode = 287, kHdr = 574, kHdrWords = 80;
constexpr int kIdat = 8192;
constexpr unsigned kMod = 65521;

// desc words per image (png.py D_*)
enum {
  D_SRC = 0, D_H, D_W, D_N, D_STREAM_OFF, D_TILE_OFF, D_NTILES, D_STRETCH_OFF, D_STRETCH_CAP,
  D_BLK_OFF, D_MAXBLK, D_BLKPOS_OFF, D_ZBUF_OFF, D_OUT_OFF, D_WBITS, D_CMF, D_FLG,
  DESC_WORDS = 20
};
// per block int64 (MRX_PNG_BLK_*) and per image int64 (MRX_PNG_IMG_*)
enum { BK_TYPE = 0, BK_LAST, BK_HDR_BITS, BK_DATA_BITS, BK_EOB, BK_BIT, BK_PBASE, BK_BITS };
enum { IM_NSYM = 0, IM_NBLK, IM_ADLER_A, IM_ADLER_B, IM_BITS, IM_ZLEN, IM_CHUNKS, IM_FILE };

__constant__ unsigned char c_extra_lbits[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2,
                                                2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ unsigned char c_extra_dbits[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6,
                                                6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ unsigned char c_extra_blbits[19] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
                                                 0, 0, 0, 0, 0, 0, 2, 3, 7};
__constant__ unsigned char c_bl_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5,
                                             11, 4, 12, 3, 13, 2, 14, 1, 15};
__constant__ unsigned char c_base_length[29] = {0,  1,  2,  3,  4,  5,   6,   7,   8,   10,
                                                12, 14, 16, 20, 24, 28,  32,  40,  48,  56,
                                                64, 80, 96, 112, 128, 160, 192, 224, 255};

__device__ __forceinline__ int length_code(int lc) {   // zlib's _length_code[lc]
  int c = 28;
  while (c_base_length[c] > lc) --c;
  return c;
}

__device__ __forceinline__ int static_llen(int c) {
  return c < 144 ? 8 : c < 256 ? 9 : c < 280 ? 7 : 8;
}

__device__ __forceinline__ unsigned bi_reverse(unsigned code, int n) {
  return __brev(code) >> (32 - n);
}

__device__ __forceinline__ unsigned static_lcode(int c) {   // gen_codes over static_llen
  if (c < 144) return bi_reverse(48 + c, 8);
  if (c < 256) return bi_reverse(400 + (c - 144), 9);
  if (c < 280) return bi_reverse(c - 256, 7);
  return bi_reverse(192 + (c - 280), 8);
}

// nbits (<= 64) of v, least significant first, at bit `bit` of a zeroed little-endian buffer
__device__ __forceinline__ void put_bits(unsigned *buf, long long bit, unsigned long long v,
                                         int nbits) {
  while (nbits > 0) {
    const int sh = int(bit & 31);
    const int take = min(32 - sh, nbits);
    const unsigned part = take == 32 ? unsigned(v) : unsigned(v & ((1ull << take) - 1));
    if (part) atomicOr(buf + (bit >> 5), part << sh);
    v >>= take;
    bit += take;
    nbits -= take;
  }
}

struct Tile {
  const long long *D;
  const unsigned char *s;
  int n, t, i0;
};

__device__ __forceinline__ bool tile_of(const long long *desc, const unsigned char *stream,
                                        Tile &T) {
  const int b = blockIdx.y;
  T.D = desc + size_t(b) * DESC_WORDS;
  T.t = blockIdx.x;
  if (T.t >= int(T.D[D_NTILES])) return false;
  T.s = stream + T.D[D_STREAM_OFF];
  T.n = int(T.D[D_N]);
  T.i0 = T.t * kTile + threadIdx.x * kItems;
  return true;
}

__device__ __forceinline__ bool eq_at(const unsigned char *s, int i) {
  return i > 0 && s[i] == s[i - 1];
}

__device__ __forceinline__ bool start_at(const unsigned char *s, int i) {
  return eq_at(s, i) && !eq_at(s, i - 1);
}

// ------------------------------------------------------------------ filter
__global__ void __launch_bounds__(kThreads) png_filter_kernel(const long long *__restrict__ desc,
                                                              unsigned char *__restrict__ stream,
                                                              int *__restrict__ blk_pos,
                                                              long long *__restrict__ img_info) {
  const int b = blockIdx.y;
  const long long *D = desc + size_t(b) * DESC_WORDS;
  const int n = int(D[D_N]), W = int(D[D_W]);
  const int rowlen = 3 * W + 1;
  const unsigned char *src = reinterpret_cast<const unsigned char *>(D[D_SRC]);
  unsigned char *s = stream + D[D_STREAM_OFF];
  const int first = blockIdx.x * kThreads + threadIdx.x;
  if (first < 8) img_info[size_t(b) * 8 + first] = 0;
  for (int k = first; k <= int(D[D_MAXBLK]); k += gridDim.x * kThreads)
    blk_pos[D[D_BLKPOS_OFF] + k] = n;
  for (int i = first; i < n; i += gridDim.x * kThreads) {
    const int r = i / rowlen, c = i - r * rowlen;
    unsigned char v;
    if (c == 0) {
      v = W > 1 ? 1 : 0;
    } else {
      const unsigned char *row = src + (long long)r * (3 * W);
      v = row[c - 1];
      if (W > 1 && c - 1 >= 3) v = (unsigned char)(v - row[c - 4]);
    }
    s[i] = v;
  }
}

// ------------------------------------------------------------------ stretch starts + Adler-32
__global__ void __launch_bounds__(kThreads) png_starts_kernel(const long long *__restrict__ desc,
                                                              const unsigned char *__restrict__ stream,
                                                              long long *__restrict__ tiles,
                                                              long long *__restrict__ img_info) {
  __shared__ long long s_warp[kThreads / 32];
  Tile T;
  if (!tile_of(desc, stream, T)) return;
  long long cnt = 0;
  unsigned long long a = 0, bsum = 0;
  for (int j = 0; j < kItems; ++j) {
    const int i = T.i0 + j;
    if (i >= T.n) break;
    cnt += start_at(T.s, i);
    const unsigned v = T.s[i];
    a += v;
    bsum += (unsigned long long)((unsigned(T.n - i)) % kMod) * v;
  }
  long long tot;
  block_exclusive_scan<long long, kThreads>(cnt, s_warp, tot);
  if (threadIdx.x == 0) tiles[T.D[D_TILE_OFF] + T.t] = tot;
  a = warp_sum(a);
  bsum = warp_sum(bsum);
  if ((threadIdx.x & 31) == 0) {
    long long *info = img_info + size_t(blockIdx.y) * 8;
    atomicAdd(reinterpret_cast<unsigned long long *>(info + IM_ADLER_A), a % kMod);
    atomicAdd(reinterpret_cast<unsigned long long *>(info + IM_ADLER_B), bsum % kMod);
  }
}

// stretch ids of a thread's positions: the exclusive count of starts before its first position
__device__ __forceinline__ long long stretch_base(const Tile &T, const long long *tiles,
                                                  long long *s_warp) {
  long long cnt = 0;
  for (int j = 0; j < kItems; ++j) {
    const int i = T.i0 + j;
    if (i >= T.n) break;
    cnt += start_at(T.s, i);
  }
  long long tot;
  const long long ex = block_exclusive_scan<long long, kThreads>(cnt, s_warp, tot);
  const long long *tb = tiles + T.D[D_TILE_OFF];
  return tb[T.t] - tb[0] + ex;
}

__global__ void __launch_bounds__(kThreads) png_stretch_kernel(const long long *__restrict__ desc,
                                                               const unsigned char *__restrict__ stream,
                                                               const long long *__restrict__ tiles,
                                                               int *__restrict__ stretch) {
  __shared__ long long s_warp[kThreads / 32];
  Tile T;
  if (!tile_of(desc, stream, T)) return;
  long long id = stretch_base(T, tiles, s_warp);
  int *st = stretch + T.D[D_STRETCH_OFF];
  int *en = st + T.D[D_STRETCH_CAP];
  for (int j = 0; j < kItems; ++j) {
    const int i = T.i0 + j;
    if (i >= T.n) break;
    if (start_at(T.s, i)) st[id++] = i;
    if (eq_at(T.s, i) && (i + 1 == T.n || !eq_at(T.s, i + 1))) en[id - 1] = i + 1;
  }
}

// deflate_rle: a stretch of L bytes is floor(L/258) matches of 258, then a match of the rest r
// when r >= 3, else r literals; every other byte is a literal.  sym: -1 inside a match, the
// literal byte, or 256 + length - 3.
__global__ void __launch_bounds__(kThreads) png_symbols_kernel(const long long *__restrict__ desc,
                                                               const unsigned char *__restrict__ stream,
                                                               const long long *__restrict__ tiles,
                                                               const int *__restrict__ stretch,
                                                               short *__restrict__ sym,
                                                               long long *__restrict__ sym_tiles) {
  __shared__ long long s_warp[kThreads / 32];
  Tile T;
  if (!tile_of(desc, stream, T)) return;
  long long id = stretch_base(T, tiles, s_warp) - 1;
  const int *st = stretch + T.D[D_STRETCH_OFF];
  const int *en = st + T.D[D_STRETCH_CAP];
  short *y = sym + T.D[D_STREAM_OFF];
  long long cnt = 0;
  for (int j = 0; j < kItems; ++j) {
    const int i = T.i0 + j;
    if (i >= T.n) break;
    short code = T.s[i];
    if (eq_at(T.s, i)) {
      id += start_at(T.s, i);
      const int a = st[id], L = en[id] - a, k = i - a;
      const int full = (L / kMaxMatch) * kMaxMatch, r = L - full;
      if (k < full) code = k % kMaxMatch == 0 ? short(256 + kMaxMatch - 3) : short(-1);
      else if (r >= 3) code = k == full ? short(256 + r - 3) : short(-1);
    }
    y[i] = code;
    cnt += code >= 0;
  }
  long long tot;
  block_exclusive_scan<long long, kThreads>(cnt, s_warp, tot);
  if (threadIdx.x == 0) sym_tiles[T.D[D_TILE_OFF] + T.t] = tot;
}

__global__ void __launch_bounds__(kThreads) png_symidx_kernel(const long long *__restrict__ desc,
                                                              const unsigned char *__restrict__ stream,
                                                              const short *__restrict__ sym,
                                                              const long long *__restrict__ sym_tiles,
                                                              int *__restrict__ blk_pos,
                                                              long long *__restrict__ img_info) {
  __shared__ long long s_warp[kThreads / 32];
  Tile T;
  if (!tile_of(desc, stream, T)) return;
  const short *y = sym + T.D[D_STREAM_OFF];
  long long cnt = 0;
  for (int j = 0; j < kItems; ++j) {
    const int i = T.i0 + j;
    if (i >= T.n) break;
    cnt += y[i] >= 0;
  }
  long long tot;
  const long long ex = block_exclusive_scan<long long, kThreads>(cnt, s_warp, tot);
  const long long *tb = sym_tiles + T.D[D_TILE_OFF];
  long long k = tb[T.t] - tb[0] + ex;
  int *bp = blk_pos + T.D[D_BLKPOS_OFF];
  for (int j = 0; j < kItems; ++j) {
    const int i = T.i0 + j;
    if (i >= T.n) break;
    if (y[i] >= 0) {
      if (k % kSyms == 0) bp[k / kSyms] = i;
      ++k;
    }
  }
  if (T.t == int(T.D[D_NTILES]) - 1 && threadIdx.x == 0) {
    const long long nsym = tb[T.t + 1] - tb[0];
    img_info[size_t(blockIdx.y) * 8 + IM_NSYM] = nsym;
    img_info[size_t(blockIdx.y) * 8 + IM_NBLK] = nsym / kSyms + 1;
  }
}

// ------------------------------------------------------------------ histogram
__global__ void __launch_bounds__(kThreads) png_hist_kernel(const long long *__restrict__ desc,
                                                            const short *__restrict__ sym,
                                                            const int *__restrict__ blk_pos,
                                                            const long long *__restrict__ img_info,
                                                            int *__restrict__ blk_tab) {
  __shared__ int h[287];
  const int b = blockIdx.y, k = blockIdx.x;
  const long long *D = desc + size_t(b) * DESC_WORDS;
  if (k >= img_info[size_t(b) * 8 + IM_NBLK]) return;
  for (int c = threadIdx.x; c < 287; c += kThreads) h[c] = c == kEndBlock;
  __syncthreads();
  const int *bp = blk_pos + D[D_BLKPOS_OFF];
  const short *y = sym + D[D_STREAM_OFF];
  for (int i = bp[k] + threadIdx.x; i < bp[k + 1]; i += kThreads) {
    const int c = y[i];
    if (c < 0) continue;
    if (c < 256) {
      atomicAdd(&h[c], 1);
    } else {
      atomicAdd(&h[257 + length_code(c - 256)], 1);
      atomicAdd(&h[286], 1);
    }
  }
  __syncthreads();
  int *tab = blk_tab + (D[D_BLK_OFF] + k) * kTabWords;
  for (int c = threadIdx.x; c < 287; c += kThreads) tab[kFreq + c] = h[c];
}

// ------------------------------------------------------------------ trees (one thread per block)
struct TreeWork {
  int freq[kHeap];
  short dad[kHeap];
  short heap[kHeap + 1];
  unsigned char len[kHeap];
  unsigned char depth[kHeap];
};

__device__ __forceinline__ bool smaller(const TreeWork &w, int n, int m) {
  return w.freq[n] < w.freq[m] || (w.freq[n] == w.freq[m] && w.depth[n] <= w.depth[m]);
}

__device__ void downheap(TreeWork &w, int heap_len, int k) {
  const int v = w.heap[k];
  int j = k << 1;
  while (j <= heap_len) {
    if (j < heap_len && smaller(w, w.heap[j + 1], w.heap[j])) ++j;
    if (smaller(w, v, w.heap[j])) break;
    w.heap[k] = w.heap[j];
    k = j;
    j <<= 1;
  }
  w.heap[k] = short(v);
}

// trees.c build_tree + gen_bitlen + gen_codes.  freq_in[0, elems) in, lens/codes out.
// kind 0: literal/length (static lengths, extra from 257), 1: distance, 2: bit lengths.
__device__ int build_tree(TreeWork &w, const int *freq_in, int elems, int kind, long long &opt_len,
                          long long &static_len, unsigned char *lens, unsigned short *codes) {
  const int max_length = kind == 2 ? 7 : 15;
  int heap_len = 0, heap_max = kHeap, max_code = -1;
  for (int n = 0; n < elems; ++n) {
    w.freq[n] = freq_in[n];
    w.depth[n] = 0;
    w.len[n] = 0;
    if (freq_in[n]) w.heap[++heap_len] = short(max_code = n);
  }
  while (heap_len < 2) {
    const int node = max_code < 2 ? ++max_code : 0;
    w.heap[++heap_len] = short(node);
    w.freq[node] = 1;
    w.depth[node] = 0;
    opt_len -= 1;
    if (kind == 0) static_len -= static_llen(node);
    if (kind == 1) static_len -= 5;
  }
  for (int n = heap_len / 2; n >= 1; --n) downheap(w, heap_len, n);
  int node = elems;
  do {
    const int n = w.heap[1];
    w.heap[1] = w.heap[heap_len--];
    downheap(w, heap_len, 1);
    const int m = w.heap[1];
    w.heap[--heap_max] = short(n);
    w.heap[--heap_max] = short(m);
    w.freq[node] = w.freq[n] + w.freq[m];
    w.depth[node] = (unsigned char)(max(w.depth[n], w.depth[m]) + 1);
    w.dad[n] = w.dad[m] = short(node);
    w.heap[1] = short(node++);
    downheap(w, heap_len, 1);
  } while (heap_len >= 2);
  w.heap[--heap_max] = w.heap[1];
  // gen_bitlen
  int bl_count[16];
  for (int i = 0; i < 16; ++i) bl_count[i] = 0;
  w.len[w.heap[heap_max]] = 0;
  int overflow = 0, h;
  for (h = heap_max + 1; h < kHeap; ++h) {
    const int n = w.heap[h];
    int bits = w.len[w.dad[n]] + 1;
    if (bits > max_length) bits = max_length, ++overflow;
    w.len[n] = (unsigned char)bits;
    if (n > max_code) continue;
    bl_count[bits]++;
    int xbits = 0;
    if (kind == 0 && n >= 257) xbits = c_extra_lbits[n - 257];
    if (kind == 1) xbits = c_extra_dbits[n];
    if (kind == 2) xbits = c_extra_blbits[n];
    const long long f = w.freq[n];
    opt_len += f * (bits + xbits);
    if (kind == 0) static_len += f * (static_llen(n) + xbits);
    if (kind == 1) static_len += f * (5 + xbits);
  }
  if (overflow) {
    do {
      int bits = max_length - 1;
      while (bl_count[bits] == 0) --bits;
      bl_count[bits]--;
      bl_count[bits + 1] += 2;
      bl_count[max_length]--;
      overflow -= 2;
    } while (overflow > 0);
    for (int bits = max_length; bits != 0; --bits) {
      int n = bl_count[bits];
      while (n != 0) {
        const int m = w.heap[--h];
        if (m > max_code) continue;
        if (w.len[m] != bits) {
          opt_len += ((long long)bits - w.len[m]) * w.freq[m];
          w.len[m] = (unsigned char)bits;
        }
        --n;
      }
    }
  }
  // gen_codes
  int next_code[16];
  int code = 0;
  next_code[0] = 0;
  for (int bits = 1; bits <= 15; ++bits) {
    code = (code + bl_count[bits - 1]) << 1;
    next_code[bits] = code;
  }
  for (int n = 0; n < elems; ++n) {
    const int l = (n <= max_code && w.freq[n]) ? w.len[n] : 0;
    lens[n] = (unsigned char)l;
    codes[n] = l ? (unsigned short)bi_reverse(next_code[l]++, l) : 0;
  }
  return max_code;
}

// scan_tree / send_tree over lens[0..max_code]; with out == nullptr only counts bl_freq
struct HdrWriter {
  unsigned *words;
  int bits;
  __device__ void put(unsigned v, int n) {
    for (int i = 0; i < n; ++i, ++bits)
      if ((v >> i) & 1) words[bits >> 5] |= 1u << (bits & 31);
  }
};

__device__ void walk_tree(const unsigned char *lens, int max_code, int *bl_freq,
                          const unsigned char *bl_len, const unsigned short *bl_code,
                          HdrWriter *out) {
  int prevlen = -1, nextlen = lens[0], count = 0;
  int max_count = 7, min_count = 4;
  if (nextlen == 0) max_count = 138, min_count = 3;
  auto emit = [&](int s, int xv, int xb) {
    if (out) {
      out->put(bl_code[s], bl_len[s]);
      if (xb) out->put(unsigned(xv), xb);
    } else {
      bl_freq[s]++;
    }
  };
  for (int n = 0; n <= max_code; ++n) {
    const int curlen = nextlen;
    nextlen = n + 1 <= max_code ? lens[n + 1] : 0xFFFF;
    if (++count < max_count && curlen == nextlen) continue;
    if (count < min_count) {
      for (; count > 0; --count) emit(curlen, 0, 0);
    } else if (curlen != 0) {
      if (curlen != prevlen) {
        emit(curlen, 0, 0);
        --count;
      }
      emit(16, count - 3, 2);
    } else if (count <= 10) {
      emit(17, count - 3, 3);
    } else {
      emit(18, count - 11, 7);
    }
    count = 0;
    prevlen = curlen;
    if (nextlen == 0) max_count = 138, min_count = 3;
    else if (curlen == nextlen) max_count = 6, min_count = 3;
    else max_count = 7, min_count = 4;
  }
}

__device__ __forceinline__ int slide_pos(const short *y, int n, int rowlen, long long w, int k) {
  // loop-top position of zlib's k-th window slide (png_oracle.slide_pos), or -1
  const long long cap = (long long)(k + 1) * w;
  long long p = cap - 262;
  if (p > n) return -1;
  long long q = p - 1;
  while (q >= 0 && y[q] < 0) --q;
  while (p < n && y[p] < 0) ++p;
  while (true) {
    if (p >= n || p >= cap - kMaxMatch) return int(p);
    const long long e = min((((q + kMaxMatch) / rowlen) + 1) * rowlen, (long long)n);
    if (min(e, cap) - p <= kMaxMatch) return int(p);
    q = p;
    ++p;
    while (p < n && y[p] < 0) ++p;
  }
}

constexpr int kTreeThreads = 32;

__global__ void __launch_bounds__(kTreeThreads) png_trees_kernel(
    const long long *__restrict__ desc, const short *__restrict__ sym,
    const int *__restrict__ blk_pos, const long long *__restrict__ img_info,
    int *__restrict__ blk_tab, long long *__restrict__ blk_info) {
  const int b = blockIdx.y, k = blockIdx.x * kTreeThreads + threadIdx.x;
  const long long *D = desc + size_t(b) * DESC_WORDS;
  const long long nblk = img_info[size_t(b) * 8 + IM_NBLK];
  if (k >= nblk) return;
  const bool last = k == nblk - 1;
  const int n = int(D[D_N]), rowlen = 3 * int(D[D_W]);
  const int *bp = blk_pos + D[D_BLKPOS_OFF];
  const int bstart = bp[k], bend = bp[k + 1];
  int *tab = blk_tab + (D[D_BLK_OFF] + k) * kTabWords;
  long long *info = blk_info + (D[D_BLK_OFF] + k) * 8;
  const short *y = sym + D[D_STREAM_OFF];

  TreeWork w;
  unsigned char llen[kLCodes], dlen[kDCodes], bllen[kBLCodes];
  unsigned short lcode[kLCodes], dcode[kDCodes], blcode[kBLCodes];
  int dfreq[kDCodes], blfreq[kBLCodes];
  long long opt_len = 0, static_len = 0;
  const int lmax = build_tree(w, tab + kFreq, kLCodes, 0, opt_len, static_len, llen, lcode);
  for (int i = 0; i < kDCodes; ++i) dfreq[i] = i == 0 ? tab[kFreq + 286] : 0;
  const int dmax = build_tree(w, dfreq, kDCodes, 1, opt_len, static_len, dlen, dcode);
  for (int i = 0; i < kBLCodes; ++i) blfreq[i] = 0;
  walk_tree(llen, lmax, blfreq, nullptr, nullptr, nullptr);
  walk_tree(dlen, dmax, blfreq, nullptr, nullptr, nullptr);
  long long bl_opt = 0, unused = 0;
  build_tree(w, blfreq, kBLCodes, 2, bl_opt, unused, bllen, blcode);
  opt_len += bl_opt;
  int max_blindex = kBLCodes - 1;
  for (; max_blindex >= 3; --max_blindex)
    if (bllen[c_bl_order[max_blindex]] != 0) break;
  opt_len += 3LL * (max_blindex + 1) + 5 + 5 + 4;
  long long opt_lenb = (opt_len + 3 + 7) >> 3;
  const long long static_lenb = (static_len + 3 + 7) >> 3;
  if (static_lenb <= opt_lenb) opt_lenb = static_lenb;

  // stored blocks need block_start >= 0: the block's first byte minus w per slide before the flush
  const long long wsize = 1LL << D[D_WBITS];
  const long long lim = last ? (long long)n + 1 : bend;
  const long long j_max = (lim - 1 + 262) / wsize - 1;
  bool can_store = true;
  if (j_max > 0) {
    long long count = j_max - 1;
    const int p = slide_pos(y, n, rowlen + 1, wsize, int(j_max));
    if (p >= 0 && p < lim) ++count;
    can_store = bstart >= count * wsize;
  }
  const long long stored_len = bend - bstart;
  int type;
  if (stored_len + 4 <= opt_lenb && can_store) type = 0;
  else if (static_lenb == opt_lenb) type = 1;
  else type = 2;

  int hdr_bits = 0;
  if (type == 2) {
    unsigned *words = reinterpret_cast<unsigned *>(tab + kHdr);
    for (int i = 0; i < kHdrWords; ++i) words[i] = 0;
    HdrWriter hw{words, 0};
    hw.put(unsigned(lmax + 1 - 257), 5);
    hw.put(unsigned(dmax + 1 - 1), 5);
    hw.put(unsigned(max_blindex + 1 - 4), 4);
    for (int r = 0; r <= max_blindex; ++r) hw.put(bllen[c_bl_order[r]], 3);
    walk_tree(llen, lmax, nullptr, bllen, blcode, &hw);
    walk_tree(dlen, dmax, nullptr, bllen, blcode, &hw);
    hdr_bits = hw.bits;
  }
  long long data_bits = 0;
  int eob = 0;
  if (type != 0) {
    for (int c = 0; c < kLCodes; ++c) {
      const int l = type == 1 ? static_llen(c) : llen[c];
      const unsigned code = type == 1 ? static_lcode(c) : lcode[c];
      tab[kCode + c] = int(code | (unsigned(l) << 16));
      const int f = tab[kFreq + c];
      if (c != kEndBlock) data_bits += (long long)f * (l + (c >= 257 ? c_extra_lbits[c - 257] : 0));
    }
    const int dl = type == 1 ? 5 : dlen[0];
    const unsigned dc = type == 1 ? 0u : dcode[0];
    tab[kCode + 286] = int(dc | (unsigned(dl) << 16));
    data_bits += (long long)tab[kFreq + 286] * dl;
    eob = tab[kCode + kEndBlock];
  }
  info[BK_TYPE] = type;
  info[BK_LAST] = last;
  info[BK_HDR_BITS] = hdr_bits;
  info[BK_DATA_BITS] = data_bits;
  info[BK_EOB] = eob;
}

// ------------------------------------------------------------------ layout (one thread per image)
__global__ void png_layout_kernel(const long long *__restrict__ desc, int B,
                                  const int *__restrict__ blk_pos,
                                  long long *__restrict__ blk_info,
                                  long long *__restrict__ img_info, long long *__restrict__ sizes) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const long long *D = desc + size_t(b) * DESC_WORDS;
  long long *im = img_info + size_t(b) * 8;
  const int *bp = blk_pos + D[D_BLKPOS_OFF];
  long long bit = 0, pbase = 0;
  for (long long k = 0; k < im[IM_NBLK]; ++k) {
    long long *info = blk_info + (D[D_BLK_OFF] + k) * 8;
    const long long start = bit;
    info[BK_BIT] = bit;
    info[BK_PBASE] = pbase;
    if (info[BK_TYPE] == 0) {
      bit = ((bit + 3 + 7) & ~7LL) + 32 + 8LL * (bp[k + 1] - bp[k]);
    } else {
      bit += 3 + info[BK_HDR_BITS] + info[BK_DATA_BITS] + (info[BK_EOB] >> 16);
      pbase += info[BK_DATA_BITS];
    }
    info[BK_BITS] = bit - start;
  }
  const long long zlen = 2 + (bit + 7) / 8 + 4;
  const long long chunks = (zlen + kIdat - 1) / kIdat;
  im[IM_BITS] = bit;
  im[IM_ZLEN] = zlen;
  im[IM_CHUNKS] = chunks;
  im[IM_FILE] = 33 + zlen + 12 * chunks + 12;
  sizes[b] = im[IM_FILE];
}

// block of position i: the last k < nblk with bp[k] <= i (binary search)
__device__ __forceinline__ int block_of(const int *bp, int nblk, int i) {
  int lo = 0, hi = nblk - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (bp[mid] <= i) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// a symbol's bits: code | extra << len | distance code << (len + extra); returns the bit count
__device__ __forceinline__ int symbol_bits(const int *tab, int c, unsigned long long &v) {
  if (c < 256) {
    const unsigned e = unsigned(tab[kCode + c]);
    v = e & 0xFFFF;
    return int(e >> 16);
  }
  const int lc = c - 256, code = length_code(lc);
  const unsigned e = unsigned(tab[kCode + 257 + code]);
  const int l = int(e >> 16), xb = c_extra_lbits[code];
  const unsigned d = unsigned(tab[kCode + 286]);
  v = (e & 0xFFFF) | ((unsigned long long)(lc - c_base_length[code]) << l) |
      ((unsigned long long)(d & 0xFFFF) << (l + xb));
  return l + xb + int(d >> 16);
}

template <bool kEmit>
__global__ void __launch_bounds__(kThreads) png_emit_kernel(
    const long long *__restrict__ desc, const unsigned char *__restrict__ stream,
    const short *__restrict__ sym, const int *__restrict__ blk_pos,
    const int *__restrict__ blk_tab, const long long *__restrict__ blk_info,
    const long long *__restrict__ img_info, long long *__restrict__ tiles,
    unsigned *__restrict__ zbuf) {
  __shared__ long long s_warp[kThreads / 32];
  Tile T;
  if (!tile_of(desc, stream, T)) return;
  const int nblk = int(img_info[size_t(blockIdx.y) * 8 + IM_NBLK]);
  const int *bp = blk_pos + T.D[D_BLKPOS_OFF];
  const short *y = sym + T.D[D_STREAM_OFF];
  const long long blk0 = T.D[D_BLK_OFF];
  int k = T.i0 < T.n ? block_of(bp, nblk, T.i0) : 0;
  const int k0 = k;
  long long cnt = 0;
  for (int j = 0; j < kItems; ++j) {
    const int i = T.i0 + j;
    if (i >= T.n) break;
    while (k + 1 < nblk && bp[k + 1] <= i) ++k;
    if (y[i] < 0 || blk_info[(blk0 + k) * 8 + BK_TYPE] == 0) continue;
    unsigned long long v;
    cnt += symbol_bits(blk_tab + (blk0 + k) * kTabWords, y[i], v);
  }
  long long tot;
  const long long ex = block_exclusive_scan<long long, kThreads>(cnt, s_warp, tot);
  if (!kEmit) {
    if (threadIdx.x == 0) tiles[T.D[D_TILE_OFF] + T.t] = tot;
    return;
  }
  const long long *tb = tiles + T.D[D_TILE_OFF];
  long long p = tb[T.t] - tb[0] + ex;
  unsigned *z = zbuf + T.D[D_ZBUF_OFF];
  k = k0;
  for (int j = 0; j < kItems; ++j) {
    const int i = T.i0 + j;
    if (i >= T.n) break;
    while (k + 1 < nblk && bp[k + 1] <= i) ++k;
    const long long *info = blk_info + (blk0 + k) * 8;
    if (info[BK_TYPE] == 0) {
      const long long byte = ((info[BK_BIT] + 3 + 7) >> 3) + 4 + (i - bp[k]);
      put_bits(z, byte * 8, T.s[i], 8);
      continue;
    }
    if (y[i] < 0) continue;
    unsigned long long v;
    const int nb = symbol_bits(blk_tab + (blk0 + k) * kTabWords, y[i], v);
    put_bits(z, info[BK_BIT] + 3 + info[BK_HDR_BITS] + p - info[BK_PBASE], v, nb);
    p += nb;
  }
}

// one warp per block: header bits, tree description, end-of-block code; LEN / NLEN when stored
__global__ void __launch_bounds__(32) png_frame_kernel(const long long *__restrict__ desc,
                                                       const int *__restrict__ blk_pos,
                                                       const int *__restrict__ blk_tab,
                                                       const long long *__restrict__ blk_info,
                                                       const long long *__restrict__ img_info,
                                                       unsigned *__restrict__ zbuf) {
  const int b = blockIdx.y, k = blockIdx.x, lane = threadIdx.x;
  const long long *D = desc + size_t(b) * DESC_WORDS;
  if (k >= img_info[size_t(b) * 8 + IM_NBLK]) return;
  const long long *info = blk_info + (D[D_BLK_OFF] + k) * 8;
  const int *tab = blk_tab + (D[D_BLK_OFF] + k) * kTabWords;
  const int *bp = blk_pos + D[D_BLKPOS_OFF];
  unsigned *z = zbuf + D[D_ZBUF_OFF];
  const long long bit = info[BK_BIT];
  const int type = int(info[BK_TYPE]);
  if (lane == 0) put_bits(z, bit, (unsigned(type) << 1) | unsigned(info[BK_LAST]), 3);
  if (type == 0) {
    if (lane == 0) {
      const unsigned len = unsigned(bp[k + 1] - bp[k]);
      put_bits(z, ((bit + 3 + 7) & ~7LL), len | ((~len & 0xFFFFu) << 16), 32);
    }
    return;
  }
  const int hb = int(info[BK_HDR_BITS]);
  for (int j = lane; j * 32 < hb; j += 32)
    put_bits(z, bit + 3 + 32LL * j, unsigned(tab[kHdr + j]), min(32, hb - 32 * j));
  if (lane == 0) {
    const unsigned e = unsigned(info[BK_EOB]);
    put_bits(z, bit + 3 + hb + info[BK_DATA_BITS], e & 0xFFFF, int(e >> 16));
  }
}

// ------------------------------------------------------------------ file
constexpr unsigned kPoly = 0xEDB88320u;

__device__ unsigned multmodp(unsigned a, unsigned b) {   // a * b modulo the CRC polynomial
  unsigned m = 1u << 31, p = 0;
  for (;;) {
    if (a & m) {
      p ^= b;
      if ((a & (m - 1)) == 0) break;
    }
    m >>= 1;
    b = b & 1 ? (b >> 1) ^ kPoly : b >> 1;
  }
  return p;
}

// crc32(A || B) from crc32(A), crc32(B) and |B|; x2n[k] = x^(2^k) modulo the polynomial
__device__ unsigned crc_combine(const unsigned *x2n, unsigned c1, unsigned c2, long long len2) {
  unsigned p = 1u << 31;
  int k = 3;
  for (long long n = len2; n; n >>= 1, ++k)
    if (n & 1) p = multmodp(x2n[k & 31], p);
  return multmodp(p, c1) ^ c2;
}

constexpr int kFileWarps = 4;

__global__ void __launch_bounds__(32 * kFileWarps) png_file_kernel(
    const long long *__restrict__ desc, const unsigned *__restrict__ zbuf,
    const long long *__restrict__ img_info, unsigned char *__restrict__ out) {
  __shared__ unsigned table[256];
  __shared__ unsigned x2n[32];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    unsigned c = unsigned(i);
    for (int j = 0; j < 8; ++j) c = c & 1 ? (c >> 1) ^ kPoly : c >> 1;
    table[i] = c;
  }
  if (threadIdx.x == 0) {
    unsigned p = 1u << 30;   // x^1
    x2n[0] = p;
    for (int i = 1; i < 32; ++i) x2n[i] = p = multmodp(p, p);
  }
  __syncthreads();
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  const long long c = (long long)blockIdx.x * kFileWarps + (threadIdx.x >> 5);
  const long long *D = desc + size_t(b) * DESC_WORDS;
  const long long *im = img_info + size_t(b) * 8;
  const long long zlen = im[IM_ZLEN], chunks = im[IM_CHUNKS];
  if (c >= chunks) return;
  const long long dlen = (im[IM_BITS] + 7) / 8;
  const unsigned a = unsigned((1 + im[IM_ADLER_A]) % kMod);
  const unsigned bb = unsigned((D[D_N] % kMod + im[IM_ADLER_B]) % kMod);
  const unsigned adler = (bb << 16) | a;
  const unsigned char *zb = reinterpret_cast<const unsigned char *>(zbuf + D[D_ZBUF_OFF]);
  unsigned char *o = out + D[D_OUT_OFF];
  auto crc_bytes = [&](unsigned crc, unsigned char v) { return table[(crc ^ v) & 0xFF] ^ (crc >> 8); };
  if (c == 0 && lane == 0) {
    const unsigned char sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1A, '\n'};
    for (int i = 0; i < 8; ++i) o[i] = sig[i];
    const unsigned H = unsigned(D[D_H]), W = unsigned(D[D_W]);
    unsigned char ih[21] = {0, 0, 0, 13, 'I', 'H', 'D', 'R',
                            (unsigned char)(W >> 24), (unsigned char)(W >> 16),
                            (unsigned char)(W >> 8), (unsigned char)W,
                            (unsigned char)(H >> 24), (unsigned char)(H >> 16),
                            (unsigned char)(H >> 8), (unsigned char)H, 8, 2, 0, 0, 0};
    unsigned crc = 0xFFFFFFFFu;
    for (int i = 4; i < 21; ++i) crc = crc_bytes(crc, ih[i]);
    crc ^= 0xFFFFFFFFu;
    for (int i = 0; i < 21; ++i) o[8 + i] = ih[i];
    for (int i = 0; i < 4; ++i) o[29 + i] = (unsigned char)(crc >> (24 - 8 * i));
  }
  const long long z0 = c * kIdat, len = min((long long)kIdat, zlen - z0);
  unsigned char *dst = o + 33 + c * (kIdat + 12);
  const int seg = kIdat / 32;
  const long long lo = min((long long)lane * seg, len), hi = min((long long)(lane + 1) * seg, len);
  unsigned crc = 0xFFFFFFFFu;
  if (lane == 0) {
    const unsigned char tag[4] = {'I', 'D', 'A', 'T'};
    for (int i = 0; i < 4; ++i) {
      crc = crc_bytes(crc, tag[i]);
      dst[4 + i] = tag[i];
      dst[i] = (unsigned char)(len >> (24 - 8 * i));
    }
  }
  for (long long j = lo; j < hi; ++j) {
    const long long zi = z0 + j;
    unsigned char v;
    if (zi < 2) v = (unsigned char)(zi == 0 ? D[D_CMF] : D[D_FLG]);
    else if (zi < 2 + dlen) v = zb[zi - 2];
    else v = (unsigned char)(adler >> (24 - 8 * (zi - 2 - dlen)));
    dst[8 + j] = v;
    crc = crc_bytes(crc, v);
  }
  crc ^= 0xFFFFFFFFu;
  unsigned total = crc;
  for (int l = 1; l < 32; ++l) {
    const unsigned cl = __shfl_sync(0xFFFFFFFFu, crc, l);
    const long long ll = min((long long)(l + 1) * seg, len) - min((long long)l * seg, len);
    if (lane == 0 && ll > 0) total = crc_combine(x2n, total, cl, ll);
  }
  if (lane == 0) {
    for (int i = 0; i < 4; ++i) dst[8 + len + i] = (unsigned char)(total >> (24 - 8 * i));
    if (c == chunks - 1) {
      const unsigned char iend[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xAE, 0x42, 0x60, 0x82};
      unsigned char *e = o + 33 + zlen + 12 * chunks;
      for (int i = 0; i < 12; ++i) e[i] = iend[i];
    }
  }
}

}  // namespace
}  // namespace mrx

using namespace mrx;

extern "C" int mrx_png_encode(const long long *d_desc, int B, long long max_n, int max_blocks,
                              long long max_chunks, long long total_tiles, long long zbuf_words,
                              unsigned char *d_stream, short *d_sym, int *d_stretch,
                              long long *d_tiles, int *d_blk_pos, int *d_blk_tab,
                              long long *d_blk_info, unsigned int *d_zbuf,
                              long long *d_img_info, unsigned char *d_out, long long *d_sizes,
                              void *stream) {
  MRX_CHECK_ARG(d_desc && d_stream && d_sym && d_stretch && d_tiles && d_blk_pos && d_blk_tab &&
                    d_blk_info && d_zbuf && d_img_info && d_out && d_sizes,
                "mrx_png_encode: null pointer");
  MRX_CHECK_ARG(B >= 0 && B <= MRX_MAX_BATCH, "mrx_png_encode: B=%d outside [0, %d]", B,
                MRX_MAX_BATCH);
  MRX_CHECK_ARG(max_n >= 4 && max_n <= MRX_PNG_MAX_STREAM,
                "mrx_png_encode: max_n=%lld outside [4, %lld]", max_n,
                (long long)MRX_PNG_MAX_STREAM);
  MRX_CHECK_ARG(max_blocks >= 1 && max_chunks >= 1 && total_tiles >= B && zbuf_words >= 1 &&
                    total_tiles <= (1LL << 30),
                "mrx_png_encode: max_blocks=%d, max_chunks=%lld, total_tiles=%lld, "
                "zbuf_words=%lld",
                max_blocks, max_chunks, total_tiles, zbuf_words);
  if (B == 0) return MRX_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  long long *tiles_a = d_tiles, *tiles_b = d_tiles + total_tiles + 1;
  const int max_tiles = int((max_n + kTile - 1) / kTile);
  const dim3 gt(max_tiles, B);
  MRX_CUDA(cudaMemsetAsync(d_zbuf, 0, sizeof(unsigned) * size_t(zbuf_words), st));
  const dim3 gf(unsigned(min((max_n + kThreads - 1) / kThreads, 4096LL)), B);
  png_filter_kernel<<<gf, kThreads, 0, st>>>(d_desc, d_stream, d_blk_pos, d_img_info);
  MRX_LAUNCH_CHECK("png_filter_kernel");
  png_starts_kernel<<<gt, kThreads, 0, st>>>(d_desc, d_stream, tiles_a, d_img_info);
  MRX_LAUNCH_CHECK("png_starts_kernel");
  if (int rc = launch_offsets_scan(tiles_a, int(total_tiles), st)) return rc;
  png_stretch_kernel<<<gt, kThreads, 0, st>>>(d_desc, d_stream, tiles_a, d_stretch);
  MRX_LAUNCH_CHECK("png_stretch_kernel");
  png_symbols_kernel<<<gt, kThreads, 0, st>>>(d_desc, d_stream, tiles_a, d_stretch, d_sym,
                                              tiles_b);
  MRX_LAUNCH_CHECK("png_symbols_kernel");
  if (int rc = launch_offsets_scan(tiles_b, int(total_tiles), st)) return rc;
  png_symidx_kernel<<<gt, kThreads, 0, st>>>(d_desc, d_stream, d_sym, tiles_b, d_blk_pos,
                                             d_img_info);
  MRX_LAUNCH_CHECK("png_symidx_kernel");
  const dim3 gb(max_blocks, B);
  png_hist_kernel<<<gb, kThreads, 0, st>>>(d_desc, d_sym, d_blk_pos, d_img_info, d_blk_tab);
  MRX_LAUNCH_CHECK("png_hist_kernel");
  const dim3 gtr((max_blocks + kTreeThreads - 1) / kTreeThreads, B);
  png_trees_kernel<<<gtr, kTreeThreads, 0, st>>>(d_desc, d_sym, d_blk_pos, d_img_info,
                                                 d_blk_tab, d_blk_info);
  MRX_LAUNCH_CHECK("png_trees_kernel");
  png_layout_kernel<<<(B + 31) / 32, 32, 0, st>>>(d_desc, B, d_blk_pos, d_blk_info, d_img_info,
                                                  d_sizes);
  MRX_LAUNCH_CHECK("png_layout_kernel");
  png_emit_kernel<false><<<gt, kThreads, 0, st>>>(d_desc, d_stream, d_sym, d_blk_pos, d_blk_tab,
                                                  d_blk_info, d_img_info, tiles_a, d_zbuf);
  MRX_LAUNCH_CHECK("png_emit_kernel<false>");
  if (int rc = launch_offsets_scan(tiles_a, int(total_tiles), st)) return rc;
  png_emit_kernel<true><<<gt, kThreads, 0, st>>>(d_desc, d_stream, d_sym, d_blk_pos, d_blk_tab,
                                                 d_blk_info, d_img_info, tiles_a, d_zbuf);
  MRX_LAUNCH_CHECK("png_emit_kernel<true>");
  png_frame_kernel<<<gb, 32, 0, st>>>(d_desc, d_blk_pos, d_blk_tab, d_blk_info, d_img_info,
                                      d_zbuf);
  MRX_LAUNCH_CHECK("png_frame_kernel");
  const dim3 gc(unsigned((max_chunks + kFileWarps - 1) / kFileWarps), B);
  png_file_kernel<<<gc, 32 * kFileWarps, 0, st>>>(d_desc, d_zbuf, d_img_info, d_out);
  MRX_LAUNCH_CHECK("png_file_kernel");
  return MRX_OK;
}
