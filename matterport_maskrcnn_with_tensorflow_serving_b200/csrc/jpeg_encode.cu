// jpeg_encode.cu -- baseline JPEG files byte for byte as cv2.imencode('.jpg', rgb[..., ::-1],
// [IMWRITE_JPEG_QUALITY, q, IMWRITE_JPEG_OPTIMIZE, opt]) writes them (libjpeg-turbo: JFIF 1.01,
// jpeg_set_quality(q, force_baseline), YCbCr 4:2:0 with h2v2 downsampling, ISLOW FDCT, one
// interleaved scan, the Annex K tables or jpeg_gen_optimal_table's, no restart markers).
//
// One stream-ordered batch (mrx.h, "JPEG encode"; tests/jpeg_encode_oracle.py restates every step):
//   coef     one thread per block of the scan (MCU order, dummy blocks included): edge replication,
//            colour conversion, h2v2 downsampling, FDCT, quantisation -> int16 zigzag coefficients
//   bits<1>  (optimize) per-image symbol histograms of the four tables
//   tables   one thread per image and table: the bits/vals (standard, or K.2 optimal) and codes
//   bits<0>  each block's coded bits, scanned over the CTA's tile of blocks -> scan over tiles
//   layout   one thread per image: coded bits, bytes, header bytes; the 1-bit padding
//   emit     every block's codes at its bit (big-endian words, word atomics)
//   stuff<0> per tile of bytes: the 0xFF bytes                          -> scan over tiles
//   stuff<1> the bytes at their file position, a 0x00 after each 0xFF
//   file     one thread per image: SOI, APP0, DQT, SOF0, DHT, SOS before the data, EOI after
#include "common.cuh"

namespace mrx {
namespace {

constexpr int kThreads = 256;       // blocks per tile of the block passes
constexpr int kItems = 8;
constexpr int kByteTile = kThreads * kItems;   // jpeg_encode.BYTE_TILE
constexpr int kTabBytes = 16 + 256;            // bits[16], vals[256] of one Huffman table

// desc words per image (jpeg_encode.py D_*)
enum {
  D_SRC = 0, D_H, D_W, D_MCUX, D_MCUY, D_NBLK, D_BLK_OFF, D_BT_OFF, D_NBT, D_WORD_OFF, D_YT_OFF,
  D_NYT, D_OUT_OFF, DESC_WORDS = 16
};
// per image int64 (MRX_JPEG_ENC_*)
enum { IM_BITS = 0, IM_BYTES, IM_FF, IM_HDR, IM_FILE, IM_BLOCKS, INFO_WORDS = 8 };

// zig-zag index -> natural (row-major) index; a constant expression once loops are unrolled
__device__ __forceinline__ constexpr int zigzag(int z) {
  constexpr unsigned char t[64] = {
      0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
      41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
      30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
  return t[z];
}

// T.81 Annex K.1, natural order
__constant__ unsigned char c_std_quant[2][64] = {
    {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,
     14, 13, 16, 24, 40,  57,  69,  56,  14, 17, 22, 29, 51,  87,  80,  62,
     18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
     49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99},
    {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99,
     99, 99, 47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99}};

// T.81 Annex K.3: bits[16] then vals, tables DC0, AC0, DC1, AC1
__constant__ unsigned char c_std_dc_bits[2][16] = {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0},
                                                   {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}};
__constant__ unsigned char c_std_ac_bits[2][16] = {
    {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d},
    {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77}};
__constant__ unsigned char c_std_ac_vals[2][162] = {
    {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61,
     0x07, 0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52,
     0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25,
     0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45,
     0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64,
     0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83,
     0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
     0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6,
     0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3,
     0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8,
     0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
    {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61,
     0x71, 0x13, 0x22, 0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33,
     0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18,
     0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44,
     0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63,
     0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a,
     0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97,
     0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4,
     0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
     0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7,
     0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa}};

// jpeg_quality_scaling + jpeg_add_quant_table(force_baseline): table t's entry at natural index i
__device__ __forceinline__ int quant_value(int quality, int t, int i) {
  const int q = quality <= 0 ? 1 : quality;
  const int scale = q < 50 ? 5000 / q : 200 - 2 * q;
  return min(max((int(c_std_quant[t][i]) * scale + 50) / 100, 1), 255);
}

// jccolor.c rgb_ycc_convert, 16-bit fixed point
__device__ __forceinline__ void rgb_ycc(const unsigned char *p, int &y, int &cb, int &cr) {
  const int r = p[0], g = p[1], b = p[2];
  constexpr int kHalf = 1 << 15, kOff = (128 << 16) + kHalf - 1;
  y = (19595 * r + 38470 * g + 7471 * b + kHalf) >> 16;
  cb = (-11059 * r - 21709 * g + 32768 * b + kOff) >> 16;
  cr = (32768 * r - 27439 * g - 5329 * b + kOff) >> 16;
}

__device__ __forceinline__ int luma_at(const unsigned char *src, int H, int W, int y, int x) {
  int Y, cb, cr;
  rgb_ycc(src + (size_t(min(y, H - 1)) * W + min(x, W - 1)) * 3, Y, cb, cr);
  return Y;
}

// h2v2_downsample of component c (1 Cb, 2 Cr) at chroma sample (cy, cx): the full-resolution
// plane replicated right and to an even row count, the chroma plane's last row replicated down
__device__ __forceinline__ int chroma_at(const unsigned char *src, int H, int W, int c, int cy,
                                         int cx) {
  cy = min(cy, (H + 1) / 2 - 1);
  int sum = 1 + (cx & 1);
#pragma unroll
  for (int dy = 0; dy < 2; ++dy)
#pragma unroll
    for (int dx = 0; dx < 2; ++dx) {
      const int y = min(2 * cy + dy, H - 1), x = min(2 * cx + dx, W - 1);
      int Y, cb, cr;
      rgb_ycc(src + (size_t(y) * W + x) * 3, Y, cb, cr);
      sum += c == 1 ? cb : cr;
    }
  return sum >> 2;
}

// jfdctint.c (ISLOW): CONST_BITS 13, PASS1_BITS 2, in place on samples - 128.  int32 holds every
// intermediate for 8-bit samples: pass 1 outputs stay below 2^13 in magnitude and each pass-2
// product sum below 2^31 (libjpeg-turbo's SIMD FDCT also computes in 32 bits).
__device__ __forceinline__ void fdct_islow(int *d) {
  constexpr int F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373,
                F1175 = 9633, F1501 = 12299, F1847 = 15137, F1961 = 16069, F2053 = 16819,
                F2562 = 20995, F3072 = 25172;
#pragma unroll
  for (int pass = 0; pass < 2; ++pass) {
    const int stride = pass == 0 ? 1 : 8, step = pass == 0 ? 8 : 1;
    const int sh = pass == 0 ? 13 - 2 : 13 + 2;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      int *p = d + r * step;
      const int t0 = p[0] + p[7 * stride], t7 = p[0] - p[7 * stride];
      const int t1 = p[stride] + p[6 * stride], t6 = p[stride] - p[6 * stride];
      const int t2 = p[2 * stride] + p[5 * stride], t5 = p[2 * stride] - p[5 * stride];
      const int t3 = p[3 * stride] + p[4 * stride], t4 = p[3 * stride] - p[4 * stride];
      const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
      if (pass == 0) {
        p[0] = (t10 + t11) << 2;
        p[4 * stride] = (t10 - t11) << 2;
      } else {
        p[0] = (t10 + t11 + 2) >> 2;
        p[4 * stride] = (t10 - t11 + 2) >> 2;
      }
      const int rnd = 1 << (sh - 1);
      int z1 = (t12 + t13) * F0541;
      p[2 * stride] = (z1 + t13 * F0765 + rnd) >> sh;
      p[6 * stride] = (z1 - t12 * F1847 + rnd) >> sh;
      z1 = t4 + t7;
      int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
      const int z5 = (z3 + z4) * F1175;
      const int a4 = t4 * F0298, a5 = t5 * F2053, a6 = t6 * F3072, a7 = t7 * F1501;
      z1 *= -F0899;
      z2 *= -F2562;
      z3 = z3 * -F1961 + z5;
      z4 = z4 * -F0390 + z5;
      p[7 * stride] = (a4 + z1 + z3 + rnd) >> sh;
      p[5 * stride] = (a5 + z2 + z4 + rnd) >> sh;
      p[3 * stride] = (a6 + z2 + z3 + rnd) >> sh;
      p[1 * stride] = (a7 + z1 + z4 + rnd) >> sh;
    }
  }
}

// quantisation: x / (8q) rounded half away from zero (libjpeg-turbo's reciprocal multiply gives
// the same quotient)
__device__ __forceinline__ int quantize(int x, int q) {
  const int d = q << 3;
  return x < 0 ? -((d / 2 - x) / d) : (x + d / 2) / d;
}

// block k of an image's scan -> (component 0/1/2, block row, block column in its component)
__device__ __forceinline__ int block_pos(const long long *D, int k, int &by, int &bx) {
  const int mcux = int(D[D_MCUX]), m = k / 6, j = k - 6 * m;
  const int my = m / mcux, mx = m - my * mcux;
  if (j < 4) {
    by = 2 * my + (j >> 1);
    bx = 2 * mx + (j & 1);
    return 0;
  }
  by = my;
  bx = mx;
  return j - 3;
}

// the quantised DC of luma block (by, bx), a block of the image (not a dummy): the FDCT's DC is
// the sum of the samples - 128
__device__ __forceinline__ int luma_dc(const unsigned char *src, int H, int W, int by, int bx,
                                       int q0) {
  int s = 0;
  for (int y = 0; y < 8; ++y)
    for (int x = 0; x < 8; ++x) s += luma_at(src, H, W, 8 * by + y, 8 * bx + x) - 128;
  return quantize(s, q0);
}

// ------------------------------------------------------------------ coefficients
__global__ void __launch_bounds__(kThreads) jpeg_coef_kernel(const long long *__restrict__ desc,
                                                             int quality,
                                                             short *__restrict__ coef) {
  __shared__ int s_q[2][64];
  for (int i = threadIdx.x; i < 128; i += kThreads) s_q[i >> 6][i & 63] = quant_value(quality, i >> 6, i & 63);
  __syncthreads();
  const long long *D = desc + size_t(blockIdx.y) * DESC_WORDS;
  const int k = blockIdx.x * kThreads + threadIdx.x;
  if (k >= int(D[D_NBLK])) return;
  const int H = int(D[D_H]), W = int(D[D_W]);
  const unsigned char *src = reinterpret_cast<const unsigned char *>(D[D_SRC]);
  int by, bx;
  const int c = block_pos(D, k, by, bx);
  const int hib = (H + 7) / 8, wib = (W + 7) / 8;
  int d[64];
  short *out = coef + (D[D_BLK_OFF] + k) * 64;
  if (c == 0 && (by >= hib || bx >= wib)) {
    // dummy block (jccoefct.c): zeros, the DC of the block before it in its row, or in a dummy
    // row the DC of the MCU's last block in the row above
    int sy = by, sx = bx - 1;
    if (by >= hib) {
      sy = by - 1;
      sx = bx | 1;
      if (sx >= wib) sx = bx & ~1;
    }
    out[0] = short(luma_dc(src, H, W, sy, sx, s_q[0][0]));
    for (int i = 1; i < 64; ++i) out[i] = 0;
    return;
  }
#pragma unroll
  for (int y = 0; y < 8; ++y)
#pragma unroll
    for (int x = 0; x < 8; ++x)
      d[8 * y + x] = (c == 0 ? luma_at(src, H, W, 8 * by + y, 8 * bx + x)
                             : chroma_at(src, H, W, c, 8 * by + y, 8 * bx + x)) - 128;
  fdct_islow(d);
  const int t = c > 0;
#pragma unroll
  for (int z = 0; z < 64; ++z) {
    const int i = zigzag(z);
    out[z] = short(quantize(d[i], s_q[t][i]));
  }
}

__device__ __forceinline__ int nbits_of(int v) {
  v = v < 0 ? -v : v;
  return v ? 32 - __clz(v) : 0;
}

// the quantised DC of the block before block k in its component, in MCU order (0 for the first)
__device__ __forceinline__ int dc_pred(const short *c0, int k) {
  const int j = k % 6;
  const int p = j == 0 ? k - 3 : j < 4 ? k - 1 : k - 6;
  return p >= 0 ? c0[size_t(p) * 64] : 0;
}

// walks block k's symbols: f(table 0..3, symbol, value bits, value length)
template <typename F>
__device__ __forceinline__ void block_symbols(const short *c0, int k, F f) {
  const short *blk = c0 + size_t(k) * 64;
  const int t = k % 6 >= 4 ? 2 : 0;   // DC table slot; AC is t + 1
  const int diff = blk[0] - dc_pred(c0, k);
  const int n = nbits_of(diff);
  f(t, n, unsigned(diff < 0 ? diff - 1 : diff) & ((1u << n) - 1), n);
  int run = 0;
  for (int z = 1; z < 64; ++z) {
    const int v = blk[z];
    if (v == 0) {
      ++run;
      continue;
    }
    for (; run > 15; run -= 16) f(t + 1, 0xF0, 0u, 0);
    const int m = nbits_of(v);
    f(t + 1, (run << 4) + m, unsigned(v < 0 ? v - 1 : v) & ((1u << m) - 1), m);
    run = 0;
  }
  if (run) f(t + 1, 0, 0u, 0);
}

// ------------------------------------------------------------------ histograms / coded bits
template <bool kHist>
__global__ void __launch_bounds__(kThreads) jpeg_bits_kernel(const long long *__restrict__ desc,
                                                             const short *__restrict__ coef,
                                                             const int *__restrict__ codes,
                                                             int *__restrict__ hist,
                                                             int *__restrict__ blk_bit,
                                                             long long *__restrict__ tiles) {
  __shared__ int s_hist[kHist ? 4 * 256 : 1];
  __shared__ long long s_warp[kThreads / 32];
  const int b = blockIdx.y;
  const long long *D = desc + size_t(b) * DESC_WORDS;
  if (blockIdx.x >= D[D_NBT]) return;
  if (kHist) {
    for (int i = threadIdx.x; i < 4 * 256; i += kThreads) s_hist[i] = 0;
    __syncthreads();
  }
  const int k = blockIdx.x * kThreads + threadIdx.x;
  const short *c0 = coef + D[D_BLK_OFF] * 64;
  const int *cd = codes + size_t(b) * 4 * 256;
  long long nb = 0;
  if (k < int(D[D_NBLK])) {
    block_symbols(c0, k, [&](int t, int sym, unsigned, int len) {
      if (kHist) atomicAdd(&s_hist[t * 256 + sym], 1);
      else nb += (unsigned(cd[t * 256 + sym]) >> 16) + len;
    });
  }
  if (kHist) {
    __syncthreads();
    int *h = hist + size_t(b) * 4 * 256;
    for (int i = threadIdx.x; i < 4 * 256; i += kThreads)
      if (s_hist[i]) atomicAdd(&h[i], s_hist[i]);
    return;
  }
  long long tot;
  const long long ex = block_exclusive_scan<long long, kThreads>(nb, s_warp, tot);
  if (k < int(D[D_NBLK])) blk_bit[D[D_BLK_OFF] + k] = int(ex);
  if (threadIdx.x == 0) tiles[D[D_BT_OFF] + blockIdx.x] = tot;
}

// ------------------------------------------------------------------ tables
// jchuff.c jpeg_gen_optimal_table (T.81 K.2) of freq[256] (symbol 256 reserves the all-ones code)
__device__ void gen_optimal_table(const int *freq_in, unsigned char *bits_out,
                                  unsigned char *vals) {
  long long freq[257];
  int codesize[257], others[257];
  short live[257];
  int nlive = 0;
  for (int i = 0; i < 257; ++i) {
    freq[i] = i < 256 ? freq_in[i] : 1;
    codesize[i] = 0;
    others[i] = -1;
    if (freq[i]) live[nlive++] = short(i);
  }
  while (true) {
    int c1 = -1, c2 = -1;
    long long v = 1000000000LL;
    for (int j = 0; j < nlive; ++j) {
      const int i = live[j];
      if (freq[i] && freq[i] <= v) v = freq[i], c1 = i;
    }
    v = 1000000000LL;
    for (int j = 0; j < nlive; ++j) {
      const int i = live[j];
      if (freq[i] && freq[i] <= v && i != c1) v = freq[i], c2 = i;
    }
    if (c2 < 0) break;
    freq[c1] += freq[c2];
    freq[c2] = 0;
    codesize[c1]++;
    while (others[c1] >= 0) {
      c1 = others[c1];
      codesize[c1]++;
    }
    others[c1] = c2;
    codesize[c2]++;
    while (others[c2] >= 0) {
      c2 = others[c2];
      codesize[c2]++;
    }
  }
  int bits[33];
  for (int i = 0; i < 33; ++i) bits[i] = 0;
  for (int i = 0; i < 257; ++i)
    if (codesize[i]) bits[codesize[i]]++;
  for (int i = 32; i > 16; --i) {
    while (bits[i] > 0) {
      int j = i - 2;
      while (bits[j] == 0) --j;
      bits[i] -= 2;
      bits[i - 1]++;
      bits[j + 1] += 2;
      bits[j]--;
    }
  }
  int i = 16;
  while (bits[i] == 0) --i;
  bits[i]--;
  for (int l = 1; l <= 16; ++l) bits_out[l - 1] = (unsigned char)bits[l];
  int p = 0;
  for (int size = 1; size <= 32; ++size)
    for (int s = 0; s < 256; ++s)
      if (codesize[s] == size) vals[p++] = (unsigned char)s;
}

// one thread per image and table (DC0, AC0, DC1, AC1): bits/vals into huff, code | length << 16
// per symbol into codes (jpeg_make_c_derived_tbl)
__global__ void jpeg_tables_kernel(int B, int optimize, const int *__restrict__ hist,
                                   unsigned char *__restrict__ huff, int *__restrict__ codes) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= 4 * B) return;
  const int t = g & 3, ac = t & 1, chroma = t >> 1;
  unsigned char *bits = huff + size_t(g) * kTabBytes, *vals = bits + 16;
  if (optimize) {
    gen_optimal_table(hist + size_t(g) * 256, bits, vals);
  } else {
    int n = 0;
    for (int l = 0; l < 16; ++l) {
      bits[l] = ac ? c_std_ac_bits[chroma][l] : c_std_dc_bits[chroma][l];
      n += bits[l];
    }
    for (int i = 0; i < n; ++i) vals[i] = ac ? c_std_ac_vals[chroma][i] : (unsigned char)i;
  }
  int *cd = codes + size_t(g) * 256;
  for (int s = 0; s < 256; ++s) cd[s] = 0;
  unsigned code = 0;
  int p = 0;
  for (int l = 1; l <= 16; ++l) {
    for (int i = 0; i < bits[l - 1]; ++i) cd[vals[p++]] = int(code++ | (unsigned(l) << 16));
    code <<= 1;
  }
}

__device__ __forceinline__ int table_values(const unsigned char *huff_b, int t) {
  int n = 0;
  for (int l = 0; l < 16; ++l) n += huff_b[t * kTabBytes + l];
  return n;
}

// big-endian bit order: stream bit p is bit 31 - (p & 31) of word p >> 5
__device__ __forceinline__ void put_bits_be(unsigned *w, long long bit, unsigned v, int n) {
  if (n <= 0) return;
  const int sh = int(bit & 31);
  unsigned *p = w + (bit >> 5);
  if (sh + n <= 32) {
    atomicOr(p, v << (32 - sh - n));
  } else {
    const int n2 = sh + n - 32;
    atomicOr(p, v >> n2);
    atomicOr(p + 1, v << (32 - n2));
  }
}

// ------------------------------------------------------------------ layout (one thread per image)
__global__ void jpeg_layout_kernel(const long long *__restrict__ desc, int B,
                                   const long long *__restrict__ tiles,
                                   const unsigned char *__restrict__ huff,
                                   unsigned *__restrict__ words, long long *__restrict__ info) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const long long *D = desc + size_t(b) * DESC_WORDS;
  const long long bits = tiles[D[D_BT_OFF] + D[D_NBT]] - tiles[D[D_BT_OFF]];
  const int pad = int((8 - (bits & 7)) & 7);
  put_bits_be(words + D[D_WORD_OFF], bits, (1u << pad) - 1, pad);
  long long hdr = 2 + 18 + 2 * 69 + 19 + 14;
  for (int t = 0; t < 4; ++t) hdr += 21 + table_values(huff + size_t(b) * 4 * kTabBytes, t);
  long long *im = info + size_t(b) * INFO_WORDS;
  im[IM_BITS] = bits;
  im[IM_BYTES] = (bits + 7) >> 3;
  im[IM_HDR] = hdr;
  im[IM_BLOCKS] = D[D_NBLK];
}

// ------------------------------------------------------------------ emit
__global__ void __launch_bounds__(kThreads) jpeg_emit_kernel(const long long *__restrict__ desc,
                                                             const short *__restrict__ coef,
                                                             const int *__restrict__ codes,
                                                             const int *__restrict__ blk_bit,
                                                             const long long *__restrict__ tiles,
                                                             unsigned *__restrict__ words) {
  const int b = blockIdx.y;
  const long long *D = desc + size_t(b) * DESC_WORDS;
  const int k = blockIdx.x * kThreads + threadIdx.x;
  if (blockIdx.x >= D[D_NBT] || k >= int(D[D_NBLK])) return;
  const short *c0 = coef + D[D_BLK_OFF] * 64;
  const int *cd = codes + size_t(b) * 4 * 256;
  const long long *tb = tiles + D[D_BT_OFF];
  long long bit = tb[blockIdx.x] - tb[0] + blk_bit[D[D_BLK_OFF] + k];
  unsigned *w = words + D[D_WORD_OFF];
  // the block's bits gathered a word at a time: acc holds fill bits at the top of the word
  // that holds `bit`
  unsigned acc = 0;
  int fill = int(bit & 31);
  long long wi = bit >> 5;
  auto push = [&](unsigned v, int n) {
    while (n > 0) {
      const int take = min(n, 32 - fill);
      const unsigned part = (v >> (n - take)) & (take == 32 ? 0xFFFFFFFFu : ((1u << take) - 1));
      acc |= part << (32 - fill - take);
      fill += take;
      n -= take;
      if (fill == 32) {
        if (acc) atomicOr(w + wi, acc);
        acc = 0;
        fill = 0;
        ++wi;
      }
    }
  };
  block_symbols(c0, k, [&](int t, int sym, unsigned v, int len) {
    const unsigned e = unsigned(cd[t * 256 + sym]);
    push(e & 0xFFFF, int(e >> 16));
    push(v, len);
  });
  if (acc) atomicOr(w + wi, acc);
}

// ------------------------------------------------------------------ byte stuffing
__device__ __forceinline__ unsigned data_byte(const unsigned *w, long long i) {
  return (w[i >> 2] >> (24 - 8 * int(i & 3))) & 0xFF;
}

template <bool kCopy>
__global__ void __launch_bounds__(kThreads) jpeg_stuff_kernel(const long long *__restrict__ desc,
                                                              const unsigned *__restrict__ words,
                                                              const long long *__restrict__ info,
                                                              long long *__restrict__ tiles,
                                                              unsigned char *__restrict__ out) {
  __shared__ long long s_warp[kThreads / 32];
  const int b = blockIdx.y;
  const long long *D = desc + size_t(b) * DESC_WORDS;
  if (blockIdx.x >= D[D_NYT]) return;
  const long long *im = info + size_t(b) * INFO_WORDS;
  const long long n = im[IM_BYTES];
  const unsigned *w = words + D[D_WORD_OFF];
  const long long i0 = (long long)blockIdx.x * kByteTile + threadIdx.x * kItems;
  unsigned v[kItems];
  long long cnt = 0;
#pragma unroll
  for (int j = 0; j < kItems; ++j) {
    v[j] = i0 + j < n ? data_byte(w, i0 + j) : 0u;
    cnt += v[j] == 0xFF;
  }
  long long tot;
  const long long ex = block_exclusive_scan<long long, kThreads>(cnt, s_warp, tot);
  long long *tb = tiles + D[D_YT_OFF];
  if (!kCopy) {
    if (threadIdx.x == 0) tb[blockIdx.x] = tot;
    return;
  }
  if (i0 >= n) return;
  unsigned char *o = out + D[D_OUT_OFF] + im[IM_HDR];
  long long p = i0 + tb[blockIdx.x] - tb[0] + ex;
#pragma unroll
  for (int j = 0; j < kItems; ++j) {
    if (i0 + j >= n) break;
    o[p++] = (unsigned char)v[j];
    if (v[j] == 0xFF) o[p++] = 0;
  }
}

// ------------------------------------------------------------------ file (one thread per image)
__global__ void jpeg_file_kernel(const long long *__restrict__ desc, int B, int quality,
                                 const unsigned char *__restrict__ huff,
                                 const long long *__restrict__ tiles,
                                 long long *__restrict__ info, unsigned char *__restrict__ out,
                                 long long *__restrict__ sizes) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const long long *D = desc + size_t(b) * DESC_WORDS;
  long long *im = info + size_t(b) * INFO_WORDS;
  const long long *tb = tiles + D[D_YT_OFF];
  const long long ff = tb[D[D_NYT]] - tb[0];
  unsigned char *o = out + D[D_OUT_OFF];
  int p = 0;
  auto put = [&](unsigned v) { o[p++] = (unsigned char)v; };
  auto put16 = [&](unsigned v) { put(v >> 8); put(v & 0xFF); };
  put16(0xFFD8);
  const unsigned char app0[18] = {0xFF, 0xE0, 0, 16, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1,
                                  0, 0};
  for (int i = 0; i < 18; ++i) put(app0[i]);
  for (int t = 0; t < 2; ++t) {
    put16(0xFFDB);
    put16(67);
    put(t);
    for (int z = 0; z < 64; ++z) put(quant_value(quality, t, zigzag(z)));
  }
  const unsigned H = unsigned(D[D_H]), W = unsigned(D[D_W]);
  const unsigned char sof[19] = {0xFF, 0xC0, 0, 17, 8, (unsigned char)(H >> 8), (unsigned char)H,
                                 (unsigned char)(W >> 8), (unsigned char)W, 3, 1, 0x22, 0, 2,
                                 0x11, 1, 3, 0x11, 1};
  for (int i = 0; i < 19; ++i) put(sof[i]);
  const unsigned char *hb = huff + size_t(b) * 4 * kTabBytes;
  for (int t = 0; t < 4; ++t) {
    const int n = table_values(hb, t);
    put16(0xFFC4);
    put16(2 + 1 + 16 + n);
    put(((t & 1) << 4) | (t >> 1));
    for (int i = 0; i < 16 + n; ++i) put(hb[t * kTabBytes + i]);
  }
  const unsigned char sos[14] = {0xFF, 0xDA, 0, 12, 3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0};
  for (int i = 0; i < 14; ++i) put(sos[i]);
  const long long end = p + im[IM_BYTES] + ff;
  o[end] = 0xFF;
  o[end + 1] = 0xD9;
  im[IM_FF] = ff;
  im[IM_FILE] = end + 2;
  sizes[b] = end + 2;
}

}  // namespace
}  // namespace mrx

using namespace mrx;

extern "C" int mrx_jpeg_encode(const long long *d_desc, int B, int quality, int optimize,
                               int min_side, int max_side, int max_blocks, long long max_bytes,
                               long long blk_tiles, long long byte_tiles, long long word_count,
                               unsigned char *d_huff, int *d_codes, int *d_hist, short *d_coef,
                               int *d_blk_bit, long long *d_tiles, unsigned int *d_words,
                               long long *d_info, unsigned char *d_out, long long *d_sizes,
                               void *stream) {
  MRX_CHECK_ARG(d_desc && d_huff && d_codes && d_hist && d_coef && d_blk_bit && d_tiles &&
                    d_words && d_info && d_out && d_sizes,
                "mrx_jpeg_encode: null pointer");
  MRX_CHECK_ARG(B >= 0 && B <= MRX_MAX_BATCH, "mrx_jpeg_encode: B=%d outside [0, %d]", B,
                MRX_MAX_BATCH);
  MRX_CHECK_ARG(quality >= 0 && quality <= 100, "mrx_jpeg_encode: quality=%d outside [0, 100]",
                quality);
  MRX_CHECK_ARG(optimize == 0 || optimize == 1, "mrx_jpeg_encode: optimize=%d", optimize);
  if (B == 0) return MRX_OK;
  MRX_CHECK_SUPPORTED(min_side >= 1 && max_side <= MRX_JPEG_ENC_MAX_SIDE,
                      "mrx_jpeg_encode: image sides in [%d, %d], outside [1, %d]", min_side,
                      max_side, MRX_JPEG_ENC_MAX_SIDE);
  MRX_CHECK_ARG(max_blocks >= 6 && max_bytes >= 1 && blk_tiles >= B && byte_tiles >= B &&
                    word_count >= 1 && blk_tiles <= (1LL << 30) && byte_tiles <= (1LL << 30),
                "mrx_jpeg_encode: max_blocks=%d, max_bytes=%lld, blk_tiles=%lld, "
                "byte_tiles=%lld, word_count=%lld",
                max_blocks, max_bytes, blk_tiles, byte_tiles, word_count);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  long long *tiles_blk = d_tiles, *tiles_byte = d_tiles + blk_tiles + 1;
  const dim3 gk((max_blocks + kThreads - 1) / kThreads, B);
  MRX_CUDA(cudaMemsetAsync(d_words, 0, sizeof(unsigned) * size_t(word_count), st));
  jpeg_coef_kernel<<<gk, kThreads, 0, st>>>(d_desc, quality, d_coef);
  MRX_LAUNCH_CHECK("jpeg_coef_kernel");
  if (optimize) {
    MRX_CUDA(cudaMemsetAsync(d_hist, 0, sizeof(int) * 4 * 256 * size_t(B), st));
    jpeg_bits_kernel<true><<<gk, kThreads, 0, st>>>(d_desc, d_coef, d_codes, d_hist, d_blk_bit,
                                                    tiles_blk);
    MRX_LAUNCH_CHECK("jpeg_bits_kernel<true>");
  }
  jpeg_tables_kernel<<<(4 * B + 127) / 128, 128, 0, st>>>(B, optimize, d_hist, d_huff, d_codes);
  MRX_LAUNCH_CHECK("jpeg_tables_kernel");
  jpeg_bits_kernel<false><<<gk, kThreads, 0, st>>>(d_desc, d_coef, d_codes, d_hist, d_blk_bit,
                                                   tiles_blk);
  MRX_LAUNCH_CHECK("jpeg_bits_kernel<false>");
  if (int rc = launch_offsets_scan(tiles_blk, int(blk_tiles), st)) return rc;
  jpeg_layout_kernel<<<(B + 31) / 32, 32, 0, st>>>(d_desc, B, tiles_blk, d_huff, d_words, d_info);
  MRX_LAUNCH_CHECK("jpeg_layout_kernel");
  jpeg_emit_kernel<<<gk, kThreads, 0, st>>>(d_desc, d_coef, d_codes, d_blk_bit, tiles_blk,
                                            d_words);
  MRX_LAUNCH_CHECK("jpeg_emit_kernel");
  const dim3 gy(unsigned((max_bytes + kByteTile - 1) / kByteTile), B);
  jpeg_stuff_kernel<false><<<gy, kThreads, 0, st>>>(d_desc, d_words, d_info, tiles_byte, d_out);
  MRX_LAUNCH_CHECK("jpeg_stuff_kernel<false>");
  if (int rc = launch_offsets_scan(tiles_byte, int(byte_tiles), st)) return rc;
  jpeg_stuff_kernel<true><<<gy, kThreads, 0, st>>>(d_desc, d_words, d_info, tiles_byte, d_out);
  MRX_LAUNCH_CHECK("jpeg_stuff_kernel<true>");
  jpeg_file_kernel<<<(B + 31) / 32, 32, 0, st>>>(d_desc, B, quality, d_huff, tiles_byte, d_info,
                                                 d_out, d_sizes);
  MRX_LAUNCH_CHECK("jpeg_file_kernel");
  return MRX_OK;
}
