// deflate.cuh -- the zlib pieces the PNG encoder (png.cu) and decoder (png_decode.cu) share:
// deflate's length / distance tables, CRC-32 with its combine step, and Adler-32's modulus.
#pragma once

namespace mrx {
namespace {

constexpr int kMaxMatch = 258;
constexpr int kLCodes = 286, kDCodes = 30, kBLCodes = 19;
constexpr int kEndBlock = 256;
constexpr unsigned kMod = 65521;           // Adler-32
constexpr unsigned kPoly = 0xEDB88320u;    // CRC-32, reflected

__constant__ unsigned char c_extra_lbits[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2,
                                                2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ unsigned char c_extra_dbits[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6,
                                                6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ unsigned char c_extra_blbits[19] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
                                                 0, 0, 0, 0, 0, 0, 2, 3, 7};
__constant__ unsigned char c_bl_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5,
                                             11, 4, 12, 3, 13, 2, 14, 1, 15};
// match length - 3 of each length code's base
__constant__ unsigned char c_base_length[29] = {0,  1,  2,  3,  4,  5,   6,   7,   8,   10,
                                                12, 14, 16, 20, 24, 28,  32,  40,  48,  56,
                                                64, 80, 96, 112, 128, 160, 192, 224, 255};
__constant__ unsigned short c_base_dist[30] = {
    1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,   65,    97,    129,
    193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};

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

// the byte table and x2n of one CTA, in shared memory; the caller synchronises afterwards
__device__ void crc_tables(unsigned *table, unsigned *x2n) {
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
}

__device__ __forceinline__ unsigned crc_byte(const unsigned *table, unsigned crc, unsigned char v) {
  return table[(crc ^ v) & 0xFF] ^ (crc >> 8);
}

}  // namespace
}  // namespace mrx
