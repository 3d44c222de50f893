// composite.cu -- mask compositing of visualize.display_instances
// (serve.py:160-169; SURVEY.md 8f rank 2: the consumer right behind
// unmold_detections).  The reference hands the [H,W,N] bool masks to matplotlib code whose
// mask part is, per instance in order,
//     for c in 0..2:  image[:,:,c] = where(mask == 1, image[:,:,c]*(1-alpha) + alpha*color[c]*255,
//                                          image[:,:,c])
// on a uint32 working copy (float64 arithmetic, truncating store), shown as uint8.
// Doing that on the device canvas mrx_mask_expand just wrote removes the 105 MB per image
// device -> host copy of the masks for callers that only want the overlay.
//
// Alternatives tried and removed again: tabulating the blend per (instance, channel, value)
// instead of evaluating it in fp64 per pixel (no gain), restricting every block of pixels to the
// instances whose box meets it (slower), and persistent CTAs with a two-stage bulk-copy ring
// (slower: four resident CTAs per SM are too few threads for the divergent walk; time went as
// 1/CTAs).  What did pay: replacing the load-and-store staging loop by ONE bulk copy per block,
// and the blend constants' load loop by a second one.
//
// HBM-read bound: N bytes of canvas per pixel (3.36 GB per config-2 batch) + 3 B in + 3 B out.
// One CTA = 256 consecutive pixels of one image: their 256*N canvas bytes are contiguous
// (N innermost) and are brought into shared memory by a single 1-D bulk copy (TMA, completion
// on an mbarrier) issued by thread 0, the image's blend constants by a second one; eight CTAs are
// resident per SM, so ~200 KB of copies are in flight per SM.  Thread t then walks pixel t's
// N bytes (4 at a time when N % 4 == 0: most words are zero) and applies the blends of the set
// instances in instance order -- fp64 with explicit _rn intrinsics in NumPy's operation
// order, truncation to uint32 after every instance: bit-exact.
#include "common.cuh"

namespace mrx {

constexpr int kCompThreads = 256;   // faster than 128, 384 or 512 threads per CTA

__global__ void __launch_bounds__(kCompThreads)
composite_masks_kernel(const Slots<const unsigned char> canvas, const int *__restrict__ counts,
                       const int *__restrict__ geom, const int4 *__restrict__ boxes, const unsigned char *__restrict__ images,
                       const long long *__restrict__ image_off, const double *__restrict__ blend,
                       double one_minus_alpha, unsigned char *__restrict__ out, int R,
                       int blend_bulk) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int b = blockIdx.y;
  const int H = geom[b * MRX_GEOM_INTS + 0], W = geom[b * MRX_GEOM_INTS + 1];
  // (the host checks H*W < 2^31: pixel indices are 32-bit, their byte offsets 64-bit)
  const unsigned npix = static_cast<unsigned>(H) * static_cast<unsigned>(W);
  const unsigned p0 = blockIdx.x * static_cast<unsigned>(kCompThreads);
  if (p0 >= npix) return;
  const int npx = static_cast<int>(min(static_cast<unsigned>(kCompThreads), npix - p0));
  const int N = counts[b];
  const int t = threadIdx.x;

  // shared memory: [blend constants R*3 doubles][skip flags R bytes, padded][canvas bytes]
  double *s_blend = reinterpret_cast<double *>(smem);
  unsigned char *s_skip = smem + ((static_cast<size_t>(R) * 3 * sizeof(double) + 15) & ~static_cast<size_t>(15));
  unsigned char *s_can = s_skip + ((R + 15) & ~15);

  // 256*N is a multiple of 16 and so is every canvas slot offset; the slot holds
  // round_up(H*W*N, 16) bytes, so the copy of the last block may take its pad bytes.  One 1-D
  // bulk copy (TMA) brings the block's canvas bytes in while the constants below are loaded.
  __shared__ __align__(8) uint64_t s_bar;
  const unsigned bytes = (static_cast<unsigned>(npx) * N + 15u) & ~15u;
  if (t == 0) {
    mbar_init(&s_bar, 1);
    fence_mbar_init();
  }
  if (t < 32) __syncwarp();
  // the image's blend constants (N x 3 doubles) come the same way when every image's block of
  // the [B,R,3] array starts 16-byte aligned (blend_bulk: R even, base aligned); otherwise the
  // threads load them
  if (t == 0) {
    const unsigned cbytes = blend_bulk ? (static_cast<unsigned>(N) * 24u + 15u) & ~15u : 0u;
    if (bytes + cbytes) {
      mbar_arrive_expect_tx(&s_bar, bytes + cbytes);
      if (bytes) bulk_g2s(s_can, canvas.base + __ldg(canvas.off + b) + static_cast<size_t>(p0) * N, bytes, &s_bar);
      if (cbytes) bulk_g2s(s_blend, blend + static_cast<size_t>(b) * R * 3, cbytes, &s_bar);
    } else {
      mbar_arrive(&s_bar);
    }
  }
  if (!blend_bulk) {
    for (int i = t; i < N * 3; i += kCompThreads)
      s_blend[i] = blend[static_cast<size_t>(b) * R * 3 + i];
  }
  for (int i = t; i < N; i += kCompThreads) {
    const int4 bx = boxes[static_cast<size_t>(b) * R + i];
    s_skip[i] = (bx.x | bx.y | bx.z | bx.w) == 0;   // upstream: `if not np.any(boxes[i]): continue`
  }
  __syncthreads();
  if (t >= npx) return;

  const unsigned char *ip = images + image_off[b] + static_cast<size_t>(p0 + t) * 3;
  unsigned v0 = ip[0], v1 = ip[1], v2 = ip[2];
  mbar_wait(&s_bar, 0);
  auto apply = [&](int i) {
    if (s_skip[i]) return;
    const double *bl = s_blend + i * 3;
    v0 = __double2uint_rz(__dadd_rn(__dmul_rn(static_cast<double>(v0), one_minus_alpha), bl[0]));
    v1 = __double2uint_rz(__dadd_rn(__dmul_rn(static_cast<double>(v1), one_minus_alpha), bl[1]));
    v2 = __double2uint_rz(__dadd_rn(__dmul_rn(static_cast<double>(v2), one_minus_alpha), bl[2]));
  };
  const unsigned char *mp = s_can + static_cast<size_t>(t) * N;
  if ((N & 3) == 0) {
    // ~3 % of the bytes are set: test five words (20 instances) with one OR before looking
    // at any of them
    const uint32_t *mw = reinterpret_cast<const uint32_t *>(mp);
    const int nw = N >> 2;
    auto word = [&](int k, uint32_t w) {
      if (w == 0u) return;
      if (w & 0x000000ffu) apply(4 * k);
      if (w & 0x0000ff00u) apply(4 * k + 1);
      if (w & 0x00ff0000u) apply(4 * k + 2);
      if (w & 0xff000000u) apply(4 * k + 3);
    };
    int k = 0;
    for (; k + 5 <= nw; k += 5) {
      const uint32_t w0 = mw[k], w1 = mw[k + 1], w2 = mw[k + 2], w3 = mw[k + 3], w4 = mw[k + 4];
      if ((w0 | w1 | w2 | w3 | w4) == 0u) continue;
      word(k, w0);
      word(k + 1, w1);
      word(k + 2, w2);
      word(k + 3, w3);
      word(k + 4, w4);
    }
    for (; k < nw; ++k) word(k, mw[k]);
  } else {
    for (int i = 0; i < N; ++i)
      if (mp[i]) apply(i);
  }
  unsigned char *op = out + image_off[b] + static_cast<size_t>(p0 + t) * 3;
  op[0] = static_cast<unsigned char>(v0);   // astype(uint8): modulo 256
  op[1] = static_cast<unsigned char>(v1);
  op[2] = static_cast<unsigned char>(v2);
}

}  // namespace mrx

extern "C" int mrx_composite_masks(const unsigned char *d_canvas, const long long *d_canvas_off,
                                   const int *d_counts, const int *d_geom, const int *d_boxes,
                                   const unsigned char *d_images, const long long *d_image_off,
                                   const double *d_blend, double one_minus_alpha,
                                   unsigned char *d_out, int B, int R, long long max_pixels,
                                   void *stream) {
  using namespace mrx;
  const char *fn = "mrx_composite_masks";
  if (int rc = check_slots(fn, d_canvas, d_canvas_off, d_counts, d_geom, B, R)) return rc;
  MRX_CHECK_ARG(d_boxes && d_images && d_image_off && d_blend && d_out, "%s: null pointer", fn);
  MRX_CHECK_ARG(max_pixels >= 0, "%s: bad max_pixels %lld", fn, max_pixels);
  if (B == 0 || max_pixels == 0) return MRX_OK;
  DevInfo dev;
  if (int rc = current_device_info(&dev)) return rc;
  const int max_optin = dev.max_smem_optin;
  const size_t smem = ((static_cast<size_t>(R) * 3 * sizeof(double) + 15) & ~static_cast<size_t>(15)) +
                      ((R + 15) & ~15) + static_cast<size_t>(kCompThreads) * R + 16;
  MRX_CHECK_SUPPORTED(smem <= static_cast<size_t>(max_optin),
                      "mrx_composite_masks: R=%d needs %zu B of shared memory (limit %d)", R, smem,
                      max_optin);
  const long long blocks = (max_pixels + kCompThreads - 1) / kCompThreads;
  MRX_CHECK_SUPPORTED(max_pixels < 0x7fffffffLL - kCompThreads, "mrx_composite_masks: image too large");
  static SmemCache cache;
  if (int rc = ensure_dynamic_smem(reinterpret_cast<const void *>(composite_masks_kernel), &cache,
                                   dev.device, static_cast<int>(smem)))
    return rc;
  dim3 grid(static_cast<unsigned>(blocks), static_cast<unsigned>(B));
  composite_masks_kernel<<<grid, kCompThreads, smem, static_cast<cudaStream_t>(stream)>>>(
      Slots<const unsigned char>{d_canvas, d_canvas_off}, d_counts, d_geom,
      reinterpret_cast<const int4 *>(d_boxes), d_images,
      d_image_off, d_blend, one_minus_alpha, d_out, R,
      ((R & 1) == 0 && (reinterpret_cast<uintptr_t>(d_blend) & 15u) == 0u) ? 1 : 0);
  MRX_LAUNCH_CHECK("composite_masks_kernel");
  return MRX_OK;
}
