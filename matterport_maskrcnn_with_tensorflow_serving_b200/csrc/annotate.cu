// annotate.cu -- the artists visualize.display_instances draws over the mask overlay
// (serve.py:160-169): per kept instance a box and its contour outlines in the instance's colour,
// then every caption in white, as the OpenCV calls of DESIGN.md section 3.25 draw them at the
// image's own resolution.
//
// Boxes and outlines go through one int32 key plane per image: every pixel an instance draws does
// atomicMax(key, k + 1), so the key alone says which instance drew a pixel last in display order
// (a box and its outlines share instance k's colour).  The resolve step then writes each keyed
// pixel's colour into the overlay and sets the caption stencils (shaped by cv2 on the host) to
// white on top.
//
//   annotate_zero_kernel     key planes cleared
//   annotate_box_kernel      CTA per (instance, image): the four edges of cv2.rectangle(thickness 1,
//                            LINE_8): rows y1 and y2 over [x1, x2], columns x1 and x2 over [y1, y2],
//                            each clipped to the image (axis-aligned, so clipping drops pixels only)
//   annotate_vertex_kernel   thread per contour vertex: polylines(shift=1, LINE_8) of a segment
//                            between edge midpoints sets exactly its two end points rounded half
//                            up, so an outline is the set of its rounded vertices; the vertex's
//                            contour and instance are found by binary search in the offsets
//   annotate_resolve_kernel  keyed pixels take their instance's colour
//   annotate_caption_kernel  CTA per caption patch: stencil bits set to 255
#include "common.cuh"

namespace mrx {

namespace annotate {

constexpr int kThreads = 256;

__device__ __forceinline__ bool box_is_zero(const int4 bx) { return (bx.x | bx.y | bx.z | bx.w) == 0; }

__global__ void __launch_bounds__(kThreads)
annotate_zero_kernel(const int *__restrict__ geom, int *__restrict__ keys,
                     const long long *__restrict__ key_off) {
  const int b = blockIdx.y;
  const long long npix = static_cast<long long>(geom[b * MRX_GEOM_INTS + 0]) * geom[b * MRX_GEOM_INTS + 1];
  int *k = keys + key_off[b];
  for (long long p = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; p < npix;
       p += static_cast<long long>(gridDim.x) * kThreads)
    k[p] = 0;
}

__global__ void __launch_bounds__(kThreads)
annotate_box_kernel(const int *__restrict__ counts, const int *__restrict__ geom,
                    const int4 *__restrict__ boxes, int *__restrict__ keys,
                    const long long *__restrict__ key_off, int R) {
  const int k = blockIdx.x, b = blockIdx.y;
  if (k >= counts[b]) return;
  const int4 bx = boxes[static_cast<size_t>(b) * R + k];   // (y1, x1, y2, x2)
  if (box_is_zero(bx)) return;                               // upstream skips all-zero boxes
  const int H = geom[b * MRX_GEOM_INTS + 0], W = geom[b * MRX_GEOM_INTS + 1];
  const int ya = min(bx.x, bx.z), yb = max(bx.x, bx.z), xa = min(bx.y, bx.w), xb = max(bx.y, bx.w);
  int *kp = keys + key_off[b];
  const int key = k + 1;
  // rows y1 and y2 over the clipped columns
  const int c0 = max(xa, 0), c1 = min(xb, W - 1);
  for (int x = c0 + static_cast<int>(threadIdx.x); x <= c1; x += kThreads) {
    if (ya >= 0 && ya < H) atomicMax(kp + static_cast<long long>(ya) * W + x, key);
    if (yb >= 0 && yb < H) atomicMax(kp + static_cast<long long>(yb) * W + x, key);
  }
  // columns x1 and x2 over the clipped rows
  const int r0 = max(ya, 0), r1 = min(yb, H - 1);
  for (int y = r0 + static_cast<int>(threadIdx.x); y <= r1; y += kThreads) {
    if (xa >= 0 && xa < W) atomicMax(kp + static_cast<long long>(y) * W + xa, key);
    if (xb >= 0 && xb < W) atomicMax(kp + static_cast<long long>(y) * W + xb, key);
  }
}

// the last index i in [0, n) with off[i] <= v (off ascending, off[0] <= v)
__device__ __forceinline__ int last_at_most(const long long *__restrict__ off, int n, long long v) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= v) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// a half-pixel coordinate u (2u an integer) rounded half up: floor((2u + 1) / 2)
__device__ __forceinline__ int round_half_up(double u) {
  return (__double2int_rn(2.0 * u) + 1) >> 1;
}

__global__ void __launch_bounds__(kThreads)
annotate_vertex_kernel(const int *__restrict__ counts, const int *__restrict__ geom,
                       const int4 *__restrict__ boxes, const double2 *__restrict__ verts,
                       const long long *__restrict__ contour_off,
                       const long long *__restrict__ inst_contour_off, long long n_vertices,
                       int *__restrict__ keys, const long long *__restrict__ key_off, int B, int R) {
  const int ni = B * R;
  const long long C = inst_contour_off[ni];
  if (C <= 0) return;
  const long long V = min(n_vertices, contour_off[C]);
  for (long long v = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; v < V;
       v += static_cast<long long>(gridDim.x) * kThreads) {
    if (v < contour_off[0]) continue;
    const int c = last_at_most(contour_off, static_cast<int>(C), v);
    const int i = last_at_most(inst_contour_off, ni, c);
    const int b = i / R, k = i - b * R;
    if (k >= counts[b] || box_is_zero(boxes[i])) continue;
    const int H = geom[b * MRX_GEOM_INTS + 0], W = geom[b * MRX_GEOM_INTS + 1];
    const double2 p = verts[v];
    const int x = round_half_up(p.x), y = round_half_up(p.y);
    if (x < 0 || x >= W || y < 0 || y >= H) continue;
    atomicMax(keys + key_off[b] + static_cast<long long>(y) * W + x, k + 1);
  }
}

__global__ void __launch_bounds__(kThreads)
annotate_resolve_kernel(const int *__restrict__ geom, const int *__restrict__ keys,
                        const long long *__restrict__ key_off, const unsigned char *__restrict__ rgb8,
                        unsigned char *__restrict__ images, const long long *__restrict__ image_off,
                        int R) {
  const int b = blockIdx.y;
  const long long npix = static_cast<long long>(geom[b * MRX_GEOM_INTS + 0]) * geom[b * MRX_GEOM_INTS + 1];
  const int *kp = keys + key_off[b];
  unsigned char *img = images + image_off[b];
  const unsigned char *tab = rgb8 + static_cast<size_t>(b) * R * 3;
  for (long long p = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; p < npix;
       p += static_cast<long long>(gridDim.x) * kThreads) {
    const int key = kp[p];
    if (key == 0) continue;
    const unsigned char *c = tab + (key - 1) * 3;
    img[p * 3 + 0] = c[0];
    img[p * 3 + 1] = c[1];
    img[p * 3 + 2] = c[2];
  }
}

__global__ void __launch_bounds__(kThreads)
annotate_caption_kernel(const int *__restrict__ geom, unsigned char *__restrict__ images,
                        const long long *__restrict__ image_off,
                        const unsigned char *__restrict__ stencils,
                        const long long *__restrict__ patches, int B) {
  const long long *rec = patches + 6ll * blockIdx.x;   // (image, y0, x0, h, w, byte offset)
  const long long b = rec[0], y0 = rec[1], x0 = rec[2], h = rec[3], w = rec[4], off = rec[5];
  if (b < 0 || b >= B || h <= 0 || w <= 0) return;
  const long long H = geom[b * MRX_GEOM_INTS + 0], W = geom[b * MRX_GEOM_INTS + 1];
  unsigned char *img = images + image_off[b];
  const unsigned char *bits = stencils + off;
  for (long long j = threadIdx.x; j < h * w; j += kThreads) {
    if (!((bits[j >> 3] >> (7 - (j & 7))) & 1)) continue;
    const long long y = y0 + j / w, x = x0 + j % w;
    if (y < 0 || y >= H || x < 0 || x >= W) continue;   // a patch is clipped to its image
    unsigned char *px = img + (y * W + x) * 3;
    px[0] = 255;
    px[1] = 255;
    px[2] = 255;
  }
}

// grid over the pixels of the largest image: enough CTAs to fill the GPU, each striding
dim3 pixel_grid(long long max_pixels, int B, const DevInfo &dev) {
  const long long want = (max_pixels + kThreads - 1) / kThreads;
  const long long cap = max(1LL, static_cast<long long>(dev.sms) * 16 / max(B, 1));
  return dim3(static_cast<unsigned>(max(1LL, min(want, cap))), static_cast<unsigned>(B));
}

}  // namespace annotate

}  // namespace mrx

using namespace mrx;

static int check_batch(const char *fn, int B, int R, long long max_pixels) {
  MRX_CHECK_ARG(B >= 0 && B <= MRX_MAX_BATCH && R >= 1 && R <= 65534,
                "%s: bad sizes B=%d R=%d (need 0<=B<=%d, 1<=R<=65534)", fn, B, R, MRX_MAX_BATCH);
  MRX_CHECK_ARG(max_pixels >= 0 && max_pixels < 0x7fffffffLL,
                "%s: bad max_pixels %lld (need 0<=max_pixels<2^31-1)", fn, max_pixels);
  return MRX_OK;
}

extern "C" int mrx_annotate_draw(const int *d_counts, const int *d_geom, const int *d_boxes,
                                 const double *d_vertices, const long long *d_contour_off,
                                 const long long *d_inst_contour_off, long long n_vertices,
                                 int show_bbox, int *d_keys, const long long *d_key_off, int B,
                                 int R, long long max_pixels, void *stream) {
  using namespace annotate;
  const char *fn = "mrx_annotate_draw";
  MRX_CHECK_ARG(d_counts && d_geom && d_boxes && d_keys && d_key_off, "%s: null pointer", fn);
  if (int rc = check_batch(fn, B, R, max_pixels)) return rc;
  MRX_CHECK_ARG(n_vertices >= 0, "%s: bad n_vertices %lld", fn, n_vertices);
  MRX_CHECK_ARG(n_vertices == 0 || (d_vertices && d_contour_off && d_inst_contour_off),
                "%s: null contour pointer", fn);
  if (B == 0 || max_pixels == 0) return MRX_OK;
  DevInfo dev;
  if (int rc = current_device_info(&dev)) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  annotate_zero_kernel<<<pixel_grid(max_pixels, B, dev), kThreads, 0, st>>>(d_geom, d_keys, d_key_off);
  MRX_LAUNCH_CHECK("annotate_zero_kernel");
  const int4 *boxes = reinterpret_cast<const int4 *>(d_boxes);
  if (show_bbox) {
    annotate_box_kernel<<<dim3(R, B), kThreads, 0, st>>>(d_counts, d_geom, boxes, d_keys, d_key_off, R);
    MRX_LAUNCH_CHECK("annotate_box_kernel");
  }
  if (n_vertices > 0) {
    const long long blocks = min((n_vertices + kThreads - 1) / kThreads, static_cast<long long>(dev.sms) * 16);
    annotate_vertex_kernel<<<static_cast<unsigned>(blocks), kThreads, 0, st>>>(
        d_counts, d_geom, boxes, reinterpret_cast<const double2 *>(d_vertices), d_contour_off,
        d_inst_contour_off, n_vertices, d_keys, d_key_off, B, R);
    MRX_LAUNCH_CHECK("annotate_vertex_kernel");
  }
  return MRX_OK;
}

extern "C" int mrx_annotate_resolve(const int *d_geom, const int *d_keys,
                                    const long long *d_key_off, const unsigned char *d_rgb8,
                                    unsigned char *d_images, const long long *d_image_off,
                                    const unsigned char *d_stencils, const long long *d_patches,
                                    int P, int B, int R, long long max_pixels, void *stream) {
  using namespace annotate;
  const char *fn = "mrx_annotate_resolve";
  MRX_CHECK_ARG(d_geom && d_keys && d_key_off && d_rgb8 && d_images && d_image_off,
                "%s: null pointer", fn);
  if (int rc = check_batch(fn, B, R, max_pixels)) return rc;
  MRX_CHECK_ARG(P >= 0, "%s: bad patch count %d", fn, P);
  MRX_CHECK_ARG(P == 0 || (d_stencils && d_patches), "%s: null stencil pointer", fn);
  if (B == 0 || max_pixels == 0) return MRX_OK;
  DevInfo dev;
  if (int rc = current_device_info(&dev)) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  annotate_resolve_kernel<<<pixel_grid(max_pixels, B, dev), kThreads, 0, st>>>(
      d_geom, d_keys, d_key_off, d_rgb8, d_images, d_image_off, R);
  MRX_LAUNCH_CHECK("annotate_resolve_kernel");
  if (P > 0) {
    annotate_caption_kernel<<<P, kThreads, 0, st>>>(d_geom, d_images, d_image_off, d_stencils,
                                                    d_patches, B);
    MRX_LAUNCH_CHECK("annotate_caption_kernel");
  }
  return MRX_OK;
}
