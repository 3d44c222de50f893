// mold.cu -- the pre-processing half of the path, preprocess_input
// (serve.py:83-107):
//   cv2_resize_kernel   cv2.resize(img, (S, S))                      serve.py:88-89
//   mold_image_kernel   utils.resize_image(square) + mold_image      serve.py:91-98
//
// cv2.resize on uint8 is OpenCV's fixed-point INTER_LINEAR: coordinates in float32,
// 11-bit coefficients, horizontal pass to int32, vertical pass
//   ((b0*(S0>>4))>>16) + ((b1*(S1>>4))>>16) + 2) >> 2
// and, for an exact 2x shrink in both axes, the INTER_AREA 2x2 box average.  Both are
// integer pipelines, restated here operation for operation -> bit-exact with cv2.
//
// resize_image scales with the zero-border bilinear of utils.resize (a4) in float64 and
// truncates to uint8; scipy's operation order is reproduced with _rn intrinsics so the
// truncation lands on the same integer:  cc = (k+0.5)*zoom - 0.5 ; t = cc - floor(cc) ;
// v = ((c00*wy0)*wx0) + ((c01*wy0)*wx1) + ((c10*wy1)*wx0) + ((c11*wy1)*wx1).
#include "common.cuh"

namespace mrx {

constexpr int kMoldThreads = 256;

struct LinCoef {
  int s;      // source index of the first tap
  int a0, a1; // 11-bit fixed-point weights of taps s and s+1
};

// OpenCV resize.cpp, linear branch of the coefficient tables (fixpt = true)
__device__ __forceinline__ LinCoef cv_lin_coef(int d, double scale, int n_src, bool clamp_w) {
  float f = __double2float_rn(__dsub_rn(__dmul_rn(static_cast<double>(d) + 0.5, scale), 0.5));
  int s = __float2int_rd(f);
  f = __fsub_rn(f, static_cast<float>(s));
  if (clamp_w) {
    if (s < 0) { f = 0.f; s = 0; }
    if (s >= n_src - 1) { f = 0.f; s = n_src - 1; }
  }
  LinCoef c;
  c.s = s;
  c.a0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
  c.a1 = __float2int_rn(__fmul_rn(f, 2048.f));
  return c;
}

// Image blockIdx.y of a batch: sources of any size at src + src_off[b] (sizes in src_hw[b]),
// destinations dh x dw each, densely packed.  src_off == nullptr: one image, sizes by value.
__global__ void __launch_bounds__(kMoldThreads)
cv2_resize_kernel(const unsigned char *__restrict__ src, const long long *__restrict__ src_off,
                  const int *__restrict__ src_hw, int sh, int sw,
                  unsigned char *__restrict__ dst, int dh, int dw) {
  const long long total = static_cast<long long>(dh) * dw;
  if (src_off != nullptr) {
    const int b = blockIdx.y;
    src += src_off[b];
    sh = src_hw[2 * b];
    sw = src_hw[2 * b + 1];
    dst += static_cast<size_t>(b) * total * 3;
  }
  // cv::resize: inv_scale = dsize/ssize (double) ; hal::resize: scale = 1./inv_scale
  const double scale_x = __ddiv_rn(1.0, __ddiv_rn(static_cast<double>(dw), static_cast<double>(sw)));
  const double scale_y = __ddiv_rn(1.0, __ddiv_rn(static_cast<double>(dh), static_cast<double>(sh)));
  // INTER_LINEAR with an exact 2x shrink in both axes is computed as INTER_AREA (2x2 box)
  const double eps = 2.220446049250313e-16;
  const bool area_fast_2x = fabs(scale_x - 2.0) < eps && fabs(scale_y - 2.0) < eps;
  for (long long i = static_cast<long long>(blockIdx.x) * kMoldThreads + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * kMoldThreads) {
    const int dy = static_cast<int>(i / dw);
    const int dx = static_cast<int>(i - static_cast<long long>(dy) * dw);
    unsigned char *o = dst + i * 3;
    if (area_fast_2x) {
      const unsigned char *p0 = src + (static_cast<size_t>(2 * dy) * sw + 2 * dx) * 3;
      const unsigned char *p1 = p0 + static_cast<size_t>(sw) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c)
        o[c] = static_cast<unsigned char>((p0[c] + p0[3 + c] + p1[c] + p1[3 + c] + 2) >> 2);
      continue;
    }
    const LinCoef cx = cv_lin_coef(dx, scale_x, sw, true);
    const LinCoef cy = cv_lin_coef(dy, scale_y, sh, false);
    const int x0 = cx.s, x1 = min(cx.s + 1, sw - 1);
    const int y0 = min(max(cy.s, 0), sh - 1), y1 = min(max(cy.s + 1, 0), sh - 1);
    const unsigned char *r0 = src + static_cast<size_t>(y0) * sw * 3;
    const unsigned char *r1 = src + static_cast<size_t>(y1) * sw * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int S0 = r0[x0 * 3 + c] * cx.a0 + r0[x1 * 3 + c] * cx.a1;   // hresize, row y0
      const int S1 = r1[x0 * 3 + c] * cx.a0 + r1[x1 * 3 + c] * cx.a1;   // hresize, row y1
      const int v = (((cy.a0 * (S0 >> 4)) >> 16) + ((cy.a1 * (S1 >> 4)) >> 16) + 2) >> 2;
      o[c] = static_cast<unsigned char>(min(max(v, 0), 255));
    }
  }
}

struct ZoomCoef {
  int i0;          // floor of the source coordinate, in [-1, n-1]
  double w0, w1;   // weights of taps i0 and i0+1
};

__device__ __forceinline__ ZoomCoef zoom_coef(int k, double zoom) {
  const double cc = __dsub_rn(__dmul_rn(static_cast<double>(k) + 0.5, zoom), 0.5);
  const double fl = floor(cc);
  const double t = __dsub_rn(cc, fl);
  ZoomCoef z;
  z.i0 = static_cast<int>(fl);
  z.w0 = __dsub_rn(1.0, t);
  z.w1 = t;
  return z;
}

// Image blockIdx.y of a batch of equally sized sources (densely packed) -> equally sized outputs.
template <typename TOut>
__global__ void __launch_bounds__(kMoldThreads)
mold_image_kernel(const unsigned char *__restrict__ src, int sh, int sw, int new_h, int new_w,
                  int top, int left, int out_h, int out_w, double zoom_y, double zoom_x,
                  double m0, double m1, double m2, TOut *__restrict__ out,
                  unsigned char *__restrict__ out_u8) {
  const long long total = static_cast<long long>(out_h) * out_w;
  src += static_cast<size_t>(blockIdx.y) * sh * sw * 3;
  out += static_cast<size_t>(blockIdx.y) * total * 3;
  if (out_u8) out_u8 += static_cast<size_t>(blockIdx.y) * total * 3;
  const bool scaled = (new_h != sh) || (new_w != sw);
  const double mean[3] = {m0, m1, m2};
  for (long long i = static_cast<long long>(blockIdx.x) * kMoldThreads + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * kMoldThreads) {
    const int oy = static_cast<int>(i / out_w);
    const int ox = static_cast<int>(i - static_cast<long long>(oy) * out_w);
    const int y = oy - top, x = ox - left;
    unsigned char px[3] = {0, 0, 0};   // np.pad(..., constant_values=0)
    if (y >= 0 && y < new_h && x >= 0 && x < new_w) {
      if (!scaled) {
        const unsigned char *s = src + (static_cast<size_t>(y) * sw + x) * 3;
        px[0] = s[0]; px[1] = s[1]; px[2] = s[2];
      } else {
        const ZoomCoef zy = zoom_coef(y, zoom_y);
        const ZoomCoef zx = zoom_coef(x, zoom_x);
        const bool y0ok = zy.i0 >= 0, y1ok = zy.i0 + 1 <= sh - 1;
        const bool x0ok = zx.i0 >= 0, x1ok = zx.i0 + 1 <= sw - 1;
        const unsigned char *r0 = src + static_cast<size_t>(max(zy.i0, 0)) * sw * 3;
        const unsigned char *r1 = src + static_cast<size_t>(min(zy.i0 + 1, sh - 1)) * sw * 3;
        const int xa = max(zx.i0, 0) * 3, xb = min(zx.i0 + 1, sw - 1) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const double c00 = (y0ok && x0ok) ? static_cast<double>(r0[xa + c]) : 0.0;
          const double c01 = (y0ok && x1ok) ? static_cast<double>(r0[xb + c]) : 0.0;
          const double c10 = (y1ok && x0ok) ? static_cast<double>(r1[xa + c]) : 0.0;
          const double c11 = (y1ok && x1ok) ? static_cast<double>(r1[xb + c]) : 0.0;
          double t = __dmul_rn(__dmul_rn(c00, zy.w0), zx.w0);
          t = __dadd_rn(t, __dmul_rn(__dmul_rn(c01, zy.w0), zx.w1));
          t = __dadd_rn(t, __dmul_rn(__dmul_rn(c10, zy.w1), zx.w0));
          t = __dadd_rn(t, __dmul_rn(__dmul_rn(c11, zy.w1), zx.w1));
          // skimage clip to [min(in,0), max(in,0)] is a no-op here; astype(uint8) truncates
          px[c] = static_cast<unsigned char>(static_cast<int>(t));
        }
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      // mold_image: images.astype(float32) - MEAN_PIXEL(float64) -> float64
      const double v = __dsub_rn(static_cast<double>(px[c]), mean[c]);
      out[i * 3 + c] = static_cast<TOut>(v);
      if (out_u8) out_u8[i * 3 + c] = px[c];
    }
  }
}

static unsigned grid_for(long long total, int threads, int sms) {
  long long blocks = (total + threads - 1) / threads;
  const long long cap = 32LL * sms;   // grid-stride over a multiple of the SM count
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return static_cast<unsigned>(blocks);
}

}  // namespace mrx

using namespace mrx;

static int cv2_resize_launch(const unsigned char *d_src, const long long *d_src_off,
                             const int *d_src_hw, int src_h, int src_w, unsigned char *d_dst,
                             int B, int dst_h, int dst_w, void *stream) {
  DevInfo dev;
  if (int rc = current_device_info(&dev)) return rc;
  const long long total = static_cast<long long>(dst_h) * dst_w;
  dim3 grid(grid_for(total, kMoldThreads, dev.sms), B);
  cv2_resize_kernel<<<grid, kMoldThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      d_src, d_src_off, d_src_hw, src_h, src_w, d_dst, dst_h, dst_w);
  MRX_LAUNCH_CHECK("cv2_resize_kernel");
  return MRX_OK;
}

extern "C" int mrx_cv2_resize_u8c3(const unsigned char *d_src, int src_h, int src_w,
                                   unsigned char *d_dst, int dst_h, int dst_w, void *stream) {
  MRX_CHECK_ARG(d_src && d_dst, "mrx_cv2_resize_u8c3: null pointer");
  MRX_CHECK_ARG(src_h >= 1 && src_w >= 1 && dst_h >= 1 && dst_w >= 1,
                "mrx_cv2_resize_u8c3: bad sizes %dx%d -> %dx%d", src_h, src_w, dst_h, dst_w);
  return cv2_resize_launch(d_src, nullptr, nullptr, src_h, src_w, d_dst, 1, dst_h, dst_w, stream);
}

extern "C" int mrx_cv2_resize_u8c3_batch(const unsigned char *d_src, const long long *d_src_off,
                                         const int *d_src_hw, unsigned char *d_dst, int B,
                                         int dst_h, int dst_w, void *stream) {
  MRX_CHECK_ARG(d_src && d_src_off && d_src_hw && d_dst, "mrx_cv2_resize_u8c3_batch: null pointer");
  MRX_CHECK_ARG(B >= 0 && B <= 65535 && dst_h >= 1 && dst_w >= 1,
                "mrx_cv2_resize_u8c3_batch: bad sizes B=%d dst %dx%d", B, dst_h, dst_w);
  if (B == 0) return MRX_OK;
  return cv2_resize_launch(d_src, d_src_off, d_src_hw, 0, 0, d_dst, B, dst_h, dst_w, stream);
}

static int mold_launch(const unsigned char *d_src, int B, int src_h, int src_w, int new_h,
                       int new_w, int top, int left, int out_h, int out_w,
                       const double *mean_pixel, int out_dtype, void *d_out,
                       unsigned char *d_molded_u8, void *stream) {
  MRX_CHECK_ARG(d_src && d_out && mean_pixel, "mrx_mold_image: null pointer");
  MRX_CHECK_ARG(src_h >= 1 && src_w >= 1 && new_h >= 1 && new_w >= 1 && out_h >= 1 && out_w >= 1,
                "mrx_mold_image: bad sizes");
  MRX_CHECK_ARG(top >= 0 && left >= 0 && top + new_h <= out_h && left + new_w <= out_w,
                "mrx_mold_image: scaled image (%d,%d)+%dx%d does not fit %dx%d", top, left,
                new_h, new_w, out_h, out_w);
  MRX_CHECK_ARG(out_dtype == MRX_F32 || out_dtype == MRX_F64, "mrx_mold_image: out_dtype %d",
                out_dtype);
  MRX_CHECK_ARG(B >= 0 && B <= 65535, "mrx_mold_image_batch: B=%d", B);
  if (B == 0) return MRX_OK;
  // scipy.ndimage.zoom(grid_mode=True): zoom = in / out per axis (float64)
  const double zoom_y = static_cast<double>(src_h) / new_h;
  const double zoom_x = static_cast<double>(src_w) / new_w;
  DevInfo dev;
  if (int rc = current_device_info(&dev)) return rc;
  const long long total = static_cast<long long>(out_h) * out_w;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  dim3 grid(grid_for(total, kMoldThreads, dev.sms), B);
  if (out_dtype == MRX_F64) {
    mold_image_kernel<double><<<grid, kMoldThreads, 0, st>>>(
        d_src, src_h, src_w, new_h, new_w, top, left, out_h, out_w, zoom_y, zoom_x,
        mean_pixel[0], mean_pixel[1], mean_pixel[2], static_cast<double *>(d_out), d_molded_u8);
  } else {
    mold_image_kernel<float><<<grid, kMoldThreads, 0, st>>>(
        d_src, src_h, src_w, new_h, new_w, top, left, out_h, out_w, zoom_y, zoom_x,
        mean_pixel[0], mean_pixel[1], mean_pixel[2], static_cast<float *>(d_out), d_molded_u8);
  }
  MRX_LAUNCH_CHECK("mold_image_kernel");
  return MRX_OK;
}

extern "C" int mrx_mold_image(const unsigned char *d_src, int src_h, int src_w, int new_h,
                              int new_w, int top, int left, int out_h, int out_w,
                              const double *mean_pixel, int out_dtype, void *d_out,
                              unsigned char *d_molded_u8, void *stream) {
  return mold_launch(d_src, 1, src_h, src_w, new_h, new_w, top, left, out_h, out_w, mean_pixel,
                     out_dtype, d_out, d_molded_u8, stream);
}

extern "C" int mrx_mold_image_batch(const unsigned char *d_src, int B, int src_h, int src_w,
                                    int new_h, int new_w, int top, int left, int out_h,
                                    int out_w, const double *mean_pixel, int out_dtype,
                                    void *d_out, unsigned char *d_molded_u8, void *stream) {
  return mold_launch(d_src, B, src_h, src_w, new_h, new_w, top, left, out_h, out_w, mean_pixel,
                     out_dtype, d_out, d_molded_u8, stream);
}
