// anchors.cu -- api_utils.get_anchors (serve.py:105): the FPN pyramid
// anchors of upstream utils.generate_pyramid_anchors + norm_boxes, one thread per anchor.
//
// Output [A,4] float32, order: level-major, then y, x, ratio innermost
//   idx = off_l + ((y * nx_l + x) * n_ratios + r)
// Arithmetic is fp64 in numpy's operation order (explicit _rn intrinsics so the
// compiler cannot contract into FMAs), rounded once to fp32 -> bit-exact with numpy.
// HBM traffic: 16 B written per anchor, no reads.
#include "common.cuh"

namespace mrx {

struct AnchorParams {
  long long level_off[MRX_MAX_LEVELS + 1];
  double scale[MRX_MAX_LEVELS];
  double ratio[MRX_MAX_RATIOS];
  int ny[MRX_MAX_LEVELS], nx[MRX_MAX_LEVELS], stride[MRX_MAX_LEVELS];
  int n_levels, n_ratios, anchor_stride;
  int img_h, img_w;
};

constexpr int kAnchorThreads = 256;

__global__ void __launch_bounds__(kAnchorThreads)
anchors_kernel(const AnchorParams p, float4 *__restrict__ out) {
  const long long total = p.level_off[p.n_levels];
  const double hm1 = static_cast<double>(p.img_h - 1);
  const double wm1 = static_cast<double>(p.img_w - 1);
  for (long long idx = static_cast<long long>(blockIdx.x) * kAnchorThreads + threadIdx.x;
       idx < total; idx += static_cast<long long>(gridDim.x) * kAnchorThreads) {
    int l = 0;
#pragma unroll
    for (int k = 1; k < MRX_MAX_LEVELS; ++k)
      if (k < p.n_levels && idx >= p.level_off[k]) l = k;
    const long long local = idx - p.level_off[l];
    const int r = static_cast<int>(local % p.n_ratios);
    const long long cell = local / p.n_ratios;
    const int x = static_cast<int>(cell % p.nx[l]);
    const int y = static_cast<int>(cell / p.nx[l]);
    // generate_anchors: heights = scales / sqrt(ratios); widths = scales * sqrt(ratios)
    const double sq = __dsqrt_rn(p.ratio[r]);
    const double h = __ddiv_rn(p.scale[l], sq);
    const double w = __dmul_rn(p.scale[l], sq);
    // shifts = arange(0, n, anchor_stride) * feature_stride  (exact integers)
    const double cy = static_cast<double>(y * p.anchor_stride * p.stride[l]);
    const double cx = static_cast<double>(x * p.anchor_stride * p.stride[l]);
    const double hh = __dmul_rn(0.5, h);
    const double hw = __dmul_rn(0.5, w);
    const double y1 = __dsub_rn(cy, hh), x1 = __dsub_rn(cx, hw);
    const double y2 = __dadd_rn(cy, hh), x2 = __dadd_rn(cx, hw);
    // norm_boxes: (boxes - [0,0,1,1]) / [h-1,w-1,h-1,w-1] -> float32
    float4 o;
    o.x = __double2float_rn(__ddiv_rn(y1, hm1));
    o.y = __double2float_rn(__ddiv_rn(x1, wm1));
    o.z = __double2float_rn(__ddiv_rn(__dsub_rn(y2, 1.0), hm1));
    o.w = __double2float_rn(__ddiv_rn(__dsub_rn(x2, 1.0), wm1));
    out[idx] = o;
  }
}

static int fill_params(AnchorParams &p, int img_h, int img_w, const double *scales,
                       const double *ratios, const int *strides, int n_levels, int n_ratios,
                       int anchor_stride) {
  MRX_CHECK_ARG(strides != nullptr, "anchors: null strides");
  MRX_CHECK_ARG(img_h >= 2 && img_w >= 2, "anchors: image %dx%d too small", img_h, img_w);
  MRX_CHECK_SUPPORTED(n_levels >= 1 && n_levels <= MRX_MAX_LEVELS,
                      "anchors: n_levels %d outside [1,%d]", n_levels, MRX_MAX_LEVELS);
  MRX_CHECK_SUPPORTED(n_ratios >= 1 && n_ratios <= MRX_MAX_RATIOS,
                      "anchors: n_ratios %d outside [1,%d]", n_ratios, MRX_MAX_RATIOS);
  MRX_CHECK_ARG(anchor_stride >= 1, "anchors: anchor_stride %d", anchor_stride);
  p.n_levels = n_levels;
  p.n_ratios = n_ratios;
  p.anchor_stride = anchor_stride;
  p.img_h = img_h;
  p.img_w = img_w;
  long long off = 0;
  for (int l = 0; l < n_levels; ++l) {
    MRX_CHECK_ARG(strides[l] >= 1, "anchors: stride[%d]=%d", l, strides[l]);
    // compute_backbone_shapes: ceil(dim / stride); arange(0, n, anchor_stride) has ceil(n/as) items
    const int fh = (img_h + strides[l] - 1) / strides[l];
    const int fw = (img_w + strides[l] - 1) / strides[l];
    p.ny[l] = (fh + anchor_stride - 1) / anchor_stride;
    p.nx[l] = (fw + anchor_stride - 1) / anchor_stride;
    p.stride[l] = strides[l];
    p.scale[l] = scales ? scales[l] : 0.0;
    p.level_off[l] = off;
    off += static_cast<long long>(p.ny[l]) * p.nx[l] * n_ratios;
  }
  for (int l = n_levels; l <= MRX_MAX_LEVELS; ++l) p.level_off[l] = off;
  p.level_off[n_levels] = off;
  for (int r = 0; r < n_ratios; ++r) p.ratio[r] = ratios ? ratios[r] : 1.0;
  return MRX_OK;
}

}  // namespace mrx

using namespace mrx;

extern "C" int mrx_anchor_count(int img_h, int img_w, const int *strides, int n_levels,
                                int n_ratios, int anchor_stride, long long *count) {
  MRX_CHECK_ARG(count != nullptr, "mrx_anchor_count: null count");
  AnchorParams p;
  if (int rc = fill_params(p, img_h, img_w, nullptr, nullptr, strides, n_levels, n_ratios,
                           anchor_stride))
    return rc;
  *count = p.level_off[n_levels];
  return MRX_OK;
}

extern "C" int mrx_anchors(float *d_out, int img_h, int img_w, const double *scales,
                           const double *ratios, const int *strides, int n_levels,
                           int n_ratios, int anchor_stride, void *stream) {
  MRX_CHECK_ARG(d_out && scales && ratios, "mrx_anchors: null pointer");
  AnchorParams p;
  if (int rc = fill_params(p, img_h, img_w, scales, ratios, strides, n_levels, n_ratios,
                           anchor_stride))
    return rc;
  const long long total = p.level_off[n_levels];
  if (total == 0) return MRX_OK;
  DevInfo dev;
  if (int rc = current_device_info(&dev)) return rc;
  long long blocks = (total + kAnchorThreads - 1) / kAnchorThreads;
  const long long cap = 16LL * dev.sms;   // grid-stride over a multiple of the SM count
  if (blocks > cap) blocks = cap;
  anchors_kernel<<<static_cast<unsigned>(blocks), kAnchorThreads, 0,
                   static_cast<cudaStream_t>(stream)>>>(p, reinterpret_cast<float4 *>(d_out));
  MRX_LAUNCH_CHECK("anchors_kernel");
  return MRX_OK;
}
