// detectnet.cu -- NVCaffe's DetectNetTransformationLayer (src/caffe/layers/detectnet_transform_layer.{cpp,cu},
// src/caffe/util/detectnet_coverage_rectangular.cpp) on the device: the image path (colour, mean, crop / rotate / scale / flip with
// the reference's bicubic) and the label path (box transform, pruning and the rectangular coverage map).  The per-image
// augmentation is an input (b2c_detectnet_aug in device memory): nothing here draws random numbers.
//
// Arithmetic follows the reference's types: coordinates and HSV in float, cubic_interpolation in double (its literals are double),
// with _rn intrinsics wherever a product feeds a sum so that nothing contracts into an FMA.  The one deliberate departure is the
// hue wrap of hsv_to_rgb (see colour_pixel).
#include <cuda_runtime.h>
#include <float.h>
#include <math_constants.h>
#include <string.h>
#include "b2c_common.cuh"

namespace b2c {

namespace {

constexpr int kImageThreads = 256;
constexpr int kLabelThreads = 256;
constexpr int kBoxWords = 16;                    // shared-memory words per box (see label_kernel)
constexpr int kMaxBoxes = 48 * 1024 / (kBoxWords * 4);

// ---- colour + mean: [N,3,H,W] -> workspace [N,3,H,W] ------------------------------------------------------------------------
// convert_rgb_to_hsv / convert_hsv_to_rgb of detectnet_transform_layer.cu:28-117, in float.  The reference's hue test
// `if (h < 0)` compares the pointer, so it never wraps, and hsv_to_rgb sends every sector outside 0..5 to its `default:` (sector 5).
// For h in [-60, 0) that is the right colour; below -60 and at 360 or above it is not.  Here h is brought into [-60, 360) by whole
// turns (fmodf, exact) before the sector is chosen, for any hue_rotation, so on [-60, 360) every bit is the reference's and outside
// it the colour is the wrapped one (what the reference's CPU path, OpenCV's cvtColor, computes).  [-60, 360) rather than [0, 360):
// h in [-60, 0) keeps the reference's own arithmetic (sector -1 taken as 5), which a wrap to [0, 360) would round differently.
__device__ __forceinline__ void colour_pixel(float& r, float& g, float& b, float hue, float sat, bool do_hue, bool do_sat) {
  const float min_v = fminf(fminf(r, g), b), max_v = fmaxf(fmaxf(r, g), b), delta = __fsub_rn(max_v, min_v);
  float h, s, v;
  if (max_v == 0.f || delta == 0.f) {
    h = 0.f; s = 0.f; v = max_v;
  } else {
    if (r == max_v) h = __fdiv_rn(__fsub_rn(g, b), delta);
    else if (g == max_v) h = __fadd_rn(2.f, __fdiv_rn(__fsub_rn(b, r), delta));
    else h = __fadd_rn(4.f, __fdiv_rn(__fsub_rn(r, g), delta));
    h = __fmul_rn(h, 60.f);
    s = __fdiv_rn(delta, max_v);
    v = max_v;
  }
  if (do_hue) h = __fsub_rn(h, hue);
  if (do_sat) s = __fmul_rn(s, sat);
  if (s == 0.f) { r = v; g = v; b = v; return; }
  if (h < -60.f || h >= 360.f) {                // fmodf is exact; for |hue_rotation| <= 300 this is one exact turn
    h = fmodf(h, 360.f);
    if (h < -60.f) h = __fadd_rn(h, 360.f);
  }
  h = __fdiv_rn(h, 60.f);
  const int i = (int)floorf(h);
  const float f = __fsub_rn(h, (float)i);
  const float p = __fmul_rn(v, __fsub_rn(1.f, s));
  const float q = __fmul_rn(v, __fsub_rn(1.f, __fmul_rn(s, f)));
  const float t = __fmul_rn(v, __fsub_rn(1.f, __fmul_rn(s, __fsub_rn(1.f, f))));
  switch (i) {
    case 0: r = v; g = t; b = p; break;
    case 1: r = q; g = v; b = p; break;
    case 2: r = p; g = v; b = t; break;
    case 3: r = p; g = q; b = v; break;
    case 4: r = t; g = p; b = v; break;
    default: r = v; g = p; b = q; break;
  }
}

// mean_kind 0: none; 1: mean_value m0..m2 per channel; 2: per-pixel mean image [3,H,W].
__global__ void __launch_bounds__(kImageThreads) colour_kernel(int N, int H, int W, const float* __restrict__ src,
                                                               const b2c_detectnet_aug* __restrict__ aug, int mean_kind,
                                                               const float* __restrict__ mean, float m0, float m1, float m2,
                                                               float* __restrict__ dst) {
  pdl_wait();
  const size_t plane = (size_t)H * W, total = (size_t)N * plane;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(i / plane);
    const size_t px = i - (size_t)n * plane, base = (size_t)n * 3 * plane + px;
    const b2c_detectnet_aug a = aug[n];
    const bool do_hue = fabsf(a.hue_rotation) > FLT_EPSILON;
    const bool do_sat = (double)a.saturation < (1.0 - 1.0 / 255);
    float r = src[base], g = src[base + plane], b = src[base + 2 * plane];
    if (do_hue || do_sat) colour_pixel(r, g, b, a.hue_rotation, a.saturation, do_hue, do_sat);
    if (mean_kind == 1) {
      r = __fsub_rn(r, m0); g = __fsub_rn(g, m1); b = __fsub_rn(b, m2);
    } else if (mean_kind == 2) {
      r = __fsub_rn(r, mean[px]); g = __fsub_rn(g, mean[px + plane]); b = __fsub_rn(b, mean[px + 2 * plane]);
    }
    dst[base] = r; dst[base + plane] = g; dst[base + 2 * plane] = b;
  }
}

// ---- spatial sampling: workspace [N,3,H,W] -> top [N,3,OH,OW] (detectnet_transform_layer.cu:211-346) -------------------------
__device__ __forceinline__ float get_value(const float* __restrict__ img, int H, int W, int y, int x) {
  if (x == -1) x = 0;
  if (x == W) x = W - 1;
  if (y == -1) y = 0;
  if (y == H) y = H - 1;
  return (x >= 0 && x < W && y >= 0 && y < H) ? img[(size_t)y * W + x] : 0.f;
}

// v2 + d * (-2 v1 - 3 v2 + 6 v3 - v4 + d * (3 v1 - 6 v2 + 3 v3 + 0 v4 + d * (-v1 + 3 v2 - 3 v3 + v4))) / 6.0, in double, rounded
// once to float as the reference's Dtype return does.
__device__ __forceinline__ float cubic(float d_, float v1_, float v2_, float v3_, float v4_) {
  const double d = d_, v1 = v1_, v2 = v2_, v3 = v3_, v4 = v4_;
  double c = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(-1.0, v1), __dmul_rn(3.0, v2)), __dmul_rn(-3.0, v3)), __dmul_rn(1.0, v4));
  double b = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(3.0, v1), __dmul_rn(-6.0, v2)), __dmul_rn(3.0, v3)), __dmul_rn(0.0, v4));
  b = __dadd_rn(b, __dmul_rn(d, c));
  double a = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(-2.0, v1), __dmul_rn(-3.0, v2)), __dmul_rn(6.0, v3)), __dmul_rn(-1.0, v4));
  a = __dadd_rn(a, __dmul_rn(d, b));
  return (float)__dadd_rn(v2, __ddiv_rn(__dmul_rn(d, a), 6.0));
}

__device__ __forceinline__ float interp_x(const float* img, int H, int W, int y, float x) {
  const float fx = floorf(x), cx = ceilf(x);
  return cubic(__fsub_rn(x, fx), get_value(img, H, W, y, (int)(fx - 1.f)), get_value(img, H, W, y, (int)fx),
               get_value(img, H, W, y, (int)cx), get_value(img, H, W, y, (int)(cx + 1.f)));
}

__device__ __forceinline__ float interp_xy(const float* img, int H, int W, float y, float x) {
  const float fy = floorf(y), cy = ceilf(y);
  return cubic(__fsub_rn(y, fy), interp_x(img, H, W, (int)(fy - 1.f), x), interp_x(img, H, W, (int)fy, x),
               interp_x(img, H, W, (int)cy, x), interp_x(img, H, W, (int)(cy + 1.f), x));
}

__global__ void __launch_bounds__(kImageThreads) sample_kernel(int N, int H, int W, int OH, int OW, const float* __restrict__ src,
                                                               const b2c_detectnet_aug* __restrict__ aug, float* __restrict__ dst) {
  pdl_wait();
  const size_t oplane = (size_t)OH * OW, total = (size_t)N * oplane, plane = (size_t)H * W;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(i / oplane);
    const size_t opx = i - (size_t)n * oplane;
    const int oy = (int)(opx / OW), ox = (int)(opx - (size_t)oy * OW);
    const b2c_detectnet_aug a = aug[n];
    float x = __fadd_rn((float)ox, (float)a.crop_x), y = __fadd_rn((float)oy, (float)a.crop_y);
    if (fabsf(a.rotation) > FLT_EPSILON) {
      const float wb = (float)(a.scale_w - 1), hb = (float)(a.scale_h - 1);
      const float angle = __fdiv_rn(__fmul_rn(a.rotation, CUDART_PI_F), 180.f);
      const float ca = cosf(angle), sa = sinf(angle);
      const float wa = __fadd_rn(fabsf(__fmul_rn(wb, ca)), fabsf(__fmul_rn(hb, sa)));
      const float ha = __fadd_rn(fabsf(__fmul_rn(wb, sa)), fabsf(__fmul_rn(hb, ca)));
      const float cxr = __fdiv_rn(wa, 2.f), cyr = __fdiv_rn(ha, 2.f);
      const float s = sinf(-angle), c = cosf(-angle);
      const float tx = __fsub_rn(x, cxr), ty = __fsub_rn(y, cyr);
      x = __fadd_rn(__fsub_rn(__fmul_rn(tx, c), __fmul_rn(ty, s)), cxr);
      y = __fadd_rn(__fadd_rn(__fmul_rn(tx, s), __fmul_rn(ty, c)), cyr);
      x = __fsub_rn(x, __fdiv_rn(__fsub_rn(wa, wb), 2.f));
      y = __fsub_rn(y, __fdiv_rn(__fsub_rn(ha, hb), 2.f));
    }
    if (W != a.scale_w) x = __fmul_rn(x, __fdiv_rn((float)(W - 1), (float)(a.scale_w - 1)));
    if (H != a.scale_h) y = __fmul_rn(y, __fdiv_rn((float)(H - 1), (float)(a.scale_h - 1)));
    if (a.flip) x = (float)__dsub_rn((double)__fsub_rn((float)W, x), 1.0);
    const float* img = src + (size_t)n * 3 * plane;
    float* out = dst + (size_t)n * 3 * oplane + opx;
    for (int ch = 0; ch < 3; ++ch) out[ch * oplane] = interp_xy(img + ch * plane, H, W, y, x);
  }
}

// ---- labels: [N,1,rows,16] -> [N, 8 + classes, GH, GW] ----------------------------------------------------------------------
struct RectF { float x, y, w, h; };

// cv::Rect_<float>::operator&= (OpenCV 2.4 / 3.x): an intersection with no area is the empty rectangle at the origin.
__device__ __forceinline__ RectF rect_and(RectF a, RectF b) {
  const float x1 = fmaxf(a.x, b.x), y1 = fmaxf(a.y, b.y);
  RectF r{x1, y1, __fsub_rn(fminf(__fadd_rn(a.x, a.w), __fadd_rn(b.x, b.w)), x1),
          __fsub_rn(fminf(__fadd_rn(a.y, a.h), __fadd_rn(b.y, b.h)), y1)};
  if (r.w <= 0.f || r.h <= 0.f) r = RectF{0.f, 0.f, 0.f, 0.f};
  return r;
}
__device__ __forceinline__ float rect_area(RectF r) { return __fmul_rn(r.w, r.h); }

// Per box, in shared memory (kBoxWords words): [0..3] the transformed, pruned bbox; [4..7] the coverage rectangle; [8..11] its
// grid cells x0, y0, x1, y1 (int; empty when x0 >= x1); [12] destination class (int, -1: dropped); [13] obj_norm; [14] 1 / width,
// [15] 1 / height (each 1.0 / w in double, rounded to float as the reference's assignment does).
__global__ void __launch_bounds__(kLabelThreads) label_kernel(int rows, int H, int W, const float* __restrict__ labels,
                                                              const b2c_detectnet_aug* __restrict__ aug, b2c_detectnet_gt gt,
                                                              int channels, int GH, int GW, float* __restrict__ top,
                                                              int* __restrict__ status) {
  extern __shared__ float boxes[];
  pdl_wait();
  const int n = blockIdx.x;
  const float* src = labels + (size_t)n * rows * 16;
  float* out = top + (size_t)n * channels * GH * GW;
  const size_t gplane = (size_t)GH * GW;
  const float h0 = src[0], h1 = src[1];
  int err = 0;
  if (!(h1 >= 16.f && h1 < 17.f)) err |= B2C_DETECTNET_BAD_BOX_LENGTH;
  if (!(h0 >= 0.f && h0 < (float)rows)) err |= B2C_DETECTNET_TOO_MANY_BOXES;  // boxes occupy rows 1 .. rows-1
  if (err) {
    if (threadIdx.x == 0) atomicOr(status, err);
    for (size_t i = threadIdx.x; i < (size_t)channels * gplane; i += blockDim.x) out[i] = 0.f;
    return;
  }
  const int nb = (int)h0;
  const b2c_detectnet_aug a = aug[n];
  const float stride = (float)gt.stride, box_area = (float)(gt.stride * gt.stride);
  for (int k = threadIdx.x; k < nb; k += blockDim.x) {
    const float* l = src + 16 * (k + 1);
    float* s = boxes + kBoxWords * k;
    int* si = reinterpret_cast<int*>(s);
    RectF bb{l[0], l[1], l[2], l[3]};
    // transform_label_cpu: flip, scale, rotate, crop (detectnet_transform_layer.cpp:450-615)
    if (a.flip) bb.x = __fsub_rn(__fsub_rn(__fsub_rn((float)W, bb.x), bb.w), 1.f);
    if (a.scale_w != W || a.scale_h != H) {
      const float sx = __fdiv_rn((float)a.scale_w, (float)W), sy = __fdiv_rn((float)a.scale_h, (float)H);
      bb = RectF{__fmul_rn(bb.x, sx), __fmul_rn(bb.y, sy), __fmul_rn(bb.w, sx), __fmul_rn(bb.h, sy)};
    }
    if (fabsf(a.rotation) > FLT_EPSILON) {
      // getTransformationMatrix: rotation by `rotation` degrees about the centre of the scaled image, then the shift that
      // brings the top-left of the rotated rectangle's integer bounding box (cv::RotatedRect::boundingRect) to the origin.
      const double th = (double)a.rotation * CUDART_PI / 180.0;
      const float bh = (float)cos(th) * 0.5f, ah = (float)sin(th) * 0.5f;
      const float ccx = __fmul_rn((float)a.scale_w, 0.5f), ccy = __fmul_rn((float)a.scale_h, 0.5f);
      const float sw = (float)a.scale_w, sh = (float)a.scale_h;
      // cv::RotatedRect::points, each product rounded (no FMA): floorf of these picks the integer corner
      const float ash = __fmul_rn(ah, sh), bsw = __fmul_rn(bh, sw), bsh = __fmul_rn(bh, sh), asw = __fmul_rn(ah, sw);
      const float p0x = __fsub_rn(__fsub_rn(ccx, ash), bsw), p0y = __fsub_rn(__fadd_rn(ccy, bsh), asw);
      const float p1x = __fsub_rn(__fadd_rn(ccx, ash), bsw), p1y = __fsub_rn(__fsub_rn(ccy, bsh), asw);
      const float c2x = __fmul_rn(2.f, ccx), c2y = __fmul_rn(2.f, ccy);
      const float p2x = __fsub_rn(c2x, p0x), p2y = __fsub_rn(c2y, p0y), p3x = __fsub_rn(c2x, p1x), p3y = __fsub_rn(c2y, p1y);
      const float tlx = floorf(fminf(fminf(p0x, p1x), fminf(p2x, p3x))), tly = floorf(fminf(fminf(p0y, p1y), fminf(p2y, p3y)));
      const double c = cos(th), sn = sin(th);
      const double cx = __dmul_rn(0.5, __dadd_rn((double)bb.x, __dadd_rn((double)bb.x, (double)bb.w)));
      const double cy = __dmul_rn(0.5, __dadd_rn((double)bb.y, __dadd_rn((double)bb.y, (double)bb.h)));
      const double dx = __dsub_rn(cx, (double)ccx), dy = __dsub_rn(cy, (double)ccy);
      const double nx = __dsub_rn(__dadd_rn(__dsub_rn(__dmul_rn(c, dx), __dmul_rn(sn, dy)), (double)ccx), (double)tlx);
      const double ny = __dsub_rn(__dadd_rn(__dadd_rn(__dmul_rn(sn, dx), __dmul_rn(c, dy)), (double)ccy), (double)tly);
      bb.x = (float)__dsub_rn(nx, __dmul_rn(0.5, (double)bb.w));
      bb.y = (float)__dsub_rn(ny, __dmul_rn(0.5, (double)bb.h));
    }
    bb.x = __fsub_rn(bb.x, (float)a.crop_x);
    bb.y = __fsub_rn(bb.y, (float)a.crop_y);
    // pruneBboxes (detectnet_coverage_rectangular.cpp:104-137)
    if (gt.crop_bboxes) bb = rect_and(bb, RectF{0.f, 0.f, (float)gt.image_size_x, (float)gt.image_size_y});
    const float cls = l[5];
    int dst = -1;
    if (cls >= 0.f && cls < 4294967296.f) {
      const unsigned key = (unsigned)cls;
      for (int m = 0; m < gt.n_classes; ++m)
        if ((unsigned)gt.class_src[m] == key) dst = gt.class_dst[m];   // later entries win, as std::map assignment does
    }
    if (rect_area(bb) < FLT_EPSILON) dst = -1;
    si[12] = dst;
    if (dst < 0) continue;
    // coverageBoundingBox
    const float ctrx = __fadd_rn(bb.x, __fadd_rn(bb.x, bb.w)) * 0.5f, ctry = __fadd_rn(bb.y, __fadd_rn(bb.y, bb.h)) * 0.5f;
    float shw = __fmul_rn(bb.w, gt.scale_cvg), shh = __fmul_rn(bb.h, gt.scale_cvg);
    if (gt.gridbox_type == 1) {                  // GRIDBOX_MIN
      shw = fminf(bb.w, fmaxf((float)gt.min_cvg_len, shw));
      shh = fminf(bb.h, fmaxf((float)gt.min_cvg_len, shh));
    } else {                                     // GRIDBOX_MAX
      shw = fminf((float)gt.max_cvg_len, shw);
      shh = fminf((float)gt.max_cvg_len, shh);
    }
    const float hw = __fmul_rn(shw, 0.5f), hh = __fmul_rn(shh, 0.5f);
    const float ax = __fadd_rn(ctrx, hw), ay = __fadd_rn(ctry, hh), bx = __fsub_rn(ctrx, hw), by = __fsub_rn(ctry, hh);
    const RectF cov{fminf(ax, bx), fminf(ay, by), __fsub_rn(fmaxf(ax, bx), fminf(ax, bx)), __fsub_rn(fmaxf(ay, by), fminf(ay, by))};
    // imageRectToGridRect, bounded by the grid
    int gx0 = (int)floorf(__fdiv_rn(cov.x, stride)), gy0 = (int)floorf(__fdiv_rn(cov.y, stride));
    int gx1 = (int)ceilf(__fdiv_rn(__fadd_rn(cov.x, cov.w), stride)), gy1 = (int)ceilf(__fdiv_rn(__fadd_rn(cov.y, cov.h), stride));
    gx0 = max(gx0, 0); gy0 = max(gy0, 0); gx1 = min(gx1, GW); gy1 = min(gy1, GH);
    s[0] = bb.x; s[1] = bb.y; s[2] = bb.w; s[3] = bb.h;
    s[4] = cov.x; s[5] = cov.y; s[6] = cov.w; s[7] = cov.h;
    si[8] = gx0; si[9] = gy0; si[10] = gx1; si[11] = gy1;
    const float norm = __fdiv_rn(box_area, rect_area(cov));
    s[13] = fmaxf(gt.obj_norm ? 0.f : 1.f, norm);
    s[14] = (float)(1.0 / (double)bb.w);
    s[15] = (float)(1.0 / (double)bb.h);
  }
  __syncthreads();
  // generate: boxes are written in list order and a later box overwrites every channel of a cell it covers, so each cell takes
  // the last box that covers it by more than FLT_EPSILON of a grid box.
  for (size_t cell = threadIdx.x; cell < gplane; cell += blockDim.x) {
    const int gy = (int)(cell / GW), gx = (int)(cell - (size_t)gy * GW);
    const float gbx = __fmul_rn((float)gx, stride), gby = __fmul_rn((float)gy, stride);
    int last = -1;
    for (int k = 0; k < nb; ++k) {
      const float* s = boxes + kBoxWords * k;
      const int* si = reinterpret_cast<const int*>(s);
      if (si[12] < 0 || gx < si[8] || gx >= si[10] || gy < si[9] || gy >= si[11]) continue;
      const RectF inter = rect_and(RectF{s[4], s[5], s[6], s[7]}, RectF{gbx, gby, stride, stride});
      if (__fdiv_rn(rect_area(inter), box_area) > FLT_EPSILON) last = k;
    }
    float* o = out + cell;
    if (last < 0) {
      for (int ch = 0; ch < channels; ++ch) o[ch * gplane] = 0.f;
      continue;
    }
    const float* s = boxes + kBoxWords * last;
    const int dst = reinterpret_cast<const int*>(s)[12];
    o[0] = 1.f;
    o[1 * gplane] = __fsub_rn(s[0], gbx);
    o[2 * gplane] = __fsub_rn(s[1], gby);
    o[3 * gplane] = __fsub_rn(__fadd_rn(s[0], s[2]), gbx);
    o[4 * gplane] = __fsub_rn(__fadd_rn(s[1], s[3]), gby);
    o[5 * gplane] = s[14];
    o[6 * gplane] = s[15];
    o[7 * gplane] = s[13];
    for (int ch = 8; ch < channels; ++ch) o[ch * gplane] = (ch - 8 == dst) ? 1.f : 0.f;
  }
}

// The class map the kernel uses: the reference's default {1 -> 0} when the parameter lists none.
b2c_detectnet_gt resolved(const b2c_detectnet_gt& g) {
  b2c_detectnet_gt r = g;
  if (r.n_classes == 0) { r.n_classes = 1; r.class_src[0] = 1; r.class_dst[0] = 0; }
  return r;
}

int check_gt(const b2c_detectnet_gt* g) {
  if (!g) return fail(B2C_ERR_INVALID, "detectnet: null ground-truth parameters");
  if (g->stride < 1 || g->image_size_x < 1 || g->image_size_y < 1)
    return fail(B2C_ERR_INVALID, "detectnet: stride %d, image_size %d x %d must be positive", g->stride, g->image_size_x,
                g->image_size_y);
  if (g->n_classes < 0 || g->n_classes > B2C_DETECTNET_MAX_CLASSES)
    return fail(B2C_ERR_INVALID, "detectnet: %d object_class entries (at most %d)", g->n_classes, B2C_DETECTNET_MAX_CLASSES);
  for (int m = 0; m < g->n_classes; ++m)
    if (g->class_src[m] < 0 || g->class_dst[m] < 0 || g->class_dst[m] >= 1024)
      return fail(B2C_ERR_INVALID, "detectnet: object_class { src: %d dst: %d } out of range", g->class_src[m], g->class_dst[m]);
  if (g->gridbox_type != 0 && g->gridbox_type != 1) return fail(B2C_ERR_INVALID, "detectnet: gridbox_type %d", g->gridbox_type);
  return 0;
}

}  // namespace

}  // namespace b2c

using namespace b2c;

extern "C" int b2c_detectnet_label_shape(const b2c_detectnet_gt* gt, int* channels, int* grid_h, int* grid_w) {
  if (int rc = check_gt(gt)) return rc;
  const b2c_detectnet_gt g = resolved(*gt);
  int mx = 0;
  for (int m = 0; m < g.n_classes; ++m) mx = g.class_dst[m] > mx ? g.class_dst[m] : mx;
  // gridROI_: the image rectangle times (float)(1.0 / stride), rounded to int as cv::Size_<float> -> cv::Size rounds
  const float inv = (float)(1.0 / g.stride);
  if (channels) *channels = 8 + mx + 1;
  if (grid_h) *grid_h = (int)rintf((float)g.image_size_y * inv);
  if (grid_w) *grid_w = (int)rintf((float)g.image_size_x * inv);
  return 0;
}

extern "C" size_t b2c_detectnet_image_workspace_bytes(int N, int H, int W) {
  return N > 0 && H > 0 && W > 0 ? (size_t)N * 3 * H * W * sizeof(float) : 0;
}

static int image_args(int N, int H, int W, int OH, int OW, int mean_kind) {
  if (N < 1 || H < 1 || W < 1 || OH < 1 || OW < 1)
    return fail(B2C_ERR_INVALID, "detectnet image: N %d, %d x %d -> %d x %d must be positive", N, H, W, OH, OW);
  if ((size_t)N * 3 * H * W >= (1ull << 40) || (size_t)N * 3 * OH * OW >= (1ull << 40))
    return fail(B2C_ERR_INVALID, "detectnet image: tensor too large");
  if (mean_kind < 0 || mean_kind > 2) return fail(B2C_ERR_INVALID, "detectnet image: mean_kind %d", mean_kind);
  return 0;
}

extern "C" int b2c_detectnet_image(int N, int H, int W, int OH, int OW, const float* bottom, const b2c_detectnet_aug* aug,
                                   int mean_kind, const float* mean_image, const float* mean_value, float* workspace,
                                   size_t workspace_bytes, float* top, void* stream) {
  if (int rc = image_args(N, H, W, OH, OW, mean_kind)) return rc;
  if (!bottom || !aug || !top || !workspace) return fail(B2C_ERR_INVALID, "detectnet image: null pointer");
  if (mean_kind == 1 && !mean_value) return fail(B2C_ERR_INVALID, "detectnet image: mean_kind 1 needs mean_value[3]");
  if (mean_kind == 2 && !mean_image) return fail(B2C_ERR_INVALID, "detectnet image: mean_kind 2 needs a mean image");
  if (workspace_bytes < b2c_detectnet_image_workspace_bytes(N, H, W))
    return fail(B2C_ERR_INVALID, "detectnet image: workspace %zu bytes < %zu", workspace_bytes,
                b2c_detectnet_image_workspace_bytes(N, H, W));
  // The reference keeps mean_values_ = mean_value / 255.f and its GPU path subtracts mean_values_ * 255: the round trip is part
  // of the value subtracted (it changes fractional means), so it is taken here.
  float m[3] = {0.f, 0.f, 0.f};
  if (mean_kind == 1)
    for (int c = 0; c < 3; ++c) m[c] = mean_value[c] / 255.f * 255.f;
  const float m0 = m[0], m1 = m[1], m2 = m[2];
  cudaStream_t st = as_stream(stream);
  launch_pdl(colour_kernel, dim3(grid_for((size_t)N * H * W, kImageThreads)), dim3(kImageThreads), 0, st, 0, N, H, W, bottom, aug,
             mean_kind, mean_image, m0, m1, m2, workspace);
  B2C_POST_LAUNCH();
  launch_pdl(sample_kernel, dim3(grid_for((size_t)N * OH * OW, kImageThreads)), dim3(kImageThreads), 0, st, 0, N, H, W, OH, OW,
             (const float*)workspace, aug, top);
  B2C_POST_LAUNCH();
  return 0;
}

extern "C" int b2c_detectnet_labels(int N, int rows, int H, int W, const float* labels, const b2c_detectnet_aug* aug,
                                    const b2c_detectnet_gt* gt, float* top, int* status, void* stream) {
  if (int rc = check_gt(gt)) return rc;
  if (N < 1 || rows < 1 || H < 1 || W < 1) return fail(B2C_ERR_INVALID, "detectnet labels: N %d, rows %d, %d x %d", N, rows, H, W);
  if (rows - 1 > kMaxBoxes) return fail(B2C_ERR_INVALID, "detectnet labels: %d box rows (at most %d)", rows - 1, kMaxBoxes);
  if (!labels || !aug || !top || !status) return fail(B2C_ERR_INVALID, "detectnet labels: null pointer");
  const b2c_detectnet_gt g = resolved(*gt);
  int channels, gh, gw;
  b2c_detectnet_label_shape(&g, &channels, &gh, &gw);
  if (gh < 1 || gw < 1) return fail(B2C_ERR_INVALID, "detectnet labels: empty %d x %d grid", gh, gw);
  const size_t smem = (size_t)(rows - 1 > 0 ? rows - 1 : 1) * kBoxWords * sizeof(float);
  launch_pdl(label_kernel, dim3(N), dim3(kLabelThreads), smem, as_stream(stream), 0, rows, H, W, labels, aug, g, channels, gh, gw,
             top, status);
  B2C_POST_LAUNCH();
  return 0;
}

extern "C" int b2c_debug_detectnet_plan(int op, int N, int H, int W, int OH, int OW, int rows, const b2c_detectnet_gt* gt, int* out,
                                        int n) {
  if (!out || n < 6) return fail(B2C_ERR_INVALID, "detectnet plan: needs out[6]");
  memset(out, 0, sizeof(int) * n);
  if (op == 0) {
    if (int rc = image_args(N, H, W, OH, OW, 0)) return rc;
    const size_t ws = b2c_detectnet_image_workspace_bytes(N, H, W);
    out[0] = 2;
    out[1] = grid_for((size_t)N * H * W, kImageThreads);
    out[2] = grid_for((size_t)N * OH * OW, kImageThreads);
    out[3] = kImageThreads;
    out[4] = (int)(ws >> 20);
    out[5] = (int)(ws & ((1u << 20) - 1));
    return 0;
  }
  if (op == 1) {
    if (int rc = check_gt(gt)) return rc;
    if (N < 1 || rows < 1) return fail(B2C_ERR_INVALID, "detectnet plan: N %d, rows %d", N, rows);
    if (rows - 1 > kMaxBoxes) return fail(B2C_ERR_INVALID, "detectnet labels: %d box rows (at most %d)", rows - 1, kMaxBoxes);
    int channels, gh, gw;
    b2c_detectnet_label_shape(gt, &channels, &gh, &gw);
    out[0] = N;
    out[1] = kLabelThreads;
    out[2] = (rows - 1 > 0 ? rows - 1 : 1) * kBoxWords * (int)sizeof(float);
    out[3] = channels;
    out[4] = gh;
    out[5] = gw;
    return 0;
  }
  return fail(B2C_ERR_INVALID, "detectnet plan: op %d (0 image, 1 labels)", op);
}
