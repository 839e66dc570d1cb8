// im2col.cu -- im2col / col2im (2-D and N-D) for sm_90a.
//
// Replaces im2col_gpu / col2im_gpu / im2col_nd_gpu / col2im_nd_gpu
// (reference src/caffe/util/im2col.cu:42-62,298-317,165-253,443-530).  These are pure
// HBM-bound copies with integer index math: the col side is kh*kw times larger than the
// image, so the kernels are organised around the col side -- one thread per col element
// for im2col (fully coalesced 4-byte stores along wo, grid.y = col row so no division by
// Ho*Wo), one thread per image element for col2im (gather, no atomics).
//
// col2im adds the contributions to a pixel in ascending (i,j) kernel-offset order starting
// from 0, which is exactly the order the reference CPU col2im_cpu (im2col.cpp:176-211)
// produces them in, so the result is bit-identical to the CPU path.
#include "b2c_common.cuh"

namespace b2c {

__global__ void __launch_bounds__(256)
im2col2d_kernel(const float* __restrict__ im, int H, int W, int kh, int kw, int ph, int pw,
                int sh, int sw, int dh, int dw, int Ho, int Wo, int row0, float* __restrict__ col) {
  const int row = row0 + blockIdx.y;          // (c*kh + i)*kw + j
  const int j = row % kw, i = (row / kw) % kh, c = row / (kw * kh);
  const int P = Ho * Wo;
  const float* src = im + (size_t)c * H * W;
  float* dst = col + (size_t)row * P;
  const int h_off = i * dh - ph, w_off = j * dw - pw;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < P; p += gridDim.x * blockDim.x) {
    const int ho = p / Wo, wo = p - ho * Wo;
    const int h = ho * sh + h_off, w = wo * sw + w_off;
    const bool in = (unsigned)h < (unsigned)H && (unsigned)w < (unsigned)W;
    dst[p] = in ? __ldg(src + (size_t)h * W + w) : 0.0f;
  }
}

__global__ void __launch_bounds__(256)
col2im2d_kernel(const float* __restrict__ col, int C, int H, int W, int kh, int kw, int ph, int pw,
                int sh, int sw, int dh, int dw, int Ho, int Wo, float* __restrict__ im) {
  const size_t total = (size_t)C * H * W;
  const int P = Ho * Wo;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x) {
    const int w = (int)(idx % W), h = (int)((idx / W) % H), c = (int)(idx / ((size_t)W * H));
    float acc = 0.0f;
    for (int i = 0; i < kh; ++i) {
      const int hh = h + ph - i * dh;
      if (hh < 0 || hh % sh) continue;
      const int ho = hh / sh;
      if (ho >= Ho) continue;
      for (int j = 0; j < kw; ++j) {
        const int ww = w + pw - j * dw;
        if (ww < 0 || ww % sw) continue;
        const int wo = ww / sw;
        if (wo >= Wo) continue;
        acc += __ldg(col + ((size_t)(c * kh + i) * kw + j) * P + (size_t)ho * Wo + wo);
      }
    }
    im[idx] = acc;
  }
}

struct NdShape {
  int nax;
  int im[11];    // [C, d0..]
  int col[11];   // [C*prod(k), o0..]
  int k[10], pad[10], stride[10], dil[10];
};

__global__ void __launch_bounds__(256)
im2col_nd_kernel(const float* __restrict__ im, NdShape s, size_t total, float* __restrict__ col) {
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x) {
    size_t t = idx;
    int opos[10];
    for (int a = s.nax - 1; a >= 0; --a) { opos[a] = (int)(t % s.col[1 + a]); t /= s.col[1 + a]; }
    int cc = (int)t;                 // col channel = c_im*prod(k) + flat kernel offset
    int koff[10];
    for (int a = s.nax - 1; a >= 0; --a) { koff[a] = cc % s.k[a]; cc /= s.k[a]; }
    size_t src = (size_t)cc;         // c_im
    bool padded = false;
    for (int a = 0; a < s.nax; ++a) {
      const int d = opos[a] * s.stride[a] - s.pad[a] + koff[a] * s.dil[a];
      padded |= (d < 0) || (d >= s.im[1 + a]);
      src = src * s.im[1 + a] + (size_t)d;
    }
    col[idx] = padded ? 0.0f : __ldg(im + src);
  }
}

__global__ void __launch_bounds__(256)
col2im_nd_kernel(const float* __restrict__ col, NdShape s, size_t total, int ksize, size_t out_sp,
                 float* __restrict__ im) {
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x) {
    size_t t = idx;
    int ipos[10];
    for (int a = s.nax - 1; a >= 0; --a) { ipos[a] = (int)(t % s.im[1 + a]); t /= s.im[1 + a]; }
    const int c_im = (int)t;
    float acc = 0.0f;
    for (int kf = 0; kf < ksize; ++kf) {          // ascending flat kernel offset == CPU order
      int r = kf;
      size_t sp = 0;
      bool ok = true;
      int koff[10];
      for (int a = s.nax - 1; a >= 0; --a) { koff[a] = r % s.k[a]; r /= s.k[a]; }
      for (int a = 0; a < s.nax && ok; ++a) {
        const int d = ipos[a] + s.pad[a] - koff[a] * s.dil[a];
        if (d < 0 || d % s.stride[a]) { ok = false; break; }
        const int o = d / s.stride[a];
        if (o >= s.col[1 + a]) { ok = false; break; }
        sp = sp * s.col[1 + a] + (size_t)o;
      }
      if (ok) acc += __ldg(col + ((size_t)c_im * ksize + kf) * out_sp + sp);
    }
    im[idx] = acc;
  }
}

int launch_im2col2d(const float* im, int C, int H, int W, int kh, int kw, int ph, int pw, int sh, int sw,
                    int dh, int dw, float* col, cudaStream_t st) {
  const int Ho = (H + 2 * ph - (dh * (kh - 1) + 1)) / sh + 1;
  const int Wo = (W + 2 * pw - (dw * (kw - 1) + 1)) / sw + 1;
  if (Ho <= 0 || Wo <= 0 || C <= 0) return fail(B2C_ERR_INVALID, "im2col: empty output");
  const int P = Ho * Wo, rows = C * kh * kw;
  int gx = (P + 255) / 256;
  if (gx > 64) gx = 64;
  for (int r0 = 0; r0 < rows; r0 += 65535) {   // grid.y limit
    const int nr = rows - r0 < 65535 ? rows - r0 : 65535;
    im2col2d_kernel<<<dim3(gx, nr), 256, 0, st>>>(im, H, W, kh, kw, ph, pw, sh, sw, dh, dw, Ho, Wo, r0, col);
    B2C_POST_LAUNCH();
  }
  return B2C_OK;
}

int launch_col2im2d(const float* col, int C, int H, int W, int kh, int kw, int ph, int pw, int sh, int sw,
                    int dh, int dw, float* im, cudaStream_t st) {
  const int Ho = (H + 2 * ph - (dh * (kh - 1) + 1)) / sh + 1;
  const int Wo = (W + 2 * pw - (dw * (kw - 1) + 1)) / sw + 1;
  if (Ho <= 0 || Wo <= 0 || C <= 0) return fail(B2C_ERR_INVALID, "col2im: empty output");
  const size_t total = (size_t)C * H * W;
  col2im2d_kernel<<<grid_for(total, 256), 256, 0, st>>>(col, C, H, W, kh, kw, ph, pw, sh, sw, dh, dw, Ho, Wo, im);
  B2C_POST_LAUNCH();
  return B2C_OK;
}

static int fill_nd(NdShape& s, int nax, const int* im_shape, const int* col_shape, const int* k, const int* pad,
                   const int* stride, const int* dil) {
  if (nax < 1 || nax > 10) return fail(B2C_ERR_INVALID, "nd im2col: num_axes %d not in [1,10]", nax);
  s.nax = nax;
  for (int a = 0; a <= nax; ++a) { s.im[a] = im_shape[a]; s.col[a] = col_shape[a]; }
  for (int a = 0; a < nax; ++a) {
    s.k[a] = k[a]; s.pad[a] = pad[a]; s.stride[a] = stride[a]; s.dil[a] = dil[a];
    if (k[a] <= 0 || stride[a] <= 0 || dil[a] <= 0 || col_shape[1 + a] <= 0)
      return fail(B2C_ERR_INVALID, "nd im2col: bad axis %d", a);
  }
  return B2C_OK;
}

}  // namespace b2c

using namespace b2c;

extern "C" int b2c_im2col(const float* im, int C, int H, int W, int kh, int kw, int ph, int pw, int sh, int sw,
                          int dh, int dw, float* col, void* stream) {
  if (!im || !col || kh <= 0 || kw <= 0 || sh <= 0 || sw <= 0 || dh <= 0 || dw <= 0)
    return fail(B2C_ERR_INVALID, "b2c_im2col: bad argument");
  return launch_im2col2d(im, C, H, W, kh, kw, ph, pw, sh, sw, dh, dw, col, as_stream(stream));
}

extern "C" int b2c_col2im(const float* col, int C, int H, int W, int kh, int kw, int ph, int pw, int sh, int sw,
                          int dh, int dw, float* im, void* stream) {
  if (!im || !col || kh <= 0 || kw <= 0 || sh <= 0 || sw <= 0 || dh <= 0 || dw <= 0)
    return fail(B2C_ERR_INVALID, "b2c_col2im: bad argument");
  return launch_col2im2d(col, C, H, W, kh, kw, ph, pw, sh, sw, dh, dw, im, as_stream(stream));
}

extern "C" int b2c_im2col_nd(const float* im, int nax, const int* im_shape, const int* col_shape, const int* k,
                             const int* pad, const int* stride, const int* dil, float* col, void* stream) {
  NdShape s;
  if (int rc = fill_nd(s, nax, im_shape, col_shape, k, pad, stride, dil)) return rc;
  size_t total = 1;
  for (int a = 0; a <= nax; ++a) total *= (size_t)col_shape[a];
  im2col_nd_kernel<<<grid_for(total, 256), 256, 0, as_stream(stream)>>>(im, s, total, col);
  B2C_POST_LAUNCH();
  return B2C_OK;
}

extern "C" int b2c_col2im_nd(const float* col, int nax, const int* im_shape, const int* col_shape, const int* k,
                             const int* pad, const int* stride, const int* dil, float* im, void* stream) {
  NdShape s;
  if (int rc = fill_nd(s, nax, im_shape, col_shape, k, pad, stride, dil)) return rc;
  size_t total = 1, out_sp = 1;
  int ksize = 1;
  for (int a = 0; a <= nax; ++a) total *= (size_t)im_shape[a];
  for (int a = 0; a < nax; ++a) { out_sp *= (size_t)col_shape[1 + a]; ksize *= k[a]; }
  col2im_nd_kernel<<<grid_for(total, 256), 256, 0, as_stream(stream)>>>(col, s, total, ksize, out_sp, im);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
