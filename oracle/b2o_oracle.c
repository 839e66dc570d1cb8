/*
 * b2o_oracle.c -- CPU ORACLE.  TEST INFRASTRUCTURE ONLY.
 *
 * A plain-C restatement of the reference's CPU algorithm for the data-parallel
 * conv + gradient-allreduce + SGD hot path.  It is the parity checker for the
 * CUDA kernels under caffe_mpi_b200/csrc.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it.  Nothing in
 * the product path calls into this file.
 *
 * Parity status: PINNED.  The functions below are checked in tests/ against
 *   - the reference's own known-answer vectors (test_util_blas.cpp:19-175 integer
 *     GEMM/GEMV, test_convolution_layer.cpp:511-604 Sobel, test_im2col_layer.cpp:63-77),
 *   - oracle/_ref (the reference's src/caffe/util/im2col.cpp compiled verbatim),
 *   - fixtures under tests/golden/ produced from oracle/_ref.
 *
 * Citations are relative to /root/reference.  All tensors fp32, dense row-major,
 * activations NCHW, weights [O, C/g, kh, kw].
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  int N, C, H, W;   /* bottom shape                                  */
  int O, G;         /* num_output, group                             */
  int kh, kw, sh, sw, ph, pw, dh, dw;
  int has_bias;
} b2o_conv_params;

/* conv_layer.cpp:7-22: truncating integer division for the output extent. */
static int out_extent(int in, int k, int s, int p, int d) {
  const int ext = d * (k - 1) + 1;
  return (in + 2 * p - ext) / s + 1;
}
int b2o_out_h(const b2o_conv_params* p) { return out_extent(p->H, p->kh, p->sh, p->ph, p->dh); }
int b2o_out_w(const b2o_conv_params* p) { return out_extent(p->W, p->kw, p->sw, p->pw, p->dw); }

/* ------------------------------------------------------------------------- *
 * im2col / col2im, 2-D.  Follows src/caffe/util/im2col.cpp:18-55 (im2col_cpu)
 * and :176-211 (col2im_cpu).  Written from the index formula
 *   col[(c*kh+i)*kw+j][ho][wo] = im[c][ho*sh-ph+i*dh][wo*sw-pw+j*dw]  (0 outside)
 * col2im zero-fills then accumulates in (c,i,j,ho,wo) order, which fixes the
 * fp32 summation order per input pixel: ascending (i,j).
 * ------------------------------------------------------------------------- */
void b2o_im2col(const float* im, int C, int H, int W, int kh, int kw,
                int ph, int pw, int sh, int sw, int dh, int dw, float* col) {
  const int Ho = out_extent(H, kh, sh, ph, dh), Wo = out_extent(W, kw, sw, pw, dw);
  size_t q = 0;
  for (int c = 0; c < C; ++c)
    for (int i = 0; i < kh; ++i)
      for (int j = 0; j < kw; ++j)
        for (int ho = 0; ho < Ho; ++ho) {
          const int h = ho * sh - ph + i * dh;
          for (int wo = 0; wo < Wo; ++wo, ++q) {
            const int w = wo * sw - pw + j * dw;
            const int inside = (h >= 0) & (h < H) & (w >= 0) & (w < W);
            col[q] = inside ? im[((size_t)c * H + h) * W + w] : 0.0f;
          }
        }
}

void b2o_col2im(const float* col, int C, int H, int W, int kh, int kw,
                int ph, int pw, int sh, int sw, int dh, int dw, float* im) {
  const int Ho = out_extent(H, kh, sh, ph, dh), Wo = out_extent(W, kw, sw, pw, dw);
  memset(im, 0, sizeof(float) * (size_t)C * H * W);
  size_t q = 0;
  for (int c = 0; c < C; ++c)
    for (int i = 0; i < kh; ++i)
      for (int j = 0; j < kw; ++j)
        for (int ho = 0; ho < Ho; ++ho) {
          const int h = ho * sh - ph + i * dh;
          for (int wo = 0; wo < Wo; ++wo, ++q) {
            const int w = wo * sw - pw + j * dw;
            if (h >= 0 && h < H && w >= 0 && w < W)
              im[((size_t)c * H + h) * W + w] += col[q];
          }
        }
}

/* ------------------------------------------------------------------------- *
 * N-D im2col / col2im (1..10 spatial axes), im2col.cpp:76-174,231-258.
 * shapes: im_shape = [C, d0, d1, ...], col_shape = [C*prod(k), o0, o1, ...].
 * Restated with a flat decode of the column index instead of the reference's
 * odometer; the visiting order (and therefore the col2im summation order per
 * image element) is identical: ascending flat column index.
 * ------------------------------------------------------------------------- */
static void nd_core(const float* in, int to_col, int nax, const int* im_shape,
                    const int* col_shape, const int* k, const int* pad,
                    const int* stride, const int* dil, float* out) {
  size_t im_size = im_shape[0], out_sp = 1;
  int ksize = 1;
  for (int a = 0; a < nax; ++a) { im_size *= im_shape[1 + a]; out_sp *= col_shape[1 + a]; ksize *= k[a]; }
  if (!to_col) memset(out, 0, sizeof(float) * im_size);
  const int ccol = col_shape[0];
  int koff[10], opos[10];
  for (int cc = 0; cc < ccol; ++cc) {
    int r = cc;
    for (int a = nax - 1; a >= 0; --a) { koff[a] = r % k[a]; r /= k[a]; }
    const int c_im = cc / ksize;
    for (size_t s = 0; s < out_sp; ++s) {
      size_t t = s;
      for (int a = nax - 1; a >= 0; --a) { opos[a] = (int)(t % col_shape[1 + a]); t /= col_shape[1 + a]; }
      size_t idx_im = c_im;
      int padded = 0;
      for (int a = 0; a < nax; ++a) {
        const int d_im = opos[a] * stride[a] - pad[a] + koff[a] * dil[a];
        padded |= (d_im < 0) || (d_im >= im_shape[1 + a]);
        idx_im = idx_im * im_shape[1 + a] + (size_t)d_im;
      }
      const size_t idx_col = (size_t)cc * out_sp + s;
      if (to_col) out[idx_col] = padded ? 0.0f : in[idx_im];
      else if (!padded) out[idx_im] += in[idx_col];
    }
  }
}
void b2o_im2col_nd(const float* im, int nax, const int* im_shape, const int* col_shape,
                   const int* k, const int* pad, const int* stride, const int* dil, float* col) {
  nd_core(im, 1, nax, im_shape, col_shape, k, pad, stride, dil, col);
}
void b2o_col2im_nd(const float* col, int nax, const int* im_shape, const int* col_shape,
                   const int* k, const int* pad, const int* stride, const int* dil, float* im) {
  nd_core(col, 0, nax, im_shape, col_shape, k, pad, stride, dil, im);
}

/* ------------------------------------------------------------------------- *
 * GEMM / GEMV with the reference's argument conventions,
 * src/caffe/util/math_functions.cpp:14-23 (caffe_cpu_gemm -> cblas_sgemm RowMajor,
 * lda = transA ? M : K, ldb = transB ? K : N, ldc = N) and :57-62 (gemv).
 * The arithmetic itself lives in OpenBLAS (not under /root/reference, unpinned:
 * Makefile.config:49 "BLAS := open"); restated as the textbook sum over k in
 * ascending order.  acc64 != 0 accumulates in double (a tighter yardstick that
 * does not depend on any BLAS's summation order).
 * ------------------------------------------------------------------------- */
void b2o_gemm(int transA, int transB, int M, int N, int K, float alpha,
              const float* A, const float* B, float beta, float* C, int acc64) {
  const int lda = transA ? M : K, ldb = transB ? K : N;
  if (!acc64 && !transB) {
    /* i-k-j order: same per-element ascending-k order, but vectorisable */
    float* row = (float*)malloc(sizeof(float) * (size_t)N);
    for (int i = 0; i < M; ++i) {
      for (int j = 0; j < N; ++j) row[j] = 0.0f;
      for (int k = 0; k < K; ++k) {
        const float a = transA ? A[(size_t)k * lda + i] : A[(size_t)i * lda + k];
        const float* b = B + (size_t)k * ldb;
        for (int j = 0; j < N; ++j) row[j] += a * b[j];
      }
      float* c = C + (size_t)i * N;
      if (beta == 0.0f) for (int j = 0; j < N; ++j) c[j] = alpha * row[j];
      else for (int j = 0; j < N; ++j) c[j] = alpha * row[j] + beta * c[j];
    }
    free(row);
    return;
  }
  for (int i = 0; i < M; ++i)
    for (int j = 0; j < N; ++j) {
      double sd = 0.0; float sf = 0.0f;
      for (int k = 0; k < K; ++k) {
        const float a = transA ? A[(size_t)k * lda + i] : A[(size_t)i * lda + k];
        const float b = transB ? B[(size_t)j * ldb + k] : B[(size_t)k * ldb + j];
        if (acc64) sd += (double)a * (double)b; else sf += a * b;
      }
      float* c = C + (size_t)i * N + j;
      if (acc64) *c = (float)((double)alpha * sd + (beta == 0.0f ? 0.0 : (double)beta * (double)*c));
      else *c = (beta == 0.0f) ? alpha * sf : alpha * sf + beta * *c;
    }
}

/* y = alpha*op(A)*x + beta*y, A is M x N row-major (math_functions.cpp:57-62). */
void b2o_gemv(int transA, int M, int N, float alpha, const float* A,
              const float* x, float beta, float* y, int acc64) {
  const int leny = transA ? N : M, lenx = transA ? M : N;
  for (int i = 0; i < leny; ++i) {
    double sd = 0.0; float sf = 0.0f;
    for (int k = 0; k < lenx; ++k) {
      const float a = transA ? A[(size_t)k * N + i] : A[(size_t)i * N + k];
      if (acc64) sd += (double)a * (double)x[k]; else sf += a * x[k];
    }
    const float s = acc64 ? (float)((double)alpha * sd) : alpha * sf;
    y[i] = (beta == 0.0f) ? s : s + beta * y[i];
  }
}

/* ------------------------------------------------------------------------- *
 * Bit-exact emulators of the product's FFMA GEMM / GEMV kernels
 * (caffe_mpi_b200/csrc/sgemm_simt.cu), so a test can compare them bit for bit:
 *   sgemm_simt_kernel: acc = fmaf(a_k, b_k, acc) for k = 0 .. 16*ceil(K/16) - 1,
 *     starting from +0, with a_k = b_k = 0 past K (the zero-padded tail of the
 *     last 16-wide K tile, which turns an acc of -0 into +0);
 *   sgemv_n_kernel: lane l of a warp runs the chain over k = l, l + 32, ... < N,
 *     then s += shfl_xor(s, o) for o = 16, 8, 4, 2, 1; lane 0's value is kept;
 *   sgemv_t_kernel: one chain over the rows r = 0 .. M - 1.
 * Then the store: beta == 0 gives fl(alpha * acc).  Otherwise the compiler may
 * contract alpha * acc + beta * c either way, so out[0..2] receive the three
 * admissible results fl(fl(a*acc) + fl(b*c)), fma(a, acc, fl(b*c)) and
 * fma(b, c, fl(a*acc)) (identical when beta == 0).  out: 3 planes of M x N
 * (GEMM) or of the length of y (GEMV).  C / y: the values before the call.
 * ------------------------------------------------------------------------- */
static void ffma_store(float alpha, float acc, float beta, float c, float* out, size_t plane, size_t idx) {
  if (beta == 0.0f) {
    const float v = alpha * acc;
    out[idx] = out[plane + idx] = out[2 * plane + idx] = v;
    return;
  }
  const float ta = alpha * acc, tb = beta * c;
  out[idx] = ta + tb;
  out[plane + idx] = fmaf(alpha, acc, tb);
  out[2 * plane + idx] = fmaf(beta, c, ta);
}
void b2o_gemm_ffma(int transA, int transB, int M, int N, int K, float alpha, const float* A, const float* B, float beta,
                   const float* C, float* out) {
  const int lda = transA ? M : K, ldb = transB ? K : N;
  const int kpad = (K + 15) / 16 * 16;
  const size_t plane = (size_t)M * N;
  /* op(B) as K x N rows so the j loop runs over contiguous memory; each element keeps its own sequential chain over k */
  float* bt = (float*)malloc(sizeof(float) * ((size_t)K * N + 1));
  float* acc = (float*)malloc(sizeof(float) * ((size_t)N + 1));
  for (int k = 0; k < K; ++k)
    for (int j = 0; j < N; ++j) bt[(size_t)k * N + j] = transB ? B[(size_t)j * ldb + k] : B[(size_t)k * ldb + j];
  for (int i = 0; i < M; ++i) {
    for (int j = 0; j < N; ++j) acc[j] = 0.0f;
    for (int k = 0; k < K; ++k) {
      const float a = transA ? A[(size_t)k * lda + i] : A[(size_t)i * lda + k];
      const float* b = bt + (size_t)k * N;
      for (int j = 0; j < N; ++j) acc[j] = fmaf(a, b[j], acc[j]);
    }
    for (int k = K; k < kpad; ++k)
      for (int j = 0; j < N; ++j) acc[j] = fmaf(0.0f, 0.0f, acc[j]);
    for (int j = 0; j < N; ++j) ffma_store(alpha, acc[j], beta, C[(size_t)i * N + j], out, plane, (size_t)i * N + j);
  }
  free(bt);
  free(acc);
}
void b2o_gemv_ffma(int transA, int M, int N, float alpha, const float* A, const float* x, float beta, const float* y,
                   float* out) {
  if (!transA) {
    for (int r = 0; r < M; ++r) {
      float s[32], t[32];
      for (int l = 0; l < 32; ++l) {
        s[l] = 0.0f;
        for (int k = l; k < N; k += 32) s[l] = fmaf(A[(size_t)r * N + k], x[k], s[l]);
      }
      for (int o = 16; o; o >>= 1) {
        for (int l = 0; l < 32; ++l) t[l] = s[l] + s[l ^ o];
        for (int l = 0; l < 32; ++l) s[l] = t[l];
      }
      ffma_store(alpha, s[0], beta, y[r], out, (size_t)M, (size_t)r);
    }
  } else {
    for (int c = 0; c < N; ++c) {
      float s = 0.0f;
      for (int r = 0; r < M; ++r) s = fmaf(A[(size_t)r * N + c], x[r], s);
      ffma_store(alpha, s, beta, y[c], out, (size_t)N, (size_t)c);
    }
  }
}

/* ------------------------------------------------------------------------- *
 * Bit-exact restatements of the product's FFMA direct-convolution kernels
 * (caffe_mpi_b200/csrc/conv_simt.cu), so a test can compare them bit for bit.
 * Each output element is one fmaf chain starting from +0; a tap that falls in
 * the padding (or, for the data gradient, off the stride grid) is skipped, not
 * multiplied by 0, so no chain ever sees a padded zero.
 * ------------------------------------------------------------------------- */
/* conv_fwd_simt_kernel: per y[n][o][ho][wo]
 *   acc = fmaf(x, w, acc) over c (0 .. Cg-1), then i, then j     (:27-35)
 *   skipping (unsigned)h >= H (:30) and (unsigned)ww >= W (:33);
 *   then one acc += bias[o] (:37), the bias never inside the chain. */
void b2o_conv_fwd_ffma(const b2o_conv_params* p, const float* x, const float* w, const float* bias, float* y) {
  const int Ho = b2o_out_h(p), Wo = b2o_out_w(p);
  const int Cg = p->C / p->G, Og = p->O / p->G, Kd = Cg * p->kh * p->kw;
  size_t idx = 0;
  for (int n = 0; n < p->N; ++n)
    for (int o = 0; o < p->O; ++o) {
      const float* xg = x + ((size_t)n * p->C + (size_t)(o / Og) * Cg) * p->H * p->W;
      const float* wr = w + (size_t)o * Kd;
      for (int ho = 0; ho < Ho; ++ho)
        for (int wo = 0; wo < Wo; ++wo, ++idx) {
          float acc = 0.0f;
          for (int c = 0; c < Cg; ++c)
            for (int i = 0; i < p->kh; ++i) {
              const int h = ho * p->sh - p->ph + i * p->dh;
              if (h < 0 || h >= p->H) continue;
              for (int j = 0; j < p->kw; ++j) {
                const int ww = wo * p->sw - p->pw + j * p->dw;
                if (ww < 0 || ww >= p->W) continue;
                acc = fmaf(xg[((size_t)c * p->H + h) * p->W + ww], wr[(c * p->kh + i) * p->kw + j], acc);
              }
            }
          if (p->has_bias && bias) acc += bias[o];
          y[idx] = acc;
        }
    }
}

/* conv_dgrad_simt_kernel: per dx[n][c][h][w], g = c / Cg, cg = c % Cg
 *   for i: hh = h + ph - i*dh; skip hh < 0 or hh % sh != 0; ho = hh / sh; skip ho >= Ho   (:53-57)
 *     for j: the same for w                                                               (:58-62)
 *       for o in the group (0 .. Og-1): acc = fmaf(dy[n][g*Og+o][ho][wo], w[g*Og+o][cg][i][j], acc)   (:65-66)
 *   then dx = acc, overwritten (:69). */
void b2o_conv_dgrad_ffma(const b2o_conv_params* p, const float* dy, const float* w, float* dx) {
  const int Ho = b2o_out_h(p), Wo = b2o_out_w(p);
  const int Cg = p->C / p->G, Og = p->O / p->G, Kd = Cg * p->kh * p->kw;
  size_t idx = 0;
  for (int n = 0; n < p->N; ++n)
    for (int c = 0; c < p->C; ++c) {
      const int g = c / Cg, cg = c - g * Cg;
      for (int h = 0; h < p->H; ++h)
        for (int ww = 0; ww < p->W; ++ww, ++idx) {
          float acc = 0.0f;
          for (int i = 0; i < p->kh; ++i) {
            const int hh = h + p->ph - i * p->dh;
            if (hh < 0 || hh % p->sh) continue;
            const int ho = hh / p->sh;
            if (ho >= Ho) continue;
            for (int j = 0; j < p->kw; ++j) {
              const int wv = ww + p->pw - j * p->dw;
              if (wv < 0 || wv % p->sw) continue;
              const int wo = wv / p->sw;
              if (wo >= Wo) continue;
              const float* dyp = dy + (((size_t)n * p->O + (size_t)g * Og) * Ho + ho) * Wo + wo;
              const float* wp = w + (((size_t)g * Og * Cg + cg) * p->kh + i) * p->kw + j;
              for (int o = 0; o < Og; ++o) acc = fmaf(dyp[(size_t)o * Ho * Wo], wp[(size_t)o * Kd], acc);
            }
          }
          dx[idx] = acc;
        }
    }
}

/* conv_wgrad_simt_kernel: one block of 256 threads per (o, cg); per tap (i, j)   (:82-83)
 *   thread t: acc = fmaf(dy[n][o][p], x[n][g*Cg+cg][h][w], acc) for q = t, t + 256, ... < N*Ho*Wo,
 *     n = q / P, p = q % P, skipping taps in the padding                          (:85-92)
 *   each warp: acc += shfl_xor(acc, off) for off = 16, 8, 4, 2, 1; lane 0 stores  (:94-95)
 *   thread 0: t = 0; t += red[k] for the 8 warps in order                         (:98-99)
 *   dw += t, once, onto what dw held (accumulated, :100). */
void b2o_conv_wgrad_ffma(const b2o_conv_params* p, const float* x, const float* dy, float* dw) {
  const int Ho = b2o_out_h(p), Wo = b2o_out_w(p), P = Ho * Wo;
  const int Cg = p->C / p->G, Og = p->O / p->G;
  const size_t Q = (size_t)p->N * P;
  float part[256], t[32];
  for (int o = 0; o < p->O; ++o)
    for (int cg = 0; cg < Cg; ++cg) {
      const int c = (o / Og) * Cg + cg;
      for (int i = 0; i < p->kh; ++i)
        for (int j = 0; j < p->kw; ++j) {
          for (int th = 0; th < 256; ++th) {
            float acc = 0.0f;
            for (size_t q = (size_t)th; q < Q; q += 256) {
              const int n = (int)(q / P), pp = (int)(q - (size_t)n * P);
              const int ho = pp / Wo, wo = pp - ho * Wo;
              const int h = ho * p->sh - p->ph + i * p->dh, ww = wo * p->sw - p->pw + j * p->dw;
              if (h < 0 || h >= p->H || ww < 0 || ww >= p->W) continue;
              acc = fmaf(dy[((size_t)n * p->O + o) * P + pp], x[(((size_t)n * p->C + c) * p->H + h) * p->W + ww], acc);
            }
            part[th] = acc;
          }
          float tot = 0.0f;
          for (int wp = 0; wp < 8; ++wp) {
            float* s = part + 32 * wp;
            for (int off = 16; off; off >>= 1) {
              for (int l = 0; l < 32; ++l) t[l] = s[l] + s[l ^ off];
              for (int l = 0; l < 32; ++l) s[l] = t[l];
            }
            tot += s[0];
          }
          float* d = dw + (((size_t)o * Cg + cg) * p->kh + i) * p->kw + j;
          *d += tot;
        }
    }
}

/* ------------------------------------------------------------------------- *
 * ConvolutionLayer::Forward_cpu (src/caffe/layers/conv_layer.cpp:24-40) with
 * forward_cpu_gemm / forward_cpu_bias (include/caffe/layers/base_conv_layer.hpp:36-60).
 * Per image: col = im2col(x_n) unless is_1x1_ (base_conv_layer.cpp:99-103),
 * per group y_{n,g} = W_g * col_g (beta=0), then y_n += bias * ones (rank-1 gemm).
 * ------------------------------------------------------------------------- */
static int is_1x1(const b2o_conv_params* p) {
  return p->kh == 1 && p->kw == 1 && p->sh == 1 && p->sw == 1 && p->ph == 0 && p->pw == 0;
}

void b2o_conv_forward(const b2o_conv_params* p, const float* x, const float* w,
                      const float* bias, float* y, int acc64) {
  const int Ho = b2o_out_h(p), Wo = b2o_out_w(p), P = Ho * Wo;
  const int Cg = p->C / p->G, Og = p->O / p->G, Kd = Cg * p->kh * p->kw;
  const size_t bottom_dim = (size_t)p->C * p->H * p->W, top_dim = (size_t)p->O * P;
  const size_t col_off = (size_t)Kd * P, out_off = (size_t)Og * P, w_off = (size_t)Og * Kd;
  float* col = is_1x1(p) ? NULL : (float*)malloc(sizeof(float) * (size_t)Kd * p->G * P);
  float* ones = (float*)malloc(sizeof(float) * (size_t)P);
  for (int i = 0; i < P; ++i) ones[i] = 1.0f;
  for (int n = 0; n < p->N; ++n) {
    const float* xn = x + n * bottom_dim;
    float* yn = y + n * top_dim;
    const float* cb = xn;
    if (col) { b2o_im2col(xn, p->C, p->H, p->W, p->kh, p->kw, p->ph, p->pw, p->sh, p->sw, p->dh, p->dw, col); cb = col; }
    for (int g = 0; g < p->G; ++g)
      b2o_gemm(0, 0, Og, P, Kd, 1.0f, w + w_off * g, cb + col_off * g, 0.0f, yn + out_off * g, acc64);
    if (p->has_bias && bias) b2o_gemm(0, 0, p->O, P, 1, 1.0f, bias, ones, 1.0f, yn, acc64);
  }
  free(ones);
  free(col);
}

/* ------------------------------------------------------------------------- *
 * ConvolutionLayer::Backward_cpu (conv_layer.cpp:42-73) with
 * backward_cpu_bias (base_conv_layer.hpp:96-100, gemv beta=1),
 * weight_cpu_gemm (:80-94, dW_g += dY_{n,g} * col_g^T, beta=1) and
 * backward_cpu_gemm (:62-78, col_g = W_g^T * dY_{n,g}, beta=0, then col2im).
 * dw/db are ACCUMULATED into; dx is OVERWRITTEN.  Null dw/db/dx skips that leg
 * (param_propagate_down_ / propagate_down).
 * ------------------------------------------------------------------------- */
void b2o_conv_backward(const b2o_conv_params* p, const float* x, const float* w,
                       const float* dy, float* dw, float* db, float* dx, int acc64) {
  const int Ho = b2o_out_h(p), Wo = b2o_out_w(p), P = Ho * Wo;
  const int Cg = p->C / p->G, Og = p->O / p->G, Kd = Cg * p->kh * p->kw;
  const size_t bottom_dim = (size_t)p->C * p->H * p->W, top_dim = (size_t)p->O * P;
  const size_t col_off = (size_t)Kd * P, out_off = (size_t)Og * P, w_off = (size_t)Og * Kd;
  const int one = is_1x1(p);
  float* col = one ? NULL : (float*)malloc(sizeof(float) * (size_t)Kd * p->G * P);
  float* ones = (float*)malloc(sizeof(float) * (size_t)P);
  for (int i = 0; i < P; ++i) ones[i] = 1.0f;
  if (p->has_bias && db)
    for (int n = 0; n < p->N; ++n)
      b2o_gemv(0, p->O, P, 1.0f, dy + n * top_dim, ones, 1.0f, db, acc64);
  if (dw || dx) {
    for (int n = 0; n < p->N; ++n) {
      const float* xn = x + n * bottom_dim;
      const float* dyn = dy + n * top_dim;
      if (dw) {
        const float* cb = xn;
        if (!one) { b2o_im2col(xn, p->C, p->H, p->W, p->kh, p->kw, p->ph, p->pw, p->sh, p->sw, p->dh, p->dw, col); cb = col; }
        for (int g = 0; g < p->G; ++g)
          b2o_gemm(0, 1, Og, Kd, P, 1.0f, dyn + out_off * g, cb + col_off * g, 1.0f, dw + w_off * g, acc64);
      }
      if (dx) {
        float* dxn = dx + n * bottom_dim;
        float* cb = one ? dxn : col;
        for (int g = 0; g < p->G; ++g)
          b2o_gemm(1, 0, Kd, P, Og, 1.0f, w + w_off * g, dyn + out_off * g, 0.0f, cb + col_off * g, acc64);
        if (!one) b2o_col2im(col, p->C, p->H, p->W, p->kh, p->kw, p->ph, p->pw, p->sh, p->sw, p->dh, p->dw, dxn);
      }
    }
  }
  free(ones);
  free(col);
}

/* ------------------------------------------------------------------------- *
 * Independent direct-definition convolution, the role caffe_conv plays in
 * src/caffe/test/test_convolution_layer.cpp:24-139 (2-D case): a second,
 * structurally different statement of the same function, used to cross-check
 * the im2col+GEMM restatement above.
 * ------------------------------------------------------------------------- */
void b2o_conv_direct(const b2o_conv_params* p, const float* x, const float* w,
                     const float* bias, float* y) {
  const int Ho = b2o_out_h(p), Wo = b2o_out_w(p);
  const int Cg = p->C / p->G, Og = p->O / p->G;
  for (int n = 0; n < p->N; ++n)
    for (int o = 0; o < p->O; ++o) {
      const int g = o / Og;
      for (int ho = 0; ho < Ho; ++ho)
        for (int wo = 0; wo < Wo; ++wo) {
          double acc = (p->has_bias && bias) ? (double)bias[o] : 0.0;
          for (int c = 0; c < Cg; ++c)
            for (int i = 0; i < p->kh; ++i)
              for (int j = 0; j < p->kw; ++j) {
                const int h = ho * p->sh - p->ph + i * p->dh, ww = wo * p->sw - p->pw + j * p->dw;
                if (h < 0 || h >= p->H || ww < 0 || ww >= p->W) continue;
                acc += (double)x[(((size_t)n * p->C + g * Cg + c) * p->H + h) * p->W + ww] *
                       (double)w[(((size_t)o * Cg + c) * p->kh + i) * p->kw + j];
              }
          y[(((size_t)n * p->O + o) * Ho + ho) * Wo + wo] = (float)acc;
        }
    }
}

/* ------------------------------------------------------------------------- *
 * SGD with momentum, CPU branch of SGDSolver::ApplyUpdate
 * (src/caffe/solvers/sgd_solver.cpp:143-149): Normalize (:152-158, x 1/iter_size),
 * Regularize (:161-192, L2: g += decay*w, L1: g += decay*sign(w)),
 * ComputeUpdateValue (:203-219: h = lr*g + m*h; g = h; Blob::Update w -= g
 * (src/caffe/blob.cpp:129-154); clear_grads -> g = 0).
 * grad_scale restates Net::ReduceAndUpdate's 1/global_grad_scale and the
 * 1/solver_count of Net::ReduceBucket (src/caffe/net.cpp:815-817,899-912): g is
 * multiplied by it first.  Pass 1 for the single-GPU fp32 case.
 * ------------------------------------------------------------------------- */
void b2o_sgd_update(size_t n, float* g, float* w, float* h, float momentum,
                    float local_rate, float local_decay, int l2, float grad_scale,
                    int iter_size, int clear_grads) {
  const float accum_norm = 1.0f / (float)iter_size;
  for (size_t i = 0; i < n; ++i) {
    float gi = g[i];
    if (grad_scale != 1.0f) gi *= grad_scale;
    if (iter_size != 1) gi *= accum_norm;
    if (local_decay != 0.0f) {
      const float reg = l2 ? w[i] : (float)((0.0f < w[i]) - (w[i] < 0.0f));
      gi += local_decay * reg;
    }
    const float hi = local_rate * gi + momentum * h[i];
    h[i] = hi;
    w[i] -= hi;
    g[i] = clear_grads ? 0.0f : hi;
  }
}

/* SGDSolver::GetLearningRate (sgd_solver.cpp:24-65).  policy: 0 fixed, 1 step,
 * 2 exp, 3 inv, 4 multistep (current_step passed in), 5 poly, 6 sigmoid.      */
float b2o_learning_rate(int policy, int iter, float base_lr, float gamma, float power,
                        int stepsize, int max_iter, float min_lr, int current_step,
                        int rampup_interval, float rampup_lr) {
  if (iter < rampup_interval) {
    const float alpha = (float)iter / (float)rampup_interval;
    return rampup_lr + (base_lr - rampup_lr) * alpha;
  }
  switch (policy) {
    case 0: return base_lr;
    case 1: return base_lr * powf(gamma, (float)(iter / stepsize));
    case 2: return base_lr * powf(gamma, (float)iter);
    case 3: return base_lr * powf(1.0f + gamma * (float)iter, -power);
    case 4: return base_lr * powf(gamma, (float)current_step);
    case 5: return min_lr + (base_lr - min_lr) * powf(1.0f - ((float)iter / (float)max_iter), power);
    case 6: return base_lr / (1.0f + (float)exp(-(double)gamma * (double)(iter - stepsize)));
    default: return -1.0f;
  }
}

/* SGDSolver::GetMomentum (sgd_solver.cpp:68-91).  policy: 0 fixed, 1 poly,
 * 2 opt; lr is GetLearningRate at iter.  "opt" squares in double what a float
 * sqrt gave, and clamps to max_momentum only when the solver file sets it.  */
float b2o_momentum(int policy, int iter, float momentum, float max_momentum, int has_max_momentum,
                   float momentum_power, int max_iter, float lr) {
  switch (policy) {
    case 0: return momentum;
    case 1: return momentum + (max_momentum - momentum) * powf((float)iter / (float)max_iter, momentum_power);
    case 2: {
      const double r = 1.0 - 0.5 * (double)sqrtf(lr);
      const float m = (float)(r * r);
      return has_max_momentum && max_momentum < m ? max_momentum : m;
    }
    default: return -1.0f;
  }
}

/* ------------------------------------------------------------------------- *
 * The fused solver updates of caffe_mpi_b200/csrc/sgd.cu, one element at a
 * time, for kind = b2c_solver_kind (0 SGD, 1 Nesterov, 2 AdaGrad, 3 RMSProp,
 * 4 AdaDelta, 5 Adam).  hp = {momentum, delta, rms_decay, beta1, beta2}; delta
 * is clamped as b2c_solver_update_arena does (AdaGrad / AdaDelta 1e-3,
 * RMSProp / Adam 1e-4).  lr for Adam carries the bias correction.
 *
 * b2o_solver_fp32 restates the kernel in fp32, in its order of operations.
 * Where a product meets a sum the compiler may contract to an fmaf; `form`
 * picks, per site, a rounded product then an add (bit clear) or the fmaf (bit
 * set).  At a site a*b + c*d at most one of its two bits may be set.
 *   bit 0  gr = fmaf(g, s, decay*reg)              bit 1  gr = fmaf(reg, decay, g*s)
 *   SGD       bit 2  h = fmaf(m, h, lr*gr)         bit 3  h = fmaf(lr, gr, m*h)
 *   Nesterov  bits 2, 3 as SGD for h';             bit 4  u = fmaf(1+m, h', -(m*h))
 *                                                  bit 5  u = fmaf(-m, h, (1+m)*h')
 *   AdaGrad   bit 2  h = fmaf(gr, gr, h)
 *   RMSProp   bit 2  h = fmaf(rd, h, (1-rd)*gr*gr) bit 3  h = fmaf((1-rd)*gr, gr, rd*h)
 *   AdaDelta  bits 2, 3 as RMSProp with m for h;   bits 4, 5 the same for h2;
 *             bit 6  w = fmaf(-lr, gr, w) (u = lr*gr rounded, for g)
 *   Adam      bit 2  m = fmaf(m, b1, gr*(1-b1))    bit 3  m = fmaf(gr, 1-b1, m*b1)
 *             bit 4  v = fmaf(v, b2, gr*gr*(1-b2)) bit 5  v = fmaf(gr*gr, 1-b2, v*b2)
 * Square roots and divisions are correctly rounded, as __fsqrt_rn and
 * __fdiv_rn.  Returns -1 for an unknown kind or an inadmissible form.
 * ------------------------------------------------------------------------- */
static float clamp_delta(int kind, float delta) {
  const float lo = (kind == 2 || kind == 4) ? 1e-3f : 1e-4f;
  return delta > lo ? delta : lo;
}
static int solver_form_ok(int kind, unsigned form) {
  static const unsigned bits[6] = {0xfu, 0x3fu, 0x7u, 0xfu, 0x7fu, 0x3fu};
  if (kind < 0 || kind > 5 || (form & ~bits[kind])) return 0;
  for (int b = 0; b < 6; b += 2)
    if (((form >> b) & 3u) == 3u) return 0;
  return 1;
}
/* a*b + c*d with bit `lo` fusing a*b and bit lo+1 fusing c*d */
static float mad2(unsigned form, int lo, float a, float b, float c, float d) {
  if (form >> lo & 1u) return fmaf(a, b, c * d);
  if (form >> (lo + 1) & 1u) return fmaf(c, d, a * b);
  return a * b + c * d;
}
int b2o_solver_fp32(int kind, unsigned form, size_t n, float* g, float* w, float* h, float* h2, const float* hp, float lr,
                    float decay, int l2, float grad_scale, int clear_grads) {
  if (!solver_form_ok(kind, form)) return -1;
  const float m = hp[0], delta = clamp_delta(kind, hp[1]), rd = hp[2], b1 = hp[3], b2 = hp[4];
  for (size_t i = 0; i < n; ++i) {
    const float reg = l2 ? w[i] : (float)((0.0f < w[i]) - (w[i] < 0.0f));
    float gr = mad2(form, 0, g[i], grad_scale, reg, decay), u = 0.0f, wn;
    int fused_w = 0;
    switch (kind) {
      case 0:
        u = h[i] = mad2(form, 2, m, h[i], lr, gr);
        break;
      case 1: {
        const float hi = h[i], hn = mad2(form, 2, m, hi, lr, gr);
        h[i] = hn;
        const float a = 1.0f + m;
        u = (form >> 4 & 1u) ? fmaf(a, hn, -(m * hi)) : (form >> 5 & 1u) ? fmaf(-m, hi, a * hn) : a * hn - m * hi;
        break;
      }
      case 2:
        h[i] = (form >> 2 & 1u) ? fmaf(gr, gr, h[i]) : h[i] + gr * gr;
        u = (lr * gr) / (sqrtf(h[i]) + delta);
        break;
      case 3:
        h[i] = mad2(form, 2, rd, h[i], (1.0f - rd) * gr, gr);
        u = (lr * gr) / (sqrtf(h[i]) + delta);
        break;
      case 4:
        h[i] = mad2(form, 2, m, h[i], (1.0f - m) * gr, gr);
        gr *= sqrtf((h2[i] + delta) / (h[i] + delta));
        h2[i] = mad2(form, 4, m, h2[i], (1.0f - m) * gr, gr);
        u = lr * gr;
        fused_w = (int)(form >> 6 & 1u);
        break;
      case 5:
        h[i] = mad2(form, 2, h[i], b1, gr, 1.0f - b1);
        h2[i] = mad2(form, 4, h2[i], b2, gr * gr, 1.0f - b2);
        u = (lr * h[i]) / (sqrtf(h2[i]) + delta);
        break;
    }
    wn = fused_w ? fmaf(-lr, gr, w[i]) : w[i] - u;
    w[i] = wn;
    g[i] = clear_grads ? 0.0f : u;
  }
  return 0;
}

/* b2o_solver_f64: the same update in float64 from the same fp32 inputs and
 * constants (1 - m, 1 + m, the clamped delta as the kernel forms them in fp32),
 * and for each output a bound on |fp32 result - float64 result| that holds for
 * every admissible form.
 *
 * Derivation.  Every fp32 operation returns fl(x) = x(1 + e) + t with |e| <=
 * u = 2^-24 and |t| <= 2^-150 (the underflow term: half the smallest fp32
 * subnormal; zero for sums and for an fmaf away from underflow, kept anyway).
 * Carry for each intermediate x its float64 value X and a bound E >= |x_fp32 -
 * X|.  Inputs and fp32 constants are exact: E = 0.  To first order, plus the
 * second-order terms where they are cheap to keep:
 *   x = a*b      E = |A| Eb + |B| Ea + Ea Eb + u|X| + 2^-150
 *   x = a +- b   E = Ea + Eb + u|X| + 2^-150
 *   x = sqrt(a)  E = min(Ea / (sqrt(A) + sqrt(max(A - Ea, 0))), sqrt(Ea)) + u|X| + 2^-150
 *                (|sqrt(a) - sqrt(A)| = |a - A| / (sqrt(a) + sqrt(A)); sqrt is
 *                1/2-Hoelder, so the second term holds at A = 0)
 *   x = a / b    E = (Ea + |X| Eb) / (|B| - Eb) + u|X| + 2^-150   (|B| > Eb:
 *                b = sqrt(h) + delta >= 1e-4 while Eb is ~1e-7 |B|)
 * An fmaf rounds once where a rounded product then an add round twice, and
 * its result deviates from X by no more than the unfused bound's terms, so the
 * bound of the unfused form covers every form.  Float64's own error (2^-53
 * per operation) is ~2^29 times smaller than each u term; the caller's test
 * multiplies the bound by 1 + 2^-20 to cover it.
 * vals, bounds: 4 x n arrays (g, w, h, h2 after the update; h2 rows are the
 * input for the one-history kinds, bound 0).
 * ------------------------------------------------------------------------- */
typedef struct { double v, e; } b2o_ve;
static const double U32 = 5.9604644775390625e-08, ETA32 = 7.006492321624085e-46;   /* 2^-24, 2^-150 */
static b2o_ve ve_exact(double v) { b2o_ve r = {v, 0.0}; return r; }
static b2o_ve ve_mul(b2o_ve a, b2o_ve b) {
  b2o_ve r; r.v = a.v * b.v;
  r.e = fabs(a.v) * b.e + fabs(b.v) * a.e + a.e * b.e + U32 * fabs(r.v) + ETA32;
  return r;
}
static b2o_ve ve_add(b2o_ve a, b2o_ve b) { b2o_ve r; r.v = a.v + b.v; r.e = a.e + b.e + U32 * fabs(r.v) + ETA32; return r; }
static b2o_ve ve_sub(b2o_ve a, b2o_ve b) { b2o_ve r; r.v = a.v - b.v; r.e = a.e + b.e + U32 * fabs(r.v) + ETA32; return r; }
static b2o_ve ve_sqrt(b2o_ve a) {
  b2o_ve r; r.v = sqrt(a.v);
  const double lo = a.v - a.e > 0.0 ? sqrt(a.v - a.e) : 0.0;
  const double lin = r.v > 0.0 ? a.e / (r.v + lo) : INFINITY, hol = sqrt(a.e);
  r.e = (lin < hol ? lin : hol) + U32 * r.v + ETA32;
  return r;
}
static b2o_ve ve_div(b2o_ve a, b2o_ve b) {
  b2o_ve r; r.v = a.v / b.v;
  r.e = (a.e + fabs(r.v) * b.e) / (fabs(b.v) - b.e) + U32 * fabs(r.v) + ETA32;
  return r;
}
int b2o_solver_f64(int kind, size_t n, const float* g, const float* w, const float* h, const float* h2, const float* hp,
                   float lr, float decay, int l2, float grad_scale, int clear_grads, double* vals, double* bounds) {
  if (kind < 0 || kind > 5) return -1;
  const float m = hp[0], rd = hp[2], b1 = hp[3], b2 = hp[4];
  const b2o_ve M = ve_exact(m), D = ve_exact(clamp_delta(kind, hp[1])), RD = ve_exact(rd), B1 = ve_exact(b1), B2 = ve_exact(b2);
  const b2o_ve LR = ve_exact(lr), DEC = ve_exact(decay), S = ve_exact(grad_scale);
  /* 1 - m, 1 + m, ... as the kernel forms them: one fp32 rounding each, so exact inputs here */
  const b2o_ve OM = ve_exact(1.0f - m), PM = ve_exact(1.0f + m), ORD = ve_exact(1.0f - rd), OB1 = ve_exact(1.0f - b1),
               OB2 = ve_exact(1.0f - b2);
  for (size_t i = 0; i < n; ++i) {
    const b2o_ve W = ve_exact(w[i]), H = ve_exact(h[i]), H2 = ve_exact(h2 ? h2[i] : 0.0f);
    const b2o_ve REG = ve_exact(l2 ? w[i] : (float)((0.0f < w[i]) - (w[i] < 0.0f)));
    b2o_ve gr = ve_add(ve_mul(ve_exact(g[i]), S), ve_mul(REG, DEC)), u, hn = H, h2n = H2;
    switch (kind) {
      case 0: u = hn = ve_add(ve_mul(M, H), ve_mul(LR, gr)); break;
      case 1:
        hn = ve_add(ve_mul(M, H), ve_mul(LR, gr));
        u = ve_sub(ve_mul(PM, hn), ve_mul(M, H));
        break;
      case 2:
        hn = ve_add(H, ve_mul(gr, gr));
        u = ve_div(ve_mul(LR, gr), ve_add(ve_sqrt(hn), D));
        break;
      case 3:
        hn = ve_add(ve_mul(RD, H), ve_mul(ve_mul(ORD, gr), gr));
        u = ve_div(ve_mul(LR, gr), ve_add(ve_sqrt(hn), D));
        break;
      case 4:
        hn = ve_add(ve_mul(M, H), ve_mul(ve_mul(OM, gr), gr));
        gr = ve_mul(gr, ve_sqrt(ve_div(ve_add(H2, D), ve_add(hn, D))));
        h2n = ve_add(ve_mul(M, H2), ve_mul(ve_mul(OM, gr), gr));
        u = ve_mul(LR, gr);
        break;
      default:
        hn = ve_add(ve_mul(H, B1), ve_mul(gr, OB1));
        h2n = ve_add(ve_mul(H2, B2), ve_mul(ve_mul(gr, gr), OB2));
        u = ve_div(ve_mul(LR, hn), ve_add(ve_sqrt(h2n), D));
        break;
    }
    const b2o_ve wn = ve_sub(W, u);
    vals[i] = clear_grads ? 0.0 : u.v;            bounds[i] = clear_grads ? 0.0 : u.e;
    vals[n + i] = wn.v;                           bounds[n + i] = wn.e;
    vals[2 * n + i] = hn.v;                       bounds[2 * n + i] = hn.e;
    vals[3 * n + i] = h2n.v;                      bounds[3 * n + i] = h2n.e;
  }
  return 0;
}

/* ------------------------------------------------------------------------- *
 * Multi-rank gradient exchange: in-place sum over ranks of a diff bucket
 * (P2PSync::allreduce_bucket, src/caffe/parallel.cpp:245-253, ncclSum) followed
 * by x 1/solver_count (Net::ReduceBucket, src/caffe/net.cpp:899-912).  One
 * process, R replicas, summed on the host in rank order.
 * ------------------------------------------------------------------------- */
void b2o_allreduce_avg(int R, size_t count, float** bufs, int solver_count) {
  const float scale = 1.0f / (float)solver_count;
  for (size_t i = 0; i < count; ++i) {
    float s = 0.0f;
    for (int r = 0; r < R; ++r) s += bufs[r][i];
    s *= scale;
    for (int r = 0; r < R; ++r) bufs[r][i] = s;
  }
}

#ifdef __cplusplus
}
#endif
