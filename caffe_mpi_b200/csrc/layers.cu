// layers.cu -- the non-convolution layers on ResNet-50's training path (SURVEY.md 8(f) rank 2), fp32 NCHW.
// All are HBM-bound elementwise / reduction kernels; each entry point cites the reference CPU code whose
// semantics it keeps (the parity oracle for them is oracle/layers_oracle.py).
//
//   ReLU            src/caffe/layers/relu_layer.cpp:10-41           y = max(x,0) + slope*min(x,0); dx = dy*(x>0 ? 1 : slope)
//   BatchNorm       src/caffe/layers/batch_norm_layer.cpp:140-300   batch statistics (biased variance, eps added before the
//                   (NVCaffe, scale_bias)                            inverse sqrt AND before the running average), x_norm kept
//                                                                    for backward; dgamma/dbeta OVERWRITTEN (compute_sum_*)
//   Pooling MAX/AVE src/caffe/layers/pooling_layer.cpp:129-318      ceil-mode extents, first-max index mask, AVE divides by the
//                                                                    padded window size
//   Eltwise SUM     src/caffe/layers/eltwise_layer.cpp
//   SoftmaxWithLoss src/caffe/layers/softmax_loss_layer.cpp:96-160  loss = -sum log p[label] / N (VALID normalisation, no
//                                                                    ignore_label); dx = (p - onehot) * loss_weight / N
//                   the _ex forms: per (outer, inner) pixel, ignore_label, FULL / VALID / BATCH_SIZE / NONE normalizers
//   Softmax         src/caffe/layers/softmax_layer.cu               over the C axis of [outer, C, inner]; dx = (dy - sum_c dy y) y
//   Sigmoid         src/caffe/layers/sigmoid_layer.cu:9-13           y = 1 / (1 + exp(-x)); dx = dy y (1 - y)
//   SigmoidCrossEntropyLoss  sigmoid_cross_entropy_loss_layer.cpp   the stable loss expression / N; dx = (sigmoid(x) - t) * loss_weight / N
//   EuclideanLoss   src/caffe/layers/euclidean_loss_layer.cu        diff = a - b, loss = sum diff^2 / N / 2; dx = +-loss_weight / N * diff
//   L1Loss          src/caffe/layers/l1_loss_layer.cu:11-43          diff = a - b, loss = sum |diff| / N; dx = +-loss_weight / N * sign(diff)
#include <float.h>
#include <type_traits>
#include <cooperative_groups.h>
#include "b2c_common.cuh"
#include "bn_common.cuh"

namespace cg = cooperative_groups;

namespace b2c {

// ---- ReLU ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) relu_fwd_kernel(size_t n, int vec, const float* __restrict__ x, float* __restrict__ y, float slope) {
  pdl_wait();
  const size_t n4 = vec ? n / 4 : 0, tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  const float4* x4 = reinterpret_cast<const float4*>(x);
  float4* y4 = reinterpret_cast<float4*>(y);
  for (size_t i = tid; i < n4; i += step) {
    float4 v = x4[i];
    v.x = v.x > 0 ? v.x : v.x * slope; v.y = v.y > 0 ? v.y : v.y * slope; v.z = v.z > 0 ? v.z : v.z * slope; v.w = v.w > 0 ? v.w : v.w * slope;
    y4[i] = v;
  }
  for (size_t i = n4 * 4 + tid; i < n; i += step) { const float v = x[i]; y[i] = v > 0 ? v : v * slope; }
}
__global__ void __launch_bounds__(256) relu_bwd_kernel(size_t n, int vec, const float* __restrict__ dy, const float* __restrict__ x,
                                                       float* __restrict__ dx, float slope) {
  pdl_wait();
  const size_t n4 = vec ? n / 4 : 0, tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  const float4* d4 = reinterpret_cast<const float4*>(dy);
  const float4* x4 = reinterpret_cast<const float4*>(x);
  float4* o4 = reinterpret_cast<float4*>(dx);
  for (size_t i = tid; i < n4; i += step) {
    const float4 d = d4[i], v = x4[i];
    float4 o;
    o.x = d.x * (v.x > 0 ? 1.f : slope); o.y = d.y * (v.y > 0 ? 1.f : slope); o.z = d.z * (v.z > 0 ? 1.f : slope); o.w = d.w * (v.w > 0 ? 1.f : slope);
    o4[i] = o;
  }
  for (size_t i = n4 * 4 + tid; i < n; i += step) dx[i] = dy[i] * (x[i] > 0 ? 1.f : slope);
}

// ---- BatchNorm --------------------------------------------------------------------------------------------------
// Per-channel reductions run as one thread-block CLUSTER of 1..8 CTAs per channel (sized by the host from the channel's
// extent): each CTA streams its share of the channel's N*S values (float4 when the planes are 16-byte aligned), the eight partial sums meet in rank 0 through
// distributed shared memory in rank order (deterministic), no scratch buffer, no atomics, one launch.
// Statistics (bn_channel_stats): sums of x - k and (x - k)^2 with k = the channel's first value, combined in double, and a second
// pass about that mean when k lies more than 4 sigma from it, so the variance's error does not depend on any one element.
// (geometry, cursors and block sums: bn_common.cuh, shared with the fused kernels of layers_fused.cu)

template <bool VEC>
__global__ void __launch_bounds__(BN_THREADS)
bn_stats_kernel(int N, int C, int S, const float* __restrict__ x, float eps, float maf, int first,
                float* __restrict__ mean, float* __restrict__ invstd, float* __restrict__ run_mean, float* __restrict__ run_var) {
  pdl_wait();
  __shared__ float2 part[2];
  cg::cluster_group cluster = cg::this_cluster();
  const int c = blockIdx.y;
  float m, var_eps;
  bn_channel_stats<VEC, 0>(cluster, N, C, S, c, x, eps, part, nullptr, m, var_eps);
  if (cluster.block_rank() == 0 && threadIdx.x == 0) {
    mean[c] = m;
    invstd[c] = 1.0f / sqrtf(var_eps);
    if (first) { run_mean[c] = m; run_var[c] = var_eps; }                         // iter_ <= 1: copy (:199-204)
    else { run_mean[c] = (1.f - maf) * m + maf * run_mean[c]; run_var[c] = (1.f - maf) * var_eps + maf * run_var[c]; }
  }
  cluster.sync();                                   // remote shared memory stays valid until every rank has read it
}
// per channel: dgamma = sum dy*xn, dbeta = sum dy (both OVERWRITTEN, batch_norm_layer.cpp:247-252)
template <bool VEC>
__global__ void __launch_bounds__(BN_THREADS)
bn_bwd_reduce_kernel(int N, int C, int S, const float* __restrict__ dy, const float* __restrict__ xnorm,
                     float* __restrict__ sum_dy_xn, float* __restrict__ sum_dy) {
  pdl_wait();
  __shared__ float2 part;
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned rank = cluster.block_rank();
  const int c = blockIdx.y;
  float a, b;
  bn_channel_partial<VEC, 1>(N, C, S, c, dy, xnorm, 0.f, rank, cluster.num_blocks(), a, b);
  block_sum2(a, b);
  if (threadIdx.x == 0) part = make_float2(a, b);
  cluster.sync();
  if (rank == 0 && threadIdx.x == 0) {
    double s1 = 0.0, s2 = 0.0;
    for (unsigned r = 0; r < cluster.num_blocks(); ++r) { const float2 v = *cluster.map_shared_rank(&part, r); s1 += v.x; s2 += v.y; }
    sum_dy_xn[c] = (float)s1; sum_dy[c] = (float)s2;
  }
  cluster.sync();
}

// Elementwise passes: each block owns BN_EW_PER_THREAD * 256 consecutive units (float4 or float) of the NCHW tensor and
// walks (plane, offset) incrementally, so there is one integer division per thread, not per element.
constexpr int BN_EW_PER_THREAD = 8;
template <bool VEC> struct ChanCursor {
  unsigned p, c;
  __device__ __forceinline__ void init(size_t i, unsigned units, unsigned C) { const size_t plane = i / units; p = (unsigned)(i - plane * units); c = (unsigned)(plane % C); }
  __device__ __forceinline__ void advance(unsigned step, unsigned units, unsigned C) { p += step; while (p >= units) { p -= units; if (++c == C) c = 0; } }
};
template <bool VEC>
__global__ void __launch_bounds__(256)
bn_norm_kernel(size_t total_units, int C, int S, const float* __restrict__ x, const float* __restrict__ mean, const float* __restrict__ invstd,
               const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ xnorm, float* __restrict__ y) {
  pdl_wait();
  const unsigned units = VEC ? S / 4 : S;
  size_t i = (size_t)blockIdx.x * (256 * BN_EW_PER_THREAD) + threadIdx.x;
  if (i >= total_units) return;
  ChanCursor<VEC> cur;
  cur.init(i, units, C);
#pragma unroll 2
  for (int k = 0; k < BN_EW_PER_THREAD && i < total_units; ++k, i += 256) {
    const float m = mean[cur.c], is = invstd[cur.c], g = gamma ? gamma[cur.c] : 1.f, bt = gamma ? beta[cur.c] : 0.f;
    if (VEC) {
      const float4 v = reinterpret_cast<const float4*>(x)[i];
      float4 n4, o4;
      const bool affine = gamma != nullptr;
      n4.x = bn_xn(v.x, m, is); n4.y = bn_xn(v.y, m, is); n4.z = bn_xn(v.z, m, is); n4.w = bn_xn(v.w, m, is);
      o4.x = bn_y(n4.x, g, bt, affine); o4.y = bn_y(n4.y, g, bt, affine); o4.z = bn_y(n4.z, g, bt, affine); o4.w = bn_y(n4.w, g, bt, affine);
      reinterpret_cast<float4*>(xnorm)[i] = n4;
      reinterpret_cast<float4*>(y)[i] = o4;
    } else {
      const float xn = bn_xn(x[i], m, is);
      xnorm[i] = xn;
      y[i] = bn_y(xn, g, bt, gamma != nullptr);
    }
    cur.advance(256, units, C);
  }
}
// dx = gamma * invstd * (dy - mean(dy) - xn * mean(dy*xn))     (means over N*S; with gamma folded: :254-281)
template <bool VEC>
__global__ void __launch_bounds__(256)
bn_bwd_dx_kernel(size_t total_units, int C, int S, float inv_cnt, const float* __restrict__ dy, const float* __restrict__ xnorm,
                 const float* __restrict__ gamma, const float* __restrict__ invstd, const float* __restrict__ sum_dy_xn,
                 const float* __restrict__ sum_dy, float* __restrict__ dx) {
  pdl_wait();
  const unsigned units = VEC ? S / 4 : S;
  size_t i = (size_t)blockIdx.x * (256 * BN_EW_PER_THREAD) + threadIdx.x;
  if (i >= total_units) return;
  ChanCursor<VEC> cur;
  cur.init(i, units, C);
#pragma unroll 2
  for (int k = 0; k < BN_EW_PER_THREAD && i < total_units; ++k, i += 256) {
    const float gi = __fmul_rn(gamma ? gamma[cur.c] : 1.f, invstd[cur.c]);
    const float mdy = bn_mean_term(sum_dy[cur.c], inv_cnt), mdx = bn_mean_term(sum_dy_xn[cur.c], inv_cnt);
    if (VEC) {
      const float4 d = reinterpret_cast<const float4*>(dy)[i], n4 = reinterpret_cast<const float4*>(xnorm)[i];
      float4 o;
      o.x = bn_dx(d.x, n4.x, gi, mdy, mdx); o.y = bn_dx(d.y, n4.y, gi, mdy, mdx); o.z = bn_dx(d.z, n4.z, gi, mdy, mdx); o.w = bn_dx(d.w, n4.w, gi, mdy, mdx);
      reinterpret_cast<float4*>(dx)[i] = o;
    } else {
      dx[i] = bn_dx(dy[i], xnorm[i], gi, mdy, mdx);
    }
    cur.advance(256, units, C);
  }
}

// ---- LRN across channels ------------------------------------------------------------------------------------------
// s^-beta: beta = 0.75 (every BASELINE net) is two reciprocal square roots instead of powf's ~30 instructions per element
__device__ __forceinline__ float lrn_pow_neg(float s, float beta) {
  if (beta == 0.75f) { const float r = rsqrtf(s); return r * sqrtf(r); }
  return powf(s, -beta);
}
// one thread per (image, pixel): walks the channels with a running window sum, loads coalesced along the pixel axis
__global__ void __launch_bounds__(256)
lrn_fwd_kernel(int N, int C, int S, int size, float alpha_over_size, float beta, float k, const float* __restrict__ x,
               float* __restrict__ scale, float* __restrict__ y) {
  pdl_wait();
  const long long total = (long long)N * S;
  const int pre = (size - 1) / 2;                              // lrn_layer.cpp: pre_pad_
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / S, sp = i - n * S;
    const float* xp = x + n * C * S + sp;
    float* sc = scale + n * C * S + sp;
    float* yp = y + n * C * S + sp;
    float acc = 0.f;                                           // window of channel c: [c - pre, c - pre + size)
    for (int c = 0; c < size - 1 - pre && c < C; ++c) { const float v = xp[(long long)c * S]; acc += v * v; }
    for (int c = 0; c < C; ++c) {
      const int head = c - pre + size - 1, tail = c - pre - 1;
      if (head < C && head >= 0) { const float v = xp[(long long)head * S]; acc += v * v; }
      if (tail >= 0 && tail < C) { const float v = xp[(long long)tail * S]; acc -= v * v; }
      const float s_ = k + alpha_over_size * acc;
      sc[(long long)c * S] = s_;
      yp[(long long)c * S] = xp[(long long)c * S] * lrn_pow_neg(s_, beta);
    }
  }
}
__global__ void __launch_bounds__(256)
lrn_bwd_kernel(int N, int C, int S, int size, float cache_ratio, float beta, const float* __restrict__ x, const float* __restrict__ y,
               const float* __restrict__ scale, const float* __restrict__ dy, float* __restrict__ dx) {
  pdl_wait();
  const long long total = (long long)N * S;
  const int ipp = size - (size + 1) / 2;                       // lrn_layer.cpp: inverse_pre_pad
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / S, sp = i - n * S, base = n * C * S + sp;
    auto ratio = [&](int c) { const long long o = base + (long long)c * S; return dy[o] * y[o] / scale[o]; };
    float acc = 0.f;                                           // window of channel c: [c - ipp, c - ipp + size)
    for (int c = 0; c < size - 1 - ipp && c < C; ++c) acc += ratio(c);
    for (int c = 0; c < C; ++c) {
      const int head = c - ipp + size - 1, tail = c - ipp - 1;
      if (head < C && head >= 0) acc += ratio(head);
      if (tail >= 0 && tail < C) acc -= ratio(tail);
      const long long o = base + (long long)c * S;
      dx[o] = dy[o] * lrn_pow_neg(scale[o], beta) - cache_ratio * x[o] * acc;
    }
  }
}

// ---- Dropout mask / elementwise product ----------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long splitmix64(unsigned long long z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__global__ void __launch_bounds__(256)
dropout_mask_kernel(size_t n, unsigned threshold24, float scale, unsigned long long seed, unsigned long long offset, float* __restrict__ mask) {
  pdl_wait();
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const unsigned u = (unsigned)(splitmix64(seed + offset + i) >> 40);      // 24 uniform bits
    mask[i] = u >= threshold24 ? scale : 0.f;
  }
}
__global__ void __launch_bounds__(256) mul_kernel(size_t n, const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ y) {
  pdl_wait();
  const size_t n4 = n / 4, tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  for (size_t i = tid; i < n4; i += step) {
    const float4 u = reinterpret_cast<const float4*>(a)[i], v = reinterpret_cast<const float4*>(b)[i];
    reinterpret_cast<float4*>(y)[i] = make_float4(u.x * v.x, u.y * v.y, u.z * v.z, u.w * v.w);
  }
  for (size_t i = n4 * 4 + tid; i < n; i += step) y[i] = a[i] * b[i];
}

// ---- Pooling ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
pool_max_fwd_kernel(size_t total, int H, int W, int Ho, int Wo, int kh, int kw, int sh, int sw, int ph, int pw,
                    const float* __restrict__ x, float* __restrict__ y, int* __restrict__ mask) {
  pdl_wait();
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int wo = (int)(i % Wo), ho = (int)((i / Wo) % Ho);
    const size_t nc = i / ((size_t)Wo * Ho);
    int hs = ho * sh - ph, ws = wo * sw - pw;
    const int he = min(hs + kh, H), we = min(ws + kw, W);
    hs = max(hs, 0); ws = max(ws, 0);
    const float* src = x + nc * H * W;
    float best = -FLT_MAX;
    int bi = -1;
    for (int h = hs; h < he; ++h)
      for (int w = ws; w < we; ++w) {
        const float v = src[h * W + w];
        if (v > best) { best = v; bi = h * W + w; }       // strict '>' keeps the FIRST maximum, as the reference
      }
    y[i] = best;
    mask[i] = bi;
  }
}
// The common window shapes with Wo % Q == 0: one thread per Q consecutive outputs of a pooled row.  The (Q-1)*SW + KW input columns
// those windows cover are loaded once per window row (27 loads instead of 36 for 3x3 / 2 with Q = 4), results leave as one 16- or
// 8-byte store each for y and the mask.  Scan order and the strict '>' are those of the scalar kernel: same first maximum.
template <int KH, int KW, int SH, int SW, int Q>
__global__ void __launch_bounds__(256)
pool_max_fwd_q_kernel(long long groups, int H, int W, int Ho, int Wo, int ph, int pw, const float* __restrict__ x,
                      float* __restrict__ y, int* __restrict__ mask) {
  pdl_wait();
  constexpr int NCOL = (Q - 1) * SW + KW;
  const int Wq = Wo / Q;
  for (long long gidx = (long long)blockIdx.x * blockDim.x + threadIdx.x; gidx < groups; gidx += (long long)gridDim.x * blockDim.x) {
    const long long orow = gidx / Wq;                             // pooled row index over (plane, ho)
    const int wo0 = (int)(gidx - orow * Wq) * Q;
    const long long nc = orow / Ho;
    const int ho = (int)(orow - nc * Ho);
    const int hs = ho * SH - ph, ws0 = wo0 * SW - pw;
    const float* src = x + nc * H * W;
    float best[Q];
    int bi[Q];
#pragma unroll
    for (int q = 0; q < Q; ++q) { best[q] = -FLT_MAX; bi[q] = -1; }
#pragma unroll
    for (int i = 0; i < KH; ++i) {
      const int h = hs + i;
      const bool hok = (unsigned)h < (unsigned)H;
      float v[NCOL];
#pragma unroll
      for (int j = 0; j < NCOL; ++j) {
        const int w = ws0 + j;
        v[j] = (hok && (unsigned)w < (unsigned)W) ? __ldg(src + (long long)h * W + w) : -FLT_MAX;
      }
#pragma unroll
      for (int q = 0; q < Q; ++q)
#pragma unroll
        for (int j = 0; j < KW; ++j) {
          const int w = ws0 + q * SW + j;
          if (hok && (unsigned)w < (unsigned)W && v[q * SW + j] > best[q]) { best[q] = v[q * SW + j]; bi[q] = h * W + w; }
        }
    }
    const long long o = orow * Wo + wo0;
    if (Q == 4) {
      *reinterpret_cast<float4*>(y + o) = make_float4(best[0], best[1], best[2], best[Q - 1]);
      *reinterpret_cast<int4*>(mask + o) = make_int4(bi[0], bi[1], bi[2], bi[Q - 1]);
    } else {
      *reinterpret_cast<float2*>(y + o) = make_float2(best[0], best[Q - 1]);
      *reinterpret_cast<int2*>(mask + o) = make_int2(bi[0], bi[Q - 1]);
    }
  }
}
// One block per input row (plane nc, row h): the row's window range in h is computed once, threads walk w, instead of decoding a
// flat 64-bit element index with three runtime divisions per element.  Ascending (a, b) summation order.
__global__ void __launch_bounds__(128)
pool_max_bwd_kernel(int rows, int H, int W, int Ho, int Wo, int kh, int kw, int sh, int sw, int ph, int pw,
                    const float* __restrict__ dy, const int* __restrict__ mask, float* __restrict__ dx) {
  pdl_wait();
  const int rpb = W >= 128 ? 1 : 128 / W;                    // input rows per block (narrow maps: several rows share the 128 threads)
  const int tr = rpb == 1 ? 0 : (int)threadIdx.x / W;        // this thread's row inside the block's group, first column
  const int tw = rpb == 1 ? (int)threadIdx.x : (int)threadIdx.x - tr * W;
  if (tr >= rpb) return;
  for (int row = blockIdx.x * rpb + tr; row < rows; row += gridDim.x * rpb) {
    const int nc = row / H, h = row - nc * H;
    const int phs = (h + ph < kh) ? 0 : (h + ph - kh) / sh + 1, phe = min((h + ph) / sh + 1, Ho);
    const float* d = dy + (size_t)nc * Ho * Wo;
    const int* m = mask + (size_t)nc * Ho * Wo;
    float* out = dx + (size_t)row * W;
    for (int w = tw; w < W; w += 128) {
      const int pws = (w + pw < kw) ? 0 : (w + pw - kw) / sw + 1, pwe = min((w + pw) / sw + 1, Wo);
      const int me = h * W + w;
      float g = 0.f;
      for (int a = phs; a < phe; ++a)
        for (int b = pws; b < pwe; ++b)
          if (m[a * Wo + b] == me) g += d[a * Wo + b];
      out[w] = g;
    }
  }
}
// The common window shapes (3x3 / stride 2, 2x2 / stride 2, 3x3 / stride 1) with W % 4 == 0: one thread per FOUR consecutive input
// columns.  The windows those four columns can sit in are MA rows x NB columns of the pooled map; their (mask, dy) pairs are loaded
// ONCE, unconditionally (12 loads for 3x3 / 2), and each of the four elements picks its own from registers -- the row kernel
// above has one element and two dependent round trips per thread (0.35 TB/s: 0.6 ms per ResNet-50 step, 5.9 ms per GoogLeNet
// step); loading per element instead of per window ran into the load/store unit (32 loads per 16-byte store, 0.94 TB/s).
// Same ascending (a, b) summation order: same bits.
template <int KH, int KW, int SH, int SW>
__global__ void __launch_bounds__(256)
pool_max_bwd_q4_kernel(long long quads, int H, int W, int Ho, int Wo, int ph, int pw, const float* __restrict__ dy,
                       const int* __restrict__ mask, float* __restrict__ dx) {
  pdl_wait();
  constexpr int MA = (KH + SH - 1) / SH;                        // pooled rows an input row can sit in
  constexpr int NB = (3 + KW - 1) / SW + 1;                    // pooled columns four consecutive input columns can sit in
  const int Wq = W / 4;
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < quads; q += (long long)gridDim.x * blockDim.x) {
    const long long row = q / Wq;
    const int w0 = (int)(q - row * Wq) * 4;
    const long long nc = row / H;
    const int h = (int)(row - nc * H);
    const int phs = (h + ph < KH) ? 0 : (h + ph - KH) / SH + 1, phe = min((h + ph) / SH + 1, Ho);
    const int b0 = (w0 + pw < KW) ? 0 : (w0 + pw - KW) / SW + 1;                    // first pooled column of input column w0
    const float* d = dy + nc * Ho * Wo;
    const int* m = mask + nc * Ho * Wo;
    int mm[MA][NB];
    float dd[MA][NB];
#pragma unroll
    for (int a = 0; a < MA; ++a)
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        const bool ok = phs + a < phe && b0 + b < Wo;
        const int idx = ok ? (phs + a) * Wo + b0 + b : 0;
        mm[a][b] = ok ? __ldg(m + idx) : -1;                    // -1 never equals an element index
        dd[a][b] = __ldg(d + idx);
      }
    float g[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int w = w0 + e;
      const int pws = (w + pw < KW) ? 0 : (w + pw - KW) / SW + 1, pwe = min((w + pw) / SW + 1, Wo);
      const int me = h * W + w;
      float acc = 0.f;
#pragma unroll
      for (int a = 0; a < MA; ++a)
#pragma unroll
        for (int b = 0; b < NB; ++b) {
          const int bb = b0 + b;
          acc += (bb >= pws && bb < pwe && mm[a][b] == me) ? dd[a][b] : 0.f;
        }
      g[e] = acc;
    }
    *reinterpret_cast<float4*>(dx + row * W + w0) = make_float4(g[0], g[1], g[2], g[3]);
  }
}
__global__ void __launch_bounds__(256)
pool_ave_fwd_kernel(size_t total, int H, int W, int Ho, int Wo, int kh, int kw, int sh, int sw, int ph, int pw,
                    const float* __restrict__ x, float* __restrict__ y) {
  pdl_wait();
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int wo = (int)(i % Wo), ho = (int)((i / Wo) % Ho);
    const size_t nc = i / ((size_t)Wo * Ho);
    int hs = ho * sh - ph, ws = wo * sw - pw;
    int he = min(hs + kh, H + ph), we = min(ws + kw, W + pw);
    const int pool_size = (he - hs) * (we - ws);          // padded window size (pooling_layer.cpp:200-206)
    hs = max(hs, 0); ws = max(ws, 0); he = min(he, H); we = min(we, W);
    const float* src = x + nc * H * W;
    float s = 0.f;
    for (int h = hs; h < he; ++h)
      for (int w = ws; w < we; ++w) s += src[h * W + w];
    y[i] = s / pool_size;
  }
}
__global__ void __launch_bounds__(256)
pool_ave_bwd_kernel(size_t total, int H, int W, int Ho, int Wo, int kh, int kw, int sh, int sw, int ph, int pw,
                    const float* __restrict__ dy, float* __restrict__ dx) {
  pdl_wait();
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int w = (int)(i % W) + pw, h = (int)((i / W) % H) + ph;
    const size_t nc = i / ((size_t)W * H);
    const int phs = (h < kh) ? 0 : (h - kh) / sh + 1, phe = min(h / sh + 1, Ho);
    const int pws = (w < kw) ? 0 : (w - kw) / sw + 1, pwe = min(w / sw + 1, Wo);
    const float* d = dy + nc * Ho * Wo;
    float g = 0.f;
    for (int a = phs; a < phe; ++a)
      for (int b = pws; b < pwe; ++b) {
        const int hs = a * sh - ph, ws = b * sw - pw;
        const int he = min(hs + kh, H + ph), we = min(ws + kw, W + pw);
        g += d[a * Wo + b] / ((he - hs) * (we - ws));
      }
    dx[i] = g;
  }
}

// ---- elementwise ----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) add_kernel(size_t n, int vec, const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ y) {
  pdl_wait();
  const size_t n4 = vec ? n / 4 : 0, tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  for (size_t i = tid; i < n4; i += step) {
    const float4 u = reinterpret_cast<const float4*>(a)[i], v = reinterpret_cast<const float4*>(b)[i];
    reinterpret_cast<float4*>(y)[i] = make_float4(u.x + v.x, u.y + v.y, u.z + v.z, u.w + v.w);
  }
  for (size_t i = n4 * 4 + tid; i < n; i += step) y[i] = a[i] + b[i];
}

// ---- softmax with loss ------------------------------------------------------------------------------------------
// one block per sample; prob[N,C]; labels are float class ids.  The loss itself is summed by softmax_loss_sum_kernel in a fixed
// order (an atomicAdd per sample made the last bit of the reported loss depend on block scheduling).  No __restrict__: the Softmax
// layer runs this kernel in place (prob == logits); every element is read by the thread that later writes it, before that write.
__global__ void __launch_bounds__(256)
softmax_loss_fwd_kernel(int C, const float* logits, float* prob) {
  pdl_wait();
  const int n = blockIdx.x;
  const float* z = logits + (size_t)n * C;
  float mx = -FLT_MAX, dummy = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) mx = fmaxf(mx, z[c]);
#pragma unroll
  for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  __shared__ float smx[32];
  if ((threadIdx.x & 31) == 0) smx[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = smx[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); ++w) mx = fmaxf(mx, smx[w]);
  float s = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) { const float e = expf(z[c] - mx); prob[(size_t)n * C + c] = e; s += e; }
  block_sum2(s, dummy);
  const float inv = 1.f / s;
  for (int c = threadIdx.x; c < C; c += blockDim.x) prob[(size_t)n * C + c] *= inv;
}
// loss = scale * sum_n -log(max(prob[n][label[n]], FLT_MIN))   (softmax_loss_layer.cpp:100-116); one block, fixed summation order
__global__ void __launch_bounds__(256)
softmax_loss_sum_kernel(int N, int C, const float* __restrict__ prob, const float* __restrict__ labels, float scale, float* __restrict__ loss) {
  pdl_wait();
  float s = 0.f, dummy = 0.f;
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    // the reference DCHECKs 0 <= label < C (:108-109); an out-of-range label must not read out of bounds
    const int lab = min(max((int)labels[n], 0), C - 1);
    s += -logf(fmaxf(prob[(size_t)n * C + lab], FLT_MIN));
  }
  block_sum2(s, dummy);
  if (threadIdx.x == 0) *loss = s * scale;
}
__global__ void __launch_bounds__(256)
softmax_loss_bwd_kernel(size_t total, int C, const float* __restrict__ prob, const float* __restrict__ labels, float scale,
                        float* __restrict__ dx) {
  pdl_wait();
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t n = i / C;
    const int c = (int)(i - n * C);
    dx[i] = (prob[i] - (c == (int)labels[n] ? 1.f : 0.f)) * scale;
  }
}

// a warp's double sum in a fixed shuffle tree (the loss reductions below)
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- Softmax ------------------------------------------------------------------------------------------------------
// Over the C axis of an [outer, C, inner] view.  inner == 1 runs softmax_loss_fwd_kernel above (alias-safe): one block per row.
// inner > 1: one thread per
// (outer, inner) column (VEC: four adjacent columns), so a warp's loads and stores run along `inner` and coalesce; each column
// takes max, then expf(z - max) and the sum, then the scale, in the row kernel's expressions.  No __restrict__: y may be x.
// softmax_col is the one column (VEC: four columns) the Softmax layer's kernel and SoftmaxWithLoss's column route both compute, so
// their prob agree bit for bit.  z and p point at channel 0 of the column; w is the channel stride in units of V.
template <bool VEC>
__device__ __forceinline__ void softmax_col(const typename std::conditional<VEC, float4, float>::type* z,
                                            typename std::conditional<VEC, float4, float>::type* p, int C, int w) {
  if constexpr (VEC) {
    float4 mx = make_float4(-FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX), s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int c = 0; c < C; ++c) { const float4 v = z[(size_t)c * w]; mx.x = fmaxf(mx.x, v.x); mx.y = fmaxf(mx.y, v.y); mx.z = fmaxf(mx.z, v.z); mx.w = fmaxf(mx.w, v.w); }
    for (int c = 0; c < C; ++c) {
      const float4 v = z[(size_t)c * w];
      const float4 e = make_float4(expf(v.x - mx.x), expf(v.y - mx.y), expf(v.z - mx.z), expf(v.w - mx.w));
      p[(size_t)c * w] = e;
      s.x += e.x; s.y += e.y; s.z += e.z; s.w += e.w;
    }
    const float4 inv = make_float4(1.f / s.x, 1.f / s.y, 1.f / s.z, 1.f / s.w);
    for (int c = 0; c < C; ++c) { float4 e = p[(size_t)c * w]; e.x *= inv.x; e.y *= inv.y; e.z *= inv.z; e.w *= inv.w; p[(size_t)c * w] = e; }
  } else {
    float mx = -FLT_MAX, s = 0.f;
    for (int c = 0; c < C; ++c) mx = fmaxf(mx, z[(size_t)c * w]);
    for (int c = 0; c < C; ++c) { const float e = expf(z[(size_t)c * w] - mx); p[(size_t)c * w] = e; s += e; }
    const float inv = 1.f / s;
    for (int c = 0; c < C; ++c) p[(size_t)c * w] *= inv;
  }
}
template <bool VEC>
__global__ void __launch_bounds__(256) softmax_col_fwd_kernel(size_t cols, int C, int inner, const float* x, float* y) {
  pdl_wait();
  using V = typename std::conditional<VEC, float4, float>::type;
  const int w = VEC ? inner / 4 : inner;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cols; i += (size_t)gridDim.x * blockDim.x) {
    const size_t o = i / w, base = o * C * w + (i - o * w);
    softmax_col<VEC>(reinterpret_cast<const V*>(x) + base, reinterpret_cast<V*>(y) + base, C, w);
  }
}

// ---- SoftmaxWithLoss over spatial positions, with ignore_label and the normalization modes (softmax_loss_layer.cpp) ----------
// A "pixel" is one (outer, inner) column of the [outer, C, inner] view; its label is labels[o * inner + i], a float class id read
// as (int).  Pixels are cut into chunks of SL_CHUNK; chunk k is one CTA, its thread t owns the four pixels 4t .. 4t+3 of the chunk
// and sums their terms as ((t0 + t1) + (t2 + t3)) in double; the CTA then sums its threads with a shuffle tree per warp and the
// warps in order into slot k.  Every slot is a function of the shape and the data alone.
constexpr int SL_CHUNK = 1024;
enum SlRoute { SL_ROW = 0, SL_COL = 1, SL_COL4 = 2 };        // b2c_softmax_loss_route
// the CTA-wide end of the chunk kernels: slot k = the CTA's double sum (threads in a fixed tree) and its integer count
__device__ __forceinline__ void sl_chunk_store(double acc, int cnt, double* __restrict__ part, int* __restrict__ valid) {
  __shared__ double wsum[8];
  __shared__ int wcnt[8];
  acc = warp_sum_d(acc);
#pragma unroll
  for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if ((threadIdx.x & 31) == 0) { wsum[threadIdx.x >> 5] = acc; wcnt[threadIdx.x >> 5] = cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    int n = 0;
    for (int w = 0; w < 8; ++w) { s += wsum[w]; n += wcnt[w]; }
    part[blockIdx.x] = s;
    valid[blockIdx.x] = n;
  }
}
// -log(max(p[label], FLT_MIN)) for one pixel (softmax_loss_layer.cpp:104-115), 0 and not counted when the label is ignored.  An
// out-of-range label that is not ignored reads the nearest class instead, as softmax_loss_sum_kernel does.
__device__ __forceinline__ float sl_term(const float* prob, size_t pix, int C, int inner, const float* labels, int has_ignore,
                                         int ignore_label, int* cnt) {
  const int lab = (int)labels[pix];
  if (has_ignore && lab == ignore_label) return 0.f;
  ++*cnt;
  const size_t o = pix / (size_t)inner, i = pix - o * inner;
  const int l = min(max(lab, 0), C - 1);
  return -logf(fmaxf(prob[(o * C + l) * inner + i], FLT_MIN));
}
// ROUTE SL_ROW: prob is already there (softmax_loss_fwd_kernel); SL_COL: the chunk's softmax first, thread t computing pixels
// t, t + 256, t + 512, t + 768 (softmax_col<false>, so a warp's loads coalesce along inner), then a barrier; SL_COL4: the thread's four
// pixels are one float4 column (inner % 4 == 0, x and prob 16-byte aligned).  Either way the terms are then formed and summed in the
// same order.  No __restrict__ on x / prob: prob elements are read back after they are written.
template <int ROUTE>
__global__ void __launch_bounds__(256)
softmax_loss_chunk_kernel(long long pixels, int C, int inner, const float* x, const float* __restrict__ labels, int has_ignore,
                          int ignore_label, float* prob, double* __restrict__ part, int* __restrict__ valid) {
  pdl_wait();
  const long long p0 = (long long)blockIdx.x * SL_CHUNK + 4 * (long long)threadIdx.x;
  float t[4] = {0.f, 0.f, 0.f, 0.f};
  int cnt = 0;
  if (ROUTE == SL_COL) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const long long pix = (long long)blockIdx.x * SL_CHUNK + k * 256 + threadIdx.x;
      if (pix < pixels) {
        const size_t o = (size_t)pix / inner, base = o * C * inner + ((size_t)pix - o * inner);
        softmax_col<false>(x + base, prob + base, C, inner);
      }
    }
    __syncthreads();                                         // the terms below read prob written by other threads of the CTA
  }
  if (p0 < pixels) {
    if (ROUTE == SL_COL4) {
      const size_t o = (size_t)p0 / inner, base = (o * C * inner + ((size_t)p0 - o * inner)) / 4;
      softmax_col<true>(reinterpret_cast<const float4*>(x) + base, reinterpret_cast<float4*>(prob) + base, C, inner / 4);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const long long pix = p0 + k;
      if (pix >= pixels) break;
      t[k] = sl_term(prob, (size_t)pix, C, inner, labels, has_ignore, ignore_label, &cnt);
    }
  }
  sl_chunk_store(((double)t[0] + (double)t[1]) + ((double)t[2] + (double)t[3]), cnt, part, valid);
}
// One CTA: the slots in index order (thread t sums slots t, t + 256, ... in double, then sl_chunk_store's tree), the normalizer of
// get_normalizer (softmax_loss_layer.cpp:65-92) floored at 1, *loss = (float)sum / normalizer; *normalizer stays on the device for
// the backward.  mode: b2c_loss_normalization.
__global__ void __launch_bounds__(256)
softmax_loss_finalize_kernel(int slots, long long outer, long long pixels, int has_ignore, int mode, const double* __restrict__ part,
                             const int* __restrict__ valid, float* __restrict__ loss, float* __restrict__ normalizer) {
  pdl_wait();
  double acc = 0.0;
  long long n = 0;
  for (int s = threadIdx.x; s < slots; s += 256) { acc += part[s]; n += valid[s]; }
  __shared__ double wsum[8];
  __shared__ long long wcnt[8];
  acc = warp_sum_d(acc);
#pragma unroll
  for (int o = 16; o; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
  if ((threadIdx.x & 31) == 0) { wsum[threadIdx.x >> 5] = acc; wcnt[threadIdx.x >> 5] = n; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    long long v = 0;
    for (int w = 0; w < 8; ++w) { s += wsum[w]; v += wcnt[w]; }
    float norm = 1.f;
    if (mode == B2C_LOSS_NORM_FULL) norm = (float)pixels;
    else if (mode == B2C_LOSS_NORM_VALID) norm = has_ignore ? (float)v : (float)pixels;
    else if (mode == B2C_LOSS_NORM_BATCH_SIZE) norm = (float)outer;
    norm = fmaxf(1.f, norm);
    *normalizer = norm;
    *loss = (float)s / norm;
  }
}
// dx = (prob - onehot) * s, s = loss_weight / *normalizer rounded once per thread; every channel of an ignored pixel is 0.  An
// out-of-range label subtracts nothing.  Column route: one thread per pixel column (VEC: four, float4 along inner); row route
// (inner == 1): one thread per element.
template <bool VEC>
__global__ void __launch_bounds__(256)
softmax_loss_bwd_col_kernel(size_t cols, int C, int inner, const float* __restrict__ prob, const float* __restrict__ labels, int has_ignore,
                            int ignore_label, const float* __restrict__ normalizer, float loss_weight, float* __restrict__ dx) {
  pdl_wait();
  using V = typename std::conditional<VEC, float4, float>::type;
  const float s = loss_weight / *normalizer;
  const int w = VEC ? inner / 4 : inner;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cols; i += (size_t)gridDim.x * blockDim.x) {
    const size_t o = i / w, base = o * C * w + (i - o * w);
    const V* p = reinterpret_cast<const V*>(prob) + base;
    V* d = reinterpret_cast<V*>(dx) + base;
    if constexpr (VEC) {
      const float4 lf = reinterpret_cast<const float4*>(labels)[i];
      const int l0 = (int)lf.x, l1 = (int)lf.y, l2 = (int)lf.z, l3 = (int)lf.w;
      const bool k0 = !(has_ignore && l0 == ignore_label), k1 = !(has_ignore && l1 == ignore_label),
                 k2 = !(has_ignore && l2 == ignore_label), k3 = !(has_ignore && l3 == ignore_label);
      for (int c = 0; c < C; ++c) {
        const float4 v = p[(size_t)c * w];
        d[(size_t)c * w] = make_float4(k0 ? __fmul_rn(v.x - (c == l0 ? 1.f : 0.f), s) : 0.f, k1 ? __fmul_rn(v.y - (c == l1 ? 1.f : 0.f), s) : 0.f,
                                       k2 ? __fmul_rn(v.z - (c == l2 ? 1.f : 0.f), s) : 0.f, k3 ? __fmul_rn(v.w - (c == l3 ? 1.f : 0.f), s) : 0.f);
      }
    } else {
      const int l = (int)labels[i];
      const bool keep = !(has_ignore && l == ignore_label);
      for (int c = 0; c < C; ++c) d[(size_t)c * w] = keep ? __fmul_rn(p[(size_t)c * w] - (c == l ? 1.f : 0.f), s) : 0.f;
    }
  }
}
__global__ void __launch_bounds__(256)
softmax_loss_bwd_row_kernel(size_t total, int C, const float* __restrict__ prob, const float* __restrict__ labels, int has_ignore,
                            int ignore_label, const float* __restrict__ normalizer, float loss_weight, float* __restrict__ dx) {
  pdl_wait();
  const float s = loss_weight / *normalizer;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t n = i / C;
    const int c = (int)(i - n * C), l = (int)labels[n];
    dx[i] = (has_ignore && l == ignore_label) ? 0.f : __fmul_rn(prob[i] - (c == l ? 1.f : 0.f), s);
  }
}
// dx = (dy - sum_c dy * y) * y  (softmax_layer.cu: channel dot, channel subtract, multiply by the top).  dx may be dy.
__global__ void __launch_bounds__(256) softmax_row_bwd_kernel(int C, const float* y, const float* dy, float* dx) {
  pdl_wait();
  const size_t off = (size_t)blockIdx.x * C;
  float dot = 0.f, dummy = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) dot += dy[off + c] * y[off + c];
  block_sum2(dot, dummy);                          // (ends on a barrier: every dy read is done before dx may overwrite it)
  for (int c = threadIdx.x; c < C; c += blockDim.x) dx[off + c] = (dy[off + c] - dot) * y[off + c];
}
template <bool VEC>
__global__ void __launch_bounds__(256) softmax_col_bwd_kernel(size_t cols, int C, int inner, const float* y, const float* dy, float* dx) {
  pdl_wait();
  using V = typename std::conditional<VEC, float4, float>::type;
  const int w = VEC ? inner / 4 : inner;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cols; i += (size_t)gridDim.x * blockDim.x) {
    const size_t o = i / w, base = o * C * w + (i - o * w);
    const V* yv = reinterpret_cast<const V*>(y) + base;
    const V* dv = reinterpret_cast<const V*>(dy) + base;
    V* xv = reinterpret_cast<V*>(dx) + base;
    if constexpr (VEC) {
      float4 d = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int c = 0; c < C; ++c) {
        const float4 a = dv[(size_t)c * w], b = yv[(size_t)c * w];
        d.x += a.x * b.x; d.y += a.y * b.y; d.z += a.z * b.z; d.w += a.w * b.w;
      }
      for (int c = 0; c < C; ++c) {
        const float4 a = dv[(size_t)c * w], b = yv[(size_t)c * w];
        xv[(size_t)c * w] = make_float4((a.x - d.x) * b.x, (a.y - d.y) * b.y, (a.z - d.z) * b.z, (a.w - d.w) * b.w);
      }
    } else {
      float d = 0.f;
      for (int c = 0; c < C; ++c) d += dv[(size_t)c * w] * yv[(size_t)c * w];
      for (int c = 0; c < C; ++c) xv[(size_t)c * w] = (dv[(size_t)c * w] - d) * yv[(size_t)c * w];
    }
  }
}

// ---- Sigmoid, SigmoidCrossEntropyLoss, EuclideanLoss, L1Loss ---------------------------------------------------------------
// sigmoid_layer.cu:9-13.  The one expression b2c_sigmoid_forward and b2c_sigmoid_ce_loss_backward share.
__device__ __forceinline__ float sigmoid_of(float x) { return 1.f / (1.f + expf(-x)); }

enum EwOp { EW_SIGMOID_FWD, EW_SIGMOID_BWD, EW_SIGCE_BWD, EW_SCALE, EW_SIGN_SCALE };
// y = op(a, b, s) per element: SIGMOID_FWD sigmoid(a); SIGMOID_BWD b * a * (1 - a) with a = y, b = dy; SIGCE_BWD (sigmoid(a) - b) * s;
// SCALE s * a; SIGN_SCALE s * sign(a) with sign(0) = sign(NaN) = 0, and +0 there (caffe_gpu_sign, then axpby's 0 * y + s * sign).
// In place allowed (no __restrict__)
template <int OP>
__device__ __forceinline__ float ew_apply(float a, float b, float s) {
  if (OP == EW_SIGMOID_FWD) return sigmoid_of(a);
  if (OP == EW_SIGMOID_BWD) return b * a * (1.f - a);
  if (OP == EW_SIGCE_BWD) return __fmul_rn(sigmoid_of(a) - b, s);
  if (OP == EW_SIGN_SCALE) return a > 0.f ? s : a < 0.f ? -s : 0.f;
  return s * a;
}
template <int OP>
__global__ void __launch_bounds__(256) ew_kernel(size_t n, int vec, const float* a, const float* b, float s, float* y) {
  pdl_wait();
  const size_t n4 = vec ? n / 4 : 0, tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  const bool two = OP == EW_SIGMOID_BWD || OP == EW_SIGCE_BWD;
  for (size_t i = tid; i < n4; i += step) {
    const float4 u = reinterpret_cast<const float4*>(a)[i];
    const float4 v = two ? reinterpret_cast<const float4*>(b)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    reinterpret_cast<float4*>(y)[i] = make_float4(ew_apply<OP>(u.x, v.x, s), ew_apply<OP>(u.y, v.y, s), ew_apply<OP>(u.z, v.z, s), ew_apply<OP>(u.w, v.w, s));
  }
  for (size_t i = n4 * 4 + tid; i < n; i += step) y[i] = ew_apply<OP>(a[i], two ? b[i] : 0.f, s);
}

// Loss sums: ONE thread-block cluster of LOSS_THREADS-thread CTAs (bn_stats_kernel's pattern: each CTA sums a contiguous slice, the
// CTA sums meet in rank 0 through distributed shared memory in rank order; no atomics, no scratch, one launch).  The cluster size
// depends only on `count`, so the summation order -- and the bits -- are the same on every call.  Terms are computed in float and
// summed in double; the float result is formed once at the end.
//   MODE 0 (SigmoidCrossEntropyLoss): term = x (t - [x >= 0]) - log(1 + exp(x - 2 x [x >= 0])), loss = -sum / N
//   MODE 1 (EuclideanLoss):           d = a - b stored to diff, term = d * d, loss = sum / N / 2
//   MODE 2 (L1Loss):                  d = a - b stored to diff, term = |d|,  loss = sum / N
constexpr int LOSS_THREADS = 512;
constexpr int LOSS_CLUSTER = 8;                    // the portable cluster limit
template <int MODE>
__device__ __forceinline__ float loss_term(float a, float b, float* d) {
  if (MODE == 0) {
    const float pos = a >= 0.f ? 1.f : 0.f;
    return a * (b - pos) - logf(1.f + expf(a - 2.f * a * pos));
  }
  const float v = a - b;
  *d = v;
  return MODE == 1 ? __fmul_rn(v, v) : fabsf(v);
}
// The reduction every loss-sum kernel ends with: each thread's double partial is summed per warp, the warp sums per CTA in warp
// order, and the CTA sums over the cluster in rank order in rank 0 through distributed shared memory.  Returns the total in rank 0's
// thread 0 (0 elsewhere).  Every thread of every CTA of the cluster must call it.
__device__ __forceinline__ double loss_cluster_sum(double acc) {
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned rank = cluster.block_rank(), nranks = cluster.num_blocks();
  __shared__ double wsum[LOSS_THREADS / 32];
  __shared__ double part;
  acc = warp_sum_d(acc);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < LOSS_THREADS / 32; ++w) s += wsum[w];
    part = s;
  }
  cluster.sync();
  double s = 0.0;
  if (rank == 0 && threadIdx.x == 0)
    for (unsigned r = 0; r < nranks; ++r) s += *cluster.map_shared_rank(&part, r);
  cluster.sync();                                   // remote shared memory stays valid until rank 0 has read it
  return s;
}
template <int MODE, bool VEC>
__global__ void __launch_bounds__(LOSS_THREADS)
loss_sum_kernel(size_t count, int N, const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ diff, float* __restrict__ loss) {
  pdl_wait();
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned rank = cluster.block_rank(), nranks = cluster.num_blocks();
  const size_t units = VEC ? count / 4 : count, len = (units + nranks - 1) / nranks;
  const size_t lo = rank * len < units ? rank * len : units, hi = lo + len < units ? lo + len : units;
  double acc = 0.0;
  for (size_t i = lo + threadIdx.x; i < hi; i += LOSS_THREADS) {
    if (VEC) {
      const float4 u = reinterpret_cast<const float4*>(a)[i], v = reinterpret_cast<const float4*>(b)[i];
      float4 d;
      const float t0 = loss_term<MODE>(u.x, v.x, &d.x), t1 = loss_term<MODE>(u.y, v.y, &d.y);
      const float t2 = loss_term<MODE>(u.z, v.z, &d.z), t3 = loss_term<MODE>(u.w, v.w, &d.w);
      if (MODE != 0) reinterpret_cast<float4*>(diff)[i] = d;
      acc += ((double)t0 + (double)t1) + ((double)t2 + (double)t3);
    } else {
      float d;
      const float t = loss_term<MODE>(a[i], b[i], &d);
      if (MODE != 0) diff[i] = d;
      acc += (double)t;
    }
  }
  if (VEC && rank == 0 && threadIdx.x < count % 4) {        // the float4 pass's tail
    const size_t i = units * 4 + threadIdx.x;
    float d;
    const float t = loss_term<MODE>(a[i], b[i], &d);
    if (MODE != 0) diff[i] = d;
    acc += (double)t;
  }
  const double s = loss_cluster_sum(acc);
  if (rank == 0 && threadIdx.x == 0) {
    const float f = (float)s;
    *loss = MODE == 0 ? -f / (float)N : MODE == 1 ? f / (float)N / 2.f : f / (float)N;
  }
}
// ContrastiveLoss (contrastive_loss_layer.cpp): one warp per pair, the lanes strided over the channels; the pair's squared distance
// is summed in double (lane partials, then warp_sum_d) and stored as float, its term formed in float and summed by
// loss_cluster_sum.  Pairs are split into contiguous CTA slices like loss_sum_kernel's units.
template <bool LEGACY>
__global__ void __launch_bounds__(LOSS_THREADS)
contrastive_loss_kernel(int N, int C, const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ y, float margin,
                        float* __restrict__ diff, float* __restrict__ dist_sq, float* __restrict__ loss) {
  pdl_wait();
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned rank = cluster.block_rank(), nranks = cluster.num_blocks();
  const int len = (int)((N + nranks - 1) / nranks);
  const int lo = min(N, (int)rank * len), hi = min(N, lo + len);
  const int lane = threadIdx.x & 31;
  double acc = 0.0;
  for (int n = lo + (int)(threadIdx.x >> 5); n < hi; n += LOSS_THREADS / 32) {
    const size_t base = (size_t)n * C;
    double s = 0.0;
    for (int c = lane; c < C; c += 32) {
      const float d = a[base + c] - b[base + c];
      diff[base + c] = d;
      s += (double)__fmul_rn(d, d);
    }
    s = warp_sum_d(s);
    if (lane == 0) {
      const float d2 = (float)s;
      dist_sq[n] = d2;
      float term;
      if ((int)y[n]) term = d2;                                    // similar pair
      else if (LEGACY) term = fmaxf(margin - d2, 0.f);
      else { const float m = fmaxf(margin - sqrtf(d2), 0.f); term = __fmul_rn(m, m); }
      acc += (double)term;
    }
  }
  const double s = loss_cluster_sum(acc);
  if (rank == 0 && threadIdx.x == 0) *loss = (float)s / (float)N / 2.f;
}
// the per-pair factor of ContrastiveLoss's backward (contrastive_loss_layer.cpp Backward_cpu); *zero: the pair's gradient is 0
__device__ __forceinline__ float contrastive_coef(float d2, float yv, float margin, int legacy, float alpha, bool* zero) {
  *zero = false;
  if ((int)yv) return alpha;
  if (legacy) { *zero = !(margin - d2 > 0.f); return -alpha; }
  const float dist = sqrtf(d2), mdist = margin - dist;
  *zero = !(mdist > 0.f);
  return -alpha * mdist / (dist + 1e-4f);
}
template <bool VEC>
__global__ void __launch_bounds__(256)
contrastive_bwd_kernel(int N, int C, const float* __restrict__ diff, const float* __restrict__ dist_sq, const float* __restrict__ y, float margin,
                       int legacy, float alpha, float* __restrict__ da, float* __restrict__ db) {
  pdl_wait();
  const size_t units = VEC ? (size_t)N * C / 4 : (size_t)N * C, tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x,
               step = (size_t)gridDim.x * blockDim.x;
  for (size_t i = tid; i < units; i += step) {
    const size_t n = (VEC ? i * 4 : i) / (size_t)C;
    bool zero;
    const float k = contrastive_coef(dist_sq[n], y[n], margin, legacy, alpha, &zero);
    if (VEC) {
      const float4 d = reinterpret_cast<const float4*>(diff)[i];
      const float4 g = zero ? make_float4(0.f, 0.f, 0.f, 0.f) : make_float4(__fmul_rn(k, d.x), __fmul_rn(k, d.y), __fmul_rn(k, d.z), __fmul_rn(k, d.w));
      reinterpret_cast<float4*>(da)[i] = g;
      if (db) reinterpret_cast<float4*>(db)[i] = zero ? g : make_float4(-g.x, -g.y, -g.z, -g.w);
    } else {
      const float g = zero ? 0.f : __fmul_rn(k, diff[i]);
      da[i] = g;
      if (db) db[i] = zero ? 0.f : -g;
    }
  }
}
// CTAs per loss cluster: one per 64K float4 units (256K values), at most LOSS_CLUSTER.  A function of the count alone.
static inline unsigned loss_cluster_size(size_t count) {
  unsigned cs = 1;
  while (cs < LOSS_CLUSTER && count / (cs * 2) >= (1u << 18)) cs *= 2;
  return cs;
}

}  // namespace b2c

using namespace b2c;
#define NEED(cond, msg) if (!(cond)) return fail(B2C_ERR_INVALID, msg)

extern "C" int b2c_relu_forward(size_t n, const float* x, float* y, float negative_slope, void* stream) {
  NEED(x && y, "b2c_relu_forward: null");
  if (!n) return B2C_OK;
  const bool al = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0;     // else one float at a time
  launch_pdl(relu_fwd_kernel, grid_for(al ? (n + 3) / 4 : n, 256), 256, 0, as_stream(stream), 0, n, al ? 1 : 0, x, y, negative_slope);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
extern "C" int b2c_relu_backward(size_t n, const float* dy, const float* x, float* dx, float negative_slope, void* stream) {
  NEED(dy && x && dx, "b2c_relu_backward: null");
  if (!n) return B2C_OK;
  const bool al = ((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dx)) & 15) == 0;
  launch_pdl(relu_bwd_kernel, grid_for(al ? (n + 3) / 4 : n, 256), 256, 0, as_stream(stream), 0, n, al ? 1 : 0, dy, x, dx, negative_slope);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
template <typename... Args>
static void launch_clustered(void (*kernel)(Args...), unsigned cs, int C, void* stream, unsigned threads, Args... args) {
  bn_launch_clustered(kernel, cs, C, 0, stream, threads, args...);
}
namespace b2c {
int launch_bn_stats(const BnPlan& p, int N, int C, int S, const float* x, float eps, float maf, int first, float* mean, float* invstd,
                    float* run_mean, float* run_var, void* stream) {
  launch_clustered(p.vec ? bn_stats_kernel<true> : bn_stats_kernel<false>, p.cs, C, stream, p.threads, N, C, S, x, eps, maf, first, mean, invstd, run_mean, run_var);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
}  // namespace b2c
extern "C" int b2c_bn_forward_train(int N, int C, int S, const float* x, const float* gamma, const float* beta, float eps,
                                    float moving_average_fraction, int first_iteration, float* running_mean, float* running_var,
                                    float* save_mean, float* save_invstd, float* xnorm, float* y, void* stream) {
  NEED(x && y && xnorm && save_mean && save_invstd && running_mean && running_var, "b2c_bn_forward_train: bad argument");
  NEED((gamma == nullptr) == (beta == nullptr), "b2c_bn_forward_train: gamma and beta go together");
  BnPlan pl;
  if (int rc = bn_plan(0, 0, N, C, S, {x, y, xnorm}, "b2c_bn_forward_train", &pl)) return rc;
  const bool vec = pl.vec;
  if (int rc = launch_bn_stats(pl, N, C, S, x, eps, moving_average_fraction, first_iteration, save_mean, save_invstd, running_mean, running_var, stream)) return rc;
  const size_t units = (size_t)N * C * (vec ? S / 4 : S);
  const unsigned blocks = (unsigned)((units + 256 * BN_EW_PER_THREAD - 1) / (256 * BN_EW_PER_THREAD));
  if (vec) launch_pdl(bn_norm_kernel<true>, blocks, 256, 0, as_stream(stream), 0, units, C, S, x, save_mean, save_invstd, gamma, beta, xnorm, y);
  else launch_pdl(bn_norm_kernel<false>, blocks, 256, 0, as_stream(stream), 0, units, C, S, x, save_mean, save_invstd, gamma, beta, xnorm, y);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
extern "C" int b2c_bn_backward(int N, int C, int S, const float* dy, const float* xnorm, const float* gamma, const float* save_invstd,
                               float* dgamma, float* dbeta, float* dx, void* stream) {
  NEED(dy && xnorm && save_invstd && dgamma && dbeta && dx, "b2c_bn_backward: null (dgamma/dbeta double as the reduction scratch)");
  BnPlan pl;
  if (int rc = bn_plan(1, 0, N, C, S, {dy, xnorm, dx}, "b2c_bn_backward", &pl)) return rc;
  const bool vec = pl.vec;
  launch_clustered(vec ? bn_bwd_reduce_kernel<true> : bn_bwd_reduce_kernel<false>, pl.cs, C, stream, pl.threads, N, C, S, dy, xnorm, dgamma, dbeta);
  B2C_POST_LAUNCH();
  const size_t units = (size_t)N * C * (vec ? S / 4 : S);
  const unsigned blocks = (unsigned)((units + 256 * BN_EW_PER_THREAD - 1) / (256 * BN_EW_PER_THREAD));
  const float inv_cnt = 1.0f / ((float)N * S);
  if (vec) launch_pdl(bn_bwd_dx_kernel<true>, blocks, 256, 0, as_stream(stream), 0, units, C, S, inv_cnt, dy, xnorm, gamma, save_invstd, dgamma, dbeta, dx);
  else launch_pdl(bn_bwd_dx_kernel<false>, blocks, 256, 0, as_stream(stream), 0, units, C, S, inv_cnt, dy, xnorm, gamma, save_invstd, dgamma, dbeta, dx);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
extern "C" int b2c_lrn_forward(int N, int C, int S, int local_size, float alpha, float beta, float k, const float* x, float* scale,
                               float* y, void* stream) {
  NEED(x && scale && y && N > 0 && C > 0 && S > 0 && local_size > 0 && (local_size & 1), "b2c_lrn_forward: bad argument (LRN only supports odd values for local_size)");
  launch_pdl(lrn_fwd_kernel, grid_for((size_t)N * S, 256), 256, 0, as_stream(stream), 0, N, C, S, local_size, alpha / local_size, beta, k, x, scale, y);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
extern "C" int b2c_lrn_backward(int N, int C, int S, int local_size, float alpha, float beta, const float* x, const float* y,
                                const float* scale, const float* dy, float* dx, void* stream) {
  NEED(x && y && scale && dy && dx && N > 0 && C > 0 && S > 0 && local_size > 0, "b2c_lrn_backward: bad argument");
  launch_pdl(lrn_bwd_kernel, grid_for((size_t)N * S, 256), 256, 0, as_stream(stream), 0, N, C, S, local_size, 2.f * alpha * beta / local_size, beta, x, y, scale, dy, dx);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
extern "C" int b2c_dropout_mask(size_t n, float ratio, unsigned long long seed, unsigned long long offset, float* mask, void* stream) {
  NEED(mask && ratio >= 0.f && ratio < 1.f, "b2c_dropout_mask: dropout_ratio must be in [0, 1)");
  if (!n) return B2C_OK;
  const unsigned thr = (unsigned)((double)ratio * 16777216.0);
  launch_pdl(dropout_mask_kernel, grid_for(n, 256), 256, 0, as_stream(stream), 0, n, thr, 1.0f / (1.0f - ratio), seed, offset, mask);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
extern "C" int b2c_mul(size_t n, const float* a, const float* b, float* y, void* stream) {
  NEED(a && b && y, "b2c_mul: null");
  if (!n) return B2C_OK;
  NEED(((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(y)) & 15) == 0, "b2c_mul: pointers must be 16-byte aligned");
  launch_pdl(mul_kernel, grid_for((n + 3) / 4, 256), 256, 0, as_stream(stream), 0, n, a, b, y);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
// PoolingLayer::Reshape's ceil-mode extent (pooling_layer.cpp:92-107), for arguments pool_route has checked
static int pool_out(int in, int k, int s, int p) {
  int o = (int)ceilf((float)(in + 2 * p - k) / s) + 1;
  if (p > 0 && (o - 1) * s >= in + p) --o;
  return o;
}
struct PoolRoute { int route, Ho, Wo, q, rpb; };
// The one place that picks the pooling kernel; b2c_pool_forward / b2c_pool_backward launch what it returns and b2c_debug_pool_plan
// reports it.  dir 0 = forward (out = y, mask = the MAX mask), 1 = backward (out = dx).  Pointers are compared, never dereferenced.
// The argument checks are PoolingLayer::LayerSetUp's and Reshape's (pooling_layer.cpp:51-52,75-76), plus non-empty maps.
static int pool_route(int method, int dir, int NC, int H, int W, int kh, int kw, int sh, int sw, int ph, int pw, const void* out,
                      const void* mask, PoolRoute* r) {
  NEED(method == 0 || method == 1, "pooling: STOCHASTIC pooling is outside this path");
  NEED(dir == 0 || dir == 1, "pooling: dir must be 0 (forward) or 1 (backward)");
  NEED(NC > 0 && H > 0 && W > 0, "pooling: empty input");
  NEED(kh > 0 && kw > 0, "pooling: Filter dimensions cannot be zero.");
  NEED(sh > 0 && sw > 0, "pooling: stride must be positive");
  NEED(ph >= 0 && pw >= 0 && ph < kh && pw < kw, "pooling: pad must lie in [0, kernel)");
  *r = PoolRoute{B2C_POOL_ROUTE_AVE, pool_out(H, kh, sh, ph), pool_out(W, kw, sw, pw), 0, 0};
  NEED(r->Ho >= 1 && r->Wo >= 1, "pooling: the kernel is larger than the padded input");
  if (method == 1) return B2C_OK;
  const bool common = kh == kw && sh == sw && ((kh == 3 && sh == 2) || (kh == 2 && sh == 2) || (kh == 3 && sh == 1));
  if (dir == 0) {
    const int q = r->Wo % 4 == 0 ? 4 : r->Wo % 2 == 0 ? 2 : 0;
    const uintptr_t al = reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(mask);
    if (common && q && (al & (q == 4 ? 15 : 7)) == 0) { r->route = B2C_POOL_ROUTE_MAX_WINDOW; r->q = q; }
    else r->route = B2C_POOL_ROUTE_MAX_SCALAR;
    return B2C_OK;
  }
  NEED((long long)NC * H < 0x7fffffffLL, "b2c_pool_backward: too many rows");
  if (common && W % 4 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0) r->route = B2C_POOL_ROUTE_MAX_BWD_QUAD;
  else { r->route = B2C_POOL_ROUTE_MAX_BWD_ROW; r->rpb = W >= 128 ? 1 : 128 / W; }
  return B2C_OK;
}
extern "C" int b2c_debug_pool_plan(int method, int dir, int NC, int H, int W, int kh, int kw, int sh, int sw, int ph, int pw,
                                   const void* out_ptr, const void* mask_ptr, int* out, int n) {
  NEED(out && n >= 5, "b2c_debug_pool_plan: needs out[5]");
  PoolRoute r;
  if (int rc = pool_route(method, dir, NC, H, W, kh, kw, sh, sw, ph, pw, out_ptr, mask_ptr, &r)) return rc;
  out[0] = r.route; out[1] = r.Ho; out[2] = r.Wo; out[3] = r.q; out[4] = r.rpb;
  return B2C_OK;
}
extern "C" int b2c_pool_forward(int method, int NC, int H, int W, int kh, int kw, int sh, int sw, int ph, int pw, const float* x,
                                float* y, int* mask, void* stream) {
  NEED(x && y, "b2c_pool_forward: null");
  NEED(mask || method != 0, "b2c_pool_forward: MAX needs a mask buffer");
  PoolRoute r;
  if (int rc = pool_route(method, 0, NC, H, W, kh, kw, sh, sw, ph, pw, y, mask, &r)) return rc;
  const int Ho = r.Ho, Wo = r.Wo;
  const size_t total = (size_t)NC * Ho * Wo;
  cudaStream_t s_ = as_stream(stream);
  if (r.route == B2C_POOL_ROUTE_MAX_WINDOW) {
    const int q = r.q;
    const long long groups = (long long)NC * Ho * (Wo / q);
    const unsigned grid = grid_for((size_t)groups, 256);
#define B2C_POOLF(KH, S, Q) launch_pdl(pool_max_fwd_q_kernel<KH, KH, S, S, Q>, grid, 256, 0, s_, 0, groups, H, W, Ho, Wo, ph, pw, x, y, mask)
    if (kh == 3 && sh == 2) { if (q == 4) B2C_POOLF(3, 2, 4); else B2C_POOLF(3, 2, 2); }
    else if (kh == 2) { if (q == 4) B2C_POOLF(2, 2, 4); else B2C_POOLF(2, 2, 2); }
    else { if (q == 4) B2C_POOLF(3, 1, 4); else B2C_POOLF(3, 1, 2); }
#undef B2C_POOLF
  } else if (r.route == B2C_POOL_ROUTE_MAX_SCALAR) {
    launch_pdl(pool_max_fwd_kernel, grid_for(total, 256), 256, 0, s_, 0, total, H, W, Ho, Wo, kh, kw, sh, sw, ph, pw, x, y, mask);
  } else {
    launch_pdl(pool_ave_fwd_kernel, grid_for(total, 256), 256, 0, s_, 0, total, H, W, Ho, Wo, kh, kw, sh, sw, ph, pw, x, y);
  }
  B2C_POST_LAUNCH();
  return B2C_OK;
}
extern "C" int b2c_pool_backward(int method, int NC, int H, int W, int kh, int kw, int sh, int sw, int ph, int pw, const float* dy,
                                 const int* mask, float* dx, void* stream) {
  NEED(dy && dx, "b2c_pool_backward: null");
  NEED(mask || method != 0, "b2c_pool_backward: MAX needs the forward mask");
  PoolRoute r;
  if (int rc = pool_route(method, 1, NC, H, W, kh, kw, sh, sw, ph, pw, dx, mask, &r)) return rc;
  const int Ho = r.Ho, Wo = r.Wo;
  cudaStream_t s_ = as_stream(stream);
  if (r.route == B2C_POOL_ROUTE_MAX_BWD_QUAD) {
    const long long quads = (long long)NC * H * (W / 4);
    const unsigned grid = grid_for((size_t)quads, 256);
    if (kh == 3 && sh == 2) launch_pdl(pool_max_bwd_q4_kernel<3, 3, 2, 2>, grid, 256, 0, s_, 0, quads, H, W, Ho, Wo, ph, pw, dy, mask, dx);
    else if (kh == 2) launch_pdl(pool_max_bwd_q4_kernel<2, 2, 2, 2>, grid, 256, 0, s_, 0, quads, H, W, Ho, Wo, ph, pw, dy, mask, dx);
    else launch_pdl(pool_max_bwd_q4_kernel<3, 3, 1, 1>, grid, 256, 0, s_, 0, quads, H, W, Ho, Wo, ph, pw, dy, mask, dx);
  } else if (r.route == B2C_POOL_ROUTE_MAX_BWD_ROW) {
    const long long rows = (long long)NC * H;
    const long long groups = (rows + r.rpb - 1) / r.rpb;
    const int grid = (int)(groups < (long long)sm_count() * 64 ? groups : (long long)sm_count() * 64);
    launch_pdl(pool_max_bwd_kernel, grid, 128, 0, s_, 0, (int)rows, H, W, Ho, Wo, kh, kw, sh, sw, ph, pw, dy, mask, dx);
  } else {
    const size_t total = (size_t)NC * H * W;
    launch_pdl(pool_ave_bwd_kernel, grid_for(total, 256), 256, 0, s_, 0, total, H, W, Ho, Wo, kh, kw, sh, sw, ph, pw, dy, dx);
  }
  B2C_POST_LAUNCH();
  return B2C_OK;
}
// dst[c][r] = src[r][c]: 32 x 32 tiles through shared memory (padded: conflict-free both ways), coalesced reads and writes
__global__ void __launch_bounds__(256)
transpose_kernel(int rows, int cols, const float* __restrict__ src, float* __restrict__ dst) {
  pdl_wait();
  __shared__ float tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;             // 32 x 8 threads
  const long long c0 = (long long)blockIdx.x * 32, r0 = (long long)blockIdx.y * 32;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const long long r = r0 + ty + 8 * j, c = c0 + tx;
    if (r < rows && c < cols) tile[ty + 8 * j][tx] = src[r * cols + c];
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const long long c = c0 + ty + 8 * j, r = r0 + tx;
    if (r < rows && c < cols) dst[c * rows + r] = tile[tx][ty + 8 * j];
  }
}
extern "C" int b2c_transpose(int rows, int cols, const float* src, float* dst, void* stream) {
  NEED(src && dst && rows > 0 && cols > 0 && src != dst, "b2c_transpose: bad argument");
  dim3 grid((cols + 31) / 32, (rows + 31) / 32);
  NEED(grid.y <= 65535, "b2c_transpose: too many rows");
  launch_pdl(transpose_kernel, grid, 256, 0, as_stream(stream), 0, rows, cols, src, dst);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
extern "C" int b2c_add(size_t n, const float* a, const float* b, float* y, void* stream) {
  NEED(a && b && y, "b2c_add: null");
  if (!n) return B2C_OK;
  const bool al = ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(y)) & 15) == 0;
  launch_pdl(add_kernel, grid_for(al ? (n + 3) / 4 : n, 256), 256, 0, as_stream(stream), 0, n, al ? 1 : 0, a, b, y);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
extern "C" int b2c_softmax_loss_forward(int N, int C, const float* logits, const float* labels, float* prob, float* loss, void* stream) {
  NEED(logits && labels && prob && loss && N > 0 && C > 0, "b2c_softmax_loss_forward: bad argument");
  launch_pdl(softmax_loss_fwd_kernel, N, 256, 0, as_stream(stream), 0, C, logits, prob);
  B2C_POST_LAUNCH();
  launch_pdl(softmax_loss_sum_kernel, 1, 256, 0, as_stream(stream), 0, N, C, prob, labels, 1.0f / (float)N, loss);   // VALID normalisation, no ignore_label
  B2C_POST_LAUNCH();
  return B2C_OK;
}
extern "C" int b2c_softmax_loss_backward(int N, int C, const float* prob, const float* labels, float loss_weight, float* dx, void* stream) {
  NEED(prob && labels && dx && N > 0 && C > 0, "b2c_softmax_loss_backward: bad argument");
  const size_t total = (size_t)N * C;
  launch_pdl(softmax_loss_bwd_kernel, grid_for(total, 256), 256, 0, as_stream(stream), 0, total, C, prob, labels, loss_weight / (float)N, dx);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
static bool al16(std::initializer_list<const void*> ptrs) {
  for (const void* p : ptrs) if (reinterpret_cast<uintptr_t>(p) & 15) return false;
  return true;
}
extern "C" int b2c_softmax_forward(int outer, int C, int inner, const float* x, float* y, void* stream) {
  NEED(x && y && outer > 0 && C > 0 && inner > 0, "b2c_softmax_forward: bad argument");
  if (inner == 1) {                                // every [N, C] use: SoftmaxWithLoss's row kernel, so prob and this top agree bit for bit
    launch_pdl(softmax_loss_fwd_kernel, outer, 256, 0, as_stream(stream), 0, C, x, y);
    B2C_POST_LAUNCH();
    return B2C_OK;
  }
  const bool vec = inner % 4 == 0 && al16({x, y});
  const size_t cols = (size_t)outer * (vec ? inner / 4 : inner);
  if (vec) launch_pdl(softmax_col_fwd_kernel<true>, grid_for(cols, 256), 256, 0, as_stream(stream), 0, cols, C, inner, x, y);
  else launch_pdl(softmax_col_fwd_kernel<false>, grid_for(cols, 256), 256, 0, as_stream(stream), 0, cols, C, inner, x, y);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
extern "C" int b2c_softmax_backward(int outer, int C, int inner, const float* y, const float* dy, float* dx, void* stream) {
  NEED(y && dy && dx && outer > 0 && C > 0 && inner > 0, "b2c_softmax_backward: bad argument");
  if (inner == 1) {
    launch_pdl(softmax_row_bwd_kernel, outer, 256, 0, as_stream(stream), 0, C, y, dy, dx);
    B2C_POST_LAUNCH();
    return B2C_OK;
  }
  const bool vec = inner % 4 == 0 && al16({y, dy, dx});
  const size_t cols = (size_t)outer * (vec ? inner / 4 : inner);
  if (vec) launch_pdl(softmax_col_bwd_kernel<true>, grid_for(cols, 256), 256, 0, as_stream(stream), 0, cols, C, inner, y, dy, dx);
  else launch_pdl(softmax_col_bwd_kernel<false>, grid_for(cols, 256), 256, 0, as_stream(stream), 0, cols, C, inner, y, dy, dx);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
struct SoftmaxLossPlan { int route; long long pixels, slots; size_t ws_bytes; };
// The one place the softmax-loss forward route is chosen: b2c_softmax_loss_forward_ex launches it, the plan query reports it.
static int softmax_loss_plan(int outer, int C, int inner, const void* logits, const void* prob, SoftmaxLossPlan* pl) {
  NEED(outer > 0 && C > 0 && inner > 0, "softmax loss: outer, C and inner must be positive");
  NEED((long long)outer * inner <= (1ll << 62) / C, "softmax loss: tensor too large");
  pl->pixels = (long long)outer * inner;
  pl->slots = (pl->pixels + SL_CHUNK - 1) / SL_CHUNK;
  NEED(pl->slots <= 0x7fffffffLL, "softmax loss: too many pixels");
  pl->route = inner == 1 ? SL_ROW : inner % 4 == 0 && al16({logits, prob}) ? SL_COL4 : SL_COL;
  pl->ws_bytes = ((size_t)pl->slots * (sizeof(double) + sizeof(int)) + 15) / 16 * 16;
  return B2C_OK;
}
extern "C" int b2c_softmax_loss_workspace(int outer, int C, int inner, size_t* bytes) {
  NEED(bytes, "b2c_softmax_loss_workspace: null");
  SoftmaxLossPlan pl{};
  if (int rc = softmax_loss_plan(outer, C, inner, nullptr, nullptr, &pl)) return rc;
  *bytes = pl.ws_bytes;
  return B2C_OK;
}
extern "C" int b2c_debug_softmax_loss_plan(int outer, int C, int inner, const void* logits, const void* prob, int* out, int n) {
  NEED(out && n >= 4, "b2c_debug_softmax_loss_plan: needs out[4]");
  SoftmaxLossPlan pl{};
  if (int rc = softmax_loss_plan(outer, C, inner, logits, prob, &pl)) return rc;
  out[0] = pl.route; out[1] = SL_CHUNK; out[2] = (int)pl.slots; out[3] = (int)pl.ws_bytes;
  return B2C_OK;
}
extern "C" int b2c_softmax_loss_forward_ex(int outer, int C, int inner, const float* logits, const float* labels, int has_ignore, int ignore_label,
                                           int norm_mode, float* prob, float* loss, float* normalizer, void* workspace, void* stream) {
  NEED(logits && labels && prob && loss && normalizer && workspace, "b2c_softmax_loss_forward_ex: null");
  NEED(norm_mode >= B2C_LOSS_NORM_FULL && norm_mode <= B2C_LOSS_NORM_NONE, "b2c_softmax_loss_forward_ex: Unknown normalization mode");
  NEED(al16({workspace}), "b2c_softmax_loss_forward_ex: workspace must be 16-byte aligned");
  SoftmaxLossPlan pl{};
  if (int rc = softmax_loss_plan(outer, C, inner, logits, prob, &pl)) return rc;
  cudaStream_t st = as_stream(stream);
  double* part = static_cast<double*>(workspace);
  int* valid = reinterpret_cast<int*>(part + pl.slots);
  const int hi = has_ignore ? 1 : 0;
  const unsigned grid = (unsigned)pl.slots;
  if (pl.route == SL_ROW) {
    launch_pdl(softmax_loss_fwd_kernel, outer, 256, 0, st, 0, C, logits, prob);
    B2C_POST_LAUNCH();
    launch_pdl(softmax_loss_chunk_kernel<SL_ROW>, grid, 256, 0, st, 0, pl.pixels, C, inner, logits, labels, hi, ignore_label, prob, part, valid);
  } else if (pl.route == SL_COL4) {
    launch_pdl(softmax_loss_chunk_kernel<SL_COL4>, grid, 256, 0, st, 0, pl.pixels, C, inner, logits, labels, hi, ignore_label, prob, part, valid);
  } else {
    launch_pdl(softmax_loss_chunk_kernel<SL_COL>, grid, 256, 0, st, 0, pl.pixels, C, inner, logits, labels, hi, ignore_label, prob, part, valid);
  }
  B2C_POST_LAUNCH();
  launch_pdl(softmax_loss_finalize_kernel, 1, 256, 0, st, 0, (int)pl.slots, (long long)outer, pl.pixels, hi, norm_mode,
             (const double*)part, (const int*)valid, loss, normalizer);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
extern "C" int b2c_softmax_loss_backward_ex(int outer, int C, int inner, const float* prob, const float* labels, int has_ignore, int ignore_label,
                                            const float* normalizer, float loss_weight, float* dx, void* stream) {
  NEED(prob && labels && normalizer && dx, "b2c_softmax_loss_backward_ex: null");
  SoftmaxLossPlan pl{};
  if (int rc = softmax_loss_plan(outer, C, inner, prob, dx, &pl)) return rc;
  cudaStream_t st = as_stream(stream);
  const int hi = has_ignore ? 1 : 0;
  if (inner == 1) {
    const size_t total = (size_t)outer * C;
    launch_pdl(softmax_loss_bwd_row_kernel, grid_for(total, 256), 256, 0, st, 0, total, C, prob, labels, hi, ignore_label, normalizer, loss_weight, dx);
  } else if (inner % 4 == 0 && al16({prob, labels, dx})) {
    const size_t cols = (size_t)pl.pixels / 4;
    launch_pdl(softmax_loss_bwd_col_kernel<true>, grid_for(cols, 256), 256, 0, st, 0, cols, C, inner, prob, labels, hi, ignore_label, normalizer, loss_weight, dx);
  } else {
    const size_t cols = (size_t)pl.pixels;
    launch_pdl(softmax_loss_bwd_col_kernel<false>, grid_for(cols, 256), 256, 0, st, 0, cols, C, inner, prob, labels, hi, ignore_label, normalizer, loss_weight, dx);
  }
  B2C_POST_LAUNCH();
  return B2C_OK;
}
template <int OP>
static int launch_ew(size_t n, const float* a, const float* b, float s, float* y, void* stream) {
  if (!n) return B2C_OK;
  const bool al = al16({a, b, y});                 // (b may be null: aligned)
  launch_pdl(ew_kernel<OP>, grid_for(al ? (n + 3) / 4 : n, 256), 256, 0, as_stream(stream), 0, n, al ? 1 : 0, a, b, s, y);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
extern "C" int b2c_sigmoid_forward(size_t n, const float* x, float* y, void* stream) {
  NEED(x && y, "b2c_sigmoid_forward: null");
  return launch_ew<EW_SIGMOID_FWD>(n, x, nullptr, 0.f, y, stream);
}
extern "C" int b2c_sigmoid_backward(size_t n, const float* y, const float* dy, float* dx, void* stream) {
  NEED(y && dy && dx, "b2c_sigmoid_backward: null");
  return launch_ew<EW_SIGMOID_BWD>(n, y, dy, 0.f, dx, stream);
}
// one cluster of loss_cluster_size(count) LOSS_THREADS-thread CTAs
template <typename... KArgs, typename... Args>
static int launch_loss_cluster(void (*kernel)(KArgs...), size_t count, void* stream, Args... args) {
  const unsigned cs = loss_cluster_size(count);
  launch_pdl(kernel, dim3(cs, 1, 1), dim3(LOSS_THREADS, 1, 1), 0, as_stream(stream), cs, args...);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
template <int MODE>
static int launch_loss_sum(int N, size_t count, const float* a, const float* b, float* diff, float* loss, void* stream) {
  const bool vec = al16({a, b, diff});
  return launch_loss_cluster(vec ? loss_sum_kernel<MODE, true> : loss_sum_kernel<MODE, false>, count, stream, count, N, a, b, diff, loss);
}
extern "C" int b2c_sigmoid_ce_loss_forward(int N, size_t count, const float* x, const float* target, float* loss, void* stream) {
  NEED(x && target && loss && N > 0 && count > 0, "b2c_sigmoid_ce_loss_forward: bad argument");
  return launch_loss_sum<0>(N, count, x, target, nullptr, loss, stream);
}
extern "C" int b2c_sigmoid_ce_loss_backward(size_t count, const float* x, const float* target, float scale, float* dx, void* stream) {
  NEED(x && target && dx, "b2c_sigmoid_ce_loss_backward: null");
  return launch_ew<EW_SIGCE_BWD>(count, x, target, scale, dx, stream);
}
extern "C" int b2c_euclidean_loss_forward(int N, size_t count, const float* a, const float* b, float* diff, float* loss, void* stream) {
  NEED(a && b && diff && loss && N > 0 && count > 0, "b2c_euclidean_loss_forward: bad argument");
  return launch_loss_sum<1>(N, count, a, b, diff, loss, stream);
}
extern "C" int b2c_euclidean_loss_backward(size_t count, const float* diff, float alpha, float* dx, void* stream) {
  NEED(diff && dx, "b2c_euclidean_loss_backward: null");
  return launch_ew<EW_SCALE>(count, diff, nullptr, alpha, dx, stream);
}
extern "C" int b2c_l1_loss_forward(int N, size_t count, const float* a, const float* b, float* diff, float* loss, void* stream) {
  NEED(a && b && diff && loss && N > 0 && count > 0, "b2c_l1_loss_forward: bad argument");
  return launch_loss_sum<2>(N, count, a, b, diff, loss, stream);
}
extern "C" int b2c_l1_loss_backward(size_t count, const float* diff, float alpha, float* dx, void* stream) {
  NEED(diff && dx, "b2c_l1_loss_backward: null");
  return launch_ew<EW_SIGN_SCALE>(count, diff, nullptr, alpha, dx, stream);
}
extern "C" int b2c_contrastive_loss_forward(int N, int C, const float* a, const float* b, const float* y, float margin, int legacy, float* diff,
                                            float* dist_sq, float* loss, void* stream) {
  NEED(a && b && y && diff && dist_sq && loss && N > 0 && C > 0, "b2c_contrastive_loss_forward: bad argument");
  return launch_loss_cluster(legacy ? contrastive_loss_kernel<true> : contrastive_loss_kernel<false>, (size_t)N * C, stream, N, C, a, b, y,
                             margin, diff, dist_sq, loss);
}
extern "C" int b2c_contrastive_loss_backward(int N, int C, const float* diff, const float* dist_sq, const float* y, float margin, int legacy,
                                             float alpha, float* da, float* db, void* stream) {
  NEED(diff && dist_sq && y && da && N > 0 && C > 0, "b2c_contrastive_loss_backward: bad argument");
  const size_t n = (size_t)N * C;
  const bool vec = C % 4 == 0 && al16({diff, da, db});
  if (vec) launch_pdl(contrastive_bwd_kernel<true>, grid_for(n / 4, 256), 256, 0, as_stream(stream), 0, N, C, diff, dist_sq, y, margin, legacy, alpha, da, db);
  else launch_pdl(contrastive_bwd_kernel<false>, grid_for(n, 256), 256, 0, as_stream(stream), 0, N, C, diff, dist_sq, y, margin, legacy, alpha, da, db);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
// y[n][o] += b[o] and db[o] += sum_n dy[n][o]: InnerProduct bias (inner_product_layer.cpp), via the conv bias kernels with P = 1
extern "C" int b2c_bias_forward(int N, int O, int P, const float* bias, float* y, void* stream) {
  NEED(bias && y, "b2c_bias_forward: null");
  return launch_bias_add(N, O, P, bias, y, as_stream(stream));
}
extern "C" int b2c_bias_backward(int N, int O, int P, const float* dy, float* db, void* stream) {
  NEED(dy && db, "b2c_bias_backward: null");
  return launch_bias_grad(N, O, P, dy, db, as_stream(stream));
}
