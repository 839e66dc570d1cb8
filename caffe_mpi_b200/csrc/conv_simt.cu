// conv_simt.cu -- fp32 SIMT direct-convolution kernels (B2C_ALGO_SIMT) and the bias kernels.
//
// Exact-fp32 (FFMA) implicit-GEMM family behind b2c_conv_forward / backward_data /
// backward_filter for shapes the tensor-core kernels do not take, and the on-device second
// opinion for them.  Same contract as the cuDNN calls they stand in for (reference
// src/caffe/layers/cudnn_conv_layer.cu:25-29,95-99,118-123): whole batch per launch,
// y / dx overwritten, dw accumulated.  Bias forward / backward replace cudnnAddTensor and
// cudnnConvolutionBackwardBias (:39-43, :73-75) and, for the CAFFE engine, the rank-1 GEMM /
// per-image GEMV of base_conv_layer.hpp:122-128,164-168.
#include "b2c_common.cuh"

namespace b2c {

// ---- forward: one thread per output element, bias fused ---------------------------------------
__global__ void __launch_bounds__(256)
conv_fwd_simt_kernel(ConvShape s, const float* __restrict__ x, const float* __restrict__ w,
                     const float* __restrict__ bias, float* __restrict__ y) {
  const size_t total = (size_t)s.N * s.O * s.Ho * s.Wo;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x) {
    const int wo = (int)(idx % s.Wo), ho = (int)((idx / s.Wo) % s.Ho);
    const int o = (int)((idx / ((size_t)s.Wo * s.Ho)) % s.O), n = (int)(idx / ((size_t)s.Wo * s.Ho * s.O));
    const int g = o / s.Og;
    const float* xg = x + ((size_t)n * s.C + (size_t)g * s.Cg) * s.H * s.W;
    const float* wr = w + (size_t)o * s.Kd;
    float acc = 0.0f;
    for (int c = 0; c < s.Cg; ++c)
      for (int i = 0; i < s.kh; ++i) {
        const int h = ho * s.sh - s.ph + i * s.dh;
        if ((unsigned)h >= (unsigned)s.H) continue;
        for (int j = 0; j < s.kw; ++j) {
          const int ww = wo * s.sw - s.pw + j * s.dw;
          if ((unsigned)ww >= (unsigned)s.W) continue;
          acc = fmaf(__ldg(xg + ((size_t)c * s.H + h) * s.W + ww), __ldg(wr + (c * s.kh + i) * s.kw + j), acc);
        }
      }
    if (bias) acc += __ldg(bias + o);
    y[idx] = acc;
  }
}

// ---- backward data: one thread per bottom element (gather, overwrite) --------------------------
__global__ void __launch_bounds__(256)
conv_dgrad_simt_kernel(ConvShape s, const float* __restrict__ dy, const float* __restrict__ w,
                       float* __restrict__ dx) {
  const size_t total = (size_t)s.N * s.C * s.H * s.W;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x) {
    const int ww = (int)(idx % s.W), h = (int)((idx / s.W) % s.H);
    const int c = (int)((idx / ((size_t)s.W * s.H)) % s.C), n = (int)(idx / ((size_t)s.W * s.H * s.C));
    const int g = c / s.Cg, cg = c - g * s.Cg;
    float acc = 0.0f;
    for (int i = 0; i < s.kh; ++i) {
      const int hh = h + s.ph - i * s.dh;
      if (hh < 0 || hh % s.sh) continue;
      const int ho = hh / s.sh;
      if (ho >= s.Ho) continue;
      for (int j = 0; j < s.kw; ++j) {
        const int wv = ww + s.pw - j * s.dw;
        if (wv < 0 || wv % s.sw) continue;
        const int wo = wv / s.sw;
        if (wo >= s.Wo) continue;
        const float* dyp = dy + (((size_t)n * s.O + (size_t)g * s.Og) * s.Ho + ho) * s.Wo + wo;
        const float* wp = w + (((size_t)g * s.Og * s.Cg + cg) * s.kh + i) * s.kw + j;
        for (int o = 0; o < s.Og; ++o)
          acc = fmaf(__ldg(dyp + (size_t)o * s.Ho * s.Wo), __ldg(wp + (size_t)o * s.Kd), acc);
      }
    }
    dx[idx] = acc;
  }
}

// ---- backward filter: one block per (o, c-in-group); threads stride (n,ho,wo); accumulate -----
__global__ void __launch_bounds__(256)
conv_wgrad_simt_kernel(ConvShape s, const float* __restrict__ x, const float* __restrict__ dy,
                       float* __restrict__ dw) {
  __shared__ float red[8];
  const int o = blockIdx.x, cg = blockIdx.y;
  const int g = o / s.Og;
  const int P = s.Ho * s.Wo;
  const size_t Q = (size_t)s.N * P;
  for (int i = 0; i < s.kh; ++i)
    for (int j = 0; j < s.kw; ++j) {
      float acc = 0.0f;
      for (size_t q = threadIdx.x; q < Q; q += blockDim.x) {
        const int n = (int)(q / P), p = (int)(q - (size_t)n * P);
        const int ho = p / s.Wo, wo = p - ho * s.Wo;
        const int h = ho * s.sh - s.ph + i * s.dh, ww = wo * s.sw - s.pw + j * s.dw;
        if ((unsigned)h >= (unsigned)s.H || (unsigned)ww >= (unsigned)s.W) continue;
        acc = fmaf(__ldg(dy + ((size_t)n * s.O + o) * P + p),
                   __ldg(x + (((size_t)n * s.C + (size_t)g * s.Cg + cg) * s.H + h) * s.W + ww), acc);
      }
#pragma unroll
      for (int off = 16; off; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
      if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
      __syncthreads();
      if (threadIdx.x == 0) {
        float t = 0.0f;
        for (int k = 0; k < (int)(blockDim.x >> 5); ++k) t += red[k];
        dw[(((size_t)o * s.Cg + cg) * s.kh + i) * s.kw + j] += t;
      }
      __syncthreads();
    }
}

// ---- bias ---------------------------------------------------------------------------------------
// y[n][o][p] += bias[o]
__global__ void __launch_bounds__(256)
bias_add_kernel(size_t total, int O, int P, const float* __restrict__ bias, float* __restrict__ y) {
  pdl_wait();
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x)
    y[idx] += __ldg(bias + (int)((idx / P) % O));
}

// db[o] += sum_{n,p} dy[n][o][p]: one block per channel, float4 loads where aligned (P % 4 == 0 and dy on a 16-byte boundary:
// then every row is), warp-shuffle tree then a cross-warp smem stage.
__global__ void __launch_bounds__(256)
bias_grad_kernel(int N, int O, int P, const float* __restrict__ dy, float* __restrict__ db) {
  pdl_wait();
  __shared__ float red[8];
  const int o = blockIdx.x;
  float acc = 0.0f;
  const bool vec = (P % 4) == 0 && (reinterpret_cast<uintptr_t>(dy) & 15) == 0;
  for (int n = 0; n < N; ++n) {
    const float* row = dy + ((size_t)n * O + o) * P;
    if (vec) {
      const float4* r4 = reinterpret_cast<const float4*>(row);
      for (int p = threadIdx.x; p < P / 4; p += blockDim.x) {
        const float4 v = __ldg(r4 + p);
        acc += (v.x + v.y) + (v.z + v.w);
      }
    } else {
      for (int p = threadIdx.x; p < P; p += blockDim.x) acc += __ldg(row + p);
    }
  }
#pragma unroll
  for (int off = 16; off; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.0f;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) t += red[k];
    db[o] += t;
  }
}

int launch_conv_fwd_simt(const ConvShape& s, const float* x, const float* w, const float* bias, float* y,
                         cudaStream_t st) {
  const size_t total = (size_t)s.N * s.O * s.Ho * s.Wo;
  conv_fwd_simt_kernel<<<grid_for(total, 256, 16), 256, 0, st>>>(s, x, w, bias, y);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
int launch_conv_dgrad_simt(const ConvShape& s, const float* dy, const float* w, float* dx, cudaStream_t st) {
  const size_t total = (size_t)s.N * s.C * s.H * s.W;
  conv_dgrad_simt_kernel<<<grid_for(total, 256, 16), 256, 0, st>>>(s, dy, w, dx);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
int launch_conv_wgrad_simt(const ConvShape& s, const float* x, const float* dy, float* dw, cudaStream_t st) {
  if (s.Cg > 65535) return fail(B2C_ERR_INVALID, "wgrad simt: C/g too large");
  conv_wgrad_simt_kernel<<<dim3(s.O, s.Cg), 256, 0, st>>>(s, x, dy, dw);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
int launch_bias_add(int N, int O, int P, const float* bias, float* y, cudaStream_t st) {
  const size_t total = (size_t)N * O * P;
  launch_pdl(bias_add_kernel, grid_for(total, 256), 256, 0, st, 0, total, O, P, bias, y);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
int launch_bias_grad(int N, int O, int P, const float* dy, float* db, cudaStream_t st) {
  launch_pdl(bias_grad_kernel, O, 256, 0, st, 0, N, O, P, dy, db);
  B2C_POST_LAUNCH();
  return B2C_OK;
}

}  // namespace b2c
