// sgemm_simt.cu -- fp32 SIMT GEMM / GEMV with the reference's row-major conventions.
//
// Replaces caffe_gpu_gemm<float> / caffe_gpu_gemv<float> (reference
// src/caffe/util/math_functions.cu:11-26,73-82 -> cublasSgemm / cublasSgemv).  This is the
// exact-fp32 (FFMA) kernel family: it serves b2c_sgemm for shapes the tensor-core GEMM does not
// take (tiny / unaligned problems such as the rank-1 bias GEMM and the integer known-answer
// vectors of test_util_blas.cpp) and is the on-device second opinion for the tensor-core
// kernels.  64x64 output tile, BK=16, 256 threads x (4x4) micro-tile, smem double buffered.
#include "b2c_common.cuh"

namespace b2c {

constexpr int TM = 64, TN = 64, TK = 16;

template <bool TA, bool TB>
__global__ void __launch_bounds__(256)
sgemm_simt_kernel(int M, int N, int K, float alpha, const float* __restrict__ A, int lda,
                  const float* __restrict__ B, int ldb, float beta, float* __restrict__ C, int ldc) {
  pdl_wait();
  __shared__ float As[2][TK][TM + 4];
  __shared__ float Bs[2][TK][TN + 4];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
  const int tx = tid % 16, ty = tid / 16;   // micro-tile: rows ty*4.., cols tx*4..

  // loader mapping: 1024 elements per operand per k-tile, 4 per thread.
  // A (not transposed) is k-contiguous -> walk k fastest; transposed -> walk m fastest.
  auto load_tile = [&](int buf, int k0) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int e = tid + r * 256;
      int m, k;
      if (TA) { m = e % TM; k = e / TM; } else { k = e % TK; m = e / TK; }
      const int gm = m0 + m, gk = k0 + k;
      float v = 0.0f;
      if (gm < M && gk < K) v = TA ? __ldg(A + (size_t)gk * lda + gm) : __ldg(A + (size_t)gm * lda + gk);
      As[buf][k][m] = v;
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int e = tid + r * 256;
      int n, k;
      if (TB) { k = e % TK; n = e / TK; } else { n = e % TN; k = e / TN; }
      const int gn = n0 + n, gk = k0 + k;
      float v = 0.0f;
      if (gn < N && gk < K) v = TB ? __ldg(B + (size_t)gn * ldb + gk) : __ldg(B + (size_t)gk * ldb + gn);
      Bs[buf][k][n] = v;
    }
  };

  float acc[4][4] = {};
  const int nk = (K + TK - 1) / TK;
  load_tile(0, 0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) load_tile(buf ^ 1, (kt + 1) * TK);
#pragma unroll
    for (int k = 0; k < TK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int gm = m0 + ty * 4 + i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gn = n0 + tx * 4 + j;
      if (gn >= N) continue;
      float* c = C + (size_t)gm * ldc + gn;
      *c = (beta == 0.0f) ? alpha * acc[i][j] : alpha * acc[i][j] + beta * *c;
    }
  }
}

int launch_sgemm_simt(bool tA, bool tB, int M, int N, int K, float alpha, const float* A, int lda, const float* B,
                      int ldb, float beta, float* C, int ldc, cudaStream_t st) {
  if (M <= 0 || N <= 0) return B2C_OK;
  dim3 grid((N + TN - 1) / TN, (M + TM - 1) / TM);
  if (grid.y > 65535) return fail(B2C_ERR_INVALID, "sgemm: M too large for the SIMT path");
  if (!tA && !tB) launch_pdl(sgemm_simt_kernel<false, false>, grid, 256, 0, st, 0, M, N, K, alpha, A, lda, B, ldb, beta, C, ldc);
  else if (tA && !tB) launch_pdl(sgemm_simt_kernel<true, false>, grid, 256, 0, st, 0, M, N, K, alpha, A, lda, B, ldb, beta, C, ldc);
  else if (!tA && tB) launch_pdl(sgemm_simt_kernel<false, true>, grid, 256, 0, st, 0, M, N, K, alpha, A, lda, B, ldb, beta, C, ldc);
  else launch_pdl(sgemm_simt_kernel<true, true>, grid, 256, 0, st, 0, M, N, K, alpha, A, lda, B, ldb, beta, C, ldc);
  B2C_POST_LAUNCH();
  return B2C_OK;
}

// ---- GEMV -------------------------------------------------------------------------------------
// NoTrans: one warp per output row, lanes stride the row (coalesced), shuffle reduction.
__global__ void __launch_bounds__(256)
sgemv_n_kernel(int M, int N, float alpha, const float* __restrict__ A, const float* __restrict__ x, float beta,
               float* __restrict__ y) {
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int row = warp; row < M; row += nwarps) {
    const float* a = A + (size_t)row * N;
    float s = 0.0f;
    for (int k = lane; k < N; k += 32) s = fmaf(__ldg(a + k), __ldg(x + k), s);
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) y[row] = (beta == 0.0f) ? alpha * s : alpha * s + beta * y[row];
  }
}
// Trans: one thread per output column (coalesced across threads), loop over rows.
__global__ void __launch_bounds__(256)
sgemv_t_kernel(int M, int N, float alpha, const float* __restrict__ A, const float* __restrict__ x, float beta,
               float* __restrict__ y) {
  pdl_wait();
  for (int col = blockIdx.x * blockDim.x + threadIdx.x; col < N; col += gridDim.x * blockDim.x) {
    float s = 0.0f;
    for (int r = 0; r < M; ++r) s = fmaf(__ldg(A + (size_t)r * N + col), __ldg(x + r), s);
    y[col] = (beta == 0.0f) ? alpha * s : alpha * s + beta * y[col];
  }
}

}  // namespace b2c

using namespace b2c;

extern "C" int b2c_sgemv(int transA, int M, int N, float alpha, const float* A, const float* x, float beta,
                         float* y, void* stream) {
  if (!A || !x || !y || M <= 0 || N <= 0) return fail(B2C_ERR_INVALID, "b2c_sgemv: bad argument");
  if (!transA) {
    launch_pdl(sgemv_n_kernel, grid_for((size_t)M * 32, 256), 256, 0, as_stream(stream), 0, M, N, alpha, A, x, beta, y);
  } else {
    launch_pdl(sgemv_t_kernel, grid_for((size_t)N, 256), 256, 0, as_stream(stream), 0, M, N, alpha, A, x, beta, y);
  }
  B2C_POST_LAUNCH();
  return B2C_OK;
}
