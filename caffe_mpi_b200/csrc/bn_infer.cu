// bn_infer.cu -- BatchNorm in the TEST phase (the reference's BatchNormLayer::Forward_gpu, phase_ == TEST, batch_norm_layer.cu:22-34,
// then stage 2 at :80-90): y = [ReLU]( (x - running_mean[c]) * (running_var[c] + eps)^-1/2 [* gamma[c] + beta[c]] [+ residual] ).
//
// Purely elementwise and HBM-bound (8 B per element, 12 with a residual), so one launch and no shared memory.  A group of G lanes
// (G = the plane's unit count rounded up to a power of two, at most a warp) walks one N x C plane: the plane's four constants and its
// inverse standard deviation are loaded and computed once, then the group streams the plane in 16-byte units when S % 4 == 0 and
// every pointer is 16-byte aligned, in 4-byte units otherwise.  Small planes (S = 1 behind an InnerProduct, S = 4) pack up to 32
// planes into one warp so the loads stay coalesced.  Every thread loads its U units before it stores any of them, which keeps U
// loads in flight and keeps y == x correct: each element is read and written by the same thread, read first.
#include "b2c_common.cuh"
#include "bn_common.cuh"

namespace b2c {

constexpr int BNI_THREADS = 256;
constexpr int BNI_U = 4;                 // units in flight per thread

template <bool VEC, bool RELU, bool RES>
__device__ __forceinline__ float bni_one(float v, float m, float is, float g, float bt, bool affine, float r) {
  float o = bn_y(bn_xn(v, m, is), g, bt, affine);
  if (RES) o = __fadd_rn(o, r);                                  // b2c_add / add_relu_kernel's a + b
  if (RELU) o = RES ? fmaxf(o, 0.f) : (o > 0.f ? o : o * 0.f);  // add_relu_kernel, relu_fwd_kernel with slope 0
  return o;
}

template <bool VEC, bool RELU, bool RES>
__global__ void __launch_bounds__(BNI_THREADS)
bn_infer_kernel(size_t planes, int C, unsigned units, int gshift, const float* x, const float* __restrict__ gamma,
                const float* __restrict__ beta, float eps, const float* __restrict__ run_mean, const float* __restrict__ run_var,
                const float* res, float* y) {
  const unsigned lane = threadIdx.x & 31, G = 1u << gshift, sub = lane & (G - 1);
  const unsigned ppw = 32u >> gshift;                            // planes per warp
  const size_t warp = ((size_t)blockIdx.x * BNI_THREADS + threadIdx.x) >> 5, nwarps = (size_t)gridDim.x * (BNI_THREADS / 32);
  const bool affine = gamma != nullptr;
  for (size_t p = warp * ppw + (lane >> gshift); p < planes; p += nwarps * ppw) {
    const int c = (int)(p % (size_t)C);
    const float m = run_mean[c];
    const float is = 1.0f / sqrtf(run_var[c] + eps);             // bn_stats_kernel's expression; run_var already holds var + eps
    const float g = affine ? gamma[c] : 1.f, bt = affine ? beta[c] : 0.f;
    const size_t base = p * units;
    for (unsigned u0 = sub; u0 < units; u0 += BNI_U * G) {
      if (VEC) {
        const float4* x4 = reinterpret_cast<const float4*>(x) + base;
        const float4* r4 = reinterpret_cast<const float4*>(res) + base;
        float4 v[BNI_U], r[BNI_U];
#pragma unroll
        for (int k = 0; k < BNI_U; ++k) {
          const unsigned u = u0 + k * G;
          if (u < units) { v[k] = x4[u]; if (RES) r[k] = r4[u]; }
        }
#pragma unroll
        for (int k = 0; k < BNI_U; ++k) {
          const unsigned u = u0 + k * G;
          if (u < units) {
            float4 o;
            o.x = bni_one<VEC, RELU, RES>(v[k].x, m, is, g, bt, affine, RES ? r[k].x : 0.f);
            o.y = bni_one<VEC, RELU, RES>(v[k].y, m, is, g, bt, affine, RES ? r[k].y : 0.f);
            o.z = bni_one<VEC, RELU, RES>(v[k].z, m, is, g, bt, affine, RES ? r[k].z : 0.f);
            o.w = bni_one<VEC, RELU, RES>(v[k].w, m, is, g, bt, affine, RES ? r[k].w : 0.f);
            reinterpret_cast<float4*>(y)[base + u] = o;
          }
        }
      } else {
        float v[BNI_U], r[BNI_U];
#pragma unroll
        for (int k = 0; k < BNI_U; ++k) {
          const unsigned u = u0 + k * G;
          if (u < units) { v[k] = x[base + u]; if (RES) r[k] = res[base + u]; }
        }
#pragma unroll
        for (int k = 0; k < BNI_U; ++k) {
          const unsigned u = u0 + k * G;
          if (u < units) y[base + u] = bni_one<VEC, RELU, RES>(v[k], m, is, g, bt, affine, RES ? r[k] : 0.f);
        }
      }
    }
  }
}

template <bool VEC, bool RELU, bool RES>
static void bni_launch(unsigned blocks, cudaStream_t st, size_t planes, int C, unsigned units, int gshift, const float* x, const float* gamma,
                       const float* beta, float eps, const float* rm, const float* rv, const float* res, float* y) {
  bn_infer_kernel<VEC, RELU, RES><<<blocks, BNI_THREADS, 0, st>>>(planes, C, units, gshift, x, gamma, beta, eps, rm, rv, res, y);
}

}  // namespace b2c

using namespace b2c;

extern "C" int b2c_bn_forward_inference(int N, int C, int S, const float* x, const float* gamma, const float* beta, float eps,
                                        const float* running_mean, const float* running_var, const float* residual, float* y, int relu,
                                        void* stream) {
  if (!(x && y && running_mean && running_var)) return fail(B2C_ERR_INVALID, "b2c_bn_forward_inference: null pointer");
  if ((gamma == nullptr) != (beta == nullptr)) return fail(B2C_ERR_INVALID, "b2c_bn_forward_inference: gamma and beta go together");
  if (!(N > 0 && C > 0 && S > 0)) return fail(B2C_ERR_INVALID, "b2c_bn_forward_inference: N, C and S must be positive");
  int dev_count = 0;
  if (cudaGetDeviceCount(&dev_count) != cudaSuccess || dev_count == 0) return fail(B2C_ERR_CUDA, "no CUDA device: this library has no CPU fallback");
  const uintptr_t addr = reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(residual);
  const bool vec = S % 4 == 0 && (addr & 15) == 0;
  const unsigned units = vec ? (unsigned)(S / 4) : (unsigned)S;
  int gshift = 0;
  while (gshift < 5 && (1u << gshift) < units) ++gshift;
  const size_t planes = (size_t)N * C, ppb = (size_t)(BNI_THREADS / 32) * (32u >> gshift);
  const size_t want = (planes + ppb - 1) / ppb, cap = (size_t)sm_count() * 64;
  const unsigned blocks = (unsigned)(want < cap ? want : cap);
  cudaStream_t st = as_stream(stream);
  const bool res = residual != nullptr;
#define B2C_BNI(V) do { \
    if (res) { if (relu) bni_launch<V, true, true>(blocks, st, planes, C, units, gshift, x, gamma, beta, eps, running_mean, running_var, residual, y); \
               else bni_launch<V, false, true>(blocks, st, planes, C, units, gshift, x, gamma, beta, eps, running_mean, running_var, residual, y); } \
    else { if (relu) bni_launch<V, true, false>(blocks, st, planes, C, units, gshift, x, gamma, beta, eps, running_mean, running_var, residual, y); \
           else bni_launch<V, false, false>(blocks, st, planes, C, units, gshift, x, gamma, beta, eps, running_mean, running_var, residual, y); } \
  } while (0)
  if (vec) B2C_BNI(true); else B2C_BNI(false);
#undef B2C_BNI
  B2C_POST_LAUNCH();
  return B2C_OK;
}
