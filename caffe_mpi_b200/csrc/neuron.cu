// neuron.cu -- the NeuronLayer family beyond ReLU / Sigmoid: one elementwise kernel template over the per-element rules of
// ELU, Power, AbsVal, BNLL, Exp, Log and Threshold, and PReLU with its per-channel slope gradient.  Each rule is the reference's
// own expression, in its operation order and types (a promotion to double where the reference writes a double literal), with
// explicit _rn intrinsics wherever a product feeds a sum, so the compiler cannot contract them into an FMA the reference does
// not have.
//
//   ELU        src/caffe/layers/elu_layer.cu        y = x > 0 ? x : alpha (exp(x) - 1.); dx = x > 0 ? dy : dy (y + alpha)
//   Power      src/caffe/layers/power_layer.cu      y = (shift + scale x)^power with its constant / power 2 / shift 0 branches
//   AbsVal     src/caffe/layers/absval_layer.cu     y = |x|; dx = sign(x) dy
//   BNLL       src/caffe/layers/bnll_layer.cu       y = log(1 + exp(x)) in its stable form; dx = dy e / (e + 1.), e = exp(min(x, 50))
//   Exp        src/caffe/layers/exp_layer.cu        y = outer_scale exp(inner_scale x); dx = inner_scale y dy
//   Log        src/caffe/layers/log_layer.cu        y = base_scale log(shift + scale x); dx = dy backward_num_scale (shift + scale x)^-1
//   Threshold  src/caffe/layers/threshold_layer.cpp y = x > threshold ? 1 : 0 (no backward)
//   PReLU      src/caffe/layers/prelu_layer.cu      y = x > 0 ? x : x slope[c]; dx = dy ((x > 0) + (x <= 0) slope[c]);
//                                                    dslope[c] += sum dy x (x <= 0), deterministically (see prelu_kernel)
#include <cuda_runtime.h>
#include "b2c_common.cuh"

namespace b2c {

// ---- elementwise family ---------------------------------------------------------------------------------------------------
template <int K>
__device__ __forceinline__ float neuron_fwd(float x, float p0, float p1, float p2) {
  if (K == B2C_NEURON_ELU) return x > 0.f ? x : (float)((double)p0 * ((double)expf(x) - 1.));
  if (K == B2C_NEURON_POWER) {                   // p0 power, p1 scale, p2 shift; diff_scale = power * scale rounded as LayerSetUp does
    const float power = p0, scale = p1, shift = p2, diff_scale = __fmul_rn(power, scale);
    if (diff_scale == 0.f) return power == 0.f ? 1.f : powf(shift, power);
    float t = x;
    if (scale != 1.f) t = __fmul_rn(scale, t);
    if (shift != 0.f) t = __fadd_rn(t, shift);
    if (power != 1.f) t = powf(t, power);
    return t;
  }
  if (K == B2C_NEURON_ABSVAL) return fabsf(x);
  if (K == B2C_NEURON_BNLL) return x > 0.f ? (float)((double)x + log(1. + (double)expf(-x))) : (float)log(1. + (double)expf(x));
  if (K == B2C_NEURON_EXP) {                     // p0 inner_scale, p1 outer_scale
    float t = p0 == 1.f ? expf(x) : expf(__fmul_rn(p0, x));
    if (p1 != 1.f) t = __fmul_rn(p1, t);
    return t;
  }
  if (K == B2C_NEURON_LOG) {                     // p0 scale, p1 shift, p2 base_scale
    float t = x;
    if (p0 != 1.f) t = __fmul_rn(p0, t);
    if (p1 != 0.f) t = __fadd_rn(t, p1);
    t = logf(t);
    if (p2 != 1.f) t = __fmul_rn(p2, t);
    return t;
  }
  return x > p0 ? 1.f : 0.f;                     // THRESHOLD: p0 threshold
}
template <int K>
__device__ __forceinline__ float neuron_bwd(float x, float y, float dy, float p0, float p1, float p2) {
  if (K == B2C_NEURON_ELU) return x > 0.f ? dy : __fmul_rn(dy, __fadd_rn(y, p0));
  if (K == B2C_NEURON_POWER) {
    const float power = p0, scale = p1, shift = p2, diff_scale = __fmul_rn(power, scale);
    float g;
    if (diff_scale == 0.f || power == 1.f) {
      g = diff_scale;
    } else if (power == 2.f) {                   // axpby(diff_scale * scale, x, 0) then + diff_scale * shift
      g = __fmul_rn(__fmul_rn(diff_scale, scale), x);
      if (shift != 0.f) g = __fadd_rn(g, __fmul_rn(diff_scale, shift));
    } else if (shift == 0.f) {                   // power * y / x
      g = __fmul_rn(power, __fdiv_rn(y, x));
    } else {                                     // diff_scale * y / (shift + scale * x)
      float t = x;
      if (scale != 1.f) t = __fmul_rn(scale, t);
      t = __fadd_rn(t, shift);
      g = __fdiv_rn(y, t);
      if (diff_scale != 1.f) g = __fmul_rn(diff_scale, g);
    }
    return __fmul_rn(dy, g);
  }
  if (K == B2C_NEURON_ABSVAL) return __fmul_rn((float)((0.f < x) - (x < 0.f)), dy);
  if (K == B2C_NEURON_BNLL) {
    const float e = expf(fminf(x, 50.f));
    return (float)((double)__fmul_rn(dy, e) / ((double)e + 1.));
  }
  if (K == B2C_NEURON_EXP) {                     // p0 inner_scale
    const float g = __fmul_rn(y, dy);
    return p0 != 1.f ? __fmul_rn(p0, g) : g;
  }
  // LOG: p0 scale, p1 shift, p2 backward_num_scale
  float t = x;
  if (p0 != 1.f) t = __fmul_rn(p0, t);
  if (p1 != 0.f) t = __fadd_rn(t, p1);
  t = powf(t, -1.f);
  if (p2 != 1.f) t = __fmul_rn(p2, t);
  return __fmul_rn(dy, t);
}

// One thread per float4 (VEC) or per element, grid-striding.  Pointers may alias (in place: y == x, dx == dy): every element is
// read before the same thread writes it.  Backward reads x / y only where the call passed them (the rule needs them).
template <int K, bool VEC>
__global__ void __launch_bounds__(256) neuron_fwd_kernel(size_t n, const float* x, float* y, float p0, float p1, float p2) {
  pdl_wait();
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  if (VEC) {
    const size_t n4 = n / 4;
    for (size_t i = tid; i < n4; i += step) {
      const float4 v = reinterpret_cast<const float4*>(x)[i];
      reinterpret_cast<float4*>(y)[i] = make_float4(neuron_fwd<K>(v.x, p0, p1, p2), neuron_fwd<K>(v.y, p0, p1, p2),
                                                    neuron_fwd<K>(v.z, p0, p1, p2), neuron_fwd<K>(v.w, p0, p1, p2));
    }
    for (size_t i = n4 * 4 + tid; i < n; i += step) y[i] = neuron_fwd<K>(x[i], p0, p1, p2);
  } else {
    for (size_t i = tid; i < n; i += step) y[i] = neuron_fwd<K>(x[i], p0, p1, p2);
  }
}
template <int K, bool VEC>
__global__ void __launch_bounds__(256) neuron_bwd_kernel(size_t n, const float* x, const float* y, const float* dy, float* dx,
                                                         float p0, float p1, float p2) {
  pdl_wait();
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  size_t i0 = tid;
  if (VEC) {
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    const size_t n4 = n / 4;
    for (size_t i = tid; i < n4; i += step) {
      const float4 d = reinterpret_cast<const float4*>(dy)[i];
      const float4 xv = x ? reinterpret_cast<const float4*>(x)[i] : z, yv = y ? reinterpret_cast<const float4*>(y)[i] : z;
      reinterpret_cast<float4*>(dx)[i] = make_float4(neuron_bwd<K>(xv.x, yv.x, d.x, p0, p1, p2), neuron_bwd<K>(xv.y, yv.y, d.y, p0, p1, p2),
                                                     neuron_bwd<K>(xv.z, yv.z, d.z, p0, p1, p2), neuron_bwd<K>(xv.w, yv.w, d.w, p0, p1, p2));
    }
    i0 = n4 * 4 + tid;
  }
  for (size_t i = i0; i < n; i += step) dx[i] = neuron_bwd<K>(x ? x[i] : 0.f, y ? y[i] : 0.f, dy[i], p0, p1, p2);
}

// What each backward rule reads: bit 0 x, bit 1 y (dy always).  Power's depends on its branch.
static int neuron_bwd_reads(int kind, float p0, float p1) {
  switch (kind) {
    case B2C_NEURON_ELU: return 3;
    case B2C_NEURON_ABSVAL: case B2C_NEURON_BNLL: case B2C_NEURON_LOG: return 1;
    case B2C_NEURON_EXP: return 2;
    case B2C_NEURON_POWER: {
      const float ds = p0 * p1;
      if (ds == 0.f || p0 == 1.f) return 0;
      if (p0 == 2.f) return 1;
      return 3;                                  // shift 0 and the general form read both
    }
    default: return -1;                          // THRESHOLD and unknown kinds: no backward
  }
}

static bool aligned16(std::initializer_list<const void*> ptrs) {
  for (const void* p : ptrs) if (p && (reinterpret_cast<uintptr_t>(p) & 15u)) return false;
  return true;
}

template <int K>
static void launch_neuron_fwd(bool vec, unsigned grid, cudaStream_t st, size_t n, const float* x, float* y, float p0, float p1, float p2) {
  if (vec) launch_pdl(neuron_fwd_kernel<K, true>, grid, 256, 0, st, 0, n, x, y, p0, p1, p2);
  else launch_pdl(neuron_fwd_kernel<K, false>, grid, 256, 0, st, 0, n, x, y, p0, p1, p2);
}
template <int K>
static void launch_neuron_bwd(bool vec, unsigned grid, cudaStream_t st, size_t n, const float* x, const float* y, const float* dy, float* dx,
                              float p0, float p1, float p2) {
  if (vec) launch_pdl(neuron_bwd_kernel<K, true>, grid, 256, 0, st, 0, n, x, y, dy, dx, p0, p1, p2);
  else launch_pdl(neuron_bwd_kernel<K, false>, grid, 256, 0, st, 0, n, x, y, dy, dx, p0, p1, p2);
}

// ---- PReLU -----------------------------------------------------------------------------------------------------------------
// Geometry (PreluPlan): a shared slope is one channel of extent C * dim (its channel index is always 0, so the layout is the
// flat array).  Each of the `channels` channels holds M = N * dim values (plane n at (n * channels + c) * dim); it is cut into
// `blocks` chunks of `chunk` consecutive values (a multiple of 4 on either path, so `blocks` and the workspace do not depend on
// the alignment), one CTA each.  Thread t of a CTA takes
// the float4 units (or values) t, t + 256, ... of its chunk: a fixed stripe of at most `stripe` values.  blocks is sized from the
// shape alone so that the launch is about PRELU_TARGET_CTAS CTAs (eight resident 256-thread CTAs on each of an H100's 132 SMs)
// whatever C is, with every thread taking at least one float4: a stem layer (C 64, 112 x 112 maps) gets 17 CTAs per channel,
// a 7 x 7 layer with C 2048 one.  The plan does not depend on the device, so neither do the bits.
constexpr int PRELU_THREADS = 256;
constexpr long long PRELU_TARGET_CTAS = 132 * 8;

struct PreluPlan {
  bool vec;
  int channels, dim, blocks;
  unsigned M, chunk, stripe;
  size_t ws_bytes;     // backward with dslope and blocks > 1: [channels u32 counters, padded to 16 B][channels * blocks fp32 partials]
};
static size_t prelu_counter_bytes(int channels) { return ((size_t)channels * 4 + 15) & ~(size_t)15; }
static int prelu_plan(int N, int C, int dim, int shared, std::initializer_list<const void*> ptrs, const char* what, PreluPlan* p) {
  if (N < 1 || C < 1 || dim < 1) return fail(B2C_ERR_INVALID, "%s: N, C and dim must be >= 1", what);
  const long long channels = shared ? 1 : C, d = shared ? (long long)C * dim : dim, M = (long long)N * d;
  if (M >= (1ll << 31)) return fail(B2C_ERR_INVALID, "%s: a channel holds N * dim >= 2^31 values", what);
  p->channels = (int)channels;
  p->dim = (int)d;
  p->M = (unsigned)M;
  p->vec = d % 4 == 0 && aligned16(ptrs);
  long long want = (PRELU_TARGET_CTAS + channels - 1) / channels;                 // CTAs per channel to fill the device
  const long long most = (M + PRELU_THREADS * 4 - 1) / (PRELU_THREADS * 4);      // ... but at least a float4 per thread
  if (want > most) want = most;
  if (want < 1) want = 1;
  long long chunk = (M + want - 1) / want;
  chunk = (chunk + 3) / 4 * 4;
  p->chunk = (unsigned)chunk;
  p->blocks = (int)((M + chunk - 1) / chunk);
  const long long unit = p->vec ? 4 : 1;
  p->stripe = (unsigned)((chunk + PRELU_THREADS * unit - 1) / (PRELU_THREADS * unit) * unit);
  if ((long long)p->blocks * channels >= (1ll << 31)) return fail(B2C_ERR_INVALID, "%s: too many channels", what);
  p->ws_bytes = p->blocks > 1 ? prelu_counter_bytes(p->channels) + sizeof(float) * (size_t)channels * p->blocks : 0;
  return B2C_OK;
}

struct PreluArgs {
  int channels, dim, blocks;
  unsigned M, chunk;
  const float* x; const float* slope; const float* dy;
  float* y; float* x_keep; float* dx; float* dslope;
  unsigned* counters; float* part;
};

// BWD: dx (may be null) and, with dslope, the slope gradient.  Each thread sums its stripe's terms dy * x * (x <= 0) in fp32 in
// stripe order; the CTA combines its threads in a fixed shuffle / shared-memory tree; with one CTA per channel that sum is added
// into dslope[c], else it goes to the channel's partial slot and the last CTA to arrive at the channel's counter adds the
// partials: each of its threads sums a fixed run of consecutive partials in double, then a fixed tree over the threads in double,
// rounded once to float and added into dslope[c], and sets the channel's counter back to zero: the workspace is zeroed once, when
// it is allocated, and no call puts a memset between two launches.  Every order is fixed by the shape, so the result is the same
// on every call.
template <bool VEC, bool BWD>
__global__ void __launch_bounds__(PRELU_THREADS) prelu_kernel(PreluArgs a) {
  pdl_wait();
  const int c = blockIdx.x / a.blocks, b = blockIdx.x - c * a.blocks;
  const unsigned j0 = (unsigned)b * a.chunk, j1 = min(a.M, j0 + a.chunk);
  const float s = a.slope[c];
  const size_t cstride = (size_t)a.channels * a.dim;
  float acc = 0.f;
  auto at = [&](unsigned j) { const unsigned n = j / (unsigned)a.dim; return (size_t)n * cstride + (size_t)c * a.dim + (j - n * (unsigned)a.dim); };
  auto term = [](float d, float v) { return __fmul_rn(__fmul_rn(d, v), (float)(v <= 0.f)); };
  auto gain = [s](float v) { return __fadd_rn((float)(v > 0.f), __fmul_rn((float)(v <= 0.f), s)); };
  if (VEC) {
    for (unsigned j = j0 + threadIdx.x * 4; j < j1; j += PRELU_THREADS * 4) {
      const size_t i = at(j);
      const float4 v = *reinterpret_cast<const float4*>(a.x + i);
      if (!BWD) {
        if (a.x_keep) *reinterpret_cast<float4*>(a.x_keep + i) = v;
        *reinterpret_cast<float4*>(a.y + i) = make_float4(v.x > 0.f ? v.x : __fmul_rn(v.x, s), v.y > 0.f ? v.y : __fmul_rn(v.y, s),
                                                         v.z > 0.f ? v.z : __fmul_rn(v.z, s), v.w > 0.f ? v.w : __fmul_rn(v.w, s));
      } else {
        const float4 d = *reinterpret_cast<const float4*>(a.dy + i);
        if (a.dslope) {
          acc = __fadd_rn(acc, term(d.x, v.x)); acc = __fadd_rn(acc, term(d.y, v.y));
          acc = __fadd_rn(acc, term(d.z, v.z)); acc = __fadd_rn(acc, term(d.w, v.w));
        }
        if (a.dx)
          *reinterpret_cast<float4*>(a.dx + i) = make_float4(__fmul_rn(d.x, gain(v.x)), __fmul_rn(d.y, gain(v.y)), __fmul_rn(d.z, gain(v.z)),
                                                            __fmul_rn(d.w, gain(v.w)));
      }
    }
  } else {
    for (unsigned j = j0 + threadIdx.x; j < j1; j += PRELU_THREADS) {
      const size_t i = at(j);
      const float v = a.x[i];
      if (!BWD) {
        if (a.x_keep) a.x_keep[i] = v;
        a.y[i] = v > 0.f ? v : __fmul_rn(v, s);
      } else {
        const float d = a.dy[i];
        if (a.dslope) acc = __fadd_rn(acc, term(d, v));
        if (a.dx) a.dx[i] = __fmul_rn(d, gain(v));
      }
    }
  }
  if constexpr (BWD) {
  if (!a.dslope) return;
  __shared__ float warp_sum[PRELU_THREADS / 32];
  __shared__ double dsum[PRELU_THREADS];
  __shared__ bool last;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc = __fadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, o));
  if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float v = warp_sum[0];
    for (int w = 1; w < PRELU_THREADS / 32; ++w) v = __fadd_rn(v, warp_sum[w]);
    if (a.blocks == 1) {
      a.dslope[c] = __fadd_rn(a.dslope[c], v);
    } else {
      a.part[(size_t)c * a.blocks + b] = v;
      __threadfence();
      last = atomicAdd(a.counters + c, 1u) == (unsigned)a.blocks - 1;
    }
  }
  if (a.blocks == 1) return;
  __syncthreads();
  if (!last) return;
  __threadfence();
  const float* part = a.part + (size_t)c * a.blocks;
  const int per = (a.blocks + PRELU_THREADS - 1) / PRELU_THREADS, k0 = threadIdx.x * per, k1 = min(a.blocks, k0 + per);
  double t = 0.;
  for (int k = k0; k < k1; ++k) t += (double)__ldcg(part + k);
  dsum[threadIdx.x] = t;
  __syncthreads();
  for (int h = PRELU_THREADS / 2; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h) dsum[threadIdx.x] += dsum[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    a.dslope[c] = __fadd_rn(a.dslope[c], (float)dsum[0]);
    a.counters[c] = 0u;                        // every CTA of the channel has arrived: the next call finds the counter zero
  }
  }
}

}  // namespace b2c

using namespace b2c;
#define NEED(cond, msg) if (!(cond)) return fail(B2C_ERR_INVALID, msg)

#define B2C_NEURON_DISPATCH(kind, F, ...)                      \
  switch (kind) {                                              \
    case B2C_NEURON_ELU: F<B2C_NEURON_ELU>(__VA_ARGS__); break; \
    case B2C_NEURON_POWER: F<B2C_NEURON_POWER>(__VA_ARGS__); break; \
    case B2C_NEURON_ABSVAL: F<B2C_NEURON_ABSVAL>(__VA_ARGS__); break; \
    case B2C_NEURON_BNLL: F<B2C_NEURON_BNLL>(__VA_ARGS__); break; \
    case B2C_NEURON_EXP: F<B2C_NEURON_EXP>(__VA_ARGS__); break; \
    case B2C_NEURON_LOG: F<B2C_NEURON_LOG>(__VA_ARGS__); break; \
    default: F<B2C_NEURON_THRESHOLD>(__VA_ARGS__); break;     \
  }

extern "C" int b2c_neuron_forward(int kind, size_t n, const float* x, float* y, float p0, float p1, float p2, void* stream) {
  NEED(kind >= B2C_NEURON_ELU && kind <= B2C_NEURON_THRESHOLD, "b2c_neuron_forward: unknown kind");
  NEED(x && y, "b2c_neuron_forward: null");
  if (!n) return B2C_OK;
  const bool vec = aligned16({x, y});
  const unsigned grid = (unsigned)grid_for(vec ? (n + 3) / 4 : n, 256);
  B2C_NEURON_DISPATCH(kind, launch_neuron_fwd, vec, grid, as_stream(stream), n, x, y, p0, p1, p2);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
extern "C" int b2c_neuron_backward(int kind, size_t n, const float* x, const float* y, const float* dy, float* dx, float p0, float p1, float p2,
                                   void* stream) {
  const int reads = neuron_bwd_reads(kind, p0, p1);
  NEED(reads >= 0, "b2c_neuron_backward: unknown kind, or a kind without a backward (Threshold)");
  NEED(dy && dx, "b2c_neuron_backward: null dy or dx");
  NEED(!(reads & 1) || x, "b2c_neuron_backward: this rule reads x");
  NEED(!(reads & 2) || y, "b2c_neuron_backward: this rule reads y");
  if (!n) return B2C_OK;
  if (!(reads & 1)) x = nullptr;
  if (!(reads & 2)) y = nullptr;
  const bool vec = aligned16({x, y, dy, dx});
  const unsigned grid = (unsigned)grid_for(vec ? (n + 3) / 4 : n, 256);
  B2C_NEURON_DISPATCH(kind, launch_neuron_bwd, vec, grid, as_stream(stream), n, x, y, dy, dx, p0, p1, p2);
  B2C_POST_LAUNCH();
  return B2C_OK;
}

extern "C" int b2c_prelu_forward(int N, int C, int dim, int shared, const float* x, const float* slope, float* y, float* x_keep, void* stream) {
  NEED(x && slope && y, "b2c_prelu_forward: null");
  NEED(x_keep != x && x_keep != y, "b2c_prelu_forward: x_keep must be a buffer of its own");
  PreluPlan pl{};
  if (int rc = prelu_plan(N, C, dim, shared, {x, y, x_keep}, "b2c_prelu_forward", &pl)) return rc;
  PreluArgs a{pl.channels, pl.dim, pl.blocks, pl.M, pl.chunk, x, slope, nullptr, y, x_keep, nullptr, nullptr, nullptr, nullptr};
  const unsigned grid = (unsigned)(pl.blocks * pl.channels);
  if (pl.vec) launch_pdl(prelu_kernel<true, false>, grid, PRELU_THREADS, 0, as_stream(stream), 0, a);
  else launch_pdl(prelu_kernel<false, false>, grid, PRELU_THREADS, 0, as_stream(stream), 0, a);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
extern "C" int b2c_prelu_workspace_bytes(int N, int C, int dim, int shared, size_t* bytes) {
  NEED(bytes, "b2c_prelu_workspace_bytes: null");
  PreluPlan pl{};
  if (int rc = prelu_plan(N, C, dim, shared, {}, "b2c_prelu_workspace_bytes", &pl)) return rc;
  *bytes = pl.ws_bytes;
  return B2C_OK;
}
extern "C" int b2c_prelu_backward(int N, int C, int dim, int shared, const float* x, const float* dy, const float* slope, float* dx,
                                  float* dslope, void* ws, size_t ws_bytes, void* stream) {
  NEED(x && dy && slope, "b2c_prelu_backward: null x, dy or slope");
  NEED(dx != x, "b2c_prelu_backward: dx may alias dy, not x");
  PreluPlan pl{};
  if (int rc = prelu_plan(N, C, dim, shared, {x, dy, dx}, "b2c_prelu_backward", &pl)) return rc;
  if (!dx && !dslope) return B2C_OK;
  const bool reduce = dslope && pl.blocks > 1;
  if (reduce) {
    if (!ws || ws_bytes < pl.ws_bytes) return fail(B2C_ERR_WORKSPACE, "b2c_prelu_backward: workspace too small (%zu < %zu bytes)", ws_bytes, pl.ws_bytes);
    NEED((reinterpret_cast<uintptr_t>(ws) & 15u) == 0, "b2c_prelu_backward: workspace must be 16-byte aligned");
  }
  unsigned* counters = reduce ? static_cast<unsigned*>(ws) : nullptr;
  float* part = reduce ? reinterpret_cast<float*>(static_cast<char*>(ws) + prelu_counter_bytes(pl.channels)) : nullptr;
  PreluArgs a{pl.channels, pl.dim, pl.blocks, pl.M, pl.chunk, x, slope, dy, nullptr, nullptr, dx, dslope, counters, part};
  const unsigned grid = (unsigned)(pl.blocks * pl.channels);
  if (pl.vec) launch_pdl(prelu_kernel<true, true>, grid, PRELU_THREADS, 0, as_stream(stream), 0, a);
  else launch_pdl(prelu_kernel<false, true>, grid, PRELU_THREADS, 0, as_stream(stream), 0, a);
  B2C_POST_LAUNCH();
  return B2C_OK;
}

extern "C" int b2c_debug_neuron_plan(int op, int kind, int N, int C, int dim, int shared, const void* const* ptrs, int nptrs, int* out, int n) {
  NEED(out && n >= 7, "b2c_debug_neuron_plan: needs out[7]");
  NEED(nptrs >= 0 && nptrs <= 4 && (nptrs == 0 || ptrs), "b2c_debug_neuron_plan: ptrs");
  const void* p[4] = {nullptr, nullptr, nullptr, nullptr};
  for (int i = 0; i < nptrs; ++i) p[i] = ptrs[i];
  if (op == 0 || op == 1) {                      // elementwise forward / backward over N values (C, dim, shared unused)
    NEED(kind >= B2C_NEURON_ELU && kind <= B2C_NEURON_THRESHOLD, "b2c_debug_neuron_plan: unknown kind");
    NEED(op == 0 || kind != B2C_NEURON_THRESHOLD, "b2c_debug_neuron_plan: Threshold has no backward");
    NEED(N >= 0, "b2c_debug_neuron_plan: negative count");
    const bool vec = aligned16({p[0], p[1], p[2], p[3]});
    const size_t cnt = (size_t)N;
    out[0] = vec ? 1 : 0;
    out[1] = cnt ? grid_for(vec ? (cnt + 3) / 4 : cnt, 256) : 0;
    out[2] = 256; out[3] = 1; out[4] = 0; out[5] = 1; out[6] = 0;
    return B2C_OK;
  }
  NEED(op == 2 || op == 3, "b2c_debug_neuron_plan: op is 0 / 1 (elementwise forward / backward) or 2 / 3 (PReLU forward / backward)");
  PreluPlan pl{};
  if (int rc = prelu_plan(N, C, dim, shared, {p[0], p[1], p[2]}, "b2c_debug_neuron_plan", &pl)) return rc;
  out[0] = pl.vec ? 1 : 0;
  out[1] = pl.blocks * pl.channels;
  out[2] = PRELU_THREADS;
  out[3] = pl.blocks;
  out[4] = (int)pl.stripe;
  out[5] = pl.channels;
  out[6] = op == 3 ? (int)pl.ws_bytes : 0;
  return B2C_OK;
}
