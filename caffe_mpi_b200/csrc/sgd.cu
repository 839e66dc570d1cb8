// sgd.cu -- fused solver updates (regularise + history + apply + clear) over the parameter arena, sm_90a.
//
// Replaces the reference's per-blob *RegUpdateAllAndClear<float,float> kernels and their launchers
// (src/caffe/solvers/{sgd,nesterov,adagrad,rmsprop,adadelta,adam}_solver.cu): there each is one unvectorised launch plus a
// host stream-sync per learnable blob (161 per iteration for ResNet-50) preceded by separate cublasSscal passes for
// 1/solver_count (net.cpp:910) and 1/global_grad_scale (net.cpp:815-817).  Here: 128-bit loads/stores, the scalings folded
// into `grad_scale`, and a multi-tensor form that walks the whole contiguous parameter arena in one or two launches.  The six
// solvers share that machinery and differ only in the per-element rule.  The kernels are HBM-bound: per element
// SGD / Nesterov / AdaGrad / RMSProp read and write g, w, h (24 B); AdaDelta and Adam also h2 (32 B).
#include "b2c_common.cuh"

namespace b2c {

// Per-element rules.  Each takes gr = g*grad_scale + decay*reg(w), updates its history in place and returns the step u;
// the caller then does w -= u, g = clear ? 0 : u.  kH2: the rule has a second history arena.  sqrt and division are the
// IEEE-rounded intrinsics so the results do not depend on fast-math flags.
struct SgdRule {                 // sgd_solver.cu:9-20
  static constexpr bool kH2 = false;
  float momentum;
  __device__ __forceinline__ float operator()(float gr, float lr, float& h, float&) const {
    gr = momentum * h + lr * gr;
    h = gr;
    return gr;
  }
};
struct NesterovRule {            // nesterov_solver.cu:12-25
  static constexpr bool kH2 = false;
  float momentum;
  __device__ __forceinline__ float operator()(float gr, float lr, float& h, float&) const {
    const float hi = h;
    h = momentum * hi + lr * gr;
    return (1.f + momentum) * h - momentum * hi;
  }
};
struct AdaGradRule {             // adagrad_solver.cu:11-23
  static constexpr bool kH2 = false;
  float delta;
  __device__ __forceinline__ float operator()(float gr, float lr, float& h, float&) const {
    h = h + gr * gr;
    return __fdiv_rn(lr * gr, __fsqrt_rn(h) + delta);
  }
};
struct RMSPropRule {             // rmsprop_solver.cu:12-23
  static constexpr bool kH2 = false;
  float rms_decay, delta;
  __device__ __forceinline__ float operator()(float gr, float lr, float& h, float&) const {
    h = rms_decay * h + (1.f - rms_decay) * gr * gr;
    return __fdiv_rn(lr * gr, __fsqrt_rn(h) + delta);
  }
};
struct AdaDeltaRule {            // adadelta_solver.cu:12-26
  static constexpr bool kH2 = true;
  float momentum, delta;
  __device__ __forceinline__ float operator()(float gr, float lr, float& h, float& h2) const {
    h = momentum * h + (1.f - momentum) * gr * gr;
    gr *= __fsqrt_rn(__fdiv_rn(h2 + delta, h + delta));
    h2 = momentum * h2 + (1.f - momentum) * gr * gr;
    return lr * gr;
  }
};
struct AdamRule {                // adam_solver.cu:11-24; lr already carries the bias correction (adam_solver.cpp:42-43)
  static constexpr bool kH2 = true;
  float beta1, beta2, eps_hat;
  __device__ __forceinline__ float operator()(float gr, float lr, float& m, float& v) const {
    m = m * beta1 + gr * (1.f - beta1);
    v = v * beta2 + gr * gr * (1.f - beta2);
    return __fdiv_rn(lr * m, __fsqrt_rn(v) + eps_hat);
  }
};

template <class R>
__device__ __forceinline__ void solver_elem(const R& rule, float& g, float& w, float& h, float& h2, float lr, float decay,
                                            bool l2, float gscale, bool clear) {
  const float reg = l2 ? w : (float)((0.0f < w) - (w < 0.0f));
  const float u = rule(g * gscale + reg * decay, lr, h, h2);
  w -= u;
  g = clear ? 0.0f : u;
}

template <class R>
__device__ __forceinline__ void solver_span(const R& rule, size_t n, float* __restrict__ g, float* __restrict__ w,
                                            float* __restrict__ h, float* __restrict__ h2, float lr, float decay, bool l2,
                                            float gscale, bool clear, size_t first, size_t step) {
  float unused = 0.f;        // h2 of the one-history rules
  // head/tail scalars keep the float4 body aligned for arbitrary segment offsets
  const unsigned mg = (unsigned)(reinterpret_cast<uintptr_t>(g) & 15u);
  const unsigned mw = (unsigned)(reinterpret_cast<uintptr_t>(w) & 15u);
  const unsigned mh = (unsigned)(reinterpret_cast<uintptr_t>(h) & 15u);
  const unsigned mh2 = R::kH2 ? (unsigned)(reinterpret_cast<uintptr_t>(h2) & 15u) : mg;
  if (mg == mw && mg == mh && mg == mh2 && (mg & 3u) == 0) {
    // peel up to 3 leading elements so the body is 16-byte aligned (arena slots are padded to an even element count,
    // reference common.hpp:723, so segments are 8-byte but not 16-byte aligned)
    size_t head = ((16u - mg) & 15u) >> 2;
    if (head > n) head = n;
    for (size_t i = first; i < head; i += step)
      solver_elem(rule, g[i], w[i], h[i], R::kH2 ? h2[i] : unused, lr, decay, l2, gscale, clear);
    g += head; w += head; h += head; n -= head;
    if (R::kH2) h2 += head;
    const size_t n4 = n / 4;
    float4* g4 = reinterpret_cast<float4*>(g);
    float4* w4 = reinterpret_cast<float4*>(w);
    float4* h4 = reinterpret_cast<float4*>(h);
    float4* h24 = reinterpret_cast<float4*>(h2);
    for (size_t i = first; i < n4; i += step) {
      float4 gv = g4[i], wv = w4[i], hv = h4[i];
      float4 h2v = R::kH2 ? h24[i] : make_float4(0.f, 0.f, 0.f, 0.f);
      solver_elem(rule, gv.x, wv.x, hv.x, h2v.x, lr, decay, l2, gscale, clear);
      solver_elem(rule, gv.y, wv.y, hv.y, h2v.y, lr, decay, l2, gscale, clear);
      solver_elem(rule, gv.z, wv.z, hv.z, h2v.z, lr, decay, l2, gscale, clear);
      solver_elem(rule, gv.w, wv.w, hv.w, h2v.w, lr, decay, l2, gscale, clear);
      g4[i] = gv; w4[i] = wv; h4[i] = hv;
      if (R::kH2) h24[i] = h2v;
    }
    for (size_t i = n4 * 4 + first; i < n; i += step)
      solver_elem(rule, g[i], w[i], h[i], R::kH2 ? h2[i] : unused, lr, decay, l2, gscale, clear);
  } else {
    for (size_t i = first; i < n; i += step)
      solver_elem(rule, g[i], w[i], h[i], R::kH2 ? h2[i] : unused, lr, decay, l2, gscale, clear);
  }
}

__global__ void __launch_bounds__(256)
sgd_update_kernel(size_t n, float* __restrict__ g, float* __restrict__ w, float* __restrict__ h, float momentum,
                  float lr, float decay, int l2, float gscale, int clear) {
  solver_span(SgdRule{momentum}, n, g, w, h, nullptr, lr, decay, l2 != 0, gscale, clear != 0,
              (size_t)blockIdx.x * blockDim.x + threadIdx.x, (size_t)gridDim.x * blockDim.x);
}

// Multi-tensor: up to SEG_MAX segments per launch described in kernel-parameter space (no device tables, no staging copies).
// Each block owns BLOCK_ELEMS consecutive elements of one segment.
constexpr int SEG_MAX = 96;
constexpr int BLOCK_ELEMS = 256 * 4 * 4;
struct SegTable {
  int nseg;
  unsigned block_start[SEG_MAX + 1];
  unsigned long long offset[SEG_MAX];
  unsigned count[SEG_MAX];
  float lr[SEG_MAX];
  float decay[SEG_MAX];
};

template <class R>
__global__ void __launch_bounds__(256)
solver_update_arena_kernel(const __grid_constant__ SegTable t, float* __restrict__ g, float* __restrict__ w,
                           float* __restrict__ h, float* __restrict__ h2, const R rule, int l2, float gscale, int clear) {
  // binary search the owning segment
  int lo = 0, hi = t.nseg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (t.block_start[mid] <= blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const size_t begin = (size_t)(blockIdx.x - t.block_start[lo]) * BLOCK_ELEMS;
  size_t len = (size_t)t.count[lo] - begin;
  if (len > BLOCK_ELEMS) len = BLOCK_ELEMS;
  const size_t off = (size_t)t.offset[lo] + begin;
  solver_span(rule, len, g + off, w + off, h + off, R::kH2 ? h2 + off : nullptr, t.lr[lo], t.decay[lo], l2 != 0, gscale,
              clear != 0, threadIdx.x, blockDim.x);
}

template <class R>
static int launch_arena(const char* who, const R& rule, int nseg, const size_t* offset, const size_t* count,
                        const float* local_rate, const float* local_decay, float* g, float* w, float* h, float* h2, int l2,
                        float grad_scale, int clear_grads, void* stream) {
  if (nseg < 0 || (nseg && (!offset || !count || !local_rate || !local_decay || !g || !w || !h || (R::kH2 && !h2))))
    return fail(B2C_ERR_INVALID, "%s: bad argument", who);
  int s = 0;
  while (s < nseg) {
    SegTable t;
    t.nseg = 0;
    unsigned blocks = 0;
    while (s < nseg && t.nseg < SEG_MAX) {
      if (count[s] > 0xffffffffull) return fail(B2C_ERR_INVALID, "segment %d too large", s);
      if (count[s] == 0) { ++s; continue; }
      t.block_start[t.nseg] = blocks;
      t.offset[t.nseg] = offset[s];
      t.count[t.nseg] = (unsigned)count[s];
      t.lr[t.nseg] = local_rate[s];
      t.decay[t.nseg] = local_decay[s];
      blocks += (unsigned)((count[s] + BLOCK_ELEMS - 1) / BLOCK_ELEMS);
      ++t.nseg;
      ++s;
    }
    if (!t.nseg) break;
    t.block_start[t.nseg] = blocks;
    solver_update_arena_kernel<R><<<blocks, 256, 0, as_stream(stream)>>>(t, g, w, h, h2, rule, l2, grad_scale, clear_grads);
    B2C_POST_LAUNCH();
  }
  return B2C_OK;
}

}  // namespace b2c

using namespace b2c;

extern "C" int b2c_sgd_update(size_t n, float* g, float* w, float* h, float momentum, float local_rate,
                              float local_decay, int l2, float grad_scale, int clear_grads, void* stream) {
  if (!g || !w || !h) return fail(B2C_ERR_INVALID, "b2c_sgd_update: null pointer");
  if (n == 0) return B2C_OK;
  sgd_update_kernel<<<grid_for((n + 3) / 4, 256), 256, 0, as_stream(stream)>>>(n, g, w, h, momentum, local_rate,
                                                                               local_decay, l2, grad_scale,
                                                                               clear_grads);
  B2C_POST_LAUNCH();
  return B2C_OK;
}

extern "C" int b2c_sgd_update_arena(int nseg, const size_t* offset, const size_t* count, const float* local_rate,
                                    const float* local_decay, float* g, float* w, float* h, float momentum, int l2,
                                    float grad_scale, int clear_grads, void* stream) {
  return launch_arena("b2c_sgd_update_arena", SgdRule{momentum}, nseg, offset, count, local_rate, local_decay, g, w, h,
                      nullptr, l2, grad_scale, clear_grads, stream);
}

extern "C" int b2c_solver_update_arena(int kind, int nseg, const size_t* offset, const size_t* count,
                                       const float* local_rate, const float* local_decay, float* g, float* w, float* h,
                                       float* h2, b2c_solver_hparams hp, int l2, float grad_scale, int clear_grads,
                                       void* stream) {
  // the reference clamps delta in each ComputeUpdateValue before the launch
  const char* who = "b2c_solver_update_arena";
#define B2C_ARENA(rule) launch_arena(who, rule, nseg, offset, count, local_rate, local_decay, g, w, h, h2, l2, grad_scale, \
                                     clear_grads, stream)
  switch (kind) {
    case B2C_SOLVER_SGD: return B2C_ARENA((SgdRule{hp.momentum}));
    case B2C_SOLVER_NESTEROV: return B2C_ARENA((NesterovRule{hp.momentum}));
    case B2C_SOLVER_ADAGRAD: return B2C_ARENA((AdaGradRule{fmaxf(hp.delta, 1e-3f)}));                 // adagrad_solver.cpp:22
    case B2C_SOLVER_RMSPROP: return B2C_ARENA((RMSPropRule{hp.rms_decay, fmaxf(hp.delta, 1e-4f)}));   // rmsprop_solver.cpp:25
    case B2C_SOLVER_ADADELTA: return B2C_ARENA((AdaDeltaRule{hp.momentum, fmaxf(hp.delta, 1e-3f)}));  // adadelta_solver.cpp:36
    case B2C_SOLVER_ADAM: return B2C_ARENA((AdamRule{hp.beta1, hp.beta2, fmaxf(hp.delta, 1e-4f)}));   // adam_solver.cpp:45
  }
#undef B2C_ARENA
  return fail(B2C_ERR_INVALID, "%s: unknown solver kind %d", who, kind);
}
