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

#include <vector>

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

// How solver_span splits a span of n elements whose arrays start at g, w, h and h2 (null for the one-history rules): when all
// share one 4-byte-aligned offset within 16 bytes, `head` (0-3) leading scalars, `body4` float4 units and `tail` trailing scalars;
// otherwise one float at a time (vec false, tail n).  Arena slots are padded to an even element count (reference common.hpp:723),
// so segments are 8-byte but not 16-byte aligned and the head peels them to a 16-byte boundary.  b2c_debug_solver_plan reports it.
struct SpanSplit {
  bool vec;
  unsigned head;
  size_t body4, tail;
};
__host__ __device__ __forceinline__ SpanSplit span_split(size_t n, const void* g, const void* w, const void* h, const void* h2) {
  const unsigned mg = (unsigned)(reinterpret_cast<uintptr_t>(g) & 15u);
  const unsigned mw = (unsigned)(reinterpret_cast<uintptr_t>(w) & 15u);
  const unsigned mh = (unsigned)(reinterpret_cast<uintptr_t>(h) & 15u);
  const unsigned mh2 = h2 ? (unsigned)(reinterpret_cast<uintptr_t>(h2) & 15u) : mg;
  SpanSplit s;
  s.vec = mg == mw && mg == mh && mg == mh2 && (mg & 3u) == 0;
  if (!s.vec) {
    s.head = 0; s.body4 = 0; s.tail = n;
    return s;
  }
  const size_t head = ((16u - mg) & 15u) >> 2;
  s.head = (unsigned)(head < n ? head : n);
  s.body4 = (n - s.head) / 4;
  s.tail = n - s.head - s.body4 * 4;
  return s;
}

template <class R>
__device__ __forceinline__ void solver_span(const R& rule, size_t n, float* __restrict__ g, float* __restrict__ w,
                                            float* __restrict__ h, float* __restrict__ h2, float lr, float decay, bool l2,
                                            float gscale, bool clear, size_t first, size_t step) {
  float unused = 0.f;        // h2 of the one-history rules
  const SpanSplit sp = span_split(n, g, w, h, R::kH2 ? h2 : nullptr);
  if (sp.vec) {
    const size_t head = sp.head;
    for (size_t i = first; i < head; i += step)
      solver_elem(rule, g[i], w[i], h[i], R::kH2 ? h2[i] : unused, lr, decay, l2, gscale, clear);
    g += head; w += head; h += head; n -= head;
    if (R::kH2) h2 += head;
    const size_t n4 = sp.body4;
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

// The launches of one arena update: segments in order, zero counts skipped, at most SEG_MAX per launch, each segment owning
// ceil(count / BLOCK_ELEMS) consecutive blocks; seg_launch[s] (when given) receives segment s's launch, -1 for an empty one.
// Every segment is checked before anything is returned, so a refused call launches nothing.  rate / decay may be null (the
// plan query): the tables then carry zeros.
static int pack_segments(const char* who, int nseg, const size_t* offset, const size_t* count, const float* local_rate,
                         const float* local_decay, std::vector<SegTable>* launches, int* seg_launch) {
  for (int s = 0; s < nseg; ++s)
    if (count[s] > 0xffffffffull) return fail(B2C_ERR_INVALID, "%s: segment %d too large", who, s);
  launches->clear();
  for (int s = 0; s < nseg; ++s) {
    if (seg_launch) seg_launch[s] = -1;
    if (count[s] == 0) continue;
    if (launches->empty() || launches->back().nseg == SEG_MAX) {
      launches->emplace_back();
      launches->back().nseg = 0;
      launches->back().block_start[0] = 0;
    }
    SegTable& t = launches->back();
    const unsigned start = t.block_start[t.nseg];
    t.offset[t.nseg] = offset[s];
    t.count[t.nseg] = (unsigned)count[s];
    t.lr[t.nseg] = local_rate ? local_rate[s] : 0.f;
    t.decay[t.nseg] = local_decay ? local_decay[s] : 0.f;
    ++t.nseg;
    t.block_start[t.nseg] = start + (unsigned)((count[s] + BLOCK_ELEMS - 1) / BLOCK_ELEMS);
    if (seg_launch) seg_launch[s] = (int)launches->size() - 1;
  }
  return B2C_OK;
}

template <class R>
static int launch_arena(const char* who, const R& rule, int nseg, const size_t* offset, const size_t* count,
                        const float* local_rate, const float* local_decay, float* g, float* w, float* h, float* h2, int l2,
                        float grad_scale, int clear_grads, void* stream) {
  if (nseg < 0 || (nseg && (!offset || !count || !local_rate || !local_decay || !g || !w || !h || (R::kH2 && !h2))))
    return fail(B2C_ERR_INVALID, "%s: bad argument", who);
  std::vector<SegTable> launches;
  if (const int rc = pack_segments(who, nseg, offset, count, local_rate, local_decay, &launches, nullptr)) return rc;
  for (const SegTable& t : launches) {
    solver_update_arena_kernel<R><<<t.block_start[t.nseg], 256, 0, as_stream(stream)>>>(t, g, w, h, h2, rule, l2, grad_scale,
                                                                                        clear_grads);
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

extern "C" int b2c_debug_solver_plan(int kind, int nseg, const size_t* offset, const size_t* count, const void* g,
                                     const void* w, const void* h, const void* h2, int* launch_out, int max_launches,
                                     int* nlaunch, long long* seg_out) {
  const char* who = "b2c_debug_solver_plan";
  bool two;
  switch (kind) {
    case B2C_SOLVER_SGD: case B2C_SOLVER_NESTEROV: case B2C_SOLVER_ADAGRAD: case B2C_SOLVER_RMSPROP: two = false; break;
    case B2C_SOLVER_ADADELTA: case B2C_SOLVER_ADAM: two = true; break;
    default: return fail(B2C_ERR_INVALID, "%s: unknown solver kind %d", who, kind);
  }
  if (nseg < 0 || (nseg && (!offset || !count || !g || !w || !h || (two && !h2))))
    return fail(B2C_ERR_INVALID, "%s: bad argument", who);
  if (!nlaunch || (nseg && !seg_out) || max_launches < 0 || (max_launches && !launch_out))
    return fail(B2C_ERR_INVALID, "%s: null output", who);
  std::vector<SegTable> launches;
  std::vector<int> seg_launch(nseg);
  if (const int rc = pack_segments(who, nseg, offset, count, nullptr, nullptr, &launches, seg_launch.data())) return rc;
  *nlaunch = (int)launches.size();
  if (*nlaunch > max_launches) return fail(B2C_ERR_INVALID, "%s: %d launches, launch_out holds %d", who, *nlaunch, max_launches);
  for (int i = 0; i < *nlaunch; ++i) {
    launch_out[2 * i] = launches[i].nseg;
    launch_out[2 * i + 1] = (int)launches[i].block_start[launches[i].nseg];
  }
  auto at = [](const void* p, size_t off) { return p ? static_cast<const void*>(static_cast<const char*>(p) + off * 4) : p; };
  for (int s = 0; s < nseg; ++s) {
    long long* o = seg_out + 6 * (size_t)s;
    o[0] = seg_launch[s];
    o[1] = o[2] = o[3] = o[4] = o[5] = 0;
    if (seg_launch[s] < 0) continue;
    // every block of the segment splits its own BLOCK_ELEMS span, as solver_update_arena_kernel does
    for (size_t begin = 0; begin < count[s]; begin += BLOCK_ELEMS) {
      const size_t len = count[s] - begin < (size_t)BLOCK_ELEMS ? count[s] - begin : (size_t)BLOCK_ELEMS;
      const size_t off = offset[s] + begin;
      const SpanSplit sp = span_split(len, at(g, off), at(w, off), at(h, off), two ? at(h2, off) : nullptr);
      o[1] = sp.vec; o[2] += 1; o[3] += sp.head; o[4] += (long long)sp.body4; o[5] += (long long)sp.tail;
    }
  }
  return B2C_OK;
}
