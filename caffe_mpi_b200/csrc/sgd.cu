// sgd.cu -- fused SGD-momentum update (regularise + history + apply + clear), sm_90a.
//
// Replaces SGDRegUpdateAllAndClear<float,float> and its launcher (reference
// src/caffe/solvers/sgd_solver.cu:9-20,57-72): there it is one unvectorised launch plus a
// host stream-sync per learnable blob (161 per iteration for ResNet-50) preceded by separate
// cublasSscal passes for 1/solver_count (net.cpp:910) and 1/global_grad_scale (net.cpp:815-817).
// Here: 128-bit loads/stores, the scalings folded into `grad_scale`, and a multi-tensor form
// that walks the whole contiguous parameter arena in one or two launches.  The kernel is
// HBM-bound: 12 B read + 12 B written per element (SURVEY 8d).
#include "b2c_common.cuh"

namespace b2c {

__device__ __forceinline__ void sgd_elem(float& g, float& w, float& h, float momentum, float lr, float decay,
                                         bool l2, float gscale, bool clear) {
  const float reg = l2 ? w : (float)((0.0f < w) - (w < 0.0f));
  float gr = g * gscale + reg * decay;
  gr = momentum * h + lr * gr;
  h = gr;
  w -= gr;
  g = clear ? 0.0f : gr;
}

__device__ __forceinline__ void sgd_span(size_t n, float* __restrict__ g, float* __restrict__ w,
                                         float* __restrict__ h, float momentum, float lr, float decay, bool l2,
                                         float gscale, bool clear, size_t first, size_t step) {
  // head/tail scalars keep the float4 body aligned for arbitrary segment offsets
  const unsigned mg = (unsigned)(reinterpret_cast<uintptr_t>(g) & 15u);
  const unsigned mw = (unsigned)(reinterpret_cast<uintptr_t>(w) & 15u);
  const unsigned mh = (unsigned)(reinterpret_cast<uintptr_t>(h) & 15u);
  if (mg == mw && mg == mh && (mg & 3u) == 0) {
    // peel up to 3 leading elements so the body is 16-byte aligned (arena slots are padded to an
    // even element count, reference common.hpp:723, so segments are 8-byte but not 16-byte aligned)
    size_t head = ((16u - mg) & 15u) >> 2;
    if (head > n) head = n;
    for (size_t i = first; i < head; i += step) sgd_elem(g[i], w[i], h[i], momentum, lr, decay, l2, gscale, clear);
    g += head; w += head; h += head; n -= head;
    const size_t n4 = n / 4;
    float4* g4 = reinterpret_cast<float4*>(g);
    float4* w4 = reinterpret_cast<float4*>(w);
    float4* h4 = reinterpret_cast<float4*>(h);
    for (size_t i = first; i < n4; i += step) {
      float4 gv = g4[i], wv = w4[i], hv = h4[i];
      sgd_elem(gv.x, wv.x, hv.x, momentum, lr, decay, l2, gscale, clear);
      sgd_elem(gv.y, wv.y, hv.y, momentum, lr, decay, l2, gscale, clear);
      sgd_elem(gv.z, wv.z, hv.z, momentum, lr, decay, l2, gscale, clear);
      sgd_elem(gv.w, wv.w, hv.w, momentum, lr, decay, l2, gscale, clear);
      g4[i] = gv; w4[i] = wv; h4[i] = hv;
    }
    for (size_t i = n4 * 4 + first; i < n; i += step) sgd_elem(g[i], w[i], h[i], momentum, lr, decay, l2, gscale, clear);
  } else {
    for (size_t i = first; i < n; i += step) sgd_elem(g[i], w[i], h[i], momentum, lr, decay, l2, gscale, clear);
  }
}

__global__ void __launch_bounds__(256)
sgd_update_kernel(size_t n, float* __restrict__ g, float* __restrict__ w, float* __restrict__ h, float momentum,
                  float lr, float decay, int l2, float gscale, int clear) {
  sgd_span(n, g, w, h, momentum, lr, decay, l2 != 0, gscale, clear != 0,
           (size_t)blockIdx.x * blockDim.x + threadIdx.x, (size_t)gridDim.x * blockDim.x);
}

// Multi-tensor: up to SEG_MAX segments per launch described in kernel-parameter space (no device
// tables, no staging copies).  Each block owns BLOCK_ELEMS consecutive elements of one segment.
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

__global__ void __launch_bounds__(256)
sgd_update_arena_kernel(const __grid_constant__ SegTable t, float* __restrict__ g, float* __restrict__ w,
                        float* __restrict__ h, float momentum, int l2, float gscale, int clear) {
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
  sgd_span(len, g + off, w + off, h + off, momentum, t.lr[lo], t.decay[lo], l2 != 0, gscale, clear != 0,
           threadIdx.x, blockDim.x);
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
  if (nseg < 0 || (nseg && (!offset || !count || !local_rate || !local_decay || !g || !w || !h)))
    return fail(B2C_ERR_INVALID, "b2c_sgd_update_arena: bad argument");
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
    sgd_update_arena_kernel<<<blocks, 256, 0, as_stream(stream)>>>(t, g, w, h, momentum, l2, grad_scale, clear_grads);
    B2C_POST_LAUNCH();
  }
  return B2C_OK;
}
