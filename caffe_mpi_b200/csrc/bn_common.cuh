// bn_common.cuh -- what the BatchNorm kernels of layers.cu (x_norm kept, the reference's form) and layers_fused.cu (x_norm
// recomputed, ReLU folded in, statistics and normalisation in ONE launch) share: the launch geometry and the per-thread
// accumulation order.  Both files produce the same bits for the same input because they run the same code in the same order.
#pragma once
#include <cooperative_groups.h>
#include <initializer_list>
#include <stdlib.h>
#include "b2c_common.cuh"

namespace b2c {

constexpr int BN_CLUSTER = 16;         // most CTAs per channel: 8 is the portable cluster limit, 16 needs the non-portable opt-in (bn_max_cluster())
constexpr int BN_THREADS = 512;        // most threads per CTA (the kernels' launch bound); bn_threads() picks the launch size per shape
constexpr int BN_U = 4;                // independent 16-byte loads in flight per thread and stream

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// block-wide sum of two values (blockDim.x multiple of 32, <= 1024); result valid in every thread
__device__ __forceinline__ void block_sum2(float& a, float& b) {
  __shared__ float sa[32], sb[32];
  a = warp_sum(a); b = warp_sum(b);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if (lane == 0) { sa[w] = a; sb[w] = b; }
  __syncthreads();
  a = lane < nw ? sa[lane] : 0.f; b = lane < nw ? sb[lane] : 0.f;
  a = warp_sum(a); b = warp_sum(b);
  __syncthreads();
}

// The elementwise expressions of the BatchNorm / ReLU / Eltwise chain, spelled with explicit-rounding intrinsics: nvcc contracts
// a * b + c into an FMA wherever it sees one, and WHICH products it sees depends on the surrounding code (the unfused dx kernel
// folded sum_dy * inv_cnt into the subtraction, the fused one folded the ReLU mask instead: 1-ulp differences in dx, found by
// tests/test_layers_gpu.py).  Every kernel that claims the same bits goes through these.
__device__ __forceinline__ float bn_xn(float x, float m, float is) { return __fmul_rn(__fsub_rn(x, m), is); }
__device__ __forceinline__ float bn_y(float xn, float g, float bt, bool affine) { return affine ? __fmaf_rn(xn, g, bt) : xn; }
__device__ __forceinline__ float relu_mask(float d, float y) { return __fmul_rn(d, y > 0.f ? 1.f : 0.f); }      // ReLU backward, slope 0
__device__ __forceinline__ float bn_mean_term(float sum, float inv_cnt) { return __fmul_rn(sum, inv_cnt); }
__device__ __forceinline__ float bn_dx(float d, float xn, float gi, float mdy, float mdx) {
  return __fmul_rn(gi, __fmaf_rn(-xn, mdx, __fsub_rn(d, mdy)));
}

struct PlaneCursor {       // walks a channel's planes: flattened unit index -> (image n, offset p)
  unsigned n, p;
  __device__ __forceinline__ void init(unsigned i, unsigned units) { n = i / units; p = i - n * units; }
  __device__ __forceinline__ void advance(unsigned step, unsigned units) { p += step; while (p >= units) { p -= units; ++n; } }
};

// The slice [lo, hi) of a channel's N * units flattened units that cluster rank `rank` owns
__device__ __forceinline__ void bn_slice(unsigned total, unsigned rank, unsigned nranks, unsigned& lo, unsigned& hi) {
  const unsigned len = (total + nranks - 1) / nranks;
  lo = min(total, rank * len); hi = min(total, lo + len);
}

// MODE 0: a = sum (x-k), b = sum (x-k)^2   (q unused)      MODE 1: a = sum dy*xn, b = sum dy   (x = dy, q = xnorm)
// CACHE 1: every unit of x this thread loads is also parked in shared memory at [unit index - slice start] (the one-launch kernels
// of layers_fused.cu read it back in their elementwise phase: same thread, same index, no barrier needed).  CACHE 2: the units
// are already there (the thread's own cp.async prefetch): read them from shared memory instead of global memory.
template <bool VEC, int MODE, int CACHE = 0>
__device__ __forceinline__ void bn_channel_partial(int N, int C, int S, int c, const float* __restrict__ x, const float* __restrict__ q,
                                                   float k, unsigned rank, unsigned nranks, float& a, float& b, void* cache = nullptr) {
  constexpr int U = BN_U;                                       // independent loads in flight per thread
  const unsigned TH = blockDim.x;                               // the launch size fixes the summation order: bn_threads() on the host
  const unsigned units = VEC ? S / 4 : S;                       // units per plane
  unsigned lo, hi;
  bn_slice((unsigned)N * units, rank, nranks, lo, hi);
  a = 0.f; b = 0.f;
  float a2 = 0.f, b2 = 0.f;
  PlaneCursor cur;
  unsigned i = lo + threadIdx.x;
  if (i < hi) cur.init(i, units);
  for (; i < hi; i += U * TH) {
    size_t off[U];
    bool ok[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      ok[u] = i + u * TH < hi;
      off[u] = ((size_t)cur.n * C + c) * units + cur.p;
      cur.advance(TH, units);
    }
    if (VEC) {
      float4 v[U], w[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (CACHE == 2) v[u] = ok[u] ? static_cast<const float4*>(cache)[i + u * TH - lo] : make_float4(k, k, k, k);
        else v[u] = ok[u] ? reinterpret_cast<const float4*>(x)[off[u]] : make_float4(k, k, k, k);
        if (MODE == 1) w[u] = ok[u] ? reinterpret_cast<const float4*>(q)[off[u]] : make_float4(0.f, 0.f, 0.f, 0.f);
        if (CACHE == 1 && ok[u]) static_cast<float4*>(cache)[i + u * TH - lo] = v[u];
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (MODE == 0) {
          const float d0 = v[u].x - k, d1 = v[u].y - k, d2 = v[u].z - k, d3 = v[u].w - k;
          a += d0 + d1; a2 += d2 + d3;
          b = fmaf(d0, d0, b); b2 = fmaf(d1, d1, b2); b = fmaf(d2, d2, b); b2 = fmaf(d3, d3, b2);
        } else {
          a = fmaf(v[u].x, w[u].x, a); a2 = fmaf(v[u].y, w[u].y, a2); a = fmaf(v[u].z, w[u].z, a); a2 = fmaf(v[u].w, w[u].w, a2);
          b += v[u].x + v[u].y; b2 += v[u].z + v[u].w;
        }
      }
    } else {
      float v[U], w[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (CACHE == 2) v[u] = ok[u] ? static_cast<const float*>(cache)[i + u * TH - lo] : k;
        else v[u] = ok[u] ? x[off[u]] : k;
        if (MODE == 1) w[u] = ok[u] ? q[off[u]] : 0.f;
        if (CACHE == 1 && ok[u]) static_cast<float*>(cache)[i + u * TH - lo] = v[u];
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (MODE == 0) { const float d = v[u] - k; a += d; b = fmaf(d, d, b); }
        else { a = fmaf(v[u], w[u], a); b += v[u]; }
      }
    }
  }
  a += a2; b += b2;
}

// the cluster's partial (a, b) pairs added in rank order, by every thread
__device__ __forceinline__ void bn_cluster_sum(cooperative_groups::cluster_group& cluster, const float2* part, unsigned nranks, double& s1, double& s2) {
  float2 v[BN_CLUSTER];
#pragma unroll
  for (unsigned r = 0; r < (unsigned)BN_CLUSTER; ++r) v[r] = r < nranks ? *cluster.map_shared_rank(part, r) : make_float2(0.f, 0.f);
  s1 = 0.0; s2 = 0.0;
#pragma unroll
  for (unsigned r = 0; r < (unsigned)BN_CLUSTER; ++r) if (r < nranks) { s1 += v[r].x; s2 += v[r].y; }
}

// Mean and variance + eps of channel c, in every thread of the cluster.  Pass 1 sums x - k and (x - k)^2 with k = the channel's
// first value; the variance s2/cnt - (s1/cnt)^2 then carries an fp32 summation error that grows as ((mean - k) / sigma)^2 (4e-4
// relative for a first value 100 sigma out).  So when k lies more than 4 sigma from the mean, pass 2 sums x - m0 and (x - m0)^2
// about pass 1's mean m0 instead: the error is then the reference's two-pass level whatever k is, and within 17x of it when pass 2
// is skipped.  Every thread of the cluster holds the same s1, s2, so all take the same branch.  CACHE (bn_channel_partial's): pass 1
// parks the slice in shared memory (1) or reads it from there (2); pass 2 reads the parked copy, else x again.  part[2]: the CTA's
// partials of each pass (pass 2 writes the second slot while peers may still read the first).
template <bool VEC, int CACHE>
__device__ __forceinline__ void bn_channel_stats(cooperative_groups::cluster_group& cluster, int N, int C, int S, int c, const float* __restrict__ x,
                                                 float eps, float2* part, void* cache, float& m, float& var_eps) {
  const unsigned rank = cluster.block_rank(), nranks = cluster.num_blocks();
  const double cnt = (double)N * S;
  const float k = x[(size_t)c * S];
  float a, b;
  double s1, s2;
  bn_channel_partial<VEC, 0, CACHE>(N, C, S, c, x, nullptr, k, rank, nranks, a, b, cache);
  block_sum2(a, b);
  if (threadIdx.x == 0) part[0] = make_float2(a, b);
  cluster.sync();
  bn_cluster_sum(cluster, part, nranks, s1, s2);
  double m1 = s1 / cnt, var = s2 / cnt - m1 * m1;
  m = (float)((double)k + m1);
  if (m1 * m1 > 16.0 * var) {
    const float m0 = m;
    bn_channel_partial<VEC, 0, CACHE ? 2 : 0>(N, C, S, c, x, nullptr, m0, rank, nranks, a, b, cache);
    block_sum2(a, b);
    if (threadIdx.x == 0) part[1] = make_float2(a, b);
    cluster.sync();
    bn_cluster_sum(cluster, part + 1, nranks, s1, s2);
    m1 = s1 / cnt;
    var = s2 / cnt - m1 * m1;
    m = (float)((double)m0 + m1);
  }
  var_eps = (float)fmax(var, 0.0) + eps;   // batch_norm_layer.cpp:183-186 (eps folded in before the average)
}

// The launch of a BatchNorm training call, chosen by bn_plan (layers_fused.cu) for every entry point and reported by
// b2c_debug_bn_plan.  threads and cs are those of the per-channel (cluster) kernel; the two-launch forms' elementwise passes
// always run 256-thread blocks.
struct BnPlan {
  int launches;            // 1: statistics / reduction and the elementwise pass in one launch; 2: two launches
  unsigned cs;             // CTAs per channel (one thread-block cluster)
  unsigned threads;        // threads per CTA
  int park;                // what stays in shared memory between the phases: bit 0 = x, bit 1 = the (masked) gradient
  int prefetch;            // the parked streams come in by cp.async before the reduction
  bool vec;                // float4 units (S % 4 == 0 and every pointer 16-byte aligned), else one float at a time
  size_t smem;             // dynamic shared memory per CTA
  unsigned slice_units;    // units in the largest (rank 0's) slice of a channel
};
// dir 0 = forward, 1 = backward; form 0 = b2c_bn_forward_train / b2c_bn_backward, 1 = *_fused, 2 = *_fused_res.  `ptrs` are the
// call's tensors (compared for alignment, never dereferenced).  Refuses what the entry points refuse about the shape.
int bn_plan(int dir, int form, int N, int C, int S, std::initializer_list<const void*> ptrs, const char* who, BnPlan* p);

// Largest cluster the per-channel kernels may use on this device: B2C_BN_CLUSTER (1..16, default 8 = the portable limit) capped by what the
// device schedules -- 16-CTA clusters are a non-portable size (cudaFuncAttributeNonPortableClusterSizeAllowed); the probe kernel
// stands for the real ones (same block size, no dynamic shared memory: the hardware limit is per GPC, not per kernel).
static __global__ void bn_cluster_probe_kernel() {}
static inline unsigned bn_max_cluster() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("B2C_BN_CLUSTER");
    int want = e ? atoi(e) : 8;
    want = want >= 16 ? 16 : want >= 8 ? 8 : want >= 4 ? 4 : want >= 2 ? 2 : 1;
    if (want > 8) {
      int clusters = 0;
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3(16, 1, 1); cfg.blockDim = dim3(BN_THREADS, 1, 1);
      cudaLaunchAttribute attr[1];
      attr[0].id = cudaLaunchAttributeClusterDimension;
      attr[0].val.clusterDim.x = 16; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
      cfg.attrs = attr; cfg.numAttrs = 1;
      if (cudaFuncSetAttribute(bn_cluster_probe_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess ||
          cudaOccupancyMaxActiveClusters(&clusters, bn_cluster_probe_kernel, &cfg) != cudaSuccess || clusters < 1) {
        (void)cudaGetLastError();
        want = 8;
      }
    }
    v = want;
  }
  return (unsigned)v;
}
// cluster size for the per-channel kernels: ~16K values or more per CTA, at least one CTA per SM, at most bn_max_cluster().
// FEWER, FATTER CTAs win: halving the slices (so that both backward streams fit shared memory) slows the 28x28 layers down,
// 16-CTA clusters slow the 56x56 ones (co-scheduling sixteen 512-thread CTAs in one GPC), and a floor of two CTAs per SM puts
// the 14x14 layers on many short CTAs in two waves (a fixed cost per launch whatever the tensor size).
static inline unsigned bn_cluster_size(int N, int C, int S) {
  const size_t E = (size_t)N * S;
  const unsigned maxc = bn_max_cluster();
  unsigned cs = 1;
  while (cs < maxc && E / (cs * 2) >= 16384) cs *= 2;
  while (cs < maxc && (size_t)C * cs < (unsigned)sm_count()) cs *= 2;
  return cs;
}
// one cluster of `cs` CTAs per channel; `smem_pad` bytes of (unused) dynamic shared memory bound the CTAs per SM
// threads per CTA: 512, or 128 for channels of at most 4 096 values (ResNet-50's 7x7 layers: 2 048 channels x 3 136 values --
// one 512-thread CTA per channel is several waves of CTAs that are all set-up and barriers)
static inline unsigned bn_threads(int N, int S, bool forward) {
  // 4 097 .. 16 384 values per channel (the 14x14 layers): 256 threads forward, 512 backward (the parked streams leave room for
  // two CTAs per SM either way)
  const size_t E = (size_t)N * S;
  return E <= 4096 ? 128u : (E <= 16384 && forward) ? 256u : (unsigned)BN_THREADS;
}
template <typename... Args>
static inline void bn_launch_clustered(void (*kernel)(Args...), unsigned cs, int C, size_t smem_pad, void* stream, unsigned threads, Args... args) {
  if (cs > 8) cudaFuncSetAttribute(kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
  launch_pdl(kernel, dim3(cs, C, 1), dim3(threads, 1, 1), smem_pad, as_stream(stream), cs, args...);
}

}  // namespace b2c
