// layers_fused.cu -- fused forms of the BatchNorm / ReLU / Eltwise chain of a residual block (HBM-bound passes; fusion is the
// only lever left once each pass runs close to the HBM roofline):
//
//   b2c_bn_forward_train_fused : batch statistics + y = [max(0, .)] (gamma * x_norm + beta).  x_norm is NOT written: the
//                                backward pass recomputes it from the layer's input x and the saved mean / inverse std
//                                (the reference keeps x_norm_, batch_norm_layer.cu:60-75).
//   b2c_bn_backward_fused      : dgamma / dbeta / dx with the ReLU mask folded in: the mask (top > 0) equals
//                                (gamma * x_norm + beta > 0) recomputed with the forward's own expression, so the result is
//                                bit-identical to ReLU::Backward followed by BatchNorm::Backward (relu_layer.cpp:27-41,
//                                batch_norm_layer.cpp:230-300).
//     Both are ONE launch: a thread-block cluster per channel reduces its slice of the channel (phase 1), the partial sums
//     meet in rank 0 through distributed shared memory, the result is broadcast back the same way, and every CTA walks ITS
//     OWN slice again for the elementwise pass (phase 2).  The slice is ~100 KB per CTA and at most two CTAs run per SM
//     (bounded by a dynamic-shared-memory pad), so what is in flight (~26 MB on 132 SMs) sits in the 50 MB L2 and the second
//     walk does not go to HBM: 8 B/element forward (read x, write y) and 12 B/element backward (read dy, x, write dx) instead of 12 / 20
//     for the two-launch form (B2C_BN_ONEPASS=0), 12 / 32 for the unfused layers.
//   b2c_add_relu               : y = max(0, a + b)                      (Eltwise SUM + in-place ReLU, one pass instead of two)
//   b2c_relu_backward2         : dx_a = dx_b = dy * (y > 0)             (ReLU backward + Eltwise SUM backward's two copies)
#include <cooperative_groups.h>
#include <initializer_list>
#include <stdlib.h>
#include "b2c_common.cuh"
#include "bn_common.cuh"

namespace cg = cooperative_groups;

namespace b2c {

constexpr int FB_EW = 8;           // units per thread of the elementwise passes (two-launch form)
struct FChanCursor {                // flattened unit index of the tensor -> (offset in plane, channel)
  unsigned p, c;
  __device__ __forceinline__ void init(size_t i, unsigned units, unsigned C) { const size_t plane = i / units; p = (unsigned)(i - plane * units); c = (unsigned)(plane % C); }
  __device__ __forceinline__ void advance(unsigned step, unsigned units, unsigned C) { p += step; while (p >= units) { p -= units; if (++c == C) c = 0; } }
};

template <bool VEC, bool RELU>
__global__ void __launch_bounds__(256)
bn_norm_fused_kernel(size_t total_units, int C, int S, const float* __restrict__ x, const float* __restrict__ mean,
                     const float* __restrict__ invstd, const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ y) {
  pdl_wait();
  const unsigned units = VEC ? S / 4 : S;
  size_t i = (size_t)blockIdx.x * (256 * FB_EW) + threadIdx.x;
  if (i >= total_units) return;
  FChanCursor cur;
  cur.init(i, units, C);
  const bool affine = gamma != nullptr;
#pragma unroll 2
  for (int k = 0; k < FB_EW && i < total_units; ++k, i += 256) {
    const float m = mean[cur.c], is = invstd[cur.c], g = affine ? gamma[cur.c] : 1.f, bt = affine ? beta[cur.c] : 0.f;
    if (VEC) {
      const float4 v = reinterpret_cast<const float4*>(x)[i];
      float4 o;
      o.x = bn_y(bn_xn(v.x, m, is), g, bt, affine); o.y = bn_y(bn_xn(v.y, m, is), g, bt, affine);
      o.z = bn_y(bn_xn(v.z, m, is), g, bt, affine); o.w = bn_y(bn_xn(v.w, m, is), g, bt, affine);
      if (RELU) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
      reinterpret_cast<float4*>(y)[i] = o;
    } else {
      const float o = bn_y(bn_xn(x[i], m, is), g, bt, affine);
      y[i] = RELU ? fmaxf(o, 0.f) : o;
    }
    cur.advance(256, units, C);
  }
}

// per channel: sum dy_eff * x_norm, sum dy_eff with dy_eff = RELU ? (y_pre > 0 ? dy : 0) : dy, one thread-block cluster per channel
// this CTA's share of sum dy_eff * x_norm (a) and sum dy_eff (b) of channel c
// MASK: 0 = dy as it is, 1 = ReLU mask recomputed from the forward's expression, 2 = ReLU mask from the tensor `ym` (the
// post-activation output of the Eltwise sum this BatchNorm feeds: ym > 0)
// CACHE bit 0: park every loaded unit of x in shared memory (cx[unit index - slice start]); bit 1: park the MASKED (and summed) gradient (cd)
// U: loads in flight per thread and stream; a thread visits its units in the same order whatever U is, so U does not change the sums
// dy2 (may be null): a second part of the upstream gradient, added to dy element by element (the shadow diff of a blob that fans
// out: SplitLayer::Backward's accumulation, b2c_add's a + b, folded into this read)
// PRE: the parked streams were brought into shared memory by the thread's own cp.async prefetch (x in cx, the RAW gradient in cd):
// they are read from there, and the masked gradient overwrites the raw one in place
template <bool VEC, int MASK, int CACHE = 0, int U = BN_U, bool PRE = false>
__device__ __forceinline__ void bn_bwd_partial_fused(int N, int C, int S, int c, const float* __restrict__ dy, const float* __restrict__ x,
                                                     const float* __restrict__ ym, float m, float is, float g, float bt, bool affine,
                                                     unsigned rank, unsigned nranks, float& a, float& b, void* cx = nullptr, void* cd = nullptr,
                                                     const float* __restrict__ dy2 = nullptr) {
  const unsigned FB_THREADS = blockDim.x;
  const unsigned units = VEC ? S / 4 : S;
  unsigned lo, hi;
  bn_slice((unsigned)N * units, rank, nranks, lo, hi);
  a = 0.f; b = 0.f;
  float a2 = 0.f, b2 = 0.f;
  PlaneCursor cur;
  unsigned i = lo + threadIdx.x;
  if (i < hi) cur.init(i, units);
  // masked upstream gradient and recomputed x_norm of one element
  auto prep = [&](float& d, float xv, float yv) {
    const float xn = bn_xn(xv, m, is);
    if (MASK == 1) d = relu_mask(d, bn_y(xn, g, bt, affine));                 // the mask ReLU::Backward applies, from the recomputed pre-activation
    if (MASK == 2) d = relu_mask(d, yv);
    return xn;
  };
  for (; i < hi; i += U * FB_THREADS) {
    size_t off[U];
    bool ok[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      ok[u] = i + u * FB_THREADS < hi;
      off[u] = ((size_t)cur.n * C + c) * units + cur.p;
      cur.advance(FB_THREADS, units);
    }
    if (VEC) {
      float4 d[U], v[U], t[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (PRE && (CACHE & 2)) d[u] = ok[u] ? static_cast<const float4*>(cd)[i + u * FB_THREADS - lo] : make_float4(0.f, 0.f, 0.f, 0.f);
        else d[u] = ok[u] ? reinterpret_cast<const float4*>(dy)[off[u]] : make_float4(0.f, 0.f, 0.f, 0.f);
        if (MASK == 2 && dy2 && ok[u]) {
          const float4 e = reinterpret_cast<const float4*>(dy2)[off[u]];
          d[u] = make_float4(__fadd_rn(d[u].x, e.x), __fadd_rn(d[u].y, e.y), __fadd_rn(d[u].z, e.z), __fadd_rn(d[u].w, e.w));
        }
        if (PRE && (CACHE & 1)) v[u] = ok[u] ? static_cast<const float4*>(cx)[i + u * FB_THREADS - lo] : make_float4(m, m, m, m);
        else v[u] = ok[u] ? reinterpret_cast<const float4*>(x)[off[u]] : make_float4(m, m, m, m);
        t[u] = (MASK == 2 && ok[u]) ? reinterpret_cast<const float4*>(ym)[off[u]] : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        // the accumulation order of layers.cu's bn_channel_partial<MODE 1>, so that fused == unfused bit for bit
        const float nx = prep(d[u].x, v[u].x, t[u].x), ny = prep(d[u].y, v[u].y, t[u].y), nz = prep(d[u].z, v[u].z, t[u].z), nw = prep(d[u].w, v[u].w, t[u].w);
        a = fmaf(d[u].x, nx, a); a2 = fmaf(d[u].y, ny, a2); a = fmaf(d[u].z, nz, a); a2 = fmaf(d[u].w, nw, a2);
        b += d[u].x + d[u].y; b2 += d[u].z + d[u].w;
        if ((CACHE & 1) && !PRE && ok[u]) static_cast<float4*>(cx)[i + u * FB_THREADS - lo] = v[u];
        if ((CACHE & 2) && ok[u]) static_cast<float4*>(cd)[i + u * FB_THREADS - lo] = d[u];
      }
    } else {
      float d[U], v[U], t[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (PRE && (CACHE & 2)) d[u] = ok[u] ? static_cast<const float*>(cd)[i + u * FB_THREADS - lo] : 0.f;
        else d[u] = ok[u] ? dy[off[u]] : 0.f;
        if (MASK == 2 && dy2 && ok[u]) d[u] = __fadd_rn(d[u], dy2[off[u]]);
        if (PRE && (CACHE & 1)) v[u] = ok[u] ? static_cast<const float*>(cx)[i + u * FB_THREADS - lo] : m;
        else v[u] = ok[u] ? x[off[u]] : m;
        t[u] = (MASK == 2 && ok[u]) ? ym[off[u]] : 0.f;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const float xn = prep(d[u], v[u], t[u]); a = fmaf(d[u], xn, a); b += d[u];
        if ((CACHE & 1) && !PRE && ok[u]) static_cast<float*>(cx)[i + u * FB_THREADS - lo] = v[u];
        if ((CACHE & 2) && ok[u]) static_cast<float*>(cd)[i + u * FB_THREADS - lo] = d[u];
      }
    }
  }
  a += a2; b += b2;
}

template <bool VEC, bool RELU>
__global__ void __launch_bounds__(BN_THREADS)
bn_bwd_reduce_fused_kernel(int N, int C, int S, const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ mean,
                           const float* __restrict__ invstd, const float* __restrict__ gamma, const float* __restrict__ beta,
                           float* __restrict__ sum_dy_xn, float* __restrict__ sum_dy) {
  pdl_wait();
  __shared__ float2 part;
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned rank = cluster.block_rank(), nranks = cluster.num_blocks();
  const int c = blockIdx.y;
  const bool affine = gamma != nullptr;
  const float m = mean[c], is = invstd[c], g = affine ? gamma[c] : 1.f, bt = affine ? beta[c] : 0.f;
  float a, b;
  bn_bwd_partial_fused<VEC, RELU ? 1 : 0>(N, C, S, c, dy, x, nullptr, m, is, g, bt, affine, rank, nranks, a, b);
  block_sum2(a, b);
  if (threadIdx.x == 0) part = make_float2(a, b);
  cluster.sync();
  if (rank == 0 && threadIdx.x == 0) {
    double s1 = 0.0, s2 = 0.0;
    for (unsigned r = 0; r < nranks; ++r) { const float2 v = *cluster.map_shared_rank(&part, r); s1 += v.x; s2 += v.y; }
    sum_dy_xn[c] = (float)s1; sum_dy[c] = (float)s2;
  }
  cluster.sync();
}

// ---- one-launch forms -----------------------------------------------------------------------------------------------------
// A cluster of 1..8 CTAs per channel.  Phase 1: every CTA streams its slice of the channel through the reduction (the very code
// and order of the two-launch kernels) and parks what it read in SHARED MEMORY (slices are <= ~100 KB at the BASELINE shapes; the
// host picks the cached variant when the slice fits).  The partial sums meet through distributed shared memory: after one
// cluster barrier EVERY thread adds the <= 8 partials in rank order (same bits everywhere, no second barrier for a broadcast).
// Phase 2: the elementwise pass over the same slice reads the parked copy -- the tensor crosses HBM once per direction
// (forward: read x, write y; backward: read dy [, mask], x, write dx [, d_res]) whatever the L2 does.  A closing cluster
// barrier keeps the partials alive until every rank has read them.
// elementwise walk of this CTA's slice of channel c: f(global unit offsets, slice-relative unit indices, validity)
template <int U, typename F>
__device__ __forceinline__ void bn_walk_slice(int N, int C, unsigned units, int c, unsigned rank, unsigned nranks, F&& f) {
  unsigned lo, hi;
  bn_slice((unsigned)N * units, rank, nranks, lo, hi);
  PlaneCursor cur;
  const unsigned TH = blockDim.x;
  unsigned i = lo + threadIdx.x;
  if (i < hi) cur.init(i, units);
  for (; i < hi; i += U * TH) {
    size_t off[U];
    unsigned idx[U];
    bool ok[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      ok[u] = i + u * TH < hi;
      idx[u] = i + u * TH - lo;
      off[u] = ((size_t)cur.n * C + c) * units + cur.p;
      cur.advance(TH, units);
    }
    f(off, idx, ok);
  }
}
// statistics (bn_stats_kernel's code and order) + normalisation [+ residual add] [+ ReLU] of one channel per cluster
// RES: y = [max(0, .)] (BatchNorm(x) + res) -- the Eltwise SUM (and its in-place ReLU) that consumes this layer, folded in
// CACHE: the slice is parked in dynamic shared memory between the phases (else phase 2 reads x again from global memory / L2)
// CACHE: 0 = phase 2 reads x again from global memory / L2; 1 = the slice is parked in dynamic shared memory by phase 1's loads;
// 2 = the whole slice is first brought in with cp.async (every thread issues ALL its units' copies at once -- ~100 KB in flight
// per CTA against 32 KB with four register loads per thread -- and waits for its own), both phases then read shared memory
__device__ __forceinline__ void bn_cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void bn_cp_async4(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
template <bool VEC, bool RELU, bool RES, int CACHE>
__global__ void __launch_bounds__(BN_THREADS, 2)
bn_fwd_onepass_kernel(int N, int C, int S, const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                      float eps, float maf, int first, float* __restrict__ mean, float* __restrict__ invstd, float* __restrict__ run_mean,
                      float* __restrict__ run_var, const float* __restrict__ res, float* __restrict__ y) {
  pdl_wait();
  extern __shared__ float4 bn_cache[];
  __shared__ float2 part[2];
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned rank = cluster.block_rank(), nranks = cluster.num_blocks();
  const int c = blockIdx.y;
  if (CACHE == 2) {
    bn_walk_slice<BN_U>(N, C, VEC ? S / 4 : S, c, rank, nranks, [&](const size_t (&off)[BN_U], const unsigned (&idx)[BN_U], const bool (&ok)[BN_U]) {
#pragma unroll
      for (int u = 0; u < BN_U; ++u)
        if (ok[u]) {
          if (VEC) bn_cp_async16(bn_cache + idx[u], reinterpret_cast<const float4*>(x) + off[u]);
          else bn_cp_async4(reinterpret_cast<float*>(bn_cache) + idx[u], x + off[u]);
        }
    });
    asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
  }
  float m, var_eps;
  bn_channel_stats<VEC, CACHE>(cluster, N, C, S, c, x, eps, part, bn_cache, m, var_eps);
  const float is = 1.0f / sqrtf(var_eps);
  if (rank == 0 && threadIdx.x == 0) {
    mean[c] = m;
    invstd[c] = is;
    if (first) { run_mean[c] = m; run_var[c] = var_eps; }                         // iter_ <= 1: copy (:199-204)
    else { run_mean[c] = (1.f - maf) * m + maf * run_mean[c]; run_var[c] = (1.f - maf) * var_eps + maf * run_var[c]; }
  }
  const bool affine = gamma != nullptr;
  const float g = affine ? gamma[c] : 1.f, bt = affine ? beta[c] : 0.f;
  auto one = [&](float v, float r) {
    float o = bn_y(bn_xn(v, m, is), g, bt, affine);
    if (RES) o = __fadd_rn(o, r);                     // add_relu_kernel's a + b
    return RELU ? fmaxf(o, 0.f) : o;
  };
  bn_walk_slice<BN_U>(N, C, VEC ? S / 4 : S, c, rank, nranks, [&](const size_t (&off)[BN_U], const unsigned (&idx)[BN_U], const bool (&ok)[BN_U]) {
    if (VEC) {
      float4 v[BN_U], r[BN_U];
#pragma unroll
      for (int u = 0; u < BN_U; ++u) {
        if (ok[u]) v[u] = CACHE ? bn_cache[idx[u]] : reinterpret_cast<const float4*>(x)[off[u]];
        r[u] = (RES && ok[u]) ? reinterpret_cast<const float4*>(res)[off[u]] : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < BN_U; ++u)
        if (ok[u]) reinterpret_cast<float4*>(y)[off[u]] = make_float4(one(v[u].x, r[u].x), one(v[u].y, r[u].y), one(v[u].z, r[u].z), one(v[u].w, r[u].w));
    } else {
      const float* cache1 = reinterpret_cast<const float*>(bn_cache);
      float v[BN_U], r[BN_U];
#pragma unroll
      for (int u = 0; u < BN_U; ++u) { if (ok[u]) v[u] = CACHE ? cache1[idx[u]] : x[off[u]]; r[u] = (RES && ok[u]) ? res[off[u]] : 0.f; }
#pragma unroll
      for (int u = 0; u < BN_U; ++u) if (ok[u]) y[off[u]] = one(v[u], r[u]);
    }
  });
  cluster.sync();                                   // nobody leaves while a peer may still be reading its partial sums
}

// dgamma / dbeta reduction + dx of one channel per cluster
// MASK == 2 (residual form): dy is the diff of the Eltwise sum's top, ym its (post-ReLU) data; the masked gradient is also what the
// sum's OTHER bottom receives: written to d_res when that is not null (EltwiseLayer::Backward's second copy)
// CACHE: bit 0 = x parked in shared memory, bit 1 = the masked (and summed) gradient parked; what is not parked is read again in
// phase 2.  When only one stream fits, the residual form parks the gradient (it stands for up to three input streams: dy, dy2,
// the mask source), the plain forms park x.
// PRE: the parked streams come in by cp.async before the reduction (all of a thread's units in flight at once), see the forward kernel
template <bool VEC, int MASK, int CACHE, bool PRE>
__global__ void __launch_bounds__(BN_THREADS, 2)
bn_bwd_onepass_kernel(int N, int C, int S, float inv_cnt, unsigned slice_units, const float* __restrict__ dy, const float* __restrict__ x,
                      const float* __restrict__ ym, const float* __restrict__ mean, const float* __restrict__ invstd,
                      const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ sum_dy_xn,
                      float* __restrict__ sum_dy, float* __restrict__ dx, float* __restrict__ d_res, const float* __restrict__ dy2) {
  pdl_wait();
  constexpr int U = MASK == 2 ? 2 : BN_U;           // three input streams in the residual form: fewer units in flight per stream (64 registers)
  extern __shared__ float4 bn_cache[];
  __shared__ float2 part;
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned rank = cluster.block_rank(), nranks = cluster.num_blocks();
  const int c = blockIdx.y;
  const bool affine = gamma != nullptr;
  const float m = mean[c], is = invstd[c], g = affine ? gamma[c] : 1.f, bt = affine ? beta[c] : 0.f;
  // the two parked streams: x first, the masked gradient behind it (slice_units units each)
  constexpr bool PX = (CACHE & 1) != 0, PD = (CACHE & 2) != 0;
  void* cx = bn_cache;
  void* cd = !PX ? static_cast<void*>(bn_cache)
                 : VEC ? static_cast<void*>(bn_cache + slice_units) : static_cast<void*>(reinterpret_cast<float*>(bn_cache) + slice_units);
  if (PRE && CACHE != 0) {
    bn_walk_slice<U>(N, C, VEC ? S / 4 : S, c, rank, nranks, [&](const size_t (&off)[U], const unsigned (&idx)[U], const bool (&ok)[U]) {
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (ok[u]) {
          if (VEC) {
            if (PX) bn_cp_async16(static_cast<float4*>(cx) + idx[u], reinterpret_cast<const float4*>(x) + off[u]);
            if (PD) bn_cp_async16(static_cast<float4*>(cd) + idx[u], reinterpret_cast<const float4*>(dy) + off[u]);
          } else {
            if (PX) bn_cp_async4(static_cast<float*>(cx) + idx[u], x + off[u]);
            if (PD) bn_cp_async4(static_cast<float*>(cd) + idx[u], dy + off[u]);
          }
        }
    });
    asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
  }
  float a, b;
  bn_bwd_partial_fused<VEC, MASK, CACHE, U, PRE && CACHE != 0>(N, C, S, c, dy, x, ym, m, is, g, bt, affine, rank, nranks, a, b, cx, cd, dy2);
  block_sum2(a, b);
  if (threadIdx.x == 0) part = make_float2(a, b);
  cluster.sync();
  double s1, s2;
  bn_cluster_sum(cluster, &part, nranks, s1, s2);
  const float sdx = (float)s1, sdy = (float)s2;
  if (rank == 0 && threadIdx.x == 0) { sum_dy_xn[c] = sdx; sum_dy[c] = sdy; }
  const float gi = __fmul_rn(g, is), mdy = bn_mean_term(sdy, inv_cnt), mdx = bn_mean_term(sdx, inv_cnt);
  // upstream gradient (masked in place unless it comes from the cache, where it already is) -> dx
  auto one = [&](float& d, float xv, float yv) {
    const float xn = bn_xn(xv, m, is);
    if (!PD) {
      if (MASK == 1) d = relu_mask(d, bn_y(xn, g, bt, affine));
      if (MASK == 2) d = relu_mask(d, yv);
    }
    return bn_dx(d, xn, gi, mdy, mdx);
  };
  bn_walk_slice<U>(N, C, VEC ? S / 4 : S, c, rank, nranks, [&](const size_t (&off)[U], const unsigned (&idx)[U], const bool (&ok)[U]) {
    if (VEC) {
      float4 d[U], v[U], t[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (ok[u]) {
          d[u] = PD ? static_cast<const float4*>(cd)[idx[u]] : reinterpret_cast<const float4*>(dy)[off[u]];
          if (MASK == 2 && !PD && dy2) {
            const float4 e = reinterpret_cast<const float4*>(dy2)[off[u]];
            d[u] = make_float4(__fadd_rn(d[u].x, e.x), __fadd_rn(d[u].y, e.y), __fadd_rn(d[u].z, e.z), __fadd_rn(d[u].w, e.w));
          }
          v[u] = PX ? static_cast<const float4*>(cx)[idx[u]] : reinterpret_cast<const float4*>(x)[off[u]];
        }
        t[u] = (MASK == 2 && !PD && ok[u]) ? reinterpret_cast<const float4*>(ym)[off[u]] : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (ok[u]) {
          float4 o;
          o.x = one(d[u].x, v[u].x, t[u].x); o.y = one(d[u].y, v[u].y, t[u].y); o.z = one(d[u].z, v[u].z, t[u].z); o.w = one(d[u].w, v[u].w, t[u].w);
          reinterpret_cast<float4*>(dx)[off[u]] = o;
          if (MASK == 2 && d_res) reinterpret_cast<float4*>(d_res)[off[u]] = d[u];
        }
    } else {
      float d[U], v[U], t[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (ok[u]) {
          d[u] = PD ? static_cast<const float*>(cd)[idx[u]] : dy[off[u]];
          if (MASK == 2 && !PD && dy2) d[u] = __fadd_rn(d[u], dy2[off[u]]);
          v[u] = PX ? static_cast<const float*>(cx)[idx[u]] : x[off[u]];
        }
        t[u] = (MASK == 2 && !PD && ok[u]) ? ym[off[u]] : 0.f;
      }
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (ok[u]) {
          dx[off[u]] = one(d[u], v[u], t[u]);
          if (MASK == 2 && d_res) d_res[off[u]] = d[u];
        }
    }
  });
  cluster.sync();                                   // nobody leaves while a peer may still be reading its partial sums
}

// dx = gamma * invstd * (dy_eff - mean(dy_eff) - x_norm * mean(dy_eff * x_norm))
template <bool VEC, bool RELU>
__global__ void __launch_bounds__(256)
bn_bwd_dx_fused_kernel(size_t total_units, int C, int S, float inv_cnt, const float* __restrict__ dy, const float* __restrict__ x,
                       const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ gamma,
                       const float* __restrict__ beta, const float* __restrict__ sum_dy_xn, const float* __restrict__ sum_dy, float* __restrict__ dx) {
  pdl_wait();
  const unsigned units = VEC ? S / 4 : S;
  size_t i = (size_t)blockIdx.x * (256 * FB_EW) + threadIdx.x;
  if (i >= total_units) return;
  FChanCursor cur;
  cur.init(i, units, C);
  const bool affine = gamma != nullptr;
#pragma unroll 2
  for (int k = 0; k < FB_EW && i < total_units; ++k, i += 256) {
    const float m = mean[cur.c], is = invstd[cur.c], g = affine ? gamma[cur.c] : 1.f, bt = affine ? beta[cur.c] : 0.f;
    const float gi = __fmul_rn(g, is), mdy = bn_mean_term(sum_dy[cur.c], inv_cnt), mdx = bn_mean_term(sum_dy_xn[cur.c], inv_cnt);
    auto one = [&](float d, float xv) {
      const float xn = bn_xn(xv, m, is);
      if (RELU) d = relu_mask(d, bn_y(xn, g, bt, affine));
      return bn_dx(d, xn, gi, mdy, mdx);
    };
    if (VEC) {
      const float4 d = reinterpret_cast<const float4*>(dy)[i], v = reinterpret_cast<const float4*>(x)[i];
      reinterpret_cast<float4*>(dx)[i] = make_float4(one(d.x, v.x), one(d.y, v.y), one(d.z, v.z), one(d.w, v.w));
    } else {
      dx[i] = one(dy[i], x[i]);
    }
    cur.advance(256, units, C);
  }
}

__global__ void __launch_bounds__(256) add_relu_kernel(size_t n, int vec, const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ y) {
  pdl_wait();
  const size_t n4 = vec ? n / 4 : 0, tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  for (size_t i = tid; i < n4; i += step) {
    const float4 u = reinterpret_cast<const float4*>(a)[i], v = reinterpret_cast<const float4*>(b)[i];
    reinterpret_cast<float4*>(y)[i] = make_float4(fmaxf(u.x + v.x, 0.f), fmaxf(u.y + v.y, 0.f), fmaxf(u.z + v.z, 0.f), fmaxf(u.w + v.w, 0.f));
  }
  for (size_t i = n4 * 4 + tid; i < n; i += step) y[i] = fmaxf(a[i] + b[i], 0.f);
}
__global__ void __launch_bounds__(256)
relu_bwd2_kernel(size_t n, int vec, const float* __restrict__ dy, const float* __restrict__ y, float* __restrict__ dxa, float* __restrict__ dxb) {
  pdl_wait();
  const size_t n4 = vec ? n / 4 : 0, tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  for (size_t i = tid; i < n4; i += step) {
    const float4 d = reinterpret_cast<const float4*>(dy)[i], v = reinterpret_cast<const float4*>(y)[i];
    const float4 o = make_float4(relu_mask(d.x, v.x), relu_mask(d.y, v.y), relu_mask(d.z, v.z), relu_mask(d.w, v.w));
    if (dxa) reinterpret_cast<float4*>(dxa)[i] = o;
    if (dxb) reinterpret_cast<float4*>(dxb)[i] = o;
  }
  for (size_t i = n4 * 4 + tid; i < n; i += step) {
    const float o = relu_mask(dy[i], y[i]);
    if (dxa) dxa[i] = o;
    if (dxb) dxb[i] = o;
  }
}

// ---- Accuracy (src/caffe/layers/accuracy_layer.cpp:44-100): a sample counts when its label is among the top_k scores; ties are
// ordered like std::greater<pair<float,int>> (equal scores: the HIGHER class index ranks first).  One warp per sample.
__global__ void __launch_bounds__(256)
accuracy_kernel(int N, int C, int top_k, const float* __restrict__ scores, const float* __restrict__ labels, unsigned int* __restrict__ hits) {
  pdl_wait();
  const int warp = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (warp >= N) return;
  const int lab = (int)labels[warp];
  if (lab < 0 || lab >= C) return;                       // the reference DCHECKs the range; out-of-range labels never hit
  const float* z = scores + (size_t)warp * C;
  const float zl = z[lab];
  int above = 0;
  for (int j = lane; j < C; j += 32) { const float v = z[j]; above += (v > zl || (v == zl && j > lab)) ? 1 : 0; }
#pragma unroll
  for (int o = 16; o; o >>= 1) above += __shfl_xor_sync(0xffffffffu, above, o);
  if (lane == 0 && above < top_k) atomicAdd(hits, 1u);
}
__global__ void accuracy_finish_kernel(const unsigned int* hits, int N, float* acc) { pdl_wait(); *acc = (float)*hits / (float)N; }
// The [outer, C, inner] form with ignore_label and the per-class counters (b2c_accuracy_ex).  cnt = {hits, counted pixels}, then
// hits_c[C] and num_c[C] when per-class counting is on (per_class != 0).  Integer atomics: the same counts in any order.
__device__ __forceinline__ void accuracy_record(int lab, int C, bool hit, int per_class, unsigned int* __restrict__ cnt) {
  atomicAdd(cnt + 1, 1u);
  if (hit) atomicAdd(cnt, 1u);
  if (per_class && lab >= 0 && lab < C) {
    atomicAdd(cnt + 2 + C + lab, 1u);
    if (hit) atomicAdd(cnt + 2 + lab, 1u);
  }
}
// inner == 1: one warp per sample, as accuracy_kernel
__global__ void __launch_bounds__(256)
accuracy_row_ex_kernel(int N, int C, int top_k, const float* __restrict__ scores, const float* __restrict__ labels, int has_ignore, int ignore_label,
                       int per_class, unsigned int* __restrict__ cnt) {
  pdl_wait();
  const int warp = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (warp >= N) return;
  const int lab = (int)labels[warp];
  if (has_ignore && lab == ignore_label) return;
  const bool in = lab >= 0 && lab < C;
  int above = 0;
  if (in) {
    const float* z = scores + (size_t)warp * C;
    const float zl = z[lab];
    for (int j = lane; j < C; j += 32) { const float v = z[j]; above += (v > zl || (v == zl && j > lab)) ? 1 : 0; }
#pragma unroll
    for (int o = 16; o; o >>= 1) above += __shfl_xor_sync(0xffffffffu, above, o);
  }
  if (lane == 0) accuracy_record(lab, C, in && above < top_k, per_class, cnt);
}
// inner > 1: one thread per pixel column, loads coalesced along inner.  Each thread keeps its hits and count in registers, the warp
// sums them and adds once per warp; the per-class counters live in shared memory (smem != 0, 8 * C bytes) and each CTA adds its
// non-zero ones to the global counters at the end, so no global address takes an atomic per pixel.
__global__ void __launch_bounds__(256)
accuracy_col_kernel(long long pixels, int C, int inner, int top_k, const float* __restrict__ scores, const float* __restrict__ labels,
                    int has_ignore, int ignore_label, int per_class, int smem, unsigned int* __restrict__ cnt) {
  pdl_wait();
  extern __shared__ unsigned int pc_smem[];                   // hits_c[C], num_c[C]
  unsigned int* pc = smem ? pc_smem : cnt + 2;
  if (smem) {
    for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) pc_smem[c] = 0u;
    __syncthreads();
  }
  unsigned int hits = 0, count = 0;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < pixels; p += (long long)gridDim.x * blockDim.x) {
    const int lab = (int)labels[p];
    if (has_ignore && lab == ignore_label) continue;
    ++count;
    if (lab < 0 || lab >= C) continue;                       // out of range: a miss, no class touched
    const long long o = p / inner;
    const float* z = scores + (size_t)o * C * inner + (size_t)(p - o * inner);
    const float zl = z[(size_t)lab * inner];
    int above = 0;
    for (int j = 0; j < C; ++j) { const float v = z[(size_t)j * inner]; above += (v > zl || (v == zl && j > lab)) ? 1 : 0; }
    const bool hit = above < top_k;
    hits += hit ? 1u : 0u;
    if (per_class) {
      atomicAdd(pc + C + lab, 1u);
      if (hit) atomicAdd(pc + lab, 1u);
    }
  }
  hits = __reduce_add_sync(0xffffffffu, hits);
  count = __reduce_add_sync(0xffffffffu, count);
  if ((threadIdx.x & 31) == 0) {
    if (hits) atomicAdd(cnt, hits);
    if (count) atomicAdd(cnt + 1, count);
  }
  if (smem) {
    __syncthreads();
    for (int c = threadIdx.x; c < 2 * C; c += blockDim.x)
      if (pc_smem[c]) atomicAdd(cnt + 2 + c, pc_smem[c]);
  }
}
// accuracy = hits / count (accuracy_layer.cpp:94, NaN for 0 / 0); per_class[c] = num_c == 0 ? 0 : hits_c / num_c (:95-100)
__global__ void __launch_bounds__(256)
accuracy_ex_finish_kernel(int C, const unsigned int* __restrict__ cnt, float* __restrict__ acc, float* __restrict__ per_class) {
  pdl_wait();
  if (blockIdx.x == 0 && threadIdx.x == 0) *acc = (float)cnt[0] / (float)cnt[1];
  if (per_class)
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < C; c += gridDim.x * blockDim.x) {
      const float num = (float)cnt[2 + C + c];
      per_class[c] = num == 0.f ? 0.f : (float)cnt[2 + c] / num;
    }
}

// the statistics kernel of layers.cu (same launch for the fused and the unfused forward)
int launch_bn_stats(const BnPlan& p, int N, int C, int S, const float* x, float eps, float maf, int first, float* mean, float* invstd,
                    float* run_mean, float* run_var, void* stream);

// B2C_BN_ONEPASS (default 1): statistics / reduction and the elementwise pass in one launch per BatchNorm direction
static bool bn_onepass() {
  static const int on = env_int("B2C_BN_ONEPASS", 1);
  return on != 0;
}
// bytes of one parked stream of the largest slice (rank 0's) of a channel, and the shared-memory budget of one CTA when two
// share an SM (228 KB per SM, 1 KB reserved per CTA, the kernels' static arrays)
static size_t bn_slice_bytes(int N, int S, bool vec, unsigned cs, unsigned* units_out) {
  const size_t total = (size_t)N * (vec ? S / 4 : S);
  const size_t units = (total + cs - 1) / cs;
  if (units_out) *units_out = (unsigned)units;
  return units * (vec ? 16 : 4);
}
static size_t bn_cache_budget() {
  static const long v = env_int("B2C_BN_CACHE_KB", 110) * 1024;   // 0: never park (phase 2 re-reads global memory)
  return (size_t)v;
}
template <typename K>
static int bn_onepass_attr(K kernel, size_t smem) {
  B2C_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return B2C_OK;
}
static bool fb_vec_ok(int S, std::initializer_list<const void*> ptrs) {
  if (S % 4) return false;
  for (const void* p : ptrs) if (reinterpret_cast<uintptr_t>(p) & 15) return false;
  return true;
}

// The one place that picks a BatchNorm training launch (bn_common.cuh).  Every switch is read here, once per process.
int bn_plan(int dir, int form, int N, int C, int S, std::initializer_list<const void*> ptrs, const char* who, BnPlan* p) {
  if (dir != 0 && dir != 1) return fail(B2C_ERR_INVALID, "%s: dir must be 0 (forward) or 1 (backward)", who);
  if (form < 0 || form > 2) return fail(B2C_ERR_INVALID, "%s: form must be 0 (unfused), 1 (fused) or 2 (fused_res)", who);
  if (!(N > 0 && C > 0 && S > 0 && (size_t)N * S < (1ull << 31) && C <= 65535)) return fail(B2C_ERR_INVALID, "%s: channel extent out of range", who);
  *p = BnPlan{2, bn_cluster_size(N, C, S), bn_threads(N, S, dir == 0), 0, 0, fb_vec_ok(S, ptrs), 0, 0};
  const size_t slice = bn_slice_bytes(N, S, p->vec, p->cs, &p->slice_units);
  if (form == 0 || (form == 1 && !bn_onepass())) return B2C_OK;
  p->launches = 1;
  const size_t budget = bn_cache_budget();
  if (dir == 0) {
    // B2C_BN_PREFETCH (default 1): cp.async the slice into shared memory before the reduction
    static const int prefetch = env_int("B2C_BN_PREFETCH", 1);
    p->park = slice <= budget ? 1 : 0;
    p->prefetch = p->park && prefetch;
  } else {
    // both streams, one (the gradient in the residual form, x otherwise), nothing
    // B2C_BN_PREFETCH_BWD (default 1; 16.03 -> 15.88 ms per ResNet-50 step): cp.async the parked streams before the reduction
    static const int prefetch = env_int("B2C_BN_PREFETCH_BWD", 1);
    p->park = 2 * slice <= budget ? 3 : slice <= budget ? (form == 2 ? 2 : 1) : 0;
    p->prefetch = p->park && prefetch;
  }
  p->smem = (size_t)(p->park == 3 ? 2 : p->park ? 1 : 0) * slice;
  return B2C_OK;
}

}  // namespace b2c

using namespace b2c;
#define FNEED(cond, msg) do { if (!(cond)) return fail(B2C_ERR_INVALID, msg); } while (0)

extern "C" int b2c_debug_bn_plan(int dir, int form, int N, int C, int S, const void* const* ptrs, int nptrs, int* out, int n) {
  FNEED(out && n >= 6, "b2c_debug_bn_plan: needs out[6]");
  FNEED(nptrs >= 0 && nptrs <= 6 && (ptrs || !nptrs), "b2c_debug_bn_plan: at most 6 pointers");
  const void* q[6] = {};
  for (int i = 0; i < nptrs; ++i) q[i] = ptrs[i];
  BnPlan p;
  if (int rc = bn_plan(dir, form, N, C, S, {q[0], q[1], q[2], q[3], q[4], q[5]}, "b2c_debug_bn_plan", &p)) return rc;
  out[0] = p.launches; out[1] = (int)p.cs; out[2] = (int)p.threads; out[3] = p.park; out[4] = p.prefetch; out[5] = p.vec ? 1 : 0;
  return B2C_OK;
}

static int bn_forward_fused_impl(int N, int C, int S, const float* x, const float* gamma, const float* beta, float eps,
                                 float moving_average_fraction, int first_iteration, float* running_mean, float* running_var,
                                 float* save_mean, float* save_invstd, const float* residual, float* y, int relu, void* stream) {
  FNEED(x && y && save_mean && save_invstd && running_mean && running_var, "b2c_bn_forward_train_fused: bad argument");
  FNEED((gamma == nullptr) == (beta == nullptr), "b2c_bn_forward_train_fused: gamma and beta go together");
  BnPlan pl;
  if (int rc = bn_plan(0, residual ? 2 : 1, N, C, S, {x, y, residual}, "b2c_bn_forward_train_fused", &pl)) return rc;
  int dev_count = 0;
  if (cudaGetDeviceCount(&dev_count) != cudaSuccess || dev_count == 0) return fail(B2C_ERR_CUDA, "no CUDA device: this library has no CPU fallback");
  const bool vec = pl.vec;
  if (pl.launches == 1) {
    const size_t smem = pl.smem;
    const int cache = pl.park ? (pl.prefetch ? 2 : 1) : 0;     // the kernel's CACHE: parked by cp.async, by the reduction's loads, not at all
#define B2C_FWD0(V, R, Q, P) do { if (int rc = bn_onepass_attr(bn_fwd_onepass_kernel<V, R, Q, P>, smem)) return rc; \
    bn_launch_clustered(bn_fwd_onepass_kernel<V, R, Q, P>, pl.cs, C, smem, stream, pl.threads, N, C, S, x, gamma, beta, eps, moving_average_fraction, first_iteration, \
                        save_mean, save_invstd, running_mean, running_var, residual, y); } while (0)
#define B2C_FWD1(V, R, Q) do { if (cache == 2) B2C_FWD0(V, R, Q, 2); else if (cache == 1) B2C_FWD0(V, R, Q, 1); else B2C_FWD0(V, R, Q, 0); } while (0)
#define B2C_FWD2(V, R) do { if (residual) B2C_FWD1(V, R, true); else B2C_FWD1(V, R, false); } while (0)
    if (vec) { if (relu) B2C_FWD2(true, true); else B2C_FWD2(true, false); }
    else { if (relu) B2C_FWD2(false, true); else B2C_FWD2(false, false); }
#undef B2C_FWD2
#undef B2C_FWD1
#undef B2C_FWD0
    B2C_POST_LAUNCH();
    return B2C_OK;
  }
  if (int rc = launch_bn_stats(pl, N, C, S, x, eps, moving_average_fraction, first_iteration, save_mean, save_invstd, running_mean, running_var, stream)) return rc;
  const size_t units = (size_t)N * C * (vec ? S / 4 : S);
  const unsigned blocks = (unsigned)((units + 256 * FB_EW - 1) / (256 * FB_EW));
  cudaStream_t st = as_stream(stream);
  if (vec) { if (relu) launch_pdl(bn_norm_fused_kernel<true, true>, blocks, 256, 0, st, 0, units, C, S, x, save_mean, save_invstd, gamma, beta, y);
             else launch_pdl(bn_norm_fused_kernel<true, false>, blocks, 256, 0, st, 0, units, C, S, x, save_mean, save_invstd, gamma, beta, y); }
  else { if (relu) launch_pdl(bn_norm_fused_kernel<false, true>, blocks, 256, 0, st, 0, units, C, S, x, save_mean, save_invstd, gamma, beta, y);
         else launch_pdl(bn_norm_fused_kernel<false, false>, blocks, 256, 0, st, 0, units, C, S, x, save_mean, save_invstd, gamma, beta, y); }
  B2C_POST_LAUNCH();
  return B2C_OK;
}

extern "C" int b2c_bn_forward_train_fused(int N, int C, int S, const float* x, const float* gamma, const float* beta, float eps,
                                          float moving_average_fraction, int first_iteration, float* running_mean, float* running_var,
                                          float* save_mean, float* save_invstd, float* y, int relu, void* stream) {
  return bn_forward_fused_impl(N, C, S, x, gamma, beta, eps, moving_average_fraction, first_iteration, running_mean, running_var, save_mean,
                               save_invstd, nullptr, y, relu, stream);
}
// y = [max(0, .)] (BatchNorm(x) + residual): BatchNorm -> Eltwise SUM [-> in-place ReLU] in one launch
extern "C" int b2c_bn_forward_train_fused_res(int N, int C, int S, const float* x, const float* gamma, const float* beta, float eps,
                                              float moving_average_fraction, int first_iteration, float* running_mean, float* running_var,
                                              float* save_mean, float* save_invstd, const float* residual, float* y, int relu, void* stream) {
  FNEED(residual, "b2c_bn_forward_train_fused_res: null residual");
  return bn_forward_fused_impl(N, C, S, x, gamma, beta, eps, moving_average_fraction, first_iteration, running_mean, running_var, save_mean,
                               save_invstd, residual, y, relu, stream);
}

static int bn_backward_fused_impl(int N, int C, int S, const float* dy, const float* dy2, const float* x, const float* y_mask, const float* save_mean,
                                  const float* save_invstd, const float* gamma, const float* beta, float* dgamma, float* dbeta, float* dx,
                                  float* d_residual, int relu, void* stream) {
  FNEED(dy && x && save_mean && save_invstd && dgamma && dbeta && dx, "b2c_bn_backward_fused: null (dgamma/dbeta double as the reduction scratch)");
  FNEED((gamma == nullptr) == (beta == nullptr), "b2c_bn_backward_fused: gamma and beta go together");
  BnPlan pl;
  if (int rc = bn_plan(1, y_mask ? 2 : 1, N, C, S, {dy, dy2, x, dx, y_mask, d_residual}, "b2c_bn_backward_fused", &pl)) return rc;
  int dev_count = 0;
  if (cudaGetDeviceCount(&dev_count) != cudaSuccess || dev_count == 0) return fail(B2C_ERR_CUDA, "no CUDA device: this library has no CPU fallback");
  const bool vec = pl.vec;
  const unsigned cs = pl.cs;
  if (pl.launches == 1) {
    const unsigned slice_units = pl.slice_units;
    const int park = pl.park;
    const size_t smem = pl.smem;
    const float inv_cnt1 = 1.0f / ((float)N * S);
#define B2C_BWDP(V, M, P, Q) do { if (int rc = bn_onepass_attr(bn_bwd_onepass_kernel<V, M, P, Q>, smem)) return rc; \
    bn_launch_clustered(bn_bwd_onepass_kernel<V, M, P, Q>, cs, C, smem, stream, pl.threads, N, C, S, inv_cnt1, slice_units, dy, x, y_mask, save_mean, save_invstd, \
                        gamma, beta, dgamma, dbeta, dx, d_residual, dy2); } while (0)
#define B2C_BWD0(V, M, P) do { if (pl.prefetch && P) B2C_BWDP(V, M, P, true); else B2C_BWDP(V, M, P, false); } while (0)
#define B2C_BWD1(V, M) do { if (park == 3) B2C_BWD0(V, M, 3); else if (park == 2) B2C_BWD0(V, M, 2); else if (park == 1) B2C_BWD0(V, M, 1); else B2C_BWD0(V, M, 0); } while (0)
    if (vec) { if (y_mask) B2C_BWD1(true, 2); else if (relu) B2C_BWD1(true, 1); else B2C_BWD1(true, 0); }
    else { if (y_mask) B2C_BWD1(false, 2); else if (relu) B2C_BWD1(false, 1); else B2C_BWD1(false, 0); }
#undef B2C_BWD1
#undef B2C_BWD0
#undef B2C_BWDP
    B2C_POST_LAUNCH();
    return B2C_OK;
  }
  if (vec) { if (relu) bn_launch_clustered(bn_bwd_reduce_fused_kernel<true, true>, cs, C, (size_t)0, stream, pl.threads, N, C, S, dy, x, save_mean, save_invstd, gamma, beta, dgamma, dbeta);
             else bn_launch_clustered(bn_bwd_reduce_fused_kernel<true, false>, cs, C, (size_t)0, stream, pl.threads, N, C, S, dy, x, save_mean, save_invstd, gamma, beta, dgamma, dbeta); }
  else { if (relu) bn_launch_clustered(bn_bwd_reduce_fused_kernel<false, true>, cs, C, (size_t)0, stream, pl.threads, N, C, S, dy, x, save_mean, save_invstd, gamma, beta, dgamma, dbeta);
         else bn_launch_clustered(bn_bwd_reduce_fused_kernel<false, false>, cs, C, (size_t)0, stream, pl.threads, N, C, S, dy, x, save_mean, save_invstd, gamma, beta, dgamma, dbeta); }
  B2C_POST_LAUNCH();
  const size_t units = (size_t)N * C * (vec ? S / 4 : S);
  const unsigned blocks = (unsigned)((units + 256 * FB_EW - 1) / (256 * FB_EW));
  const float inv_cnt = 1.0f / ((float)N * S);
  cudaStream_t st = as_stream(stream);
  if (vec) { if (relu) launch_pdl(bn_bwd_dx_fused_kernel<true, true>, blocks, 256, 0, st, 0, units, C, S, inv_cnt, dy, x, save_mean, save_invstd, gamma, beta, dgamma, dbeta, dx);
             else launch_pdl(bn_bwd_dx_fused_kernel<true, false>, blocks, 256, 0, st, 0, units, C, S, inv_cnt, dy, x, save_mean, save_invstd, gamma, beta, dgamma, dbeta, dx); }
  else { if (relu) launch_pdl(bn_bwd_dx_fused_kernel<false, true>, blocks, 256, 0, st, 0, units, C, S, inv_cnt, dy, x, save_mean, save_invstd, gamma, beta, dgamma, dbeta, dx);
         else launch_pdl(bn_bwd_dx_fused_kernel<false, false>, blocks, 256, 0, st, 0, units, C, S, inv_cnt, dy, x, save_mean, save_invstd, gamma, beta, dgamma, dbeta, dx); }
  B2C_POST_LAUNCH();
  return B2C_OK;
}

extern "C" int b2c_bn_backward_fused(int N, int C, int S, const float* dy, const float* x, const float* save_mean, const float* save_invstd,
                                     const float* gamma, const float* beta, float* dgamma, float* dbeta, float* dx, int relu, void* stream) {
  return bn_backward_fused_impl(N, C, S, dy, nullptr, x, nullptr, save_mean, save_invstd, gamma, beta, dgamma, dbeta, dx, nullptr, relu, stream);
}
// backward of BatchNorm -> Eltwise SUM -> ReLU run as one layer: d_sum (+ d_sum2 when not null: the second part of a fanned-out
// blob's gradient, added on the fly) / y_sum are the diff and the (post-ReLU) data of the sum's top;
// dx = BatchNorm backward of d_sum * (y_sum > 0); that masked gradient is also written to d_residual (the sum's other bottom) when
// d_residual is not null
extern "C" int b2c_bn_backward_fused_res(int N, int C, int S, const float* d_sum, const float* d_sum2, const float* y_sum, const float* x,
                                         const float* save_mean, const float* save_invstd, const float* gamma, const float* beta,
                                         float* dgamma, float* dbeta, float* dx, float* d_residual, void* stream) {
  FNEED(y_sum, "b2c_bn_backward_fused_res: null y_sum");
  return bn_backward_fused_impl(N, C, S, d_sum, d_sum2, x, y_sum, save_mean, save_invstd, gamma, beta, dgamma, dbeta, dx, d_residual, 1, stream);
}

extern "C" int b2c_add_relu(size_t n, const float* a, const float* b, float* y, void* stream) {
  FNEED(a && b && y, "b2c_add_relu: null pointer");
  int dev_count = 0;
  if (cudaGetDeviceCount(&dev_count) != cudaSuccess || dev_count == 0) return fail(B2C_ERR_CUDA, "no CUDA device: this library has no CPU fallback");
  if (!n) return B2C_OK;
  const bool al = ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(y)) & 15) == 0;
  launch_pdl(add_relu_kernel, grid_for(al ? n / 4 + 1 : n, 256), 256, 0, as_stream(stream), 0, n, al ? 1 : 0, a, b, y);
  B2C_POST_LAUNCH();
  return B2C_OK;
}

extern "C" int b2c_relu_backward2(size_t n, const float* dy, const float* y, float* dx_a, float* dx_b, void* stream) {
  FNEED(dy && y && (dx_a || dx_b), "b2c_relu_backward2: null pointer");
  int dev_count = 0;
  if (cudaGetDeviceCount(&dev_count) != cudaSuccess || dev_count == 0) return fail(B2C_ERR_CUDA, "no CUDA device: this library has no CPU fallback");
  if (!n) return B2C_OK;
  const bool al = ((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(dx_a) | reinterpret_cast<uintptr_t>(dx_b)) & 15) == 0;
  launch_pdl(relu_bwd2_kernel, grid_for(al ? n / 4 + 1 : n, 256), 256, 0, as_stream(stream), 0, n, al ? 1 : 0, dy, y, dx_a, dx_b);
  B2C_POST_LAUNCH();
  return B2C_OK;
}

// accuracy = (#samples whose label is in the top_k scores) / N; `scratch` is 4 bytes of device memory
extern "C" int b2c_accuracy(int N, int C, int top_k, const float* scores, const float* labels, float* accuracy, void* scratch, void* stream) {
  FNEED(scores && labels && accuracy && scratch && N > 0 && C > 0 && top_k > 0 && top_k <= C, "b2c_accuracy: bad argument");
  int dev_count = 0;
  if (cudaGetDeviceCount(&dev_count) != cudaSuccess || dev_count == 0) return fail(B2C_ERR_CUDA, "no CUDA device: this library has no CPU fallback");
  cudaStream_t st = as_stream(stream);
  B2C_CUDA_OK(cudaMemsetAsync(scratch, 0, 4, st));
  launch_pdl(accuracy_kernel, (N * 32 + 255) / 256, 256, 0, st, 0, N, C, top_k, scores, labels, static_cast<unsigned int*>(scratch));
  B2C_POST_LAUNCH();
  launch_pdl(accuracy_finish_kernel, 1, 1, 0, st, 0, static_cast<const unsigned int*>(scratch), N, accuracy);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
extern "C" int b2c_accuracy_ex(int outer, int C, int inner, int top_k, const float* scores, const float* labels, int has_ignore, int ignore_label,
                               float* accuracy, float* per_class, void* scratch, void* stream) {
  FNEED(scores && labels && accuracy && scratch, "b2c_accuracy_ex: null");
  FNEED(outer > 0 && C > 0 && inner > 0 && (long long)outer * inner <= (1ll << 62) / C, "b2c_accuracy_ex: bad shape");
  FNEED(top_k > 0 && top_k <= C, "b2c_accuracy_ex: top_k must be less than or equal to the number of classes.");
  FNEED(inner > 1 || outer <= 0x7fffffff / 32, "b2c_accuracy_ex: too many samples");
  int dev_count = 0;
  if (cudaGetDeviceCount(&dev_count) != cudaSuccess || dev_count == 0) return fail(B2C_ERR_CUDA, "no CUDA device: this library has no CPU fallback");
  cudaStream_t st = as_stream(stream);
  unsigned int* cnt = static_cast<unsigned int*>(scratch);
  const int pc = per_class ? 1 : 0;
  B2C_CUDA_OK(cudaMemsetAsync(scratch, 0, sizeof(unsigned int) * (2 + (pc ? 2 * (size_t)C : 0)), st));
  const int hi = has_ignore ? 1 : 0;
  if (inner == 1) {
    launch_pdl(accuracy_row_ex_kernel, (unsigned)(((long long)outer * 32 + 255) / 256), 256, 0, st, 0, outer, C, top_k, scores, labels, hi, ignore_label, pc, cnt);
  } else {
    const long long pixels = (long long)outer * inner;
    const int smem = pc && C <= 6144 ? 1 : 0;                // per-class counters in shared memory up to the 48 KB default
    launch_pdl(accuracy_col_kernel, grid_for((size_t)pixels, 256), 256, smem ? 8 * (size_t)C : 0, st, 0, pixels, C, inner, top_k, scores, labels,
               hi, ignore_label, pc, smem, cnt);
  }
  B2C_POST_LAUNCH();
  launch_pdl(accuracy_ex_finish_kernel, pc ? (C + 255) / 256 : 1, 256, 0, st, 0, C, (const unsigned int*)cnt, accuracy, per_class);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
