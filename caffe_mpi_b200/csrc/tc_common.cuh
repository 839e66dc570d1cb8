// tc_common.cuh -- Hopper (sm_90a) building blocks for the tensor-core kernels: mbarrier, proxy fences,
// wgmma shared-memory matrix descriptors, wgmma fence / commit / wait and the accumulator fragment map,
// and the TF32 hi/lo split used by the fp32-equivalent (3xTF32) math mode; TMA loads, shared-memory accessors, the bf16 hi/lo
// split and the fused split-K reduction; and the host plumbing around them (tc_host.cu): tensor-map encoding, the split-K
// planner and workspace, B2C_PROF buffers.
//
// Shared-memory operand layout used by every kernel here: K-major, no swizzle ("interleave"),
// canonical form ((8,m),(4,2)):((4,SBO),(1,LBO)) in fp32 elements, i.e. 8-row x 16-byte core
// matrices of 128 contiguous bytes; consecutive 8-row groups SBO = 128 B apart, consecutive
// 16-byte K chunks LBO = rows*16 + 16 B apart.  The +16 pad makes the eight K chunks of one row
// land in eight different 16-byte bank groups, so both producer mappings (lanes along rows, and
// lanes along K) store conflict-free with 128-bit st.shared.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "b2c_common.cuh"
#include "wgmma_ops.cuh"

namespace b2c {
namespace tc {

constexpr int BK = 32;              // fp32 elements of K per pipeline stage (8 chunks of 16 B)
constexpr int KCHUNKS = BK / 4;

__host__ __device__ constexpr uint32_t tile_lbo(int rows) { return (uint32_t)rows * 16u + 16u; }
__host__ __device__ constexpr uint32_t tile_bytes(int rows) { return KCHUNKS * tile_lbo(rows); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier ------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// Every wait is bounded: a protocol bug (a missed arrive, a wrong parity) must fail the launch with a trap
// ("unspecified launch failure" on the host) instead of hanging the GPU.  The bound is ~2^31 SM cycles (about a
// second), three orders of magnitude beyond the longest legitimate wait in any of these kernels.
__device__ __forceinline__ bool mbar_try(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}" : "=r"(done) : "r"(bar), "r"(parity) : "memory");
  return done != 0;
}
// Timeout handling (cold path).  Default: kill the kernel with `trap` (the host sees "illegal instruction").
// A translation unit that defines B2C_MBAR_DEBUG before including this header records the stuck waits instead:
// g_mbar_dbg[0] = number of timeouts, then up to 31 records of {block, thread, barrier smem address, parity}; with
// B2C_MBAR_TRAP=0 (b2c_debug_mbar_set_trap) the wait then gives up, so a deadlocked kernel drains and
// b2c_debug_mbar_timeouts() can say which role was stuck on which barrier.  (Off by default: the out-of-line call costs the
// register-tight gather kernels a few spilled registers.)
#ifdef B2C_MBAR_DEBUG
static __device__ unsigned int g_mbar_dbg[128];
static __device__ unsigned int g_mbar_trap = 1;
static __device__ __noinline__ void mbar_timeout_trap(uint32_t bar, uint32_t parity) {
  const unsigned int slot = atomicAdd(&g_mbar_dbg[0], 1u);
  if (slot < 31u) {
    unsigned int* r = &g_mbar_dbg[4 + 4 * slot];
    r[0] = blockIdx.x | (blockIdx.y << 16); r[1] = threadIdx.x; r[2] = bar; r[3] = parity;
  }
  __threadfence_system();
  if (g_mbar_trap) asm volatile("trap;");
}
#define TC_DEBUG_EXPORT(name)                                                                                   \
  int name(unsigned int* out, int cap_words, int set_trap) {                                                    \
    if (set_trap >= 0) { const unsigned int v = set_trap ? 1u : 0u; cudaMemcpyToSymbol(::b2c::tc::g_mbar_trap, &v, sizeof(v)); } \
    if (!out) return 0;                                                                                          \
    unsigned int h[128];                                                                                         \
    if (cudaMemcpyFromSymbol(h, ::b2c::tc::g_mbar_dbg, sizeof(h)) != cudaSuccess) return -1;                    \
    for (int i = 0; i < cap_words && i < 128; ++i) out[i] = h[i];                                                \
    unsigned int z[128] = {0};                                                                                   \
    cudaMemcpyToSymbol(::b2c::tc::g_mbar_dbg, z, sizeof(z));                                                     \
    return (int)h[0];                                                                                            \
  }
#else
__device__ __forceinline__ void mbar_timeout_trap(uint32_t, uint32_t) { asm volatile("trap;"); }
#define TC_DEBUG_EXPORT(name)                                                          \
  int name(unsigned int* out, int cap_words, int) {                                    \
    for (int i = 0; out && i < cap_words && i < 128; ++i) out[i] = 0;                  \
    return 0;                                                                          \
  }
#endif
constexpr long long MBAR_TIMEOUT_CYCLES = 1ll << 31;
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try(bar, parity)) {
    if ((++spins & 0x3ffu) == 0 && clock64() - t0 > MBAR_TIMEOUT_CYCLES) { mbar_timeout_trap(bar, parity); return; }
  }
}
// Waiters that are not on the critical path (epilogue warps waiting a whole tile for the accumulator,
// producers waiting for a free stage) must not spin hot: the warp scheduler prefers high warp ids, and a
// try_wait loop in 4-20 warps starves the single MMA-issuing thread of issue slots.  Back off with nanosleep.
__device__ __forceinline__ void mbar_wait_backoff(uint32_t bar, uint32_t parity, unsigned ns) {
  if (mbar_try(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t spins = 0;
  for (;;) {
    __nanosleep(ns);
    if (mbar_try(bar, parity)) break;
    if ((++spins & 0xffu) == 0 && clock64() - t0 > MBAR_TIMEOUT_CYCLES) { mbar_timeout_trap(bar, parity); return; }
  }
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// generic-proxy st.shared -> visible to the async proxy (wgmma operand reads, TMA stores)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// One lane of a CONVERGED warp.  TMA issue is a uniform-datapath instruction: issued under `if (lane == 0)` the
// compiler wraps it in an ELECT/branch loop over the active lanes; with elect.sync on a converged warp it is
// straight-line code.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}" : "=r"(pred));
  return pred != 0;
}

// ---- wgmma ------------------------------------------------------------------------------------------
// 64-bit shared-memory matrix descriptor (sm_90a layout): start address, LBO (K-direction core-matrix stride for
// K-major SWIZZLE_NONE; ignored for swizzled K-major), SBO (stride between 8-row groups), layout type in bits 62-63.
__device__ __forceinline__ uint64_t smem_desc(uint32_t addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  return d;
}
// K-major SWIZZLE_128B tile (what TMA writes with CU_TENSOR_MAP_SWIZZLE_128B): 128-byte rows, 8-row groups 1024 B apart,
// tile base 1024-byte aligned; a K step inside the 128-byte row advances the start address.
__device__ __forceinline__ uint64_t smem_desc_sw128(uint32_t addr) {
  return smem_desc(addr, 16u, 1024u) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R>
__device__ __forceinline__ void wgmma_reg_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Accumulator fragment of m64nN (fp32): element i of thread t of the warpgroup is row frag_row(t, i) (0..63), column
// frag_col(t, i) (0..N-1).
__device__ __forceinline__ int frag_row(int t, int i) { return ((t >> 5) << 4) + ((t & 31) >> 2) + ((i & 2) ? 8 : 0); }
__device__ __forceinline__ int frag_col(int t, int i) { return ((i >> 2) << 3) + ((t & 3) << 1) + (i & 1); }
// named barrier over `n` threads (the consumer warpgroups of a kernel)
__device__ __forceinline__ void named_bar(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
// signal side of a named barrier: counts the calling warp towards `n` without waiting (the waiting side calls named_bar)
__device__ __forceinline__ void named_bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }
// per-warpgroup register budget (all four warps of the warpgroup execute it): .dec returns registers to the CTA's pool,
// .inc waits until the pool holds enough.  The budgets of all warpgroups must fit the registers the CTA was launched with.
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// ---- TF32 split ------------------------------------------------------------------------------------
// fp32-equivalent mode: hi = a with the 13 low mantissa bits cleared (exactly a TF32 value), lo = a - hi
// (exact in fp32, |lo| < 2^-10 |a|; the tensor core reads its top 19 bits).  hi*hi' + hi*lo' + lo*hi'
// then carries ~2^-20 relative error per product -- fp32-class accuracy on the TF32 pipe for two ALU
// ops per element (cvt.rna.tf32 runs at 1/4 rate and made the producers conversion-bound).
// TF32 mode: round-to-nearest (ties away) on the integer pipe: (bits + 0x1000) & ~0x1fff.
__device__ __forceinline__ float to_tf32(float a) {
  return __uint_as_float((__float_as_uint(a) + 0x1000u) & 0xffffe000u);
}
__device__ __forceinline__ void split_tf32(float a, float& hi, float& lo) {
  hi = __uint_as_float(__float_as_uint(a) & 0xffffe000u);
  lo = a - hi;
}

__device__ __forceinline__ void sts128(uint32_t addr, float a, float b, float c, float d) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// store a 4-element K chunk of one row into the hi (and lo) tile
template <bool SPLIT>
__device__ __forceinline__ void store_chunk(uint32_t hi_addr, uint32_t lo_addr, float v0, float v1, float v2, float v3) {
  if (SPLIT) {
    float h0, h1, h2, h3, l0, l1, l2, l3;
    split_tf32(v0, h0, l0); split_tf32(v1, h1, l1); split_tf32(v2, h2, l2); split_tf32(v3, h3, l3);
    sts128(hi_addr, h0, h1, h2, h3);
    sts128(lo_addr, l0, l1, l2, l3);
  } else {
    sts128(hi_addr, to_tf32(v0), to_tf32(v1), to_tf32(v2), to_tf32(v3));
  }
}

__device__ __forceinline__ void sts128u(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
// addr + OFF as an immediate: a run of loads at fixed offsets shares one base register
template <int OFF>
__device__ __forceinline__ float lds32i(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1+%2];" : "=f"(v) : "r"(addr), "n"(OFF));
  return v;
}

// ---- bf16x3 split ------------------------------------------------------------------------------------
// fp32 pair (k even, k odd) -> packed bf16 hi word and packed bf16 lo word; element k sits in the LOW half
// (two consecutive K elements per 32-bit word of the K-major operand tile, little endian)
__device__ __forceinline__ void split_pack_bf16(float e, float o, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(e, o);            // .x = e (low half), .y = o
  const uint32_t hb = *reinterpret_cast<const uint32_t*>(&h);
  const float he = __uint_as_float(hb << 16), ho = __uint_as_float(hb & 0xffff0000u);
  const __nv_bfloat162 l = __floats2bfloat162_rn(e - he, o - ho);   // a - hi is exact in fp32
  hi = hb;
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

// ---- TMA ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_3d(uint32_t smem_dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}

// ---- split-K reduction fused into the tile's own CTAs (the weight-gradient kernels and the NT GEMM) -------------------------
// Round 1 ran a second kernel per layer (wgrad_reduce_kernel, 53 launches / 0.58 ms per ResNet-50 step).  Here the `splits` CTAs
// of an output tile meet at a counter in the workspace once their partial tiles are in global memory -- the whole grid is one
// wave by construction (plan_splitk: never more CTAs than SMs), so every CTA of the tile is resident -- and then each CTA adds
// up its 1/splits slice of the tile over the partials IN SPLIT ORDER and accumulates it into dW: the summation order of every
// element is fixed, so the result is bit-reproducible and equal to what the separate kernel produced.
__device__ __forceinline__ void splitk_fused_reduce(const float* __restrict__ part, float* __restrict__ dw, unsigned int* counter,
                                                    int split, int splits, long long plane, long long tile_base, int ld, int nrows, int ncols) {
  __syncthreads();                                   // this CTA's partial tile is complete (epilogue warps)
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(counter, 1u);
    const long long t0 = clock64();
    unsigned int seen;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(counter) : "memory");
      if (seen < (unsigned)splits) {
        __nanosleep(64);
        if (clock64() - t0 > MBAR_TIMEOUT_CYCLES) asm volatile("trap;");
      }
    } while (seen < (unsigned)splits);
  }
  __syncthreads();
  const int total = nrows * ncols;
  const int per = (total + splits - 1) / splits;
  const int e_end = min(total, (split + 1) * per);
  for (int e = split * per + (int)threadIdx.x; e < e_end; e += (int)blockDim.x) {
    const int r = e / ncols, c = e - r * ncols;
    const long long idx = tile_base + (long long)r * ld + c;
    // loads of 8 splits in flight, added in split order (the order, not the batching, fixes the rounding)
    float acc = 0.0f;
    int s2 = 0;
    for (; s2 + 8 <= splits; s2 += 8) {
      float v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) v[u] = __ldcg(part + (long long)(s2 + u) * plane + idx);
#pragma unroll
      for (int u = 0; u < 8; ++u) acc += v[u];
    }
    for (; s2 < splits; ++s2) acc += __ldcg(part + (long long)s2 * plane + idx);
    dw[idx] += acc;
  }
}

// ---- host side (tc_host.cu) ----------------------------------------------------------------------------
// cuTensorMapEncodeTiled of a 3-D tensor (no interleave, 256-byte L2 promotion, no OOB NaN fill: out-of-range elements read as
// zero and are not written); `what` names the map in the failure message
int make_tensor_map_3d(CUtensorMap* map, CUtensorMapDataType dtype, const void* base, const cuuint64_t (&dims)[3],
                       const cuuint64_t (&byte_strides)[2], const cuuint32_t (&box)[3], CUtensorMapSwizzle swizzle, const char* what);

// One wave of split-K CTAs: every CTA pays a fixed prologue + epilogue (partial tile write), so fewer, longer CTAs win; never more
// CTAs than SMs (a partial second wave costs a full CTA time), at least min_kb_per_split of the nkb K blocks per split, and the
// split length rebalanced so no split is empty.  `tiles`: output tiles of the launch (CTAs per split).
void plan_splitk(long long nkb, long long tiles, int min_kb_per_split, int* splits, int* kb_per_split);

// split-K workspace: [arrival counters, one u32 per output tile (<= #SMs)][partials: splits x plane_elems fp32]; 0 for one split
constexpr size_t SPLITK_COUNTER_BYTES = 1024;
inline size_t splitk_workspace_bytes(int splits, long long plane_elems) {
  return splits > 1 ? SPLITK_COUNTER_BYTES + sizeof(float) * (size_t)splits * (size_t)plane_elems : 0;
}
// Points a split-K kernel's parameters at the workspace: `out` at the partials (splits > 1) or at dW itself, `grad` at dW,
// `counters` at the zeroed counters.  `what` names the kernel in the failure message.
template <class P>
int bind_splitk(P& p, int splits, long long plane_elems, float* dw, void* ws, size_t ws_bytes, cudaStream_t st, const char* what) {
  const size_t need = splitk_workspace_bytes(splits, plane_elems);
  if (need && (!ws || ws_bytes < need)) return fail(B2C_ERR_WORKSPACE, "%s: workspace too small", what);
  p.out = splits > 1 ? reinterpret_cast<float*>(static_cast<char*>(ws) + SPLITK_COUNTER_BYTES) : dw;
  p.grad = dw;
  p.counters = static_cast<unsigned int*>(ws);
  if (splits > 1) B2C_CUDA_OK(cudaMemsetAsync(ws, 0, SPLITK_COUNTER_BYTES, st));
  return B2C_OK;
}

// B2C_PROF=1: a 32-word device buffer for the kernels' clock64 phase counters, zeroed on `st`; null when the switch is off
long long* prof_buffer(cudaStream_t st);
// the counters the last launch wrote (synchronous)
void prof_read(const long long* buf, long long (&h)[32]);

}  // namespace tc
}  // namespace b2c
