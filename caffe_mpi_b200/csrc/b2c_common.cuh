// b2c_common.cuh -- shared helpers for the sm_90a kernels behind include/b2c.h.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include <string>
#include <utility>

#include "../../include/b2c.h"

namespace b2c {

// ---- error plumbing (thread-local message, b2c_last_error()) -----------------------------
std::string& last_error();
int fail(int code, const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;

#define B2C_CUDA_OK(expr)                                                            \
  do {                                                                               \
    cudaError_t e__ = (expr);                                                        \
    if (e__ != cudaSuccess)                                                          \
      return ::b2c::fail(B2C_ERR_CUDA, "%s:%d %s: %s", __FILE__, __LINE__, #expr,    \
                         cudaGetErrorString(e__));                                   \
  } while (0)

// Count the launch and pick up launch-configuration errors (no sync).
#define B2C_POST_LAUNCH()                                                            \
  do {                                                                               \
    ::b2c::g_launches.fetch_add(1, std::memory_order_relaxed);                       \
    cudaError_t e__ = cudaGetLastError();                                            \
    if (e__ != cudaSuccess)                                                          \
      return ::b2c::fail(B2C_ERR_CUDA, "%s:%d kernel launch: %s", __FILE__, __LINE__,\
                         cudaGetErrorString(e__));                                   \
  } while (0)

inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// ---- programmatic dependent launch (DESIGN §3b) ----------------------------------------------------------------
// Every kernel of a training step is launched by launch_pdl, so its launch overlaps the end of the kernel before it on the
// stream instead of following that kernel's completion.  Such a kernel touches no global memory before pdl_wait(), which
// returns once every prerequisite grid has completed and its writes are visible; it is a no-op in a kernel launched without
// the attribute.  No kernel issues griddepcontrol.launch_dependents: each grid lets the next one launch as its CTAs exit, which
// measured faster than triggering early (DESIGN §3b), and it keeps the chain transitive.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// kernel<<<grid, block, smem, st>>>(args...) with programmatic stream serialization; cluster > 0: in thread-block clusters of
// `cluster` CTAs along x.  The caller follows it with B2C_POST_LAUNCH(), which counts the launch and reports a launch error.
template <typename... KArgs, typename... Args>
inline void launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, unsigned cluster,
                       Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  attr[1].id = cudaLaunchAttributeClusterDimension;
  attr[1].val.clusterDim.x = cluster; attr[1].val.clusterDim.y = 1; attr[1].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = cluster ? 2 : 1;
  cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// The reference sizes grids as ceil(n/512) with 512-thread blocks
// (include/caffe/util/device_alternate.hpp:91-96).  Here element-wise grids are capped at a
// multiple of the SM count and kernels grid-stride.
int sm_count();
inline int grid_for(size_t n, int block, int per_sm = 8) {
  size_t want = (n + block - 1) / block;
  size_t cap = (size_t)sm_count() * per_sm;
  return (int)(want < cap ? (want ? want : 1) : cap);
}

struct ConvShape {
  int N, C, H, W, O, G, kh, kw, sh, sw, ph, pw, dh, dw, has_bias;
  int Ho, Wo, Cg, Og, Kd;  // derived
  bool is_1x1;             // k=1, s=1, p=0 on every axis (base_conv_layer.cpp:99-103)
};

// A weight-gradient kernel's split-K plan as b2c_debug_wgrad_plan reports it: split i walks K blocks
// [i * kb_per_split, min(nkb, (i + 1) * kb_per_split)); bpi = K blocks per image (0: blocks run over the flattened pixels).
struct WgradPlanInfo {
  int splits, kb_per_split;
  long long nkb;
  int cols, bpi, taps;
  bool plane;
  int presplit;          // staged kernel: 1 where dY is split to bf16 hi / lo before the launch
  size_t split_bytes;    // the buffer that split needs (b2c_conv_wgrad_split_bytes)
};

// A forward / data-gradient kernel's tile plan as b2c_debug_conv_plan reports it: 128 x n_tile output tiles, m_tiles x n_tiles
// per group, `tiles` in all (run by persistent_grid(tiles) CTAs); nkb K blocks per tile.  variant: KMODE of the gather kernel
// (conv_tc.cu), BWT of the staged kernel (conv_tc_stg.cu).
struct ConvPlanInfo {
  int n_tile, m_tiles, n_tiles, tiles, nkb, variant;
};

// CTAs of a persistent kernel: one per SM, never more than there are tiles
inline int persistent_grid(int tiles) {
  const int sms = sm_count();
  return tiles < sms ? tiles : sms;
}

// A B2C_* switch: atol of the variable, `dflt` when it is unset.  Switches are read once per process, into a function-local
// `static const` (thread-safe initialisation).
long env_int(const char* name, long dflt);

// ---- kernels in the other translation units -----------------------------------------------------------------
struct PrepEntry;
int launch_im2col2d(const float*, int, int, int, int, int, int, int, int, int, int, int, float*, cudaStream_t);
int launch_col2im2d(const float*, int, int, int, int, int, int, int, int, int, int, int, float*, cudaStream_t);
int launch_sgemm_simt(bool, bool, int, int, int, float, const float*, int, const float*, int, float, float*, int,
                      cudaStream_t);
int launch_conv_fwd_simt(const ConvShape&, const float*, const float*, const float*, float*, cudaStream_t);
int launch_conv_dgrad_simt(const ConvShape&, const float*, const float*, float*, cudaStream_t);
int launch_conv_wgrad_simt(const ConvShape&, const float*, const float*, float*, cudaStream_t);
int launch_bias_add(int, int, int, const float*, float*, cudaStream_t);
int launch_bias_grad(int, int, int, const float*, float*, cudaStream_t);
// tensor-core family (conv_tc*.cu)
bool tc_conv_supported(const ConvShape&, int op);
size_t tc_conv_workspace(const ConvShape&, int op, int math);
int launch_conv_tc(const ConvShape&, int op, int math, const float* a, const float* b, const float* bias, float* out,
                   void* ws, size_t ws_bytes, const void* prepared, cudaStream_t);
void tc_conv_prep_entry(const ConvShape&, int op, int math, const float* w, void* dst, PrepEntry* q);
void tc_conv_plan_info(const ConvShape&, int op, ConvPlanInfo*);   // the launch's plan; the shape must be tc_conv_supported
bool tc_conv_scatter(const ConvShape&, int op);   // the data gradient of a strided 1x1 layer: rows scattered into a zeroed dx
bool tc_stg_prep_entry(const ConvShape&, int op, const float* w, void* dst, PrepEntry* q);
// bulk-copy-staged bf16x3 kernel (conv_tc_stg.cu): forward / dgrad of stride-1 "same" convolutions
bool tc_stg_supported(const ConvShape&, int op);
size_t tc_stg_workspace(const ConvShape&, int op);
bool tc_stg_plan_info(const ConvShape&, int op, ConvPlanInfo*);     // false: the shape is not staged-eligible
int launch_conv_tc_stg(const ConvShape&, int op, const float* a, const float* w, const float* bias, float* out, void* ws,
                       size_t ws_bytes, const void* prepared, bool accumulate, cudaStream_t);
// gather-family weight gradient (conv_tc_wgrad.cu): the gather kernel, the TMA-fed 1x1 kernel, compaction of strided 1x1 layers
bool tc_wgrad_supported(const ConvShape&);
size_t tc_wgrad_workspace(const ConvShape&);
int launch_conv_tc_wgrad(const ConvShape&, int math, const float* x, const float* dy, float* dw, void* ws, size_t ws_bytes,
                         cudaStream_t);
// weight-gradient route among the gather-family kernels and its plan
int tc_wgrad_route(const ConvShape&, int math, bool x_ok, bool dy_ok, bool ws_ok);
void tc_wgrad_plan_info(const ConvShape&, int route, WgradPlanInfo*);
// TMA-staged bf16x3 weight gradient (conv_tc_wgrad_stg.cu): stride-1 "same" convolutions with 1 or 9 taps
bool tc_wgrad_stg_supported(const ConvShape&);
size_t tc_wgrad_stg_workspace(const ConvShape&);
// split: the buffer for dY's bf16 hi / lo planes where the plan pre-splits it (WgradPlanInfo::split_bytes), or null to convert
// both operands in the kernel
int launch_conv_tc_wgrad_stg(const ConvShape&, const float* x, const float* dy, float* dw, void* ws, size_t ws_bytes, cudaStream_t,
                             void* split = nullptr, size_t split_bytes = 0);
bool tc_wgrad_stg_plan_info(const ConvShape&, WgradPlanInfo*);
// One output phase of a strided transposed convolution along one axis (deconv.cu): the outputs t = t0 + s*m, m < M, are the
// stride-1 correlation of the bottom with n taps of the filter (tap l reads filter tap i0 + (n-1-l)*L), dilation dd, pad `pad`
// (negative where the phase's first output lies beyond the pad).  n == 0: no tap reaches these outputs.
struct DeconvPhaseAxis { int t0, M, n, i0, L, dd, pad; };
// The gather kernel (conv_tc.cu) on phase (a, b) of the transposed convolution whose dual convolution is `dual` (dual input = the
// transposed convolution's top, dual output = its bottom): x = bottom, out = top (only the phase's lattice is written, + bias).
bool tc_deconv_phase_supported(const ConvShape& dual, const DeconvPhaseAxis& a, const DeconvPhaseAxis& b);
size_t tc_deconv_phase_prep_bytes(const ConvShape& dual, const DeconvPhaseAxis& a, const DeconvPhaseAxis& b, int math);
void tc_deconv_phase_prep_entry(const ConvShape& dual, const DeconvPhaseAxis& a, const DeconvPhaseAxis& b, int math, const float* w,
                                void* dst, PrepEntry* q);
void tc_deconv_phase_plan_info(const ConvShape& dual, const DeconvPhaseAxis& a, const DeconvPhaseAxis& b, ConvPlanInfo* q);
int launch_deconv_phase_tc(const ConvShape& dual, const DeconvPhaseAxis& a, const DeconvPhaseAxis& b, int math, const float* x,
                           const float* bias, float* out, const PrepEntry& q, cudaStream_t st);
bool tc_gemm_supported(bool tA, bool tB, int M, int N, int K);
size_t tc_gemm_workspace(bool tA, bool tB, int M, int N, int K);
// The kernel b2c_sgemm_ex runs and its plan, decided in one place (sgemm_route) for the launch and for b2c_debug_sgemm_plan.
// tc: the staged 1x1 kernel (wgrad_stg_kernel<1, cols>) on 128 x cols tiles, bpi K blocks of 64, split over `splits` CTAs of
// kb_per_split blocks each; else the FFMA kernel (sgemm_simt_kernel) on 64 x 64 tiles, bpi = kb_per_split = K steps of 16.
struct GemmPlan {
  bool tc;
  int cols, bpi, splits, kb_per_split, m_tiles, n_tiles;
};
// tc_allowed: the default algo and math let the tensor cores run (not SIMT, fp32 math).  Pointers are only tested for alignment.
void sgemm_route(bool tc_allowed, bool tA, bool tB, int M, int N, int K, float alpha, float beta, const void* A, const void* B,
                 const void* ws, size_t ws_bytes, GemmPlan* g);
int launch_sgemm_tc(const GemmPlan& g, int M, int N, int K, const float* A, const float* B, float beta, float* C, void* ws,
                    size_t ws_bytes, cudaStream_t);

}  // namespace b2c

struct b2c_conv_desc {
  b2c::ConvShape s;
  int engine;
  int math;
  int algo;
  const void* filter_cache;   // b2c_conv_desc_bind_filter_cache: prepared forward / dgrad filters, or null
};
