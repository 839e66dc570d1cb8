// b2c_common.cuh -- shared helpers for the sm_90a kernels behind include/b2c.h.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include <string>

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
};

}  // namespace b2c

struct b2c_conv_desc {
  b2c::ConvShape s;
  int engine;
  int math;
  int algo;
  const void* filter_cache;   // b2c_conv_desc_bind_filter_cache: prepared forward / dgrad filters, or null
};
