// api.cu -- C-ABI glue: error plumbing, convolution descriptors and engine/algo dispatch.
//
// The dispatch mirrors GetConvolutionLayer (reference src/caffe/layer_factory.cpp:53-88):
//   engine CAFFE          -> explicit per-image im2col + GEMM + bias, the literal structure of
//                            ConvolutionLayer::Forward_gpu/Backward_gpu (conv_layer.cu:7-57).
//   engine DEFAULT/CUDNN  -> whole-batch implicit GEMM (the cuDNN role): wgmma tensor-core kernels
//                            (conv_tc.cu) when the shape qualifies, else the SIMT direct kernels.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "b2c_common.cuh"
#include "filter_prep.cuh"

namespace b2c {

std::string& last_error() {
  thread_local std::string e;
  return e;
}
std::atomic<uint64_t> g_launches{0};

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  last_error() = buf;
  return code;
}

int sm_count() {
  // cached per device (a process may drive several GPUs, like the reference's solver threads)
  static int cache[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (!cache[dev]) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cache[dev] = n;
  }
  return cache[dev];
}

static std::atomic<int> g_default_math{B2C_MATH_FP32};
static std::atomic<int> g_default_algo{B2C_ALGO_AUTO};

static bool have_device() {
  static int ok = -1;
  if (ok < 0) {
    int n = 0;
    ok = (cudaGetDeviceCount(&n) == cudaSuccess && n > 0) ? 1 : 0;
  }
  return ok == 1;
}

// the staged kernels run bf16x3 math: only in the fp32 math mode of the implicit engine, and not where the FFMA kernels are asked for
static bool staged_allowed(const b2c_conv_desc* d) {
  return d->engine != B2C_ENGINE_CAFFE && d->algo != B2C_ALGO_SIMT && d->math == B2C_MATH_FP32;
}
static bool use_staged(const b2c_conv_desc* d, int op) {
  if (!staged_allowed(d)) return false;
  return op == B2C_OP_BACKWARD_FILTER ? tc_wgrad_stg_supported(d->s) : tc_stg_supported(d->s, op);
}
// math mode handed to the gather kernels (conv_tc.cu / conv_tc_wgrad.cu), which know FP32 (= 3xTF32) and TF32
static int gather_math(const b2c_conv_desc* d) { return d->math == B2C_MATH_TF32 ? B2C_MATH_TF32 : B2C_MATH_FP32; }

// The kernel b2c_conv_backward_filter runs (b2c_wgrad_route), decided in one place for the launch and for b2c_debug_wgrad_plan.
// x_ok / dy_ok / ws_ok: those pointers are 16-byte aligned (the staged and TMA-fed kernels need it; otherwise the gather kernel).
static int wgrad_route(const b2c_conv_desc* d, bool x_ok, bool dy_ok, bool ws_ok) {
  if (d->engine == B2C_ENGINE_CAFFE) return B2C_WGRAD_ROUTE_CAFFE;
  if (use_staged(d, B2C_OP_BACKWARD_FILTER) && x_ok && dy_ok) {
    WgradPlanInfo q{};
    tc_wgrad_stg_plan_info(d->s, &q);
    if (q.taps == 9) return q.plane ? B2C_WGRAD_ROUTE_STAGED_3X3_PLANE : B2C_WGRAD_ROUTE_STAGED_3X3;
    return q.plane ? B2C_WGRAD_ROUTE_STAGED_1X1_PLANE : B2C_WGRAD_ROUTE_STAGED_1X1;
  }
  if (tc_conv_supported(d->s, B2C_OP_BACKWARD_FILTER) && d->algo != B2C_ALGO_SIMT)
    return tc_wgrad_route(d->s, gather_math(d), x_ok, dy_ok, ws_ok);
  return B2C_WGRAD_ROUTE_SIMT;
}

// The kernel b2c_conv_forward (op B2C_OP_FORWARD) or b2c_conv_backward_data (B2C_OP_BACKWARD_DATA) runs (b2c_conv_route), decided
// in one place for the launches, the workspace and filter-cache sizes and b2c_debug_conv_plan.  aligned: the activation operands
// (x and y, or dy and dx) are 16-byte aligned, which the staged kernel needs; otherwise the gather kernel.
static int conv_route(const b2c_conv_desc* d, int op, bool aligned) {
  if (d->engine == B2C_ENGINE_CAFFE) return B2C_CONV_ROUTE_CAFFE;
  ConvPlanInfo q;
  if (aligned && staged_allowed(d) && tc_stg_plan_info(d->s, op, &q))
    return q.variant < 128 ? B2C_CONV_ROUTE_STAGED_PLANE : B2C_CONV_ROUTE_STAGED;
  if (tc_conv_supported(d->s, op) && d->algo != B2C_ALGO_SIMT)
    return tc_conv_scatter(d->s, op) ? B2C_CONV_ROUTE_GATHER_SCATTER : B2C_CONV_ROUTE_GATHER;
  return B2C_CONV_ROUTE_SIMT;
}
static bool staged_route(int route) { return route == B2C_CONV_ROUTE_STAGED || route == B2C_CONV_ROUTE_STAGED_PLANE; }
static bool gather_route(int route) { return route == B2C_CONV_ROUTE_GATHER || route == B2C_CONV_ROUTE_GATHER_SCATTER; }

// ---- prepared-filter cache: [forward layout | dgrad layout], each region 256-byte aligned -------------------------------
// (the layout of the route for aligned operands: a call with unaligned ones runs its own prepass)
static size_t cache_region_bytes(const b2c_conv_desc* d, int op) {
  const int route = conv_route(d, op, true);
  size_t n = 0;
  if (staged_route(route)) n = tc_stg_workspace(d->s, op);
  else if (gather_route(route)) n = tc_conv_workspace(d->s, op, gather_math(d));
  return (n + 255) & ~(size_t)255;
}
static const void* prepared_filter(const b2c_conv_desc* d, int op) {
  if (!d->filter_cache) return nullptr;
  const char* base = static_cast<const char*>(d->filter_cache);
  return op == B2C_OP_FORWARD ? base : base + cache_region_bytes(d, B2C_OP_FORWARD);
}
// the prepared filter for a gather-kernel launch: none where the cache holds the staged kernel's layout
static const void* cached_gather_filter(const b2c_conv_desc* d, int op) {
  return staged_route(conv_route(d, op, true)) ? nullptr : prepared_filter(d, op);
}
static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// A layer of the implicit engine that no tensor-core kernel takes (K = C/g*kh*kw beyond the filter tile limit, a strided k > 1 data
// gradient, ...) runs on the FFMA kernels: correct, an order of magnitude slower.  Say so instead of doing it silently -- the
// first few times per process, on stderr; b2c_conv_algo_used() is the programmatic form.  B2C_QUIET=1 turns the notes off.
static void note_simt_fallback(const b2c_conv_desc* d, int op) {
  if (d->algo == B2C_ALGO_SIMT) return;                       // the caller asked for these kernels
  static std::atomic<int> notes{0};
  static const bool quiet = [] { const char* e = getenv("B2C_QUIET"); return e && *e && *e != '0'; }();
  if (quiet || notes.fetch_add(1) >= 4) return;
  const ConvShape& s = d->s;
  static const char* const names[] = {"forward", "data gradient", "weight gradient"};   // b2c_conv_op order
  fprintf(stderr, "b2c: note: convolution C=%d %dx%d -> O=%d k=%dx%d s=%dx%d p=%dx%d g=%d, %s: no tensor-core kernel takes this shape, "
                  "using the FFMA kernels\n", s.C, s.H, s.W, s.O, s.kh, s.kw, s.sh, s.sw, s.ph, s.pw, s.G,
          op >= 0 && op < 3 ? names[op] : "?");
}

static int resolve_algo(const b2c_conv_desc* d, int op) {
  if (d->engine == B2C_ENGINE_CAFFE) return B2C_ALGO_SIMT;  // reported family of the explicit path's GEMM
  if (op != B2C_OP_BACKWARD_FILTER) return conv_route(d, op, true) == B2C_CONV_ROUTE_SIMT ? B2C_ALGO_SIMT : B2C_ALGO_TCGEN05;
  if (d->algo == B2C_ALGO_SIMT) return B2C_ALGO_SIMT;
  if (use_staged(d, op)) return B2C_ALGO_TCGEN05;
  return tc_conv_supported(d->s, op) ? B2C_ALGO_TCGEN05 : B2C_ALGO_SIMT;
}

}  // namespace b2c

using namespace b2c;

extern "C" const char* b2c_last_error(void) { return last_error().c_str(); }
extern "C" const char* b2c_version(void) { return "b2c 0.1 (sm_90a)"; }
extern "C" uint64_t b2c_launch_count(void) { return g_launches.load(); }
extern "C" int b2c_set_default_math(int m) {
  if (m < B2C_MATH_FP32 || m > B2C_MATH_FP32_3XTF32) return fail(B2C_ERR_INVALID, "bad math mode %d", m);
  g_default_math = m;
  return B2C_OK;
}
extern "C" int b2c_set_default_algo(int a) {
  if (a < B2C_ALGO_AUTO || a > B2C_ALGO_TCGEN05) return fail(B2C_ERR_INVALID, "bad algo %d", a);
  g_default_algo = a;
  return B2C_OK;
}

extern "C" int b2c_conv_desc_create(const b2c_conv_params* p, int engine, b2c_conv_desc** out) {
  if (!p || !out) return fail(B2C_ERR_INVALID, "b2c_conv_desc_create: null");
  if (engine < B2C_ENGINE_DEFAULT || engine > B2C_ENGINE_CUDNN) return fail(B2C_ERR_INVALID, "bad engine %d", engine);
  // the CHECKs of BaseConvolutionLayer::LayerSetUp (base_conv_layer.cpp:44-118)
  if (p->N <= 0 || p->C <= 0 || p->H <= 0 || p->W <= 0 || p->O <= 0)
    return fail(B2C_ERR_INVALID, "conv: non-positive blob dimension");
  if (p->kh <= 0 || p->kw <= 0) return fail(B2C_ERR_INVALID, "conv: Filter dimensions must be nonzero");
  if (p->sh <= 0 || p->sw <= 0) return fail(B2C_ERR_INVALID, "conv: Stride dimensions must be nonzero");
  if (p->dh <= 0 || p->dw <= 0) return fail(B2C_ERR_INVALID, "conv: dilation must be positive");
  if (p->ph < 0 || p->pw < 0) return fail(B2C_ERR_INVALID, "conv: negative pad");
  if (p->G <= 0 || p->C % p->G) return fail(B2C_ERR_INVALID, "conv: channels %d not divisible by group %d", p->C, p->G);
  if (p->O % p->G) return fail(B2C_ERR_INVALID, "conv: Number of output should be multiples of group");
  b2c_conv_desc* d = new b2c_conv_desc;
  ConvShape& s = d->s;
  s.N = p->N; s.C = p->C; s.H = p->H; s.W = p->W; s.O = p->O; s.G = p->G;
  s.kh = p->kh; s.kw = p->kw; s.sh = p->sh; s.sw = p->sw; s.ph = p->ph; s.pw = p->pw; s.dh = p->dh; s.dw = p->dw;
  s.has_bias = p->has_bias;
  s.Ho = (s.H + 2 * s.ph - (s.dh * (s.kh - 1) + 1)) / s.sh + 1;   // conv_layer.cpp:14-21
  s.Wo = (s.W + 2 * s.pw - (s.dw * (s.kw - 1) + 1)) / s.sw + 1;
  if (s.Ho <= 0 || s.Wo <= 0) { delete d; return fail(B2C_ERR_INVALID, "conv: kernel larger than padded input"); }
  s.Cg = s.C / s.G; s.Og = s.O / s.G; s.Kd = s.Cg * s.kh * s.kw;
  s.is_1x1 = s.kh == 1 && s.kw == 1 && s.sh == 1 && s.sw == 1 && s.ph == 0 && s.pw == 0;
  d->engine = engine;
  d->math = g_default_math;
  d->algo = g_default_algo;
  d->filter_cache = nullptr;
  *out = d;
  return B2C_OK;
}
extern "C" int b2c_conv_desc_destroy(b2c_conv_desc* d) { delete d; return B2C_OK; }
extern "C" int b2c_conv_desc_set_math(b2c_conv_desc* d, int m) {
  if (!d || m < B2C_MATH_FP32 || m > B2C_MATH_FP32_3XTF32) return fail(B2C_ERR_INVALID, "set_math: bad argument");
  d->math = m;
  return B2C_OK;
}
extern "C" int b2c_conv_desc_set_algo(b2c_conv_desc* d, int a) {
  if (!d || a < B2C_ALGO_AUTO || a > B2C_ALGO_TCGEN05) return fail(B2C_ERR_INVALID, "set_algo: bad argument");
  d->algo = a;
  return B2C_OK;
}
extern "C" int b2c_conv_out_shape(const b2c_conv_desc* d, int* Ho, int* Wo) {
  if (!d) return fail(B2C_ERR_INVALID, "null desc");
  if (Ho) *Ho = d->s.Ho;
  if (Wo) *Wo = d->s.Wo;
  return B2C_OK;
}
extern "C" int b2c_conv_algo_used(const b2c_conv_desc* d, int op) {
  if (!d) return B2C_ERR_INVALID;
  return resolve_algo(d, op);
}

extern "C" size_t b2c_conv_workspace_bytes(const b2c_conv_desc* d, int op) {
  if (!d) return 0;
  const ConvShape& s = d->s;
  if (d->engine == B2C_ENGINE_CAFFE)   // one image's col buffer [Kd*G, Ho, Wo] (base_conv_layer.cpp:225-233)
    return s.is_1x1 ? 0 : sizeof(float) * (size_t)s.Kd * s.G * s.Ho * s.Wo;
  if (op != B2C_OP_BACKWARD_FILTER) {
    const int route = conv_route(d, op, true);
    if (!staged_route(route)) return gather_route(route) ? tc_conv_workspace(s, op, gather_math(d)) : 0;
    // the gather kernel is the fallback for unaligned activation pointers: size for both
    const size_t a = tc_stg_workspace(s, op);
    const size_t b = gather_route(conv_route(d, op, false)) ? tc_conv_workspace(s, op, gather_math(d)) : 0;
    return a > b ? a : b;
  }
  if (use_staged(d, op)) {   // as above, for the staged weight-gradient kernel
    const size_t a = tc_wgrad_stg_workspace(s);
    const size_t b = tc_conv_supported(s, op) ? tc_conv_workspace(s, op, gather_math(d)) : 0;
    return a > b ? a : b;
  }
  if (resolve_algo(d, op) == B2C_ALGO_TCGEN05) return tc_conv_workspace(s, op, gather_math(d));
  return 0;
}

#define REQUIRE_DEVICE() \
  if (!have_device()) return fail(B2C_ERR_CUDA, "no CUDA device: this library has no CPU fallback")

extern "C" int b2c_conv_forward(const b2c_conv_desc* d, const float* x, const float* w, const float* bias, float* y,
                                void* ws, size_t ws_bytes, void* stream) {
  if (!d || !x || !w || !y) return fail(B2C_ERR_INVALID, "b2c_conv_forward: null pointer");
  REQUIRE_DEVICE();
  const ConvShape& s = d->s;
  if (s.has_bias && !bias) return fail(B2C_ERR_INVALID, "b2c_conv_forward: bias_term set but bias is null");
  if (!s.has_bias) bias = nullptr;
  cudaStream_t st = as_stream(stream);
  const size_t need = b2c_conv_workspace_bytes(d, B2C_OP_FORWARD);
  if (ws_bytes < need || (need && !ws)) return fail(B2C_ERR_WORKSPACE, "forward workspace too small");
  if (d->engine == B2C_ENGINE_CAFFE) {
    const int P = s.Ho * s.Wo;
    const size_t bdim = (size_t)s.C * s.H * s.W, tdim = (size_t)s.O * P;
    float* col = static_cast<float*>(ws);
    for (int n = 0; n < s.N; ++n) {
      const float* cb = x + n * bdim;
      if (!s.is_1x1) {
        if (int rc = launch_im2col2d(x + n * bdim, s.C, s.H, s.W, s.kh, s.kw, s.ph, s.pw, s.sh, s.sw, s.dh, s.dw, col, st)) return rc;
        cb = col;
      }
      for (int g = 0; g < s.G; ++g)
        if (int rc = b2c_sgemm(0, 0, s.Og, P, s.Kd, 1.0f, w + (size_t)g * s.Og * s.Kd, cb + (size_t)g * s.Kd * P, 0.0f,
                               y + n * tdim + (size_t)g * s.Og * P, stream)) return rc;
    }
    if (bias) return launch_bias_add(s.N, s.O, P, bias, y, st);
    return B2C_OK;
  }
  const int route = conv_route(d, B2C_OP_FORWARD, aligned16(x) && aligned16(y));
  if (staged_route(route))
    return launch_conv_tc_stg(s, B2C_OP_FORWARD, x, w, bias, y, ws, ws_bytes, prepared_filter(d, B2C_OP_FORWARD), false, st);
  // a staged layer that falls back here (unaligned activation pointers) has the staged kernel's bf16 layout in its cache: of no use
  if (gather_route(route))
    return launch_conv_tc(s, B2C_OP_FORWARD, gather_math(d), x, w, bias, y, ws, ws_bytes, cached_gather_filter(d, B2C_OP_FORWARD), st);
  note_simt_fallback(d, B2C_OP_FORWARD);
  return launch_conv_fwd_simt(s, x, w, bias, y, st);
}

extern "C" int b2c_conv_backward_data(const b2c_conv_desc* d, const float* dy, const float* w, float* dx, void* ws,
                                      size_t ws_bytes, void* stream) {
  if (!d || !dy || !w || !dx) return fail(B2C_ERR_INVALID, "b2c_conv_backward_data: null pointer");
  REQUIRE_DEVICE();
  const ConvShape& s = d->s;
  cudaStream_t st = as_stream(stream);
  const size_t need = b2c_conv_workspace_bytes(d, B2C_OP_BACKWARD_DATA);
  if (ws_bytes < need || (need && !ws)) return fail(B2C_ERR_WORKSPACE, "backward_data workspace too small");
  if (d->engine == B2C_ENGINE_CAFFE) {
    const int P = s.Ho * s.Wo;
    const size_t bdim = (size_t)s.C * s.H * s.W, tdim = (size_t)s.O * P;
    float* col = static_cast<float*>(ws);
    for (int n = 0; n < s.N; ++n) {
      float* cb = s.is_1x1 ? dx + n * bdim : col;
      for (int g = 0; g < s.G; ++g)
        if (int rc = b2c_sgemm(1, 0, s.Kd, P, s.Og, 1.0f, w + (size_t)g * s.Og * s.Kd, dy + n * tdim + (size_t)g * s.Og * P,
                               0.0f, cb + (size_t)g * s.Kd * P, stream)) return rc;
      if (!s.is_1x1)
        if (int rc = launch_col2im2d(col, s.C, s.H, s.W, s.kh, s.kw, s.ph, s.pw, s.sh, s.sw, s.dh, s.dw, dx + n * bdim, st)) return rc;
    }
    return B2C_OK;
  }
  const int route = conv_route(d, B2C_OP_BACKWARD_DATA, aligned16(dy) && aligned16(dx));
  if (staged_route(route))
    return launch_conv_tc_stg(s, B2C_OP_BACKWARD_DATA, dy, w, nullptr, dx, ws, ws_bytes, prepared_filter(d, B2C_OP_BACKWARD_DATA), false, st);
  if (gather_route(route))
    return launch_conv_tc(s, B2C_OP_BACKWARD_DATA, gather_math(d), dy, w, nullptr, dx, ws, ws_bytes,
                          cached_gather_filter(d, B2C_OP_BACKWARD_DATA), st);
  note_simt_fallback(d, B2C_OP_BACKWARD_DATA);
  return launch_conv_dgrad_simt(s, dy, w, dx, st);
}

// dx += dgrad(dy, w): the accumulation Net::Backward performs where a blob fans out (SplitLayer::Backward in the reference),
// folded into the kernel's TMA reduce-add store.  Only the staged kernel has it; the caller asks first.
extern "C" int b2c_conv_backward_data_accumulate_supported(const b2c_conv_desc* d) {
  return d && staged_route(conv_route(d, B2C_OP_BACKWARD_DATA, true)) ? 1 : 0;
}
extern "C" int b2c_conv_backward_data_accumulate(const b2c_conv_desc* d, const float* dy, const float* w, float* dx, void* ws,
                                                 size_t ws_bytes, void* stream) {
  if (!d || !dy || !w || !dx) return fail(B2C_ERR_INVALID, "b2c_conv_backward_data_accumulate: null pointer");
  REQUIRE_DEVICE();
  if (!staged_route(conv_route(d, B2C_OP_BACKWARD_DATA, aligned16(dy) && aligned16(dx))))
    return fail(B2C_ERR_INVALID, "b2c_conv_backward_data_accumulate: not available for this layer (see ..._accumulate_supported)");
  const size_t need = b2c_conv_workspace_bytes(d, B2C_OP_BACKWARD_DATA);
  if (!prepared_filter(d, B2C_OP_BACKWARD_DATA) && (ws_bytes < need || (need && !ws))) return fail(B2C_ERR_WORKSPACE, "backward_data workspace too small");
  return launch_conv_tc_stg(d->s, B2C_OP_BACKWARD_DATA, dy, w, nullptr, dx, ws, ws_bytes, prepared_filter(d, B2C_OP_BACKWARD_DATA), true,
                            as_stream(stream));
}

extern "C" size_t b2c_conv_wgrad_split_bytes(const b2c_conv_desc* d) {
  if (!d) return 0;
  const int route = wgrad_route(d, true, true, true);
  WgradPlanInfo q;
  tc_wgrad_plan_info(d->s, route, &q);
  return q.split_bytes;
}

extern "C" int b2c_conv_backward_filter_split(const b2c_conv_desc* d, const float* x, const float* dy, float* dw, void* ws,
                                              size_t ws_bytes, void* split, size_t split_bytes, void* stream) {
  if (!d || !x || !dy || !dw) return fail(B2C_ERR_INVALID, "b2c_conv_backward_filter: null pointer");
  REQUIRE_DEVICE();
  const ConvShape& s = d->s;
  cudaStream_t st = as_stream(stream);
  const size_t need = b2c_conv_workspace_bytes(d, B2C_OP_BACKWARD_FILTER);
  if (ws_bytes < need || (need && !ws)) return fail(B2C_ERR_WORKSPACE, "backward_filter workspace too small");
  auto aligned = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
  const int route = wgrad_route(d, aligned(x), aligned(dy), ws && aligned(ws));
  if (route == B2C_WGRAD_ROUTE_CAFFE) {
    const int P = s.Ho * s.Wo;
    const size_t bdim = (size_t)s.C * s.H * s.W, tdim = (size_t)s.O * P;
    float* col = static_cast<float*>(ws);
    for (int n = 0; n < s.N; ++n) {
      const float* cb = x + n * bdim;
      if (!s.is_1x1) {
        if (int rc = launch_im2col2d(x + n * bdim, s.C, s.H, s.W, s.kh, s.kw, s.ph, s.pw, s.sh, s.sw, s.dh, s.dw, col, st)) return rc;
        cb = col;
      }
      for (int g = 0; g < s.G; ++g)
        if (int rc = b2c_sgemm(0, 1, s.Og, s.Kd, P, 1.0f, dy + n * tdim + (size_t)g * s.Og * P, cb + (size_t)g * s.Kd * P,
                               1.0f, dw + (size_t)g * s.Og * s.Kd, stream)) return rc;
    }
    return B2C_OK;
  }
  if (route >= B2C_WGRAD_ROUTE_STAGED_3X3 && route <= B2C_WGRAD_ROUTE_STAGED_1X1_PLANE)
    return launch_conv_tc_wgrad_stg(s, x, dy, dw, ws, ws_bytes, st, split, split_bytes);
  if (route != B2C_WGRAD_ROUTE_SIMT)   // the gather kernel or the TMA-fed 1x1 kernel, with or without compaction (conv_tc_wgrad.cu)
    return launch_conv_tc(s, B2C_OP_BACKWARD_FILTER, gather_math(d), x, dy, nullptr, dw, ws, ws_bytes, nullptr, st);
  note_simt_fallback(d, B2C_OP_BACKWARD_FILTER);
  return launch_conv_wgrad_simt(s, x, dy, dw, st);
}

extern "C" int b2c_conv_backward_filter(const b2c_conv_desc* d, const float* x, const float* dy, float* dw, void* ws,
                                        size_t ws_bytes, void* stream) {
  return b2c_conv_backward_filter_split(d, x, dy, dw, ws, ws_bytes, nullptr, 0, stream);
}

extern "C" int b2c_debug_wgrad_plan(const b2c_conv_desc* d, int* out, int n) {
  if (!d || !out || n < 6) return fail(B2C_ERR_INVALID, "b2c_debug_wgrad_plan: need a descriptor and 6 ints");
  const int route = wgrad_route(d, true, true, true);
  WgradPlanInfo q;
  tc_wgrad_plan_info(d->s, route, &q);
  out[0] = route; out[1] = q.splits; out[2] = q.kb_per_split; out[3] = (int)q.nkb; out[4] = q.cols; out[5] = q.bpi;
  if (n >= 7) out[6] = q.presplit;
  return B2C_OK;
}

extern "C" int b2c_debug_conv_plan(const b2c_conv_desc* d, int op, int* out, int n) {
  if (!d || !out || n < 8) return fail(B2C_ERR_INVALID, "b2c_debug_conv_plan: need a descriptor and 8 ints");
  if (op != B2C_OP_FORWARD && op != B2C_OP_BACKWARD_DATA) return fail(B2C_ERR_INVALID, "b2c_debug_conv_plan: op %d is not forward or backward data", op);
  const int route = conv_route(d, op, true);
  ConvPlanInfo q{};
  if (staged_route(route)) tc_stg_plan_info(d->s, op, &q);
  else if (gather_route(route)) tc_conv_plan_info(d->s, op, &q);
  out[0] = route; out[1] = q.n_tile; out[2] = q.m_tiles; out[3] = q.n_tiles; out[4] = q.tiles; out[5] = persistent_grid(q.tiles);
  out[6] = q.nkb; out[7] = q.variant;
  return B2C_OK;
}

namespace b2c {
int debug_mbar_fwd(unsigned int*, int, int);
int debug_mbar_stg(unsigned int*, int, int);
int debug_mbar_wgrad(unsigned int*, int, int);
int debug_mbar_wstg(unsigned int*, int, int);
}
// out: four consecutive blocks of 128 words (gather fwd/dgrad kernel, staged fwd/dgrad kernel, gather weight-gradient kernels,
// staged weight-gradient kernel)
extern "C" int b2c_debug_mbar_timeouts(unsigned int* out, int cap_words) {
  REQUIRE_DEVICE();
  if (!out || cap_words < 512) return fail(B2C_ERR_INVALID, "b2c_debug_mbar_timeouts: need 512 words");
  const int a = debug_mbar_fwd(out, 128, -1), b = debug_mbar_stg(out + 128, 128, -1), c = debug_mbar_wgrad(out + 256, 128, -1),
            e = debug_mbar_wstg(out + 384, 128, -1);
  return (a < 0 || b < 0 || c < 0 || e < 0) ? -1 : a + b + c + e;
}
extern "C" int b2c_debug_mbar_set_trap(int on) {
  REQUIRE_DEVICE();
  debug_mbar_fwd(nullptr, 0, on != 0); debug_mbar_stg(nullptr, 0, on != 0); debug_mbar_wgrad(nullptr, 0, on != 0); debug_mbar_wstg(nullptr, 0, on != 0);
  return B2C_OK;
}

extern "C" size_t b2c_conv_filter_cache_bytes(const b2c_conv_desc* d) {
  if (!d) return 0;
  return cache_region_bytes(d, B2C_OP_FORWARD) + cache_region_bytes(d, B2C_OP_BACKWARD_DATA);
}
extern "C" int b2c_conv_desc_bind_filter_cache(b2c_conv_desc* d, const void* cache) {
  if (!d) return fail(B2C_ERR_INVALID, "bind_filter_cache: null descriptor");
  if (cache && (reinterpret_cast<uintptr_t>(cache) & 255u)) return fail(B2C_ERR_INVALID, "bind_filter_cache: the cache must be 256-byte aligned");
  d->filter_cache = cache;
  return B2C_OK;
}
static int collect_prep_entries(const b2c_conv_desc* d, const float* w, void* cache, PrepEntry* out) {
  int n = 0;
  char* base = static_cast<char*>(cache);
  for (int op = B2C_OP_FORWARD; op <= B2C_OP_BACKWARD_DATA; ++op) {
    const size_t bytes = cache_region_bytes(d, op);
    if (!bytes) continue;
    void* dst = op == B2C_OP_FORWARD ? base : base + cache_region_bytes(d, B2C_OP_FORWARD);
    if (staged_route(conv_route(d, op, true))) tc_stg_prep_entry(d->s, op, w, dst, &out[n++]);
    else tc_conv_prep_entry(d->s, op, gather_math(d), w, dst, &out[n++]);
  }
  return n;
}
extern "C" int b2c_conv_prepare_filters(int n, const b2c_conv_desc* const* descs, const float* const* ws, void* const* caches,
                                        void* stream) {
  if (n < 0 || (n && (!descs || !ws || !caches))) return fail(B2C_ERR_INVALID, "b2c_conv_prepare_filters: bad argument");
  REQUIRE_DEVICE();
  std::vector<PrepEntry> entries;
  entries.reserve(2 * (size_t)n);
  for (int i = 0; i < n; ++i) {
    if (!descs[i] || !ws[i]) return fail(B2C_ERR_INVALID, "b2c_conv_prepare_filters: null entry %d", i);
    if (!b2c_conv_filter_cache_bytes(descs[i])) continue;
    if (!caches[i] || (reinterpret_cast<uintptr_t>(caches[i]) & 255u)) return fail(B2C_ERR_INVALID, "b2c_conv_prepare_filters: cache %d null or not 256-byte aligned", i);
    PrepEntry e[2];
    const int m = collect_prep_entries(descs[i], ws[i], caches[i], e);
    for (int k = 0; k < m; ++k) entries.push_back(e[k]);
  }
  if (entries.empty()) return B2C_OK;
  return launch_filter_prep(entries.data(), (int)entries.size(), as_stream(stream));
}
extern "C" int b2c_conv_prepare_filter(const b2c_conv_desc* d, const float* w, void* cache, size_t cache_bytes, void* stream) {
  if (!d || !w) return fail(B2C_ERR_INVALID, "b2c_conv_prepare_filter: null pointer");
  if (cache_bytes < b2c_conv_filter_cache_bytes(d)) return fail(B2C_ERR_WORKSPACE, "b2c_conv_prepare_filter: cache too small");
  return b2c_conv_prepare_filters(1, &d, &w, &cache, stream);
}

extern "C" int b2c_conv_backward_bias(const b2c_conv_desc* d, const float* dy, float* db, void* stream) {
  if (!d || !dy || !db) return fail(B2C_ERR_INVALID, "b2c_conv_backward_bias: null pointer");
  REQUIRE_DEVICE();
  return launch_bias_grad(d->s.N, d->s.O, d->s.Ho * d->s.Wo, dy, db, as_stream(stream));
}

extern "C" int b2c_sgemm_tc_supported(int transA, int transB, int M, int N, int K) {
  return M > 0 && N > 0 && K > 0 && have_device() && g_default_algo != B2C_ALGO_SIMT && g_default_math == B2C_MATH_FP32 &&
         tc_gemm_supported(transA != 0, transB != 0, M, N, K) ? 1 : 0;
}
extern "C" size_t b2c_sgemm_workspace_bytes(int transA, int transB, int M, int N, int K) {
  if (M <= 0 || N <= 0 || K <= 0 || !have_device()) return 0;
  return tc_gemm_workspace(transA != 0, transB != 0, M, N, K);
}
extern "C" int b2c_sgemm(int transA, int transB, int M, int N, int K, float alpha, const float* A, const float* B,
                         float beta, float* C, void* stream) {
  return b2c_sgemm_ex(transA, transB, M, N, K, alpha, A, B, beta, C, nullptr, 0, stream);
}
extern "C" int b2c_sgemm_ex(int transA, int transB, int M, int N, int K, float alpha, const float* A, const float* B,
                            float beta, float* C, void* workspace, size_t workspace_bytes, void* stream) {
  if (!A || !B || !C || M < 0 || N < 0 || K < 0) return fail(B2C_ERR_INVALID, "b2c_sgemm: bad argument");
  REQUIRE_DEVICE();
  if (M == 0 || N == 0) return B2C_OK;
  const bool tA = transA != 0, tB = transB != 0;
  // NoTrans x Trans products (InnerProduct forward) on the tensor cores, fp32-equivalent bf16x3 math; everything else -- and any
  // alpha / beta / alignment the staged kernel does not take -- on the exact-fp32 FFMA kernel
  if (g_default_algo != B2C_ALGO_SIMT && g_default_math == B2C_MATH_FP32 && alpha == 1.0f && (beta == 0.0f || beta == 1.0f) &&
      ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B)) & 15u) == 0 && tc_gemm_supported(tA, tB, M, N, K))
    return launch_sgemm_tc(tA, tB, M, N, K, alpha, A, B, beta, C, g_default_math, workspace, workspace_bytes, as_stream(stream));
  return launch_sgemm_simt(tA, tB, M, N, K, alpha, A, tA ? M : K, B, tB ? K : N, beta, C, N, as_stream(stream));
}
