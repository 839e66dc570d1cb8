// deconv.cu -- transposed convolution (DeconvolutionLayer, deconv_layer.cpp / .cu) and Crop (crop_layer.cpp / .cu), sm_90a.
//
// A transposed convolution is the data gradient of its dual convolution: the dual's input is the deconvolution's top
// (Ht = sh*(Hb-1) + dh*(kh-1) + 1 - 2*ph, deconv_layer.cpp:7-22), its output the bottom, its filter [C_in, num_output/G, kh, kw]
// -- exactly the deconvolution's weight blob.  Forward is the dual's data gradient, backward data the dual's forward, the weight
// gradient the dual's with X = top diff and dY = bottom data (deconv_layer.cu Backward_gpu: weight_gpu_gemm(top_diff, bottom_data)).
// Routes (b2c_deconv_route):
//   DUAL       the dual convolution's own routes (CAFFE engine, stride 1, strided 1x1 pad 0, and every backward op).
//   PHASE      forward of a strided layer with k > 1: the sub-pixel decomposition.  Along an axis, output t takes taps i with
//              i*d == (t + p) (mod s).  For the outputs t = t0 + s*m of one residue the taps are consecutive members of a
//              progression with step L = s / gcd(s, d), and the outputs form a stride-1 correlation of the bottom with the flipped
//              sub-filter, dilation d / gcd(s, d) (DeconvPhaseAxis).  Each of the sh*sw phases is one gather-kernel launch
//              (conv_tc.cu) writing its lattice of the top through the epilogue's row / column strides, bias fused.  A phase
//              that no tap reaches (k < s, or a residue the dilation never hits) holds only the bias, or 0.
//   DEPTHWISE  group == C_in == num_output (the bilinear upsampler of filler.hpp's BilinearFiller): direct fp32 kernels below.
#include <algorithm>
#include <vector>
#include "b2c_common.cuh"
#include "filter_prep.cuh"

namespace b2c {
struct Phase { DeconvPhaseAxis a, b; };
}

struct b2c_deconv_desc {
  b2c_conv_desc* dual;   // owned
  int N, C, H, W, O, G, has_bias;   // the layer's view: bottom [N, C, H, W], num_output O
  std::vector<b2c::Phase> phases;   // the sh*sw output phases, computed once at creation
};

namespace b2c {

// ---- phase geometry -----------------------------------------------------------------------------------------------------
static int gcd_int(int a, int b) { while (b) { const int t = a % b; a = b; b = t; } return a; }
// outputs t0, t0 + s, ... < T of a transposed convolution with kernel k, stride s, pad p, dilation d along one axis
static DeconvPhaseAxis phase_axis(int t0, int T, int k, int s, int p, int d) {
  DeconvPhaseAxis a{};
  const int g = gcd_int(s, d);
  a.t0 = t0;
  a.M = t0 < T ? (T - t0 + s - 1) / s : 0;
  a.L = s / g; a.dd = d / g;
  const int r = (t0 + p) % s;
  for (int i = 0; i < k && i < a.L; ++i)
    if ((long long)i * d % s == r) { a.i0 = i; a.n = (k - 1 - i) / a.L + 1; break; }
  if (a.n) {
    const int q0 = (int)(((long long)a.i0 * d - r) / s);
    a.pad = q0 + (a.n - 1) * a.dd - (t0 + p - r) / s;
  }
  return a;
}
static std::vector<Phase> phases(const ConvShape& s) {
  std::vector<Phase> v;
  for (int th = 0; th < s.sh; ++th)
    for (int tw = 0; tw < s.sw; ++tw)
      v.push_back(Phase{phase_axis(th, s.H, s.kh, s.sh, s.ph, s.dh), phase_axis(tw, s.W, s.kw, s.sw, s.pw, s.dw)});
  return v;
}
static bool phase_has_gemm(const Phase& f) { return f.a.M > 0 && f.b.M > 0 && f.a.n > 0 && f.b.n > 0; }
static size_t phase_region(const ConvShape& s, const Phase& f, int math) {
  return phase_has_gemm(f) ? (tc_deconv_phase_prep_bytes(s, f.a, f.b, math) + 255) & ~(size_t)255 : 0;
}
static int phase_math(const b2c_deconv_desc* d) { return d->dual->math == B2C_MATH_TF32 ? B2C_MATH_TF32 : B2C_MATH_FP32; }

static bool depthwise(const b2c_deconv_desc* d) { return d->G == d->C && d->C == d->O; }

// The route of `op` (b2c_deconv_route), decided in one place for the launches, the workspace size and b2c_debug_deconv_plan.
static int deconv_route(const b2c_deconv_desc* d, int op) {
  const ConvShape& s = d->dual->s;
  if (d->dual->engine == B2C_ENGINE_CAFFE) return B2C_DECONV_ROUTE_DUAL;
  if (depthwise(d)) return B2C_DECONV_ROUTE_DEPTHWISE;
  if (op != B2C_OP_FORWARD) return B2C_DECONV_ROUTE_DUAL;
  if (s.sh == 1 && s.sw == 1) return B2C_DECONV_ROUTE_DUAL;                                    // dgrad-as-forward routes
  if (s.kh == 1 && s.kw == 1 && s.ph == 0 && s.pw == 0) return B2C_DECONV_ROUTE_DUAL;         // the scatter route
  if (d->dual->algo == B2C_ALGO_SIMT) return B2C_DECONV_ROUTE_DUAL;                           // the caller asked for FFMA
  for (const Phase& f : d->phases)
    if (phase_has_gemm(f) && !tc_deconv_phase_supported(s, f.a, f.b)) return B2C_DECONV_ROUTE_DUAL;
  return B2C_DECONV_ROUTE_PHASE;
}

// ---- kernels ---------------------------------------------------------------------------------------------------------------
// Depthwise shapes: bottom [N, C, Hb, Wb], top [N, C, Ht, Wt], filter [C, 1, kh, kw].
struct DwShape { int N, C, Hb, Wb, Ht, Wt, kh, kw, sh, sw, ph, pw, dh, dw, Lh, Lw; };

// the smallest tap i in [0, k) with i*d == r (mod s), or -1 (L = s / gcd(s, d): the taps of one residue are L apart)
__device__ __forceinline__ int first_tap(int r, int k, int s, int d, int L) {
  if (d == 1) return r < k ? r : -1;
  for (int i = 0; i < k && i < L; ++i)
    if ((i * d) % s == r) return i;
  return -1;
}

// Forward: one thread per top element.  Tap order: i ascending, then j ascending, over the on-grid in-bounds taps only; each
// product rounded to fp32 and added to the running sum (no FMA contraction), starting from +0; the bias added last.
__global__ void __launch_bounds__(256)
deconv_dw_fwd_kernel(const DwShape s, const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                     float* __restrict__ y) {
  const size_t total = (size_t)s.N * s.C * s.Ht * s.Wt;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int tw = (int)(idx % s.Wt);
    const size_t r1 = idx / s.Wt;
    const int th = (int)(r1 % s.Ht);
    const size_t nc = r1 / s.Ht;
    const int c = (int)(nc % s.C);
    const float* xp = x + nc * s.Hb * s.Wb;
    const float* wp = w + (size_t)c * s.kh * s.kw;
    float acc = 0.0f;
    const int i0 = first_tap((th + s.ph) % s.sh, s.kh, s.sh, s.dh, s.Lh);
    const int j0 = first_tap((tw + s.pw) % s.sw, s.kw, s.sw, s.dw, s.Lw);
    if (i0 >= 0 && j0 >= 0) {
      for (int i = i0; i < s.kh; i += s.Lh) {
        const int nh = th + s.ph - i * s.dh;
        if (nh < 0) break;
        const int h = nh / s.sh;
        if (h >= s.Hb) continue;
        for (int j = j0; j < s.kw; j += s.Lw) {
          const int nw = tw + s.pw - j * s.dw;
          if (nw < 0) break;
          const int ww = nw / s.sw;
          if (ww >= s.Wb) continue;
          acc = __fadd_rn(acc, __fmul_rn(__ldg(xp + h * s.Wb + ww), __ldg(wp + i * s.kw + j)));
        }
      }
    }
    if (bias) acc = __fadd_rn(acc, __ldg(bias + c));
    y[idx] = acc;
  }
}

// Data gradient: the depthwise strided convolution of the top diff, one thread per bottom element, the same tap order and
// rounding as the forward (no bias).
__global__ void __launch_bounds__(256)
deconv_dw_dgrad_kernel(const DwShape s, const float* __restrict__ dy, const float* __restrict__ w, float* __restrict__ dx) {
  const size_t total = (size_t)s.N * s.C * s.Hb * s.Wb;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int wb = (int)(idx % s.Wb);
    const size_t r1 = idx / s.Wb;
    const int hb = (int)(r1 % s.Hb);
    const size_t nc = r1 / s.Hb;
    const int c = (int)(nc % s.C);
    const float* dp = dy + nc * s.Ht * s.Wt;
    const float* wp = w + (size_t)c * s.kh * s.kw;
    float acc = 0.0f;
    for (int i = 0; i < s.kh; ++i) {
      const int th = hb * s.sh - s.ph + i * s.dh;
      if ((unsigned)th >= (unsigned)s.Ht) continue;
      for (int j = 0; j < s.kw; ++j) {
        const int tw = wb * s.sw - s.pw + j * s.dw;
        if ((unsigned)tw >= (unsigned)s.Wt) continue;
        acc = __fadd_rn(acc, __fmul_rn(__ldg(dp + th * s.Wt + tw), __ldg(wp + i * s.kw + j)));
      }
    }
    dx[idx] = acc;
  }
}

// Weight gradient, dW[c][i][j] += sum_{n,h,w} x[n][c][h][w] * dy[n][c][h*sh - ph + i*dh][w*sw - pw + j*dw]: one 256-thread block
// per (tap, channel).  Thread t sums the elements e = t, t + 256, ... of the flattened (n, h, w) range in order (products rounded,
// then added); then an xor butterfly per warp, the 8 warp partials summed in warp order by thread 0, and one add onto dW.  Fixed
// slots and a fixed combine order, no atomics: the same bits on every call.
constexpr int DW_WG_THREADS = 256;
__global__ void __launch_bounds__(DW_WG_THREADS)
deconv_dw_wgrad_kernel(const DwShape s, const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dw) {
  __shared__ float part[DW_WG_THREADS / 32];
  const int tap = blockIdx.x, c = blockIdx.y;
  const int i = tap / s.kw, j = tap - i * s.kw;
  const long long P = (long long)s.Hb * s.Wb, total = (long long)s.N * P;
  float acc = 0.0f;
  for (long long e = threadIdx.x; e < total; e += DW_WG_THREADS) {
    const int n = (int)(e / P);
    const int pix = (int)(e - (long long)n * P);
    const int hb = pix / s.Wb, wb = pix - hb * s.Wb;
    const int th = hb * s.sh - s.ph + i * s.dh, tw = wb * s.sw - s.pw + j * s.dw;
    if ((unsigned)th >= (unsigned)s.Ht || (unsigned)tw >= (unsigned)s.Wt) continue;
    const long long nc = (long long)n * s.C + c;
    acc = __fadd_rn(acc, __fmul_rn(__ldg(x + nc * P + pix), __ldg(dy + nc * s.Ht * s.Wt + (long long)th * s.Wt + tw)));
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) acc = __fadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, o));
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = part[0];
#pragma unroll
    for (int k = 1; k < DW_WG_THREADS / 32; ++k) t = __fadd_rn(t, part[k]);
    float* o = dw + (size_t)c * s.kh * s.kw + tap;
    *o = __fadd_rn(*o, t);
  }
}

// A phase of the PHASE route that no tap reaches: top[n][o][t0h + sh*m][t0w + sw*m'] = bias[o] (or 0).
__global__ void __launch_bounds__(256)
deconv_phase_fill_kernel(int NO, int O, int Ht, int Wt, int t0h, int t0w, int sh, int sw, int Mh, int Mw,
                         const float* __restrict__ bias, float* __restrict__ y) {
  const size_t total = (size_t)NO * Mh * Mw;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int mw = (int)(idx % Mw);
    const size_t r1 = idx / Mw;
    const int mh = (int)(r1 % Mh);
    const size_t no = r1 / Mh;
    y[no * Ht * Wt + (size_t)(t0h + sh * mh) * Wt + t0w + sw * mw] = bias ? __ldg(bias + no % O) : 0.0f;
  }
}

// ---- Crop ------------------------------------------------------------------------------------------------------------------
constexpr int CROP_MAX_AXES = 32;   // Blob's kMaxBlobAxes
struct CropGeom {
  int nax, vec;                      // vec: units of 4 floats
  int tshape[CROP_MAX_AXES], off[CROP_MAX_AXES];
  long long bstride[CROP_MAX_AXES];
};
// One thread per unit of the top window (a float, or 4 when vec); dir 0: top = bottom[window], dir 1: bottom[window] = top.
__global__ void __launch_bounds__(256)
crop_kernel(const __grid_constant__ CropGeom g, long long units, int dir, const float* __restrict__ src, float* __restrict__ dst) {
  for (long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x; u < units; u += (long long)gridDim.x * blockDim.x) {
    long long t = g.vec ? 4 * u : u, rem = t, b = 0;
    for (int a = g.nax - 1; a >= 0; --a) {
      const int e = (int)(rem % g.tshape[a]);
      rem /= g.tshape[a];
      b += (long long)(e + g.off[a]) * g.bstride[a];
    }
    const long long si = dir == 0 ? b : t, di = dir == 0 ? t : b;
    if (g.vec) *reinterpret_cast<float4*>(dst + di) = __ldg(reinterpret_cast<const float4*>(src + si));
    else dst[di] = __ldg(src + si);
  }
}

static int crop_geom(const char* who, int nax, const int* bshape, const int* tshape, const int* offsets, const void* a, const void* b,
                     CropGeom* g, long long* count) {
  if (nax < 1 || nax > CROP_MAX_AXES || !bshape || !tshape || !offsets) return fail(B2C_ERR_INVALID, "%s: bad shape arguments", who);
  *g = CropGeom{};
  g->nax = nax;
  long long n = 1, stride = 1;
  for (int i = nax - 1; i >= 0; --i) {
    if (bshape[i] < 0 || tshape[i] < 0 || offsets[i] < 0) return fail(B2C_ERR_INVALID, "%s: negative extent or offset on axis %d", who, i);
    if (bshape[i] - offsets[i] < tshape[i])   // CropLayer::Reshape's CHECK_GE(bottom - crop, top)
      return fail(B2C_ERR_INVALID, "%s: invalid crop parameters in dimension: %d", who, i);
    g->tshape[i] = tshape[i]; g->off[i] = offsets[i]; g->bstride[i] = stride;
    stride *= bshape[i];
    n *= tshape[i];
  }
  const int last = nax - 1;
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
  g->vec = tshape[last] % 4 == 0 && offsets[last] % 4 == 0 && bshape[last] % 4 == 0 && al16(a) && al16(b) ? 1 : 0;
  *count = n;
  return B2C_OK;
}

static DwShape dw_shape(const b2c_deconv_desc* d) {
  const ConvShape& s = d->dual->s;
  return DwShape{s.N, d->C, s.Ho, s.Wo, s.H, s.W, s.kh, s.kw, s.sh, s.sw, s.ph, s.pw, s.dh, s.dw,
                 s.sh / gcd_int(s.sh, s.dh), s.sw / gcd_int(s.sw, s.dw)};
}

static bool have_device_() {
  static int ok = -1;
  if (ok < 0) { int n = 0; ok = (cudaGetDeviceCount(&n) == cudaSuccess && n > 0) ? 1 : 0; }
  return ok == 1;
}

}  // namespace b2c

using namespace b2c;

#define REQUIRE_DEVICE() \
  if (!have_device_()) return fail(B2C_ERR_CUDA, "no CUDA device: this library has no CPU fallback")

extern "C" int b2c_deconv_desc_create(const b2c_conv_params* p, int engine, b2c_deconv_desc** out) {
  if (!p || !out) return fail(B2C_ERR_INVALID, "b2c_deconv_desc_create: null");
  if (p->N <= 0 || p->C <= 0 || p->H <= 0 || p->W <= 0 || p->O <= 0) return fail(B2C_ERR_INVALID, "deconv: non-positive blob dimension");
  if (p->kh <= 0 || p->kw <= 0) return fail(B2C_ERR_INVALID, "deconv: Filter dimensions must be nonzero");
  if (p->sh <= 0 || p->sw <= 0) return fail(B2C_ERR_INVALID, "deconv: Stride dimensions must be nonzero");
  if (p->dh <= 0 || p->dw <= 0) return fail(B2C_ERR_INVALID, "deconv: dilation must be positive");
  if (p->ph < 0 || p->pw < 0) return fail(B2C_ERR_INVALID, "deconv: negative pad");
  // deconv_layer.cpp:7-22
  const long long Ht = (long long)p->sh * (p->H - 1) + (long long)p->dh * (p->kh - 1) + 1 - 2LL * p->ph;
  const long long Wt = (long long)p->sw * (p->W - 1) + (long long)p->dw * (p->kw - 1) + 1 - 2LL * p->pw;
  if (Ht <= 0 || Wt <= 0)
    return fail(B2C_ERR_INVALID, "deconv: output extent %lld x %lld is not positive (pad larger than the upsampled input)", Ht, Wt);
  if (Ht > 0x7fffffffLL || Wt > 0x7fffffffLL) return fail(B2C_ERR_INVALID, "deconv: output extent too large");
  // the dual convolution: input = the top [N, O, Ht, Wt], output = the bottom, filter [C, O/G, kh, kw]
  b2c_conv_params q = *p;
  q.C = p->O; q.O = p->C; q.H = (int)Ht; q.W = (int)Wt; q.has_bias = 0;
  b2c_conv_desc* dual = nullptr;
  if (int rc = b2c_conv_desc_create(&q, engine, &dual)) return rc;
  if (dual->s.Ho != p->H || dual->s.Wo != p->W) {
    b2c_conv_desc_destroy(dual);
    return fail(B2C_ERR_INVALID, "deconv: the dual convolution does not map %dx%d back to the bottom", (int)Ht, (int)Wt);
  }
  *out = new b2c_deconv_desc{dual, p->N, p->C, p->H, p->W, p->O, p->G, p->has_bias, phases(dual->s)};
  return B2C_OK;
}
extern "C" int b2c_deconv_desc_destroy(b2c_deconv_desc* d) {
  if (d) { b2c_conv_desc_destroy(d->dual); delete d; }
  return B2C_OK;
}
extern "C" int b2c_deconv_desc_set_math(b2c_deconv_desc* d, int math) {
  if (!d) return fail(B2C_ERR_INVALID, "deconv set_math: null descriptor");
  return b2c_conv_desc_set_math(d->dual, math);
}
extern "C" int b2c_deconv_desc_set_algo(b2c_deconv_desc* d, int algo) {
  if (!d) return fail(B2C_ERR_INVALID, "deconv set_algo: null descriptor");
  return b2c_conv_desc_set_algo(d->dual, algo);
}
extern "C" int b2c_deconv_out_shape(const b2c_deconv_desc* d, int* Ht, int* Wt) {
  if (!d) return fail(B2C_ERR_INVALID, "null desc");
  if (Ht) *Ht = d->dual->s.H;
  if (Wt) *Wt = d->dual->s.W;
  return B2C_OK;
}

extern "C" size_t b2c_deconv_workspace_bytes(const b2c_deconv_desc* d, int op) {
  if (!d) return 0;
  const int route = deconv_route(d, op);
  if (route == B2C_DECONV_ROUTE_DEPTHWISE) return 0;
  if (route == B2C_DECONV_ROUTE_PHASE) {
    size_t n = 256;   // alignment slack
    for (const Phase& f : d->phases) n += phase_region(d->dual->s, f, phase_math(d));
    return n;
  }
  const int dual_op = op == B2C_OP_FORWARD ? B2C_OP_BACKWARD_DATA : op == B2C_OP_BACKWARD_DATA ? B2C_OP_FORWARD : B2C_OP_BACKWARD_FILTER;
  return b2c_conv_workspace_bytes(d->dual, dual_op);
}

extern "C" int b2c_deconv_forward(const b2c_deconv_desc* d, const float* x, const float* w, const float* bias, float* y, void* ws,
                                  size_t ws_bytes, void* stream) {
  if (!d || !x || !w || !y) return fail(B2C_ERR_INVALID, "b2c_deconv_forward: null pointer");
  REQUIRE_DEVICE();
  if (d->has_bias && !bias) return fail(B2C_ERR_INVALID, "b2c_deconv_forward: bias_term set but bias is null");
  if (!d->has_bias) bias = nullptr;
  const ConvShape& s = d->dual->s;
  cudaStream_t st = as_stream(stream);
  const size_t need = b2c_deconv_workspace_bytes(d, B2C_OP_FORWARD);
  if (ws_bytes < need || (need && !ws)) return fail(B2C_ERR_WORKSPACE, "deconv forward workspace too small");
  const int route = deconv_route(d, B2C_OP_FORWARD);
  if (route == B2C_DECONV_ROUTE_DEPTHWISE) {
    const DwShape g = dw_shape(d);
    const size_t total = (size_t)g.N * g.C * g.Ht * g.Wt;
    deconv_dw_fwd_kernel<<<grid_for(total, 256), 256, 0, st>>>(g, x, w, bias, y);
    B2C_POST_LAUNCH();
    return B2C_OK;
  }
  if (route == B2C_DECONV_ROUTE_PHASE) {
    const int math = phase_math(d);
    const std::vector<Phase>& ph = d->phases;
    std::vector<PrepEntry> q(ph.size());
    std::vector<PrepEntry> gemm;
    char* base = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~(uintptr_t)255);
    for (size_t k = 0; k < ph.size(); ++k) {
      if (!phase_has_gemm(ph[k])) continue;
      tc_deconv_phase_prep_entry(s, ph[k].a, ph[k].b, math, w, base, &q[k]);
      gemm.push_back(q[k]);
      base += phase_region(s, ph[k], math);
    }
    if (!gemm.empty())
      if (int rc = launch_filter_prep(gemm.data(), (int)gemm.size(), st)) return rc;
    for (size_t k = 0; k < ph.size(); ++k) {
      const Phase& f = ph[k];
      if (f.a.M == 0 || f.b.M == 0) continue;
      if (!phase_has_gemm(f)) {
        const size_t total = (size_t)s.N * s.C * f.a.M * f.b.M;
        deconv_phase_fill_kernel<<<grid_for(total, 256), 256, 0, st>>>(s.N * s.C, s.C, s.H, s.W, f.a.t0, f.b.t0, s.sh, s.sw, f.a.M,
                                                                       f.b.M, bias, y);
        B2C_POST_LAUNCH();
        continue;
      }
      if (int rc = launch_deconv_phase_tc(s, f.a, f.b, math, x, bias, y, q[k], st)) return rc;
    }
    return B2C_OK;
  }
  if (int rc = b2c_conv_backward_data(d->dual, x, w, y, ws, ws_bytes, stream)) return rc;
  if (bias) return launch_bias_add(s.N, s.C, s.H * s.W, bias, y, st);
  return B2C_OK;
}

extern "C" int b2c_deconv_backward_data(const b2c_deconv_desc* d, const float* dy, const float* w, float* dx, void* ws, size_t ws_bytes,
                                        void* stream) {
  if (!d || !dy || !w || !dx) return fail(B2C_ERR_INVALID, "b2c_deconv_backward_data: null pointer");
  REQUIRE_DEVICE();
  if (deconv_route(d, B2C_OP_BACKWARD_DATA) == B2C_DECONV_ROUTE_DEPTHWISE) {
    const DwShape g = dw_shape(d);
    const size_t total = (size_t)g.N * g.C * g.Hb * g.Wb;
    deconv_dw_dgrad_kernel<<<grid_for(total, 256), 256, 0, as_stream(stream)>>>(g, dy, w, dx);
    B2C_POST_LAUNCH();
    return B2C_OK;
  }
  return b2c_conv_forward(d->dual, dy, w, nullptr, dx, ws, ws_bytes, stream);
}

extern "C" size_t b2c_deconv_wgrad_split_bytes(const b2c_deconv_desc* d) {
  if (!d || deconv_route(d, B2C_OP_BACKWARD_FILTER) != B2C_DECONV_ROUTE_DUAL) return 0;
  return b2c_conv_wgrad_split_bytes(d->dual);
}

extern "C" int b2c_deconv_backward_filter_split(const b2c_deconv_desc* d, const float* x, const float* dy, float* dw, void* ws,
                                                size_t ws_bytes, void* split, size_t split_bytes, void* stream) {
  if (!d || !x || !dy || !dw) return fail(B2C_ERR_INVALID, "b2c_deconv_backward_filter: null pointer");
  REQUIRE_DEVICE();
  if (deconv_route(d, B2C_OP_BACKWARD_FILTER) == B2C_DECONV_ROUTE_DEPTHWISE) {
    const DwShape g = dw_shape(d);
    if (g.C > 65535) return fail(B2C_ERR_INVALID, "b2c_deconv_backward_filter: %d channels exceed the depthwise grid", g.C);
    deconv_dw_wgrad_kernel<<<dim3((unsigned)(g.kh * g.kw), (unsigned)g.C), DW_WG_THREADS, 0, as_stream(stream)>>>(g, x, dy, dw);
    B2C_POST_LAUNCH();
    return B2C_OK;
  }
  // the dual's weight gradient: its input is the top diff, its output gradient the bottom data
  return b2c_conv_backward_filter_split(d->dual, dy, x, dw, ws, ws_bytes, split, split_bytes, stream);
}
extern "C" int b2c_deconv_backward_filter(const b2c_deconv_desc* d, const float* x, const float* dy, float* dw, void* ws,
                                          size_t ws_bytes, void* stream) {
  return b2c_deconv_backward_filter_split(d, x, dy, dw, ws, ws_bytes, nullptr, 0, stream);
}

extern "C" int b2c_deconv_backward_bias(const b2c_deconv_desc* d, const float* dy, float* db, void* stream) {
  if (!d || !dy || !db) return fail(B2C_ERR_INVALID, "b2c_deconv_backward_bias: null pointer");
  REQUIRE_DEVICE();
  const ConvShape& s = d->dual->s;
  return launch_bias_grad(s.N, s.C, s.H * s.W, dy, db, as_stream(stream));
}

extern "C" int b2c_debug_deconv_plan(const b2c_deconv_desc* d, int op, int* out, int n) {
  if (!d || !out || n < 3) return fail(B2C_ERR_INVALID, "b2c_debug_deconv_plan: need a descriptor and 3 ints");
  if (op < B2C_OP_FORWARD || op > B2C_OP_BACKWARD_FILTER) return fail(B2C_ERR_INVALID, "b2c_debug_deconv_plan: bad op %d", op);
  const int route = deconv_route(d, op);
  out[0] = route; out[1] = -1; out[2] = 0;
  if (route == B2C_DECONV_ROUTE_DUAL) {
    int q[8] = {0};
    int rc = op == B2C_OP_BACKWARD_FILTER ? b2c_debug_wgrad_plan(d->dual, q, 7)
                                          : b2c_debug_conv_plan(d->dual, op == B2C_OP_FORWARD ? B2C_OP_BACKWARD_DATA : B2C_OP_FORWARD, q, 8);
    if (rc) return rc;
    out[1] = q[0];
  } else if (route == B2C_DECONV_ROUTE_PHASE) {
    const ConvShape& s = d->dual->s;
    const std::vector<Phase>& ph = d->phases;
    if (n < 3 + 2 * (int)ph.size())
      return fail(B2C_ERR_INVALID, "b2c_debug_deconv_plan: the phase route needs %d ints", 3 + 2 * (int)ph.size());
    out[2] = (int)ph.size();
    for (size_t k = 0; k < ph.size(); ++k) {
      const Phase& f = ph[k];
      ConvPlanInfo q{};
      if (phase_has_gemm(f)) tc_deconv_phase_plan_info(s, f.a, f.b, &q);
      out[3 + 2 * k] = f.a.n * f.b.n;
      out[4 + 2 * k] = q.tiles;
    }
  }
  return B2C_OK;
}

extern "C" int b2c_crop_forward(int num_axes, const int* bottom_shape, const int* top_shape, const int* offsets, const float* bottom,
                                float* top, void* stream) {
  CropGeom g;
  long long n = 0;
  if (int rc = crop_geom("b2c_crop_forward", num_axes, bottom_shape, top_shape, offsets, bottom, top, &g, &n)) return rc;
  if (n == 0) return B2C_OK;
  if (!bottom || !top) return fail(B2C_ERR_INVALID, "b2c_crop_forward: null pointer");
  REQUIRE_DEVICE();
  const long long units = g.vec ? n / 4 : n;
  crop_kernel<<<grid_for((size_t)units, 256), 256, 0, as_stream(stream)>>>(g, units, 0, bottom, top);
  B2C_POST_LAUNCH();
  return B2C_OK;
}

extern "C" int b2c_crop_backward(int num_axes, const int* bottom_shape, const int* top_shape, const int* offsets, const float* top_diff,
                                 float* bottom_diff, void* stream) {
  CropGeom g;
  long long n = 0;
  if (int rc = crop_geom("b2c_crop_backward", num_axes, bottom_shape, top_shape, offsets, top_diff, bottom_diff, &g, &n)) return rc;
  if (!top_diff || !bottom_diff) return fail(B2C_ERR_INVALID, "b2c_crop_backward: null pointer");
  REQUIRE_DEVICE();
  size_t bcount = 1;
  for (int i = 0; i < num_axes; ++i) bcount *= (size_t)bottom_shape[i];
  cudaStream_t st = as_stream(stream);
  B2C_CUDA_OK(cudaMemsetAsync(bottom_diff, 0, sizeof(float) * bcount, st));
  if (n == 0) return B2C_OK;
  const long long units = g.vec ? n / 4 : n;
  crop_kernel<<<grid_for((size_t)units, 256), 256, 0, st>>>(g, units, 1, top_diff, bottom_diff);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
