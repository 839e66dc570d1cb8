/*
 * b2c.h -- C ABI of the H100-native Caffe-MPI data-parallel hot path
 *          (ConvolutionLayer forward/backward, im2col/col2im, SGEMM/SGEMV, fused
 *          SGD-momentum update, NCCL gradient exchange).
 *
 * This is the drop-in boundary (SURVEY.md 8b): plain pointers and sizes, no torch or
 * C++ types.  Every entry point names the reference interface it replaces (paths
 * relative to the Caffe-MPI tree).  All tensor pointers are DEVICE pointers, fp32,
 * dense row-major; activations NCHW, weights [O, C/g, kh, kw], bias [O].  `stream`
 * is the caller's cudaStream_t passed as void* (NULL = legacy default stream).
 * Calls are asynchronous on `stream`; nothing host-synchronises (the reference syncs
 * after every BLAS call, math_functions.cu:25 -- callers that need that behaviour
 * synchronise the stream themselves).
 *
 * Error model: the reference aborts through glog CHECK / CUDA_CHECK
 * (include/caffe/util/nccl.hpp:10-15).  Here every function returns 0 on success or
 * a negative b2c_status and leaves a thread-local message readable with
 * b2c_last_error(); the C++ layer shim turns non-zero into a fatal check.
 * There is NO CPU fallback: on a machine without a CUDA device every compute entry
 * point returns B2C_ERR_CUDA.
 */
#ifndef B2C_H_
#define B2C_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  B2C_OK = 0,
  B2C_ERR_INVALID = -1,     /* bad argument / unsupported shape            */
  B2C_ERR_CUDA = -2,        /* CUDA runtime / launch error                 */
  B2C_ERR_NCCL = -3,        /* NCCL error                                  */
  B2C_ERR_WORKSPACE = -4    /* workspace too small                         */
} b2c_status;

/* ConvolutionParameter.engine, src/caffe/proto/caffe.proto:745-750 (same values).
 * CAFFE  -> explicit per-image im2col + GEMM (base_conv_layer.hpp:105-168).
 * CUDNN / DEFAULT -> implicit-GEMM kernels (replaces cudnn_conv_layer.cu:13-132). */
typedef enum { B2C_ENGINE_DEFAULT = 0, B2C_ENGINE_CAFFE = 1, B2C_ENGINE_CUDNN = 2 } b2c_engine;

/* Math mode of the tensor-core kernels (NetParameter default_forward_math /
 * default_backward_math, caffe.proto:124-127, is the reference's analogous knob).
 * FP32        : split-precision wgmma, fp32-equivalent results (default): bf16 hi/lo split, three
 *               bf16 MMAs per K step, on the layers the bulk-copy-staged kernel takes (stride-1 "same"
 *               convolutions, forward and dgrad); 3xTF32 split everywhere else.  Blob error ~1e-6..1e-5.
 * TF32        : single-pass TF32 (round-to-nearest operands), ~1e-3 relative.
 * FP32_3XTF32 : the 3xTF32 split on every layer (the round-1 default; ~1e-7..4e-5).          */
typedef enum { B2C_MATH_FP32 = 0, B2C_MATH_TF32 = 1, B2C_MATH_FP32_3XTF32 = 2 } b2c_math;

/* Kernel family used by the implicit-GEMM engine (diagnostics / tests); B2C_ALGO_TCGEN05 names the tensor-core
 * kernels (wgmma on sm_90a). */
typedef enum { B2C_ALGO_AUTO = 0, B2C_ALGO_SIMT = 1, B2C_ALGO_TCGEN05 = 2 } b2c_algo;

typedef enum { B2C_OP_FORWARD = 0, B2C_OP_BACKWARD_DATA = 1, B2C_OP_BACKWARD_FILTER = 2 } b2c_conv_op;

/* Shape of one ConvolutionLayer call: ConvolutionParameter (caffe.proto:718-786) plus
 * the bottom shape BaseConvolutionLayer::Reshape reads (base_conv_layer.cpp:172-239). */
typedef struct {
  int N, C, H, W;     /* bottom blob                                              */
  int O, G;           /* num_output, group                                        */
  int kh, kw;         /* kernel_size / kernel_h,kernel_w                          */
  int sh, sw;         /* stride                                                   */
  int ph, pw;         /* pad                                                      */
  int dh, dw;         /* dilation                                                 */
  int has_bias;       /* bias_term                                                */
} b2c_conv_params;

typedef struct b2c_conv_desc b2c_conv_desc;
typedef struct b2c_comm b2c_comm;

/* ---- library ------------------------------------------------------------------- */
const char* b2c_last_error(void);
const char* b2c_version(void);
/* number of kernels THIS library has launched in this process (all threads).      */
uint64_t b2c_launch_count(void);
/* process-wide defaults used by descriptors created afterwards                    */
int b2c_set_default_math(int math /* b2c_math */);
int b2c_set_default_algo(int algo /* b2c_algo */);

/* ---- convolution descriptor -------------------------------------------------------
 * Replaces BaseConvolutionLayer::LayerSetUp/Reshape bookkeeping (base_conv_layer.cpp:12-239)
 * and CuDNNConvolutionLayer's descriptor set-up (cudnn_conv_layer.cpp:78-210).        */
int b2c_conv_desc_create(const b2c_conv_params* p, int engine, b2c_conv_desc** out);
int b2c_conv_desc_destroy(b2c_conv_desc* d);
int b2c_conv_desc_set_math(b2c_conv_desc* d, int math);
int b2c_conv_desc_set_algo(b2c_conv_desc* d, int algo);
/* output extent, conv_layer.cpp:7-22 (truncating division)                          */
int b2c_conv_out_shape(const b2c_conv_desc* d, int* Ho, int* Wo);
/* scratch bytes the given op needs (col buffer for CAFFE engine: base_conv_layer.cpp:225-233;
 * split-K partials / transformed weights for the implicit engine).                   */
size_t b2c_conv_workspace_bytes(const b2c_conv_desc* d, int op);
/* which kernel family the op will run (b2c_algo) -- lets tests assert "the tensor cores ran". */
int b2c_conv_algo_used(const b2c_conv_desc* d, int op);

/* Prepared filters.  The tensor-core forward / dgrad kernels read the filter through TMA in a GEMM-ordered, hi/lo-split copy
 * that b2c_conv_forward / b2c_conv_backward_data otherwise rebuild on every call.  Weights change once per iteration
 * (SGDSolver::ApplyUpdate, sgd_solver.cpp:143-149), so a caller that owns the iteration can build the copies ONCE:
 *   bytes = b2c_conv_filter_cache_bytes(d);            cudaMalloc(&cache, bytes)  (256-byte aligned; 0 = nothing to cache)
 *   b2c_conv_desc_bind_filter_cache(d, cache);          forward / backward_data now trust the cache
 *   b2c_conv_prepare_filters(n, descs, ws, caches, s)   after every weight update: ONE multi-tensor launch per 24 layouts
 * Binding NULL restores the self-contained behaviour.  The cache is the caller's promise that it was prepared from the `w`
 * passed to forward / backward_data; nothing checks it.  (cuDNN's analogue: cudnnTransformFilter + a persistent
 * filter descriptor; the reference re-reads the blob each call, cudnn_conv_layer.cu:25-29.) */
size_t b2c_conv_filter_cache_bytes(const b2c_conv_desc* d);
int b2c_conv_desc_bind_filter_cache(b2c_conv_desc* d, const void* cache);
int b2c_conv_prepare_filter(const b2c_conv_desc* d, const float* w, void* cache, size_t cache_bytes, void* stream);
int b2c_conv_prepare_filters(int n, const b2c_conv_desc* const* descs, const float* const* ws, void* const* caches,
                             void* stream);


/* Y = conv(X, W) (+ bias).  y OVERWRITTEN.
 * Replaces ConvolutionLayer::Forward_gpu (conv_layer.cu:7-23) = forward_gpu_gemm +
 * forward_gpu_bias (base_conv_layer.hpp:105-128) and CuDNNConvolutionLayer::Forward_gpu
 * (cudnn_conv_layer.cu:13-58: cudnnConvolutionForward beta=0 + cudnnAddTensor).      */
int b2c_conv_forward(const b2c_conv_desc* d, const float* x, const float* w, const float* bias,
                     float* y, void* ws, size_t ws_bytes, void* stream);
/* dX = conv_bwd_data(dY, W).  dx OVERWRITTEN.
 * Replaces backward_gpu_gemm + col2im (base_conv_layer.hpp:130-146) /
 * cudnnConvolutionBackwardData beta=0 (cudnn_conv_layer.cu:118-123).                 */
int b2c_conv_backward_data(const b2c_conv_desc* d, const float* dy, const float* w, float* dx,
                           void* ws, size_t ws_bytes, void* stream);
/* dW += conv_bwd_filter(X, dY).  dw ACCUMULATED (beta = 1).
 * Replaces weight_gpu_gemm (base_conv_layer.hpp:148-162) /
 * cudnnConvolutionBackwardFilter beta=1 (cudnn_conv_layer.cu:95-99).                 */
/* dx += the bottom gradient (instead of dx = ...): where a blob feeds several layers the reference sums their bottom diffs
 * in SplitLayer::Backward (split_layer.cpp); here the second and later writers add straight into the blob's diff through
 * the kernel's TMA reduce-add store.  Available for the layers the staged kernel takes; ask first. */
int b2c_conv_backward_data_accumulate_supported(const b2c_conv_desc* d);
int b2c_conv_backward_data_accumulate(const b2c_conv_desc* d, const float* dy, const float* w, float* dx,
                                      void* ws, size_t ws_bytes, void* stream);
int b2c_conv_backward_filter(const b2c_conv_desc* d, const float* x, const float* dy, float* dw,
                             void* ws, size_t ws_bytes, void* stream);
/* The same dW += ..., with a second scratch buffer of b2c_conv_wgrad_split_bytes(d) bytes (16-byte aligned, disjoint from ws):
 * on the 3x3 layers where many thread blocks of the TMA-staged kernel would each convert the same dY block to bf16 hi / lo, one
 * pass converts dY once into `split` before the kernel runs.  Same bits as b2c_conv_backward_filter.  split == NULL (and every
 * layer whose size query is 0) runs exactly b2c_conv_backward_filter. */
size_t b2c_conv_wgrad_split_bytes(const b2c_conv_desc* d);
int b2c_conv_backward_filter_split(const b2c_conv_desc* d, const float* x, const float* dy, float* dw,
                                   void* ws, size_t ws_bytes, void* split, size_t split_bytes, void* stream);
/* db[o] += sum_{n,h,w} dY.  db ACCUMULATED (beta = 1).
 * Replaces backward_gpu_bias (base_conv_layer.hpp:164-168, gemv per image) /
 * cudnnConvolutionBackwardBias beta=1 (cudnn_conv_layer.cu:73-75).                   */
int b2c_conv_backward_bias(const b2c_conv_desc* d, const float* dy, float* db, void* stream);

/* ---- transposed convolution (DeconvolutionLayer, src/caffe/layers/deconv_layer.{cpp,cu}) ----------------------------------
 * The descriptor takes the deconvolution's own parameters and bottom shape: b2c_conv_params with C = bottom channels, H, W = bottom
 * extent, O = num_output.  Top extent Ht = sh*(H-1) + dh*(kh-1) + 1 - 2*ph (deconv_layer.cpp:7-22; a non-positive extent is
 * refused), weights [C, O/G, kh, kw], bias [O].  Internally it holds the DUAL convolution (input = the top [N, O, Ht, Wt], output =
 * the bottom, filter = the same weight blob), so math / algo / engine mean what they mean for b2c_conv_desc.  Same calling rules
 * as the b2c_conv_* entry points: y and dx overwritten, dw and db accumulated. */
typedef struct b2c_deconv_desc b2c_deconv_desc;
int b2c_deconv_desc_create(const b2c_conv_params* p, int engine, b2c_deconv_desc** out);
int b2c_deconv_desc_destroy(b2c_deconv_desc* d);
int b2c_deconv_desc_set_math(b2c_deconv_desc* d, int math);
int b2c_deconv_desc_set_algo(b2c_deconv_desc* d, int algo);
int b2c_deconv_out_shape(const b2c_deconv_desc* d, int* Ht, int* Wt);
size_t b2c_deconv_workspace_bytes(const b2c_deconv_desc* d, int op);
/* y = deconv(x, W) (+ bias): the dual's data gradient. */
int b2c_deconv_forward(const b2c_deconv_desc* d, const float* x, const float* w, const float* bias, float* y, void* ws,
                       size_t ws_bytes, void* stream);
/* dx = the dual's forward of dy (no bias). */
int b2c_deconv_backward_data(const b2c_deconv_desc* d, const float* dy, const float* w, float* dx, void* ws, size_t ws_bytes,
                             void* stream);
/* dW += the dual's weight gradient with X = dy (top diff) and dY = x (bottom data); the _split form as
 * b2c_conv_backward_filter_split, with a buffer of b2c_deconv_wgrad_split_bytes(d) bytes. */
int b2c_deconv_backward_filter(const b2c_deconv_desc* d, const float* x, const float* dy, float* dw, void* ws, size_t ws_bytes,
                               void* stream);
size_t b2c_deconv_wgrad_split_bytes(const b2c_deconv_desc* d);
int b2c_deconv_backward_filter_split(const b2c_deconv_desc* d, const float* x, const float* dy, float* dw, void* ws, size_t ws_bytes,
                                     void* split, size_t split_bytes, void* stream);
/* db[o] += sum_{n,h,w} dy[n][o][h][w] (b2c_bias_backward over the top diff). */
int b2c_deconv_backward_bias(const b2c_deconv_desc* d, const float* dy, float* db, void* stream);
typedef enum {
  B2C_DECONV_ROUTE_DUAL = 0,       /* the dual convolution's routes: forward = b2c_conv_backward_data (+ one bias pass), backward    */
                                   /* data = b2c_conv_forward, weight gradient = b2c_conv_backward_filter[_split]                    */
  B2C_DECONV_ROUTE_PHASE = 1,      /* forward of a strided layer with k > 1 (not engine CAFFE): sh*sw stride-1 gather-kernel launches */
                                   /* on the bottom, one per output phase, each writing its lattice of the top with the bias fused   */
  B2C_DECONV_ROUTE_DEPTHWISE = 2   /* group == C == num_output, every op, except under engine CAFFE (always the DUAL route): direct  */
                                   /* fp32 kernels.  Forward and data gradient: per                                                  */
                                   /* output, taps i ascending then j ascending (on-grid, in-bounds taps only), each product rounded  */
                                   /* to fp32 then added (no FMA) from +0, bias added last.  Weight gradient per (c, i, j): 256       */
                                   /* lane-strided chains over the flattened (n, h, w), an xor butterfly per warp, the 8 warp         */
                                   /* partials in order, one add onto dW -- the same bits on every call                               */
} b2c_deconv_route;
/* The route of op (b2c_conv_op) for this descriptor: out[0] route (b2c_deconv_route), [1] for the DUAL route the dual's own route
 * (b2c_conv_route of its b2c_debug_conv_plan, or b2c_wgrad_route for the weight gradient), else -1; [2] phases (sh*sw on the PHASE
 * route, else 0); then per phase k (phase (t0h, t0w) = (k / sw, k % sw): outputs t0h + sh*m, t0w + sw*m'), [3 + 2k] its taps
 * (0: only the bias is written) and [4 + 2k] its gather-kernel tiles.  Needs n >= 3, and n >= 3 + 2*phases on the PHASE route.
 * Pure host computation. */
int b2c_debug_deconv_plan(const b2c_deconv_desc* d, int op, int* out, int n);

/* ---- Crop (CropLayer, src/caffe/layers/crop_layer.{cpp,cu}) ------------------------------------------------------------------
 * N-D (1..32 axes) window copy; shapes and per-axis offsets are HOST int arrays over every axis (0 offset on the uncropped ones).
 * Forward: top = bottom[offsets : offsets + top_shape].  Backward: bottom_diff zero-filled, then the top diff copied into the
 * window.  16-byte units when the innermost top extent, offset and bottom extent are multiples of 4 and both pointers 16-byte
 * aligned, else one float at a time (the same values).  Refuses (B2C_ERR_INVALID) num_axes outside [1, 32], negative extents or
 * offsets, and a window that leaves the bottom ("invalid crop parameters in dimension: i", crop_layer.cpp). */
int b2c_crop_forward(int num_axes, const int* bottom_shape, const int* top_shape, const int* offsets, const float* bottom, float* top,
                     void* stream);
int b2c_crop_backward(int num_axes, const int* bottom_shape, const int* top_shape, const int* offsets, const float* top_diff,
                      float* bottom_diff, void* stream);

/* ---- im2col / col2im ----------------------------------------------------------------
 * One image [C,H,W] <-> [C*kh*kw, Ho, Wo].  Replace im2col_gpu / col2im_gpu
 * (src/caffe/util/im2col.cu:42-62, 298-317).  col2im OVERWRITES im and adds the
 * contributions of each pixel in ascending (kh,kw) order (bit-identical to the
 * reference's col2im_cpu, im2col.cpp:176-211).                                         */
int b2c_im2col(const float* im, int C, int H, int W, int kh, int kw, int ph, int pw,
               int sh, int sw, int dh, int dw, float* col, void* stream);
int b2c_col2im(const float* col, int C, int H, int W, int kh, int kw, int ph, int pw,
               int sh, int sw, int dh, int dw, float* im, void* stream);
/* N-D (1..10 spatial axes): im2col_nd_gpu / col2im_nd_gpu (im2col.cu:165-253, 443-530).
 * Shape arrays are HOST int arrays: im_shape [C, d0..], col_shape [C*prod(k), o0..].   */
int b2c_im2col_nd(const float* im, int num_axes, const int* im_shape, const int* col_shape,
                  const int* kernel, const int* pad, const int* stride, const int* dilation,
                  float* col, void* stream);
int b2c_col2im_nd(const float* col, int num_axes, const int* im_shape, const int* col_shape,
                  const int* kernel, const int* pad, const int* stride, const int* dilation,
                  float* im, void* stream);

/* ---- BLAS-shaped entry points -----------------------------------------------------------
 * Row-major C[MxN] = alpha*op(A)*op(B) + beta*C with the reference's leading
 * dimensions (lda = transA ? M : K, ldb = transB ? K : N, ldc = N).
 * Replaces caffe_gpu_gemm<float> -> cublasSgemm (src/caffe/util/math_functions.cu:11-26). */
int b2c_sgemm(int transA, int transB, int M, int N, int K, float alpha, const float* A,
              const float* B, float beta, float* C, void* stream);
/* The same product with caller-provided scratch (b2c_sgemm_workspace_bytes(...) bytes, 16-byte aligned; may be null / short: then
 * as b2c_sgemm).  With it the NoTrans x Trans tensor-core path splits the K loop over one wave of CTAs and reduces the partial
 * tiles in a fixed order (deterministic) -- InnerProduct forward at small batch is otherwise one CTA per 128 x 128 output tile. */
/* 1 when b2c_sgemm_ex with its workspace would run this product (alpha = 1, beta in {0, 1}, 16-byte aligned operands) on the
 * tensor cores: NoTrans x Trans, K >= 64, K % 4 == 0, default math = fp32-equivalent.  Callers that can choose their operand layout
 * (InnerProductLayer::Backward_gpu with transposed copies) ask before preparing them.  Without a usable workspace a product whose
 * K loop the planner would split runs unsplit, and on the FFMA kernel once K exceeds 256 blocks of 64 (one fp32 accumulator
 * chain that long is not fp32-accurate); b2c_debug_sgemm_plan tells. */
int b2c_sgemm_tc_supported(int transA, int transB, int M, int N, int K);
size_t b2c_sgemm_workspace_bytes(int transA, int transB, int M, int N, int K);
/* dst[c][r] = src[r][c] (rows x cols -> cols x rows), src != dst. */
int b2c_transpose(int rows, int cols, const float* src, float* dst, void* stream);
int b2c_sgemm_ex(int transA, int transB, int M, int N, int K, float alpha, const float* A, const float* B, float beta, float* C,
                 void* workspace, size_t workspace_bytes, void* stream);
/* The kernel b2c_sgemm_ex runs (b2c_debug_sgemm_plan out[0]). */
typedef enum {
  B2C_SGEMM_ROUTE_FFMA = 0,   /* exact-fp32 FFMA kernel: one sequential fmaf chain over k per element, 64 x 64 tiles, K steps of 16 */
  B2C_SGEMM_ROUTE_TC = 1      /* NoTrans x Trans on the staged bf16x3 tensor-core kernel: 128 x cols tiles, K blocks of 64        */
} b2c_sgemm_route;
/* Which kernel b2c_sgemm_ex takes for these arguments and its plan; A, B and workspace are only tested for alignment, never
 * dereferenced.  out[0] route (b2c_sgemm_route), [1] tile columns (64 or 128), [2] K blocks in all (64 wide on the tensor cores, 16
 * on the FFMA kernel), [3] split count of the K loop, [4] K blocks per split (1 split after a null, short or misaligned workspace),
 * [5] M tiles, [6] N tiles.  Reads the default math and algo like the entry point.  Needs n >= 7.  Pure host computation: splits
 * follow the current device's SM count (132 without a device). */
int b2c_debug_sgemm_plan(int transA, int transB, int M, int N, int K, float alpha, float beta, const void* A, const void* B,
                         const void* workspace, size_t workspace_bytes, int* out, int n);
/* y = alpha*op(A)*x + beta*y, A row-major MxN.
 * Replaces caffe_gpu_gemv<float> -> cublasSgemv (math_functions.cu:73-82).               */
int b2c_sgemv(int transA, int M, int N, float alpha, const float* A, const float* x,
              float beta, float* y, void* stream);

/* ---- the non-convolution layers on ResNet-50's training path (SURVEY.md 8(f) rank 2) ----------------------------
 * fp32 NCHW, asynchronous on `stream`.  Each keeps the semantics of the reference layer's CPU code.                */
/* ReLULayer::Forward/Backward (src/caffe/layers/relu_layer.cpp:10-41); may run in place (y == x).  Any 4-byte-aligned
 * pointers: float4 passes when all of them are 16-byte aligned, one float at a time otherwise (same values either way).     */
int b2c_relu_forward(size_t n, const float* x, float* y, float negative_slope, void* stream);
int b2c_relu_backward(size_t n, const float* dy, const float* x, float* dx, float negative_slope, void* stream);
/* BatchNormLayer (NVCaffe, src/caffe/layers/batch_norm_layer.cpp:140-300), TRAIN phase.  x,y,xnorm: [N,C,S].
 * gamma/beta null <=> scale_bias false.  running_var stores (variance + eps) like the reference's blobs_[1].
 * backward OVERWRITES dgamma/dbeta (also the reduction scratch when gamma is null) and dx.                          */
int b2c_bn_forward_train(int N, int C, int S, const float* x, const float* gamma, const float* beta, float eps,
                         float moving_average_fraction, int first_iteration, float* running_mean, float* running_var,
                         float* save_mean, float* save_invstd, float* xnorm, float* y, void* stream);
int b2c_bn_backward(int N, int C, int S, const float* dy, const float* xnorm, const float* gamma, const float* save_invstd,
                    float* dgamma, float* dbeta, float* dx, void* stream);
/* PoolingLayer (src/caffe/layers/pooling_layer.cpp:129-318): method 0 = MAX (mask = argmax index inside the H*W
 * plane, first maximum), 1 = AVE.  NC = N*C planes; output extent is the reference's ceil mode.  dx overwritten.
 * Refused like PoolingLayer::LayerSetUp / Reshape's CHECKs: kernel and stride >= 1, 0 <= pad < kernel, H, W >= 1,
 * Ho, Wo >= 1.  The kernel chosen is b2c_debug_pool_plan's.                                                         */
/* DataTransformer::Transform on a batch of uint8 datums (data_transformer.cpp:178-312): crop window and mirror flag per image
 * (device arrays of N), per-channel mean_values[C] or a per-pixel mean_image[C*Hd*Wd] in datum coordinates (or neither), scale.
 * out[n][c][h][w] = (datum[n][c][h_off[n]+h][w_off[n] + (mirror[n] ? crop_w-1-w : w)] - mean) * scale. */
int b2c_transform_u8(const unsigned char* src, int N, int C, int Hd, int Wd, int crop_h, int crop_w, const int* h_off,
                     const int* w_off, const unsigned char* mirror, const float* mean_values, const float* mean_image,
                     float scale, float* dst, void* stream);

/* Fused forms of the BatchNorm -> ReLU and Eltwise(SUM) -> ReLU chains (csrc/layers_fused.cu): bit-identical to the unfused
 * layer sequence, one HBM pass less each way; x_norm is recomputed in backward from the layer input and the saved statistics. */
int b2c_bn_forward_train_fused(int N, int C, int S, const float* x, const float* gamma, const float* beta, float eps,
                               float moving_average_fraction, int first_iteration, float* running_mean, float* running_var,
                               float* save_mean, float* save_invstd, float* y, int relu, void* stream);
int b2c_bn_backward_fused(int N, int C, int S, const float* dy, const float* x, const float* save_mean, const float* save_invstd,
                          const float* gamma, const float* beta, float* dgamma, float* dbeta, float* dx, int relu, void* stream);
/* The residual tail of a ResNet block -- BatchNorm -> Eltwise(SUM, 2 bottoms) -> in-place ReLU (batch_norm_layer.cpp,
 * eltwise_layer.cpp:47-60,100-140, relu_layer.cpp) -- as one launch each way.  Forward: y = [max(0, .)] (BatchNorm(x) + residual).
 * Backward: d_sum / y_sum are the diff and the post-ReLU data of the sum's top; dx = BatchNorm::Backward of d_sum * (y_sum > 0), and
 * that masked gradient is also written to d_residual (the sum's other bottom) unless it is null.  d_sum2 (may be null) is a second
 * part of the sum's top diff -- the shadow diff of a blob with two consumers -- added to d_sum on the fly (SplitLayer::Backward's
 * accumulation without its pass over memory).  Same bits as the layers run one by one. */
int b2c_bn_forward_train_fused_res(int N, int C, int S, const float* x, const float* gamma, const float* beta, float eps,
                                   float moving_average_fraction, int first_iteration, float* running_mean, float* running_var,
                                   float* save_mean, float* save_invstd, const float* residual, float* y, int relu, void* stream);
int b2c_bn_backward_fused_res(int N, int C, int S, const float* d_sum, const float* d_sum2, const float* y_sum, const float* x,
                              const float* save_mean, const float* save_invstd, const float* gamma, const float* beta,
                              float* dgamma, float* dbeta, float* dx, float* d_residual, void* stream);
/* BatchNormLayer TEST phase (batch_norm_layer.cu:22-34 and stage 2, :80-90), one elementwise launch (csrc/bn_infer.cu):
 *   y = [ReLU]( bn_y(bn_xn(x, running_mean[c], invstd[c]), gamma[c], beta[c]) [+ residual] ),  invstd[c] = 1 / sqrtf(running_var[c] + eps).
 * DOUBLE eps: running_var already holds variance + eps (the TRAIN kernels fold eps in before the running average, as the reference's
 * CAFFE engine does, batch_norm_layer.cpp:183-186), and the TEST branch adds eps again (powx(var + eps, -0.5)); this reproduces both.
 * gamma/beta null <=> scale_bias false.  residual (may be null): the other bottom of an Eltwise SUM fed by this layer.  relu: the
 * in-place ReLU after the layer (or after the sum).  Bit-identical to this entry point without relu / residual followed by
 * b2c_relu_forward (slope 0), b2c_add or b2c_add_relu.  y may alias x.  Writes y only; the running statistics are read-only. */
int b2c_bn_forward_inference(int N, int C, int S, const float* x, const float* gamma, const float* beta, float eps,
                             const float* running_mean, const float* running_var, const float* residual, float* y, int relu,
                             void* stream);
/* AccuracyLayer::Forward (accuracy_layer.cpp:44-100), labels as float class ids, ties ranked like the reference's
 * std::greater<pair<score, index>>; `scratch`: 4 bytes of device memory. */
int b2c_accuracy(int N, int C, int top_k, const float* scores, const float* labels, float* accuracy, void* scratch, void* stream);
int b2c_add_relu(size_t n, const float* a, const float* b, float* y, void* stream);
int b2c_relu_backward2(size_t n, const float* dy, const float* y, float* dx_a, float* dx_b, void* stream);
int b2c_pool_forward(int method, int NC, int H, int W, int kh, int kw, int sh, int sw, int ph, int pw, const float* x,
                     float* y, int* mask, void* stream);
int b2c_pool_backward(int method, int NC, int H, int W, int kh, int kw, int sh, int sw, int ph, int pw, const float* dy,
                      const int* mask, float* dx, void* stream);
/* y = a + b: EltwiseLayer SUM forward (eltwise_layer.cpp) and the diff accumulation of SplitLayer::Backward.  Alignment
 * as b2c_relu_forward; may run in place (y == a or y == b).                                                         */
int b2c_add(size_t n, const float* a, const float* b, float* y, void* stream);
/* SoftmaxWithLossLayer (src/caffe/layers/softmax_loss_layer.cpp:96-160), VALID normalisation, labels as float ids:
 * forward writes prob [N,C] and *loss (device scalar); backward writes dx = (prob - onehot) * loss_weight / N.       */
int b2c_softmax_loss_forward(int N, int C, const float* logits, const float* labels, float* prob, float* loss, void* stream);
int b2c_softmax_loss_backward(int N, int C, const float* prob, const float* labels, float loss_weight, float* dx, void* stream);
/* SoftmaxWithLossLayer over an [outer, C, inner] view (softmax_loss_layer.cpp:44-160): one softmax over C per (outer, inner)
 * pixel, LossParameter.ignore_label and .normalization (caffe.proto NormalizationMode).  labels[outer * inner] are float class ids
 * read as (int).  A pixel whose label equals ignore_label (has_ignore != 0) adds no term and is not counted.
 * Forward: prob as b2c_softmax_forward on the same logits, bit for bit; *loss (device) = (float)S / norm with S = the sum over the
 * counted pixels of -log(max(prob[label], FLT_MIN)), taken in double in a fixed order: pixels in chunks of 1024, one double per
 * chunk (its threads' four-pixel sums in a fixed tree), the chunks in index order.  The bits depend on the shape and the data
 * only, never on the device or the alignment.  norm (get_normalizer, floored at 1): FULL outer * inner; VALID the counted
 * pixels when has_ignore, else outer * inner; BATCH_SIZE outer; NONE 1.  *normalizer (device float) receives it for the backward;
 * nothing is read back to the host.  workspace: b2c_softmax_loss_workspace bytes of device memory, 16-byte aligned.
 * Backward: dx = (prob - onehot) * s with s = loss_weight / *normalizer rounded once; every channel of an ignored pixel is 0.
 * A label that is not ignored and lies outside [0, C): the forward reads class min(max(label, 0), C - 1) and the backward
 * subtracts nothing, so no access leaves the tensors (the reference DCHECKs the range).
 * Routes (b2c_debug_softmax_loss_plan): inner == 1 the row kernel of b2c_softmax_loss_forward, then a masked pass over the rows;
 * inner > 1 one fused pass, a thread per pixel column, four columns as float4 when inner % 4 == 0 and logits, prob are 16-byte
 * aligned.  The backward takes float4 along inner when inner % 4 == 0 and prob, labels, dx are aligned.
 * outer, C, inner >= 1 and outer * C * inner < 2^62, else B2C_ERR_INVALID. */
typedef enum {
  B2C_LOSS_NORM_FULL = 0, B2C_LOSS_NORM_VALID = 1, B2C_LOSS_NORM_BATCH_SIZE = 2, B2C_LOSS_NORM_NONE = 3
} b2c_loss_normalization;
typedef enum { B2C_SOFTMAX_LOSS_ROUTE_ROW = 0, B2C_SOFTMAX_LOSS_ROUTE_COLUMN = 1, B2C_SOFTMAX_LOSS_ROUTE_COLUMN_F4 = 2 } b2c_softmax_loss_route;
int b2c_softmax_loss_workspace(int outer, int C, int inner, size_t* bytes);
int b2c_softmax_loss_forward_ex(int outer, int C, int inner, const float* logits, const float* labels, int has_ignore, int ignore_label,
                                int norm_mode, float* prob, float* loss, float* normalizer, void* workspace, void* stream);
int b2c_softmax_loss_backward_ex(int outer, int C, int inner, const float* prob, const float* labels, int has_ignore, int ignore_label,
                                 const float* normalizer, float loss_weight, float* dx, void* stream);
/* The forward route b2c_softmax_loss_forward_ex takes with logits and prob at these addresses (only tested for alignment):
 * out[0] route (b2c_softmax_loss_route), [1] pixels per chunk, [2] chunks (the workspace's slots), [3] workspace bytes.  Needs
 * n >= 4.  Refuses what the entry points refuse.  Pure host computation. */
int b2c_debug_softmax_loss_plan(int outer, int C, int inner, const void* logits, const void* prob, int* out, int n);
/* AccuracyLayer over an [outer, C, inner] view (accuracy_layer.cpp:21-101) with AccuracyParameter.ignore_label and the per-class
 * top.  A pixel is a hit when fewer than top_k classes rank above its label in the order of std::greater<pair<score, index>> (on
 * equal scores the larger index ranks first).  Pixels whose label is ignored are skipped; a label outside [0, C) that is not
 * ignored is counted as a miss and touches no per-class counter.  *accuracy = hits / counted pixels (NaN when none is counted,
 * as the reference's accuracy / count); per_class[c] (may be null) = hits_c / pixels labelled c, or 0 when none is.  Counts are
 * integers: the result is exact and the same on every call.  scratch: 8 + 8 * C bytes of device memory (8 without per_class).
 * top_k in [1, C]. */
int b2c_accuracy_ex(int outer, int C, int inner, int top_k, const float* scores, const float* labels, int has_ignore, int ignore_label,
                    float* accuracy, float* per_class, void* scratch, void* stream);
/* SoftmaxLayer (src/caffe/layers/softmax_layer.cpp / .cu): softmax over the C axis of an [outer, C, inner] view.  inner == 1
 * runs b2c_softmax_loss_forward's row kernel, so y is bit-identical to its prob.  Backward: dx = (dy - sum_c dy * y) * y.  Both
 * may run in place (y == x; dx == dy).  Alignment as b2c_relu_forward (the float4 path takes four columns when inner % 4 == 0). */
int b2c_softmax_forward(int outer, int C, int inner, const float* x, float* y, void* stream);
int b2c_softmax_backward(int outer, int C, int inner, const float* y, const float* dy, float* dx, void* stream);
/* SigmoidLayer (src/caffe/layers/sigmoid_layer.cu:9-13): y = 1 / (1 + exp(-x)); backward dx = dy * y * (1 - y).  Both may
 * run in place.  Alignment as b2c_relu_forward.                                                                                */
int b2c_sigmoid_forward(size_t n, const float* x, float* y, void* stream);
int b2c_sigmoid_backward(size_t n, const float* y, const float* dy, float* dx, void* stream);
/* The elementwise NeuronLayers (src/caffe/layers/{elu,power,absval,bnll,exp,log,threshold}_layer): one kernel template over
 * the per-element rules, each the reference's own expression in its operation order and types, with no contraction into FMA.
 * p0..p2 per kind -- the derived constants as the layer's LayerSetUp computes them in float on the host:
 *   ELU        p0 alpha.                                  dx = x > 0 ? dy : dy * (y + alpha); reads x, y
 *   POWER      p0 power, p1 scale, p2 shift; diff_scale = power * scale rounded to float in the kernel, as LayerSetUp does.
 *              Forward: diff_scale == 0 gives the constant (power == 0 ? 1 : powf(shift, power)), else powf(shift + scale x, power)
 *              with the scale / shift / power steps skipped where they are 1 / 0 / 1.  Backward (power_layer.cu):
 *              diff_scale == 0 or power == 1: dx = dy * diff_scale (reads neither x nor y); power == 2: dy * (diff_scale * scale * x
 *              [+ diff_scale * shift]) (reads x); shift == 0: dy * (power * (y / x)); else dy * (diff_scale * (y / (shift + scale x)))
 *              (both read x and y)
 *   ABSVAL     no parameter.                              dx = sign(x) * dy; reads x
 *   BNLL       no parameter; exp(min(x, 50)) in the backward.   reads x
 *   EXP        p0 inner_scale = log(base) * scale, p1 outer_scale = base^shift.   dx = inner_scale * (y * dy); reads y
 *   LOG        p0 scale, p1 shift, p2 base_scale = 1 / log(base) (forward) or backward_num_scale = scale / log(base) (backward).
 *              dx = dy * (p2 * powf(shift + scale x, -1)); reads x
 *   THRESHOLD  p0 threshold; y = x > threshold ? 1 : 0.  Forward only: b2c_neuron_backward refuses it.
 * expf / logf / powf, built without fast-math.  Backward reads only the pointers its rule needs (listed above); the others may be
 * null.  Both directions may run in place (y == x; dx == dy): each element is read before the same thread writes it.  Alignment as
 * b2c_relu_forward: float4 when every pointer the call reads or writes is 16-byte aligned, one float at a time otherwise, the same
 * values either way.  Refuses (B2C_ERR_INVALID) an unknown kind and a null pointer the rule needs. */
typedef enum {
  B2C_NEURON_ELU = 0, B2C_NEURON_POWER = 1, B2C_NEURON_ABSVAL = 2, B2C_NEURON_BNLL = 3, B2C_NEURON_EXP = 4, B2C_NEURON_LOG = 5,
  B2C_NEURON_THRESHOLD = 6
} b2c_neuron_kind;
int b2c_neuron_forward(int kind, size_t n, const float* x, float* y, float p0, float p1, float p2, void* stream);
int b2c_neuron_backward(int kind, size_t n, const float* x, const float* y, const float* dy, float* dx, float p0, float p1, float p2,
                        void* stream);
/* PReLULayer (src/caffe/layers/prelu_layer.cu) over x [N, C, dim] (channels = shape(1), dim = count(2)); slope has C values, or
 * one when `shared` (channel_shared: every value uses slope[0]).
 * Forward: y = x > 0 ? x : x * slope[c].  y may be x.  x_keep (may be null; not x or y): the same pass also writes a copy of x
 * there -- what the backward of an in-place layer needs (the reference's caffe_copy into bottom_memory_).
 * Backward, one pass reading x and dy: dx = dy * ((x > 0) + (x <= 0) * slope[c]) when dx is not null (dx may be dy, not x); when
 * dslope is not null, dslope[c] += sum over the channel of dy * x * (x <= 0) -- ADDED, as Caffe accumulates parameter diffs.  The
 * sum is deterministic, with no float atomics: each thread adds a fixed stripe of the channel in fp32, the CTA a fixed tree of its
 * threads; with several CTAs per channel the last to arrive at the channel's counter sums their partials in double (fixed runs,
 * then a fixed tree) and rounds once.  The orders depend on the shape only, never on the device or the data: the same bits on
 * every call.  ws: b2c_prelu_workspace_bytes of device memory, 16-byte aligned (may be null when that is 0, or when dslope is
 * null), ZEROED BEFORE ITS FIRST USE: each call leaves its counters zero again, so a workspace is zeroed once, when it is
 * allocated, and nothing but the kernel runs on `stream`.  The workspace size depends on the shape only, not on the pointers'
 * alignment.  Both null dx and dslope: nothing is launched.
 * Float4 units when dim (C * dim when shared) % 4 == 0 and every tensor pointer is 16-byte aligned, else one float at a time.
 * Refuses (B2C_ERR_INVALID) N, C or dim < 1 and a channel of N * dim >= 2^31 values (N * C * dim when shared). */
int b2c_prelu_forward(int N, int C, int dim, int shared, const float* x, const float* slope, float* y, float* x_keep, void* stream);
int b2c_prelu_workspace_bytes(int N, int C, int dim, int shared, size_t* bytes);
int b2c_prelu_backward(int N, int C, int dim, int shared, const float* x, const float* dy, const float* slope, float* dx, float* dslope,
                       void* ws, size_t ws_bytes, void* stream);
/* The launch of a neuron call.  op 0 / 1: b2c_neuron_forward / _backward of `kind` over N values (C, dim, shared unused); op 2 / 3:
 * b2c_prelu_forward / _backward.  ptrs[nptrs] (nptrs <= 4): the call's tensors, only tested for 16-byte alignment, null entries
 * ignored (for PReLU the first three: x, y or dy, x_keep or dx).  out[0] 1 for float4 units, [1] CTAs, [2] threads per CTA,
 * [3] CTAs per channel (PReLU; 1 otherwise), [4] stripe: values per thread (PReLU; 0 otherwise), [5] channels of the reduction
 * (C, or 1 when shared), [6] workspace bytes (op 3; 0 otherwise).  Needs n >= 7.  Refuses what the entry points refuse about the
 * shape and kind.  Pure host computation, independent of the device for PReLU. */
int b2c_debug_neuron_plan(int op, int kind, int N, int C, int dim, int shared, const void* const* ptrs, int nptrs, int* out, int n);
/* SigmoidCrossEntropyLossLayer (src/caffe/layers/sigmoid_cross_entropy_loss_layer.cpp): *loss (device scalar) =
 * -sum_i [x (t - [x >= 0]) - log(1 + exp(x - 2 x [x >= 0]))] / N, one launch, the same bits on every call (fixed reduction
 * order for a given count and alignment); no sigmoid tensor is stored.  Backward: dx = (sigmoid(x) - t) * scale with
 * scale = loss_weight / N, where sigmoid(x) is THE SAME EXPRESSION as b2c_sigmoid_forward's: dx equals
 * (b2c_sigmoid_forward(x) - t) * scale bit for bit.  dx may be x.                                                              */
int b2c_sigmoid_ce_loss_forward(int N, size_t count, const float* x, const float* target, float* loss, void* stream);
int b2c_sigmoid_ce_loss_backward(size_t count, const float* x, const float* target, float scale, float* dx, void* stream);
/* EuclideanLossLayer (src/caffe/layers/euclidean_loss_layer.cu): diff = a - b (kept for backward), *loss = sum diff^2 / N / 2
 * (device scalar, same reduction as b2c_sigmoid_ce_loss_forward).  Backward, once per bottom that propagates: dx = alpha * diff
 * with alpha = +-loss_weight / N.  dx may be diff.                                                                             */
int b2c_euclidean_loss_forward(int N, size_t count, const float* a, const float* b, float* diff, float* loss, void* stream);
int b2c_euclidean_loss_backward(size_t count, const float* diff, float alpha, float* dx, void* stream);
/* L1LossLayer (NVCaffe's l1_loss_layer.cu:11-43): diff = a - b (kept for backward), *loss = float(sum |diff|) / N (device scalar,
 * the same deterministic reduction as b2c_euclidean_loss_forward: the same bits on every call).  Backward, once per bottom that
 * propagates: dx = alpha * sign(diff) with alpha = +-loss_weight / N and sign(0) = sign(NaN) = 0 (written as +0).  dx may be diff. */
int b2c_l1_loss_forward(int N, size_t count, const float* a, const float* b, float* diff, float* loss, void* stream);
int b2c_l1_loss_backward(size_t count, const float* diff, float alpha, float* dx, void* stream);
/* ---- DetectNetTransformationLayer (NVCaffe's src/caffe/layers/detectnet_transform_layer.{cpp,cu} and
 * src/caffe/util/detectnet_coverage_rectangular.cpp); GPU parity: tests/test_detectnet_transform_gpu.py.
 * One image's augmentation, the reference's AugmentSelection (include/caffe/layers/detectnet_transform_layer.hpp:29-45):
 * hue_rotation in degrees (applied when |h| > FLT_EPSILON), saturation factor (applied when < 1 - 1/255), flip, the scaled size
 * (scale_w x scale_h; scaling applies where it differs from the bottom's W x H), rotation in degrees (applied when
 * |r| > FLT_EPSILON) and the crop offset.  The entry points read an array of N of them in DEVICE memory and draw nothing. */
typedef struct {
  float hue_rotation, saturation;
  int flip, scale_w, scale_h;
  float rotation;
  int crop_x, crop_y;
} b2c_detectnet_aug;
/* DetectNetGroundTruthParameter (caffe.proto), RECTANGULAR coverage.  gridbox_type 0 GRIDBOX_MAX, 1 GRIDBOX_MIN.  class_src[m] ->
 * class_dst[m] for m < n_classes is the object_class map (a later entry with the same src wins); n_classes 0 is the reference's
 * default {1 -> 0}. */
#define B2C_DETECTNET_MAX_CLASSES 32
typedef struct {
  int image_size_x, image_size_y, stride, gridbox_type, max_cvg_len, min_cvg_len, obj_norm, crop_bboxes;
  float scale_cvg;
  int n_classes;
  int class_src[B2C_DETECTNET_MAX_CLASSES], class_dst[B2C_DETECTNET_MAX_CLASSES];
} b2c_detectnet_gt;
/* Image path (detectnet_transform_layer.cu:121-346, replacing its three kernels and their cudaStreamSynchronize): bottom
 * [N, 3, H, W] of 0-255 values -> top [N, 3, OH, OW].  Per pixel: RGB -> HSV -> RGB with the hue rotation and desaturation, then
 * the mean (mean_kind 0 none, 1 mean_value[3]: the transform_param values as written, host floats, of which the kernel subtracts
 * float(float(m / 255) * 255) as the reference's GPU path does; 2 mean_image [3, H, W] device, subtracted as given), into `workspace`
 * (b2c_detectnet_image_workspace_bytes); then per output pixel: crop offset, rotation, scale and flip in the reference's order and
 * its bicubic (1-pixel replicated border, 0 beyond).  Float coordinates and HSV, the cubic in double, no FMA contraction: without
 * rotation the result is bit-exact against a float32 / double restatement.  One departure: hue is wrapped into [-60, 360) by whole
 * turns, for any hue_rotation, before the HSV sector is chosen (the reference never wraps it; DESIGN §4).  Two launches.  Refuses (B2C_ERR_INVALID) non-positive
 * sizes, null pointers and a small workspace. */
size_t b2c_detectnet_image_workspace_bytes(int N, int H, int W);
int b2c_detectnet_image(int N, int H, int W, int OH, int OW, const float* bottom, const b2c_detectnet_aug* aug, int mean_kind,
                        const float* mean_image, const float* mean_value, float* workspace, size_t workspace_bytes, float* top,
                        void* stream);
/* Label path (transform_label_cpu, detectnet_transform_layer.cpp:450-615, and CoverageGenerator::generate,
 * detectnet_coverage_rectangular.cpp:292-360, which the reference runs on the host): labels [N, 1, rows, 16], the DIGITS layout
 * (row 0 [num_boxes, 16, ...], then one BboxLabel_ per row), of images H x W -> top [N, C, GH, GW] (b2c_detectnet_label_shape):
 * foreground, the box corners relative to the cell, 1 / width, 1 / height, obj_norm, then one coverage channel per class.  One CTA
 * per image, the boxes in shared memory; each cell takes the last box in list order that covers it, which is what the reference's
 * in-order overwrite leaves (no atomics, the same bits on every call).  A malformed header is never read as boxes: the image's
 * labels are zeroed and *status (device int, zeroed by the caller; sticky) gains B2C_DETECTNET_BAD_BOX_LENGTH (the reference's
 * CHECK bboxLen == 16) or B2C_DETECTNET_TOO_MANY_BOXES (CHECK numOfBbox <= height; boxes are the rows after the header, so
 * num_boxes == rows is refused too).  rows - 1 <= 768.  Refuses (B2C_ERR_INVALID) bad shapes and parameters. */
#define B2C_DETECTNET_BAD_BOX_LENGTH 1
#define B2C_DETECTNET_TOO_MANY_BOXES 2
int b2c_detectnet_label_shape(const b2c_detectnet_gt* gt, int* channels, int* grid_h, int* grid_w);
int b2c_detectnet_labels(int N, int rows, int H, int W, const float* labels, const b2c_detectnet_aug* aug, const b2c_detectnet_gt* gt,
                         float* top, int* status, void* stream);
/* The launches of a DetectNet call.  op 0 (image; gt and rows unused): out[0] launches (2), [1] colour CTAs, [2] sampling CTAs,
 * [3] threads per CTA, [4] workspace MiB, [5] workspace bytes beyond them.  op 1 (labels; OH, OW unused): [0] CTAs (N), [1] threads,
 * [2] shared-memory bytes, [3] channels, [4] GH, [5] GW.  Needs n >= 6.  Pure host computation. */
int b2c_debug_detectnet_plan(int op, int N, int H, int W, int OH, int OW, int rows, const b2c_detectnet_gt* gt, int* out, int n);
/* ContrastiveLossLayer (src/caffe/layers/contrastive_loss_layer.cpp), N pairs of C-channel features a, b [N, C] and labels y [N]
 * read as (int)y (0.7 is dissimilar, -1 similar).  Forward, one launch: diff = a - b [N, C] (kept for backward), dist_sq [N], and
 * *loss (device scalar) = sum_n (y_n ? d2_n : max(margin - sqrt(d2_n), 0)^2) / N / 2; legacy != 0 takes max(margin - d2_n, 0) as
 * the dissimilar term.  Rounding: dist_sq[n] = float( sum_c float(diff^2) ), each square rounded to float and the sum over the
 * channels taken in double, then rounded once; every term is formed in float from that dist_sq and the terms are summed in
 * double over the pairs with b2c_euclidean_loss_forward's cluster reduction (no atomics: the same bits on every call).
 * Backward, one elementwise launch, alpha = loss_weight / N: similar pairs da = alpha * diff; dissimilar pairs with
 * mdist = margin - sqrt(d2) > 0: da = (-alpha * mdist / (sqrt(d2) + 1e-4)) * diff (the 1e-4 is the reference's), else 0.  Legacy:
 * da = -alpha * diff where margin - d2 > 0, else 0 -- the reference's Backward_cpu.  Its .cu kernel writes the constant -alpha
 * with no diff factor there, which is not the derivative of the loss it computes; this follows the CPU form.  db (may be null)
 * = -da bit for bit, except that both are +0 where the hinge zeroes a pair (as the reference's caffe_set(0)).  float4 path when diff, da and db are 16-byte aligned and C % 4 == 0, else one float at a
 * time.  N >= 1 and C >= 1, else B2C_ERR_INVALID.                                                                           */
int b2c_contrastive_loss_forward(int N, int C, const float* a, const float* b, const float* y, float margin, int legacy, float* diff,
                                 float* dist_sq, float* loss, void* stream);
int b2c_contrastive_loss_backward(int N, int C, const float* diff, const float* dist_sq, const float* y, float margin, int legacy,
                                  float alpha, float* da, float* db, void* stream);
/* y[n][o][p] += bias[o];  db[o] += sum_{n,p} dy[n][o][p]  (InnerProduct bias with P = 1; conv bias with P = Ho*Wo). */
int b2c_bias_forward(int N, int O, int P, const float* bias, float* y, void* stream);
int b2c_bias_backward(int N, int O, int P, const float* dy, float* db, void* stream);
/* ---- layers the AlexNet / GoogLeNet / VGG-16 BASELINE nets add (SURVEY 8f rank 2, second half);
 * GPU parity: tests/test_layers_extra_gpu.py.
 * LRNLayer ACROSS_CHANNELS (src/caffe/layers/lrn_layer.cpp CrossChannelForward_cpu / CrossChannelBackward_cpu):
 * scale = k + alpha/size * sum_{window} x^2, y = x * scale^-beta; x,y,scale,dy,dx: [N,C,S].                          */
int b2c_lrn_forward(int N, int C, int S, int local_size, float alpha, float beta, float k, const float* x, float* scale,
                    float* y, void* stream);
int b2c_lrn_backward(int N, int C, int S, int local_size, float alpha, float beta, const float* x, const float* y,
                     const float* scale, const float* dy, float* dx, void* stream);
/* DropoutLayer TRAIN (src/caffe/layers/dropout_layer.cpp): mask[i] = keep ? 1/(1-ratio) : 0 with
 * keep = (splitmix64(seed + offset + i) >> 40) >= ratio * 2^24  (counter based: reproducible, no state);
 * forward y = x * mask and backward dx = dy * mask are b2c_mul.                                                        */
int b2c_dropout_mask(size_t n, float ratio, unsigned long long seed, unsigned long long offset, float* mask, void* stream);
int b2c_mul(size_t n, const float* a, const float* b, float* y, void* stream);

/* ---- fused SGD-momentum update -----------------------------------------------------------
 * h = momentum*h + local_rate*(grad_scale*g + local_decay*reg(w)); w -= h;
 * g = clear_grads ? 0 : h.   reg(w) = w (l2 != 0) or sign(w).
 * Replaces SGDRegUpdateAllAndClear + its launcher (src/caffe/solvers/sgd_solver.cu:9-72),
 * with Net::ReduceBucket's 1/solver_count scal (net.cpp:910), the 1/global_grad_scale
 * scal (net.cpp:815-817) and SGDSolver::Normalize's 1/iter_size (sgd_solver.cpp:152-158)
 * folded into grad_scale.                                                                 */
int b2c_sgd_update(size_t n, float* g, float* w, float* h, float momentum, float local_rate,
                   float local_decay, int l2, float grad_scale, int clear_grads, void* stream);
/* Multi-tensor form over a contiguous arena (Net::InitializeLearnableDiffSpace,
 * net.cpp:1350-1373): nseg segments, segment s covers elements [offset[s], offset[s]+count[s])
 * of g, w and h (same offsets in all three arenas) with its own local_rate / local_decay
 * (lr_mult / decay_mult, sgd_solver.cpp:208-210,254-259).  The four arrays are HOST arrays.
 * One launch replaces one SGDRegUpdateAllAndClear launch per learnable blob.               */
int b2c_sgd_update_arena(int nseg, const size_t* offset, const size_t* count,
                         const float* local_rate, const float* local_decay,
                         float* g, float* w, float* h, float momentum, int l2,
                         float grad_scale, int clear_grads, void* stream);

/* ---- the other solvers, fused over the arena ------------------------------------------------
 * Same segments, host arrays and folded grad_scale as b2c_sgd_update_arena; per element, with
 * gr = grad_scale*g + local_decay*reg(w), lr = local_rate[s]:
 *   SGD       h = momentum*h + lr*gr; u = h                    (b2c_sgd_update_arena, bit for bit)
 *   NESTEROV  h' = momentum*h + lr*gr; u = (1+momentum)*h' - momentum*h
 *             replaces NesterovRegUpdateAllAndClear (src/caffe/solvers/nesterov_solver.cu:12-25)
 *   ADAGRAD   h += gr^2; u = lr*gr / (sqrt(h) + max(delta, 1e-3))
 *             replaces AdaGradRegUpdateAllAndClear (adagrad_solver.cu:11-23, delta clamp adagrad_solver.cpp:22)
 *   RMSPROP   h = rms_decay*h + (1-rms_decay)*gr^2; u = lr*gr / (sqrt(h) + max(delta, 1e-4))
 *             replaces RMSPropRegUpdateAllAndClear (rmsprop_solver.cu:12-23, rmsprop_solver.cpp:25)
 *   ADADELTA  h = momentum*h + (1-momentum)*gr^2; gr *= sqrt((h2+d)/(h+d)); h2 = momentum*h2 + (1-momentum)*gr^2;
 *             u = lr*gr, d = max(delta, 1e-3)
 *             replaces AdaDeltaRegUpdateAllAndClear (adadelta_solver.cu:12-26, adadelta_solver.cpp:36)
 *   ADAM      h = beta1*h + (1-beta1)*gr; h2 = beta2*h2 + (1-beta2)*gr^2; u = lr*h / (sqrt(h2) + max(delta, 1e-4))
 *             replaces AdamRegUpdateAllAndClear (adam_solver.cu:11-24).  The bias correction
 *             sqrt(1-beta2^t)/(1-beta1^t) is NOT applied here: fold it into local_rate (adam_solver.cpp:42-43).
 * then w -= u; g = clear_grads ? 0 : u.  h2 (same offsets as h) is read only by ADADELTA and ADAM and may be NULL
 * otherwise.  sqrt and division are IEEE-rounded.  Fields of b2c_solver_hparams a kind does not name are ignored. */
enum b2c_solver_kind {
  B2C_SOLVER_SGD = 0, B2C_SOLVER_NESTEROV = 1, B2C_SOLVER_ADAGRAD = 2, B2C_SOLVER_RMSPROP = 3,
  B2C_SOLVER_ADADELTA = 4, B2C_SOLVER_ADAM = 5
};
typedef struct b2c_solver_hparams {
  float momentum;   /* SGD, NESTEROV, ADADELTA */
  float delta;      /* ADAGRAD, RMSPROP, ADADELTA, ADAM (epsilon); clamped as above */
  float rms_decay;  /* RMSPROP */
  float beta1;      /* ADAM (SolverParameter.momentum) */
  float beta2;      /* ADAM (SolverParameter.momentum2) */
} b2c_solver_hparams;
int b2c_solver_update_arena(int kind, int nseg, const size_t* offset, const size_t* count,
                            const float* local_rate, const float* local_decay,
                            float* g, float* w, float* h, float* h2, b2c_solver_hparams hp,
                            int l2, float grad_scale, int clear_grads, void* stream);
/* The launches b2c_solver_update_arena (and, for kind SGD, b2c_sgd_update_arena) makes for this layout with the arenas at g, w,
 * h and h2 (only tested for alignment, never dereferenced).  Segments are taken in order, zero counts skipped, at most 96 per
 * launch, each segment owning ceil(count / 4096) blocks of 4096 elements.  *nlaunch = launches; launch_out[2i], [2i+1] = launch
 * i's segments and blocks (max_launches entries fit).  seg_out[6s..6s+5] for segment s: its launch (-1 when count is 0), 1 when
 * its blocks take the float4 path (g, w, h and h2 at one 4-byte-aligned offset within 16 bytes) else 0, its blocks, and summed
 * over them the leading scalars (0-3 per block), float4 units and trailing scalars.  Refuses (B2C_ERR_INVALID) what the entry
 * points refuse: an unknown kind, nseg < 0, a null g / w / h (h2 for ADADELTA and ADAM) or layout array, a count >= 2^32.
 * Pure host computation. */
int b2c_debug_solver_plan(int kind, int nseg, const size_t* offset, const size_t* count, const void* g, const void* w,
                          const void* h, const void* h2, int* launch_out, int max_launches, int* nlaunch, long long* seg_out);

/* ---- gradient clipping (SolverParameter.clip_gradients) -----------------------------------------------------------------
 * Replaces SGDSolver::ClipGradients (sgd_solver.cpp:111-128): there one float sumsq_diff per learnable blob (a cuBLAS sdot each),
 * summed on the host, then a cublasSscal per blob.  Here the squared L2 norm of the whole diff arena is accumulated in double,
 * bucket by bucket on the stream that reduces the gradients; one CTA turns it into a factor in device memory; the update reads
 * the factor.  The host reads nothing on the training path.  Partials depend only on each segment's address and count, so the
 * norm is the same whichever buckets carry the segments. */
#define B2C_SUMSQ_BLOCK_ELEMS 4096
/* sum(g^2) over segment s, one double per block of B2C_SUMSQ_BLOCK_ELEMS elements: block b of segment s (ceil(count[s] / 4096)
 * blocks) writes partials[slot[s] + b].  Within a block each of 256 threads sums its elements in order in double (the head
 * scalars that peel g to 16 bytes, its float4 units, the tail), then a shuffle tree per warp, then the eight warps in order.
 * Segments are taken as b2c_solver_update_arena takes them: in order, zero counts skipped, at most 96 per launch.  Refuses
 * (B2C_ERR_INVALID) nseg < 0, a null layout array, g or partials, a count >= 2^32; a refused call launches nothing. */
int b2c_arena_sumsq(int nseg, const size_t* offset, const size_t* count, const size_t* slot, const float* g, double* partials,
                    void* stream);
typedef struct b2c_clip_state {
  float norm;         /* the last iteration's L2 norm of the scaled gradient */
  float factor;       /* the last iteration's scale: clip / norm when norm > clip, else 1 */
  long long clipped;  /* iterations with norm > clip so far */
} b2c_clip_state;
/* One CTA: S = the sum of partials[0..nslots) (thread t sums the slots t mod 256 in order, then the fixed tree of
 * b2c_arena_sumsq); norm = (float)sqrt(s_n^2 * S) formed in double, s_n = 1/(solver_count * global_grad_scale), the scale the
 * net applies before ClipGradients (net.cpp:815-817,910); factor = norm > clip ? clip / norm : 1 in IEEE float, so a NaN norm
 * does not scale (sgd_solver.cpp:118-127).  Writes state->norm and ->factor and counts a clipped iteration in ->clipped, which
 * the caller zeroes once.  Refuses a null state, null partials with nslots > 0, clip < 0 or NaN, s_n not positive and finite. */
int b2c_clip_factor(const double* partials, size_t nslots, double s_n, float clip, b2c_clip_state* state, void* stream);
/* b2c_solver_update_arena with grad_scale replaced, once per thread, by the rounded product grad_scale * *factor (a device
 * address, normally &state->factor of b2c_clip_factor).  Weight decay is not scaled: Regularize follows ClipGradients
 * (sgd_solver.cpp:143-149).  A factor of 1 gives b2c_solver_update_arena's bits.  Refuses what b2c_solver_update_arena
 * refuses, and a null factor. */
int b2c_solver_update_arena_scaled(int kind, int nseg, const size_t* offset, const size_t* count,
                                   const float* local_rate, const float* local_decay,
                                   float* g, float* w, float* h, float* h2, b2c_solver_hparams hp,
                                   int l2, float grad_scale, const float* factor, int clear_grads, void* stream);
/* The launches b2c_arena_sumsq makes for this layout with the diff arena at g (only tested for alignment).  *nlaunch,
 * launch_out as b2c_debug_solver_plan.  seg_out[7s..7s+6] for segment s: its launch (-1 when count is 0), 1 when its blocks take
 * the float4 path, its blocks, its first slot, and summed over its blocks the head scalars, float4 units and tail scalars.
 * *npartials = max(slot[s] + blocks) over the segments: the partials a workspace needs.  Refuses what b2c_arena_sumsq refuses.
 * Pure host computation. */
int b2c_debug_sumsq_plan(int nseg, const size_t* offset, const size_t* count, const size_t* slot, const void* g, int* launch_out,
                         int max_launches, int* nlaunch, long long* seg_out, long long* npartials);

/* ---- gradient exchange ---------------------------------------------------------------------
 * Replaces P2PManager/P2PSync's NCCL use (src/caffe/parallel.cpp:36-87,145-253) and the MPI
 * bootstrap (src/caffe/clusters.cpp:8-16; parallel.cpp:42-45,163-172).  One communicator per
 * process (one process per GPU).  The 128-byte id is produced on rank 0 and carried to the
 * other ranks by the caller (MPI_Bcast in the reference; any byte transport here).           */
/* Debugging aid for the mbarrier-synchronised kernels: every wait is bounded (~1 s); a timeout records
 * {block, thread, barrier, parity} and kills the kernel with a trap.  b2c_debug_mbar_set_trap(0) makes timeouts non-fatal so
 * that a deadlocked kernel drains; b2c_debug_mbar_timeouts fills four 128-word blocks (gather fwd/dgrad, staged fwd/dgrad,
 * gather weight-gradient, staged weight-gradient kernels), each {count, -, -, -, records...}, clears them and returns the
 * total count (cap_words >= 512). */
int b2c_debug_mbar_timeouts(unsigned int* out, int cap_words);
int b2c_debug_mbar_set_trap(int on);

/* The kernel b2c_conv_backward_filter runs for a descriptor (b2c_debug_wgrad_plan out[0]). */
typedef enum {
  B2C_WGRAD_ROUTE_CAFFE = 0,             /* engine CAFFE: per-image im2col + b2c_sgemm                                   */
  B2C_WGRAD_ROUTE_SIMT = 1,              /* FFMA direct kernel                                                           */
  B2C_WGRAD_ROUTE_GATHER = 2,            /* implicit-GEMM gather kernel (3xTF32, or TF32 in that math mode)              */
  B2C_WGRAD_ROUTE_STAGED_3X3 = 3,        /* TMA-staged bf16x3 kernel, 3x3 / pad 1: 8 channels x 9 taps per tile          */
  B2C_WGRAD_ROUTE_STAGED_3X3_PLANE = 4,  /* the same on 7x7 maps, one image per K block                                  */
  B2C_WGRAD_ROUTE_STAGED_1X1 = 5,        /* TMA-staged bf16x3 kernel, 1x1                                                */
  B2C_WGRAD_ROUTE_STAGED_1X1_PLANE = 6,  /* the same on 7x7 maps                                                         */
  B2C_WGRAD_ROUTE_TMA_1X1 = 7,           /* TMA-fed 3xTF32 1x1 kernel                                                    */
  B2C_WGRAD_ROUTE_COMPACT_STAGED = 8,    /* strided 1x1: X subsampled into the workspace, then the staged 1x1 kernel     */
  B2C_WGRAD_ROUTE_COMPACT_TMA = 9        /* strided 1x1: X subsampled, then the TMA-fed 1x1 kernel                       */
} b2c_wgrad_route;
/* Which weight-gradient route b2c_conv_backward_filter takes for this descriptor with 16-byte-aligned x / dy (and workspace),
 * and its split-K plan: out[0] route (b2c_wgrad_route), [1] splits, [2] K blocks per split, [3] K blocks in total,
 * [4] tile columns (channels x taps, or N_TILE), [5] K blocks per image (0 where the route has no per-image blocking).
 * For the compaction routes the plan is that of the dense 1x1 problem; the CAFFE and SIMT routes report zeros.
 * With n >= 7, out[6] is 1 where b2c_conv_backward_filter_split splits dY before the staged kernel, else 0.
 * Needs n >= 6.  Pure host computation: splits follow the current device's SM count (132 without a device). */
int b2c_debug_wgrad_plan(const b2c_conv_desc* d, int* out, int n);

/* The kernel b2c_conv_forward or b2c_conv_backward_data runs for a descriptor (b2c_debug_conv_plan out[0]). */
typedef enum {
  B2C_CONV_ROUTE_CAFFE = 0,           /* engine CAFFE: per-image im2col / col2im + b2c_sgemm                               */
  B2C_CONV_ROUTE_SIMT = 1,            /* FFMA direct kernels                                                               */
  B2C_CONV_ROUTE_GATHER = 2,          /* implicit-GEMM gather kernel: the forward, or the data gradient as a stride-1       */
                                      /* forward of dy with the flipped filter                                             */
  B2C_CONV_ROUTE_GATHER_SCATTER = 3,  /* the gather kernel on the data gradient of a strided 1x1 layer: rows scattered     */
                                      /* onto the stride grid of dx, the rest of dx zeroed                                  */
  B2C_CONV_ROUTE_STAGED = 4,          /* TMA-staged bf16x3 kernel (stride-1 "same" convolutions)                            */
  B2C_CONV_ROUTE_STAGED_PLANE = 5     /* the same in plane mode (7x7 maps: whole image planes staged)                       */
} b2c_conv_route;
/* Which route op B2C_OP_FORWARD or B2C_OP_BACKWARD_DATA takes for this descriptor with 16-byte-aligned activations (x and y,
 * or dy and dx), and its tile plan: out[0] route (b2c_conv_route), [1] N_TILE, [2] 128-row M tiles, [3] N tiles per group,
 * [4] tiles in all (x groups), [5] grid = min(tiles, SMs), [6] K blocks per tile, [7] variant: KMODE of the gather kernel
 * (1: K in chunks of 4 channels, 0: per-element K order), BWT of the staged kernel (staged pixels per channel: 49 in plane
 * mode, else 128, 160, 192 or 256).  The CAFFE and SIMT routes report zeros.  Needs n >= 8.  Pure host computation: the
 * grid follows the current device's SM count (132 without a device), N_TILE the B2C_NTILE switch as the launch does. */
int b2c_debug_conv_plan(const b2c_conv_desc* d, int op, int* out, int n);

/* The kernel b2c_pool_forward (dir 0) or b2c_pool_backward (dir 1) runs (b2c_debug_pool_plan out[0]). */
typedef enum {
  B2C_POOL_ROUTE_MAX_SCALAR = 0,    /* MAX forward, one thread per output                                                      */
  B2C_POOL_ROUTE_MAX_WINDOW = 1,    /* MAX forward, 3x3/2, 2x2/2 or 3x3/1 with Wo % Q == 0 (Q = 4 or 2) and y, mask aligned   */
                                    /* to 4Q bytes: one thread per Q outputs of a pooled row                                  */
  B2C_POOL_ROUTE_MAX_BWD_ROW = 2,   /* MAX backward, one 128-thread block per input row (several rows per block when W < 128) */
  B2C_POOL_ROUTE_MAX_BWD_QUAD = 3,  /* MAX backward, the same three windows with W % 4 == 0 and dx 16-byte aligned: one        */
                                    /* thread per four input columns                                                          */
  B2C_POOL_ROUTE_AVE = 4            /* AVE forward or backward, one thread per output element                                 */
} b2c_pool_route;
/* Which kernel the pooling call with these arguments takes; out_ptr is y (dir 0) or dx (dir 1), mask_ptr the MAX mask.  The
 * pointers are only tested for alignment, never dereferenced.  out[0] route (b2c_pool_route), [1] Ho, [2] Wo, [3] Q of the
 * window kernel (else 0), [4] input rows per block of the row kernel (else 0).  Needs n >= 5.  Refuses (B2C_ERR_INVALID) what
 * the entry points refuse: kernel or stride < 1, pad outside [0, kernel), H or W < 1, an empty output.  Pure host computation. */
int b2c_debug_pool_plan(int method, int dir, int NC, int H, int W, int kh, int kw, int sh, int sw, int ph, int pw,
                        const void* out_ptr, const void* mask_ptr, int* out, int n);

/* The launch a BatchNorm training call with these arguments takes.  dir 0 = forward, 1 = backward; form 0 = b2c_bn_forward_train /
 * b2c_bn_backward, 1 = b2c_bn_*_fused, 2 = b2c_bn_*_fused_res.  ptrs[nptrs] (nptrs <= 6) are the call's tensors -- forward: x, y,
 * and xnorm or residual; backward: dy, d_sum2, x or xnorm, dx, y_sum, d_residual -- only tested for 16-byte alignment, never
 * dereferenced; null entries are ignored.  out[0] launches (1: statistics / reduction and elementwise pass in one launch, 2: two),
 * [1] CTAs per channel (one cluster), [2] threads per CTA of the per-channel kernel, [3] what stays in shared memory between the
 * two phases (bit 0 = x, bit 1 = the masked gradient), [4] 1 when the parked streams come in by cp.async, [5] 1 for float4 units
 * (S % 4 == 0 and every pointer aligned), 0 for one float at a time.  Reads the B2C_BN_* switches like the entry points and the
 * current device's SM count (132 without a device).  Needs n >= 6.  Refuses (B2C_ERR_INVALID) what the entry points refuse about
 * the shape: N, C or S < 1, N * S >= 2^31, C > 65535.  Pure host computation. */
int b2c_debug_bn_plan(int dir, int form, int N, int C, int S, const void* const* ptrs, int nptrs, int* out, int n);

#define B2C_UNIQUE_ID_BYTES 128
int b2c_comm_get_unique_id(void* id_out /* B2C_UNIQUE_ID_BYTES */);
int b2c_comm_init(int nranks, int rank, const void* id, b2c_comm** out);
int b2c_comm_destroy(b2c_comm* c);
int b2c_comm_nranks(const b2c_comm* c);
/* ncclBcast of parameter data from `root` (P2PSync::on_start, parallel.cpp:208-227).        */
int b2c_comm_bcast(b2c_comm* c, float* buf, size_t count, int root, void* stream);
/* in-place ncclSum allreduce of a diff bucket (P2PSync::allreduce_bucket, parallel.cpp:245-253) */
int b2c_comm_allreduce_sum(b2c_comm* c, float* buf, size_t count, void* stream);
/* NVLS-capable buffers: ncclMemAlloc / ncclMemFree and ncclCommRegister (handles are released by b2c_comm_destroy).  An
 * in-place allreduce on a registered ncclMemAlloc buffer can be reduced inside the NVSwitch without NCCL's staging copies.
 * Environment: B2C_NCCL_MAX_CTAS / B2C_NCCL_MIN_CTAS set ncclConfig_t.maxCTAs / minCTAs of b2c_comm_init. */
int b2c_comm_mem_alloc(void** ptr, size_t bytes);
int b2c_comm_mem_free(void* ptr);
int b2c_comm_register(b2c_comm* c, void* buf, size_t bytes);

#ifdef __cplusplus
}
#endif
#endif  /* B2C_H_ */
