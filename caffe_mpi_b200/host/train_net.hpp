// train_net.hpp -- the non-convolution layers of the BASELINE nets as caffe::LayerBase subclasses, and TrainNet: a
// caffe::Net executor (forward / backward over the prototxt graph with automatic diff accumulation where a blob fans
// out, i.e. what insert_splits.cpp + SplitLayer do in the reference) wired to SGDSolver / ReduceScheduler / P2PSync.
//
// Reference map: src/caffe/layers/{relu,batch_norm,pooling,eltwise,inner_product,softmax_loss,split}_layer.cpp,
// Net::ForwardFromTo / BackwardFromToAu (src/caffe/net.cpp:669-751), Solver::Step (src/caffe/solver.cpp:187-353).
#pragma once
#include "b2caffe.hpp"
#include "prototxt.hpp"
#include "data_layer.hpp"

namespace caffe {

class ReLULayer : public LayerBase {
 public:
  using LayerBase::LayerBase;
  const char* type() const override { return "ReLU"; }
  void Reshape(const vector<Blob*>& b, const vector<Blob*>& t) override { if (t[0] != b[0]) t[0]->ReshapeLike(*b[0]); }
 protected:
  void Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) override;
  bool fused_away_ = false;
 public:
  float negative_slope() const { return layer_param_.relu_param.negative_slope; }   // relu_layer.cpp:13-16
  void set_fused_away(bool v) { fused_away_ = v; }   // the producing BatchNorm / Eltwise layer applies (and back-propagates) this ReLU
};

class BatchNormLayer : public LayerBase {      // NVCaffe BatchNorm with scale_bias (batch_norm_layer.cpp)
 public:
  // TEST phase: normalise with the running statistics (b2c_bn_forward_inference), never write blobs 0-4
  explicit BatchNormLayer(const LayerParameter& p)
      : LayerBase(p), scale_bias_(p.batch_norm_param.scale_bias), eps_(p.batch_norm_param.eps),
        maf_(p.batch_norm_param.moving_average_fraction) {}
  const char* type() const override { return "BatchNorm"; }
  void LayerSetUp(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Reshape(const vector<Blob*>& b, const vector<Blob*>& t) override;
 protected:
  void Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) override;
  bool scale_bias_;
  float eps_, maf_;
  bool fuse_relu_ = false;   // an in-place ReLU on the top blob is folded into this layer's kernels (TrainNet's fusion pass)
  bool recompute_ = false;   // do not store x_norm: backward recomputes it from the bottom blob (needs top != bottom)
  int iter_ = 0;
 public:
  void set_iter(int i) { iter_ = i; }
  void set_fusion(bool recompute_xnorm, bool fuse_relu) { recompute_ = recompute_xnorm; fuse_relu_ = fuse_relu; }
  bool recompute() const { return recompute_; }
  bool fuse_relu() const { return fuse_relu_; }
  // Residual tail: this layer also does the Eltwise SUM (+ in-place ReLU) that consumes its top.  Forward writes
  // max(0, BatchNorm(x) + other) into sum_top; backward takes sum_top's diff / data and also writes other's diff.
  void set_residual(Blob* other, Blob* sum_top, bool propagate_other) { res_other_ = other; res_sum_ = sum_top; res_prop_ = propagate_other; }
  Blob* residual_sum() const { return res_sum_; }
  // the sum's top has a second consumer whose bottom gradient lands in a shadow blob: this layer's backward reads both parts and
  // adds them on the fly instead of TrainNet running b2c_add over them first
  void set_sum_diff_part2(Blob* shadow) { res_part2_ = shadow; }
 protected:
  Blob* res_other_ = nullptr;
  Blob* res_sum_ = nullptr;
  Blob* res_part2_ = nullptr;
  bool res_prop_ = false;
  Blob xnorm_, save_mean_, save_invstd_, scratch_;
};

class PoolingLayer : public LayerBase {
 public:
  using LayerBase::LayerBase;
  const char* type() const override { return "Pooling"; }
  void Reshape(const vector<Blob*>& b, const vector<Blob*>& t) override;
 protected:
  void Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) override;
  PoolingParameter eff_;
  int* mask_ = nullptr;
  size_t mask_cap_ = 0;
 public:
  ~PoolingLayer() override;
};

class EltwiseLayer : public LayerBase {        // SUM with unit coefficients (the only use in the BASELINE nets)
 public:
  explicit EltwiseLayer(const LayerParameter& p) : LayerBase(p) {
    B2_CHECK(p.eltwise_param.operation == 1, "TrainNet: Eltwise PROD / MAX are not built (the BASELINE nets use SUM)");
    for (float c : p.eltwise_param.coeff) B2_CHECK(c == 1.f, "TrainNet: Eltwise SUM is built for unit coefficients only");
  }
  void set_fuse_relu(bool v) { fuse_relu_ = v; }
  bool fuse_relu() const { return fuse_relu_; }
  void set_fused_away(bool v) { fused_away_ = v; }     // the BatchNorm layer that produces one of the bottoms does the sum (TrainNet's fusion pass)
 protected:
  bool fuse_relu_ = false;
  bool fused_away_ = false;
 public:
  const char* type() const override { return "Eltwise"; }
  void Reshape(const vector<Blob*>& b, const vector<Blob*>& t) override { t[0]->ReshapeLike(*b[0]); }
 protected:
  void Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) override;
};

class InnerProductLayer : public LayerBase {
 public:
  explicit InnerProductLayer(const LayerParameter& p)
      : LayerBase(p), num_output_(p.inner_product_param.num_output), bias_(p.inner_product_param.bias_term) {}
  const char* type() const override { return "InnerProduct"; }
  void LayerSetUp(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Reshape(const vector<Blob*>& b, const vector<Blob*>& t) override;
 protected:
  void Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) override;
  int num_output_, K_ = 0, M_ = 0;
  bool bias_;
  // forward runs on the tensor-core NoTrans x Trans GEMM (b2c_sgemm_ex): split-K scratch, and a 16-byte aligned copy of the
  // weights when their slot in the parameter arena is only 8-byte aligned (slots are padded to even counts, net.cpp:1356-1371;
  // TMA wants 16).  The copy is 4 bytes per weight once per forward -- against a 4x slower FFMA kernel.
  Blob gemm_ws_, w_aligned_;
  // backward on the same GEMM: dW[N x K] += dy^T x and dx[M x K] = dy W are NoTrans x Trans products of TRANSPOSED operand copies
  // (dy^T [N x M], x^T [K x M]; W^T [K x N]) -- the reduction axis must be the contiguous one.  The copies are one pass over
  // each operand; the FFMA kernel they replace runs at ~20 TFLOP/s (2.9 of AlexNet's 17 ms step, 1.4 of VGG-16's 19).
  Blob dyt_, xt_, wt_, bwd_ws_;
  bool bwd_w_tc_ = false, bwd_x_tc_ = false;
};

// ---- layers the AlexNet / GoogLeNet / VGG-16 nets add (parity: tests/test_layers_extra_gpu.py, test_inception_style_net_matches_oracle) ----
class LRNLayer : public LayerBase {            // ACROSS_CHANNELS only (the BASELINE nets' use)
 public:
  explicit LRNLayer(const LayerParameter& p) : LayerBase(p) {
    B2_CHECK(p.lrn_param.norm_region == 0, "TrainNet: LRN WITHIN_CHANNEL is not built (the BASELINE nets use ACROSS_CHANNELS)");
  }
  const char* type() const override { return "LRN"; }
  void Reshape(const vector<Blob*>& b, const vector<Blob*>& t) override { t[0]->ReshapeLike(*b[0]); scale_.ReshapeLike(*b[0]); }
 protected:
  void Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) override;
  Blob scale_;
};

class DropoutLayer : public LayerBase {        // TRAIN phase: y = x * mask, mask in {0, 1/(1-ratio)}; TEST phase: y = x
 public:
  DropoutLayer(const LayerParameter& p, uint64_t seed) : LayerBase(p), seed_(seed) {}
  const char* type() const override { return "Dropout"; }
  void Reshape(const vector<Blob*>& b, const vector<Blob*>& t) override { if (t[0] != b[0]) t[0]->ReshapeLike(*b[0]); mask_.ReshapeLike(*b[0]); }
 protected:
  void Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) override;
  uint64_t seed_, offset_ = 0;
  Blob mask_;
};

class ConcatLayer : public LayerBase {         // along the channel axis (axis 1), strided 2-D copies
 public:
  explicit ConcatLayer(const LayerParameter& p) : LayerBase(p) {
    B2_CHECK(p.concat_param.axis == 1, "TrainNet: Concat is built for the channel axis only");
  }
  const char* type() const override { return "Concat"; }
  void Reshape(const vector<Blob*>& b, const vector<Blob*>& t) override;
 protected:
  void Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) override;
};

// slice_layer.cpp: the bottom split along one axis into the tops, in order; Concat's strided 2-D copies with the roles swapped.
// Backward writes the whole bottom diff: a top whose diff no layer writes contributes its zero-initialised diff.
class SliceLayer : public LayerBase {
 public:
  SliceLayer(const LayerParameter& p, const vector<vector<int>>& top_shapes) : LayerBase(p), shapes_(top_shapes) {}
  const char* type() const override { return "Slice"; }
  void Reshape(const vector<Blob*>& b, const vector<Blob*>& t) override;
 protected:
  void Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) override;
  vector<vector<int>> shapes_;
};

// softmax_loss_layer.cpp over the [outer, C, inner] view of softmax_param.axis (canonical: Net resolved it), with loss_param's
// ignore_label and normalization; top 1 (optional) shares prob_.  The legacy case -- inner == 1, no ignore_label, a normalizer of
// outer (VALID, FULL or BATCH_SIZE), one top -- runs b2c_softmax_loss_forward / _backward with the arguments it always had; every
// other case b2c_softmax_loss_forward_ex / _backward_ex, with the normalizer kept on the device between the two.
class SoftmaxWithLossLayer : public LayerBase {
 public:
  using LayerBase::LayerBase;
  const char* type() const override { return "SoftmaxWithLoss"; }
  void Reshape(const vector<Blob*>& b, const vector<Blob*>& t) override;
 protected:
  void Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) override;
  Blob prob_, workspace_, normalizer_;
  int outer_ = 0, C_ = 0, inner_ = 0;
  bool legacy_ = true;
};

// ---- layers the deploy / TEST nets and the MNIST autoencoder add (softmax_layer, sigmoid_layer, flatten_layer, euclidean_loss_layer,
// sigmoid_cross_entropy_loss_layer .cpp) ----
class SoftmaxLayer : public LayerBase {        // over softmax_param.axis: an [outer, C, inner] view of the bottom
 public:
  using LayerBase::LayerBase;
  const char* type() const override { return "Softmax"; }
  void Reshape(const vector<Blob*>& b, const vector<Blob*>& t) override { if (t[0] != b[0]) t[0]->ReshapeLike(*b[0]); }
 protected:
  void Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) override;
};

class SigmoidLayer : public LayerBase {
 public:
  using LayerBase::LayerBase;
  const char* type() const override { return "Sigmoid"; }
  void Reshape(const vector<Blob*>& b, const vector<Blob*>& t) override { if (t[0] != b[0]) t[0]->ReshapeLike(*b[0]); }
 protected:
  void Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) override;
};

// ELU, Power, AbsVal, BNLL, Exp, Log and Threshold (their *_layer.cpp / .cu): b2c_neuron_forward / _backward with the constants
// each reference LayerSetUp derives, in float.  In place: AbsVal refuses it always (absval_layer.cpp); BNLL, Log and the Power
// branches that read x refuse it when the layer runs backward (TrainNet checks that at build time), where the reference would
// differentiate at the overwritten bottom.  ELU in place reads the top as the bottom, as the reference does.  Threshold has no
// backward: TrainNet refuses a net in which its bottom would need a gradient.
class NeuronLayer : public LayerBase {
 public:
  explicit NeuronLayer(const LayerParameter& p);
  const char* type() const override { return layer_param_.type.c_str(); }
  void LayerSetUp(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Reshape(const vector<Blob*>& b, const vector<Blob*>& t) override { if (t[0] != b[0]) t[0]->ReshapeLike(*b[0]); }
  bool backward_reads_bottom() const;   // the backward rule reads x (so an in-place layer would read y in its place)
 protected:
  void Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) override;
  int kind_ = 0;
  float fwd_[3] = {0.f, 0.f, 0.f}, bwd_[3] = {0.f, 0.f, 0.f};   // p0..p2 of b2c_neuron_forward / _backward
};

// prelu_layer.cpp / .cu: blobs_[0] the slopes, [C] or the 0-axis blob when channel_shared, filled by prelu_param.filler.  In place
// with a backward, the forward also keeps a copy of x (x_keep, the reference's bottom_memory_) in the same pass.  The backward is
// one pass for dx and the slope gradient, which it adds into blobs_[0]'s diff (b2c_prelu_backward, deterministic).
class PReLULayer : public LayerBase {
 public:
  using LayerBase::LayerBase;
  const char* type() const override { return "PReLU"; }
  void LayerSetUp(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Reshape(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void set_keep_bottom(bool v) { keep_bottom_ = v; }   // TrainNet: in place and running backward
 protected:
  void Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) override;
  void view(const Blob* b, int* N, int* C, int* dim) const;
  bool keep_bottom_ = false;
  Blob x_keep_, workspace_;
  size_t workspace_bytes_ = 0;
};

// Launches nothing.  Forward: the top aliases the bottom's data (Blob::ShareData), re-pointed every call in case the bottom's
// memory moved.  Backward: ONE device-to-device copy of the top's diff into the bottom's diff, not an alias: the bottom handed
// to Backward may be a fan-out shadow blob with a private diff, and the arena may re-point diffs (set_gpu_diff) after set-up,
// so a diff alias fixed at set-up could write a gradient nobody reads.
class FlattenLayer : public LayerBase {
 public:
  FlattenLayer(const LayerParameter& p, const vector<int>& top_shape) : LayerBase(p), shape_(top_shape) {}
  const char* type() const override { return "Flatten"; }
  void Reshape(const vector<Blob*>& b, const vector<Blob*>& t) override;
 protected:
  void Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) override;
  vector<int> shape_;
};

class EuclideanLossLayer : public LayerBase {  // loss = sum (a - b)^2 / N / 2; gradient to each propagating bottom with its sign
 public:
  using LayerBase::LayerBase;
  const char* type() const override { return "EuclideanLoss"; }
  void Reshape(const vector<Blob*>& b, const vector<Blob*>& t) override { diff_.ReshapeLike(*b[0]); t[0]->Reshape({1}); }
 protected:
  void Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) override;
  Blob diff_;
};

class L1LossLayer : public LayerBase {         // loss = sum |a - b| / N; gradient +-loss_weight / N * sign(a - b) to each propagating bottom
 public:
  using LayerBase::LayerBase;
  const char* type() const override { return "L1Loss"; }
  void Reshape(const vector<Blob*>& b, const vector<Blob*>& t) override { diff_.ReshapeLike(*b[0]); t[0]->Reshape({1}); }
 protected:
  void Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) override;
  Blob diff_;                                   // a - b; the backward takes its sign (the reference keeps a separate sign_ blob)
};

class SigmoidCrossEntropyLossLayer : public LayerBase {   // no sigmoid tensor: backward recomputes sigmoid(x)
 public:
  using LayerBase::LayerBase;
  const char* type() const override { return "SigmoidCrossEntropyLoss"; }
  void Reshape(const vector<Blob*>&, const vector<Blob*>& t) override { t[0]->Reshape({1}); }
 protected:
  void Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) override;
};

// contrastive_loss_layer.cpp: bottoms a, b [N, C(, 1, 1)] and the similarity label [N]; diff = a - b and dist_sq are kept for backward
// CropLayer (crop_layer.cpp / .cu): top = bottom[0]'s window of bottom[1]'s extents (CropShape); backward zero-fills bottom[0]'s
// diff and copies the top diff into the window.  bottom[1] supplies only a shape and never receives a gradient (LabelBottom).
class CropLayer : public LayerBase {
 public:
  using LayerBase::LayerBase;
  const char* type() const override { return "Crop"; }
  int MinBottomBlobs() const override { return 2; }
  void Reshape(const vector<Blob*>& b, const vector<Blob*>& t) override;
 protected:
  void Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) override;
  vector<int> offsets_;
};

class ContrastiveLossLayer : public LayerBase {
 public:
  using LayerBase::LayerBase;
  const char* type() const override { return "ContrastiveLoss"; }
  void Reshape(const vector<Blob*>& b, const vector<Blob*>& t) override {
    diff_.Reshape({b[0]->shape(0), (int)b[0]->count(1)}); dist_sq_.Reshape({b[0]->shape(0)}); t[0]->Reshape({1});
  }
 protected:
  void Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) override;
  Blob diff_, dist_sq_;
};

// forward only (accuracy_layer.cpp) over the [outer, C, inner] view of accuracy_param.axis (canonical); top[0] is a scalar, top[1]
// (optional) the per-class accuracy [C].  The legacy case -- inner == 1, no ignore_label, one top -- runs b2c_accuracy as it always
// did; every other case b2c_accuracy_ex.
class AccuracyLayer : public LayerBase {
 public:
  using LayerBase::LayerBase;
  const char* type() const override { return "Accuracy"; }
  void Reshape(const vector<Blob*>& b, const vector<Blob*>& t) override;
 protected:
  void Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Backward_gpu(const vector<Blob*>&, const vector<bool>&, const vector<Blob*>&) override {}   // "Accuracy cannot backpropagate"
  Blob hits_;
  int outer_ = 0, C_ = 0, inner_ = 0;
  bool legacy_ = true;
};

// Synthetic in-memory source standing in for DataLayer's LMDB reader (SURVEY 8d / 8f rank 4).  Two forms:
//   * float: N(0,1) images from mt19937(seed), uniform labels (Input / DummyData layers, nets without transform_param);
//   * datum: a pinned batch of uint8 datums (crop_size + 32 on a side, like the 256x256 ImageNet LMDBs for a 224 crop) that
//     goes through the reference's own path every e2e step: host -> device copy of the BYTES, then DataTransformer::Transform
//     on the device (b2c_transform_u8: random crop window and mirror per image drawn with Caffe's rule rand % (extent), mean
//     values, scale) into the float data blob.
class SyntheticDataLayer : public LayerBase {
 public:
  // transform_param: crop, mirror, mean_value, scale; the TEST phase takes the centre crop window (data_transformer.cpp:219-229)
  SyntheticDataLayer(const LayerParameter& p, const vector<vector<int>>& shapes, int num_classes, uint64_t seed)
      : LayerBase(p), shapes_(shapes), classes_(num_classes), seed_(seed) {}
  const char* type() const override { return "Data"; }
  void LayerSetUp(const vector<Blob*>& b, const vector<Blob*>& t) override;
  void Reshape(const vector<Blob*>&, const vector<Blob*>&) override {}
  // one batch from pinned host memory into top[0] on `stream` (the e2e step): float copy, or uint8 copy + device transform
  void LoadBatch(Blob* top, cudaStream_t stream);
  size_t h2d_bytes() const { return datum_mode_ ? u8_bytes_ + 9 * (size_t)shapes_[0][0] : sizeof(float) * n0_; }
  bool datum_mode() const { return datum_mode_; }
  ~SyntheticDataLayer() override;
 protected:
  void Forward_gpu(const vector<Blob*>&, const vector<Blob*>&) override {}
  void Backward_gpu(const vector<Blob*>&, const vector<bool>&, const vector<Blob*>&) override {}
  vector<vector<int>> shapes_;
  int classes_;
  uint64_t seed_;
  float* host_ = nullptr;
  size_t n0_ = 0;
  // datum mode
  bool datum_mode_ = false;
  int hd_ = 0, wd_ = 0;
  size_t u8_bytes_ = 0;
  unsigned char* host_u8_ = nullptr;      // pinned [N][C][hd][wd]
  float* dev_mean_ = nullptr;
  uint64_t draws_ = 0;                    // batches drawn so far (crop / mirror stream position)
  // Prefetch (BasePrefetchingDataLayer's thread, as a copy stream): while step i computes, batch i+1's datums and its crop / mirror
  // draws travel host -> device into the other of two slots; LoadBatch makes the compute stream wait for its slot, transforms out
  // of it and starts the next copy.  Every step still moves one batch over PCIe; the copy no longer sits in front of the forward.
  struct Slot {
    unsigned char* dev_u8 = nullptr;
    int* host_off = nullptr;              // pinned: h_off[N], w_off[N], then mirror[N] as bytes
    int* dev_off = nullptr;
    cudaEvent_t copied = nullptr, consumed = nullptr;
    bool in_flight = false, used = false;
  } slot_[2];
  int cur_ = 0;
  cudaStream_t copy_stream_ = nullptr;
  void IssueCopy(int s);
};

// A Net built with phase TEST makes a forward-only instance (the reference's test net, net.cpp / tools/caffe.cpp test()): no
// SGDSolver, ReduceScheduler or parameter arena, no backward bookkeeping, BatchNorm on its running statistics, Dropout the identity,
// Data layers on the centre crop window.  Its parameters come from a .caffemodel (CopyTrainedLayersFrom) or are the blobs of a TRAIN
// instance (ShareTrainedLayersWith), and Test() scores it.
class TrainNet {
 public:
  TrainNet(const Net& net, const SolverParameter& sp, int num_classes, uint64_t seed, int math);
  ~TrainNet();
  void AttachSync(P2PSync* sync);                  // weights broadcast from rank 0, gradients exchanged per bucket
  float ForwardBackward();                         // Net::ForwardBackward (net.cpp:711-716); returns the loss (host sync)
  void ClearParamDiffs();                          // Net::ClearParamDiffs (net.cpp:1256-1270): zero every learnable blob's diff
  void Step(bool copy_input_from_host);            // one Solver::Step iteration, fully asynchronous on the thread stream
  // n Steps bracketed by CUDA events on the thread stream; returns milliseconds (end-of-iteration makes the compute
  // stream wait for the last update, so the closing event covers reduce + update too)
  float TimedSteps(int n, bool copy_input, bool read_loss);
  // n Steps with CUDA events around every layer call (and around the conv weight- / data-gradient calls inside Backward);
  // per (layer, EventProfiler::Op) mean milliseconds per step.  Events serialise nothing, but the numbers are per-call device
  // times on the compute stream, not a decomposition of the overlapped step.
  void ProfileSteps(int n, vector<int>* layer, vector<int>* op, vector<float>* ms);
  const string& layer_name(int i) const { return layer_names_[i]; }
  const string& layer_type(int i) const { return layer_types_[i]; }
  float last_loss();                               // device -> host read of the loss blob
  SGDSolver& solver() { return *solver_; }
  Blob* blob(const string& name);
  int num_layers() const { return (int)layers_.size(); }
  LayerBase* layer(int i) { return layers_[i].get(); }
  // Net::learnable_params(): every layer blob that owns its storage (a blob sharing a named parameter is not listed: it aliases its
  // owner's data and diff, and its gradient adds into the owner's)
  const vector<shared_ptr<Blob>>& learnable_params() const { return learnable_; }
  const vector<int>& trainable_ids() const { return trainable_ids_; }               // ids the layers differentiate
  size_t activation_floats() const;
  size_t input_bytes() const {                     // host -> device bytes of one e2e step's batch
    size_t n = data_ ? data_->h2d_bytes() : 0;
    for (auto& d : db_data_) n += d.first->h2d_bytes();
    return n;
  }
  // the first Data layer that reads its LMDB (data_layer.hpp), or null
  DataLayer* database_layer() { return db_data_.empty() ? nullptr : db_data_[0].first; }
  // Solver::Snapshot (solver.cpp:447-520): <prefix>_iter_<N>.caffemodel (every layer's blobs, NVCaffe raw BlobProto) and
  // <prefix>_iter_<N>.solverstate (iter, learned_net, one history blob per learnable parameter, current_step).
  // Returns the .solverstate path.
  string Snapshot(const string& prefix);
  void Restore(const string& solverstate_path);          // SGDSolver::RestoreSolverStateFromBinaryProto + weights
  // Net::CopyTrainedLayersFrom (net.cpp): layers matched by name, blob shapes must agree; returns the number of layers copied
  int CopyTrainedLayersFrom(const string& caffemodel_path);
  const string& name() const { return name_; }
  bool test_phase() const { return test_; }
  bool has_solver() const { return solver_ != nullptr; }
  // ---- TEST phase only ----
  // Net::ShareTrainedLayersWith (net.cpp): a layer matched by name takes `train`'s parameter blobs by pointer (shapes must agree), so
  // this net reads the weights and BatchNorm statistics the trainer keeps updating.  `train` must outlive this net.  When `train` has
  // a P2PSync attached (call this after AttachSync), this net's database reads the rank's stripe and TestPass sums over the ranks.
  void ShareTrainedLayersWith(TrainNet& train);
  // Net::output_blobs (Net::Init's available_blobs: tops no later layer consumes, in name order) with their loss weights: the layer's
  // loss_weight, else 1 for a loss layer's first top and 0 otherwise
  struct Output { string name; Blob* blob; float loss_weight; };
  const vector<Output>& outputs() const { return outputs_; }
  void ForwardTest();                              // one forward: the database's next batch (when the net reads one), then every layer
  // tools/caffe.cpp test(): `iterations` forwards on freshly prepared filter caches; per_batch gets every output element of every
  // batch (iterations x sum of output counts), mean their means; returns the mean loss (sum of loss_weight * output per batch)
  float Test(int iterations, vector<float>* per_batch, vector<float>* mean);
  // Solver::Test (solver.cpp:445-540) without a host read per batch: `iterations` forwards on the thread stream, each batch's outputs
  // added (b2c_add, output order) into a device score vector -- the float sums of Test(), bit for bit.  With a trainer's P2PSync
  // (ShareTrainedLayersWith) the vector is then summed over the ranks by one allreduce on the comm stream, ordered after the last batch
  // by an event.  One device -> host read at the end: mean = sum / batches / ranks, loss = sum_k loss_weight_k * mean_k.
  // before_batch (may be empty) is asked before every batch; false stops the pass.  Returns the batches run; mean and loss are
  // written only when all `iterations` ran.  Every rank of a multi-GPU trainer must run the whole pass (the allreduce waits for all).
  int TestPass(int iterations, const std::function<bool(int)>& before_batch, vector<float>* mean, float* loss);
  // TestPass in its two halves: everything up to the read (returns the batches enqueued; the reduction only follows a whole pass),
  // then the read.  Several ranks driven from one host thread enqueue every rank's pass before reading any.
  int EnqueueTestPass(int iterations, const std::function<bool(int)>& before_batch);
  void ReadTestPass(vector<float>* mean, float* loss);
  float TimedForwards(int n);                     // n ForwardTest calls bracketed by CUDA events; milliseconds
  void ProfileForwards(int n, vector<int>* layer, vector<int>* op, vector<float>* ms);   // ProfileSteps for ForwardTest
 private:
  struct Node {
    vector<Blob*> bottom, top;
    vector<bool> propagate_down;
    vector<Blob*> bottom_diff_tmp;                 // per bottom: null = write the blob's own diff, else accumulate through this
    vector<bool> accumulate_bottom;                // per bottom: the layer itself adds into the blob's diff (no shadow blob)
    vector<bool> deferred_add;                     // per bottom: the shadow diff is added by the blob's producer (fused BatchNorm residual tail)
    bool need_backward = false;
    // per layer blob: its learnable id (the owner's for a shared blob; the reference's learnable_param_ids_) and whether this layer
    // owns it.  first_owned: the lowest learnable id this layer owns, -1 when it owns none (it then releases nothing to the reducer)
    vector<int> param_ids;
    vector<bool> param_owned;
    int first_owned = -1;
  };
  // set-up, in this order: the layers and their parameter ids (sharing included), BatchNorm / Eltwise fused with the ReLU that
  // follows, shadow diffs where a blob fans out, residual tails with their deferred shadow adds, the output blobs
  vector<ParamSpec> BuildNodes(const Net& net, int num_classes, uint64_t seed, int math);   // returns the learnable blobs' specs
  void FuseReLU();
  void PlanFanOutDiffs();
  void FuseResidualTails(bool fuse_split);
  void CollectOutputs(const Net& net);
  void Forward(bool copy_input);
  void Backward(bool update);
  void PrepareFilters();                           // b2c_conv_prepare_filters over every cached conv layer (weights changed)
  // a blob that shares a named parameter (Net::param_owners_): blob `blob` of layer `layer` aliases blob `owner_blob` of `owner_layer`
  struct Share { int layer, blob, owner_layer, owner_blob; };
  vector<Share> shares_;
  void AliasShare(const Share& sh);                // the sharer's data and diff alias the owner's (ShareData + ShareDiff, no copy)
  void Profile(int n, const std::function<void()>& iteration, vector<int>* layer, vector<int>* op, vector<float>* ms);
 public:
  void MarkParamsDirty() { filters_dirty_ = true; } // call after writing parameter data behind the net's back
 private:
  bool filters_dirty_ = true;
  bool test_ = false;                              // built from a TEST-phase Net: forward only
  vector<Output> outputs_;
  P2PSync* test_sync_ = nullptr;                   // TEST phase: the P2PSync of the trainer this net shares (TestPass's reduction)
  Blob scores_;                                    // TEST phase: TestPass's device score vector
  int pass_batches_ = 0;                           // batches of the enqueued, unread pass
  cudaEvent_t pass_scored_ = nullptr, pass_reduced_ = nullptr;   // its score allreduce: after the last batch, before the read
  bool fuse_fanout_ = true;                        // B2C_FUSE: conv layers add their bottom gradient into a fan-out blob's diff directly
  vector<ConvolutionLayer*> cached_convs_;
  float host_loss_ = 0.f;
  string name_;
  vector<string> layer_names_, layer_types_;
  std::map<string, shared_ptr<Blob>> blobs_;
  vector<shared_ptr<LayerBase>> layers_;
  vector<Node> nodes_;
  vector<shared_ptr<Blob>> tmp_diffs_;
  vector<shared_ptr<Blob>> learnable_;
  vector<int> trainable_ids_;
  std::unique_ptr<SGDSolver> solver_;
  std::unique_ptr<ReduceScheduler> sched_;
  P2PSync* sync_ = nullptr;
  Blob* loss_blob_ = nullptr;
  SyntheticDataLayer* data_ = nullptr;
  vector<std::pair<DataLayer*, int>> db_data_;     // the LMDB-backed sources (data_param.source opened) and their nodes
};

}  // namespace caffe
