// prototxt.hpp -- protobuf TEXT-format reader for the subset of caffe.proto the BASELINE models use, and the
// Net graph builder on top of it (SURVEY.md 8(f) rank 1: there is no protoc / libprotobuf in the toolchain, so
// the reference's models/*.prototxt and solver.prototxt files are read by this hand-written parser, unmodified).
//
// Reference map:
//   text format / ReadProtoFromTextFile      src/caffe/util/io.cpp, src/caffe/proto/caffe.proto
//   NetParameter / LayerParameter / NetState  caffe.proto:88-146, 303-337, 368-481
//   phase filtering (include / exclude)       Net::FilterNet, Net::StateMeetsRule  (src/caffe/net.cpp)
//   graph build, shapes, need-backward,       Net::Init, Net::AppendTop/AppendBottom/AppendParam (net.cpp:64-667)
//   learnable-parameter list in layer order
//   SolverParameter                           caffe.proto:147-301
#pragma once
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "b2caffe.hpp"

namespace caffe {

// ---- generic text-format tree --------------------------------------------------------------------------------
struct PMessage;
struct PField {
  std::string scalar;                 // for `name: value` (quotes removed)
  std::shared_ptr<PMessage> msg;      // for `name { ... }`
  bool is_msg() const { return (bool)msg; }
};
struct PMessage {
  std::vector<std::pair<std::string, PField>> fields;   // in file order, repeated fields repeat
  bool has(const std::string& k) const;
  std::vector<const PField*> all(const std::string& k) const;
  const PMessage* sub(const std::string& k) const;      // first sub-message or null
  std::string str(const std::string& k, const std::string& d = "") const;
  double num(const std::string& k, double d = 0) const;
  long long integer(const std::string& k, long long d = 0) const;
  bool boolean(const std::string& k, bool d = false) const;
  std::vector<long long> ints(const std::string& k) const;
};
PMessage ParseTextProto(const std::string& text);        // throws FatalError with line number on bad input
PMessage ParseTextProtoFile(const std::string& path);

// ---- net description --------------------------------------------------------------------------------------------
struct NetLayer {                       // one LayerParameter after phase filtering
  LayerParameter param;
  bool use_database = false;            // a Data layer whose source opened: it reads it (else the synthetic in-memory source stands in)
  // Net::Init's need-backward result (net.cpp:160-330), loss pruning included: whether the layer runs backward, and per bottom
  // whether it receives a gradient.  TrainNet reads these; nothing else restates the rule.
  bool need_backward = false;
  std::vector<bool> propagate_down;
  bool label_wants_gradient = false;    // the LabelBottom bottom needs a gradient (and the layer runs backward)
};

// The bottom a loss-like layer reads its labels / targets from, which never receives a gradient (-1: none; EuclideanLoss sends
// gradient to both of its bottoms).  SoftmaxWithLoss, SigmoidCrossEntropyLoss and Accuracy: bottom 1; ContrastiveLoss: bottom 2;
// Crop: bottom 1, which only supplies the shape (CropLayer::Backward_gpu never writes it).
int LabelBottom(const std::string& type);
// A layer type whose name ends in "Loss" (LossLayer's subclasses)
bool IsLossType(const std::string& type);
// LayerParameter.loss_weight of top t, defaulting as Layer::SetLossWeights / LossLayer::LayerSetUp do: 1 for the first top of a
// layer whose type ends in "Loss", 0 otherwise
float TopLossWeight(const LayerParameter& p, size_t t);
// PoolingLayer::Reshape's output extent: ceil mode, and the last window clipped when it would start in the padding
int pooled_extent(int in, int k, int s, int p);
// q over an h x w bottom: global_pooling makes the whole plane one window (stride 1, no padding)
PoolingParameter EffectivePooling(const PoolingParameter& q, int h, int w);
// CropLayer::Reshape (crop_layer.cpp): the top takes `ref`'s extents from crop_param.axis on (negative counts from the end), the
// axes before keep the bottom's; one offset for every cropped axis or one per cropped axis, none = 0.  Fills the top shape and
// the offset of every axis; fatal with the reference's messages where it CHECK-fails.
void CropShape(const std::vector<int>& bottom, const std::vector<int>& ref, const CropParameter& q, std::vector<int>* top,
               std::vector<int>* offsets);

// One parameter blob of a layer.  blob_id counts the layer's learnable blobs; layer_blob is its index among the layer's blobs
// (BatchNorm's scale / bias are blobs 3 and 4).  Named blobs are shared (Net::AppendParam, net.cpp:576-666): the first blob with
// a name owns it, a later one is a sharer with owner = the owner's index in net_params(); learnable_id indexes learnable_params().
struct LearnableParam {
  std::string layer; int layer_id, blob_id; size_t count; std::vector<int> shape; float lr_mult, decay_mult;
  int layer_blob = 0;
  std::string name;                     // ParamSpec.name, empty when anonymous
  int owner = -1;                       // -1: this blob owns its storage
  int learnable_id = 0;
};

struct ConvEntry { std::string name; int layer_id; b2c_conv_params p; bool propagate_down; };

class Net {
 public:
  // batch_override > 0 replaces the Data layer's batch_size (the reference divides the prototxt batch by the GPU
  // count, parallel.cpp:284-293; callers pass the per-rank batch)
  Net(const PMessage& net_param, Phase phase, int batch_override = 0, int default_channels = 3, int default_size = 224);
  static Net FromFile(const std::string& path, Phase phase, int batch_override = 0);
  const std::string& name() const { return name_; }
  Phase phase() const { return phase_; }
  const std::vector<NetLayer>& layers() const { return layers_; }
  const std::map<std::string, std::vector<int>>& blob_shapes() const { return shapes_; }
  const std::vector<int>& top_shape(int layer, int top = 0) const { return layer_top_shapes_[layer][top]; }
  // owners only, in layer order (Net::learnable_params_); a sharer's lr_mult / decay_mult fill in what its owner left unset
  const std::vector<LearnableParam>& learnable_params() const { return params_; }
  const std::vector<LearnableParam>& net_params() const { return net_params_; }   // every layer's blobs, sharers included (Net::params_)
  // the owner of blob `layer_blob` of layer `layer_id` as (layer_id, layer_blob); (-1, -1) when the blob owns itself
  std::pair<int, int> param_owner(int layer_id, int layer_blob) const;
  const std::vector<ConvEntry>& conv_layers() const { return convs_; }
  int reduce_buckets() const { return reduce_buckets_; }
  float global_grad_scale() const { return global_grad_scale_; }
  size_t learnable_count() const;
  // the training loss a trainer reports: the first top of the last layer whose type ends in "Loss" and whose first top has a
  // non-zero loss weight (empty: none)
  const std::string& loss_blob() const { return loss_blob_; }
 private:
  std::string loss_blob_;
  std::string name_;
  Phase phase_ = TRAIN;
  std::vector<NetLayer> layers_;
  std::map<std::string, std::vector<int>> shapes_;
  std::vector<std::vector<std::vector<int>>> layer_top_shapes_;
  std::vector<LearnableParam> params_, net_params_;
  std::vector<ConvEntry> convs_;
  int reduce_buckets_ = 6;
  float global_grad_scale_ = 1.f;
};

// caffe.proto SolverParameter -> the struct SGDSolver takes; `net_path` receives SolverParameter.net
SolverParameter ReadSolverParameter(const PMessage& m, std::string* net_path = nullptr);

}  // namespace caffe
