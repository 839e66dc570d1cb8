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
enum Phase { TRAIN = 0, TEST = 1 };

struct PoolingParameter { int pool = 0, kernel_h = 0, kernel_w = 0, stride_h = 1, stride_w = 1, pad_h = 0, pad_w = 0; bool global_pooling = false; };

struct NetLayer {                       // one LayerParameter after phase filtering
  LayerParameter param;                 // name, type, bottom, top, ParamSpecs, convolution_param
  PoolingParameter pooling;
  int ip_num_output = 0;
  bool ip_bias = true;
  bool bn_scale_bias = false;           // NVCaffe BatchNormParameter.scale_bias
  float bn_eps = 1e-5f, bn_maf = 0.999f; // BatchNormParameter.eps / moving_average_fraction
  FillerParameter ip_weight_filler, ip_bias_filler;
  float relu_slope = 0.f;
  int eltwise_op = 1;                   // EltwiseParameter.operation: PROD = 0, SUM = 1, MAX = 2
  std::vector<float> eltwise_coeff;
  FillerParameter bn_scale_filler, bn_bias_filler; bool bn_has_scale_filler = false, bn_has_bias_filler = false;
  int lrn_size = 5; float lrn_alpha = 1.f, lrn_beta = 0.75f, lrn_k = 1.f; int lrn_region = 0;   // LRNParameter (caffe.proto:1039-1055)
  float dropout_ratio = 0.5f;           // DropoutParameter.dropout_ratio
  std::vector<float> loss_weight;        // LayerParameter.loss_weight (one per top)
  int concat_axis = 1;
  int accuracy_top_k = 1;               // AccuracyParameter.top_k
  int batch_size = 0, crop_size = 0;    // Data layers
  bool has_transform = false, mirror = false;   // TransformationParameter (caffe.proto:436-470)
  float transform_scale = 1.f;
  std::vector<float> mean_value;
  // DataParameter / TransformationParameter fields the database-backed DataLayer reads (caffe.proto:436-470, 806-849)
  std::string data_source, mean_file;
  int data_backend = 0;                 // DataParameter.DB: LEVELDB = 0 (the proto's default), LMDB = 1
  int parser_threads = 0;               // 0 = automatic in the reference; one parser thread here
  bool force_encoded_color = false;     // DataParameter.force_encoded_color
  bool data_cache = false, data_shuffle = false;   // DataParameter.cache / shuffle (accepted; see DataLayer::LayerSetUp)
  long long transform_random_seed = -1; // TransformationParameter.random_seed
  bool use_database = false;            // the source opened: this layer reads it (else the synthetic in-memory source stands in)
  std::vector<int> input_shape;         // Input / DummyData layers
  int softmax_axis = 1;                 // SoftmaxParameter.axis, canonicalised against the bottom's axes
  int flatten_axis = 1, flatten_end_axis = -1;   // FlattenParameter.axis / end_axis, canonicalised
  int slice_axis = 1;                   // SliceParameter.axis (canonicalised) or slice_dim; the tops' shapes carry the split
  float contrastive_margin = 1.f;       // ContrastiveLossParameter.margin / legacy_version (caffe.proto)
  bool contrastive_legacy = false;
  // Net::Init's need-backward result (net.cpp:160-330), loss pruning included: whether the layer runs backward, and per bottom
  // whether it receives a gradient.  TrainNet reads these; nothing else restates the rule.
  bool need_backward = false;
  std::vector<bool> propagate_down;
  bool label_wants_gradient = false;    // the LabelBottom bottom needs a gradient (and the layer runs backward)
};

// The bottom a loss-like layer reads its labels / targets from, which never receives a gradient (-1: none; EuclideanLoss sends
// gradient to both of its bottoms).  SoftmaxWithLoss, SigmoidCrossEntropyLoss and Accuracy: bottom 1; ContrastiveLoss: bottom 2.
int LabelBottom(const std::string& type);
// A layer type whose name ends in "Loss" (LossLayer's subclasses)
bool IsLossType(const std::string& type);
// LayerParameter.loss_weight of top t, defaulting as Layer::SetLossWeights / LossLayer::LayerSetUp do: 1 for the first top of a
// layer whose type ends in "Loss", 0 otherwise
float TopLossWeight(const NetLayer& L, size_t t);

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
