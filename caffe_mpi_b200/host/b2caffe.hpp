// b2caffe.hpp -- C++ host layer of the H100-native Caffe-MPI hot path.
//
// Mirrors, for this path only, the reference's operator / plugin surface so that code written against
// caffe::Blob / caffe::Layer / caffe::LayerRegistry / caffe::SGDSolver / caffe::P2PSync reads the same:
//   Blob                      include/caffe/blob.hpp:37-603, src/caffe/blob.cpp, syncedmem.hpp:19-89
//   FillerParameter, Filler   include/caffe/filler.hpp (constant, gaussian, xavier, msra)
//   ConvolutionParameter      src/caffe/proto/caffe.proto:718-786
//   LayerBase / Layer         include/caffe/layer.hpp:43-120,279-303,472-611
//   LayerRegistry             include/caffe/layer_factory.hpp:114-202, src/caffe/layer_factory.cpp:53-88
//   ConvolutionLayer          src/caffe/layers/{base_conv_layer.cpp,conv_layer.cpp,conv_layer.cu}
//   ParamArena                Net::InitializeLearnableDiffSpace, src/caffe/net.cpp:1350-1373
//   ReduceScheduler           Net::ReduceAndUpdate / ReduceBucket, src/caffe/net.cpp:757-912
//   SolverParameter/SGDSolver src/caffe/solvers/sgd_solver.cpp:24-259, include/caffe/solver.hpp:81-97
//   P2PSync                   src/caffe/parallel.cpp:36-253, src/caffe/clusters.cpp:8-16
// All device work goes through the C ABI of include/b2c.h (libb2c.so); this layer owns no kernels.
// Differences by design: fp32 only (the BASELINE configs), one process per GPU, no host syncs on the hot
// path (CUDA events order compute stream -> comm stream), errors throw caffe::FatalError where the
// reference LOG(FATAL)s.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <functional>
#include <map>
#include <memory>
#include <random>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/b2c.h"

namespace caffe {

using std::shared_ptr;
using std::string;
using std::vector;

struct FatalError : std::runtime_error {
  using std::runtime_error::runtime_error;
};
[[noreturn]] void Fatal(const char* file, int line, const string& msg);
#define B2_CHECK(cond, msg)                                            \
  do {                                                                 \
    if (!(cond)) ::caffe::Fatal(__FILE__, __LINE__, std::string("Check failed: " #cond " ") + (msg)); \
  } while (0)
void CudaCheck(cudaError_t e, const char* file, int line);
#define CUDA_CHECK(expr) ::caffe::CudaCheck((expr), __FILE__, __LINE__)
void B2cCheck(int rc, const char* file, int line);   // NCCL_CHECK / CUBLAS_CHECK analogue for libb2c calls
#define B2C_CHECK(expr) ::caffe::B2cCheck((expr), __FILE__, __LINE__)

// common.hpp:723 -- arena slots are padded to an even element count
inline size_t even(size_t n) { return n + (n & 1); }

// Thread-local runtime state, the part of the `Caffe` singleton (common.hpp:334-353) this path needs.
// Per-call CUDA-event timing of a training step (the `caffe time` benchmark of the reference, tools/caffe.cpp:289-379, times
// layers the same way, with host timers).  TrainNet brackets every layer's Forward / Backward; ConvolutionLayer additionally
// brackets its weight-gradient and data-gradient calls.  Off (null) outside TrainNet::ProfileSteps.
class EventProfiler {
 public:
  enum Op { FWD = 0, BWD = 1, WGRAD = 2, DGRAD = 3 };
  struct Rec { int layer, op; cudaEvent_t a, b; };
  ~EventProfiler();
  void set_layer(int l) { layer_ = l; }
  size_t begin(int op, cudaStream_t st);        // returns the record handle for end()
  void end(size_t h, cudaStream_t st);
  // synchronises, then sums elapsed ms per (layer, op); clears the records
  void collect(std::map<std::pair<int, int>, float>* out);
 private:
  int layer_ = -1;
  vector<Rec> recs_;
};

class Caffe {
 public:
  static Caffe& Get();
  static EventProfiler* profiler() { return Get().profiler_; }
  static void set_profiler(EventProfiler* p) { Get().profiler_ = p; }
  static cudaStream_t thread_stream() { return Get().stream_; }
  static void set_thread_stream(cudaStream_t s) { Get().stream_ = s; }
  static int solver_count() { return Get().solver_count_; }
  static void set_solver_count(int n) { Get().solver_count_ = n; }
  static bool root_solver() { return Get().root_solver_; }
  static void set_root_solver(bool v) { Get().root_solver_ = v; }
  static std::mt19937& rng() { return Get().rng_; }
  static void set_random_seed(uint64_t seed) { Get().rng_.seed(seed); }

 private:
  cudaStream_t stream_ = nullptr;
  EventProfiler* profiler_ = nullptr;
  int solver_count_ = 1;
  bool root_solver_ = true;
  std::mt19937 rng_{1701};
};

// ---------------------------------------------------------------------------------------------- Blob
// N-D fp32 array with data + diff, lazily mirrored between host and device (SyncedMemory head state).
// Device pointers must be re-fetched on every call: the arena re-points diffs with set_gpu_diff.
class Blob {
 public:
  Blob() = default;
  explicit Blob(const vector<int>& shape) { Reshape(shape); }
  Blob(int n, int c, int h, int w) { Reshape(vector<int>{n, c, h, w}); }
  ~Blob();
  Blob(const Blob&) = delete;
  Blob& operator=(const Blob&) = delete;

  void Reshape(const vector<int>& shape);
  void ReshapeLike(const Blob& o) { Reshape(o.shape_); }
  const vector<int>& shape() const { return shape_; }
  int shape(int i) const { return shape_[CanonicalAxisIndex(i)]; }
  int num_axes() const { return (int)shape_.size(); }
  size_t count() const { return count_; }
  size_t count(int start, int end) const;
  size_t count(int start) const { return count(start, num_axes()); }
  int CanonicalAxisIndex(int i) const;
  string shape_string() const;

  const float* cpu_data();
  const float* cpu_diff();
  float* mutable_cpu_data();
  float* mutable_cpu_diff();
  const float* gpu_data();
  const float* gpu_diff();
  float* mutable_gpu_data();
  float* mutable_gpu_diff();
  // alias external device memory (Net::InitializeLearnableDiffSpace uses this for diffs; the arena here
  // also re-homes data so the fused multi-tensor SGD sees one contiguous parameter space)
  void set_gpu_data(float* p);
  void set_gpu_diff(float* p);
  void ShareData(Blob& other);        // alias other's device data without copying (Blob::ShareData, blob.hpp)
  void ShareDiff(Blob& other);        // alias other's device diff without copying (Blob::ShareDiff)
  void Update();                      // data -= diff (blob.cpp:129-154), on the thread stream
  void set_diff(float v);

 private:
  enum Head { UNINIT, AT_CPU, AT_GPU, SYNCED };
  struct Mem {
    float* cpu = nullptr;
    float* gpu = nullptr;
    bool own_gpu = true;
    Head head = UNINIT;
    size_t cap = 0;
  };
  void to_cpu(Mem& m);
  void to_gpu(Mem& m);
  void release(Mem& m);
  vector<int> shape_;
  size_t count_ = 0;
  Mem data_, diff_;
};

// ---------------------------------------------------------------------------------------------- params
struct FillerParameter {   // caffe.proto FillerParameter
  string type = "constant";
  float value = 0.f, min = 0.f, max = 1.f, mean = 0.f, std = 1.f;
  int variance_norm = 0;   // FAN_IN
};
void Fill(const FillerParameter& f, Blob* b);   // filler.hpp:33,100,278,381

struct ConvolutionParameter {   // caffe.proto:718-786 (same names / defaults)
  int num_output = 0;
  bool bias_term = true;
  vector<int> pad, kernel_size, stride, dilation;
  int pad_h = -1, pad_w = -1, kernel_h = -1, kernel_w = -1, stride_h = -1, stride_w = -1;   // -1 == !has_*
  int group = 1;
  FillerParameter weight_filler, bias_filler;
  int engine = B2C_ENGINE_DEFAULT;    // DEFAULT = 0, CAFFE = 1, CUDNN = 2
  int axis = 1;
  bool force_nd_im2col = false;
  int math = B2C_MATH_FP32;           // forward_math / backward_math analogue (b2c_math)
};
struct ParamSpec {
  float lr_mult = 1.f, decay_mult = 1.f;
  bool statistic = false;   // set by TrainNet for blobs their layer never differentiates (BatchNorm mean / variance / correction)
  // caffe.proto ParamSpec.name / share_mode and whether lr_mult / decay_mult were given: blobs that carry one name are one
  // parameter (Net::AppendParam, net.cpp:576-666).  share_mode: STRICT = 0, PERMISSIVE = 1
  string name;
  bool has_lr_mult = false, has_decay_mult = false;
  int share_mode = 0;
};
// The sub-messages of caffe.proto's LayerParameter the built layers read, with the proto's names and defaults.  Net (prototxt.hpp)
// fills them and stores what it resolves against the bottoms: canonical axes, global pooling's window, BatchNorm's eps floor.
struct PoolingParameter { int pool = 0, kernel_h = 0, kernel_w = 0, stride_h = 1, stride_w = 1, pad_h = 0, pad_w = 0; bool global_pooling = false; };   // pool: MAX = 0, AVE = 1, STOCHASTIC = 2
struct InnerProductParameter { int num_output = 0; bool bias_term = true; FillerParameter weight_filler, bias_filler; };
struct BatchNormParameter {     // NVCaffe's; a scale_filler or bias_filler implies scale_bias.  The fillers' defaults: scale 1, bias 0
  bool scale_bias = false; float eps = 1e-5f, moving_average_fraction = 0.999f; FillerParameter scale_filler{"constant", 1.f}, bias_filler;
};
struct ReLUParameter { float negative_slope = 0.f; };
struct LRNParameter { int local_size = 5; float alpha = 1.f, beta = 0.75f, k = 1.f; int norm_region = 0; };   // ACROSS_CHANNELS = 0, WITHIN_CHANNEL = 1
struct DropoutParameter { float dropout_ratio = 0.5f; };
struct EltwiseParameter { int operation = 1; vector<float> coeff; };   // PROD = 0, SUM = 1, MAX = 2
struct ConcatParameter { int axis = 1; };
struct SliceParameter { int axis = 1; bool slice_dim_given = false; vector<int> slice_point; };   // axis: SliceParameter.axis or slice_dim
struct SoftmaxParameter { int axis = 1; };
struct FlattenParameter { int axis = 1, end_axis = -1; };
struct AccuracyParameter { int top_k = 1; };
struct ContrastiveLossParameter { float margin = 1.f; bool legacy_version = false; };
struct TransformationParameter { float scale = 1.f; bool mirror = false; int crop_size = 0; vector<float> mean_value; string mean_file; long long random_seed = -1; };
struct DataParameter {   // batch_size after Net's batch override; backend: LEVELDB = 0, LMDB = 1; parser_threads 0: automatic (see DataLayer)
  string source; int batch_size = 0, backend = 0, parser_threads = 0; bool force_encoded_color = false, cache = false, shuffle = false;
};
enum Phase { TRAIN = 0, TEST = 1 };
struct LayerParameter {
  string name, type;
  vector<string> bottom, top;
  vector<float> loss_weight;            // one per top; see TopLossWeight (prototxt.hpp) for the default
  vector<ParamSpec> param;
  Phase phase = TRAIN;                  // the net's phase: TEST runs BatchNorm on its running statistics and Dropout as the identity
  ConvolutionParameter convolution_param;
  PoolingParameter pooling_param;
  InnerProductParameter inner_product_param;
  BatchNormParameter batch_norm_param;
  ReLUParameter relu_param;
  LRNParameter lrn_param;
  DropoutParameter dropout_param;
  EltwiseParameter eltwise_param;
  ConcatParameter concat_param;
  SliceParameter slice_param;
  SoftmaxParameter softmax_param;
  FlattenParameter flatten_param;
  AccuracyParameter accuracy_param;
  ContrastiveLossParameter contrastive_loss_param;
  TransformationParameter transform_param;
  DataParameter data_param;
};

// ---------------------------------------------------------------------------------------------- Layer
class LayerBase {
 public:
  explicit LayerBase(const LayerParameter& p) : layer_param_(p) {}
  virtual ~LayerBase() {}
  // layer.hpp:76-81: checks blob counts, LayerSetUp, Reshape
  void SetUp(const vector<Blob*>& bottom, const vector<Blob*>& top);
  virtual void LayerSetUp(const vector<Blob*>& bottom, const vector<Blob*>& top) {}
  virtual void Reshape(const vector<Blob*>& bottom, const vector<Blob*>& top) = 0;
  // layer.hpp:555-611: Reshape before every forward, then the device implementation
  float Forward(const vector<Blob*>& bottom, const vector<Blob*>& top);
  void Backward(const vector<Blob*>& top, const vector<bool>& propagate_down, const vector<Blob*>& bottom);
  vector<shared_ptr<Blob>>& blobs() { return blobs_; }
  const LayerParameter& layer_param() const { return layer_param_; }
  float loss_weight() const;            // the loss weight of top 0 (TopLossWeight: 1 for a *Loss type unless the prototxt says)
  virtual const char* type() const { return ""; }
  virtual int MinBottomBlobs() const { return -1; }
  virtual int MinTopBlobs() const { return -1; }
  virtual bool EqualNumBottomTopBlobs() const { return false; }
  virtual bool bias_term() const { return false; }
  bool param_propagate_down(int i) const { return i < (int)param_propagate_down_.size() ? param_propagate_down_[i] : false; }
  // Net::Backward's fan-out accumulation folded into the layer: when true for bottom i, Backward ADDS its gradient to
  // bottom[i]'s diff instead of overwriting it.  Only layers that answer SupportsBottomDiffAccumulate() may be asked to.
  virtual bool SupportsBottomDiffAccumulate(int /*bottom*/) const { return false; }
  void set_accumulate_bottom_diff(const vector<bool>& v) { accumulate_bottom_ = v; }
  void set_param_propagate_down(int i, bool v) { if ((int)param_propagate_down_.size() <= i) param_propagate_down_.resize(i + 1, true); param_propagate_down_[i] = v; }

 protected:
  virtual void Forward_gpu(const vector<Blob*>& bottom, const vector<Blob*>& top) = 0;
  virtual void Backward_gpu(const vector<Blob*>& top, const vector<bool>& propagate_down, const vector<Blob*>& bottom) = 0;
  LayerParameter layer_param_;
  vector<shared_ptr<Blob>> blobs_;
  vector<bool> param_propagate_down_;
  vector<bool> accumulate_bottom_;       // per bottom; empty = overwrite everywhere (the reference's semantics)
};

class LayerRegistry {   // layer_factory.hpp:114-202
 public:
  typedef shared_ptr<LayerBase> (*Creator)(const LayerParameter&);
  static void AddCreator(const string& type, Creator c);   // duplicate registration is fatal (:127-128)
  static shared_ptr<LayerBase> CreateLayer(const LayerParameter& p);
  static vector<string> LayerTypeList();
 private:
  static std::map<string, Creator>& Registry();
};
struct LayerRegisterer { LayerRegisterer(const string& t, LayerRegistry::Creator c) { LayerRegistry::AddCreator(t, c); } };
#define REGISTER_LAYER_CREATOR(type, creator) static ::caffe::LayerRegisterer g_creator_##type(#type, creator)

// ---------------------------------------------------------------------------------------------- Convolution
class ConvolutionLayer : public LayerBase {
 public:
  explicit ConvolutionLayer(const LayerParameter& p) : LayerBase(p) {}
  ~ConvolutionLayer() override;
  void LayerSetUp(const vector<Blob*>& bottom, const vector<Blob*>& top) override;   // base_conv_layer.cpp:12-170
  void Reshape(const vector<Blob*>& bottom, const vector<Blob*>& top) override;      // base_conv_layer.cpp:172-239
  const char* type() const override { return "Convolution"; }
  int MinBottomBlobs() const override { return 1; }
  int MinTopBlobs() const override { return 1; }
  bool EqualNumBottomTopBlobs() const override { return true; }
  bool bias_term() const override { return bias_term_; }
  int algo_used(int op) const;
  // Prepared-filter cache (include/b2c.h "Prepared filters"): an owner of the iteration (TrainNet) enables it and then calls
  // b2c_conv_prepare_filters for all layers after every weight change; without it every Forward / Backward call re-derives
  // the GEMM-ordered filter copy itself.  Returns false when the layer has nothing to cache (CAFFE engine, SIMT, N-D).
  bool EnableFilterCache();
  bool SupportsBottomDiffAccumulate(int) const override { return desc_ && b2c_conv_backward_data_accumulate_supported(desc_) != 0; }
  const b2c_conv_desc* desc() const { return desc_; }
  void* filter_cache() const { return fcache_; }

 protected:
  void Forward_gpu(const vector<Blob*>& bottom, const vector<Blob*>& top) override;     // conv_layer.cu:7-23
  void Backward_gpu(const vector<Blob*>& top, const vector<bool>& propagate_down,
                    const vector<Blob*>& bottom) override;                              // conv_layer.cu:25-57
  void compute_output_shape();                                                          // conv_layer.cpp:7-22
  void* workspace(size_t bytes);

  vector<int> kernel_shape_, stride_, pad_, dilation_, output_shape_, bottom_shape_;
  int num_spatial_axes_ = 0, channel_axis_ = 1, num_ = 0, channels_ = 0, group_ = 1, num_output_ = 0;
  bool bias_term_ = false, is_1x1_ = false;
  b2c_conv_desc* desc_ = nullptr;
  b2c_conv_params desc_params_{};
  void* ws_ = nullptr;
  size_t ws_bytes_ = 0;
  void* fcache_ = nullptr;
  size_t fcache_bytes_ = 0;
  bool fcache_on_ = false;
};
shared_ptr<LayerBase> GetConvolutionLayer(const LayerParameter& p);   // layer_factory.cpp:53-88

// ---------------------------------------------------------------------------------------------- arena
// One contiguous device space each for parameter data, diffs and solver history; every learnable blob's
// data/diff is re-pointed into it at even(count) stride (net.cpp:1350-1373; the reference does diffs only).
// AdaDelta and Adam keep a second history (history2) with the same layout; the other solvers allocate none.
class ParamArena {
 public:
  ~ParamArena();
  void Init(const vector<shared_ptr<Blob>>& params, bool second_history = false);
  void InitLayout(const vector<size_t>& counts);   // offsets only, no device memory (planning / CPU tests)
  size_t total() const { return total_; }
  size_t offset(int i) const { return offset_[i]; }
  size_t count(int i) const { return count_[i]; }
  int size() const { return (int)offset_.size(); }
  float* data() const { return data_; }
  float* diff() const { return diff_; }
  float* history() const { return hist_; }
  float* history2() const { return hist2_; }     // nullptr unless Init(..., second_history)
  bool diff_is_nccl_memory() const { return diff_nccl_; }
 private:
  vector<size_t> offset_, count_;
  size_t total_ = 0;
  float *data_ = nullptr, *diff_ = nullptr, *hist_ = nullptr, *hist2_ = nullptr;
  bool diff_nccl_ = false;
};

// ---------------------------------------------------------------------------------------------- solver
struct SolverParameter {   // caffe.proto SolverParameter (fields this path reads)
  string type = "SGD";             // caffe.proto:269; the legacy solver_type enum (:288-297) is read into it
  float delta = 1e-8f, momentum2 = 0.999f, rms_decay = 0.f;   // caffe.proto:272,274,278 (rms_decay declares no default)
  float base_lr = 0.01f, gamma = 0.1f, power = 1.f, momentum = 0.f, weight_decay = 0.f, min_lr = 0.f;
  float rampup_lr = 0.f, max_momentum = 0.99f, momentum_power = 1.f, clip_gradients = -1.f;
  int stepsize = 1, max_iter = 1, iter_size = 1, rampup_interval = 0;
  vector<int> stepvalue;
  string lr_policy = "fixed", momentum_policy = "fixed", regularization_type = "L2";
  bool snapshot_diff = false;
  bool has_max_momentum = false;   // max_momentum was given: the "opt" momentum policy clamps to it only then (sgd_solver.cpp:83-86)
  float global_grad_scale = 1.f;   // NetParameter.global_grad_scale (caffe.proto:130)
  int reduce_buckets = 6;          // NetParameter.reduce_buckets (caffe.proto:140)
  // testing (caffe.proto:184-188): one TEST net per test_iter entry, built from `net`; a pass every test_interval iterations
  vector<int> test_iter;
  int test_interval = 0;
  bool test_compute_loss = false;
  vector<string> test_fields_not_built;   // test_net, test_net_param, test_state when present: test nets from those are not built
};

// b2c_solver_kind of a SolverParameter.type (REGISTER_SOLVER_CLASS names); an unknown type is fatal and lists the known ones
int SolverKind(const string& type);
// SolverKind plus the constructor sanity checks of the reference's solvers (include/caffe/sgd_solvers.hpp:84-113): AdaGrad
// and RMSProp take no momentum, rms_decay lies in [0, 1).  Fatal on violation.
void CheckSolverParameter(const SolverParameter& p);

class P2PSync;

// SGDSolver and the five solvers derived from it in the reference (Nesterov, AdaGrad, RMSProp, AdaDelta, Adam): they share the
// lr policy, arena, bucket walk and snapshot code and differ only in the fused update ApplyUpdate launches (dispatched on
// param().type) and in the number of history arenas.
class SGDSolver {
 public:
  explicit SGDSolver(const SolverParameter& p) : param_(p), kind_(SolverKind(p.type)) { CheckSolverParameter(p); }
  const SolverParameter& param() const { return param_; }
  int kind() const { return kind_; }
  // history blobs per learnable blob: 2 for AdaDelta and Adam (AdaDeltaPreSolve / AdamPreSolve), 1 otherwise
  int num_histories() const { return kind_ == B2C_SOLVER_ADADELTA || kind_ == B2C_SOLVER_ADAM ? 2 : 1; }
  int iter() const { return iter_; }
  void set_iter(int i) { iter_ = i; }
  int current_step() const { return current_step_; }
  void set_current_step(int s) { current_step_ = s; }
  float GetLearningRate();   // sgd_solver.cpp:24-65
  float GetMomentum();       // sgd_solver.cpp:68-91
  // Register the learnable blobs in layer order with their lr_mult / decay_mult (Net::AppendParam).
  void SetParams(const vector<shared_ptr<Blob>>& params, const vector<ParamSpec>& specs);
  ParamArena& arena() { return arena_; }
  // ApplyUpdate for params [from, to] on `stream` (sgd_solver.cpp:143-149 + sgd_solver.cu:57-72), fused
  // over the arena; grad_scale folds 1/solver_count, 1/global_grad_scale and 1/iter_size.
  void ApplyUpdate(int id_from, int id_to, cudaStream_t stream);
  void ApplyUpdateAll(cudaStream_t stream) { ApplyUpdate(0, arena_.size() - 1, stream); }
  void increment_iter() { ++iter_; }
 private:
  SolverParameter param_;
  int kind_;
  ParamArena arena_;
  vector<ParamSpec> specs_;
  int iter_ = 0, current_step_ = 0;
};

// Bucket plan of Net::ReduceAndUpdate (net.cpp:772-783,824-862): params arrive in reverse order (last
// layer first); adjacent ids are coalesced until received_count >= bucket_space_count.
struct Bucket { int id_from, id_to; size_t offset, count; };
vector<Bucket> PlanBuckets(const ParamArena& arena, int reduce_buckets);

// ---------------------------------------------------------------------------------------------- P2PSync
// One NCCL communicator per process over b2c_comm; carries the rank-0 weight broadcast and the bucket
// allreduce.  The unique id travels through the `bcast_bytes` callable supplied by the launcher
// (MPI_Bcast in the reference, parallel.cpp:42-45; torch.distributed / a file here).
// Solver::Callback (include/caffe/solver.hpp:81-97): what the solver invokes at fixed points of an iteration.  The
// reference's P2PSync implements it with NCCL + host barriers; here the bucket exchange is stream-ordered, so the two
// barriers have nothing to wait for on the host and only order the comm stream.
class SolverCallback {
 public:
  virtual ~SolverCallback() {}
  virtual void on_start(ParamArena& arena) = 0;                    // Callback::on_start: weights from the root solver
  virtual void allreduce_bucket(float* buf, size_t count) = 0;     // Callback::allreduce_bucket (async, comm stream)
  virtual void soft_barrier() {}                                    // Callback::soft_barrier
  virtual void reduce_barrier() {}                                  // Callback::reduce_barrier
  virtual cudaStream_t comm_stream() const = 0;
};

class P2PSync : public SolverCallback {
 public:
  typedef std::function<void(void* buf, size_t bytes, int root)> BcastBytes;
  P2PSync(int nranks, int rank, const BcastBytes& bcast);
  ~P2PSync();
  int nranks() const { return nranks_; }
  int rank() const { return rank_; }
  cudaStream_t comm_stream() const override { return comm_stream_; }
  void on_start(ParamArena& arena) override;                          // parallel.cpp:208-227
  void allreduce_bucket(float* buf, size_t count) override;           // parallel.cpp:245-253 (async, comm stream)
  // the test scores' sum over the ranks (saveTestResults / aggregateTestResults, parallel.cpp:256-282), async on the comm stream;
  // a sibling of allreduce_bucket so that bucket timing never counts it as a gradient bucket
  void allreduce_scores(float* buf, size_t count);
  void soft_barrier() override;                                      // parallel.cpp: MPI_Barrier -> comm-stream drain
  void reduce_barrier() override;
  // batch division of parallel.cpp:284-293: per-rank batch, rounded up to a multiple
  static int divide_batch_size(int total, int solver_count);
  // measurement: CUDA events around every bucket's allreduce on the comm stream (off by default; bench.py's in-step bus bandwidth)
  void set_bucket_timing(bool on) { timing_ = on; }
  void collect_bucket_times(vector<size_t>* bytes, vector<float>* ms);   // drains the comm stream, returns and clears the records
 private:
  int nranks_, rank_;
  b2c_comm* comm_ = nullptr;
  cudaStream_t comm_stream_ = nullptr;
  bool timing_ = false;
  struct TimedBucket { size_t bytes; cudaEvent_t a, b; };
  vector<TimedBucket> timed_;
};

// Event-driven Net::ReduceAndUpdate: after the backward pass has produced the diffs of bucket b on the
// compute stream, the comm stream allreduces it and runs the fused update for its params, overlapping
// with the remaining backward work.  No host thread, no host barrier.
class ReduceScheduler {
 public:
  ReduceScheduler(SGDSolver* solver, SolverCallback* sync);
  ~ReduceScheduler();
  const vector<Bucket>& buckets() const { return buckets_; }
  // call after the backward of the layer owning param `id` has been enqueued on `compute` (ids arrive in
  // descending order, net.cpp:738-746); flushes a bucket when its lowest id has arrived
  void on_param_ready(int id, cudaStream_t compute);
  // END_OF_ITERATION (net.cpp:748-750,866-874): leftovers, then make `compute` wait for the updates
  void end_of_iteration(cudaStream_t compute);
 private:
  void flush(int b, cudaStream_t compute);
  SGDSolver* solver_;
  SolverCallback* sync_;
  vector<Bucket> buckets_;
  int next_bucket_ = 0;
  cudaEvent_t ev_ready_ = nullptr, ev_done_ = nullptr;
  cudaStream_t update_stream_ = nullptr;
};

}  // namespace caffe
