// b2caffe.cpp -- implementation of the C++ host layer (see b2caffe.hpp for the reference map).
#include "b2caffe.hpp"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <sstream>

namespace caffe {

void Fatal(const char* file, int line, const string& msg) {
  std::ostringstream os;
  os << file << ":" << line << "] " << msg;
  throw FatalError(os.str());
}
void CudaCheck(cudaError_t e, const char* file, int line) {
  if (e != cudaSuccess) Fatal(file, line, string("CUDA: ") + cudaGetErrorString(e));
}
void B2cCheck(int rc, const char* file, int line) {
  if (rc != 0) Fatal(file, line, string("libb2c: ") + b2c_last_error());
}

Caffe& Caffe::Get() {
  thread_local Caffe inst;
  return inst;
}

// ================================================================================================ Blob
Blob::~Blob() {
  release(data_);
  release(diff_);
}
void Blob::release(Mem& m) {
  if (m.cpu) cudaFreeHost(m.cpu);
  if (m.gpu && m.own_gpu) cudaFree(m.gpu);
  m = Mem();
}
void Blob::Reshape(const vector<int>& shape) {
  B2_CHECK(shape.size() <= 32, "blob has too many axes");
  size_t c = 1;
  for (int d : shape) { B2_CHECK(d >= 0, "negative blob dimension"); c *= (size_t)d; }
  shape_ = shape;
  count_ = c;
  for (Mem* m : {&data_, &diff_}) {
    if (c > m->cap) {            // grow only (blob.cpp Reshape keeps capacity)
      B2_CHECK(m->own_gpu || m->gpu == nullptr, "cannot grow a blob that aliases external memory");
      release(*m);
      m->cap = c;
    }
  }
}
size_t Blob::count(int start, int end) const {
  size_t c = 1;
  for (int i = start; i < end; ++i) c *= (size_t)shape_[i];
  return c;
}
int Blob::CanonicalAxisIndex(int i) const {
  B2_CHECK(i >= -num_axes() && i < num_axes(), "axis out of range");
  return i < 0 ? i + num_axes() : i;
}
string Blob::shape_string() const {
  std::ostringstream os;
  for (int d : shape_) os << d << " ";
  os << "(" << count_ << ")";
  return os.str();
}
void Blob::to_cpu(Mem& m) {
  const size_t bytes = sizeof(float) * (m.cap ? m.cap : 1);
  if (!m.cpu) {
    CUDA_CHECK(cudaMallocHost(reinterpret_cast<void**>(&m.cpu), bytes));
    if (m.head == UNINIT) memset(m.cpu, 0, bytes);
  }
  if (m.head == UNINIT) m.head = AT_CPU;
  if (m.head == AT_GPU) {
    cudaStream_t st = Caffe::thread_stream();
    CUDA_CHECK(cudaMemcpyAsync(m.cpu, m.gpu, sizeof(float) * count_, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));   // the only host sync: a CPU reader asked for device results
    m.head = SYNCED;
  }
}
void Blob::to_gpu(Mem& m) {
  const size_t bytes = sizeof(float) * (m.cap ? m.cap : 1);
  if (!m.gpu) {
    CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&m.gpu), bytes));
    m.own_gpu = true;
    if (m.head == UNINIT) CUDA_CHECK(cudaMemsetAsync(m.gpu, 0, bytes, Caffe::thread_stream()));
  }
  if (m.head == UNINIT) m.head = AT_GPU;
  if (m.head == AT_CPU) {
    CUDA_CHECK(cudaMemcpyAsync(m.gpu, m.cpu, sizeof(float) * count_, cudaMemcpyHostToDevice, Caffe::thread_stream()));
    m.head = SYNCED;
  }
}
const float* Blob::cpu_data() { to_cpu(data_); return data_.cpu; }
const float* Blob::cpu_diff() { to_cpu(diff_); return diff_.cpu; }
float* Blob::mutable_cpu_data() { to_cpu(data_); data_.head = AT_CPU; return data_.cpu; }
float* Blob::mutable_cpu_diff() { to_cpu(diff_); diff_.head = AT_CPU; return diff_.cpu; }
const float* Blob::gpu_data() { to_gpu(data_); return data_.gpu; }
const float* Blob::gpu_diff() { to_gpu(diff_); return diff_.gpu; }
float* Blob::mutable_gpu_data() { to_gpu(data_); data_.head = AT_GPU; return data_.gpu; }
float* Blob::mutable_gpu_diff() { to_gpu(diff_); diff_.head = AT_GPU; return diff_.gpu; }

void Blob::set_gpu_data(float* p) {
  // keep the current contents: copy them into the new home first
  const float* cur = count_ ? gpu_data() : nullptr;
  if (cur && cur != p) CUDA_CHECK(cudaMemcpyAsync(p, cur, sizeof(float) * count_, cudaMemcpyDeviceToDevice, Caffe::thread_stream()));
  CUDA_CHECK(cudaStreamSynchronize(Caffe::thread_stream()));
  if (data_.gpu && data_.own_gpu) cudaFree(data_.gpu);
  data_.gpu = p; data_.own_gpu = false; data_.head = AT_GPU;
}
void Blob::set_gpu_diff(float* p) {
  const float* cur = count_ ? gpu_diff() : nullptr;
  if (cur && cur != p) CUDA_CHECK(cudaMemcpyAsync(p, cur, sizeof(float) * count_, cudaMemcpyDeviceToDevice, Caffe::thread_stream()));
  CUDA_CHECK(cudaStreamSynchronize(Caffe::thread_stream()));
  if (diff_.gpu && diff_.own_gpu) cudaFree(diff_.gpu);
  diff_.gpu = p; diff_.own_gpu = false; diff_.head = AT_GPU;
}
void Blob::ShareData(Blob& other) {
  B2_CHECK(count_ == other.count(), "ShareData: count mismatch");
  if (data_.gpu && data_.own_gpu) cudaFree(data_.gpu);
  data_.gpu = other.mutable_gpu_data(); data_.own_gpu = false; data_.head = AT_GPU;
}
void Blob::ShareDiff(Blob& other) {
  B2_CHECK(count_ == other.count(), "ShareDiff: count mismatch");
  if (diff_.gpu && diff_.own_gpu) cudaFree(diff_.gpu);
  diff_.gpu = other.mutable_gpu_diff(); diff_.own_gpu = false; diff_.head = AT_GPU;
}
void Blob::Update() {
  // data = data - 1*diff, expressed with the fused kernel: momentum 0, rate 1, no decay, keep diff
  B2C_CHECK(b2c_sgd_update(count_, mutable_gpu_diff(), mutable_gpu_data(), mutable_gpu_diff(), 0.f, 1.f, 0.f, 1, 1.f, 0,
                           Caffe::thread_stream()));
}
void Blob::set_diff(float v) {
  float* d = mutable_cpu_diff();
  for (size_t i = 0; i < count_; ++i) d[i] = v;
}

// ================================================================================================ Filler
void Fill(const FillerParameter& f, Blob* b) {
  float* d = b->mutable_cpu_data();
  const size_t n = b->count();
  std::mt19937& rng = Caffe::rng();
  const int fan_in = (int)(n / std::max(1, b->num_axes() > 0 ? b->shape(0) : 1));   // a 0-axis blob (count 1) has fan-in 1
  const int fan_out = b->num_axes() > 1 ? (int)(n / std::max(1, b->shape(1))) : (int)n;
  float nval = (float)fan_in;                          // FAN_IN
  if (f.variance_norm == 2) nval = (fan_in + fan_out) / 2.f;   // AVERAGE
  else if (f.variance_norm == 1) nval = (float)fan_out;        // FAN_OUT
  if (f.type == "constant") {
    for (size_t i = 0; i < n; ++i) d[i] = f.value;
  } else if (f.type == "uniform") {
    std::uniform_real_distribution<float> u(f.min, f.max);
    for (size_t i = 0; i < n; ++i) d[i] = u(rng);
  } else if (f.type == "gaussian") {
    std::normal_distribution<float> g(f.mean, f.std);
    for (size_t i = 0; i < n; ++i) d[i] = g(rng);
  } else if (f.type == "xavier") {                     // filler.hpp:278: U(-sqrt(3/n), sqrt(3/n))
    const float s = std::sqrt(3.f / nval);
    std::uniform_real_distribution<float> u(-s, s);
    for (size_t i = 0; i < n; ++i) d[i] = u(rng);
  } else if (f.type == "msra") {                       // filler.hpp:381: N(0, sqrt(2/n))
    std::normal_distribution<float> g(0.f, std::sqrt(2.f / nval));
    for (size_t i = 0; i < n; ++i) d[i] = g(rng);
  } else if (f.type == "bilinear") {                   // filler.hpp BilinearFiller, as the modelled reference writes it:
    B2_CHECK(b->num_axes() == 4, "Blob must be 4 dim.");
    B2_CHECK(b->shape(3) == b->shape(2), "Filter must be square");
    const int k = b->shape(3);
    const int f2 = k / 2;                                // ceil(width / 2) with integer division: k / 2 for odd k too
    const float c = (2 * f2 - 1 - f2 % 2) / (2.f * f2);
    for (size_t i = 0; i < n; ++i) {
      const float x = (float)(i % k), y = (float)((i / k) % k);
      d[i] = (float)((1. - std::fabs(x / f2 - c)) * (1. - std::fabs(y / f2 - c)));
    }
  } else {
    B2_CHECK(false, "Unknown filler name: " + f.type);
  }
}

// ================================================================================================ Layer
void LayerBase::SetUp(const vector<Blob*>& bottom, const vector<Blob*>& top) {
  if (MinBottomBlobs() >= 0) B2_CHECK((int)bottom.size() >= MinBottomBlobs(), string(type()) + " Layer takes at least " + std::to_string(MinBottomBlobs()) + " bottom blob(s) as input.");
  if (MinTopBlobs() >= 0) B2_CHECK((int)top.size() >= MinTopBlobs(), string(type()) + " Layer produces at least " + std::to_string(MinTopBlobs()) + " top blob(s) as output.");
  if (EqualNumBottomTopBlobs()) B2_CHECK(bottom.size() == top.size(), string(type()) + " Layer produces one top blob as output for each bottom blob input.");
  LayerSetUp(bottom, top);
  Reshape(bottom, top);
}
float LayerBase::Forward(const vector<Blob*>& bottom, const vector<Blob*>& top) {
  Reshape(bottom, top);
  Forward_gpu(bottom, top);
  return 0.f;
}
void LayerBase::Backward(const vector<Blob*>& top, const vector<bool>& propagate_down, const vector<Blob*>& bottom) {
  Backward_gpu(top, propagate_down, bottom);
}

std::map<string, LayerRegistry::Creator>& LayerRegistry::Registry() {
  static std::map<string, Creator> r;
  return r;
}
void LayerRegistry::AddCreator(const string& type, Creator c) {
  B2_CHECK(Registry().count(type) == 0, "Layer type " + type + " already registered.");
  Registry()[type] = c;
}
shared_ptr<LayerBase> LayerRegistry::CreateLayer(const LayerParameter& p) {
  auto it = Registry().find(p.type);
  if (it == Registry().end()) {
    string known;
    for (auto& kv : Registry()) known += kv.first + " ";
    B2_CHECK(false, "Unknown layer type: " + p.type + " (known types: " + known + ")");
  }
  return it->second(p);
}
vector<string> LayerRegistry::LayerTypeList() {
  vector<string> v;
  for (auto& kv : Registry()) v.push_back(kv.first);
  return v;
}

// ================================================================================================ profiler
EventProfiler::~EventProfiler() { for (auto& r : recs_) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); } }
size_t EventProfiler::begin(int op, cudaStream_t st) {
  Rec r{layer_, op, nullptr, nullptr};
  CUDA_CHECK(cudaEventCreate(&r.a)); CUDA_CHECK(cudaEventCreate(&r.b));
  CUDA_CHECK(cudaEventRecord(r.a, st));
  recs_.push_back(r);
  return recs_.size() - 1;
}
void EventProfiler::end(size_t h, cudaStream_t st) { CUDA_CHECK(cudaEventRecord(recs_[h].b, st)); }
void EventProfiler::collect(std::map<std::pair<int, int>, float>* out) {
  CUDA_CHECK(cudaDeviceSynchronize());
  for (auto& r : recs_) {
    float ms = 0.f;
    CUDA_CHECK(cudaEventElapsedTime(&ms, r.a, r.b));
    (*out)[{r.layer, r.op}] += ms;
    cudaEventDestroy(r.a); cudaEventDestroy(r.b);
  }
  recs_.clear();
}

// ================================================================================================ Convolution
shared_ptr<LayerBase> GetConvolutionLayer(const LayerParameter& p) {
  // layer_factory.cpp:53-88: DEFAULT resolves to the implicit-GEMM ("CUDNN") engine unless the layer is
  // dilated, in which case the reference falls back to the CAFFE engine.  The implicit kernels here handle
  // dilation, so DEFAULT keeps them; an explicit `engine: CAFFE` still selects im2col + GEMM.
  return shared_ptr<LayerBase>(new ConvolutionLayer(p));
}
REGISTER_LAYER_CREATOR(Convolution, GetConvolutionLayer);

ConvolutionLayer::~ConvolutionLayer() {
  if (desc_) b2c_conv_desc_destroy(desc_);
  if (ws_) cudaFree(ws_);
  if (fcache_) cudaFree(fcache_);
}
bool ConvolutionLayer::EnableFilterCache() {
  fcache_on_ = true;
  if (!desc_) return false;
  const size_t need = b2c_conv_filter_cache_bytes(desc_);
  if (!need) { B2C_CHECK(b2c_conv_desc_bind_filter_cache(desc_, nullptr)); return false; }
  if (need > fcache_bytes_) {
    if (fcache_) CUDA_CHECK(cudaFree(fcache_));
    CUDA_CHECK(cudaMalloc(&fcache_, need));          // cudaMalloc: 256-byte aligned
    fcache_bytes_ = need;
  }
  B2C_CHECK(b2c_conv_desc_bind_filter_cache(desc_, fcache_));
  return true;
}

static void per_axis(const char* what, const vector<int>& rep, int h, int w, int naxes, int dflt, bool need, vector<int>* out) {
  out->assign(naxes, dflt);
  if (h >= 0 || w >= 0) {
    B2_CHECK(naxes == 2, string(what) + "_h & " + what + "_w can only be used for 2D convolution.");
    B2_CHECK(rep.empty(), string("Either ") + what + " or " + what + "_h/w should be specified; not both.");
    (*out)[0] = h; (*out)[1] = w;
    return;
  }
  const int nd = (int)rep.size();
  if (need) B2_CHECK(nd == 1 || nd == naxes, string(what) + " must be specified once, or once per spatial dimension");
  else B2_CHECK(nd == 0 || nd == 1 || nd == naxes, string(what) + " must be specified once, or once per spatial dimension");
  for (int i = 0; i < naxes; ++i)
    if (nd) (*out)[i] = rep[nd == 1 ? 0 : i];
}

void ConvolutionLayer::LayerSetUp(const vector<Blob*>& bottom, const vector<Blob*>& top) {
  const ConvolutionParameter& cp = layer_param_.convolution_param;
  channel_axis_ = bottom[0]->CanonicalAxisIndex(cp.axis);
  num_spatial_axes_ = bottom[0]->num_axes() - (channel_axis_ + 1);
  B2_CHECK(num_spatial_axes_ >= 1, "convolution needs at least one spatial axis");
  per_axis("kernel_size", cp.kernel_size, cp.kernel_h, cp.kernel_w, num_spatial_axes_, 0, true, &kernel_shape_);
  for (int k : kernel_shape_) B2_CHECK(k > 0, "Filter dimensions must be nonzero.");
  per_axis("stride", cp.stride, cp.stride_h, cp.stride_w, num_spatial_axes_, 1, false, &stride_);
  for (int s : stride_) B2_CHECK(s > 0, "Stride dimensions must be nonzero.");
  per_axis("pad", cp.pad, cp.pad_h, cp.pad_w, num_spatial_axes_, 0, false, &pad_);
  per_axis("dilation", cp.dilation, -1, -1, num_spatial_axes_, 1, false, &dilation_);
  is_1x1_ = true;
  for (int i = 0; i < num_spatial_axes_; ++i) is_1x1_ &= kernel_shape_[i] == 1 && stride_[i] == 1 && pad_[i] == 0;
  channels_ = bottom[0]->shape(channel_axis_);
  num_output_ = cp.num_output;
  B2_CHECK(num_output_ > 0, "num_output must be positive");
  group_ = cp.group;
  B2_CHECK(channels_ % group_ == 0, "channels not divisible by group");
  B2_CHECK(num_output_ % group_ == 0, "Number of output should be multiples of group.");
  vector<int> wshape = reverse_dimensions() ? vector<int>{channels_, num_output_ / group_} : vector<int>{num_output_, channels_ / group_};
  for (int k : kernel_shape_) wshape.push_back(k);
  bias_term_ = cp.bias_term;
  if (!blobs_.empty()) {
    B2_CHECK((int)blobs_.size() == 1 + (bias_term_ ? 1 : 0), "Incorrect number of weight blobs.");
    B2_CHECK(blobs_[0]->shape() == wshape, "Incorrect weight shape: expected " + Blob(wshape).shape_string() + "; instead, shape was " + blobs_[0]->shape_string());
    if (bias_term_) B2_CHECK(blobs_[1]->shape() == vector<int>{num_output_}, "Incorrect bias shape");
  } else {
    blobs_.resize(bias_term_ ? 2 : 1);
    blobs_[0].reset(new Blob(wshape));
    Fill(cp.weight_filler, blobs_[0].get());
    if (bias_term_) {
      blobs_[1].reset(new Blob(vector<int>{num_output_}));
      Fill(cp.bias_filler, blobs_[1].get());
    }
  }
  param_propagate_down_.resize(blobs_.size(), true);
}

void ConvolutionLayer::compute_output_shape() {
  output_shape_.clear();
  for (int i = 0; i < num_spatial_axes_; ++i) {
    const int in = bottom_shape_[channel_axis_ + 1 + i];
    const int ext = dilation_[i] * (kernel_shape_[i] - 1) + 1;
    output_shape_.push_back((in + 2 * pad_[i] - ext) / stride_[i] + 1);
  }
}

void ConvolutionLayer::Reshape(const vector<Blob*>& bottom, const vector<Blob*>& top) {
  const int first_spatial = channel_axis_ + 1;
  B2_CHECK(bottom[0]->num_axes() == first_spatial + num_spatial_axes_, "bottom num_axes may not change.");
  num_ = (int)bottom[0]->count(0, channel_axis_);
  B2_CHECK(bottom[0]->shape(channel_axis_) == channels_, "Input size incompatible with convolution kernel.");
  for (size_t i = 1; i < bottom.size(); ++i) B2_CHECK(bottom[0]->shape() == bottom[i]->shape(), "All inputs must have the same shape.");
  bottom_shape_ = bottom[0]->shape();
  compute_output_shape();
  vector<int> tshape(bottom_shape_.begin(), bottom_shape_.begin() + channel_axis_);
  tshape.push_back(num_output_);
  for (int o : output_shape_) { B2_CHECK(o > 0, "kernel larger than padded input"); tshape.push_back(o); }
  for (Blob* t : top) t->Reshape(tshape);
  if (num_spatial_axes_ == 2 && !layer_param_.convolution_param.force_nd_im2col) {
    b2c_conv_params p{num_, channels_, bottom_shape_[first_spatial], bottom_shape_[first_spatial + 1], num_output_, group_,
                      kernel_shape_[0], kernel_shape_[1], stride_[0], stride_[1], pad_[0], pad_[1], dilation_[0], dilation_[1],
                      bias_term_ ? 1 : 0};
    if (!desc_ || memcmp(&p, &desc_params_, sizeof(p)) != 0) {   // shapes may change between iterations
      if (desc_) b2c_conv_desc_destroy(desc_);
      desc_ = nullptr;
      B2C_CHECK(b2c_conv_desc_create(&p, layer_param_.convolution_param.engine, &desc_));
      B2C_CHECK(b2c_conv_desc_set_math(desc_, layer_param_.convolution_param.math));
      desc_params_ = p;
      if (fcache_on_) EnableFilterCache();           // new descriptor (shape change): re-bind; the owner re-prepares
    }
  }
}

void* ConvolutionLayer::workspace(size_t bytes) {
  if (bytes > ws_bytes_) {
    if (ws_) CUDA_CHECK(cudaFree(ws_));
    CUDA_CHECK(cudaMalloc(&ws_, bytes));
    ws_bytes_ = bytes;
  }
  return ws_;
}
int ConvolutionLayer::algo_used(int op) const { return desc_ ? b2c_conv_algo_used(desc_, op) : B2C_ALGO_SIMT; }

void ConvolutionLayer::Forward_gpu(const vector<Blob*>& bottom, const vector<Blob*>& top) {
  cudaStream_t st = Caffe::thread_stream();
  const float* w = blobs_[0]->gpu_data();
  const float* b = bias_term_ ? blobs_[1]->gpu_data() : nullptr;
  for (size_t i = 0; i < bottom.size(); ++i) {       // several bottom/top pairs share one weight set
    if (desc_) {
      const size_t need = b2c_conv_workspace_bytes(desc_, B2C_OP_FORWARD);
      void* ws = need ? workspace(need) : nullptr;     // (sequenced before ws_bytes_ is read)
      B2C_CHECK(b2c_conv_forward(desc_, bottom[i]->gpu_data(), w, b, top[i]->mutable_gpu_data(), ws, ws_bytes_, st));
      continue;
    }
    // N-D path: the literal per-image im2col_nd + GEMM of base_conv_layer.hpp:105-128
    vector<int> im_shape{channels_}, col_shape{(int)(blobs_[0]->count(1)) * group_};
    for (int a = 0; a < num_spatial_axes_; ++a) { im_shape.push_back(bottom_shape_[channel_axis_ + 1 + a]); col_shape.push_back(output_shape_[a]); }
    size_t P = 1;
    for (int o : output_shape_) P *= (size_t)o;
    const int Kd = (int)blobs_[0]->count(1), Og = num_output_ / group_;
    float* col = static_cast<float*>(workspace(sizeof(float) * (size_t)Kd * group_ * P));
    const size_t bdim = bottom[i]->count(channel_axis_), tdim = top[i]->count(channel_axis_);
    for (int n = 0; n < num_; ++n) {
      B2C_CHECK(b2c_im2col_nd(bottom[i]->gpu_data() + n * bdim, num_spatial_axes_, im_shape.data(), col_shape.data(), kernel_shape_.data(),
                              pad_.data(), stride_.data(), dilation_.data(), col, st));
      for (int g = 0; g < group_; ++g)
        B2C_CHECK(b2c_sgemm(0, 0, Og, (int)P, Kd, 1.f, w + (size_t)g * Og * Kd, col + (size_t)g * Kd * P, 0.f,
                            top[i]->mutable_gpu_data() + n * tdim + (size_t)g * Og * P, st));
      if (b) {
        // y_n += bias x ones: rank-1 update expressed as GEMM with K = 1 against a ones row held in `col`'s tail
        // (base_conv_layer.hpp:122-128); done with sgemv-free broadcast: C = bias[Ox1] * ones[1xP] + C
        static thread_local float* ones = nullptr;
        static thread_local size_t ones_n = 0;
        if (ones_n < P) {
          if (ones) cudaFree(ones);
          CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&ones), sizeof(float) * P));
          vector<float> h(P, 1.f);
          CUDA_CHECK(cudaMemcpy(ones, h.data(), sizeof(float) * P, cudaMemcpyHostToDevice));
          ones_n = P;
        }
        B2C_CHECK(b2c_sgemm(0, 0, num_output_, (int)P, 1, 1.f, b, ones, 1.f, top[i]->mutable_gpu_data() + n * tdim, st));
      }
    }
  }
}

void ConvolutionLayer::Backward_gpu(const vector<Blob*>& top, const vector<bool>& propagate_down, const vector<Blob*>& bottom) {
  cudaStream_t st = Caffe::thread_stream();
  const float* w = blobs_[0]->gpu_data();
  for (size_t i = 0; i < top.size(); ++i) {
    const float* dy = top[i]->gpu_diff();
    if (desc_) {
      if (bias_term_ && param_propagate_down_[1]) B2C_CHECK(b2c_conv_backward_bias(desc_, dy, blobs_[1]->mutable_gpu_diff(), st));
      EventProfiler* prof = Caffe::profiler();
      if (param_propagate_down_[0]) {
        // [the kernel's workspace | the buffer its operands are split into], both 256-byte aligned
        const size_t need = (b2c_conv_workspace_bytes(desc_, B2C_OP_BACKWARD_FILTER) + 255) & ~(size_t)255;
        // (only the tensor-core weight-gradient kernels take a split buffer)
        const size_t split = algo_used(B2C_OP_BACKWARD_FILTER) == B2C_ALGO_TCGEN05 ? b2c_conv_wgrad_split_bytes(desc_) : 0;
        char* ws = need + split ? static_cast<char*>(workspace(need + split)) : nullptr;
        const size_t h = prof ? prof->begin(EventProfiler::WGRAD, st) : 0;
        if (split)
          B2C_CHECK(b2c_conv_backward_filter_split(desc_, bottom[i]->gpu_data(), dy, blobs_[0]->mutable_gpu_diff(), ws, need, ws + need, split, st));
        else
          B2C_CHECK(b2c_conv_backward_filter(desc_, bottom[i]->gpu_data(), dy, blobs_[0]->mutable_gpu_diff(), ws, need, st));
        if (prof) prof->end(h, st);
      }
      if (propagate_down[i]) {
        const size_t need = b2c_conv_workspace_bytes(desc_, B2C_OP_BACKWARD_DATA);
        void* ws = need ? workspace(need) : nullptr;
        const size_t h = prof ? prof->begin(EventProfiler::DGRAD, st) : 0;
        if (i < accumulate_bottom_.size() && accumulate_bottom_[i])
          B2C_CHECK(b2c_conv_backward_data_accumulate(desc_, dy, w, bottom[i]->mutable_gpu_diff(), ws, ws_bytes_, st));
        else
          B2C_CHECK(b2c_conv_backward_data(desc_, dy, w, bottom[i]->mutable_gpu_diff(), ws, ws_bytes_, st));
        if (prof) prof->end(h, st);
      }
      continue;
    }
    // N-D path (base_conv_layer.hpp:130-168)
    vector<int> im_shape{channels_}, col_shape{(int)(blobs_[0]->count(1)) * group_};
    for (int a = 0; a < num_spatial_axes_; ++a) { im_shape.push_back(bottom_shape_[channel_axis_ + 1 + a]); col_shape.push_back(output_shape_[a]); }
    size_t P = 1;
    for (int o : output_shape_) P *= (size_t)o;
    const int Kd = (int)blobs_[0]->count(1), Og = num_output_ / group_;
    float* col = static_cast<float*>(workspace(sizeof(float) * ((size_t)Kd * group_ * P + P)));
    float* ones = col + (size_t)Kd * group_ * P;
    {
      vector<float> h(P, 1.f);
      CUDA_CHECK(cudaMemcpyAsync(ones, h.data(), sizeof(float) * P, cudaMemcpyHostToDevice, st));
      CUDA_CHECK(cudaStreamSynchronize(st));
    }
    const size_t bdim = bottom[i]->count(channel_axis_), tdim = top[i]->count(channel_axis_);
    if (bias_term_ && param_propagate_down_[1])
      for (int n = 0; n < num_; ++n)
        B2C_CHECK(b2c_sgemv(0, num_output_, (int)P, 1.f, dy + n * tdim, ones, 1.f, blobs_[1]->mutable_gpu_diff(), st));
    for (int n = 0; n < num_; ++n) {
      if (param_propagate_down_[0]) {
        B2C_CHECK(b2c_im2col_nd(bottom[i]->gpu_data() + n * bdim, num_spatial_axes_, im_shape.data(), col_shape.data(), kernel_shape_.data(),
                                pad_.data(), stride_.data(), dilation_.data(), col, st));
        for (int g = 0; g < group_; ++g)
          B2C_CHECK(b2c_sgemm(0, 1, Og, Kd, (int)P, 1.f, dy + n * tdim + (size_t)g * Og * P, col + (size_t)g * Kd * P, 1.f,
                              blobs_[0]->mutable_gpu_diff() + (size_t)g * Og * Kd, st));
      }
      if (propagate_down[i]) {
        for (int g = 0; g < group_; ++g)
          B2C_CHECK(b2c_sgemm(1, 0, Kd, (int)P, Og, 1.f, w + (size_t)g * Og * Kd, dy + n * tdim + (size_t)g * Og * P, 0.f,
                              col + (size_t)g * Kd * P, st));
        B2C_CHECK(b2c_col2im_nd(col, num_spatial_axes_, im_shape.data(), col_shape.data(), kernel_shape_.data(), pad_.data(),
                                stride_.data(), dilation_.data(), bottom[i]->mutable_gpu_diff() + n * bdim, st));
      }
    }
  }
}

// ================================================================================================ Deconvolution
static shared_ptr<LayerBase> GetDeconvolutionLayer(const LayerParameter& p) { return shared_ptr<LayerBase>(new DeconvolutionLayer(p)); }
REGISTER_LAYER_CREATOR(Deconvolution, GetDeconvolutionLayer);

DeconvolutionLayer::~DeconvolutionLayer() { if (ddesc_) b2c_deconv_desc_destroy(ddesc_); }

void DeconvolutionLayer::compute_output_shape() {   // deconv_layer.cpp:7-22
  output_shape_.clear();
  for (int i = 0; i < num_spatial_axes_; ++i) {
    const int in = bottom_shape_[channel_axis_ + 1 + i];
    const int ext = dilation_[i] * (kernel_shape_[i] - 1) + 1;
    output_shape_.push_back(stride_[i] * (in - 1) + ext - 2 * pad_[i]);
  }
}

void DeconvolutionLayer::Reshape(const vector<Blob*>& bottom, const vector<Blob*>& top) {
  const int first_spatial = channel_axis_ + 1;
  B2_CHECK(bottom[0]->num_axes() == first_spatial + num_spatial_axes_, "bottom num_axes may not change.");
  num_ = (int)bottom[0]->count(0, channel_axis_);
  B2_CHECK(bottom[0]->shape(channel_axis_) == channels_, "Input size incompatible with convolution kernel.");
  for (size_t i = 1; i < bottom.size(); ++i) B2_CHECK(bottom[0]->shape() == bottom[i]->shape(), "All inputs must have the same shape.");
  bottom_shape_ = bottom[0]->shape();
  compute_output_shape();
  vector<int> tshape(bottom_shape_.begin(), bottom_shape_.begin() + channel_axis_);
  tshape.push_back(num_output_);
  for (int o : output_shape_) { B2_CHECK(o > 0, "Deconvolution: non-positive output extent (pad larger than the upsampled input)"); tshape.push_back(o); }
  for (Blob* t : top) t->Reshape(tshape);
  if (num_spatial_axes_ == 2 && !layer_param_.convolution_param.force_nd_im2col) {
    b2c_conv_params p{num_, channels_, bottom_shape_[first_spatial], bottom_shape_[first_spatial + 1], num_output_, group_,
                      kernel_shape_[0], kernel_shape_[1], stride_[0], stride_[1], pad_[0], pad_[1], dilation_[0], dilation_[1],
                      bias_term_ ? 1 : 0};
    if (!ddesc_ || memcmp(&p, &ddesc_params_, sizeof(p)) != 0) {
      if (ddesc_) b2c_deconv_desc_destroy(ddesc_);
      ddesc_ = nullptr;
      B2C_CHECK(b2c_deconv_desc_create(&p, layer_param_.convolution_param.engine, &ddesc_));
      B2C_CHECK(b2c_deconv_desc_set_math(ddesc_, layer_param_.convolution_param.math));
      ddesc_params_ = p;
    }
  }
}

// N-D helpers: the top is the dual convolution's "image" [O, top spatial], the col buffer [Kd*G, bottom spatial] with
// Kd = (O/G)*prod(k) (BaseConvolutionLayer with reverse_dimensions: conv_in_channels_ = O, conv_out_channels_ = C)
void DeconvolutionLayer::Forward_gpu(const vector<Blob*>& bottom, const vector<Blob*>& top) {
  cudaStream_t st = Caffe::thread_stream();
  const float* w = blobs_[0]->gpu_data();
  const float* b = bias_term_ ? blobs_[1]->gpu_data() : nullptr;
  for (size_t i = 0; i < bottom.size(); ++i) {
    if (ddesc_) {
      const size_t need = b2c_deconv_workspace_bytes(ddesc_, B2C_OP_FORWARD);
      void* ws = need ? workspace(need) : nullptr;
      B2C_CHECK(b2c_deconv_forward(ddesc_, bottom[i]->gpu_data(), w, b, top[i]->mutable_gpu_data(), ws, ws_bytes_, st));
      continue;
    }
    // deconv_layer.cu Forward_gpu: backward_gpu_gemm (GEMM + col2im_nd) per image, then the bias (one add per element)
    vector<int> im_shape{num_output_}, col_shape{(int)blobs_[0]->count(1) * group_};
    size_t Pb = 1, Pt = 1;
    for (int a = 0; a < num_spatial_axes_; ++a) {
      im_shape.push_back(output_shape_[a]); col_shape.push_back(bottom_shape_[channel_axis_ + 1 + a]);
      Pb *= (size_t)bottom_shape_[channel_axis_ + 1 + a]; Pt *= (size_t)output_shape_[a];
    }
    const int Kd = (int)blobs_[0]->count(1), Cg = channels_ / group_;
    float* col = static_cast<float*>(workspace(sizeof(float) * (size_t)Kd * group_ * Pb));
    const size_t bdim = bottom[i]->count(channel_axis_), tdim = top[i]->count(channel_axis_);
    for (int n = 0; n < num_; ++n) {
      for (int g = 0; g < group_; ++g)
        B2C_CHECK(b2c_sgemm(1, 0, Kd, (int)Pb, Cg, 1.f, w + (size_t)g * Cg * Kd, bottom[i]->gpu_data() + n * bdim + (size_t)g * Cg * Pb, 0.f,
                            col + (size_t)g * Kd * Pb, st));
      B2C_CHECK(b2c_col2im_nd(col, num_spatial_axes_, im_shape.data(), col_shape.data(), kernel_shape_.data(), pad_.data(), stride_.data(),
                              dilation_.data(), top[i]->mutable_gpu_data() + n * tdim, st));
    }
    if (b) B2C_CHECK(b2c_bias_forward(num_, num_output_, (int)Pt, b, top[i]->mutable_gpu_data(), st));
  }
}

void DeconvolutionLayer::Backward_gpu(const vector<Blob*>& top, const vector<bool>& propagate_down, const vector<Blob*>& bottom) {
  cudaStream_t st = Caffe::thread_stream();
  const float* w = blobs_[0]->gpu_data();
  for (size_t i = 0; i < top.size(); ++i) {
    const float* dy = top[i]->gpu_diff();
    if (ddesc_) {
      if (bias_term_ && param_propagate_down_[1]) B2C_CHECK(b2c_deconv_backward_bias(ddesc_, dy, blobs_[1]->mutable_gpu_diff(), st));
      if (param_propagate_down_[0]) {
        const size_t need = (b2c_deconv_workspace_bytes(ddesc_, B2C_OP_BACKWARD_FILTER) + 255) & ~(size_t)255;
        const size_t split = b2c_deconv_wgrad_split_bytes(ddesc_);
        char* ws = need + split ? static_cast<char*>(workspace(need + split)) : nullptr;
        B2C_CHECK(b2c_deconv_backward_filter_split(ddesc_, bottom[i]->gpu_data(), dy, blobs_[0]->mutable_gpu_diff(), ws, need,
                                                   split ? ws + need : nullptr, split, st));
      }
      if (propagate_down[i]) {
        const size_t need = b2c_deconv_workspace_bytes(ddesc_, B2C_OP_BACKWARD_DATA);
        void* ws = need ? workspace(need) : nullptr;
        B2C_CHECK(b2c_deconv_backward_data(ddesc_, dy, w, bottom[i]->mutable_gpu_diff(), ws, ws_bytes_, st));
      }
      continue;
    }
    // deconv_layer.cu Backward_gpu: bias gradient; per image im2col_nd of the top diff, then the weight GEMM
    // (weight_gpu_gemm(top_diff, bottom_data)) and the bottom GEMM (forward_gpu_gemm(top_diff, weights))
    vector<int> im_shape{num_output_}, col_shape{(int)blobs_[0]->count(1) * group_};
    size_t Pb = 1, Pt = 1;
    for (int a = 0; a < num_spatial_axes_; ++a) {
      im_shape.push_back(output_shape_[a]); col_shape.push_back(bottom_shape_[channel_axis_ + 1 + a]);
      Pb *= (size_t)bottom_shape_[channel_axis_ + 1 + a]; Pt *= (size_t)output_shape_[a];
    }
    const int Kd = (int)blobs_[0]->count(1), Cg = channels_ / group_;
    float* col = static_cast<float*>(workspace(sizeof(float) * (size_t)Kd * group_ * Pb));
    const size_t bdim = bottom[i]->count(channel_axis_), tdim = top[i]->count(channel_axis_);
    if (bias_term_ && param_propagate_down_[1]) B2C_CHECK(b2c_bias_backward(num_, num_output_, (int)Pt, dy, blobs_[1]->mutable_gpu_diff(), st));
    if (!param_propagate_down_[0] && !propagate_down[i]) continue;
    for (int n = 0; n < num_; ++n) {
      B2C_CHECK(b2c_im2col_nd(dy + n * tdim, num_spatial_axes_, im_shape.data(), col_shape.data(), kernel_shape_.data(), pad_.data(),
                              stride_.data(), dilation_.data(), col, st));
      for (int g = 0; g < group_; ++g) {
        if (param_propagate_down_[0])
          B2C_CHECK(b2c_sgemm(0, 1, Cg, Kd, (int)Pb, 1.f, bottom[i]->gpu_data() + n * bdim + (size_t)g * Cg * Pb, col + (size_t)g * Kd * Pb,
                              1.f, blobs_[0]->mutable_gpu_diff() + (size_t)g * Cg * Kd, st));
        if (propagate_down[i])
          B2C_CHECK(b2c_sgemm(0, 0, Cg, (int)Pb, Kd, 1.f, w + (size_t)g * Cg * Kd, col + (size_t)g * Kd * Pb, 0.f,
                              bottom[i]->mutable_gpu_diff() + n * bdim + (size_t)g * Cg * Pb, st));
      }
    }
  }
}

// ================================================================================================ arena
ParamArena::~ParamArena() {
  if (data_) cudaFree(data_);
  if (diff_) { if (diff_nccl_) b2c_comm_mem_free(diff_); else cudaFree(diff_); }
  if (hist_) cudaFree(hist_);
  if (hist2_) cudaFree(hist2_);
}
void ParamArena::InitLayout(const vector<size_t>& counts) {
  offset_.clear(); count_.clear();
  size_t off = 0;
  for (size_t c : counts) { offset_.push_back(off); count_.push_back(c); off += even(c); }
  total_ = off;
}
void ParamArena::Init(const vector<shared_ptr<Blob>>& params, bool second_history) {
  B2_CHECK(!data_, "arena already initialised");
  offset_.clear(); count_.clear();
  size_t off = 0;
  for (auto& b : params) {
    offset_.push_back(off);
    count_.push_back(b->count());
    off += even(b->count());
  }
  total_ = off;
  const size_t bytes = sizeof(float) * (total_ ? total_ : 1);
  CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&data_), bytes));
  // the diff arena is what the gradient allreduce runs on: allocate it with ncclMemAlloc so that, once registered with the
  // communicator (P2PSync::on_start), NCCL can reduce it inside the NVSwitch (NVLS) in place.  B2C_NCCL_ARENA=0: cudaMalloc.
  {
    const char* e = getenv("B2C_NCCL_ARENA");
    if ((!e || atoi(e) != 0) && b2c_comm_mem_alloc(reinterpret_cast<void**>(&diff_), bytes) == B2C_OK) diff_nccl_ = true;
    else { diff_ = nullptr; CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&diff_), bytes)); }
  }
  CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&hist_), bytes));
  CUDA_CHECK(cudaMemset(data_, 0, bytes));
  CUDA_CHECK(cudaMemset(diff_, 0, bytes));     // net.cpp:1367
  CUDA_CHECK(cudaMemset(hist_, 0, bytes));
  if (second_history) {
    CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&hist2_), bytes));
    CUDA_CHECK(cudaMemset(hist2_, 0, bytes));
  }
  for (size_t i = 0; i < params.size(); ++i) {
    params[i]->set_gpu_data(data_ + offset_[i]);
    params[i]->set_gpu_diff(diff_ + offset_[i]);
  }
}

// ================================================================================================ solver
int SolverKind(const string& type) {
  static const char* const names[] = {"SGD", "Nesterov", "AdaGrad", "RMSProp", "AdaDelta", "Adam"};   // b2c_solver_kind order
  for (int k = 0; k < 6; ++k) if (type == names[k]) return k;
  Fatal(__FILE__, __LINE__, "Unknown solver type: " + type + " (known types: SGD, Nesterov, AdaGrad, RMSProp, AdaDelta, Adam)");
}
void CheckSolverParameter(const SolverParameter& p) {
  const int k = SolverKind(p.type);
  if (k == B2C_SOLVER_ADAGRAD) B2_CHECK(p.momentum == 0.f, "Momentum cannot be used with AdaGrad.");
  if (k == B2C_SOLVER_RMSPROP) {
    B2_CHECK(p.momentum == 0.f, "Momentum cannot be used with RMSProp.");
    B2_CHECK(p.rms_decay >= 0.f && p.rms_decay < 1.f, "rms_decay should lie between 0 and 1.");
  }
}
float SGDSolver::GetLearningRate() {
  const SolverParameter& p = param_;
  if (iter_ < p.rampup_interval) {
    const float alpha = float(iter_) / p.rampup_interval;
    return p.rampup_lr + (p.base_lr - p.rampup_lr) * alpha;
  }
  const string& pol = p.lr_policy;
  if (pol == "fixed") return p.base_lr;
  if (pol == "step") {
    B2_CHECK(p.stepsize > 0, "lr_policy \"step\" needs a positive stepsize");      // the reference divides by it unchecked (sgd_solver.cpp:40)
    current_step_ = iter_ / p.stepsize;
    return p.base_lr * std::pow(p.gamma, (float)current_step_);
  }
  if (pol == "exp") return p.base_lr * std::pow(p.gamma, (float)iter_);
  if (pol == "inv") return p.base_lr * std::pow(1.f + p.gamma * float(iter_), -p.power);
  if (pol == "multistep") {
    if (current_step_ < (int)p.stepvalue.size() && iter_ >= p.stepvalue[current_step_]) ++current_step_;
    return p.base_lr * std::pow(p.gamma, (float)current_step_);
  }
  if (pol == "poly") return p.min_lr + (p.base_lr - p.min_lr) * std::pow(1.f - (float(iter_) / float(p.max_iter)), p.power);
  if (pol == "sigmoid") return p.base_lr / (1.f + (float)std::exp(-(double)p.gamma * (double)(iter_ - p.stepsize)));
  B2_CHECK(false, "Unknown learning rate policy: " + pol);
}
float SGDSolver::GetMomentum() {
  const SolverParameter& p = param_;
  if (p.momentum_policy == "fixed") return p.momentum;
  if (p.momentum_policy == "poly")
    return p.momentum + (p.max_momentum - p.momentum) * std::pow(float(iter_) / float(p.max_iter), p.momentum_power);
  if (p.momentum_policy == "opt") {
    // as the reference: a float square root, the square in double, and a clamp only when max_momentum is given
    const float lr = GetLearningRate();
    const double r = 1. - 0.5 * std::sqrt(lr);
    const float m = (float)(r * r);
    return p.has_max_momentum ? std::min(p.max_momentum, m) : m;
  }
  B2_CHECK(false, "Unknown momentum policy: " + p.momentum_policy);
}
SGDSolver::~SGDSolver() {
  if (clip_partials_) cudaFree(clip_partials_);
  if (clip_state_) cudaFree(clip_state_);
}
void SGDSolver::SetParams(const vector<shared_ptr<Blob>>& params, const vector<ParamSpec>& specs) {
  B2_CHECK(params.size() == specs.size(), "one ParamSpec per learnable blob");
  specs_ = specs;
  arena_.Init(params, num_histories() == 2);
  if (clipping()) {
    vector<size_t> counts;
    for (int i = 0; i < arena_.size(); ++i) counts.push_back(arena_.count(i));
    clip_nslots_ = ClipSlots(counts, &clip_slot_);
    CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&clip_partials_), sizeof(double) * (clip_nslots_ ? clip_nslots_ : 1)));
    CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&clip_state_), sizeof(b2c_clip_state)));
    CUDA_CHECK(cudaMemset(clip_state_, 0, sizeof(b2c_clip_state)));
  }
}
void SGDSolver::set_clip_gradients(float clip) {
  B2_CHECK(arena_.size() == 0 && !arena_.data(), "clip_gradients must be set before the solver's parameters");
  param_.clip_gradients = clip;
}
size_t SGDSolver::ClipSlots(const vector<size_t>& counts, vector<size_t>* slot) {
  slot->clear();
  size_t n = 0;
  for (size_t c : counts) {
    slot->push_back(n);
    n += (c + B2C_SUMSQ_BLOCK_ELEMS - 1) / B2C_SUMSQ_BLOCK_ELEMS;
  }
  return n;
}
void SGDSolver::ClipNorm(int id_from, int id_to, cudaStream_t stream) {
  B2_CHECK(clip_state_, "ClipNorm without clip_gradients");
  if (id_to < id_from) return;
  // every param, BatchNorm statistics included: their diffs stay 0, so they add exact zeros and keep the slots contiguous
  vector<size_t> off, cnt, slot;
  for (int id = id_from; id <= id_to; ++id) {
    off.push_back(arena_.offset(id)); cnt.push_back(arena_.count(id)); slot.push_back(clip_slot_[id]);
  }
  B2C_CHECK(b2c_arena_sumsq((int)off.size(), off.data(), cnt.data(), slot.data(), arena_.diff(), clip_partials_, stream));
}
void SGDSolver::ClipFactor(cudaStream_t stream) {
  B2_CHECK(clip_state_, "ClipFactor without clip_gradients");
  // the scale the net applies before ClipGradients (net.cpp:815-817,910); Normalize's 1/iter_size comes after it
  const double s_n = 1.0 / ((double)Caffe::solver_count() * (double)param_.global_grad_scale);
  B2C_CHECK(b2c_clip_factor(clip_partials_, clip_nslots_, s_n, param_.clip_gradients, clip_state_, stream));
}
b2c_clip_state SGDSolver::ClipState() {
  B2_CHECK(clipping(), "the solver does not clip gradients (clip_gradients < 0)");
  B2_CHECK(clip_state_, "the solver clips gradients but has no parameters yet");
  b2c_clip_state st;
  CUDA_CHECK(cudaDeviceSynchronize());
  CUDA_CHECK(cudaMemcpy(&st, clip_state_, sizeof(st), cudaMemcpyDeviceToHost));
  return st;
}
void SGDSolver::ApplyUpdate(int id_from, int id_to, cudaStream_t stream) {
  B2_CHECK(!clipping() || (id_from == 0 && id_to == arena_.size() - 1),
           "with clip_gradients the update covers the whole arena: every parameter takes the one global factor");
  B2_CHECK(param_.regularization_type == "L2" || param_.regularization_type == "L1", "Unknown regularization type");
  const float rate = GetLearningRate();
  // SGD keeps its momentum policy; Nesterov, AdaDelta and Adam (as beta1) read param_.momentum() directly
  // (nesterov_solver.cpp:22, adadelta_solver.cpp:37, adam_solver.cpp:33)
  const float momentum = kind_ == B2C_SOLVER_SGD ? GetMomentum() : param_.momentum;
  // Adam's bias correction, folded into every segment's rate (adam_solver.cpp:42-43)
  float correction = 1.f;
  if (kind_ == B2C_SOLVER_ADAM) {
    const float t = (float)(iter_ + 1);
    correction = std::sqrt(1.f - std::pow(param_.momentum2, t)) / (1.f - std::pow(param_.momentum, t));
  }
  if (id_to < id_from) return;
  vector<size_t> off, cnt;
  vector<float> lr, dc;
  for (int id = id_from; id <= id_to; ++id) {
    const float l = rate * specs_[id].lr_mult;                        // sgd_solver.cpp:208-210
    const float d = param_.weight_decay * specs_[id].decay_mult;      // :254-259
    // lr_mult = decay_mult = 0 (BatchNorm statistics, batch_norm_layer.cpp): the diff is never written, so it stays 0 and
    // gr = 0; every rule then leaves its histories at 0 and steps by u = 0 (each delta is clamped positive, so no 0/0), so
    // the update is the identity for every solver type -- left out of the fused launch
    if (specs_[id].statistic && l == 0.f && d == 0.f) continue;
    off.push_back(arena_.offset(id)); cnt.push_back(arena_.count(id)); lr.push_back(kind_ == B2C_SOLVER_ADAM ? l * correction : l);
    dc.push_back(d);
  }
  const int n = (int)off.size();
  if (n == 0) return;
  const float grad_scale = 1.f / (float)Caffe::solver_count() / param_.global_grad_scale / (float)param_.iter_size;
  const int l2 = param_.regularization_type == "L2" ? 1 : 0, clear = param_.snapshot_diff ? 0 : 1;
  b2c_solver_hparams hp;
  hp.momentum = momentum; hp.delta = param_.delta; hp.rms_decay = param_.rms_decay; hp.beta1 = param_.momentum; hp.beta2 = param_.momentum2;
  if (clipping()) {
    B2C_CHECK(b2c_solver_update_arena_scaled(kind_, n, off.data(), cnt.data(), lr.data(), dc.data(), arena_.diff(), arena_.data(),
                                             arena_.history(), arena_.history2(), hp, l2, grad_scale, &clip_state_->factor, clear, stream));
    return;
  }
  if (kind_ == B2C_SOLVER_SGD) {
    B2C_CHECK(b2c_sgd_update_arena(n, off.data(), cnt.data(), lr.data(), dc.data(), arena_.diff(), arena_.data(), arena_.history(),
                                   momentum, l2, grad_scale, clear, stream));
    return;
  }
  B2C_CHECK(b2c_solver_update_arena(kind_, n, off.data(), cnt.data(), lr.data(), dc.data(), arena_.diff(), arena_.data(), arena_.history(),
                                    arena_.history2(), hp, l2, grad_scale, clear, stream));
}

// The streaming bucket logic of Net::ReduceAndUpdate (net.cpp:772-783,824-862), replayed over an arrival order.
static void bucket_walk(const ParamArena& a, int reduce_buckets, const vector<int>& arrival,
                        const std::function<void(int, int)>& flush) {
  const int np = a.size();
  if (np == 0) return;
  B2_CHECK(reduce_buckets > 0, "reduce_buckets must be positive");
  int max_params_per_bucket = (np + 1) / reduce_buckets;
  if (max_params_per_bucket < 1) max_params_per_bucket = 1;
  const size_t bucket_space_count = (size_t)((float)(a.total() + 1) / np * max_params_per_bucket);
  int id_from = -1, id_to = -1;
  size_t received = 0;
  for (int pid : arrival) {
    if (received >= bucket_space_count || (id_from != -1 && pid < id_from - 1) || (id_to != -1 && pid > id_to + 1)) {
      if (id_from != -1) flush(id_from, id_to);
      id_from = id_to = pid;
      received = even(a.count(pid));
    } else {
      if (id_from == -1 || pid < id_from) id_from = pid;
      if (id_to == -1 || pid > id_to) id_to = pid;
      received += even(a.count(pid));
    }
  }
  if (id_from != -1) flush(id_from, id_to);     // END_OF_ITERATION leftovers
}
vector<Bucket> PlanBuckets(const ParamArena& a, int reduce_buckets) {
  vector<int> arrival;
  for (int i = a.size() - 1; i >= 0; --i) arrival.push_back(i);
  vector<Bucket> out;
  bucket_walk(a, reduce_buckets, arrival, [&](int f, int t) {
    size_t cnt = 0;
    for (int i = f; i <= t; ++i) cnt += even(a.count(i));
    out.push_back(Bucket{f, t, a.offset(f), cnt});
  });
  return out;
}

// ================================================================================================ P2PSync
P2PSync::P2PSync(int nranks, int rank, const BcastBytes& bcast) : nranks_(nranks), rank_(rank) {
  unsigned char id[B2C_UNIQUE_ID_BYTES];
  if (rank == 0) B2C_CHECK(b2c_comm_get_unique_id(id));
  bcast(id, sizeof(id), 0);                      // MPI_Bcast(&nccl_id) in the reference (parallel.cpp:45)
  B2C_CHECK(b2c_comm_init(nranks, rank, id, &comm_));
  int lo = 0, hi = 0;
  CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
  CUDA_CHECK(cudaStreamCreateWithPriority(&comm_stream_, cudaStreamNonBlocking, hi));   // parallel.cpp:119-132
  Caffe::set_solver_count(nranks);
  Caffe::set_root_solver(rank == 0);
}
P2PSync::~P2PSync() {
  if (comm_) b2c_comm_destroy(comm_);
  if (comm_stream_) cudaStreamDestroy(comm_stream_);
}
void P2PSync::on_start(ParamArena& arena) {
  // the reference broadcasts blob by blob; the arena makes it one call.  The comm stream knows nothing of the compute stream yet (the
  // per-iteration events come later): whatever filled or uploaded the parameters there must have landed before they travel.
  CUDA_CHECK(cudaStreamSynchronize(Caffe::thread_stream()));
  B2C_CHECK(b2c_comm_bcast(comm_, arena.data(), arena.total(), 0, comm_stream_));
  CUDA_CHECK(cudaStreamSynchronize(comm_stream_));
  if (arena.diff_is_nccl_memory()) {
    // user-buffer registration of the whole diff arena (every bucket is a sub-range of it); a failure only costs the
    // zero-copy path, so it is reported on stderr and training goes on
    if (b2c_comm_register(comm_, arena.diff(), sizeof(float) * arena.total()) != B2C_OK)
      fprintf(stderr, "P2PSync: ncclCommRegister of the diff arena failed (%s); continuing unregistered\n", b2c_last_error());
  }
}
void P2PSync::allreduce_bucket(float* buf, size_t count) {
  if (!timing_) { B2C_CHECK(b2c_comm_allreduce_sum(comm_, buf, count, comm_stream_)); return; }
  TimedBucket t{sizeof(float) * count, nullptr, nullptr};
  CUDA_CHECK(cudaEventCreate(&t.a)); CUDA_CHECK(cudaEventCreate(&t.b));
  CUDA_CHECK(cudaEventRecord(t.a, comm_stream_));
  B2C_CHECK(b2c_comm_allreduce_sum(comm_, buf, count, comm_stream_));
  CUDA_CHECK(cudaEventRecord(t.b, comm_stream_));
  timed_.push_back(t);
}
void P2PSync::allreduce_scores(float* buf, size_t count) { B2C_CHECK(b2c_comm_allreduce_sum(comm_, buf, count, comm_stream_)); }
void P2PSync::collect_bucket_times(vector<size_t>* bytes, vector<float>* ms) {
  CUDA_CHECK(cudaStreamSynchronize(comm_stream_));
  for (TimedBucket& t : timed_) {
    float v = 0.f;
    CUDA_CHECK(cudaEventElapsedTime(&v, t.a, t.b));
    bytes->push_back(t.bytes); ms->push_back(v);
    cudaEventDestroy(t.a); cudaEventDestroy(t.b);
  }
  timed_.clear();
}
int P2PSync::divide_batch_size(int total, int solver_count) {
  // parallel.cpp:284-293: total/solver_count, rounded up so that no sample is dropped
  int b = total / solver_count;
  if (total % solver_count) ++b;
  return b;
}

// ================================================================================================ scheduler
void P2PSync::soft_barrier() { CUDA_CHECK(cudaStreamSynchronize(comm_stream_)); }
void P2PSync::reduce_barrier() { CUDA_CHECK(cudaStreamSynchronize(comm_stream_)); }

ReduceScheduler::ReduceScheduler(SGDSolver* solver, SolverCallback* sync) : solver_(solver), sync_(sync) {
  buckets_ = PlanBuckets(solver->arena(), solver->param().reduce_buckets);
  CUDA_CHECK(cudaEventCreateWithFlags(&ev_ready_, cudaEventDisableTiming));
  CUDA_CHECK(cudaEventCreateWithFlags(&ev_done_, cudaEventDisableTiming));
  if (!sync_) CUDA_CHECK(cudaStreamCreateWithFlags(&update_stream_, cudaStreamNonBlocking));
}
ReduceScheduler::~ReduceScheduler() {
  if (ev_ready_) cudaEventDestroy(ev_ready_);
  if (ev_done_) cudaEventDestroy(ev_done_);
  if (update_stream_) cudaStreamDestroy(update_stream_);
}
void ReduceScheduler::flush(int b, cudaStream_t compute) {
  const Bucket& bk = buckets_[b];
  cudaStream_t side = sync_ ? sync_->comm_stream() : update_stream_;
  CUDA_CHECK(cudaEventRecord(ev_ready_, compute));           // diffs of this bucket are complete on `compute`
  CUDA_CHECK(cudaStreamWaitEvent(side, ev_ready_, 0));
  if (sync_) sync_->allreduce_bucket(solver_->arena().diff() + bk.offset, bk.count);
  if (solver_->clipping()) solver_->ClipNorm(bk.id_from, bk.id_to, side);   // the update waits for the global norm
  else solver_->ApplyUpdate(bk.id_from, bk.id_to, side);     // chained on the same side stream
}
void ReduceScheduler::on_param_ready(int id, cudaStream_t compute) {
  while (next_bucket_ < (int)buckets_.size() && id <= buckets_[next_bucket_].id_from) {
    flush(next_bucket_, compute);
    ++next_bucket_;
  }
}
void ReduceScheduler::end_of_iteration(cudaStream_t compute) {
  while (next_bucket_ < (int)buckets_.size()) { flush(next_bucket_, compute); ++next_bucket_; }
  cudaStream_t side = sync_ ? sync_->comm_stream() : update_stream_;
  if (solver_->clipping()) {
    // behind every bucket's partials on the same stream: every rank holds the same reduced diffs, so the same factor
    solver_->ClipFactor(side);
    solver_->ApplyUpdateAll(side);
  }
  CUDA_CHECK(cudaEventRecord(ev_done_, side));
  CUDA_CHECK(cudaStreamWaitEvent(compute, ev_done_, 0));     // next forward sees the updated weights
  next_bucket_ = 0;
  solver_->increment_iter();
}

}  // namespace caffe
