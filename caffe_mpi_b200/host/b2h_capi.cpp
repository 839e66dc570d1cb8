// b2h_capi.cpp -- flat C entry points over the C++ host layer, used by tests/ and bench.py through ctypes.
// (The C++ classes in b2caffe.hpp are the interface a Caffe maintainer codes against; this file only
// marshals arrays so Python can drive them.)  Every function returns 0 / a handle, or -1 / NULL with the
// message available from b2h_last_error().
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include "b2caffe.hpp"
#include "prototxt.hpp"
#include "train_net.hpp"
#include "proto_wire.hpp"

using namespace caffe;

static thread_local std::string g_err;
#define B2H_TRY(body)                          \
  try { body; return 0; }                      \
  catch (const std::exception& e) { g_err = e.what(); return -1; }

struct ConvHandle {
  shared_ptr<LayerBase> layer;
  Blob bottom, top;
  bool set_up = false;
};
struct SolverHandle {
  std::unique_ptr<SGDSolver> solver;
  vector<shared_ptr<Blob>> params;
  std::unique_ptr<P2PSync> sync;
  std::unique_ptr<ReduceScheduler> sched;
};

extern "C" {

const char* b2h_last_error() { return g_err.c_str(); }

int b2h_registry_has(const char* type) {
  for (auto& t : LayerRegistry::LayerTypeList()) if (t == type) return 1;
  return 0;
}

// ---- ConvolutionLayer through LayerRegistry::CreateLayer --------------------------------------------------
void* b2h_conv_create(int num_output, int bias_term, int nk, const int* kernel, int ns, const int* stride, int np, const int* pad,
                      int nd, const int* dilation, int group, int engine, int math, int force_nd) {
  try {
    LayerParameter lp;
    lp.name = "conv"; lp.type = "Convolution";
    ConvolutionParameter& c = lp.convolution_param;
    c.num_output = num_output; c.bias_term = bias_term != 0; c.group = group; c.engine = engine; c.math = math;
    c.force_nd_im2col = force_nd != 0;
    c.kernel_size.assign(kernel, kernel + nk);
    c.stride.assign(stride, stride + ns);
    c.pad.assign(pad, pad + np);
    c.dilation.assign(dilation, dilation + nd);
    c.weight_filler.type = "gaussian"; c.weight_filler.std = 0.01f;
    c.bias_filler.type = "constant"; c.bias_filler.value = 0.1f;
    auto* h = new ConvHandle;
    h->layer = LayerRegistry::CreateLayer(lp);
    return h;
  } catch (const std::exception& e) { g_err = e.what(); return nullptr; }
}
int b2h_conv_setup(void* hv, int naxes, const int* bottom_shape) {
  auto* h = static_cast<ConvHandle*>(hv);
  B2H_TRY({
    h->bottom.Reshape(vector<int>(bottom_shape, bottom_shape + naxes));
    h->layer->SetUp({&h->bottom}, {&h->top});
    h->set_up = true;
  });
}
int b2h_conv_top_shape(void* hv, int* naxes, int* shape) {
  auto* h = static_cast<ConvHandle*>(hv);
  *naxes = h->top.num_axes();
  for (int i = 0; i < h->top.num_axes(); ++i) shape[i] = h->top.shape(i);
  return 0;
}
int b2h_conv_num_blobs(void* hv) { return (int)static_cast<ConvHandle*>(hv)->layer->blobs().size(); }
long long b2h_conv_blob_count(void* hv, int i) { return (long long)static_cast<ConvHandle*>(hv)->layer->blobs()[i]->count(); }
int b2h_conv_set_blob(void* hv, int i, int diff, const float* src) {
  auto* h = static_cast<ConvHandle*>(hv);
  B2H_TRY({
    Blob& b = *h->layer->blobs()[i];
    memcpy(diff ? b.mutable_cpu_diff() : b.mutable_cpu_data(), src, sizeof(float) * b.count());
  });
}
int b2h_conv_get_blob(void* hv, int i, int diff, float* dst) {
  auto* h = static_cast<ConvHandle*>(hv);
  B2H_TRY({
    Blob& b = *h->layer->blobs()[i];
    memcpy(dst, diff ? b.cpu_diff() : b.cpu_data(), sizeof(float) * b.count());
  });
}
int b2h_conv_forward(void* hv, const float* x, float* y) {
  auto* h = static_cast<ConvHandle*>(hv);
  B2H_TRY({
    memcpy(h->bottom.mutable_cpu_data(), x, sizeof(float) * h->bottom.count());
    h->layer->Forward({&h->bottom}, {&h->top});
    memcpy(y, h->top.cpu_data(), sizeof(float) * h->top.count());
  });
}
int b2h_conv_backward(void* hv, const float* dy, float* dx, int propagate_down) {
  auto* h = static_cast<ConvHandle*>(hv);
  B2H_TRY({
    memcpy(h->top.mutable_cpu_diff(), dy, sizeof(float) * h->top.count());
    h->layer->Backward({&h->top}, {propagate_down != 0}, {&h->bottom});
    if (dx && propagate_down) memcpy(dx, h->bottom.cpu_diff(), sizeof(float) * h->bottom.count());
    else CUDA_CHECK(cudaStreamSynchronize(Caffe::thread_stream()));
  });
}
int b2h_conv_algo_used(void* hv, int op) {
  auto* c = dynamic_cast<ConvolutionLayer*>(static_cast<ConvHandle*>(hv)->layer.get());
  return c ? c->algo_used(op) : -1;
}
void b2h_conv_destroy(void* hv) { delete static_cast<ConvHandle*>(hv); }

// ---- solver / scheduler ---------------------------------------------------------------------------------------
// a solver of any type (SGD, Nesterov, AdaGrad, RMSProp, AdaDelta, Adam) with its hyperparameters; NULL on a bad type or a failed
// sanity check
void* b2h_solver_create_typed(const char* type, float base_lr, const char* lr_policy, float gamma, float power, int stepsize,
                              int max_iter, float momentum, float weight_decay, const char* reg_type, int iter_size, int reduce_buckets,
                              int nstep, const int* stepvalue, int rampup_interval, float rampup_lr, float min_lr, float delta,
                              float momentum2, float rms_decay) {
  try {
    SolverParameter p;
    p.type = type; p.delta = delta; p.momentum2 = momentum2; p.rms_decay = rms_decay;
    p.base_lr = base_lr; p.lr_policy = lr_policy; p.gamma = gamma; p.power = power; p.stepsize = stepsize; p.max_iter = max_iter;
    p.momentum = momentum; p.weight_decay = weight_decay; p.regularization_type = reg_type; p.iter_size = iter_size;
    p.reduce_buckets = reduce_buckets; p.rampup_interval = rampup_interval; p.rampup_lr = rampup_lr; p.min_lr = min_lr;
    if (nstep) p.stepvalue.assign(stepvalue, stepvalue + nstep);
    auto* h = new SolverHandle;
    h->solver.reset(new SGDSolver(p));
    return h;
  } catch (const std::exception& e) { g_err = e.what(); return nullptr; }
}
// an SGD solver (b2h_solver_create_typed with type "SGD" and the SolverParameter defaults of the other solvers' fields)
void* b2h_solver_create(float base_lr, const char* lr_policy, float gamma, float power, int stepsize, int max_iter,
                        float momentum, float weight_decay, const char* reg_type, int iter_size, int reduce_buckets,
                        int nstep, const int* stepvalue, int rampup_interval, float rampup_lr, float min_lr) {
  const SolverParameter d;
  return b2h_solver_create_typed("SGD", base_lr, lr_policy, gamma, power, stepsize, max_iter, momentum, weight_decay, reg_type, iter_size,
                                 reduce_buckets, nstep, stepvalue, rampup_interval, rampup_lr, min_lr, d.delta, d.momentum2, d.rms_decay);
}
void b2h_solver_destroy(void* hv) { delete static_cast<SolverHandle*>(hv); }
float b2h_solver_lr_at(void* hv, int iter) {
  auto* h = static_cast<SolverHandle*>(hv);
  try { h->solver->set_iter(iter); return h->solver->GetLearningRate(); } catch (const std::exception& e) { g_err = e.what(); return -1.f; }
}
// SGD's momentum at `iter` under its momentum_policy (fixed, poly, opt); NaN with the error set on an unknown policy
float b2h_solver_momentum_at(void* hv, int iter) {
  auto* h = static_cast<SolverHandle*>(hv);
  try { h->solver->set_iter(iter); return h->solver->GetMomentum(); } catch (const std::exception& e) { g_err = e.what(); return NAN; }
}
// bucket plan over a layout of `n` params with the given element counts (no device memory needed)
int b2h_plan_buckets(int n, const size_t* counts, int reduce_buckets, int max_out, int* id_from, int* id_to, size_t* offset, size_t* count) {
  try {
    ParamArena a;
    a.InitLayout(vector<size_t>(counts, counts + n));
    vector<Bucket> b = PlanBuckets(a, reduce_buckets);
    for (int i = 0; i < (int)b.size() && i < max_out; ++i) { id_from[i] = b[i].id_from; id_to[i] = b[i].id_to; offset[i] = b[i].offset; count[i] = b[i].count; }
    return (int)b.size();
  } catch (const std::exception& e) { g_err = e.what(); return -1; }
}
int b2h_divide_batch_size(int total, int solver_count) { return P2PSync::divide_batch_size(total, solver_count); }

int b2h_solver_set_params(void* hv, int n, const size_t* counts, const float* lr_mult, const float* decay_mult) {
  auto* h = static_cast<SolverHandle*>(hv);
  B2H_TRY({
    vector<ParamSpec> specs(n);
    h->params.clear();
    for (int i = 0; i < n; ++i) {
      h->params.emplace_back(new Blob(vector<int>{(int)counts[i]}));
      specs[i].lr_mult = lr_mult[i]; specs[i].decay_mult = decay_mult[i];
    }
    h->solver->SetParams(h->params, specs);
  });
}
int b2h_solver_set(void* hv, int i, int diff, const float* src) {
  auto* h = static_cast<SolverHandle*>(hv);
  B2H_TRY({
    Blob& b = *h->params[i];
    CUDA_CHECK(cudaMemcpy(diff ? b.mutable_gpu_diff() : b.mutable_gpu_data(), src, sizeof(float) * b.count(), cudaMemcpyHostToDevice));
  });
}
// the device address of history `what` (2: history, 3: second history -- AdaDelta / Adam only) of arena slot i
static float* history_at(SGDSolver& s, int what, int i) {
  float* base = what == 2 ? s.arena().history() : s.arena().history2();
  B2_CHECK(base != nullptr, "solver type " + s.param().type + " keeps no second history");
  return base + s.arena().offset(i);
}
int b2h_solver_get(void* hv, int i, int what, float* dst) {   // what: 0 data, 1 diff, 2 history, 3 second history
  auto* h = static_cast<SolverHandle*>(hv);
  B2H_TRY({
    Blob& b = *h->params[i];
    CUDA_CHECK(cudaDeviceSynchronize());
    const float* src = what == 0 ? b.gpu_data() : what == 1 ? b.gpu_diff() : history_at(*h->solver, what, i);
    CUDA_CHECK(cudaMemcpy(dst, src, sizeof(float) * b.count(), cudaMemcpyDeviceToHost));
  });
}
// multi-GPU: rank 0 fills `id` (128 B) when create_id != 0; every rank then passes the same bytes
int b2h_solver_attach_sync(void* hv, int nranks, int rank, unsigned char* id, int create_id) {
  auto* h = static_cast<SolverHandle*>(hv);
  B2H_TRY({
    if (create_id) { B2C_CHECK(b2c_comm_get_unique_id(id)); return 0; }
    // the launcher has already carried rank 0's id to every rank: the bcast hook only hands it over
    unsigned char* idp = id;
    // P2PSync asks rank 0 for a fresh id and then "broadcasts"; here the broadcast overwrites with the carried id
    h->sync.reset(new P2PSync(nranks, rank, [idp](void* buf, size_t bytes, int) { memcpy(buf, idp, bytes); }));
    h->sync->on_start(h->solver->arena());
  });
}
// one iteration of the reduce-and-update schedule: params become ready last-to-first on the thread stream
int b2h_solver_step(void* hv) {
  auto* h = static_cast<SolverHandle*>(hv);
  B2H_TRY({
    if (!h->sched) h->sched.reset(new ReduceScheduler(h->solver.get(), h->sync.get()));
    cudaStream_t st = Caffe::thread_stream();
    for (int i = (int)h->params.size() - 1; i >= 0; --i) h->sched->on_param_ready(i, st);
    h->sched->end_of_iteration(st);
    CUDA_CHECK(cudaStreamSynchronize(st));
  });
}
int b2h_solver_iter(void* hv) { return static_cast<SolverHandle*>(hv)->solver->iter(); }
// SolverParameter.clip_gradients of a solver handle (negative: off); before b2h_solver_set_params
int b2h_solver_set_clip_gradients(void* hv, float clip) { B2H_TRY(static_cast<SolverHandle*>(hv)->solver->set_clip_gradients(clip)); }
static int clip_state(SGDSolver& s, float* norm, float* factor, long long* clipped) {
  B2H_TRY({
    const b2c_clip_state st = s.ClipState();
    *norm = st.norm; *factor = st.factor; *clipped = st.clipped;
  });
}
// the last iteration's gradient norm and factor, and the clipped iterations so far; synchronises the device
int b2h_solver_clip_state(void* hv, float* norm, float* factor, long long* clipped) {
  return clip_state(*static_cast<SolverHandle*>(hv)->solver, norm, factor, clipped);
}
// the first norm partial of each of `n` params with these counts, in arena order (no device memory); returns the partial count
long long b2h_clip_slots(int n, const size_t* counts, size_t* slot) {
  vector<size_t> s;
  const size_t total = SGDSolver::ClipSlots(vector<size_t>(counts, counts + n), &s);
  std::copy(s.begin(), s.end(), slot);
  return (long long)total;
}

// ---- prototxt / Net -----------------------------------------------------------------------------------------------
void* b2h_net_create(const char* path_or_text, int is_text, int phase, int batch_override, int def_channels, int def_size) {
  try {
    PMessage m = is_text ? ParseTextProto(path_or_text) : ParseTextProtoFile(path_or_text);
    return new Net(m, phase ? TEST : TRAIN, batch_override, def_channels, def_size);
  } catch (const std::exception& e) { g_err = e.what(); return nullptr; }
}
void b2h_net_destroy(void* h) { delete static_cast<Net*>(h); }
int b2h_net_num_layers(void* h) { return (int)static_cast<Net*>(h)->layers().size(); }
int b2h_net_layer(void* h, int i, char* name, char* type, int cap, int* naxes, int* top_shape) {
  Net* n = static_cast<Net*>(h);
  if (i < 0 || i >= (int)n->layers().size()) return -1;
  const NetLayer& L = n->layers()[i];
  snprintf(name, cap, "%s", L.param.name.c_str());
  snprintf(type, cap, "%s", L.param.type.c_str());
  const std::vector<int>& s = n->top_shape(i, 0);
  *naxes = (int)s.size();
  for (size_t k = 0; k < s.size() && k < 8; ++k) top_shape[k] = s[k];
  return 0;
}
// top t of layer i: its shape as Net inferred it (-1 when there is no such top)
int b2h_net_top_shape(void* h, int i, int t, int* naxes, int* top_shape) {
  Net* n = static_cast<Net*>(h);
  if (i < 0 || i >= (int)n->layers().size() || t < 0 || t >= (int)n->layers()[i].param.top.size()) return -1;
  const std::vector<int>& s = n->top_shape(i, t);
  *naxes = (int)s.size();
  for (size_t k = 0; k < s.size() && k < 8; ++k) top_shape[k] = s[k];
  return 0;
}
// the class-axis parameters of layer i as the layers read them (axes canonical): out[0] softmax_param.axis, [1] loss_param has
// ignore_label, [2] its ignore_label, [3] its normalization (b2c_loss_normalization, `normalize` folded in), [4] accuracy_param.axis,
// [5] top_k, [6] has ignore_label, [7] its ignore_label
int b2h_net_loss_params(void* h, int i, int* out, int n) {
  Net* net = static_cast<Net*>(h);
  if (i < 0 || i >= (int)net->layers().size() || n < 8) return -1;
  const LayerParameter& p = net->layers()[i].param;
  const int v[8] = {p.softmax_param.axis, p.loss_param.has_ignore_label, p.loss_param.ignore_label, p.loss_param.normalization,
                    p.accuracy_param.axis, p.accuracy_param.top_k, p.accuracy_param.has_ignore_label, p.accuracy_param.ignore_label};
  for (int k = 0; k < 8; ++k) out[k] = v[k];
  return 0;
}
int b2h_net_num_convs(void* h) { return (int)static_cast<Net*>(h)->conv_layers().size(); }
int b2h_net_conv(void* h, int i, b2c_conv_params* out, int* propagate_down, char* name, int cap) {
  Net* n = static_cast<Net*>(h);
  if (i < 0 || i >= (int)n->conv_layers().size()) return -1;
  const ConvEntry& c = n->conv_layers()[i];
  *out = c.p; *propagate_down = c.propagate_down ? 1 : 0;
  snprintf(name, cap, "%s", c.name.c_str());
  return 0;
}
int b2h_net_num_params(void* h) { return (int)static_cast<Net*>(h)->learnable_params().size(); }
int b2h_net_param(void* h, int i, size_t* count, float* lr_mult, float* decay_mult, char* layer, int cap) {
  Net* n = static_cast<Net*>(h);
  if (i < 0 || i >= (int)n->learnable_params().size()) return -1;
  const LearnableParam& p = n->learnable_params()[i];
  *count = p.count; *lr_mult = p.lr_mult; *decay_mult = p.decay_mult;
  snprintf(layer, cap, "%s", p.layer.c_str());
  return 0;
}
// every layer's parameter blobs, sharers included (Net::params_): blob i's layer, ParamSpec.name, its owner's index in this list
// (-1: it owns its storage) and its index in b2h_net_param's list (the owner's, for a sharer)
int b2h_net_num_net_params(void* h) { return (int)static_cast<Net*>(h)->net_params().size(); }
int b2h_net_net_param(void* h, int i, int* owner, int* learnable_id, char* layer, char* name, int cap) {
  Net* n = static_cast<Net*>(h);
  if (i < 0 || i >= (int)n->net_params().size()) return -1;
  const LearnableParam& p = n->net_params()[i];
  *owner = p.owner; *learnable_id = p.learnable_id;
  snprintf(layer, cap, "%s", p.layer.c_str());
  snprintf(name, cap, "%s", p.name.c_str());
  return 0;
}
// 1 when layer i is a Data layer whose data_param.source opened (it will read the database), 0 otherwise
int b2h_net_layer_uses_database(void* h, int i) {
  const auto& ls = static_cast<Net*>(h)->layers();
  return i >= 0 && i < (int)ls.size() && ls[i].use_database ? 1 : 0;
}
int b2h_net_reduce_buckets(void* h) { return static_cast<Net*>(h)->reduce_buckets(); }
// layer i's need-backward result (loss pruning included): bit 0 = the layer runs backward, bit 1 + b = bottom b gets a gradient
long long b2h_net_layer_backward(void* h, int i) {
  const auto& ls = static_cast<Net*>(h)->layers();
  if (i < 0 || i >= (int)ls.size()) return -1;
  long long v = ls[i].need_backward ? 1 : 0;
  for (size_t b = 0; b < ls[i].propagate_down.size() && b < 62; ++b) if (ls[i].propagate_down[b]) v |= 2ll << b;
  return v;
}
int b2h_net_layer_bottoms(void* h, int i) {
  const auto& ls = static_cast<Net*>(h)->layers();
  return i >= 0 && i < (int)ls.size() ? (int)ls[i].param.bottom.size() : -1;
}
// the blob the trainer reports as its loss (Net::loss_blob); empty when the net has none
int b2h_net_loss_blob(void* h, char* name, int cap) {
  snprintf(name, cap, "%s", static_cast<Net*>(h)->loss_blob().c_str());
  return 0;
}

// SolverParameter from a solver.prototxt of any type (SGD, Nesterov, AdaGrad, RMSProp, AdaDelta, Adam; `type` or the legacy
// `solver_type`); returns a solver handle like b2h_solver_create_typed
void* b2h_solver_open(const char* path_or_text, int is_text, char* net_path, int cap) {
  try {
    PMessage m = is_text ? ParseTextProto(path_or_text) : ParseTextProtoFile(path_or_text);
    std::string np;
    SolverParameter p = ReadSolverParameter(m, &np);
    if (net_path) snprintf(net_path, cap, "%s", np.c_str());
    auto* h = new SolverHandle;
    h->solver.reset(new SGDSolver(p));
    return h;
  } catch (const std::exception& e) { g_err = e.what(); return nullptr; }
}
// the same, for SGD solver files only: a caller that asked for an SGD solver is refused a file of another type
void* b2h_solver_from_file(const char* path_or_text, int is_text, char* net_path, int cap) {
  auto* h = static_cast<SolverHandle*>(b2h_solver_open(path_or_text, is_text, net_path, cap));
  if (h && h->solver->kind() != B2C_SOLVER_SGD) {
    g_err = "solver type '" + h->solver->param().type + "' asked of an SGD solver handle (SGD only; b2h_solver_open reads every type)";
    delete h;
    return nullptr;
  }
  return h;
}
int b2h_solver_describe(void* hv, float* base_lr, float* momentum, float* weight_decay, int* max_iter, int* iter_size, char* policy, int cap) {
  const SolverParameter& p = static_cast<SolverHandle*>(hv)->solver->param();
  *base_lr = p.base_lr; *momentum = p.momentum; *weight_decay = p.weight_decay; *max_iter = p.max_iter; *iter_size = p.iter_size;
  snprintf(policy, cap, "%s", p.lr_policy.c_str());
  return 0;
}
int b2h_solver_hparams(void* hv, char* type, int cap, float* delta, float* momentum2, float* rms_decay) {
  const SolverParameter& p = static_cast<SolverHandle*>(hv)->solver->param();
  snprintf(type, cap, "%s", p.type.c_str());
  *delta = p.delta; *momentum2 = p.momentum2; *rms_decay = p.rms_decay;
  return 0;
}
// the testing fields: returns the number of test_iter entries (the first `cap` of them land in test_iter); not_built gets the names of
// the test-net sources present that are not built (test_net, test_net_param, test_state), space-separated
int b2h_solver_testing(void* hv, int* test_iter, int cap, int* test_interval, int* test_compute_loss, char* not_built, int nb_cap) {
  const SolverParameter& p = static_cast<SolverHandle*>(hv)->solver->param();
  for (int i = 0; i < (int)p.test_iter.size() && i < cap; ++i) test_iter[i] = p.test_iter[i];
  *test_interval = p.test_interval;
  *test_compute_loss = p.test_compute_loss ? 1 : 0;
  std::string nb;
  for (const std::string& f : p.test_fields_not_built) nb += (nb.empty() ? "" : " ") + f;
  snprintf(not_built, nb_cap, "%s", nb.c_str());
  return (int)p.test_iter.size();
}

// first scalar value of a top-level field of a text-format message (tools/caffe.py reads SolverParameter.display / snapshot /
// snapshot_prefix / snapshot_after_train / random_seed with it); returns 1 if present, 0 if absent, -1 on a parse error
int b2h_textproto_scalar(const char* path_or_text, int is_text, const char* key, char* value, int cap) {
  try {
    PMessage m = is_text ? ParseTextProto(path_or_text) : ParseTextProtoFile(path_or_text);
    for (const PField* f : m.all(key))
      if (!f->is_msg()) { snprintf(value, cap, "%s", f->scalar.c_str()); return 1; }
    return 0;
  } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// ---- TrainNet: the whole prototxt net + solver ------------------------------------------------------------------
struct TrainerHandle {
  std::unique_ptr<Net> desc;
  std::unique_ptr<TrainNet> net;
  std::unique_ptr<P2PSync> sync;
};
void* b2h_trainer_create(const char* net_src, int net_is_text, const char* solver_src, int solver_is_text, int batch, int num_classes,
                         unsigned long long seed, int math, int def_channels, int def_size) {
  try {
    auto* h = new TrainerHandle;
    PMessage nm = net_is_text ? ParseTextProto(net_src) : ParseTextProtoFile(net_src);
    h->desc.reset(new Net(nm, TRAIN, batch, def_channels, def_size));
    PMessage sm = solver_is_text ? ParseTextProto(solver_src) : ParseTextProtoFile(solver_src);
    SolverParameter sp = ReadSolverParameter(sm);
    sp.reduce_buckets = h->desc->reduce_buckets();
    sp.global_grad_scale = h->desc->global_grad_scale();
    h->net.reset(new TrainNet(*h->desc, sp, num_classes, seed, math));
    return h;
  } catch (const std::exception& e) { g_err = e.what(); return nullptr; }
}
void b2h_trainer_destroy(void* hv) { delete static_cast<TrainerHandle*>(hv); }
int b2h_trainer_attach_sync(void* hv, int nranks, int rank, unsigned char* id, int create_id) {
  auto* h = static_cast<TrainerHandle*>(hv);
  B2H_TRY({
    if (create_id) { B2C_CHECK(b2c_comm_get_unique_id(id)); return 0; }
    unsigned char* idp = id;
    h->sync.reset(new P2PSync(nranks, rank, [idp](void* buf, size_t bytes, int) { memcpy(buf, idp, bytes); }));
    h->net->AttachSync(h->sync.get());
  });
}
// in-step exchange timing: CUDA events around every bucket's allreduce on the comm stream (bench.py)
int b2h_trainer_bucket_timing(void* hv, int on) {
  auto* h = static_cast<TrainerHandle*>(hv);
  B2H_TRY({ B2_CHECK(h->sync != nullptr, "bucket timing needs an attached P2PSync"); h->sync->set_bucket_timing(on != 0); });
}
int b2h_trainer_bucket_times(void* hv, int cap, unsigned long long* bytes, float* ms, int* count) {
  auto* h = static_cast<TrainerHandle*>(hv);
  B2H_TRY({
    B2_CHECK(h->sync != nullptr, "bucket timing needs an attached P2PSync");
    vector<size_t> by;
    vector<float> t;
    h->sync->collect_bucket_times(&by, &t);
    *count = (int)by.size();
    for (int i = 0; i < *count && i < cap; ++i) { bytes[i] = by[i]; ms[i] = t[i]; }
  });
}
int b2h_trainer_step(void* hv, int nsteps, int copy_input) {
  auto* h = static_cast<TrainerHandle*>(hv);
  B2H_TRY({ for (int i = 0; i < nsteps; ++i) h->net->Step(copy_input != 0); });
}
int b2h_trainer_timed_steps(void* hv, int nsteps, int copy_input, int read_loss, float* ms) {
  auto* h = static_cast<TrainerHandle*>(hv);
  B2H_TRY({ *ms = h->net->TimedSteps(nsteps, copy_input != 0, read_loss != 0); });
}
long long b2h_trainer_input_bytes(void* hv) { return (long long)static_cast<TrainerHandle*>(hv)->net->input_bytes(); }
int b2h_trainer_forward_backward(void* hv, float* loss) {
  auto* h = static_cast<TrainerHandle*>(hv);
  B2H_TRY({ *loss = h->net->ForwardBackward(); });
}
int b2h_trainer_clear_param_diffs(void* hv) {
  auto* h = static_cast<TrainerHandle*>(hv);
  B2H_TRY({ h->net->ClearParamDiffs(); });
}
int b2h_trainer_sync(void* hv) { (void)hv; B2H_TRY({ CUDA_CHECK(cudaStreamSynchronize(Caffe::thread_stream())); CUDA_CHECK(cudaDeviceSynchronize()); }); }
int b2h_trainer_loss(void* hv, float* loss) {
  auto* h = static_cast<TrainerHandle*>(hv);
  B2H_TRY({ *loss = h->net->last_loss(); });
}
long long b2h_trainer_blob_count(void* hv, const char* name) {
  Blob* b = static_cast<TrainerHandle*>(hv)->net->blob(name);
  return b ? (long long)b->count() : -1;
}
int b2h_trainer_blob(void* hv, const char* name, int diff, int set, float* buf) {
  auto* h = static_cast<TrainerHandle*>(hv);
  B2H_TRY({
    Blob* b = h->net->blob(name);
    B2_CHECK(b != nullptr, std::string("no blob named ") + name);
    if (set) memcpy(diff ? b->mutable_cpu_diff() : b->mutable_cpu_data(), buf, sizeof(float) * b->count());
    else memcpy(buf, diff ? b->cpu_diff() : b->cpu_data(), sizeof(float) * b->count());
  });
}
// parameter access by TRAINABLE index (conv / fc weights + biases, BatchNorm scale + bias -- the blobs the layers
// differentiate); b2h_trainer_num_learnable counts every layer blob like Net::learnable_params() (BatchNorm: 5)
// blob `blob` of layer `layer` (execution order): the Blob object's address and its device data / diff pointers.  Two layers that
// share a named parameter report distinct objects over one storage (test_net.cpp TestSharedWeightsUpdate)
int b2h_trainer_layer_blob(void* hv, int layer, int blob, unsigned long long* object, unsigned long long* data, unsigned long long* diff) {
  B2H_TRY({
    TrainNet& n = *static_cast<TrainerHandle*>(hv)->net;
    B2_CHECK(layer >= 0 && layer < n.num_layers(), "layer index out of range");
    auto& bl = n.layer(layer)->blobs();
    B2_CHECK(blob >= 0 && blob < (int)bl.size(), "blob index out of range");
    *object = (unsigned long long)(uintptr_t)bl[blob].get();
    *data = (unsigned long long)(uintptr_t)bl[blob]->gpu_data();
    *diff = (unsigned long long)(uintptr_t)bl[blob]->gpu_diff();
  });
}
int b2h_trainer_num_params(void* hv) { return (int)static_cast<TrainerHandle*>(hv)->net->trainable_ids().size(); }
int b2h_trainer_num_learnable(void* hv) { return (int)static_cast<TrainerHandle*>(hv)->net->learnable_params().size(); }
long long b2h_trainer_param_count(void* hv, int i) {
  auto* h = static_cast<TrainerHandle*>(hv);
  return (long long)h->net->learnable_params()[h->net->trainable_ids()[i]]->count();
}
int b2h_trainer_param(void* hv, int i, int what, int set, float* buf) {   // what: 0 data, 1 diff, 2 history, 3 second history
  auto* h = static_cast<TrainerHandle*>(hv);
  B2H_TRY({
    const int id = h->net->trainable_ids().at(i);
    Blob& b = *h->net->learnable_params()[id];
    CUDA_CHECK(cudaDeviceSynchronize());
    float* dev = what == 0 ? b.mutable_gpu_data() : what == 1 ? b.mutable_gpu_diff() : history_at(h->net->solver(), what, id);
    if (set) { CUDA_CHECK(cudaMemcpy(dev, buf, sizeof(float) * b.count(), cudaMemcpyHostToDevice)); if (what == 0) h->net->MarkParamsDirty(); }
    else CUDA_CHECK(cudaMemcpy(buf, dev, sizeof(float) * b.count(), cudaMemcpyDeviceToHost));
  });
}
int b2h_trainer_clip_state(void* hv, float* norm, float* factor, long long* clipped) {
  return clip_state(static_cast<TrainerHandle*>(hv)->net->solver(), norm, factor, clipped);
}
int b2h_trainer_snapshot(void* hv, const char* prefix, char* state_path, int len) {
  auto* h = static_cast<TrainerHandle*>(hv);
  B2H_TRY({ const std::string p = h->net->Snapshot(prefix); snprintf(state_path, len, "%s", p.c_str()); });
}
int b2h_trainer_restore(void* hv, const char* state_path) {
  auto* h = static_cast<TrainerHandle*>(hv);
  B2H_TRY({ h->net->Restore(state_path); });
}
int b2h_trainer_copy_from(void* hv, const char* model_path, int* copied) {
  auto* h = static_cast<TrainerHandle*>(hv);
  B2H_TRY({ *copied = h->net->CopyTrainedLayersFrom(model_path); });
}
long long b2h_trainer_arena_floats(void* hv) { return (long long)static_cast<TrainerHandle*>(hv)->net->solver().arena().total(); }
int b2h_trainer_num_layers(void* hv) { return static_cast<TrainerHandle*>(hv)->net->num_layers(); }
int b2h_trainer_layer(void* hv, int i, char* name, char* type, int len) {
  auto* h = static_cast<TrainerHandle*>(hv);
  B2H_TRY({ snprintf(name, len, "%s", h->net->layer_name(i).c_str()); snprintf(type, len, "%s", h->net->layer_type(i).c_str()); });
}
// per (layer, op) mean ms per step over nsteps profiled steps; op: 0 forward, 1 backward (whole layer), 2 conv wgrad, 3 conv dgrad
int b2h_trainer_profile(void* hv, int nsteps, int cap, int* layer, int* op, float* ms, int* count) {
  auto* h = static_cast<TrainerHandle*>(hv);
  B2H_TRY({
    std::vector<int> l; std::vector<int> o; std::vector<float> m;
    h->net->ProfileSteps(nsteps, &l, &o, &m);
    *count = (int)l.size();
    for (int i = 0; i < *count && i < cap; ++i) { layer[i] = l[i]; op[i] = o[i]; ms[i] = m[i]; }
  });
}
int b2h_trainer_iter(void* hv) { return static_cast<TrainerHandle*>(hv)->net->solver().iter(); }

// ---- .caffemodel / .solverstate wire format on host arrays (no device needed; tests/test_snapshot_cpu.py) ----------------
struct WireHandle { NetWeights net; SolverStateData st; };
void* b2h_wire_new() { return new WireHandle; }
void b2h_wire_destroy(void* hv) { delete static_cast<WireHandle*>(hv); }
int b2h_wire_add_layer(void* hv, const char* name, const char* type) {
  auto* h = static_cast<WireHandle*>(hv);
  LayerWeights l; l.name = name; l.type = type;
  h->net.layers.push_back(l);
  return (int)h->net.layers.size() - 1;
}
int b2h_wire_add_blob(void* hv, int layer, int ndim, const int* shape, const float* data) {   // layer < 0: solver history
  auto* h = static_cast<WireHandle*>(hv);
  B2H_TRY({
    BlobData b;
    size_t cnt = 1;
    for (int i = 0; i < ndim; ++i) { b.shape.push_back(shape[i]); cnt *= (size_t)shape[i]; }
    b.data.assign(data, data + cnt);
    if (layer < 0) h->st.history.push_back(b);
    else { B2_CHECK(layer < (int)h->net.layers.size(), "no such layer"); h->net.layers[layer].blobs.push_back(b); }
  });
}
int b2h_wire_save_model(void* hv, const char* path, const char* net_name, int raw) {
  auto* h = static_cast<WireHandle*>(hv);
  B2H_TRY({ h->net.name = net_name; WriteBinaryFile(path, SerializeNetWeights(h->net, raw != 0)); });
}
int b2h_wire_save_state(void* hv, const char* path, int iter, int current_step, const char* learned_net, int raw) {
  auto* h = static_cast<WireHandle*>(hv);
  B2H_TRY({ h->st.iter = iter; h->st.current_step = current_step; h->st.learned_net = learned_net; WriteBinaryFile(path, SerializeSolverState(h->st, raw != 0)); });
}
void* b2h_wire_load(const char* path, int is_state) {
  try {
    auto* h = new WireHandle;
    if (is_state) h->st = ParseSolverState(ReadBinaryFile(path)); else h->net = ParseNetWeights(ReadBinaryFile(path));
    return h;
  } catch (const std::exception& e) { g_err = e.what(); return nullptr; }
}
int b2h_wire_num_layers(void* hv) { return (int)static_cast<WireHandle*>(hv)->net.layers.size(); }
int b2h_wire_layer(void* hv, int i, char* name, char* type, int len, int* nblobs) {
  auto* h = static_cast<WireHandle*>(hv);
  B2H_TRY({
    const LayerWeights& l = h->net.layers.at(i);
    snprintf(name, len, "%s", l.name.c_str()); snprintf(type, len, "%s", l.type.c_str());
    *nblobs = (int)l.blobs.size();
  });
}
int b2h_wire_num_history(void* hv) { return (int)static_cast<WireHandle*>(hv)->st.history.size(); }
int b2h_wire_blob(void* hv, int layer, int j, int* ndim, int* shape, long long* count, float* data) {   // data may be null (query)
  auto* h = static_cast<WireHandle*>(hv);
  B2H_TRY({
    const BlobData& b = layer < 0 ? h->st.history.at(j) : h->net.layers.at(layer).blobs.at(j);
    *ndim = (int)b.shape.size();
    for (size_t k = 0; k < b.shape.size() && k < 8; ++k) shape[k] = b.shape[k];
    *count = (long long)b.data.size();
    if (data) memcpy(data, b.data.data(), sizeof(float) * b.data.size());
  });
}
int b2h_wire_state(void* hv, int* iter, int* current_step, char* learned_net, int len, char* net_name, int nlen) {
  auto* h = static_cast<WireHandle*>(hv);
  B2H_TRY({ *iter = h->st.iter; *current_step = h->st.current_step; snprintf(learned_net, len, "%s", h->st.learned_net.c_str());
            snprintf(net_name, nlen, "%s", h->net.name.c_str()); });
}

// batches the database-backed Data layer has loaded so far; -1 when the net runs on the synthetic source
long long b2h_trainer_database_batches(void* hv) {
  DataLayer* d = static_cast<TrainerHandle*>(hv)->net->database_layer();
  return d ? (long long)d->batches_loaded() : -1;
}
long long b2h_trainer_activation_floats(void* hv) { return (long long)static_cast<TrainerHandle*>(hv)->net->activation_floats(); }

// ---- TEST-phase net (TrainNet over a Net filtered for TEST): forward only, scored like tools/caffe.cpp test() -------------------
struct TesterHandle {
  std::unique_ptr<Net> desc;
  std::unique_ptr<TrainNet> net;
};
void* b2h_tester_create(const char* net_src, int net_is_text, int batch, int num_classes, unsigned long long seed, int math, int def_channels,
                        int def_size) {
  try {
    auto* h = new TesterHandle;
    PMessage nm = net_is_text ? ParseTextProto(net_src) : ParseTextProtoFile(net_src);
    h->desc.reset(new Net(nm, TEST, batch, def_channels, def_size));
    h->net.reset(new TrainNet(*h->desc, SolverParameter(), num_classes, seed, math));
    return h;
  } catch (const std::exception& e) { g_err = e.what(); return nullptr; }
}
void b2h_tester_destroy(void* hv) { delete static_cast<TesterHandle*>(hv); }
int b2h_tester_copy_from(void* hv, const char* model_path, int* copied) {
  auto* h = static_cast<TesterHandle*>(hv);
  B2H_TRY({ *copied = h->net->CopyTrainedLayersFrom(model_path); });
}
// the trainer handle must outlive the tester: the tester reads the trainer's parameter blobs
int b2h_tester_share_from(void* hv, void* trainer) {
  auto* h = static_cast<TesterHandle*>(hv);
  B2H_TRY({ h->net->ShareTrainedLayersWith(*static_cast<TrainerHandle*>(trainer)->net); });
}
int b2h_tester_forward(void* hv) {
  auto* h = static_cast<TesterHandle*>(hv);
  B2H_TRY({ h->net->MarkParamsDirty(); h->net->ForwardTest(); CUDA_CHECK(cudaStreamSynchronize(Caffe::thread_stream())); });
}
int b2h_tester_num_outputs(void* hv) { return (int)static_cast<TesterHandle*>(hv)->net->outputs().size(); }
int b2h_tester_output(void* hv, int i, char* name, int cap, float* loss_weight, long long* count) {
  auto* h = static_cast<TesterHandle*>(hv);
  B2H_TRY({
    const TrainNet::Output& o = h->net->outputs().at(i);
    snprintf(name, cap, "%s", o.name.c_str());
    *loss_weight = o.loss_weight;
    *count = (long long)o.blob->count();
  });
}
// per_batch: iterations x (sum of the output counts), output order; mean: one value per output element
int b2h_tester_test(void* hv, int iterations, float* per_batch, float* mean, float* loss) {
  auto* h = static_cast<TesterHandle*>(hv);
  B2H_TRY({
    vector<float> pb;
    vector<float> m;
    *loss = h->net->Test(iterations, &pb, &m);
    memcpy(per_batch, pb.data(), sizeof(float) * pb.size());
    memcpy(mean, m.data(), sizeof(float) * m.size());
  });
}
// Solver::Test's pass (TrainNet::TestPass): scores summed on the device (over the ranks too when the tester shares a multi-GPU trainer),
// one read at the end.  between (may be null) is called before every batch with its index; a zero return stops the pass there.
// Returns the number of batches run (= iterations unless stopped), -1 on error; means / loss are written only for a whole pass.
int b2h_tester_test_pass(void* hv, int iterations, float* means, float* loss, int (*between)(int)) {
  auto* h = static_cast<TesterHandle*>(hv);
  try {
    vector<float> m;
    std::function<bool(int)> hook;
    if (between) hook = [between](int i) { return between(i) != 0; };
    const int ran = h->net->TestPass(iterations, hook, &m, loss);
    if (ran == iterations) memcpy(means, m.data(), sizeof(float) * m.size());
    return ran;
  } catch (const std::exception& e) { g_err = e.what(); return -1; }
}
long long b2h_tester_blob_count(void* hv, const char* name) {
  Blob* b = static_cast<TesterHandle*>(hv)->net->blob(name);
  return b ? (long long)b->count() : -1;
}
int b2h_tester_blob(void* hv, const char* name, int set, float* buf) {
  auto* h = static_cast<TesterHandle*>(hv);
  B2H_TRY({
    Blob* b = h->net->blob(name);
    B2_CHECK(b != nullptr, std::string("no blob named ") + name);
    if (set) memcpy(b->mutable_cpu_data(), buf, sizeof(float) * b->count());
    else memcpy(buf, b->cpu_data(), sizeof(float) * b->count());
  });
}
int b2h_tester_has_solver(void* hv) { return static_cast<TesterHandle*>(hv)->net->has_solver() ? 1 : 0; }
int b2h_tester_num_layers(void* hv) { return static_cast<TesterHandle*>(hv)->net->num_layers(); }
int b2h_tester_layer(void* hv, int i, char* name, char* type, int len) {
  auto* h = static_cast<TesterHandle*>(hv);
  B2H_TRY({ snprintf(name, len, "%s", h->net->layer_name(i).c_str()); snprintf(type, len, "%s", h->net->layer_type(i).c_str()); });
}
int b2h_tester_timed_forwards(void* hv, int n, float* ms) {
  auto* h = static_cast<TesterHandle*>(hv);
  B2H_TRY({ *ms = h->net->TimedForwards(n); });
}
// per layer mean forward ms over n profiled forwards (b2h_trainer_profile's layout, op 0 only)
int b2h_tester_profile(void* hv, int n, int cap, int* layer, float* ms, int* count) {
  auto* h = static_cast<TesterHandle*>(hv);
  B2H_TRY({
    std::vector<int> l;
    std::vector<int> o;
    std::vector<float> m;
    h->net->ProfileForwards(n, &l, &o, &m);
    *count = (int)l.size();
    for (int i = 0; i < *count && i < cap; ++i) { layer[i] = l[i]; ms[i] = m[i]; }
  });
}
long long b2h_tester_database_batches(void* hv) {
  DataLayer* d = static_cast<TesterHandle*>(hv)->net->database_layer();
  return d ? (long long)d->batches_loaded() : -1;
}

}  // extern "C"
