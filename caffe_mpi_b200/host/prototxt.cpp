// prototxt.cpp -- text-format protobuf reader + Net graph builder (see prototxt.hpp for the reference map).
#include "prototxt.hpp"
#include "data_reader.hpp"

#include <cctype>
#include <cmath>
#include <algorithm>
#include <cstdlib>
#include <fstream>
#include <set>
#include <sstream>

namespace caffe {

// ================================================================================================ tokenizer
namespace {
struct Tok { enum Kind { IDENT, STRING, NUMBER, COLON, LBRACE, RBRACE, END } kind; std::string text; int line; };

class Lexer {
 public:
  explicit Lexer(const std::string& s) : s_(s) {}
  Tok next() {
    skip();
    if (i_ >= s_.size()) return {Tok::END, "", line_};
    const char c = s_[i_];
    if (c == ':') { ++i_; return {Tok::COLON, ":", line_}; }
    if (c == '{' || c == '<') { ++i_; return {Tok::LBRACE, "{", line_}; }
    if (c == '}' || c == '>') { ++i_; return {Tok::RBRACE, "}", line_}; }
    if (c == '"' || c == '\'') {
      const char q = c;
      std::string out;
      ++i_;
      while (i_ < s_.size() && s_[i_] != q) {
        if (s_[i_] == '\\' && i_ + 1 < s_.size()) {
          const char e = s_[++i_];
          out += e == 'n' ? '\n' : e == 't' ? '\t' : e;
        } else {
          if (s_[i_] == '\n') ++line_;
          out += s_[i_];
        }
        ++i_;
      }
      if (i_ >= s_.size()) Fatal(__FILE__, __LINE__, "prototxt line " + std::to_string(line_) + ": unterminated string");
      ++i_;
      return {Tok::STRING, out, line_};
    }
    if (std::isalpha((unsigned char)c) || c == '_') {
      size_t b = i_;
      while (i_ < s_.size() && (std::isalnum((unsigned char)s_[i_]) || s_[i_] == '_' || s_[i_] == '.')) ++i_;
      return {Tok::IDENT, s_.substr(b, i_ - b), line_};
    }
    if (std::isdigit((unsigned char)c) || c == '-' || c == '+' || c == '.') {
      size_t b = i_;
      ++i_;
      while (i_ < s_.size() && (std::isalnum((unsigned char)s_[i_]) || s_[i_] == '.' || s_[i_] == '-' || s_[i_] == '+')) {
        // allow exponents like 1e-4; stop a sign that is not part of an exponent
        if ((s_[i_] == '-' || s_[i_] == '+') && !(s_[i_ - 1] == 'e' || s_[i_ - 1] == 'E')) break;
        ++i_;
      }
      return {Tok::NUMBER, s_.substr(b, i_ - b), line_};
    }
    Fatal(__FILE__, __LINE__, "prototxt line " + std::to_string(line_) + ": unexpected character '" + std::string(1, c) + "'");
  }
 private:
  void skip() {
    for (;;) {
      while (i_ < s_.size() && (std::isspace((unsigned char)s_[i_]) || s_[i_] == ',' || s_[i_] == ';')) { if (s_[i_] == '\n') ++line_; ++i_; }
      if (i_ < s_.size() && s_[i_] == '#') { while (i_ < s_.size() && s_[i_] != '\n') ++i_; continue; }
      break;
    }
  }
  const std::string& s_;
  size_t i_ = 0;
  int line_ = 1;
};

void parse_message(Lexer& lx, PMessage& m, bool top) {
  for (;;) {
    Tok t = lx.next();
    if (t.kind == Tok::END) { if (!top) Fatal(__FILE__, __LINE__, "prototxt: missing '}'"); return; }
    if (t.kind == Tok::RBRACE) { if (top) Fatal(__FILE__, __LINE__, "prototxt line " + std::to_string(t.line) + ": unmatched '}'"); return; }
    if (t.kind != Tok::IDENT) Fatal(__FILE__, __LINE__, "prototxt line " + std::to_string(t.line) + ": expected a field name, got '" + t.text + "'");
    Tok v = lx.next();
    if (v.kind == Tok::COLON) v = lx.next();
    PField f;
    if (v.kind == Tok::LBRACE) {
      f.msg.reset(new PMessage);
      parse_message(lx, *f.msg, false);
    } else if (v.kind == Tok::STRING || v.kind == Tok::NUMBER || v.kind == Tok::IDENT) {
      f.scalar = v.text;
    } else {
      Fatal(__FILE__, __LINE__, "prototxt line " + std::to_string(v.line) + ": expected a value for '" + t.text + "'");
    }
    m.fields.emplace_back(t.text, std::move(f));
  }
}
}  // namespace

PMessage ParseTextProto(const std::string& text) {
  Lexer lx(text);
  PMessage m;
  parse_message(lx, m, true);
  return m;
}
PMessage ParseTextProtoFile(const std::string& path) {
  std::ifstream in(path);
  if (!in) Fatal(__FILE__, __LINE__, "File not found: " + path);   // ReadProtoFromTextFile CHECK
  std::stringstream ss;
  ss << in.rdbuf();
  return ParseTextProto(ss.str());
}

bool PMessage::has(const std::string& k) const { for (auto& f : fields) if (f.first == k) return true; return false; }
std::vector<const PField*> PMessage::all(const std::string& k) const {
  std::vector<const PField*> v;
  for (auto& f : fields) if (f.first == k) v.push_back(&f.second);
  return v;
}
const PMessage* PMessage::sub(const std::string& k) const {
  for (auto& f : fields) if (f.first == k && f.second.is_msg()) return f.second.msg.get();
  return nullptr;
}
std::string PMessage::str(const std::string& k, const std::string& d) const {
  for (auto& f : fields) if (f.first == k && !f.second.is_msg()) return f.second.scalar;
  return d;
}
double PMessage::num(const std::string& k, double d) const { const std::string s = str(k); return s.empty() ? d : std::atof(s.c_str()); }
long long PMessage::integer(const std::string& k, long long d) const { const std::string s = str(k); return s.empty() ? d : std::atoll(s.c_str()); }
bool PMessage::boolean(const std::string& k, bool d) const { const std::string s = str(k); return s.empty() ? d : (s == "true" || s == "1" || s == "True"); }
std::vector<long long> PMessage::ints(const std::string& k) const {
  std::vector<long long> v;
  for (auto* f : all(k)) if (!f->is_msg()) v.push_back(std::atoll(f->scalar.c_str()));
  return v;
}

// ================================================================================================ Net
namespace {
bool rule_met(const PMessage& rule, Phase phase) {     // Net::StateMeetsRule with level 0 and no stages
  if (rule.has("phase")) {
    const std::string p = rule.str("phase");
    const Phase rp = (p == "TEST" || p == "1") ? TEST : TRAIN;
    if (rp != phase) return false;
  }
  if (rule.has("min_level") && rule.integer("min_level") > 0) return false;
  if (rule.has("max_level") && rule.integer("max_level") < 0) return false;
  if (rule.has("stage")) return false;                  // the net state carries no stages
  return true;
}
bool layer_included(const PMessage& lp, Phase phase) {  // Net::FilterNet
  const auto inc = lp.all("include"), exc = lp.all("exclude");
  if (!inc.empty() && !exc.empty()) Fatal(__FILE__, __LINE__, "Specify either include rules or exclude rules; not both.");
  if (inc.empty()) {
    for (auto* e : exc) if (e->is_msg() && rule_met(*e->msg, phase)) return false;
    return true;
  }
  for (auto* i : inc) if (i->is_msg() && rule_met(*i->msg, phase)) return true;
  return false;
}
int engine_of(const std::string& s) { return s == "CAFFE" || s == "1" ? B2C_ENGINE_CAFFE : s == "CUDNN" || s == "2" ? B2C_ENGINE_CUDNN : B2C_ENGINE_DEFAULT; }
FillerParameter filler_of(const PMessage* m) {
  FillerParameter f;
  if (!m) return f;
  f.type = m->str("type", "constant");
  f.value = (float)m->num("value", 0); f.min = (float)m->num("min", 0); f.max = (float)m->num("max", 1);
  f.mean = (float)m->num("mean", 0); f.std = (float)m->num("std", 1);
  const std::string vn = m->str("variance_norm", "FAN_IN");
  f.variance_norm = vn == "FAN_OUT" ? 1 : vn == "AVERAGE" ? 2 : 0;
  return f;
}
std::vector<int> to_int(const std::vector<long long>& v) { return std::vector<int>(v.begin(), v.end()); }
size_t prod(const std::vector<int>& s, size_t from = 0) { size_t c = 1; for (size_t i = from; i < s.size(); ++i) c *= (size_t)s[i]; return c; }
int canonical_axis(int axis, const std::vector<int>& s) {  // Blob::CanonicalAxisIndex, with its message
  const int n = (int)s.size();
  if (axis < -n || axis >= n) {
    std::string shp;
    for (int d : s) shp += std::to_string(d) + " ";
    Fatal(__FILE__, __LINE__, "axis " + std::to_string(axis) + " out of range for " + std::to_string(n) + "-D Blob with shape " + shp + "(" +
                                  std::to_string(prod(s)) + ")");
  }
  return axis < 0 ? axis + n : axis;
}
// Step one of Net::Net for a layer: the LayerParameter message as written, every sub-message the built layers read included.
// What depends on the bottoms' shapes (canonical axes, global pooling) is resolved by the shape step.
LayerParameter read_layer(const PMessage& lp, Phase phase, int batch_override) {
  static const PMessage none;                           // an absent sub-message reads as its defaults
  auto sub = [&](const char* k) -> const PMessage& { const PMessage* m = lp.sub(k); return m ? *m : none; };
  LayerParameter p;
  p.name = lp.str("name");
  p.type = lp.str("type");
  p.phase = phase;
  for (const PField* f : lp.all("loss_weight")) p.loss_weight.push_back((float)std::atof(f->scalar.c_str()));
  for (auto* b : lp.all("bottom")) p.bottom.push_back(b->scalar);
  for (auto* t : lp.all("top")) p.top.push_back(t->scalar);
  for (auto* ps : lp.all("param")) {
    ParamSpec s;
    if (ps->is_msg()) {
      const PMessage& m = *ps->msg;
      s.lr_mult = (float)m.num("lr_mult", 1.0); s.decay_mult = (float)m.num("decay_mult", 1.0);
      s.has_lr_mult = m.has("lr_mult"); s.has_decay_mult = m.has("decay_mult");
      s.name = m.str("name");
      const std::string sm = m.str("share_mode", "STRICT");
      s.share_mode = (sm == "PERMISSIVE" || sm == "1") ? 1 : 0;
    }
    p.param.push_back(s);
  }
  const PMessage& cp = sub("convolution_param");
  ConvolutionParameter& c = p.convolution_param;
  c.num_output = (int)cp.integer("num_output");
  c.bias_term = cp.boolean("bias_term", true);
  c.pad = to_int(cp.ints("pad")); c.kernel_size = to_int(cp.ints("kernel_size"));
  c.stride = to_int(cp.ints("stride")); c.dilation = to_int(cp.ints("dilation"));
  c.pad_h = (int)cp.integer("pad_h", -1);
  c.pad_w = (int)cp.integer("pad_w", -1);
  c.kernel_h = (int)cp.integer("kernel_h", -1);
  c.kernel_w = (int)cp.integer("kernel_w", -1);
  c.stride_h = (int)cp.integer("stride_h", -1);
  c.stride_w = (int)cp.integer("stride_w", -1);
  c.group = (int)cp.integer("group", 1);
  c.weight_filler = filler_of(cp.sub("weight_filler"));
  c.bias_filler = filler_of(cp.sub("bias_filler"));
  c.engine = engine_of(cp.str("engine", "DEFAULT"));
  c.axis = (int)cp.integer("axis", 1);
  c.force_nd_im2col = cp.boolean("force_nd_im2col", false);
  const PMessage& pp = sub("pooling_param");
  PoolingParameter& q = p.pooling_param;
  const std::string pool = pp.str("pool", "MAX");
  q.pool = pool == "AVE" || pool == "1" ? 1 : pool == "STOCHASTIC" || pool == "2" ? 2 : 0;
  q.global_pooling = pp.boolean("global_pooling", false);
  const int k = (int)pp.integer("kernel_size", 0), s = (int)pp.integer("stride", 1), pad = (int)pp.integer("pad", 0);
  q.kernel_h = (int)pp.integer("kernel_h", k); q.kernel_w = (int)pp.integer("kernel_w", k);
  q.stride_h = (int)pp.integer("stride_h", s); q.stride_w = (int)pp.integer("stride_w", s);
  q.pad_h = (int)pp.integer("pad_h", pad); q.pad_w = (int)pp.integer("pad_w", pad);
  const PMessage& ip = sub("inner_product_param");
  p.inner_product_param.num_output = (int)ip.integer("num_output");
  p.inner_product_param.bias_term = ip.boolean("bias_term", true);
  p.inner_product_param.weight_filler = filler_of(ip.sub("weight_filler"));
  p.inner_product_param.bias_filler = filler_of(ip.sub("bias_filler"));
  const PMessage& bp = sub("batch_norm_param");
  BatchNormParameter& bn = p.batch_norm_param;
  bn.scale_bias = bp.boolean("scale_bias", false) || bp.has("scale_filler") || bp.has("bias_filler");
  bn.eps = std::max((float)bp.num("eps", 1e-5), 1e-5f);
  bn.moving_average_fraction = (float)bp.num("moving_average_fraction", 0.999);
  if (bp.has("scale_filler")) bn.scale_filler = filler_of(bp.sub("scale_filler"));
  if (bp.has("bias_filler")) bn.bias_filler = filler_of(bp.sub("bias_filler"));
  p.relu_param.negative_slope = (float)sub("relu_param").num("negative_slope", 0.0);
  if (sub("prelu_param").has("filler")) p.prelu_param.filler = filler_of(sub("prelu_param").sub("filler"));
  p.prelu_param.channel_shared = sub("prelu_param").boolean("channel_shared", false);
  p.elu_param.alpha = (float)sub("elu_param").num("alpha", 1.0);
  const PMessage& pw = sub("power_param");
  p.power_param.power = (float)pw.num("power", 1.0); p.power_param.scale = (float)pw.num("scale", 1.0); p.power_param.shift = (float)pw.num("shift", 0.0);
  const PMessage& ep = sub("exp_param");
  p.exp_param.base = (float)ep.num("base", -1.0); p.exp_param.scale = (float)ep.num("scale", 1.0); p.exp_param.shift = (float)ep.num("shift", 0.0);
  const PMessage& lg = sub("log_param");
  p.log_param.base = (float)lg.num("base", -1.0); p.log_param.scale = (float)lg.num("scale", 1.0); p.log_param.shift = (float)lg.num("shift", 0.0);
  p.threshold_param.threshold = (float)sub("threshold_param").num("threshold", 0.0);
  const PMessage& lrn = sub("lrn_param");
  LRNParameter& l = p.lrn_param;
  l.local_size = (int)lrn.integer("local_size", 5); l.alpha = (float)lrn.num("alpha", 1.0); l.beta = (float)lrn.num("beta", 0.75);
  l.k = (float)lrn.num("k", 1.0);
  const std::string region = lrn.str("norm_region", "ACROSS_CHANNELS");
  l.norm_region = (region == "WITHIN_CHANNEL" || region == "1") ? 1 : 0;
  p.dropout_param.dropout_ratio = (float)sub("dropout_param").num("dropout_ratio", 0.5);
  const std::string op = sub("eltwise_param").str("operation", "SUM");
  p.eltwise_param.operation = (op == "PROD" || op == "0") ? 0 : (op == "MAX" || op == "2") ? 2 : 1;
  for (auto* f : sub("eltwise_param").all("coeff")) if (!f->is_msg()) p.eltwise_param.coeff.push_back((float)std::atof(f->scalar.c_str()));
  p.concat_param.axis = (int)sub("concat_param").integer("axis", 1);
  p.crop_param.axis = (int)sub("crop_param").integer("axis", 2);
  for (long long v : sub("crop_param").ints("offset")) p.crop_param.offset.push_back((int)v);
  const PMessage& sp = sub("slice_param");
  B2_CHECK(!(sp.has("axis") && sp.has("slice_dim")), "Either axis or slice_dim should be specified; not both.");   // slice_layer.cpp:12-13
  p.slice_param.slice_dim_given = sp.has("slice_dim");
  p.slice_param.axis = (int)(sp.has("slice_dim") ? sp.integer("slice_dim") : sp.integer("axis", 1));
  p.slice_param.slice_point = to_int(sp.ints("slice_point"));
  p.softmax_param.axis = (int)sub("softmax_param").integer("axis", 1);
  p.flatten_param.axis = (int)sub("flatten_param").integer("axis", 1);
  p.flatten_param.end_axis = (int)sub("flatten_param").integer("end_axis", -1);
  const PMessage& ap = sub("accuracy_param");
  p.accuracy_param.top_k = (int)ap.integer("top_k", 1);
  p.accuracy_param.axis = (int)ap.integer("axis", 1);
  p.accuracy_param.has_ignore_label = ap.has("ignore_label");
  p.accuracy_param.ignore_label = (int)ap.integer("ignore_label", 0);
  const PMessage& lsp = sub("loss_param");                     // softmax_loss_layer.cpp:29-40
  p.loss_param.has_ignore_label = lsp.has("ignore_label");
  p.loss_param.ignore_label = (int)lsp.integer("ignore_label", 0);
  if (lsp.has("normalization")) {
    const std::string nm = lsp.str("normalization");
    static const char* names[] = {"FULL", "VALID", "BATCH_SIZE", "NONE"};
    p.loss_param.normalization = -1;
    for (int i = 0; i < 4; ++i) if (nm == names[i] || nm == std::to_string(i)) p.loss_param.normalization = i;
    B2_CHECK(p.loss_param.normalization >= 0, "Unknown normalization mode: " + nm);
  } else if (lsp.has("normalize")) {
    p.loss_param.normalization = lsp.boolean("normalize", true) ? 1 : 2;
  }
  p.contrastive_loss_param.margin = (float)sub("contrastive_loss_param").num("margin", 1.0);
  p.contrastive_loss_param.legacy_version = sub("contrastive_loss_param").boolean("legacy_version", false);
  const PMessage& tp = sub("transform_param");
  TransformationParameter& t = p.transform_param;
  t.crop_size = (int)tp.integer("crop_size", 0);
  t.mirror = tp.boolean("mirror", false);
  t.scale = (float)tp.num("scale", 1.0);
  for (auto* f : tp.all("mean_value")) if (!f->is_msg()) t.mean_value.push_back((float)std::atof(f->scalar.c_str()));
  t.mean_file = tp.str("mean_file");
  t.random_seed = tp.integer("random_seed", -1);
  const PMessage& dp = lp.sub("data_param") ? sub("data_param") : sub("image_data_param");
  DataParameter& d = p.data_param;
  d.batch_size = batch_override > 0 ? batch_override : (int)dp.integer("batch_size", 1);
  d.source = dp.str("source");
  const std::string be = dp.str("backend", "LEVELDB");
  d.backend = (be == "LMDB" || be == "1") ? 1 : 0;
  d.parser_threads = (int)dp.integer("parser_threads", 0);
  d.force_encoded_color = dp.boolean("force_encoded_color", false);
  d.cache = dp.boolean("cache", false);
  d.shuffle = dp.boolean("shuffle", false);
  return p;
}
}  // namespace

int LabelBottom(const std::string& type) {
  if (type == "ContrastiveLoss") return 2;          // the similarity label (ContrastiveLossLayer::AllowForceBackward(2) is false)
  if (type == "Crop") return 1;                     // the reference blob: a shape, never a gradient
  return type == "SoftmaxWithLoss" || type == "SigmoidCrossEntropyLoss" || type == "Accuracy" ? 1 : -1;
}
bool IsLossType(const std::string& ty) { return ty.size() >= 4 && ty.compare(ty.size() - 4, 4, "Loss") == 0; }
float TopLossWeight(const LayerParameter& p, size_t t) {
  return t < p.loss_weight.size() ? p.loss_weight[t] : (IsLossType(p.type) && t == 0 ? 1.f : 0.f);
}
float LayerBase::loss_weight() const { return TopLossWeight(layer_param_, 0); }
int pooled_extent(int in, int k, int s, int p) {
  int o = (int)std::ceil((float)(in + 2 * p - k) / s) + 1;
  if (p > 0 && (o - 1) * s >= in + p) --o;
  return o;
}
void CropShape(const std::vector<int>& bottom, const std::vector<int>& ref, const CropParameter& q, std::vector<int>* top,
               std::vector<int>* offsets) {
  const int nax = (int)bottom.size();
  auto check_eq = [](long long u, long long v, const std::string& what) {
    if (u != v) Fatal(__FILE__, __LINE__, "Check failed: " + what + " (" + std::to_string(u) + " vs. " + std::to_string(v) + ") ");
  };
  check_eq(nax, (long long)ref.size(), "bottom[0]->num_axes() == bottom[1]->num_axes()");
  if (q.axis < -nax || q.axis >= nax)                                 // Blob::CanonicalAxisIndex
    Fatal(__FILE__, __LINE__, "axis " + std::to_string(q.axis) + " out of range for " + std::to_string(nax) + "-D Blob with shape");
  const int start = q.axis < 0 ? q.axis + nax : q.axis;
  if (q.offset.size() > 1)
    check_eq((long long)q.offset.size(), nax - start,
             "param.offset_size() == num_dims - start_axis number of offset values specified must be equal to the number of dimensions "
             "following axis.");
  *top = bottom;
  offsets->assign(nax, 0);
  for (int i = start; i < nax; ++i) {
    const int o = q.offset.empty() ? 0 : q.offset.size() == 1 ? q.offset[0] : q.offset[i - start];
    (*top)[i] = ref[i];
    if (!(bottom[i] - o >= ref[i]))
      Fatal(__FILE__, __LINE__, "Check failed: bottom[0]->shape(i) - crop_offset >= bottom[1]->shape(i) (" + std::to_string(bottom[i] - o) +
                                    " vs. " + std::to_string(ref[i]) + ") invalid crop parameters in dimension: " + std::to_string(i));
    B2_CHECK(o >= 0, "Crop: negative offset in dimension " + std::to_string(i));
    (*offsets)[i] = o;
  }
}
PoolingParameter EffectivePooling(const PoolingParameter& q, int h, int w) {
  PoolingParameter e = q;
  if (q.global_pooling) { e.kernel_h = h; e.kernel_w = w; e.stride_h = e.stride_w = 1; e.pad_h = e.pad_w = 0; }
  return e;
}

Net Net::FromFile(const std::string& path, Phase phase, int batch_override) {
  return Net(ParseTextProtoFile(path), phase, batch_override);
}
size_t Net::learnable_count() const { size_t c = 0; for (auto& p : params_) c += p.count; return c; }
std::pair<int, int> Net::param_owner(int layer_id, int layer_blob) const {
  for (const LearnableParam& p : net_params_)
    if (p.layer_id == layer_id && p.layer_blob == layer_blob && p.owner >= 0)
      return {net_params_[p.owner].layer_id, net_params_[p.owner].layer_blob};
  return {-1, -1};
}

Net::Net(const PMessage& np, Phase phase, int batch_override, int default_channels, int default_size) {
  name_ = np.str("name");
  phase_ = phase;
  reduce_buckets_ = (int)np.integer("reduce_buckets", 6);          // caffe.proto:140
  global_grad_scale_ = (float)np.num("global_grad_scale", 1.0);    // caffe.proto:130
  if (!np.all("layers").empty()) Fatal(__FILE__, __LINE__, "V1 'layers' prototxt: run upgrade_net_proto_text first (not on this path)");
  // net-level inputs (deploy-style prototxts): input: "data" input_shape { dim: ... } / input_dim: ...
  {
    const auto names = np.all("input");
    const auto shp = np.all("input_shape");
    const auto dims = np.ints("input_dim");
    for (size_t i = 0; i < names.size(); ++i) {
      std::vector<int> s;
      if (i < shp.size() && shp[i]->is_msg()) s = to_int(shp[i]->msg->ints("dim"));
      else if (dims.size() >= 4 * (i + 1)) s.assign(dims.begin() + 4 * i, dims.begin() + 4 * i + 4);
      if (batch_override > 0 && !s.empty()) s[0] = batch_override;
      shapes_[names[i]->scalar] = s;
    }
  }
  std::map<std::string, bool> need_bw;
  std::map<std::string, int> param_names;               // param name -> its owner's index in net_params_ (Net::param_names_index_)
  std::map<std::string, std::string> bn_stat_names;     // names given to BatchNorm statistics blobs -> the layer
  std::vector<bool> has_lr, has_decay;                  // per learnable param: lr_mult / decay_mult given (Net::has_params_lr_)
  for (auto* lf : np.all("layer")) {
    if (!lf->is_msg()) continue;
    const PMessage& lp = *lf->msg;
    if (!layer_included(lp, phase)) continue;
    NetLayer L;
    L.param = read_layer(lp, phase, batch_override);
    LayerParameter& P = L.param;
    const std::string& type = P.type;
    const int id = (int)layers_.size();
    auto bottom_shape = [&](int i) -> const std::vector<int>& {
      B2_CHECK(i < (int)P.bottom.size(), "layer " + P.name + " has too few bottoms");
      auto it = shapes_.find(P.bottom[i]);
      if (it == shapes_.end()) Fatal(__FILE__, __LINE__, "Unknown bottom blob '" + P.bottom[i] + "' (layer '" + P.name + "')");
      return it->second;
    };
    std::vector<std::vector<int>> tops;
    std::vector<std::pair<std::vector<int>, int>> blobs;   // learnable blob shapes (+ index into ParamSpecs)
    bool is_data = false;

    if (type == "Data" || type == "ImageData" || type == "HDF5Data") {
      is_data = true;
      const DataParameter& dp = P.data_param;
      const int crop = P.transform_param.crop_size;
      int dc = default_channels, dh = default_size, dw = default_size;
      if (type == "Data") {
        // DataLayerSetUp reads one datum to size the top blob (data_layer.cpp:176-183); so does this, when the database is there
        L.use_database = UseDatabase(dp.source, dp.backend);
        bool float_data = false;
        if (L.use_database) PeekDatumShape(dp.source, &dc, &dh, &dw, dp.force_encoded_color, nullptr, &float_data);
        const TransformationParameter& tp = P.transform_param;
        B2_CHECK(!float_data || FloatDatumsTakeNoTransform(tp.scale, tp.mirror, tp.crop_size, !tp.mean_value.empty() || !tp.mean_file.empty()),
                 "Data layer '" + P.name + "': " + kFloatDatumTransformMsg);
      }
      if (crop > 0) {
        if (L.use_database) B2_CHECK(dh >= crop && dw >= crop, "crop_size larger than the datums of " + dp.source);
        dh = dw = crop;
      }
      tops.push_back({dp.batch_size, dc, dh, dw});
      tops.push_back({dp.batch_size});
    } else if (type == "Input" || type == "DummyData") {
      is_data = true;
      const PMessage* ip = lp.sub(type == "Input" ? "input_param" : "dummy_data_param");
      B2_CHECK(ip != nullptr, type + " layer needs its parameter message");
      const auto shp = ip->all("shape");
      for (size_t i = 0; i < P.top.size(); ++i) {
        B2_CHECK(!shp.empty(), "Input layer needs shape");
        const PField* sf = shp[std::min(i, shp.size() - 1)];
        B2_CHECK(sf->is_msg(), type + " layer: `shape` must be a message { dim: ... }");
        std::vector<int> s = to_int(sf->msg->ints("dim"));
        if (batch_override > 0 && !s.empty()) s[0] = batch_override;
        tops.push_back(s);
      }
    } else if (type == "Convolution") {
      const PMessage* cp = lp.sub("convolution_param");
      B2_CHECK(cp != nullptr, "Convolution layer without convolution_param");
      const ConvolutionParameter& c = P.convolution_param;
      const std::vector<int>& bs = bottom_shape(0);
      B2_CHECK(bs.size() == 4, "2-D convolution expects a 4-D bottom");
      auto ax = [&](const std::vector<int>& rep, int hv, int wv, int dflt, int which) {
        if (hv >= 0 || wv >= 0) return which == 0 ? hv : wv;
        if (rep.empty()) return dflt;
        return rep[rep.size() == 1 ? 0 : which];
      };
      b2c_conv_params p{};
      p.N = bs[0]; p.C = bs[1]; p.H = bs[2]; p.W = bs[3]; p.O = c.num_output; p.G = c.group;
      p.kh = ax(c.kernel_size, c.kernel_h, c.kernel_w, 0, 0); p.kw = ax(c.kernel_size, c.kernel_h, c.kernel_w, 0, 1);
      p.sh = ax(c.stride, c.stride_h, c.stride_w, 1, 0); p.sw = ax(c.stride, c.stride_h, c.stride_w, 1, 1);
      p.ph = ax(c.pad, c.pad_h, c.pad_w, 0, 0); p.pw = ax(c.pad, c.pad_h, c.pad_w, 0, 1);
      p.dh = ax(c.dilation, -1, -1, 1, 0); p.dw = ax(c.dilation, -1, -1, 1, 1);
      p.has_bias = c.bias_term;
      B2_CHECK(p.kh > 0 && p.kw > 0, "Filter dimensions must be nonzero.");
      B2_CHECK(p.sh > 0 && p.sw > 0, "Stride dimensions must be nonzero.");                 // base_conv_layer.cpp:66-69
      B2_CHECK(p.dh > 0 && p.dw > 0 && p.ph >= 0 && p.pw >= 0, "dilation must be positive and pad non-negative");
      B2_CHECK(p.G > 0 && p.O > 0, "num_output and group must be positive");
      B2_CHECK(p.C % p.G == 0 && p.O % p.G == 0, "channels / num_output must be multiples of group");
      const int Ho = (p.H + 2 * p.ph - (p.dh * (p.kh - 1) + 1)) / p.sh + 1;     // conv_layer.cpp:7-22
      const int Wo = (p.W + 2 * p.pw - (p.dw * (p.kw - 1) + 1)) / p.sw + 1;
      tops.push_back({p.N, p.O, Ho, Wo});
      blobs.push_back({{p.O, p.C / p.G, p.kh, p.kw}, 0});
      if (c.bias_term) blobs.push_back({{p.O}, 1});
      convs_.push_back(ConvEntry{P.name, id, p, false});   // propagate_down: set once need-backward is final, below
    } else if (type == "Deconvolution") {
      // ConvolutionLayer's checks (base_conv_layer.cpp), the output extent of deconv_layer.cpp:7-22, weights [C, O/G, k...]
      B2_CHECK(lp.sub("convolution_param") != nullptr, "Deconvolution layer without convolution_param");
      const ConvolutionParameter& c = P.convolution_param;
      const std::vector<int>& bs = bottom_shape(0);
      const int caxis = canonical_axis(c.axis, bs), nsp = (int)bs.size() - caxis - 1;
      B2_CHECK(nsp >= 1, "convolution needs at least one spatial axis");
      auto ax = [&](const std::vector<int>& rep, int hv, int wv, int dflt, int i, const char* what) {
        if (hv >= 0 || wv >= 0) {
          B2_CHECK(nsp == 2, std::string(what) + "_h & " + what + "_w can only be used for 2D convolution.");
          B2_CHECK(rep.empty(), std::string("Either ") + what + " or " + what + "_h/w should be specified; not both.");
          return std::max(i == 0 ? hv : wv, 0);       // the unset one of the pair reads as the proto's 0
        }
        B2_CHECK(rep.size() <= 1 || (int)rep.size() == nsp, std::string(what) + " must be specified once, or once per spatial dimension");
        return rep.empty() ? dflt : rep[rep.size() == 1 ? 0 : i];
      };
      B2_CHECK(c.num_output > 0 && c.group > 0, "num_output and group must be positive");
      B2_CHECK(bs[caxis] % c.group == 0 && c.num_output % c.group == 0, "channels / num_output must be multiples of group");
      std::vector<int> top(bs.begin(), bs.begin() + caxis + 1), wshape{bs[caxis], c.num_output / c.group};
      top[caxis] = c.num_output;
      for (int i = 0; i < nsp; ++i) {
        const int k = ax(c.kernel_size, c.kernel_h, c.kernel_w, 0, i, "kernel_size"), s = ax(c.stride, c.stride_h, c.stride_w, 1, i, "stride");
        const int pd = ax(c.pad, c.pad_h, c.pad_w, 0, i, "pad"), d = ax(c.dilation, -1, -1, 1, i, "dilation");
        B2_CHECK(k > 0, "Filter dimensions must be nonzero.");
        B2_CHECK(s > 0, "Stride dimensions must be nonzero.");
        B2_CHECK(d > 0 && pd >= 0, "dilation must be positive and pad non-negative");
        const int o = s * (bs[caxis + 1 + i] - 1) + d * (k - 1) + 1 - 2 * pd;
        B2_CHECK(o > 0, "Deconvolution: non-positive output extent (pad larger than the upsampled input)");
        top.push_back(o);
        wshape.push_back(k);
      }
      tops.push_back(top);
      blobs.push_back({wshape, 0});
      if (c.bias_term) blobs.push_back({{c.num_output}, 1});
    } else if (type == "Crop") {
      std::vector<int> top, offsets;
      B2_CHECK(P.bottom.size() == 2, "Crop Layer takes 2 bottom blobs: the blob to crop and the one whose shape it takes");
      CropShape(bottom_shape(0), bottom_shape(1), P.crop_param, &top, &offsets);
      tops.push_back(top);
    } else if (type == "Pooling") {
      const std::vector<int>& bs = bottom_shape(0);
      B2_CHECK(bs.size() == 4, "Pooling expects a 4-D bottom (num, channels, height, width)");   // pooling_layer.cpp:84-86
      PoolingParameter& q = P.pooling_param;
      q = EffectivePooling(q, bs[2], bs[3]);
      B2_CHECK(q.kernel_h > 0 && q.kernel_w > 0, "Filter dimensions cannot be zero.");
      B2_CHECK(q.stride_h > 0 && q.stride_w > 0 && q.pad_h >= 0 && q.pad_w >= 0, "Pooling stride must be positive and pad non-negative");
      tops.push_back({bs[0], bs[1], pooled_extent(bs[2], q.kernel_h, q.stride_h, q.pad_h), pooled_extent(bs[3], q.kernel_w, q.stride_w, q.pad_w)});
    } else if (type == "InnerProduct") {
      const PMessage* ip = lp.sub("inner_product_param");
      B2_CHECK(ip != nullptr, "InnerProduct layer without inner_product_param");
      const InnerProductParameter& q = P.inner_product_param;
      const std::vector<int>& bs = bottom_shape(0);
      B2_CHECK(bs.size() >= 2 && q.num_output > 0, "InnerProduct needs a bottom with at least 2 axes and a positive num_output");
      tops.push_back({bs[0], q.num_output});
      blobs.push_back({{q.num_output, (int)prod(bs, 1)}, 0});
      if (q.bias_term) blobs.push_back({{q.num_output}, 1});
    } else if (type == "BatchNorm") {
      const std::vector<int>& bs = bottom_shape(0);
      B2_CHECK(bs.size() >= 2, "BatchNorm needs a bottom with a channel axis");
      tops.push_back(bs);
      // blobs_[0..2] = running mean / variance / correction (statistics, not exchanged with the cuDNN engine:
      // include/caffe/layers/cudnn_batch_norm_layer.hpp:30-32); [3], [4] = scale, bias when scale_bias
      if (P.batch_norm_param.scale_bias) { blobs.push_back({{bs[1]}, 3}); blobs.push_back({{bs[1]}, 4}); }
    } else if (type == "Scale") {
      const PMessage* sp = lp.sub("scale_param");
      const std::vector<int>& bs = bottom_shape(0);
      B2_CHECK(bs.size() >= 2, "Scale needs a bottom with a channel axis");
      tops.push_back(bs);
      if (P.bottom.size() == 1) {
        blobs.push_back({{bs[1]}, 0});
        if (sp && sp->boolean("bias_term", false)) blobs.push_back({{bs[1]}, 1});
      }
    } else if (type == "Concat") {
      const int axis = P.concat_param.axis;
      std::vector<int> s = bottom_shape(0);
      B2_CHECK(axis >= 0 && axis < (int)s.size(), "Concat: axis outside the bottom's axes");
      for (size_t i = 1; i < P.bottom.size(); ++i) {
        const std::vector<int>& b = bottom_shape((int)i);
        B2_CHECK(b.size() == s.size(), "Concat: all inputs must have the same #axes.");
        s[axis] += b[axis];
      }
      tops.push_back(s);
    } else if (type == "Flatten") {
      FlattenParameter& f = P.flatten_param;
      const std::vector<int>& bs = bottom_shape(0);
      B2_CHECK(P.top.empty() || P.top[0] != P.bottom[0], "Flatten Layer does not allow in-place computation.");
      f.axis = canonical_axis(f.axis, bs);                                                          // flatten_layer.cpp:8-30
      f.end_axis = canonical_axis(f.end_axis, bs);
      std::vector<int> s(bs.begin(), bs.begin() + f.axis);
      int flat = 1;
      for (int a = f.axis; a <= f.end_axis; ++a) flat *= bs[a];
      s.push_back(flat);
      for (int a = f.end_axis + 1; a < (int)bs.size(); ++a) s.push_back(bs[a]);
      tops.push_back(s);
    } else if (type == "Softmax") {
      P.softmax_param.axis = canonical_axis(P.softmax_param.axis, bottom_shape(0));                 // softmax_layer.cpp:12-13
      tops.push_back(bottom_shape(0));
    } else if (type == "SoftmaxWithLoss" || type == "EuclideanLoss" || type == "L1Loss" || type == "SigmoidCrossEntropyLoss" || type == "Accuracy") {
      if (type == "EuclideanLoss" || type == "L1Loss" || type == "SigmoidCrossEntropyLoss") {
        const std::vector<int>& a = bottom_shape(0);
        const std::vector<int>& b = bottom_shape(1);
        B2_CHECK(!a.empty() && !b.empty() && a[0] == b[0], "The data and label should have the same number.");   // loss_layer.cpp:19-20
        if (type != "SigmoidCrossEntropyLoss") B2_CHECK(prod(a, 1) == prod(b, 1), "Inputs must have the same dimension.");  // l1_loss_layer.cpp:14-15 too
        else B2_CHECK(prod(a) == prod(b), "SIGMOID_CROSS_ENTROPY_LOSS layer inputs must have the same count.");
      }
      for (size_t i = 0; i < P.top.size(); ++i) tops.push_back({});
      if (type == "SoftmaxWithLoss" || type == "Accuracy") {
        // softmax_loss_layer.cpp:47-61, accuracy_layer.cpp:21-42: the class axis, the [outer, C, inner] view, one label per pixel
        const std::vector<int>& a = bottom_shape(0);
        const size_t labels = prod(bottom_shape(1));
        if (type == "Accuracy")
          B2_CHECK(labels > 0 && P.accuracy_param.top_k <= (long long)(prod(a) / labels), "top_k must be less than or equal to the number of classes.");
        int& axis = type == "Accuracy" ? P.accuracy_param.axis : P.softmax_param.axis;
        axis = canonical_axis(axis, a);
        const size_t outer = prod(std::vector<int>(a.begin(), a.begin() + axis)), inner = prod(a, axis + 1);
        // nets of the [N, C] form without ignore_label or a second top are checked by the layers' Reshape, as they always were
        const bool spatial = inner > 1 || tops.size() > 1 || (type == "Accuracy" ? P.accuracy_param.has_ignore_label : P.loss_param.has_ignore_label);
        if (spatial && outer * inner != labels)
          Fatal(__FILE__, __LINE__, "Check failed: outer_num_ * inner_num_ == bottom[1]->count() (" + std::to_string(outer * inner) + " vs. " +
                                        std::to_string(labels) + ") Number of labels must match number of predictions; e.g., if " +
                                        (type == "Accuracy" ? "label" : "softmax") + " axis == 1 and prediction shape is (N, C, H, W), label count "
                                        "(number of labels) must be N*H*W, with integer values in {0, 1, ..., C-1}.");
        if (tops.size() > 1) tops[1] = type == "Accuracy" ? std::vector<int>{a[axis]} : a;
      }
    } else if (type == "Slice") {
      SliceParameter& sp = P.slice_param;
      const std::vector<int> bs = bottom_shape(0);
      const size_t ntop = P.top.size();
      B2_CHECK(ntop >= 1, "Slice layer needs at least one top");
      if (sp.slice_dim_given) {                                                                                          // slice_layer.cpp:26-33
        B2_CHECK(sp.axis >= 0, "casting slice_dim from uint32 to int32 produced negative result; slice_dim must satisfy 0 <= slice_dim < 32");
        B2_CHECK(sp.axis < (int)bs.size(), "slice_dim out of range.");
      } else {
        sp.axis = canonical_axis(sp.axis, bs);
      }
      const int extent = bs[sp.axis];
      const std::vector<int>& points = sp.slice_point;
      std::vector<int> slices;
      if (!points.empty()) {                                                                                              // :40-56
        if (points.size() != ntop - 1)
          Fatal(__FILE__, __LINE__, "Check failed: slice_point_.size() == top.size() - 1 (" + std::to_string(points.size()) + " vs. " +
                                        std::to_string(ntop - 1) + ") ");
        if ((int)ntop > extent)
          Fatal(__FILE__, __LINE__, "Check failed: top.size() <= bottom_slice_axis (" + std::to_string(ntop) + " vs. " + std::to_string(extent) + ") ");
        int prev = 0;
        for (int p : points) {
          if (!(p > prev)) Fatal(__FILE__, __LINE__, "Check failed: slice_point_[i] > prev (" + std::to_string(p) + " vs. " + std::to_string(prev) + ") ");
          slices.push_back(p - prev);
          prev = p;
        }
        slices.push_back(extent - prev);
        if (slices.back() < 0)                                                                                            // Blob::Reshape's CHECK
          Fatal(__FILE__, __LINE__, "Check failed: shape[i] >= 0 (" + std::to_string(slices.back()) + " vs. 0) ");
      } else {                                                                                                            // :57-64
        if (extent % (int)ntop != 0)
          Fatal(__FILE__, __LINE__, "Check failed: bottom_slice_axis % top.size() == 0 (" + std::to_string(extent % (int)ntop) + " vs. 0) Number of top blobs (" +
                                        std::to_string(ntop) + ") should evenly divide input slice axis (" + std::to_string(extent) + ")");
        slices.assign(ntop, extent / (int)ntop);
      }
      for (int s : slices) {
        std::vector<int> t = bs;
        t[sp.axis] = s;
        tops.push_back(t);
      }
    } else if (type == "ContrastiveLoss") {
      // contrastive_loss_layer.cpp:13-20 and LossLayer::Reshape, on the legacy num / channels / height / width view (Blob::LegacyShape:
      // a missing axis reads as 1, so an [N, C] feature blob is [N, C, 1, 1])
      const std::vector<int>& a = bottom_shape(0);
      const std::vector<int>& b = bottom_shape(1);
      const std::vector<int>& y = bottom_shape(2);
      for (const std::vector<int>* s : {&a, &b, &y})
        B2_CHECK(s->size() <= 4, "Cannot use legacy accessors on Blobs with > 4 axes.");
      auto legacy = [](const std::vector<int>& s, int i) { return i < (int)s.size() ? s[i] : 1; };
      auto check_eq = [](int u, int v, const char* what) {
        if (u != v) Fatal(__FILE__, __LINE__, std::string("Check failed: ") + what + " (" + std::to_string(u) + " vs. " + std::to_string(v) + ") ");
      };
      check_eq(legacy(a, 1), legacy(b, 1), "bottom[0]->channels() == bottom[1]->channels()");
      check_eq(legacy(a, 2), 1, "bottom[0]->height() == 1");
      check_eq(legacy(a, 3), 1, "bottom[0]->width() == 1");
      check_eq(legacy(b, 2), 1, "bottom[1]->height() == 1");
      check_eq(legacy(b, 3), 1, "bottom[1]->width() == 1");
      check_eq(legacy(y, 1), 1, "bottom[2]->channels() == 1");
      check_eq(legacy(y, 2), 1, "bottom[2]->height() == 1");
      check_eq(legacy(y, 3), 1, "bottom[2]->width() == 1");
      B2_CHECK(!a.empty() && !b.empty() && a[0] == b[0], "The data and label should have the same number.");     // loss_layer.cpp:19-20
      // not in the reference, which reads bottom[2][i] for every pair without checking: one label per pair
      B2_CHECK(!y.empty() && y[0] == a[0], "ContrastiveLoss: the similarity blob needs one label per pair");
      for (size_t i = 0; i < P.top.size(); ++i) tops.push_back({});
    } else if (type == "PReLU") {
      const std::vector<int>& bs = bottom_shape(0);
      B2_CHECK(bs.size() >= 2, "Number of axes of bottom blob must be >=2.");                              // prelu_layer.cpp:12-13
      tops.push_back(bs);
      // blobs_[0]: the negative slopes, one per channel, or a 0-axis blob (count 1) when channel_shared (prelu_layer.cpp:20-25)
      blobs.push_back({P.prelu_param.channel_shared ? std::vector<int>{} : std::vector<int>{bs[1]}, 0});
    } else if (type == "Exp" || type == "Log") {
      const float base = type == "Exp" ? P.exp_param.base : P.log_param.base;
      B2_CHECK(base == -1.f || base > 0.f, "base must be strictly positive.");                            // exp_layer.cpp:13-15, log_layer.cpp:13-15
      tops.push_back(bottom_shape(0));
    } else if (type == "ReLU" || type == "Dropout" || type == "LRN" || type == "Eltwise" || type == "Sigmoid" ||
               type == "TanH" || type == "Power" || type == "Bias" || type == "ELU" || type == "Split" || type == "AbsVal" ||
               type == "BNLL" || type == "Threshold") {
      for (size_t i = 0; i < std::max<size_t>(1, P.top.size()); ++i) tops.push_back(bottom_shape(0));
    } else {
      Fatal(__FILE__, __LINE__, "Unknown layer type: " + type + " (layer '" + P.name + "')");
    }


    // need-backward analysis (Net::Init, net.cpp:160-283): data tops never need it; a layer needs backward if a
    // bottom does or it owns a parameter with a non-zero lr_mult
    bool layer_bw = false;
    for (auto& b : L.param.bottom) layer_bw |= need_bw.count(b) ? need_bw[b] : false;
    for (auto& bl : blobs) {
      const ParamSpec spec = bl.second < (int)L.param.param.size() ? L.param.param[bl.second] : ParamSpec();
      if (spec.lr_mult != 0.f) layer_bw = true;
    }
    if (is_data) layer_bw = false;
    L.need_backward = layer_bw;
    for (size_t i = 0; i < L.param.bottom.size(); ++i) {     // a label / target bottom never receives a gradient (LabelBottom)
      const bool want = layer_bw && (need_bw.count(L.param.bottom[i]) ? need_bw[L.param.bottom[i]] : false);
      L.propagate_down.push_back(want && (int)i != LabelBottom(type));
      if (want && (int)i == LabelBottom(type)) L.label_wants_gradient = true;
    }
    for (size_t i = 0; i < L.param.top.size(); ++i) {
      B2_CHECK(i < tops.size(), "layer '" + L.param.name + "' declares more tops than its type produces");
      shapes_[L.param.top[i]] = tops[i];
      need_bw[L.param.top[i]] = layer_bw;
    }
    // parameter sharing (Net::AppendParam, net.cpp:576-666).  BatchNorm's statistics (blobs 0-2) are not learnable blobs here; a
    // name on one of them is refused as soon as a second blob would carry it: two layers would update one running mean
    if (type == "BatchNorm")
      for (int i = 0; i < 3 && i < (int)L.param.param.size(); ++i) {
        const std::string& nm = L.param.param[i].name;
        if (nm.empty()) continue;
        B2_CHECK(!param_names.count(nm) && !bn_stat_names.count(nm),
                 "Cannot share param '" + nm + "' with BatchNorm layer '" + L.param.name + "' statistics blob " + std::to_string(i) +
                     ": two layers would update one running statistic");
        bn_stat_names[nm] = L.param.name;
      }
    int bid = 0;
    for (auto& bl : blobs) {
      const ParamSpec spec = bl.second < (int)L.param.param.size() ? L.param.param[bl.second] : ParamSpec();
      LearnableParam p{L.param.name, id, bid++, prod(bl.first), bl.first, spec.lr_mult, spec.decay_mult};
      p.layer_blob = bl.second;
      p.name = spec.name;
      if (!spec.name.empty() && bn_stat_names.count(spec.name))
        Fatal(__FILE__, __LINE__, "Cannot share param '" + spec.name + "' with BatchNorm layer '" + bn_stat_names[spec.name] +
                                      "' statistics blob: two layers would update one running statistic");
      auto it = spec.name.empty() ? param_names.end() : param_names.find(spec.name);
      if (it == param_names.end()) {                    // anonymous, or a name seen for the first time: this blob owns it
        if (!spec.name.empty()) param_names[spec.name] = (int)net_params_.size();
        p.learnable_id = (int)params_.size();
        params_.push_back(p);
        has_lr.push_back(spec.has_lr_mult);
        has_decay.push_back(spec.has_decay_mult);
      } else {                                          // a sharer: same storage, same update
        const LearnableParam& o = net_params_[it->second];
        auto shape_str = [](const std::vector<int>& s) {
          std::string r;
          for (int d : s) r += std::to_string(d) + " ";
          return r + "(" + std::to_string(prod(s)) + ")";
        };
        const std::string who = "Cannot share param '" + spec.name + "' owned by layer '" + o.layer + "' with layer '" + L.param.name + "'; ";
        if (spec.share_mode == 1) {                     // PERMISSIVE: the reference then reshapes the sharer; only STRICT is built
          B2_CHECK(p.count == o.count, who + "count mismatch.  Owner layer param shape is " + shape_str(o.shape) + "; sharing layer shape is " +
                                           shape_str(p.shape));
          B2_CHECK(p.shape == o.shape, who + "share_mode PERMISSIVE with a different shape is not built (only STRICT sharing is).  Owner "
                                           "layer param shape is " + shape_str(o.shape) + "; sharing layer expects shape " + shape_str(p.shape));
        }
        B2_CHECK(p.shape == o.shape, who + "shape mismatch.  Owner layer param shape is " + shape_str(o.shape) + "; sharing layer expects shape " +
                                         shape_str(p.shape));
        p.owner = it->second;
        p.learnable_id = o.learnable_id;
        LearnableParam& lo = params_[o.learnable_id];
        if (spec.has_lr_mult) {                         // net.cpp:647-664: agree where both are given, else the sharer's value is adopted
          B2_CHECK(!has_lr[o.learnable_id] || spec.lr_mult == lo.lr_mult, "Shared param '" + spec.name + "' has mismatched lr_mult.");
          has_lr[o.learnable_id] = true;
          lo.lr_mult = spec.lr_mult;
        }
        if (spec.has_decay_mult) {
          B2_CHECK(!has_decay[o.learnable_id] || spec.decay_mult == lo.decay_mult, "Shared param '" + spec.name + "' has mismatched decay_mult.");
          has_decay[o.learnable_id] = true;
          lo.decay_mult = spec.decay_mult;
        }
      }
      net_params_.push_back(p);
    }
    layer_top_shapes_.push_back(tops);
    layers_.push_back(std::move(L));
  }
  // loss pruning (net.cpp:285-330, blobs_under_loss): walking back from the last layer, a layer none of whose tops has a non-zero
  // loss weight or feeds a layer that reaches one does not run backward, and none of its bottoms gets a gradient.  (The
  // reference's skip-propagate-down half needs propagate_down params, which this parser does not take.)
  std::set<std::string> under_loss;
  for (int li = (int)layers_.size() - 1; li >= 0; --li) {
    NetLayer& L = layers_[li];
    bool contributes = false;
    for (size_t t = 0; t < L.param.top.size(); ++t)
      contributes |= TopLossWeight(L.param, t) != 0.f || under_loss.count(L.param.top[t]) > 0;
    if (!contributes) {
      L.need_backward = false;
      L.label_wants_gradient = false;
      L.propagate_down.assign(L.param.bottom.size(), false);
    } else {
      for (auto& b : L.param.bottom) under_loss.insert(b);
    }
  }
  // force_backward (net.cpp:342-360, after the pruning): every layer runs backward and every bottom gets a gradient except the ones
  // a loss layer refuses (LossLayer::AllowForceBackward: the label bottom).  Data layers have nothing to propagate to.
  if (np.boolean("force_backward", false)) {
    for (NetLayer& L : layers_) {
      const std::string& ty = L.param.type;
      if (ty == "Data" || ty == "ImageData" || ty == "HDF5Data" || ty == "Input" || ty == "DummyData") continue;
      L.need_backward = true;
      for (size_t i = 0; i < L.propagate_down.size(); ++i)
        if ((int)i != LabelBottom(ty)) L.propagate_down[i] = true;
    }
  }
  for (ConvEntry& c : convs_) c.propagate_down = layers_[c.layer_id].propagate_down[0];
  for (const NetLayer& L : layers_)
    if (IsLossType(L.param.type) && !L.param.top.empty() && TopLossWeight(L.param, 0) != 0.f) loss_blob_ = L.param.top[0];
}

// ================================================================================================ solver
SolverParameter ReadSolverParameter(const PMessage& m, std::string* net_path) {
  SolverParameter p;
  p.base_lr = (float)m.num("base_lr", p.base_lr);
  p.lr_policy = m.str("lr_policy", "fixed");
  p.gamma = (float)m.num("gamma", p.gamma);
  p.power = (float)m.num("power", p.power);
  p.momentum = (float)m.num("momentum", 0.0);
  p.momentum_policy = m.str("momentum_policy", "fixed");
  p.max_momentum = (float)m.num("max_momentum", 0.99);
  p.has_max_momentum = m.has("max_momentum");
  p.momentum_power = (float)m.num("momentum_power", 1.0);
  p.weight_decay = (float)m.num("weight_decay", 0.0);
  p.regularization_type = m.str("regularization_type", "L2");
  p.stepsize = (int)m.integer("stepsize", 1);
  for (long long v : m.ints("stepvalue")) p.stepvalue.push_back((int)v);
  p.max_iter = (int)m.integer("max_iter", 1);
  p.iter_size = (int)m.integer("iter_size", 1);
  p.clip_gradients = (float)m.num("clip_gradients", -1.0);
  p.rampup_interval = (int)m.integer("rampup_interval", 0);
  p.rampup_lr = (float)m.num("rampup_lr", 0.0);
  p.min_lr = (float)m.num("min_lr", 0.0);
  p.snapshot_diff = m.boolean("snapshot_diff", false);
  p.delta = (float)m.num("delta", 1e-8);
  p.momentum2 = (float)m.num("momentum2", 0.999);
  p.rms_decay = (float)m.num("rms_decay", 0.0);
  // the legacy solver_type enum (caffe.proto:288-297) becomes `type` as in UpgradeSolverType (upgrade_proto.cpp:1002-1040)
  p.type = m.str("type", "SGD");
  if (m.has("solver_type")) {
    B2_CHECK(!m.has("type"), "Failed to upgrade solver: old solver_type field (enum) and new type field (string) cannot be both "
                             "specified in solver proto text.");
    static const char* const legacy[][2] = {{"SGD", "SGD"}, {"NESTEROV", "Nesterov"}, {"ADAGRAD", "AdaGrad"},
                                            {"RMSPROP", "RMSProp"}, {"ADADELTA", "AdaDelta"}, {"ADAM", "Adam"}};
    const std::string e = m.str("solver_type");
    p.type.clear();
    for (auto& l : legacy) if (e == l[0] || e == std::to_string(&l - legacy)) p.type = l[1];
    if (p.type.empty()) Fatal(__FILE__, __LINE__, "Unknown SolverParameter solver_type: " + e + " (known: SGD, NESTEROV, ADAGRAD, RMSPROP, ADADELTA, ADAM)");
  }
  // testing: test nets come from the generic `net` only (Solver::InitTestNets, solver.cpp:107-185; the reference's model files
  // use nothing else), with phase TEST and no stages.  The other sources are recorded, and refused where test nets are built
  for (const char* f : {"test_net", "test_net_param", "test_state"})
    if (m.has(f)) p.test_fields_not_built.push_back(f);
  for (long long v : m.ints("test_iter")) p.test_iter.push_back((int)v);
  p.test_interval = (int)m.integer("test_interval", 0);
  p.test_compute_loss = m.boolean("test_compute_loss", false);
  if (!p.test_iter.empty()) B2_CHECK(p.test_interval > 0, "(test_interval > 0 when test_iter is given)");   // solver.cpp:135-137 CHECK_GT
  if (net_path) *net_path = m.str("net", m.str("train_net"));
  return p;
}

}  // namespace caffe
