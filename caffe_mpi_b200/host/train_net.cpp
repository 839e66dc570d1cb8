// train_net.cpp -- see train_net.hpp.
#include "train_net.hpp"
#include "proto_wire.hpp"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <cstdlib>
#include <set>

namespace caffe {

static cudaStream_t S() { return Caffe::thread_stream(); }
static bool env_on(const char* name, bool dflt) {        // a 0 / 1 switch from the environment
  const char* e = getenv(name);
  return e ? atoi(e) != 0 : dflt;
}

// ================================================================================================ ReLU
void ReLULayer::Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) {
  if (fused_away_) return;
  B2C_CHECK(b2c_relu_forward(b[0]->count(), b[0]->gpu_data(), t[0]->mutable_gpu_data(), negative_slope(), S()));
}
void ReLULayer::Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) {
  if (!pd[0] || fused_away_) return;
  // in place: bottom data == top data (post-activation), same (x > 0) mask for slope 0 (relu_layer.cpp:27-41)
  B2C_CHECK(b2c_relu_backward(b[0]->count(), t[0]->gpu_diff(), b[0]->gpu_data(), b[0]->mutable_gpu_diff(), negative_slope(), S()));
}

// ================================================================================================ BatchNorm
void BatchNormLayer::LayerSetUp(const vector<Blob*>& b, const vector<Blob*>&) {
  const int C = b[0]->num_axes() > 1 ? b[0]->shape(1) : 1;
  blobs_.resize(scale_bias_ ? 5 : 3);
  blobs_[0].reset(new Blob(vector<int>{C}));      // running mean
  blobs_[1].reset(new Blob(vector<int>{C}));      // running variance (+eps)
  blobs_[2].reset(new Blob(vector<int>{1}));      // variance correction (kept for blob-count compatibility)
  if (scale_bias_) {
    blobs_[3].reset(new Blob(vector<int>{C}));
    blobs_[4].reset(new Blob(vector<int>{C}));
    Fill(layer_param_.batch_norm_param.scale_filler, blobs_[3].get());   // batch_norm_layer.cpp:52-63
    Fill(layer_param_.batch_norm_param.bias_filler, blobs_[4].get());
  }
  param_propagate_down_.assign(blobs_.size(), false);
  if (scale_bias_) param_propagate_down_[3] = param_propagate_down_[4] = true;
}
void BatchNormLayer::Reshape(const vector<Blob*>& b, const vector<Blob*>& t) {
  if (t[0] != b[0]) t[0]->ReshapeLike(*b[0]);
  const int C = b[0]->shape(1);
  if (layer_param_.phase != TEST && !(recompute_ && t[0] != b[0])) xnorm_.ReshapeLike(*b[0]);
  save_mean_.Reshape({C}); save_invstd_.Reshape({C}); scratch_.Reshape({2 * C});
}
void BatchNormLayer::Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) {
  const int N = b[0]->shape(0), C = b[0]->shape(1), Sp = (int)(b[0]->count() / ((size_t)N * C));
  if (layer_param_.phase == TEST) {
    // TEST: normalise with the running statistics (batch_norm_layer.cu:22-34), [+ the residual tail's other operand], [ReLU]
    B2C_CHECK(b2c_bn_forward_inference(N, C, Sp, b[0]->gpu_data(), scale_bias_ ? blobs_[3]->gpu_data() : nullptr,
                                       scale_bias_ ? blobs_[4]->gpu_data() : nullptr, eps_, blobs_[0]->gpu_data(), blobs_[1]->gpu_data(),
                                       res_sum_ ? res_other_->gpu_data() : nullptr,
                                       res_sum_ ? res_sum_->mutable_gpu_data() : t[0]->mutable_gpu_data(), res_sum_ || fuse_relu_ ? 1 : 0, S()));
    return;
  }
  if (res_sum_) {
    // residual tail: sum_top = max(0, BatchNorm(x) + other); this layer's own top blob is not materialised
    B2C_CHECK(b2c_bn_forward_train_fused_res(N, C, Sp, b[0]->gpu_data(), scale_bias_ ? blobs_[3]->gpu_data() : nullptr,
                                             scale_bias_ ? blobs_[4]->gpu_data() : nullptr, eps_, maf_, iter_ <= 1 ? 1 : 0,
                                             blobs_[0]->mutable_gpu_data(), blobs_[1]->mutable_gpu_data(), save_mean_.mutable_gpu_data(),
                                             save_invstd_.mutable_gpu_data(), res_other_->gpu_data(), res_sum_->mutable_gpu_data(), 1, S()));
    ++iter_;
    return;
  }
  if (recompute_ && t[0] != b[0]) {
    // fused form: no x_norm blob (backward recomputes it from the bottom), optional ReLU on the way out
    B2C_CHECK(b2c_bn_forward_train_fused(N, C, Sp, b[0]->gpu_data(), scale_bias_ ? blobs_[3]->gpu_data() : nullptr,
                                         scale_bias_ ? blobs_[4]->gpu_data() : nullptr, eps_, maf_, iter_ <= 1 ? 1 : 0,
                                         blobs_[0]->mutable_gpu_data(), blobs_[1]->mutable_gpu_data(), save_mean_.mutable_gpu_data(),
                                         save_invstd_.mutable_gpu_data(), t[0]->mutable_gpu_data(), fuse_relu_ ? 1 : 0, S()));
    ++iter_;
    return;
  }
  B2_CHECK(!fuse_relu_, "BatchNorm: ReLU fusion needs the recompute form (top != bottom)");
  B2C_CHECK(b2c_bn_forward_train(N, C, Sp, b[0]->gpu_data(), scale_bias_ ? blobs_[3]->gpu_data() : nullptr,
                                 scale_bias_ ? blobs_[4]->gpu_data() : nullptr, eps_, maf_, iter_ <= 1 ? 1 : 0,
                                 blobs_[0]->mutable_gpu_data(), blobs_[1]->mutable_gpu_data(), save_mean_.mutable_gpu_data(),
                                 save_invstd_.mutable_gpu_data(), xnorm_.mutable_gpu_data(), t[0]->mutable_gpu_data(), S()));
  ++iter_;
}
void BatchNormLayer::Backward_gpu(const vector<Blob*>& t, const vector<bool>&, const vector<Blob*>& b) {
  const int N = b[0]->shape(0), C = b[0]->shape(1), Sp = (int)(b[0]->count() / ((size_t)N * C));
  float* dg = scale_bias_ ? blobs_[3]->mutable_gpu_diff() : scratch_.mutable_gpu_data();
  float* db = scale_bias_ ? blobs_[4]->mutable_gpu_diff() : scratch_.mutable_gpu_data() + C;
  if (res_sum_) {
    B2C_CHECK(b2c_bn_backward_fused_res(N, C, Sp, res_sum_->gpu_diff(), res_part2_ ? res_part2_->gpu_diff() : nullptr, res_sum_->gpu_data(),
                                        b[0]->gpu_data(), save_mean_.gpu_data(),
                                        save_invstd_.gpu_data(), scale_bias_ ? blobs_[3]->gpu_data() : nullptr,
                                        scale_bias_ ? blobs_[4]->gpu_data() : nullptr, dg, db, b[0]->mutable_gpu_diff(),
                                        res_prop_ ? res_other_->mutable_gpu_diff() : nullptr, S()));
    return;
  }
  if (recompute_ && t[0] != b[0]) {
    B2C_CHECK(b2c_bn_backward_fused(N, C, Sp, t[0]->gpu_diff(), b[0]->gpu_data(), save_mean_.gpu_data(), save_invstd_.gpu_data(),
                                    scale_bias_ ? blobs_[3]->gpu_data() : nullptr, scale_bias_ ? blobs_[4]->gpu_data() : nullptr, dg, db,
                                    b[0]->mutable_gpu_diff(), fuse_relu_ ? 1 : 0, S()));
    return;
  }
  B2C_CHECK(b2c_bn_backward(N, C, Sp, t[0]->gpu_diff(), xnorm_.gpu_data(), scale_bias_ ? blobs_[3]->gpu_data() : nullptr,
                            save_invstd_.gpu_data(), dg, db, b[0]->mutable_gpu_diff(), S()));
}

// ================================================================================================ Pooling
PoolingLayer::~PoolingLayer() { if (mask_) cudaFree(mask_); }
void PoolingLayer::Reshape(const vector<Blob*>& b, const vector<Blob*>& t) {
  eff_ = EffectivePooling(layer_param_.pooling_param, b[0]->shape(2), b[0]->shape(3));
  t[0]->Reshape({b[0]->shape(0), b[0]->shape(1), pooled_extent(b[0]->shape(2), eff_.kernel_h, eff_.stride_h, eff_.pad_h),
                 pooled_extent(b[0]->shape(3), eff_.kernel_w, eff_.stride_w, eff_.pad_w)});
  if (eff_.pool == 0 && t[0]->count() > mask_cap_) {
    if (mask_) CUDA_CHECK(cudaFree(mask_));
    CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&mask_), sizeof(int) * t[0]->count()));
    mask_cap_ = t[0]->count();
  }
}
void PoolingLayer::Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) {
  B2C_CHECK(b2c_pool_forward(eff_.pool, b[0]->shape(0) * b[0]->shape(1), b[0]->shape(2), b[0]->shape(3), eff_.kernel_h, eff_.kernel_w,
                             eff_.stride_h, eff_.stride_w, eff_.pad_h, eff_.pad_w, b[0]->gpu_data(), t[0]->mutable_gpu_data(), mask_, S()));
}
void PoolingLayer::Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) {
  if (!pd[0]) return;
  B2C_CHECK(b2c_pool_backward(eff_.pool, b[0]->shape(0) * b[0]->shape(1), b[0]->shape(2), b[0]->shape(3), eff_.kernel_h, eff_.kernel_w,
                              eff_.stride_h, eff_.stride_w, eff_.pad_h, eff_.pad_w, t[0]->gpu_diff(), mask_, b[0]->mutable_gpu_diff(), S()));
}

// ================================================================================================ Eltwise SUM
void EltwiseLayer::Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) {
  B2_CHECK(b.size() >= 2, "Eltwise needs two bottoms");
  if (fused_away_) return;
  if (fuse_relu_ && b.size() == 2) {        // y = max(0, a + b): the in-place ReLU that follows is folded in
    B2C_CHECK(b2c_add_relu(t[0]->count(), b[0]->gpu_data(), b[1]->gpu_data(), t[0]->mutable_gpu_data(), S()));
    return;
  }
  B2C_CHECK(b2c_add(t[0]->count(), b[0]->gpu_data(), b[1]->gpu_data(), t[0]->mutable_gpu_data(), S()));
  for (size_t i = 2; i < b.size(); ++i) B2C_CHECK(b2c_add(t[0]->count(), t[0]->gpu_data(), b[i]->gpu_data(), t[0]->mutable_gpu_data(), S()));
}
void EltwiseLayer::Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) {
  if (fused_away_) return;
  if (fuse_relu_ && b.size() == 2) {        // dx_a = dx_b = dy * (y > 0): ReLU backward + the two copies of SUM's backward
    if (pd[0] || pd[1])
      B2C_CHECK(b2c_relu_backward2(t[0]->count(), t[0]->gpu_diff(), t[0]->gpu_data(), pd[0] ? b[0]->mutable_gpu_diff() : nullptr,
                                   pd[1] ? b[1]->mutable_gpu_diff() : nullptr, S()));
    return;
  }
  for (size_t i = 0; i < b.size(); ++i)
    if (pd[i]) CUDA_CHECK(cudaMemcpyAsync(b[i]->mutable_gpu_diff(), t[0]->gpu_diff(), sizeof(float) * t[0]->count(), cudaMemcpyDeviceToDevice, S()));
}

// ================================================================================================ InnerProduct
void InnerProductLayer::LayerSetUp(const vector<Blob*>& b, const vector<Blob*>&) {
  K_ = (int)b[0]->count(1);
  blobs_.resize(bias_ ? 2 : 1);
  blobs_[0].reset(new Blob(vector<int>{num_output_, K_}));
  Fill(layer_param_.inner_product_param.weight_filler, blobs_[0].get());
  if (bias_) { blobs_[1].reset(new Blob(vector<int>{num_output_})); Fill(layer_param_.inner_product_param.bias_filler, blobs_[1].get()); }
  param_propagate_down_.assign(blobs_.size(), true);
}
void InnerProductLayer::Reshape(const vector<Blob*>& b, const vector<Blob*>& t) {
  M_ = b[0]->shape(0);
  B2_CHECK((int)b[0]->count(1) == K_, "Input size incompatible with inner product parameters.");
  t[0]->Reshape({M_, num_output_});
  const size_t wsb = b2c_sgemm_workspace_bytes(0, 1, M_, num_output_, K_);
  if (wsb) gemm_ws_.Reshape({(int)((wsb + 3) / 4)});
  // backward: dW = dy^T[N x M] * (x^T[K x M])^T (reduction over the batch), dx = dy[M x N] * (W^T[K x N])^T (reduction over the outputs)
  const bool on = env_on("B2C_IP_BWD_TC", true);
  // dW: the reduction runs over the batch -- only a few K blocks per 128 x 128 output tile unless the batch is large; on AlexNet
  // (batch 256, 4096 x 9216 outputs) the tile set-up and the read-modify-write epilogue cost more than the FFMA kernel saves,
  // so the batch has to be at least 512
  bwd_w_tc_ = on && M_ >= 512 && b2c_sgemm_tc_supported(0, 1, num_output_, K_, M_) != 0;
  bwd_x_tc_ = on && b2c_sgemm_tc_supported(0, 1, M_, K_, num_output_) != 0;
  size_t bws = 0;
  if (bwd_w_tc_) { dyt_.Reshape({num_output_, M_}); xt_.Reshape({K_, M_}); bws = std::max(bws, b2c_sgemm_workspace_bytes(0, 1, num_output_, K_, M_)); }
  if (bwd_x_tc_) { wt_.Reshape({K_, num_output_}); bws = std::max(bws, b2c_sgemm_workspace_bytes(0, 1, M_, K_, num_output_)); }
  if (bws) bwd_ws_.Reshape({(int)((bws + 3) / 4)});
}
void InnerProductLayer::Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) {
  // y[M x N] = x[M x K] * W[N x K]^T (+ bias)   (inner_product_layer.cpp: caffe_gpu_gemm(NoTrans, Trans, M, N, K))
  const float* w = blobs_[0]->gpu_data();
  if ((reinterpret_cast<uintptr_t>(w) & 15u) && K_ >= 64 && K_ % 4 == 0) {     // arena slot on an 8-byte boundary: aligned copy for the TMA-fed GEMM
    if (w_aligned_.count() != blobs_[0]->count()) w_aligned_.Reshape(blobs_[0]->shape());
    CUDA_CHECK(cudaMemcpyAsync(w_aligned_.mutable_gpu_data(), w, sizeof(float) * blobs_[0]->count(), cudaMemcpyDeviceToDevice, S()));
    w = w_aligned_.gpu_data();
  }
  B2C_CHECK(b2c_sgemm_ex(0, 1, M_, num_output_, K_, 1.f, b[0]->gpu_data(), w, 0.f, t[0]->mutable_gpu_data(),
                         gemm_ws_.count() ? gemm_ws_.mutable_gpu_data() : nullptr, sizeof(float) * gemm_ws_.count(), S()));
  if (bias_) B2C_CHECK(b2c_bias_forward(M_, num_output_, 1, blobs_[1]->gpu_data(), t[0]->mutable_gpu_data(), S()));
}
void InnerProductLayer::Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) {
  // dW[N x K] += dy^T[N x M] * x[M x K];  db += sum_m dy;  dx[M x K] = dy[M x N] * W[N x K]
  float* ws = bwd_ws_.count() ? bwd_ws_.mutable_gpu_data() : nullptr;
  const size_t wsb = sizeof(float) * bwd_ws_.count();
  float* dw = blobs_[0]->mutable_gpu_diff();
  if (bwd_w_tc_) {                                  // (the GEMM's output has no alignment requirement: 4-byte stores)
    B2C_CHECK(b2c_transpose(M_, num_output_, t[0]->gpu_diff(), dyt_.mutable_gpu_data(), S()));
    B2C_CHECK(b2c_transpose(M_, K_, b[0]->gpu_data(), xt_.mutable_gpu_data(), S()));
    B2C_CHECK(b2c_sgemm_ex(0, 1, num_output_, K_, M_, 1.f, dyt_.gpu_data(), xt_.gpu_data(), 1.f, dw, ws, wsb, S()));
  } else {
    B2C_CHECK(b2c_sgemm(1, 0, num_output_, K_, M_, 1.f, t[0]->gpu_diff(), b[0]->gpu_data(), 1.f, dw, S()));
  }
  if (bias_) B2C_CHECK(b2c_bias_backward(M_, num_output_, 1, t[0]->gpu_diff(), blobs_[1]->mutable_gpu_diff(), S()));
  if (pd[0]) {
    if (bwd_x_tc_) {
      B2C_CHECK(b2c_transpose(num_output_, K_, blobs_[0]->gpu_data(), wt_.mutable_gpu_data(), S()));
      B2C_CHECK(b2c_sgemm_ex(0, 1, M_, K_, num_output_, 1.f, t[0]->gpu_diff(), wt_.gpu_data(), 0.f, b[0]->mutable_gpu_diff(), ws, wsb, S()));
    } else {
      B2C_CHECK(b2c_sgemm(0, 0, M_, K_, num_output_, 1.f, t[0]->gpu_diff(), blobs_[0]->gpu_data(), 0.f, b[0]->mutable_gpu_diff(), S()));
    }
  }
}

// ================================================================================================ LRN / Dropout / Concat
void LRNLayer::Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) {
  const LRNParameter& q = layer_param_.lrn_param;
  const int N = b[0]->shape(0), C = b[0]->shape(1), Sp = (int)(b[0]->count() / ((size_t)N * C));
  B2C_CHECK(b2c_lrn_forward(N, C, Sp, q.local_size, q.alpha, q.beta, q.k, b[0]->gpu_data(), scale_.mutable_gpu_data(), t[0]->mutable_gpu_data(), S()));
}
void LRNLayer::Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) {
  if (!pd[0]) return;
  const LRNParameter& q = layer_param_.lrn_param;
  const int N = b[0]->shape(0), C = b[0]->shape(1), Sp = (int)(b[0]->count() / ((size_t)N * C));
  B2C_CHECK(b2c_lrn_backward(N, C, Sp, q.local_size, q.alpha, q.beta, b[0]->gpu_data(), t[0]->gpu_data(), scale_.gpu_data(), t[0]->gpu_diff(),
                             b[0]->mutable_gpu_diff(), S()));
}
void DropoutLayer::Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) {
  if (layer_param_.phase == TEST) {          // TEST: the identity (dropout_layer.cu); no mask is drawn and the stream offset stays
    if (t[0] != b[0])
      CUDA_CHECK(cudaMemcpyAsync(t[0]->mutable_gpu_data(), b[0]->gpu_data(), sizeof(float) * b[0]->count(), cudaMemcpyDeviceToDevice, S()));
    return;
  }
  B2C_CHECK(b2c_dropout_mask(b[0]->count(), layer_param_.dropout_param.dropout_ratio, seed_, offset_, mask_.mutable_gpu_data(), S()));
  offset_ += b[0]->count();
  B2C_CHECK(b2c_mul(b[0]->count(), b[0]->gpu_data(), mask_.gpu_data(), t[0]->mutable_gpu_data(), S()));
}
void DropoutLayer::Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) {
  if (!pd[0]) return;
  B2C_CHECK(b2c_mul(b[0]->count(), t[0]->gpu_diff(), mask_.gpu_data(), b[0]->mutable_gpu_diff(), S()));
}
void ConcatLayer::Reshape(const vector<Blob*>& b, const vector<Blob*>& t) {
  vector<int> s = b[0]->shape();
  B2_CHECK(s.size() >= 2, "Concat: need at least 2 axes");
  for (size_t i = 1; i < b.size(); ++i) {
    B2_CHECK(b[i]->shape().size() == s.size() && b[i]->shape(0) == s[0] && b[i]->count(2) == b[0]->count(2),
             "All inputs must have the same shape, except at concat_axis.");
    s[1] += b[i]->shape(1);
  }
  t[0]->Reshape(s);
}
// The copies of Concat and Slice: `whole` is the parts laid side by side along `axis`, as count(0, axis) rows of which part i
// holds a window of shape(axis) * count(axis + 1) floats.  One strided 2-D copy per part: into whole's window (gather) or out of
// it; diff selects the diffs instead of the data.  Parts with copy[i] false (when given) are skipped but keep their window.
static void axis_copy(Blob* whole, const vector<Blob*>& parts, int axis, bool gather, bool diff, const vector<bool>* copy) {
  const size_t inner = whole->count(axis + 1), rows = whole->count(0, axis), pitch = sizeof(float) * whole->shape(axis) * inner;
  size_t off = 0;
  for (size_t i = 0; i < parts.size(); ++i) {
    Blob* p = parts[i];
    const size_t w = sizeof(float) * p->shape(axis) * inner;
    if (!copy || (*copy)[i]) {
      if (gather)
        CUDA_CHECK(cudaMemcpy2DAsync((diff ? whole->mutable_gpu_diff() : whole->mutable_gpu_data()) + off * inner, pitch,
                                     diff ? p->gpu_diff() : p->gpu_data(), w, w, rows, cudaMemcpyDeviceToDevice, S()));
      else
        CUDA_CHECK(cudaMemcpy2DAsync(diff ? p->mutable_gpu_diff() : p->mutable_gpu_data(), w,
                                     (diff ? whole->gpu_diff() : whole->gpu_data()) + off * inner, pitch, w, rows, cudaMemcpyDeviceToDevice, S()));
    }
    off += p->shape(axis);
  }
}
void ConcatLayer::Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) { axis_copy(t[0], b, 1, true, false, nullptr); }
void ConcatLayer::Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) { axis_copy(t[0], b, 1, false, true, &pd); }
void SliceLayer::Reshape(const vector<Blob*>& b, const vector<Blob*>& t) {
  size_t count = 0;
  for (size_t i = 0; i < t.size(); ++i) {
    B2_CHECK(t[i] != b[0], "Slice Layer does not allow in-place computation.");
    t[i]->Reshape(shapes_[i]);
    count += t[i]->count();
  }
  B2_CHECK(count == b[0]->count(), "Slice: the tops do not cover the bottom");   // slice_layer.cpp:65
}
void SliceLayer::Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) { axis_copy(b[0], t, layer_param_.slice_param.axis, false, false, nullptr); }
void SliceLayer::Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) {
  if (!pd[0]) return;
  axis_copy(b[0], t, layer_param_.slice_param.axis, true, true, nullptr);
}

// ================================================================================================ SoftmaxWithLoss
static void softmax_view(Blob* b, int axis, int* outer, int* C, int* inner) {
  *outer = (int)b->count(0, axis); *C = b->shape(axis); *inner = (int)b->count(axis + 1);
}
void SoftmaxWithLossLayer::Reshape(const vector<Blob*>& b, const vector<Blob*>& t) {
  const LossParameter& q = layer_param_.loss_param;
  softmax_view(b[0], layer_param_.softmax_param.axis, &outer_, &C_, &inner_);
  B2_CHECK((size_t)outer_ * inner_ == b[1]->count(), "Number of labels must match number of predictions; e.g., if softmax axis == 1 and "
           "prediction shape is (N, C, H, W), label count (number of labels) must be N*H*W, with integer values in {0, 1, ..., C-1}.");
  legacy_ = inner_ == 1 && !q.has_ignore_label && q.normalization != B2C_LOSS_NORM_NONE && t.size() == 1;
  prob_.ReshapeLike(*b[0]);
  t[0]->Reshape({1});
  if (t.size() > 1) t[1]->ReshapeLike(*b[0]);
  if (!legacy_) {
    size_t bytes = 0;
    B2C_CHECK(b2c_softmax_loss_workspace(outer_, C_, inner_, &bytes));
    workspace_.Reshape({(int)(bytes / sizeof(float))});
    normalizer_.Reshape({1});
  }
}
void SoftmaxWithLossLayer::Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) {
  const LossParameter& q = layer_param_.loss_param;
  if (legacy_)
    B2C_CHECK(b2c_softmax_loss_forward(outer_, C_, b[0]->gpu_data(), b[1]->gpu_data(), prob_.mutable_gpu_data(), t[0]->mutable_gpu_data(), S()));
  else
    B2C_CHECK(b2c_softmax_loss_forward_ex(outer_, C_, inner_, b[0]->gpu_data(), b[1]->gpu_data(), q.has_ignore_label ? 1 : 0, q.ignore_label,
                                          q.normalization, prob_.mutable_gpu_data(), t[0]->mutable_gpu_data(), normalizer_.mutable_gpu_data(),
                                          workspace_.mutable_gpu_data(), S()));
  if (t.size() > 1) t[1]->ShareData(prob_);
}
void SoftmaxWithLossLayer::Backward_gpu(const vector<Blob*>&, const vector<bool>& pd, const vector<Blob*>& b) {
  if (!pd[0]) return;
  const LossParameter& q = layer_param_.loss_param;
  if (legacy_)
    B2C_CHECK(b2c_softmax_loss_backward(outer_, C_, prob_.gpu_data(), b[1]->gpu_data(), loss_weight(), b[0]->mutable_gpu_diff(), S()));
  else
    B2C_CHECK(b2c_softmax_loss_backward_ex(outer_, C_, inner_, prob_.gpu_data(), b[1]->gpu_data(), q.has_ignore_label ? 1 : 0, q.ignore_label,
                                           normalizer_.gpu_data(), loss_weight(), b[0]->mutable_gpu_diff(), S()));
}

// ================================================================================================ Softmax / Sigmoid / Flatten
void SoftmaxLayer::Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) {
  int outer, C, inner;
  softmax_view(b[0], layer_param_.softmax_param.axis, &outer, &C, &inner);
  B2C_CHECK(b2c_softmax_forward(outer, C, inner, b[0]->gpu_data(), t[0]->mutable_gpu_data(), S()));
}
void SoftmaxLayer::Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) {
  if (!pd[0]) return;
  int outer, C, inner;
  softmax_view(t[0], layer_param_.softmax_param.axis, &outer, &C, &inner);
  B2C_CHECK(b2c_softmax_backward(outer, C, inner, t[0]->gpu_data(), t[0]->gpu_diff(), b[0]->mutable_gpu_diff(), S()));
}
void CropLayer::Reshape(const vector<Blob*>& b, const vector<Blob*>& t) {
  vector<int> top;
  CropShape(b[0]->shape(), b[1]->shape(), layer_param_.crop_param, &top, &offsets_);
  t[0]->Reshape(top);
}
void CropLayer::Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) {
  B2C_CHECK(b2c_crop_forward(b[0]->num_axes(), b[0]->shape().data(), t[0]->shape().data(), offsets_.data(), b[0]->gpu_data(),
                             t[0]->mutable_gpu_data(), Caffe::thread_stream()));
}
void CropLayer::Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) {
  if (!pd[0]) return;
  B2C_CHECK(b2c_crop_backward(b[0]->num_axes(), b[0]->shape().data(), t[0]->shape().data(), offsets_.data(), t[0]->gpu_diff(),
                              b[0]->mutable_gpu_diff(), Caffe::thread_stream()));
}
void SigmoidLayer::Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) {
  B2C_CHECK(b2c_sigmoid_forward(b[0]->count(), b[0]->gpu_data(), t[0]->mutable_gpu_data(), S()));
}
void SigmoidLayer::Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) {
  if (!pd[0]) return;
  B2C_CHECK(b2c_sigmoid_backward(t[0]->count(), t[0]->gpu_data(), t[0]->gpu_diff(), b[0]->mutable_gpu_diff(), S()));
}

// ================================================================================================ NeuronLayer / PReLU
NeuronLayer::NeuronLayer(const LayerParameter& p) : LayerBase(p) {
  const string& t = p.type;
  if (t == "ELU") {
    kind_ = B2C_NEURON_ELU;
    fwd_[0] = bwd_[0] = p.elu_param.alpha;
  } else if (t == "Power") {                              // power_layer.cpp:9-16 (diff_scale = power * scale: the kernel rounds it)
    kind_ = B2C_NEURON_POWER;
    fwd_[0] = bwd_[0] = p.power_param.power; fwd_[1] = bwd_[1] = p.power_param.scale; fwd_[2] = bwd_[2] = p.power_param.shift;
  } else if (t == "AbsVal") {
    kind_ = B2C_NEURON_ABSVAL;
  } else if (t == "BNLL") {
    kind_ = B2C_NEURON_BNLL;
  } else if (t == "Exp") {                                // exp_layer.cpp:9-29
    kind_ = B2C_NEURON_EXP;
    const ExpParameter& q = p.exp_param;
    B2_CHECK(q.base == -1.f || q.base > 0.f, "base must be strictly positive.");
    const float log_base = q.base == -1.f ? 1.f : std::log(q.base);
    B2_CHECK(!std::isnan(log_base) && !std::isinf(log_base), "NaN / Inf result: log(base)");
    const float inner = log_base * q.scale;
    const float outer = q.shift == 0.f ? 1.f : (q.base != -1.f ? std::pow(q.base, q.shift) : std::exp(q.shift));
    fwd_[0] = bwd_[0] = inner;
    fwd_[1] = outer;
  } else if (t == "Log") {                                // log_layer.cpp:9-35
    kind_ = B2C_NEURON_LOG;
    const LogParameter& q = p.log_param;
    B2_CHECK(q.base == -1.f || q.base > 0.f, "base must be strictly positive.");
    const float log_base = q.base == -1.f ? 1.f : std::log(q.base);
    B2_CHECK(!std::isnan(log_base) && !std::isinf(log_base), "NaN / Inf result: log(base)");
    const float base_scale = 1.f / log_base;
    B2_CHECK(!std::isnan(base_scale) && !std::isinf(base_scale), "NaN / Inf result: 1/log(base)");
    fwd_[0] = bwd_[0] = q.scale; fwd_[1] = bwd_[1] = q.shift;
    fwd_[2] = base_scale;
    bwd_[2] = q.scale / log_base;                         // backward_num_scale
  } else if (t == "Threshold") {
    kind_ = B2C_NEURON_THRESHOLD;
    fwd_[0] = p.threshold_param.threshold;
  } else {
    B2_CHECK(false, "NeuronLayer: unknown type " + t);
  }
}
void NeuronLayer::LayerSetUp(const vector<Blob*>& b, const vector<Blob*>& t) {
  if (kind_ == B2C_NEURON_ABSVAL) B2_CHECK(t[0] != b[0], "AbsVal Layer does not allow in-place computation.");   // absval_layer.cpp:10-11
}
bool NeuronLayer::backward_reads_bottom() const {
  switch (kind_) {
    case B2C_NEURON_ABSVAL: case B2C_NEURON_BNLL: case B2C_NEURON_LOG: return true;
    case B2C_NEURON_POWER: {
      const float power = bwd_[0], diff_scale = bwd_[0] * bwd_[1];
      return !(diff_scale == 0.f || power == 1.f);       // the constant branch reads neither x nor y
    }
    default: return false;                                // ELU: in place the top stands in for x (same sign for alpha >= 0); Exp reads y
  }
}
void NeuronLayer::Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) {
  B2C_CHECK(b2c_neuron_forward(kind_, b[0]->count(), b[0]->gpu_data(), t[0]->mutable_gpu_data(), fwd_[0], fwd_[1], fwd_[2], S()));
}
void NeuronLayer::Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) {
  if (!pd[0]) return;
  B2_CHECK(kind_ != B2C_NEURON_THRESHOLD, "Threshold Layer has no backward.");
  B2C_CHECK(b2c_neuron_backward(kind_, b[0]->count(), b[0]->gpu_data(), t[0]->gpu_data(), t[0]->gpu_diff(), b[0]->mutable_gpu_diff(), bwd_[0],
                                bwd_[1], bwd_[2], S()));
}
void PReLULayer::view(const Blob* b, int* N, int* C, int* dim) const {
  *N = b->shape(0); *C = b->shape(1); *dim = (int)b->count(2);
}
void PReLULayer::LayerSetUp(const vector<Blob*>& b, const vector<Blob*>&) {
  B2_CHECK(b[0]->num_axes() >= 2, "Number of axes of bottom blob must be >=2.");   // prelu_layer.cpp:12-38
  const PReLUParameter& q = layer_param_.prelu_param;
  blobs_.resize(1);
  blobs_[0].reset(new Blob(q.channel_shared ? vector<int>{} : vector<int>{b[0]->shape(1)}));
  Fill(q.filler, blobs_[0].get());
  param_propagate_down_.assign(1, true);
}
void PReLULayer::Reshape(const vector<Blob*>& b, const vector<Blob*>& t) {
  B2_CHECK(b[0]->num_axes() >= 2, "Number of axes of bottom blob must be >=2.");
  if (t[0] != b[0]) t[0]->ReshapeLike(*b[0]);
  if (keep_bottom_) x_keep_.ReshapeLike(*b[0]);
  int N, C, dim;
  view(b[0], &N, &C, &dim);
  size_t bytes = 0;
  B2C_CHECK(b2c_prelu_workspace_bytes(N, C, dim, layer_param_.prelu_param.channel_shared ? 1 : 0, &bytes));
  if (bytes != workspace_bytes_) {            // b2c_prelu_backward wants its counters zero once; every call leaves them so
    workspace_bytes_ = bytes;
    workspace_.Reshape({(int)((bytes + sizeof(float) - 1) / sizeof(float))});
    if (bytes) CUDA_CHECK(cudaMemsetAsync(workspace_.mutable_gpu_data(), 0, bytes, S()));
  }
}
void PReLULayer::Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) {
  int N, C, dim;
  view(b[0], &N, &C, &dim);
  B2C_CHECK(b2c_prelu_forward(N, C, dim, layer_param_.prelu_param.channel_shared ? 1 : 0, b[0]->gpu_data(), blobs_[0]->gpu_data(),
                              t[0]->mutable_gpu_data(), keep_bottom_ ? x_keep_.mutable_gpu_data() : nullptr, S()));
}
void PReLULayer::Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) {
  const bool dslope = param_propagate_down_[0];
  if (!pd[0] && !dslope) return;
  int N, C, dim;
  view(b[0], &N, &C, &dim);
  // in place: the backward reads the x the forward kept; dx is written over dy element by element (top diff == bottom diff)
  const float* x = keep_bottom_ ? x_keep_.gpu_data() : b[0]->gpu_data();
  B2C_CHECK(b2c_prelu_backward(N, C, dim, layer_param_.prelu_param.channel_shared ? 1 : 0, x, t[0]->gpu_diff(), blobs_[0]->gpu_data(),
                               pd[0] ? b[0]->mutable_gpu_diff() : nullptr, dslope ? blobs_[0]->mutable_gpu_diff() : nullptr,
                               workspace_.count() ? workspace_.mutable_gpu_data() : nullptr, sizeof(float) * workspace_.count(), S()));
}

void FlattenLayer::Reshape(const vector<Blob*>& b, const vector<Blob*>& t) {
  B2_CHECK(t[0] != b[0], "Flatten Layer does not allow in-place computation.");
  t[0]->Reshape(shape_);
  B2_CHECK(t[0]->count() == b[0]->count(), "Flatten: top and bottom counts differ");
}
void FlattenLayer::Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) { t[0]->ShareData(*b[0]); }
void FlattenLayer::Backward_gpu(const vector<Blob*>& t, const vector<bool>& pd, const vector<Blob*>& b) {
  if (!pd[0]) return;
  CUDA_CHECK(cudaMemcpyAsync(b[0]->mutable_gpu_diff(), t[0]->gpu_diff(), sizeof(float) * t[0]->count(), cudaMemcpyDeviceToDevice, S()));
}

// ================================================================================================ EuclideanLoss / L1Loss / SigmoidCrossEntropyLoss
void EuclideanLossLayer::Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) {
  B2C_CHECK(b2c_euclidean_loss_forward(b[0]->shape(0), b[0]->count(), b[0]->gpu_data(), b[1]->gpu_data(), diff_.mutable_gpu_data(),
                                       t[0]->mutable_gpu_data(), S()));
}
void EuclideanLossLayer::Backward_gpu(const vector<Blob*>&, const vector<bool>& pd, const vector<Blob*>& b) {
  for (int i = 0; i < 2; ++i) {                    // euclidean_loss_layer.cu:24-35: alpha = sign * loss_weight / num
    if (!pd[i]) continue;
    const float alpha = (i == 0 ? 1.f : -1.f) * loss_weight() / (float)b[i]->shape(0);
    B2C_CHECK(b2c_euclidean_loss_backward(b[i]->count(), diff_.gpu_data(), alpha, b[i]->mutable_gpu_diff(), S()));
  }
}
void L1LossLayer::Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) {
  B2C_CHECK(b2c_l1_loss_forward(b[0]->shape(0), b[0]->count(), b[0]->gpu_data(), b[1]->gpu_data(), diff_.mutable_gpu_data(),
                                t[0]->mutable_gpu_data(), S()));
}
void L1LossLayer::Backward_gpu(const vector<Blob*>&, const vector<bool>& pd, const vector<Blob*>& b) {
  for (int i = 0; i < 2; ++i) {                    // l1_loss_layer.cu:31-41: alpha = sign * loss_weight / num, times sign(diff)
    if (!pd[i]) continue;
    const float alpha = (i == 0 ? 1.f : -1.f) * loss_weight() / (float)b[i]->shape(0);
    B2C_CHECK(b2c_l1_loss_backward(b[i]->count(), diff_.gpu_data(), alpha, b[i]->mutable_gpu_diff(), S()));
  }
}
void SigmoidCrossEntropyLossLayer::Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) {
  B2C_CHECK(b2c_sigmoid_ce_loss_forward(b[0]->shape(0), b[0]->count(), b[0]->gpu_data(), b[1]->gpu_data(), t[0]->mutable_gpu_data(), S()));
}
void SigmoidCrossEntropyLossLayer::Backward_gpu(const vector<Blob*>&, const vector<bool>& pd, const vector<Blob*>& b) {
  B2_CHECK(!pd[1], "SigmoidCrossEntropyLoss Layer cannot backpropagate to label inputs.");
  if (!pd[0]) return;
  const float scale = loss_weight() / (float)b[0]->shape(0);     // caffe_scal(count, loss_weight / num, bottom_diff)
  B2C_CHECK(b2c_sigmoid_ce_loss_backward(b[0]->count(), b[0]->gpu_data(), b[1]->gpu_data(), scale, b[0]->mutable_gpu_diff(), S()));
}

// ================================================================================================ ContrastiveLoss
void ContrastiveLossLayer::Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) {
  const ContrastiveLossParameter& q = layer_param_.contrastive_loss_param;
  B2C_CHECK(b2c_contrastive_loss_forward(b[0]->shape(0), (int)b[0]->count(1), b[0]->gpu_data(), b[1]->gpu_data(), b[2]->gpu_data(), q.margin,
                                         q.legacy_version ? 1 : 0, diff_.mutable_gpu_data(), dist_sq_.mutable_gpu_data(), t[0]->mutable_gpu_data(), S()));
}
void ContrastiveLossLayer::Backward_gpu(const vector<Blob*>&, const vector<bool>& pd, const vector<Blob*>& b) {
  if (!pd[0] && !pd[1]) return;
  // contrastive_loss_layer.cpp Backward_cpu: alpha = +-loss_weight / num; bottom 1's gradient is bottom 0's negated
  const ContrastiveLossParameter& q = layer_param_.contrastive_loss_param;
  const int N = b[0]->shape(0), C = (int)b[0]->count(1);
  const float alpha = loss_weight() / (float)N;
  if (pd[0])
    B2C_CHECK(b2c_contrastive_loss_backward(N, C, diff_.gpu_data(), dist_sq_.gpu_data(), b[2]->gpu_data(), q.margin, q.legacy_version ? 1 : 0, alpha,
                                            b[0]->mutable_gpu_diff(), pd[1] ? b[1]->mutable_gpu_diff() : nullptr, S()));
  else
    B2C_CHECK(b2c_contrastive_loss_backward(N, C, diff_.gpu_data(), dist_sq_.gpu_data(), b[2]->gpu_data(), q.margin, q.legacy_version ? 1 : 0, -alpha,
                                            b[1]->mutable_gpu_diff(), nullptr, S()));
}

// ================================================================================================ Accuracy
void AccuracyLayer::Reshape(const vector<Blob*>& b, const vector<Blob*>& t) {
  const AccuracyParameter& q = layer_param_.accuracy_param;
  B2_CHECK(q.top_k <= (int)(b[0]->count() / b[1]->count()), "top_k must be less than or equal to the number of classes.");
  softmax_view(b[0], q.axis, &outer_, &C_, &inner_);
  B2_CHECK((size_t)outer_ * inner_ == b[1]->count(), "Number of labels must match number of predictions; e.g., if label axis == 1 and "
           "prediction shape is (N, C, H, W), label count (number of labels) must be N*H*W, with integer values in {0, 1, ..., C-1}.");
  legacy_ = inner_ == 1 && !q.has_ignore_label && t.size() == 1;
  t[0]->Reshape({1});
  if (t.size() > 1) t[1]->Reshape({C_});
  hits_.Reshape({legacy_ ? 1 : 2 + (t.size() > 1 ? 2 * C_ : 0)});        // b2c_accuracy_ex's scratch: 8 + 8 * C bytes with the per-class top
}
void AccuracyLayer::Forward_gpu(const vector<Blob*>& b, const vector<Blob*>& t) {
  const AccuracyParameter& q = layer_param_.accuracy_param;
  if (legacy_)
    B2C_CHECK(b2c_accuracy(outer_, C_, q.top_k, b[0]->gpu_data(), b[1]->gpu_data(), t[0]->mutable_gpu_data(), hits_.mutable_gpu_data(), S()));
  else
    B2C_CHECK(b2c_accuracy_ex(outer_, C_, inner_, q.top_k, b[0]->gpu_data(), b[1]->gpu_data(), q.has_ignore_label ? 1 : 0, q.ignore_label,
                              t[0]->mutable_gpu_data(), t.size() > 1 ? t[1]->mutable_gpu_data() : nullptr, hits_.mutable_gpu_data(), S()));
}

// ================================================================================================ synthetic data
SyntheticDataLayer::~SyntheticDataLayer() {
  if (host_) cudaFreeHost(host_);
  if (copy_stream_) cudaStreamSynchronize(copy_stream_);
  if (host_u8_) cudaFreeHost(host_u8_);
  for (Slot& sl : slot_) {
    if (sl.host_off) cudaFreeHost(sl.host_off);
    if (sl.dev_u8) cudaFree(sl.dev_u8);
    if (sl.dev_off) cudaFree(sl.dev_off);
    if (sl.copied) cudaEventDestroy(sl.copied);
    if (sl.consumed) cudaEventDestroy(sl.consumed);
  }
  if (copy_stream_) cudaStreamDestroy(copy_stream_);
  if (dev_mean_) cudaFree(dev_mean_);
}
static inline uint64_t splitmix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
void SyntheticDataLayer::LayerSetUp(const vector<Blob*>&, const vector<Blob*>& t) {
  std::mt19937 rng((uint32_t)seed_);
  for (size_t i = 0; i < t.size(); ++i) t[i]->Reshape(shapes_[i]);
  n0_ = t[0]->count();
  if (t.size() > 1) {
    std::uniform_int_distribution<int> u(0, classes_ - 1);
    float* l = t[1]->mutable_cpu_data();
    for (size_t i = 0; i < t[1]->count(); ++i) l[i] = (float)u(rng);
  }
  const TransformationParameter& tf = layer_param_.transform_param;
  datum_mode_ = tf.crop_size > 0 && shapes_[0].size() == 4 && shapes_[0][2] == tf.crop_size && shapes_[0][3] == tf.crop_size;
  if (datum_mode_) {
    const int N = shapes_[0][0], C = shapes_[0][1];
    hd_ = wd_ = tf.crop_size + 32;
    u8_bytes_ = (size_t)N * C * hd_ * wd_;
    CUDA_CHECK(cudaMallocHost(reinterpret_cast<void**>(&host_u8_), u8_bytes_));
    CUDA_CHECK(cudaStreamCreateWithFlags(&copy_stream_, cudaStreamNonBlocking));
    for (Slot& sl : slot_) {
      CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&sl.dev_u8), u8_bytes_));
      CUDA_CHECK(cudaMallocHost(reinterpret_cast<void**>(&sl.host_off), sizeof(int) * 3 * N));
      CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&sl.dev_off), sizeof(int) * 3 * N));
      CUDA_CHECK(cudaEventCreateWithFlags(&sl.copied, cudaEventDisableTiming));
      CUDA_CHECK(cudaEventCreateWithFlags(&sl.consumed, cudaEventDisableTiming));
    }
    for (size_t i = 0; i < u8_bytes_; i += 8) {          // uniform bytes, 8 per draw
      uint64_t r = splitmix64(seed_ * 0x100000001B3ull + i);
      for (size_t k = 0; k < 8 && i + k < u8_bytes_; ++k, r >>= 8) host_u8_[i + k] = (unsigned char)(r & 0xff);
    }
    if (!tf.mean_value.empty()) {
      B2_CHECK(tf.mean_value.size() == 1 || (int)tf.mean_value.size() == C, "Specify either 1 mean_value or as many as channels");
      vector<float> mv(C, tf.mean_value[0]);
      if ((int)tf.mean_value.size() == C) mv = tf.mean_value;
      CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&dev_mean_), sizeof(float) * C));
      CUDA_CHECK(cudaMemcpy(dev_mean_, mv.data(), sizeof(float) * C, cudaMemcpyHostToDevice));
    }
    for (Blob* b : t) b->gpu_data();
    LoadBatch(t[0], Caffe::thread_stream());              // the resident batch of the non-e2e steps
    CUDA_CHECK(cudaStreamSynchronize(Caffe::thread_stream()));
    return;
  }
  CUDA_CHECK(cudaMallocHost(reinterpret_cast<void**>(&host_), sizeof(float) * n0_));
  std::normal_distribution<float> g(0.f, 1.f);
  for (size_t i = 0; i < n0_; ++i) host_[i] = g(rng);
  memcpy(t[0]->mutable_cpu_data(), host_, sizeof(float) * n0_);
  for (Blob* b : t) b->gpu_data();   // upload once; the blobs stay resident
}
void SyntheticDataLayer::LoadBatch(Blob* top, cudaStream_t st) {
  if (!datum_mode_) {
    CUDA_CHECK(cudaMemcpyAsync(top->mutable_gpu_data(), host_, sizeof(float) * n0_, cudaMemcpyHostToDevice, st));
    return;
  }
  const int N = shapes_[0][0], C = shapes_[0][1], crop = layer_param_.transform_param.crop_size;
  Slot& sl = slot_[cur_];
  if (!sl.in_flight) IssueCopy(cur_);                    // first batch, or nothing was prefetched
  CUDA_CHECK(cudaStreamWaitEvent(st, sl.copied, 0));
  B2C_CHECK(b2c_transform_u8(sl.dev_u8, N, C, hd_, wd_, crop, crop, sl.dev_off, sl.dev_off + N,
                             reinterpret_cast<const unsigned char*>(sl.dev_off + 2 * N), dev_mean_, nullptr, layer_param_.transform_param.scale, top->mutable_gpu_data(), st));
  CUDA_CHECK(cudaEventRecord(sl.consumed, st));
  sl.in_flight = false; sl.used = true;
  cur_ ^= 1;
  IssueCopy(cur_);                                       // the next batch travels while this one is being computed on
}
void SyntheticDataLayer::IssueCopy(int s) {
  const int N = shapes_[0][0];
  const int crop = layer_param_.transform_param.crop_size;
  Slot& sl = slot_[s];
  if (sl.used) {
    CUDA_CHECK(cudaEventSynchronize(sl.copied));         // the previous copy out of this slot's pinned offsets finished long ago
    CUDA_CHECK(cudaStreamWaitEvent(copy_stream_, sl.consumed, 0));   // ... and the transform that read the slot has to be done before it is overwritten
  }
  // DataTransformer's draws (data_transformer.cpp:129-135,187,224-225): mirror = rand0 % 2, offsets = rand % (extent - crop + 1)
  unsigned char* mir = reinterpret_cast<unsigned char*>(sl.host_off + 2 * N);
  for (int i = 0; i < N; ++i) {
    const uint64_t base = (draws_ * (uint64_t)N + (uint64_t)i) * 3;
    const unsigned r0 = (unsigned)(splitmix64(seed_ + base) >> 33) + 1, r1 = (unsigned)(splitmix64(seed_ + base + 1) >> 33) + 1,
                   r2 = (unsigned)(splitmix64(seed_ + base + 2) >> 33) + 1;
    mir[i] = (layer_param_.transform_param.mirror && (r0 % 2)) ? 1 : 0;
    sl.host_off[i] = layer_param_.phase != TEST ? (int)(r1 % (unsigned)(hd_ - crop + 1)) : (hd_ - crop) / 2;
    sl.host_off[N + i] = layer_param_.phase != TEST ? (int)(r2 % (unsigned)(wd_ - crop + 1)) : (wd_ - crop) / 2;
  }
  ++draws_;
  CUDA_CHECK(cudaMemcpyAsync(sl.dev_u8, host_u8_, u8_bytes_, cudaMemcpyHostToDevice, copy_stream_));
  CUDA_CHECK(cudaMemcpyAsync(sl.dev_off, sl.host_off, sizeof(int) * 3 * N, cudaMemcpyHostToDevice, copy_stream_));
  CUDA_CHECK(cudaEventRecord(sl.copied, copy_stream_));
  sl.in_flight = true;
}

// ================================================================================================ TrainNet
// Every layer type TrainNet builds except the data layers, from its LayerParameter.  top_shapes: the tops Net inferred
// (Flatten and Slice take them); dropout_seed keys that layer's mask stream.
static shared_ptr<LayerBase> CreateLayer(const LayerParameter& p, const vector<vector<int>>& top_shapes, uint64_t dropout_seed) {
  const string& t = p.type;
  if (t == "Convolution") return LayerRegistry::CreateLayer(p);
  if (t == "ReLU") return std::make_shared<ReLULayer>(p);
  if (t == "BatchNorm") return std::make_shared<BatchNormLayer>(p);
  if (t == "Pooling") return std::make_shared<PoolingLayer>(p);
  if (t == "Eltwise") return std::make_shared<EltwiseLayer>(p);
  if (t == "InnerProduct") return std::make_shared<InnerProductLayer>(p);
  if (t == "SoftmaxWithLoss") return std::make_shared<SoftmaxWithLossLayer>(p);
  if (t == "Accuracy") return std::make_shared<AccuracyLayer>(p);
  if (t == "Softmax") return std::make_shared<SoftmaxLayer>(p);
  if (t == "Sigmoid") return std::make_shared<SigmoidLayer>(p);
  if (t == "Flatten") return std::make_shared<FlattenLayer>(p, top_shapes[0]);
  if (t == "EuclideanLoss") return std::make_shared<EuclideanLossLayer>(p);
  if (t == "L1Loss") return std::make_shared<L1LossLayer>(p);
  if (t == "SigmoidCrossEntropyLoss") return std::make_shared<SigmoidCrossEntropyLossLayer>(p);
  if (t == "LRN") return std::make_shared<LRNLayer>(p);
  if (t == "Dropout") return std::make_shared<DropoutLayer>(p, dropout_seed);
  if (t == "Concat") return std::make_shared<ConcatLayer>(p);
  if (t == "Slice") return std::make_shared<SliceLayer>(p, top_shapes);
  if (t == "ContrastiveLoss") return std::make_shared<ContrastiveLossLayer>(p);
  if (t == "Deconvolution") return LayerRegistry::CreateLayer(p);
  if (t == "Crop") return std::make_shared<CropLayer>(p);
  if (t == "PReLU") return std::make_shared<PReLULayer>(p);
  if (t == "ELU" || t == "Power" || t == "AbsVal" || t == "BNLL" || t == "Exp" || t == "Log" || t == "Threshold") return std::make_shared<NeuronLayer>(p);
  B2_CHECK(false, "TrainNet: layer type '" + t + "' is not built yet (SURVEY 8f rank 2 covers the ResNet-50 set)");
  return nullptr;
}

TrainNet::TrainNet(const Net& net, const SolverParameter& sp, int num_classes, uint64_t seed, int math) {
  name_ = net.name();
  test_ = net.phase() == TEST;
  Caffe::set_random_seed(seed);
  const vector<ParamSpec> specs = BuildNodes(net, num_classes, seed, math);
  // B2C_FUSE=0 disables every graph fusion; each pass below has its own switch as well
  const bool fuse = env_on("B2C_FUSE", true);
  // conv layers adding their bottom gradient straight into a fan-out blob's diff (TMA reduce-add store): measured SLOWER than
  // the shadow blob + add pass on ResNet-50 (dgrad 3.04 -> 3.82 ms/step against 0.50 ms of adds saved; the L2 reduction
  // units retire the 16 large accumulating stores at about half the plain-store rate), so it is opt-in: B2C_FUSE_FANOUT=1
  fuse_fanout_ = fuse && env_on("B2C_FUSE_FANOUT", false);
  if (fuse) FuseReLU();
  PlanFanOutDiffs();
  const bool fuse_res = fuse && env_on("B2C_FUSE_RES", true);
  if (fuse_res) FuseResidualTails(env_on("B2C_FUSE_SPLIT", true));
  if (!net.loss_blob().empty()) loss_blob_ = blobs_[net.loss_blob()].get();
  if (!test_) {
    solver_.reset(new SGDSolver(sp));
    solver_->SetParams(learnable_, specs);
  }
  // Net::ShareWeights (net.cpp:1270-1287), after the arena re-homed the owners: every sharer blob aliases its owner's data and diff.
  // The sharer's filler ran in SetUp; the owner's values win, with no copy either way
  for (const Share& sh : shares_) AliasShare(sh);
  for (auto& l : layers_)
    if (auto* c = dynamic_cast<ConvolutionLayer*>(l.get()))
      if (c->EnableFilterCache()) cached_convs_.push_back(c);
  if (!test_) sched_.reset(new ReduceScheduler(solver_.get(), nullptr));
  CollectOutputs(net);
  CUDA_CHECK(cudaStreamSynchronize(S()));
}
vector<ParamSpec> TrainNet::BuildNodes(const Net& net, int num_classes, uint64_t seed, int math) {
  vector<ParamSpec> specs;
  // Data layers that each read an LMDB (DetectNet's images and labels): batch n of every one must hold the same record positions.
  // DataReader's partition gives that when they share the batch size and, with several solvers, the parser thread count, so they
  // all run the largest count any of them asks for or resolves to.  A net reads either its databases or one synthetic source: a
  // synthetic layer next to a database one (an Input, or a Data layer whose source does not open) would never be reloaded, and the
  // net would train on its placeholder values without a word
  int db_layers = 0, db_parsers = 0, db_batch = 0;
  string synthetic;
  for (const NetLayer& L : net.layers()) {
    const string& t = L.param.type;
    if (!(t == "Data" && L.use_database)) {
      if (synthetic.empty() && (t == "Data" || t == "Input" || t == "DummyData" || t == "ImageData")) synthetic = L.param.name;
      continue;
    }
    B2_CHECK(db_layers == 0 || L.param.data_param.batch_size == db_batch,
             "TrainNet: Data layers that read databases must have one batch_size, so that their batches hold the same records");
    db_batch = L.param.data_param.batch_size;
    db_parsers = std::max(db_parsers, DataLayer::ParserThreads(L));
    ++db_layers;
  }
  B2_CHECK(db_layers == 0 || synthetic.empty(),
           "TrainNet: layer '" + synthetic + "' feeds synthetic data next to Data layers that read databases (an Input / DummyData layer, "
           "or a Data layer whose source does not open): one data source per net");
  int db_index = 0;
  for (size_t li = 0; li < net.layers().size(); ++li) {
    const NetLayer& L = net.layers()[li];
    const string& type = L.param.type;
    Node node;
    for (auto& bn : L.param.bottom) {
      auto it = blobs_.find(bn);
      B2_CHECK(it != blobs_.end(), "Unknown bottom blob '" + bn + "'");
      node.bottom.push_back(it->second.get());
    }
    for (auto& tn : L.param.top) {
      auto& sp_ = blobs_[tn];
      if (!sp_) sp_.reset(new Blob());
      node.top.push_back(sp_.get());
    }
    vector<vector<int>> shapes;
    for (size_t t = 0; t < L.param.top.size(); ++t) shapes.push_back(net.top_shape((int)li, (int)t));
    shared_ptr<LayerBase> layer;
    if (type == "Data" && L.use_database) {
      // data_param.source opened: the layer reads it (parser threads -> pinned batch -> device transform), data_layer.hpp
      // Several such layers (DetectNet's images and labels) each read their own LMDB; every one loads a batch per step, so with equal
      // batch sizes batch i of each holds the same record positions
      // each layer its own crop / mirror stream (the first keeps `seed`), as the reference's layers each draw Caffe::next_seed()
      auto* d = new DataLayer(L, seed + 0x9E3779B97F4A7C15ull * (uint64_t)db_index++, db_layers > 1 ? db_parsers : 0);
      layer.reset(d);
      db_data_.push_back({d, (int)layers_.size()});
    } else if (type == "Data" || type == "Input" || type == "DummyData" || type == "ImageData") {
      auto* d = new SyntheticDataLayer(L.param, shapes, num_classes, seed);
      layer.reset(d);
      data_ = d;
    } else {
      LayerParameter lp = L.param;
      lp.convolution_param.math = math;
      layer = CreateLayer(lp, shapes, seed * 0x100000001B3ull + li);
    }
    layer->SetUp(node.bottom, node.top);
    // learnable blobs in layer order: Net::AppendParam (net.cpp:573-606) appends EVERY blob of every layer, so param ids,
    // reduce-bucket boundaries and the SolverState history list (5 blobs per BatchNorm layer) match the reference.
    // Blobs the layer never differentiates (BatchNorm mean / variance / correction, batch_norm_layer.cpp: lr_mult forced
    // to 0) are marked `statistic`; trainable_ids_ lists the rest for the trainer API.
    // A blob that shares a named parameter (Net::AppendParam, net.cpp:611-666; Net checked shapes and multipliers) is not appended:
    // it maps to its owner's id, keeps its own Blob object, and aliases the owner's storage once the arena exists (ShareNamedParams).
    for (size_t bi = 0; bi < layer->blobs().size(); ++bi) {
      const ParamSpec& own = bi < L.param.param.size() ? L.param.param[bi] : ParamSpec();
      const std::pair<int, int> owner = net.param_owner((int)li, (int)bi);
      if (owner.first >= 0) {
        const Node& on = nodes_[owner.first];
        const int id = on.param_ids[owner.second];
        node.param_ids.push_back(id);
        node.param_owned.push_back(false);
        shares_.push_back({(int)li, (int)bi, owner.first, owner.second});
        if (own.has_lr_mult && !specs[id].statistic) specs[id].lr_mult = own.lr_mult;   // the owner left it unset (else Net found them equal)
        if (own.has_decay_mult && !specs[id].statistic) specs[id].decay_mult = own.decay_mult;
        continue;
      }
      ParamSpec ps = own;
      if (!layer->param_propagate_down((int)bi)) { ps.lr_mult = 0.f; ps.decay_mult = 0.f; ps.statistic = true; }
      else trainable_ids_.push_back((int)learnable_.size());
      if (node.first_owned < 0) node.first_owned = (int)learnable_.size();
      node.param_ids.push_back((int)learnable_.size());
      node.param_owned.push_back(true);
      learnable_.push_back(layer->blobs()[bi]);
      specs.push_back(ps);
    }
    // need-backward (net.cpp:160-330, loss pruning included) is Net's result; a TEST net runs no backward at all.  Accuracy is
    // forward-only (accuracy_layer.hpp: "cannot backpropagate"): its top carries no loss weight, so pruning already stops it
    node.need_backward = L.need_backward && !test_ && type != "Accuracy";
    for (size_t i = 0; i < node.bottom.size(); ++i) {
      node.propagate_down.push_back(node.need_backward && L.propagate_down[i]);
    }
    // the reference refuses at backward time (sigmoid_cross_entropy_loss_layer.cpp:52-55); here the graph is known up front
    // (softmax_loss_layer.cpp:128-130 likewise)
    B2_CHECK(!((type == "SigmoidCrossEntropyLoss" || type == "SoftmaxWithLoss") && node.need_backward && L.label_wants_gradient),
             type + " Layer cannot backpropagate to label inputs.");
    // the neuron layers' in-place and backward limits, known once need-backward is (the reference meets them at run time, or not at all)
    const bool in_place = !node.top.empty() && !node.bottom.empty() && node.top[0] == node.bottom[0];
    if (auto* nl = dynamic_cast<NeuronLayer*>(layer.get())) {
      B2_CHECK(!(type == "Threshold" && node.propagate_down[0]), "Threshold Layer cannot backpropagate: its bottom '" + L.param.bottom[0] +
                                                                     "' needs a gradient, and the layer has no backward.");
      B2_CHECK(!(in_place && node.propagate_down[0] && nl->backward_reads_bottom()),
               type + " Layer does not allow in-place computation when it runs backward: its backward reads the bottom the top overwrites.");
    }
    if (auto* pr = dynamic_cast<PReLULayer*>(layer.get())) pr->set_keep_bottom(in_place && node.need_backward);
    node.bottom_diff_tmp.assign(node.bottom.size(), nullptr);
    layers_.push_back(layer);
    layer_names_.push_back(L.param.name);
    layer_types_.push_back(type);
    nodes_.push_back(node);
  }
  return specs;
}
// Fusion: BatchNorm -> in-place ReLU and Eltwise(SUM, 2 bottoms) -> in-place ReLU run as one kernel each way, and BatchNorm stops
// materialising x_norm (csrc/layers_fused.cu).  The ReLU layer stays in the graph as a no-op so that layer indices, names and blobs
// are those of the prototxt.  Results are bit-identical to the unfused graph.
void TrainNet::FuseReLU() {
  for (size_t i = 0; i < layers_.size(); ++i) {
    auto* bn = dynamic_cast<BatchNormLayer*>(layers_[i].get());
    auto* el = dynamic_cast<EltwiseLayer*>(layers_[i].get());
    if (!bn && !el) continue;
    const bool out_of_place = nodes_[i].top[0] != nodes_[i].bottom[0];
    ReLULayer* relu = nullptr;
    if (i + 1 < layers_.size()) {
      relu = dynamic_cast<ReLULayer*>(layers_[i + 1].get());
      if (relu && !(nodes_[i + 1].bottom[0] == nodes_[i].top[0] && nodes_[i + 1].top[0] == nodes_[i].top[0] && relu->negative_slope() == 0.f))
        relu = nullptr;
    }
    if (bn && (out_of_place || test_)) {           // (TEST: the inference kernel also runs in place)
      bn->set_fusion(true, relu != nullptr);
      bn->Reshape(nodes_[i].bottom, nodes_[i].top);
      if (relu) relu->set_fused_away(true);
    } else if (el && relu && nodes_[i].bottom.size() == 2) {
      el->set_fuse_relu(true);
      relu->set_fused_away(true);
    }
  }
}
// diff accumulation where a blob fans out (insert_splits.cpp / SplitLayer::Backward): the consumer that runs FIRST in
// the backward pass writes the blob's diff; every other consumer writes a shadow diff that is then added in
void TrainNet::PlanFanOutDiffs() {
  std::map<Blob*, int> writers;
  for (int li = (int)nodes_.size() - 1; li >= 0; --li) {
    Node& nd = nodes_[li];
    if (!nd.need_backward) continue;
    for (size_t i = 0; i < nd.bottom.size(); ++i) {
      if (!nd.propagate_down[i]) continue;
      const bool in_place = i < nd.top.size() && nd.top[i] == nd.bottom[i];
      if (in_place) continue;
      if (writers[nd.bottom[i]]++ > 0) {
        if (fuse_fanout_ && layers_[li]->SupportsBottomDiffAccumulate((int)i)) {
          nd.accumulate_bottom.resize(nd.bottom.size(), false);       // the layer adds into the blob's diff itself
          nd.accumulate_bottom[i] = true;
        } else {
          tmp_diffs_.emplace_back(new Blob(nd.bottom[i]->shape()));
          nd.bottom_diff_tmp[i] = tmp_diffs_.back().get();
        }
      }
    }
  }
}
// Residual tails (B2C_FUSE_RES=0 disables): BatchNorm -> Eltwise(SUM, 2 bottoms) -> in-place ReLU.  The BatchNorm that runs LAST
// among the producers of the sum's bottoms takes over the sum and the ReLU in both directions (csrc/layers_fused.cu, *_res): its
// top is not materialised, four passes over a block-output-sized tensor go away per block and step.  Conditions: the
// BatchNorm's top has no other consumer, nothing between it and the sum rewrites the other operand, the sum is the first
// backward writer of both bottoms (no shadow diffs).  A TEST net has no backward: there only the first two conditions apply.
void TrainNet::FuseResidualTails(bool fuse_split) {
  for (size_t i = 0; i < layers_.size(); ++i) {
    auto* el = dynamic_cast<EltwiseLayer*>(layers_[i].get());
    Node& en = nodes_[i];
    if (!el || !el->fuse_relu() || en.bottom.size() != 2 || (!test_ && !en.need_backward)) continue;
    if (!en.accumulate_bottom.empty() || en.bottom_diff_tmp[0] || en.bottom_diff_tmp[1]) continue;
    int prod[2] = {-1, -1};
    for (int k = 0; k < 2; ++k)
      for (int j = (int)i - 1; j >= 0 && prod[k] < 0; --j)
        for (Blob* tb : nodes_[j].top) if (tb == en.bottom[k]) prod[k] = j;
    if (prod[0] < 0 || prod[1] < 0 || prod[0] == prod[1]) continue;
    const int k = prod[0] > prod[1] ? 0 : 1, j = prod[k];
    auto* bn = dynamic_cast<BatchNormLayer*>(layers_[j].get());
    if (!bn || !bn->recompute() || bn->fuse_relu() || nodes_[j].top[0] == nodes_[j].bottom[0] || (!test_ && !en.propagate_down[k])) continue;
    int consumers = 0;
    for (size_t l = 0; l < nodes_.size(); ++l)
      for (Blob* bb : nodes_[l].bottom) if (bb == en.bottom[k]) ++consumers;
    bool other_rewritten = false;
    for (size_t l = (size_t)j + 1; l < i; ++l) {       // ... nor reads it (its backward would add into a diff this layer has yet to write)
      for (Blob* tb : nodes_[l].top) if (tb == en.bottom[1 - k]) other_rewritten = true;
      if (!test_) for (Blob* bb : nodes_[l].bottom) if (bb == en.bottom[1 - k]) other_rewritten = true;
    }
    if (consumers != 1 || other_rewritten) continue;
    bn->set_residual(en.bottom[1 - k], en.top[0], en.propagate_down[1 - k]);
    el->set_fused_away(true);
  }
  // a fused tail's sum blob with a second backward writer: hand the shadow diff to the tail instead of adding it in a pass of its own
  std::map<Blob*, BatchNormLayer*> tails;
  for (size_t j = 0; j < layers_.size(); ++j)
    if (auto* bn = dynamic_cast<BatchNormLayer*>(layers_[j].get()))
      if (bn->residual_sum()) tails[bn->residual_sum()] = bn;
  std::map<Blob*, int> shadows;
  for (Node& nd : nodes_)
    for (size_t i = 0; i < nd.bottom.size(); ++i) if (nd.bottom_diff_tmp[i]) ++shadows[nd.bottom[i]];
  for (Node& nd : nodes_) {
    nd.deferred_add.assign(nd.bottom.size(), false);
    for (size_t i = 0; fuse_split && i < nd.bottom.size(); ++i) {
      if (!nd.bottom_diff_tmp[i] || shadows[nd.bottom[i]] != 1) continue;       // exactly one shadow per blob
      auto it = tails.find(nd.bottom[i]);
      if (it == tails.end()) continue;
      it->second->set_sum_diff_part2(nd.bottom_diff_tmp[i]);
      nd.deferred_add[i] = true;
    }
  }
}
// output blobs and loss weights (Net::Init, net.cpp: available_blobs; Layer::SetLossWeights, LossLayer::LayerSetUp)
void TrainNet::CollectOutputs(const Net& net) {
  std::set<string> available;
  std::map<string, float> weight;
  for (const NetLayer& L : net.layers()) {
    for (auto& bn : L.param.bottom) available.erase(bn);
    for (size_t t = 0; t < L.param.top.size(); ++t) {
      available.insert(L.param.top[t]);
      weight[L.param.top[t]] = TopLossWeight(L.param, t);
    }
  }
  for (const string& n : available) outputs_.push_back({n, blobs_[n].get(), weight[n]});
}
TrainNet::~TrainNet() {
  if (pass_scored_) cudaEventDestroy(pass_scored_);
  if (pass_reduced_) cudaEventDestroy(pass_reduced_);
}

void TrainNet::AttachSync(P2PSync* sync) {
  sync_ = sync;
  for (auto& d : db_data_) d.first->set_solver(sync->nranks(), sync->rank());     // each solver reads its own stripe of the database
  sync_->on_start(solver_->arena());
  filters_dirty_ = true;
  sched_.reset(new ReduceScheduler(solver_.get(), sync_));
}
Blob* TrainNet::blob(const string& name) {
  auto it = blobs_.find(name);
  return it == blobs_.end() ? nullptr : it->second.get();
}
size_t TrainNet::activation_floats() const {
  size_t c = 0;
  for (auto& kv : blobs_) c += kv.second->count();
  return c;
}
void TrainNet::AliasShare(const Share& sh) {
  Blob* sharer = layers_[sh.layer]->blobs()[sh.blob].get();
  Blob& owner = *layers_[sh.owner_layer]->blobs()[sh.owner_blob];
  sharer->ShareData(owner);
  sharer->ShareDiff(owner);
}
void TrainNet::PrepareFilters() {
  // one multi-tensor launch per 24 filter layouts instead of one prepass per forward and per dgrad call
  vector<const b2c_conv_desc*> descs;
  vector<const float*> ws;
  vector<void*> caches;
  for (ConvolutionLayer* c : cached_convs_) {
    if (!c->desc() || !c->filter_cache()) continue;
    descs.push_back(c->desc()); ws.push_back(c->blobs()[0]->gpu_data()); caches.push_back(c->filter_cache());
  }
  if (!descs.empty()) B2C_CHECK(b2c_conv_prepare_filters((int)descs.size(), descs.data(), ws.data(), caches.data(), S()));
  filters_dirty_ = false;
}
void TrainNet::Forward(bool copy_input) {
  if (filters_dirty_) PrepareFilters();
  if (!db_data_.empty()) {                                               // database sources: a new batch per e2e step; the first one always
    for (auto& d : db_data_)
      if (copy_input || !d.first->loaded()) d.first->LoadBatch(nodes_[d.second].top, S());
  } else if (copy_input && data_) data_->LoadBatch(nodes_[0].top[0], S());     // H2D of the batch (+ the device transform of uint8 datums)
  EventProfiler* prof = Caffe::profiler();
  for (size_t i = 0; i < layers_.size(); ++i) {
    size_t h = 0;
    if (prof) { prof->set_layer((int)i); h = prof->begin(EventProfiler::FWD, S()); }
    layers_[i]->Forward(nodes_[i].bottom, nodes_[i].top);
    if (prof) prof->end(h, S());
  }
}
void TrainNet::Backward(bool update) {
  for (int li = (int)layers_.size() - 1; li >= 0; --li) {
    Node& nd = nodes_[li];
    EventProfiler* prof = Caffe::profiler();
    size_t ph = 0;
    if (prof && nd.need_backward) { prof->set_layer(li); ph = prof->begin(EventProfiler::BWD, S()); }
    if (nd.need_backward) {
      // redirect fan-out bottoms to their shadow blobs (data shared, private diff), run, then accumulate
      vector<Blob*> bvec = nd.bottom;
      for (size_t i = 0; i < bvec.size(); ++i)
        if (nd.bottom_diff_tmp[i]) { nd.bottom_diff_tmp[i]->ShareData(*nd.bottom[i]); bvec[i] = nd.bottom_diff_tmp[i]; }
      if (!nd.accumulate_bottom.empty()) layers_[li]->set_accumulate_bottom_diff(nd.accumulate_bottom);
      layers_[li]->Backward(nd.top, nd.propagate_down, bvec);
      for (size_t i = 0; i < bvec.size(); ++i)
        if (nd.bottom_diff_tmp[i] && !(i < nd.deferred_add.size() && nd.deferred_add[i]))
          B2C_CHECK(b2c_add(nd.bottom[i]->count(), nd.bottom[i]->gpu_diff(), nd.bottom_diff_tmp[i]->gpu_diff(), nd.bottom[i]->mutable_gpu_diff(), S()));
      if (prof) prof->end(ph, S());
    }
    // net.cpp:738-746: only the owner of a parameter releases it, after its own backward.  The owner of a shared parameter is the
    // earliest layer that uses the name, so its backward runs after every sharer's has added into the shared diff; a layer that
    // owns nothing releases nothing.  Owned ids grow with the layer index, so releases still arrive in descending id order.
    if (update && nd.first_owned >= 0) sched_->on_param_ready(nd.first_owned, S());
  }
}
float TrainNet::ForwardBackward() {
  Forward(false);
  Backward(false);              // diffs stay in place for inspection; Step() is the path that reduces + updates
  return last_loss();
}
void TrainNet::ClearParamDiffs() {
  // the reference's solver relies on ApplyUpdate clearing the diffs (solver.cpp:237-239) and so does Step(); a caller that
  // ran ForwardBackward() for inspection clears them before stepping, as with Net::ClearParamDiffs
  CUDA_CHECK(cudaMemsetAsync(solver_->arena().diff(), 0, sizeof(float) * solver_->arena().total(), S()));
}
void TrainNet::Step(bool copy_input_from_host) {
  // Solver::Step (solver.cpp:277-288): iter_size micro-batches accumulate into the parameter diffs (weight / bias
  // gradients are accumulated by every layer, as in the reference); only the last one releases parameters to the
  // reduction queue (ForwardBackward(apply_update = i + 1 == iter_size)), and the update folds 1/iter_size in.
  const int iter_size = std::max(1, solver_->param().iter_size);
  for (int i = 0; i < iter_size; ++i) {
    Forward(copy_input_from_host);
    Backward(i + 1 == iter_size);
  }
  sched_->end_of_iteration(S());
  filters_dirty_ = true;          // the update changed every weight: the next Forward re-prepares (after the compute stream's wait)
}
float TrainNet::TimedSteps(int n, bool copy_input, bool read_loss) {
  cudaEvent_t a, b;
  CUDA_CHECK(cudaEventCreate(&a)); CUDA_CHECK(cudaEventCreate(&b));
  CUDA_CHECK(cudaStreamSynchronize(S()));
  CUDA_CHECK(cudaEventRecord(a, S()));
  for (int i = 0; i < n; ++i) {
    Step(copy_input);
    if (read_loss) {                               // device -> host read of the step's result, on the same stream
      CUDA_CHECK(cudaMemcpyAsync(&host_loss_, loss_blob_->gpu_data(), sizeof(float), cudaMemcpyDeviceToHost, S()));
      CUDA_CHECK(cudaStreamSynchronize(S()));
    }
  }
  CUDA_CHECK(cudaEventRecord(b, S()));
  CUDA_CHECK(cudaEventSynchronize(b));
  float ms = 0.f;
  CUDA_CHECK(cudaEventElapsedTime(&ms, a, b));
  cudaEventDestroy(a); cudaEventDestroy(b);
  return ms;
}
void TrainNet::ProfileSteps(int n, vector<int>* layer, vector<int>* op, vector<float>* ms) {
  Profile(n, [this] { Step(false); }, layer, op, ms);
}
void TrainNet::Profile(int n, const std::function<void()>& iteration, vector<int>* layer, vector<int>* op, vector<float>* ms) {
  EventProfiler prof;
  CUDA_CHECK(cudaDeviceSynchronize());
  Caffe::set_profiler(&prof);
  try { for (int i = 0; i < n; ++i) iteration(); } catch (...) { Caffe::set_profiler(nullptr); throw; }
  Caffe::set_profiler(nullptr);
  std::map<std::pair<int, int>, float> acc;
  prof.collect(&acc);
  for (auto& kv : acc) { layer->push_back(kv.first.first); op->push_back(kv.first.second); ms->push_back(kv.second / (float)n); }
}
// ---- snapshot / restore -------------------------------------------------------------------------------------------
static BlobData to_blob_data(const vector<int>& shape, const float* host, size_t count) {
  BlobData b;
  b.shape = shape;
  b.data.assign(host, host + count);
  return b;
}
string TrainNet::Snapshot(const string& prefix) {
  CUDA_CHECK(cudaDeviceSynchronize());
  NetWeights nw;
  nw.name = name_;
  for (size_t i = 0; i < layers_.size(); ++i) {
    LayerWeights lw;
    lw.name = layer_names_[i]; lw.type = layer_types_[i];
    // read the DEVICE copy explicitly: the fused SGD kernel updates the arena behind the Blob's back, so a blob whose
    // head was left SYNCED by an earlier cpu_data() would hand out stale host values (second snapshot of a process)
    for (auto& b : layers_[i]->blobs()) {
      vector<float> h(b->count());
      CUDA_CHECK(cudaMemcpy(h.data(), b->gpu_data(), sizeof(float) * h.size(), cudaMemcpyDeviceToHost));
      lw.blobs.push_back(to_blob_data(b->shape(), h.data(), h.size()));
    }
    nw.layers.push_back(std::move(lw));
  }
  const string stem = prefix + "_iter_" + std::to_string(solver_->iter());
  WriteBinaryFile(stem + ".caffemodel", SerializeNetWeights(nw));
  SolverStateData st;
  st.iter = solver_->iter(); st.current_step = solver_->current_step(); st.learned_net = stem + ".caffemodel";
  // the reference's history_ layout: [h_0 .. h_np-1], then for AdaDelta / Adam [h2_0 .. h2_np-1] (AdamPreSolve, adam_solver.cpp:8-16)
  ParamArena& ar = solver_->arena();
  for (int k = 0; k < solver_->num_histories(); ++k)
    for (size_t i = 0; i < learnable_.size(); ++i) {
      vector<float> h(learnable_[i]->count());
      CUDA_CHECK(cudaMemcpy(h.data(), (k ? ar.history2() : ar.history()) + ar.offset((int)i), sizeof(float) * h.size(), cudaMemcpyDeviceToHost));
      st.history.push_back(to_blob_data(learnable_[i]->shape(), h.data(), h.size()));
    }
  WriteBinaryFile(stem + ".solverstate", SerializeSolverState(st));
  return stem + ".solverstate";
}
int TrainNet::CopyTrainedLayersFrom(const string& path) {
  const NetWeights nw = ParseNetWeights(ReadBinaryFile(path));
  CUDA_CHECK(cudaDeviceSynchronize());
  int copied = 0;
  for (const LayerWeights& lw : nw.layers) {
    size_t li = 0;
    while (li < layer_names_.size() && layer_names_[li] != lw.name) ++li;
    if (li == layer_names_.size() || lw.blobs.empty()) continue;          // "Ignoring source layer" (net.cpp)
    auto& target = layers_[li]->blobs();
    B2_CHECK(target.size() == lw.blobs.size(), "Incompatible number of blobs for layer " + lw.name);
    for (size_t j = 0; j < target.size(); ++j) {
      B2_CHECK(target[j]->count() == lw.blobs[j].data.size(), "Cannot copy param " + std::to_string(j) + " weights from layer '" + lw.name +
                                                                  "'; shape mismatch.");
      CUDA_CHECK(cudaMemcpy(target[j]->mutable_gpu_data(), lw.blobs[j].data.data(), sizeof(float) * target[j]->count(), cudaMemcpyHostToDevice));
    }
    ++copied;
  }
  filters_dirty_ = true;
  return copied;
}
void TrainNet::Restore(const string& state_path) {
  const SolverStateData st = ParseSolverState(ReadBinaryFile(state_path));
  if (!st.learned_net.empty()) CopyTrainedLayersFrom(st.learned_net);
  const size_t np = learnable_.size();
  B2_CHECK(st.history.size() == np * solver_->num_histories(), "Incorrect length of history blobs.");      // sgd_solver.cpp:334
  ParamArena& ar = solver_->arena();
  for (size_t j = 0; j < st.history.size(); ++j) {
    const size_t i = j % np;
    B2_CHECK(st.history[j].data.size() == learnable_[i]->count(), "history blob " + std::to_string(j) + ": size mismatch");
    CUDA_CHECK(cudaMemcpy((j < np ? ar.history() : ar.history2()) + ar.offset((int)i), st.history[j].data.data(),
                          sizeof(float) * learnable_[i]->count(), cudaMemcpyHostToDevice));
  }
  solver_->set_iter(st.iter);
  solver_->set_current_step(st.current_step);
  for (auto& l : layers_)
    if (auto* bn = dynamic_cast<BatchNormLayer*>(l.get())) bn->set_iter(st.iter + 1);   // running statistics are warm
}
float TrainNet::last_loss() { return loss_blob_ ? loss_blob_->cpu_data()[0] : 0.f; }

// ---- TEST phase --------------------------------------------------------------------------------------------------------
void TrainNet::ShareTrainedLayersWith(TrainNet& train) {
  B2_CHECK(test_, "ShareTrainedLayersWith: only a TEST-phase net takes another net's parameters");
  CUDA_CHECK(cudaStreamSynchronize(S()));
  vector<bool> taken(layers_.size(), false);
  for (size_t i = 0; i < layers_.size(); ++i) {
    size_t k = 0;
    while (k < train.layer_names_.size() && train.layer_names_[k] != layer_names_[i]) ++k;
    if (k == train.layer_names_.size() || train.layers_[k]->blobs().empty()) continue;     // "Ignoring source layer" (net.cpp)
    auto& src = train.layers_[k]->blobs();
    auto& dst = layers_[i]->blobs();
    B2_CHECK(src.size() == dst.size(), "Incompatible number of blobs for layer " + layer_names_[i]);
    for (size_t j = 0; j < src.size(); ++j) {
      B2_CHECK(src[j]->shape() == dst[j]->shape(), "Cannot share param " + std::to_string(j) + " weights from layer '" + layer_names_[i] +
                                                       "'; shape mismatch.  Source param shape is " + src[j]->shape_string() +
                                                       "; target param shape is " + dst[j]->shape_string());
      dst[j] = src[j];                             // a sharer takes the trainer's sharer blob, which aliases the trainer's owner
      if (nodes_[i].param_owned[j]) learnable_[nodes_[i].param_ids[j]] = src[j];
    }
    taken[i] = true;
  }
  // a sharer in a layer the trainer does not have kept its own blob, which aliased an owner blob that may just have been replaced
  // (and freed): point it at the owner's current storage
  for (const Share& sh : shares_)
    if (!taken[sh.layer]) AliasShare(sh);
  // a multi-GPU trainer: rank r scores its stripe of the validation database (Net::Init's TEST DataReader gets (solver_count, rank))
  test_sync_ = train.sync_;
  if (test_sync_)
    for (auto& d : db_data_) d.first->set_solver(test_sync_->nranks(), test_sync_->rank());
  filters_dirty_ = true;
}
void TrainNet::ForwardTest() {
  B2_CHECK(test_, "ForwardTest: the net was built for the TRAIN phase");
  for (auto& d : db_data_) d.first->LoadBatch(nodes_[d.second].top, S());   // every TEST forward reads the next batch
  Forward(false);
}
float TrainNet::Test(int iterations, vector<float>* per_batch, vector<float>* mean) {
  B2_CHECK(iterations > 0, "Test: iterations must be positive");
  filters_dirty_ = true;          // shared weights change under this net between calls: never score on a stale filter cache
  size_t width = 0;
  for (const Output& o : outputs_) width += o.blob->count();
  per_batch->clear();
  vector<float> sum(width, 0.f);
  float loss = 0.f;
  for (int i = 0; i < iterations; ++i) {
    ForwardTest();
    float iter_loss = 0.f;
    size_t idx = 0;
    for (const Output& o : outputs_) {
      const float* v = o.blob->cpu_data();
      for (size_t k = 0; k < o.blob->count(); ++k, ++idx) {
        per_batch->push_back(v[k]);
        sum[idx] += v[k];                                   // tools/caffe.cpp:272-289: float sums, then / iterations
        iter_loss += o.loss_weight * v[k];                  // Layer::Forward's loss: loss_weight . top
      }
    }
    loss += iter_loss;
  }
  mean->resize(width);
  for (size_t k = 0; k < width; ++k) (*mean)[k] = sum[k] / iterations;
  return loss / iterations;
}
int TrainNet::TestPass(int iterations, const std::function<bool(int)>& before_batch, vector<float>* mean, float* loss) {
  const int ran = EnqueueTestPass(iterations, before_batch);
  if (ran == iterations) ReadTestPass(mean, loss);
  return ran;
}
int TrainNet::EnqueueTestPass(int iterations, const std::function<bool(int)>& before_batch) {
  B2_CHECK(test_, "TestPass: the net was built for the TRAIN phase");
  B2_CHECK(iterations > 0, "TestPass: iterations must be positive");
  B2_CHECK(pass_batches_ == 0, "TestPass: the previous pass was never read");
  // the shared weights changed since the last pass.  This stream waited for the trainer's last update at the end of its step
  // (ReduceScheduler::end_of_iteration), so the forwards below read the updated weights; the trainer's next step is enqueued
  // behind them on the same stream, so its updates cannot overtake them.
  filters_dirty_ = true;
  size_t width = 0;
  for (const Output& o : outputs_) width += o.blob->count();
  if (scores_.count() != std::max<size_t>(width, 1)) scores_.Reshape({(int)std::max<size_t>(width, 1)});
  float* score = scores_.mutable_gpu_data();
  CUDA_CHECK(cudaMemsetAsync(score, 0, sizeof(float) * scores_.count(), S()));
  for (int i = 0; i < iterations; ++i) {
    if (before_batch && !before_batch(i)) return i;
    ForwardTest();
    size_t idx = 0;
    for (const Output& o : outputs_) {                   // 0 + v, then + v per batch: Test()'s host sums (tools/caffe.cpp:272-289)
      B2C_CHECK(b2c_add(o.blob->count(), score + idx, o.blob->gpu_data(), score + idx, S()));
      idx += o.blob->count();
    }
  }
  if (test_sync_ && test_sync_->nranks() > 1 && width) {
    CUDA_CHECK(cudaEventCreateWithFlags(&pass_scored_, cudaEventDisableTiming));
    CUDA_CHECK(cudaEventCreateWithFlags(&pass_reduced_, cudaEventDisableTiming));
    CUDA_CHECK(cudaEventRecord(pass_scored_, S()));                  // the last batch's scores are in the vector ...
    CUDA_CHECK(cudaStreamWaitEvent(test_sync_->comm_stream(), pass_scored_, 0));
    test_sync_->allreduce_scores(score, width);                      // ... before it travels
    CUDA_CHECK(cudaEventRecord(pass_reduced_, test_sync_->comm_stream()));
    CUDA_CHECK(cudaStreamWaitEvent(S(), pass_reduced_, 0));
  }
  pass_batches_ = iterations;
  return iterations;
}
void TrainNet::ReadTestPass(vector<float>* mean, float* loss) {
  B2_CHECK(pass_batches_ > 0, "ReadTestPass: no whole pass was enqueued");
  const int batches = pass_batches_, nranks = test_sync_ ? test_sync_->nranks() : 1;
  pass_batches_ = 0;
  size_t width = 0;
  for (const Output& o : outputs_) width += o.blob->count();
  vector<float> sum(width);
  if (width) CUDA_CHECK(cudaMemcpyAsync(sum.data(), scores_.gpu_data(), sizeof(float) * width, cudaMemcpyDeviceToHost, S()));
  CUDA_CHECK(cudaStreamSynchronize(S()));
  if (pass_scored_) {
    cudaEventDestroy(pass_scored_); cudaEventDestroy(pass_reduced_);
    pass_scored_ = pass_reduced_ = nullptr;
  }
  // solver.cpp:527: score / test_iterations / solver_count, with the score summed over every rank (DESIGN.md section 8)
  mean->resize(width);
  float l = 0.f;
  size_t idx = 0;
  for (const Output& o : outputs_)
    for (size_t k = 0; k < o.blob->count(); ++k, ++idx) {
      (*mean)[idx] = sum[idx] / batches / nranks;
      l += o.loss_weight * sum[idx];
    }
  *loss = l / batches / nranks;
}
float TrainNet::TimedForwards(int n) {
  cudaEvent_t a, b;
  CUDA_CHECK(cudaEventCreate(&a)); CUDA_CHECK(cudaEventCreate(&b));
  CUDA_CHECK(cudaStreamSynchronize(S()));
  CUDA_CHECK(cudaEventRecord(a, S()));
  for (int i = 0; i < n; ++i) ForwardTest();
  CUDA_CHECK(cudaEventRecord(b, S()));
  CUDA_CHECK(cudaEventSynchronize(b));
  float ms = 0.f;
  CUDA_CHECK(cudaEventElapsedTime(&ms, a, b));
  cudaEventDestroy(a); cudaEventDestroy(b);
  return ms;
}
void TrainNet::ProfileForwards(int n, vector<int>* layer, vector<int>* op, vector<float>* ms) {
  Profile(n, [this] { ForwardTest(); }, layer, op, ms);
}

}  // namespace caffe
