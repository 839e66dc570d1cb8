// data_layer.cpp -- see data_layer.hpp.
#include "data_layer.hpp"

#include <algorithm>
#include <cstdio>

#include "proto_wire.hpp"

namespace caffe {

DataLayer::DataLayer(const NetLayer& L, uint64_t seed, int parser_threads)
    : LayerBase(L.param), parsers_(parser_threads > 0 ? parser_threads : 0), seed_(seed) {}

int DataLayer::ParserThreads(const NetLayer& L) {
  const DataParameter& dp = L.param.data_param;
  if (dp.parser_threads > 0) return dp.parser_threads;
  int c = 0, h = 0, w = 0;
  bool encoded = false;
  PeekDatumShape(dp.source, &c, &h, &w, dp.force_encoded_color, &encoded);
  return encoded ? 6 : 1;
}

DataLayer::~DataLayer() {
  if (copy_stream_) cudaStreamSynchronize(copy_stream_);
  cudaStreamSynchronize(Caffe::thread_stream());     // a transform may still be reading a device slot
  reader_.reset();                                   // joins the parser threads before their pinned buffers are released
  for (Slot& sl : slot_) {
    if (sl.buf.data) cudaFreeHost(sl.buf.data);
    if (sl.buf.label) cudaFreeHost(sl.buf.label);
    if (sl.buf.record_id) cudaFreeHost(sl.buf.record_id);
    if (sl.host_off) cudaFreeHost(sl.host_off);
    if (sl.dev_u8) cudaFree(sl.dev_u8);
    if (sl.dev_off) cudaFree(sl.dev_off);
    if (sl.dev_label) cudaFree(sl.dev_label);
    if (sl.copied) cudaEventDestroy(sl.copied);
    if (sl.consumed) cudaEventDestroy(sl.consumed);
  }
  if (dev_mean_values_) cudaFree(dev_mean_values_);
  if (dev_mean_image_) cudaFree(dev_mean_image_);
  if (copy_stream_) cudaStreamDestroy(copy_stream_);
}

void DataLayer::LayerSetUp(const vector<Blob*>&, const vector<Blob*>& top) {
  const DataParameter& dp = layer_param_.data_param;
  const TransformationParameter& tp = layer_param_.transform_param;
  B2_CHECK(top.size() == 1 || top.size() == 2, "Data layer produces data, or data and label");
  B2_CHECK(dp.batch_size > 0, "Data layer needs a positive batch_size");
  N_ = dp.batch_size;
  bool encoded = false;
  PeekDatumShape(dp.source, &C_, &Hd_, &Wd_, dp.force_encoded_color, &encoded, &float_);    // data_layer.cpp:176-183: shape from one datum
  B2_CHECK(!float_ || FloatDatumsTakeNoTransform(tp.scale, tp.mirror, tp.crop_size, !tp.mean_value.empty() || !tp.mean_file.empty()),
           "Data layer '" + layer_param_.name + "': " + kFloatDatumTransformMsg);
  crop_h_ = tp.crop_size > 0 ? tp.crop_size : Hd_;
  crop_w_ = tp.crop_size > 0 ? tp.crop_size : Wd_;
  B2_CHECK(Hd_ >= crop_h_ && Wd_ >= crop_w_, "crop_size larger than the datum");   // data_transformer.cpp:192-193
  host_crop_ = encoded && tp.crop_size > 0 && tp.mean_file.empty();
  if (host_crop_) Hd_ = Wd_ = tp.crop_size;                                        // the slots hold crop windows
  top[0]->Reshape({N_, C_, crop_h_, crop_w_});
  if (top.size() > 1) top[1]->Reshape({N_});
  batch_bytes_ = (size_t)N_ * C_ * Hd_ * Wd_ * (float_ ? sizeof(float) : 1);

  // DataTransformer's constructor (data_transformer.cpp:17-40)
  if (!tp.mean_file.empty()) {
    B2_CHECK(tp.mean_value.empty(), "Cannot specify mean_file and mean_value at the same time");
    const BlobData mean = ParseBlobProto(ReadBinaryFile(tp.mean_file));
    vector<int> shp = mean.shape;
    while (shp.size() > 3 && shp.front() == 1) shp.erase(shp.begin());   // (1, C, H, W) as compute_image_mean writes it
    B2_CHECK(shp.size() == 3 && shp[0] == C_ && shp[1] == Hd_ && shp[2] == Wd_,
             "mean_file " + tp.mean_file + " does not have the datums' channels x height x width");   // data_transformer.cpp:198-200
    CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&dev_mean_image_), sizeof(float) * mean.data.size()));
    CUDA_CHECK(cudaMemcpy(dev_mean_image_, mean.data.data(), sizeof(float) * mean.data.size(), cudaMemcpyHostToDevice));
  } else if (!tp.mean_value.empty()) {
    B2_CHECK(tp.mean_value.size() == 1 || (int)tp.mean_value.size() == C_, "Specify either 1 mean_value or as many as channels: " + std::to_string(C_));
    vector<float> mv(C_, tp.mean_value[0]);
    if ((int)tp.mean_value.size() == C_) mv = tp.mean_value;
    CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&dev_mean_values_), sizeof(float) * C_));
    CUDA_CHECK(cudaMemcpy(dev_mean_values_, mv.data(), sizeof(float) * C_, cudaMemcpyHostToDevice));
  }

  if (dp.cache || dp.shuffle)
    fprintf(stderr, "DataLayer '%s': data_param { cache: %s shuffle: %s } -- the database is a read-only mapping of the page cache, "
                    "so `cache` has nothing to add; `shuffle` is not built: records are read in key order (shuffle when converting)\n",
            layer_param_.name.c_str(), dp.cache ? "true" : "false", dp.shuffle ? "true" : "false");
  if (parsers_ == 0) parsers_ = dp.parser_threads > 0 ? dp.parser_threads : (encoded ? 6 : 1);   // as ParserThreads
  const int K = std::max(2, parsers_ + 1);
  slot_.resize(K);
  CUDA_CHECK(cudaStreamCreateWithFlags(&copy_stream_, cudaStreamNonBlocking));
  for (Slot& sl : slot_) {
    CUDA_CHECK(cudaMallocHost(reinterpret_cast<void**>(&sl.buf.data), batch_bytes_));
    CUDA_CHECK(cudaMallocHost(reinterpret_cast<void**>(&sl.buf.label), sizeof(float) * N_));
    CUDA_CHECK(cudaMallocHost(reinterpret_cast<void**>(&sl.buf.record_id), sizeof(uint32_t) * N_));
    CUDA_CHECK(cudaMallocHost(reinterpret_cast<void**>(&sl.host_off), sizeof(int) * 3 * N_));
    CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&sl.dev_u8), batch_bytes_));
    CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&sl.dev_off), sizeof(int) * 3 * N_));
    CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&sl.dev_label), sizeof(float) * N_));
    CUDA_CHECK(cudaEventCreateWithFlags(&sl.copied, cudaEventDisableTiming));
    CUDA_CHECK(cudaEventCreateWithFlags(&sl.consumed, cudaEventDisableTiming));
  }
  for (Blob* b : top) b->mutable_gpu_data();          // allocate; the first Forward loads the first batch
}

void DataLayer::set_solver(int solver_count, int solver_rank) {
  B2_CHECK(!reader_, "DataLayer::set_solver after the first batch: the parser threads already read as rank " + std::to_string(solver_rank_));
  B2_CHECK(solver_count > 0 && solver_rank >= 0 && solver_rank < solver_count, "DataLayer::set_solver: rank outside count");
  solver_count_ = solver_count;
  solver_rank_ = solver_rank;
}

size_t DataLayer::h2d_bytes() const { return batch_bytes_ + sizeof(int) * 3 * (size_t)N_ + sizeof(float) * (size_t)N_; }

void DataLayer::EnsureStarted() {
  if (reader_) return;
  const TransformationParameter& tp = layer_param_.transform_param;
  DataReaderParam p;
  p.source = layer_param_.data_param.source;
  p.batch_size = N_;
  p.solver_count = (size_t)solver_count_;
  p.solver_rank = (size_t)solver_rank_;
  p.parser_threads = (size_t)parsers_;
  p.force_encoded_color = layer_param_.data_param.force_encoded_color;
  p.host_crop = host_crop_ ? tp.crop_size : 0;
  p.train = layer_param_.phase != TEST;
  reader_.reset(new DataReader(p));
  B2_CHECK(reader_->channels() == C_ && reader_->height() == Hd_ && reader_->width() == Wd_ && reader_->float_data() == float_,
           "database changed shape between set-up and start");
  // random_seed >= 0: "Use random_seed setting for deterministic transformations" (data_transformer.cpp:733-736); otherwise every
  // solver gets its own stream (the reference: Caffe::next_seed() of a solver seeded with seed + rank, parallel.cpp:179-187)
  const uint64_t s = tp.random_seed >= 0 ? (uint64_t)tp.random_seed : seed_ + 0x9E3779B9ull * (uint64_t)(solver_rank_ + 1);
  draws_.reset(new TransformDraws(s, tp.mirror, tp.crop_size, p.train));
  for (int s = 0; s < (int)slot_.size(); ++s) HandToReader(s);   // slot k assembles batch k, k + K, k + 2K, ...
}

void DataLayer::HandToReader(int s) {
  Slot& sl = slot_[s];
  if (host_crop_) {                                      // Fill3Randoms per item, in batch order: the stream one transformer thread draws
    sl.rand.resize((size_t)3 * N_);
    for (int i = 0; i < N_; ++i) draws_->Fill3Randoms(sl.rand.data() + 3 * i);
    sl.buf.rand = sl.rand.data();
  }
  reader_->free_push(&sl.buf);
}

void DataLayer::IssueCopy(int s) {
  Slot& sl = slot_[s];
  BatchBuf* b = reader_->full_pop();                     // blocks until the parser thread has assembled the batch
  B2_CHECK(b == &sl.buf, "DataLayer: batch order and slot order diverged");
  if (sl.used) CUDA_CHECK(cudaStreamWaitEvent(copy_stream_, sl.consumed, 0));   // the transform that read this device slot is done
  // crop / mirror draws in item order (one parser thread pops datums in record order, so pop order == item order;
  // data_layer.cpp:283-296).  host_off is free: LoadBatch waited for this slot's previous copy before handing the slot back.
  unsigned char* mir = reinterpret_cast<unsigned char*>(sl.host_off + 2 * N_);
  if (host_crop_) {                                      // the windows are cut already; what is left for the device is the flip
    for (int i = 0; i < N_; ++i) { sl.host_off[i] = sl.host_off[N_ + i] = 0; mir[i] = (layer_param_.transform_param.mirror && (sl.rand[3 * i] % 2)) ? 1 : 0; }
  } else {
    for (int i = 0; i < N_; ++i) draws_->Draw(Hd_, Wd_, sl.host_off + i, sl.host_off + N_ + i, mir + i);
  }
  CUDA_CHECK(cudaMemcpyAsync(sl.dev_u8, sl.buf.data, batch_bytes_, cudaMemcpyHostToDevice, copy_stream_));
  CUDA_CHECK(cudaMemcpyAsync(sl.dev_off, sl.host_off, sizeof(int) * 3 * N_, cudaMemcpyHostToDevice, copy_stream_));
  CUDA_CHECK(cudaMemcpyAsync(sl.dev_label, sl.buf.label, sizeof(float) * N_, cudaMemcpyHostToDevice, copy_stream_));
  CUDA_CHECK(cudaEventRecord(sl.copied, copy_stream_));
  sl.in_flight = true;
}

void DataLayer::LoadBatch(const vector<Blob*>& top, cudaStream_t st) {
  EnsureStarted();
  Slot& sl = slot_[cur_];
  if (!sl.in_flight) IssueCopy(cur_);                    // the first batch: nothing was prefetched yet
  CUDA_CHECK(cudaStreamWaitEvent(st, sl.copied, 0));
  if (float_)                                            // float_data datums are the top's values already
    CUDA_CHECK(cudaMemcpyAsync(top[0]->mutable_gpu_data(), sl.dev_u8, batch_bytes_, cudaMemcpyDeviceToDevice, st));
  else
    B2C_CHECK(b2c_transform_u8(sl.dev_u8, N_, C_, Hd_, Wd_, crop_h_, crop_w_, sl.dev_off, sl.dev_off + N_,
                               reinterpret_cast<const unsigned char*>(sl.dev_off + 2 * N_), dev_mean_values_, dev_mean_image_, layer_param_.transform_param.scale,
                               top[0]->mutable_gpu_data(), st));
  if (top.size() > 1)
    CUDA_CHECK(cudaMemcpyAsync(top[1]->mutable_gpu_data(), sl.dev_label, sizeof(float) * N_, cudaMemcpyDeviceToDevice, st));
  CUDA_CHECK(cudaEventRecord(sl.consumed, st));
  // the pinned half of the slot goes back to the parser threads as soon as its bytes have left the host (the copy was issued a
  // whole step ago, so this wait is normally already satisfied)
  CUDA_CHECK(cudaEventSynchronize(sl.copied));
  sl.in_flight = false;
  sl.used = true;
  HandToReader(cur_);
  ++batches_;
  cur_ = (cur_ + 1) % (int)slot_.size();
  IssueCopy(cur_);                                       // the next batch crosses PCIe while this one is computed on
}

}  // namespace caffe
