// data_layer.hpp -- DataLayer: LMDB datums -> pinned host batch -> device -> DataTransformer on the device -> top blobs
// (SURVEY 8(f) rank 4; the device half, behind the DataReader of data_reader.hpp).
//
// Reference: src/caffe/layers/data_layer.cpp:127-200 (DataLayerSetUp: shape from one datum, top[0] = {batch, C, crop|H, crop|W},
// top[1] = {batch}), :203-326 (load_batch: pop batch_size datums, item_id = record_id % batch_size, Fill3Randoms per datum in pop
// order, copy the bytes, TransformGPU), src/caffe/layers/base_data_layer.cpp (the prefetch thread and its Batch queue),
// src/caffe/data_transformer.{cpp,cu} (crop / mirror / mean_file | mean_value / scale; "Cannot specify mean_file and mean_value at
// the same time").
//
// GPU-first shape of the same pipeline:
//   parser threads (DataReader)  --memcpy from the file mapping-->  pinned slot k  --cudaMemcpyAsync, copy stream-->  device slot k
//   --b2c_transform_u8 on the compute stream, first thing of the step-->  top[0];   labels ride along and are copied into top[1].
// float_data datums take the same path with 4 bytes per value and no transform (a transform_param is refused).
// K = max(2, parser_threads + 1) slots circulate: while step i computes, batch i+1 is crossing PCIe and batches i+2.. are being
// assembled by the parser threads.  A step moves 1 byte per pixel over PCIe (the reference's GPU transform moves Ftype-sized
// elements, data_layer.cpp:235-237) and no host thread touches a pixel after the parser's one memcpy.
#pragma once
#include "b2caffe.hpp"
#include "data_reader.hpp"
#include "prototxt.hpp"

namespace caffe {

class DataLayer : public LayerBase {
 public:
  // reads L.param's data_param and transform_param.  `seed` feeds the crop / mirror stream when transform_param.random_seed is unset
  // (the reference draws Caffe::next_seed()); the TEST phase takes the centre crop window.  parser_threads > 0 overrides
  // ParserThreads(L) (a net whose Data layers must read in step gives them one count)
  DataLayer(const NetLayer& L, uint64_t seed, int parser_threads = 0);
  // the parser threads the layer runs: data_param.parser_threads, or the automatic count for its datums (see parsers_)
  static int ParserThreads(const NetLayer& L);
  ~DataLayer() override;
  const char* type() const override { return "Data"; }
  void LayerSetUp(const vector<Blob*>& bottom, const vector<Blob*>& top) override;
  void Reshape(const vector<Blob*>&, const vector<Blob*>&) override {}
  // Caffe::solver_count() / solver_rank_ of the reader (parallel.cpp:284-293); must be called before the first batch is loaded
  void set_solver(int solver_count, int solver_rank);
  // the next batch into top[0] (and top[1] when the layer has a label top), ordered on `stream`
  void LoadBatch(const vector<Blob*>& top, cudaStream_t stream);
  bool loaded() const { return batches_ > 0; }
  size_t batches_loaded() const { return batches_; }
  size_t h2d_bytes() const;                       // bytes one batch moves host -> device
  const DataReader* reader() const { return reader_.get(); }

 protected:
  void Forward_gpu(const vector<Blob*>&, const vector<Blob*>&) override {}   // TrainNet::Forward calls LoadBatch (prefetch-aware)
  void Backward_gpu(const vector<Blob*>&, const vector<bool>&, const vector<Blob*>&) override {}

 private:
  struct Slot {
    BatchBuf buf;                 // pinned: data, label (and record ids)
    int* host_off = nullptr;      // pinned: h_off[N], w_off[N], mirror[N] (bytes)
    vector<unsigned> rand;        // host-crop mode: Fill3Randoms' draws of the batch this slot is assembling (3 per item)
    unsigned char* dev_u8 = nullptr;   // the batch on the device, as the slot's pinned `buf.data` holds it
    int* dev_off = nullptr;
    float* dev_label = nullptr;
    cudaEvent_t copied = nullptr, consumed = nullptr;
    bool in_flight = false, used = false;
  };
  void EnsureStarted();
  void IssueCopy(int s);
  void HandToReader(int s);         // host-crop mode: draw the batch's randoms, then free_push the slot
  // Encoded datums with a crop_size and no mean_file: the parser threads -- which decode anyway -- also cut the crop window, so the
  // database may hold images of different sizes (original files) and only crop^2 bytes per image cross PCIe.  Raw datums keep the
  // whole-datum path (one memcpy per datum, crop on the device); a mean_file is indexed in datum coordinates and needs it too.
  bool host_crop_ = false;
  // DataParameter.parser_threads; 0 ("Caffe optimizes it automatically", caffe.proto:841-844; the reference's auto mode ends between 1
  // and 4, data_layer.cpp:85-95) becomes 1 for raw datums -- one thread's memcpy outruns the GPU -- and 6 for encoded ones: at
  // ~0.8 k decoded 256x256 JPEGs per second and thread that is what a GPU training ResNet-50 at a few thousand img/s asks for
  int parsers_ = 1;
  uint64_t seed_;
  int solver_count_ = 1, solver_rank_ = 0;
  int N_ = 0, C_ = 0, Hd_ = 0, Wd_ = 0, crop_h_ = 0, crop_w_ = 0;
  // float_data datums (DIGITS' label databases): the slots carry floats, and LoadBatch copies the device slot into top[0] as it is
  bool float_ = false;
  size_t batch_bytes_ = 0;                 // one batch in a slot: N*C*Hd*Wd bytes, or floats for float_data datums
  std::unique_ptr<DataReader> reader_;
  std::unique_ptr<TransformDraws> draws_;
  vector<Slot> slot_;
  int cur_ = 0;
  size_t batches_ = 0;
  cudaStream_t copy_stream_ = nullptr;
  float* dev_mean_values_ = nullptr;   // [C]
  float* dev_mean_image_ = nullptr;    // [C*Hd*Wd], datum coordinates
};

}  // namespace caffe
