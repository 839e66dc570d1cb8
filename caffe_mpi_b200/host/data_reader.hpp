// data_reader.hpp -- DataReader: the parser threads between the LMDB and the data layer (SURVEY 8(f) rank 4, 8(e) "data
// reader stride").
//
// Reference: src/caffe/data_reader.cpp:16-124 (DataReader, InternalThreadEntryN), :206-310 (CursorManager: which records a
// (node, solver, parser thread) triple reads), include/caffe/data_reader.hpp.  Kept from it, exactly:
//   * the partition.  With B = batch_size, P = parser threads per solver, S = solvers per node, N = nodes:
//         rank_cycle = P*B,  full_cycle = P*B*S*N
//         parser thread t of solver s on node n starts at record  P*B*s + P*B*S*n + t*B   (CursorManager::rewind)
//         reads B consecutive records, then jumps full_cycle - B ahead                     (CursorManager::next)
//     so every record of the database is read by exactly one (n, s, t) per full cycle, and a thread's k-th run of B records is
//     one whole batch: batch number k*P + t of its solver (data_reader.cpp:96-98), item_id = record_id % B (data_layer.cpp:256);
//   * wrap-around by cursor stepping: Next(), and SeekToFirst() when the cursor runs off the end (data_reader.cpp:246-258,
//     300-305), i.e. positions are record ids modulo the number of entries;
//   * Datum::record_id numbering (data_reader.cpp:239).
// GPU-first differences: the unit handed between threads is a BATCH, not a Datum -- a parser thread owns the B records of its
// batch anyway -- and it is assembled in place in a buffer the consumer provides (the data layer passes pinned host memory), the
// datum's pixel bytes being copied once, from the file mapping.  The reference moves every datum three times (LMDB value ->
// Datum string -> batch blob -> device).  DataParameter.cache / shuffle are accepted and ignored with a note: the mapping is the
// cache; shuffling is not built.  ENCODED datums (convert_imageset --encoded) are decoded by the parser threads with the baseline
// JPEG decoder of jpeg_decode.hpp -- bit-identical to the reference's cv::imdecode on the files it takes; PNG-encoded datums and
// the JPEG variants that decoder lists are fatal.  Raw datums are the fast path: a decode costs a few milliseconds per image and
// thread, so an encoded database wants `parser_threads` raised accordingly.
#pragma once
#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <deque>
#include <memory>
#include <mutex>
#include <random>
#include <string>
#include <thread>
#include <vector>

#include "lmdb_reader.hpp"
#include "proto_wire.hpp"

namespace caffe {

struct DataReaderParam {
  std::string source;
  int batch_size = 1;
  size_t solver_count = 1, solver_rank = 0;     // Caffe::solver_count(), solver_rank_
  size_t node_count = 1, node_rank = 0;         // Clusters::node_count() / node_rank()
  size_t parser_threads = 1;                    // DataParameter.parser_threads (0 = auto in the reference; 1 here)
  bool force_encoded_color = false;             // DataParameter.force_encoded_color: decode one-channel files to three channels
  // > 0: the parser threads cut the crop_size x crop_size window out of every datum themselves, from the draws the consumer hands
  // over with the buffer (BatchBuf::rand), and the batch holds only the windows.  This is what lets datums of DIFFERENT sizes share a
  // batch -- the reference's "crop might help here" (data_layer.cpp:262-271), i.e. databases of original, un-resized image files --
  // and it moves crop^2 instead of H x W bytes per image over PCIe.  0: whole datums, one size, cropped on the device.
  int host_crop = 0;
  bool train = true;                            // TRAIN: random window; TEST: the centre window (data_transformer.cpp:219-229)
};

// One batch under assembly / assembled.  `data` is [batch][C][H][W] uint8 in datum layout (float for float_data datums), `label`
// one float per item (the reference's label blob is Ftype), `record_id` the reader's numbering of the records it holds.
struct BatchBuf {
  uint8_t* data = nullptr;
  float* label = nullptr;
  uint32_t* record_id = nullptr;    // may be null
  // host_crop only: DataTransformer::Fill3Randoms' three draws per item (rand[3i + 1], rand[3i + 2] place the window), filled by the
  // consumer in batch order before free_push -- the draws do not depend on the datum, so the stream is the one a single transformer
  // thread would produce however many parser threads cut the windows
  const unsigned* rand = nullptr;
  size_t batch_id = 0;              // k*P + t, set by the reader
};

class DataReader {
 public:
  explicit DataReader(const DataReaderParam& p);
  ~DataReader();
  DataReader(const DataReader&) = delete;
  DataReader& operator=(const DataReader&) = delete;
  // shape of the first datum of the database (DataReader::sample(), used by DataLayerSetUp to size the top blob)
  int channels() const { return c_; }
  int height() const { return h_; }
  int width() const { return w_; }
  // float_data datums (a datum with float_data and no `data`): the batch holds c*h*w floats per item instead of bytes
  bool float_data() const { return float_; }
  size_t datum_bytes() const { return (size_t)c_ * h_ * w_ * (float_ ? sizeof(float) : 1); }
  size_t entries() const { return db_->entries(); }
  size_t full_cycle() const { return full_cycle_; }
  // Hand an empty buffer to the reader: the n-th buffer pushed receives batch n (filled by parser thread n % P).  The buffer must
  // stay valid until it comes back from full_pop() or the reader is destroyed: destroy the reader first, then free the buffers.
  void free_push(BatchBuf* b);
  // Next assembled batch, in batch order 0, 1, 2, ...  Blocks; rethrows a parser thread's failure as caffe::FatalError.
  BatchBuf* full_pop();
  // first record id of batch n of this solver (what CursorManager's rec_id_ is when the batch starts)
  size_t first_record_of_batch(size_t n) const;

 private:
  struct Queue {
    std::mutex m;
    std::condition_variable cv;
    std::deque<BatchBuf*> q;
  };
  void thread_entry(size_t t);
  void fill(db::LMDBCursor* cur, size_t rec_id, BatchBuf* b);
  DataReaderParam p_;
  std::unique_ptr<db::LMDB> db_;
  int c_ = 0, h_ = 0, w_ = 0;
  bool float_ = false;              // the first datum's kind; every datum of the database must be of it
  size_t full_cycle_ = 0;
  std::vector<std::unique_ptr<Queue>> free_, full_;
  std::vector<std::thread> threads_;
  size_t pushed_ = 0, popped_ = 0;
  std::atomic<bool> stop_{false};
  std::mutex err_m_;
  std::string error_;
};

// Which source a Data layer reads.  B2C_DATA = "synthetic": never the database; "db": the database, a missing one is fatal (the
// reference's behaviour, db_lmdb.cpp:19); unset / "auto": the database when <source>/data.mdb exists, else the synthetic source
// (bench.py and the tests run the reference's prototxts on machines that do not hold ImageNet).
bool UseDatabase(const std::string& source, int backend);
// A Data layer over float_data datums takes no transform_param: its values reach the top as they are stored
inline bool FloatDatumsTakeNoTransform(float scale, bool mirror, int crop_size, bool has_mean) {
  return scale == 1.f && !mirror && crop_size == 0 && !has_mean;
}
constexpr const char* kFloatDatumTransformMsg =
    "its datums carry float_data, which are copied as they are: transform_param (crop_size, mirror, mean_file, mean_value, scale) is not built for them";
// channels / height / width of the first datum (DataReader::sample()); an encoded first datum is decoded to learn them.
// *float_data: the datum carries float_data and no `data`
void PeekDatumShape(const std::string& source, int* c, int* h, int* w, bool force_encoded_color = false, bool* encoded = nullptr,
                    bool* float_data = nullptr);

// DataTransformer's random draws (src/caffe/data_transformer.cpp:127-137 Fill3Randoms, :187,219-226 their use, :729-749
// InitRand / Rand): per datum  rand0 = Rand() + 1 if mirror;  rand1 = Rand() + 1, rand2 = Rand() + 1 if TRAIN and crop_size;
// do_mirror = mirror && rand0 % 2;  h_off = rand1 % (H - crop + 1), w_off = rand2 % (W - crop + 1) in TRAIN, the centre
// window in TEST.  Rand() is one draw of a mt19937 (caffe::rng_t = boost::mt19937) seeded with transform_param.random_seed
// when that is >= 0 -- the same stream as std::mt19937 -- so a seeded reference run and this one crop and flip identically.
class TransformDraws {
 public:
  TransformDraws(uint64_t seed, bool mirror, int crop, bool train) : rng_((uint32_t)seed), mirror_(mirror), crop_(crop), train_(train) {}
  void Fill3Randoms(unsigned* r);
  // one datum: consumes Fill3Randoms and applies the rules above
  void Draw(int datum_h, int datum_w, int* h_off, int* w_off, unsigned char* do_mirror);
 private:
  std::mt19937 rng_;
  bool mirror_;
  int crop_;
  bool train_;
};

}  // namespace caffe
