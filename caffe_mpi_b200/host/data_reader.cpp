// data_reader.cpp -- see data_reader.hpp.
#include "data_reader.hpp"

#include <sys/stat.h>

#include <cstdlib>
#include <cstring>

#include "b2caffe.hpp"
#include "jpeg_decode.hpp"

namespace caffe {

namespace {
// CursorManager::next / rewind step the cursor one record at a time and restart from the first record when it runs off the
// end (data_reader.cpp:246-258, 300-305); n steps on a ring of `entries` records end where n % entries steps do.
void step(db::LMDBCursor* cur) {
  cur->Next();
  if (!cur->valid()) cur->SeekToFirst();
}
void advance(db::LMDBCursor* cur, size_t n, size_t entries) {
  for (size_t i = n % entries; i > 0; --i) step(cur);
}
}  // namespace

namespace {
// What a datum contributes to a batch: its own bytes, the decoded image of an encoded one (DecodeDatumToCVMat[Native] +
// CVMatToDatum, io.cpp:167-230), or its float_data when it carries floats and no `data` (the label databases DIGITS writes for
// DetectNet; DataTransformer::Copy moves them to the device as they are, data_transformer.cpp:92-110).  Returns whether the values are floats;
// *px then points at c*h*w floats, else at c*h*w bytes.  `img` is scratch that keeps the decoded pixels alive.
bool datum_values(const Datum& d, bool force_color, DecodedImage* img, const void** px, int* c, int* h, int* w) {
  if (d.encoded) {
    DecodeImage(d.data, d.data_size, force_color, img);        // JPEG or PNG, by the file's own signature (cv::imdecode does the same)
    *px = img->chw.data(); *c = img->channels; *h = img->height; *w = img->width;
    return false;
  }
  B2_CHECK(d.channels > 0 && d.height > 0 && d.width > 0, "DataReader: datum has no shape");
  const size_t n = (size_t)d.channels * d.height * d.width;
  *c = d.channels; *h = d.height; *w = d.width;
  if (d.data_size == 0 && !d.float_data.empty()) {
    B2_CHECK(d.float_data.size() == n, "DataReader: datum float_data size disagrees with channels*height*width");
    *px = d.float_data.data();
    return true;
  }
  B2_CHECK(d.data_size == n, "DataReader: datum data size disagrees with channels*height*width");
  *px = d.data;
  return false;
}
}  // namespace

DataReader::DataReader(const DataReaderParam& p) : p_(p) {
  B2_CHECK(p_.batch_size > 0, "DataReader: batch_size must be positive");
  B2_CHECK(p_.solver_count > 0 && p_.solver_rank < p_.solver_count, "DataReader: solver_rank outside solver_count");
  B2_CHECK(p_.node_count > 0 && p_.node_rank < p_.node_count, "DataReader: node_rank outside node_count");
  if (p_.parser_threads == 0) p_.parser_threads = 1;
  db_.reset(new db::LMDB());
  db_->Open(p_.source, db::READ);
  B2_CHECK(db_->entries() > 0, "DataReader: database " + p_.source + " is empty");
  {  // DataReader::sample(): the first datum fixes the batch geometry
    std::unique_ptr<db::LMDBCursor> cur(db_->NewCursor());
    B2_CHECK(cur->valid(), "DataReader: database " + p_.source + " has no first record");
    Datum d;
    B2_CHECK(ParseDatum(cur->data(), cur->size(), &d), "Database cursor failed to parse Datum record");
    DecodedImage img;
    const void* px = nullptr;
    float_ = datum_values(d, p_.force_encoded_color, &img, &px, &c_, &h_, &w_);
    if (p_.host_crop > 0) {
      B2_CHECK(!float_, "DataReader: float_data datums are copied whole (no crop)");
      B2_CHECK(h_ >= p_.host_crop && w_ >= p_.host_crop, "crop_size larger than the datum");
      h_ = w_ = p_.host_crop;                            // the batch holds windows
    }
  }
  full_cycle_ = p_.parser_threads * (size_t)p_.batch_size * p_.solver_count * p_.node_count;
  for (size_t t = 0; t < p_.parser_threads; ++t) {
    free_.emplace_back(new Queue());
    full_.emplace_back(new Queue());
  }
  for (size_t t = 0; t < p_.parser_threads; ++t) threads_.emplace_back(&DataReader::thread_entry, this, t);
}

DataReader::~DataReader() {
  for (auto& q : free_) { std::lock_guard<std::mutex> g(q->m); stop_ = true; }
  for (auto& q : free_) q->cv.notify_all();
  for (auto& q : full_) q->cv.notify_all();
  for (auto& th : threads_) th.join();
}

size_t DataReader::first_record_of_batch(size_t n) const {
  const size_t P = p_.parser_threads, B = (size_t)p_.batch_size;
  const size_t t = n % P, k = n / P;
  const size_t rank_cycle_per_solver = P * B, rank_cycle_per_node = rank_cycle_per_solver * p_.solver_count;
  return rank_cycle_per_solver * p_.solver_rank + rank_cycle_per_node * p_.node_rank + t * B + k * full_cycle_;
}

void DataReader::free_push(BatchBuf* b) {
  Queue& q = *free_[pushed_ % p_.parser_threads];
  ++pushed_;
  { std::lock_guard<std::mutex> g(q.m); q.q.push_back(b); }
  q.cv.notify_one();
}

BatchBuf* DataReader::full_pop() {
  B2_CHECK(popped_ < pushed_, "DataReader::full_pop: no buffer is with the reader (free_push one first)");
  Queue& q = *full_[popped_ % p_.parser_threads];
  std::unique_lock<std::mutex> g(q.m);
  q.cv.wait(g, [&] { return !q.q.empty() || stop_; });
  if (q.q.empty()) {                       // a parser thread died
    std::lock_guard<std::mutex> e(err_m_);
    Fatal(__FILE__, __LINE__, "DataReader: " + (error_.empty() ? std::string("reader stopped") : error_));
  }
  BatchBuf* b = q.q.front();
  q.q.pop_front();
  ++popped_;
  return b;
}

void DataReader::fill(db::LMDBCursor* cur, size_t rec_id, BatchBuf* b) {
  const size_t B = (size_t)p_.batch_size, bytes = datum_bytes();
  Datum d;
  DecodedImage img;
  for (size_t j = 0; j < B; ++j) {
    B2_CHECK(ParseDatum(cur->data(), cur->size(), &d), "Database cursor failed to parse Datum record");
    const void* vals = nullptr;
    int c = 0, h = 0, w = 0;
    B2_CHECK(datum_values(d, p_.force_encoded_color, &img, &vals, &c, &h, &w) == float_,
             "DataReader: " + p_.source + " mixes float_data datums and uint8 datums");
    const uint8_t* px = static_cast<const uint8_t*>(vals);
    B2_CHECK(c == c_, "Number of channels can't vary in the same batch");
    const size_t item = (rec_id + j) % B;                              // data_layer.cpp:256
    if (p_.host_crop > 0) {
      // the window of DataTransformer::Transform (data_transformer.cpp:216-229), cut here so that datums of any size fit the batch
      const int crop = p_.host_crop;
      B2_CHECK(h >= crop && w >= crop, "crop_size larger than a datum of " + p_.source);        // data_transformer.cpp:192-193
      B2_CHECK(b->rand != nullptr || !p_.train, "DataReader: host_crop needs the consumer's draws (BatchBuf::rand)");
      const int h_off = p_.train ? (int)(b->rand[3 * item + 1] % (unsigned)(h - crop + 1)) : (h - crop) / 2;
      const int w_off = p_.train ? (int)(b->rand[3 * item + 2] % (unsigned)(w - crop + 1)) : (w - crop) / 2;
      uint8_t* dst = b->data + item * bytes;
      for (int cc = 0; cc < c; ++cc)
        for (int y = 0; y < crop; ++y) memcpy(dst + ((size_t)cc * crop + y) * crop, px + ((size_t)cc * h + h_off + y) * w + w_off, (size_t)crop);
    } else {
      B2_CHECK(h == h_, "Image height can't vary in the same batch (crop might help here)");   // data_layer.cpp:262-271; all
      B2_CHECK(w == w_, "Image width can't vary in the same batch (crop might help here)");     // datums share the sample's shape
      memcpy(b->data + item * bytes, px, bytes);
    }
    b->label[item] = (float)d.label;
    if (b->record_id) b->record_id[item] = (uint32_t)(rec_id + j);
    step(cur);
  }
}

void DataReader::thread_entry(size_t t) {
  try {
    const size_t P = p_.parser_threads, B = (size_t)p_.batch_size, entries = db_->entries();
    std::unique_ptr<db::LMDBCursor> cur(db_->NewCursor());
    size_t rec_id = first_record_of_batch(t);                           // CursorManager::rewind
    cur->SeekToFirst();
    advance(cur.get(), rec_id, entries);
    for (size_t k = 0;; ++k) {
      Queue& fq = *free_[t];
      BatchBuf* b = nullptr;
      {
        std::unique_lock<std::mutex> g(fq.m);
        fq.cv.wait(g, [&] { return !fq.q.empty() || stop_; });
        if (stop_) return;
        b = fq.q.front();
        fq.q.pop_front();
      }
      fill(cur.get(), rec_id, b);
      b->batch_id = k * P + t;
      advance(cur.get(), full_cycle_ - B, entries);                     // CursorManager::next: rec_id_ += full_cycle_ - batch_size_
      rec_id += full_cycle_;
      Queue& uq = *full_[t];
      { std::lock_guard<std::mutex> g(uq.m); uq.q.push_back(b); }
      uq.cv.notify_one();
    }
  } catch (const std::exception& e) {
    { std::lock_guard<std::mutex> g(err_m_); if (error_.empty()) error_ = e.what(); }
    for (auto& q : full_) { std::lock_guard<std::mutex> g(q->m); stop_ = true; }
    for (auto& q : full_) q->cv.notify_all();
    for (auto& q : free_) q->cv.notify_all();
  }
}

bool UseDatabase(const std::string& source, int backend) {
  const char* e = std::getenv("B2C_DATA");
  const std::string mode = e ? e : "auto";
  if (mode == "synthetic" || source.empty() || source == "synthetic") return false;   // "synthetic": the name caffe_mpi_b200/models.py gives its stand-in source
  const bool there = db::LMDB::Exists(source);
  if (mode == "db") B2_CHECK(there, "Failed to open lmdb " + source + ": no data.mdb (B2C_DATA=db)");
  if (!there) {
    // a directory that is there but holds no data.mdb is a LevelDB or a wrong path: training on the synthetic stand-in instead would be
    // a silent surprise.  (A source that does not exist at all is the benchmark / test case: the reference's prototxts on a machine
    // without ImageNet.)
    struct stat st;
    B2_CHECK(!(stat(source.c_str(), &st) == 0 && S_ISDIR(st.st_mode)),
             "Data layer source " + source + " exists but holds no data.mdb (LevelDB databases are not built; B2C_DATA=synthetic ignores the source)");
    return false;
  }
  B2_CHECK(backend == 1, "Data layer source " + source + " exists but its backend is LEVELDB: only `backend: LMDB` is built");
  return true;
}

void PeekDatumShape(const std::string& source, int* c, int* h, int* w, bool force_encoded_color, bool* encoded, bool* float_data) {
  db::LMDB env;
  env.Open(source, db::READ);
  std::unique_ptr<db::LMDBCursor> cur(env.NewCursor());
  B2_CHECK(cur->valid(), "database " + source + " is empty");
  Datum d;
  B2_CHECK(ParseDatum(cur->data(), cur->size(), &d), "Database cursor failed to parse Datum record");
  DecodedImage img;
  const void* px = nullptr;
  const bool f = datum_values(d, force_encoded_color, &img, &px, c, h, w);
  if (encoded) *encoded = d.encoded;
  if (float_data) *float_data = f;
}

// ------------------------------------------------------------------------------------------------ TransformDraws
void TransformDraws::Fill3Randoms(unsigned* r) {
  r[0] = r[1] = r[2] = 0;
  if (mirror_) r[0] = (unsigned)rng_() + 1u;
  if (train_ && crop_) {
    r[1] = (unsigned)rng_() + 1u;
    r[2] = (unsigned)rng_() + 1u;
  }
}

void TransformDraws::Draw(int datum_h, int datum_w, int* h_off, int* w_off, unsigned char* do_mirror) {
  unsigned r[3];
  Fill3Randoms(r);
  *do_mirror = (mirror_ && (r[0] % 2)) ? 1 : 0;
  *h_off = *w_off = 0;
  if (crop_) {
    B2_CHECK(datum_h >= crop_ && datum_w >= crop_, "crop_size larger than the datum");   // data_transformer.cpp:192-193
    if (train_) {
      *h_off = (int)(r[1] % (unsigned)(datum_h - crop_ + 1));
      *w_off = (int)(r[2] % (unsigned)(datum_w - crop_ + 1));
    } else {
      *h_off = (datum_h - crop_) / 2;
      *w_off = (datum_w - crop_) / 2;
    }
  }
}

}  // namespace caffe
