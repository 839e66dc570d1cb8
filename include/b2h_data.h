/* b2h_data.h -- flat C entry points of the input pipeline's HOST half (libb2caffe.so: caffe_mpi_b200/host/b2h_data_capi.cpp).
 *
 * SURVEY.md 8(f) rank 4.  The C++ classes a Caffe-MPI maintainer codes against keep the reference's names (caffe::db::LMDB,
 * caffe::db::LMDBCursor, caffe::DataReader, caffe::DataLayer -- host/lmdb_reader.hpp, data_reader.hpp, data_layer.hpp; binding
 * table in INTEGRATION.md section 8); these functions marshal them for ctypes (tests/test_data_cpu.py) and for any other FFI.
 * None of them touches the device.  Conventions: plain pointers and sizes; 0 / a handle on success, -1 / NULL on failure with the
 * message in b2h_data_last_error() (the reference aborts through glog CHECK / MDB_CHECK instead).  The device half of the
 * pipeline is b2c_transform_u8 in include/b2c.h. */
#ifndef B2H_DATA_H_
#define B2H_DATA_H_
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

const char* b2h_data_last_error(void);

/* ---- db::LMDB / LMDBCursor / LMDBTransaction (include/caffe/util/db_lmdb.hpp:27-106, src/caffe/util/db_lmdb.cpp) --------------------
 * `source` is the environment directory (holding data.mdb) or the data file itself.  The handle owns the environment (an mmap of
 * the file, as mdb_env_open(MDB_RDONLY | MDB_NOLOCK) makes) and one cursor, positioned on the first record like LMDBCursor's
 * constructor leaves it. */
int b2h_lmdb_exists(const char* source);                       /* data.mdb present?  (what B2C_DATA=auto tests) */
void* b2h_lmdb_open(const char* source);                       /* LMDB::Open(source, READ) + NewCursor() */
void* b2h_lmdb_open_mode(const char* source, int mode);        /* LMDB::Open(source, mode): 0 READ, 1 WRITE, 2 NEW (mkdir must succeed) */
/* LMDBTransaction::Put / Commit (src/caffe/util/db_lmdb.cpp:52-96) on the handle's pending transaction.  A commit whose keys all sort
 * after the database's last key appends (convert_imageset's pattern); any other rewrites the file -- see host/lmdb_reader.hpp. */
int b2h_lmdb_put(void* env, const void* key, size_t key_size, const void* value, size_t value_size);
int b2h_lmdb_commit(void* env);
void b2h_lmdb_close(void* env);                                /* LMDB::Close() */
int b2h_lmdb_stat(void* env, long long* entries, unsigned* page_size, unsigned* depth, unsigned long long* txnid);   /* mdb_env_stat */
int b2h_lmdb_seek_to_first(void* env);                         /* LMDBCursor::SeekToFirst(); returns valid() as 1 / 0, -1 on error */
int b2h_lmdb_next(void* env);                                  /* LMDBCursor::Next(); returns valid() */
int b2h_lmdb_valid(void* env);                                 /* LMDBCursor::valid() */
/* LMDBCursor::key() / data() / size(): pointers INTO the mapping, valid until b2h_lmdb_close */
int b2h_lmdb_current(void* env, const void** key, size_t* key_size, const void** value, size_t* value_size);

/* ---- Datum (src/caffe/proto/caffe.proto:43-56) and the mean_file BlobProto (caffe.proto:15-35) ------------------------------------
 * b2h_datum_parse = Datum::ParseFromArray as CursorManager::fetch calls it (src/caffe/data_reader.cpp:312-316): returns 1 if the
 * bytes parse, 0 if not.  out[0..5] = channels, height, width, label, encoded, record_id; *data / *data_size view the input buffer
 * (zero copy); float_data is copied when float_cap > 0. */
int b2h_datum_parse(const void* bytes, size_t n, long long* out, const void** data, size_t* data_size, float* float_data, int float_cap,
                    int* n_float);
/* what convert_imageset stores per image (tools/convert_imageset.cpp, CVMatToDatum in src/caffe/util/io.cpp): returns the length
 * written to `out`, -1 if it does not fit */
long long b2h_datum_serialize(int channels, int height, int width, const void* data, size_t data_size, int label, int encoded,
                              const float* float_data, int n_float, void* out, size_t cap);
/* An ENCODED datum's image: DecodeDatumToCVMatNative / DecodeDatumToCVMat(force_color) (src/caffe/util/io.cpp:167-190, cv::imdecode)
 * followed by CVMatToDatum's [channel][row][column] layout with OpenCV's channel order B, G, R (io.cpp:205-230).  Baseline and progressive
 * Huffman JPEG and non-interlaced 8-bit PNG, picked by the file's signature (host/jpeg_decode.hpp, png_decode.cpp).  chw[0..2] = channels, height, width; `out` may be NULL to learn the shape. */
int b2h_jpeg_decode(const void* bytes, size_t n, int force_color, int* chw, unsigned char* out, size_t cap);
/* ReadProtoFromBinaryFileOrDie(mean_file) + Blob::FromProto (src/caffe/data_transformer.cpp:21-30, src/caffe/blob.cpp:352-414):
 * shape gets up to 8 axes; call with data == NULL to learn the count first */
int b2h_blobproto_load(const char* path, int* ndim, int* shape, long long* count, float* data);
int b2h_blobproto_save(const char* path, int ndim, const int* shape, const float* data, int raw_format);   /* compute_image_mean's output */

/* ---- DataReader (src/caffe/data_reader.cpp:16-124 threads and queues, :206-310 CursorManager) ---------------------------------------
 * Same arguments as the reference's constructor: which solver of how many (Caffe::solver_count(), solver_rank_), which node of how
 * many (Clusters::node_count() / node_rank()), parser threads per solver, batch size.  `depth` = batches in flight per parser
 * thread (queue_depth); force_encoded_color = DataParameter.force_encoded_color (encoded datums are decoded by the parser threads).  Batches come back in the order the data layer consumes them: batch n of this solver = records
 * [first_record(n), first_record(n) + batch_size) of the (node, solver, thread) partition, positions taken modulo the entries. */
void* b2h_data_reader_create(const char* source, int batch_size, int solver_count, int solver_rank, int node_count, int node_rank,
                             int parser_threads, int depth, int force_encoded_color);
void b2h_data_reader_destroy(void* reader);
int b2h_data_reader_info(void* reader, int* chw, long long* entries, long long* full_cycle);   /* DataReader::sample() shape */
long long b2h_data_reader_first_record(void* reader, long long batch);                           /* CursorManager::rewind / next */
/* DataLayer::load_batch's view of one batch (src/caffe/layers/data_layer.cpp:232-296): uint8 datums [B][C][H][W] (floats when the
 * database's datums carry float_data and no `data`, as DIGITS' label databases do) at item_id = record_id % B, labels as floats,
 * Datum::record_id per item */
int b2h_data_reader_next(void* reader, unsigned char* data, float* label, unsigned* record_id, long long* batch_id);

/* ---- DataTransformer::Fill3Randoms + the crop / mirror rules of Transform (src/caffe/data_transformer.cpp:127-137,187,219-228) ------
 * n consecutive datums of a transformer seeded with `seed` (transform_param.random_seed; caffe::rng_t = mt19937) */
int b2h_transform_draws(unsigned long long seed, int mirror, int crop, int train, int n, int datum_h, int datum_w, int* h_off, int* w_off,
                        unsigned char* do_mirror);

#ifdef __cplusplus
}
#endif
#endif  /* B2H_DATA_H_ */
