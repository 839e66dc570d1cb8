// tc_host.cu -- host plumbing the tensor-core kernel files share (declared in tc_common.cuh): tensor-map encoding, the one-wave
// split-K planner, B2C_PROF counter buffers; and env_int (b2c_common.cuh), how every B2C_* switch of the library is read.
#include <stdlib.h>
#include "b2c_common.cuh"
#include "tc_common.cuh"

namespace b2c {

long env_int(const char* name, long dflt) {
  const char* e = getenv(name);
  return e ? atol(e) : dflt;
}

namespace tc {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// the driver's cuTensorMapEncodeTiled, looked up once (no link dependency on libcuda)
static EncodeTiledFn encode_tiled() {
  static const EncodeTiledFn fn = [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      return reinterpret_cast<EncodeTiledFn>(f);
    return (EncodeTiledFn) nullptr;
  }();
  return fn;
}

int make_tensor_map_3d(CUtensorMap* map, CUtensorMapDataType dtype, const void* base, const cuuint64_t (&dims)[3],
                       const cuuint64_t (&byte_strides)[2], const cuuint32_t (&box)[3], CUtensorMapSwizzle swizzle, const char* what) {
  EncodeTiledFn enc = encode_tiled();
  if (!enc) return fail(B2C_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
  const cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, dtype, 3, const_cast<void*>(base), dims, byte_strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(B2C_ERR_CUDA, "cuTensorMapEncodeTiled (%s) failed (%d)", what, (int)r);
  return B2C_OK;
}

void plan_splitk(long long nkb, long long tiles, int min_kb_per_split, int* splits, int* kb_per_split) {
  long long n = sm_count() / tiles;
  const long long max_splits = nkb / min_kb_per_split > 0 ? nkb / min_kb_per_split : 1;
  if (n > max_splits) n = max_splits;
  if (n < 1) n = 1;
  const long long per = (nkb + n - 1) / n;
  *splits = (int)((nkb + per - 1) / per);
  *kb_per_split = (int)per;
}

long long* prof_buffer(cudaStream_t st) {
  static const bool on = env_int("B2C_PROF", 0) != 0;
  if (!on) return nullptr;
  static long long* const buf = [] { long long* b = nullptr; cudaMalloc(&b, 32 * sizeof(long long)); return b; }();
  cudaMemsetAsync(buf, 0, 32 * sizeof(long long), st);
  return buf;
}

void prof_read(const long long* buf, long long (&h)[32]) { cudaMemcpy(h, buf, sizeof(h), cudaMemcpyDeviceToHost); }

}  // namespace tc
}  // namespace b2c
