// filter_prep.cu -- see filter_prep.cuh.
#include <cuda_bf16.h>
#include "b2c_common.cuh"
#include "tc_common.cuh"
#include "filter_prep.cuh"

namespace b2c {
using namespace tc;

__global__ void __launch_bounds__(256)
filter_prep_multi_kernel(const __grid_constant__ PrepBatch b) {
  pdl_wait();
  const PrepEntry& q = b.e[blockIdx.y];
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < q.total; idx += (long long)gridDim.x * blockDim.x) {
    const int kp = (int)(idx % q.Kp);
    const long long rg = idx / q.Kp;
    const int row = (int)(rg % q.rows);
    const int g = (int)(rg / q.rows);
    int ch, tap;
    bool valid;
    if (q.kind == 1) {                                  // (channel group of 32, tap, channel in group)
      const int hb = kp >> 5;
      const int cg = hb / q.taps;
      tap = hb - cg * q.taps;
      ch = cg * 32 + (kp & 31);
      valid = ch < q.kch;
    } else {
      valid = kp < q.K;
      if (q.tap_major) { const int cb = kp / (4 * q.taps); const int r = kp - cb * 4 * q.taps; tap = r >> 2; ch = cb * 4 + (r & 3); }
      else { ch = kp / q.taps; tap = kp - ch * q.taps; }
    }
    float v = 0.0f;
    if (valid) {
      if (q.flip) tap = q.taps - 1 - tap;
      const int o = q.mode == 0 ? row : ch, c = q.mode == 0 ? ch : row;
      int taps = q.taps;
      if (q.mode == 2) {
        const int a = tap / q.sub_kw, bb = tap - a * q.sub_kw;
        tap = (q.i0h + (q.sub_kh - 1 - a) * q.Lh) * q.src_kw + q.i0w + (q.sub_kw - 1 - bb) * q.Lw;
        taps = q.src_taps;
      }
      v = __ldg(q.w + (((long long)g * q.Og + o) * q.Cg + c) * taps + tap);
    }
    if (q.kind == 1) {
      const __nv_bfloat16 h = __float2bfloat16_rn(v);
      static_cast<__nv_bfloat16*>(q.hi)[idx] = h;
      static_cast<__nv_bfloat16*>(q.lo)[idx] = __float2bfloat16_rn(v - __bfloat162float(h));
    } else if (q.lo) {
      float h, l;
      split_tf32(v, h, l);
      static_cast<float*>(q.hi)[idx] = h;
      static_cast<float*>(q.lo)[idx] = l;
    } else {
      static_cast<float*>(q.hi)[idx] = to_tf32(v);
    }
  }
}

int launch_filter_prep(const PrepEntry* entries, int n, cudaStream_t st) {
  for (int i0 = 0; i0 < n; i0 += PREP_BATCH) {
    PrepBatch b;
    const int m = n - i0 < PREP_BATCH ? n - i0 : PREP_BATCH;
    long long biggest = 0;
    for (int i = 0; i < m; ++i) { b.e[i] = entries[i0 + i]; if (b.e[i].total > biggest) biggest = b.e[i].total; }
    for (int i = m; i < PREP_BATCH; ++i) { b.e[i] = PrepEntry{}; }
    dim3 grid((unsigned)grid_for((size_t)biggest, 256, 4), (unsigned)m);
    launch_pdl(filter_prep_multi_kernel, grid, 256, 0, st, 0, b);
    B2C_POST_LAUNCH();
  }
  return B2C_OK;
}

}  // namespace b2c
