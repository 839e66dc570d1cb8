// transform.cu -- DataTransformer on the device (SURVEY 8f rank 4: the input pipeline's compute half).
//
// Replaces DataTransformer<Dtype>::Transform(const Datum&, Dtype*, rand) (reference src/caffe/data_transformer.cpp:178-312,
// the uint8 branch; data_transformer.cu is its batched GPU twin): per image a crop window (h_off, w_off), an optional
// horizontal mirror, mean subtraction (per-channel mean_value or a per-pixel mean image in datum coordinates) and a scale:
//     out[n][c][h][w] = (datum[n][c][h_off + h][w_off + (mirror ? crop_w - 1 - w : w)] - mean) * scale
// The batch arrives as uint8 datums (a quarter of the bytes of the float blob it produces), so the host -> device copy of a
// 64 x 3 x 256 x 256 batch is 12.6 MB instead of the 38.5 MB of the cropped float blob.  HBM-bound: 1 B read + 4 B written
// per output element; one thread per 4 consecutive output pixels (16-byte stores).
#include "b2c_common.cuh"

namespace b2c {

__global__ void __launch_bounds__(256)
transform_u8_kernel(const unsigned char* __restrict__ src, int N, int C, int Hd, int Wd, int Hc, int Wc, const int* __restrict__ h_off,
                    const int* __restrict__ w_off, const unsigned char* __restrict__ mirror, const float* __restrict__ mean_values,
                    const float* __restrict__ mean_image, float scale, float* __restrict__ dst) {
  pdl_wait();
  const int wq = (Wc + 3) / 4;                              // 4-pixel groups per output row
  const long long total = (long long)N * C * Hc * wq;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % wq);
    long long t = i / wq;
    const int h = (int)(t % Hc); t /= Hc;
    const int c = (int)(t % C);
    const int n = (int)(t / C);
    const int ho = h_off[n], wo = w_off[n];
    const bool mir = mirror[n] != 0;
    const long long row = (((long long)n * C + c) * Hd + ho + h) * Wd;         // datum row of this output row
    const long long mrow = ((long long)c * Hd + ho + h) * Wd;                  // same row in the mean image
    const float mv = mean_values ? mean_values[c] : 0.f;
    float v[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int w = g * 4 + e;
      v[e] = 0.f;
      if (w < Wc) {
        const int ws = wo + (mir ? Wc - 1 - w : w);
        const float x = (float)src[row + ws];
        const float m = mean_image ? mean_image[mrow + ws] : mv;
        v[e] = (x - m) * scale;
      }
    }
    float* o = dst + (((long long)n * C + c) * Hc + h) * Wc + g * 4;
    if ((Wc & 3) == 0 && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
    else
      for (int e = 0; e < 4 && g * 4 + e < Wc; ++e) o[e] = v[e];
  }
}

}  // namespace b2c

using namespace b2c;

extern "C" int b2c_transform_u8(const unsigned char* src, int N, int C, int Hd, int Wd, int crop_h, int crop_w, const int* h_off,
                                const int* w_off, const unsigned char* mirror, const float* mean_values, const float* mean_image,
                                float scale, float* dst, void* stream) {
  if (!src || !dst || !h_off || !w_off || !mirror || N <= 0 || C <= 0 || Hd <= 0 || Wd <= 0)
    return fail(B2C_ERR_INVALID, "b2c_transform_u8: bad argument");
  if (crop_h <= 0 || crop_w <= 0 || crop_h > Hd || crop_w > Wd) return fail(B2C_ERR_INVALID, "b2c_transform_u8: crop larger than the datum");
  if (mean_values && mean_image) return fail(B2C_ERR_INVALID, "b2c_transform_u8: Cannot specify mean_file and mean_value at the same time");
  int dev_count = 0;
  if (cudaGetDeviceCount(&dev_count) != cudaSuccess || dev_count == 0) return fail(B2C_ERR_CUDA, "no CUDA device: this library has no CPU fallback");
  const size_t units = (size_t)N * C * crop_h * ((crop_w + 3) / 4);
  launch_pdl(transform_u8_kernel, grid_for(units, 256), 256, 0, as_stream(stream), 0, src, N, C, Hd, Wd, crop_h, crop_w, h_off, w_off, mirror, mean_values,
                                                                         mean_image, scale, dst);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
