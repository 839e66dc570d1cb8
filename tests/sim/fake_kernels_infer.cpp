// fake_kernels_infer.cpp -- host stand-in for b2c_bn_forward_inference (BatchNorm in the TEST phase), written from its contract in
// include/b2c.h and enqueued on tests/sim/fake_cuda.cpp's streams like the real launch.  Linked with the other stand-ins into
// libinfersim.so (Makefile.infer), on which a TEST-phase TrainNet runs its forward on the CPU and is held against
// tests/infer_oracle.py (tests/test_infer_cpu.py).  TEST INFRASTRUCTURE ONLY; the real kernel is checked on hardware
// (tests/test_infer_gpu.py).
#include <cuda_runtime.h>

#include <cmath>
#include <functional>

#include "../../include/b2c.h"

void fakecuda_launch(cudaStream_t st, std::function<void()> fn);

// y = [relu]((x - mean) * 1/sqrt(running_var + eps) [* gamma + beta] [+ residual]); y may alias x
extern "C" int b2c_bn_forward_inference(int N, int C, int Sp, const float* x, const float* gamma, const float* beta, float eps,
                                        const float* run_mean, const float* run_var, const float* residual, float* y, int relu, void* stream) {
  fakecuda_launch(static_cast<cudaStream_t>(stream), [=] {
    for (int n = 0; n < N; ++n)
      for (int c = 0; c < C; ++c) {
        const float is = 1.0f / std::sqrt(run_var[c] + eps);
        for (int i = 0; i < Sp; ++i) {
          const size_t at = ((size_t)n * C + c) * Sp + i;
          float v = (x[at] - run_mean[c]) * is;
          if (gamma) v = (float)((double)v * gamma[c] + beta[c]);
          if (residual) v += residual[at];
          y[at] = relu && !(v > 0.f) ? 0.f : v;
        }
      }
  });
  return B2C_OK;
}
