// fake_kernels_solvers.cpp -- host stand-in for b2c_solver_update_arena (the Nesterov, AdaGrad, RMSProp, AdaDelta and Adam updates
// over the parameter arena), enqueued on tests/sim/fake_cuda.cpp's streams like the real launch.  Linked into libsolversim.so
// (Makefile.solvers) so that TrainNet::Step with every solver type runs end to end on the stream-order model
// (tests/test_solvers_sim.py).  TEST INFRASTRUCTURE ONLY: fp32 loops written from the per-element rules of include/b2c.h; the
// real kernel is checked against the oracle on hardware (tests/test_solvers_gpu.py).
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <functional>
#include <vector>

#include "../../include/b2c.h"

void fakecuda_launch(cudaStream_t st, std::function<void()> fn);

extern "C" int b2c_solver_update_arena(int kind, int nseg, const size_t* offset, const size_t* count, const float* local_rate,
                                       const float* local_decay, float* g, float* w, float* h, float* h2, b2c_solver_hparams hp, int l2,
                                       float grad_scale, int clear_grads, void* stream) {
  if (kind < B2C_SOLVER_SGD || kind > B2C_SOLVER_ADAM || ((kind == B2C_SOLVER_ADADELTA || kind == B2C_SOLVER_ADAM) && !h2)) return B2C_ERR_INVALID;
  std::vector<size_t> off(offset, offset + nseg), cnt(count, count + nseg);
  std::vector<float> rate(local_rate, local_rate + nseg), decay(local_decay, local_decay + nseg);
  const float d3 = std::max(hp.delta, 1e-3f), d4 = std::max(hp.delta, 1e-4f), m = hp.momentum;
  fakecuda_launch(static_cast<cudaStream_t>(stream), [=] {
    for (int s = 0; s < nseg; ++s)
      for (size_t i = off[s]; i < off[s] + cnt[s]; ++i) {
        const float reg = l2 ? w[i] : (w[i] > 0.f ? 1.f : w[i] < 0.f ? -1.f : 0.f);
        float gr = g[i] * grad_scale + decay[s] * reg, u = 0.f;
        const float lr = rate[s];
        switch (kind) {
          case B2C_SOLVER_SGD: h[i] = m * h[i] + lr * gr; u = h[i]; break;
          case B2C_SOLVER_NESTEROV: { const float hp0 = h[i]; h[i] = m * hp0 + lr * gr; u = (1.f + m) * h[i] - m * hp0; break; }
          case B2C_SOLVER_ADAGRAD: h[i] += gr * gr; u = lr * gr / (std::sqrt(h[i]) + d3); break;
          case B2C_SOLVER_RMSPROP: h[i] = hp.rms_decay * h[i] + (1.f - hp.rms_decay) * gr * gr; u = lr * gr / (std::sqrt(h[i]) + d4); break;
          case B2C_SOLVER_ADADELTA:
            h[i] = m * h[i] + (1.f - m) * gr * gr;
            gr *= std::sqrt((h2[i] + d3) / (h[i] + d3));
            h2[i] = m * h2[i] + (1.f - m) * gr * gr;
            u = lr * gr;
            break;
          default:
            h[i] = hp.beta1 * h[i] + (1.f - hp.beta1) * gr;
            h2[i] = hp.beta2 * h2[i] + (1.f - hp.beta2) * gr * gr;
            u = lr * h[i] / (std::sqrt(h2[i]) + d4);
        }
        w[i] -= u;
        g[i] = clear_grads ? 0.f : u;
      }
  });
  return B2C_OK;
}
