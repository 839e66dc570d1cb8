// fake_kernels_clip.cpp -- host stand-ins for the clip_gradients entry points (b2c_arena_sumsq, b2c_clip_factor,
// b2c_solver_update_arena_scaled), enqueued on tests/sim/fake_cuda.cpp's streams like the real launches.  Linked into libclipsim.so
// (Makefile.clip) with fake_kernels_solvers.cpp so that TrainNet::Step with clipping runs end to end on the stream-order model
// (tests/test_clip_sim.py).  TEST INFRASTRUCTURE ONLY: the norm keeps the kernels' structure -- one double partial per 4096-element
// block of each segment, the partials summed in slot order -- so it does not depend on the bucket plan; the arithmetic inside a
// block is a plain ordered sum.  The update is fake_kernels_solvers.cpp's rule with grad_scale * factor read when the launch runs.
// The real kernels are checked against the oracle on hardware (tests/test_clip_gpu.py).
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <functional>
#include <vector>

#include "../../include/b2c.h"

void fakecuda_launch(cudaStream_t st, std::function<void()> fn);
static cudaStream_t S(void* s) { return static_cast<cudaStream_t>(s); }

extern "C" {

int b2c_arena_sumsq(int nseg, const size_t* offset, const size_t* count, const size_t* slot, const float* g, double* partials,
                    void* stream) {
  if (nseg < 0 || (nseg && (!offset || !count || !slot || !g || !partials))) return B2C_ERR_INVALID;
  std::vector<size_t> off(offset, offset + nseg), cnt(count, count + nseg), sl(slot, slot + nseg);
  fakecuda_launch(S(stream), [=] {
    for (int s = 0; s < nseg; ++s)
      for (size_t b = 0; b * B2C_SUMSQ_BLOCK_ELEMS < cnt[s]; ++b) {
        double acc = 0.0;
        const size_t end = std::min(cnt[s], (b + 1) * B2C_SUMSQ_BLOCK_ELEMS);
        for (size_t i = b * B2C_SUMSQ_BLOCK_ELEMS; i < end; ++i) acc += (double)g[off[s] + i] * (double)g[off[s] + i];
        partials[sl[s] + b] = acc;
      }
  });
  return B2C_OK;
}

int b2c_clip_factor(const double* partials, size_t nslots, double s_n, float clip, b2c_clip_state* state, void* stream) {
  if ((nslots && !partials) || !state || !(clip >= 0.f) || !(s_n > 0.0)) return B2C_ERR_INVALID;
  fakecuda_launch(S(stream), [=] {
    double sum = 0.0;
    for (size_t i = 0; i < nslots; ++i) sum += partials[i];
    const float norm = (float)std::sqrt((s_n * s_n) * sum);
    const bool clipped = norm > clip;
    state->norm = norm;
    state->factor = clipped ? clip / norm : 1.0f;
    if (clipped) state->clipped += 1;
  });
  return B2C_OK;
}

int b2c_solver_update_arena_scaled(int kind, int nseg, const size_t* offset, const size_t* count, const float* local_rate,
                                   const float* local_decay, float* g, float* w, float* h, float* h2, b2c_solver_hparams hp, int l2,
                                   float grad_scale, const float* factor, int clear_grads, void* stream) {
  if (kind < B2C_SOLVER_SGD || kind > B2C_SOLVER_ADAM || ((kind == B2C_SOLVER_ADADELTA || kind == B2C_SOLVER_ADAM) && !h2) || !factor)
    return B2C_ERR_INVALID;
  std::vector<size_t> off(offset, offset + nseg), cnt(count, count + nseg);
  std::vector<float> rate(local_rate, local_rate + nseg), decay(local_decay, local_decay + nseg);
  const float d3 = std::max(hp.delta, 1e-3f), d4 = std::max(hp.delta, 1e-4f), m = hp.momentum;
  fakecuda_launch(S(stream), [=] {
    const float gs = grad_scale * *factor;
    for (int s = 0; s < nseg; ++s)
      for (size_t i = off[s]; i < off[s] + cnt[s]; ++i) {
        const float reg = l2 ? w[i] : (w[i] > 0.f ? 1.f : w[i] < 0.f ? -1.f : 0.f);
        float gr = g[i] * gs + decay[s] * reg, u = 0.f;
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

}  // extern "C"
