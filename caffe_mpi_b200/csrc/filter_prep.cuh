// filter_prep.cuh -- the filter operand of the tensor-core forward / dgrad kernels in its GEMM layout, as ONE multi-tensor launch.
//
// Both kernels read the filter through TMA as a [rows][Kp] matrix in GEMM-K order, pre-split into hi / lo parts:
//   kind GATHER (conv_tc.cu)     fp32 TF32-hi / lo planes [G][rows][Kp], K = (c,i,j) natural or (c/4, tap, c%4) "tap major"
//   kind STAGED (conv_tc_stg.cu) bf16 hi / lo planes [rows][Kp], K = (channel group of 32, tap, channel in group)
// mode 0 (forward): row = o, K channel = c;  mode 1 (dgrad): row = c, K channel = o (taps flipped when `flip`).
// mode 2 (one phase of a strided transposed convolution, deconv.cu): as mode 1, over the phase's sub_kh x sub_kw taps; sub-filter
// tap (a, b) reads filter tap (i0h + (sub_kh-1-a)*Lh, i0w + (sub_kw-1-b)*Lw) of the full src_kw-wide, src_taps-tap filter.
// Weights change once per iteration, so the host layer prepares every layer's filters once per iteration with
// b2c_conv_prepare_filters (chained after the SGD update) instead of once per forward and once per dgrad call
// (105 launches of ~8 us per ResNet-50 step in round 1, 0.85 ms).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b2c {

struct PrepEntry {
  const float* w;        // [G*Og][Cg][taps]
  void* hi;
  void* lo;              // null: single plane of round-to-nearest TF32 (GATHER, TF32 math mode)
  long long total;       // elements of one plane
  int kind;              // 0 GATHER, 1 STAGED
  int G, Og, Cg, taps, rows, K, Kp, mode, tap_major, flip, kch;
  int src_taps, src_kw, sub_kh, sub_kw, i0h, i0w, Lh, Lw;   // mode 2 only
};
constexpr int PREP_BATCH = 24;
struct PrepBatch { PrepEntry e[PREP_BATCH]; };

// enqueue the prepass for n entries (ceil(n / PREP_BATCH) launches)
int launch_filter_prep(const PrepEntry* entries, int n, cudaStream_t st);

}  // namespace b2c
