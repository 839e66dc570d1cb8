// conv_tc_wgrad.cu -- wgmma implicit-GEMM weight-gradient kernels (sm_90a).
//
// Replaces cudnnConvolutionBackwardFilter beta=1 (reference src/caffe/layers/cudnn_conv_layer.cu:95-99)
// and, semantically, the per-image weight_gpu_gemm loop (base_conv_layer.hpp:148-162):
//     dW[o][k'=(c,i,j)] += sum_{q=(n,ho,wo)} dY[n,o,ho,wo] * X[n,c,ho*s-p+i*d,wo*s-p+j*d]
// GEMM view: M = output channels of one group (tile 128), N = K_dim = (C/g)*kh*kw (tile N_TILE), the
// reduction runs over q = N*Ho*Wo, which is the CONTIGUOUS axis of both operands in NCHW memory, so both
// smem tiles are filled "lanes along K": dY with 128-bit loads, X through the im2col gather.  Two consumer
// warpgroups (warps 0-7) issue wgmma from the two tiles and keep the fp32 accumulators in registers.  The
// reduction is split across CTAs (grid.x); partial tiles go to a workspace and the tile's CTAs then add them
// to dW in split order (splitk_fused_reduce; the reference accumulates image by image, also a fixed order).
#include <stdio.h>
#include "b2c_common.cuh"
#include "tc_common.cuh"

namespace b2c {
using namespace tc;

constexpr int NCONS = 8;                        // consumer warps: two warpgroups (wgmma + epilogue), tile rows [64 cw, 64 cw + 64)
constexpr int WG_YW = 8;                        // dY producer warps
constexpr int WG_GW = 8;                        // X-gather producer warps
constexpr int WG_THREADS = (NCONS + WG_YW + WG_GW) * 32;   // 768

struct WgradParams {
  const float* dy;   // [N, O, Ho, Wo]
  const float* x;    // [N, C, H, W]
  int N, C, H, W, O, Cg, Og, Kd;
  int kh, kw, sh, sw, ph, pw, dh, dw, Ho, Wo;
  long long Q;       // N*Ho*Wo
  int kb_per_split;  // k-blocks (of 32 q) per split
  int splits;
  float* out;        // splits == 1: dW (accumulated);  else partials [splits][O*Kd] (overwritten)
  float* grad;       // splits > 1: the gradient blob the fused reduction accumulates into
  unsigned int* counters;   // splits > 1: one zeroed arrival counter per output tile
  long long* prof;   // optional cycle counters from CTA (0,0,0) (B2C_PROF=1)
};

template <int N_TILE, bool SPLIT>
struct WgradSmem {
  static constexpr uint32_t A_BYTES = tile_bytes(128);
  static constexpr uint32_t B_BYTES = tile_bytes(N_TILE);
  static constexpr uint32_t STAGE = (SPLIT ? 2u : 1u) * (A_BYTES + B_BYTES);
  static constexpr uint32_t TABLE = N_TILE * 8u;
  static constexpr uint32_t PROM_BYTES = NCONS * 32u * (N_TILE / 2) * 4u;   // the consumers' promoted accumulators
  static constexpr int STAGES_ = (int)((216u * 1024u - PROM_BYTES) / STAGE);
  static constexpr int STAGES = STAGES_ > 6 ? 6 : STAGES_;
  static constexpr uint32_t BAR_OFF = STAGES * STAGE;
  static constexpr uint32_t TAB_OFF = BAR_OFF + 256;
  static constexpr uint32_t PROM_OFF = TAB_OFF + TABLE;
  static constexpr uint32_t TOTAL = PROM_OFF + PROM_BYTES;
};

template <int N_TILE, bool SPLIT, bool X1X1>
__global__ void __launch_bounds__(WG_THREADS, 1)
igemm_wgrad_kernel(const __grid_constant__ WgradParams p) {
  using S = WgradSmem<N_TILE, SPLIT>;
  using MMA = WgmmaTf32<N_TILE>;
  constexpr int STAGES = S::STAGES;
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bar_full = sbase + S::BAR_OFF;
  const uint32_t bar_empty = bar_full + 8 * STAGES;
  int2* rowtab = reinterpret_cast<int2*>(smem + S::TAB_OFF);   // per B row: {channel offset, hoff | woff<<16}

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int split = blockIdx.x;
  const int n0 = blockIdx.y * N_TILE;                 // k' tile
  const int mtiles = (p.Og + 127) / 128;
  const int g = blockIdx.z / mtiles, m0 = (blockIdx.z % mtiles) * 128;
  const int P = p.Ho * p.Wo;
  const long long HW = (long long)p.H * p.W;
  const long long nkb_total = (p.Q + BK - 1) / BK;
  const long long kb_begin = (long long)split * p.kb_per_split;
  long long kb_end = kb_begin + p.kb_per_split;
  if (kb_end > nkb_total) kb_end = nkb_total;
  const int nkb = (int)(kb_end - kb_begin);           // >= 1 by construction

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(bar_full + 8 * s, WG_YW + WG_GW); mbar_init(bar_empty + 8 * s, NCONS); }   // one elected arrive per producer / consumer warp
    fence_barrier_init();
  }
  // row table for the X gather: k' = (c,i,j)
  for (int r = tid; r < N_TILE; r += WG_THREADS) {
    const int kp = n0 + r;
    int2 e = make_int2(-1, 0);
    if (kp < p.Kd) {
      const int j = kp % p.kw, i = (kp / p.kw) % p.kh, c = kp / (p.kw * p.kh);
      e.x = (int)(((long long)g * p.Cg + c) * HW);      // channel offset inside one image (C*H*W < 2^31)
      e.y = (i * p.dh) | ((j * p.dw) << 16);
    }
    rowtab[r] = e;
  }
  __syncthreads();
  pdl_wait();      // everything above is shared-memory and barrier set-up

  constexpr uint32_t LBO_A = tile_lbo(128), LBO_B = tile_lbo(N_TILE);
  auto stage_a_hi = [&](int s) { return sbase + s * S::STAGE; };
  auto stage_a_lo = [&](int s) { return sbase + s * S::STAGE + S::A_BYTES; };
  auto stage_b_hi = [&](int s) { return sbase + s * S::STAGE + (SPLIT ? 2u : 1u) * S::A_BYTES; };
  auto stage_b_lo = [&](int s) { return stage_b_hi(s) + S::B_BYTES; };

  if (warp >= NCONS && warp < NCONS + WG_YW) {
    // ================= A producer: dY rows (output channels), lanes along q ==========================
    const int ytid = tid - NCONS * 32;
    const int kc = ytid & 7, rb = ytid >> 3;            // rb in [0, 32): rows r*32 + rb, r < 4
    const bool vec_ok = (P % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.dy) & 15u) == 0);
    // loads of k-block kb+1 are issued before the stores of k-block kb (register double buffer)
    // q = n*P + p of this thread's first element; advanced by BK per K block with 32-bit arithmetic only
    // (the 64-bit q / P per block made the load phase ~2000 cycles)
    int cur_n, cur_p;
    {
      const long long q0 = kb_begin * BK + kc * 4;
      cur_n = (int)(q0 / P); cur_p = (int)(q0 - (long long)cur_n * P);
    }
    auto load_block = [&](int /*kb*/, float (&v)[16]) {
      int nn[4], pp[4];
      bool qv[4];
      {
        int n_ = cur_n, p_ = cur_p;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          qv[e] = n_ < p.N;
          nn[e] = n_; pp[e] = p_;
          if (++p_ == P) { p_ = 0; ++n_; }
        }
        cur_p += BK;
        while (cur_p >= P) { cur_p -= P; ++cur_n; }
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int o = m0 + r * 32 + rb;
        float* vv = v + r * 4;
        vv[0] = vv[1] = vv[2] = vv[3] = 0.f;
        if (o < p.Og) {
          const long long ch = (long long)g * p.Og + o;
          if (vec_ok && qv[3] && nn[3] == nn[0]) {
            const float4 t4 = __ldg(reinterpret_cast<const float4*>(p.dy + ((long long)nn[0] * p.O + ch) * P + pp[0]));
            vv[0] = t4.x; vv[1] = t4.y; vv[2] = t4.z; vv[3] = t4.w;
          } else {
#pragma unroll
            for (int e = 0; e < 4; ++e)
              if (qv[e]) vv[e] = __ldg(p.dy + ((long long)nn[e] * p.O + ch) * P + pp[e]);
          }
        }
      }
    };
    long long pa_wait = 0, pa_store = 0;
    const long long pa_t0 = clock64();
    auto store_block = [&](int kb, const float (&v)[16]) {
      const int s = kb % STAGES, it = kb / STAGES;
      const long long w0 = clock64();
      mbar_wait_backoff(bar_empty + 8 * s, (it & 1) ^ 1, 40);
      const long long w1 = clock64();
      pa_wait += w1 - w0;
      const uint32_t a_hi = stage_a_hi(s) + kc * LBO_A, a_lo = stage_a_lo(s) + kc * LBO_A;
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int row = r * 32 + rb;
        store_chunk<SPLIT>(a_hi + row * 16, a_lo + row * 16, v[r * 4], v[r * 4 + 1], v[r * 4 + 2], v[r * 4 + 3]);
      }
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_full + 8 * s);
      pa_store += clock64() - w1;
    };
    {
      float va[16], vb[16];
      load_block(0, va);
      int kb = 0;
      for (; kb + 2 <= nkb; kb += 2) {
        load_block(kb + 1, vb);
        store_block(kb, va);
        if (kb + 2 < nkb) load_block(kb + 2, va);
        store_block(kb + 1, vb);
      }
      if (kb < nkb) store_block(kb, va);
    }
    if (p.prof && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && ytid == 0) {
      p.prof[0] = clock64() - pa_t0; p.prof[1] = pa_wait; p.prof[2] = pa_store; p.prof[5] = nkb;
    }
  } else if (warp >= NCONS + WG_YW) {
    // ================= B producer: im2col gather of X, rows k'=(c,i,j), lanes along q ==================
    const int t = tid - (NCONS + WG_YW) * 32;
    const int kc = t & 7, rb = t >> 3;                 // rb in [0, 32): rows r*32 + rb, r < N_TILE / 32
    const bool vec_ok = X1X1 && (P % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.x) & 15u) == 0);
    constexpr int RB = N_TILE / 32;
    const bool row_active = true;
    int cur_n, cur_ho, cur_wo;
    {
      const long long q0 = kb_begin * BK + kc * 4;
      cur_n = (int)(q0 / P);
      const int p0 = (int)(q0 - (long long)cur_n * P);
      cur_ho = p0 / p.Wo; cur_wo = p0 - cur_ho * p.Wo;
    }
    const long long img = (long long)p.C * HW;
    auto load_block = [&](int /*kb*/, float (&v)[RB * 4]) {
      long long base[4];
      int ihb[4], iwb[4];
      bool qv[4];
      {
        int n_ = cur_n, ho = cur_ho, wo = cur_wo;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          qv[e] = n_ < p.N;
          base[e] = n_ * img;
          ihb[e] = ho * p.sh - p.ph; iwb[e] = wo * p.sw - p.pw;
          if (++wo == p.Wo) { wo = 0; if (++ho == p.Ho) { ho = 0; ++n_; } }
        }
        // advance the cursor by BK pixels (32-bit divisions only)
        int w2 = cur_wo + BK;
        const int dh = w2 / p.Wo;
        cur_wo = w2 - dh * p.Wo;
        int h2 = cur_ho + dh;
        const int dn = h2 / p.Ho;
        cur_ho = h2 - dn * p.Ho;
        cur_n += dn;
      }
#pragma unroll
      for (int r = 0; r < RB; ++r) {
        float* vv = v + r * 4;
        vv[0] = vv[1] = vv[2] = vv[3] = 0.f;
        if (!row_active) continue;
        const int2 rt = rowtab[r * 32 + rb];
        if (rt.x >= 0) {
          if (X1X1) {
            // k=1, s=1, p=0: X rows are contiguous in q exactly like dY
            if (vec_ok && qv[3] && base[3] == base[0]) {
              const float4 t4 = __ldg(reinterpret_cast<const float4*>(p.x + base[0] + rt.x + (long long)ihb[0] * p.W + iwb[0]));
              vv[0] = t4.x; vv[1] = t4.y; vv[2] = t4.z; vv[3] = t4.w;
            } else {
#pragma unroll
              for (int e = 0; e < 4; ++e)
                if (qv[e]) vv[e] = __ldg(p.x + base[e] + rt.x + (long long)ihb[e] * p.W + iwb[e]);
            }
          } else {
            const int hoff = rt.y & 0xffff, woff = rt.y >> 16;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const int ih = ihb[e] + hoff, iw = iwb[e] + woff;
              if (qv[e] && (unsigned)ih < (unsigned)p.H && (unsigned)iw < (unsigned)p.W)
                v[r * 4 + e] = __ldg(p.x + base[e] + rt.x + ih * p.W + iw);
            }
          }
        }
      }
    };
    long long pb_wait = 0, pb_store = 0;
    const long long pb_t0 = clock64();
    auto store_block = [&](int kb, const float (&v)[RB * 4]) {
      const int s = kb % STAGES, it = kb / STAGES;
      const long long w0 = clock64();
      mbar_wait_backoff(bar_empty + 8 * s, (it & 1) ^ 1, 40);
      const long long w1 = clock64();
      pb_wait += w1 - w0;
      const uint32_t b_hi = stage_b_hi(s) + kc * LBO_B, b_lo = stage_b_lo(s) + kc * LBO_B;
      if (row_active) {
#pragma unroll
        for (int r = 0; r < RB; ++r) {
          const int row = r * 32 + rb;
          store_chunk<SPLIT>(b_hi + row * 16, b_lo + row * 16, v[r * 4], v[r * 4 + 1], v[r * 4 + 2], v[r * 4 + 3]);
        }
      }
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_full + 8 * s);
      pb_store += clock64() - w1;
    };
    {
      float va[RB * 4], vb[RB * 4];
      load_block(0, va);
      int kb = 0;
      for (; kb + 2 <= nkb; kb += 2) {
        load_block(kb + 1, vb);
        store_block(kb, va);
        if (kb + 2 < nkb) load_block(kb + 2, va);
        store_block(kb + 1, vb);
      }
      if (kb < nkb) store_block(kb, va);
    }
    if (p.prof && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && t == 0) {  // first X-gather thread
      p.prof[8] = clock64() - pb_t0; p.prof[9] = pb_wait; p.prof[10] = pb_store;
    }
  } else if (warp < NCONS) {
    // ================= consumers: wgmma over the CTA's K range, then the partial tile from registers =================
    // Every PROMOTE K blocks (512 pixels) the wgmma accumulator is added into a promoted sum on the CUDA cores and restarted.
    // Accumulating a whole split in the wgmma accumulator measured outside the 3e-4 dW bar of test_full_size_vs_reference_loop
    // on an H100 where the one-wave split plan leaves each CTA a long reduction: AlexNet conv2 (g = 2, N = 256) 4.3e-4, conv3
    // 3.1e-4 (43k pixels per CTA); with the promotion both pass.
    // The promoted sum lives in shared memory, element i of consumer thread tid at prom[i * 256 + tid] (conflict-free): the
    // 80 registers a thread of this 768-thread kernel has hold the wgmma accumulators, not a second copy of them.
    constexpr int PROMOTE = 16;
    const int cw = warp >> 2, t = tid & 127;
    float acc[N_TILE / 2];
    float* prom = reinterpret_cast<float*>(smem + S::PROM_OFF) + tid;
#pragma unroll
    for (int i = 0; i < N_TILE / 2; ++i) prom[i * NCONS * 32] = 0.f;
    int prev = -1;
    // chunks of PROMOTE K blocks: the wait for the whole chunk's MMAs is unconditional (a wgmma wait under a data-dependent
    // branch makes ptxas serialize every wgmma of the kernel)
    for (int kb0 = 0; kb0 < nkb; kb0 += PROMOTE) {
      const int kend = min(nkb, kb0 + PROMOTE);
      for (int kb = kb0; kb < kend; ++kb) {
        const int s = kb % STAGES, it = kb / STAGES;
        mbar_wait(bar_full + 8 * s, it & 1);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < BK / 8; ++kk) {
          const uint32_t a = stage_a_hi(s) + 2u * kk * LBO_A + (uint32_t)cw * 1024u;
          const uint64_t ah = smem_desc(a, LBO_A, 128);
          const uint64_t bh = smem_desc(stage_b_hi(s) + 2 * kk * LBO_B, LBO_B, 128);
          if (SPLIT) {
            const uint64_t al = smem_desc(stage_a_lo(s) + 2u * kk * LBO_A + (uint32_t)cw * 1024u, LBO_A, 128);
            const uint64_t bl = smem_desc(stage_b_lo(s) + 2 * kk * LBO_B, LBO_B, 128);
            MMA::mma(acc, al, bh, kb != kb0 || kk != 0);
            MMA::mma(acc, ah, bl, 1);
            MMA::mma(acc, ah, bh, 1);
          } else {
            MMA::mma(acc, ah, bh, kb != kb0 || kk != 0);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(bar_empty + 8 * prev); }
        prev = s;
      }
      wgmma_wait<0>();
      wgmma_reg_fence(acc);
#pragma unroll
      for (int i = 0; i < N_TILE / 2; ++i) prom[i * NCONS * 32] += acc[i];
    }
    // row = output channel, column = k'; lanes of a quad write 8 consecutive columns of a row
    const bool accumulate = p.splits == 1;
#pragma unroll
    for (int i = 0; i < N_TILE / 2; ++i) {
      const int r = m0 + cw * 64 + frag_row(t, i), c = n0 + frag_col(t, i);
      if (r < p.Og && c < p.Kd) {
        float* dst = p.out + (p.splits > 1 ? (long long)split * p.O * p.Kd : 0LL) + ((long long)g * p.Og + r) * p.Kd + c;
        const float v = prom[i * NCONS * 32];
        *dst = accumulate ? *dst + v : v;
      }
    }
  }
  if (p.splits > 1) {
    const int tile_id = blockIdx.z * gridDim.y + blockIdx.y;
    splitk_fused_reduce(p.out, p.grad, p.counters + tile_id, split, p.splits, (long long)p.O * p.Kd,
                        ((long long)g * p.Og + m0) * p.Kd + n0, p.Kd, min(128, p.Og - m0), min(N_TILE, p.Kd - n0));
  }
}

// =====================================================================================================================
// 1x1 / stride 1 / pad 0 layers (24 of ResNet-50's 53): per image both operands are plain row-major matrices with the
// reduction axis q = (ho,wo) contiguous -- dY[n] is [O x P], X[n] is [C x P] -- so neither needs a gather:
//   * one elected thread drops [128 x 32] (dY) and [N_TILE x 32] (X) fp32 boxes into shared memory with TMA
//     (3-D tensor maps {P, rows, N}, SWIZZLE_128B = a canonical K-major wgmma layout; rows past O / C and columns
//     past P are zero-filled by the TMA unit, which is exactly the padding the GEMM needs);
//   * the RAW tile is the TF32 "hi" operand as it stands: the tf32 MMA reads the top 19 bits of each fp32 word, i.e.
//     a & 0xffffe000 -- the same truncation split_tf32() applies in software;
//   * 8 converter warps produce the "lo" tiles, lo = a - (a & 0xffffe000), position by position (the copy is
//     layout-agnostic: same swizzled offset in a second buffer), 12 x (LDS.128 + 8 ALU + STS.128) per thread and K block;
//   * two consumer warpgroups issue lo*hi + hi*lo + hi*hi from shared-memory descriptors as in the gather kernel.
// K blocks are enumerated per image (ceil(P/32) chunks, the last one zero padded) and split across CTAs in one wave.
// fp32-equivalent math only: single-pass TF32 mode needs round-to-nearest operands and keeps the gather kernel.
constexpr int WT_CW = 8;                               // converter warps
constexpr int WT_THREADS = (NCONS + WT_CW + 1) * 32;   // consumers + converters + TMA warp = 544

struct WgradTmaParams {
  int O, C;              // rows of dY / X per image (G = 1)
  int cpi;               // K chunks of 32 per image = ceil(P / 32)
  long long nkb_total;   // N * cpi
  int kb_per_split, splits;
  float* out;            // splits == 1: dW (accumulated);  else partials [splits][O*C] (overwritten)
  float* grad;           // splits > 1: the gradient blob the fused reduction accumulates into
  unsigned int* counters;   // splits > 1: one zeroed arrival counter per output tile
};

template <int N_TILE>
struct WgradTmaSmem {
  static constexpr uint32_t A_BYTES = 128u * 128u;                     // [128 rows][32 fp32], SW128
  static constexpr uint32_t B_BYTES = (uint32_t)N_TILE * 128u;
  static constexpr uint32_t RAW_BYTES = A_BYTES + B_BYTES;             // one TMA transaction pair
  static constexpr uint32_t STAGE = 2u * RAW_BYTES;                    // raw (= hi) tiles, then lo tiles at +RAW_BYTES
  static constexpr int STAGES_ = (int)((208u * 1024u) / STAGE);
  static constexpr int STAGES = STAGES_ > 6 ? 6 : STAGES_;
  static constexpr uint32_t BAR_OFF = STAGES * STAGE;
  static constexpr uint32_t TOTAL = BAR_OFF + 256 + 1024;              // + 1024-byte alignment slack
};

template <int N_TILE>
__global__ void __launch_bounds__(WT_THREADS, 1)
wgrad1x1_tma_kernel(const __grid_constant__ WgradTmaParams p, const __grid_constant__ CUtensorMap map_dy,
                    const __grid_constant__ CUtensorMap map_x) {
  using S = WgradTmaSmem<N_TILE>;
  using MMA = WgmmaTf32<N_TILE>;
  constexpr int STAGES = S::STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;        // SW128 tiles need 1024-byte alignment
  uint8_t* sptr = smem_raw + (sbase - smem_u32(smem_raw));
  const uint32_t bar_raw = sbase + S::BAR_OFF;                         // TMA bytes have landed
  const uint32_t bar_full = bar_raw + 8 * STAGES;                      // lo tiles written
  const uint32_t bar_empty = bar_full + 8 * STAGES;                    // MMAs of the stage have completed

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int split = blockIdx.x;
  const int n0 = blockIdx.y * N_TILE;                                   // input-channel tile (GEMM N)
  const int m0 = blockIdx.z * 128;                                      // output-channel tile (GEMM M)
  const long long kb_begin = (long long)split * p.kb_per_split;
  long long kb_end = kb_begin + p.kb_per_split;
  if (kb_end > p.nkb_total) kb_end = p.nkb_total;
  const int nkb = (int)(kb_end - kb_begin);                             // >= 1 by construction

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(bar_raw + 8 * s, 1);
      mbar_init(bar_full + 8 * s, WT_CW);
      mbar_init(bar_empty + 8 * s, NCONS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();      // everything above is shared-memory and barrier set-up

  auto stage_a = [&](int s) { return sbase + (uint32_t)s * S::STAGE; };            // raw dY tile (hi operand)
  auto stage_b = [&](int s) { return sbase + (uint32_t)s * S::STAGE + S::A_BYTES; };  // raw X tile

  if (warp >= NCONS && warp < NCONS + WT_CW) {
    // ================= converters: lo = a - trunc_tf32(a), same offset in the lo half of the stage =============
    constexpr int UNITS = (int)(S::RAW_BYTES / 16u);                   // 16-byte units per stage, multiple of 256
    for (int kb = 0; kb < nkb; ++kb) {
      const int s = kb % STAGES, it = kb / STAGES;
      mbar_wait_backoff(bar_raw + 8 * s, it & 1, 20);
      const uint32_t src = stage_a(s);
#pragma unroll 4
      for (int u = tid - NCONS * 32; u < UNITS; u += WT_CW * 32) {
        const float4 v = lds128(src + (uint32_t)u * 16u);
        float h, l0, l1, l2, l3;
        split_tf32(v.x, h, l0); split_tf32(v.y, h, l1); split_tf32(v.z, h, l2); split_tf32(v.w, h, l3);
        sts128(src + S::RAW_BYTES + (uint32_t)u * 16u, l0, l1, l2, l3);
      }
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_full + 8 * s);
    }
  } else if (warp == NCONS + WT_CW) {
    // ================= TMA producer (whole warp converged, one elected lane issues) ============================
    int n = (int)(kb_begin / p.cpi), j = (int)(kb_begin - (long long)n * p.cpi);
    for (int kb = 0; kb < nkb; ++kb) {
      const int s = kb % STAGES, it = kb / STAGES;
      mbar_wait_backoff(bar_empty + 8 * s, (it & 1) ^ 1, 20);
      if (elect_one()) {
        arrive_expect_tx(bar_raw + 8 * s, S::RAW_BYTES);
        tma_load_3d(stage_a(s), &map_dy, bar_raw + 8 * s, j * 32, m0, n);
        tma_load_3d(stage_b(s), &map_x, bar_raw + 8 * s, j * 32, n0, n);
      }
      __syncwarp();
      if (++j == p.cpi) { j = 0; ++n; }
    }
  } else if (warp < NCONS) {
    // ================= consumers: wgmma over the CTA's K range, then the partial tile from registers =================
    const int cw = warp >> 2, t = tid & 127;
    float acc[N_TILE / 2];
    int prev = -1;
    for (int kb = 0; kb < nkb; ++kb) {
      const int s = kb % STAGES, it = kb / STAGES;
      mbar_wait(bar_full + 8 * s, it & 1);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BK / 8; ++kk) {
        const uint32_t a = stage_a(s) + (uint32_t)cw * 8192u + kk * 32;     // rows [64 cw, 64 cw + 64): 8 groups of 8 rows x 128 B
        const uint64_t ah = smem_desc_sw128(a), al = smem_desc_sw128(a + S::RAW_BYTES);
        const uint64_t bh = smem_desc_sw128(stage_b(s) + kk * 32), bl = smem_desc_sw128(stage_b(s) + S::RAW_BYTES + kk * 32);
        MMA::mma(acc, al, bh, (kb | kk) != 0);
        MMA::mma(acc, ah, bl, 1);
        MMA::mma(acc, ah, bh, 1);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(bar_empty + 8 * prev); }
      prev = s;
    }
    wgmma_wait<0>();
    wgmma_reg_fence(acc);
    // row = output channel, column = k'; lanes of a quad write 8 consecutive columns of a row
    const bool accumulate = p.splits == 1;
#pragma unroll
    for (int i = 0; i < N_TILE / 2; ++i) {
      const int r = m0 + cw * 64 + frag_row(t, i), c = n0 + frag_col(t, i);
      if (r < p.O && c < p.C) {
        float* dst = p.out + (p.splits > 1 ? (long long)split * p.O * p.C : 0LL) + (long long)r * p.C + c;
        *dst = accumulate ? *dst + acc[i] : acc[i];
      }
    }
  }
  if (p.splits > 1) {
    const int tile_id = blockIdx.z * gridDim.y + blockIdx.y;
    splitk_fused_reduce(p.out, p.grad, p.counters + tile_id, split, p.splits, (long long)p.O * p.C, (long long)m0 * p.C + n0, p.C,
                        min(128, p.O - m0), min(N_TILE, p.C - n0));
  }
}

struct WgradPlan { int n_tile, splits, kb_per_split; long long nkb; };

static WgradPlan wgrad_plan(const ConvShape& s) {
  WgradPlan pl;
  pl.n_tile = s.Kd > 32 ? 64 : 32;                  // 768 threads leave 80 registers: 32 accumulators per consumer thread
  const long long Q = (long long)s.N * s.Ho * s.Wo;
  pl.nkb = (Q + BK - 1) / BK;
  const long long mn = (long long)((s.Og + 127) / 128) * ((s.Kd + pl.n_tile - 1) / pl.n_tile) * s.G;
  plan_splitk(pl.nkb, mn, 8, &pl.splits, &pl.kb_per_split);
  return pl;
}

bool tc_wgrad_supported(const ConvShape& s) {
  if ((long long)s.C * s.H * s.W >= 0x7fffffffLL) return false;
  if ((s.kh - 1) * s.dh > 0xffff || (s.kw - 1) * s.dw > 0x7fff) return false;
  const long long nkb = ((long long)s.N * s.Ho * s.Wo + BK - 1) / BK;
  return nkb < 0x7fffffffLL;
}

static WgradPlan wgrad_tma_plan(const ConvShape& s, int* cpi_out);
static bool wgrad_tma_shape_ok(const ConvShape& s);
static bool wgrad_compact_shape_ok(const ConvShape& s);
static ConvShape wgrad_compact_dense_shape(const ConvShape& s);
size_t tc_wgrad_workspace(const ConvShape& s) {
  size_t need = splitk_workspace_bytes(wgrad_plan(s).splits, (long long)s.O * s.Kd);
  if (wgrad_tma_shape_ok(s)) {                       // the TMA path of 1x1 layers plans its own split count
    const size_t nt = splitk_workspace_bytes(wgrad_tma_plan(s, nullptr).splits, (long long)s.O * s.C);
    if (nt > need) need = nt;
  }
  if (wgrad_compact_shape_ok(s)) {                   // strided 1x1: compacted input + the TMA path's partials
    const ConvShape d = wgrad_compact_dense_shape(s);
    const size_t part = tc_wgrad_stg_supported(d) ? tc_wgrad_stg_workspace(d)
                                                  : splitk_workspace_bytes(wgrad_tma_plan(d, nullptr).splits, (long long)s.O * s.C);
    const size_t nt = part + 256 + sizeof(float) * (size_t)s.N * s.C * s.Ho * s.Wo;
    if (nt > need) need = nt;
  }
  return need;
}

// ---- TMA path for 1x1 layers: eligibility, plan, launch -----------------------------------------------------------
static bool wgrad_tma_enabled() {
  static const int on = env_int("B2C_WGRAD_TMA", 1);
  return on != 0;
}
static bool wgrad_tma_shape_ok(const ConvShape& s) {
  const long long P = (long long)s.Ho * s.Wo;
  return wgrad_tma_enabled() && s.is_1x1 && s.G == 1 && P % 4 == 0 && P >= 32 && s.H == s.Ho && s.W == s.Wo;
}
static WgradPlan wgrad_tma_plan(const ConvShape& s, int* cpi_out) {
  WgradPlan pl;
  pl.n_tile = s.C > 64 ? 128 : s.C > 32 ? 64 : 32;  // 128 x 128 fp32 accumulators = 64 registers per consumer thread
  const int cpi = (s.Ho * s.Wo + BK - 1) / BK;
  pl.nkb = (long long)s.N * cpi;
  const long long mn = (long long)((s.O + 127) / 128) * ((s.C + pl.n_tile - 1) / pl.n_tile);
  plan_splitk(pl.nkb, mn, 8, &pl.splits, &pl.kb_per_split);
  if (cpi_out) *cpi_out = cpi;
  return pl;
}
template <int N_TILE>
static int launch_wgrad_tma_inst(const WgradTmaParams& p, const CUtensorMap& mdy, const CUtensorMap& mx, cudaStream_t st) {
  using S = WgradTmaSmem<N_TILE>;
  // per-device attribute: set on every launch (a process may drive several GPUs)
  B2C_CUDA_OK(cudaFuncSetAttribute(wgrad1x1_tma_kernel<N_TILE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)S::TOTAL));
  dim3 grid(p.splits, (p.C + N_TILE - 1) / N_TILE, (p.O + 127) / 128);
  launch_pdl(wgrad1x1_tma_kernel<N_TILE>, grid, WT_THREADS, S::TOTAL, st, 0, p, mdy, mx);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
static int launch_conv_tc_wgrad_tma(const ConvShape& s, const float* x, const float* dy, float* dw, void* ws, size_t ws_bytes,
                                    cudaStream_t st) {
  int cpi = 0;
  const WgradPlan pl = wgrad_tma_plan(s, &cpi);
  WgradTmaParams p;
  p.O = s.O; p.C = s.C; p.cpi = cpi; p.nkb_total = (long long)s.N * cpi;
  p.kb_per_split = pl.kb_per_split; p.splits = pl.splits;
  if (int rc = bind_splitk(p, pl.splits, (long long)s.O * s.C, dw, ws, ws_bytes, st, "wgrad (tma)")) return rc;
  alignas(64) CUtensorMap mdy, mx;
  // [N][rows][P] fp32, box {32, box rows, 1}, SWIZZLE_128B
  const cuuint64_t P = (cuuint64_t)s.Ho * s.Wo;
  int rc = make_tensor_map_3d(&mdy, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, dy, {P, (cuuint64_t)s.O, (cuuint64_t)s.N}, {P * 4, P * 4 * (cuuint64_t)s.O},
                              {32, 128, 1}, CU_TENSOR_MAP_SWIZZLE_128B, "wgrad");
  if (rc) return rc;
  rc = make_tensor_map_3d(&mx, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, x, {P, (cuuint64_t)s.C, (cuuint64_t)s.N}, {P * 4, P * 4 * (cuuint64_t)s.C},
                          {32, (cuuint32_t)pl.n_tile, 1}, CU_TENSOR_MAP_SWIZZLE_128B, "wgrad");
  if (rc) return rc;
  switch (pl.n_tile) {
    case 128: return launch_wgrad_tma_inst<128>(p, mdy, mx, st);
    case 64: return launch_wgrad_tma_inst<64>(p, mdy, mx, st);
    default: return launch_wgrad_tma_inst<32>(p, mdy, mx, st);
  }
}

// ---- strided 1x1 layers (pad 0, stride > 1): subsample, then the TMA path ------------------------------------------
// On by default for layers with more than 128 output channels (B2C_WGRAD_COMPACT=0 switches it off, =2 forces it for every
// eligible layer).  On ResNet-50's strided projections the wide layers gain, while for C256->O128@56 the extra pass over X
// costs more than the gather it replaces (the GEMM is that small).  dW[o][c] = sum_q dY[o][q] * X[c][ho*sh][wo*sw]: the gather
// kernel reads X with 8-byte-strided 4-byte loads, far slower than its MMAs.  Copying the
// sampled pixels into a dense [N][C][Ho*Wo] buffer first is one HBM-bound pass over half of X's rows, after which the
// layer is an ordinary 1x1 / stride 1 weight gradient for the TMA-fed kernel.
static int wgrad_compact_mode() {
  static const int on = env_int("B2C_WGRAD_COMPACT", 1);
  return on;
}
static bool wgrad_compact_shape_ok(const ConvShape& s) {
  const long long P = (long long)s.Ho * s.Wo;
  const int mode = wgrad_compact_mode();
  if (!(mode != 0 && wgrad_tma_enabled() && s.kh == 1 && s.kw == 1 && s.ph == 0 && s.pw == 0 && (s.sh > 1 || s.sw > 1) && s.G == 1))
    return false;
  // with the staged kernel behind it the extra pass over X pays for every layer it takes; with the 3xTF32 TMA kernel only for
  // the wide ones (measurements above).  7x7 outputs (P = 49) exist only on the staged kernel (plane mode).
  const bool staged = tc_wgrad_stg_supported(wgrad_compact_dense_shape(s));
  if (!(P % 4 == 0 && P >= 32)) return staged && P == 49;
  return mode == 2 || s.O > 128 || staged;
}
static ConvShape wgrad_compact_dense_shape(const ConvShape& s) {
  ConvShape d = s;
  d.H = s.Ho; d.W = s.Wo; d.sh = d.sw = 1; d.is_1x1 = true;
  return d;
}
__global__ void __launch_bounds__(256)
subsample_kernel(const float* __restrict__ x, float* __restrict__ y, long long planes, int H, int W, int Ho, int Wo, int sh, int sw) {
  pdl_wait();
  const long long total = planes * Ho * Wo;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int wo = (int)(i % Wo);
    const long long t = i / Wo;
    const int ho = (int)(t % Ho);
    const long long pl = t / Ho;
    y[i] = __ldg(x + (pl * H + (long long)ho * sh) * W + (long long)wo * sw);
  }
}

template <int N_TILE, bool SPLIT, bool X1X1>
static int launch_wgrad_inst(const WgradParams& p, int G, cudaStream_t st) {
  using S = WgradSmem<N_TILE, SPLIT>;
  // per-device attribute: set on every launch (a process may drive several GPUs)
  B2C_CUDA_OK(cudaFuncSetAttribute(igemm_wgrad_kernel<N_TILE, SPLIT, X1X1>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)S::TOTAL));
  dim3 grid(p.splits, (p.Kd + N_TILE - 1) / N_TILE, G * ((p.Og + 127) / 128));
  launch_pdl(igemm_wgrad_kernel<N_TILE, SPLIT, X1X1>, grid, WG_THREADS, S::TOTAL, st, 0, p);
  B2C_POST_LAUNCH();
  return B2C_OK;
}

template <int N_TILE>
static int launch_wgrad_n(const WgradParams& p, int G, int math, bool x1, cudaStream_t st) {
  if (math == B2C_MATH_FP32)
    return x1 ? launch_wgrad_inst<N_TILE, true, true>(p, G, st) : launch_wgrad_inst<N_TILE, true, false>(p, G, st);
  return x1 ? launch_wgrad_inst<N_TILE, false, true>(p, G, st) : launch_wgrad_inst<N_TILE, false, false>(p, G, st);
}

// The kernel launch_conv_tc_wgrad runs, decided in one place for the launch and for b2c_debug_wgrad_plan.  x_ok / dy_ok: the
// operands are 16-byte aligned (the TMA maps need it); ws_ok: a 16-byte aligned workspace, which holds the compacted X.
int tc_wgrad_route(const ConvShape& s, int math, bool x_ok, bool dy_ok, bool ws_ok) {
  if (math == B2C_MATH_FP32 && wgrad_tma_shape_ok(s) && x_ok && dy_ok) return B2C_WGRAD_ROUTE_TMA_1X1;
  if (math == B2C_MATH_FP32 && wgrad_compact_shape_ok(s) && dy_ok && ws_ok)
    return tc_wgrad_stg_supported(wgrad_compact_dense_shape(s)) ? B2C_WGRAD_ROUTE_COMPACT_STAGED : B2C_WGRAD_ROUTE_COMPACT_TMA;
  return B2C_WGRAD_ROUTE_GATHER;
}

// the plan the planner of `route`'s kernel makes for s (compaction routes: for the dense 1x1 problem)
void tc_wgrad_plan_info(const ConvShape& s, int route, WgradPlanInfo* q) {
  *q = WgradPlanInfo{};
  const bool compact = route == B2C_WGRAD_ROUTE_COMPACT_STAGED || route == B2C_WGRAD_ROUTE_COMPACT_TMA;
  const ConvShape d = compact ? wgrad_compact_dense_shape(s) : s;
  if (route == B2C_WGRAD_ROUTE_TMA_1X1 || route == B2C_WGRAD_ROUTE_COMPACT_TMA) {
    int cpi = 0;
    const WgradPlan pl = wgrad_tma_plan(d, &cpi);
    q->splits = pl.splits; q->kb_per_split = pl.kb_per_split; q->nkb = pl.nkb; q->cols = pl.n_tile; q->bpi = cpi; q->taps = 1;
  } else if (route == B2C_WGRAD_ROUTE_GATHER) {
    const WgradPlan pl = wgrad_plan(d);
    q->splits = pl.splits; q->kb_per_split = pl.kb_per_split; q->nkb = pl.nkb; q->cols = pl.n_tile; q->taps = s.kh * s.kw;
  } else if (route != B2C_WGRAD_ROUTE_CAFFE && route != B2C_WGRAD_ROUTE_SIMT) {
    tc_wgrad_stg_plan_info(d, q);
  }
}

int launch_conv_tc_wgrad(const ConvShape& s, int math, const float* x, const float* dy, float* dw, void* ws,
                         size_t ws_bytes, cudaStream_t st) {
  auto aligned = [](const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15u) == 0; };
  const int route = tc_wgrad_route(s, math, aligned(x), aligned(dy), ws && aligned(ws));
  if (route == B2C_WGRAD_ROUTE_TMA_1X1) return launch_conv_tc_wgrad_tma(s, x, dy, dw, ws, ws_bytes, st);
  if (route == B2C_WGRAD_ROUTE_COMPACT_STAGED || route == B2C_WGRAD_ROUTE_COMPACT_TMA) {
    const ConvShape d = wgrad_compact_dense_shape(s);
    const bool staged = route == B2C_WGRAD_ROUTE_COMPACT_STAGED;
    const size_t part = staged ? tc_wgrad_stg_workspace(d) : splitk_workspace_bytes(wgrad_tma_plan(d, nullptr).splits, (long long)s.O * s.C);
    const size_t xoff = (part + 255) & ~(size_t)255;
    const size_t xbytes = sizeof(float) * (size_t)s.N * s.C * s.Ho * s.Wo;
    if (ws_bytes < xoff + xbytes) return fail(B2C_ERR_WORKSPACE, "wgrad (compact): workspace too small");
    float* xc = reinterpret_cast<float*>(static_cast<char*>(ws) + xoff);       // 16-byte aligned: ws is, xoff is a multiple of 256
    const long long planes = (long long)s.N * s.C;
    launch_pdl(subsample_kernel, grid_for((size_t)(planes * s.Ho * s.Wo), 256), 256, 0, st, 0, x, xc, planes, s.H, s.W, s.Ho, s.Wo, s.sh, s.sw);
    B2C_POST_LAUNCH();
    if (staged) return launch_conv_tc_wgrad_stg(d, xc, dy, dw, ws, part, st);
    return launch_conv_tc_wgrad_tma(d, xc, dy, dw, ws, part, st);
  }
  const WgradPlan pl = wgrad_plan(s);
  WgradParams p;
  p.dy = dy; p.x = x;
  p.N = s.N; p.C = s.C; p.H = s.H; p.W = s.W; p.O = s.O; p.Cg = s.Cg; p.Og = s.Og; p.Kd = s.Kd;
  p.kh = s.kh; p.kw = s.kw; p.sh = s.sh; p.sw = s.sw; p.ph = s.ph; p.pw = s.pw; p.dh = s.dh; p.dw = s.dw;
  p.Ho = s.Ho; p.Wo = s.Wo;
  p.Q = (long long)s.N * s.Ho * s.Wo;
  p.kb_per_split = pl.kb_per_split; p.splits = pl.splits;
  if (int rc = bind_splitk(p, pl.splits, (long long)s.O * s.Kd, dw, ws, ws_bytes, st, "wgrad")) return rc;
  p.prof = prof_buffer(st);
  int rc;
  switch (pl.n_tile) {
    case 64: rc = launch_wgrad_n<64>(p, s.G, math, s.is_1x1, st); break;
    default: rc = launch_wgrad_n<32>(p, s.G, math, s.is_1x1, st); break;
  }
  if (rc) return rc;
  if (p.prof) {
    long long h[32];
    prof_read(p.prof, h);
    fprintf(stderr, "[wprof] N_TILE=%d splits=%d nkb=%lld | dY-prod: loop=%lld wait_empty=%lld store=%lld | X-prod: loop=%lld wait_empty=%lld store=%lld\n",
            pl.n_tile, pl.splits, h[5], h[0], h[1], h[2], h[8], h[9], h[10]);
  }
  return B2C_OK;
}

TC_DEBUG_EXPORT(debug_mbar_wgrad)

}  // namespace b2c
