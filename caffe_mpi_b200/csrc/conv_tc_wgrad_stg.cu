// conv_tc_wgrad_stg.cu -- wgmma weight gradient with TMA-STAGED operands and bf16x3 math (sm_90a), for the stride-1
// "same" convolutions with 1 or 9 taps (1x1 / pad 0 and 3x3 / pad 1: 40 of ResNet-50's 53 layers, all of VGG-16's).
//
// Replaces cudnnConvolutionBackwardFilter beta=1 (reference src/caffe/layers/cudnn_conv_layer.cu:95-99) and, semantically,
// the per-image weight_gpu_gemm loop (base_conv_layer.hpp:148-162):
//     dW[o][c][tap] += sum_{n,p} dY[n][o][p] * X[n][c][p + off(tap)]        (X read as zero outside the image)
// GEMM view: M = 128 output channels, N = CN input channels x T taps (columns ordered (c, tap) = dW's own memory order, so
// a tile row is one contiguous run of dW), K = pixels.  The gather kernel (conv_tc_wgrad.cu) builds the X operand with
// per-thread predicated 4-byte loads.  Here, per K block of 64 pixels of one image:
//   * TMA brings in dY as two [128 o][32 px] fp32 boxes (SWIZZLE_128B) and X as ONE [CN c][64 + 2*halo px] fp32 box; pixels
//     past the image end and channels past O / C read as zero, which is the padding both the K tail and the M / N tails need;
//   * 8 converter warps split dY into bf16 hi / lo and write it into shared memory as the A operand (K-major, no swizzle;
//     the swizzled 16-byte chunks make the row-wise ld.shared.v4 conflict-free), and build the B operand in shared memory:
//     row (c, tap) of the K-major SWIZZLE_128B tile is the staged row of channel c shifted by the tap offset, masked where
//     the tap leaves the image (zero padding / row wrap; one bit per pixel and tap, computed once per K block), split into
//     bf16 hi / lo; lanes run along the pixels, so both the reads and the 4-byte writes are conflict-free;
//   * two consumer warpgroups issue wgmma.mma_async.m64nNk16.bf16: lo*hi + hi*lo + hi*hi per 16-pixel K step, N = 128 / 64
//     (1x1) or 72 (8 channels x 9 taps), fp32 accumulators in registers for the whole K range of the CTA (pixels past the
//     image end are zeros in both tiles, so every K block runs all four K steps);
//   * the reduction over pixels is split across CTAs in one wave; partial tiles meet through the fused, deterministic
//     split-K reduction of tc_common.cuh (arrival counter + per-CTA slice, fixed split order).
// Three bf16 MMAs per MAC cost 1.5 TF32 MMAs (3xTF32: 3); dropped terms ~2^-17 per product.
#include <stdio.h>
#include "b2c_common.cuh"
#define B2C_MBAR_DEBUG 1     // this kernel records stuck mbarrier waits (tc_common.cuh)
#include "tc_common.cuh"

namespace b2c {
using namespace tc;

namespace wstg {

constexpr int NCONS = 8;                      // consumer warps: two warpgroups (wgmma + epilogue), rows [64 cw, 64 cw + 64)
constexpr int NCW = 8;                        // converter warps
constexpr int W_CONV0 = NCONS;
constexpr int W_TMA = NCONS + NCW;
constexpr int THREADS = (NCONS + NCW + 1) * 32;   // 544
constexpr int KPX = 64;                       // pixels per K block
constexpr uint32_t DY_BYTES = 2u * 128u * 128u;   // two [128 rows][32 px] fp32 boxes

struct Params {
  int N, HW, H, W, C, O;
  int halo;                // pad*W + pad
  int bwx;                 // staged pixels per X channel row (multiple of 4)
  int bpi;                 // K blocks per image = ceil(HW / 64)
  long long nkb_total;     // N * bpi
  int kb_per_split, splits;
  int Kd;                  // C * T (row length of dW)
  float* out;              // splits == 1: dW (accumulated); else partials [splits][O*Kd] (overwritten)
  float* grad;             // dW (fused reduction target when splits > 1)
  unsigned int* counters;
};

// A_PRE: dY arrives already split into bf16 hi / lo planes (wstg_split_kernel) and TMA lands it straight in the A tiles as
// K-major SWIZZLE_128B boxes: no raw dY ring and no converter work for it.  The freed space goes to a deeper A / B ring.
template <int T, int CN, bool A_PRE>
struct Cfg {
  static constexpr int NROWS = T * CN;                                  // B rows = GEMM N (one wgmma)
  static constexpr uint32_t B_PLANE = (uint32_t)NROWS * 128u;           // [NROWS][64 bf16], SW128
  static constexpr uint32_t B_STAGE = 2u * B_PLANE;                     // hi + lo
  // [128 rows][64 bf16]: SW128 as TMA writes it (A_PRE), else K-major no swizzle as the converters write it
  static constexpr uint32_t A_BYTES = A_PRE ? 128u * 128u : tile_bytes(128);
  // raw operands as TMA delivers them.  dY and X have their own rings: the converters are done with a dY stage early
  // (it is converted into the A tile first), while X is read until the end of the block and wants two stages.
  // 3x3: X pool = 2 x [CN c][184 px] (W <= 56; wider maps, up to the 256-column TMA box, run with one X stage).
  static constexpr int NDY = 1;
  static constexpr uint32_t XMAX = (uint32_t)CN * (T == 1 ? 64u : 256u) * 4u;   // raw X box upper bound (1x1: no halo; else bwx <= 256)
  static constexpr uint32_t XPOOL = T == 1 ? 2u * XMAX : 2u * (uint32_t)CN * 184u * 4u;
  static constexpr uint32_t DYPOOL = A_PRE ? 0u : NDY * DY_BYTES;
  static_assert(XPOOL >= XMAX, "one X stage always fits");
  static constexpr uint32_t FIXED = DYPOOL + XPOOL + 256 + 1024;
  static constexpr uint32_t STAGE = B_STAGE + 2u * A_BYTES;
  static constexpr uint32_t FIT = (227u * 1024u - FIXED) / STAGE;
  static constexpr int BSTAGES = A_PRE ? (FIT < 4u ? (int)FIT : 4) : 2;
  static constexpr uint32_t B_OFF = 0;                                  // SW128 tiles: 1024-byte aligned
  static constexpr uint32_t DY_OFF = BSTAGES * B_STAGE;                 // SW128 boxes: 1024-byte aligned
  static constexpr uint32_t A_OFF = DY_OFF + DYPOOL;                    // A_PRE: SW128, 1024-byte aligned
  static constexpr uint32_t X_OFF = A_OFF + BSTAGES * 2u * A_BYTES;    // 128-byte aligned
  static constexpr uint32_t BAR_OFF = X_OFF + XPOOL;
  static constexpr uint32_t TOTAL = BAR_OFF + 256 + 1024;
  static_assert(NROWS % 8 == 0 && NROWS <= 256, "wgmma N");
  static_assert(BSTAGES >= 2 && BSTAGES <= 4, "A / B ring depth (4 barriers per ring)");
  static_assert(B_PLANE % 1024u == 0 && A_OFF % 1024u == 0, "SW128 tiles are 1024-byte aligned");
  static_assert(X_OFF % 128u == 0, "TMA destinations are 128-byte aligned");
  static_assert(TOTAL <= 227u * 1024u, "shared memory budget");
};

__device__ __forceinline__ float lds32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ float2 lds64(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
// PLANE (7x7 maps: a 196-byte channel pitch is not a TMA stride): one K block = one whole image.  The blobs are viewed as
// {4*H*W, channels/4, N} (four channels per tensor row), so a box of 32 rows is 128 channels x H*W pixels, contiguous; dY is read
// with 4-byte loads (odd word pitch: conflict-free), pixels H*W..63 of the 64-wide K block are written as zeros on both operands.
template <int T, int CN, bool PLANE, bool A_PRE>
__global__ void __launch_bounds__(THREADS, 1)
wgrad_stg_kernel(const __grid_constant__ Params p, const __grid_constant__ CUtensorMap map_dy, const __grid_constant__ CUtensorMap map_x) {
  using S = Cfg<T, CN, A_PRE>;
  using MMA = WgmmaBf16<S::NROWS>;
  constexpr int NROWS = S::NROWS, NDY = S::NDY, BST = S::BSTAGES;
  constexpr uint32_t LBO_A = tile_lbo(128);
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_dy_full = sbase + S::BAR_OFF;         // 2: dY boxes landed
  const uint32_t bar_dy_empty = bar_dy_full + 16;          // 2: converters have read the dY stage
  const uint32_t bar_x_full = bar_dy_empty + 16;           // 2: X box landed
  const uint32_t bar_x_empty = bar_x_full + 16;            // 2: converters have read the X stage
  const uint32_t bar_b_full = bar_x_empty + 16;            // BST (<= 4): A and B tiles written / landed
  const uint32_t bar_b_empty = bar_b_full + 32;            // BST: the MMAs of the stage have completed

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int split = blockIdx.x;
  const int c0 = blockIdx.y * CN;                          // input-channel tile
  const int m0 = blockIdx.z * 128;                         // output-channel tile
  const long long kb_begin = (long long)split * p.kb_per_split;
  long long kb_end = kb_begin + p.kb_per_split;
  if (kb_end > p.nkb_total) kb_end = p.nkb_total;
  const int nkb = (int)(kb_end - kb_begin);                // >= 1 by construction
  const uint32_t x_bytes = (uint32_t)CN * (uint32_t)p.bwx * 4u;      // plane mode: bwx = H*W (the channel pitch of the box)
  const uint32_t x_stride = (x_bytes + 127u) & ~127u;      // TMA destinations are 128-byte aligned
  const uint32_t dy_bytes = PLANE ? 128u * (uint32_t)p.HW * 4u : DY_BYTES;
  const int nx = 2u * x_stride <= S::XPOOL ? 2 : 1;        // X stages

  if (tid == 0) {
    for (int s = 0; s < 2; ++s) {
      mbar_init(bar_dy_full + 8 * s, 1); mbar_init(bar_dy_empty + 8 * s, NCW);
      mbar_init(bar_x_full + 8 * s, 1); mbar_init(bar_x_empty + 8 * s, NCW);
    }
    // b_full: the converter warps that write a tile, plus the TMA warp's expect_tx for the pre-split dY boxes
    constexpr uint32_t b_arrivals = A_PRE ? NCW + 1u : NCW;
    for (int s = 0; s < BST; ++s) { mbar_init(bar_b_full + 8 * s, b_arrivals); mbar_init(bar_b_empty + 8 * s, NCONS); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();      // everything above is shared-memory and barrier set-up

  auto b_hi = [&](int s) { return sbase + S::B_OFF + (uint32_t)s * S::B_STAGE; };
  auto b_lo = [&](int s) { return sbase + S::B_OFF + (uint32_t)s * S::B_STAGE + S::B_PLANE; };
  auto a_hi = [&](int s) { return sbase + S::A_OFF + (uint32_t)s * 2u * S::A_BYTES; };
  auto raw_dy = [&](int r) { return sbase + S::DY_OFF + (uint32_t)r * DY_BYTES; };
  auto raw_x = [&](int r) { return sbase + S::X_OFF + (uint32_t)r * x_stride; };
  // first pixel of the staged X row for K block j of an image: 16-byte aligned, never negative
  auto x_start = [&](int j) { return max((j * KPX - p.halo) & ~3, 0); };

  if (warp >= W_CONV0 && warp < W_CONV0 + NCW) {
    // ================= converters ===============================================================================
    const int cw = warp - W_CONV0;
    const int rq = cw & 3, ch2 = cw >> 2;                  // dY: row quarter / 32-pixel half of the K block
    const int row = rq * 32 + lane;
    const uint32_t a_row = (uint32_t)(row >> 3) * 128u + (uint32_t)(row & 7) * 16u;
    int n_img = (int)(kb_begin / p.bpi), j = (int)(kb_begin - (long long)n_img * p.bpi);
    const uint32_t lq = (uint32_t)lane >> 2, wr_off = (uint32_t)(lane & 3) * 4u;   // 16-byte chunk / byte inside it of this lane's pixel pair
    for (int i = 0; i < nkb; ++i) {
      const int rd = i % NDY, rx = i % nx, s = i % BST;
      // ---- (a) dY -> bf16 hi / lo: this thread's row (output channel), pixels [ch2*32, ch2*32 + 32)
      uint32_t hi[16], lo[16];
      if constexpr (!A_PRE) mbar_wait(bar_dy_full + 8 * rd, (i / NDY) & 1);
      if constexpr (A_PRE) {
        // dY arrives split: the TMA warp lands it in the A tile
      } else if constexpr (PLANE) {
        const uint32_t rowb = raw_dy(rd) + (uint32_t)row * (uint32_t)(p.HW * 4) + (uint32_t)(ch2 * 128);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          float v[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) v[e] = ch2 * 32 + q * 4 + e < p.HW ? lds32(rowb + (uint32_t)((q * 4 + e) * 4)) : 0.f;
          split_pack_bf16(v[0], v[1], hi[2 * q], lo[2 * q]);
          split_pack_bf16(v[2], v[3], hi[2 * q + 1], lo[2 * q + 1]);
        }
      } else {
        const uint32_t box = raw_dy(rd) + (uint32_t)ch2 * (128u * 128u) + (uint32_t)row * 128u;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const uint32_t chunk = (uint32_t)q ^ (uint32_t)(row & 7);
          const float4 v = lds128(box + chunk * 16u);
          split_pack_bf16(v.x, v.y, hi[2 * q], lo[2 * q]);
          split_pack_bf16(v.z, v.w, hi[2 * q + 1], lo[2 * q + 1]);
        }
      }
      if constexpr (!A_PRE) {
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_dy_empty + 8 * rd);    // the dY stage reloads while the B tile is built
      }
      mbar_wait_backoff(bar_b_empty + 8 * s, ((i / BST) & 1) ^ 1, 32);
      if constexpr (!A_PRE) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {                          // 16-byte K chunk = 8 pixels
          const uint32_t a = a_hi(s) + (uint32_t)(ch2 * 4 + q) * LBO_A + a_row;
          sts128u(a, hi[4 * q], hi[4 * q + 1], hi[4 * q + 2], hi[4 * q + 3]);
          sts128u(a + S::A_BYTES, lo[4 * q], lo[4 * q + 1], lo[4 * q + 2], lo[4 * q + 3]);
        }
      }
      // ---- (b) X -> B tile rows (c, tap): lanes run along the pixels, two adjacent pixels per lane
      const int col0 = j * KPX - x_start(j) + 2 * lane;       // staged column of this lane's first pixel at tap offset 0
      const uint32_t bh = b_hi(s);
      if constexpr (T == 9) {
        // per-tap validity of this lane's two pixels as an AND mask over the packed pair (zero padding, image borders, row
        // wrap, pixels past the image end), once per K block
        uint32_t mw[9];
        {
          uint32_t rb[2], cb[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int pp = j * KPX + 2 * lane + e;
            const int h = pp / p.W, w = pp - h * p.W;
            rb[e] = pp < p.HW ? ((h > 0 ? 1u : 0u) | 2u | (h + 1 < p.H ? 4u : 0u)) : 0u;
            cb[e] = (w > 0 ? 1u : 0u) | 2u | (w + 1 < p.W ? 4u : 0u);
          }
#pragma unroll
          for (int t = 0; t < 9; ++t)
            mw[t] = (((rb[0] >> (t / 3)) & (cb[0] >> (t % 3)) & 1u) ? 0x0000ffffu : 0u) |
                    (((rb[1] >> (t / 3)) & (cb[1] >> (t % 3)) & 1u) ? 0xffff0000u : 0u);
        }
        mbar_wait(bar_x_full + 8 * rx, (i / nx) & 1);
        constexpr int CPW = CN / NCW;                           // channels per warp (all 9 taps of each)
        const int w4 = p.W * 4;
#pragma unroll
        for (int c = 0; c < CPW; ++c) {
          const int cl = cw * CPW + c;
          const uint32_t srcc = raw_x(rx) + (uint32_t)((cl * p.bwx + col0) * 4);
          const uint32_t n0 = (uint32_t)cl * 9u;
#pragma unroll
          for (int ti = 0; ti < 3; ++ti) {
            // the three taps of a filter row read a 4-pixel window [-1, +2] around the pair
            const uint32_t srow = srcc + (uint32_t)((ti - 1) * w4);
            float v[4];
            v[0] = lds32i<-4>(srow); v[1] = lds32i<0>(srow); v[2] = lds32i<4>(srow); v[3] = lds32i<8>(srow);
#pragma unroll
            for (int tj = 0; tj < 3; ++tj) {
              const int t = ti * 3 + tj;
              uint32_t hw, lw;
              split_pack_bf16(v[tj], v[tj + 1], hw, lw);
              hw &= mw[t]; lw &= mw[t];                         // exact zeros whatever the staged bytes were
              const uint32_t n = n0 + (uint32_t)t;
              const uint32_t dst = bh + n * 128u + ((lq ^ (n & 7u)) << 4) + wr_off;
              sts32(dst, hw);
              sts32(dst + S::B_PLANE, lw);
            }
          }
        }
      } else {
        mbar_wait(bar_x_full + 8 * rx, (i / nx) & 1);
        constexpr int RPW = CN / NCW;                           // channels (= B rows) per warp
        // 1x1: no halo, the box starts at the K block's first pixel: the pair is 8-byte aligned
        const uint32_t srcw = raw_x(rx) + (uint32_t)((cw * RPW * KPX + 2 * lane) * 4);
#pragma unroll
        for (int k = 0; k < RPW; ++k) {
          float2 v;
          if constexpr (PLANE) {
            // channel pitch H*W*4 bytes (4-byte aligned only); pixels past the image are the next channel's: zeros instead
            const uint32_t a = raw_x(rx) + (uint32_t)(((cw * RPW + k) * p.HW + 2 * lane) * 4);
            v.x = 2 * lane < p.HW ? lds32(a) : 0.f;
            v.y = 2 * lane + 1 < p.HW ? lds32(a + 4u) : 0.f;
          } else {
            v = lds64(srcw + (uint32_t)(k * KPX * 4));
          }
          uint32_t hw, lw;
          split_pack_bf16(v.x, v.y, hw, lw);
          const uint32_t n = (uint32_t)(cw * RPW + k);
          const uint32_t dst = bh + n * 128u + ((lq ^ (n & 7u)) << 4) + wr_off;
          sts32(dst, hw);
          sts32(dst + S::B_PLANE, lw);
        }
      }
      // X stage fully read by this warp: hand it back to the TMA warp
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_x_empty + 8 * rx);
      fence_proxy_async();                                  // st.shared A / B tiles -> visible to the MMA's async-proxy reads
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_b_full + 8 * s);
      if (++j == p.bpi) { j = 0; ++n_img; }
    }
  } else if (warp == W_TMA) {
    // ================= TMA producer ================================================================================
    int n_img = (int)(kb_begin / p.bpi), j = (int)(kb_begin - (long long)n_img * p.bpi);
    for (int i = 0; i < nkb; ++i) {
      const int rd = i % NDY, rx = i % nx, s = i % BST;
      mbar_wait_backoff(bar_x_empty + 8 * rx, ((i / nx) & 1) ^ 1, 32);
      if (elect_one()) {
        arrive_expect_tx(bar_x_full + 8 * rx, x_bytes);
        if constexpr (PLANE) tma_load_3d(raw_x(rx), &map_x, bar_x_full + 8 * rx, 0, c0 / 4, n_img);
        else tma_load_3d(raw_x(rx), &map_x, bar_x_full + 8 * rx, x_start(j), c0, n_img);
      }
      __syncwarp();
      if constexpr (A_PRE) {
        // pre-split planes {HWp, O, 2N}: hi of image n at n, lo at N + n; rows past O read as zeros
        mbar_wait_backoff(bar_b_empty + 8 * s, ((i / BST) & 1) ^ 1, 32);
        if (elect_one()) {
          const uint32_t bar = bar_b_full + 8 * s;
          arrive_expect_tx(bar, 2u * S::A_BYTES);
          tma_load_3d(a_hi(s), &map_dy, bar, j * KPX, m0, n_img);
          tma_load_3d(a_hi(s) + S::A_BYTES, &map_dy, bar, j * KPX, m0, p.N + n_img);
        }
        __syncwarp();
      } else {
      mbar_wait_backoff(bar_dy_empty + 8 * rd, ((i / NDY) & 1) ^ 1, 32);
      if (elect_one()) {
        arrive_expect_tx(bar_dy_full + 8 * rd, dy_bytes);
        if constexpr (PLANE) {
          tma_load_3d(raw_dy(rd), &map_dy, bar_dy_full + 8 * rd, 0, m0 / 4, n_img);
        } else {
          tma_load_3d(raw_dy(rd), &map_dy, bar_dy_full + 8 * rd, j * KPX, m0, n_img);
          tma_load_3d(raw_dy(rd) + 128u * 128u, &map_dy, bar_dy_full + 8 * rd, j * KPX + 32, m0, n_img);
        }
      }
      __syncwarp();
      }
      if (++j == p.bpi) { j = 0; ++n_img; }
    }
  } else if (warp >= 4 && warp < NCONS && p.O - m0 <= 64) {
    // ================= second consumer warpgroup of a tile whose rows [m0 + 64, m0 + 128) are all past O ==========
    // nothing to multiply (its rows are never stored): it only keeps the stage protocol, releasing each stage as it fills
    for (int i = 0; i < nkb; ++i) {
      const int s = i % BST;
      mbar_wait_backoff(bar_b_full + 8 * s, (i / BST) & 1, 32);
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_b_empty + 8 * s);
    }
  } else if (warp < NCONS) {
    // ================= consumers: wgmma over the CTA's K range, then the partial tile from registers ==============
    // For T = 9 the wgmma accumulator is added into `tot` on the CUDA cores every PROMOTE K blocks (512 pixels) and restarted.
    // Accumulating a whole split in the wgmma accumulator measured 7.5e-4 against the 3e-4 dW bar of
    // test_full_size_vs_reference_loop on an H100 for VGG-16 conv1_2 (N = 32, ~10^5 pixels per CTA); with the promotion it passes.
    // (The 1x1 tiles are wider -- no registers for a second copy -- and have enough tiles to keep their chains short.)
    constexpr int PROMOTE = T == 9 ? 8 : 1 << 30;
    constexpr int NT = T == 9 ? NROWS / 2 : 1;
    const int cwg = warp >> 2, t = tid & 127;
    float acc[NROWS / 2], tot[NT];
#pragma unroll
    for (int q = 0; q < NROWS / 2; ++q) acc[q] = 0.f;
#pragma unroll
    for (int q = 0; q < NT; ++q) tot[q] = 0.f;
    int prev = -1;
    for (int i = 0; i < nkb; ++i) {
      const int s = i % BST;
      const int fresh = i % PROMOTE == 0;
      mbar_wait(bar_b_full + 8 * s, (i / BST) & 1);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < KPX / 16; ++kk) {
        uint64_t ah, al;
        if constexpr (A_PRE) {                     // SW128 [128 rows][64 px]: this warpgroup's 64 rows start 8 KB in
          const uint32_t a = a_hi(s) + (uint32_t)cwg * (64u * 128u) + kk * 32;
          ah = smem_desc_sw128(a); al = smem_desc_sw128(a + S::A_BYTES);
        } else {
          const uint32_t a = a_hi(s) + 2u * kk * LBO_A + (uint32_t)cwg * 1024u;
          ah = smem_desc(a, LBO_A, 128); al = smem_desc(a + S::A_BYTES, LBO_A, 128);
        }
        const uint64_t bh = smem_desc_sw128(b_hi(s) + kk * 32), bl = smem_desc_sw128(b_lo(s) + kk * 32);
        MMA::mma(acc, al, bh, !fresh || kk != 0);  // lo * hi
        MMA::mma(acc, ah, bl, 1);                 // hi * lo
        MMA::mma(acc, ah, bh, 1);                 // hi * hi
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(bar_b_empty + 8 * prev); }
      prev = s;
      if constexpr (T == 9) {
        if (i % PROMOTE == PROMOTE - 1 || i == nkb - 1) {
          wgmma_wait<0>();
          wgmma_reg_fence(acc);
#pragma unroll
          for (int q = 0; q < NT; ++q) tot[q] += acc[q];
        }
      }
    }
    wgmma_wait<0>();
    wgmma_reg_fence(acc);
    // row = output channel, column = (c, tap) = dW's own order; lanes of a quad write 8 consecutive columns of a row
    float* obase = p.out + (p.splits > 1 ? (long long)split * p.O * p.Kd : 0LL) + (long long)c0 * T;
    const int cols_valid = min(NROWS, (p.C - c0) * T);
    const bool accumulate = p.splits == 1;
#pragma unroll
    for (int q = 0; q < NROWS / 2; ++q) {
      const int r = m0 + cwg * 64 + frag_row(t, q), c = frag_col(t, q);
      if (r < p.O && c < cols_valid) {
        float* dst = obase + (long long)r * p.Kd + c;
        const float v = T == 9 ? tot[q < NT ? q : 0] : acc[q];
        *dst = accumulate ? *dst + v : v;
      }
    }
  }
  if (p.splits > 1) {
    const int tile_id = blockIdx.z * gridDim.y + blockIdx.y;
    splitk_fused_reduce(p.out, p.grad, p.counters + tile_id, split, p.splits, (long long)p.O * p.Kd, (long long)m0 * p.Kd + (long long)c0 * T, p.Kd,
                        min(128, p.O - m0), min(NROWS, (p.C - c0) * T));
  }
}

// fp32 [N][channels][HW] -> bf16 hi plane [N][channels][HWp] followed by the lo plane (same shape), pixels HW..HWp-1 zero:
// the dY operand wgrad_stg_kernel's A_PRE variant reads.  The split is the converters' split_pack_bf16, so the MMA tiles
// hold the same bits either way.  One thread per 8 output pixels (one 16-byte store per plane).
__global__ void __launch_bounds__(256)
wstg_split_kernel(const float* __restrict__ src, uint4* __restrict__ dst, long long rows, int HW, int HWp) {
  pdl_wait();
  const int per_row = HWp / 8;
  const long long total = rows * per_row;
  const long long plane = total;                            // 16-byte units per plane
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / per_row;
    const int p0 = (int)(i - r * per_row) * 8;
    const float* row = src + r * HW;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = p0 + e < HW ? __ldg(row + p0 + e) : 0.f;
    uint32_t hi[4], lo[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) split_pack_bf16(v[2 * q], v[2 * q + 1], hi[q], lo[q]);
    dst[i] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    dst[plane + i] = make_uint4(lo[0], lo[1], lo[2], lo[3]);
  }
}

}  // namespace wstg


// ---- host side ------------------------------------------------------------------------------------------------------
static bool wstg_enabled() {
  static const int on = env_int("B2C_WGRAD_STAGED", 1);
  return on != 0;
}
// a_pre: dY goes through wstg_split_kernel first (only when the caller brings the split buffer)
struct WstgPlan { int T, cn, bwx, bpi, splits, kb_per_split; long long nkb; bool plane, a_pre; };
// dY of a 3x3 layer is split into bf16 hi / lo planes once per call, instead of once per CTA in the converter warps, when at least
// this many input-channel tiles (8 channels each) would convert each of its K blocks.  The split pass moves 8 bytes of HBM per
// element.  Measured on an H100 SXM (700 W), ResNet-50 at N = 64: every 3x3 layer gains (c_tiles 8 to 64; 250 -> 210 us for res2,
// 221 -> 167 us for res4), while no 1x1 layer does in the training step: their tiles are 64 or 128 channels wide, so a block is
// converted by at most 16 CTAs, and the split pass over their larger dY / X costs as much as it saves.  1x1 layers never pre-split.
constexpr int PRESPLIT_MIN_TILES = 8;
static bool wstg_plane_enabled() {
  static const int on = env_int("B2C_WGRAD_STAGED_PLANE", 1);
  return on != 0;
}
static bool wstg_plan(const ConvShape& s, WstgPlan* pl) {
  if (!wstg_enabled()) return false;
  if (s.G != 1 || s.sh != 1 || s.sw != 1 || s.dh != 1 || s.dw != 1 || s.Ho != s.H || s.Wo != s.W) return false;
  const bool k1 = s.kh == 1 && s.kw == 1 && s.ph == 0 && s.pw == 0;
  const bool k3 = s.kh == 3 && s.kw == 3 && s.ph == 1 && s.pw == 1;
  if (!k1 && !k3) return false;
  const long long HW = (long long)s.H * s.W;
  if ((long long)s.N * HW > 0x7fffffffLL - 256) return false;
  // 7x7 maps: plane mode (one image per K block, blobs viewed four channels per tensor row)
  const bool plane = HW == 49 && s.C % 4 == 0 && s.O % 4 == 0 && wstg_plane_enabled();
  if (!plane && (HW % 4 != 0 || HW < 64)) return false;
  const int T = k1 ? 1 : 9;
  const int halo = s.ph * s.W + s.pw;
  const int need = wstg::KPX + 2 * halo + ((4 - halo % 4) % 4);
  if (!plane && need > 256) return false;
  if (!pl) return true;
  pl->T = T;
  pl->plane = plane;
  pl->cn = k1 ? (s.C > 64 ? 128 : 64) : 8;           // N = 128 / 64 / 72 columns: <= 64 accumulator registers per consumer thread
  pl->bwx = plane ? (int)HW : (need + 3) & ~3;
  pl->bpi = (int)((HW + wstg::KPX - 1) / wstg::KPX);
  pl->nkb = (long long)s.N * pl->bpi;
  const int c_tiles = (s.C + pl->cn - 1) / pl->cn, o_tiles = (s.O + 127) / 128;
  plan_splitk(pl->nkb, (long long)o_tiles * c_tiles, 4, &pl->splits, &pl->kb_per_split);
  pl->a_pre = T == 9 && c_tiles >= PRESPLIT_MIN_TILES;
  return true;
}
// pre-split dY: hi and lo planes of [N][O][bpi * 64] bf16
static size_t wstg_split_bytes(const ConvShape& s, const WstgPlan& pl) {
  return pl.a_pre ? (size_t)4 * s.N * s.O * pl.bpi * wstg::KPX : 0;
}
bool tc_wgrad_stg_supported(const ConvShape& s) { return wstg_plan(s, nullptr); }
bool tc_wgrad_stg_plan_info(const ConvShape& s, WgradPlanInfo* q) {
  WstgPlan pl;
  if (!wstg_plan(s, &pl)) return false;
  q->splits = pl.splits; q->kb_per_split = pl.kb_per_split; q->nkb = pl.nkb;
  q->cols = pl.cn * pl.T; q->bpi = pl.bpi; q->taps = pl.T; q->plane = pl.plane;
  q->presplit = pl.a_pre ? 1 : 0;
  q->split_bytes = wstg_split_bytes(s, pl);
  return true;
}
size_t tc_wgrad_stg_workspace(const ConvShape& s) {
  WstgPlan pl;
  if (!wstg_plan(s, &pl)) return 0;
  return splitk_workspace_bytes(pl.splits, (long long)s.O * s.Kd);
}

template <int T, int CN, bool PLANE, bool A_PRE = false>
static int wstg_launch(const wstg::Params& p, const CUtensorMap& mdy, const CUtensorMap& mx, int c_tiles, int o_tiles, cudaStream_t st) {
  using S = wstg::Cfg<T, CN, A_PRE>;
  B2C_CUDA_OK(cudaFuncSetAttribute(wstg::wgrad_stg_kernel<T, CN, PLANE, A_PRE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)S::TOTAL));
  dim3 grid(p.splits, c_tiles, o_tiles);
  launch_pdl(wstg::wgrad_stg_kernel<T, CN, PLANE, A_PRE>, grid, wstg::THREADS, S::TOTAL, st, 0, p, mdy, mx);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
static int launch_wstg_planned(const ConvShape& s, const WstgPlan& pl, const float* x, const float* dy, float* dw, void* ws, size_t ws_bytes,
                               void* split, cudaStream_t st);
int launch_conv_tc_wgrad_stg(const ConvShape& s, const float* x, const float* dy, float* dw, void* ws, size_t ws_bytes, cudaStream_t st,
                             void* split, size_t split_bytes) {
  WstgPlan pl;
  if (!wstg_plan(s, &pl)) return fail(B2C_ERR_INVALID, "staged wgrad: shape not eligible");
  if (!split) {
    pl.a_pre = false;
  } else if (split_bytes < wstg_split_bytes(s, pl) || (reinterpret_cast<uintptr_t>(split) & 15u)) {
    return fail(B2C_ERR_WORKSPACE, "staged wgrad: split buffer too small or not 16-byte aligned");
  }
  return launch_wstg_planned(s, pl, x, dy, dw, ws, ws_bytes, split, st);
}

// ---- caffe_gpu_gemm, NoTrans x Trans (math_functions.cu:11-26 as InnerProductLayer::Forward_gpu calls it): C[M][N] (+)= A[M][K] * B[N][K]^T.
// Both operands have the reduction axis contiguous, which is exactly the 1x1 weight-gradient problem with one "image" of K
// "pixels": A plays dY (rows = M), B plays X (rows = N), C is dW with row length N.  No workspace in the BLAS signature, so
// the reduction is not split (one CTA per 128 x 128 output tile walks all of K).
bool tc_gemm_supported(bool tA, bool tB, int M, int N, int K) {
  return wstg_enabled() && !tA && tB && M > 0 && N > 0 && K >= 64 && K % 4 == 0 && (long long)M * N * 4 < (1ll << 40);
}
// split count of the K loop when the caller brings a workspace (b2c_sgemm_ex): one wave of CTAs, >= 4 K blocks per split
static void gemm_tc_plan(int M, int N, int K, WstgPlan* pl) {
  pl->T = 1; pl->plane = false; pl->a_pre = false; pl->cn = N > 64 ? 128 : 64; pl->bwx = wstg::KPX; pl->bpi = (K + wstg::KPX - 1) / wstg::KPX; pl->nkb = pl->bpi;
  plan_splitk(pl->nkb, (long long)((M + 127) / 128) * ((N + pl->cn - 1) / pl->cn), 4, &pl->splits, &pl->kb_per_split);
}
size_t tc_gemm_workspace(bool tA, bool tB, int M, int N, int K) {
  if (!tc_gemm_supported(tA, tB, M, N, K)) return 0;
  WstgPlan pl;
  gemm_tc_plan(M, N, K, &pl);
  return splitk_workspace_bytes(pl.splits, (long long)M * N);
}
// The wgmma accumulator of the 1x1 tiles is never promoted (no registers for a second copy): its error grows with the K blocks
// one CTA walks.  Measured on an H100 SXM (700 W), N(0, 1) operands, blob error max|err| / max|ref| of one unsplit chain: 144 blocks
// 3.7e-5, 392 blocks 8.9e-5, 784 blocks (K = 50176) 1.9e-4 against the 1e-4 bar.  A product the planner would split, but that runs
// unsplit because the caller brought no usable workspace (b2c_sgemm: the CAFFE engine's per-image weight gradient), goes to the
// FFMA kernel past this many K blocks instead.
constexpr int TC_GEMM_MAX_UNSPLIT_KB = 256;
void sgemm_route(bool tc_allowed, bool tA, bool tB, int M, int N, int K, float alpha, float beta, const void* A, const void* B,
                 const void* ws, size_t ws_bytes, GemmPlan* g) {
  bool tc = tc_allowed && alpha == 1.0f && (beta == 0.0f || beta == 1.0f) &&
            ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B)) & 15u) == 0 && tc_gemm_supported(tA, tB, M, N, K);
  if (tc) {
    WstgPlan pl;
    gemm_tc_plan(M, N, K, &pl);
    // no workspace, a short one or a misaligned one: one CTA per tile walks all of K
    if (pl.splits > 1 &&
        (!ws || ws_bytes < splitk_workspace_bytes(pl.splits, (long long)M * N) || (reinterpret_cast<uintptr_t>(ws) & 15u))) {
      pl.splits = 1;
      pl.kb_per_split = pl.bpi;
      tc = pl.bpi <= TC_GEMM_MAX_UNSPLIT_KB;
    }
    if (tc) {
      *g = GemmPlan{true, pl.cn, pl.bpi, pl.splits, pl.kb_per_split, (M + 127) / 128, (N + pl.cn - 1) / pl.cn};
      return;
    }
  }
  const int nk = (K + 15) / 16;                       // sgemm_simt_kernel: 64 x 64 tiles, K in steps of 16
  *g = GemmPlan{false, 64, nk, 1, nk, (M + 63) / 64, (N + 63) / 64};
}
int launch_sgemm_tc(const GemmPlan& g, int M, int N, int K, const float* A, const float* B, float beta, float* Cm, void* ws,
                    size_t ws_bytes, cudaStream_t st) {
  if (!g.tc) return fail(B2C_ERR_INVALID, "tensor-core GEMM: the plan is not a tensor-core one");
  if (beta == 0.0f) B2C_CUDA_OK(cudaMemsetAsync(Cm, 0, sizeof(float) * (size_t)M * N, st));
  ConvShape s{};
  s.N = 1; s.C = N; s.H = 1; s.W = K; s.O = M; s.G = 1; s.kh = s.kw = 1; s.sh = s.sw = 1; s.ph = s.pw = 0; s.dh = s.dw = 1; s.has_bias = 0;
  s.Ho = 1; s.Wo = K; s.Cg = N; s.Og = M; s.Kd = N; s.is_1x1 = true;
  WstgPlan pl;
  gemm_tc_plan(M, N, K, &pl);
  pl.splits = g.splits; pl.kb_per_split = g.kb_per_split;
  if (g.splits == 1) { ws = nullptr; ws_bytes = 0; }
  return launch_wstg_planned(s, pl, B, A, Cm, ws, ws_bytes, nullptr, st);
}

static int launch_wstg_split(const float* src, void* dst, long long rows, int HW, int HWp, cudaStream_t st) {
  launch_pdl(wstg::wstg_split_kernel, grid_for((size_t)rows * (HWp / 8), 256), 256, 0, st, 0, src, static_cast<uint4*>(dst), rows, HW, HWp);
  B2C_POST_LAUNCH();
  return B2C_OK;
}

static int launch_wstg_planned(const ConvShape& s, const WstgPlan& pl, const float* x, const float* dy, float* dw, void* ws, size_t ws_bytes,
                               void* split, cudaStream_t st) {
  wstg::Params p;
  p.N = s.N; p.HW = s.H * s.W; p.H = s.H; p.W = s.W; p.C = s.C; p.O = s.O;
  p.halo = s.ph * s.W + s.pw; p.bwx = pl.bwx; p.bpi = pl.bpi; p.nkb_total = pl.nkb;
  p.kb_per_split = pl.kb_per_split; p.splits = pl.splits; p.Kd = s.Kd;
  if (int rc = bind_splitk(p, pl.splits, (long long)s.O * s.Kd, dw, ws, ws_bytes, st, "staged wgrad")) return rc;
  alignas(64) CUtensorMap mdy, mx;
  const cuuint64_t HW = (cuuint64_t)p.HW;
  const int c_tiles = (s.C + pl.cn - 1) / pl.cn, o_tiles = (s.O + 127) / 128;
  if (pl.a_pre) {
    // pre-split dY: {HWp, O, 2N} bf16 (hi planes of the N images, then their lo planes), [128 o][64 px] SW128 boxes
    const int HWp = pl.bpi * wstg::KPX;
    if (int rc = launch_wstg_split(dy, split, (long long)s.N * s.O, p.HW, HWp, st)) return rc;
    const cuuint64_t pitch = (cuuint64_t)HWp * 2;
    if (int rc = make_tensor_map_3d(&mdy, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, split, {(cuuint64_t)HWp, (cuuint64_t)s.O, 2 * (cuuint64_t)s.N},
                                    {pitch, pitch * (cuuint64_t)s.O}, {(cuuint32_t)wstg::KPX, 128, 1}, CU_TENSOR_MAP_SWIZZLE_128B,
                                    "staged wgrad (pre-split dY)"))
      return rc;
  } else if (pl.plane) {
    // {4*HW, channels/4, N}: four channels per tensor row (a 16-byte-multiple pitch); box rows = tile channels / 4
    if (int rc = make_tensor_map_3d(&mdy, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, dy, {HW * 4, (cuuint64_t)s.O / 4, (cuuint64_t)s.N},
                                    {HW * 16, HW * 16 * (cuuint64_t)(s.O / 4)}, {(cuuint32_t)HW * 4, 32, 1}, CU_TENSOR_MAP_SWIZZLE_NONE, "staged wgrad"))
      return rc;
  } else {
    // [N][channels][HW] fp32: dY in [128 o][32 px] SWIZZLE_128B boxes
    if (int rc = make_tensor_map_3d(&mdy, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, dy, {HW, (cuuint64_t)s.O, (cuuint64_t)s.N}, {HW * 4, HW * 4 * (cuuint64_t)s.O},
                                    {32, 128, 1}, CU_TENSOR_MAP_SWIZZLE_128B, "staged wgrad"))
      return rc;
  }
  if (pl.plane) {
    if (int rc = make_tensor_map_3d(&mx, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, x, {HW * 4, (cuuint64_t)s.C / 4, (cuuint64_t)s.N},
                                    {HW * 16, HW * 16 * (cuuint64_t)(s.C / 4)}, {(cuuint32_t)HW * 4, (cuuint32_t)pl.cn / 4, 1},
                                    CU_TENSOR_MAP_SWIZZLE_NONE, "staged wgrad"))
      return rc;
  } else {
    // X in [CN c][bwx px] boxes
    if (int rc = make_tensor_map_3d(&mx, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, x, {HW, (cuuint64_t)s.C, (cuuint64_t)s.N}, {HW * 4, HW * 4 * (cuuint64_t)s.C},
                                    {(cuuint32_t)pl.bwx, (cuuint32_t)pl.cn, 1}, CU_TENSOR_MAP_SWIZZLE_NONE, "staged wgrad"))
      return rc;
  }
  if (pl.plane) {
    if (pl.T == 9) return pl.a_pre ? wstg_launch<9, 8, true, true>(p, mdy, mx, c_tiles, o_tiles, st) : wstg_launch<9, 8, true>(p, mdy, mx, c_tiles, o_tiles, st);
    if (pl.cn == 128) return wstg_launch<1, 128, true>(p, mdy, mx, c_tiles, o_tiles, st);
    return wstg_launch<1, 64, true>(p, mdy, mx, c_tiles, o_tiles, st);
  }
  if (pl.T == 9) return pl.a_pre ? wstg_launch<9, 8, false, true>(p, mdy, mx, c_tiles, o_tiles, st) : wstg_launch<9, 8, false>(p, mdy, mx, c_tiles, o_tiles, st);
  if (pl.cn == 128) return wstg_launch<1, 128, false>(p, mdy, mx, c_tiles, o_tiles, st);
  return wstg_launch<1, 64, false>(p, mdy, mx, c_tiles, o_tiles, st);
}

TC_DEBUG_EXPORT(debug_mbar_wstg)

}  // namespace b2c
