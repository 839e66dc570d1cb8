// conv_tc_stg.cu -- wgmma implicit-GEMM convolution with BULK-COPY-STAGED activations and bf16x3 math (sm_90a):
// forward and data-gradient of stride-1 "same" convolutions (1x1 / pad 0, 3x3 / pad 1, 5x5 / pad 2 ...), which are
// 43 of ResNet-50's 53 layers and every VGG-16 / GoogLeNet inception convolution with C % 32 == 0.
//
// Replaces cudnnConvolutionForward / cudnnConvolutionBackwardData as the reference's CuDNNConvolutionLayer calls them
// (src/caffe/layers/cudnn_conv_layer.cu:25-29,118-123); same contract as conv_tc.cu: NCHW fp32 in and out, whole
// batch per launch, y / dx overwritten, bias fused.
//
// Why a second kernel.  conv_tc.cu gathers the im2col rows with per-thread __ldg and re-reads every input pixel kh*kw
// times through L1/L2.  Here no thread touches global memory for the activation operand:
//   * GEMM rows are 128 CONSECUTIVE flattened pixels q = n*H*W + p.  For 32 input channels the pixels a tile needs --
//     its own 128 plus a halo of pad*W + pad on either side -- are ONE TMA box per image the tile touches (at most two):
//     a 3-D tensor map {H*W, C, N} over the NCHW blob, box {BWT pixels, 32 channels, 1 image}, start column
//     p0 - halo; columns outside the image read as zero.  (One 1-D bulk copy per channel instead would cost one small
//     bulk operation per channel, which the TMA unit retires far more slowly than one box.)
//   * All kh*kw taps of those 32 channels are then served from that ONE staged copy: tap (i,j) of row r is the staged
//     value at column r + halo + (i-pad)*W + (j-pad); rows whose tap falls outside the image (zero padding, image
//     borders, row wrap) are masked with a per-row bit computed once per tile.  Global->smem traffic per tile is
//     (128 + 2*halo)/128 of the input instead of kh*kw times it.
//   * 8 converter warps read the staged fp32 values (lanes = consecutive pixels: conflict-free; the row pitch BWT is a
//     template parameter so the sixteen channel loads of a thread are one base register + immediates), split each into
//     bf16 hi + bf16 lo (hi = rn(a), lo = rn(a - hi)), pack pairs along K and write the A operand into shared memory
//     (K-major, no swizzle, tc_common.cuh), 64 K-elements per stage.
//   * The filter is pre-split into bf16 hi / lo in GEMM-K order (channel group, tap, channel) by a prepass and streamed
//     by TMA (SWIZZLE_128B, [N_TILE x 64] boxes).  Two consumer warpgroups take turns over the CTA's tiles (ping-pong):
//     each issues wgmma.mma_async.m64nNk16.bf16 for both 64-row halves of its own tile (fp32 accumulators in registers,
//     N_TILE per thread): lo*hi + hi*lo + hi*hi per K step -- three bf16 MMAs cost 1.5 TF32-MMA equivalents (3xTF32
//     costs 3), and the operand bytes in shared memory halve.  Dropped terms (lo*lo and the bf16 rounding of lo) are
//     ~2^-17 per product, far inside the 1e-3 blob tolerance.
//   * Epilogue (the tile's warpgroup, after its last K block, while the other warpgroup runs the next tile's MMAs):
//     (+ bias), 32-channel chunks transposed through the warpgroup's own shared-memory buffer [channel][128 pixels] and
//     written by the TMA unit when the tile lies inside one image: one tensor store per chunk (box {128, 32, 1} of the
//     output blob, clipped by the hardware at the image end and the channel count; the start column is never negative).
//     Tiles that span two images write the staged chunk with 16-byte st.global.
//   * Plane mode (BWT < 128): 7x7 maps, whole image planes staged -- see Smem below.
// dgrad of a stride-1 same convolution is the same kernel on dY with the transposed + flipped filter.
#include <cuda_bf16.h>
#include <limits.h>
#include <stdio.h>
#include "b2c_common.cuh"
#define B2C_MBAR_DEBUG 1     // this kernel records stuck mbarrier waits (tc_common.cuh)
#include "tc_common.cuh"
#include "filter_prep.cuh"

namespace b2c {
using namespace tc;

namespace stg {

// Five whole warpgroups, so that setmaxnreg can give each role its own register budget:
//   WG0, WG1  consumers (wgmma + epilogue), ping-pong: each owns whole 128 x N_TILE tiles, the CTA's even / odd ones
//   WG2, WG3  the 8 converter warps
//   WG4       filter TMA warp, activation TMA warp, two idle warps
constexpr int NCW = 8;                        // converter warps
constexpr int W_CONV0 = 8;                    // first converter warp
constexpr int W_BTMA = 16;                    // filter TMA warp
constexpr int W_STG = 17;                     // activation TMA warp
constexpr int THREADS = 5 * 128;              // 640
// registers per thread after setmaxnreg: the consumers hold two m64 x N_TILE accumulator sets (N_TILE fp32 per thread).
// All budgets together must fit what the CTA is launched with: 65536 / 640 rounded down to the allocation unit of 8 = 96.
constexpr int REG_CONS = 176, REG_CONV = 48, REG_TMA = 32;
static_assert(2 * 128 * REG_CONS + 2 * 128 * REG_CONV + 128 * REG_TMA <= THREADS * ((65536 / THREADS) & ~7), "register budget");
// named barriers: 1 + w = warpgroup w's epilogue, 3 + w = "warpgroup w may start its next tile's MMAs"
constexpr int BAR_EPI = 1, BAR_ORDER = 3;
constexpr int CB = 32;                        // channels per staged group
constexpr int BKE = 64;                       // bf16 K elements per pipeline stage (two (group, tap) half blocks)
constexpr uint32_t STG_POOL = 64u * 1024u;    // activation staging pool, carved into slots of one TMA box each
constexpr int MAX_SLOTS = 6;
constexpr int MAX_TAPS = 32;                  // per-row validity mask is one 32-bit word
constexpr int PLANE_IMGS = 4;                 // plane mode: images per staging slot (a 128-row tile of 7x7 maps touches <= 4)

struct Params {
  int HW, H, W;
  int kh, kw, ph, pw;
  int Mtot;                // Nimg * H * W (output pixel grid == input pixel grid)
  int Ntot;                // GEMM columns (output channels)
  int taps, groups;        // kh*kw, Cin / 32
  int nhb, nkb;            // half blocks = groups * taps, K blocks = ceil(nhb / 2)
  int halo;                // pad*W + pad
  const float* bias;       // [Ntot] or null
  float* out;              // [Nimg, Ntot, H, W]: the epilogue's st.global path (tiles that span two images)
  int m_tiles, n_tiles, total_tiles;
  int dbg;                 // B2C_STG_DBG bit 0: never use TMA stores (st.global epilogue for every tile)
  int accumulate;          // out += result instead of out = result (TMA reduce-add store; the fan-out accumulation of Net::Backward)
  long long* prof;
};

template <int N_TILE, int BWT>
struct Smem {
  static constexpr uint32_t B_BYTES = (uint32_t)N_TILE * 128u;              // [N_TILE rows][64 bf16], SW128
  static constexpr uint32_t A_BYTES = tile_bytes(128);                      // [128 rows][64 bf16], K-major no swizzle
  static constexpr uint32_t STAGE = 2u * B_BYTES + 2u * A_BYTES;           // B hi, B lo, A hi, A lo
  // BWT >= 128: one box = [32 channels][BWT pixels] fp32.  BWT < 128 ("plane mode", maps of BWT = H*W pixels whose
  // channel pitch TMA cannot address, 7x7 = 196 bytes): one slot = up to PLANE_IMGS whole images x [32 channels][H*W]
  static constexpr bool PLANE = BWT < 128;
  static constexpr uint32_t IMG_BYTES = (uint32_t)CB * (uint32_t)BWT * 4u;
  static constexpr uint32_t SLOT_BYTES = PLANE ? PLANE_IMGS * IMG_BYTES : IMG_BYTES;
  static constexpr uint32_t PITCH = (uint32_t)BWT * 4u;                     // bytes between channels of a staged box
  static_assert(!PLANE || IMG_BYTES % 128u == 0, "TMA destinations are 128-byte aligned");
  static_assert(!PLANE || 127 / BWT + 2 <= PLANE_IMGS, "a 128-row tile touches at most PLANE_IMGS images");
  static constexpr int NSLOT_ = (int)(STG_POOL / SLOT_BYTES);
  static constexpr int NSLOT = NSLOT_ > MAX_SLOTS ? MAX_SLOTS : NSLOT_;
  static constexpr uint32_t EPI_BYTES = 32u * 128u * 4u;                    // [32 channels][128 pixels] fp32, one per consumer warpgroup
  static constexpr uint32_t FIXED = STG_POOL + 2u * EPI_BYTES + 256u + MAX_TAPS * 4u + 1024u;
  static constexpr int STAGES_ = (int)((227u * 1024u - FIXED) / STAGE);
  static constexpr int STAGES = STAGES_ > 3 ? 3 : STAGES_;                  // operand pipeline depth
  // the B tiles of every stage first (SWIZZLE_128B wants 1024-byte alignment), then the A tiles, packed
  static constexpr uint32_t A_OFF = STAGES * 2u * B_BYTES;
  static constexpr uint32_t STG_OFF = A_OFF + STAGES * 2u * A_BYTES;
  static constexpr uint32_t EPI_OFF = STG_OFF + STG_POOL;
  static constexpr uint32_t BAR_OFF = EPI_OFF + 2u * EPI_BYTES;
  static_assert(STG_OFF % 128u == 0, "TMA destinations are 128-byte aligned");
  static constexpr uint32_t TAP_OFF = BAR_OFF + 256;                        // int tap offsets [MAX_TAPS]
  static constexpr uint32_t TOTAL = TAP_OFF + MAX_TAPS * 4 + 1024;          // + alignment slack
  static constexpr uint32_t TX_BYTES = 2u * B_BYTES;
  static_assert(STAGES >= 2, "shared memory budget");
  static_assert(NSLOT >= 2, "a tile that spans two images needs two boxes per channel group");
};

__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, uint32_t smem_src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_src), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// out[box] += smem tile: the TMA unit's reduction store (fp32 add in L2), same clipping as the plain store
__device__ __forceinline__ void tma_reduce_add_3d(const CUtensorMap* map, uint32_t smem_src, int c0, int c1, int c2) {
  asm volatile("cp.reduce.async.bulk.tensor.3d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_src), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
template <int N_TILE, int BWT>
__global__ void __launch_bounds__(THREADS, 1)
igemm_stg_kernel(const __grid_constant__ Params p, const __grid_constant__ CUtensorMap map_hi, const __grid_constant__ CUtensorMap map_lo,
                 const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_y) {
  using S = Smem<N_TILE, BWT>;
  using MMA = WgmmaBf16<N_TILE>;
  constexpr int STAGES = S::STAGES;
  constexpr int NSLOT = S::NSLOT;
  constexpr bool PLANE = S::PLANE;
  constexpr uint32_t LBO_A = tile_lbo(128);
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* sptr = smem_raw + (sbase - smem_u32(smem_raw));
  const uint32_t bar_full = sbase + S::BAR_OFF;                 // STAGES: 8 converter warps + the filter TMA's expect_tx
  const uint32_t bar_empty = bar_full + 8 * STAGES;             // STAGES: the 4 warps of the consumer warpgroup that owns the stage's tile are done with it
  const uint32_t bar_sfull = bar_empty + 8 * STAGES;            // MAX_SLOTS: staged box landed
  const uint32_t bar_sempty = bar_sfull + 8 * MAX_SLOTS;        // MAX_SLOTS: the converters are done with the box
  int* tapoff = reinterpret_cast<int*>(sptr + S::TAP_OFF);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(bar_full + 8 * s, NCW + 1); mbar_init(bar_empty + 8 * s, 4); }
    for (int b = 0; b < MAX_SLOTS; ++b) { mbar_init(bar_sfull + 8 * b, 1); mbar_init(bar_sempty + 8 * b, NCW); }
    fence_barrier_init();
  }
  if (tid < p.taps) {
    const int i = tid / p.kw, j = tid - i * p.kw;
    tapoff[tid] = ((i - p.ph) * p.W + (j - p.pw)) * 4;          // byte offset inside a staged channel row
  }
  __syncthreads();
  pdl_wait();      // everything above is shared-memory and barrier set-up

  auto stage_b_hi = [&](int s) { return sbase + (uint32_t)s * 2u * S::B_BYTES; };
  auto stage_b_lo = [&](int s) { return sbase + (uint32_t)s * 2u * S::B_BYTES + S::B_BYTES; };
  auto stage_a_hi = [&](int s) { return sbase + S::A_OFF + (uint32_t)s * 2u * S::A_BYTES; };
  auto slot_addr = [&](int slot) { return sbase + S::STG_OFF + (uint32_t)slot * S::SLOT_BYTES; };
  auto tile_coords = [&](int tile, int& m0, int& n0) {
    const int nt = tile % p.n_tiles;
    m0 = (tile / p.n_tiles) * 128; n0 = nt * N_TILE;
  };
  // images a tile touches: 1 or 2 (H*W >= 128); the second one starts at tile row `split`
  // plane mode: nseg = 1 (all the tile's images share one slot), nimg = how many of them there are (<= PLANE_IMGS)
  auto tile_images = [&](int m0, int& n_first, int& nseg, int& split, int& nimg) {
    const int q_last = min(m0 + 128, p.Mtot) - 1;
    n_first = m0 / p.HW;
    nimg = q_last / p.HW - n_first + 1;
    nseg = PLANE ? 1 : nimg;
    split = PLANE ? 128 : (n_first + 1) * p.HW - m0;          // >= 128 when nseg == 1
  };
  const bool prof = p.prof != nullptr && blockIdx.x == 0;

  if (warp >= W_CONV0 && warp < W_CONV0 + NCW) {
    // ================= converters: staged fp32 -> bf16 hi/lo -> A tile in shared memory ========================
    // thread = (GEMM row, channel octets sub and sub + 2 of every 32-channel half block)
    setmaxnreg_dec<REG_CONV>();
    const int cw = warp - W_CONV0;
    const int rq = cw & 3, sub = cw >> 2;
    const int row = rq * 32 + lane;
    const uint32_t a_row = (uint32_t)(row >> 3) * 128u + (uint32_t)(row & 7) * 16u;
    long long c_t0 = 0;
    if (prof) c_t0 = clock64();
    int kbg = 0;                                               // K blocks processed by this CTA (stage ring position)
    int u_base = 0;                                            // staged boxes consumed before this tile
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      int m0, n0, n_first, nseg, split, nimg;
      tile_coords(tile, m0, n0);
      tile_images(m0, n_first, nseg, split, nimg);
      // per-row tap validity (zero padding / image borders / row wrap), once per tile
      uint32_t mask = 0;
      const int seg_r = row >= split ? 1 : 0;                  // which of the tile's images this row belongs to
      // plane mode: the row's image relative to the tile's first one (rows past the batch: any staged address will do)
      const int img_r = PLANE ? (m0 + row < p.Mtot ? (m0 + row) / p.HW - n_first : 0) : seg_r;
      {
        const int q = m0 + row;
        if (q < p.Mtot) {
          const int pp = q - (n_first + img_r) * p.HW;
          const int h = pp / p.W, w = pp - h * p.W;
          if (p.taps == 1) mask = 1u;
          else {
            int t = 0;
            for (int i = 0; i < p.kh; ++i) {
              const bool hok = (unsigned)(h + i - p.ph) < (unsigned)p.H;
              for (int j = 0; j < p.kw; ++j, ++t)
                if (hok && (unsigned)(w + j - p.pw) < (unsigned)p.W) mask |= 1u << t;
            }
          }
        }
      }
      // byte offset of this row at tap offset 0 inside its image's box, plus the channel octet of this warp.  Box column 0
      // is pixel max(first pixel of the segment - halo, 0) of the image rounded DOWN to a multiple of 4: the innermost TMA
      // coordinate has to be 16-byte aligned and never negative; the TMA unit zero-fills past the image END; taps that reach
      // before pixel 0 belong to masked rows, whatever they read is discarded
      // plane mode: whole images are staged, [image][32 channels][H*W]
      const int pp_r = m0 + row - (n_first + img_r) * p.HW;                       // this row's pixel inside its image
      const int start_r = (PLANE || seg_r) ? 0 : max((m0 - n_first * p.HW - p.halo) & ~3, 0);
      const uint32_t row_off = (uint32_t)((pp_r - start_r) * 4) + (uint32_t)(sub * 8) * S::PITCH + (PLANE ? (uint32_t)img_r * S::IMG_BYTES : 0u);
      int g = 0, tap = 0;
      uint32_t src_base = 0;
      for (int kb = 0; kb < p.nkb; ++kb, ++kbg) {
        // one half block at a time: 8 + 8 words live, not 16 + 16.  The first one is converted before waiting for the stage.
        const int s = kbg % STAGES, it = kbg / STAGES;
        const uint32_t a0 = stage_a_hi(s) + a_row;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          uint32_t hi[8], lo[8];                               // [octet o][4 words]
          if (2 * kb + h < p.nhb) {
            const int u0 = u_base + g * nseg;
            if (tap == 0) {                                    // first tap of a channel group: its box(es) must have landed
              mbar_wait(bar_sfull + 8 * (u0 % NSLOT), (u0 / NSLOT) & 1);
              if (nseg == 2) mbar_wait(bar_sfull + 8 * ((u0 + 1) % NSLOT), ((u0 + 1) / NSLOT) & 1);
              src_base = slot_addr((u0 + seg_r) % NSLOT) + row_off;
            }
            const bool ok = (mask >> tap) & 1u;
            const uint32_t src = src_base + (uint32_t)tapoff[tap];
            constexpr int CP = (int)S::PITCH;
            float v[16];
            v[0] = lds32i<0>(src); v[1] = lds32i<CP>(src); v[2] = lds32i<2 * CP>(src); v[3] = lds32i<3 * CP>(src);
            v[4] = lds32i<4 * CP>(src); v[5] = lds32i<5 * CP>(src); v[6] = lds32i<6 * CP>(src); v[7] = lds32i<7 * CP>(src);
            v[8] = lds32i<16 * CP>(src); v[9] = lds32i<17 * CP>(src); v[10] = lds32i<18 * CP>(src); v[11] = lds32i<19 * CP>(src);
            v[12] = lds32i<20 * CP>(src); v[13] = lds32i<21 * CP>(src); v[14] = lds32i<22 * CP>(src); v[15] = lds32i<23 * CP>(src);
#pragma unroll
            for (int o = 0; o < 2; ++o)
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                uint32_t hw, lw;
                split_pack_bf16(v[o * 8 + 2 * e], v[o * 8 + 2 * e + 1], hw, lw);
                hi[o * 4 + e] = ok ? hw : 0u;                  // masked taps contribute exact zeros (never NaN from stale smem)
                lo[o * 4 + e] = ok ? lw : 0u;
              }
            if (++tap == p.taps) {                             // group fully consumed by this warp: hand its box(es) back
              tap = 0;
              __syncwarp();
              if (lane == 0) {
                mbar_arrive(bar_sempty + 8 * (u0 % NSLOT));
                if (nseg == 2) mbar_arrive(bar_sempty + 8 * ((u0 + 1) % NSLOT));
              }
              ++g;
            }
          } else {
#pragma unroll
            for (int o = 0; o < 2; ++o)
#pragma unroll
              for (int e = 0; e < 4; ++e) { hi[o * 4 + e] = 0u; lo[o * 4 + e] = 0u; }   // K padding: finite zeros
          }
          if (h == 0) mbar_wait_backoff(bar_empty + 8 * s, (it & 1) ^ 1, 32);
#pragma unroll
          for (int o = 0; o < 2; ++o) {
            const uint32_t a = a0 + (uint32_t)(h * 4 + sub + 2 * o) * LBO_A;      // 16-byte K chunk = 8 channels
            sts128u(a, hi[o * 4], hi[o * 4 + 1], hi[o * 4 + 2], hi[o * 4 + 3]);
            sts128u(a + S::A_BYTES, lo[o * 4], lo[o * 4 + 1], lo[o * 4 + 2], lo[o * 4 + 3]);
          }
        }
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_full + 8 * s);
      }
      u_base += p.groups * nseg;
    }
    if (prof && cw == 0 && lane == 0) { p.prof[0] = clock64() - c_t0; p.prof[3] = kbg; }
  } else if (warp >= W_BTMA) {
    setmaxnreg_dec<REG_TMA>();
    if (warp == W_BTMA) {
      // ================= filter TMA producer ====================================================================
      int kbg = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        int m0, n0;
        tile_coords(tile, m0, n0);
        for (int kb = 0; kb < p.nkb; ++kb, ++kbg) {
          const int s = kbg % STAGES, it = kbg / STAGES;
          mbar_wait_backoff(bar_empty + 8 * s, (it & 1) ^ 1, 32);
          if (elect_one()) {
            arrive_expect_tx(bar_full + 8 * s, S::TX_BYTES);
            tma_load_3d(stage_b_hi(s), &map_hi, bar_full + 8 * s, kb * BKE, n0, 0);
            tma_load_3d(stage_b_lo(s), &map_lo, bar_full + 8 * s, kb * BKE, n0, 0);
          }
          __syncwarp();
        }
      }
    } else if (warp == W_STG) {
      // ================= activation TMA producer: one box per channel group and image ==============================
      int u = 0;
      long long s_wait = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        int m0, n0, n_first, nseg, split, nimg;
        tile_coords(tile, m0, n0);
        tile_images(m0, n_first, nseg, split, nimg);
        for (int g = 0; g < p.groups; ++g) {
          for (int seg = 0; seg < nseg; ++seg, ++u) {
            const int slot = u % NSLOT;
            if (prof) { const long long t0 = clock64(); mbar_wait_backoff(bar_sempty + 8 * slot, ((u / NSLOT) & 1) ^ 1, 32); s_wait += clock64() - t0; }
            else mbar_wait_backoff(bar_sempty + 8 * slot, ((u / NSLOT) & 1) ^ 1, 32);
            if (elect_one()) {
              if constexpr (PLANE) {
                // the blob viewed as {4*H*W, C/4, N} (four channels per row: a 16-byte multiple pitch); box {4*H*W, 8, 1} is
                // 32 channels of one image, contiguous
                arrive_expect_tx(bar_sfull + 8 * slot, (uint32_t)nimg * S::IMG_BYTES);
                for (int k = 0; k < nimg; ++k)
                  tma_load_3d(slot_addr(slot) + (uint32_t)k * S::IMG_BYTES, &map_x, bar_sfull + 8 * slot, 0, g * (CB / 4), n_first + k);
              } else {
                arrive_expect_tx(bar_sfull + 8 * slot, S::SLOT_BYTES);
                const int col0 = seg ? 0 : max((m0 - n_first * p.HW - p.halo) & ~3, 0);   // 16-byte aligned; columns past the image end read as zero
                tma_load_3d(slot_addr(slot), &map_x, bar_sfull + 8 * slot, col0, g * CB, n_first + seg);
              }
            }
            __syncwarp();
          }
        }
      }
      if (prof && lane == 0) { p.prof[4] = s_wait; p.prof[5] = u; }
    }                                                    // warps 18 and 19: no work
  } else {
    // ================= consumers: ping-pong wgmma + epilogue =====================================================
    // Warpgroup cw owns the CTA's tiles of ordinal j = cw, cw + 2, ... and issues both m64 row halves of each (rows [0, 64)
    // into acc0, [64, 128) into acc1).  Its epilogue then runs while the other warpgroup issues the next tile's MMAs.
    setmaxnreg_inc<REG_CONS>();
    const int cw = warp >> 2, wq = warp & 3, t = tid & 127;
    float* epi = reinterpret_cast<float*>(sptr + S::EPI_OFF + (uint32_t)cw * S::EPI_BYTES);
    const bool issuer = wq == 0;
    float acc0[N_TILE / 2], acc1[N_TILE / 2];
#pragma unroll
    for (int i = 0; i < N_TILE / 2; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
    // profile counters of CTA 0 (B2C_PROF), SM cycles added straight into the zeroed buffer: no registers held across the loop
    long long* const pc = p.prof + 8 + 8 * cw;
    const bool tally = prof && t == 0;
    long long m_t0 = 0;
    if (tally) m_t0 = clock64();
    for (int j = cw, tile = blockIdx.x + cw * (int)gridDim.x; tile < p.total_tiles; j += 2, tile += 2 * (int)gridDim.x) {
      int m0, n0, n_first, nseg, split, nimg;
      tile_coords(tile, m0, n0);
      tile_images(m0, n_first, nseg, split, nimg);
      // Start only once the other warpgroup has seen every K block of tile j - 1 land: the producers fill the stage ring in
      // tile order, so every earlier fill of this tile's stages is then complete and the parity waits below cannot match a
      // phase two behind.  It also keeps the tensor core working on one tile at a time.
      if (j > 0) {
        const long long t0 = tally ? clock64() : 0;
        named_bar(BAR_ORDER + cw, 256);
        if (tally) pc[2] += clock64() - t0;
      }
      int kbg = j * p.nkb;                                 // this tile's position in the stage ring
      int prev = -1;
      for (int kb = 0; kb < p.nkb; ++kb, ++kbg) {
        const int s = kbg % STAGES, it = kbg / STAGES;
        const long long t0 = tally ? clock64() : 0;
        mbar_wait(bar_full + 8 * s, it & 1);
        if (tally) pc[1] += clock64() - t0;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < BKE / 16; ++kk) {
          const uint32_t a = stage_a_hi(s) + 2u * kk * LBO_A;
          const uint64_t ah0 = smem_desc(a, LBO_A, 128), al0 = smem_desc(a + S::A_BYTES, LBO_A, 128);
          const uint64_t ah1 = smem_desc(a + 1024u, LBO_A, 128), al1 = smem_desc(a + 1024u + S::A_BYTES, LBO_A, 128);
          const uint64_t bh = smem_desc_sw128(stage_b_hi(s) + kk * 32), bl = smem_desc_sw128(stage_b_lo(s) + kk * 32);
          MMA::mma(acc0, al0, bh, (kb | kk) != 0);   // lo * hi
          MMA::mma(acc0, ah0, bl, 1);                // hi * lo
          MMA::mma(acc0, ah0, bh, 1);                // hi * hi
          MMA::mma(acc1, al1, bh, (kb | kk) != 0);
          MMA::mma(acc1, ah1, bl, 1);
          MMA::mma(acc1, ah1, bh, 1);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(bar_empty + 8 * prev); }
        prev = s;
      }
      if (tally) pc[5] += p.nkb;
      if (tile + (int)gridDim.x < p.total_tiles) named_bar_arrive(BAR_ORDER + (cw ^ 1), 256);   // tile j + 1 may start
      long long e0 = tally ? clock64() : 0;
      wgmma_wait<0>();
      wgmma_reg_fence(acc0);
      wgmma_reg_fence(acc1);
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty + 8 * prev);
      if (tally) { const long long e1 = clock64(); pc[3] += e1 - e0; e0 = e1; }

      // ---- epilogue: (+ bias) -> 32-channel chunks transposed into this warpgroup's [channel][128 pixels] buffer -> one
      // TMA tensor store per chunk when the tile lies inside one image, else 16-byte st.global; plane mode: per-pixel stores
      // A warp's fragment covers 16 rows and the buffer's row pitch is 128 words, so at best 16 banks take a store: lanes
      // of odd column pairs write element i ^ 2 (row + 8) where the others write element i (2-way conflicts, not 4-way).
      const int sw = (lane & 1) << 1;
      const int nrem = p.Ntot - n0;                        // channels of this tile inside the output
#pragma unroll
      for (int c = 0; c < N_TILE / 32; ++c) {
        const int c0 = c * 32;
        if (c0 >= nrem) break;                             // uniform over the warpgroup
        // the TMA store of the previous chunk has finished reading the buffer (elect.sync on a converged warp always elects
        // the same lane, which owns the bulk-async groups)
        if (issuer && elect_one()) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        named_bar(BAR_EPI + cw, 128);
#pragma unroll
        for (int i = 0; i < N_TILE / 2; ++i)
          if ((i >> 4) == c) {
            const int col = frag_col(t, i), row = frag_row(t, i ^ sw);   // frag_col(t, i ^ 2) == frag_col(t, i)
            float v0 = sw ? acc0[i ^ 2] : acc0[i];
            float v1 = sw ? acc1[i ^ 2] : acc1[i];
            if (p.bias && col < nrem) { const float b = __ldg(p.bias + n0 + col); v0 += b; v1 += b; }
            epi[(col - c0) * 128 + row] = v0;
            epi[(col - c0) * 128 + 64 + row] = v1;
          }
        fence_proxy_async();                               // generic-proxy writes -> visible to the TMA store
        named_bar(BAR_EPI + cw, 128);
        if constexpr (PLANE) {
          // thread = pixel: every channel's store is one (unaligned) 128-byte run per warp
          const int q = m0 + t;
          if (q < p.Mtot) {
            const int nq = q / p.HW;
            float* ob = p.out + ((size_t)nq * p.Ntot + n0 + c0) * p.HW + (q - nq * p.HW);
#pragma unroll 4
            for (int ch = 0; ch < 32; ++ch)
              if (c0 + ch < nrem) { float* d = ob + (size_t)ch * p.HW; const float v = epi[ch * 128 + t]; *d = p.accumulate ? *d + v : v; }
          }
        } else if (nseg == 1 && !(p.dbg & 1)) {
          // the tile lies inside one image: box column 0 = tile row 0 = pixel m0 - n*HW >= 0; columns past the image end
          // (last tile of an image, rows past the batch) and channels past Ntot are clipped by the TMA unit
          if (issuer && elect_one()) {
            if (p.accumulate) tma_reduce_add_3d(&map_y, smem_u32(epi), m0 - n_first * p.HW, n0 + c0, n_first);
            else tma_store_3d(&map_y, smem_u32(epi), m0 - n_first * p.HW, n0 + c0, n_first);
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
          }
        } else {
          // the tile spans two images: 16-byte st.global from the staged chunk, warp = 8 channels, lane = 4 pixels
          const int mv = m0 + lane * 4;                    // H*W % 4 == 0: never across an image end
          if (mv < p.Mtot) {
            const int nv = mv / p.HW, pv = mv - nv * p.HW;
            float* vbase = p.out + ((size_t)nv * p.Ntot + n0 + c0) * p.HW + pv;
#pragma unroll
            for (int q = 0; q < 8; ++q) {
              const int ch = wq * 8 + q;
              if (c0 + ch < nrem) {
                float4 v = *reinterpret_cast<const float4*>(epi + ch * 128 + lane * 4);
                float4* dst = reinterpret_cast<float4*>(vbase + (size_t)ch * p.HW);
                if (p.accumulate) { const float4 o = *dst; v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w; }
                *dst = v;
              }
            }
          }
        }
      }
      if (tally) pc[4] += clock64() - e0;
    }
    if (issuer && elect_one()) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    if (tally) pc[0] = clock64() - m_t0;
  }
  __syncthreads();
}

}  // namespace stg


// ---- host side ------------------------------------------------------------------------------------------------------
static bool stg_enabled() {
  static const int on = env_int("B2C_CONV_STAGED", 1);
  return on != 0;
}

static bool stg_plane_enabled() {
  static const int on = env_int("B2C_CONV_STAGED_PLANE", 1);
  return on != 0;
}

// geometry shared by the eligibility test, the workspace size and the launch
struct StgGeom { int Cin, Cout, halo, bwt, taps, groups, nhb, nkb, Kp; };
static bool stg_geom(const ConvShape& s, int op, StgGeom* g) {
  if (!stg_enabled()) return false;
  if (op != B2C_OP_FORWARD && op != B2C_OP_BACKWARD_DATA) return false;
  if (s.G != 1 || s.sh != 1 || s.sw != 1 || s.dh != 1 || s.dw != 1) return false;
  if (s.Ho != s.H || s.Wo != s.W || 2 * s.ph != s.kh - 1 || 2 * s.pw != s.kw - 1) return false;     // "same" convolution
  const long long HW = (long long)s.H * s.W;
  if ((long long)s.N * HW > 0x7fffffffLL - 256) return false;
  const int Cin = op == B2C_OP_FORWARD ? s.C : s.O, Cout = op == B2C_OP_FORWARD ? s.O : s.C;
  if (Cin % stg::CB != 0 || Cout < 32) return false;
  const int taps = s.kh * s.kw;
  if (taps > stg::MAX_TAPS) return false;
  const int halo = s.ph * s.W + s.pw;
  int bwt;
  if (HW == 49) {
    // 7x7 maps (ResNet-50 res5, GoogLeNet inception 5): a 196-byte channel pitch is not a TMA stride; whole image planes are
    // staged instead ("plane mode", template parameter BWT = H*W)
    if (!stg_plane_enabled()) return false;
    bwt = 49;
  } else {
    if (HW % 4 != 0 || HW < 128) return false;               // 16-byte TMA pitches; <= 2 images per tile
    const int need = 128 + 2 * halo + ((4 - halo % 4) % 4);   // staged pixels per channel (+ what rounding the box start down to 16 bytes costs)
    bwt = need <= 128 ? 128 : need <= 160 ? 160 : need <= 192 ? 192 : need <= 256 ? 256 : 0;   // TMA boxes are <= 256 wide
    if (!bwt) return false;
  }
  if (g) {
    g->Cin = Cin; g->Cout = Cout; g->halo = halo; g->bwt = bwt; g->taps = taps;
    g->groups = Cin / stg::CB; g->nhb = g->groups * taps; g->nkb = (g->nhb + 1) / 2; g->Kp = g->nkb * stg::BKE;
  }
  return true;
}
bool tc_stg_supported(const ConvShape& s, int op) { return stg_geom(s, op, nullptr); }

// The launch's tile plan: 128 consecutive flattened pixels x N_TILE output channels per tile, BWT as the variant
static void stg_plan(const ConvShape& s, const StgGeom& g, ConvPlanInfo* q) {
  *q = ConvPlanInfo{};
  q->n_tile = g.Cout > 64 ? 128 : g.Cout > 32 ? 64 : 32;
  q->m_tiles = (s.N * s.H * s.W + 127) / 128; q->n_tiles = (g.Cout + q->n_tile - 1) / q->n_tile;
  q->tiles = q->m_tiles * q->n_tiles;
  q->nkb = g.nkb;
  q->variant = g.bwt;
}
bool tc_stg_plan_info(const ConvShape& s, int op, ConvPlanInfo* q) {
  StgGeom g;
  if (!stg_geom(s, op, &g)) return false;
  stg_plan(s, g, q);
  return true;
}
size_t tc_stg_workspace(const ConvShape& s, int op) {
  StgGeom g;
  if (!stg_geom(s, op, &g)) return 0;
  return 2 * sizeof(__nv_bfloat16) * (size_t)g.Cout * g.Kp + 256;
}

template <int N_TILE, int BWT>
static int stg_launch_inst(const stg::Params& p, const CUtensorMap& mh, const CUtensorMap& ml, const CUtensorMap& mx, const CUtensorMap& my,
                           cudaStream_t st) {
  using S = stg::Smem<N_TILE, BWT>;
  B2C_CUDA_OK(cudaFuncSetAttribute(stg::igemm_stg_kernel<N_TILE, BWT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)S::TOTAL));
  const int grid = persistent_grid(p.total_tiles);
  launch_pdl(stg::igemm_stg_kernel<N_TILE, BWT>, grid, stg::THREADS, S::TOTAL, st, 0, p, mh, ml, mx, my);
  B2C_POST_LAUNCH();
  return B2C_OK;
}
template <int N_TILE>
static int stg_launch_n(int bwt, const stg::Params& p, const CUtensorMap& mh, const CUtensorMap& ml, const CUtensorMap& mx,
                        const CUtensorMap& my, cudaStream_t st) {
  switch (bwt) {
    case 49: return stg_launch_inst<N_TILE, 49>(p, mh, ml, mx, my, st);
    case 128: return stg_launch_inst<N_TILE, 128>(p, mh, ml, mx, my, st);
    case 160: return stg_launch_inst<N_TILE, 160>(p, mh, ml, mx, my, st);
    case 192: return stg_launch_inst<N_TILE, 192>(p, mh, ml, mx, my, st);
    default: return stg_launch_inst<N_TILE, 256>(p, mh, ml, mx, my, st);
  }
}

// The filter operand of `op` in this kernel's GEMM layout, written into `dst` (tc_stg_workspace(s, op) bytes).
bool tc_stg_prep_entry(const ConvShape& s, int op, const float* w, void* dst, PrepEntry* q) {
  StgGeom g;
  if (!stg_geom(s, op, &g)) return false;
  __nv_bfloat16* wbase = reinterpret_cast<__nv_bfloat16*>((reinterpret_cast<uintptr_t>(dst) + 255) & ~(uintptr_t)255);
  q->w = w; q->kind = 1; q->G = 1; q->Og = s.O; q->Cg = s.C; q->taps = g.taps; q->rows = g.Cout; q->K = g.Cin * g.taps; q->Kp = g.Kp;
  q->mode = op == B2C_OP_FORWARD ? 0 : 1; q->tap_major = 0; q->flip = q->mode; q->kch = g.Cin;
  q->total = (long long)g.Cout * g.Kp;
  q->hi = wbase; q->lo = wbase + q->total;
  return true;
}

// a = x (forward) or dy (dgrad); b = w; out = y or dx; `prepared`: filter already in GEMM layout, or null = prepass here
int launch_conv_tc_stg(const ConvShape& s, int op, const float* a, const float* w, const float* bias, float* out, void* ws,
                       size_t ws_bytes, const void* prepared, bool accumulate, cudaStream_t st) {
  StgGeom g;
  if (!stg_geom(s, op, &g)) return fail(B2C_ERR_INVALID, "staged tensor-core conv: shape not eligible");
  if (!prepared && (!ws || ws_bytes < tc_stg_workspace(s, op))) return fail(B2C_ERR_WORKSPACE, "staged tensor-core conv: workspace too small");
  if ((reinterpret_cast<uintptr_t>(a) & 15u) || (reinterpret_cast<uintptr_t>(out) & 15u))
    return fail(B2C_ERR_INVALID, "staged tensor-core conv: activations must be 16-byte aligned");
  PrepEntry q;
  tc_stg_prep_entry(s, op, w, prepared ? const_cast<void*>(prepared) : ws, &q);
  if (!prepared)
    if (int rc = launch_filter_prep(&q, 1, st)) return rc;

  stg::Params p;
  p.H = s.H; p.W = s.W; p.HW = s.H * s.W;
  p.kh = s.kh; p.kw = s.kw; p.ph = s.ph; p.pw = s.pw;
  p.Mtot = s.N * p.HW; p.Ntot = g.Cout;
  p.taps = g.taps; p.groups = g.groups; p.nhb = g.nhb; p.nkb = g.nkb;
  p.halo = g.halo;
  p.bias = op == B2C_OP_FORWARD ? bias : nullptr;
  p.out = out;
  p.accumulate = accumulate ? 1 : 0;
  static const int dbg = env_int("B2C_STG_DBG", 0);
  p.dbg = dbg;
  ConvPlanInfo plan;
  stg_plan(s, g, &plan);
  const int n_tile = plan.n_tile;
  p.m_tiles = plan.m_tiles; p.n_tiles = plan.n_tiles; p.total_tiles = plan.tiles;
  p.prof = prof_buffer(st);
  alignas(64) CUtensorMap mh, ml, mx, my;
  {
    // filter: [Cout][Kp] bf16, box {64, N_TILE}, SWIZZLE_128B
    const cuuint64_t dims[3] = {(cuuint64_t)g.Kp, (cuuint64_t)g.Cout, 1};
    const cuuint64_t strides[2] = {(cuuint64_t)g.Kp * 2, (cuuint64_t)g.Kp * 2 * (cuuint64_t)g.Cout};
    const cuuint32_t box[3] = {64, (cuuint32_t)n_tile, 1};
    if (int rc = make_tensor_map_3d(&mh, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, q.hi, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B, "staged conv filter"))
      return rc;
    if (int rc = make_tensor_map_3d(&ml, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, q.lo, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B, "staged conv filter"))
      return rc;
  }
  const cuuint64_t HW = (cuuint64_t)p.HW;
  if (g.bwt < 128) {
    // plane mode: the [N][C][HW] blob viewed as {4*HW, C/4, N}; box {4*HW, 8, 1} = 32 channels of one image
    if (int rc = make_tensor_map_3d(&mx, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, a, {HW * 4, (cuuint64_t)g.Cin / 4, (cuuint64_t)s.N},
                                    {HW * 16, HW * 4 * (cuuint64_t)g.Cin}, {(cuuint32_t)HW * 4, (cuuint32_t)stg::CB / 4, 1},
                                    CU_TENSOR_MAP_SWIZZLE_NONE, "staged conv, plane mode"))
      return rc;
    my = mx;                                                  // plane mode stores with st.global
  } else {
    // [N][channels][HW] fp32, box {bw, 32, 1}, no swizzle
    if (int rc = make_tensor_map_3d(&mx, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, a, {HW, (cuuint64_t)g.Cin, (cuuint64_t)s.N},
                                    {HW * 4, HW * 4 * (cuuint64_t)g.Cin}, {(cuuint32_t)g.bwt, (cuuint32_t)stg::CB, 1},
                                    CU_TENSOR_MAP_SWIZZLE_NONE, "staged conv activations"))
      return rc;
    if (int rc = make_tensor_map_3d(&my, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, out, {HW, (cuuint64_t)g.Cout, (cuuint64_t)s.N},
                                    {HW * 4, HW * 4 * (cuuint64_t)g.Cout}, {128, (cuuint32_t)stg::CB, 1},
                                    CU_TENSOR_MAP_SWIZZLE_NONE, "staged conv activations"))
      return rc;
  }
  int rc;
  switch (n_tile) {
    case 128: rc = stg_launch_n<128>(g.bwt, p, mh, ml, mx, my, st); break;
    case 64: rc = stg_launch_n<64>(g.bwt, p, mh, ml, mx, my, st); break;
    default: rc = stg_launch_n<32>(g.bwt, p, mh, ml, mx, my, st); break;
  }
  if (rc == B2C_OK && p.prof) {
    long long h[32];
    prof_read(p.prof, h);
    fprintf(stderr, "[stg-prof] N_TILE=%d BWT=%d nkb=%d groups=%d taps=%d tiles=%d | conv(t0): total=%lld kblocks=%lld | act-tma: wait_empty=%lld boxes=%lld\n",
            n_tile, g.bwt, g.nkb, g.groups, g.taps, p.total_tiles, h[0], h[3], h[4], h[5]);
    // CTA 0's consumer warpgroups, SM cycles: issue = total - wait_full - wait_order - mma_drain - epilogue (issuing MMAs, and
    // waiting behind the other warpgroup's MMAs in the tensor core)
    for (int w = 0; w < 2; ++w) {
      const long long* c = h + 8 + 8 * w;
      fprintf(stderr, "[stg-prof]   consumer wg%d: total=%lld wait_full=%lld wait_order=%lld mma_drain=%lld epilogue=%lld issue=%lld kblocks=%lld\n",
              w, c[0], c[1], c[2], c[3], c[4], c[0] - c[1] - c[2] - c[3] - c[4], c[5]);
    }
  }
  return rc;
}

TC_DEBUG_EXPORT(debug_mbar_stg)

}  // namespace b2c
