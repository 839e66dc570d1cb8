// conv_tc.cu -- wgmma (Hopper tensor core) implicit-GEMM convolution, forward and data-gradient (sm_90a).
//
// Replaces cudnnConvolutionForward / cudnnConvolutionBackwardData as called by the reference's
// CuDNNConvolutionLayer (src/caffe/layers/cudnn_conv_layer.cu:25-29,118-123) and, semantically, the
// per-image forward_gpu_gemm / backward_gpu_gemm loops (base_conv_layer.hpp:105-146): whole batch per
// launch, NCHW fp32 in and out, y / dx overwritten, bias fused, no col buffer in HBM.
//
// GEMM view (batch folded into the pixel dimension):
//   forward : D[q=(n,ho,wo)][o] = sum_k A[q][k] * B[o][k],  A = im2col gather of X, B = filter
//   dgrad   : the same kernel run on dY with the transposed (+ flipped) filter for stride-1 layers, or
//             on the top grid with a strided scatter epilogue for 1x1 / stride>1 / pad 0 layers.
//
// Kernel anatomy -- persistent, one CTA per SM, 128 x N_TILE output tiles, 544 threads:
//   warps 0-7  two consumer warpgroups: wgmma.mma_async.m64nNk8.tf32 from shared-memory descriptors, the fp32
//              accumulators of rows [64 cw, 64 cw + 64) in registers; then the epilogue: accumulators -> shared
//              memory [channel][pixel] -> bias -> coalesced NCHW stores.
//   warps 8-15 A producers.  Two threads per GEMM row (pixel), each owning four of the eight 16-byte K
//              chunks of a K block; the im2col gather reads NCHW global memory directly (coalesced along
//              W) from a per-kernel smem table of chunk offsets (the (c,i,j) decode is the same for every
//              tile), keeps two K blocks of loads in flight in registers across tile boundaries, splits
//              to TF32 hi (+ lo) on the ALU pipe and writes its row of the A tile into shared memory (K-major,
//              no swizzle).  K is ordered (channel/4, tap, channel%4) when C/g % 4 == 0.
//   warp  16   TMA producer for the filter operand: a prepass kernel writes the filter in GEMM-K order,
//              already split into TF32 hi / lo and zero padded to a multiple of 32; cp.async.bulk.tensor
//              (SWIZZLE_128B) drops [N_TILE x 32] boxes into smem, completion on the stage mbarrier.
// The activation operand is not TMA-staged: with NCHW the GEMM-K axis (c,i,j) is not unit-stride and
// 7x7 maps have 196-byte channel pitches (TMA needs 16-byte multiples); see DESIGN.md.
// fp32 math mode = 3 TF32 MMAs per K step (lo*hi, hi*lo, hi*hi); TF32 mode = 1.
#include <limits.h>
#include <stdio.h>
#include "b2c_common.cuh"
#include "tc_common.cuh"
#include "filter_prep.cuh"

namespace b2c {
using namespace tc;

constexpr int NCONS = 8;                    // consumer warps: two warpgroups, tile rows [0, 64) and [64, 128)
constexpr int NPW = 8;                      // A-producer warps
constexpr int W_PROD0 = NCONS;              // first A-producer warp
constexpr int W_TMA = NCONS + NPW;          // filter TMA warp
constexpr int FW_THREADS = (NCONS + NPW + 1) * 32;  // 544
constexpr int TAB_ENTRIES = 1152;   // gather table: one entry per K chunk (KMODE 1) or per K element (KMODE 0)

struct FwdParams {
  // A: activations [Nimg, Cin_tot, H, W]; group g reads channels [g*Cg, (g+1)*Cg)
  const float* x;
  int Cin_tot, H, W, Cg;
  int kh, kw, sh, sw, ph, pw, dh, dw;
  int Ho, Wo;        // pixel grid of the GEMM rows: m = (n*Ho + ho)*Wo + wo
  int Mtot;          // Nimg*Ho*Wo
  int Ntot;          // GEMM columns per group
  int K, Kp;         // true / padded (multiple of 32) reduction length
  // out[(n*Cout_tot + g*Ntot + col)*out_plane + ho*out_hs + wo*out_ws]
  float* out;
  int Cout_tot, out_hs, out_ws;
  long long out_plane;
  const float* bias;  // [G*Ntot] or null
  int m_tiles, n_tiles, G, total_tiles;
  long long* prof;    // optional cycle counters written by CTA 0 (B2C_PROF=1), else null
  int dbg;            // B2C_DBG experiments: 1 = skip the global gather (producer-side ceiling), 2 = skip the MMAs
};

// One pipeline stage: [B hi | B lo | A hi | A lo].  B (filter) is a TMA box in the SWIZZLE_128B K-major layout (1024-byte
// aligned); A (activations) is written by the producers in the padded K-major no-swizzle layout of tc_common.cuh.
template <int N_TILE, bool SPLIT>
struct FwdSmem {
  static constexpr uint32_t B_BYTES = N_TILE * 128u;                       // [N_TILE rows][32 fp32], SW128
  static constexpr uint32_t A_BYTES = tile_bytes(128);                     // [128 rows][32 fp32]
  static constexpr uint32_t NP = SPLIT ? 2u : 1u;
  static constexpr uint32_t B_STAGE = NP * B_BYTES;
  static constexpr uint32_t STAGE = B_STAGE + ((NP * A_BYTES + 1023u) & ~1023u);
  static constexpr uint32_t EPI_BYTES = 32u * 128u * 4u;                   // [32 channels][128 pixels] fp32 (epilogue transpose)
  static constexpr uint32_t FIXED = 256u + TAB_ENTRIES * 8u + EPI_BYTES + 1024u;   // + alignment slack
  static constexpr int STAGES_ = (int)((227u * 1024u - FIXED) / STAGE);
  static constexpr int STAGES = STAGES_ > 6 ? 6 : STAGES_;
  static constexpr uint32_t BAR_OFF = STAGES * STAGE;
  static constexpr uint32_t TAB_OFF = BAR_OFF + 256;
  static constexpr uint32_t EPI_OFF = TAB_OFF + TAB_ENTRIES * 8;
  static constexpr uint32_t TOTAL = EPI_OFF + EPI_BYTES + 1024;
  static constexpr uint32_t TX_BYTES = B_STAGE;
  static_assert(STAGES >= 2, "shared memory budget");
};

// KMODE 0: natural K order (c,i,j), per-element decode (any C/g).
// KMODE 1 (C/g % 4 == 0): K order (c/4, i, j, c%4): a 16-byte chunk = 4 channels of one tap (one bounds check),
// and the kh*kw taps of a channel block are consecutive chunks, so their overlapping pixel windows hit in L1
// instead of re-reading L2 kh*kw times.
template <int N_TILE, bool SPLIT, int KMODE>
__global__ void __launch_bounds__(FW_THREADS, 1)
igemm_fwd_kernel(const __grid_constant__ FwdParams p, const __grid_constant__ CUtensorMap map_hi,
                 const __grid_constant__ CUtensorMap map_lo) {
  using S = FwdSmem<N_TILE, SPLIT>;
  using MMA = WgmmaTf32<N_TILE>;
  constexpr int STAGES = S::STAGES;
  constexpr uint32_t LBO_A = tile_lbo(128);
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;   // SW128 tiles need 1024-byte alignment
  uint8_t* sptr = smem_raw + (sbase - smem_u32(smem_raw));
  const uint32_t bar_full = sbase + S::BAR_OFF;
  const uint32_t bar_empty = bar_full + 8 * STAGES;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nkb = p.Kp / BK;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(bar_full + 8 * s, NPW + 1);   // one elected arrive per producer warp + the TMA thread's expect_tx
      mbar_init(bar_empty + 8 * s, NCONS);    // one arrive per consumer warp once its MMAs have read the stage
    }
    fence_barrier_init();
  }
  // gather table (identical for every tile): element offset inside one image's group slab + tap offsets
  {
    int2* tab = reinterpret_cast<int2*>(sptr + S::TAB_OFF);
    const int HWi = p.H * p.W;
    const int entries = KMODE == 1 ? p.Kp / 4 : p.Kp;
    for (int e = tid; e < entries; e += FW_THREADS) {
      int2 t = make_int2(INT_MIN, 0);
      const int k = KMODE == 1 ? e * 4 : e;
      if (k < p.K) {
        int c, i, j;
        if (KMODE == 1) { const int taps = p.kh * p.kw; const int cb = k / (4 * taps); const int tap = (k - cb * 4 * taps) >> 2;
                          c = cb * 4; i = tap / p.kw; j = tap - i * p.kw; }
        else { c = k / (p.kh * p.kw); const int tap = k - c * p.kh * p.kw; i = tap / p.kw; j = tap - i * p.kw; }
        t.x = c * HWi + i * p.dh * p.W + j * p.dw;
        t.y = (i * p.dh) | ((j * p.dw) << 16);
      }
      tab[e] = t;
    }
  }
  __syncthreads();
  pdl_wait();      // everything above is shared-memory and barrier set-up

  auto stage_b_hi = [&](int s) { return sbase + s * S::STAGE; };
  auto stage_b_lo = [&](int s) { return sbase + s * S::STAGE + S::B_BYTES; };
  auto stage_a_hi = [&](int s) { return sbase + s * S::STAGE + S::B_STAGE; };

  auto tile_coords = [&](int tile, int& m0, int& n0, int& g) {
    const int nt = tile % p.n_tiles;
    const int r = tile / p.n_tiles;
    const int mt = r % p.m_tiles;
    g = r / p.m_tiles;
    m0 = mt * 128; n0 = nt * N_TILE;
  };

  if (warp >= W_PROD0 && warp < W_PROD0 + NPW) {
    // ================= A producers =====================================================================
    // 8 warps: two threads per GEMM row, each owning four of the eight 16-byte K chunks of every K block.  (Twice as
    // many, lighter warps would shorten each warp's dependent chain per K block, but their registers are what the
    // consumers' 128 x 128 fp32 accumulators need.)
    const int2* tab = reinterpret_cast<const int2*>(sptr + S::TAB_OFF);
    const long long HW = (long long)p.H * p.W;
    const int P = p.Ho * p.Wo;
    const int ptid = tid - W_PROD0 * 32;
    const int row = ptid & 127, cp = ptid >> 7;            // chunk quad 0..1 -> chunks 4cp .. 4cp+3 (16 K columns)
    const uint32_t a_off = (uint32_t)(4 * cp) * LBO_A + (uint32_t)(row >> 3) * 128u + (uint32_t)(row & 7) * 16u;
    const int my_tiles = (p.total_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    const int total_blocks = my_tiles * nkb;
    const float* xrow = p.x;
    int ih0 = 0, iw0 = 0;
    bool mvalid = false;
    int lt = 0, lkb = 0;       // load cursor: local tile index, K block inside it

    long long pw_load = 0;
    auto load_block_ = [&](float (&v)[16]) {
      if (lkb == 0) {
        int m0, n0, g;
        tile_coords((int)blockIdx.x + lt * (int)gridDim.x, m0, n0, g);
        const int m = m0 + row;
        mvalid = m < p.Mtot;
        const int mm = mvalid ? m : 0;
        const int n = mm / P, pix = mm - n * P;
        const int ho = pix / p.Wo, wo = pix - ho * p.Wo;
        ih0 = ho * p.sh - p.ph; iw0 = wo * p.sw - p.pw;
        xrow = p.x + ((long long)n * p.Cin_tot + (long long)g * p.Cg) * HW + (long long)ih0 * p.W + iw0;
      }
      if (p.dbg & 1) {
#pragma unroll
        for (int e = 0; e < 16; ++e) v[e] = 1.0f;
      } else if (KMODE == 1) {
        const int2* te = tab + lkb * KCHUNKS + cp * 4;
#pragma unroll
        for (int ch = 0; ch < 4; ++ch) {
          const int2 tt = te[ch];
          const bool ok = mvalid && tt.x != INT_MIN && (unsigned)(ih0 + (tt.y & 0xffff)) < (unsigned)p.H &&
                          (unsigned)(iw0 + (tt.y >> 16)) < (unsigned)p.W;
          const float* src = xrow + tt.x;
#pragma unroll
          for (int e = 0; e < 4; ++e) v[ch * 4 + e] = ok ? __ldg(src + e * HW) : 0.0f;
        }
      } else {
        const int2* te = tab + lkb * BK + cp * 16;
#pragma unroll
        for (int e = 0; e < 16; ++e) {
          const int2 tt = te[e];
          const bool ok = mvalid && tt.x != INT_MIN && (unsigned)(ih0 + (tt.y & 0xffff)) < (unsigned)p.H &&
                          (unsigned)(iw0 + (tt.y >> 16)) < (unsigned)p.W;
          v[e] = ok ? __ldg(xrow + tt.x) : 0.0f;
        }
      }
      if (++lkb == nkb) { lkb = 0; ++lt; }
    };
    auto load_block = [&](float (&v)[16]) { const long long a0 = clock64(); load_block_(v); pw_load += clock64() - a0; };
    int kbg = 0;   // pipeline position of the store cursor
    long long pw_empty = 0, pw_store = 0;
    const long long pt0 = clock64();
    auto store_block = [&](const float (&v)[16]) {
      const int s = kbg % STAGES, it = kbg / STAGES;
      const long long t0 = clock64();
      mbar_wait_backoff(bar_empty + 8 * s, (it & 1) ^ 1, 40);
      const long long t1 = clock64();
      const uint32_t a_hi = stage_a_hi(s) + a_off;
#pragma unroll
      for (int ch = 0; ch < 4; ++ch)
        store_chunk<SPLIT>(a_hi + ch * LBO_A, a_hi + ch * LBO_A + S::A_BYTES, v[4 * ch], v[4 * ch + 1], v[4 * ch + 2], v[4 * ch + 3]);
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_full + 8 * s);
      ++kbg;
      pw_empty += t1 - t0; pw_store += clock64() - t1;
    };

    // two K blocks of loads in flight ahead of the block being stored, across tile boundaries
    float v0[16], v1[16], v2[16];
    int issued = 0;
    if (issued < total_blocks) { load_block(v0); ++issued; }
    if (issued < total_blocks) { load_block(v1); ++issued; }
    for (int j = 0; j < total_blocks; j += 3) {
      if (issued < total_blocks) { load_block(v2); ++issued; }
      store_block(v0);
      if (j + 1 >= total_blocks) break;
      if (issued < total_blocks) { load_block(v0); ++issued; }
      store_block(v1);
      if (j + 2 >= total_blocks) break;
      if (issued < total_blocks) { load_block(v1); ++issued; }
      store_block(v2);
    }
    if (p.prof && blockIdx.x == 0 && ptid == 0) {
      p.prof[0] = clock64() - pt0; p.prof[1] = pw_empty; p.prof[2] = pw_store; p.prof[3] = pw_load; p.prof[4] = total_blocks;
    }
  } else if (warp == W_TMA) {
    // ================= TMA producer (filter operand) ===================================================
    // (whole warp runs the loop converged; one elected lane issues)
    int kbg = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      int m0, n0, g;
      tile_coords(tile, m0, n0, g);
      for (int kb = 0; kb < nkb; ++kb, ++kbg) {
        const int s = kbg % STAGES, it = kbg / STAGES;
        mbar_wait_backoff(bar_empty + 8 * s, (it & 1) ^ 1, 40);
        if (elect_one()) {
          arrive_expect_tx(bar_full + 8 * s, S::TX_BYTES);
          tma_load_3d(stage_b_hi(s), &map_hi, bar_full + 8 * s, kb * BK, n0, g);
          if (SPLIT) tma_load_3d(stage_b_lo(s), &map_lo, bar_full + 8 * s, kb * BK, n0, g);
        }
        __syncwarp();
      }
    }
  } else if (warp < NCONS) {
    // ================= consumers: wgmma (accumulators in registers) + epilogue ==============================
    // warpgroup cw owns tile rows [64 cw, 64 cw + 64); a stage is released once the MMAs of the NEXT stage are
    // issued (wgmma.wait_group 1), so the tensor core always has the following K block queued.
    const int cw = warp >> 2, t = tid & 127;
    const int P = p.Ho * p.Wo;
    float* epi = reinterpret_cast<float*>(sptr + S::EPI_OFF);
    const bool vec_epi = p.out_ws == 1 && p.out_hs == p.Wo && (P & 3) == 0 && (p.out_plane & 3) == 0 &&
                         (reinterpret_cast<uintptr_t>(p.out) & 15u) == 0 && !(p.dbg & 16);
    float acc[N_TILE / 2];
#pragma unroll
    for (int i = 0; i < N_TILE / 2; ++i) acc[i] = 0.f;
    int kbg = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      int m0, n0, g;
      tile_coords(tile, m0, n0, g);
      int prev = -1;
      for (int kb = 0; kb < nkb; ++kb, ++kbg) {
        const int s = kbg % STAGES, it = kbg / STAGES;
        mbar_wait(bar_full + 8 * s, it & 1);
        wgmma_fence();
        if (!(p.dbg & 2)) {
#pragma unroll
          for (int kk = 0; kk < BK / 8; ++kk) {
            const uint32_t a = stage_a_hi(s) + 2u * kk * LBO_A + (uint32_t)cw * 1024u;
            const uint64_t ah = smem_desc(a, LBO_A, 128);
            const uint64_t bh = smem_desc_sw128(stage_b_hi(s) + kk * 32);
            if (SPLIT) {
              const uint64_t al = smem_desc(a + S::A_BYTES, LBO_A, 128);
              const uint64_t bl = smem_desc_sw128(stage_b_lo(s) + kk * 32);
              MMA::mma(acc, al, bh, (kb | kk) != 0);   // lo * hi
              MMA::mma(acc, ah, bl, 1);                // hi * lo
              MMA::mma(acc, ah, bh, 1);                // hi * hi
            } else {
              MMA::mma(acc, ah, bh, (kb | kk) != 0);
            }
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(bar_empty + 8 * prev); }
        prev = s;
      }
      wgmma_wait<0>();
      wgmma_reg_fence(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty + 8 * prev);

      // ---- epilogue: 32-channel chunks transposed through shared memory [channel][128 pixels], then stored
      const float* brow = p.bias ? p.bias + (long long)g * p.Ntot + n0 : nullptr;
      const int r = tid & 127, half = tid >> 7;            // row-per-thread store path: channels [16 half, 16 half + 16)
      const int m = m0 + r;
      const bool mvalid = m < p.Mtot;
      float* orow;
      {
        const int mm = mvalid ? m : 0;
        const int n = mm / P, pix = mm - n * P;
        const int ho = pix / p.Wo, wo = pix - ho * p.Wo;
        orow = p.out + ((long long)n * p.Cout_tot + (long long)g * p.Ntot + n0) * p.out_plane +
               (long long)ho * p.out_hs + (long long)wo * p.out_ws;
      }
      const int mv = m0 + lane * 4;                        // vector path: this lane's 4 pixels
      const bool mv_ok = mv < p.Mtot;                      // P % 4 == 0: the group is valid or not as a whole
      float* vbase;
      {
        const int nv = (mv_ok ? mv : 0) / P, pv = (mv_ok ? mv : 0) - ((mv_ok ? mv : 0) / P) * P;
        vbase = p.out + ((long long)nv * p.Cout_tot + (long long)g * p.Ntot + n0) * p.out_plane + pv;
      }
#pragma unroll
      for (int c = 0; c < N_TILE / 32; ++c) {
        const int c0 = c * 32;
        if (n0 + c0 >= p.Ntot) break;                      // uniform over the consumers
        named_bar(1, NCONS * 32);                          // the previous chunk's stores have read the staging buffer
#pragma unroll
        for (int i = 0; i < N_TILE / 2; ++i)
          if ((i >> 4) == c) epi[(frag_col(t, i) - c0) * 128 + cw * 64 + frag_row(t, i)] = acc[i];
        named_bar(1, NCONS * 32);
        if (p.dbg & 4) continue;
        if (vec_epi) {
          // contiguous output planes: one warp instruction writes 128 consecutive pixels of a channel (512 B per request)
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int ch = warp * 4 + q;
            if (mv_ok && n0 + c0 + ch < p.Ntot) {
              float4 v = *reinterpret_cast<const float4*>(epi + ch * 128 + lane * 4);
              if (brow) { const float b = __ldg(brow + c0 + ch); v.x += b; v.y += b; v.z += b; v.w += b; }
              *reinterpret_cast<float4*>(vbase + (long long)(c0 + ch) * p.out_plane) = v;
            }
          }
        } else if (mvalid) {
#pragma unroll 4
          for (int j = 0; j < 16; ++j) {
            const int ch = half * 16 + j;
            if (n0 + c0 + ch < p.Ntot) {
              float v = epi[ch * 128 + r];
              if (brow) v += __ldg(brow + c0 + ch);
              orow[(long long)(c0 + ch) * p.out_plane] = v;
            }
          }
        }
      }
    }
  }
  __syncthreads();
}

// ---- host side ---------------------------------------------------------------------------------------------
template <int N_TILE, bool SPLIT, int KMODE>
static int launch_fwd_inst(const FwdParams& p, const CUtensorMap& mh, const CUtensorMap& ml, cudaStream_t st) {
  using S = FwdSmem<N_TILE, SPLIT>;
  // per-device attribute: set on every launch (a process may drive several GPUs)
  B2C_CUDA_OK(cudaFuncSetAttribute(igemm_fwd_kernel<N_TILE, SPLIT, KMODE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)S::TOTAL));
  const int grid = persistent_grid(p.total_tiles);
  launch_pdl(igemm_fwd_kernel<N_TILE, SPLIT, KMODE>, grid, FW_THREADS, S::TOTAL, st, 0, p, mh, ml);
  B2C_POST_LAUNCH();
  return B2C_OK;
}

template <int N_TILE>
static int launch_fwd_n(const FwdParams& p, const CUtensorMap& mh, const CUtensorMap& ml, int math, int kmode,
                        cudaStream_t st) {
  if (math == B2C_MATH_FP32)
    return kmode ? launch_fwd_inst<N_TILE, true, 1>(p, mh, ml, st) : launch_fwd_inst<N_TILE, true, 0>(p, mh, ml, st);
  return kmode ? launch_fwd_inst<N_TILE, false, 1>(p, mh, ml, st) : launch_fwd_inst<N_TILE, false, 0>(p, mh, ml, st);
}

// N tile choice: the producers stage 16 KB of TF32 hi/lo per K block regardless of N, so narrow tiles are
// staging-bound; 128 (64 accumulator registers per consumer thread) whenever the layer has more than 64 output
// columns, else the smallest tile that covers them.
static int pick_n_tile(int Ntot) {
  if (Ntot > 64) return 128;
  if (Ntot > 32) return 64;
  return 32;
}

static bool dgrad_as_fwd(const ConvShape& s) { return s.sh == 1 && s.sw == 1; }
static bool dgrad_scatter(const ConvShape& s) { return s.kh == 1 && s.kw == 1 && s.ph == 0 && s.pw == 0 && (s.sh > 1 || s.sw > 1); }

static int padded_k(int K) { return (K + BK - 1) / BK * BK; }

bool tc_conv_supported(const ConvShape& s, int op) {
  const long long Mtot = (long long)s.N * s.Ho * s.Wo;
  if (Mtot > 0x7fffffffLL || (long long)s.N * s.H * s.W > 0x7fffffffLL) return false;
  if ((long long)s.C * s.H * s.W >= 0x7fffffffLL || (long long)s.O * s.Ho * s.Wo >= 0x7fffffffLL) return false;
  if ((s.kh - 1) * s.dh > 0x7fff || (s.kw - 1) * s.dw > 0x7fff) return false;
  auto table_fits = [](int K, int chan) { const int Kp = (K + 31) / 32 * 32; return (chan % 4 == 0 ? Kp / 4 : Kp) <= TAB_ENTRIES; };
  if (op == B2C_OP_FORWARD) return table_fits(s.Kd, s.Cg);
  if (op == B2C_OP_BACKWARD_DATA) return (dgrad_as_fwd(s) || dgrad_scatter(s)) && table_fits(s.Og * s.kh * s.kw, s.Og);
  return tc_wgrad_supported(s);
}

size_t tc_conv_workspace(const ConvShape& s, int op, int math) {
  const size_t np = math == B2C_MATH_FP32 ? 2 : 1;
  if (op == B2C_OP_FORWARD) return sizeof(float) * np * (size_t)s.O * padded_k(s.Kd) + 256;
  if (op == B2C_OP_BACKWARD_DATA) return sizeof(float) * np * (size_t)s.C * padded_k(s.Og * s.kh * s.kw) + 256;
  return tc_wgrad_workspace(s);
}

// The filter operand of `op` in this kernel's GEMM layout, written into `dst` (tc_conv_workspace(s, op, math) bytes).
void tc_conv_prep_entry(const ConvShape& s, int op, int math, const float* w, void* dst, PrepEntry* q) {
  float* wbase = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(dst) + 255) & ~(uintptr_t)255);
  const int chan = op == B2C_OP_FORWARD ? s.Cg : s.Og;
  q->w = w; q->kind = 0; q->G = s.G; q->Og = s.Og; q->Cg = s.Cg; q->taps = s.kh * s.kw;
  q->mode = op == B2C_OP_FORWARD ? 0 : 1;
  q->rows = op == B2C_OP_FORWARD ? s.Og : s.Cg;
  q->K = chan * s.kh * s.kw; q->Kp = padded_k(q->K);
  q->tap_major = (chan % 4 == 0) ? 1 : 0;
  q->flip = (op == B2C_OP_BACKWARD_DATA && dgrad_as_fwd(s)) ? 1 : 0;
  q->kch = chan;
  q->total = (long long)s.G * q->rows * q->Kp;
  q->hi = wbase;
  q->lo = math == B2C_MATH_FP32 ? static_cast<void*>(wbase + q->total) : nullptr;
}

// The kernel's view of `op` on shape `s`: gather geometry, GEMM extents and output strides.  Pointers, bias and the tile plan
// are left to the caller.
static FwdParams fwd_params(const ConvShape& s, int op) {
  FwdParams p{};
  if (op == B2C_OP_FORWARD) {
    p.Cin_tot = s.C; p.H = s.H; p.W = s.W; p.Cg = s.Cg;
    p.kh = s.kh; p.kw = s.kw; p.sh = s.sh; p.sw = s.sw; p.ph = s.ph; p.pw = s.pw; p.dh = s.dh; p.dw = s.dw;
    p.Ho = s.Ho; p.Wo = s.Wo; p.Mtot = s.N * s.Ho * s.Wo;
    p.Ntot = s.Og; p.K = s.Kd;
    p.Cout_tot = s.O; p.out_plane = (long long)s.Ho * s.Wo; p.out_hs = s.Wo; p.out_ws = 1;
  } else {
    // x = dy [N,O,Ho,Wo], out = dx [N,C,H,W]
    p.Cin_tot = s.O; p.Cg = s.Og;
    p.Ntot = s.Cg; p.K = s.Og * s.kh * s.kw;
    p.Cout_tot = s.C; p.out_plane = (long long)s.H * s.W;
    if (dgrad_as_fwd(s)) {
      // stride-1 conv of dY with the flipped filter, pad' = (k-1)*d - p, rows = bottom pixels
      p.H = s.Ho; p.W = s.Wo;
      p.kh = s.kh; p.kw = s.kw; p.sh = 1; p.sw = 1; p.dh = s.dh; p.dw = s.dw;
      p.ph = (s.kh - 1) * s.dh - s.ph; p.pw = (s.kw - 1) * s.dw - s.pw;
      p.Ho = s.H; p.Wo = s.W; p.Mtot = s.N * s.H * s.W;
      p.out_hs = s.W; p.out_ws = 1;
    } else {
      // 1x1, stride > 1, pad 0: rows = top pixels, scatter to bottom[ho*sh][wo*sw]; the rest of dx is 0 (memset by the launch)
      p.H = s.Ho; p.W = s.Wo;
      p.kh = 1; p.kw = 1; p.sh = 1; p.sw = 1; p.dh = 1; p.dw = 1; p.ph = 0; p.pw = 0;
      p.Ho = s.Ho; p.Wo = s.Wo; p.Mtot = s.N * s.Ho * s.Wo;
      p.out_hs = s.sh * s.W; p.out_ws = s.sw;
    }
  }
  p.Kp = padded_k(p.K);
  p.G = s.G;
  return p;
}

// The tile plan of the launch for these GEMM extents: N_TILE (pick_n_tile, or the B2C_NTILE override where it is wider than half
// the columns), tile counts, K blocks and KMODE.
static void plan_tiles(const FwdParams& p, ConvPlanInfo* q) {
  int n_tile = pick_n_tile(p.Ntot);
  static const int force = env_int("B2C_NTILE", 0);
  if ((force == 32 || force == 64 || force == 128) && force / 2 < p.Ntot) n_tile = force;
  q->n_tile = n_tile;
  q->m_tiles = (p.Mtot + 127) / 128; q->n_tiles = (p.Ntot + n_tile - 1) / n_tile;
  q->tiles = q->m_tiles * q->n_tiles * p.G;
  q->nkb = p.Kp / BK;
  q->variant = (p.Cg % 4 == 0) ? 1 : 0;
}

void tc_conv_plan_info(const ConvShape& s, int op, ConvPlanInfo* q) {
  *q = ConvPlanInfo{};
  plan_tiles(fwd_params(s, op), q);
}
bool tc_conv_scatter(const ConvShape& s, int op) { return op == B2C_OP_BACKWARD_DATA && !dgrad_as_fwd(s); }

static int launch_gather(FwdParams& p, const PrepEntry& q, int math, cudaStream_t st);

// `prepared`: the filter already in GEMM layout (b2c_conv_prepare_filter) or null = run the prepass here into `ws`
int launch_conv_tc(const ConvShape& s, int op, int math, const float* a, const float* b, const float* bias, float* out,
                   void* ws, size_t ws_bytes, const void* prepared, cudaStream_t st) {
  if (op == B2C_OP_BACKWARD_FILTER) return launch_conv_tc_wgrad(s, math, a, b, out, ws, ws_bytes, st);
  if (!prepared && (ws_bytes < tc_conv_workspace(s, op, math) || !ws)) return fail(B2C_ERR_WORKSPACE, "tensor-core conv: workspace too small");
  PrepEntry q;
  tc_conv_prep_entry(s, op, math, b, prepared ? const_cast<void*>(prepared) : ws, &q);
  FwdParams p = fwd_params(s, op);
  p.x = a; p.out = out;
  p.bias = op == B2C_OP_FORWARD ? bias : nullptr;
  if (tc_conv_scatter(s, op))
    B2C_CUDA_OK(cudaMemsetAsync(out, 0, sizeof(float) * (size_t)s.N * s.C * s.H * s.W, st));
  static const int dbg = env_int("B2C_DBG", 0);
  p.dbg = dbg;
  if (!prepared)
    if (int rc = launch_filter_prep(&q, 1, st)) return rc;
  return launch_gather(p, q, math, st);
}

// The gather kernel on the GEMM `p` describes, its filter operand prepared in q's planes (geometry, pointers and bias set by the
// caller; the tile plan and the debug switches set here).
static int launch_gather(FwdParams& p, const PrepEntry& q, int math, cudaStream_t st) {
  ConvPlanInfo plan;
  plan_tiles(p, &plan);
  const int n_tile = plan.n_tile, kmode = plan.variant;
  p.m_tiles = plan.m_tiles; p.n_tiles = plan.n_tiles; p.total_tiles = plan.tiles;
  alignas(64) CUtensorMap mh, ml;
  const cuuint64_t dims[3] = {(cuuint64_t)p.Kp, (cuuint64_t)q.rows, (cuuint64_t)p.G};
  const cuuint64_t strides[2] = {(cuuint64_t)p.Kp * 4, (cuuint64_t)p.Kp * 4 * (cuuint64_t)q.rows};
  const cuuint32_t box[3] = {32, (cuuint32_t)n_tile, 1};
  if (int rc = make_tensor_map_3d(&mh, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, q.hi, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B, "conv filter"))
    return rc;
  if (int rc = make_tensor_map_3d(&ml, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, q.lo ? q.lo : q.hi, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                                  "conv filter"))
    return rc;
  p.prof = prof_buffer(st);
  int rc;
  switch (n_tile) {
    case 128: rc = launch_fwd_n<128>(p, mh, ml, math, kmode, st); break;
    case 64: rc = launch_fwd_n<64>(p, mh, ml, math, kmode, st); break;
    default: rc = launch_fwd_n<32>(p, mh, ml, math, kmode, st); break;
  }
  if (p.prof) {
    long long h[32];
    prof_read(p.prof, h);
    fprintf(stderr, "[prof] N_TILE=%d nkb=%d tiles=%d | producer(t0): total=%lld wait_empty=%lld store=%lld load=%lld blocks=%lld\n",
            n_tile, p.Kp / 32, p.total_tiles, h[0], h[1], h[2], h[3], h[4]);
  }
  return rc;
}

// ---- transposed convolution, one output phase (deconv.cu): a stride-1 gather GEMM over the bottom whose epilogue writes the
// phase's lattice of the top through out_hs / out_ws, starting at (a.t0, b.t0)
static FwdParams deconv_phase_params(const ConvShape& dual, const DeconvPhaseAxis& a, const DeconvPhaseAxis& b) {
  FwdParams p{};
  p.Cin_tot = dual.O; p.Cg = dual.Og; p.H = dual.Ho; p.W = dual.Wo;
  p.kh = a.n; p.kw = b.n; p.sh = 1; p.sw = 1; p.ph = a.pad; p.pw = b.pad; p.dh = a.dd; p.dw = b.dd;
  p.Ho = a.M; p.Wo = b.M; p.Mtot = dual.N * a.M * b.M;
  p.Ntot = dual.Cg; p.K = dual.Og * a.n * b.n; p.Kp = padded_k(p.K);
  p.Cout_tot = dual.C; p.out_plane = (long long)dual.H * dual.W; p.out_hs = dual.sh * dual.W; p.out_ws = dual.sw;
  p.G = dual.G;
  return p;
}
bool tc_deconv_phase_supported(const ConvShape& dual, const DeconvPhaseAxis& a, const DeconvPhaseAxis& b) {
  if ((long long)dual.N * a.M * b.M > 0x7fffffffLL || (long long)dual.N * dual.Ho * dual.Wo > 0x7fffffffLL) return false;
  if ((long long)dual.O * dual.Ho * dual.Wo >= 0x7fffffffLL || (long long)dual.C * dual.H * dual.W >= 0x7fffffffLL) return false;
  if ((a.n - 1) * a.dd > 0x7fff || (b.n - 1) * b.dd > 0x7fff) return false;
  const int Kp = padded_k(dual.Og * a.n * b.n);
  return (dual.Og % 4 == 0 ? Kp / 4 : Kp) <= TAB_ENTRIES;
}
size_t tc_deconv_phase_prep_bytes(const ConvShape& dual, const DeconvPhaseAxis& a, const DeconvPhaseAxis& b, int math) {
  const size_t np = math == B2C_MATH_FP32 ? 2 : 1;
  return sizeof(float) * np * (size_t)dual.G * dual.Cg * padded_k(dual.Og * a.n * b.n);
}
// dst: 256-byte aligned, tc_deconv_phase_prep_bytes long
void tc_deconv_phase_prep_entry(const ConvShape& dual, const DeconvPhaseAxis& a, const DeconvPhaseAxis& b, int math, const float* w,
                                void* dst, PrepEntry* q) {
  *q = PrepEntry{};
  float* wbase = static_cast<float*>(dst);
  q->w = w; q->kind = 0; q->G = dual.G; q->Og = dual.Og; q->Cg = dual.Cg; q->taps = a.n * b.n;
  q->mode = 2; q->rows = dual.Cg;
  q->K = dual.Og * a.n * b.n; q->Kp = padded_k(q->K);
  q->tap_major = (dual.Og % 4 == 0) ? 1 : 0;
  q->flip = 0; q->kch = dual.Og;
  q->src_taps = dual.kh * dual.kw; q->src_kw = dual.kw; q->sub_kh = a.n; q->sub_kw = b.n;
  q->i0h = a.i0; q->i0w = b.i0; q->Lh = a.L; q->Lw = b.L;
  q->total = (long long)dual.G * q->rows * q->Kp;
  q->hi = wbase;
  q->lo = math == B2C_MATH_FP32 ? static_cast<void*>(wbase + q->total) : nullptr;
}
void tc_deconv_phase_plan_info(const ConvShape& dual, const DeconvPhaseAxis& a, const DeconvPhaseAxis& b, ConvPlanInfo* q) {
  *q = ConvPlanInfo{};
  plan_tiles(deconv_phase_params(dual, a, b), q);
}
int launch_deconv_phase_tc(const ConvShape& dual, const DeconvPhaseAxis& a, const DeconvPhaseAxis& b, int math, const float* x,
                           const float* bias, float* out, const PrepEntry& q, cudaStream_t st) {
  FwdParams p = deconv_phase_params(dual, a, b);
  p.x = x; p.bias = bias;
  p.out = out + (long long)a.t0 * dual.W + b.t0;
  return launch_gather(p, q, math, st);
}

TC_DEBUG_EXPORT(debug_mbar_fwd)

}  // namespace b2c
