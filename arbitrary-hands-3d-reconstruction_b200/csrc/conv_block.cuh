// One HRNet BasicBlock (conv3x3-BN-ReLU, conv3x3-BN, + block input, ReLU) as ONE wgmma launch, sm_90a.
//
// Two conv_tc launches move five activation passes through HBM per block (read x, write y, read y, write the output,
// read x again as the residual); this kernel moves two (read x, write the output; the residual re-read of the tile just
// loaded hits L2).  The intermediate y never leaves shared memory.
//
// Per 16x16 output super-tile (persistent CTAs, the conv_tc_kernel warp layout: four consumer warpgroups, one producer):
//   * Input: ONE TMA box {64 ch, 24-pixel pitch, 20 rows} from (x0-2, y0-2): a two-pixel halo, TMA's out-of-bounds
//     zeros are conv1's padding.  x-paired blocks (dense 32-channel tensors, ACR_CONV_XPAIR) count the box in pixel pairs.
//   * conv1 over the 18x18 intermediate region (the tile plus conv2's one-pixel halo), "flat M": the pitch-24 box is a
//     flat array of pixels and intermediate pixel p = r * 24 + c reads input pixel p + ky * 24 + kx for tap (ky, kx), a
//     constant offset.  So every M = 64 block is 64 consecutive flat pixels (8 core groups of 8, SBO = 1024 B) and a tap
//     is a descriptor start (ky * 24 + kx) * 128 B into the box -- an unaligned start, like MODE_P1 (the 128B swizzle
//     follows the absolute address).  18 x 24 = 432 flat pixels take 7 M blocks; warpgroup g owns blocks g and g + 4,
//     so warpgroup 3 also computes a discarded 8th block: a warpgroup-dependent branch around the wgmmas makes ptxas
//     serialise them, and warpgroup 3 would wait at the barrier after conv1 anyway.  The last blocks read up to 82
//     pixels past the box: a zeroed slack region (those reads only feed discarded flat rows).
//   * conv1 epilogue IN PLACE: once every conv1 wgmma of the tile has completed (a barrier over the consumers), bias +
//     ReLU, rounded to 16 bits, is stored over the box in the 128B-swizzled K-major layout TMA would have written (16-byte
//     chunk index ^= pixel & 7), 18 rows at pitch 24.  Pixels outside the image are stored as ZERO: they are conv2's
//     padding.  Columns 18..23 are never read.  Then fence.proxy.async and a second barrier: conv2's taps read rows
//     written by other warpgroups.
//   * conv2 reads the intermediate with the MODE_P1 addressing (8x8-pixel M blocks at pitch 24, taps = descriptor
//     starts); once its wgmmas completed the box is handed back to the producer, whose next load overlaps conv2's
//     epilogue (bias, residual from global, ReLU, NHWC stores).
//   * Both weight sets stay resident (2 x 72 KB); box 60 KB + slack.  That is why the intermediate overwrites the box.
//   * Bit-identical to the two conv_tc launches: every accumulator sums its taps and k-steps in the standalone order
//     (ky-major, kx 0,1,2; x-paired: kx 1,0,2, side taps as full-width MMAs over zero weight quarters), the epilogues do
//     the same float operations, and the intermediate is rounded to 16 bits in both paths.
//   * `mid` (optional): conv1's output is also stored for the tile's own 16x16 pixels, so an observable intermediate
//     (teacher-forced checks, kept tensors) is still written.
#pragma once
#include "conv_tc.cuh"

namespace acr {

constexpr int BLK_PITCH = 24, BLK_ROWS = 20;                       // input box: 24 x 20 pixels (pairs), two-pixel halo
constexpr int BLK_MID = 18;                                        // intermediate region: 18 x 18 at pitch 24
constexpr uint32_t BLK_ROW_BYTES = 128;                            // 64 16-bit channels
constexpr uint32_t BLK_W_BYTES = 9u * 64u * BLK_ROW_BYTES;         // one conv's resident weights: 9 taps x [64][64]
constexpr uint32_t BLK_BOX_BYTES = (uint32_t)BLK_PITCH * BLK_ROWS * BLK_ROW_BYTES;
constexpr int BLK_M_BLOCKS = 8;   // 7 cover the 432 flat pixels; the 8th keeps every warpgroup's wgmma sequence identical
constexpr int BLK_SLACK_PIX = BLK_M_BLOCKS * 64 + 2 * BLK_PITCH + 2 - BLK_PITCH * BLK_ROWS;
constexpr uint32_t BLK_SLACK_BYTES = (uint32_t)BLK_SLACK_PIX * BLK_ROW_BYTES;
constexpr uint32_t BLK_OFF_B2 = BLK_W_BYTES;
constexpr uint32_t BLK_OFF_A = 2 * BLK_W_BYTES;
constexpr uint32_t BLK_OFF_BIAS = BLK_OFF_A + BLK_BOX_BYTES + BLK_SLACK_BYTES;
constexpr uint32_t BLK_OFF_BAR = BLK_OFF_BIAS + 2 * 64 * 4;
constexpr size_t BLK_SMEM = 1024 /*alignment slack*/ + BLK_OFF_BAR + 64;
static_assert(BLK_SLACK_PIX == 82 && (BLK_M_BLOCKS - 1) * 64 >= BLK_MID * BLK_PITCH, "flat-M plan: 8 M blocks of 64 read 82 pixels past the box");
static_assert(BLK_MID * BLK_PITCH * BLK_ROW_BYTES <= BLK_BOX_BYTES, "the intermediate fits in the box it overwrites");
static_assert(BLK_SMEM <= (size_t)SMEM_BUDGET, "fused-block shared-memory plan exceeds the budget");
constexpr int BLK_BAR = 1;   // named barrier over the 512 consumer threads

struct ConvBlockParams {
  CUtensorMap tmA;          // block input x {C, W, H, B}, box {64, 24, 20}
  CUtensorMap tmB1, tmB2;   // packed weights of conv1 / conv2 [64][9 * 64], box {64, 64}
  const float* bias1;
  const float* bias2;
  const void* res;          // the block input again (residual of conv2)
  void* out;
  void* mid;                // conv1's output buffer, or nullptr when nothing reads it
  int res_stride, out_stride, mid_stride;
  int H, W, tiles_x, tiles_per_img, total_tiles;
};

// the wgmmas of one tap of one accumulator (x-paired side taps: the two k-steps of their K half, see conv_tc_kernel)
template <typename T, bool XPAIR>
__device__ __forceinline__ void blk_tap(float* acc, uint32_t a_lo, uint32_t hi_a, uint32_t b_lo, uint32_t hi_b, int kx,
                                        bool first) {
  if (XPAIR && kx != 1) {
    const int ks0 = kx == 0 ? 2 : 0;
#pragma unroll
    for (int ks = ks0; ks < ks0 + 2; ++ks) wgmma_m64k16<64, T>(acc, desc_lohi(a_lo + ks * 2, hi_a), desc_lohi(b_lo + ks * 2, hi_b));
  } else {
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
      wgmma_m64k16<64, T>(acc, desc_lohi(a_lo + ks * 2, hi_a), desc_lohi(b_lo + ks * 2, hi_b), (first && ks == 0) ? 0u : 1u);
  }
}

// all nine taps of NB accumulators (NB = 1 or 2), tap-interleaved; a_lo[i] = tap (0,0) of accumulator i
template <typename T, bool XPAIR, int NB>
__device__ __forceinline__ void blk_conv(float* acc0, float* acc1, uint32_t a_lo0, uint32_t a_lo1, uint32_t hi_a,
                                         uint32_t a_row16, uint32_t b_lo, uint32_t hi_b) {
#pragma unroll
  for (int ky = 0; ky < 3; ++ky)
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const int kx = XPAIR ? (i == 0 ? 1 : (i == 1 ? 0 : 2)) : i;
      const uint32_t off = (uint32_t)ky * a_row16 + (uint32_t)kx * (BLK_ROW_BYTES >> 4);
      const uint32_t bt = b_lo + (uint32_t)(ky * 3 + kx) * ((64u * BLK_ROW_BYTES) >> 4);
      const bool first = ky == 0 && i == 0;
      blk_tap<T, XPAIR>(acc0, a_lo0 + off, hi_a, bt, hi_b, kx, first);
      if (NB == 2) blk_tap<T, XPAIR>(acc1, a_lo1 + off, hi_a, bt, hi_b, kx, first);
    }
}

template <typename T, bool XPAIR>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_block_kernel(const __grid_constant__ ConvBlockParams P) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const uint32_t b1_base = base, b2_base = base + BLK_OFF_B2, a_base = base + BLK_OFF_A;
  const uint32_t full_bar = base + BLK_OFF_BAR, empty_bar = full_bar + 8, bres_bar = full_bar + 16;
  float* s_bias = reinterpret_cast<float*>(smem_raw + (base + BLK_OFF_BIAS - raw));   // [2][64]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    mbar_init(full_bar, 1);
    mbar_init(empty_bar, CONSUMER_WARPS);
    mbar_init(bres_bar, 1);
    fence_barrier_init();
    tma_prefetch_desc(&P.tmA);
    tma_prefetch_desc(&P.tmB1);
    tma_prefetch_desc(&P.tmB2);
  }
  for (int i = threadIdx.x; i < 128; i += TC_THREADS) s_bias[i] = i < 64 ? P.bias1[i] : P.bias2[i - 64];
  // the slack past the box is never written by TMA: zero it once
  for (uint32_t i = threadIdx.x; i < BLK_SLACK_BYTES / 4; i += TC_THREADS) sts32(a_base + BLK_BOX_BYTES + 4 * i, 0u);
  __syncthreads();
  pdl_launch_dependents();

  if (warp >= CONSUMER_WARPS) {
    // ===================================================================== TMA producer
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp != PRODUCER_WARP) return;
    if (elect_one_sync()) {   // both weight sets, once per CTA
      mbar_expect_tx(bres_bar, 2 * BLK_W_BYTES);
      for (int t = 0; t < 9; ++t) {
        tma_load_2d(b1_base + (uint32_t)t * 64u * BLK_ROW_BYTES, &P.tmB1, bres_bar, t * 64, 0);
        tma_load_2d(b2_base + (uint32_t)t * 64u * BLK_ROW_BYTES, &P.tmB2, bres_bar, t * 64, 0);
      }
    }
    __syncwarp();
    pdl_wait();
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < P.total_tiles; tile += gridDim.x) {
      const int n = tile / P.tiles_per_img, rem = tile % P.tiles_per_img;
      const int y0 = (rem / P.tiles_x) * TILE_Y, x0 = (rem % P.tiles_x) * TILE_X;
      mbar_wait_parity(empty_bar, ph ^ 1u);
      if (elect_one_sync()) {
        mbar_expect_tx(full_bar, BLK_BOX_BYTES);
        tma_load_4d(a_base, &P.tmA, full_bar, 0, x0 - 2, y0 - 2, n);
      }
      __syncwarp();
      ph ^= 1u;
    }
    return;
  }

  // ========================================================================= consumer warpgroups
  setmaxnreg_inc<CONSUMER_REGS>();
  const int wg = warp >> 2, wq = warp & 3;
  const int h = wg & 1, rg = wg >> 1;
  mbar_wait_parity(bres_bar, 0);
  pdl_wait();
  constexpr uint32_t sw = 1u << 30;                                  // 128B swizzle
  const uint32_t hi_flat = ((8u * BLK_ROW_BYTES) >> 4) | sw;         // conv1: SBO = next 8 flat pixels
  const uint32_t hi_p1 = (((uint32_t)BLK_PITCH * BLK_ROW_BYTES) >> 4) | sw;   // conv2: SBO = next image row
  const uint32_t hi_b = ((8u * BLK_ROW_BYTES) >> 4) | sw;
  const uint32_t lo_flags = 1u << 16;
  const uint32_t a_lo = ((a_base >> 4) & 0x3FFF) | lo_flags;
  const uint32_t b1_lo = ((b1_base >> 4) & 0x3FFF) | lo_flags, b2_lo = ((b2_base >> 4) & 0x3FFF) | lo_flags;
  constexpr uint32_t pix16 = BLK_ROW_BYTES >> 4, row16 = (uint32_t)BLK_PITCH * pix16;
  const int blk0 = wg, blk1 = wg + 4;                                // conv1 M blocks of this warpgroup (block 7: discarded)
  const int cq = 2 * (lane & 3);
  const uint32_t is_lane0 = lane == 0 ? 1u : 0u;
  const T* res = reinterpret_cast<const T*>(P.res);
  T* out = reinterpret_cast<T*>(P.out);
  T* mid = reinterpret_cast<T*>(P.mid);
  float acc0[32], acc1[32];

  // conv1 epilogue of one M block, in place over the box
  auto mid_store = [&](const float* acc, int blk, int y0, int x0, int n) {
#pragma unroll
    for (int r2 = 0; r2 < 2; ++r2) {
      const int q = 64 * blk + 16 * wq + (lane >> 2) + 8 * r2;    // flat intermediate pixel
      const int r = q / BLK_PITCH, c = q - r * BLK_PITCH;
      if (r >= BLK_MID || c >= BLK_MID) continue;
      const int y = y0 - 1 + r, x = x0 - 1 + c;
      const bool inside = y >= 0 && y < P.H && x >= 0 && x < P.W;
      const bool keep = mid != nullptr && r >= 1 && r <= TILE_Y && c >= 1 && c <= TILE_X;
      T* mp = keep ? mid + (((size_t)n * P.H + y) * P.W + x) * P.mid_stride : nullptr;
      const uint32_t row = a_base + (uint32_t)q * BLK_ROW_BYTES;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int ch = 8 * j + cq;
        uint32_t v = 0u;
        if (inside) {
          float f0 = acc[4 * j + 2 * r2] + s_bias[ch], f1 = acc[4 * j + 2 * r2 + 1] + s_bias[ch + 1];
          f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f);
          v = pack2<T>(f0, f1);
          if (keep) *reinterpret_cast<uint32_t*>(mp + ch) = v;
        }
        sts32(row + ((((uint32_t)j ^ ((uint32_t)q & 7u))) << 4) + (uint32_t)cq * 2u, v);
      }
    }
  };

  uint32_t ph = 0;
  for (int tile = blockIdx.x; tile < P.total_tiles; tile += gridDim.x) {
    const int n = tile / P.tiles_per_img, rem = tile % P.tiles_per_img;
    const int y0 = (rem / P.tiles_x) * TILE_Y, x0 = (rem % P.tiles_x) * TILE_X;
    mbar_wait_parity(full_bar, ph);
    ph ^= 1u;
    // ---- conv1 over the flat 18 x 24 region
    wgmma_fence();
    blk_conv<T, XPAIR, 2>(acc0, acc1, a_lo + (uint32_t)(64 * blk0) * pix16, a_lo + (uint32_t)(64 * blk1) * pix16, hi_flat, row16,
                          b1_lo, hi_b);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_acc_fence<32>(acc0);
    wgmma_acc_fence<32>(acc1);
    named_bar_sync(BLK_BAR, 512);   // every conv1 wgmma of the tile has read the box: overwrite it
    mid_store(acc0, blk0, y0, x0, n);
    mid_store(acc1, blk1, y0, x0, n);
    fence_proxy_async();            // generic-proxy stores -> wgmma operand reads
    named_bar_sync(BLK_BAR, 512);
    // ---- conv2 over the intermediate, MODE_P1 addressing
    wgmma_fence();
    blk_conv<T, XPAIR, 1>(acc0, acc0, a_lo + (uint32_t)h * 8u * pix16 + (uint32_t)(rg * 8) * row16, 0u, hi_p1, row16, b2_lo, hi_b);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_acc_fence<32>(acc0);
    __syncwarp();
    mbar_arrive_if(empty_bar, is_lane0);   // the box is free: the next tile's load overlaps this epilogue
    // ---- conv2 epilogue: + bias + residual, ReLU
    const int oy0 = y0 + rg * 8 + 2 * wq, ox = x0 + h * HALF_X + (lane >> 2);
#pragma unroll
    for (int r2 = 0; r2 < 2; ++r2) {
      const size_t pix = ((size_t)n * P.H + oy0 + r2) * P.W + ox;
      const T* rp = res + pix * P.res_stride;
      T* op = out + pix * P.out_stride;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = 8 * j + cq;
        float f0 = acc0[4 * j + 2 * r2] + s_bias[64 + c], f1 = acc0[4 * j + 2 * r2 + 1] + s_bias[64 + c + 1];
        float x0f, x1f;
        unpack2<T>(*reinterpret_cast<const uint32_t*>(rp + c), x0f, x1f);
        f0 += x0f; f1 += x1f;
        f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f);
        *reinterpret_cast<uint32_t*>(op + c) = pack2<T>(f0, f1);
      }
    }
  }
}

// --------------------------------------------------------------------------------- host side
struct ConvBlockPlan {
  ConvBlockParams p;
  int act_dtype, xpair, grid;
};

// conv_block_prepare (ops.cuh): conv1 = a1 (3x3 s1 64 -> 64, ReLU, or its x-paired form), conv2 = a2 (same geometry, input
// = a1's output, residual = a1's input, ReLU); `store_mid`: also write conv1's output to a1.out

}  // namespace acr
