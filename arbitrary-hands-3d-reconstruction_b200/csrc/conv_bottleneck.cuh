// One Bottleneck (1x1 C_in -> 64 BN ReLU, 3x3 64 -> 64 BN ReLU, 1x1 64 -> 256 BN + residual, ReLU) as ONE wgmma launch,
// sm_90a.
//
// Three conv_tc launches move the 256-channel tensors through HBM three times per block (read x, read x again as conv3's
// residual, write the output) plus both 64-channel intermediates twice; this kernel reads x once, writes the output once
// and re-reads the residual of the tile it just loaded (an L2 hit).  Block 0 of a layer reads its 64-channel input and
// the downsample's output as the residual.  The intermediates never leave shared memory.
//
// Per 16-wide x 8-tall output tile (persistent CTAs, the conv_tc_kernel warp layout: four consumer warpgroups as two
// teams of two, one producer warp per team):
//   * Tiles.  The CTA's k-th tile is blockIdx.x + k * gridDim.x; team k & 1 computes it in input box k & 1, with that
//     box's own full / empty mbarrier pair, its own producer warp and its own named barrier.  The teams share nothing
//     but the resident weights, so they issue freely: while one team waits for a chunk to land, or runs an epilogue, the
//     other team's wgmmas use the tensor cores.
//   * Input: per 64-channel chunk of x, ONE TMA box {64 ch, 24-pixel pitch, 10 rows} from (x0-1, y0-1): the tile plus
//     conv2's one-pixel halo.  K = 256 inputs stream their four chunks through the team's box, in the standalone chunk
//     order; K = 64 inputs load one.  Chunk c + 1 of a team lands once chunk c's wgmmas have read the box.
//   * conv1 over the whole 10 x 24 box, "flat M" as conv_block.cuh's conv1 (a 1x1 conv has no tap offsets): 240 flat
//     pixels in the team's 4 M blocks of 64, warpgroup w of the team owns blocks w and w + 2 (the last block reads 16
//     pixels of zeroed slack past the box, which only feed the discarded flat row 10).  Its k-steps sum chunk-major,
//     k16-minor, as conv_tc's resident 1x1 form.
//   * conv1 epilogue IN PLACE over the box once every conv1 wgmma of the team's tile has completed: bias + ReLU, rounded
//     to 16 bits, in the 128B-swizzled K-major layout TMA writes.  Pixels outside the image are stored as ZERO: they are
//     conv2's padding (a 1x1 conv of TMA's zero fill would be ReLU(bias), not zero).  Columns 18..23 are never read.
//   * conv2 reads that intermediate with the MODE_P1 addressing (one 8 x 8 M block per warpgroup at pitch 24, taps =
//     descriptor starts).
//   * conv2 epilogue IN PLACE again, once every conv2 wgmma of the team has completed: the 8 x 16 x 64 result at the same
//     pitch 24 (rows 0..7, columns 0..15).  conv3's M block of a warpgroup is exactly the 64 pixels its conv2 produced,
//     so a warpgroup barrier orders those stores before its conv3 wgmmas.
//   * conv3 in two N halves of 128 (a 64-register accumulator, as conv_tc's nsplit = 2 virtual tiles): MMAs, then the
//     epilogue (bias, residual from global one output row at a time, ReLU, NHWC stores straight from the register
//     fragment).  Once the second half's wgmmas have completed the box goes back to the team's producer, whose next load
//     overlaps that epilogue.
//   * Shared memory: all three weight sets resident, conv1 32 KB (4 chunks x [64][64]) + conv2 72 KB (9 taps x [64][64])
//     + conv3 32 KB ([256][64]) = 136 KB; two boxes of 10 x 24 x 128 B = 30 KB, each followed by 2 KB of slack (so box 1
//     starts on the 1024 B swizzle boundary) = 64 KB; biases 1.5 KB: 201.5 KB + barriers + alignment.  A separate conv2
//     output does not fit next to the weights, which is why both intermediates overwrite the team's box and the chunks
//     of a K = 256 input take turns in it.
//   * Bit-identical to the three conv_tc launches: every accumulator sums its chunks, taps and k-steps in the standalone
//     order, both intermediates are rounded to 16 bits, and the epilogues do the same float operations.
#pragma once
#include "conv_tc.cuh"

namespace acr {

constexpr int BNK_TILE_Y = 8;                                      // output tile: TILE_X (16) x 8 pixels
constexpr int BNK_PITCH = 24, BNK_ROWS = BNK_TILE_Y + 2;           // input box: 24 x 10 pixels, one-pixel halo
constexpr int BNK_MID_ROWS = BNK_ROWS, BNK_MID_COLS = TILE_X + 2;  // conv1's region: 10 x 18 at pitch 24
constexpr int BNK_MAX_CHUNKS = 4;                                  // C_in = 64 or 256
constexpr uint32_t BNK_ROW_BYTES = 128;                            // 64 16-bit channels
constexpr uint32_t BNK_BLK_BYTES = 64u * BNK_ROW_BYTES;            // one [64][64] weight block
constexpr uint32_t BNK_BOX_BYTES = (uint32_t)BNK_PITCH * BNK_ROWS * BNK_ROW_BYTES;
constexpr int BNK_M_BLOCKS = 4;                                    // conv1 M blocks of a tile: 2 per warpgroup of the team
constexpr int BNK_SLACK_PIX = BNK_M_BLOCKS * 64 - BNK_PITCH * BNK_ROWS;
constexpr uint32_t BNK_SLACK_BYTES = (uint32_t)BNK_SLACK_PIX * BNK_ROW_BYTES;
constexpr uint32_t BNK_BOX_STRIDE = (BNK_BOX_BYTES + BNK_SLACK_BYTES + 1023u) & ~1023u;   // box 1 starts 1024-aligned
constexpr uint32_t BNK_OFF_B2 = BNK_MAX_CHUNKS * BNK_BLK_BYTES;
constexpr uint32_t BNK_OFF_B3 = BNK_OFF_B2 + 9u * BNK_BLK_BYTES;
constexpr uint32_t BNK_OFF_A = BNK_OFF_B3 + 4u * BNK_BLK_BYTES;    // box t at BNK_OFF_A + t * BNK_BOX_STRIDE
constexpr uint32_t BNK_OFF_BIAS = BNK_OFF_A + BNK_BOX_STRIDE + BNK_BOX_BYTES + BNK_SLACK_BYTES;
constexpr uint32_t BNK_OFF_BAR = BNK_OFF_BIAS + (64 + 64 + 256) * 4;
constexpr size_t BNK_SMEM = 1024 /*alignment slack*/ + BNK_OFF_BAR + 64;
static_assert(BNK_M_BLOCKS * 64 >= BNK_MID_ROWS * BNK_PITCH && (BNK_M_BLOCKS - 1) * 64 < BNK_MID_ROWS * BNK_PITCH,
              "flat-M plan: 4 M blocks of 64 cover the 240 flat pixels, none discarded");
static_assert(BNK_SLACK_PIX == 16 && BNK_BOX_STRIDE == 32768, "flat-M plan: the last M block reads 16 pixels past the box");
static_assert(BNK_OFF_A % 1024 == 0 && BNK_BOX_STRIDE % 1024 == 0, "128B swizzle: every box starts on a 1024 B boundary");
static_assert(BNK_TILE_Y * BNK_PITCH <= BNK_PITCH * BNK_ROWS, "conv2's output fits in the box it overwrites");
static_assert(BNK_SMEM == 207424 && BNK_SMEM <= (size_t)SMEM_BUDGET,
              "fused-Bottleneck shared-memory plan: 136 KB weights + two 1024-aligned boxes with slack + biases + barriers");
static_assert(TILE_Y % BNK_TILE_Y == 0, "the 16-row super-tile precondition covers the 8-row tiles");
constexpr int BNK_BAR = 1;        // named barrier BNK_BAR + t over the 256 threads of team t
constexpr int BNK_WG_BAR = 3;     // named barrier BNK_WG_BAR + g over warpgroup g alone

struct ConvBottleneckParams {
  CUtensorMap tmA;                // block input x {C_in, W, H, B}, box {64, 24, 10}
  CUtensorMap tmB1, tmB2, tmB3;   // packed weights: conv1 [64][C_in], conv2 [64][9 * 64], conv3 [256][64]
  const float* bias1;
  const float* bias2;
  const float* bias3;
  const void* res;                // conv3's residual: x, or the downsample's output
  void* out;
  int res_stride, out_stride;
  int H, W, tiles_x, tiles_per_img, total_tiles;   // 16 x 8 tiles
};

// CCHUNKS = 64-channel chunks of x (1 or 4), a compile-time count: a runtime chunk loop keeps both conv1 accumulators live
// across a loop back-edge, and ptxas spills them
template <typename T, int CCHUNKS>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_bottleneck_kernel(const __grid_constant__ ConvBottleneckParams P) {
  static_assert(CCHUNKS == 1 || CCHUNKS == BNK_MAX_CHUNKS, "C_in = 64 or 256");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const uint32_t b1_base = base, b2_base = base + BNK_OFF_B2, b3_base = base + BNK_OFF_B3, a_base0 = base + BNK_OFF_A;
  // mbarriers: full[t], empty[t] of box t, then the resident weights
  const uint32_t full_bar0 = base + BNK_OFF_BAR, empty_bar0 = full_bar0 + 16, bres_bar = full_bar0 + 32;
  float* s_bias = reinterpret_cast<float*>(smem_raw + (base + BNK_OFF_BIAS - raw));   // [64 | 64 | 256]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int cchunks = CCHUNKS;
  // tiles of this CTA: blockIdx.x + k * gridDim.x for k < ntiles
  const int ntiles = (int)blockIdx.x < P.total_tiles ? (P.total_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;

  if (threadIdx.x == 0) {
    for (int t = 0; t < 2; ++t) {
      mbar_init(full_bar0 + 8 * t, 1);
      mbar_init(empty_bar0 + 8 * t, CONSUMER_WARPS / 2);
    }
    mbar_init(bres_bar, 1);
    fence_barrier_init();
    tma_prefetch_desc(&P.tmA);
    tma_prefetch_desc(&P.tmB1);
    tma_prefetch_desc(&P.tmB2);
    tma_prefetch_desc(&P.tmB3);
  }
  for (int i = threadIdx.x; i < 384; i += TC_THREADS) s_bias[i] = i < 64 ? P.bias1[i] : (i < 128 ? P.bias2[i - 64] : P.bias3[i - 128]);
  // the slack past each box is never written by TMA: zero it once
  for (uint32_t i = threadIdx.x; i < 2 * (BNK_SLACK_BYTES / 4); i += TC_THREADS) {
    const uint32_t t = i / (BNK_SLACK_BYTES / 4), j = i - t * (BNK_SLACK_BYTES / 4);
    sts32(a_base0 + t * BNK_BOX_STRIDE + BNK_BOX_BYTES + 4 * j, 0u);
  }
  __syncthreads();
  pdl_launch_dependents();

  if (warp >= CONSUMER_WARPS) {
    // ===================================================================== TMA producers: warp PRODUCER_WARP + t feeds box t
    setmaxnreg_dec<PRODUCER_REGS>();
    const int team = warp - PRODUCER_WARP;
    if (team > 1) return;
    if (team == 0 && elect_one_sync()) {   // all three weight sets, once per CTA
      mbar_expect_tx(bres_bar, (uint32_t)(cchunks + 9 + 4) * BNK_BLK_BYTES);
      for (int c = 0; c < cchunks; ++c) tma_load_2d(b1_base + (uint32_t)c * BNK_BLK_BYTES, &P.tmB1, bres_bar, c * 64, 0);
      for (int t = 0; t < 9; ++t) tma_load_2d(b2_base + (uint32_t)t * BNK_BLK_BYTES, &P.tmB2, bres_bar, t * 64, 0);
      tma_load_2d(b3_base, &P.tmB3, bres_bar, 0, 0);
    }
    __syncwarp();
    pdl_wait();
    const uint32_t a_base = a_base0 + (uint32_t)team * BNK_BOX_STRIDE;
    const uint32_t full_bar = full_bar0 + 8 * team, empty_bar = empty_bar0 + 8 * team;
    uint32_t ph = 0;
    for (int k = team; k < ntiles; k += 2) {
      const int tile = (int)blockIdx.x + k * (int)gridDim.x;
      const int n = tile / P.tiles_per_img, rem = tile % P.tiles_per_img;
      const int y0 = (rem / P.tiles_x) * BNK_TILE_Y, x0 = (rem % P.tiles_x) * TILE_X;
      for (int c = 0; c < cchunks; ++c) {
        mbar_wait_parity(empty_bar, ph ^ 1u);
        if (elect_one_sync()) {
          mbar_expect_tx(full_bar, BNK_BOX_BYTES);
          tma_load_4d(a_base, &P.tmA, full_bar, c * 64, x0 - 1, y0 - 1, n);
        }
        __syncwarp();
        ph ^= 1u;
      }
    }
    return;
  }

  // ========================================================================= consumer warpgroups
  setmaxnreg_inc<CONSUMER_REGS>();
  const int wg = warp >> 2, wq = warp & 3;
  const int team = wg >> 1, w = wg & 1;   // team (box, tiles k with k & 1 == team), warpgroup of the team (left / right 8 columns)
  mbar_wait_parity(bres_bar, 0);
  pdl_wait();
  constexpr uint32_t sw = 1u << 30;                                   // 128B swizzle
  const uint32_t hi_flat = ((8u * BNK_ROW_BYTES) >> 4) | sw;          // conv1: SBO = next 8 flat pixels
  const uint32_t hi_p1 = (((uint32_t)BNK_PITCH * BNK_ROW_BYTES) >> 4) | sw;   // conv2 / conv3: SBO = next image row
  const uint32_t hi_b = ((8u * BNK_ROW_BYTES) >> 4) | sw;
  const uint32_t lo_flags = 1u << 16;
  const uint32_t a_base = a_base0 + (uint32_t)team * BNK_BOX_STRIDE;   // this team's box
  const uint32_t full_bar = full_bar0 + 8 * team, empty_bar = empty_bar0 + 8 * team;
  const uint32_t a_lo = ((a_base >> 4) & 0x3FFF) | lo_flags;
  const uint32_t b1_lo = ((b1_base >> 4) & 0x3FFF) | lo_flags, b2_lo = ((b2_base >> 4) & 0x3FFF) | lo_flags;
  const uint32_t b3_lo = ((b3_base >> 4) & 0x3FFF) | lo_flags;
  constexpr uint32_t pix16 = BNK_ROW_BYTES >> 4, row16 = (uint32_t)BNK_PITCH * pix16, blk16 = BNK_BLK_BYTES >> 4;
  const uint32_t a_tile = a_lo + (uint32_t)w * 8u * pix16;            // this warpgroup's 8 x 8 pixels
  const int blk0 = w, blk1 = w + 2;                                   // conv1 M blocks of this warpgroup
  const int cq = 2 * (lane & 3);
  const uint32_t is_lane0 = lane == 0 ? 1u : 0u;
  const T* res = reinterpret_cast<const T*>(P.res);
  T* out = reinterpret_cast<T*>(P.out);

  // (each accumulator is declared where it is used: one declared across tiles would stay live through the other convs)
  uint32_t ph = 0;
  for (int k = team; k < ntiles; k += 2) {
    const int tile = (int)blockIdx.x + k * (int)gridDim.x;
    const int n = tile / P.tiles_per_img, rem = tile % P.tiles_per_img;
    const int y0 = (rem / P.tiles_x) * BNK_TILE_Y, x0 = (rem % P.tiles_x) * TILE_X;
    // ---- conv1 over the flat 10 x 24 box, one 64-channel chunk at a time
    float acc0[32], acc1[32];
#pragma unroll
    for (int c = 0; c < cchunks; ++c) {
      mbar_wait_parity(full_bar, ph);
      ph ^= 1u;
      wgmma_fence();
      const uint32_t bc = b1_lo + (uint32_t)c * blk16;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const uint32_t sc = (c == 0 && ks == 0) ? 0u : 1u;
        wgmma_m64k16<64, T>(acc0, desc_lohi(a_lo + (uint32_t)(64 * blk0) * pix16 + ks * 2, hi_flat), desc_lohi(bc + ks * 2, hi_b), sc);
        wgmma_m64k16<64, T>(acc1, desc_lohi(a_lo + (uint32_t)(64 * blk1) * pix16 + ks * 2, hi_flat), desc_lohi(bc + ks * 2, hi_b), sc);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_acc_fence<32>(acc0);
      wgmma_acc_fence<32>(acc1);
      if (c + 1 < cchunks) {   // the next chunk may land in the box
        __syncwarp();
        mbar_arrive_if(empty_bar, is_lane0);
      }
    }
    named_bar_sync(BNK_BAR + team, 256);   // every conv1 wgmma of the team's tile has read the box: overwrite it
    // conv1 epilogue of both M blocks, in place over the box
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      const float* acc = b ? acc1 : acc0;
#pragma unroll
      for (int r2 = 0; r2 < 2; ++r2) {
        const int q = 64 * (b ? blk1 : blk0) + 16 * wq + (lane >> 2) + 8 * r2;    // flat pixel
        const int r = q / BNK_PITCH, c = q - r * BNK_PITCH;
        if (r >= BNK_MID_ROWS || c >= BNK_MID_COLS) continue;
        const int y = y0 - 1 + r, x = x0 - 1 + c;
        const bool inside = y >= 0 && y < P.H && x >= 0 && x < P.W;
        const uint32_t row = a_base + (uint32_t)q * BNK_ROW_BYTES;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int ch = 8 * j + cq;
          uint32_t v = 0u;
          if (inside) {
            float f0 = acc[4 * j + 2 * r2] + s_bias[ch], f1 = acc[4 * j + 2 * r2 + 1] + s_bias[ch + 1];
            f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f);
            v = pack2<T>(f0, f1);
          }
          sts32(row + (((uint32_t)j ^ ((uint32_t)q & 7u)) << 4) + (uint32_t)cq * 2u, v);
        }
      }
    }
    fence_proxy_async();                   // generic-proxy stores -> wgmma operand reads
    named_bar_sync(BNK_BAR + team, 256);   // conv2's taps read rows written by the team's other warpgroup
    // ---- conv2 over the intermediate, MODE_P1 addressing
    float acc2[32];
    wgmma_fence();
#pragma unroll
    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
      for (int kx = 0; kx < 3; ++kx)
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
          wgmma_m64k16<64, T>(acc2, desc_lohi(a_tile + (uint32_t)ky * row16 + (uint32_t)kx * pix16 + ks * 2, hi_p1),
                              desc_lohi(b2_lo + (uint32_t)(ky * 3 + kx) * blk16 + ks * 2, hi_b), (ky == 0 && kx == 0 && ks == 0) ? 0u : 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_acc_fence<32>(acc2);
    named_bar_sync(BNK_BAR + team, 256);   // every conv2 wgmma of the team has read the intermediate: overwrite it
    // conv2 epilogue in place: this warpgroup's 64 pixels (row 2 wq + r2, column w * 8 + lane / 4)
#pragma unroll
    for (int r2 = 0; r2 < 2; ++r2) {
      const int q = (2 * wq + r2) * BNK_PITCH + w * HALF_X + (lane >> 2);
      const uint32_t row = a_base + (uint32_t)q * BNK_ROW_BYTES;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int ch = 8 * j + cq;
        float f0 = acc2[4 * j + 2 * r2] + s_bias[64 + ch], f1 = acc2[4 * j + 2 * r2 + 1] + s_bias[64 + ch + 1];
        f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f);
        sts32(row + (((uint32_t)j ^ ((uint32_t)q & 7u)) << 4) + (uint32_t)cq * 2u, pack2<T>(f0, f1));
      }
    }
    fence_proxy_async();
    named_bar_sync(BNK_WG_BAR + wg, 128);   // conv3 of this warpgroup reads exactly the pixels it just stored
    // ---- conv3: two N halves of 128, epilogue straight from the register fragment
    const int oy0 = y0 + 2 * wq, ox = x0 + w * HALF_X + (lane >> 2);
#pragma unroll 1
    for (int v = 0; v < 2; ++v) {
      float acc3[64];
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks)
        wgmma_m64k16<128, T>(acc3, desc_lohi(a_tile + ks * 2, hi_p1), desc_lohi(b3_lo + (uint32_t)v * 2u * blk16 + ks * 2, hi_b), ks == 0 ? 0u : 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_acc_fence<64>(acc3);
      if (v == 1) {   // every read of the box is done: the team's next tile may land
        __syncwarp();
        mbar_arrive_if(empty_bar, is_lane0);
      }
      // the residual is loaded one output row (16 registers) at a time, all 16 loads in flight before the first use.  It
      // is not loaded under the wgmmas: the 64-register accumulator and one such row already exceed the 96 registers
      // ptxas allots a 640-thread CTA, and the spill it then makes costs more than the L2 round trip it would hide
      const int n_off = 128 * v;
#pragma unroll
      for (int r2 = 0; r2 < 2; ++r2) {
        const size_t pix = ((size_t)n * P.H + oy0 + r2) * P.W + ox;
        const T* rp = res + pix * P.res_stride + n_off;
        uint32_t rv[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) rv[j] = *reinterpret_cast<const uint32_t*>(rp + 8 * j + cq);
        T* op = out + pix * P.out_stride + n_off;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int c = 8 * j + cq;
          float f0 = acc3[4 * j + 2 * r2] + s_bias[128 + n_off + c], f1 = acc3[4 * j + 2 * r2 + 1] + s_bias[128 + n_off + c + 1];
          float x0f, x1f;
          unpack2<T>(rv[j], x0f, x1f);
          f0 += x0f; f1 += x1f;
          f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f);
          *reinterpret_cast<uint32_t*>(op + c) = pack2<T>(f0, f1);
        }
      }
    }
  }
}

// --------------------------------------------------------------------------------- host side
struct ConvBottleneckPlan {
  ConvBottleneckParams p;
  int act_dtype, cchunks, grid;
};

// conv_bottleneck_prepare (ops.cuh): a1 = 1x1 C_in -> 64 (C_in 64 or 256), ReLU; a2 = 3x3 s1 64 -> 64 on a1's output, ReLU;
// a3 = 1x1 64 -> 256 on a2's output, residual, ReLU

}  // namespace acr
