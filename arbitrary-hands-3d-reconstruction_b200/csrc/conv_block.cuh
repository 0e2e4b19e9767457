// One HRNet BasicBlock (conv3x3-BN-ReLU, conv3x3-BN, + block input, ReLU) as ONE wgmma launch, sm_90a.
//
// Two conv_tc launches move five activation passes through HBM per block (read x, write y, read y, write the output,
// read x again as the residual); this kernel moves two (read x, write the output; the residual is read from the input
// box).  The intermediate y never leaves shared memory.
//
// Per 16-wide x 8-tall output tile (persistent CTAs, the conv_tc_kernel warp layout: four consumer warpgroups as two
// ping-pong teams of two, one producer warp):
//   * Tiles.  The CTA's k-th tile is blockIdx.x + k * gridDim.x; team k & 1 computes it, in input box k & 1, with that
//     box's own full / empty mbarrier pair.  The producer refills a box as soon as its team's conv2 wgmmas completed, and
//     when it issues a box's load it also pulls the team's next box (tile k + 2) into L2, so that refill waits on L2, not
//     on HBM.  x-paired blocks (dense 32-channel tensors, ACR_CONV_XPAIR) count the tile and the box in pixel pairs (a
//     32 x 8 pixel tile).
//   * Input: one TMA box {64 ch, 24-pixel pitch, 12 rows} from (x0-2, y0-2): a two-pixel halo, TMA's out-of-bounds zeros
//     are conv1's padding.
//   * conv1 over the 10 x 18 intermediate region (the tile plus conv2's one-pixel halo), "flat": the pitch-24 box is a
//     flat array of pixels and intermediate pixel p = r * 24 + c reads input pixel p + ky * 24 + kx for tap (ky, kx), a
//     constant offset.  The resident weights ([tap][cout][64 ch], K-major) are the wgmma A operand, M = the 64 output
//     channels, and N = 120 consecutive flat pixels are B (15 core groups of 8, SBO = 1024 B); a tap is a descriptor
//     start (ky * 24 + kx) * 128 B into the box -- an unaligned start, like MODE_P1 (the 128B swizzle follows the
//     absolute address).  10 x 24 = 240 flat pixels are exactly the team's two N ranges: warpgroup w of the team issues
//     one m64n120k16 per tap and k-step over pixels [120 w, 120 w + 120).  The accumulator is the standalone conv's,
//     transposed: each element is the same dot product over the same k-steps in the same order, and the tensor core
//     reduces it the same way from either operand side (checked bit for bit on H100, bf16 and fp16).  Pixel 239 reads 2
//     pixels past the box: a zeroed slack (those reads only feed flat columns 22..23, which conv2 never reads).
//   * conv1 epilogue IN PLACE: once every conv1 wgmma of the team's tile has completed (a barrier over the team), bias +
//     ReLU, rounded to 16 bits, is stored over the box in the 128B-swizzled K-major layout TMA would have written (16-byte
//     chunk index ^= pixel & 7), with stmatrix.trans: a fragment of 8 channels x 8 pixels, transposed, is those pixels'
//     16-byte chunks, so a thread issues 8 shared stores for its 30 pixel pairs x 2 channels (the epilogue runs while
//     the other team streams wgmmas, which leave its instructions few issue and shared-memory slots).  Pixels outside
//     the image are stored as ZERO: they are conv2's padding; tiles whose 10 x 18 region lies inside the image skip the
//     masks.  Flat columns 18..23 get values too; conv2 never reads them.  Then fence.proxy.async and a second team
//     barrier: conv2's taps read rows written by the team's other warpgroup.
//   * conv2 reads the intermediate with the MODE_P1 addressing (one 8x8-pixel M block per warpgroup at pitch 24, taps =
//     descriptor starts); once its wgmmas completed the box is handed back to the producer, then the conv2 epilogue
//     (bias, residual, ReLU, NHWC stores).  The residual is read from the box into registers (ldmatrix) before the conv1
//     epilogue overwrites it.
//   * Ping-pong: the teams take turns issuing one group of wgmmas each (a tile's conv1, or its conv2), so the turns run
//     team 0 conv1, team 1 conv1, team 0 conv2, team 1 conv2, team 0 conv1 of its next tile, ...  A team holds the turn
//     only while it issues and hands it over before it waits for its wgmmas, so its waits, barriers and epilogues run
//     under the other team's MMAs.  Turn s belongs to team s & 1 and is the conv1 (s & 2 == 0) or conv2 of the CTA's
//     tile 2 (s >> 2) + (s & 1).  Barrier TEAM_BAR + t completes when team t may issue: a team waits on it only when
//     the previous turn exists and arrives on the other team's only when the next turn exists, so every barrier phase
//     completes by kernel exit for any tile count per CTA.
//   * Shared memory: both weight sets stay resident (2 x 72 KB), two boxes of 36 KB, each followed by its slack and
//     starting on a 1024 B boundary (the 128B swizzle).  That is why the intermediate overwrites the box.
//   * Bit-identical to the two conv_tc launches: every accumulator sums its taps and k-steps in the standalone order
//     (ky-major, kx 0,1,2; x-paired: kx 1,0,2, side taps as full-width MMAs over zero weight quarters), the epilogues do
//     the same float operations, and the intermediate is rounded to 16 bits in both paths.
//   * `mid` (optional): conv1's output for the tile's own 16x8 pixels is also copied from the box to global (16-byte
//     chunks, unswizzled) while conv2's wgmmas run, so an observable intermediate (teacher-forced checks, kept tensors)
//     is still written.
#pragma once
#include <type_traits>

#include "conv_tc.cuh"

namespace acr {

constexpr int BLK_TILE_Y = 8;                                      // output tile: TILE_X (16) x 8 pixels (pairs)
constexpr int BLK_PITCH = 24, BLK_ROWS = BLK_TILE_Y + 4;           // input box: 24 x 12 pixels (pairs), two-pixel halo
constexpr int BLK_MID_ROWS = BLK_TILE_Y + 2, BLK_MID_COLS = TILE_X + 2;   // intermediate region: 10 x 18 at pitch 24
constexpr uint32_t BLK_ROW_BYTES = 128;                            // 64 16-bit channels
constexpr uint32_t BLK_W_BYTES = 9u * 64u * BLK_ROW_BYTES;         // one conv's resident weights: 9 taps x [64][64]
constexpr uint32_t BLK_BOX_BYTES = (uint32_t)BLK_PITCH * BLK_ROWS * BLK_ROW_BYTES;
constexpr int BLK_CONV1_N = 120;   // conv1 flat pixels per warpgroup: the N of its m64n120k16 (A = the 64 output channels)
constexpr int BLK_SLACK_PIX = 2 * BLK_CONV1_N + 2 * BLK_PITCH + 2 - BLK_PITCH * BLK_ROWS;
constexpr uint32_t BLK_SLACK_BYTES = (uint32_t)BLK_SLACK_PIX * BLK_ROW_BYTES;
constexpr uint32_t BLK_BOX_STRIDE = (BLK_BOX_BYTES + BLK_SLACK_BYTES + 1023u) & ~1023u;   // box 1 starts 1024-aligned
constexpr uint32_t BLK_OFF_B2 = BLK_W_BYTES;
constexpr uint32_t BLK_OFF_A = 2 * BLK_W_BYTES;                    // box t at BLK_OFF_A + t * BLK_BOX_STRIDE
constexpr uint32_t BLK_OFF_BIAS = BLK_OFF_A + BLK_BOX_STRIDE + BLK_BOX_BYTES + BLK_SLACK_BYTES;
constexpr uint32_t BLK_OFF_BAR = BLK_OFF_BIAS + 2 * 64 * 4;
constexpr size_t BLK_SMEM = 1024 /*alignment slack*/ + BLK_OFF_BAR + 64;
static_assert(2 * BLK_CONV1_N == BLK_MID_ROWS * BLK_PITCH && BLK_CONV1_N % BLK_PITCH == 0 && BLK_CONV1_N % 16 == 8,
              "flat conv1: the team's two N = 120 ranges are the 240 flat intermediate pixels, 5 whole rows each");
static_assert(BLK_SLACK_PIX == 2 && BLK_BOX_STRIDE == 37888, "flat conv1: pixel 239 reads 2 pixels past the box");
static_assert(BLK_OFF_A % 1024 == 0 && BLK_BOX_STRIDE % 1024 == 0, "128B swizzle: every box starts on a 1024 B boundary");
static_assert(BLK_MID_ROWS * BLK_PITCH * BLK_ROW_BYTES <= BLK_BOX_BYTES, "the intermediate fits in the box it overwrites");
static_assert(BLK_SMEM == 224064 && BLK_SMEM <= (size_t)SMEM_BUDGET,
              "fused-block shared-memory plan: 144 KB weights + two 1024-aligned boxes with slack + biases + barriers");
static_assert(TILE_Y % BLK_TILE_Y == 0, "the 16-row super-tile precondition covers the 8-row tiles");
constexpr int BLK_BAR = 1;   // named barrier BLK_BAR + t over the 256 threads of team t

struct ConvBlockParams {
  CUtensorMap tmA;          // block input x {C, W, H, B}, box {64, 24, 12}
  CUtensorMap tmB1, tmB2;   // packed weights of conv1 / conv2 [64][9 * 64], box {64, 64}
  const float* bias1;
  const float* bias2;
  void* out;
  void* mid;                // conv1's output buffer, or nullptr when nothing reads it
  int out_stride, mid_stride;
  int H, W, tiles_x, tiles_per_img, total_tiles;   // 16 x 8 tiles
};

// the wgmmas of one tap, D[64][N] += A * B (x-paired side taps: the two k-steps of their K half, see conv_tc_kernel)
template <typename T, bool XPAIR, int N>
__device__ __forceinline__ void blk_tap(float* acc, uint32_t a_lo, uint32_t hi_a, uint32_t b_lo, uint32_t hi_b, int kx,
                                        bool first) {
  if (XPAIR && kx != 1) {
    const int ks0 = kx == 0 ? 2 : 0;
#pragma unroll
    for (int ks = ks0; ks < ks0 + 2; ++ks) wgmma_m64k16<N, T>(acc, desc_lohi(a_lo + ks * 2, hi_a), desc_lohi(b_lo + ks * 2, hi_b));
  } else {
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
      wgmma_m64k16<N, T>(acc, desc_lohi(a_lo + ks * 2, hi_a), desc_lohi(b_lo + ks * 2, hi_b), (first && ks == 0) ? 0u : 1u);
  }
}

// all nine taps of one accumulator; px_lo = the pixels of tap (0,0), w_lo = the weights of tap 0.  W_AS_A (conv1): the
// weights are A (M = the 64 output channels) and BLK_CONV1_N pixels are B; else (conv2) 64 pixels are A and the weights B
template <typename T, bool XPAIR, bool W_AS_A>
__device__ __forceinline__ void blk_conv(float* acc, uint32_t px_lo, uint32_t hi_px, uint32_t w_lo, uint32_t hi_w) {
  constexpr uint32_t pix16 = BLK_ROW_BYTES >> 4, row16 = (uint32_t)BLK_PITCH * pix16;
#pragma unroll
  for (int ky = 0; ky < 3; ++ky)
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const int kx = XPAIR ? (i == 0 ? 1 : (i == 1 ? 0 : 2)) : i;
      const uint32_t px = px_lo + (uint32_t)ky * row16 + (uint32_t)kx * pix16;
      const uint32_t wt = w_lo + (uint32_t)(ky * 3 + kx) * ((64u * BLK_ROW_BYTES) >> 4);
      const bool first = ky == 0 && i == 0;
      if constexpr (W_AS_A) blk_tap<T, XPAIR, BLK_CONV1_N>(acc, wt, hi_w, px, hi_px, kx, first);
      else blk_tap<T, XPAIR, 64>(acc, px, hi_px, wt, hi_w, kx, first);
    }
}

// pull one TMA box into L2 (no shared-memory destination, no completion to wait for)
__device__ __forceinline__ void tma_prefetch_l2_4d(const CUtensorMap* map, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.prefetch.tensor.4d.L2.global.tile [%0, {%1, %2, %3, %4}];"
               ::"l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}

// 8x8 16-bit fragments (r_i = this thread's pair of fragment i: row lane >> 2, columns 2 (lane & 3) + {0, 1}) to shared
// memory TRANSPOSED: column c of fragment i goes to the 16 bytes at the address of lane 8 i + c
__device__ __forceinline__ void stsm_x4_trans(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1),
               "r"(r2), "r"(r3) : "memory");
}
__device__ __forceinline__ void stsm_x2_trans(uint32_t addr, uint32_t r0, uint32_t r1) {
  asm volatile("stmatrix.sync.aligned.m8n8.x2.trans.shared.b16 [%0], {%1, %2};" ::"r"(addr), "r"(r0), "r"(r1) : "memory");
}
// four 8x8 16-bit fragments from shared memory (r_i: row lane >> 2, columns 2 (lane & 3) + {0, 1} of fragment i); lane l
// gives the address of row l & 7 of fragment l >> 3
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}

// wait on named barrier `id` when pred != 0; one asm statement, no branch between the wgmma groups
__device__ __forceinline__ void named_bar_sync_if(int id, int nthreads, uint32_t pred) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.u32 p, %2, 0;\n@p bar.sync %0, %1;\n}\n" ::"r"(id), "r"(nthreads), "r"(pred) : "memory");
}

template <typename T, bool XPAIR>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_block_kernel(const __grid_constant__ ConvBlockParams P) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const uint32_t b1_base = base, b2_base = base + BLK_OFF_B2, a_base0 = base + BLK_OFF_A;
  // mbarriers: full[t], empty[t] of box t, then the resident weights
  const uint32_t full_bar0 = base + BLK_OFF_BAR, empty_bar0 = full_bar0 + 16, bres_bar = full_bar0 + 32;
  float* s_bias = reinterpret_cast<float*>(smem_raw + (base + BLK_OFF_BIAS - raw));   // [2][64]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
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
  }
  for (int i = threadIdx.x; i < 128; i += TC_THREADS) s_bias[i] = i < 64 ? P.bias1[i] : P.bias2[i - 64];
  // the slack past each box is never written by TMA: zero it once
  for (uint32_t i = threadIdx.x; i < 2 * (BLK_SLACK_BYTES / 4); i += TC_THREADS) {
    const uint32_t t = i / (BLK_SLACK_BYTES / 4), j = i - t * (BLK_SLACK_BYTES / 4);
    sts32(a_base0 + t * BLK_BOX_STRIDE + BLK_BOX_BYTES + 4 * j, 0u);
  }
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
    for (int k = 0; k < ntiles; ++k) {
      const int tile = (int)blockIdx.x + k * (int)gridDim.x, bx = k & 1;
      const int n = tile / P.tiles_per_img, rem = tile % P.tiles_per_img;
      const int y0 = (rem / P.tiles_x) * BLK_TILE_Y, x0 = (rem % P.tiles_x) * TILE_X;
      mbar_wait_parity(empty_bar0 + 8 * bx, ((uint32_t)(k >> 1) & 1u) ^ 1u);
      if (elect_one_sync()) {
        mbar_expect_tx(full_bar0 + 8 * bx, BLK_BOX_BYTES);
        tma_load_4d(a_base0 + (uint32_t)bx * BLK_BOX_STRIDE, &P.tmA, full_bar0 + 8 * bx, 0, x0 - 2, y0 - 2, n);
        if (k + 2 < ntiles) {   // the box's next tile, into L2
          const int t2 = tile + 2 * (int)gridDim.x, rem2 = t2 % P.tiles_per_img;
          tma_prefetch_l2_4d(&P.tmA, 0, (rem2 % P.tiles_x) * TILE_X - 2, (rem2 / P.tiles_x) * BLK_TILE_Y - 2,
                             t2 / P.tiles_per_img);
        }
      }
      __syncwarp();
    }
    return;
  }

  // ========================================================================= consumer warpgroups
  setmaxnreg_inc<CONSUMER_REGS>();
  const int wg = warp >> 2, wq = warp & 3;
  const int team = wg >> 1, w = wg & 1;   // team (box, tiles k with k & 1 == team), warpgroup of the team (left / right 8 columns)
  mbar_wait_parity(bres_bar, 0);
  pdl_wait();
  constexpr uint32_t sw = 1u << 30;                                  // 128B swizzle
  const uint32_t hi_flat = ((8u * BLK_ROW_BYTES) >> 4) | sw;         // conv1: SBO = next 8 flat pixels
  const uint32_t hi_p1 = (((uint32_t)BLK_PITCH * BLK_ROW_BYTES) >> 4) | sw;   // conv2: SBO = next image row
  const uint32_t hi_b = ((8u * BLK_ROW_BYTES) >> 4) | sw;
  const uint32_t lo_flags = 1u << 16;
  const uint32_t a_base = a_base0 + (uint32_t)team * BLK_BOX_STRIDE;   // this team's box
  const uint32_t full_bar = full_bar0 + 8 * team, empty_bar = empty_bar0 + 8 * team;
  const uint32_t a_lo = ((a_base >> 4) & 0x3FFF) | lo_flags;
  const uint32_t b1_lo = ((b1_base >> 4) & 0x3FFF) | lo_flags, b2_lo = ((b2_base >> 4) & 0x3FFF) | lo_flags;
  constexpr uint32_t pix16 = BLK_ROW_BYTES >> 4;
  const int cq = 2 * (lane & 3);
  const uint32_t is_lane0 = lane == 0 ? 1u : 0u;
  T* out = reinterpret_cast<T*>(P.out);
  T* mid = reinterpret_cast<T*>(P.mid);
  // conv1's accumulator is transposed (M = channels): this thread holds channels ch1 and ch1 + 8 of the warpgroup's flat
  // pixels 120 w + 8 j + cq + {0, 1}, j < 15, which are row 5 w + j / 3, columns 8 (j % 3) + cq + {0, 1}
  const int ch1 = 16 * wq + (lane >> 2);
  const float bias1_lo = s_bias[ch1], bias1_hi = s_bias[ch1 + 8];
  // stmatrix.trans of the fragments (channels 8 h.., pixels 8 j..) stores those 8 pixels' 16-byte chunk 2 wq + h.  For
  // fragment pair t, lane l gives the row of pixel 8 (2 t + (l >> 4)) + (l & 7), chunk 2 wq + ((l >> 3) & 1) ^ (l & 7)
  const uint32_t epi_row = a_base + (uint32_t)(BLK_CONV1_N * w + 8 * (lane >> 4) + (lane & 7)) * BLK_ROW_BYTES +
                           (((uint32_t)(2 * wq + ((lane >> 3) & 1)) ^ (uint32_t)(lane & 7)) << 4);
  float acc1[BLK_CONV1_N / 2], acc2[32];
  // turn s exists when the CTA has its tile (see the header); turn_pre / turn_post: wait for the turn, hand it on
  auto turn_exists = [&](int s) -> uint32_t { return (s >= 0 && 2 * (s >> 2) + (s & 1) < ntiles) ? 1u : 0u; };
  auto turn_pre = [&](int s) { named_bar_sync_if(TEAM_BAR + team, 512, turn_exists(s - 1)); };
  auto turn_post = [&](int s) { named_bar_arrive_if(TEAM_BAR + (team ^ 1), 512, turn_exists(s + 1)); };

  // conv1 epilogue in place over the box: bias + ReLU, rounded to 16 bits.  `masked` (std::true_type) zeroes the pixels
  // outside the image (conv2's padding); columns 18..23 are never read, so an interior tile masks nothing.
  auto conv1_epilogue = [&](auto masked, int y0, int x0) {
    uint32_t colm[3], rowm[5];   // per j % 3: the (pixel, pixel + 1) halves of a packed word; per j / 3: the row
    if constexpr (decltype(masked)::value) {
#pragma unroll
      for (int jm = 0; jm < 3; ++jm) {
        const int x = x0 - 1 + 8 * jm + cq;
        colm[jm] = (x >= 0 && x < P.W ? 0xFFFFu : 0u) | (x + 1 >= 0 && x + 1 < P.W ? 0xFFFF0000u : 0u);
      }
#pragma unroll
      for (int jr = 0; jr < 5; ++jr) {
        const int y = y0 - 1 + (BLK_CONV1_N / BLK_PITCH) * w + jr;
        rowm[jr] = y >= 0 && y < P.H ? ~0u : 0u;
      }
    }
    uint32_t v[2][BLK_CONV1_N / 8];
#pragma unroll
    for (int j = 0; j < BLK_CONV1_N / 8; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float b = h ? bias1_hi : bias1_lo;
        float f0 = acc1[4 * j + 2 * h] + b, f1 = acc1[4 * j + 2 * h + 1] + b;
        f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f);
        v[h][j] = pack2<T>(f0, f1);
        if constexpr (decltype(masked)::value) v[h][j] &= colm[j % 3] & rowm[j / 3];
      }
#pragma unroll
    for (int t = 0; t < BLK_CONV1_N / 16; ++t)
      stsm_x4_trans(epi_row + (uint32_t)t * 16u * BLK_ROW_BYTES, v[0][2 * t], v[1][2 * t], v[0][2 * t + 1], v[1][2 * t + 1]);
    stsm_x2_trans(epi_row + (uint32_t)(BLK_CONV1_N / 16) * 16u * BLK_ROW_BYTES, v[0][BLK_CONV1_N / 8 - 1],
                  v[1][BLK_CONV1_N / 8 - 1]);
  };

  for (int k = team; k < ntiles; k += 2) {
    const int tile = (int)blockIdx.x + k * (int)gridDim.x;
    const int n = tile / P.tiles_per_img, rem = tile % P.tiles_per_img;
    const int y0 = (rem / P.tiles_x) * BLK_TILE_Y, x0 = (rem % P.tiles_x) * TILE_X;
    const int s = 2 * k - team;   // this tile's conv1 turn; its conv2 turn is s + 2
    mbar_wait_parity(full_bar, (uint32_t)(k >> 1) & 1u);
    // ---- conv1 over the flat 10 x 24 region: the weights are A, this warpgroup's 120 flat pixels are B
    turn_pre(s);
    wgmma_fence();
    blk_conv<T, XPAIR, true>(acc1, a_lo + (uint32_t)(BLK_CONV1_N * w) * pix16, hi_flat, b1_lo, hi_b);
    wgmma_commit();
    turn_post(s);
    wgmma_wait<0>();
    wgmma_acc_fence<BLK_CONV1_N / 2>(acc1);
    // conv2's residual is the block input at the tile's own pixels, which the box holds (rows 2 wq + r2 + 2, columns
    // 8 w + 2 + (lane >> 2)) until the epilogue overwrites it.  An 8-pixel x 8-channel ldmatrix fragment is the
    // accumulator's layout: rv[r2][j] = channels 8 j + cq, + 1.  From global, each tile's residual loads took thousands
    // of cycles to land, and the team's next tile waited for them.
    uint32_t rv[2][8];
#pragma unroll
    for (int r2 = 0; r2 < 2; ++r2) {
      const uint32_t q = (uint32_t)((2 * wq + r2 + 2) * BLK_PITCH + HALF_X * w + 2 + (lane & 7));
#pragma unroll
      for (int h = 0; h < 2; ++h)
        ldsm_x4(a_base + q * BLK_ROW_BYTES + (((uint32_t)(4 * h + (lane >> 3)) ^ (q & 7u)) << 4), rv[r2][4 * h],
                rv[r2][4 * h + 1], rv[r2][4 * h + 2], rv[r2][4 * h + 3]);
    }
    named_bar_sync(BLK_BAR + team, 256);   // every conv1 wgmma and residual read of the tile is done: overwrite the box
    if (x0 >= 1 && x0 + BLK_MID_COLS - 1 <= P.W && y0 >= 1 && y0 + BLK_MID_ROWS - 1 <= P.H)
      conv1_epilogue(std::false_type{}, y0, x0);
    else
      conv1_epilogue(std::true_type{}, y0, x0);
    fence_proxy_async();                   // generic-proxy stores -> wgmma operand reads
    named_bar_sync(BLK_BAR + team, 256);
    // ---- conv2 over the intermediate, MODE_P1 addressing
    turn_pre(s + 2);
    wgmma_fence();
    blk_conv<T, XPAIR, false>(acc2, a_lo + (uint32_t)w * 8u * pix16, hi_p1, b2_lo, hi_b);
    wgmma_commit();
    turn_post(s + 2);
    if (mid != nullptr) {   // the tile's own 16 x 8 intermediate pixels: 16-byte chunks, unswizzled, from the box
      const int tt = 128 * w + (threadIdx.x & 127);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int e = tt + 256 * i, pix = e >> 3, g = e & 7;
        const int r = 1 + pix / TILE_X, c = 1 + pix % TILE_X, q = r * BLK_PITCH + c;
        const int y = y0 - 1 + r, x = x0 - 1 + c;
        const uint4 u = lds128(a_base + (uint32_t)q * BLK_ROW_BYTES + (((uint32_t)g ^ (uint32_t)(q & 7)) << 4));
        if (y < P.H && x < P.W) {   // 4-byte stores: the buffer's pixel stride is only known to be even
          uint32_t* mp = reinterpret_cast<uint32_t*>(mid + (((size_t)n * P.H + y) * P.W + x) * P.mid_stride + 8 * g);
          mp[0] = u.x; mp[1] = u.y; mp[2] = u.z; mp[3] = u.w;
        }
      }
    }
    wgmma_wait<0>();
    wgmma_acc_fence<32>(acc2);
    __syncwarp();
    mbar_arrive_if(empty_bar, is_lane0);   // the box is free: the team's next tile loads under the other team's MMAs
    // ---- conv2 epilogue: + bias + residual, ReLU
    const int oy0 = y0 + 2 * wq, ox = x0 + w * HALF_X + (lane >> 2);
#pragma unroll
    for (int r2 = 0; r2 < 2; ++r2) {
      T* op = out + (((size_t)n * P.H + oy0 + r2) * P.W + ox) * P.out_stride;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = 8 * j + cq;
        float f0 = acc2[4 * j + 2 * r2] + s_bias[64 + c], f1 = acc2[4 * j + 2 * r2 + 1] + s_bias[64 + c + 1];
        float x0f, x1f;
        unpack2<T>(rv[r2][j], x0f, x1f);
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
