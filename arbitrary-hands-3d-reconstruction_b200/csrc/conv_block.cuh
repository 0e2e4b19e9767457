// One HRNet BasicBlock (conv3x3-BN-ReLU, conv3x3-BN, + block input, ReLU) as ONE wgmma launch, sm_90a.
//
// Two conv_tc launches move five activation passes through HBM per block (read x, write y, read y, write the output,
// read x again as the residual); this kernel moves two (read x, write the output; the residual re-read of the tile just
// loaded hits L2).  The intermediate y never leaves shared memory.
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
//   * conv1 over the 10 x 18 intermediate region (the tile plus conv2's one-pixel halo), "flat M": the pitch-24 box is a
//     flat array of pixels and intermediate pixel p = r * 24 + c reads input pixel p + ky * 24 + kx for tap (ky, kx), a
//     constant offset.  So every M = 64 block is 64 consecutive flat pixels (8 core groups of 8, SBO = 1024 B) and a tap
//     is a descriptor start (ky * 24 + kx) * 128 B into the box -- an unaligned start, like MODE_P1 (the 128B swizzle
//     follows the absolute address).  10 x 24 = 240 flat pixels take exactly the team's 4 M blocks; warpgroup w of the
//     team owns blocks w and w + 2.  The last block reads up to 18 pixels past the box: a zeroed slack region (those
//     reads only feed the discarded flat row 10 and columns 18..23).
//   * conv1 epilogue IN PLACE: once every conv1 wgmma of the team's tile has completed (a barrier over the team), bias +
//     ReLU, rounded to 16 bits, is stored over the box in the 128B-swizzled K-major layout TMA would have written (16-byte
//     chunk index ^= pixel & 7), with stmatrix: one instruction stores four 8-pixel x 16-byte fragments, so the
//     epilogue issues 8 shared stores per thread instead of 32 (it runs while the other team streams wgmmas, which
//     leave its instructions few issue and shared-memory slots).  Pixels outside the image are stored as ZERO: they are
//     conv2's padding.  stmatrix writes whole M blocks, so flat row 10 and columns 18..23 get values too; conv2 never
//     reads them.  Then fence.proxy.async and a second team barrier: conv2's taps read rows written by the team's other
//     warpgroup.
//   * conv2 reads the intermediate with the MODE_P1 addressing (one 8x8-pixel M block per warpgroup at pitch 24, taps =
//     descriptor starts); once its wgmmas completed the box is handed back to the producer, then the conv2 epilogue
//     (bias, residual from global, ReLU, NHWC stores).
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
//   * `mid` (optional): conv1's output is also stored for the tile's own 16x8 pixels, so an observable intermediate
//     (teacher-forced checks, kept tensors) is still written.
#pragma once
#include "conv_tc.cuh"

namespace acr {

constexpr int BLK_TILE_Y = 8;                                      // output tile: TILE_X (16) x 8 pixels (pairs)
constexpr int BLK_PITCH = 24, BLK_ROWS = BLK_TILE_Y + 4;           // input box: 24 x 12 pixels (pairs), two-pixel halo
constexpr int BLK_MID_ROWS = BLK_TILE_Y + 2, BLK_MID_COLS = TILE_X + 2;   // intermediate region: 10 x 18 at pitch 24
constexpr uint32_t BLK_ROW_BYTES = 128;                            // 64 16-bit channels
constexpr uint32_t BLK_W_BYTES = 9u * 64u * BLK_ROW_BYTES;         // one conv's resident weights: 9 taps x [64][64]
constexpr uint32_t BLK_BOX_BYTES = (uint32_t)BLK_PITCH * BLK_ROWS * BLK_ROW_BYTES;
constexpr int BLK_M_BLOCKS = 4;                                    // conv1 M blocks of a tile: 2 per warpgroup of the team
constexpr int BLK_SLACK_PIX = BLK_M_BLOCKS * 64 + 2 * BLK_PITCH + 2 - BLK_PITCH * BLK_ROWS;
constexpr uint32_t BLK_SLACK_BYTES = (uint32_t)BLK_SLACK_PIX * BLK_ROW_BYTES;
constexpr uint32_t BLK_BOX_STRIDE = (BLK_BOX_BYTES + BLK_SLACK_BYTES + 1023u) & ~1023u;   // box 1 starts 1024-aligned
constexpr uint32_t BLK_OFF_B2 = BLK_W_BYTES;
constexpr uint32_t BLK_OFF_A = 2 * BLK_W_BYTES;                    // box t at BLK_OFF_A + t * BLK_BOX_STRIDE
constexpr uint32_t BLK_OFF_BIAS = BLK_OFF_A + BLK_BOX_STRIDE + BLK_BOX_BYTES + BLK_SLACK_BYTES;
constexpr uint32_t BLK_OFF_BAR = BLK_OFF_BIAS + 2 * 64 * 4;
constexpr size_t BLK_SMEM = 1024 /*alignment slack*/ + BLK_OFF_BAR + 64;
static_assert(BLK_M_BLOCKS * 64 >= BLK_MID_ROWS * BLK_PITCH && (BLK_M_BLOCKS - 1) * 64 < BLK_MID_ROWS * BLK_PITCH,
              "flat-M plan: 4 M blocks of 64 cover the 240 flat intermediate pixels, none discarded");
static_assert(BLK_SLACK_PIX == 18 && BLK_BOX_STRIDE == 39936, "flat-M plan: the last M block reads 18 pixels past the box");
static_assert(BLK_OFF_A % 1024 == 0 && BLK_BOX_STRIDE % 1024 == 0, "128B swizzle: every box starts on a 1024 B boundary");
static_assert(BLK_MID_ROWS * BLK_PITCH * BLK_ROW_BYTES <= BLK_BOX_BYTES, "the intermediate fits in the box it overwrites");
static_assert(BLK_M_BLOCKS * 64 <= BLK_PITCH * BLK_ROWS, "the conv1 epilogue's whole-block stores stay inside the box");
static_assert(BLK_SMEM == 228160 && BLK_SMEM <= (size_t)SMEM_BUDGET,
              "fused-block shared-memory plan: 144 KB weights + two 1024-aligned boxes with slack + biases + barriers");
static_assert(TILE_Y % BLK_TILE_Y == 0, "the 16-row super-tile precondition covers the 8-row tiles");
constexpr int BLK_BAR = 1;   // named barrier BLK_BAR + t over the 256 threads of team t

struct ConvBlockParams {
  CUtensorMap tmA;          // block input x {C, W, H, B}, box {64, 24, 12}
  CUtensorMap tmB1, tmB2;   // packed weights of conv1 / conv2 [64][9 * 64], box {64, 64}
  const float* bias1;
  const float* bias2;
  const void* res;          // the block input again (residual of conv2)
  void* out;
  void* mid;                // conv1's output buffer, or nullptr when nothing reads it
  int res_stride, out_stride, mid_stride;
  int H, W, tiles_x, tiles_per_img, total_tiles;   // 16 x 8 tiles
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

// pull one TMA box into L2 (no shared-memory destination, no completion to wait for)
__device__ __forceinline__ void tma_prefetch_l2_4d(const CUtensorMap* map, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.prefetch.tensor.4d.L2.global.tile [%0, {%1, %2, %3, %4}];"
               ::"l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}

// four 8x8 16-bit fragments (r_i = this thread's pair of fragment i) to shared memory; lane l gives the address of row
// l & 7 of fragment l >> 3
__device__ __forceinline__ void stsm_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1), "r"(r2),
               "r"(r3) : "memory");
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
  constexpr uint32_t pix16 = BLK_ROW_BYTES >> 4, row16 = (uint32_t)BLK_PITCH * pix16;
  const int blk0 = w, blk1 = w + 2;                                  // conv1 M blocks of this warpgroup
  const int cq = 2 * (lane & 3);
  const uint32_t is_lane0 = lane == 0 ? 1u : 0u;
  const T* res = reinterpret_cast<const T*>(P.res);
  T* out = reinterpret_cast<T*>(P.out);
  T* mid = reinterpret_cast<T*>(P.mid);
  float acc0[32], acc1[32];
  // turn s exists when the CTA has its tile (see the header); turn_pre / turn_post: wait for the turn, hand it on
  auto turn_exists = [&](int s) -> uint32_t { return (s >= 0 && 2 * (s >> 2) + (s & 1) < ntiles) ? 1u : 0u; };
  auto turn_pre = [&](int s) { named_bar_sync_if(TEAM_BAR + team, 512, turn_exists(s - 1)); };
  auto turn_post = [&](int s) { named_bar_arrive_if(TEAM_BAR + (team ^ 1), 512, turn_exists(s + 1)); };

  // conv1 epilogue of one M block, in place over the box; bb[j] = conv1's bias of channels 8 j + cq, + 1
  auto mid_store = [&](const float* acc, const float2* bb, int blk, int y0, int x0, int n) {
#pragma unroll
    for (int r2 = 0; r2 < 2; ++r2) {
      const int q = 64 * blk + 16 * wq + (lane >> 2) + 8 * r2;    // flat intermediate pixel of this thread's values
      const int r = q / BLK_PITCH, c = q - r * BLK_PITCH;
      const int y = y0 - 1 + r, x = x0 - 1 + c;
      const bool inside = r < BLK_MID_ROWS && c < BLK_MID_COLS && y >= 0 && y < P.H && x >= 0 && x < P.W;
      uint32_t v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float f0 = acc[4 * j + 2 * r2] + bb[j].x, f1 = acc[4 * j + 2 * r2 + 1] + bb[j].y;
        f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f);
        v[j] = inside ? pack2<T>(f0, f1) : 0u;
      }
      if (mid != nullptr && inside && r >= 1 && r <= BLK_TILE_Y && c >= 1 && c <= TILE_X) {
        T* mp = mid + (((size_t)n * P.H + y) * P.W + x) * P.mid_stride + cq;
#pragma unroll
        for (int j = 0; j < 8; ++j) *reinterpret_cast<uint32_t*>(mp + 8 * j) = v[j];
      }
      // lane l stores row l & 7 of chunks 4 h + (l >> 3); that pixel's swizzle is l & 7
      const uint32_t row = a_base + (uint32_t)(64 * blk + 16 * wq + 8 * r2 + (lane & 7)) * BLK_ROW_BYTES;
#pragma unroll
      for (int h = 0; h < 2; ++h)
        stsm_x4(row + (((uint32_t)(4 * h + (lane >> 3)) ^ (uint32_t)(lane & 7)) << 4), v[4 * h], v[4 * h + 1], v[4 * h + 2],
                v[4 * h + 3]);
    }
  };

  for (int k = team; k < ntiles; k += 2) {
    const int tile = (int)blockIdx.x + k * (int)gridDim.x;
    const int n = tile / P.tiles_per_img, rem = tile % P.tiles_per_img;
    const int y0 = (rem / P.tiles_x) * BLK_TILE_Y, x0 = (rem % P.tiles_x) * TILE_X;
    const int s = 2 * k - team;   // this tile's conv1 turn; its conv2 turn is s + 2
    mbar_wait_parity(full_bar, (uint32_t)(k >> 1) & 1u);
    // ---- conv1 over the flat 10 x 24 region
    turn_pre(s);
    wgmma_fence();
    blk_conv<T, XPAIR, 2>(acc0, acc1, a_lo + (uint32_t)(64 * blk0) * pix16, a_lo + (uint32_t)(64 * blk1) * pix16, hi_flat, row16,
                          b1_lo, hi_b);
    wgmma_commit();
    turn_post(s);
    wgmma_wait<0>();
    wgmma_acc_fence<32>(acc0);
    wgmma_acc_fence<32>(acc1);
    named_bar_sync(BLK_BAR + team, 256);   // every conv1 wgmma of the tile has read the box: overwrite it
    float2 bb[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) bb[j] = *reinterpret_cast<const float2*>(s_bias + 8 * j + cq);
    mid_store(acc0, bb, blk0, y0, x0, n);
    mid_store(acc1, bb, blk1, y0, x0, n);
    fence_proxy_async();                   // generic-proxy stores -> wgmma operand reads
    named_bar_sync(BLK_BAR + team, 256);
    // ---- conv2 over the intermediate, MODE_P1 addressing
    turn_pre(s + 2);
    wgmma_fence();
    blk_conv<T, XPAIR, 1>(acc0, acc0, a_lo + (uint32_t)w * 8u * pix16, 0u, hi_p1, row16, b2_lo, hi_b);
    wgmma_commit();
    turn_post(s + 2);
    // the residual (conv2's epilogue) is loaded while conv2's wgmmas run: all 16 loads in flight at once, where loads
    // interleaved with the output stores would each wait out an L2 round trip
    const int oy0 = y0 + 2 * wq, ox = x0 + w * HALF_X + (lane >> 2);
    uint32_t rv[2][8];
#pragma unroll
    for (int r2 = 0; r2 < 2; ++r2) {
      const T* rp = res + (((size_t)n * P.H + oy0 + r2) * P.W + ox) * P.res_stride;
#pragma unroll
      for (int j = 0; j < 8; ++j) rv[r2][j] = *reinterpret_cast<const uint32_t*>(rp + 8 * j + cq);
    }
    wgmma_wait<0>();
    wgmma_acc_fence<32>(acc0);
    __syncwarp();
    mbar_arrive_if(empty_bar, is_lane0);   // the box is free: the team's next tile loads under the other team's MMAs
    // ---- conv2 epilogue: + bias + residual, ReLU
#pragma unroll
    for (int r2 = 0; r2 < 2; ++r2) {
      T* op = out + (((size_t)n * P.H + oy0 + r2) * P.W + ox) * P.out_stride;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = 8 * j + cq;
        float f0 = acc0[4 * j + 2 * r2] + s_bias[64 + c], f1 = acc0[4 * j + 2 * r2 + 1] + s_bias[64 + c + 1];
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
