// Implicit-GEMM NHWC convolution on the Hopper tensor cores (wgmma + TMA + mbarrier), sm_90a.
//
// Replaces every nn.Conv2d + BatchNorm2d (+ReLU, +residual add) of the reference network (acr/model.py: BasicBlock,
// Bottleneck, transition / fuse convs, SegmNet, head stacks, contact conv), which the reference dispatches to cuDNN +
// separate ATen elementwise kernels.
//
// GEMM view:  D[M = 64 output pixels][N = nsub] += A[M][K] * B[N][K],  K = taps * cin_pad.
//   * Work unit = a 16x16-pixel SUPER-TILE of one image, computed by four consumer warpgroups: warpgroup g owns the M = 64
//     block of half g & 1 (left / right 8 columns) and image rows 8 (g >> 1) .. 8 (g >> 1) + 7 (8 swizzle atoms of 8 pixels
//     at a uniform stride).  Each holds its 64 x nsub fp32 accumulator in registers (nsub <= 128: wider layers run as
//     "virtual tiles" of nsub channels, ConvTcParams::nsplit), so activations are never re-read across more N tiles than that.
//   * A operand by TMA, the conv padding by TMA's out-of-bounds zero fill.  3x3 stride-1 convs with 64-channel chunks load
//     ONE haloed box {64, 24, 18} per chunk and address all nine taps inside it through wgmma descriptors whose start is
//     NOT aligned to the swizzle repeat (MODE_P1; the 128B swizzle follows the absolute shared-memory address, as the TMA
//     unit wrote it); narrower chunks use three kx-shifted boxes {CK, 16, 18} with the ky taps as row offsets
//     (MODE_PATCH).  Dense 32-channel tensors are convolved as x-pairs (two pixels per 128-byte row): stride 1 as a
//     64->64 conv with block-sparse weights whose side taps are 32x32 corners (MODE_XPAIR), stride 2 from two row-parity
//     boxes with taps = row offset + pair-column offset + K half (MODE_S2X).  Other stride-2 convs read four parity views
//     (even/odd rows x columns, own tensor maps), 1x1 convs a single tap.
//   * B operand: packed weights [cout_pad][taps*cin_pad] (BN folded), 2-D TMA boxes {CK, N}; resident in shared memory for
//     the whole kernel when they fit (all 32/64-channel layers), otherwise streamed through their own mbarrier ring.
//   * Both land in shared memory in the canonical K-major swizzled layout (128B / 64B / 32B swizzle for CK = 64 / 32 / 16)
//     that wgmma descriptors address directly.
//   * 1x1 stride-2 convs read parity view 0 at offset 0 (padding 0); transposed convs (MODE_DECONV) are four 2x2 convs
//     on the input grid, one per output parity.
//   * Persistent CTAs (one per SM): warps 0..15 = the four consumer warpgroups (wgmma issue, then the epilogue straight
//     from the accumulator registers: +bias (+residual) (+extra terms) (ReLU) -> 16-bit / fp32 NHWC); warps 16..19 = the
//     producer warpgroup, whose first warp issues the TMA loads and runs ahead into the next tile's operands.  The producer
//     gives registers to the consumers (setmaxnreg).
//   * Resident weights: the consumers run as two ping-pong teams by row group (warpgroups {0,1} and {2,3}), so one team's
//     epilogue overlaps the other team's MMAs.  Streamed weights: all four warpgroups issue in lockstep.
//   * T = float (the TF32 plan): fp32 activations and weights, tf32 MMAs with fp32 accumulation.  All shared-memory geometry
//     is in bytes, and CK counts 16-bit channels: an fp32 NHWC tensor with C channels is, for the TMA boxes, the swizzle
//     and the descriptors, byte-identical to a 16-bit tensor with 2C channels (CK = 64 / 32 hold 32 / 16 fp32 channels),
//     and one k8 tf32 step reads the 32 bytes of K of one k16 16-bit step.  The three otherwise idle producer warps round
//     every landed A stage to the nearest tf32 before the consumers read it (readyA).  The residual is read and the output
//     stored as fp32.  No x-paired, x-paired stride-2 or transposed form, no extra terms, no TMA-store epilogue.
#pragma once
#include <cuda.h>
#include <stdlib.h>

#include "ops.cuh"
#include "wgmma.cuh"

namespace acr {

// ------------------------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// one lane of a converged warp issues (keeps TMA issue on the uniform datapath)
__device__ __forceinline__ bool elect_one_sync() {
  uint32_t pred;
  asm volatile("{\n.reg .pred p;\nelect.sync _|p, 0xffffffff;\nselp.u32 %0, 1, 0, p;\n}" : "=r"(pred));
  return pred != 0;
}
// Programmatic dependent launch: a kernel launched with the programmatic-stream-serialisation attribute may
// start while its predecessor is still draining; everything that touches the predecessor's outputs (or
// writes memory the predecessor may still read) comes after pdl_wait().
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
// TMA store of one shared-memory slab (shared -> global, bulk async-group completion)
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(map), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }
// arrive (without waiting) when pred != 0; one asm statement, so it may sit between wgmma commit and wait
__device__ __forceinline__ void named_bar_arrive_if(int id, int nthreads, uint32_t pred) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.u32 p, %2, 0;\n@p bar.arrive %0, %1;\n}\n" ::"r"(id), "r"(nthreads), "r"(pred) : "memory");
}
// per-thread register budget of the executing warpgroup (warpgroup-collective)
template <int N> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
__device__ __forceinline__ void sts32(uint32_t addr, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
__device__ __forceinline__ uint64_t desc_lohi(uint32_t lo, uint32_t hi) { return ((uint64_t)hi << 32) | lo; }

// two 16-bit values <-> two floats through one 32-bit access
template <typename T>
__device__ __forceinline__ void unpack2(uint32_t u, float& a, float& b) {
  const T* p = reinterpret_cast<const T*>(&u);
  a = to_f32<T>(p[0]);
  b = to_f32<T>(p[1]);
}
template <typename T>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  uint32_t u;
  T* p = reinterpret_cast<T*>(&u);
  p[0] = from_f32<T>(a);
  p[1] = from_f32<T>(b);
  return u;
}

// ------------------------------------------------------------------------------------ kernel
// The CTA works on 16x16-pixel super-tiles: ONE TMA box per (channel chunk, kx) (or per channel chunk, MODE_P1) feeds all
// four M = 64 blocks and three (nine) taps.
constexpr int TILE_Y = 16, TILE_X = 16, HALF_X = 8;
constexpr int CONSUMER_WARPS = 16;                 // four warpgroups, one M = 64 block of the super-tile each
constexpr int PRODUCER_WARP = CONSUMER_WARPS;      // first warp of the producer warpgroup: the TMA issuer
constexpr int TC_THREADS = 32 * (CONSUMER_WARPS + 4);
// Register split: 640 threads launch with 96 registers each (61440 of the SM's 64K).  The producer warpgroup drops to 32,
// which lets the consumers rise to 112 (16 x 32 x 112 + 4 x 32 x 32 = 61440): room for a 64-register accumulator (NT = 128)
// without spilling.
constexpr int PRODUCER_REGS = 32, CONSUMER_REGS = 112;
static_assert(CONSUMER_WARPS * 32 * CONSUMER_REGS + 4 * 32 * PRODUCER_REGS <= (65536 / TC_THREADS) / 8 * 8 * TC_THREADS,
              "setmaxnreg split exceeds the launch allocation");
// named barriers of the ping-pong teams (ids 1..4 are the TMA-store epilogue's per-warpgroup barriers): barrier
// TEAM_BAR + t completes when team t may issue its next tile
constexpr int TEAM_BAR = 5;
constexpr int MAX_NSUB = 128;                      // accumulator columns per warpgroup (64 fp32 registers per thread)
constexpr int SMEM_BUDGET = 224 * 1024;            // of the 227 KB a Hopper block may opt into

struct ConvTcParams {
  CUtensorMap tmA[4];
  CUtensorMap tmB;
  const void* ext[3];  // extra terms added before the activation (folded fuse sums), read at (oy >> shift, ox >> shift)
  int n_ext, ext_shift[3], ext_stride[3], ext_W[3], ext_H[3];
  CUtensorMap tmOut;   // TMA-store epilogue: output as {C, W, H, B}, box {64, 8, 8, 1}, 128B swizzle
  int tma_out;         // epilogue stages 64-channel slabs in shared memory and stores them with TMA (16-bit, nsub % 64 == 0)
  uint32_t stage_out_bytes;
  const float* bias;
  const void* res;
  void* out;
  int taps, ksz, stride, cchunks, cin_pad, npad, relu, has_res, out_f32, bias_per_image, pow11_ch0;
  uint32_t bias_bytes;  // shared-memory bias region (cout_pad floats, rounded to 1 KB)
  int nsplit, nsub;     // N split: every super-tile is computed as nsplit "virtual tiles" of nsub output channels (the last
                        // one may extend past cout_pad: those columns are computed from zero / unused weights and not stored)
  int xpair;    // x-paired 32->32 conv run as 64->64 (see below): side taps are quarter blocks
  int patch_mode, b_resident, SA, SB;
  int pingpong;   // resident weights and a tile's A loads fit in the ring: the consumer teams alternate (see the kernel)
  int patch1;   // MODE_P1: ONE 24-wide haloed box per channel chunk, kx shifts = unaligned descriptor starts
  int s2x;      // MODE_S2X: 3x3 stride-2 conv of a dense 32-channel tensor read as x-pairs: two row-parity boxes per tile
  int deconv;   // MODE_DECONV: transposed conv k4 s2 p1; tiles_x / tiles_per_img count INPUT super-tiles, Ho / Wo the output
  uint32_t a_stage_bytes, b_block_bytes, b_region_bytes;
  int tiles_x, tiles_per_img, total_tiles, Ho, Wo, out_stride, res_stride;
};

// kx served by the i-th A patch of a channel chunk (x-paired convs take the centre tap first, as the weights are packed)
__device__ __forceinline__ int patch_kx(int i, int xpair) { return xpair ? (i == 0 ? 1 : (i == 1 ? 0 : 2)) : i; }

template <int CK>
struct SwizzleCfg {
  static constexpr uint32_t kRowBytes = CK * 2;
  static constexpr uint32_t kAtom = 8 * kRowBytes;          // 8 pixels of one image row = one swizzle atom
  static constexpr uint32_t kSBO_A = TILE_X * kRowBytes;    // next image row of the 16-wide box
  static constexpr uint32_t kSwizzle = gmma_swizzle(kRowBytes);
};

// MODE bits (compile-time specialisation of the issue loop)
constexpr int MODE_PATCH = 1, MODE_RESIDENT = 2, MODE_XPAIR = 4;
// MODE_P1 (with MODE_PATCH, CK = 64): the whole haloed input patch of a super-tile is ONE TMA box {64, 24, 18} per channel
// chunk (x0-1 .. x0+22, y0-1 .. y0+16; the row pitch of 24 pixels keeps every image row on a swizzle-atom boundary).
// The nine taps are nine descriptors into it: ky moves the start by whole image rows, kx by single pixels -- a start
// address that is NOT aligned to the 1024-byte swizzle repeat.  The 128-byte swizzle is a function of the ABSOLUTE
// shared-memory address bits (chunk ^= (addr >> 7) & 7), exactly like the TMA unit wrote the box, so any 128-byte-aligned
// start works with base offset 0.  One box instead of three: a third of the TMA issues, half the L2 -> smem bytes.
constexpr int MODE_P1 = 16;
constexpr int P1_PITCH = 24;   // pixels per image row of the single box
// MODE_S2X (CK = 64): 3x3 STRIDE-2 conv whose input is a dense 32-channel tensor, viewed as (H, W/2, 64): one 128-byte
// row = an even pixel's 32 channels followed by its odd neighbour's.  Output pixel (oy, ox) reads input columns
// 2ox-1, 2ox, 2ox+1 = [pair ox-1, odd half], [pair ox, even half], [pair ox, odd half] and rows 2oy-1, 2oy, 2oy+1 =
// odd-row view row oy-1, even-row view row oy, odd-row view row oy+1.  So a 16x16 output tile needs TWO boxes
// {64, 24 pair columns from x0-1, 17 rows} (even rows from y0, odd rows from y0-1) instead of nine 64-byte-row
// boxes of four parity views: the nine taps are descriptor starts inside them (row offset 0/1, pair-column offset
// 0/1 = an unaligned start, K half 0/1 = k-steps {0,1} or {2,3}).  The packed weights carry the 32 input channels
// of tap (ky,kx) at K offset 32*(kx != 1) (engine._pack_conv(s2x=True)).
constexpr int MODE_S2X = 32;
// MODE_DECONV (CK = 64, streamed weights, lockstep): ConvTranspose2d kernel 4 stride 2 padding 1.  Output pixel
// (2m+py, 2n+px) is a 2x2 conv of the input at offsets {py-1, py} x {px-1, px}, so every output parity is an ordinary
// conv on the INPUT grid: the super-tile is 16x16 input pixels, read as the MODE_P1 haloed box {64, 24, 18} from
// (x0-1, y0-1), and parity (py,px) issues only its 4 live taps, tap (ty,tx) = descriptor start (py+ty) rows and (px+tx)
// pixels into the box.  Parity x N split are virtual tiles (parity-major within a super-tile); the weights are
// [4 parities][cout_pad][4 taps][cin_pad], so parity p streams rows p * cout_pad + n_off.  The epilogue stores at
// stride 2: pixel (2 oy + py, 2 ox + px) of the output.
constexpr int MODE_DECONV = 64;

template <int CK, typename T, int MODE, int NT>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_tc_kernel(const __grid_constant__ ConvTcParams P) {
  using Cfg = SwizzleCfg<CK>;
  constexpr bool PATCH = (MODE & MODE_PATCH) != 0, RESIDENT = (MODE & MODE_RESIDENT) != 0, XPAIR = (MODE & MODE_XPAIR) != 0;
  constexpr bool P1 = (MODE & MODE_P1) != 0, S2X = (MODE & MODE_S2X) != 0, DECONV = (MODE & MODE_DECONV) != 0;
  constexpr int NPAR = DECONV ? 4 : 1;   // virtual tiles per (super-tile, N split)
  static_assert(!P1 || (PATCH && CK == 64 && !XPAIR), "the single-box form exists for CK = 64 patch convs (not x-paired)");
  static_assert(!S2X || (!PATCH && !P1 && !XPAIR && CK == 64), "the x-paired stride-2 form is a CK = 64 mode of its own");
  static_assert(!DECONV || (MODE == MODE_DECONV && CK == 64), "the transposed conv is a CK = 64 streamed-weight mode of its own");
  static_assert((NT == 64 || NT == 128) && (!XPAIR || NT == 64), "MMA width: 64 or 128 columns (x-paired convs: 64)");
  // a 32-channel fp32 pixel already fills a 128-byte row: nothing to pair, and stride-2 convs read the four parity views
  static_assert(!IsF32<T>::value || !(XPAIR || S2X || DECONV), "fp32 (tf32) operands: no x-paired, stride-2 x-paired or transposed form");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;  // swizzle atoms need 1024-byte alignment
  const int SA = P.SA, SB = P.SB;
  const uint32_t b_base = base;
  const uint32_t a_base = base + P.b_region_bytes;
  const uint32_t stage_base = a_base + (uint32_t)SA * P.a_stage_bytes;  // TMA-store epilogue: 4 x 8 KB output slabs
  const uint32_t bias_base = stage_base + P.stage_out_bytes;             // fp32 bias[npad]
  const uint32_t bar_base = bias_base + P.bias_bytes;
  // barrier map: fullA[SA] emptyA[SA] fullB[SB] emptyB[SB] bres
  auto fullA = [&](int s) { return bar_base + 8u * s; };
  auto emptyA = [&](int s) { return bar_base + 8u * (SA + s); };
  auto fullB = [&](int s) { return bar_base + 8u * (2 * SA + s); };
  auto emptyB = [&](int s) { return bar_base + 8u * (2 * SA + SB + s); };
  const uint32_t bres_bar = bar_base + 8u * (2 * SA + 2 * SB);
  const uint32_t dummy_bar = bres_bar + 8u;   // target of the "no stage" arrivals of the consumers (never waited on)
  // T = float: readyA[SA] after the dummy -- stage s rounded to tf32 (see the producer); the consumers wait on it instead
  // of fullA
  auto readyA = [&](int s) { return dummy_bar + 8u * (1 + s); };
  auto stageA = [&](int s) {
    if constexpr (IsF32<T>::value) return readyA(s);
    else return fullA(s);
  };
  float* s_bias = reinterpret_cast<float*>(smem_raw + (bias_base - raw));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nA = DECONV ? P.cchunks : (P.s2x ? 2 : (P.patch1 ? P.cchunks : (P.patch_mode ? P.cchunks * 3 : P.taps * P.cchunks)));  // A loads per super-tile
  const int nsub_taps = DECONV ? 4 : (P.patch1 ? 9 : (P.patch_mode ? 3 : 1));                  // taps served by one A load

  if (threadIdx.x == 0) {
    // a stage is free again once every consumer warp has seen the wgmmas that read it complete
    for (int s = 0; s < SA; ++s) { mbar_init(fullA(s), 1); mbar_init(emptyA(s), CONSUMER_WARPS); }
    for (int s = 0; s < SB; ++s) { mbar_init(fullB(s), 1); mbar_init(emptyB(s), CONSUMER_WARPS); }
    mbar_init(bres_bar, 1);
    mbar_init(dummy_bar, 1);
    if constexpr (IsF32<T>::value)
      for (int s = 0; s < SA; ++s) mbar_init(readyA(s), 3);
    fence_barrier_init();
    tma_prefetch_desc(&P.tmB);
    tma_prefetch_desc(&P.tmA[0]);
    if (P.tma_out) tma_prefetch_desc(&P.tmOut);
  }
  if (!P.bias_per_image)
    for (int i = threadIdx.x; i < P.npad; i += TC_THREADS) s_bias[i] = P.bias[i];
  __syncthreads();
  // let the next kernel of the stream begin its own prologue as soon as SMs drain; our own prologue above touched
  // nothing the previous kernel produces
  pdl_launch_dependents();

  if (warp >= CONSUMER_WARPS) {
    // ===================================================================== TMA producer warpgroup
    // (one warp issues: it stays converged and one elected lane issues; the other three only give up registers)
    setmaxnreg_dec<PRODUCER_REGS>();
    if constexpr (IsF32<T>::value) {
      if (warp != PRODUCER_WARP) {
        // the other three warps: once a stage has landed, round its fp32 activations in place to the nearest tf32
        // (cvt.rna: ties away from zero), make the writes visible to the MMAs (async proxy) and release the stage to the
        // consumers.  Fed as stored, the tensor cores would drop the low 13 bits of every activation: a bias of half a
        // tf32 ulp per product, which the network accumulates (DESIGN.md, TF32 plan).  The weights are rounded on the host.
        const int ct = threadIdx.x - 32 * (PRODUCER_WARP + 1);
        int sa = 0;
        uint32_t pha = 0;
        for (int vt = blockIdx.x; vt < P.total_tiles * P.nsplit; vt += gridDim.x)
          for (int a = 0; a < nA; ++a) {
            mbar_wait_parity(fullA(sa), pha);
            {
              uint4* st = reinterpret_cast<uint4*>(smem_raw + (a_base - raw) + (uint32_t)sa * P.a_stage_bytes);
              for (uint32_t i = ct; i < P.a_stage_bytes / 16u; i += 96) {
                const float4 v = reinterpret_cast<const float4*>(st)[i];
                uint4 r;
                asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r.x) : "f"(v.x));
                asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r.y) : "f"(v.y));
                asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r.z) : "f"(v.z));
                asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r.w) : "f"(v.w));
                st[i] = r;
              }
              fence_proxy_async();
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(readyA(sa));
            if (++sa == SA) { sa = 0; pha ^= 1u; }
          }
        return;
      }
    }
    if (warp != PRODUCER_WARP) return;
    if (P.b_resident && elect_one_sync()) {  // whole weight tensor once per CTA
      const int nblk = P.taps * P.cchunks;
      mbar_expect_tx(bres_bar, (uint32_t)nblk * P.b_block_bytes);
      for (int i = 0; i < nblk; ++i)
        tma_load_2d(b_base + (uint32_t)i * P.b_block_bytes, &P.tmB, bres_bar, (i / P.cchunks) * P.cin_pad + (i % P.cchunks) * CK, 0);
    }
    __syncwarp();
    pdl_wait();   // weights are constants; the activations below are the previous kernel's output
    int sa = 0, sb = 0;
    uint32_t pha = 0, phb = 0;
    for (int vt = blockIdx.x; vt < P.total_tiles * P.nsplit * NPAR; vt += gridDim.x) {
      const int tile = vt / (P.nsplit * NPAR), vr = vt - tile * (P.nsplit * NPAR);
      const int par = DECONV ? vr / P.nsplit : 0;
      const int n_off = (vr - par * P.nsplit) * P.nsub;
      const int b_row = DECONV ? par * P.npad + n_off : n_off;   // first weight row of this virtual tile
      const int n = tile / P.tiles_per_img, rem = tile % P.tiles_per_img;
      const int y0 = (rem / P.tiles_x) * TILE_Y, x0 = (rem % P.tiles_x) * TILE_X;
      for (int a = 0; a < nA; ++a) {
        int cc, view = 0, dy = 0, dx = 0, tap0;
        int nsub_a = nsub_taps;
        if (DECONV) {                 // one 18x24 box per channel chunk, as MODE_P1; the parity picks taps inside it
          cc = a; dy = -1; dx = -1; tap0 = 0;
        } else if (P.s2x) {                // a = row parity: even rows from y0 (taps ky=1), odd rows from y0-1 (ky=0,2)
          cc = 0; view = a; dy = a ? -1 : 0; dx = -1; tap0 = 0; nsub_a = a ? 6 : 3;
        } else if (P.patch1) {        // one 18x24 box per channel chunk: rows y0-1 .. y0+16, columns x0-1 .. x0+22
          cc = a; dy = -1; dx = -1; tap0 = 0;
        } else if (P.patch_mode) {    // one 18x16 box per (channel chunk, kx); rows y0-1 .. y0+16
          cc = a / 3; const int kx = patch_kx(a % 3, P.xpair);
          dy = -1; dx = kx - 1; tap0 = kx;
        } else {
          const int tap = a / P.cchunks; cc = a % P.cchunks; tap0 = tap;
          if (P.ksz == 3) {
            const int ky = tap / 3, kx = tap % 3;
            if (P.stride == 1) { dy = ky - 1; dx = kx - 1; }
            else {  // input row 2*oy + ky - 1 = 2*(oy + dy) + py
              const int py = (ky == 1) ? 0 : 1, px = (kx == 1) ? 0 : 1;
              dy = (ky == 0) ? -1 : 0; dx = (kx == 0) ? -1 : 0;
              view = py * 2 + px;
            }
          }
        }
        mbar_wait_parity(emptyA(sa), pha ^ 1u);
        if (elect_one_sync()) {
          mbar_expect_tx(fullA(sa), P.a_stage_bytes);
          tma_load_4d(a_base + (uint32_t)sa * P.a_stage_bytes, &P.tmA[view], fullA(sa), cc * CK, x0 + dx, y0 + dy, n);
        }
        __syncwarp();
        if (++sa == SA) { sa = 0; pha ^= 1u; }
        if (!P.b_resident) {
          for (int sub = 0; sub < nsub_a; ++sub) {
            // weight block order = the consumers' tap order (single box: ky-major, kx 1,0,2 for x-paired convs;
            // stride-2 pairs: ky=1 with the even-row box, then ky=0 and ky=2 with the odd-row box)
            // (transposed conv: the 4 taps (ty,tx) of this parity, row-major)
            const int tap = DECONV ? sub : P.s2x ? (a == 0 ? 3 + sub : (sub < 3 ? sub : 3 + sub))
                                  : (P.patch1 ? (sub / 3) * 3 + patch_kx(sub % 3, P.xpair) : (P.patch_mode ? sub * 3 + tap0 : tap0));
            mbar_wait_parity(emptyB(sb), phb ^ 1u);
            if (elect_one_sync()) {
              mbar_expect_tx(fullB(sb), P.b_block_bytes);
              tma_load_2d(b_base + (uint32_t)sb * P.b_block_bytes, &P.tmB, fullB(sb), tap * P.cin_pad + cc * CK, b_row);
            }
            __syncwarp();
            if (++sb == SB) { sb = 0; phb ^= 1u; }
          }
        }
      }
    }
    return;
  }

  // ========================================================================= consumer warpgroups
  // Every thread of a warpgroup runs the same issue loop (wgmma is warpgroup-collective).  Per group of wgmmas (one tap, or
  // a whole A stage when the weights are resident): wait for the operands, fence, the k16 steps of the chunk as wgmma
  // m64nNTk16 into the register accumulator, commit.  A committed group is known complete one group later
  // (wgmma.wait_group 1); only then are the operand stages it read handed back to the producer.  Between the wgmmas there
  // is no C++ branch or call (waits and arrivals are single asm statements, NT and the tap pattern are compile-time):
  // otherwise ptxas serialises the wgmmas.
  //
  // Ping-pong (resident weights): team rg (warpgroups 2 rg, 2 rg + 1) issues ALL wgmmas of a tile, then hands the turn
  // to the other team and only then waits for its own MMAs and runs its epilogue, which so overlaps the other team's
  // MMAs.  Barrier TEAM_BAR + t: team t waits on it (bar.sync) before a tile, the other team arrives after issuing its
  // own tile.  Team 1 pre-arrives once so that team 0 goes first, and skips its arrival after its last tile, so every
  // barrier phase completes by kernel exit.  Both teams read the same A stages, which the producer refills only after
  // all 16 consumer warps released them, so the A ring must hold all loads of a tile (P.pingpong, set by the plan):
  // otherwise the first team would wait for a stage that only the second team, still waiting for its turn, can free.
  // Streamed weights stay in lockstep: staggered teams would read every streamed B block a team phase apart, so the
  // B ring would have to hold a whole tile of weights.
  constexpr bool PINGPONG = RESIDENT;
  const bool pingpong = PINGPONG && P.pingpong != 0;
  setmaxnreg_inc<CONSUMER_REGS>();
  const int wg = warp >> 2, wq = warp & 3;
  const int h = wg & 1, rg = wg >> 1;           // half (left / right 8 columns), row group (image rows 0..7 / 8..15)
  if (RESIDENT) mbar_wait_parity(bres_bar, 0);
  pdl_wait();   // residual / extra-term / per-image bias reads and every output write wait for the previous kernel
  constexpr uint32_t pitch16 = ((P1 || S2X || DECONV) ? P1_PITCH * Cfg::kRowBytes : Cfg::kSBO_A) >> 4;   // image row pitch of the A box
  const uint32_t hi_a = pitch16 | (Cfg::kSwizzle << 30);          // SBO = next image row (= next 8-pixel core-matrix group)
  const uint32_t hi_b = (Cfg::kAtom >> 4) | (Cfg::kSwizzle << 30);
  const uint32_t lo_flags = 1u << 16;                              // LBO (unused by swizzled K-major operands)
  // this warpgroup's 64 rows start h * 8 pixels and rg * 8 image rows into the box
  const uint32_t a_lo_base = (((a_base >> 4) & 0x3FFF) | lo_flags) + (uint32_t)h * (Cfg::kAtom >> 4) + (uint32_t)(rg * 8) * pitch16;
  const uint32_t b_lo_base0 = ((b_base >> 4) & 0x3FFF) | lo_flags;
  const uint32_t b_block16 = P.b_block_bytes >> 4, a_stage16 = P.a_stage_bytes >> 4;
  const int cchunks = P.cchunks, taps = P.taps, nsub = P.nsub;
  const bool tma_out = P.tma_out != 0;   // (16-bit outputs only: conv_tc_prepare)
  const bool plain = !tma_out && !P.has_res && !P.pow11_ch0 && P.n_ext == 0;   // short epilogue (see below)
  const int wg_thread = threadIdx.x & 127;
  const uint32_t stage_wg = stage_base + (uint32_t)wg * 8192u;      // this warpgroup's output slab (TMA-store epilogue)
  const uint32_t is_lane0 = lane == 0 ? 1u : 0u;
  float acc[NT / 2];
  uint32_t scale = 0;   // 0 for the first wgmma of a tile (overwrites the accumulator), then 1

  // the wgmmas of one (A stage, tap)
  auto issue = [&](uint32_t a_tap, uint32_t b_lo, int kx) {
    if (XPAIR && kx != 1) {
      // side taps of the x-paired conv connect ONE pixel of the neighbouring pair to ONE of ours: a 32x32 corner of the
      // 64x64 block.  left pair (kx 0): K 32..63 -> N 0..31; right pair (kx 2): K 0..31 -> N 32..63.  Only the corner's
      // two k-steps are issued, at full width: the packed weights are zero outside the corner, so the other 32 columns
      // receive exact zeros (bit-identical to corner-only MMAs, which ptxas would serialise next to full-width ones for
      // lack of registers).  Never the first tap of a tile: the centre tap is issued first.
      const int ks0 = kx == 0 ? 2 : 0;
#pragma unroll
      for (int ks = ks0; ks < ks0 + 2; ++ks)
        wgmma_m64k16<NT, T>(acc, desc_lohi(a_tap + ks * 2, hi_a), desc_lohi(b_lo + ks * 2, hi_b));
    } else {
#pragma unroll
      for (int ks = 0; ks < CK / 16; ++ks) {
        wgmma_m64k16<NT, T>(acc, desc_lohi(a_tap + ks * 2, hi_a), desc_lohi(b_lo + ks * 2, hi_b), scale);
        scale = 1;
      }
    }
  };
  // barriers of the stages read by the newest committed group (not yet known complete); `dummy` when there is none
  uint32_t pend_a = dummy_bar, pend_b = dummy_bar;
  auto release = [&]() {
    __syncwarp();
    mbar_arrive_if(pend_b, is_lane0);
    mbar_arrive_if(pend_a, is_lane0);
    pend_a = pend_b = dummy_bar;
  };
  // close the group of wgmmas just issued; the previous group has then completed: free what it read
  auto group_done = [&](uint32_t a_bar, uint32_t b_bar) {
    wgmma_commit();
    wgmma_wait<1>();
    release();
    pend_a = a_bar; pend_b = b_bar;
  };

  int sa = 0, sb = 0;
  uint32_t pha = 0, phb = 0;
  uint32_t xa_bar[3];   // x-paired form: the three A stages of the tile, released once its MMAs completed
  const int nvt = P.total_tiles * P.nsplit * NPAR;
  if (pingpong && rg == 1) named_bar_arrive_if(TEAM_BAR, 512, 1u);
  for (int vt = blockIdx.x; vt < nvt; vt += gridDim.x) {
    if (pingpong) named_bar_sync(TEAM_BAR + rg, 512);
    scale = 0;
    // resident weights hold all N rows: this virtual tile multiplies rows [n_off, n_off + NT)
    const uint32_t b_lo_base = b_lo_base0 + (RESIDENT ? (uint32_t)((vt % P.nsplit) * nsub) * (Cfg::kRowBytes >> 4) : 0u);
    if (DECONV) {
      // one A stage per channel chunk; parity (py,px) reads taps (ty,tx) at (py + ty) rows, (px + tx) pixels into it
      const int par = (vt / P.nsplit) & 3;
      const uint32_t a_par = a_lo_base + (uint32_t)(par >> 1) * pitch16 + (uint32_t)(par & 1) * (Cfg::kRowBytes >> 4);
      for (int cc = 0; cc < cchunks; ++cc) {
        mbar_wait_parity(stageA(sa), pha);
        const uint32_t a_lo = a_par + (uint32_t)sa * a_stage16;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          mbar_wait_parity(fullB(sb), phb);
          wgmma_fence();
          issue(a_lo + (uint32_t)(t >> 1) * pitch16 + (uint32_t)(t & 1) * (Cfg::kRowBytes >> 4), b_lo_base + (uint32_t)sb * b_block16, 1);
          group_done(t == 3 ? emptyA(sa) : dummy_bar, emptyB(sb));
          if (++sb == SB) { sb = 0; phb ^= 1u; }
        }
        if (++sa == SA) { sa = 0; pha ^= 1u; }
      }
    } else if (S2X) {
      // two A stages per tile (even-row box, odd-row box); tap (ky,kx): row offset (ky == 2), pair-column offset
      // (kx != 0), K half (kx != 1) -> k-steps {0,1} or {2,3} of the 64-wide row, same k-steps of the weight block
#pragma unroll
      for (int v = 0; v < 2; ++v) {
        mbar_wait_parity(stageA(sa), pha);
        const uint32_t a_lo = a_lo_base + (uint32_t)sa * a_stage16;
        if (RESIDENT) wgmma_fence();
#pragma unroll
        for (int t9 = 0; t9 < 6; ++t9) {
          if (v == 0 && t9 >= 3) continue;
          const int ky = v == 0 ? 1 : (t9 < 3 ? 0 : 2), kx = t9 % 3;
          const bool last = t9 == (v == 0 ? 2 : 5);
          uint32_t b_lo;
          if (RESIDENT) b_lo = b_lo_base + (uint32_t)(ky * 3 + kx) * b_block16;
          else { mbar_wait_parity(fullB(sb), phb); wgmma_fence(); b_lo = b_lo_base + (uint32_t)sb * b_block16; }
          const uint32_t a_tap = a_lo + (uint32_t)(ky == 2 ? pitch16 : 0u) + (uint32_t)(kx != 0 ? 1 : 0) * (Cfg::kRowBytes >> 4);
          const int ks0 = kx == 1 ? 0 : 2;
#pragma unroll
          for (int ks = ks0; ks < ks0 + 2; ++ks) {
            wgmma_m64k16<NT, T>(acc, desc_lohi(a_tap + ks * 2, hi_a), desc_lohi(b_lo + ks * 2, hi_b), scale);
            scale = 1;
          }
          if (!RESIDENT || last) group_done(last ? emptyA(sa) : dummy_bar, RESIDENT ? dummy_bar : emptyB(sb));
          if (!RESIDENT && ++sb == SB) { sb = 0; phb ^= 1u; }
        }
        if (++sa == SA) { sa = 0; pha ^= 1u; }
      }
    } else if (P1) {
      // one A stage per channel chunk; tap (ky,kx) starts (ky * 24 + kx) pixels into it
      for (int cc = 0; cc < cchunks; ++cc) {
        mbar_wait_parity(stageA(sa), pha);
        const uint32_t a_lo = a_lo_base + (uint32_t)sa * a_stage16;
        if (RESIDENT) wgmma_fence();
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
#pragma unroll
          for (int i = 0; i < 3; ++i) {
            const int kx = XPAIR ? (i == 0 ? 1 : (i == 1 ? 0 : 2)) : i;
            const bool last = ky == 2 && i == 2;
            const bool close = !RESIDENT || last;
            uint32_t b_lo;
            if (RESIDENT) b_lo = b_lo_base + (uint32_t)((ky * 3 + kx) * cchunks + cc) * b_block16;
            else { mbar_wait_parity(fullB(sb), phb); wgmma_fence(); b_lo = b_lo_base + (uint32_t)sb * b_block16; }
            issue(a_lo + (uint32_t)ky * pitch16 + (uint32_t)kx * (Cfg::kRowBytes >> 4), b_lo, kx);
            if (close) group_done(last ? emptyA(sa) : dummy_bar, RESIDENT ? dummy_bar : emptyB(sb));
            if (!RESIDENT && ++sb == SB) { sb = 0; phb ^= 1u; }
          }
        }
        if (++sa == SA) { sa = 0; pha ^= 1u; }
      }
    } else if (PATCH && XPAIR) {
      // x-paired (resident weights, one 64-channel chunk: conv_tc_prepare): the three kx boxes, then the nine taps
      // ky-major with kx 1, 0, 2 -- the summation order of the single-box form -- in one group
      uint32_t a_lo[3];
#pragma unroll
      for (int i = 0; i < 3; ++i) {   // box i holds kx = patch_kx(i) = 1, 0, 2
        mbar_wait_parity(stageA(sa), pha);
        a_lo[i] = a_lo_base + (uint32_t)sa * a_stage16;
        xa_bar[i] = emptyA(sa);
        if (++sa == SA) { sa = 0; pha ^= 1u; }
      }
      wgmma_fence();
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          const int kx = i == 0 ? 1 : (i == 1 ? 0 : 2);
          issue(a_lo[i] + (uint32_t)ky * pitch16, b_lo_base + (uint32_t)(ky * 3 + kx) * b_block16, kx);
        }
      wgmma_commit();
    } else if (PATCH) {
      // one A stage per (channel chunk, kx): rows y0-1 .. y0+16, the three ky taps are 16-pixel row shifts
      for (int cc = 0; cc < cchunks; ++cc) {
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          const int kx = XPAIR ? (i == 0 ? 1 : (i == 1 ? 0 : 2)) : i;
          mbar_wait_parity(stageA(sa), pha);
          const uint32_t a_lo = a_lo_base + (uint32_t)sa * a_stage16;
          if (RESIDENT) wgmma_fence();
#pragma unroll
          for (int sub = 0; sub < 3; ++sub) {
            uint32_t b_lo;
            if (RESIDENT) b_lo = b_lo_base + (uint32_t)((sub * 3 + kx) * cchunks + cc) * b_block16;
            else { mbar_wait_parity(fullB(sb), phb); wgmma_fence(); b_lo = b_lo_base + (uint32_t)sb * b_block16; }
            issue(a_lo + (uint32_t)sub * pitch16, b_lo, kx);
            if (!RESIDENT || sub == 2) group_done(sub == 2 ? emptyA(sa) : dummy_bar, RESIDENT ? dummy_bar : emptyB(sb));
            if (!RESIDENT && ++sb == SB) { sb = 0; phb ^= 1u; }
          }
          if (++sa == SA) { sa = 0; pha ^= 1u; }
        }
      }
    } else {
      // one A stage per (tap, channel chunk)
      uint32_t b_res = b_lo_base;
      for (int tap = 0; tap < taps; ++tap) {
        for (int cc = 0; cc < cchunks; ++cc) {
          mbar_wait_parity(stageA(sa), pha);
          uint32_t b_lo;
          if (RESIDENT) { b_lo = b_res; b_res += b_block16; }
          else { mbar_wait_parity(fullB(sb), phb); b_lo = b_lo_base + (uint32_t)sb * b_block16; }
          wgmma_fence();
          issue(a_lo_base + (uint32_t)sa * a_stage16, b_lo, 1);
          group_done(emptyA(sa), RESIDENT ? dummy_bar : emptyB(sb));
          if (!RESIDENT && ++sb == SB) { sb = 0; phb ^= 1u; }
          if (++sa == SA) { sa = 0; pha ^= 1u; }
        }
      }
    }
    // every wgmma of this tile is issued: the other team may issue its tile while this one's complete
    if (PINGPONG) named_bar_arrive_if(TEAM_BAR + (rg ^ 1), 512, (pingpong && (rg == 0 || vt + (int)gridDim.x < nvt)) ? 1u : 0u);
    wgmma_wait<0>();
    release();
    if (XPAIR) {
#pragma unroll
      for (int i = 0; i < 3; ++i) mbar_arrive_if(xa_bar[i], is_lane0);
    }
    wgmma_acc_fence<NT / 2>(acc);

    // ---------------------------------------------------------------- epilogue, straight from the register fragment
    // thread: pixels (image row 2 wq + r2 of this warpgroup's 8, column lane / 4), channels 8 j + 2 (lane % 4) + {0, 1}
    // (transposed conv: oy / ox below are input-grid coordinates, stored at output pixel (2 oy + py, 2 ox + px))
    const int tile = vt / (P.nsplit * NPAR), vr = vt - tile * (P.nsplit * NPAR);
    const int par = DECONV ? vr / P.nsplit : 0;
    const int n_off = (vr - par * P.nsplit) * nsub;
    const int n = tile / P.tiles_per_img, rem = tile % P.tiles_per_img;
    const int oy0 = (rem / P.tiles_x) * TILE_Y + rg * 8 + 2 * wq, ox = (rem % P.tiles_x) * TILE_X + h * HALF_X + (lane >> 2);
    const int cq = 2 * (lane & 3);
    const int ty0 = (rem / P.tiles_x) * TILE_Y + rg * 8, tx0 = (rem % P.tiles_x) * TILE_X + h * HALF_X;   // slab origin
    if constexpr (!IsF32<T>::value) {
      if (plain) {
        // Plain layers (stores from the fragment, no residual, no cam-scale channel, no extra terms): one short
        // straight-line body per channel pair.  The general loop below carries every optional term; inlined for all
        // 32 channel pairs of a thread, it is most of the kernel's code, far more than the instruction cache holds,
        // and it ran several times slower than this loop (DESIGN.md, Conv).  The float operations are those of the
        // general loop, in the same order.  Columns [0, cols) of the virtual tile are stored: inside it (nsub) and
        // below cout_pad (npad and n_off are multiples of 16, so the bound holds for a whole group of 8 channels).
        const int cols = min(nsub, P.npad - n_off);
        const float* pbias = P.bias_per_image ? P.bias + (size_t)n * P.npad + n_off : s_bias + n_off;
#pragma unroll
        for (int g = 0; g < NT / 64; ++g) {
          if (64 * g >= cols) break;
#pragma unroll
          for (int r2 = 0; r2 < 2; ++r2) {
            const int oy = oy0 + r2;
            const size_t pix = DECONV ? ((size_t)n * P.Ho + 2 * oy + (par >> 1)) * P.Wo + 2 * ox + (par & 1)
                                      : ((size_t)n * P.Ho + oy) * P.Wo + ox;
            const size_t o = pix * P.out_stride + n_off + cq;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int j = 8 * g + jj;
              if (8 * j >= cols) break;
              const float2 b = *reinterpret_cast<const float2*>(pbias + 8 * j + cq);
              float f0 = acc[4 * j + 2 * r2] + b.x, f1 = acc[4 * j + 2 * r2 + 1] + b.y;
              if (P.relu) { f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f); }
              if (P.out_f32) *reinterpret_cast<float2*>(reinterpret_cast<float*>(P.out) + o + 8 * j) = make_float2(f0, f1);
              else *reinterpret_cast<uint32_t*>(reinterpret_cast<T*>(P.out) + o + 8 * j) = pack2<T>(f0, f1);
            }
          }
        }
        continue;
      }
    }
    // bias: per CTA from shared memory, or (folded part-head conv) one row per image from global
    const float* bsrc = P.bias_per_image ? P.bias + (size_t)n * P.npad + n_off : s_bias + n_off;
    // the channels come in groups of 64: with the TMA-store epilogue one group of the warpgroup's 64 pixels is one
    // 8 KB slab (box {64 ch, 8 px, 8 rows}, 128B swizzle) in this warpgroup's staging buffer
#pragma unroll
    for (int g = 0; g < NT / 64; ++g) {
      if (64 * g >= nsub) break;
      if (tma_out) {   // the previous slab's TMA store must have finished READING the staging buffer
        if (wg_thread == 0) bulk_wait_read0();
        named_bar_sync(1 + wg, 128);
      }
#pragma unroll
      for (int r2 = 0; r2 < 2; ++r2) {
        const int oy = oy0 + r2;
        const size_t pix = DECONV ? ((size_t)n * P.Ho + 2 * oy + (par >> 1)) * P.Wo + 2 * ox + (par & 1)
                                  : ((size_t)n * P.Ho + oy) * P.Wo + ox;
        const T* resp = P.has_res ? reinterpret_cast<const T*>(P.res) + pix * P.res_stride + n_off : nullptr;
        const uint32_t srow = stage_wg + (uint32_t)(16 * wq + (lane >> 2) + 8 * r2) * 128u;   // slab row = pixel (row-major 8 x 8)
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int j = 8 * g + jj;
          const int c = 8 * j + cq;                      // channel inside the virtual tile
          // columns past this virtual tile or past cout_pad are not computed from real weights: the direct path skips
          // them, the TMA-store path writes zeros into the slab (the TMA unit clips channels >= cout_pad)
          const bool valid = 8 * j < nsub && n_off + c < P.npad;
          if (!valid && !tma_out) continue;
          float f0 = 0.f, f1 = 0.f;
          if (valid) {
            f0 = acc[4 * j + 2 * r2] + bsrc[c]; f1 = acc[4 * j + 2 * r2 + 1] + bsrc[c + 1];
            if (P.pow11_ch0 && n_off + c == 0) f0 = powf(1.1f, f0);   // cam scale channel (acr/model.py:95-96)
            if (resp) {
              float x0, x1;
              if constexpr (IsF32<T>::value) {
                const float2 r = *reinterpret_cast<const float2*>(resp + c);
                x0 = r.x; x1 = r.y;
              } else {
                unpack2<T>(*reinterpret_cast<const uint32_t*>(resp + c), x0, x1);
              }
              f0 += x0; f1 += x1;
            }
            if constexpr (!IsF32<T>::value)   // (extra terms: 16-bit plans only)
            for (int e = 0; e < P.n_ext; ++e) {   // folded fuse sum: the other terms, nearest-upsampled (warp-uniform loop)
              const T* xp = reinterpret_cast<const T*>(P.ext[e]) +
                            (((size_t)n * P.ext_H[e] + (oy >> P.ext_shift[e])) * P.ext_W[e] + (ox >> P.ext_shift[e])) * P.ext_stride[e] + n_off + c;
              float x0, x1;
              unpack2<T>(*reinterpret_cast<const uint32_t*>(xp), x0, x1);
              f0 += x0; f1 += x1;
            }
            if (P.relu) { f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f); }
          }
          if constexpr (IsF32<T>::value) {
            *reinterpret_cast<float2*>(reinterpret_cast<float*>(P.out) + pix * P.out_stride + n_off + c) = make_float2(f0, f1);
          } else if (tma_out) {   // 16-byte chunk jj of the 128-byte row lives at chunk jj ^ (row & 7) (row & 7 = lane / 4)
            sts32(srow + (((uint32_t)jj ^ (uint32_t)(lane >> 2)) << 4) + (uint32_t)cq * 2u, pack2<T>(f0, f1));
          } else if (P.out_f32) {
            *reinterpret_cast<float2*>(reinterpret_cast<float*>(P.out) + pix * P.out_stride + n_off + c) = make_float2(f0, f1);
          } else {
            *reinterpret_cast<uint32_t*>(reinterpret_cast<T*>(P.out) + pix * P.out_stride + n_off + c) = pack2<T>(f0, f1);
          }
        }
      }
      if (tma_out) {   // slab complete in shared memory: one thread hands it to the TMA unit
        fence_proxy_async();
        named_bar_sync(1 + wg, 128);
        if (wg_thread == 0) {
          tma_store_4d(&P.tmOut, stage_wg, n_off + 64 * g, tx0, ty0, n);
          bulk_commit();
        }
      }
    }
  }
  if (tma_out && wg_thread == 0) bulk_wait_all();   // the staging buffer must outlive the stores
}

// --------------------------------------------------------------------------------- host side
struct ConvTcPlan {
  ConvTcParams p;
  int ck, act_dtype, grid, nt;
  size_t smem;
};

// One launch of a conv-family kernel (conv_tc_kernel, conv_block_kernel, conv_bottleneck_kernel) with programmatic
// dependent launch: it may start while the previous kernel on the stream drains (see pdl_wait).
template <typename Kernel, typename Params>
static int launch_pdl(Kernel kernel, const Params& p, int grid, size_t smem, cudaStream_t st) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(TC_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  ACR_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kernel, p));
  return ACR_B200_OK;
}

template <int CK, typename T, int MODE, int NT>
static int launch_nt(const ConvTcPlan* pl, cudaStream_t st) {
  static unsigned long long configured = 0;
  ACR_CHECK_CUDA(ensure_dynamic_smem(conv_tc_kernel<CK, T, MODE, NT>, SMEM_BUDGET, &configured));
  return launch_pdl(conv_tc_kernel<CK, T, MODE, NT>, pl->p, pl->grid, pl->smem, st);
}

template <int CK, typename T, int MODE>
static int launch_inst(const ConvTcPlan* pl, cudaStream_t st) {
  if constexpr ((MODE & MODE_XPAIR) != 0) return launch_nt<CK, T, MODE, 64>(pl, st);
  else return pl->nt == 64 ? launch_nt<CK, T, MODE, 64>(pl, st) : launch_nt<CK, T, MODE, 128>(pl, st);
}

template <int CK, typename T>
static int launch_mode(const ConvTcPlan* pl, cudaStream_t st) {
  const int mode = (pl->p.patch_mode ? MODE_PATCH : 0) | (pl->p.b_resident ? MODE_RESIDENT : 0);
  if constexpr (IsF32<T>::value) {   // tf32: the single-box form and the four generic modes
    if (pl->p.deconv || pl->p.s2x || pl->p.xpair) { set_error("conv_tc: no tf32 form of the transposed or x-paired convs"); return ACR_B200_EINVAL; }
    if constexpr (CK == 64)
      if (pl->p.patch1)
        return pl->p.b_resident ? launch_inst<64, T, MODE_PATCH | MODE_RESIDENT | MODE_P1>(pl, st)
                                : launch_inst<64, T, MODE_PATCH | MODE_P1>(pl, st);
  } else if constexpr (CK == 64) {
    if (pl->p.deconv) return launch_inst<64, T, MODE_DECONV>(pl, st);
    if (pl->p.s2x)
      return pl->p.b_resident ? launch_inst<64, T, MODE_RESIDENT | MODE_S2X>(pl, st) : launch_inst<64, T, MODE_S2X>(pl, st);
    if (pl->p.patch1)
      return pl->p.b_resident ? launch_inst<64, T, MODE_PATCH | MODE_RESIDENT | MODE_P1>(pl, st)
                              : launch_inst<64, T, MODE_PATCH | MODE_P1>(pl, st);
    if (pl->p.xpair) {
      if (mode != (MODE_PATCH | MODE_RESIDENT)) { set_error("conv_tc: x-paired conv needs resident weights"); return ACR_B200_EINVAL; }
      return launch_inst<64, T, MODE_PATCH | MODE_RESIDENT | MODE_XPAIR>(pl, st);
    }
  }
  if constexpr (CK == 64) {   // every 64-channel-chunk 3x3 stride-1 conv is one of the single-box or x-paired forms above
    if (pl->p.patch_mode) { set_error("conv_tc: no three-box form of a 64-channel-chunk conv"); return ACR_B200_EINVAL; }
    return pl->p.b_resident ? launch_inst<64, T, MODE_RESIDENT>(pl, st) : launch_inst<64, T, 0>(pl, st);
  } else {
    switch (mode) {
      case 0: return launch_inst<CK, T, 0>(pl, st);
      case 1: return launch_inst<CK, T, 1>(pl, st);
      case 2: return launch_inst<CK, T, 2>(pl, st);
      default: return launch_inst<CK, T, 3>(pl, st);
    }
  }
}

// the kernel instances of one (CK, activation type), each in its own translation unit (conv_tc_inst_*.cu)
int conv_tc_launch_64_bf16(const ConvTcPlan* pl, cudaStream_t st);
int conv_tc_launch_64_f16(const ConvTcPlan* pl, cudaStream_t st);
int conv_tc_launch_32(const ConvTcPlan* pl, cudaStream_t st);
int conv_tc_launch_16(const ConvTcPlan* pl, cudaStream_t st);
int conv_tc_launch_tf32(const ConvTcPlan* pl, cudaStream_t st);   // T = float, CK = 64 and 32

}  // namespace acr
