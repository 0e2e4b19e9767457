// Stem conv on the Hopper tensor cores WITHOUT the im2col round trip (sm_90a).
//
// HigherResolutionNet.forward (acr/model.py of the reference): x/255*2-1, conv1 3x3 stride 2 (3 -> 64) + bn1 + ReLU.
// As im2col_stem_kernel (uint8 frame -> 32-channel 16-bit tensor of the 27 normalised taps, 1.07 GB at batch 256) + a
// 1x1 conv it would write and read that tensor back.  Here the A operand of that GEMM is built IN SHARED MEMORY by
// producer warps straight from the uint8 frame, in the K-major SWIZZLE_64B layout a TMA box {32, 16, 16} would have
// produced (row = output pixel, 32 channels = 27 taps + 5 zeros = 64 bytes; 16-byte chunk c of row r lives at chunk
// c ^ ((r >> 1) & 3): the swizzle is a function of the absolute shared-memory address), so the intermediate tensor never
// exists: 0.2 GB in + 2.15 GB out instead of 0.2 + 1.07 + 1.07 + 2.15 GB.
//
// Persistent CTAs, one per SM, tile = 16x16 output pixels:
//   warps 0..7   two consumer warpgroups; warpgroup g takes image rows 8g .. 8g+7 of the tile as two M = 64 blocks:
//                2 k-steps of wgmma m64n64k16 each into 32 fp32 registers per thread, then ReLU -> 16-bit pairs -> NHWC
//   warps 8..23  producers, two groups of 8 warps taking alternate tiles (a group converts one tile at a time, so one group
//                alone leaves the load latency exposed): thread = output pixel; its 27 uint8 taps straight from the frame
//                (L1 shares them between neighbours; the next tile's patch is prefetched), (float)v / 255.f * 2.f - 1.f
//                in three FMA-pipe operations (bit-identical to the reference's normalisation), round to the storage
//                type, write the swizzled 64-byte row; generic -> async proxy fence, one mbarrier arrive per warp.
// The BN bias rides in two spare K channels (hi + lo 16-bit parts against constant-one taps).
//
// KS = 7 is the ResNet stem (conv1 7x7 stride 2 padding 3, 3 -> 64): K = 147 taps + the bias pair + 11 zeros = 160, five
// 32-channel SWIZZLE_64B slabs per operand (A: 5 x 16 KB per stage, two stages; weights: 5 x 4 KB), 10 k-steps per M = 64
// block.  Its producers gather the 147 bytes of their pixel's 7x7x3 window with bounds checks (zeros in the padding).
#include <cuda.h>

#include "ops.cuh"
#include "wgmma.cuh"

namespace acr {
namespace {

__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mb_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count)); }
__device__ __forceinline__ void mb_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
// ReLU, then two fp32 -> packed 16-bit pair (round to nearest even)
template <typename T>
__device__ __forceinline__ uint32_t pack2_relu(float a, float b) {
  uint32_t u;
  T* p = reinterpret_cast<T*>(&u);
  p[0] = from_f32<T>(fmaxf(a, 0.f));
  p[1] = from_f32<T>(fmaxf(b, 0.f));
  return u;
}
// (float)b / 255.f * 2.f - 1.f for a byte b, bit for bit (the reference's normalisation, acr/model.py:832), without a division
// or a table: b as a float through the 2^23 trick, the correctly rounded quotient as fma(x, rh, x * rl) with rh + rl = 1/255
// to 48 bits (exact for all 256 inputs: tests/test_cpu_round2.py), then 2q - 1 in one rounding (2q is exact).
__device__ __forceinline__ float normalised(uint32_t b) {
  const float x = __uint_as_float(0x4B000000u | b) - 8388608.f;
  const float q = __fmaf_rn(x, __uint_as_float(0x3B808081u), __fmul_rn(x, __uint_as_float(0xAF7EFEFFu)));
  return __fmaf_rn(q, 2.f, -1.f);
}
constexpr int CONS_WARPS = 8, PROD_WARPS = 16;   // two consumer warpgroups; two producer groups of 8 warps take alternate tiles
constexpr int THREADS = 32 * (CONS_WARPS + PROD_WARPS);
template <int KS>
struct StemCfg {
  static constexpr int BIAS_CH = KS * KS * 3;              // channels: (ky*KS+kx)*3+ci, then the bias pair (hi, lo)
  static constexpr int KCH = (BIAS_CH + 2 + 31) / 32 * 32; // K: 32 (3x3) or 160 (7x7)
  static constexpr int NSLAB = KCH / 32;                   // 64-byte-row SWIZZLE_64B slabs of K
  static constexpr int NS = KS == 3 ? 4 : 2;               // operand stages
  static constexpr int SLAB_A = 256 * 64;                  // one slab of one A stage: 256 pixel rows x 64 B
  static constexpr int A_BYTES = NSLAB * SLAB_A;
  static constexpr int SLAB_W = 64 * 64;                   // one slab of the weights: 64 output channels x 64 B
  static constexpr int SMEM = 1024 + NS * A_BYTES + NSLAB * SLAB_W + 256 /*barriers*/;
  static_assert(BIAS_CH % 8 < 7, "the bias pair shares one 16-byte chunk");
};

struct StemTcParams {
  const uint8_t* img;     // (B, H, W, 3) uint8
  void* out;              // (B, H/2, W/2, out_stride) 16-bit
  const void* w;          // packed [64][KCH] 16-bit, K-major (channel (ky*KS+kx)*3+ci, then zeros), BN folded
  const float* bias;      // [64]
  int H, W, out_stride, total_tiles;
  int tx_log2, tpi_log2;  // tiles per output row / per image are powers of two (512 x 512 frames: 16, 256): shifts, no divisions in the tile loops
};

template <typename T, int KS>
__global__ void __launch_bounds__(THREADS, 1) stem_tc_kernel(const __grid_constant__ StemTcParams P) {
  using Cfg = StemCfg<KS>;
  constexpr int NS = Cfg::NS, A_BYTES = Cfg::A_BYTES, NSLAB = Cfg::NSLAB;
  extern __shared__ uint8_t raw_smem[];
  const uint32_t raw = s32(raw_smem);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gen = raw_smem + (base - raw);                 // generic pointer to the aligned base
  const uint32_t a_base = base;
  const uint32_t w_base = base + NS * A_BYTES;
  const uint32_t bar_base = w_base + NSLAB * Cfg::SLAB_W;
  auto fullA = [&](int s) { return bar_base + 8u * s; };
  auto emptyA = [&](int s) { return bar_base + 8u * (NS + s); };
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < NS; ++s) { mb_init(fullA(s), 8); mb_init(emptyA(s), CONS_WARPS); }   // one arrival per producer warp of a group / consumer warp
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // weights [64 rows][KCH] into NSLAB SWIZZLE_64B slabs of [64 rows][64 B]: 256 16-byte chunks per slab
  for (int i = threadIdx.x; i < 256 * NSLAB; i += THREADS) {
    const int r = i / (4 * NSLAB), q = i % (4 * NSLAB), slab = q >> 2, c = q & 3;
    uint4 v = reinterpret_cast<const uint4*>(P.w)[i];
    if (q == Cfg::BIAS_CH / 8) {   // the bias rides in two spare K channels (the producers write 1.0 there): hi + lo parts,
                                   // so the fp32 accumulator receives it to 2^-17 (bf16) / 2^-22 (fp16) relative and the
                                   // epilogue needs no add
      T* e = reinterpret_cast<T*>(&v);
      const float b = P.bias[r];
      e[Cfg::BIAS_CH % 8] = from_f32<T>(b);
      e[Cfg::BIAS_CH % 8 + 1] = from_f32<T>(b - to_f32<T>(e[Cfg::BIAS_CH % 8]));
    }
    *reinterpret_cast<uint4*>(gen + NS * A_BYTES + slab * Cfg::SLAB_W + r * 64 + ((c ^ ((r >> 1) & 3)) << 4)) = v;
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // the weights were written through the generic proxy
  __syncthreads();

  if (warp < CONS_WARPS) {
    // ================================================================== consumers: wgmma + epilogue
    // warpgroup g takes pixel rows 128 g .. 128 g + 127 of the tile (image rows 8 g .. 8 g + 7), as two M = 64 blocks
    const int g = warp >> 2, wq = warp & 3;
    int it = 0, s = 0;
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < P.total_tiles; tile += gridDim.x, ++it) {
      const int n = tile >> P.tpi_log2, rem = tile & ((1 << P.tpi_log2) - 1);
      const int y0 = (rem >> P.tx_log2) * 16, x0 = (rem & ((1 << P.tx_log2) - 1)) * 16;
      mbar_wait_parity(fullA(s), ph);
      const uint32_t a0 = a_base + (uint32_t)s * A_BYTES;
#pragma unroll
      for (int blk = 0; blk < 2; ++blk) {
        const int row0 = 128 * g + 64 * blk;    // first pixel row of this M = 64 block (4 image rows x 16 pixels)
        float acc[32];
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 2 * NSLAB; ++ks)  // K = 32 per slab (3x3: 27 taps, the bias pair, 3 zeros); 8-row core-matrix groups 512 B apart
          wgmma_m64n64k16<T>(acc, gmma_desc(a0 + (uint32_t)(ks >> 1) * Cfg::SLAB_A + (uint32_t)row0 * 64u + (ks & 1) * 32, 16, 512, gmma_swizzle(64)),
                             gmma_desc(w_base + (uint32_t)(ks >> 1) * Cfg::SLAB_W + (ks & 1) * 32, 16, 512, gmma_swizzle(64)), ks ? 1u : 0u);   // ks 0 overwrites
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_acc_fence<32>(acc);
        if (blk == 1) {   // both blocks have read the stage
          __syncwarp();
          mbar_arrive_if(emptyA(s), lane == 0 ? 1u : 0u);
        }
        // thread: pixel rows row0 + 16 wq + lane / 4 (+ 8), channels 8 j + 2 (lane % 4) + {0, 1}; the accumulator already
        // holds conv + bias: ReLU, round, store
#pragma unroll
        for (int r2 = 0; r2 < 2; ++r2) {
          const int r = row0 + 16 * wq + (lane >> 2) + 8 * r2;
          const size_t pix = ((size_t)n * (P.H >> 1) + y0 + (r >> 4)) * (size_t)(P.W >> 1) + x0 + (r & 15);
          uint32_t* o = reinterpret_cast<uint32_t*>(static_cast<T*>(P.out) + pix * P.out_stride + 2 * (lane & 3));
#pragma unroll
          for (int j = 0; j < 8; ++j) o[4 * j] = pack2_relu<T>(acc[4 * j + 2 * r2], acc[4 * j + 2 * r2 + 1]);
        }
      }
      if (++s == NS) { s = 0; ph ^= 1u; }
    }
  } else {
    // ===================================================================================== producers
    const int pt = threadIdx.x - 32 * CONS_WARPS;    // 0..511
    const int grp = pt >> 8, t = pt & 255;          // group 0 / 1 builds the even / odd tiles of this CTA; t = output pixel
    const int py = t >> 4, px = t & 15;
    int s = grp;                                    // stage of tile number it = it % NS; this group's tiles: it = grp, grp + 2, ..
    uint32_t ph = 0;
    const int r = py * 16 + px;
    const int sw = (r >> 1) & 3;
    const int tmask = (1 << P.tpi_log2) - 1, xmask = (1 << P.tx_log2) - 1;
    const size_t img_bytes = (size_t)P.H * P.W * 3;
    // Only the top and the left frame edges pad (the patch of tile (y0, x0) starts at input pixel (2*y0 - 1, 2*x0 - 1) and ends
    // inside the frame): filter row 0 of pixel row 0 of the tiles with y0 == 0, filter column 0 of pixel column 0 where x0 == 0.
    for (int tile = blockIdx.x + grp * (int)gridDim.x; tile < P.total_tiles; tile += 2 * (int)gridDim.x) {
      const int n = tile >> P.tpi_log2, rem = tile & tmask;
      const int y0 = (rem >> P.tx_log2) * 16, x0 = (rem & xmask) * 16;
      if constexpr (KS == 3) {
        const bool pad_top = (y0 | py) == 0, pad_left = (x0 | px) == 0;
        const int iy = 2 * (y0 + py) - (pad_top ? 0 : 1), ix = 2 * (x0 + px) - (pad_left ? 0 : 1);   // first tap that exists
        const uint8_t* p0 = P.img + (size_t)n * img_bytes + ((size_t)iy * P.W + ix) * 3;
        {  // pull the NEXT tile's 33 x 99-byte patch towards L1 while this one is converted
          const int nt = tile + 2 * (int)gridDim.x;
          if (nt < P.total_tiles && t < 66) {
            const int nrem = nt & tmask;
            int piy = 2 * (nrem >> P.tx_log2) * 16 - 1 + (t >> 1), pix = 2 * (nrem & xmask) * 16 - 1;
            piy = piy < 0 ? 0 : piy; pix = pix < 0 ? 0 : pix;
            asm volatile("prefetch.global.L1 [%0];" ::"l"(P.img + (size_t)(nt >> P.tpi_log2) * img_bytes + ((size_t)piy * P.W + pix) * 3 + (t & 1) * 96));
          }
        }
        mbar_wait_parity(emptyA(s), ph ^ 1u);                                         // the MMAs that read this stage are done
        // ---- this thread's pixel: 3 filter rows x 9 contiguous bytes straight from the frame (neighbouring pixels share them
        // through L1); a padded row / column reads the next one instead (always inside the frame) and is zeroed afterwards
        uint32_t raw9[3][9];
        if (x0 != 0) {        // (uniform) no left padding: the row starts at an odd address -> one byte + four aligned 16-bit loads
  #pragma unroll
          for (int ky = 0; ky < 3; ++ky) {
            const uint8_t* prow = p0 + (size_t)(pad_top ? (ky ? ky - 1 : 0) : ky) * P.W * 3;
            raw9[ky][0] = (uint32_t)__ldg(prow);
  #pragma unroll
            for (int j = 0; j < 4; ++j) {
              const uint32_t w = (uint32_t)__ldg(reinterpret_cast<const unsigned short*>(prow + 1 + 2 * j));
              raw9[ky][1 + 2 * j] = w & 0xffu;
              raw9[ky][2 + 2 * j] = w >> 8;
            }
          }
        } else {
  #pragma unroll
          for (int ky = 0; ky < 3; ++ky) {
            const uint8_t* prow = p0 + (size_t)(pad_top ? (ky ? ky - 1 : 0) : ky) * P.W * 3 - (pad_left ? 3 : 0);
            const uint8_t* pcol0 = prow + (pad_left ? 3 : 0);                 // filter column 0 (or its stand-in)
  #pragma unroll
            for (int j = 0; j < 9; ++j) raw9[ky][j] = (uint32_t)__ldg((j < 3 ? pcol0 : prow) + j);
          }
        }
        float vch[32];
  #pragma unroll
        for (int i = 27; i < 32; ++i) vch[i] = i < 29 ? 1.f : 0.f;           // channels 27 / 28 carry the bias (hi / lo)
  #pragma unroll
        for (int ky = 0; ky < 3; ++ky)
  #pragma unroll
          for (int j = 0; j < 9; ++j) {
            const float v = normalised(raw9[ky][j]);
            vch[ky * 9 + j] = (ky == 0 && j < 3) ? ((pad_top || pad_left) ? 0.f : v) : ky == 0 ? (pad_top ? 0.f : v) : j < 3 ? (pad_left ? 0.f : v) : v;
          }
        uint8_t* arow = gen + s * A_BYTES + r * 64;
  #pragma unroll
        for (int c = 0; c < 4; ++c) *reinterpret_cast<uint4*>(arow + ((c ^ sw) << 4)) = pack8<T>(vch + c * 8);
      } else {
        // 7x7 stride 2 padding 3: input rows 2(y0+py)-3 .. +3, columns 2(x0+px)-3 .. +3, zero outside the frame; channel
        // c = (ky*7+kx)*3+ci, one slab of 32 channels at a time
        const int iy0 = 2 * (y0 + py) - 3, ix0 = 2 * (x0 + px) - 3;
        const uint8_t* pimg = P.img + (size_t)n * img_bytes;
        mbar_wait_parity(emptyA(s), ph ^ 1u);                                       // the MMAs that read this stage are done
        uint8_t* arow = gen + s * A_BYTES + r * 64;
#pragma unroll 1
        for (int slab = 0; slab < NSLAB; ++slab) {   // (not unrolled: five unrolled slabs of address arithmetic would spill)
          float vch[32];
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const int c = slab * 32 + i;
            float v = 0.f;
            if (c < Cfg::BIAS_CH) {
              const int ky = c / (3 * KS), kx = (c % (3 * KS)) / 3, ci = c % 3;
              const int iy = iy0 + ky, ix = ix0 + kx;
              if ((unsigned)iy < (unsigned)P.H && (unsigned)ix < (unsigned)P.W)
                v = normalised((uint32_t)__ldg(pimg + ((size_t)iy * P.W + ix) * 3 + ci));
            } else if (c < Cfg::BIAS_CH + 2) {
              v = 1.f;                                                              // the bias pair (hi / lo)
            }
            vch[i] = v;
          }
#pragma unroll
          for (int c = 0; c < 4; ++c) *reinterpret_cast<uint4*>(arow + slab * Cfg::SLAB_A + ((c ^ sw) << 4)) = pack8<T>(vch + c * 8);
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");         // generic-proxy writes -> visible to the tensor core
      __syncwarp();
      if (lane == 0) mb_arrive(fullA(s));                                  // 8 arrivals (this group's warps) complete the stage
      s += 2;
      if (s >= NS) { s -= NS; ph ^= 1u; }
    }
  }
}

}  // namespace

template <typename T, int KS>
static int launch_ks(const StemTcParams& p, int grid, cudaStream_t st) {
  static unsigned long long done = 0;
  ACR_CHECK_CUDA(ensure_dynamic_smem(stem_tc_kernel<T, KS>, StemCfg<KS>::SMEM, &done));
  stem_tc_kernel<T, KS><<<grid, THREADS, StemCfg<KS>::SMEM, st>>>(p);
  return ACR_B200_OK;
}

int launch_stem_tc(const TensorRef& img, const TensorRef& out, const void* w, const float* bias, int batch, int act_dtype,
                   int ks, cudaStream_t st) {
  ACR_CHECK_ARG(ks == 3 || ks == 7, "stem_tc: kernel size %d (3 or 7)", ks);
  ACR_CHECK_ARG(out.C == 64 && out.H * 2 == img.H && out.W * 2 == img.W && img.dtype == ACR_DT_U8 && out.H % 16 == 0 &&
                    out.W % 16 == 0 && out.pix_stride % 16 == 0 && (uintptr_t)out.ptr % 32 == 0 && (uintptr_t)w % 16 == 0 &&
                    out.dtype == act_dtype && (uintptr_t)img.ptr % 2 == 0, "stem_tc: shape / alignment");
  StemTcParams p;
  p.img = static_cast<const uint8_t*>(img.ptr); p.out = out.ptr; p.w = w; p.bias = bias;
  p.H = img.H; p.W = img.W; p.out_stride = out.pix_stride;
  const int tiles_x = out.W / 16, tiles_per_img = tiles_x * (out.H / 16);
  ACR_CHECK_ARG((tiles_x & (tiles_x - 1)) == 0 && (tiles_per_img & (tiles_per_img - 1)) == 0, "stem_tc: tiles per row / image must be powers of two");
  p.tx_log2 = __builtin_ctz(tiles_x); p.tpi_log2 = __builtin_ctz(tiles_per_img); p.total_tiles = tiles_per_img * batch;
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) sms = 132;
  const int grid = p.total_tiles < sms ? p.total_tiles : sms;
  int rc;
  if (act_dtype == ACR_DT_BF16) {
    rc = ks == 7 ? launch_ks<__nv_bfloat16, 7>(p, grid, st) : launch_ks<__nv_bfloat16, 3>(p, grid, st);
  } else if (act_dtype == ACR_DT_F16) {
    rc = ks == 7 ? launch_ks<__half, 7>(p, grid, st) : launch_ks<__half, 3>(p, grid, st);
  } else {
    set_error("stem_tc: activation dtype %d", act_dtype);
    return ACR_B200_EINVAL;
  }
  if (rc) return rc;
  ACR_CHECK_LAUNCH();
  return ACR_B200_OK;
}

}  // namespace acr
