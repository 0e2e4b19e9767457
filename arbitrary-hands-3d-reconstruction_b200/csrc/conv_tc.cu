// Host side of the implicit-GEMM conv (conv_tc.cuh): tensor maps, N split, shared-memory plan, launch dispatch; and of
// the fused BasicBlock (conv_block.cuh) and Bottleneck (conv_bottleneck.cuh).
#include "conv_block.cuh"
#include "conv_bottleneck.cuh"

namespace acr {

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

static int num_sms() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

static int encode(CUtensorMap* m, int act_dtype, int rank, const void* ptr, const cuuint64_t* dims,
                  const cuuint64_t* strides, const cuuint32_t* box, int ck) {
  PFN_encodeTiled fn = get_encode();
  if (!fn) { set_error("conv_tc: cuTensorMapEncodeTiled unavailable (no CUDA driver?)"); return ACR_B200_ECUDA; }
  cuuint32_t es[5] = {1, 1, 1, 1, 1};
  const CUtensorMapSwizzle sw = ck == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (ck == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
  // (TF32 plan: fp32 tensors are described as 16-bit words, two per channel; see conv_tc_prepare)
  const CUtensorMapDataType dt = act_dtype == ACR_DT_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                 : (act_dtype == ACR_DT_TF32 ? CU_TENSOR_MAP_DATA_TYPE_UINT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
  CUresult r = fn(m, dt, (cuuint32_t)rank, const_cast<void*>(ptr), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("conv_tc: cuTensorMapEncodeTiled failed (%d)", (int)r); return ACR_B200_ECUDA; }
  return ACR_B200_OK;
}

// The TMA-store epilogue is opt-in (ACR_B200_TMA_OUT=1, read at plan creation): every consumer warpgroup stages each
// 64-channel group of its 64 pixels as one swizzled 8 KB slab and hands it to the TMA unit instead of storing channel
// pairs from the register fragment.  It needs 32 KB of shared memory next to the operand stages.
static bool tma_out_enabled() {
  const char* e = getenv("ACR_B200_TMA_OUT");
  return e && atoi(e) != 0;
}

int conv_tc_prepare(const ConvArgs& a, int act_dtype, ConvTcPlan** out) {
  ACR_CHECK_ARG(a.out.H % TILE_Y == 0 && a.out.W % TILE_X == 0, "conv_tc: output %dx%d is not a multiple of the 16x16 super-tile", a.out.H, a.out.W);
  ACR_CHECK_ARG(a.in.pix_stride % 8 == 0 && a.cin_pad % 16 == 0 && a.cout_pad % 16 == 0 && a.cout_pad <= 2048 && a.cin_pad <= 2048,
                "conv_tc: channel alignment");
  // TF32 plan (act_dtype ACR_DT_TF32): fp32 tensors and weights, described to the TMA unit as 16-bit words, two per
  // channel -- byte-identical, for boxes, swizzle and descriptors, to a 16-bit tensor of twice the channels.  So every
  // channel count, chunk (ck) and stride below is in 16-bit units: ck = 64 / 32 holds 32 / 16 fp32 channels.
  const bool tf32 = act_dtype == ACR_DT_TF32;
  const int ew = tf32 ? 2 : 1;   // 16-bit words per element
  ACR_CHECK_ARG(a.in.dtype == (tf32 ? ACR_DT_F32 : act_dtype), "conv_tc: input dtype mismatch");
  ACR_CHECK_ARG(!tf32 || (a.out.dtype == ACR_DT_F32 && (!a.has_res || a.res.dtype == ACR_DT_F32) && !a.xpair && !a.s2x &&
                          !a.deconv && a.n_ext == 0),
                "conv_tc: the tf32 conv reads and writes fp32 tensors and has no x-paired, transposed or extra-term form");
  const int cin_pad = a.cin_pad * ew, in_stride = a.in.pix_stride * ew;
  ACR_CHECK_ARG(!a.deconv || (a.k == 4 && a.stride == 2 && a.cin_pad % 64 == 0 && !a.has_res && a.n_ext == 0 && !a.xpair &&
                              !a.s2x && !a.bias_per_image && !a.pow11_ch0 && a.out.H == 2 * a.in.H && a.out.W == 2 * a.in.W &&
                              a.in.H % TILE_Y == 0 && a.in.W % TILE_X == 0),
                "conv_tc: the transposed conv is k4 s2 p1 over whole 16x16 input tiles, 64-channel K chunks, no residual");
  ACR_CHECK_ARG(a.deconv || a.k == 1 || a.k == 3, "conv_tc: kernel size %d", a.k);
  ACR_CHECK_ARG(!a.xpair || (a.k == 3 && a.stride == 1 && a.cin_pad == 64 && a.cout_pad == 64 && a.in.pix_stride >= 64),
                "conv_tc: the x-paired form is a 3x3 stride-1 64->64 conv");
  ACR_CHECK_ARG(!a.s2x || (a.k == 3 && a.stride == 2 && a.cin_pad == 64 && a.in.pix_stride == 64 && a.in.C == 64 && !a.xpair &&
                           a.in.H == 2 * a.out.H && a.in.W == a.out.W),
                "conv_tc: the x-paired stride-2 form reads a dense 32-channel tensor as (H, W/2, 64)");
  ACR_CHECK_ARG(a.out.pix_stride % 2 == 0 && (!a.has_res || a.res.pix_stride % 2 == 0), "conv_tc: output / residual rows must hold channel pairs");
  const int ck = (cin_pad % 64 == 0) ? 64 : ((cin_pad % 32 == 0) ? 32 : 16);
  ConvTcPlan* pl = new ConvTcPlan();
  ConvTcParams& p = pl->p;
  pl->ck = ck; pl->act_dtype = act_dtype;
  p.patch_mode = (a.k == 3 && a.stride == 1) ? 1 : 0;
  // x-paired convs keep the three-box form: their single-box instance mixes full-width and corner MMAs on accumulator
  // subsets within a tap row, which ptxas serialises for lack of registers
  p.patch1 = (p.patch_mode && ck == 64 && !a.xpair) ? 1 : 0;
  p.s2x = a.s2x ? 1 : 0;
  p.deconv = a.deconv ? 1 : 0;
  const cuuint32_t box_rows = p.s2x ? TILE_Y + 1 : ((p.patch_mode || p.deconv) ? TILE_Y + 2 : TILE_Y);
  const cuuint32_t box_cols = (p.patch1 || p.s2x || p.deconv) ? P1_PITCH : TILE_X;
  const cuuint64_t esz = 2;
  const cuuint64_t dim0 = (cuuint64_t)(cin_pad < in_stride ? cin_pad : in_stride);
  int rc = ACR_B200_OK;
  if (a.s2x) {   // two row-parity views of the x-paired input (H, W/2, 64): rows 2r + py
    for (int v = 0; v < 2 && !rc; ++v) {
      const char* ptr = static_cast<const char*>(a.in.ptr) + (size_t)v * a.in.W * in_stride * esz;
      cuuint64_t dims[4] = {dim0, (cuuint64_t)a.in.W, (cuuint64_t)a.in.H / 2, (cuuint64_t)a.batch};
      cuuint64_t str[3] = {(cuuint64_t)in_stride * esz, (cuuint64_t)2 * a.in.W * in_stride * esz,
                           (cuuint64_t)a.in.H * a.in.W * in_stride * esz};
      cuuint32_t box[4] = {(cuuint32_t)ck, box_cols, box_rows, 1};
      rc = encode(&p.tmA[v], act_dtype, 4, ptr, dims, str, box, ck);
    }
    for (int v = 2; v < 4 && !rc; ++v) p.tmA[v] = p.tmA[0];
  } else if (a.stride == 1 || a.deconv) {   // (the transposed conv reads its input at stride 1)
    cuuint64_t dims[4] = {dim0, (cuuint64_t)a.in.W, (cuuint64_t)a.in.H, (cuuint64_t)a.batch};
    cuuint64_t str[3] = {(cuuint64_t)in_stride * esz, (cuuint64_t)a.in.W * in_stride * esz,
                         (cuuint64_t)a.in.H * a.in.W * in_stride * esz};
    cuuint32_t box[4] = {(cuuint32_t)ck, box_cols, box_rows, 1};
    rc = encode(&p.tmA[0], act_dtype, 4, a.in.ptr, dims, str, box, ck);
    for (int v = 1; v < 4 && !rc; ++v) p.tmA[v] = p.tmA[0];
  } else {
    // four parity views (even / odd rows x columns); a 1x1 stride-2 conv (padding 0) reads view 0 at offset 0 only
    for (int v = 0; v < 4 && !rc; ++v) {
      const int py = v >> 1, px = v & 1;
      const char* ptr = static_cast<const char*>(a.in.ptr) + ((size_t)py * a.in.W + px) * in_stride * esz;
      cuuint64_t dims[4] = {dim0, (cuuint64_t)a.in.W / 2, (cuuint64_t)a.in.H / 2, (cuuint64_t)a.batch};
      cuuint64_t str[3] = {(cuuint64_t)2 * in_stride * esz, (cuuint64_t)2 * a.in.W * in_stride * esz,
                           (cuuint64_t)a.in.H * a.in.W * in_stride * esz};
      cuuint32_t box[4] = {(cuuint32_t)ck, TILE_X, box_rows, 1};
      rc = encode(&p.tmA[v], act_dtype, 4, ptr, dims, str, box, ck);
    }
  }
  if (rc) { delete pl; return rc; }
  // N split (see ConvTcParams::nsplit): the register accumulator of a warpgroup holds at most 128 columns; wider layers
  // are cut into nsplit balanced virtual tiles
  const int nsplit = (a.cout_pad + MAX_NSUB - 1) / MAX_NSUB;
  const int nsub = ((a.cout_pad + nsplit - 1) / nsplit + 15) / 16 * 16;
  p.n_ext = a.n_ext;
  for (int e = 0; e < a.n_ext; ++e) {
    ACR_CHECK_ARG((uintptr_t)a.ext[e].ptr % 4 == 0 && a.ext[e].pix_stride % 2 == 0 && a.out.dtype != ACR_DT_F32,
                  "conv_tc: extra term %d must be a 16-bit tensor with channel-pair aligned rows", e);
    p.ext[e] = a.ext[e].ptr; p.ext_shift[e] = a.ext_shift[e]; p.ext_stride[e] = a.ext[e].pix_stride;
    p.ext_W[e] = a.ext[e].W; p.ext_H[e] = a.ext[e].H;
  }
  p.tma_out = (tma_out_enabled() && !a.deconv && a.out.dtype != ACR_DT_F32 && nsub % 64 == 0 && (uintptr_t)a.out.ptr % 16 == 0 &&
               a.out.pix_stride % 8 == 0) ? 1 : 0;
  if (p.tma_out) {
    cuuint64_t dims[4] = {(cuuint64_t)a.cout_pad, (cuuint64_t)a.out.W, (cuuint64_t)a.out.H, (cuuint64_t)a.batch};
    cuuint64_t str[3] = {(cuuint64_t)a.out.pix_stride * esz, (cuuint64_t)a.out.W * a.out.pix_stride * esz,
                         (cuuint64_t)a.out.H * a.out.W * a.out.pix_stride * esz};
    cuuint32_t box[4] = {64, HALF_X, 8, 1};
    rc = encode(&p.tmOut, act_dtype, 4, a.out.ptr, dims, str, box, 64);
    if (rc) { delete pl; return rc; }
  }
  p.stage_out_bytes = p.tma_out ? 4u * 8192u : 0u;
  p.bias = a.bias; p.res = a.has_res ? a.res.ptr : nullptr; p.out = a.out.ptr;
  p.taps = a.deconv ? 4 : a.k * a.k; p.ksz = a.k; p.stride = a.stride; p.cchunks = cin_pad / ck; p.cin_pad = cin_pad;
  p.npad = a.cout_pad; p.nsplit = nsplit; p.nsub = nsub;
  pl->nt = nsub <= 64 ? 64 : 128;   // MMA width (a compile-time kernel parameter): the columns past nsub are not stored
  p.relu = a.relu; p.has_res = a.has_res; p.out_f32 = a.out.dtype == ACR_DT_F32;
  p.bias_per_image = a.bias_per_image; p.pow11_ch0 = a.pow11_ch0;
  p.xpair = a.xpair;
  // super-tiles cover the output grid, or the input grid of a transposed conv (each input tile feeds 4 output parities)
  const int grid_h = a.deconv ? a.in.H : a.out.H, grid_w = a.deconv ? a.in.W : a.out.W;
  p.tiles_x = grid_w / TILE_X; p.tiles_per_img = p.tiles_x * (grid_h / TILE_Y);
  p.total_tiles = p.tiles_per_img * a.batch;
  const int npar = a.deconv ? 4 : 1;
  p.Ho = a.out.H; p.Wo = a.out.W; p.out_stride = a.out.pix_stride;
  p.res_stride = a.has_res ? a.res.pix_stride : 0;
  // shared-memory plan
  p.a_stage_bytes = (uint32_t)(box_rows * box_cols) * ck * 2;
  // resident weights: every output channel of a (tap, chunk) in one box (<= 256 rows); streamed: one virtual tile's rows
  // (the transposed conv always streams: its [4 parities][cout_pad] rows are read one virtual tile at a time)
  const size_t b_total = (a.cout_pad <= 256 && !a.deconv) ?(size_t)p.taps * p.cchunks * a.cout_pad * ck * 2 : (size_t)1 << 40;
  p.bias_bytes = (uint32_t)(((size_t)a.cout_pad * 4 + 1023) & ~(size_t)1023);
  const size_t fixed = 1024 /*alignment slack*/ + p.bias_bytes + 512 /*barriers*/ + p.stage_out_bytes;
  const int nA = p.deconv ? p.cchunks : (p.s2x ? 2 : (p.patch1 ? p.cchunks : (p.patch_mode ? p.cchunks * 3 : p.taps * p.cchunks)));
  // stages that must fit next to resident weights: a tile's worth of kx patches (3) for 3x3 stride-1 convs, 2 otherwise
  const size_t min_a = (size_t)((p.patch_mode && !p.patch1) ? 3 : 2) * (size_t)p.a_stage_bytes;
  p.b_resident = (b_total + min_a + fixed <= (size_t)SMEM_BUDGET) ? 1 : 0;
  p.b_block_bytes = (uint32_t)(p.b_resident ? a.cout_pad : pl->nt) * ck * 2;
  {
    const int taps = p.taps;
    cuuint64_t dims[2] = {(cuuint64_t)taps * cin_pad, (cuuint64_t)npar * a.cout_pad};
    cuuint64_t str[1] = {(cuuint64_t)taps * cin_pad * esz};
    cuuint32_t box[2] = {(cuuint32_t)ck, (cuuint32_t)(p.b_resident ? a.cout_pad : pl->nt)};   // rows past cout_pad: zero fill
    rc = encode(&p.tmB, act_dtype, 2, a.w, dims, str, box, ck);
    if (rc) { delete pl; return rc; }
  }
  if (p.b_resident) {
    // the last virtual tile reads NT rows from its offset, possibly past cout_pad: keep them inside the region
    const int last_row = (nsplit - 1) * nsub + pl->nt;
    const size_t over = (size_t)(last_row > a.cout_pad ? last_row - a.cout_pad : 0) * ck * 2;
    p.b_region_bytes = (uint32_t)((b_total + over + 1023) & ~(size_t)1023);
    p.SB = 0;
  } else {
    p.SB = 4;
    while (p.SB > 2 && (size_t)p.SB * p.b_block_bytes + min_a + fixed > (size_t)SMEM_BUDGET) --p.SB;
    p.b_region_bytes = (uint32_t)(((size_t)p.SB * p.b_block_bytes + 1023) & ~(size_t)1023);
  }
  int SA = (int)(((size_t)SMEM_BUDGET - fixed - p.b_region_bytes) / p.a_stage_bytes);
  if (SA > 8) SA = 8;
  if (SA > 2 * nA && !p.patch1) SA = 2 * nA;  // no point in more stages than two super-tiles' worth of loads
  if ((p.patch1 || p.s2x || p.deconv) && SA > 4) SA = 4;
  if (SA < 2) { set_error("conv_tc: shared memory plan does not fit (cout_pad %d, ck %d)", a.cout_pad, ck); delete pl; return ACR_B200_EINVAL; }
  p.SA = SA;
  // ping-pong teams need every A load of a tile in the ring at once (conv_tc_kernel); the four-view stride-2 convs
  // (9 loads per channel chunk) and the 16-channel-chunk patch convs with several chunks stay in lockstep
  p.pingpong = (p.b_resident && nA <= SA) ? 1 : 0;
  pl->smem = fixed + p.b_region_bytes + (size_t)SA * p.a_stage_bytes;
  const int nvt = p.total_tiles * nsplit * npar;
  pl->grid = nvt < num_sms() ? nvt : num_sms();
  *out = pl;
  return ACR_B200_OK;
}

int conv_tc_launch(const ConvTcPlan* pl, cudaStream_t st) {
  if (pl->act_dtype == ACR_DT_TF32) return conv_tc_launch_tf32(pl, st);
  const bool bf = pl->act_dtype == ACR_DT_BF16;
  switch (pl->ck) {
    case 64: return bf ? conv_tc_launch_64_bf16(pl, st) : conv_tc_launch_64_f16(pl, st);
    case 32: return conv_tc_launch_32(pl, st);
    default: return conv_tc_launch_16(pl, st);
  }
}

void conv_tc_free(ConvTcPlan* p) { delete p; }

int conv_block_prepare(const ConvArgs& a1, const ConvArgs& a2, int act_dtype, int store_mid, ConvBlockPlan** out) {
  auto is_3x3_64 = [&](const ConvArgs& a) {
    return a.k == 3 && a.stride == 1 && a.cin_pad == 64 && a.cout_pad == 64 && a.relu && !a.bias_per_image && !a.pow11_ch0 &&
           a.n_ext == 0 && !a.s2x && !a.deconv && a.in.dtype == act_dtype && a.out.dtype == act_dtype;
  };
  ACR_CHECK_ARG(act_dtype == ACR_DT_BF16 || act_dtype == ACR_DT_F16, "conv_block: 16-bit activations only");
  ACR_CHECK_ARG(is_3x3_64(a1) && is_3x3_64(a2) && !a1.has_res && a2.has_res && a1.xpair == a2.xpair,
                "conv_block: a BasicBlock of two 3x3 stride-1 64->64 convs (or their x-paired form), ReLU, residual on conv2");
  ACR_CHECK_ARG(a2.in.ptr == a1.out.ptr && a2.res.ptr == a1.in.ptr && a2.res.pix_stride == a1.in.pix_stride,
                "conv_block: conv2 must read conv1's output, with conv1's input as the residual");
  const int H = a1.in.H, W = a1.in.W;
  ACR_CHECK_ARG(a1.out.H == H && a1.out.W == W && a2.out.H == H && a2.out.W == W && H % TILE_Y == 0 && W % TILE_X == 0,
                "conv_block: %dx%d is not a multiple of the 16x16 super-tile", H, W);
  ACR_CHECK_ARG(a1.in.pix_stride % 8 == 0 && a1.in.pix_stride >= 64 && a2.out.pix_stride % 2 == 0 && a1.out.pix_stride % 2 == 0,
                "conv_block: row alignment");
  ConvBlockPlan* pl = new ConvBlockPlan();
  ConvBlockParams& p = pl->p;
  pl->act_dtype = act_dtype; pl->xpair = a1.xpair;
  const cuuint64_t esz = 2;
  int rc;
  {
    cuuint64_t dims[4] = {64, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)a1.batch};
    cuuint64_t str[3] = {(cuuint64_t)a1.in.pix_stride * esz, (cuuint64_t)W * a1.in.pix_stride * esz,
                         (cuuint64_t)H * W * a1.in.pix_stride * esz};
    cuuint32_t box[4] = {64, BLK_PITCH, BLK_ROWS, 1};
    rc = encode(&p.tmA, act_dtype, 4, a1.in.ptr, dims, str, box, 64);
  }
  for (int c = 0; c < 2 && !rc; ++c) {
    cuuint64_t dims[2] = {9 * 64, 64};
    cuuint64_t str[1] = {9 * 64 * esz};
    cuuint32_t box[2] = {64, 64};
    rc = encode(c ? &p.tmB2 : &p.tmB1, act_dtype, 2, c ? a2.w : a1.w, dims, str, box, 64);
  }
  if (rc) { delete pl; return rc; }
  p.bias1 = a1.bias; p.bias2 = a2.bias;
  p.out = a2.out.ptr; p.mid = store_mid ? a1.out.ptr : nullptr;   // the residual is the input box (checked above)
  p.out_stride = a2.out.pix_stride; p.mid_stride = a1.out.pix_stride;
  p.H = H; p.W = W;
  p.tiles_x = W / TILE_X; p.tiles_per_img = p.tiles_x * (H / BLK_TILE_Y);   // 16 x 8 tiles
  p.total_tiles = p.tiles_per_img * a1.batch;
  pl->grid = p.total_tiles < num_sms() ? p.total_tiles : num_sms();
  *out = pl;
  return ACR_B200_OK;
}

void conv_block_free(ConvBlockPlan* p) { delete p; }

int conv_bottleneck_prepare(const ConvArgs& a1, const ConvArgs& a2, const ConvArgs& a3, int act_dtype, ConvBottleneckPlan** out) {
  auto plain = [&](const ConvArgs& a, int k, int cout_pad) {
    return a.k == k && a.stride == 1 && a.cout_pad == cout_pad && a.relu && !a.bias_per_image && !a.pow11_ch0 && a.n_ext == 0 &&
           !a.xpair && !a.s2x && !a.deconv && a.in.dtype == act_dtype && a.out.dtype == act_dtype;
  };
  ACR_CHECK_ARG(act_dtype == ACR_DT_BF16 || act_dtype == ACR_DT_F16, "conv_bottleneck: 16-bit activations only");
  ACR_CHECK_ARG(plain(a1, 1, 64) && plain(a2, 3, 64) && plain(a3, 1, 256) && !a1.has_res && !a2.has_res && a3.has_res &&
                    (a1.cin_pad == 64 || a1.cin_pad == 256) && a2.cin_pad == 64 && a3.cin_pad == 64 && a3.res.dtype == act_dtype,
                "conv_bottleneck: 1x1 (64 or 256) -> 64, 3x3 64 -> 64, 1x1 64 -> 256 + residual, stride 1, ReLU on all three");
  ACR_CHECK_ARG(a2.in.ptr == a1.out.ptr && a3.in.ptr == a2.out.ptr, "conv_bottleneck: each conv must read the previous one's output");
  const int H = a1.in.H, W = a1.in.W;
  ACR_CHECK_ARG(a1.out.H == H && a1.out.W == W && a2.out.H == H && a2.out.W == W && a3.out.H == H && a3.out.W == W &&
                    H % TILE_Y == 0 && W % TILE_X == 0,
                "conv_bottleneck: %dx%d is not a multiple of the 16x16 super-tile", H, W);
  ACR_CHECK_ARG(a1.in.pix_stride % 8 == 0 && a1.in.pix_stride >= a1.cin_pad && a3.out.pix_stride % 2 == 0 && a3.out.pix_stride >= 256 &&
                    a3.res.pix_stride % 2 == 0 && a3.res.pix_stride >= 256,
                "conv_bottleneck: row alignment");
  ConvBottleneckPlan* pl = new ConvBottleneckPlan();
  ConvBottleneckParams& p = pl->p;
  pl->act_dtype = act_dtype;
  const cuuint64_t esz = 2;
  int rc;
  {
    cuuint64_t dims[4] = {(cuuint64_t)a1.cin_pad, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)a1.batch};
    cuuint64_t str[3] = {(cuuint64_t)a1.in.pix_stride * esz, (cuuint64_t)W * a1.in.pix_stride * esz,
                         (cuuint64_t)H * W * a1.in.pix_stride * esz};
    cuuint32_t box[4] = {64, BNK_PITCH, BNK_ROWS, 1};
    rc = encode(&p.tmA, act_dtype, 4, a1.in.ptr, dims, str, box, 64);
  }
  // packed weights [cout_pad][taps * cin_pad]: conv1 [64][C_in], conv2 [64][9 * 64], conv3 [256][64] (one box)
  const ConvArgs* as[3] = {&a1, &a2, &a3};
  CUtensorMap* tms[3] = {&p.tmB1, &p.tmB2, &p.tmB3};
  for (int c = 0; c < 3 && !rc; ++c) {
    const ConvArgs& a = *as[c];
    const cuuint64_t kk = (cuuint64_t)a.k * a.k * a.cin_pad;
    cuuint64_t dims[2] = {kk, (cuuint64_t)a.cout_pad};
    cuuint64_t str[1] = {kk * esz};
    cuuint32_t box[2] = {64, (cuuint32_t)a.cout_pad};
    rc = encode(tms[c], act_dtype, 2, a.w, dims, str, box, 64);
  }
  if (rc) { delete pl; return rc; }
  p.bias1 = a1.bias; p.bias2 = a2.bias; p.bias3 = a3.bias;
  p.res = a3.res.ptr; p.out = a3.out.ptr;
  pl->cchunks = a1.cin_pad / 64;
  p.res_stride = a3.res.pix_stride; p.out_stride = a3.out.pix_stride;
  p.H = H; p.W = W;
  p.tiles_x = W / TILE_X; p.tiles_per_img = p.tiles_x * (H / BNK_TILE_Y);   // 16 x 8 tiles
  p.total_tiles = p.tiles_per_img * a1.batch;
  pl->grid = p.total_tiles < num_sms() ? p.total_tiles : num_sms();
  *out = pl;
  return ACR_B200_OK;
}

void conv_bottleneck_free(ConvBottleneckPlan* p) { delete p; }

}  // namespace acr
