// Frame pre-processing on the device (SURVEY.md 8f-2): BGR -> RGB, white pad to a square, bicubic resize to
// input_size x input_size, all in one kernel reading the raw frame once.
// Replaces (reference, /root/reference/acr/utils.py): img_preprocess :1315-1337 (image[:,:,::-1],
// process_image_ori :1310-1313 -> image_pad_white_bg :1303-1308 with imgaug's
// compute_paddings_to_reach_aspect_ratio and pad_cval=255, cv2.resize(..., INTER_CUBIC) :1320).
//
// Arithmetic = OpenCV's generic 8-bit cubic path (third-party, absent from the reference tree: opencv-python,
// resize.cpp HResizeCubic/VResizeCubic with INTER_RESIZE_COEF_BITS = 11): per axis 4 taps with short
// coefficients round(c*2048) of the A=-0.75 cubic at fx = (d+0.5)*scale-0.5, border = replicate, horizontal
// pass exact in int32, vertical pass (sum + 2^21) >> 22, saturate to uint8.  The coefficient / offset tables
// are built on the host in float32 exactly like OpenCV (acr_b200/preprocess.py) and passed in, so the kernel
// is pure integer work and bit-reproducible.  (OpenCV builds that dispatch to IPP differ from this generic
// path by +-1 grey level on ~5 % of the pixels -- the reference itself is only defined up to that.)
#include "common.cuh"

namespace acr {

struct PreArgs {
  const uint8_t* src;   // (n, H, W, 3) BGR
  uint8_t* dst;         // (n, S, S, 3) RGB
  const int16_t* cx;    // (S,4) horizontal coefficients
  const int32_t* ox;    // (S) first-tap-plus-one source column in the PADDED square
  const int16_t* cy;
  const int32_t* oy;
  int n, H, W, S, side, pad_t, pad_l;
};

__global__ void __launch_bounds__(256) preprocess_kernel(PreArgs a) {
  const long long gid = (long long)blockIdx.x * 256 + threadIdx.x;
  const long long total = (long long)a.n * a.S * a.S;
  if (gid >= total) return;
  const int dx = (int)(gid % a.S), dy = (int)((gid / a.S) % a.S);
  const int img = (int)(gid / ((long long)a.S * a.S));
  const uint8_t* src = a.src + (size_t)img * a.H * a.W * 3;
  int acc[3] = {0, 0, 0};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int py = min(max(a.oy[dy] + j - 1, 0), a.side - 1);   // replicate border of the padded square
    const int sy = py - a.pad_t;
    int hor[3] = {0, 0, 0};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int px = min(max(a.ox[dx] + k - 1, 0), a.side - 1);
      const int sx = px - a.pad_l;
      const int w = a.cx[dx * 4 + k];
      if (sy >= 0 && sy < a.H && sx >= 0 && sx < a.W) {
        const uint8_t* p = src + ((size_t)sy * a.W + sx) * 3;
        hor[0] += w * p[2]; hor[1] += w * p[1]; hor[2] += w * p[0];   // BGR -> RGB
      } else {
        hor[0] += w * 255; hor[1] += w * 255; hor[2] += w * 255;      // white padding
      }
    }
    const int wy = a.cy[dy * 4 + j];
    acc[0] += wy * hor[0]; acc[1] += wy * hor[1]; acc[2] += wy * hor[2];
  }
  uint8_t* o = a.dst + (size_t)gid * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c] = (uint8_t)min(max((acc[c] + (1 << 21)) >> 22, 0), 255);
}

// ---- ragged batches: per-frame geometry and tables are device data ------------------------------------------------
// acr_b200/preprocess.py::cubic_tables, one thread per (frame, d).  Every operation is the numpy one, rounded to
// nearest on its own: fx in double, then the A = -0.75 polynomials in float32 left to right (numpy's order), so
// nothing may be contracted into an FMA.  5A, 8A, 4A, A+2 and A+3 are exact in float32.
__global__ void __launch_bounds__(256) cubic_tables_kernel(const int32_t* n_src, int n, int S, int16_t* coef,
                                                           int32_t* ofs) {
  const long long gid = (long long)blockIdx.x * 256 + threadIdx.x;
  if (gid >= (long long)n * S) return;
  const int src = n_src[gid / S], d = (int)(gid % S);
  int16_t* c_out = coef + gid * 4;
  if (src < 1) {
    c_out[0] = c_out[1] = c_out[2] = c_out[3] = 0;
    ofs[gid] = 0;
    return;
  }
  const double scale = __ddiv_rn((double)src, (double)S);
  const float fx = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), 0.5));
  const float s = floorf(fx);
  const float x = __fsub_rn(fx, s);
  const float x1 = __fadd_rn(x, 1.f), u = __fsub_rn(1.f, x);
  float c[4];
  c[0] = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(-0.75f, x1), -3.75f), x1), -6.f), x1), -3.f);
  c[1] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(1.25f, x), 2.25f), x), x), 1.f);
  c[2] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(1.25f, u), 2.25f), u), u), 1.f);
  c[3] = __fsub_rn(__fsub_rn(__fsub_rn(1.f, c[0]), c[1]), c[2]);
#pragma unroll
  for (int k = 0; k < 4; ++k) c_out[k] = (int16_t)rintf(__fmul_rn(c[k], 2048.f));
  ofs[gid] = (int32_t)s;
}

struct RaggedArgs {
  const uint8_t* src;               // packed BGR frames, src_bytes bytes
  long long src_bytes;
  const acr_b200_frame* frames;     // (n)
  const int16_t* coef;              // (n,S,4), both axes of a frame
  const int32_t* ofs;               // (n,S)
  uint8_t* dst;                     // (n,S,S,3) RGB
  float* offsets;                   // (n,10) or null
  int S;
};

// side - H and side - W are >= 0 once side == max(H, W), so no sum below can overflow
__device__ __forceinline__ bool frame_ok(const acr_b200_frame& f, long long src_bytes) {
  return f.H >= 1 && f.W >= 1 && f.side == max(f.H, f.W) && f.pad_t >= 0 && f.pad_l >= 0 &&
         f.pad_t <= f.side - f.H && f.pad_l <= f.side - f.W && f.offset >= 0 && f.offset <= src_bytes &&
         (long long)f.H * f.W <= (src_bytes - f.offset) / 3;
}

// grid (pixel blocks, n): blockIdx.y is the frame.  Per pixel the arithmetic of preprocess_kernel.
__global__ void __launch_bounds__(256) preprocess_ragged_kernel(RaggedArgs a) {
  const int img = blockIdx.y, S = a.S;
  const acr_b200_frame f = a.frames[img];
  const bool ok = frame_ok(f, a.src_bytes);
  if (a.offsets && blockIdx.x == 0 && threadIdx.x < 10) {
    const int i = threadIdx.x;
    const int v = !ok ? 0 : i < 2 ? f.side : i == 6 ? f.pad_t : i == 7 ? f.side - f.W - f.pad_l
                : i == 8 ? f.side - f.H - f.pad_t : i == 9 ? f.pad_l : 0;
    a.offsets[img * 10 + i] = (float)v;
  }
  const int pix = blockIdx.x * 256 + threadIdx.x;
  if (pix >= S * S) return;
  uint8_t* o = a.dst + ((size_t)img * S * S + pix) * 3;
  if (!ok) {
    o[0] = o[1] = o[2] = 0;
    return;
  }
  const int dx = pix % S, dy = pix / S;
  const int16_t* cf = a.coef + (size_t)img * S * 4;
  const int32_t* of = a.ofs + (size_t)img * S;
  const uint8_t* src = a.src + f.offset;
  int acc[3] = {0, 0, 0};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int py = min(max(of[dy] + j - 1, 0), f.side - 1);   // replicate border of the padded square
    const int sy = py - f.pad_t;
    int hor[3] = {0, 0, 0};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int px = min(max(of[dx] + k - 1, 0), f.side - 1);
      const int sx = px - f.pad_l;
      const int w = cf[dx * 4 + k];
      if (sy >= 0 && sy < f.H && sx >= 0 && sx < f.W) {
        const uint8_t* p = src + ((size_t)sy * f.W + sx) * 3;
        hor[0] += w * p[2]; hor[1] += w * p[1]; hor[2] += w * p[0];   // BGR -> RGB
      } else {
        hor[0] += w * 255; hor[1] += w * 255; hor[2] += w * 255;      // white padding
      }
    }
    const int wy = cf[dy * 4 + j];
    acc[0] += wy * hor[0]; acc[1] += wy * hor[1]; acc[2] += wy * hor[2];
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c] = (uint8_t)min(max((acc[c] + (1 << 21)) >> 22, 0), 255);
}

}  // namespace acr

using namespace acr;

extern "C" int acr_b200_preprocess(const uint8_t* frames_bgr, int n, int H, int W, const int16_t* coef_x,
                                   const int32_t* ofs_x, const int16_t* coef_y, const int32_t* ofs_y, int side,
                                   int pad_t, int pad_l, int out_size, uint8_t* out_rgb, void* stream) {
  ACR_CHECK_ARG(frames_bgr && out_rgb && coef_x && ofs_x && coef_y && ofs_y, "preprocess: null argument");
  ACR_CHECK_ARG(n > 0 && H > 0 && W > 0 && out_size > 0 && side >= H && side >= W && pad_t >= 0 && pad_l >= 0 &&
                    pad_t + H <= side && pad_l + W <= side, "preprocess: inconsistent geometry");
  PreArgs a{frames_bgr, out_rgb, coef_x, ofs_x, coef_y, ofs_y, n, H, W, out_size, side, pad_t, pad_l};
  const long long total = (long long)n * out_size * out_size;
  preprocess_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a);
  ACR_CHECK_LAUNCH();
  return ACR_B200_OK;
}

extern "C" int acr_b200_cubic_tables(const int32_t* n_src, int n, int out_size, int16_t* coef, int32_t* ofs,
                                     void* stream) {
  ACR_CHECK_ARG(n_src && coef && ofs, "cubic_tables: null argument");
  const long long total = (long long)n * out_size;
  ACR_CHECK_ARG(n > 0 && out_size > 0 && (total + 255) / 256 <= 0x7fffffff, "cubic_tables: bad n=%d / out_size=%d",
                n, out_size);
  cubic_tables_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(n_src, n, out_size, coef, ofs);
  ACR_CHECK_LAUNCH();
  return ACR_B200_OK;
}

extern "C" int acr_b200_preprocess_ragged(const uint8_t* frames_bgr, int64_t src_bytes, const acr_b200_frame* frames,
                                          int n, const int16_t* coef, const int32_t* ofs, int out_size,
                                          uint8_t* out_rgb, float* offsets, void* stream) {
  ACR_CHECK_ARG(frames_bgr && frames && coef && ofs && out_rgb, "preprocess_ragged: null argument");
  // grid.y carries the frame; S * S must fit the int pixel index
  ACR_CHECK_ARG(n > 0 && n <= 65535 && out_size > 0 && out_size <= 16384 && src_bytes >= 0,
                "preprocess_ragged: bad n=%d / out_size=%d / src_bytes=%lld", n, out_size, (long long)src_bytes);
  RaggedArgs a{frames_bgr, (long long)src_bytes, frames, coef, ofs, out_rgb, offsets, out_size};
  const dim3 grid((unsigned)(((long long)out_size * out_size + 255) / 256), (unsigned)n);
  preprocess_ragged_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a);
  ACR_CHECK_LAUNCH();
  return ACR_B200_OK;
}
