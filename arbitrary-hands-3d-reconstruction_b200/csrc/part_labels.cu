// Part labels on the device: SegmNet's 33-class logits (the arena's `segms`, M x M NHWC, 16-bit or fp32) ->
// bilinear resize to each frame's padded square (F.interpolate, align_corners=False) -> argmax -> uint8 labels of the
// frame's own H x W pixels, packed frame after frame.  tests/part_labels_ref.py is the statement.
//
// Each CTA owns a 16 x 16 block of source quads (quad (i, j): cells i, i+1 by j, j+1, the upper neighbour clamped to
// M - 1) of one image, and every output pixel whose bilinear footprint is that quad.  The CTA stages the 17 x 17 cells
// of its quads in shared memory as fp32, once, then:
//   * labels each cell with its winner c when c beats the runner-up by more than 2^-20 of the cell's largest |logit|,
//     else "mixed";
//   * labels a quad c when all four corners are c: every bilinear weight set is a convex combination of the corners,
//     so c wins the exact interpolation, and the 2^-20 margin is four times the fp32 rounding of the interpolation
//     below (<= 8u of the corners' largest |logit| between two channels), so c wins the computed one too;
//   * stores the quad's label for the pixels of uniform quads and runs the 33-channel interpolation + argmax (strict
//     >, so ties go to the lowest channel as torch.argmax) only for the pixels of mixed quads.
// The output pixels of a quad block are a rectangle (the source index is monotone in the output index), found by a
// binary search over the fp32 source index.  Blocks that no pixel of the frame maps to return before loading.  Source
// tiling keeps the staged footprint at 17 x 17 cells for every frame size, small frames included.
#include <math.h>

#include "common.cuh"

namespace acr {

constexpr int PL_CH = 33;          // background, 16 right-hand parts, 16 left-hand parts
constexpr int PL_Q = 16;           // quads per CTA and axis
constexpr int PL_F = PL_Q + 1;     // staged cells per axis
constexpr int PL_THREADS = 256;
constexpr int PL_PREFIX_THREADS = 1024;
constexpr unsigned char PL_MIXED = 255;

struct PartGeom {
  int side, pad_t, pad_l, H, W;
};

// The offsets row [side, side, 0,0,0,0, pad_t, pad_r, pad_b, pad_l] as a frame, or false: every entry a non-negative
// integer (NaN fails), both sides equal and in 1..ACR_B200_PART_LABELS_MAX_SIDE, pad_t + pad_b < side,
// pad_l + pad_r < side.  The pads are compared in float first so that no huge value reaches an int conversion.
__device__ __forceinline__ bool part_geom(const float* o, PartGeom& g) {
#pragma unroll
  for (int i = 0; i < 10; ++i)
    if (!(o[i] >= 0.f) || o[i] != floorf(o[i])) return false;
  if (o[0] != o[1] || o[0] < 1.f || o[0] > (float)ACR_B200_PART_LABELS_MAX_SIDE) return false;
  if (o[6] + o[8] >= o[0] || o[7] + o[9] >= o[0]) return false;   // exact: integers below 2^15
  g.side = (int)o[0];
  g.pad_t = (int)o[6];
  g.pad_l = (int)o[9];
  g.H = g.side - g.pad_t - (int)o[8];
  g.W = g.side - g.pad_l - (int)o[7];
  return true;
}

// torch's area_pixel_compute_source_index (align_corners=False, not cubic) in fp32
__device__ __forceinline__ float part_src(float scale, int d) {
  return fmaxf(__fmaf_rn(scale, (float)d + 0.5f, -0.5f), 0.f);
}

// one CTA: exclusive prefix of H*W over the valid frames, the flags, and each frame's first label byte
__global__ void __launch_bounds__(PL_PREFIX_THREADS) part_labels_prefix_kernel(const float* offsets, int n,
                                                                               long long capacity,
                                                                               long long* frame_offset, int* flags) {
  __shared__ long long part[PL_PREFIX_THREADS];
  const int t = threadIdx.x, per = (n + PL_PREFIX_THREADS - 1) / PL_PREFIX_THREADS;
  const int b = min(t * per, n), e = min(b + per, n);
  long long s = 0;
  for (int i = b; i < e; ++i) {
    PartGeom g;
    if (part_geom(offsets + (size_t)i * 10, g)) s += (long long)g.H * g.W;
  }
  part[t] = s;
  __syncthreads();
  for (int d = 1; d < PL_PREFIX_THREADS; d <<= 1) {   // inclusive Hillis-Steele scan
    const long long v = t >= d ? part[t - d] : 0;
    __syncthreads();
    part[t] += v;
    __syncthreads();
  }
  long long pos = part[t] - s;
  for (int i = b; i < e; ++i) {
    PartGeom g;
    const bool ok = part_geom(offsets + (size_t)i * 10, g);
    const long long size = ok ? (long long)g.H * g.W : 0;
    frame_offset[i] = pos;
    flags[i] = !ok ? ACR_B200_PART_LABELS_INVALID : pos + size > capacity ? ACR_B200_PART_LABELS_OVER_CAPACITY : 0;
    pos += size;
  }
}

struct PartArgs {
  const void* segms;        // (n, M, M, pix_stride) NHWC
  const float* offsets;     // (n, 10)
  const long long* frame_offset;
  const int* flags;
  uint8_t* labels;
  int M, pix_stride;
};

template <typename T>
__global__ void __launch_bounds__(PL_THREADS) part_labels_kernel(PartArgs a) {
  __shared__ float cell[PL_F * PL_F][PL_CH];   // odd row length: a thread per cell reads without bank conflicts
  __shared__ unsigned char sure[PL_F * PL_F];
  __shared__ unsigned char quad[PL_Q * PL_Q];
  __shared__ int range[4];                     // output rows [range[0], range[1]), columns [range[2], range[3])
  const int img = blockIdx.y, tid = threadIdx.x, M = a.M;
  if (a.flags[img]) return;
  PartGeom g;
  part_geom(a.offsets + (size_t)img * 10, g);  // valid: the prefix kernel flagged it otherwise
  const int nb = (M + PL_Q - 1) / PL_Q;
  const int qy0 = (blockIdx.x / nb) * PL_Q, qx0 = (blockIdx.x % nb) * PL_Q;
  const float scale = __fdiv_rn((float)M, (float)g.side);
  if (tid < 4) {   // first padded index in [lo, hi) whose source index reaches q, or hi
    const int q = (tid < 2 ? qy0 : qx0) + (tid & 1) * PL_Q;
    int lo = tid < 2 ? g.pad_t : g.pad_l;
    int hi = lo + (tid < 2 ? g.H : g.W);
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if ((int)part_src(scale, mid) >= q) hi = mid; else lo = mid + 1;
    }
    range[tid] = lo;
  }
  __syncthreads();
  const int Y0 = range[0], X0 = range[2], rows = range[1] - Y0, cols = range[3] - X0;
  if (rows <= 0 || cols <= 0) return;

  // stage the 17 x 17 cells (rows / columns past M - 1 repeat M - 1: torch's clamped upper neighbour)
  constexpr int E = 16 / sizeof(T);                 // channels per 16-byte load
  constexpr int U = (PL_CH + E - 1) / E;            // loads per cell
  const T* src = reinterpret_cast<const T*>(a.segms) + (size_t)img * M * M * a.pix_stride;
  for (int i = tid; i < PL_F * PL_F * U; i += PL_THREADS) {
    const int c = i / U, u = i - c * U;
    const int gy = min(qy0 + c / PL_F, M - 1), gx = min(qx0 + c % PL_F, M - 1);
    const uint4 v = *reinterpret_cast<const uint4*>(src + ((size_t)gy * M + gx) * a.pix_stride + u * E);
    const T* p = reinterpret_cast<const T*>(&v);
#pragma unroll
    for (int j = 0; j < E; ++j)
      if (u * E + j < PL_CH) cell[c][u * E + j] = to_f32<T>(p[j]);
  }
  __syncthreads();
  for (int c = tid; c < PL_F * PL_F; c += PL_THREADS) {
    float best = cell[c][0], second = -INFINITY, amax = fabsf(best);
    int arg = 0;
    bool nan = best != best;
#pragma unroll
    for (int k = 1; k < PL_CH; ++k) {
      const float v = cell[c][k];
      nan |= v != v;
      amax = fmaxf(amax, fabsf(v));
      if (v > best) {
        second = best;
        best = v;
        arg = k;
      } else {
        second = fmaxf(second, v);
      }
    }
    sure[c] = !nan && best - second > fmaxf(amax * 0x1p-20f, 1e-30f) ? (unsigned char)arg : PL_MIXED;
  }
  __syncthreads();
  {
    const int i = tid / PL_Q, j = tid % PL_Q, c = i * PL_F + j;
    const unsigned char s = sure[c];
    quad[tid] = s == sure[c + 1] && s == sure[c + PL_F] && s == sure[c + PL_F + 1] ? s : PL_MIXED;
  }
  __syncthreads();

  // threads take `span` consecutive columns of `step` rows at a time: the column's source index once per column, the
  // row's once per pixel, and consecutive threads store consecutive bytes of a row
  uint8_t* out = a.labels + a.frame_offset[img] + (size_t)(Y0 - g.pad_t) * g.W + (X0 - g.pad_l);
  const int span = min(cols, PL_THREADS), step = PL_THREADS / span, r_first = tid / span;
  if (r_first >= step) return;
  for (int x = tid - r_first * span; x < cols; x += span) {
    const float sx = part_src(scale, X0 + x);
    const int x0 = (int)sx, qx = x0 - qx0;
    const float lx = sx - (float)x0, hx = 1.f - lx;   // torch's weights: lambda = src - (int)src, 1 - lambda
    for (int r = r_first; r < rows; r += step) {
      const float sy = part_src(scale, Y0 + r);
      const int y0 = (int)sy, qy = y0 - qy0;
      int lab = quad[qy * PL_Q + qx];
      if (lab == PL_MIXED) {
        const float ly = sy - (float)y0, hy = 1.f - ly;
        const int c = qy * PL_F + qx;
        const float* c00 = cell[c];
        const float* c01 = cell[c + 1];
        const float* c10 = cell[c + PL_F];
        const float* c11 = cell[c + PL_F + 1];
        float best = 0.f;
#pragma unroll
        for (int k = 0; k < PL_CH; ++k) {
          const float v = __fmaf_rn(hy, __fmaf_rn(lx, c01[k], hx * c00[k]), ly * __fmaf_rn(lx, c11[k], hx * c10[k]));
          if (k == 0 || v > best) {
            best = v;
            lab = k;
          }
        }
      }
      out[(size_t)r * g.W + x] = (uint8_t)lab;
    }
  }
}

}  // namespace acr

using namespace acr;

extern "C" int acr_b200_part_labels(const void* segms, int dtype, int pix_stride, int map_size, const float* offsets,
                                    int n, int64_t capacity, uint8_t* labels, int64_t* frame_offset, int32_t* flags,
                                    void* stream) {
  ACR_CHECK_ARG(segms && offsets && labels && frame_offset && flags, "part_labels: null argument");
  ACR_CHECK_ARG(dtype == ACR_DT_BF16 || dtype == ACR_DT_F16 || dtype == ACR_DT_F32,
                "part_labels: dtype %d is not bf16, fp16 or fp32", dtype);
  const int esz = dtype == ACR_DT_F32 ? 4 : 2, E = 16 / esz;
  ACR_CHECK_ARG(pix_stride >= (PL_CH + E - 1) / E * E && pix_stride * esz % 16 == 0 &&
                    reinterpret_cast<uintptr_t>(segms) % 16 == 0,
                "part_labels: the map needs a 16-byte aligned base and pixel stride covering 33 channels in 16-byte "
                "loads (pix_stride=%d)", pix_stride);
  ACR_CHECK_ARG(map_size >= 1 && map_size <= 4096 && n >= 1 && n <= 65535 && capacity >= 0,
                "part_labels: bad map_size=%d / n=%d / capacity=%lld", map_size, n, (long long)capacity);
  const cudaStream_t s = (cudaStream_t)stream;
  part_labels_prefix_kernel<<<1, PL_PREFIX_THREADS, 0, s>>>(offsets, n, (long long)capacity,
                                                            reinterpret_cast<long long*>(frame_offset), flags);
  ACR_CHECK_LAUNCH();
  const int nb = (map_size + PL_Q - 1) / PL_Q;
  const PartArgs a{segms, offsets, reinterpret_cast<const long long*>(frame_offset), flags, labels, map_size, pix_stride};
  const dim3 grid((unsigned)(nb * nb), (unsigned)n);
  if (dtype == ACR_DT_BF16)
    part_labels_kernel<__nv_bfloat16><<<grid, PL_THREADS, 0, s>>>(a);
  else if (dtype == ACR_DT_F16)
    part_labels_kernel<__half><<<grid, PL_THREADS, 0, s>>>(a);
  else
    part_labels_kernel<float><<<grid, PL_THREADS, 0, s>>>(a);
  ACR_CHECK_LAUNCH();
  return ACR_B200_OK;
}
