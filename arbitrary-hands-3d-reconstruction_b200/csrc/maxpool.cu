// nn.MaxPool2d(kernel 3, stride 2, padding 1) of the ResNet trunk (after conv1 + bn1 + ReLU) on 16-bit NHWC.
//
// Thread = 8 channels (one 16-byte vector) of one output pixel.  The max runs over the taps that lie inside the input
// only, as PyTorch's padding never wins; the centre tap (2y, 2x) always exists and seeds it.  16-bit -> fp32 -> 16-bit is
// exact, so the result is bit-identical to F.max_pool2d on the same 16-bit input.
#include "ops.cuh"

namespace acr {
namespace {

template <typename T>
__global__ void __launch_bounds__(256) maxpool3s2_kernel(const T* __restrict__ in, T* __restrict__ out, int H, int W,
                                                         int in_stride, int out_stride, int groups, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int g = (int)(i % groups);
  long long p = i / groups;
  const int Wo = W >> 1, Ho = H >> 1;
  const int ox = (int)(p % Wo); p /= Wo;
  const int oy = (int)(p % Ho);
  const int n = (int)(p / Ho);
  const T* base = in + (size_t)n * H * W * in_stride + 8 * g;
  float m[8];
  unpack8<T>(*reinterpret_cast<const uint4*>(base + ((size_t)(2 * oy) * W + 2 * ox) * in_stride), m);
#pragma unroll
  for (int dy = -1; dy <= 1; ++dy) {
    const int iy = 2 * oy + dy;
    if (iy < 0 || iy >= H) continue;
#pragma unroll
    for (int dx = -1; dx <= 1; ++dx) {
      const int ix = 2 * ox + dx;
      if ((dy == 0 && dx == 0) || ix < 0 || ix >= W) continue;
      float v[8];
      unpack8<T>(*reinterpret_cast<const uint4*>(base + ((size_t)iy * W + ix) * in_stride), v);
#pragma unroll
      for (int c = 0; c < 8; ++c) m[c] = fmaxf(m[c], v[c]);
    }
  }
  *reinterpret_cast<uint4*>(out + (((size_t)n * Ho + oy) * Wo + ox) * out_stride + 8 * g) = pack8<T>(m);
}

}  // namespace

int launch_maxpool(const TensorRef& in, const TensorRef& out, int batch, int act_dtype, cudaStream_t st) {
  ACR_CHECK_ARG(in.dtype == act_dtype && out.dtype == act_dtype && (act_dtype == ACR_DT_BF16 || act_dtype == ACR_DT_F16),
                "maxpool: 16-bit tensors of the plan's dtype");
  ACR_CHECK_ARG(in.C == out.C && in.C % 8 == 0 && in.pix_stride % 8 == 0 && out.pix_stride % 8 == 0 && in.H % 2 == 0 &&
                    in.W % 2 == 0 && out.H * 2 == in.H && out.W * 2 == in.W && (uintptr_t)in.ptr % 16 == 0 &&
                    (uintptr_t)out.ptr % 16 == 0,
                "maxpool: shape / alignment (C %d -> %d, %dx%d -> %dx%d)", in.C, out.C, in.H, in.W, out.H, out.W);
  const int groups = in.C / 8;
  const long long total = (long long)batch * out.H * out.W * groups;
  const int threads = 256;
  const unsigned blocks = (unsigned)((total + threads - 1) / threads);
  if (act_dtype == ACR_DT_BF16)
    maxpool3s2_kernel<__nv_bfloat16><<<blocks, threads, 0, st>>>(static_cast<const __nv_bfloat16*>(in.ptr),
                                                                 static_cast<__nv_bfloat16*>(out.ptr), in.H, in.W,
                                                                 in.pix_stride, out.pix_stride, groups, total);
  else
    maxpool3s2_kernel<__half><<<blocks, threads, 0, st>>>(static_cast<const __half*>(in.ptr), static_cast<__half*>(out.ptr),
                                                          in.H, in.W, in.pix_stride, out.pix_stride, groups, total);
  ACR_CHECK_LAUNCH();
  return ACR_B200_OK;
}

}  // namespace acr
