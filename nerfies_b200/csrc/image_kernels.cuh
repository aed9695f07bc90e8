// Rendered frames -> 8- and 16-bit images on the device, value for value what numpy computes in
// image_utils.image_to_uint8 / image_to_uint16 (image_utils.py:114-131) and save_depth
// (image_utils.py:172-174):  (src / scale * max).clip(0, max).astype(uintN),  max = 255 | 65535.
// Division and product are single IEEE float32 operations, the cast truncates (numpy's astype
// does not round: 0.999 * 255 = 254.745 -> 254).  -inf and negatives clip to 0, +inf to max.
// NaN passes through numpy's clip and its cast to an unsigned integer on x86-64 is 0 (cvttss2si
// yields 0x80000000, whose low 8 / 16 bits are 0); fmaxf(NaN, 0) = 0 gives the same value here.
// One pass, no workspace: a thread converts 16 output bytes from 16-byte loads and writes them
// with one 16-byte store; unaligned pointers and the tail take the scalar path.
#pragma once

namespace nfb {
namespace image {

constexpr int kThreads = 256;

template <typename Out>
__device__ __forceinline__ unsigned quantize_one(float x, float scale) {
  constexpr float kMax = sizeof(Out) == 1 ? 255.0f : 65535.0f;
  const float v = __fmul_rn(__fdiv_rn(x, scale), kMax);
  return __float2uint_rz(fminf(fmaxf(v, 0.0f), kMax));
}

// Out = unsigned char | unsigned short.  `vec` is the number of 16-byte output groups taken by the
// vector path (0 when src or dst is not 16-byte aligned); elements past them are converted one by one.
template <typename Out>
__global__ void __launch_bounds__(kThreads)
image_quantize_kernel(const float* __restrict__ src, long long n, long long vec, float scale,
                      Out* __restrict__ dst) {
  constexpr int kPer = 16 / sizeof(Out);       // outputs of one 16-byte store
  constexpr int kPack = 4 / sizeof(Out);       // outputs of one 32-bit word
  const long long stride = (long long)gridDim.x * kThreads;
  const long long tid = (long long)blockIdx.x * kThreads + threadIdx.x;
  for (long long g = tid; g < vec; g += stride) {
    const float4* in = reinterpret_cast<const float4*>(src) + g * (kPer / 4);
    float x[kPer];
#pragma unroll
    for (int i = 0; i < kPer / 4; ++i) {
      const float4 f = __ldg(in + i);
      x[4 * i] = f.x; x[4 * i + 1] = f.y; x[4 * i + 2] = f.z; x[4 * i + 3] = f.w;
    }
    unsigned w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      w[i] = 0;
#pragma unroll
      for (int j = 0; j < kPack; ++j)
        w[i] |= quantize_one<Out>(x[i * kPack + j], scale) << (8 * sizeof(Out) * j);
    }
    reinterpret_cast<uint4*>(dst)[g] = make_uint4(w[0], w[1], w[2], w[3]);
  }
  for (long long i = vec * kPer + tid; i < n; i += stride)
    dst[i] = static_cast<Out>(quantize_one<Out>(src[i], scale));
}

}  // namespace image
}  // namespace nfb
