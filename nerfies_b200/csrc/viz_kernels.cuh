// Colour maps on the device: value for value what numpy computes in the reference's
// visualization.colorize (visualization.py:177-219) followed by image_utils.image_to_uint8
// (image_utils.py:114-121), for a caller's 256-entry float64 table.  Under numpy 2 (NEP 50):
//   x = (v - cmin) / d           float32, cmin rounded to float32; d = float32(max(cmax - cmin, eps))
//                                (the subtraction is the caller's when both bounds are given: fp64 for
//                                Python floats; float32 when a bound is the frame's min / max)
//   y = invert ? 1 - x : x       float32
//   t = y * 255, a = floor(t), b = min(a + 1, 255), f = t - a          float32
//   c = table[a] + (table[b] - table[a]) * f                           float64, no contraction
//   x > 1 -> 1.0 (0.0 inverted), x < 0 -> 0.0 (1.0 inverted); NaN -> a NaN colour
//   uint8: trunc(clip(c * 255, 0, 255)) with a float64 product; NaN -> 0 (as x86-64's cast).
// The value v comes from a source: the array, its IEEE reciprocal, or the per-pixel error sums of
// two (h, w, 3) images in numpy's order ((e0 + e1) + e2).  kRgb is not a colour map: it writes an
// (h, w, 3) float32 image as uint8 through the same float64 product, the rgb half of
// image_to_uint8(concatenate([rgb, depth_viz], 1)).
//
// Bounds from the frame: colorize_range_kernel reduces the source to kRangeBlocks (min, max) pairs
// (NaN when the block saw a NaN, as np.min / np.max); every colorize block folds the pairs itself, so
// nothing returns to the host between the two launches.
//
// uint8 output goes through a row pitch and a column offset (a half of a wider frame).  A thread
// writes one 16-byte-aligned group of output bytes with one 16-byte store: it computes the <= 7
// pixels that touch the group (bytes 3p..3p+2 of pixel p).  Each row's unaligned head and tail bytes
// take a scalar path.  The table sits in shared memory as [256][3] doubles (6 KB); neighbouring
// pixels of a smooth image share bins, so a warp's reads are mostly broadcasts.  The grid is a few
// blocks per SM with a grid-stride loop, so the table is loaded a few hundred times per frame, not
// once per row.
#pragma once

#include <cstdint>

namespace nfb {
namespace viz {

constexpr int kThreads = 256;
constexpr int kRangeBlocks = 256;   // (min, max) partials: workspace of 2 * kRangeBlocks floats

enum Source { kValue = 0, kReciprocal = 1, kAbsError = 2, kSqError = 3, kRgb = 4 };
enum Flags { kInvert = 1, kFrameMin = 2, kFrameMax = 4 };

template <int S>
__device__ __forceinline__ float source_value(const float* __restrict__ a, const float* __restrict__ b, long long p) {
  if constexpr (S == kValue) return __ldg(a + p);
  else if constexpr (S == kReciprocal) return __fdiv_rn(1.0f, __ldg(a + p));
  else {
    float e[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float d = __fsub_rn(__ldg(a + 3 * p + c), __ldg(b + 3 * p + c));
      e[c] = S == kAbsError ? fabsf(d) : __fmul_rn(d, d);
    }
    return __fadd_rn(__fadd_rn(e[0], e[1]), e[2]);
  }
}

template <int S>
__global__ void __launch_bounds__(kThreads)
colorize_range_kernel(const float* __restrict__ a, const float* __restrict__ b, long long n,
                      float* __restrict__ partials) {
  float lo = INFINITY, hi = -INFINITY;
  bool nan = false;
  for (long long p = (long long)blockIdx.x * kThreads + threadIdx.x; p < n; p += (long long)kRangeBlocks * kThreads) {
    const float v = source_value<S>(a, b, p);
    nan |= v != v;
    lo = fminf(lo, v);
    hi = fmaxf(hi, v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  nan = __any_sync(0xffffffffu, nan);
  __shared__ float s_lo[kThreads / 32], s_hi[kThreads / 32];
  __shared__ int s_nan;
  if (threadIdx.x == 0) s_nan = 0;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) {
    s_lo[threadIdx.x >> 5] = lo;
    s_hi[threadIdx.x >> 5] = hi;
    if (nan) s_nan = 1;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kThreads / 32; ++w) {
      lo = fminf(lo, s_lo[w]);
      hi = fmaxf(hi, s_hi[w]);
    }
    partials[blockIdx.x] = s_nan ? NAN : lo;
    partials[kRangeBlocks + blockIdx.x] = s_nan ? NAN : hi;
  }
}

// One pixel's three colour components (float64).
__device__ __forceinline__ void colour(float v, float cmin, float d, bool invert, const double* table, double c[3]) {
  const float x = __fdiv_rn(__fsub_rn(v, cmin), d);
  if (x > 1.0f || x < 0.0f) {
    const double fill = (x > 1.0f) != invert ? 1.0 : 0.0;
    c[0] = c[1] = c[2] = fill;
    return;
  }
  const float y = invert ? __fsub_rn(1.0f, x) : x;
  const float t = __fmul_rn(y, 255.0f);
  const float af = floorf(t);
  const float f = __fsub_rn(t, af);
  const int ia = min(max(__float2int_rz(af), 0), 255);       // NaN: any bin; the colour is NaN
  const int ib = min(ia + 1, 255);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double ca = table[3 * ia + k];
    c[k] = __dadd_rn(ca, __dmul_rn(__dsub_rn(table[3 * ib + k], ca), (double)f));
  }
}

__device__ __forceinline__ unsigned to_u8(double c) {
  return (unsigned)__double2uint_rz(fmin(fmax(__dmul_rn(c, 255.0), 0.0), 255.0));
}

// The three uint8 components of pixel p.
template <int S>
__device__ __forceinline__ void pixel_u8(const float* __restrict__ a, const float* __restrict__ b, long long p,
                                         float cmin, float d, bool invert, const double* table, unsigned u[3]) {
  if (S == kRgb) {
#pragma unroll
    for (int k = 0; k < 3; ++k) u[k] = to_u8((double)__ldg(a + 3 * p + k));
    return;
  }
  double c[3];
  colour(source_value<S>(a, b, p), cmin, d, invert, table, c);
#pragma unroll
  for (int k = 0; k < 3; ++k) u[k] = to_u8(c[k]);
}

// The scale of this call: (cmin, d), the block folding the range partials (one pair per thread)
// when a bound comes from the frame.  Every thread of the block calls it.
__device__ __forceinline__ float2 scale_of(const float* __restrict__ partials, float cmin, float cmax, float d,
                                           int flags) {
  static_assert(kRangeBlocks == kThreads, "one partial per thread");
  if (!(flags & (kFrameMin | kFrameMax))) return make_float2(cmin, d);
  __shared__ float s_lo[kThreads / 32], s_hi[kThreads / 32];
  float lo = partials[threadIdx.x], hi = partials[kRangeBlocks + threadIdx.x];
  const bool nan = __syncthreads_or(lo != lo);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  if ((threadIdx.x & 31) == 0) {
    s_lo[threadIdx.x >> 5] = lo;
    s_hi[threadIdx.x >> 5] = hi;
  }
  __syncthreads();
  for (int w = 0; w < kThreads / 32; ++w) {
    lo = fminf(lo, s_lo[w]);
    hi = fmaxf(hi, s_hi[w]);
  }
  if (flags & kFrameMin) cmin = nan ? NAN : lo;
  if (flags & kFrameMax) cmax = nan ? NAN : hi;
  const float diff = __fsub_rn(cmax, cmin);
  return make_float2(cmin, d > diff ? d : diff);             // d is float32(eps) here; NaN stays NaN
}

template <int S>
__device__ __forceinline__ void load_table(const double* __restrict__ table, double* s_table) {
  if (S != kRgb)
    for (int i = threadIdx.x; i < 768; i += kThreads) s_table[i] = table[i];
  __syncthreads();
}

// uint8 output: rows of `width` pixels at dst + row * pitch (bytes; the column offset is applied by
// the caller).  Work unit u of a row: 0 = the unaligned head bytes, 1..groups = 16-byte groups,
// groups + 1 = the tail bytes.
template <int S>
__global__ void __launch_bounds__(kThreads)
colorize_u8_kernel(const float* __restrict__ a, const float* __restrict__ b, int height, int width,
                   const double* __restrict__ table, const float* __restrict__ partials, float cmin, float cmax,
                   float d, int flags, unsigned char* __restrict__ dst, long long pitch) {
  __shared__ double s_table[768];
  load_table<S>(table, s_table);
  const float2 sc = scale_of(partials, cmin, cmax, d, flags);
  const bool invert = flags & kInvert;
  const int row_bytes = 3 * width;
  const int max_units = row_bytes / 16 + 2;
  const int total = height * max_units;                      // < 2^31: checked by the caller
  for (int w = blockIdx.x * kThreads + threadIdx.x; w < total; w += gridDim.x * kThreads) {
    const int row = w / max_units, u = w - row * max_units;
    unsigned char* out = dst + row * pitch;
    const long long pix0 = (long long)row * width;
    const int head = min((int)((16 - (reinterpret_cast<uintptr_t>(out) & 15)) & 15), row_bytes);
    const int groups = (row_bytes - head) / 16;
    if (u == 0 || u == groups + 1) {
      const int lo = u == 0 ? 0 : head + 16 * groups;
      const int hi = u == 0 ? head : row_bytes;
      for (int byte = lo; byte < hi; ++byte) {
        unsigned c[3];
        pixel_u8<S>(a, b, pix0 + byte / 3, sc.x, sc.y, invert, s_table, c);
        const int k = byte % 3;
        out[byte] = (unsigned char)(k == 0 ? c[0] : k == 1 ? c[1] : c[2]);
      }
    } else if (u <= groups) {
      const int first = head + 16 * (u - 1);                 // the group's first byte in the row
      unsigned long long lo = 0ull, hi = 0ull;             // bytes 0-7 and 8-15 of the group
      for (int p = first / 3; 3 * p < first + 16; ++p) {
        unsigned c[3];
        pixel_u8<S>(a, b, pix0 + p, sc.x, sc.y, invert, s_table, c);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const int j = 3 * p + k - first;
          if (j >= 0 && j < 8) lo |= (unsigned long long)c[k] << (8 * j);
          else if (j >= 8 && j < 16) hi |= (unsigned long long)c[k] << (8 * (j - 8));
        }
      }
      *reinterpret_cast<uint4*>(out + first) =
          make_uint4((unsigned)lo, (unsigned)(lo >> 32), (unsigned)hi, (unsigned)(hi >> 32));
    }
  }
}

// float64 (n, 3) output, what colorize returns.
template <int S>
__global__ void __launch_bounds__(kThreads)
colorize_f64_kernel(const float* __restrict__ a, const float* __restrict__ b, long long n,
                    const double* __restrict__ table, const float* __restrict__ partials, float cmin, float cmax,
                    float d, int flags, double* __restrict__ dst) {
  __shared__ double s_table[768];
  load_table<S>(table, s_table);
  const float2 sc = scale_of(partials, cmin, cmax, d, flags);
  for (long long p = (long long)blockIdx.x * kThreads + threadIdx.x; p < n; p += (long long)gridDim.x * kThreads) {
    double c[3];
    colour(source_value<S>(a, b, p), sc.x, sc.y, flags & kInvert, s_table, c);
#pragma unroll
    for (int k = 0; k < 3; ++k) dst[3 * p + k] = c[k];
  }
}

// The range pass when a bound comes from the frame, then the colour pass; `sms` sizes the grid.
template <int S>
void launch(const float* a, const float* b, int height, int width, const double* table,
                            float cmin, float cmax, float d, int flags, float* partials, double* out_f64,
                            unsigned char* out_u8, long long pitch, int sms, cudaStream_t s) {
  const long long n = (long long)height * width;
  if (flags & (kFrameMin | kFrameMax))
    colorize_range_kernel<S><<<kRangeBlocks, kThreads, 0, s>>>(a, b, n, partials);
  if (out_f64) {
    const long long blocks = std::min<long long>((n + kThreads - 1) / kThreads, 4ll * sms);
    colorize_f64_kernel<S><<<(unsigned)blocks, kThreads, 0, s>>>(a, b, n, table, partials, cmin, cmax, d, flags,
                                                                   out_f64);
  } else {
    const long long units = (long long)height * (3 * width / 16 + 2);
    const long long blocks = std::min<long long>((units + kThreads - 1) / kThreads, 4ll * sms);
    colorize_u8_kernel<S><<<(unsigned)blocks, kThreads, 0, s>>>(a, b, height, width, table, partials, cmin, cmax,
                                                                  d, flags, out_u8, pitch);
  }
}

}  // namespace viz
}  // namespace nfb
