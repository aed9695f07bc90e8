// Self-test of the tensor-core plumbing the field kernel relies on: the 128-byte
// swizzled operand images, GMMA descriptors with K stepping inside a K-block, and
// the wgmma accumulator fragment layout.  One warpgroup computes C (128 x N) =
// A (128 x K, fp32 -> operand images) x W (the packed weight units, copied in as the
// field kernel's weight ring receives them), N in 16-column chunks.
//   kX3 = false: bf16 operands (nfb_selftest_gemm).
//   kX3 = true : the fp16x3 chains x_hi W_hi + x_hi W_lo + x_lo W_hi of the field
//                kernel, A split by round-to-nearest (nfb_selftest_gemm3).  As in the
//                field kernel's hidden layers, x_lo is the register A operand: each
//                thread loads its values in the accumulator fragment layout (x3_lo_reg).
#pragma once
#include "field_tc3.cuh"
#include "tc_common.cuh"

namespace nfb {
namespace tc {

constexpr int kSelfMaxKb = 5;                                        // K <= 320
constexpr int kSelfSmemBytes = 2 * kSelfMaxKb * kABlockBytes + 2 * kSelfMaxKb * 2048 + 64;

template <bool kX3>
__global__ void __launch_bounds__(128, 1)
tc_selftest_kernel(const float* __restrict__ A, int K, const uint8_t* __restrict__ w, int nkb, int n_rows, int N,
                   float scale, int reps, float* __restrict__ C, long long* __restrict__ out) {
  extern __shared__ __align__(1024) uint8_t sm[];
  uint8_t* a_hi = sm;                                       // [kb][128 rows x 128 B]
  uint8_t* a_lo = sm + kSelfMaxKb * kABlockBytes;
  uint8_t* ws = sm + 2 * kSelfMaxKb * kABlockBytes;         // [kb][part][16 rows x 128 B]
  const int tid = threadIdx.x, lane = tid & 31, wq = tid >> 5, lq = lane & 3;
  constexpr int parts = kX3 ? 2 : 1;
  for (int i = tid; i < 128 * nkb * 8; i += 128) {
    const int r = i / (nkb * 8), kb = (i / 8) % nkb, ch = i % 8;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = kb * kBlockK + ch * 8 + j;
      v[j] = k < K ? A[(size_t)r * K + k] : 0.f;
    }
    if constexpr (kX3) tc3::store_chunk_x3(a_hi + kb * kABlockBytes, a_lo + kb * kABlockBytes, r, ch, v);
    else store_chunk(a_hi + kb * kABlockBytes, r, ch, v);
  }
  const long long t0 = clock64();
  for (int nc = 0; nc < n_rows / 16; ++nc) {
    __syncthreads();                                        // the previous chunk's MMAs are complete
    for (int i = tid; i < nkb * parts * 128; i += 128) {    // 16 rows x 128 B = 128 uint4 per unit
      const int unit = i / 128, q = i % 128;
      const uint4* src = reinterpret_cast<const uint4*>(w + ((size_t)unit * n_rows + nc * 16) * kRowBytes);
      reinterpret_cast<uint4*>(ws + unit * 2048)[q] = src[q];
    }
    fence_proxy_async();
    __syncthreads();
    for (int mt = 0; mt < 2; ++mt) {
      float d[8];
      const int row = mt * 64 + 16 * wq + (lane >> 2);
      uint32_t lo[kX3 ? kSelfMaxKb * 16 : 1];
      if constexpr (kX3) {
#pragma unroll
        for (int kb = 0; kb < kSelfMaxKb; ++kb)
#pragma unroll
          for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int k = kb * kBlockK + 8 * j + 2 * lq;
              const float* ar = A + (size_t)(row + 8 * h) * K;
              uint32_t hi;
              tc3::split_pair(k < K ? ar[k] : 0.f, k + 1 < K ? ar[k + 1] : 0.f, hi, lo[x3_lo_reg(kb, j, h)]);
            }
      }
      wg_fence();
      for (int rep = 0; rep < reps; ++rep)
#pragma unroll
        for (int kb = 0; kb < kSelfMaxKb; ++kb) {
          if (kb >= nkb) break;
          const uint32_t a0 = smem_u32(a_hi + kb * kABlockBytes) + mt * 8192;
          const uint32_t b0 = smem_u32(ws + kb * parts * 2048);
          if constexpr (kX3) wg_unit<true, 16>(d, a0, lo + x3_lo_reg(kb, 0, 0), b0, b0 + 2048, (rep | kb) != 0);
          else wg_unit<false, 16>(d, a0, 0u, b0, b0 + 2048, (rep | kb) != 0);
        }
      wg_commit();
      wg_wait<0>();
      wg_fence_regs<8>(d);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int rr = row + 8 * ((i >> 1) & 1), col = nc * 16 + 8 * (i >> 2) + 2 * lq + (i & 1);
        if (col < N) C[(size_t)rr * N + col] = d[i] * scale;
      }
    }
  }
  if (out && tid == 0) {
    out[0] = clock64() - t0;
    out[1] = (long long)nkb * 4 * (kX3 ? 3 : 1);            // MMAs per 64 x 16 output block and repetition
  }
}

}  // namespace tc
}  // namespace nfb
