// Training tier, tf32x3 mode (NFB_TRAIN_TF32X3, opt-in per handle): the GEMM of train.cuh on the
// tensor cores.  Same contract as sgemm128_kernel - C(m, n) (+)= sum_k A(m, k) B(k, n), A and B read
// through the element functors, C written through the epilogue functor, gridDim.z splitting the
// reduction into slices of k_per_split - so every launch_gemm call site runs either kernel unchanged.
//
// Split arithmetic: every operand value a becomes big = tf32(a), small = tf32(a - big) (cvt.rna;
// a - big is exact in fp32).  Per k-block of 32 the three chains go, in this fixed order, into a fresh
// fp32 register partial: A_small B_big, A_big B_small, A_big B_big (each over the block's four k8
// steps); the partial is then added to the running fp32 sum (FADD, round to nearest).  tf32 x tf32
// products are exact in fp32 (11 x 11 significant bits); what is lost per product is A_small B_small
// and the rounding of the two small parts, together at most ~3 x 2^-22 |a||b|.  TF32 keeps fp32's
// 8-bit exponent, so operands over any range that fp32 holds need no scaling.
// Why a partial per k-block: the tensor cores' fp32 accumulation is not round-to-nearest; with one
// accumulator carried over a whole reduction (up to 3 x 256 / 8 wgmma steps for a layer, 3 x 8192 / 8 for
// a dW slice) its error drifts one way, and the gin-size gradient checks (test_training_scale_gpu.py)
// measured 2-4x their tolerance.  Twelve steps per partial keep that error at the block's own scale.
//
// Tile: 128 x 128 of C per CTA, two consumer warpgroups of 64 rows (wgmma m64n128k8), k-blocks of 32
// (one 128-byte swizzle row of fp32).  All 256 threads stage: they read a k-block of A and B through
// the functors into registers, split, and store big and small into K-major swizzled images (tc_common.cuh
// operand format).  Two stages of 64 KB (A big, A small, B big, B small, 16 KB each): while the MMAs of
// block k run, block k+1 is stored into the other stage and the global loads of block k+2 are issued.
// Rows, columns and k beyond the shape (or the slice) are staged as zeros.
#pragma once
#include "tc_common.cuh"
#include "train.cuh"

namespace nfb {
namespace train {

constexpr int kTcBK = 32;                               // fp32 per 128-byte swizzle row: one k-block
constexpr int kTcImage = kT2 * tc::kRowBytes;           // 16 KB: 128 rows of one k-block
constexpr int kTcStage = 4 * kTcImage;                  // A big, A small, B big, B small
constexpr int kTcSmem = 2 * kTcStage + 1024;            // two stages + slack to align to 1024 bytes

// (row, k) of element e (0..15) of this thread's share of a 128 x 32 k-block.  Contiguous-k operands:
// a warp takes 32 consecutive k of one row (128-byte global reads, 32 distinct banks in the swizzled
// row).  Contiguous-row operands: a warp takes 8 consecutive rows x 4 consecutive k (32-byte global
// segments; the swizzle spreads the 8 rows over 8 chunks, so the stores hit 32 distinct banks).
template <bool kKFast>
__device__ __forceinline__ void tc_slot(int warp, int lane, int e, int& row, int& k) {
  if (kKFast) {
    row = warp + 8 * e; k = lane;
  } else {
    const int q = warp + 8 * e;
    row = (q & 15) * 8 + (lane & 7); k = (q >> 4) * 4 + (lane >> 3);
  }
}

// Byte offset in a k-block image of element e of tc_slot<kKFast>(warp, lane, e): tc::swz_off(row, k >> 2) +
// (k & 3) * 4 as a per-thread base (tc_stage_base) and a step that is an immediate or one XOR
// (tc_stage_off).  With warp < 8: contiguous-k, row & 7 = warp and the rows of e are 8 e apart (1 KB);
// contiguous-row, row & 7 = lane & 7, chunk e >> 1 (bits 4-6, disjoint from the other terms) and
// e & 1 selects rows 64 apart (8 KB).
template <bool kKFast>
__device__ __forceinline__ uint32_t tc_stage_base(int warp, int lane) {
  return kKFast ? warp * 128 + (((lane >> 2) ^ (warp & 7)) << 4) + (lane & 3) * 4
                : warp * 1024 + (lane & 7) * 128 + ((lane & 7) << 4) + (lane >> 3) * 4;
}
template <bool kKFast>
__device__ __forceinline__ uint32_t tc_stage_off(uint32_t base, int e) {
  return kKFast ? base + e * 1024 : (base ^ ((e >> 1) << 4)) + (e & 1) * 8192;
}

__device__ __forceinline__ void st_shared(uint32_t addr, float v) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}

// One k-block of one chain: four k8 steps; `first` overwrites d instead of accumulating into it.
__device__ __forceinline__ void tf32_chain(float* d, uint32_t a, uint32_t b, bool first = false) {
  const uint64_t da = tc::make_wg_desc(a), db = tc::make_wg_desc(b);
#pragma unroll
  for (int ks = 0; ks < kTcBK / 8; ++ks) tc::wg_mma_n128_tf32(d, da + 2 * ks, db + 2 * ks, (first && ks == 0) ? 0u : 1u);
}

template <bool kAKFast, bool kBNFast, class FA, class FB, class FC>
__global__ void __launch_bounds__(256, 1)
tf32x3_gemm_kernel(GemmShape sh, FA fa, FB fb, FC fc, long long k_per_split) {
  extern __shared__ uint8_t tc_smem_raw[];
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(tc_smem_raw) + 1023) & ~uintptr_t(1023));
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = tid >> 7;
  const long long m0 = (long long)blockIdx.x * kT2;
  const int n0 = blockIdx.y * kT2;
  const long long k_begin = (long long)blockIdx.z * k_per_split;
  const long long k_end = min(sh.K, k_begin + k_per_split);
  float acc[64], part[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = part[i] = 0.f;
  float ra[16], rb[16];
  // Opaque copies of the per-thread indices: the address arithmetic of the 32 staged elements is redone per
  // k-block instead of being held in registers across the loop (which spills beside the 64 accumulators).
  // A k-block wholly inside the shape and the slice is read without the per-element bounds checks.
  auto fetch = [&](long long k0) {
    int w = warp, l = lane, nb = n0;
    long long mb = m0;
    asm volatile("" : "+r"(w), "+r"(l), "+r"(nb), "+l"(mb));
    if (mb + kT2 <= sh.M && nb + kT2 <= sh.N && k0 + kTcBK <= k_end) {
#pragma unroll
      for (int e = 0; e < 16; ++e) {
        int r, k;
        tc_slot<kAKFast>(w, l, e, r, k);
        ra[e] = fa(mb + r, k0 + k);
        tc_slot<!kBNFast>(w, l, e, r, k);
        rb[e] = fb(k0 + k, nb + r);
      }
    } else {
#pragma unroll
      for (int e = 0; e < 16; ++e) {
        int r, k;
        tc_slot<kAKFast>(w, l, e, r, k);
        const long long m = mb + r, ka = k0 + k;
        ra[e] = (m < sh.M && ka < k_end) ? fa(m, ka) : 0.f;
        tc_slot<!kBNFast>(w, l, e, r, k);
        const long long kb = k0 + k;
        const int n = nb + r;
        rb[e] = (kb < k_end && n < sh.N) ? fb(kb, n) : 0.f;
      }
    }
  };
  auto stash = [&](int buf) {
    const uint32_t st = tc::smem_u32(sm + buf * kTcStage);
    int w = warp, l = lane;
    asm volatile("" : "+r"(w), "+r"(l));
    const uint32_t base_a = tc_stage_base<kAKFast>(w, l), base_b = tc_stage_base<!kBNFast>(w, l);
#pragma unroll
    for (int e = 0; e < 16; ++e) {
      uint32_t off = tc_stage_off<kAKFast>(base_a, e);
      float big = tc::round_tf32(ra[e]);
      st_shared(st + off, big);
      st_shared(st + kTcImage + off, tc::round_tf32(ra[e] - big));
      off = tc_stage_off<!kBNFast>(base_b, e);       // B is stored as its transpose: row n, K-major
      big = tc::round_tf32(rb[e]);
      st_shared(st + 2 * kTcImage + off, big);
      st_shared(st + 3 * kTcImage + off, tc::round_tf32(rb[e] - big));
    }
  };
  // Pipeline: block k+1 sits in registers while block k's MMAs run; it is stored into the other stage under
  // them, and the loads of block k+2 are issued at once, so they have a whole iteration to arrive.
  int buf = 0;
  if (k_begin < k_end) {
    fetch(k_begin);
    stash(0);
    if (k_begin + kTcBK < k_end) fetch(k_begin + kTcBK);
  }
  tc::fence_proxy_async();                            // generic-proxy stores -> wgmma (async proxy) reads
  __syncthreads();
  for (long long k0 = k_begin; k0 < k_end; k0 += kTcBK) {
    const bool more = k0 + kTcBK < k_end;
    const uint32_t st = tc::smem_u32(sm + buf * kTcStage);
    const uint32_t a_big = st + wg * 64 * tc::kRowBytes, a_small = a_big + kTcImage;
    const uint32_t b_big = st + 2 * kTcImage, b_small = b_big + kTcImage;
    tc::wg_fence();
    tf32_chain(part, a_small, b_big, true);
    tf32_chain(part, a_big, b_small);
    tf32_chain(part, a_big, b_big);
    tc::wg_commit();
    if (more) {
      stash(buf ^ 1);                                 // the other stage: its MMAs were waited for below
      if (k0 + 2 * kTcBK < k_end) fetch(k0 + 2 * kTcBK);
    }
    tc::wg_wait<0>();
    tc::wg_fence_regs<64>(part);
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] += part[i];
    if (more) {
      tc::fence_proxy_async();
      __syncthreads();
      buf ^= 1;
    }
  }
  // accumulator fragment (nfb_selftest_gemm): element i of this thread is row 16 warp + lane / 4 + 8 ((i >> 1) & 1)
  // of its warpgroup's 64, column 8 (i >> 2) + 2 (lane & 3) + (i & 1)
  const long long mrow = m0 + wg * 64 + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const long long m = mrow + 8 * ((i >> 1) & 1);
    const int n = n0 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
    if (m < sh.M && n < sh.N) fc(m, n, acc[i]);
  }
}

}  // namespace train
}  // namespace nfb
