// mbarrier / bulk-copy / wgmma primitives (inline PTX, sm_90a) and the
// shared-memory operand format used by the tensor-core field kernel.
//
// Operand format ("K-major, 128-byte swizzle", the GMMA canonical layout
// Swizzle<3,4,3> o ((8,m),(8,2)) of 16-byte units): an operand with R rows and
// K columns of bf16 / fp16 is cut into K-blocks of 64 columns.  One K-block is R
// rows of 128 bytes; inside each row the eight 16-byte chunks are XOR-permuted with
// (row & 7).  Blocks start on 1024-byte boundaries, 8-row groups are 1024 bytes
// apart (the descriptor's stride byte offset).  One wgmma consumes K=16 (32 bytes
// of every row), so stepping K inside a block adds 32 bytes to the descriptor's
// start address.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

namespace nfb {
namespace tc {

constexpr int kBlockK = 64;              // bf16 columns per 128-byte swizzle row
constexpr int kRowBytes = 128;
constexpr int kTileRows = 128;           // rows of one A operand / accumulator
constexpr int kABlockBytes = kTileRows * kRowBytes;   // 16 KB

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}

// Byte offset of logical 16-byte chunk `chunk` (0..7) of row `row` in a K-block.
__device__ __host__ __forceinline__ uint32_t swz_off(int row, int chunk) {
  return (uint32_t)(row * kRowBytes + ((chunk ^ (row & 7)) << 4));
}

// Warp-uniform leader election (elect.sync): control flow stays uniform for the whole warp.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .b32 rx;\n\t.reg .pred px;\n\t"
      "elect.sync rx|px, %1;\n\t"
      "selp.u32 %0, 1, 0, px;\n\t}"
      : "=r"(pred)
      : "r"(0xffffffffu));
  return pred != 0;
}
// ---- mbarrier ----------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
// Host-visible abort flag: a mapped pinned int (one per process, set up by
// ensure_abort_flag() in nfb_api.cu).  Nonzero = some mbarrier wait timed out.
__device__ int* g_nfb_abort = nullptr;

// Waits for the completion of the phase with the given parity.  A wait that
// spins "forever" (a protocol bug, not a condition that can occur in a correct
// run) does not hang the GPU: after 2^22 probes (tens of milliseconds at least; a
// legitimate wait is over within microseconds) the thread raises the host-visible
// abort flag, marks itself `dead` and returns; a dead thread returns from every
// later wait at once.  All roles of a CTA wait concurrently, so their time-outs
// expire together and the kernel drains; the host API then reports the error.
// Deliberately no __trap()/printf here: trap exits inside the consumer warpgroups keep
// ptxas from allocating the registers that setmaxnreg.inc hands to them.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, uint32_t& dead) {
  if (dead) return;
  const uint32_t addr = smem_u32(bar);
  uint32_t done;
  constexpr uint32_t kWaitProbes = 1u << 22;
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .u32 n;\n\t"
      "mov.u32 n, 0;\n"
      "NFB_W: mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "@p bra NFB_D;\n\t"
      "add.u32 n, n, 1;\n\t"
      "setp.ne.u32 p, n, %3;\n\t"
      "@p bra NFB_W;\n\t"
      "setp.eq.u32 p, n, 0;\n"
      "NFB_D: selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(done)
      : "r"(addr), "r"(parity), "r"(kWaitProbes)
      : "memory");
  if (!done) {                       // time-out: raise the abort flag, give up for good
    volatile int* ab = g_nfb_abort;
    if (ab) *ab = 1;
    dead = 1;
  }
}
// ---- bulk async copy (TMA engine, 1-D) -----------------------------------------
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes,
                                         uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_u32(smem_dst)),
      "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---- wgmma (warpgroup MMA, sm_90a) ----------------------------------------------
// Shared-memory matrix descriptor: K-major, SWIZZLE_128B, 8-row groups 1024 B apart
// (GMMA descriptor: start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), layout [62,64) = 1).
__device__ __forceinline__ uint64_t make_wg_desc(uint32_t saddr) {
  uint64_t d = (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;            // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;  // stride byte offset
  d |= (uint64_t)1 << 62;            // SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Keeps the compiler from moving accumulator reads across a wgmma wait.
template <int N>
__device__ __forceinline__ void wg_fence_regs(float* d) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define NFB_WG_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), \
                     "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
// D(64 x 16, fp32 registers) (+)= A(64 x 16, smem) * B(16 x 16, smem)^T
template <bool kBf16>
__device__ __forceinline__ void wg_mma_n16(float* d, uint64_t a, uint64_t b, uint32_t accumulate) {
  if constexpr (kBf16)
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
                 : NFB_WG_D8(0) : "l"(a), "l"(b), "r"(accumulate));
  else
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
                 : NFB_WG_D8(0) : "l"(a), "l"(b), "r"(accumulate));
}
#define NFB_WG_N128_REGS                                                                            \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "                        \
  "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "                \
  "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "                \
  "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
#define NFB_WG_N128_OPS                                                                              \
  : NFB_WG_D8(0), NFB_WG_D8(8), NFB_WG_D8(16), NFB_WG_D8(24), NFB_WG_D8(32), NFB_WG_D8(40),          \
    NFB_WG_D8(48), NFB_WG_D8(56)                                                                     \
  : "l"(a), "l"(b), "r"(accumulate)
// D(64 x 128, fp32 registers) (+)= A(64 x 16, smem) * B(128 x 16, smem)^T
template <bool kBf16>
__device__ __forceinline__ void wg_mma_n128(float* d, uint64_t a, uint64_t b, uint32_t accumulate) {
  if constexpr (kBf16)
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " NFB_WG_N128_REGS NFB_WG_N128_OPS);
  else
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " NFB_WG_N128_REGS NFB_WG_N128_OPS);
}
// D (+)= A * B^T with the fp16 A operand (64 x 16) in registers: 4 x b32 per thread,
// a[0] = (row, k = 2 lq + {0,1}), a[1] = (row + 8, same k), a[2] / a[3] = the same at k + 8,
// row = 16 * warp + lane / 4.  That is the accumulator fragment layout of columns
// 8j + 2lq + {0,1}, j = 0, 1: see x3_lo_reg.
// Always accumulates (it is never the first product of a K-block).
__device__ __forceinline__ void wg_mma_n16_rs(float* d, const uint32_t* a, uint64_t b) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
               "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, 0;\n\t}"
               : NFB_WG_D8(0) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(1u));
}
__device__ __forceinline__ void wg_mma_n128_rs(float* d, const uint32_t* a, uint64_t b) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
               "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
               "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
               "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
               "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
               "{%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
               : NFB_WG_D8(0), NFB_WG_D8(8), NFB_WG_D8(16), NFB_WG_D8(24), NFB_WG_D8(32), NFB_WG_D8(40),
                 NFB_WG_D8(48), NFB_WG_D8(56)
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(1u));
}
// D(64 x 128, fp32 registers) (+)= A(64 x 8, smem) * B(128 x 8, smem)^T with tf32 operands (the
// top 19 bits of each fp32 word).  PTX allows no transpose for .tf32: both operands are K-major.  A
// 128-byte swizzle row holds 32 fp32 and one K step of 8 is 32 bytes, the same step as the k16
// forms above, so make_wg_desc and its +2 (16-byte units) per step apply unchanged.
__device__ __forceinline__ void wg_mma_n128_tf32(float* d, uint64_t a, uint64_t b, uint32_t accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
               "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
               "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
               "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
               "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
               "%64, %65, p, 1, 1;\n\t}" NFB_WG_N128_OPS);
}
// x rounded to tf32 (round to nearest, ties away; the low 13 bits of the result are zero).
__device__ __forceinline__ float round_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
#undef NFB_WG_N128_REGS
#undef NFB_WG_N128_OPS
#undef NFB_WG_D8

// fp16x3: index in a thread's register copy of a 64-row activation operand (uint32_t[16 per
// K-block], fp16 pairs) of the pair at row arow + 8h, columns 64 kb + 8j + 2lq + {0, 1}
// (j = 0..7) - the pair an accumulator fragment holds as elements 4j + 2h + {0, 1}.  Entries
// 16 kb + 4 ks .. + 3 are the register A operand of K step ks of K-block kb.
__host__ __device__ constexpr int x3_lo_reg(int kb, int j, int h) { return 16 * kb + 2 * j + h; }

// One K-block (64 columns = 4 K-steps) of a warpgroup's 64 rows against one weight
// unit.  bf16: x W.  fp16x3: per K step x_hi W_hi, x_hi W_lo, x_lo W_hi into the same
// accumulator.  a_hi / b_* are shared-memory byte addresses of the K-block images; a_lo
// is either that of the x_lo image (uint32_t) or this thread's 16 registers of x_lo
// (const uint32_t*, fp16x3 only, see x3_lo_reg).
template <bool kX3, int N, typename ALo>
__device__ __forceinline__ void wg_unit(float* d, uint32_t a_hi, ALo a_lo, uint32_t b_hi, uint32_t b_lo,
                                        uint32_t accumulate) {
  constexpr bool kLoRegs = !std::is_integral<ALo>::value;
  static_assert(kX3 || !kLoRegs, "register x_lo operand is fp16x3 only");
  const uint64_t ah = make_wg_desc(a_hi);
  const uint64_t bh = make_wg_desc(b_hi), bl = make_wg_desc(b_lo);
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    const uint64_t o = (uint64_t)(2 * ks);     // +32 bytes per K step, in 16-byte units
    const uint32_t acc = (accumulate || ks) ? 1u : 0u;
    if constexpr (N == 16) {
      wg_mma_n16<!kX3>(d, ah + o, bh + o, acc);
      if constexpr (kX3) {
        wg_mma_n16<false>(d, ah + o, bl + o, 1u);
        if constexpr (kLoRegs) wg_mma_n16_rs(d, a_lo + 4 * ks, bh + o);
        else wg_mma_n16<false>(d, make_wg_desc(a_lo) + o, bh + o, 1u);
      }
    } else {
      wg_mma_n128<!kX3>(d, ah + o, bh + o, acc);
      if constexpr (kX3) {
        wg_mma_n128<false>(d, ah + o, bl + o, 1u);
        if constexpr (kLoRegs) wg_mma_n128_rs(d, a_lo + 4 * ks, bh + o);
        else wg_mma_n128<false>(d, make_wg_desc(a_lo) + o, bh + o, 1u);
      }
    }
  }
}

// ---- bf16 helpers ---------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
// Stores 8 consecutive K-columns (one 16-byte chunk) of `row` into a K-block.
__device__ __forceinline__ void store_chunk(uint8_t* block, int row, int chunk, const float* v) {
  uint4 q;
  q.x = pack_bf16x2(v[0], v[1]);
  q.y = pack_bf16x2(v[2], v[3]);
  q.z = pack_bf16x2(v[4], v[5]);
  q.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(block + swz_off(row, chunk)) = q;
}

// Weight packing (global memory image of the shared-memory operand): the
// (in,out) fp32 kernel W[k][n] of a Dense layer becomes, per K-block kb, a
// contiguous unit of `n_rows` rows x 128 bytes holding W^T (row n, column k),
// chunk-swizzled, zero-padded in K and N.  `k_map` lists for each of the nkb*64
// packed K columns the source row of W (or -1 for padding), which is how the
// skip concat [x, inputs] and the 64-column padding of the input block are laid
// out.
__global__ void pack_weight_kernel(const float* __restrict__ w_packed_fp32, int ld,
                                   const int* __restrict__ k_map, int nkb, int n, int n_rows,
                                   __nv_bfloat16* __restrict__ dst) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)nkb * n_rows * kBlockK;
  if (idx >= total) return;
  const int kk = (int)(idx % kBlockK);
  const int row = (int)((idx / kBlockK) % n_rows);
  const int kb = (int)(idx / ((long long)kBlockK * n_rows));
  const int src_k = k_map[kb * kBlockK + kk];
  float v = 0.f;
  if (src_k >= 0 && row < n) v = w_packed_fp32[(size_t)src_k * ld + row];
  uint8_t* unit = reinterpret_cast<uint8_t*>(dst) + (size_t)kb * n_rows * kRowBytes;
  *reinterpret_cast<__nv_bfloat16*>(unit + swz_off(row, kk >> 3) + (kk & 7) * 2) =
      __float2bfloat16_rn(v);
}

// fp16x3 mode: every layer's weights are multiplied by a power of two s so that
// max |W| s lies in [2, 4) before the fp16 hi/lo split, and the epilogue multiplies
// the accumulator by 1/s (exact).  Without it small weights (the warp heads are
// ~1e-3) push W_lo into fp16's subnormal range (absolute floor 2^-25) and the
// split loses up to 10 bits; with it the split error is ~3e-7 of the layer output.
__host__ __device__ __forceinline__ float x3_weight_scale(float absmax) {
  if (!(absmax > 0.f) || !(absmax < 3.0e38f)) return 1.f;
  int e = 0;
  frexpf(absmax, &e);                      // absmax = f * 2^e, f in [0.5, 1)
  e = 2 - e;
  e = e < -100 ? -100 : (e > 100 ? 100 : e);
  return ldexpf(1.f, e);
}
// max |w| over a float range (one slot per layer; non-negative floats order like uints).
__global__ void absmax_kernel(const float* __restrict__ w, long long n, float* __restrict__ out) {
  float m = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    m = fmaxf(m, fabsf(w[i]));
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<unsigned int*>(out), __float_as_uint(m));
}

// fp16x3 mode: fp32 (K x N, row-major, leading dimension ld) -> fp16 hi and lo units,
// hi = rn(w), lo = rn(w - hi), interleaved per K-block: unit (kb, part) at
// ((kb * 2 + part) * n_rows) rows x 128 bytes.
__global__ void pack_weight_x3_kernel(const float* __restrict__ w, int ld, const int* __restrict__ k_map,
                                      int nkb, int n, int n_rows, const float* __restrict__ absmax,
                                      uint8_t* __restrict__ dst) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)nkb * n_rows * kBlockK;
  if (idx >= total) return;
  const int kk = (int)(idx % kBlockK);
  const int row = (int)((idx / kBlockK) % n_rows);
  const int kb = (int)(idx / ((long long)kBlockK * n_rows));
  const int src_k = k_map[kb * kBlockK + kk];
  float v = 0.f;
  if (src_k >= 0 && row < n) v = w[(size_t)src_k * ld + row] * x3_weight_scale(*absmax);
  const __half hi = __float2half_rn(v);
  const __half lo = __float2half_rn(v - __half2float(hi));
  uint8_t* unit = dst + (size_t)kb * 2 * n_rows * kRowBytes;
  const uint32_t off = swz_off(row, kk >> 3) + (kk & 7) * 2;
  *reinterpret_cast<__half*>(unit + off) = hi;
  *reinterpret_cast<__half*>(unit + (size_t)n_rows * kRowBytes + off) = lo;
}

}  // namespace tc
}  // namespace nfb
