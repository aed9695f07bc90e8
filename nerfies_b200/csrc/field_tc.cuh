// Fused per-sample field evaluation on the Hopper tensor cores (wgmma) for the two
// tensor-core precisions: bf16 (NFB_PREC_BF16: bf16 operands, fp32 accumulation) and
// fp16x3 (NFB_PREC_FP16X3: three fp16 chains per layer, see field_tc3.cuh).  Every Dense
// layer of the warp MLP and the NeRF MLP is a chain of wgmma over 64-column K-blocks:
//   A = the tile's activations (or the encoded-input block) in shared memory, in the
//       GMMA K-major 128B-swizzle format, written in place by the epilogue;
//   B = pre-swizzled weight units streamed from L2 by cp.async.bulk through an
//       mbarrier ring, each unit used by both consumer warpgroups;
//   D = fp32 accumulators in registers.
// Activations never leave the SM; per sample 16 B (r,g,b,sigma) go to HBM, or with the
// fused composite 24 B per ray.
#pragma once
#include "field_simt.cuh"   // FieldArgs
#include "field_tc3.cuh"
#include "nfb_handle.h"
#include "tc_common.cuh"
#include "tc_program.cuh"

namespace nfb {
namespace tc {

// bf16 mode: the encoded features are rounded to bf16 (rel. 4e-3) before they
// reach the tensor cores, so the octave recurrence
//   sin 2a = 2 sin a cos a,  cos 2a = 1 - 2 sin^2 a
// (error doubles per octave: < 1e-4 at 2^9) replaces 6F libm calls by 3 sincosf.
__device__ __forceinline__ void posenc_fast_to_block(uint8_t* block, int r, const float* x, int F,
                                                  const float* __restrict__ window,
                                                  const float* __restrict__ extra, int n_extra,
                                                  int c_begin = 0, int c_end = 8) {
  float feat[64];
#pragma unroll
  for (int k = 0; k < 64; ++k) feat[k] = 0.f;
  float sn[3], cs[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    feat[c] = x[c];
    sincosf(x[c], &sn[c], &cs[c]);
  }
#pragma unroll
  for (int f = 0; f < 10; ++f) {
    if (f < F) {
      const float w = window ? __ldg(window + f) : 1.f;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        feat[3 + f * 6 + c] = w * sn[c];
        feat[3 + f * 6 + 3 + c] = w * cs[c];
        const float s2 = 2.f * sn[c] * cs[c];
        const float c2 = 1.f - 2.f * sn[c] * sn[c];
        sn[c] = s2; cs[c] = c2;
      }
    }
  }
  const int d = 3 + 6 * F;
#pragma unroll
  for (int k = 0; k < 64; ++k) {
    // `extra` (GLO code) sits right after the encoding; k is compile-time, d is not.
    if (k >= d && k < d + n_extra) feat[k] = __ldg(extra + (k - d));
  }
#pragma unroll
  for (int c = 0; c < 8; ++c)
    if (c >= c_begin && c < c_end) store_chunk(block, r, c, feat + c * 8);
}
// This thread's half `hs` (32 columns) of row r of the input block, [x | window * posenc(x) | extra | 0...],
// in the kernel's precision: fp16 hi / lo images (kX3) or bf16.  Inlined: a call with a literal null `extra`
// and n_extra = 0 carries no extra-column code (register pressure).  The lo image follows the hi
// image at kBlkBytes.
template <bool kX3, uint32_t kBlkBytes>
__device__ __forceinline__ void encode_input(uint8_t* in_block, int r, int hs, const float* x, int F,
                                             const float* __restrict__ window,
                                             const float* __restrict__ extra, int n_extra) {
  if constexpr (kX3) {
    if (hs == 0) tc3::posenc_block_x3<0>(in_block, in_block + kBlkBytes, r, x, F, window, extra, n_extra);
    else tc3::posenc_block_x3<1>(in_block, in_block + kBlkBytes, r, x, F, window, extra, n_extra);
  } else {
    posenc_fast_to_block(in_block, r, x, F, window, extra, n_extra, 4 * hs, 4 * hs + 4);
  }
}

// One 128-column accumulator chunk of a hidden layer (this thread's fragment: rows
// arow, arow + 8; columns c*128 + 8j + 2*lq + {0, 1}) -> + bias, activation, (alpha
// head dot product in fp32) -> the activation image of the next layer, in place; in
// fp16x3 the lo half goes to this thread's register operand `lo` (x3_lo_reg) instead.
// `inv_s` undoes the fp16x3 power-of-two weight scale (x3_weight_scale; 1 in bf16
// mode): acc * inv_s is exact, so fma(acc, inv_s, bias) rounds like acc + bias.
// fp16x3 split: hi = v with the fp32 mantissa truncated to fp16's 11 significant bits
// (the conversion is then exact), lo = fp16(v - hi) (exact subtraction):
// v - (hi + lo) <= 2^-23 |v|, the bound of a round-to-nearest split.  ReLU rides on the
// conversions: for v < 0 both hi and v - hi are <= 0 and convert to +0.  Conversions
// saturate: |v| > 65504 does not become inf.  kBlkBytes: bytes of one K-block of the tile's
// activation image (128 or 256 rows).  kRows: bit h set = write row arow + 8h (a layer whose two rows
// take different biases runs one call per row, so only one bias pointer is live at a time).
template <bool kX3, uint32_t kBlkBytes, int kRows = 3>
__device__ __forceinline__ void epi_chunk(const float* acc, int c, const float* __restrict__ bias, float inv_s,
                                          bool relu, bool adot, const float* __restrict__ aw, float& al0,
                                          float& al1, uint8_t* act_hi, uint32_t* lo, int arow, int lq) {
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int col = c * 128 + 8 * j + 2 * lq;
    const float2 b = __ldg(reinterpret_cast<const float2*>(bias + col));
    float v[4] = {fmaf(acc[4 * j], inv_s, b.x), fmaf(acc[4 * j + 1], inv_s, b.y),
                  fmaf(acc[4 * j + 2], inv_s, b.x), fmaf(acc[4 * j + 3], inv_s, b.y)};
    if (adot) {
      // bf16 mode: bf16-rounded alpha weights, fp32 activations and accumulation
      float2 w = __ldg(reinterpret_cast<const float2*>(aw + col));
      if constexpr (!kX3) w = __bfloat1622float2(__floats2bfloat162_rn(w.x, w.y));
      al0 = fmaf(relu ? fmaxf(v[0], 0.f) : v[0], w.x, al0);
      al0 = fmaf(relu ? fmaxf(v[1], 0.f) : v[1], w.y, al0);
      al1 = fmaf(relu ? fmaxf(v[2], 0.f) : v[2], w.x, al1);
      al1 = fmaf(relu ? fmaxf(v[3], 0.f) : v[3], w.y, al1);
    }
    const uint32_t blk = (uint32_t)(2 * c + (j >> 3)) * kBlkBytes + 4 * lq;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!((kRows >> h) & 1)) continue;
      const uint32_t off = blk + swz_off(arow + 8 * h, j & 7);
      const float a = v[2 * h], bb = v[2 * h + 1];
      uint32_t hi;
      if constexpr (kX3) {
        const float ta = __uint_as_float(__float_as_uint(a) & 0xFFFFE000u);
        const float tb = __uint_as_float(__float_as_uint(bb) & 0xFFFFE000u);
        const float da = a - ta, db = bb - tb;
        uint32_t& l = lo[x3_lo_reg(2 * c + (j >> 3), j & 7, h)];
        if (relu) {
          asm("cvt.rn.relu.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(tb), "f"(ta));
          asm("cvt.rn.relu.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(l) : "f"(db), "f"(da));
        } else {
          asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(tb), "f"(ta));
          asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(l) : "f"(db), "f"(da));
        }
      } else {
        if (relu) asm("cvt.rn.relu.bf16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(bb), "f"(a));
        else asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(bb), "f"(a));
      }
      *reinterpret_cast<uint32_t*>(act_hi + off) = hi;
    }
  }
}

// bf16: the rgb condition into chunks [c_begin, c_end) of row r of the input block.
__device__ __forceinline__ void cond_to_block(uint8_t* block, int r, const float* __restrict__ cond,
                                              int n, int c_begin, int c_end) {
#pragma unroll 1
  for (int c = c_begin; c < c_end; ++c) {
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = c * 8 + j;
      v[j] = k < n ? __ldg(cond + k) : 0.f;
    }
    store_chunk(block, r, c, v);
  }
}

// bf16: the per-ray part of the alpha head with an alpha condition, cond . w with bf16-rounded weights.
// Out of line: it runs once per row and tile, and inlined it costs the hot loop registers.
__device__ __noinline__ float alpha_cond_dot(const float* __restrict__ cond, const float* __restrict__ w, int n) {
  float a = 0.f;
  for (int j = 0; j < n; ++j) a = fmaf(__ldg(cond + j), __bfloat162float(__float2bfloat16_rn(__ldg(w + j))), a);
  return a;
}

// Row state owned by the two row threads of a row for the lifetime of a tile.
struct RowState {
  float x[3];        // current (possibly warped) sample point
  long long m;       // global row (clamped to a valid row)
  long long ray;
  bool valid;
  float z, dist;     // fused composite: z of the sample, (z_next - z) * |d| (or the last-sample constant)
  bool last;         // last sample of its ray
};

// Fused per-sample field evaluation on the Hopper tensor cores (wgmma), one kernel for
// both tensor-core precisions (kX3: fp16x3, else bf16).
//
// A launch runs one of the program's two nets (TcProgram::n_warp): the warp pass (FieldArgs::
// warp_only) evaluates the warp MLP and the SE(3) / translation tail and writes the warped
// points; the NeRF pass reads them (FieldArgs::points), or forms o + z d without a warp.
//
// Persistent, one CTA per SM, 384 threads, one tile of 128 kMB rows at a time:
//   warpgroup 0     : warp 0 streams the weight units (one cp.async.bulk per unit into a
//                     ring of mbarrier-guarded slots: 32 KB fp16x3 [W_hi | W_lo], 16 KB
//                     bf16); the other warps idle (setmaxnreg 24 / 240).
//   kMB = 2         : (warp pass of a warp MLP no wider than 128) each consumer warpgroup
//                     owns two 64-row blocks, rows 128 cw + {0..63, 64..127}, with one
//                     accumulator set (acc0 / acc1) and 32 x_lo registers per block; every
//                     unit issues block 0's chain, then block 1's, so a row sees the same
//                     products in the same order as at kMB = 1, and each weight unit feeds
//                     256 rows.  One row thread per row.  Below, the kMB = 1 kernel:
//   warpgroups 1, 2 : rows 0-63 / 64-127.  Each issues its own wgmma (M = 64, N = 128 per
//                     chunk, fp32 accumulators in registers: a 256-wide layer is 128 of them
//                     per thread), A = its rows of the activation image in shared memory,
//                     B = the weight slot shared by both.  A layer's epilogue writes the
//                     next layer's activation image in place once the warpgroup's MMAs of
//                     the layer are complete, so no second image is needed.  fp16x3: the
//                     x_lo operand of the activations is not in shared memory but in the
//                     registers of the thread whose accumulators produced it (64 per thread,
//                     epi_chunk -> lo -> the register-A form of wgmma), under the same rule.
// Shared memory (225 KB), in 16 KB units; the activation image is 64 KB at both kMB (4 K-blocks
// of 128 rows or 2 of 256), an input-block K-block is 128 kMB rows:
//   fp16x3 kMB = 1: activation image hi 64 KB | input block (the encoded points / conditions)
//                   hi | lo, 32 KB | weight ring 4 x 32 KB;
//   fp16x3 kMB = 2: activation image hi 64 KB | input block hi | lo, 64 KB (the skip layer reads
//                   it again, so it stays resident) | weight ring 3 x 32 KB;
//   bf16   kMB = 1: activation image 64 KB | 64 KB unused | input block 32 KB (its lo half
//                   unused) | weight ring 4 x 16 KB;
//   bf16   kMB = 2: activation image 64 KB | 32 KB unused | input block 64 KB (lo unused) |
//                   weight ring 4 x 16 KB;
// then for all alpha partials | composite scratch | barriers.  The weight units are 128-column
// N-chunks at both kMB, so a 256-row fp16x3 tile keeps 32 KB slots and drops to three of them.
// Per-row work (positional encodings, SE(3) exp-map, sigmoid / sigma activation, fused
// volumetric rendering) is done by "row threads".  kMB = 1: two per row (hs = which half of the
// input block's columns), thread t of warpgroup w owns row 64 (w - 1) + (t & 63); kMB = 2: one
// per row, thread t owns row 128 (w - 1) + t and writes both halves.
// Head layers (N = 16) leave their accumulators in a per-warpgroup scratch inside
// activation block 0 (free at that point: the step after a head reads the input block only).
constexpr int kWgThreads = 384;
constexpr int kAlphaOff = 14 * kABlockBytes;          // per-row alpha-head partial (128 floats)
constexpr int kScanOff = kAlphaOff + 512;             // fused composite: cross-warp partials (40 floats)
constexpr int kRayOff = kScanOff + 256;               // NeRF pass: each row's ray (128 ints, TcStep::ray_bias)
constexpr int kBarOff = kRayOff + 512;
constexpr int kWgSmemBytes = kBarOff + 256;
template <bool kX3, int kMB>
struct WgSmem {
  static constexpr int kRows = kMB * kTileRows;                 // rows of a tile
  static constexpr uint32_t kBlkBytes = kRows * kRowBytes;      // one K-block of the tile
  static constexpr int kSlots = (kX3 && kMB == 2) ? 3 : 4;
  static constexpr int kSlotBytes = (kX3 ? 2 : 1) * kABlockBytes;
  static constexpr int kRingOff = kAlphaOff - kSlots * kSlotBytes;   // the ring ends at the alpha partials
  static constexpr int kInOff = kRingOff - 2 * (int)kBlkBytes;
  static_assert(kInOff >= 4 * kABlockBytes, "input block overlaps the activation image");
};
static_assert(kWgSmemBytes <= 232448, "shared memory");

// One weight unit of a layer into the accumulators d, A = K-block `src` (an activation
// block or kSrcIn).  fp16x3 takes x_lo of an activation block from the registers `lo`, that
// of the input block (written by the row threads) from its shared image at in_lo; the switch
// keeps every register index a compile-time constant.  kActKb: K-blocks of the activation image
// (4, or 2 in a 256-row tile, whose `lo` holds 32 registers per row block).
template <bool kX3, int N, int kActKb>
__device__ __forceinline__ void wg_layer_unit(float* d, int src, uint32_t a_hi, uint32_t in_lo, const uint32_t* lo,
                                              uint32_t b_hi, uint32_t b_lo, uint32_t accumulate) {
  if constexpr (kX3) {
    switch (src) {
      case 0: wg_unit<true, N>(d, a_hi, lo + x3_lo_reg(0, 0, 0), b_hi, b_lo, accumulate); break;
      case 1: wg_unit<true, N>(d, a_hi, lo + x3_lo_reg(1, 0, 0), b_hi, b_lo, accumulate); break;
      case 2:
        if constexpr (kActKb > 2) wg_unit<true, N>(d, a_hi, lo + x3_lo_reg(2, 0, 0), b_hi, b_lo, accumulate);
        break;
      case 3:
        if constexpr (kActKb > 2) wg_unit<true, N>(d, a_hi, lo + x3_lo_reg(3, 0, 0), b_hi, b_lo, accumulate);
        break;
      default: wg_unit<true, N>(d, a_hi, in_lo, b_hi, b_lo, accumulate); break;
    }
  } else {
    wg_unit<false, N>(d, a_hi, 0u, b_hi, b_lo, accumulate);
  }
}

struct WgBars {
  uint64_t full[4];
  uint64_t empty[4];       // 8 arrivals: every consumer warp, after its wgmma reading the slot completed
  uint64_t never;          // never completes: the abort-path test hook waits on it
};

template <bool kX3, int kMB>
__global__ void __launch_bounds__(kWgThreads, 1)
field_wg_kernel(const __grid_constant__ TcProgram prog, const FieldArgs args, const uint8_t* __restrict__ wpack,
                const float* __restrict__ aux, int num_tiles) {
  static_assert(kMB == 1 || kMB == 2, "one or two 64-row blocks per consumer warpgroup");
  using Smem = WgSmem<kX3, kMB>;
  constexpr int kSlots = Smem::kSlots, kSlotBytes = Smem::kSlotBytes, kRows = Smem::kRows;
  constexpr uint32_t kBlk = Smem::kBlkBytes;
  constexpr int kActKb = 4 / kMB;                 // K-blocks of the activation image
  // Registers per thread: 128 * producer + 256 * consumer <= 64 K.  fp16x3 consumers hold 64
  // x_lo registers on top of a 256-wide layer's 128 accumulators.
  constexpr int kProducerRegs = kX3 ? 24 : 40, kConsumerRegs = kX3 ? 240 : 232;
  // A consumer warp frees the slot of unit u-1 after issuing unit u, so the MMAs of u-1 and u
  // overlap; with four slots the copies of u+1 .. u+3 can be in flight meanwhile.  (Freeing it
  // before waiting for unit u, which drains the MMA pipeline on every unit, measured slower in
  // both precisions: DESIGN 5.1.)
  extern __shared__ __align__(1024) uint8_t base[];
  if ((smem_u32(base) & 1023u) != 0) {
    if (threadIdx.x == 0) printf("nfb: dynamic shared memory is not 1024-byte aligned\n");
    __trap();
  }
  WgBars* bars = reinterpret_cast<WgBars*>(base + kBarOff);
  const int tid = threadIdx.x, wg = tid >> 7, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    for (int i = 0; i < kSlots; ++i) { mbar_init(&bars->full[i], 1); mbar_init(&bars->empty[i], 8); }
    mbar_init(&bars->never, 1);
    fence_barrier_init();
  }
  __syncthreads();
  // the warp pass runs steps [0, n_warp), the NeRF pass the rest (build_tc_program)
  const bool warp_pass = args.warp_only != 0;
  const int first_step = warp_pass ? 0 : prog.n_warp, end_step = warp_pass ? prog.n_warp : prog.n_steps;
  // Tiles of this CTA: blockIdx.x, + gridDim.x, ...  With the fused composite a CTA takes whole
  // rays - the S / 128 tiles of a ray back to back - so that transmittance and the partial sums
  // are carried in registers from tile to tile.
  const bool fuse = kMB == 1 && args.ray_out != nullptr && !warp_pass;
  const int tpr = fuse ? args.samples_per_ray / kTileRows : 1;          // tiles per group
  const int groups = num_tiles / tpr;
  const int bid = (int)blockIdx.x;
  const int my_groups = bid < groups ? (groups - bid + (int)gridDim.x - 1) / (int)gridDim.x : 0;
  const int n_my = my_groups * tpr;
  auto tile_of = [&](int i) { return (bid + (i / tpr) * (int)gridDim.x) * tpr + (i % tpr); };

  if (wg == 0) {
    // ===================== weight producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
    if (warp == 0) {
      uint32_t sg = 0, ph = 0, dead = 0;
      if (args.debug & kDebugTimeout) mbar_wait(&bars->never, 0, dead);   // test hook: provoke a wait time-out
      uint8_t* ring = base + Smem::kRingOff;
      for (int ti = 0; ti < n_my; ++ti) {
        for (int si = first_step; si < end_step; ++si) {
          const TcStep& st = prog.steps[si];
          const uint32_t bytes = (kX3 ? 2u : 1u) * (uint32_t)st.chunk_n * kRowBytes;
          const uint8_t* src = wpack + st.w_off;
          const int n = st.n_chunks * st.nkb;
          for (int u = 0; u < n; ++u) {
            mbar_wait(&bars->empty[sg], ph ^ 1, dead);
            if (!dead && elect_one()) {
              mbar_arrive_expect_tx(&bars->full[sg], bytes);
              bulk_g2s(ring + sg * kSlotBytes, src + (size_t)u * bytes, bytes, &bars->full[sg]);
            }
            __syncwarp();
            if (++sg == kSlots) { sg = 0; ph ^= 1; }
          }
        }
      }
    }
  } else {
    // ===================== consumers: MMAs + epilogue of 64 kMB rows =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
    constexpr int kWgRows = 64 * kMB;                    // rows of a consumer warpgroup
    const int cw = wg - 1, t = tid & 127, wq = t >> 5, lq = lane & 3;
    // accumulator rows arow, arow + 8 of block 0; block b adds 64 b
    const int arow = kWgRows * cw + 16 * wq + (lane >> 2);
    // row thread: row r, input-block halves [h0, h1)
    const int lr = kMB == 2 ? t : (t & 63);              // row within the warpgroup
    const int r = kWgRows * cw + lr;
    const int h0 = kMB == 2 ? 0 : t >> 6, h1 = kMB == 2 ? 2 : h0 + 1;
    uint8_t* act_hi = base;
    uint8_t* inh = base + Smem::kInOff;
    float* alpha_s = reinterpret_cast<float*>(base + kAlphaOff);
    float* scan_s = reinterpret_cast<float*>(base + kScanOff);
    int* ray_s = reinterpret_cast<int*>(base + kRayOff);
    const uint32_t rows_off = (uint32_t)(kWgRows * cw * kRowBytes); // this warpgroup's rows in a K-block
    // head accumulators, kWgRows x 16 floats over this warpgroup's own rows of activation block 0
    // (the other warpgroup's MMAs may still read its rows)
    float* scr = reinterpret_cast<float*>(base + rows_off);
    const uint32_t ring_a = smem_u32(base + Smem::kRingOff);
    const uint32_t act_a = smem_u32(act_hi) + rows_off, in_a = smem_u32(inh) + rows_off;
    // fp16x3: x_lo of the activation image of this thread's accumulator rows, see epi_chunk
    // (kMB = 2: lo[32 b ..] for block b)
    uint32_t lo[kX3 ? 64 : 1];
    const float alpha_b = __ldg(aux + prog.alpha_b_off);
    const int S = args.samples_per_ray;
    uint32_t sg = 0, ph = 0, dead = 0;
    auto wg_sync = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory"); };
    RowState row;

    // Row state of tile `tile` (model_utils.py:72-73) and this thread's half of its first
    // input block (warping.py:325-326 / models.py:270).  With FieldArgs::points the row's point
    // is the given (already warped) one and the NeRF net's inputs come first.
    auto begin_tile = [&](int tile) {
      long long m = (long long)tile * kRows + r;
      row.valid = m < args.num_rows;
      if (!row.valid) m = args.num_rows - 1;
      row.m = m;
      row.ray = m / S;
      if (!warp_pass && h0 == 0) ray_s[r] = (int)row.ray;   // read by the ray_bias epilogue
      const float z = args.z_vals ? __ldg(args.z_vals + m) : 0.f;
      float org[3], dir[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        dir[c] = __ldg(args.directions + row.ray * 3 + c);
        org[c] = __ldg(args.origins + row.ray * 3 + c);
      }
      if (args.points) {
#pragma unroll
        for (int c = 0; c < 3; ++c) row.x[c] = __ldg(args.points + m * 3 + c);
      } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) row.x[c] = org[c] + z * dir[c];
      }
      if (fuse) {
        // dists of volumetric_rendering (model_utils.py:98-104)
        row.z = z;
        row.last = m + 1 == (row.ray + 1) * S;
        const float zn = (!row.last && args.z_vals) ? __ldg(args.z_vals + m + 1) : 0.f;
        const float dnorm = sqrtf(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]);
        const float d = row.last ? (args.sample_at_infinity ? 1e10f : 1e-19f) : (zn - z);
        row.dist = d * dnorm;
      }
      if (!warp_pass && args.warped && row.valid && h0 == 0) {
#pragma unroll
        for (int c = 0; c < 3; ++c) args.warped[m * 3 + c] = row.x[c];
      }
      const float* cond = args.cond + row.ray * prog.cond_stride;
      // warp net: [posenc | GLO code]; NeRF net: [posenc | trunk condition]
#pragma unroll
      for (int hs = h0; hs < h1; ++hs)
        encode_input<kX3, kBlk>(inh, r, hs, row.x, warp_pass ? prog.Fw : prog.Fp, warp_pass ? args.window : nullptr,
                                warp_pass ? cond : cond + prog.G, warp_pass ? prog.G : prog.tc);
    };

    // fused composite: running state of the ray this CTA is on (replicated in every row thread)
    float c_T = 1.f, c_cw = 0.f, a_r = 0.f, a_g = 0.f, a_b = 0.f, a_d = 0.f, a_w = 0.f, a_wnl = 0.f, a_med = 0.f;
    bool c_med = false;   // the ray's median sample has been found
    if (n_my > 0) begin_tile(tile_of(0));
    fence_proxy_async();
    wg_sync();
    for (int ti = 0; ti < n_my; ++ti) {
      const int tile = tile_of(ti);
      const bool has_next = ti + 1 < n_my;
      for (int si = first_step; si < end_step; ++si) {
        const TcStep& st = prog.steps[si];
        const float* bias = aux + st.b_off;
        const float inv_s = kX3 ? 1.f / x3_weight_scale(__ldg(aux + prog.scale_off + si)) : 1.f;
        const bool hidden = st.epi == kEpiHidden;
        // kMB = 1: acc0 / acc1 = N-chunk 0 / 1; kMB = 2: acc0 / acc1 = row block 0 / 1 (one N-chunk).
        // A head (N = 16) accumulates into acc0[0..7] (and acc1[0..7] for row block 1).
        float acc0[64], acc1[64];
        // ---- the layer's MMAs: one weight unit per (chunk, K-block), one unit in flight ----
        uint32_t prev_sg = 0;
        const int n_units = st.n_chunks * st.nkb;
        for (int u = 0; u < n_units; ++u) {
          const int c = u >= st.nkb ? 1 : 0, kb = u - c * st.nkb;
          const int src = st.src[kb];
          const uint32_t a_hi = src == kSrcIn ? in_a : act_a + (uint32_t)src * kBlk;
          const uint32_t b_hi = ring_a + sg * kSlotBytes, b_lo = b_hi + (uint32_t)st.chunk_n * kRowBytes;
          mbar_wait(&bars->full[sg], ph, dead);
          wg_fence();
          const uint32_t in_lo = in_a + kBlk;
          if constexpr (kMB == 1) {
            if (!hidden) wg_layer_unit<kX3, 16, kActKb>(acc0, src, a_hi, in_lo, lo, b_hi, b_lo, kb);
            else if (c == 0) wg_layer_unit<kX3, 128, kActKb>(acc0, src, a_hi, in_lo, lo, b_hi, b_lo, kb);
            else wg_layer_unit<kX3, 128, kActKb>(acc1, src, a_hi, in_lo, lo, b_hi, b_lo, kb);
          } else {
            // row block 1's rows are 64 rows (8 KB) after block 0's in every K-block
            if (!hidden) {
              wg_layer_unit<kX3, 16, kActKb>(acc0, src, a_hi, in_lo, lo, b_hi, b_lo, kb);
              wg_layer_unit<kX3, 16, kActKb>(acc1, src, a_hi + 8192u, in_lo + 8192u, lo + 32, b_hi, b_lo, kb);
            } else {
              wg_layer_unit<kX3, 128, kActKb>(acc0, src, a_hi, in_lo, lo, b_hi, b_lo, kb);
              wg_layer_unit<kX3, 128, kActKb>(acc1, src, a_hi + 8192u, in_lo + 8192u, lo + 32, b_hi, b_lo, kb);
            }
          }
          wg_commit();
          if (u > 0) {
            wg_wait<1>();
            if (lane == 0) mbar_arrive(&bars->empty[prev_sg]);
          }
          prev_sg = sg;
          if (++sg == kSlots) { sg = 0; ph ^= 1; }
        }
        wg_wait<0>();
        wg_fence_regs<64>(acc0); wg_fence_regs<64>(acc1);
        if (lane == 0) mbar_arrive(&bars->empty[prev_sg]);
        wg_sync();      // every MMA of the warpgroup is complete: its activation rows may be overwritten

        if (hidden) {
          // ---- hidden layer: the output overwrites the input in place ----
          const bool relu = st.relu != 0, adot = st.alpha_dot != 0;
          const float* aw = aux + prog.alpha_w_off;
          if constexpr (kMB == 1) {
            float al0 = 0.f, al1 = 0.f;
            if (kX3 && st.ray_bias) {
              // the bias of each accumulator row's own ray: a tile of the staged path with S % 128 != 0
              // spans rays (with the fused composite the tile is one ray)
              const int cols = 128 * st.n_chunks;
              const float* rb = args.ray_bias + (size_t)ray_s[arow] * cols;
              epi_chunk<kX3, kBlk, 1>(acc0, 0, rb, inv_s, relu, false, aw, al0, al1, act_hi, lo, arow, lq);
              if (st.n_chunks == 2) epi_chunk<kX3, kBlk, 1>(acc1, 1, rb, inv_s, relu, false, aw, al0, al1, act_hi, lo, arow, lq);
              rb = args.ray_bias + (size_t)ray_s[arow + 8] * cols;
              epi_chunk<kX3, kBlk, 2>(acc0, 0, rb, inv_s, relu, false, aw, al0, al1, act_hi, lo, arow, lq);
              if (st.n_chunks == 2) epi_chunk<kX3, kBlk, 2>(acc1, 1, rb, inv_s, relu, false, aw, al0, al1, act_hi, lo, arow, lq);
            } else {
              epi_chunk<kX3, kBlk>(acc0, 0, bias, inv_s, relu, adot, aw, al0, al1, act_hi, lo, arow, lq);
              if (st.n_chunks == 2)
                epi_chunk<kX3, kBlk>(acc1, 1, bias, inv_s, relu, adot, aw, al0, al1, act_hi, lo, arow, lq);
            }
            if (adot) {
              // the four threads of a quad hold the row's columns
              al0 += __shfl_xor_sync(0xffffffffu, al0, 1); al0 += __shfl_xor_sync(0xffffffffu, al0, 2);
              al1 += __shfl_xor_sync(0xffffffffu, al1, 1); al1 += __shfl_xor_sync(0xffffffffu, al1, 2);
              if (lq == 0) { alpha_s[arow] = al0; alpha_s[arow + 8] = al1; }
            }
            if constexpr (!kX3) {
              if (st.write_cond) {   // bf16: the rgb condition, the input block of the next step
                const float* cond = args.cond + row.ray * prog.cond_stride + prog.rc_off;
                cond_to_block(inh, r, cond, prog.rc, 4 * h0, 4 * h0 + 4);
              }
            }
          } else {
            // warp net: one 128-column chunk per row block, no alpha head, no rgb condition
            float al0 = 0.f, al1 = 0.f;
            epi_chunk<kX3, kBlk>(acc0, 0, bias, inv_s, relu, false, aw, al0, al1, act_hi, lo, arow, lq);
            epi_chunk<kX3, kBlk>(acc1, 0, bias, inv_s, relu, false, aw, al0, al1, act_hi, lo + 32, arow + 64, lq);
          }
        } else {
          // ---- heads: N = 16 accumulator columns through the scratch to the row threads ----
          const int l0 = 16 * wq + (lane >> 2);
#pragma unroll
          for (int b = 0; b < kMB; ++b) {
            const float* a16 = b == 0 ? acc0 : acc1;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float* sr = scr + (l0 + 64 * b + 8 * h) * 16 + 2 * lq;
              sr[0] = a16[2 * h]; sr[1] = a16[2 * h + 1];
              sr[8] = a16[4 + 2 * h]; sr[9] = a16[5 + 2 * h];
            }
          }
          wg_sync();
          float v[12];
#pragma unroll
          for (int j = 0; j < 12; ++j) v[j] = fmaf(scr[lr * 16 + j], inv_s, __ldg(bias + j));
          wg_sync();      // the scratch has been read before anything overwrites block 0
          if (st.epi == kEpiWarpHeads) {
            float y[3];
            warp_tail(prog.warp_type, v, row.x, prog.warp_pivot, prog.warp_trans, y);
            if (row.valid && h0 == 0) {
#pragma unroll
              for (int c = 0; c < 3; ++c) args.warped[row.m * 3 + c] = y[c];
            }
            if (has_next) begin_tile(tile_of(ti + 1));
          } else if constexpr (kMB == 1) {
            float4 o;
            o.x = sigmoidf(v[0]); o.y = sigmoidf(v[1]); o.z = sigmoidf(v[2]);
            float a;
            if constexpr (kX3) {
              // with an alpha condition the head's bias, the bottleneck's and the condition's terms are one
              // per-ray constant
              a = (prog.ac ? __ldg(args.ray_alpha + row.ray) : alpha_b) + alpha_s[r];
            } else {
              // bf16: the alpha condition's part of Dense(1) on [bottleneck | alpha condition]
              const float a_cond = prog.ac ? alpha_cond_dot(args.cond + row.ray * prog.cond_stride + prog.ac_off,
                                                            aux + prog.alpha_w_off + kAlphaCondOff, prog.ac)
                                           : 0.f;
              a = alpha_b + (alpha_s[r] + a_cond);
            }
            o.w = apply_act(a, prog.sigma_act);
            if (h0 == 0 && row.valid && args.samples) reinterpret_cast<float4*>(args.samples)[row.m] = o;
            if (fuse && h0 == 0) {
              // ---- volumetric_rendering (model_utils.py:104-136) + median depth (:231-239, 262-263)
              //      over the 128 samples of this tile; one sample per row thread of half 0 ----
              const int qd = r >> 5;
              auto bar128 = [&]() { asm volatile("bar.sync 3, 128;" ::: "memory"); };
              if ((tile % tpr) == 0) {
                c_T = 1.f; c_cw = 0.f; a_r = a_g = a_b = a_d = a_w = a_wnl = a_med = 0.f; c_med = false;
              }
              // alpha = 1 - exp(-sigma * dist) as -expm1(-x) (see composite_kernel)
              const float al = -expm1f(-o.w * row.dist);
              const float tf = 1.0f - al + 1e-10f;
              float P = tf;                                    // inclusive product scan of tf
#pragma unroll
              for (int sh = 1; sh < 32; sh <<= 1) {
                const float q = __shfl_up_sync(0xffffffffu, P, sh);
                if (lane >= sh) P = P * q;
              }
              float excl = __shfl_up_sync(0xffffffffu, P, 1);
              if (lane == 0) excl = 1.f;
              if (lane == 31) scan_s[qd] = P;
              bar128();
              float Wq = 1.f, Wall = 1.f;
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                const float f = scan_s[q];
                if (q < qd) Wq = Wq * f;
                Wall = Wall * f;
              }
              const float Ti = (c_T * Wq) * excl;              // accum_prod (model_utils.py:110-113)
              const float w = al * Ti;
              if (args.ray_weights) args.ray_weights[row.m] = w;
              float C = w;                                     // inclusive cumsum of the weights
#pragma unroll
              for (int sh = 1; sh < 32; sh <<= 1) {
                const float q = __shfl_up_sync(0xffffffffu, C, sh);
                if (lane >= sh) C = C + q;
              }
              float red[6] = {w * o.x, w * o.y, w * o.z, w * row.z, w, row.last ? 0.f : w};
#pragma unroll
              for (int k = 0; k < 6; ++k)
#pragma unroll
                for (int sh = 16; sh > 0; sh >>= 1) red[k] += __shfl_xor_sync(0xffffffffu, red[k], sh);
              if (lane == 0) {
#pragma unroll
                for (int k = 0; k < 6; ++k) scan_s[8 + qd * 8 + k] = red[k];
              }
              bar128();
              float pre = c_cw, tot[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                if (q < qd) pre += scan_s[8 + q * 8 + 4];
#pragma unroll
                for (int k = 0; k < 6; ++k) tot[k] += scan_s[8 + q * 8 + k];
              }
              const float cwt = pre + C;                       // cumsum over the ray up to this sample
              // Median depth: the first sample in ray order whose cumulative weight reaches 0.5
              // (opaque xor shifted, :231-238).  cwt is summed in three associations (the shfl_up scan,
              // the quarter totals, the tile carry), so it is not monotone across lanes, quarters and
              // tiles: comparing each sample with its predecessor can fire no sample or two near 0.5.
              // The median is the lowest firing lane of the lowest firing quarter of the ray's first
              // firing tile, taken once.
              const unsigned hit = __ballot_sync(0xffffffffu, cwt >= 0.5f);
              const float zhit = __shfl_sync(0xffffffffu, row.z, hit ? __ffs(hit) - 1 : 0);
              if (lane == 0) { scan_s[4 + qd] = zhit; scan_s[8 + qd * 8 + 6] = hit ? 1.f : 0.f; }
              bar128();
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                if (!c_med && scan_s[8 + q * 8 + 6] != 0.f) { a_med = scan_s[4 + q]; c_med = true; }
              }
              a_r += tot[0]; a_g += tot[1]; a_b += tot[2]; a_d += tot[3]; a_w += tot[4]; a_wnl += tot[5];
              c_T = c_T * Wall; c_cw += tot[4];
              if ((tile % tpr) == tpr - 1 && r == 0) {
                float rr = a_r, gg = a_g, bb = a_b;
                if (args.white_bg) { const float bg = 1.f - a_w; rr = rr + bg; gg = gg + bg; bb = bb + bg; }
                float* ro = args.ray_out + row.ray * 6;
                ro[0] = rr; ro[1] = gg; ro[2] = bb; ro[3] = a_d; ro[4] = a_med;
                ro[5] = args.sample_at_infinity ? a_wnl : a_w;
              }
              bar128();   // scan_s is read by every row thread before the next tile writes it
            }
            if (has_next) begin_tile(tile_of(ti + 1));
          }
          // The step after a head reads the input block only (build_tc_program), so the head was
          // the last reader of the x_lo registers.  Redefining them here, after the row-thread work,
          // lets the compiler see that they are dead during it (64 registers for the fp64 encoder).
          if constexpr (kX3) {
#pragma unroll
            for (int i = 0; i < 64; ++i) lo[i] = 0u;
          }
        }
        fence_proxy_async();   // this thread's shared-memory stores are visible to the next MMAs ...
        wg_sync();             // ... of every warp of the warpgroup
      }
    }
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------
// Host side: translate the model's layer list (FieldProgram, built for every
// precision in nfb_api.cu) into TcPrograms, pack the weights, launch.
// ---------------------------------------------------------------------------
inline int tc_fail(const char* what) {
  return fail("the tensor-core paths (precision bf16 / fp16x3) do not support this model: %s; use precision fp32", what);
}

inline int build_tc_program(nfb_handle* h, int level, long long* wbytes, long long* aux_floats,
                            long long* fold_floats) {
  const FieldProgram& fp = h->prog[level];
  TcProgram& tp = h->tcprog[level];
  memset(&tp, 0, sizeof(tp));
  TcFold& fo = h->tc_fold[level];
  memset(&fo, 0, sizeof(fo));
  // fp16x3: every unit is [W_hi | W_lo]
  const int wparts = h->cfg.precision == NFB_PREC_FP16X3 ? 2 : 1;
  tp.warp_pivot = fp.warp_pivot; tp.warp_trans = fp.warp_trans;
  tp.warp_type = fp.warp_type; tp.Fw = fp.Fw; tp.G = fp.G; tp.Fp = fp.Fp;
  tp.cond_stride = fp.cond_stride; tp.sigma_act = fp.sigma_act;
  tp.tc = fp.tc; tp.ac = fp.ac; tp.rc = fp.rc; tp.ac_off = fp.G + fp.tc; tp.rc_off = fp.G + fp.tc + fp.ac;
  // per-ray condition vector: [glo | trunk | alpha | rgb] (nfb_api.cu: build_programs)
  fo.ac_off = fp.G + fp.tc; fo.rc_off = fp.G + fp.tc + fp.ac;
  if (fp.rc > kBlockK) return tc_fail("rgb condition wider than 64 channels");
  if (fp.ac > kBlockK) return tc_fail("alpha condition wider than 64 channels");
  if (fp.Dp + fp.tc > kBlockK || (fp.warp_type && fp.Dw > kBlockK)) return tc_fail("encoded inputs wider than 64");
  if (fp.hidden_act != kRelu) return tc_fail("hidden activation other than relu");
  auto new_bias = [&](const Step& st) {
    int off = (int)*aux_floats;
    *aux_floats += 256;
    h->tc_aux_jobs.push_back({st.b_off, st.n, 1, off});
    return off;
  };
  // The folded bottleneck still counts against kMaxTcSteps, so the fold does not change which models
  // the tensor-core paths accept.
  int folded = 0;
  // fold: the layer that reads the bottleneck, its weights W_b W_r[:W] in d_fold and its bias per ray
  auto add = [&](const Step& st, int epi, int cur_width, bool fold = false) -> int {
    if (tp.n_steps + folded >= kMaxTcSteps) return tc_fail("too many layers");
    TcStep& t = tp.steps[tp.n_steps];
    memset(&t, 0, sizeof(t));
    if (st.k_x > 256 || st.k_in > kBlockK) return tc_fail("layer wider than 256 or inputs wider than 64");
    if (st.k_x && st.k_x != cur_width) return tc_fail("unexpected layer input width");
    t.nkb = 0;
    if (st.k_in) t.src[t.nkb++] = kSrcIn;
    for (int b = 0; b < (st.k_x + kBlockK - 1) / kBlockK; ++b) t.src[t.nkb++] = b;
    t.epi = epi;
    if (epi == kEpiHidden) {
      // N is issued in chunks of 128 columns; a narrower layer is zero-padded (zero weight rows
      // and biases give zero output columns, which the next layer's zero-padded K rows ignore)
      if (st.n < 1 || st.n > 256) return tc_fail("hidden widths must be 1..256");
      t.n_chunks = (st.n + 127) / 128; t.chunk_n = 128;
      if (st.act != kRelu && st.act != kNone) return tc_fail("hidden activation other than relu");
      t.relu = st.act == kRelu;
    } else {
      // a head follows a hidden layer and is followed by a step that reads the input block only
      // (its accumulators pass through activation block 0, see field_wg_kernel)
      t.n_chunks = 1; t.chunk_n = 16;
      if (st.n > 12) return tc_fail("head wider than 12");
      if (st.k_in) return tc_fail("head reading the encoded inputs");
    }
    if (fold) t.ray_bias = 1;
    else t.b_off = new_bias(st);
    // weight units: for chunk c, for kb: wparts x chunk_n rows x 128 B
    t.w_off = (uint32_t)*wbytes;
    for (int c = 0; c < t.n_chunks; ++c) {
      nfb_handle::TcPackJob job;
      job.level = level; job.step = tp.n_steps; job.chunk = c;
      job.simt_w_off = st.w_off; job.ld = st.npad; job.n = st.n; job.n0 = c * t.chunk_n;
      job.k_total = st.k_x + st.k_in;
      job.fold = fold;
      job.k_map.assign((size_t)t.nkb * kBlockK, -1);
      for (int kb = 0; kb < t.nkb; ++kb)
        for (int j = 0; j < kBlockK; ++j) {
          int srck = -1;
          if (t.src[kb] < kSrcIn) srck = t.src[kb] * kBlockK + j < st.k_x ? t.src[kb] * kBlockK + j : -1;
          else if (j < st.k_in) srck = st.k_x + j;
          job.k_map[(size_t)kb * kBlockK + j] = srck;
        }
      h->tc_jobs.push_back(job);
      *wbytes += (long long)wparts * t.nkb * t.chunk_n * kRowBytes;
    }
    ++tp.n_steps;
    return 0;
  };
  // warp net
  int width = 0;
  for (int i = 0; i < fp.warp.n_steps; ++i) {
    const Step& st = fp.warp.steps[i];
    const bool head = st.dst == kOut0 || st.dst == kOut1;
    if (add(st, head ? kEpiWarpHeads : kEpiHidden, width)) return -1;
    if (!head) width = st.n;
  }
  tp.n_warp = tp.n_steps;
  // A warp net no wider than 128 runs in 256-row tiles: its layers are one N-chunk, so two row
  // blocks fit the accumulator and x_lo registers of one 256-wide layer.
  tp.warp_mb = 2;
  for (int i = 0; i < tp.n_warp; ++i)
    if (tp.steps[i].n_chunks != 1) tp.warp_mb = 1;
  // nerf net: trunk..., alpha head (an epilogue dot product), rgb branch.  A bottleneck (a Dense(W) with no
  // activation, present when there is an alpha or rgb condition, modules.py:149-161) is linear, so it is
  // folded into the layers that read it and has no step: the rgb branch's first layer reads
  //   relu([x W_b + b_b | cond] W_r + b_r) = relu(x (W_b W_r[:W]) + (b_b W_r[:W] + b_r + cond W_r[W:])),
  // x = the trunk's last activation; the second term is one vector per ray (ray_bias_kernel).  With an
  // alpha condition the alpha head is folded the same way: weights W_b w_a[:W] over x, and a per-ray
  // constant b_a + b_b w_a[:W] + cond w_a[W:].
  // bf16 keeps the bottleneck as a layer: that mode's arithmetic is bf16 operands per layer (the rgb
  // condition enters as a K-block the bottleneck's epilogue writes, the alpha condition's dot product is
  // added by the row threads), which a folded product cannot reproduce.
  const bool fold = h->cfg.precision == NFB_PREC_FP16X3;
  width = 0;
  int last_hidden = -1;
  bool seen_alpha = false, fold_pending = false, seen_bottleneck = false;
  for (int i = 0; i < fp.nerf.n_steps; ++i) {
    const Step& st = fp.nerf.steps[i];
    if (st.dst == fp.alpha_slot && st.n == 1 && !seen_alpha) {
      // alpha = Dense(1)(trunk_out), or with an alpha condition Dense(1)([bottleneck_out | alpha_cond])
      // (models.py:206-207, modules.py:152-157): the dot product over the trunk's last layer is folded into
      // that layer's epilogue.
      if (st.k_in != fp.ac) return tc_fail("alpha head inputs");
      seen_alpha = true;
      // Unfolded, the program runs the bottleneck before alpha: without an alpha condition the alpha head
      // reads the trunk's last layer, the hidden step before the bottleneck.
      const int src_step = (!fold && seen_bottleneck && !st.k_in) ? last_hidden - 1 : last_hidden;
      if (src_step < 0) return tc_fail("alpha head without a trunk layer");
      tp.steps[src_step].alpha_dot = 1;
      tp.alpha_w_off = (int)*aux_floats; *aux_floats += kAlphaCondOff + kBlockK;
      tp.alpha_b_off = (int)*aux_floats; *aux_floats += 4;
      if (st.k_in && !fold) {
        h->tc_aux_jobs.push_back({st.w_off, st.k_x, st.npad, tp.alpha_w_off, false});
        h->tc_aux_jobs.push_back({st.w_off + st.k_x * st.npad, st.k_in, st.npad, tp.alpha_w_off + kAlphaCondOff, false});
      } else if (st.k_in) {
        fo.ac = st.k_in; fo.lda = st.npad; fo.wa = st.w_off; fo.ba = st.b_off;
        h->tc_aux_jobs.push_back({fo.fwa, st.k_x, 1, tp.alpha_w_off, true});
      } else {
        h->tc_aux_jobs.push_back({st.w_off, st.k_x, st.npad, tp.alpha_w_off, false});
      }
      h->tc_aux_jobs.push_back({st.b_off, 1, 1, tp.alpha_b_off, false});
      continue;
    }
    const bool out = st.dst == fp.rgb_slot;
    if (!out && st.act == kNone && !fold) {        // bottleneck, bf16
      seen_bottleneck = true;
      if (add(st, kEpiHidden, width)) return -1;
      last_hidden = tp.n_steps - 1;
      tp.steps[last_hidden].write_cond = 1;
      continue;
    }
    if (!out && st.act == kNone) {                 // bottleneck, fp16x3
      fo.active = 1; fo.W = st.n; fo.ldb = st.npad; fo.wb = st.w_off; fo.bb = st.b_off;
      // d_fold: [W_b w_a[:W] (W) | constant (4) | rgb constant (256) | W_b W_r[:W] (W x ldr)]
      fo.fwa = (int)*fold_floats; fo.fca = fo.fwa + (fo.W + 3) / 4 * 4; fo.fc = fo.fca + 4; fo.fw = fo.fc + 256;
      *fold_floats = fo.fw;
      ++folded;
      fold_pending = true;
      continue;
    }
    if (fold_pending) {                            // the layer that reads the bottleneck
      fold_pending = false;
      if (out) return tc_fail(st.k_in ? "head reading the encoded inputs" : "rgb logit reading the bottleneck");
      fo.nr = st.n; fo.ldr = st.npad; fo.rc = st.k_in; fo.wr = st.w_off; fo.br = st.b_off;
      fo.cols = 128 * ((st.n + 127) / 128);
      *fold_floats += (long long)fo.W * fo.ldr;
      Step f = st;
      f.k_in = 0; f.w_off = fo.fw;
      if (add(f, kEpiHidden, width, true)) return -1;
      last_hidden = tp.n_steps - 1;
      width = st.n;
      continue;
    }
    if (add(st, out ? kEpiRgbOut : kEpiHidden, width)) return -1;
    if (!out) {
      last_hidden = tp.n_steps - 1;
      width = st.n;
    }
  }
  if (!seen_alpha) return tc_fail("model without alpha head");
  for (int si = 0; si < tp.n_steps; ++si) {
    const bool after_head = si > 0 && tp.steps[si - 1].epi != kEpiHidden;
    if ((si == 0 || after_head) && (tp.steps[si].nkb != 1 || tp.steps[si].src[0] != kSrcIn))
      return tc_fail("first layer of an MLP reading more than the encoded inputs");
  }
  tp.scale_off = (int)*aux_floats; *aux_floats += kMaxTcSteps;
  return 0;
}

inline int create_tc(nfb_handle* h) {
  long long wbytes = 0, auxf = 0, foldf = 0;
  h->tc_jobs.clear(); h->tc_aux_jobs.clear();
  const int levels = h->cfg.num_fine_samples > 0 ? 2 : 1;
  for (int lv = 0; lv < levels; ++lv)
    if (build_tc_program(h, lv, &wbytes, &auxf, &foldf)) return -1;
  if (levels == 1) { h->tcprog[1] = h->tcprog[0]; h->tc_fold[1] = h->tc_fold[0]; }
  h->wpack_bytes = wbytes; h->aux_floats = auxf;
  if (cudaMalloc(&h->d_wpack, (size_t)wbytes) != cudaSuccess) return fail("cudaMalloc wpack failed");
  if (cudaMalloc(&h->d_aux, (size_t)auxf * sizeof(float)) != cudaSuccess) return fail("cudaMalloc aux failed");
  if (cudaMemset(h->d_aux, 0, (size_t)auxf * sizeof(float)) != cudaSuccess) return fail("cudaMemset failed");
  if (h->tc_fold[0].active) {
    // both levels have the same widths, so one per-ray buffer serves both
    const size_t rb = (size_t)h->max_rays * (h->tc_fold[0].cols + 1);
    if (cudaMalloc(&h->d_fold, (size_t)foldf * sizeof(float)) != cudaSuccess ||
        cudaMalloc(&h->d_ray_bias, rb * sizeof(float)) != cudaSuccess)
      return fail("cudaMalloc of the bottleneck fold buffers failed");
  }
  const auto smem_attr = cudaFuncAttributeMaxDynamicSharedMemorySize;
  if (cudaFuncSetAttribute(field_wg_kernel<true, 1>, smem_attr, kWgSmemBytes) != cudaSuccess ||
      cudaFuncSetAttribute(field_wg_kernel<true, 2>, smem_attr, kWgSmemBytes) != cudaSuccess ||
      cudaFuncSetAttribute(field_wg_kernel<false, 1>, smem_attr, kWgSmemBytes) != cudaSuccess ||
      cudaFuncSetAttribute(field_wg_kernel<false, 2>, smem_attr, kWgSmemBytes) != cudaSuccess)
    return fail("cannot reserve %d bytes of shared memory for the tensor-core kernel", kWgSmemBytes);
  return 0;
}

inline void destroy_tc(nfb_handle* h) {
  if (h->d_wpack) cudaFree(h->d_wpack);
  if (h->d_aux) cudaFree(h->d_aux);
  if (h->d_fold) cudaFree(h->d_fold);
  if (h->d_ray_bias) cudaFree(h->d_ray_bias);
  h->d_wpack = nullptr; h->d_aux = nullptr; h->d_fold = nullptr; h->d_ray_bias = nullptr;
}

__global__ void aux_copy_kernel(const float* __restrict__ src, int count, int stride,
                                float* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) dst[i] = src[(size_t)i * stride];
}

// The bottleneck fold of one level (TcFold) from the fp32 parameters p, in fp64, each output rounded once.
// Thread (i, j) of (W + 1) x (ldr + 1): row i < W is the bottleneck's weight row i (its output is row i of
// the folded weights), row W its bias (the folded constants); column j < ldr is column j of the rgb layer
// (zero past nr), column ldr the alpha head (alpha condition only).
__global__ void fold_kernel(const float* __restrict__ p, const TcFold f, float* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int cols = f.ldr + 1;
  if (idx >= (f.W + 1) * cols) return;
  const int i = idx / cols, j = idx - i * cols;
  const bool alpha = j == f.ldr, bias = i == f.W;
  if (alpha && !f.ac) return;
  float* o = alpha ? out + (bias ? f.fca : f.fwa + i) : out + (bias ? f.fc : f.fw + i * f.ldr) + j;
  if (!alpha && j >= f.nr) { *o = 0.f; return; }
  const float* x = bias ? p + f.bb : p + f.wb + (size_t)i * f.ldb;
  const float* y = alpha ? p + f.wa : p + f.wr + j;
  const int ldy = alpha ? f.lda : f.ldr;
  double v = bias ? (double)p[alpha ? f.ba : f.br + j] : 0.0;
  for (int k = 0; k < f.W; ++k) v = fma((double)x[k], (double)y[(size_t)k * ldy], v);
  *o = (float)v;
}

// Called from nfb_set_params after the fp32 layout has been filled.
inline int pack_tc(nfb_handle* h, cudaStream_t s) {
  // k_maps are small; one staging buffer, stream-ordered.
  size_t total_map = 0;
  for (auto& j : h->tc_jobs) total_map += j.k_map.size();
  int* d_maps = nullptr;
  if (cudaMalloc(&d_maps, total_map * sizeof(int)) != cudaSuccess) return fail("cudaMalloc k_map failed");
  std::vector<int> all;
  all.reserve(total_map);
  for (auto& j : h->tc_jobs) all.insert(all.end(), j.k_map.begin(), j.k_map.end());
  cudaError_t e = cudaMemcpyAsync(d_maps, all.data(), total_map * sizeof(int), cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);   // `all` is pageable and local
  if (e != cudaSuccess) { cudaFree(d_maps); return fail("k_map upload failed: %s", cudaGetErrorString(e)); }
  size_t map_off = 0;
  const bool x3 = h->cfg.precision == NFB_PREC_FP16X3;
  // the folded weights first: the pack jobs of the layers that read the bottleneck read them
  for (int lv = 0; lv < (h->cfg.num_fine_samples > 0 ? 2 : 1); ++lv) {
    const TcFold& f = h->tc_fold[lv];
    if (!f.active) continue;
    const int n = (f.W + 1) * (f.ldr + 1);
    fold_kernel<<<(n + 127) / 128, 128, 0, s>>>(h->d_packed, f, h->d_fold);
    h->launches++;
  }
  auto src = [&](bool fold) { return fold ? h->d_fold : h->d_packed; };
  if (x3) {
    // per-layer max |W| -> power-of-two scale (x3_weight_scale), computed on the device
    for (int lv = 0; lv < 2; ++lv)
      cudaMemsetAsync(h->d_aux + h->tcprog[lv].scale_off, 0, kMaxTcSteps * sizeof(float), s);
    for (auto& j : h->tc_jobs) {
      if (j.chunk != 0) continue;
      const long long n = (long long)j.k_total * j.ld;
      absmax_kernel<<<(unsigned)std::min<long long>((n + 255) / 256, 64), 256, 0, s>>>(
          src(j.fold) + j.simt_w_off, n, h->d_aux + h->tcprog[j.level].scale_off + j.step);
      h->launches++;
    }
  }
  for (auto& j : h->tc_jobs) {
    const TcStep& t = h->tcprog[j.level].steps[j.step];
    const long long total = (long long)t.nkb * t.chunk_n * kBlockK;
    uint8_t* dst = h->d_wpack + t.w_off + (size_t)(x3 ? 2 : 1) * j.chunk * t.nkb * t.chunk_n * kRowBytes;
    // source columns n0.. of the fp32 (K x npad) matrix: shift the base pointer.
    if (x3)
      pack_weight_x3_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(
          src(j.fold) + j.simt_w_off + j.n0, j.ld, d_maps + map_off, t.nkb, j.n - j.n0, t.chunk_n,
          h->d_aux + h->tcprog[j.level].scale_off + j.step, dst);
    else
      pack_weight_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(
          src(j.fold) + j.simt_w_off + j.n0, j.ld, d_maps + map_off, t.nkb, j.n - j.n0, t.chunk_n,
          reinterpret_cast<__nv_bfloat16*>(dst));
    h->launches++;
    map_off += j.k_map.size();
  }
  for (auto& a : h->tc_aux_jobs) {
    aux_copy_kernel<<<(a.count + 127) / 128, 128, 0, s>>>(src(a.fold) + a.src_off, a.count, a.stride,
                                                          h->d_aux + a.dst_off);
    h->launches++;
  }
  e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  cudaFree(d_maps);
  if (e != cudaSuccess) return fail("tensor-core weight packing failed: %s", cudaGetErrorString(e));
  return 0;
}

// One pass of field_wg_kernel: the warp net (a.warp_only, into a.warped) or the NeRF net.  The NeRF
// pass of a warped model reads the warp pass's points (a.points); nothing warps inside it.  The NeRF pass
// of a model with a bottleneck first forms its rays' folded bias (ray_bias_kernel, from a.cond).
inline int run_field_tc(nfb_handle* h, int level, const FieldArgs& args, cudaStream_t s) {
  const TcProgram& prog = h->tcprog[level];
  FieldArgs a = args;
  const TcFold& f = h->tc_fold[level];
  if (!a.warp_only && f.active && a.num_rows > 0) {
    RayBiasArgs r{};
    r.num_rays = (int)((a.num_rows + a.samples_per_ray - 1) / a.samples_per_ray);
    r.cond = a.cond; r.stride = prog.cond_stride;
    r.w_rc = h->d_packed + f.wr + (size_t)f.W * f.ldr; r.ldr = f.ldr; r.rc = f.rc; r.rc_off = f.rc_off;
    r.c_r = h->d_fold + f.fc; r.nr = f.nr; r.cols = f.cols;
    r.w_ac = h->d_packed + f.wa + (size_t)f.W * f.lda; r.lda = f.lda; r.ac = f.ac; r.ac_off = f.ac_off;
    r.c_a = h->d_fold + f.fca;
    r.bias = h->d_ray_bias; r.alpha = h->d_ray_bias + (size_t)h->max_rays * f.cols;
    const long long n = (long long)r.num_rays * (f.cols + (f.ac > 0));
    ray_bias_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(r);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail("ray_bias_kernel launch failed: %s", cudaGetErrorString(e));
    h->launches++;
    a.ray_bias = r.bias; a.ray_alpha = r.alpha;
  }
  if (a.warp_only && (prog.n_warp == 0 || !a.warped)) return fail("warp pass without a warp net or an output");
  if (!a.warp_only && a.use_warp && prog.n_warp > 0 && !a.points)
    return fail("the NeRF pass of a warped model needs the warp pass's points");
  const int mb = (a.warp_only && prog.warp_mb == 2 && !(a.debug & kDebugOneRowBlock)) ? 2 : 1;
  const long long rows_per_tile = (long long)mb * kTileRows;
  const long long tiles = (a.num_rows + rows_per_tile - 1) / rows_per_tile;
  if (tiles > 0x7fffffffLL) return fail("too many rows for one launch");
  const bool fuse = a.ray_out != nullptr && !a.warp_only;
  if (fuse && (a.samples_per_ray % kTileRows != 0 || a.num_rows % a.samples_per_ray != 0))
    return fail("fused composite needs samples_per_ray to be a multiple of %d", kTileRows);
  const long long groups = fuse ? a.num_rows / a.samples_per_ray : tiles;
  const int grid = (int)std::min<long long>(groups, h->sm_count);
  const bool x3 = h->cfg.precision == NFB_PREC_FP16X3;
  auto kernel = x3 ? (mb == 2 ? field_wg_kernel<true, 2> : field_wg_kernel<true, 1>)
                   : (mb == 2 ? field_wg_kernel<false, 2> : field_wg_kernel<false, 1>);
  kernel<<<grid, kWgThreads, kWgSmemBytes, s>>>(prog, a, h->d_wpack, h->d_aux, (int)tiles);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("field_wg_kernel launch failed: %s", cudaGetErrorString(e));
  h->launches++;
  return 0;
}

}  // namespace tc
}  // namespace nfb
