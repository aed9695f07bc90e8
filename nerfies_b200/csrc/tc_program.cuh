// Step list interpreted by the tensor-core field kernel (field_tc.cuh).
#pragma once
#include <stdint.h>

namespace nfb {
namespace tc {

constexpr int kMaxTcSteps = 24;
constexpr int kSrcIn = 4;     // K-block source: 0..3 = activation block, 4 = input block
constexpr int kAlphaCondOff = 256;   // bf16: alpha-condition weights, after the 256 trunk weights

enum Epi { kEpiHidden = 0, kEpiWarpHeads = 1, kEpiRgbOut = 2 };

// One Dense layer as a chain of wgmma over K-blocks of 64 columns.  A weight unit is
// one (N-chunk, K-block) pair; units are packed and streamed chunk-major.
struct TcStep {
  uint32_t w_off;      // byte offset of the first weight unit (pre-swizzled)
  int nkb;             // K-blocks
  int src[6];          // per K-block source
  int n_chunks;        // the N dimension is issued as 1 or 2 chunks ...
  int chunk_n;         // ... of this many columns (128, or 16 for a head)
  int b_off;           // float offset of the bias (256 floats reserved) in the aux buffer
  int epi;             // Epi
  int relu;            // hidden activation (relu) or identity (bf16: the bottleneck)
  int alpha_dot;       // this epilogue also accumulates the alpha head (Dense(1))
  int ray_bias;        // the bias is per ray (FieldArgs::ray_bias, 128 n_chunks floats per ray), not b_off:
                       // the rgb branch's first layer with the bottleneck folded into it (build_tc_program)
  int write_cond;      // bf16: this epilogue also writes the rgb condition into the input block
};

struct TcProgram {
  int n_steps;
  TcStep steps[kMaxTcSteps];
  int n_warp;                     // steps [0, n_warp) are the warp net, the rest the NeRF net
  int warp_mb;                    // 64-row blocks per consumer warpgroup in the warp pass (1 or 2)
  int warp_type, Fw, G, Fp, rc, cond_stride, sigma_act;
  int tc, ac;                     // trunk / alpha condition widths (fp16x3, ac > 0: the alpha head's constant
                                  // is per ray, FieldArgs::ray_alpha)
  int ac_off, rc_off;             // bf16: offsets of the alpha / rgb condition in the per-ray condition vector
  int warp_pivot, warp_trans;     // SE3Field use_pivot / use_translation
  int alpha_w_off, alpha_b_off;   // aux float offsets of the alpha weights (over the layer it reads, then bf16:
                                  // the condition part at kAlphaCondOff) and bias
  int scale_off;                  // fp16x3: aux offset of the per-step max |W| (kMaxTcSteps floats)
};

// A NeRF net's bottleneck (Dense(W), no activation) folded into the layers that read it: the rgb branch's
// first layer r (reading [bottleneck | rgb condition]) and, with an alpha condition, the alpha head a
// (reading [bottleneck | alpha condition]).  Offsets: `w*` / `b*` in the fp32 parameter buffer, `f*` in
// the handle's fold buffer.
struct TcFold {
  int active;
  int W, ldb;                     // trunk width = bottleneck width, row stride of the bottleneck's weights
  int nr, ldr, rc;                // rgb layer: outputs, row stride of its weights, rgb condition width
  int cols;                       // 128 n_chunks: per-ray bias floats (columns >= nr are zero)
  int lda, ac;                    // alpha head: row stride of its weights, alpha condition width (0: none)
  int rc_off, ac_off;             // rgb / alpha condition offsets in the per-ray condition vector
  int wb, bb, wr, br, wa, ba;
  int fw, fc, fwa, fca;           // W_b W_r[:W] (W x ldr) | b_b W_r[:W] + b_r (ldr) | W_b w_a[:W] (W) | constant
};

}  // namespace tc
}  // namespace nfb
