// Step list interpreted by the tensor-core field kernel (field_tc.cuh).
#pragma once
#include <stdint.h>

namespace nfb {
namespace tc {

constexpr int kMaxTcSteps = 24;
constexpr int kSrcIn = 4;     // K-block source: 0..3 = activation block, 4 = input block
constexpr int kAlphaCondOff = 256;   // alpha-condition weights, after the 256 trunk weights

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
  int relu;            // hidden activation (relu) or identity (bottleneck)
  int alpha_dot;       // this epilogue also accumulates the alpha head (Dense(1))
  int write_cond;      // this epilogue also writes the rgb condition into the input block
};

struct TcProgram {
  int n_steps;
  TcStep steps[kMaxTcSteps];
  int n_warp;                     // steps [0, n_warp) are the warp net, the rest the NeRF net
  int warp_mb;                    // 64-row blocks per consumer warpgroup in the warp pass (1 or 2)
  int warp_type, Fw, G, Fp, rc, cond_stride, sigma_act;
  int tc, ac;                     // trunk / alpha condition widths
  int ac_off, rc_off;             // offsets of the alpha / rgb condition in the per-ray condition vector
  int warp_pivot, warp_trans;     // SE3Field use_pivot / use_translation
  int alpha_w_off, alpha_b_off;   // aux float offsets (alpha weights: trunk part, then the condition part)
  int scale_off;                  // fp16x3: aux offset of the per-step max |W| (kMaxTcSteps floats)
};

}  // namespace tc
}  // namespace nfb
