// Shared definitions for the nerfies_b200 render kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nfb {

constexpr int kMaxSteps = 16;     // GEMM steps per network
constexpr int kMaxWidth = 256;    // widest hidden layer
constexpr int kMaxIn = 128;       // widest input-feature block (posenc + conds)
constexpr float kHalfPiF = 1.57079637050628662109375f;  // fl32(pi/2), modules.py:221-223

enum Act { kNone = 0, kRelu = 1, kElu = 2, kLeakyRelu = 3, kTanh = 4,
           kSigmoid = 5, kSoftplus = 6 };
enum Buf { kB0 = 0, kB1 = 1, kOut0 = 2, kOut1 = 3 };

// One Dense layer: out = act([X[:, :k_x], IN[:, in_off:in_off+k_in]] @ W + b).
// W is packed (k_x + k_in) x npad row-major (columns zero-padded to npad).
struct Step {
  int w_off, b_off;        // float offsets into the packed parameter buffer
  int k_x, k_in, in_off;   // K rows taken from the source buffer / input block
  int n, npad;             // true and padded output width (npad % 32 == 0)
  int act;
  int src, dst;            // Buf ids
};

struct Net {
  int n_steps;
  Step steps[kMaxSteps];
};

// Everything the fused field kernel needs to know about the model.
struct FieldProgram {
  Net warp;                // SE3Field / TranslationField trunk + heads
  Net nerf;                // NerfMLP trunk, bottleneck, alpha head, rgb branch
  int warp_type;           // 0 none, 1 translation, 2 se3
  int warp_pivot, warp_trans;  // SE3Field use_pivot / use_translation: heads [w v (p) (t)]
  int Fw, G, Dw;           // warp inputs: [3 + 6 Fw posenc | G glo code]
  int Fp, Dp;              // nerf inputs: [3 + 6 Fp posenc | tc | ac | rc]
  int tc, ac, rc;
  int cond_stride;         // per-ray condition vector: [glo | tc | ac | rc]
  int hidden_act, sigma_act;
  int alpha_slot, rgb_slot;  // kOut0 / kOut1
};

// ---------------------------------------------------------------------------
// Scalar math shared by every precision mode.  Compiled with -fmad=false so
// that a*b+c keeps the two roundings of the reference's fp32 arithmetic;
// GEMM inner loops call fmaf() explicitly.
// ---------------------------------------------------------------------------
__device__ __forceinline__ float softplusf(float x) {
  // jax.nn.softplus = logaddexp(x, 0) = max(x,0) + log1p(exp(-|x|)).
  return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x)));
}

__device__ __forceinline__ float sigmoidf(float x) {
  // jax.nn.sigmoid = lax.logistic = 1 / (1 + exp(-x)).
  return 1.f / (1.f + expf(-x));
}

__device__ __forceinline__ float apply_act(float v, int act) {
  switch (act) {
    case kRelu: return fmaxf(v, 0.f);
    case kElu: return v > 0.f ? v : expm1f(v);
    case kLeakyRelu: return v >= 0.f ? v : 0.01f * v;
    case kTanh: return tanhf(v);
    case kSigmoid: return sigmoidf(v);
    case kSoftplus: return softplusf(v);
    default: return v;
  }
}

// Feature f (0 <= f < 6F) of SinusoidalEncoder after the identity block
// (modules.py:213-228): f = freq*6 + which*3 + c, value sin(2^freq x_c [+pi/2]).
__device__ __forceinline__ float posenc_feature(const float x[3], int f) {
  int freq = f / 6;
  int rem = f - freq * 6;
  int which = rem / 3;
  int c = rem - which * 3;
  float a = x[c] * exp2f((float)freq);   // exact: power of two
  if (which) a = a + kHalfPiF;
  return sinf(a);
}

// ---------------------------------------------------------------------------
// Scalar interface of the warp tail: float in the render kernels, forward-mode
// numbers (train.cuh: Fwd) in the training kernels.  Num<S>::c makes a constant.
// ---------------------------------------------------------------------------
template <class S> struct Num;
template <> struct Num<float> {
  static __device__ __forceinline__ float c(float x) { return x; }
};
__device__ __forceinline__ float nsqrt(float x) { return sqrtf(x); }
__device__ __forceinline__ float nsin(float x) { return sinf(x); }
__device__ __forceinline__ float ncos(float x) { return cosf(x); }

// SE3Field.warp tail (warping.py:330-352) + rigid_body.exp_se3 (rigid_body.py:54-97),
// written exactly as the reference does (no small-angle guard).  in[0..5] = w, v raw
// head outputs, in[6..] = (pivot), (translation); x = the sample point:
// x + pivot -> rigid transform -> - pivot -> + translation.
template <class S>
__device__ __forceinline__ void se3_tail(const S* in, const S* x_in, bool pivot, bool trans, S* out) {
  const S zero = Num<S>::c(0.f), one = Num<S>::c(1.f);
  const S theta = nsqrt(in[0] * in[0] + in[1] * in[1] + in[2] * in[2]);
  const S w[3] = {in[0] / theta, in[1] / theta, in[2] / theta};
  const S v[3] = {in[3] / theta, in[4] / theta, in[5] / theta};
  S x[3] = {x_in[0], x_in[1], x_in[2]};
  const S* pv = in + 6;
  const S* tr = in + (pivot ? 9 : 6);
  if (pivot)
    for (int c = 0; c < 3; ++c) x[c] = x[c] + pv[c];
  // W = skew(w); W2 = W @ W.
  const S W[3][3] = {{zero, zero - w[2], w[1]}, {w[2], zero, zero - w[0]}, {zero - w[1], w[0], zero}};
  S W2[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) W2[i][j] = W[i][0] * W[0][j] + W[i][1] * W[1][j] + W[i][2] * W[2][j];
  const S s = nsin(theta), c = ncos(theta);
  const S omc = one - c, tms = theta - s;
  for (int i = 0; i < 3; ++i) {
    S rx = zero, p = zero;
    for (int j = 0; j < 3; ++j) {
      const S eye = (i == j) ? one : zero;
      const S R = eye + s * W[i][j] + omc * W2[i][j];
      const S M = theta * eye + omc * W[i][j] + tms * W2[i][j];
      rx = rx + R * x[j];
      p = p + M * v[j];
    }
    out[i] = rx + p;
    if (pivot) out[i] = out[i] - pv[i];
    if (trans) out[i] = out[i] + tr[i];
  }
}

// The warp of both field types: SE(3) (warp_type 2, heads [w v (p) (t)]) or the
// TranslationField's y = x + t (warping.py:156).
template <class S>
__device__ __forceinline__ void warp_tail(int warp_type, const S* head, const S* x, bool pivot, bool trans,
                                          S* y) {
  if (warp_type == 2) {
    se3_tail(head, x, pivot, trans, y);
  } else {
    for (int c = 0; c < 3; ++c) y[c] = x[c] + head[c];
  }
}

}  // namespace nfb
