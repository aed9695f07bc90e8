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

// SE3Field.warp tail (warping.py:330-345) + rigid_body.exp_se3
// (rigid_body.py:54-89), written exactly as the reference does (no small-angle
// guard).  wv = [w(3), v(3)] raw head outputs, x the sample point.
// pivot / trans (nullable): SE3Field use_pivot / use_translation (warping.py:339-352):
// x + pivot -> rigid transform -> - pivot -> + trans.
__device__ __forceinline__ void se3_apply(const float wv[6], const float x_in[3],
                                          float out[3], const float* pivot = nullptr,
                                          const float* trans = nullptr) {
  float x[3] = {x_in[0], x_in[1], x_in[2]};
  if (pivot) { x[0] = x[0] + pivot[0]; x[1] = x[1] + pivot[1]; x[2] = x[2] + pivot[2]; }
  float theta = sqrtf(wv[0] * wv[0] + wv[1] * wv[1] + wv[2] * wv[2]);
  float w0 = wv[0] / theta, w1 = wv[1] / theta, w2 = wv[2] / theta;
  float v0 = wv[3] / theta, v1 = wv[4] / theta, v2 = wv[5] / theta;
  // W = skew(w); W2 = W @ W.
  float W[3][3] = {{0.f, -w2, w1}, {w2, 0.f, -w0}, {-w1, w0, 0.f}};
  float W2[3][3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      W2[i][j] = W[i][0] * W[0][j] + W[i][1] * W[1][j] + W[i][2] * W[2][j];
  float s = sinf(theta), c = cosf(theta);
  float omc = 1.0f - c, tms = theta - s;
  float v[3] = {v0, v1, v2};
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    float R[3], M[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      float eye = (i == j) ? 1.f : 0.f;
      R[j] = eye + s * W[i][j] + omc * W2[i][j];
      M[j] = theta * eye + omc * W[i][j] + tms * W2[i][j];
    }
    float p = M[0] * v[0] + M[1] * v[1] + M[2] * v[2];
    float rx = R[0] * x[0] + R[1] * x[1] + R[2] * x[2];
    out[i] = (rx + p) / 1.0f;
  }
  if (pivot) { out[0] = out[0] - pivot[0]; out[1] = out[1] - pivot[1]; out[2] = out[2] - pivot[2]; }
  if (trans) { out[0] = out[0] + trans[0]; out[1] = out[1] + trans[1]; out[2] = out[2] + trans[2]; }
}

}  // namespace nfb
