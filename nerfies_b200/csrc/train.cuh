// Training tier (SURVEY §8(f) #1): value_and_grad of the photometric loss of
// training.py:171-212 (mean squared error of the coarse and the fine rgb,
// training.py:173) through NerfModel.__call__, in fp32.
//
// Unlike the fused forward kernels this path is layer-wise: the forward pass keeps a
// TAPE in HBM (every Dense layer's output, the encoded inputs, the sample points) and
// the backward pass walks it in reverse.  All kernels are hand-written fp32 SIMT:
//   * sgemm128_kernel: one tiled GEMM template for the three shapes of a Dense layer
//       forward   Y  = act([X | IN] W + b)
//       backward  dX = dZ W^T         (dZ = dY * act'(Y), formed while loading)
//                 dW = [X | IN]^T dZ  (reduction over the rows: split + atomicAdd)
//   * colsum_kernel (bias gradients), encode / se3 / raw-activation kernels and their
//     adjoints, the adjoint of volumetric_rendering, embedding scatter-add, the TimeEncoder's input and
//     output stages and their adjoint ('time' / 'blend' warp metadata encoders), Adam.
// 80 GB of HBM holds the tape of a whole gpu_fullhd training batch (~31 GB); the
// caller may still process a batch in ray chunks (gradients accumulate).
// z_fine is a constant of the fine level (lax.stop_gradient, model_utils.py:211).
#pragma once
#include "common.cuh"
#include "nfb_handle.h"
#include "ray_kernels.cuh"

namespace nfb {

// ---------------------------------------------------------------------------
// Forward-mode numbers with N tangent directions over a scalar type T (float or
// another Fwd, for second derivatives): the scalar type of the warp tail's
// derivatives (se3_tail, common.cuh).
// ---------------------------------------------------------------------------
template <int N, class T>
struct Fwd {
  T v;
  T d[N];
};
template <int N, class T> struct Num<Fwd<N, T>> {
  static __device__ __forceinline__ Fwd<N, T> c(float x) {
    Fwd<N, T> r;
    r.v = Num<T>::c(x);
#pragma unroll
    for (int i = 0; i < N; ++i) r.d[i] = Num<T>::c(0.f);
    return r;
  }
};
template <int N, class T> __device__ __forceinline__ Fwd<N, T> operator+(const Fwd<N, T>& a, const Fwd<N, T>& b) {
  Fwd<N, T> r; r.v = a.v + b.v;
#pragma unroll
  for (int i = 0; i < N; ++i) r.d[i] = a.d[i] + b.d[i];
  return r;
}
template <int N, class T> __device__ __forceinline__ Fwd<N, T> operator-(const Fwd<N, T>& a, const Fwd<N, T>& b) {
  Fwd<N, T> r; r.v = a.v - b.v;
#pragma unroll
  for (int i = 0; i < N; ++i) r.d[i] = a.d[i] - b.d[i];
  return r;
}
template <int N, class T> __device__ __forceinline__ Fwd<N, T> operator*(const Fwd<N, T>& a, const Fwd<N, T>& b) {
  Fwd<N, T> r; r.v = a.v * b.v;
#pragma unroll
  for (int i = 0; i < N; ++i) r.d[i] = a.d[i] * b.v + a.v * b.d[i];
  return r;
}
template <int N, class T> __device__ __forceinline__ Fwd<N, T> operator/(const Fwd<N, T>& a, const Fwd<N, T>& b) {
  Fwd<N, T> r; r.v = a.v / b.v;
#pragma unroll
  for (int i = 0; i < N; ++i) r.d[i] = (a.d[i] - r.v * b.d[i]) / b.v;
  return r;
}
template <int N, class T> __device__ __forceinline__ Fwd<N, T> nsqrt(const Fwd<N, T>& a) {
  Fwd<N, T> r; r.v = nsqrt(a.v);
  const T k = Num<T>::c(0.5f) / r.v;
#pragma unroll
  for (int i = 0; i < N; ++i) r.d[i] = a.d[i] * k;
  return r;
}
template <int N, class T> __device__ __forceinline__ Fwd<N, T> nsin(const Fwd<N, T>& a) {
  Fwd<N, T> r; r.v = nsin(a.v);
  const T c = ncos(a.v);
#pragma unroll
  for (int i = 0; i < N; ++i) r.d[i] = a.d[i] * c;
  return r;
}
template <int N, class T> __device__ __forceinline__ Fwd<N, T> ncos(const Fwd<N, T>& a) {
  Fwd<N, T> r; r.v = ncos(a.v);
  const T s = Num<T>::c(0.f) - nsin(a.v);
#pragma unroll
  for (int i = 0; i < N; ++i) r.d[i] = a.d[i] * s;
  return r;
}

namespace train {

// activation derivative expressed through the OUTPUT y = act(z) (every registered
// activation is invertible enough for that: configs.py:27-32).
__device__ __forceinline__ float act_grad_from_output(float y, int act) {
  switch (act) {
    case kRelu: return y > 0.f ? 1.f : 0.f;
    case kElu: return y > 0.f ? 1.f : y + 1.f;
    case kLeakyRelu: return y >= 0.f ? 1.f : 0.01f;
    case kTanh: return 1.f - y * y;
    case kSigmoid: return y * (1.f - y);
    case kSoftplus: return 1.f - expf(-y);          // sigmoid(z) with y = log(1 + e^z)
    default: return 1.f;
  }
}

// ---------------------------------------------------------------------------
// One GEMM template.  C(m, n) (+)= sum_k A(m, k) * B(k, n) with element functors:
// slow address arithmetic, fast inner product.  gridDim.z splits the reduction
// (k_per_split; the caller's FC then atomicAdd-s).
// The layer-wise training tier is GEMM-bound (3 x the forward FLOPs per step), so the
// inner product is shaped for shared-memory bandwidth: a 128 x 128 C tile, an 8 x 8
// register tile per thread (two 4 x 4 quadrant pairs, so that every shared-memory read
// is a 16-byte vector and the A reads are warp broadcasts: 64 FMAs per 4 LDS.128),
// k-steps of 8 and a register prefetch of the next k-step's operands under the
// arithmetic of the current one (one __syncthreads per step).
// ---------------------------------------------------------------------------
struct GemmShape { long long M; int N; long long K; };

// kAKFast / kBNFast: which index of the element functor is contiguous in memory (k for a row-major A, n for a
// row-major B) - the loader walks that index with consecutive threads.
constexpr int kT2 = 128, kBK2 = 8, kPad2 = 4;
template <bool kAKFast, bool kBNFast, class FA, class FB, class FC>
__global__ void __launch_bounds__(256, 2)
sgemm128_kernel(GemmShape sh, FA fa, FB fb, FC fc, long long k_per_split) {
  __shared__ __align__(16) float As[2][kBK2][kT2 + kPad2];
  __shared__ __align__(16) float Bs[2][kBK2][kT2 + kPad2];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const long long m0 = (long long)blockIdx.x * kT2;
  const int n0 = blockIdx.y * kT2;
  const long long k_begin = (long long)blockIdx.z * k_per_split;
  const long long k_end = min(sh.K, k_begin + k_per_split);
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  float ra[4], rb[4];
  auto fetch = [&](long long k0) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int idx = tid + e * 256;
      {
        const int mm = kAKFast ? idx / kBK2 : idx % kT2, kk = kAKFast ? idx % kBK2 : idx / kT2;
        const long long m = m0 + mm, k = k0 + kk;
        ra[e] = (m < sh.M && k < k_end) ? fa(m, k) : 0.f;
      }
      {
        const int kk = kBNFast ? idx / kT2 : idx % kBK2, nn = kBNFast ? idx % kT2 : idx / kBK2;
        const long long k = k0 + kk;
        const int n = n0 + nn;
        rb[e] = (k < k_end && n < sh.N) ? fb(k, n) : 0.f;
      }
    }
  };
  auto stash = [&](int buf) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int idx = tid + e * 256;
      As[buf][kAKFast ? idx % kBK2 : idx / kT2][kAKFast ? idx / kBK2 : idx % kT2] = ra[e];
      Bs[buf][kBNFast ? idx / kT2 : idx % kBK2][kBNFast ? idx % kT2 : idx / kBK2] = rb[e];
    }
  };
  int buf = 0;
  if (k_begin < k_end) {
    fetch(k_begin);
    stash(0);
  }
  __syncthreads();
  for (long long k0 = k_begin; k0 < k_end; k0 += kBK2) {
    const bool more = k0 + kBK2 < k_end;
    if (more) fetch(k0 + kBK2);                       // global loads in flight under the FMAs below
#pragma unroll
    for (int kk = 0; kk < kBK2; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][kk][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (more) {
      stash(buf ^ 1);                                 // the other buffer: its last readers passed the previous barrier
      __syncthreads();
      buf ^= 1;
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const long long m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
      const int n = n0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
      if (m < sh.M && n < sh.N) fc(m, n, acc[i][j]);
    }
}

// [X (rows x k_x, ld ldx) | IN (rows x k_in, ld ldin, column offset folded into the pointer)]
struct ConcatA {
  const float* x; int ldx, k_x; const float* in; int ldin;
  __device__ float operator()(long long m, long long k) const {
    return k < k_x ? x[m * ldx + k] : in[m * ldin + (k - k_x)];
  }
};
struct ConcatAT {                  // transposed view for dW: A^T(k, row)
  ConcatA a;
  __device__ float operator()(long long k, long long m) const { return a(m, k); }
};
struct WeightB {                   // W (K x npad) row-major
  const float* w; int ld;
  __device__ float operator()(long long k, int n) const { return w[k * ld + n]; }
};
struct WeightBT {                  // W^T: (n, k) -> W[k][n]; "k" of the GEMM is the layer's n
  const float* w; int ld;
  __device__ float operator()(long long n, int k) const { return w[(long long)k * ld + n]; }
};
struct DZ {                        // dZ(m, n) = dY(m, n) * act'(Y(m, n))
  const float* dy; const float* y; int ld; int act;
  __device__ float operator()(long long m, long long n) const {
    return dy[m * ld + n] * act_grad_from_output(y[m * ld + n], act);
  }
};
struct DZB {                       // same as a B operand (k = row)
  DZ z;
  __device__ float operator()(long long m, int n) const { return z(m, n); }
};
struct StoreBiasAct {
  float* y; int ld; const float* bias; int act;
  __device__ void operator()(long long m, int n, float v) const { y[m * ld + n] = apply_act(v + bias[n], act); }
};
struct AccumSplit {                // dX / dIN: += into the producer's gradient buffer(s)
  float* dx; int ldx, k_x; float* din; int ldin;
  __device__ void operator()(long long m, int k, float v) const {
    if (k < k_x) dx[m * ldx + k] += v;
    else din[m * ldin + (k - k_x)] += v;
  }
};
struct AtomicAdd {
  float* c; int ld;
  __device__ void operator()(long long m, int n, float v) const { atomicAdd(c + m * ld + n, v); }
};

// db[n] += sum_m dZ(m, n)
__global__ void colsum_kernel(DZ z, long long rows, int n, float* __restrict__ db) {
  const int col = blockIdx.x * 32 + (threadIdx.x & 31);
  const int lane_row = threadIdx.x >> 5;              // 8 row lanes
  float s = 0.f;
  if (col < n)
    for (long long m = (long long)blockIdx.y * 8 + lane_row; m < rows; m += (long long)gridDim.y * 8) s += z(m, col);
  __shared__ float red[8][33];
  red[lane_row][threadIdx.x & 31] = s;
  __syncthreads();
  if (lane_row == 0 && col < n) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i][threadIdx.x & 31];
    atomicAdd(db + col, t);
  }
}

// ---------------------------------------------------------------------------
// Encoded inputs (R3 / R6) and their adjoints.
// ---------------------------------------------------------------------------
struct EncodeArgs {
  const float* origins; const float* directions; const float* z;   // rays / (B,S) z; z null = free points
  const float* pts_in;        // (rows,3) points to encode instead of o + z d (the warped points), or null
  const float* cond;          // (B, cond_stride)
  const float* window;        // (F) or null
  float* pts_out;             // (rows,3) the encoded point (tape), or null
  float* in;                  // (rows, ld)
  int F, ld, S, cond_stride, cond_off, n_cond;     // cond[cond_off .. +n_cond) follows the encoding
  long long rows;
};
__global__ void encode_kernel(const EncodeArgs a) {
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= a.rows) return;
  const long long ray = m / a.S;
  float x[3];
  if (a.pts_in) {
#pragma unroll
    for (int c = 0; c < 3; ++c) x[c] = a.pts_in[m * 3 + c];
  } else {
    const float z = a.z ? a.z[m] : 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) x[c] = a.origins[ray * 3 + c] + z * a.directions[ray * 3 + c];
  }
  if (a.pts_out) {
#pragma unroll
    for (int c = 0; c < 3; ++c) a.pts_out[m * 3 + c] = x[c];
  }
  float* o = a.in + m * a.ld;
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c] = x[c];
  const int nf = 6 * a.F;
  for (int f = 0; f < nf; ++f) {
    float v = posenc_feature(x, f);
    if (a.window) v = a.window[f / 6] * v;
    o[3 + f] = v;
  }
  const float* c = a.cond + ray * a.cond_stride + a.cond_off;
  for (int q = 0; q < a.n_cond; ++q) o[3 + nf + q] = c[q];
  for (int q = 3 + nf + a.n_cond; q < a.ld; ++q) o[q] = 0.f;
}

// dIN -> dx (rows,3) (+= when accumulate) and per-ray dcond (atomicAdd over the ray's samples).
struct EncodeBwdArgs {
  const float* pts;           // (rows,3) the point that was encoded
  const float* window; const float* din; int F, ld, S, cond_stride, cond_off, n_cond;
  float* dpts;                // (rows,3) or null
  float* dcond;               // (B, cond_stride) or null
  long long rows;
};
__global__ void encode_bwd_kernel(const EncodeBwdArgs a) {
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= a.rows) return;
  const float* g = a.din + m * a.ld;
  if (a.dpts) {
    float x[3], dx[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) { x[c] = a.pts[m * 3 + c]; dx[c] = g[c]; }
    for (int f = 0; f < a.F; ++f) {
      const float w = a.window ? a.window[f] : 1.f;
      const float s = exp2f((float)f);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float ang = x[c] * s;
        // d/dx sin(s x) = s cos(s x);  d/dx sin(s x + hp) = s cos(s x + hp)
        dx[c] = fmaf(g[3 + f * 6 + c] * w * s, cosf(ang), dx[c]);
        dx[c] = fmaf(g[3 + f * 6 + 3 + c] * w * s, cosf(ang + kHalfPiF), dx[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) a.dpts[m * 3 + c] = dx[c];
  }
  if (a.dcond) {
    const long long ray = m / a.S;
    for (int q = 0; q < a.n_cond; ++q) {
      const float v = g[3 + 6 * a.F + q];
      if (v != 0.f) atomicAdd(a.dcond + ray * a.cond_stride + a.cond_off + q, v);
    }
  }
}

// ---------------------------------------------------------------------------
// Warp tail (R5) and its adjoint by forward mode (one direction per head output:
// w, v, (pivot), (translation)).
// ---------------------------------------------------------------------------
struct WarpTailArgs {
  const float* head; int ld;  // (rows, ld): [w v (p) (t)] or the translation (3)
  const float* pts;           // (rows,3)
  float* warped;              // (rows,3)
  int warp_type, pivot, trans;
  long long rows;
};
__global__ void warp_tail_kernel(const WarpTailArgs a) {
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= a.rows) return;
  const float x[3] = {a.pts[m * 3], a.pts[m * 3 + 1], a.pts[m * 3 + 2]};
  float y[3];
  warp_tail(a.warp_type, a.head + m * a.ld, x, a.pivot != 0, a.trans != 0, y);
#pragma unroll
  for (int c = 0; c < 3; ++c) a.warped[m * 3 + c] = y[c];
}

// The SE(3) tail y at (h, x) with one tangent direction per head output:
// y[i].d[q] = d y_i / d head_q for q < nh (zero beyond; h[q] = 0 there).
__device__ __forceinline__ void se3_head_jacobian(const float h[12], const float x[3], int nh, bool pivot,
                                                  bool trans, Fwd<12, float> y[3]) {
  using S = Fwd<12, float>;
  S in[12], xs[3];
  for (int q = 0; q < 12; ++q) { in[q] = Num<S>::c(h[q]); if (q < nh) in[q].d[q] = 1.f; }
  for (int c = 0; c < 3; ++c) xs[c] = Num<S>::c(x[c]);
  se3_tail(in, xs, pivot, trans, y);
}

struct WarpTailBwdArgs {
  const float* head; int ld; const float* pts; const float* dwarped;   // (rows,3)
  float* dhead;               // (rows, ld): += the gradient of the head outputs
  int warp_type, pivot, trans;
  long long rows;
};
__global__ void warp_tail_bwd_kernel(const WarpTailBwdArgs a) {
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= a.rows) return;
  const float g[3] = {a.dwarped[m * 3], a.dwarped[m * 3 + 1], a.dwarped[m * 3 + 2]};
  float* dh = a.dhead + m * a.ld;
  if (a.warp_type != 2) {
#pragma unroll
    for (int c = 0; c < 3; ++c) dh[c] += g[c];       // warped = x + t
    return;
  }
  // The points carry no parameter upstream: x = o + z d with z a constant.
  const int nh = 6 + (a.pivot ? 3 : 0) + (a.trans ? 3 : 0);
  float h[12], x[3];
  Fwd<12, float> y[3];
  for (int q = 0; q < 12; ++q) h[q] = q < nh ? a.head[m * a.ld + q] : 0.f;
  for (int c = 0; c < 3; ++c) x[c] = a.pts[m * 3 + c];
  se3_head_jacobian(h, x, nh, a.pivot != 0, a.trans != 0, y);
  for (int q = 0; q < nh; ++q) dh[q] += g[0] * y[0].d[q] + g[1] * y[1].d[q] + g[2] * y[2].d[q];
}

// ---------------------------------------------------------------------------
// R8: raw -> (sigmoid(rgb), sigma_act(alpha)); the photometric loss; R9 adjoint.
// ---------------------------------------------------------------------------
__global__ void raw_to_samples_kernel(const float* __restrict__ rgb_raw, int ld_rgb,
                                      const float* __restrict__ alpha_raw, int ld_a, int sigma_act,
                                      float4* __restrict__ samples, long long rows) {
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= rows) return;
  float4 o;
  o.x = sigmoidf(rgb_raw[m * ld_rgb]); o.y = sigmoidf(rgb_raw[m * ld_rgb + 1]); o.z = sigmoidf(rgb_raw[m * ld_rgb + 2]);
  o.w = apply_act(alpha_raw[m * ld_a], sigma_act);
  samples[m] = o;
}

// loss = mean((rgb - target)^2) over the LOCAL batch (training.py:173), one thread per ray: adds the ray's share
// to *loss and writes its row of d_out (R,6), the cotangents of rgb, depth, med_depth and acc that seed
// composite_vjp_kernel.
__global__ void photometric_loss_kernel(const float* __restrict__ out, const float* __restrict__ target, float scale,
                                        int num_rays, float* __restrict__ d_out, float* __restrict__ loss) {
  const int ray = blockIdx.x * blockDim.x + threadIdx.x;
  if (ray >= num_rays) return;
  float l = 0.f;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float diff = out[ray * 6 + c] - target[ray * 3 + c];
    d_out[ray * 6 + c] = 2.f * diff * scale;
    l += diff * diff * scale;
  }
#pragma unroll
  for (int c = 3; c < 6; ++c) d_out[ray * 6 + c] = 0.f;
  atomicAdd(loss, l);
}

// The depth loss (no reference counterpart): L1 between the expected depth sum_i w_i z_i and a per-ray target,
// averaged over the rays whose target is finite and > 0.
__device__ __forceinline__ bool depth_target_valid(float t) { return isfinite(t) && t > 0.f; }

// The number of valid targets of the whole local batch into *count, before the tape's chunk loop: one block, a
// fixed reduction order, no host synchronisation.  Exact in float up to 2^24 rays.
__global__ void __launch_bounds__(256) depth_count_kernel(const float* __restrict__ target, int num_rays,
                                                          float* __restrict__ count) {
  __shared__ int part[8];
  int n = 0;
  for (int i = threadIdx.x; i < num_rays; i += 256) n += depth_target_valid(target[i]) ? 1 : 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = n;
  __syncthreads();
  if (threadIdx.x == 0) {
    int total = 0;
    for (int w = 0; w < 8; ++w) total += part[w];
    *count = (float)total;
  }
}

// One level's share, launched after photometric_loss_kernel: adds |depth - target| / count of each valid ray to
// *loss (unweighted) and writes weight * sign(depth - target) / count into column 3 of d_out, beside the
// photometric seed (sign(0) = 0: torch's subgradient of abs).  An invalid ray keeps the 0 photometric_loss_kernel
// wrote; with no valid ray nothing is added.
__global__ void __launch_bounds__(128) depth_loss_kernel(const float* __restrict__ out, const float* __restrict__ target,
                                                         const float* __restrict__ count, float weight, int num_rays,
                                                         float* __restrict__ d_out, float* __restrict__ loss) {
  const int ray = blockIdx.x * blockDim.x + threadIdx.x;
  float l = 0.f;
  if (ray < num_rays) {
    const float t = target[ray];
    if (depth_target_valid(t)) {
      const float inv = 1.f / *count;       // >= 1: this ray is counted
      const float e = out[ray * 6 + 3] - t;
      d_out[ray * 6 + 3] = e > 0.f ? weight * inv : (e < 0.f ? -weight * inv : 0.f);
      l = fabsf(e) * inv;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
  if ((threadIdx.x & 31) == 0 && l != 0.f) atomicAdd(loss, l);
}

// The adjoint of volumetric_rendering (model_utils.py:104-126) for given cotangents of its outputs: the seed of
// every backward (the caller's cotangents in nfb_render_vjp, photometric_loss_kernel's in training).  Per ray
//   d/dw_i = g_rgb . c_i - [white_bg] sum(g_rgb) + g_depth z_i + g_acc [i < S-1 or !sample_at_infinity] + g_w_i
// (the white background adds 1 - sum w, the acc before sample_at_infinity drops the last sample), then through
// w_i = alpha_i T_i to the raw rgb and density.  med_depth is piecewise constant: no cotangent.
struct CompositeVjpArgs {
  const float4* samples; const float* z; const float* directions;   // the taped forward
  const float* d_out;         // (R,6) cotangents of rgb, depth, med_depth (ignored), acc; or null
  const float* d_weights;     // (R,S) or null
  const float* rgb_raw; int ld_rgb; const float* alpha_raw; int ld_a;
  float* d_rgb_raw; float* d_alpha_raw;     // same layouts: = (not +=)
  int num_rays, S, white_bg, sample_at_infinity, sigma_act;
  // (R) or null: = dL/d|d| of each ray, through dist_i = dz_i |d| in alpha_i = 1 - exp(-sigma_i dist_i)
  float* d_dnorm;
};
// Shared memory: three floats per sample of each of kRaysPerBlock rays.
constexpr size_t composite_vjp_smem(int S) { return (size_t)kRaysPerBlock * 3 * S * sizeof(float); }

// One warp per ray, S <= kMaxSamples.  Lane l owns the contiguous samples [l p, l p + p), p = ceil(S / 32): the
// transmittance T_i = prod_{j<i} (1 - alpha_j + eps) is an exclusive product scan and sum_{k>i} gw_k w_k an
// exclusive suffix-sum scan, each as a serial pass over the lane's own samples around one shuffle scan of the
// 32 lane totals.
__global__ void __launch_bounds__(32 * kRaysPerBlock) composite_vjp_kernel(const CompositeVjpArgs a) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ray = blockIdx.x * kRaysPerBlock + warp;
  if (ray >= a.num_rays) return;
  extern __shared__ float sh[];
  const int S = a.S;
  float* gw = sh + warp * 3 * S;       // d / d w_i
  float* al = gw + S;                  // alpha_i
  float* tr = al + S;                  // T_i
  float g[3] = {0.f, 0.f, 0.f}, gd = 0.f, ga = 0.f;
  if (a.d_out) {
    const float* o = a.d_out + (size_t)ray * 6;
    g[0] = o[0]; g[1] = o[1]; g[2] = o[2]; gd = o[3]; ga = o[5];
  }
  const float gsum = g[0] + g[1] + g[2];
  const float dx = a.directions[ray * 3], dy = a.directions[ray * 3 + 1], dz = a.directions[ray * 3 + 2];
  const float dnorm = sqrtf(dx * dx + dy * dy + dz * dz);
  const float last = a.sample_at_infinity ? 1e10f : 1e-19f;
  const size_t base = (size_t)ray * S;
  for (int i = lane; i < S; i += 32) {
    const float4 c = a.samples[base + i];
    const float z = a.z[base + i];
    float v = g[0] * c.x + g[1] * c.y + g[2] * c.z;
    if (a.white_bg) v -= gsum;
    v += gd * z;
    if (i + 1 < S || !a.sample_at_infinity) v += ga;
    if (a.d_weights) v += a.d_weights[base + i];
    gw[i] = v;
    const float dist = (i + 1 < S) ? (a.z[base + i + 1] - z) : last;
    al[i] = -expm1f(-c.w * (dist * dnorm));
  }
  __syncwarp();
  const int per = (S + 31) / 32;
  const int b = min(S, lane * per), e = min(S, b + per);
  // T: product of the lane's factors, exclusive scan over the lanes, then the lane's own samples
  float p = 1.f;
  for (int i = b; i < e; ++i) p = p * (1.0f - al[i] + 1e-10f);
  float incl = p;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl = incl * u;
  }
  float t = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0) t = 1.f;
  float s = 0.f;                       // the lane's sum of gw_k w_k
  for (int i = b; i < e; ++i) {
    tr[i] = t;
    s += gw[i] * (al[i] * t);
    t = t * (1.0f - al[i] + 1e-10f);
  }
  // sum over the lanes to the right: an inclusive suffix scan, shifted by one lane.  (Not the inclusive sum minus
  // the lane's own: dalpha divides this sum by 1 - alpha_i + eps, down to 1e-10 behind an opaque sample, where
  // the cancellation's error of ~2^-24 |s| would swamp the true, tiny remainder.)
  float incl_suf = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float u = __shfl_down_sync(0xffffffffu, incl_suf, o);
    if (lane + o < 32) incl_suf += u;
  }
  float acc = __shfl_down_sync(0xffffffffu, incl_suf, 1);
  if (lane == 31) acc = 0.f;
  float sd = 0.f;                      // the lane's sum of dsigma_i sigma_i (d_dnorm)
  for (int i = e - 1; i >= b; --i) {
    const size_t m = base + i;
    const float4 c = a.samples[m];
    const float dist = ((i + 1 < S) ? (a.z[m + 1] - a.z[m]) : last) * dnorm;
    const float w = al[i] * tr[i];
    // w_i = alpha_i T_i: dL/dalpha_i = gw_i T_i - (sum_{k>i} gw_k w_k) / (1 - alpha_i + eps)
    const float dalpha = gw[i] * tr[i] - acc / (1.0f - al[i] + 1e-10f);
    acc += gw[i] * w;
    const float dsigma = dalpha * dist * expf(-c.w * dist);      // alpha = 1 - exp(-sigma dist)
    const float raw = a.alpha_raw[m * a.ld_a];
    float dact;                                                    // sigma = act(raw)
    if (a.sigma_act == kSoftplus) dact = 1.f / (1.f + expf(-raw));
    else if (a.sigma_act == kRelu) dact = raw > 0.f ? 1.f : 0.f;
    else dact = act_grad_from_output(c.w, a.sigma_act);
    a.d_alpha_raw[m * a.ld_a] = dsigma * dact;
    a.d_rgb_raw[m * a.ld_rgb + 0] = g[0] * w * c.x * (1.f - c.x);
    a.d_rgb_raw[m * a.ld_rgb + 1] = g[1] * w * c.y * (1.f - c.y);
    a.d_rgb_raw[m * a.ld_rgb + 2] = g[2] * w * c.z * (1.f - c.z);
    // dL/d|d| = sum_i dL/d dist_i dz_i = sum_i dsigma_i sigma_i / |d|.  The last sample (dz 1e10 or 1e-19)
    // counts like the others: where sigma is finite its exp(-sigma dist) makes it 0 (or leaves its true
    // value), as the reference's autograd does.
    if (a.d_dnorm) sd = fmaf(dsigma, c.w, sd);
  }
  if (a.d_dnorm) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sd += __shfl_xor_sync(0xffffffffu, sd, o);
    if (lane == 0) a.d_dnorm[ray] = sd / dnorm;
  }
}

// ---------------------------------------------------------------------------
// Ray adjoints (nfb_render_ray_vjp): the sample points x_{r,s} = o_r + z_{r,s} d_r with z a constant.
// ---------------------------------------------------------------------------
// The warp tail's direct term in the point gradient: dpts += (d warped / d x)^T dwarped at the head outputs
// of the tape, by forward mode on x (three tangents; the head is a constant here, its own adjoint is
// warp_tail_bwd_kernel's).  The identity for the TranslationField.
struct WarpTailDxArgs {
  const float* head; int ld; const float* pts; const float* dwarped;   // (rows,3)
  float* dpts;                // (rows,3): +=
  int warp_type, pivot, trans;
  long long rows;
};
__global__ void warp_tail_dx_kernel(const WarpTailDxArgs a) {
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= a.rows) return;
  const float g[3] = {a.dwarped[m * 3], a.dwarped[m * 3 + 1], a.dwarped[m * 3 + 2]};
  float* dx = a.dpts + m * 3;
  if (a.warp_type != 2) {
#pragma unroll
    for (int c = 0; c < 3; ++c) dx[c] += g[c];
    return;
  }
  using S = Fwd<3, float>;
  const int nh = 6 + (a.pivot ? 3 : 0) + (a.trans ? 3 : 0);
  S in[12], xs[3], y[3];
  for (int q = 0; q < 12; ++q) in[q] = Num<S>::c(q < nh ? a.head[m * a.ld + q] : 0.f);
  for (int c = 0; c < 3; ++c) { xs[c] = Num<S>::c(a.pts[m * 3 + c]); xs[c].d[c] = 1.f; }
  se3_tail(in, xs, a.pivot != 0, a.trans != 0, y);
#pragma unroll
  for (int c = 0; c < 3; ++c) dx[c] += g[0] * y[0].d[c] + g[1] * y[1].d[c] + g[2] * y[2].d[c];
}

// Per ray of S samples (one warp per ray, shuffle sums), += over the levels:
//   d_origins    += sum_s g_s
//   d_directions += sum_s z_s g_s + (dL/d|d|) d / |d|
// with g the level's point gradient (rows,3) and dL/d|d| from composite_vjp_kernel (nullable).
struct RayReduceArgs {
  const float* dpts; const float* z; const float* directions; const float* d_dnorm;
  float* d_origins; float* d_directions;   // (R,3), nullable
  int num_rays, S;
};
__global__ void __launch_bounds__(32 * kRaysPerBlock) ray_reduce_kernel(const RayReduceArgs a) {
  const int lane = threadIdx.x & 31;
  const int ray = blockIdx.x * kRaysPerBlock + (threadIdx.x >> 5);
  if (ray >= a.num_rays) return;
  float so[3] = {0.f, 0.f, 0.f}, sd[3] = {0.f, 0.f, 0.f};
  const size_t base = (size_t)ray * a.S;
  for (int i = lane; i < a.S; i += 32) {
    const float z = a.z[base + i];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float g = a.dpts[(base + i) * 3 + c];
      so[c] += g;
      sd[c] = fmaf(z, g, sd[c]);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      so[c] += __shfl_xor_sync(0xffffffffu, so[c], o);
      sd[c] += __shfl_xor_sync(0xffffffffu, sd[c], o);
    }
  if (lane != 0) return;
  if (a.d_origins)
#pragma unroll
    for (int c = 0; c < 3; ++c) a.d_origins[ray * 3 + c] += so[c];
  if (a.d_directions) {
    const float* d = a.directions + ray * 3;
    float k = 0.f;
    if (a.d_dnorm) k = a.d_dnorm[ray] / sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
#pragma unroll
    for (int c = 0; c < 3; ++c) a.d_directions[ray * 3 + c] += fmaf(k, d[c], sd[c]);
  }
}

// The adjoint of the viewdir block of the rgb condition (ray_cond_kernel: identity, then sin(2^f v_c [+pi/2])
// with no window), one thread per ray: out (B,3) = (accumulate ? += : =) dL/d viewdirs.
struct ViewdirVjpArgs {
  const float* dcond; int stride, off, F;  // the block is dcond[:, off .. off + 3 + 6F)
  const float* viewdirs; float* out;
  int accumulate, num_rays;
};
__global__ void viewdir_vjp_kernel(const ViewdirVjpArgs a) {
  const int ray = blockIdx.x * blockDim.x + threadIdx.x;
  if (ray >= a.num_rays) return;
  const float* g = a.dcond + (size_t)ray * a.stride + a.off;
  float v[3], dv[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) { v[c] = a.viewdirs[ray * 3 + c]; dv[c] = g[c]; }
  for (int f = 0; f < a.F; ++f) {
    const float s = exp2f((float)f);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float ang = v[c] * s;
      dv[c] = fmaf(g[3 + f * 6 + c] * s, cosf(ang), dv[c]);
      dv[c] = fmaf(g[3 + f * 6 + 3 + c] * s, cosf(ang + kHalfPiF), dv[c]);
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    if (a.accumulate) a.out[ray * 3 + c] += dv[c];
    else a.out[ray * 3 + c] = dv[c];
  }
}

// out[i] += x[i]
__global__ void add_into_kernel(float* __restrict__ out, const float* __restrict__ x, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] += x[i];
}

// ---------------------------------------------------------------------------
// Embedding gradients: dcond (B, stride) -> table rows (glo.py:41-53), the adjoint of
// ray_cond_kernel over the same layout.
// ---------------------------------------------------------------------------
struct CondBwdArgs {
  const float* dcond; int num_rays;
  const unsigned* warp_id; const unsigned* app_id; const unsigned* cam_id;
  float* d_warp_table; float* d_app_table; float* d_cam_table;
  int n_warp, n_app, n_cam;
  CondLayout layout;
  // d(warp block) / d(GLO row): 1 ('glo'), 1 - time_alpha ('blend'), 0 ('time': no table; nothing is scattered)
  float warp_scale;
};
__global__ void cond_bwd_kernel(const CondBwdArgs a) {
  const CondLayout& L = a.layout;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)a.num_rays * L.stride) return;
  const int ray = (int)(idx / L.stride);
  const float v = a.dcond[idx];
  if (v == 0.f) return;
  int j;
  const CondSource src = cond_source(L, (int)(idx - (long long)ray * L.stride), j);
  if (src == kCondWarp) {
    if (a.warp_scale != 0.f) atomicAdd(a.d_warp_table + embed_row(a.warp_id, ray, a.n_warp) * L.G + j, a.warp_scale * v);
  } else if (src == kCondApp) atomicAdd(a.d_app_table + embed_row(a.app_id, ray, a.n_app) * L.A + j, v);
  else if (src == kCondCam) atomicAdd(a.d_cam_table + embed_row(a.cam_id, ray, a.n_cam) * L.C + j, v);
  // view directions carry no parameter
}

// The same adjoint with metadata_encoded=True (models.py:198-213, warping.py:186-187): the condition vector holds
// the caller's per-ray codes, so dcond goes (+=) to the dense code gradients d_warp (B,G), d_app (B,A), d_cam
// (B,C).  An appearance code feeding several blocks (trunk, alpha and, under the use_alpha_condition quirk of
// models.py:206-207, rgb) receives their sum.  A code the call did not pass is row 0 of its table
// (ray_cond_kernel), whose gradient goes to that row; a null gradient pointer drops its code's share.
struct CondVjpEncodedArgs {
  const float* dcond; int num_rays;
  int has_warp, has_app, has_cam;                   // the call passed that code
  float* d_warp; float* d_app; float* d_cam;        // dense code gradients, or null
  float* d_warp_table; float* d_app_table; float* d_cam_table;   // row 0 of the tables, or null
  CondLayout layout;
};
__global__ void cond_vjp_encoded_kernel(const CondVjpEncodedArgs a) {
  const CondLayout& L = a.layout;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)a.num_rays * L.stride) return;
  const int ray = (int)(idx / L.stride);
  const float v = a.dcond[idx];
  if (v == 0.f) return;
  int j;
  const CondSource src = cond_source(L, (int)(idx - (long long)ray * L.stride), j);
  auto to = [&](int has, float* dense, float* table, int width) {
    if (has && dense) atomicAdd(dense + (size_t)ray * width + j, v);
    else if (!has && table) atomicAdd(table + j, v);
  };
  if (src == kCondWarp) to(a.has_warp, a.d_warp, a.d_warp_table, L.G);
  else if (src == kCondApp) to(a.has_app, a.d_app, a.d_app_table, L.A);
  else if (src == kCondCam) to(a.has_cam, a.d_cam, a.d_cam_table, L.C);
}

// ---------------------------------------------------------------------------
// The TimeEncoder of the 'time' / 'blend' warp metadata encoders on the time tape (train_api.cuh,
// time_forward / time_backward): its Dense layers run through net_forward / net_backward like every other
// MLP; these kernels are the stages around them.  The timestamp is a constant (it is data), so nothing is
// differentiated below the first layer.
// ---------------------------------------------------------------------------
struct TimeEncodeArgs {
  const float* time_f;        // (n) timestamps, or null
  const unsigned* time_id;    // (n) ids used as timestamps (float(id)), or null
  float window[20];           // cosine_easing_window(F, alpha)
  float* in;                  // (n, ld): the tape's input rows
  int din, ld, n;             // din = 1 + 2 F
};
__global__ void time_encode_kernel(const __grid_constant__ TimeEncodeArgs a) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)a.n * a.din) return;
  const int r = (int)(idx / a.din), k = (int)(idx - (long long)r * a.din);
  const float t = a.time_f ? a.time_f[r] : (float)a.time_id[r];
  a.in[(long long)r * a.ld + k] = time_encoding(t, k, a.window);
}

// cond[:, 0:G] = Y ('time'), or (1 - time_alpha) cond + time_alpha Y over the GLO rows already there
// ('blend', warping.py:132-133): the output stage of time_embed_kernel.
struct TimeCondArgs {
  const float* y; int ld;     // (n, ld): the TimeEncoder's output layer
  float* cond; int stride, G, n;
  int blend; float time_alpha;
};
__global__ void time_cond_kernel(const TimeCondArgs a) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)a.n * a.G) return;
  const int r = (int)(idx / a.G), q = (int)(idx - (long long)r * a.G);
  float v = a.y[(long long)r * a.ld + q];
  float* c = a.cond + (long long)r * a.stride + q;
  if (a.blend) v = (1.0f - a.time_alpha) * *c + a.time_alpha * v;
  *c = v;
}

// Its adjoint towards the TimeEncoder: dY = dcond[:, 0:G] ('time'), time_alpha dcond[:, 0:G] ('blend').
// (The GLO rows' share, (1 - time_alpha) dcond, is cond_bwd_kernel's warp_scale.)
__global__ void time_cond_bwd_kernel(const float* __restrict__ dcond, int stride, int G, float scale,
                                     float* __restrict__ dy, int ld, int n) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)n * G) return;
  const int r = (int)(idx / G), q = (int)(idx - (long long)r * G);
  dy[(long long)r * ld + q] = scale * dcond[(long long)r * stride + q];
}

// packed (K x ld, column offset) gradient -> the caller's dense (rows x cols) tensor (+=).
__global__ void unpack_grad_kernel(const float* __restrict__ packed, float* __restrict__ dst, long long rows,
                                   long long cols, int ld, int c_off) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * cols) return;
  const long long r = idx / cols, c = idx - r * cols;
  dst[idx] += packed[r * ld + c_off + c];
}

// flax.optim.Adam (beta1 0.9, beta2 0.999, eps 1e-8, no weight decay): one fused pass.
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                            float* __restrict__ v, long long n, float lr, float b1, float b2, float eps,
                            float bc1, float bc2) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float gi = g[i];
  const float mi = b1 * m[i] + (1.f - b1) * gi;
  const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
  m[i] = mi; v[i] = vi;
  const float mhat = mi / bc1, vhat = vi / bc2;
  p[i] = p[i] - lr * mhat / (sqrtf(vhat) + eps);
}

}  // namespace train
}  // namespace nfb
