// Fused per-sample field evaluation, fp32 CUDA-core path (NFB_PREC_FP32).
//
// One CTA evaluates a tile of 64 consecutive (ray, sample) rows end to end:
//   point = o + z d                                   (model_utils.py:72-73)
//   windowed posenc + GLO code -> warp MLP -> SE(3)/translation warp
//                                                     (warping.py:322-353)
//   posenc of the warped point + per-ray conditions -> NerfMLP
//                                                     (modules.py:104-169)
//   sigmoid(rgb), sigma_activation(alpha)             (models.py:276-277)
// and writes 16 B per sample (r, g, b, sigma).  Activations never leave shared
// memory; weights stream from L2 through a cp.async double buffer.
//
// Shared-memory activations are kept TRANSPOSED, X[k][row] with a padded row
// stride of 68 floats, so that a thread's 8 rows are two 128-bit loads
// (broadcast across the warp) and the epilogue's column-strided 128-bit stores
// are bank-conflict free.  Thread mapping: warp g owns rows 8g..8g+7, lane l
// owns columns l, l+32, ... (8 x NJ register tile, NJ = npad / 32).
#pragma once
#include "common.cuh"

namespace nfb {

constexpr int kTM = 64;             // rows per tile
constexpr int kRS = kTM + 4;        // padded row stride (floats)
constexpr int kKS = 16;             // K rows per weight slab
constexpr int kSimtThreads = 256;
constexpr int kSimtSmemFloats =
    2 * kMaxWidth * kRS      // B0, B1
    + kMaxIn * kRS           // IN
    + 64 * kRS               // OUT (2 slots x 32 columns)
    + 2 * kKS * kMaxWidth    // weight slabs
    + 3 * kTM;               // warped points
constexpr int kSimtSmemBytes = kSimtSmemFloats * 4;

// FieldArgs::debug bits.  kDebugTimeout: the weight producer of the tensor-core kernel first waits
// on a barrier that never completes.  kDebugOneRowBlock: the tensor-core warp pass runs in 128-row
// tiles (kMB = 1) even where the warp net fits 256-row tiles.
constexpr int kDebugTimeout = 8, kDebugOneRowBlock = 16;

struct FieldArgs {
  const float* params;       // packed weights/biases
  const float* origins;      // (B,3)
  const float* directions;   // (B,3)
  const float* z_vals;       // (B,S) or nullptr (= 0: free-point mode)
  const float* points;       // (B*S, 3) already-warped sample points, or nullptr.  When set, a row's
                             // point is read from here instead of o + z d and the warp net is skipped;
                             // z_vals still gives the composite's dists and depth.
  const float* cond;         // (B, cond_stride) per-ray [glo | tc | ac | rc]
  const float* window;       // (Fw) cosine-easing window
  float* samples;            // (B*S, 4) out: r,g,b,sigma  (nullable)
  float* warped;             // (B*S, 3) out: warped points (nullable)
  long long num_rows;        // B*S
  int samples_per_ray;       // S
  int use_warp;              // run the warp net
  int warp_only;             // stop after the warp (nfb_warp_forward)
  int debug;                 // test hooks: kDebugTimeout (nfb_debug_provoke_timeout), kDebugOneRowBlock
                             // (nfb_debug_one_row_block)
  // fp16x3 kernel: volumetric rendering fused into the rgb epilogue (samples_per_ray a multiple
  // of 128): per-ray (rgb3, depth, med_depth, acc) and, optionally, the weights.
  float* ray_out;            // (B,6) or nullptr = no fused composite
  float* ray_weights;        // (B,S) or nullptr
  int white_bg, sample_at_infinity;
  // tensor-core NeRF pass of a model with a bottleneck (ray_bias_kernel): the bias of the layer with
  // TcStep::ray_bias, (B, 128 n_chunks), and with an alpha condition the alpha head's constant, (B)
  const float* ray_bias;
  const float* ray_alpha;
};

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() {
  asm volatile("cp.async.commit_group;\n" ::);
}
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

struct SimtSmem {
  float* buf[2];
  float* in;
  float* out;
  float* slab[2];
  float* wp;
  __device__ float* ptr(int id) const {
    return id == kB0 ? buf[0] : id == kB1 ? buf[1] : id == kOut0 ? out : out + 32 * kRS;
  }
};

// One Dense step on the CTA's 64-row tile.
template <int NJ>
__device__ __forceinline__ void simt_dense(const Step& st, const float* __restrict__ params,
                                           const SimtSmem& sm) {
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int g = tid >> 5;                 // row group: rows 8g..8g+7
  const int npad = 32 * NJ;
  const int ktot = st.k_x + st.k_in;
  const float* __restrict__ W = params + st.w_off;
  const float* src = sm.ptr(st.src);
  const float* in = sm.in + st.in_off * kRS;

  float acc[8][NJ];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < NJ; ++j) acc[i][j] = 0.f;

  const int nslab = (ktot + kKS - 1) / kKS;
  auto load_slab = [&](int s) {
    const int k0 = s * kKS;
    const int rows = min(kKS, ktot - k0);
    const int chunks = rows * (npad / 4);
    float* dst = sm.slab[s & 1];
    const float* gsrc = W + (size_t)k0 * npad;
    for (int c = tid; c < chunks; c += kSimtThreads) cp_async16(dst + c * 4, gsrc + c * 4);
    cp_async_commit();
  };

  load_slab(0);
  for (int s = 0; s < nslab; ++s) {
    if (s + 1 < nslab) {
      load_slab(s + 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const float* slab = sm.slab[s & 1];
    const int k0 = s * kKS;
    const int rows = min(kKS, ktot - k0);
#pragma unroll 4
    for (int kk = 0; kk < rows; ++kk) {
      const int k = k0 + kk;
      const float* ap = (k < st.k_x) ? (src + k * kRS) : (in + (k - st.k_x) * kRS);
      const float4 a0 = *reinterpret_cast<const float4*>(ap + 8 * g);
      const float4 a1 = *reinterpret_cast<const float4*>(ap + 8 * g + 4);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      float b[NJ];
#pragma unroll
      for (int j = 0; j < NJ; ++j) b[j] = slab[kk * npad + lane + 32 * j];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < NJ; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }

  // Epilogue: bias + activation, transposed store.
  float* dst = sm.ptr(st.dst);
  const int act = st.act;
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int col = lane + 32 * j;
    const float bias = __ldg(params + st.b_off + col);
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = apply_act(acc[i][j] + bias, act);
    float* p = dst + col * kRS + 8 * g;
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
  }
  __syncthreads();
}

__device__ __forceinline__ void simt_run_net(const Net& net, const float* params,
                                             const SimtSmem& sm) {
  for (int s = 0; s < net.n_steps; ++s) {
    const Step& st = net.steps[s];
    switch (st.npad / 32) {
      case 1: simt_dense<1>(st, params, sm); break;
      case 2: simt_dense<2>(st, params, sm); break;
      case 3: simt_dense<3>(st, params, sm); break;
      case 4: simt_dense<4>(st, params, sm); break;
      case 5: simt_dense<5>(st, params, sm); break;
      case 6: simt_dense<6>(st, params, sm); break;
      case 7: simt_dense<7>(st, params, sm); break;
      default: simt_dense<8>(st, params, sm); break;
    }
  }
}

__global__ void __launch_bounds__(kSimtThreads, 1)
field_simt_kernel(const __grid_constant__ FieldProgram prog, const FieldArgs args) {
  extern __shared__ __align__(16) float smem[];
  SimtSmem sm;
  sm.buf[0] = smem;
  sm.buf[1] = sm.buf[0] + kMaxWidth * kRS;
  sm.in = sm.buf[1] + kMaxWidth * kRS;
  sm.out = sm.in + kMaxIn * kRS;
  sm.slab[0] = sm.out + 64 * kRS;
  sm.slab[1] = sm.slab[0] + kKS * kMaxWidth;
  sm.wp = sm.slab[1] + kKS * kMaxWidth;

  const int tid = threadIdx.x;
  const int r = tid & (kTM - 1);        // row within the tile
  const int part = tid >> 6;            // 0..3: feature slice handled for row r
  const long long row0 = (long long)blockIdx.x * kTM;
  long long m = row0 + r;
  const bool valid = m < args.num_rows;
  if (!valid) m = args.num_rows - 1;    // compute on a valid row, never store
  const int S = args.samples_per_ray;
  const long long ray = m / S;

  // Sample point x = o + z d, or the given (warped) point.
  float x[3];
  if (args.points) {
#pragma unroll
    for (int c = 0; c < 3; ++c) x[c] = __ldg(args.points + m * 3 + c);
  } else {
    const float z = args.z_vals ? __ldg(args.z_vals + m) : 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c)
      x[c] = __ldg(args.origins + ray * 3 + c) + z * __ldg(args.directions + ray * 3 + c);
  }
  const float* cond = args.cond + ray * prog.cond_stride;

  const bool do_warp = args.use_warp && prog.warp_type != 0 && !args.points;
  if (do_warp) {
    // Warp-field inputs: identity, windowed posenc, GLO code (warping.py:325-326,
    // modules.py:240-272).
    const int nf = 6 * prog.Fw;
    if (part == 0) {
#pragma unroll
      for (int c = 0; c < 3; ++c) sm.in[c * kRS + r] = x[c];
    }
    for (int f = part; f < nf; f += 4)
      sm.in[(3 + f) * kRS + r] = __ldg(args.window + f / 6) * posenc_feature(x, f);
    for (int q = part; q < prog.G; q += 4) sm.in[(3 + nf + q) * kRS + r] = __ldg(cond + q);
    __syncthreads();
    simt_run_net(prog.warp, args.params, sm);
    if (part == 0) {
      float h[12], y[3];
#pragma unroll
      for (int q = 0; q < 12; ++q) h[q] = sm.out[q * kRS + r];
      warp_tail(prog.warp_type, h, x, prog.warp_pivot, prog.warp_trans, y);
#pragma unroll
      for (int c = 0; c < 3; ++c) sm.wp[c * kTM + r] = y[c];
      if (args.warped && valid) {
#pragma unroll
        for (int c = 0; c < 3; ++c) args.warped[m * 3 + c] = y[c];
      }
    }
    __syncthreads();
#pragma unroll
    for (int c = 0; c < 3; ++c) x[c] = sm.wp[c * kTM + r];
  } else if (args.warped && valid && part == 0) {
#pragma unroll
    for (int c = 0; c < 3; ++c) args.warped[m * 3 + c] = x[c];
  }
  if (args.warp_only) return;

  // NerfMLP inputs: point posenc, then the per-ray condition blocks.
  {
    const int nf = 6 * prog.Fp;
    if (part == 0) {
#pragma unroll
      for (int c = 0; c < 3; ++c) sm.in[c * kRS + r] = x[c];
    }
    for (int f = part; f < nf; f += 4) sm.in[(3 + f) * kRS + r] = posenc_feature(x, f);
    const int nc = prog.tc + prog.ac + prog.rc;
    for (int q = part; q < nc; q += 4)
      sm.in[(prog.Dp + q) * kRS + r] = __ldg(cond + prog.G + q);
    __syncthreads();
  }
  simt_run_net(prog.nerf, args.params, sm);

  if (part == 0 && valid && args.samples) {
    const float* oa = sm.ptr(prog.alpha_slot);
    const float* orgb = sm.ptr(prog.rgb_slot);
    float4 o;
    o.x = sigmoidf(orgb[0 * kRS + r]);
    o.y = sigmoidf(orgb[1 * kRS + r]);
    o.z = sigmoidf(orgb[2 * kRS + r]);
    o.w = apply_act(oa[r], prog.sigma_act);
    reinterpret_cast<float4*>(args.samples)[m] = o;
  }
}

}  // namespace nfb
