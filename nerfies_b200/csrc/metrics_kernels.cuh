// Per-frame metrics of eval.py:process_batch on the GPU (eval.py:58-62, 120-122, 140):
//   MS-SSIM   = tf.image.ssim_multiscale(target, image, max_val=1) with TF's defaults
//               (tensorflow/python/ops/image_ops_impl.py: ssim_multiscale, _ssim_per_channel,
//               _ssim_helper, _fspecial_gauss);
//   MSE       = mean((image - target)^2);
//   depth_abs = nanmean(|depth_target - depth|) per pixel.
// One call = 4 downsample launches (the level-0 one also sums the squared error and the depth
// error, so MSE and depth cost no extra pass), one filter + SSIM launch per scale that keeps the
// filtered moments in shared memory and writes one fp64 partial per CTA and channel, and one
// finalize launch that sums the partials in a fixed order.  No atomics: results are bitwise
// reproducible.  Images are (N, h, w, C) float32, channels interleaved.
#pragma once

namespace nfb {
namespace metrics {

constexpr int kScales = 5;
constexpr int kTaps = 11;                  // _fspecial_gauss(11, 1.5)
constexpr int kHalo = kTaps - 1;           // padding='VALID': output (h - 10) x (w - 10)
constexpr int kMinSize = 161;              // 161 -> 81 -> 41 -> 21 -> 11: scale 4 is still >= 11
constexpr int kTileW = 32, kTileH = 16;    // output pixels of one SSIM CTA
constexpr int kInW = kTileW + kHalo, kInH = kTileH + kHalo;
constexpr int kThreads = 256;
__constant__ double kPowerFactors[kScales] = {0.0448, 0.2856, 0.3001, 0.2363, 0.1333};

struct SsimArgs {
  const float* x;          // (N, h, w, C) one level of each image
  const float* y;
  int h, w, tiles_x, tiles_y;
  double* part;            // (N, C, tiles_y * tiles_x, 2): sums of luminance * cs and of cs
  float g[kTaps];          // normalised 1-D Gaussian
};

struct PoolArgs {
  const float* x;          // (N, h, w, C) level k
  const float* y;
  float* x_out;            // (N, ceil(h/2), ceil(w/2), C) level k + 1
  float* y_out;
  int h, w;
  // level 0 only (nullptr otherwise): per-CTA sums over the pixels of level 0
  double* err_part;        // (N, gridDim.x, 3): sum (x - y)^2, sum |dt - d| (non-NaN), count
  const float* depth;      // (N, h, w) or nullptr
  const float* depth_target;
};

struct FinalArgs {
  int C, pool_blocks;
  int tiles[kScales];
  long long outputs[kScales];   // (h_k - 10) (w_k - 10)
  long long values;             // h w C of level 0
  const double* part[kScales];
  const double* err_part;
  float* ms_ssim;               // (N) each nullable
  float* mse;
  float* depth_abs;
};

// Sum of one double per thread of a kThreads block, in a fixed order; the result is valid in
// every thread.  s_red holds kThreads / 32 doubles.
__device__ __forceinline__ double block_sum(double v, double* s_red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();                                   // s_red may still be read by a previous call
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
#pragma unroll
  for (int i = 0; i < kThreads / 32; ++i) s += s_red[i];
  return s;
}

// Level k -> k + 1 (ssim_multiscale between scales): pad an odd side at its end by one in
// SYMMETRIC mode (the edge pixel again), then avg_pool 2x2 stride 2 VALID.  One thread per output
// pixel of image blockIdx.y.  On level 0 every input pixel belongs to exactly one thread, which
// also accumulates its squared error and depth error (a padded duplicate is not counted).
template <int C>
__global__ void __launch_bounds__(kThreads) downsample_kernel(const PoolArgs a) {
  __shared__ double s_red[kThreads / 32];
  const int n = blockIdx.y;
  const int h2 = (a.h + 1) >> 1, w2 = (a.w + 1) >> 1;
  const long long p = (long long)blockIdx.x * kThreads + threadIdx.x;
  double sq = 0.0, dsum = 0.0, dcnt = 0.0;
  if (p < (long long)h2 * w2) {
    const long long i = p / w2, j = p - i * w2;
    const long long r0 = 2 * i, c0 = 2 * j;
    const bool row1 = r0 + 1 < a.h, col1 = c0 + 1 < a.w;
    const long long img = (long long)n * a.h * a.w;
    const long long q00 = img + r0 * a.w + c0;
    const long long q01 = col1 ? q00 + 1 : q00;
    const long long q10 = row1 ? q00 + a.w : q00;
    const long long q11 = row1 ? q01 + a.w : q01;
    const long long o = ((long long)n * h2 * w2 + p) * C;
    const bool stats = a.err_part != nullptr;
#pragma unroll
    for (int ch = 0; ch < C; ++ch) {
      const float x00 = __ldg(a.x + q00 * C + ch), x01 = __ldg(a.x + q01 * C + ch);
      const float x10 = __ldg(a.x + q10 * C + ch), x11 = __ldg(a.x + q11 * C + ch);
      const float y00 = __ldg(a.y + q00 * C + ch), y01 = __ldg(a.y + q01 * C + ch);
      const float y10 = __ldg(a.y + q10 * C + ch), y11 = __ldg(a.y + q11 * C + ch);
      a.x_out[o + ch] = ((x00 + x01) + (x10 + x11)) * 0.25f;
      a.y_out[o + ch] = ((y00 + y01) + (y10 + y11)) * 0.25f;
      if (stats) {
        float d = x00 - y00;
        sq += (double)(d * d);
        if (col1) { d = x01 - y01; sq += (double)(d * d); }
        if (row1) { d = x10 - y10; sq += (double)(d * d); }
        if (row1 && col1) { d = x11 - y11; sq += (double)(d * d); }
      }
    }
    if (stats && a.depth) {
      const long long q[4] = {q00, q01, q10, q11};
      const bool real[4] = {true, col1, row1, row1 && col1};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float e = fabsf(__ldg(a.depth_target + q[k]) - __ldg(a.depth + q[k]));
        if (real[k] && !isnan(e)) { dsum += (double)e; dcnt += 1.0; }
      }
    }
  }
  if (a.err_part == nullptr) return;                 // uniform over the grid
  sq = block_sum(sq, s_red);
  dsum = block_sum(dsum, s_red);
  dcnt = block_sum(dcnt, s_red);
  if (threadIdx.x == 0) {
    double* out = a.err_part + ((long long)n * gridDim.x + blockIdx.x) * 3;
    out[0] = sq; out[1] = dsum; out[2] = dcnt;
  }
}

// One scale of _ssim_per_channel for a kTileH x kTileW block of output pixels of image
// blockIdx.z: load the tile and its 10-pixel halo of both images (all channels), filter x, y,
// x*y and x^2 + y^2 with the separable Gaussian (along w, then along h; fp32), evaluate
// _ssim_helper per pixel and write this CTA's per-channel sums of luminance * cs and cs.
//
// Both images are first shifted by the tile's top-left pixel (a per-channel constant; each image
// by its own).  Covariances do not change under a shift, but their fp32 evaluation as
// F(xy) - F(x)F(y) does: unshifted, the difference of two ~mu^2 quantities is taken over c2 =
// 9e-4, which moves cs by ~1e-4 on flat regions (TF's own fp32 result included).  The luminance
// uses the unshifted means.  Identical images still give exactly 1: x' == y' bit for bit.
template <int C>
__global__ void __launch_bounds__(kThreads) ssim_level_kernel(const SsimArgs a) {
  __shared__ float s_x[C][kInH][kInW];
  __shared__ float s_y[C][kInH][kInW];
  __shared__ float s_h[4][kInH][kTileW];             // horizontally filtered x, y, xy, x^2 + y^2
  __shared__ float s_ref[2][C];
  __shared__ double s_red[kThreads / 32];
  const int n = blockIdx.z;
  const int r0 = blockIdx.y * kTileH, c0 = blockIdx.x * kTileW;
  const int oh = a.h - kHalo, ow = a.w - kHalo;
  const long long img = (long long)n * a.h * a.w * C;
  const long long corner = img + ((long long)r0 * a.w + c0) * C;
  if (threadIdx.x < C) {
    s_ref[0][threadIdx.x] = __ldg(a.x + corner + threadIdx.x);
    s_ref[1][threadIdx.x] = __ldg(a.y + corner + threadIdx.x);
  }
  __syncthreads();
  // Pixels outside the image only feed outputs outside [0, oh) x [0, ow), which are not summed.
  for (int e = threadIdx.x; e < kInH * kInW * C; e += kThreads) {
    const int r = e / (kInW * C), rem = e - r * (kInW * C);
    const int col = rem / C, ch = rem - col * C;
    float vx = 0.f, vy = 0.f;
    if (r0 + r < a.h && c0 + col < a.w) {
      const long long gi = corner + (long long)r * a.w * C + rem;
      vx = __ldg(a.x + gi) - s_ref[0][ch];
      vy = __ldg(a.y + gi) - s_ref[1][ch];
    }
    s_x[ch][r][col] = vx;
    s_y[ch][r][col] = vy;
  }
  const float c1 = 0.01f * 0.01f, c2 = 0.03f * 0.03f;   // (k * max_val)^2, max_val = 1
  const int tile = blockIdx.y * a.tiles_x + blockIdx.x;
  const int tiles = a.tiles_x * a.tiles_y;
#pragma unroll 1
  for (int ch = 0; ch < C; ++ch) {
    __syncthreads();                                  // s_x / s_y loaded, s_h free
    for (int e = threadIdx.x; e < kInH * kTileW; e += kThreads) {
      const int r = e / kTileW, j = e - r * kTileW;
      float mx = 0.f, my = 0.f, mxy = 0.f, mss = 0.f;
#pragma unroll
      for (int t = 0; t < kTaps; ++t) {
        const float xv = s_x[ch][r][j + t], yv = s_y[ch][r][j + t], g = a.g[t];
        mx = mx + g * xv;
        my = my + g * yv;
        mxy = mxy + g * (xv * yv);
        mss = mss + g * (xv * xv + yv * yv);
      }
      s_h[0][r][j] = mx; s_h[1][r][j] = my; s_h[2][r][j] = mxy; s_h[3][r][j] = mss;
    }
    __syncthreads();
    double lcs_sum = 0.0, cs_sum = 0.0;
    for (int e = threadIdx.x; e < kTileH * kTileW; e += kThreads) {
      const int i = e / kTileW, j = e - i * kTileW;
      if (r0 + i >= oh || c0 + j >= ow) continue;
      float mx = 0.f, my = 0.f, mxy = 0.f, mss = 0.f;
#pragma unroll
      for (int t = 0; t < kTaps; ++t) {
        const float g = a.g[t];
        mx = mx + g * s_h[0][i + t][j];
        my = my + g * s_h[1][i + t][j];
        mxy = mxy + g * s_h[2][i + t][j];
        mss = mss + g * s_h[3][i + t][j];
      }
      // _ssim_helper, in its expression order
      const float mean0 = s_ref[0][ch] + mx, mean1 = s_ref[1][ch] + my;
      const float lum = (mean0 * mean1 * 2.f + c1) / (mean0 * mean0 + mean1 * mean1 + c1);
      const float num0 = mx * my * 2.f, den0 = mx * mx + my * my;
      const float num1 = mxy * 2.f, den1 = mss;
      const float cs = (num1 - num0 + c2) / (den1 - den0 + c2);
      lcs_sum += (double)(lum * cs);
      cs_sum += (double)cs;
    }
    lcs_sum = block_sum(lcs_sum, s_red);
    cs_sum = block_sum(cs_sum, s_red);
    if (threadIdx.x == 0) {
      double* out = a.part + (((long long)n * C + ch) * tiles + tile) * 2;
      out[0] = lcs_sum; out[1] = cs_sum;
    }
  }
}

// Sum of part[i * stride] for i in [0, count) over the block, in a fixed order.
__device__ __forceinline__ double sum_slots(const double* part, long long count, int stride, double* s_red) {
  double v = 0.0;
  for (long long i = threadIdx.x; i < count; i += kThreads) v += part[i * stride];
  return block_sum(v, s_red);
}

// Image blockIdx.x: per-channel means of every scale, then ssim_multiscale's combination
//   mcs = [relu(cs_0), ..., relu(cs_3), relu(ssim_4)],  ms_ssim = mean_c prod_k mcs_k ^ p_k,
// and MSE / depth_abs from the level-0 downsample partials.  fp64 throughout.
__global__ void __launch_bounds__(kThreads) finalize_kernel(const FinalArgs a) {
  __shared__ double s_red[kThreads / 32];
  const int n = blockIdx.x;
  if (a.ms_ssim) {
    double ms = 0.0;
    for (int ch = 0; ch < a.C; ++ch) {
      double prod = 1.0;
      for (int k = 0; k < kScales; ++k) {
        const double* p = a.part[k] + ((long long)n * a.C + ch) * a.tiles[k] * 2;
        const double s = sum_slots(p + (k == kScales - 1 ? 0 : 1), a.tiles[k], 2, s_red);
        prod *= pow(fmax(s / (double)a.outputs[k], 0.0), kPowerFactors[k]);
      }
      ms += prod;
    }
    if (threadIdx.x == 0) a.ms_ssim[n] = (float)(ms / a.C);
  }
  const double* e = a.err_part + (long long)n * a.pool_blocks * 3;
  const double sq = sum_slots(e, a.pool_blocks, 3, s_red);
  const double dsum = sum_slots(e + 1, a.pool_blocks, 3, s_red);
  const double dcnt = sum_slots(e + 2, a.pool_blocks, 3, s_red);
  if (threadIdx.x == 0) {
    if (a.mse) a.mse[n] = (float)(sq / (double)a.values);
    if (a.depth_abs) a.depth_abs[n] = dcnt > 0.0 ? (float)(dsum / dcnt) : __int_as_float(0x7fc00000);
  }
}

}  // namespace metrics
}  // namespace nfb
