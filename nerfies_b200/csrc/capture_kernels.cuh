// Capture processing on the GPU: the hot steps of the reference's capture notebook
// (notebooks/Nerfies_Capture_Processing.ipynb, "Resize images" through "Compute near/far planes").
//   frame_pyramid_kernel   every level of one uint8 RGB frame, read once
//   blur_sums_kernel       grey -> 3x3 Laplacian -> exact int64 sum and sum of squares per frame
//   blur_finalize_kernel   fp64 variance of the Laplacian per frame
//   near_far_*             per-camera depth quantiles of the projected point cloud by radix select
// DESIGN.md §5.5d records what each one reproduces and why.
#pragma once
#include "../../include/nerfies_b200.h"
#include "camera_kernels.cuh"

namespace nfb {
namespace capture {

constexpr int kMaxLevels = 8;

// ---------------------------------------------------------------------------------------------
// Pyramid.  cv2.resize(image, (w, h)) with its default INTER_LINEAR for an even factor s maps each
// output pixel to the rounded mean (a + b + c + d + 2) >> 2 of the 2x2 block at source offsets
// s/2 - 1 and s/2; scale 1 is the frame itself.  One thread owns one S x S block of the source
// (S the largest scale) and writes every level's pixels inside it.
// ---------------------------------------------------------------------------------------------
struct PyramidArgs {
  const unsigned char* src;
  long long src_pitch;                 // bytes between source rows
  int height, width, max_scale;        // cropped size, a multiple of max_scale
  int num_levels;
  int scale[kMaxLevels];
  unsigned char* dst[kMaxLevels];      // (height / scale, width / scale, 3), contiguous
};

__global__ void __launch_bounds__(256) frame_pyramid_kernel(const PyramidArgs a) {
  const int S = a.max_scale;
  const int bw = a.width / S;
  const long long b = (long long)blockIdx.x * 256 + threadIdx.x;
  if (b >= (long long)bw * (a.height / S)) return;
  const int by = (int)(b / bw), bx = (int)(b - (long long)by * bw);
  const int y0 = by * S, x0 = bx * S;
  for (int l = 0; l < a.num_levels; ++l) {
    const int s = a.scale[l];
    const int ow = a.width / s;
    unsigned char* dst = a.dst[l];
    if (s == 1) {
      for (int r = 0; r < S; ++r) {
        const unsigned char* in = a.src + (long long)(y0 + r) * a.src_pitch + 3LL * x0;
        unsigned char* out = dst + ((long long)(y0 + r) * ow + x0) * 3;
        for (int e = 0; e < 3 * S; ++e) out[e] = __ldg(in + e);
      }
      continue;
    }
    const int n = S / s, h = s / 2 - 1;
    for (int i = 0; i < n; ++i) {
      const unsigned char* r0 = a.src + (long long)(y0 + i * s + h) * a.src_pitch;
      const unsigned char* r1 = r0 + a.src_pitch;
      unsigned char* out = dst + ((long long)(y0 / s + i) * ow + x0 / s) * 3;
      for (int j = 0; j < n; ++j) {
        const int cx = 3 * (x0 + j * s + h);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
          const int sum = __ldg(r0 + cx + ch) + __ldg(r0 + cx + 3 + ch) + __ldg(r1 + cx + ch) +
                          __ldg(r1 + cx + 3 + ch);
          out[3 * j + ch] = (unsigned char)((sum + 2) >> 2);
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Blur score: cv2.Laplacian(cv2.cvtColor(rgb, COLOR_RGB2GRAY), CV_64F).var().
//   grey = (9798 R + 19235 G + 3735 B + 16384) >> 15   (cv2's 15-bit rule, exact for all 2^24 triples)
//   lap  = g[y-1][x] + g[y+1][x] + g[y][x-1] + g[y][x+1] - 4 g[y][x], BORDER_REFLECT_101
// Integer values: the int64 sums of lap and lap^2 are exact in any order, so the launch shape does
// not change the result.
// ---------------------------------------------------------------------------------------------
struct BlurArgs {
  const unsigned char* frames;   // (num_frames, height, width, 3)
  int num_frames, height, width;
  unsigned long long* sums;      // (num_frames, 2): sum, sum of squares (two's complement int64)
  double* scores;                // (num_frames)
};

__device__ __forceinline__ int reflect101(int i, int n) {
  if (n == 1) return 0;
  if (i < 0) return -i;
  if (i >= n) return 2 * n - 2 - i;
  return i;
}

__device__ __forceinline__ int grey_of(const unsigned char* f, int width, int y, int x) {
  const unsigned char* p = f + 3LL * ((long long)y * width + x);
  return (9798 * (int)__ldg(p) + 19235 * (int)__ldg(p + 1) + 3735 * (int)__ldg(p + 2) + 16384) >> 15;
}

__global__ void __launch_bounds__(256) blur_sums_kernel(const BlurArgs a) {
  const int frame = blockIdx.y;
  const unsigned char* f = a.frames + 3LL * a.height * a.width * frame;
  const long long n = (long long)a.height * a.width;
  long long s1 = 0, s2 = 0;
  for (long long p = (long long)blockIdx.x * 256 + threadIdx.x; p < n; p += (long long)gridDim.x * 256) {
    const int y = (int)(p / a.width), x = (int)(p - (long long)y * a.width);
    const int lap = grey_of(f, a.width, reflect101(y - 1, a.height), x) +
                    grey_of(f, a.width, reflect101(y + 1, a.height), x) +
                    grey_of(f, a.width, y, reflect101(x - 1, a.width)) +
                    grey_of(f, a.width, y, reflect101(x + 1, a.width)) - 4 * grey_of(f, a.width, y, x);
    s1 += lap;
    s2 += (long long)lap * lap;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  __shared__ long long part[2][8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { part[0][warp] = s1; part[1][warp] = s2; }
  __syncthreads();
  if (threadIdx.x == 0) {
    long long t1 = 0, t2 = 0;
    for (int w = 0; w < 8; ++w) { t1 += part[0][w]; t2 += part[1][w]; }
    atomicAdd(a.sums + 2 * frame, (unsigned long long)t1);
    atomicAdd(a.sums + 2 * frame + 1, (unsigned long long)t2);
  }
}

// var = (n * S2 - S1^2) / n^2: the numerator exactly in 128 bits, then one division in fp64.
__global__ void blur_finalize_kernel(const BlurArgs a) {
  const int frame = blockIdx.x * blockDim.x + threadIdx.x;
  if (frame >= a.num_frames) return;
  const long long n = (long long)a.height * a.width;
  const long long s1 = (long long)a.sums[2 * frame], s2 = (long long)a.sums[2 * frame + 1];
  const __int128 num = (__int128)n * s2 - (__int128)s1 * s1;       // >= 0 (Cauchy-Schwarz)
  const unsigned long long hi = (unsigned long long)(num >> 64), lo = (unsigned long long)num;
  const double numd = (double)hi * 18446744073709551616.0 + (double)lo;
  a.scores[frame] = numd / ((double)n * (double)n);
}

// ---------------------------------------------------------------------------------------------
// Near/far planes.  For camera c, the depths of the points that project into [0, W] x [0, H] with
// depth > 0 are a multiset of positive doubles; numpy's 'linear' quantile of it needs the order
// statistics at floor(v) and floor(v) + 1 (clamped), v = n q + (1 - q) - 1.  Positive doubles
// order as their uint64 bit patterns, so each of the four ranks (two per quantile) is found by
// radix select on 8-bit digits from the top: every pass recomputes the fp64 projection of every
// point (cheap against a sort) and counts the digits of the points whose higher digits match the
// rank's prefix so far, in a shared-memory histogram per (camera, rank).  Pass 0 counts every
// accepted point (all ranks share an empty prefix), which also gives n.  Workspace: the per-camera
// histograms and selection state, independent of the number of points.
// ---------------------------------------------------------------------------------------------
constexpr int kRanks = 4;
constexpr int kDigitBits = 8;
constexpr int kBins = 1 << kDigitBits;
constexpr int kPasses = 64 / kDigitBits;

struct NearFarState {
  unsigned long long prefix[kRanks];   // bits selected so far (the high digits)
  unsigned long long k[kRanks];        // rank still to find among the points matching the prefix
  long long count;                     // points accepted for this camera
};

struct NearFarArgs {
  const nfb_camera* cameras;   // device (num_cameras)
  int num_cameras;
  const double* points;        // (num_points, 3)
  long long num_points;
  double q[2];                 // near and far quantiles
  unsigned int* hist;          // (num_cameras, kRanks, kBins)
  NearFarState* state;         // (num_cameras)
  double* near;
  double* far;
  long long* counts;
};

// The depth bits of point p for camera c, or 0 if the point is rejected (0 is no positive double).
__device__ __forceinline__ unsigned long long accepted_depth_bits(const nfb_camera& c, const double* pts,
                                                                  long long p) {
  double px, py, depth;
  camera_project_point<double>(c, __ldg(pts + 3 * p), __ldg(pts + 3 * p + 1), __ldg(pts + 3 * p + 2), px, py,
                               depth);
  const bool in = px >= 0.0 && px <= (double)c.image_size[0] && py >= 0.0 && py <= (double)c.image_size[1] &&
                  depth > 0.0;
  return in ? (unsigned long long)__double_as_longlong(depth) : 0ull;
}

// grid (blocks per camera, num_cameras): histogram of digit `pass` for each rank.
__global__ void __launch_bounds__(256) near_far_hist_kernel(const NearFarArgs a, int pass) {
  __shared__ unsigned int h[kRanks][kBins];
  __shared__ nfb_camera cam;
  __shared__ unsigned long long prefix[kRanks];
  const int c = blockIdx.y;
  for (int i = threadIdx.x; i < kRanks * kBins; i += 256) (&h[0][0])[i] = 0u;
  if (threadIdx.x == 0) cam = a.cameras[c];
  if (threadIdx.x < kRanks) prefix[threadIdx.x] = pass ? a.state[c].prefix[threadIdx.x] : 0ull;
  __syncthreads();
  const int shift = 64 - kDigitBits * (pass + 1);
  const int ranks = pass ? kRanks : 1;
  for (long long p = (long long)blockIdx.x * 256 + threadIdx.x; p < a.num_points; p += (long long)gridDim.x * 256) {
    const unsigned long long bits = accepted_depth_bits(cam, a.points, p);
    if (!bits) continue;
    const unsigned int digit = (unsigned int)(bits >> shift) & (kBins - 1);
    for (int r = 0; r < ranks; ++r)
      if (pass == 0 || (bits >> (shift + kDigitBits)) == (prefix[r] >> (shift + kDigitBits)))
        atomicAdd(&h[r][digit], 1u);
  }
  __syncthreads();
  unsigned int* g = a.hist + (long long)c * kRanks * kBins;
  for (int i = threadIdx.x; i < ranks * kBins; i += 256) {
    const unsigned int v = (&h[0][0])[i];
    if (v) atomicAdd(g + i, v);
  }
}

// One block of 32 threads per camera: thread r < kRanks picks rank r's digit, then the block clears
// the histograms for the next pass.  After the last pass, thread 0 writes numpy's lerp.
__global__ void __launch_bounds__(32) near_far_select_kernel(const NearFarArgs a, int pass) {
  const int c = blockIdx.x;
  unsigned int* g = a.hist + (long long)c * kRanks * kBins;
  NearFarState& st = a.state[c];
  const int shift = 64 - kDigitBits * (pass + 1);
  const int r = threadIdx.x;
  if (pass == 0 && r == 0) {
    long long n = 0;
    for (int b = 0; b < kBins; ++b) n += g[b];
    st.count = n;
    for (int qi = 0; qi < 2; ++qi) {                 // numpy _compute_virtual_index / _get_indexes
      const double q = a.q[qi];
      const double v = (double)n * q + (1.0 + q * (1.0 - 1.0 - 1.0)) - 1.0;
      long long lo = (long long)floor(v), hi = lo + 1;
      if (v >= (double)(n - 1)) lo = hi = n - 1;
      if (v < 0) lo = hi = 0;
      st.k[2 * qi] = (unsigned long long)lo;
      st.k[2 * qi + 1] = (unsigned long long)hi;
      st.prefix[2 * qi] = st.prefix[2 * qi + 1] = 0ull;
    }
  }
  __syncwarp();
  if (r < kRanks && st.count > 0) {
    const unsigned int* row = g + (pass ? r : 0) * kBins;
    unsigned long long k = st.k[r], below = 0;
    int b = 0;
    for (; b < kBins - 1; ++b) {
      if (below + row[b] > k) break;
      below += row[b];
    }
    st.k[r] = k - below;
    st.prefix[r] |= (unsigned long long)b << shift;
  }
  __syncwarp();
  for (int i = threadIdx.x; i < kRanks * kBins; i += 32) g[i] = 0u;
  if (pass == kPasses - 1 && r == 0) {
    a.counts[c] = st.count;
    double out[2];
    for (int qi = 0; qi < 2; ++qi) {
      if (st.count == 0) { out[qi] = __longlong_as_double(0x7ff8000000000000ll); continue; }
      const double lo = __longlong_as_double((long long)st.prefix[2 * qi]);
      const double hi = __longlong_as_double((long long)st.prefix[2 * qi + 1]);
      const double q = a.q[qi], n = (double)st.count;
      const double v = n * q + (1.0 + q * (1.0 - 1.0 - 1.0)) - 1.0;
      const double t = v - floor(v);                 // numpy _get_gamma; unused when clamped (lo == hi)
      const double diff = hi - lo;                   // numpy _lerp
      out[qi] = t >= 0.5 ? hi - diff * (1.0 - t) : lo + diff * t;
    }
    a.near[c] = out[0];
    a.far[c] = out[1];
  }
}

}  // namespace capture
}  // namespace nfb
