// Camera -> rays on the GPU (SURVEY §8(f) row 3): what the reference does on the
// host in numpy for every evaluated frame,
//   datasets/core.py:50-75  camera_to_rays
//   camera.py:317-321       get_pixel_centers
//   camera.py:225-269       pixel_to_local_rays / pixels_to_rays
//   camera.py:26-105        radial + tangential undistortion (10 Newton steps)
// HBM-bound elementwise work: 0 or 8 B read and 24-32 B written per pixel; one
// thread per pixel, fully coalesced stores of consecutive pixels.  fp32, written
// operation for operation as the reference's float32 numpy (the build uses
// -fmad=false and IEEE division / sqrt).
#pragma once
#include "../../include/nerfies_b200.h"

namespace nfb {

struct CameraArgs {
  nfb_camera cam;
  const float* pixels_in;   // (n,2) or nullptr: pixel centres of the linear range
  long long first, count;
  float* origins;           // (n,3) nullable
  float* directions;        // (n,3)
  float* pixels_out;        // (n,2) nullable
  int has_distortion;
};

__device__ __forceinline__ void undistort_point(float xd, float yd, float k1, float k2, float k3,
                                                float p1, float p2, float& xo, float& yo) {
  float x = xd, y = yd;
  const float eps = 1e-9f;
  const float two_p1 = 2.f * p1, two_p2 = 2.f * p2, six_p1 = 6.f * p1, six_p2 = 6.f * p2;
  const float two_k2 = 2.f * k2, three_k3 = 3.f * k3;
#pragma unroll 1
  for (int it = 0; it < 10; ++it) {                       // camera.py:90 (no early exit)
    const float r = x * x + y * y;                        // camera.py:42
    const float d = 1.f + r * (k1 + r * (k2 + k3 * r));   // camera.py:43
    const float fx = d * x + two_p1 * x * y + p2 * (r + 2.f * x * x) - xd;   // camera.py:55
    const float fy = d * y + two_p2 * x * y + p1 * (r + 2.f * y * y) - yd;   // camera.py:56
    const float d_r = k1 + r * (two_k2 + three_k3 * r);   // camera.py:59
    const float d_x = 2.f * x * d_r;
    const float d_y = 2.f * y * d_r;
    const float fx_x = d + d_x * x + two_p1 * y + six_p2 * x;   // camera.py:64
    const float fx_y = d_y * x + two_p1 * x + two_p2 * y;
    const float fy_x = d_x * y + two_p2 * y + two_p1 * x;       // camera.py:68
    const float fy_y = d + d_y * y + two_p2 * x + six_p1 * y;
    const float den = fy_x * fx_y - fx_x * fy_y;                // camera.py:93-95
    const float xn = fx * fy_y - fy * fx_y;
    const float yn = fy * fx_x - fx * fy_x;
    const bool ok = fabsf(den) > eps;
    x = x + (ok ? xn / den : 0.f);
    y = y + (ok ? yn / den : 0.f);
  }
  xo = x; yo = y;
}

// camera.py:201-207: undistortion runs only when a coefficient is non-zero.
__host__ __device__ __forceinline__ int camera_has_distortion(const nfb_camera& c) {
  return c.radial_distortion[0] != 0.f || c.radial_distortion[1] != 0.f || c.radial_distortion[2] != 0.f ||
         c.tangential_distortion[0] != 0.f || c.tangential_distortion[1] != 0.f;
}

// Pixel centre of row-major pixel p (camera.py:319-321).
__device__ __forceinline__ void camera_pixel_center(const nfb_camera& c, long long p, float& px, float& py) {
  const long long row = p / c.image_size[0];
  px = (float)(p - row * c.image_size[0]) + 0.5f;
  py = (float)row + 0.5f;
}

// Unit world-space direction of the pixel position (px, py) (camera.py:225-269).
__device__ __forceinline__ void camera_pixel_direction(const nfb_camera& c, int has_distortion, float px, float py,
                                                       float* out_d) {
  const float sy = c.focal_length * c.pixel_aspect_ratio;  // camera.py:186-187
  float y = (py - c.principal_point[1]) / sy;              // camera.py:227
  float x = (px - c.principal_point[0] - y * c.skew) / c.focal_length;   // camera.py:228-229
  if (has_distortion)
    undistort_point(x, y, c.radial_distortion[0], c.radial_distortion[1], c.radial_distortion[2],
                    c.tangential_distortion[0], c.tangential_distortion[1], x, y);
  // camera.py:241-242: dirs / ||dirs||, dirs = (x, y, 1)
  const float n = sqrtf(x * x + y * y + 1.f);
  const float l0 = x / n, l1 = y / n, l2 = 1.f / n;
  // camera.py:262: orientation^T @ local (orientation is world-to-camera, row-major)
  float d[3];
#pragma unroll
  for (int j = 0; j < 3; ++j)
    d[j] = c.orientation[j] * l0 + c.orientation[3 + j] * l1 + c.orientation[6 + j] * l2;
  const float n2 = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);        // camera.py:266
#pragma unroll
  for (int j = 0; j < 3; ++j) d[j] = d[j] / n2;
  out_d[0] = d[0]; out_d[1] = d[1]; out_d[2] = d[2];
}

// One pixel of CameraArgs: unit world-space direction and the pixel position used.
__device__ __forceinline__ void camera_ray_of_pixel(const CameraArgs& a, long long i, float* out_d, float* out_p) {
  float px, py;
  if (a.pixels_in) {
    px = __ldg(a.pixels_in + 2 * i);
    py = __ldg(a.pixels_in + 2 * i + 1);
  } else {
    camera_pixel_center(a.cam, a.first + i, px, py);
  }
  camera_pixel_direction(a.cam, a.has_distortion, px, py, out_d);
  out_p[0] = px; out_p[1] = py;
}

// 12-byte-per-pixel outputs are staged through shared memory so that a block
// writes its 256 x 12 B as 192 aligned 16-byte vectors (a per-thread stride-12
// scalar store pattern leaves HBM sectors partially written: 208 GB/s measured on
// an 8K frame before this, see profiles/).
__global__ void __launch_bounds__(256) camera_rays_kernel(const CameraArgs a) {
  __shared__ __align__(16) float s_dir[256 * 3];
  const long long block0 = (long long)blockIdx.x * 256;
  const long long i = block0 + threadIdx.x;
  const bool valid = i < a.count;
  float d[3] = {0.f, 0.f, 0.f}, p[2] = {0.f, 0.f};
  if (valid) camera_ray_of_pixel(a, i, d, p);
  s_dir[threadIdx.x * 3 + 0] = d[0];
  s_dir[threadIdx.x * 3 + 1] = d[1];
  s_dir[threadIdx.x * 3 + 2] = d[2];
  if (valid && a.pixels_out)
    reinterpret_cast<float2*>(a.pixels_out)[i] = make_float2(p[0], p[1]);   // 8 B/thread: coalesced as is
  __syncthreads();
  const long long n_here = min((long long)256, a.count - block0);          // pixels of this block
  if (n_here == 256) {
    // block0 * 12 B is a multiple of 3072 B: 16-byte aligned if the buffer is
    if (threadIdx.x < 192) {
      reinterpret_cast<float4*>(a.directions + block0 * 3)[threadIdx.x] =
          reinterpret_cast<const float4*>(s_dir)[threadIdx.x];
      if (a.origins) {
        // origins repeat (x,y,z): element e of the block's 768 floats is position[e % 3]
        const int e = threadIdx.x * 4;
        const float* q = a.cam.position;
        reinterpret_cast<float4*>(a.origins + block0 * 3)[threadIdx.x] =
            make_float4(q[e % 3], q[(e + 1) % 3], q[(e + 2) % 3], q[(e + 3) % 3]);   // datasets/core.py:66-67
      }
    }
  } else {
    for (int e = threadIdx.x; e < n_here * 3; e += 256) {
      a.directions[block0 * 3 + e] = s_dir[e];
      if (a.origins) a.origins[block0 * 3 + e] = a.cam.position[e % 3];
    }
  }
}

// Training batches and eval items of a preloaded capture (datasets/core.py:392-447 with flatten
// and shuffle, then repeat + batch): output i is ray order[(first + i) mod num_rays] of the
// image-after-image, row-major concatenation of the table's items.  Every output is nullable.
struct GatherArgs {
  nfb_ray_table t;
  long long first, count;
  float* origins;      // (count,3)
  float* directions;   // (count,3)
  float* pixels;       // (count,2)
  float* rgb;          // (count,3)
  int *appearance, *camera, *warp;   // (count)
  float* time;         // (count)
};

__global__ void __launch_bounds__(256) gather_rays_kernel(const GatherArgs a) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= a.count) return;
  const nfb_ray_table& t = a.t;
  const long long g = (a.first + i) % t.num_rays;
  long long r = g;
  if (t.order)
    r = t.order_is_64 ? __ldg(static_cast<const long long*>(t.order) + g) : __ldg(static_cast<const int*>(t.order) + g);
  // image k: pixel_offsets[k] <= r < pixel_offsets[k + 1]
  int lo = 0, hi = t.num_images;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(t.pixel_offsets + mid) <= r) lo = mid; else hi = mid;
  }
  const nfb_camera& c = t.cameras[lo];
  if (a.origins || a.directions || a.pixels) {
    float px, py;
    camera_pixel_center(c, r - __ldg(t.pixel_offsets + lo), px, py);
    if (a.directions) {
      float d[3];
      camera_pixel_direction(c, camera_has_distortion(c), px, py, d);
      for (int j = 0; j < 3; ++j) a.directions[3 * i + j] = d[j];
    }
    if (a.pixels) { a.pixels[2 * i] = px; a.pixels[2 * i + 1] = py; }
    if (a.origins)
      for (int j = 0; j < 3; ++j) a.origins[3 * i + j] = c.position[j];   // datasets/core.py:176
  }
  if (a.rgb)   // datasets/nerfies.py:62: float32(u8) / 255.0, an IEEE division
    for (int j = 0; j < 3; ++j) a.rgb[3 * i + j] = (float)__ldg(t.rgb + 3 * r + j) / 255.f;
  if (a.appearance) a.appearance[i] = __ldg(t.appearance + lo);
  if (a.camera) a.camera[i] = __ldg(t.camera + lo);
  if (a.warp) a.warp[i] = __ldg(t.warp + lo);
  if (a.time) a.time[i] = __ldg(t.time + lo);
}

}  // namespace nfb
