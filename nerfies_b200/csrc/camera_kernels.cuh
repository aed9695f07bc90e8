// Camera -> rays on the GPU (SURVEY §8(f) row 3): what the reference does on the
// host in numpy for every evaluated frame,
//   datasets/core.py:50-75  camera_to_rays
//   camera.py:317-321       get_pixel_centers
//   camera.py:225-269       pixel_to_local_rays / pixels_to_rays
//   camera.py:26-105        radial + tangential undistortion (10 Newton steps)
// HBM-bound elementwise work: 0 or 8 B read and 24-32 B written per pixel; one
// thread per pixel, fully coalesced stores of consecutive pixels.  fp32, written
// operation for operation as the reference's float32 numpy (the build uses
// -fmad=false and IEEE division / sqrt).  refined_camera applies an intrinsics delta (nfb_gather_rays_refined,
// nfb_pixels_to_rays_refined); intrinsics_kernels.cuh holds its adjoint.
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
  const float* intrinsics;  // (8) device or null: cam refined by this delta (refined_camera)
};

// The Newton system of camera.py:42-68 at (x, y): the residual F = D(x, y) - (xd, yd) of the distortion D and
// its 2x2 Jacobian J = dD/d(x, y) = [fx_x, fx_y, fy_x, fy_y].  T = float is the ray kernels' arithmetic
// operation for operation; T = double serves the intrinsics adjoint (intrinsics_kernels.cuh).
template <typename T>
__device__ __forceinline__ void distortion_newton_terms(T x, T y, T xd, T yd, T k1, T k2, T k3, T p1, T p2,
                                                        T& fx, T& fy, T J[4]) {
  const T two_p1 = (T)2 * p1, two_p2 = (T)2 * p2, six_p1 = (T)6 * p1, six_p2 = (T)6 * p2;
  const T two_k2 = (T)2 * k2, three_k3 = (T)3 * k3;
  const T r = x * x + y * y;                              // camera.py:42
  const T d = (T)1 + r * (k1 + r * (k2 + k3 * r));        // camera.py:43
  fx = d * x + two_p1 * x * y + p2 * (r + (T)2 * x * x) - xd;   // camera.py:55
  fy = d * y + two_p2 * x * y + p1 * (r + (T)2 * y * y) - yd;   // camera.py:56
  const T d_r = k1 + r * (two_k2 + three_k3 * r);         // camera.py:59
  const T d_x = (T)2 * x * d_r;
  const T d_y = (T)2 * y * d_r;
  J[0] = d + d_x * x + two_p1 * y + six_p2 * x;           // camera.py:64
  J[1] = d_y * x + two_p1 * x + two_p2 * y;
  J[2] = d_x * y + two_p2 * y + two_p1 * x;               // camera.py:68
  J[3] = d + d_y * y + two_p2 * x + six_p1 * y;
}

template <typename T>
__device__ __forceinline__ void undistort_point(T xd, T yd, T k1, T k2, T k3, T p1, T p2, T& xo, T& yo) {
  T x = xd, y = yd;
  const T eps = (T)1e-9f;
#pragma unroll 1
  for (int it = 0; it < 10; ++it) {                       // camera.py:90 (no early exit)
    T fx, fy, J[4];
    distortion_newton_terms<T>(x, y, xd, yd, k1, k2, k3, p1, p2, fx, fy, J);
    const T den = J[2] * J[1] - J[0] * J[3];              // camera.py:93-95
    const T xn = fx * J[3] - fy * J[1];
    const T yn = fy * J[0] - fx * J[2];
    const bool ok = fabs(den) > eps;
    x = x + (ok ? xn / den : (T)0);
    y = y + (ok ? yn / den : (T)0);
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
    undistort_point<float>(x, y, c.radial_distortion[0], c.radial_distortion[1], c.radial_distortion[2],
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

// Image k's camera refined by its intrinsics delta q = (s, dcx, dcy, dk1, dk2, dk3, dp1, dp2)
// (nfb_gather_rays_refined): focal f0 exp(s), principal point c0 + f0 dc, radial k0 + dk, tangential p0 + dp;
// skew, pixel aspect ratio, pose and image size stay.  q = 0 gives c0's ray bit for bit: exp(0) = 1 and
// x + 0 = x, and camera_has_distortion reads the refined coefficients.
__host__ __device__ __forceinline__ nfb_camera refined_camera(const nfb_camera& c0, const float* q) {
  nfb_camera c = c0;
  c.focal_length = c0.focal_length * expf(q[0]);
  for (int j = 0; j < 2; ++j) c.principal_point[j] = c0.principal_point[j] + c0.focal_length * q[1 + j];
  for (int j = 0; j < 3; ++j) c.radial_distortion[j] = c0.radial_distortion[j] + q[3 + j];
  for (int j = 0; j < 2; ++j) c.tangential_distortion[j] = c0.tangential_distortion[j] + q[6 + j];
  return c;
}

// camera_pixel_direction of c0 refined by q (refined_camera); q null: c0's own.
__device__ __forceinline__ void refined_pixel_direction(const nfb_camera& c0, const float* q, float px, float py,
                                                        float* out_d) {
  if (!q) {
    camera_pixel_direction(c0, camera_has_distortion(c0), px, py, out_d);
    return;
  }
  const nfb_camera c = refined_camera(c0, q);
  camera_pixel_direction(c, camera_has_distortion(c), px, py, out_d);
}

// Camera.project (camera.py:279-315) of the world point (X, Y, Z) in arithmetic T, written operation
// for operation as numpy evaluates it: T = float is float32 numpy on float32 points; T = double is
// float64 points against the camera's float32 fields, which numpy widens per operation.  Products of
// two camera fields (2 * p1, focal * aspect) stay float32 as numpy computes them on float32 scalars.
// Returns the pixel position and the local depth (points_to_local_points(.)[..., 2]).  The elementwise
// operations keep each a*b+c at two roundings (the build's -fmad=false), as numpy's ufuncs do.  The
// rotation is np.matmul, which numpy hands to BLAS: OpenBLAS's x86-64 GEMM kernels accumulate the
// three products as fma(o2, t2, fma(o1, t1, o0 * t0)), and that chain reproduces the recorded
// projections (tests/golden/camera_*.npz) bit for bit where two roundings per step miss by up to 384 ulp.
template <typename T>
__device__ __forceinline__ void camera_project_point(const nfb_camera& c, T X, T Y, T Z, T& px, T& py,
                                                     T& depth) {
  const T t0 = X - (T)c.position[0], t1 = Y - (T)c.position[1], t2 = Z - (T)c.position[2];   // camera.py:280
  T l[3];
#pragma unroll
  for (int i = 0; i < 3; ++i)                                                               // camera.py:281
    l[i] = fma((T)c.orientation[3 * i + 2], t2, fma((T)c.orientation[3 * i + 1], t1, (T)c.orientation[3 * i] * t0));
  const T x = l[0] / l[2], y = l[1] / l[2];                                                 // camera.py:291-292
  const T r2 = x * x + y * y;
  const T k1 = (T)c.radial_distortion[0], k2 = (T)c.radial_distortion[1], k3 = (T)c.radial_distortion[2];
  const T d = (T)1 + r2 * (k1 + r2 * (k2 + k3 * r2));                                       // camera.py:296-298
  const T xy = x * y;
  const float p1 = c.tangential_distortion[0], p2 = c.tangential_distortion[1];
  const T xd = x * d + (T)(2.f * p1) * xy + (T)p2 * (r2 + (T)2 * (x * x));                  // camera.py:302-304
  const T yd = y * d + (T)(2.f * p2) * xy + (T)p1 * (r2 + (T)2 * (y * y));                  // camera.py:305-307
  px = (T)c.focal_length * xd + (T)c.skew * yd + (T)c.principal_point[0];                   // camera.py:310
  py = (T)(c.focal_length * c.pixel_aspect_ratio) * yd + (T)c.principal_point[1];           // camera.py:311-312
  depth = l[2];
}

// Camera.project of float32 points (n, 3) -> pixels (n, 2), float32 throughout.
__global__ void __launch_bounds__(256) camera_project_kernel(const nfb_camera c, const float* __restrict__ points,
                                                             long long n, float* __restrict__ pixels) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  float px, py, depth;
  camera_project_point<float>(c, __ldg(points + 3 * i), __ldg(points + 3 * i + 1), __ldg(points + 3 * i + 2),
                              px, py, depth);
  pixels[2 * i] = px;
  pixels[2 * i + 1] = py;
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
  if (a.intrinsics)
    refined_pixel_direction(a.cam, a.intrinsics, px, py, out_d);
  else
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
  const float* pose;   // (num_images,6) [omega | v] or null: image k's camera moved by pose k (pose_moved_ray)
  int* image;          // (count) the table image of each ray
  const float* intrinsics;   // (num_groups,8) or null: image k's camera refined by intrinsics[group[k]]
  const int* group;          // (num_images) each image's intrinsics group; one outside [0, num_groups): none
  int num_groups;
};

// exp([w]x) of a rotation vector, as geometry.rotvec_to_matrix: I + a K + b K^2 with a = sin(t)/t and
// b = 2 sin^2(t/2)/t^2, their Taylor series to t^4 below t^2 = 1e-4.  Row-major.
__host__ __device__ __forceinline__ void rotvec_matrix(const float w[3], float R[9]) {
  const float t2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
  float a, b;
  if (t2 < 1e-4f) {
    a = 1.f - t2 / 6.f + t2 * t2 / 120.f;
    b = 0.5f - t2 / 24.f + t2 * t2 / 720.f;
  } else {
    const float t = sqrtf(t2), h = sinf(0.5f * t);
    a = sinf(t) / t;
    b = 2.f * h * h / t2;
  }
  const float K[9] = {0.f, -w[2], w[1], w[2], 0.f, -w[0], -w[1], w[0], 0.f};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const float kk = K[3 * i] * K[j] + K[3 * i + 1] * K[3 + j] + K[3 * i + 2] * K[6 + j];
      R[3 * i + j] = (i == j ? 1.f : 0.f) + a * K[3 * i + j] + b * kk;
    }
}

// A ray of a camera moved by the pose p = (omega, v) (geometry.pose_rays): d <- exp(omega) d, o <- o + v.
// A zero pose gives exp(0) = I exactly, so the ray is returned bit for bit.
__device__ __forceinline__ void pose_moved_ray(const float* p, float* o, float* d) {
  float R[9];
  rotvec_matrix(p, R);
  const float x = d[0], y = d[1], z = d[2];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    d[j] = R[3 * j] * x + R[3 * j + 1] * y + R[3 * j + 2] * z;
    o[j] = o[j] + p[3 + j];
  }
}

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
  if (a.image) a.image[i] = lo;
  if (a.origins || a.directions || a.pixels) {
    float px, py;
    camera_pixel_center(c, r - __ldg(t.pixel_offsets + lo), px, py);
    float o[3] = {c.position[0], c.position[1], c.position[2]}, d[3] = {0.f, 0.f, 0.f};   // datasets/core.py:176
    if (a.directions) {
      const int gk = a.intrinsics ? __ldg(a.group + lo) : -1;
      refined_pixel_direction(c, gk >= 0 && gk < a.num_groups ? a.intrinsics + 8 * gk : nullptr, px, py, d);
    }
    if (a.pose) pose_moved_ray(a.pose + 6 * lo, o, d);
    if (a.directions)
      for (int j = 0; j < 3; ++j) a.directions[3 * i + j] = d[j];
    if (a.pixels) { a.pixels[2 * i] = px; a.pixels[2 * i + 1] = py; }
    if (a.origins)
      for (int j = 0; j < 3; ++j) a.origins[3 * i + j] = o[j];
  }
  if (a.rgb)   // datasets/nerfies.py:62: float32(u8) / 255.0, an IEEE division
    for (int j = 0; j < 3; ++j) a.rgb[3 * i + j] = (float)__ldg(t.rgb + 3 * r + j) / 255.f;
  if (a.appearance) a.appearance[i] = __ldg(t.appearance + lo);
  if (a.camera) a.camera[i] = __ldg(t.camera + lo);
  if (a.warp) a.warp[i] = __ldg(t.warp + lo);
  if (a.time) a.time[i] = __ldg(t.time + lo);
}

}  // namespace nfb
