// Per-group camera intrinsics gradient (nfb_intrinsics_grad): the ray-direction gradients of a batch taken back
// through pixel -> ray (camera_pixel_direction of refined_camera, then pose_moved_ray) to the intrinsics delta
// q = (s, dcx, dcy, dk1, dk2, dk3, dp1, dp2) of each ray's image group, and summed over each group's rays.
//
// Per ray, in fp64 at the refined camera (f = f0 e^s, c = c0 + f0 dc, k, p):
//   g      <- exp(omega)^T g                     the pose's rotation undone
//   g'      = g - d (d . g)                      d = d'/|d'|, |d'| = 1: the world normalisation
//   g_l     = R0 g'                              d' = R0^T l
//   g_u     = (g_l - l (l . g_l)) / |u|          l = u/|u|, u = (x, y, 1)
//   g_x0    = J_D^-T g_u                         (x, y) = D^-1(x0, y0) at Newton's fixed point (implicit
//   g_(k,p) = -(dD/d(k,p))^T g_x0                 function theorem), J_D the Newton step's Jacobian
//   then y0 = (py - cy) / (f a), x0 = (px - cx - y0 skew) / f to s and dc.
// Deterministic: per-block fp64 partials in ray order, then one fixed-order column sum per group; no atomics.
#pragma once
#include "camera_kernels.cuh"

namespace nfb {

constexpr int kIntrinsicsRays = 256;   // rays (and threads) per block of intrinsics_partials_kernel

struct IntrinsicsGradArgs {
  const nfb_camera* cameras;   // (num_images) the capture cameras
  int num_images;
  const float* pose;           // (num_images,6) or null (zero poses)
  const float* intrinsics;     // (num_groups,8) or null (zero deltas)
  const int* group;            // (num_images) image -> group
  int num_groups;
  unsigned parts;              // NFB_INTRINSICS_* bits: the fitted entries
  const int* image;            // (count)
  const float* pixels;         // (count,2)
  const float* directions;     // (count,3) the posed world directions
  const float* d_directions;   // (count,3)
  long long count;
  double* partial;             // (blocks, num_groups, 8)
  float* grad;                 // (num_groups,8): +=
};

// dL/dq of ray r of image k in group gk (see the file comment).  0 where J_D is singular.
__device__ __forceinline__ void intrinsics_ray_grad(const IntrinsicsGradArgs& a, long long r, int k, int gk,
                                                    double out[8]) {
  const nfb_camera& c = a.cameras[k];
  double q[8];
  for (int j = 0; j < 8; ++j) q[j] = a.intrinsics ? (double)a.intrinsics[8 * gk + j] : 0.0;
  const double f0 = c.focal_length, f = f0 * exp(q[0]), fy = f * (double)c.pixel_aspect_ratio;
  const double cx = c.principal_point[0] + f0 * q[1], cy = c.principal_point[1] + f0 * q[2];
  const double k1 = c.radial_distortion[0] + q[3], k2 = c.radial_distortion[1] + q[4];
  const double k3 = c.radial_distortion[2] + q[5];
  const double p1 = c.tangential_distortion[0] + q[6], p2 = c.tangential_distortion[1] + q[7];
  const double sk = c.skew;
  const double y0 = ((double)a.pixels[2 * r + 1] - cy) / fy;
  const double x0 = ((double)a.pixels[2 * r] - cx - y0 * sk) / f;
  double x, y;
  undistort_point<double>(x0, y0, k1, k2, k3, p1, p2, x, y);
  double g[3], d[3];
  for (int j = 0; j < 3; ++j) {
    g[j] = a.d_directions[3 * r + j];
    d[j] = a.directions[3 * r + j];
  }
  if (a.pose) {   // exp(omega)^T on both: the capture camera's direction and its gradient
    float R[9];
    rotvec_matrix(a.pose + 6 * k, R);
    double gr[3], dr[3];
    for (int j = 0; j < 3; ++j) {
      gr[j] = R[j] * g[0] + R[3 + j] * g[1] + R[6 + j] * g[2];
      dr[j] = R[j] * d[0] + R[3 + j] * d[1] + R[6 + j] * d[2];
    }
    for (int j = 0; j < 3; ++j) { g[j] = gr[j]; d[j] = dr[j]; }
  }
  const double dg = d[0] * g[0] + d[1] * g[1] + d[2] * g[2];
  double gl[3];
  for (int i = 0; i < 3; ++i) {
    gl[i] = 0.0;
    for (int j = 0; j < 3; ++j) gl[i] += (double)c.orientation[3 * i + j] * (g[j] - d[j] * dg);
  }
  const double n = sqrt(x * x + y * y + 1.0);
  const double lg = (x * gl[0] + y * gl[1] + gl[2]) / n;
  const double gux = (gl[0] - x / n * lg) / n, guy = (gl[1] - y / n * lg) / n;
  double fx, fyr, J[4];
  distortion_newton_terms<double>(x, y, x0, y0, k1, k2, k3, p1, p2, fx, fyr, J);
  const double det = J[0] * J[3] - J[1] * J[2];
  for (int j = 0; j < 8; ++j) out[j] = 0.0;
  if (!(fabs(det) > 1e-12)) return;
  const double gx0 = (J[3] * gux - J[2] * guy) / det, gy0 = (J[0] * guy - J[1] * gux) / det;
  const double r2 = x * x + y * y, w = -(x * gx0 + y * gy0);
  out[3] = r2 * w;
  out[4] = r2 * r2 * w;
  out[5] = r2 * r2 * r2 * w;
  out[6] = -(2.0 * x * y * gx0 + (r2 + 2.0 * y * y) * gy0);
  out[7] = -((r2 + 2.0 * x * x) * gx0 + 2.0 * x * y * gy0);
  const double gy0t = gy0 - gx0 * sk / f;   // y0 also enters x0 through the skew
  out[0] = -(x0 * gx0 + y0 * gy0t);
  out[1] = -f0 * gx0 / f;
  out[2] = -f0 * gy0t / fy;
}

// Block b: each group's sum of dL/dq over the block's rays [b kIntrinsicsRays, +kIntrinsicsRays), in ray order.
__global__ void __launch_bounds__(kIntrinsicsRays) intrinsics_partials_kernel(const IntrinsicsGradArgs a) {
  __shared__ int s_grp[kIntrinsicsRays];
  __shared__ double s_val[kIntrinsicsRays][8];
  const long long r0 = (long long)blockIdx.x * kIntrinsicsRays;
  const long long r = r0 + threadIdx.x;
  const int n = (int)min((long long)kIntrinsicsRays, a.count - r0);
  if (r < a.count) {
    const int k = a.image[r];
    const int gk = k >= 0 && k < a.num_images ? a.group[k] : -1;
    s_grp[threadIdx.x] = gk >= 0 && gk < a.num_groups ? gk : -1;
    if (s_grp[threadIdx.x] >= 0) intrinsics_ray_grad(a, r, k, gk, s_val[threadIdx.x]);
  }
  __syncthreads();
  for (int gk = threadIdx.x; gk < a.num_groups; gk += kIntrinsicsRays) {
    double acc[8] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int i = 0; i < n; ++i)
      if (s_grp[i] == gk)
        for (int c = 0; c < 8; ++c) acc[c] += s_val[i][c];
    double* out = a.partial + ((size_t)blockIdx.x * a.num_groups + gk) * 8;
    for (int c = 0; c < 8; ++c) out[c] = acc[c];
  }
}

// One thread per group: the column sum over the blocks, added to the fitted entries only.
__global__ void intrinsics_finish_kernel(const IntrinsicsGradArgs a, int blocks) {
  const int gk = blockIdx.x * blockDim.x + threadIdx.x;
  if (gk >= a.num_groups) return;
  double s[8] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int b = 0; b < blocks; ++b)
    for (int c = 0; c < 8; ++c) s[c] += a.partial[((size_t)b * a.num_groups + gk) * 8 + c];
  // entry -> part: s focal, dc principal point, dk radial, dp tangential
  const unsigned bit[8] = {NFB_INTRINSICS_FOCAL, NFB_INTRINSICS_PRINCIPAL_POINT, NFB_INTRINSICS_PRINCIPAL_POINT,
                           NFB_INTRINSICS_RADIAL, NFB_INTRINSICS_RADIAL, NFB_INTRINSICS_RADIAL,
                           NFB_INTRINSICS_TANGENTIAL, NFB_INTRINSICS_TANGENTIAL};
  float* g = a.grad + 8 * (size_t)gk;
  for (int c = 0; c < 8; ++c)
    if (a.parts & bit[c]) g[c] += (float)s[c];
}

}  // namespace nfb
