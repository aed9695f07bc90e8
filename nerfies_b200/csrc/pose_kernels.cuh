// Per-image camera pose gradient (nfb_pose_grad): the ray gradients of a training batch reduced over the
// rays of each table image, then taken through the pose parameterisation of pose_moved_ray
// (geometry.pose_rays), d = exp(omega) d0, o = o0 + v:
//   dL/dv     = sum_r g_o,r
//   dL/domega = J_l(omega)^T sum_r (d_r x g_d,r)
// with J_l SO(3)'s left Jacobian.  Deterministic: per-block partials in ray order, then one fixed-order
// column sum per image; no atomics.
#pragma once
#include "camera_kernels.cuh"

namespace nfb {

constexpr int kPoseRays = 256;   // rays (and threads) per block of pose_partials_kernel

struct PoseGradArgs {
  int num_images;
  long long count;
  const float* pose;          // (num_images,6) or null (zero poses)
  const int* image;           // (count)
  const float* directions;    // (count,3) the posed directions d_r
  const float* d_origins;     // (count,3) or null
  const float* d_directions;  // (count,3) or null
  double* partial;            // (blocks, num_images, 6)
  float* grad;                // (num_images,6): +=
};

// Block b: the images' sums [sum d x g_d | sum g_o] over its rays [b kPoseRays, +kPoseRays), in ray order.
__global__ void __launch_bounds__(kPoseRays) pose_partials_kernel(const PoseGradArgs a) {
  __shared__ int s_img[kPoseRays];
  __shared__ double s_val[kPoseRays][6];
  const long long r0 = (long long)blockIdx.x * kPoseRays;
  const long long r = r0 + threadIdx.x;
  const int n = (int)min((long long)kPoseRays, a.count - r0);
  if (r < a.count) {
    double g[3] = {0.0, 0.0, 0.0}, go[3] = {0.0, 0.0, 0.0};
    if (a.d_directions)
      for (int c = 0; c < 3; ++c) g[c] = a.d_directions[3 * r + c];
    if (a.d_origins)
      for (int c = 0; c < 3; ++c) go[c] = a.d_origins[3 * r + c];
    const double d[3] = {a.directions[3 * r], a.directions[3 * r + 1], a.directions[3 * r + 2]};
    s_img[threadIdx.x] = a.image[r];
    s_val[threadIdx.x][0] = d[1] * g[2] - d[2] * g[1];
    s_val[threadIdx.x][1] = d[2] * g[0] - d[0] * g[2];
    s_val[threadIdx.x][2] = d[0] * g[1] - d[1] * g[0];
    for (int c = 0; c < 3; ++c) s_val[threadIdx.x][3 + c] = go[c];
  }
  __syncthreads();
  for (int k = threadIdx.x; k < a.num_images; k += kPoseRays) {
    double acc[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int i = 0; i < n; ++i)
      if (s_img[i] == k)
        for (int c = 0; c < 6; ++c) acc[c] += s_val[i][c];
    double* out = a.partial + ((size_t)blockIdx.x * a.num_images + k) * 6;
    for (int c = 0; c < 6; ++c) out[c] = acc[c];
  }
}

// One thread per image: the column sum over the blocks, then J_l(omega)^T on the rotation part,
//   J_l^T s = s - b (omega x s) + c (omega x (omega x s)),  b = (1 - cos t)/t^2,  c = (t - sin t)/t^3,
// both by their Taylor series to t^4 below t^2 = 1e-4 (rotvec_matrix's threshold).
__global__ void pose_finish_kernel(const PoseGradArgs a, int blocks) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= a.num_images) return;
  double s[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int b = 0; b < blocks; ++b)
    for (int c = 0; c < 6; ++c) s[c] += a.partial[((size_t)b * a.num_images + k) * 6 + c];
  double w[3] = {0.0, 0.0, 0.0};
  if (a.pose)
    for (int c = 0; c < 3; ++c) w[c] = a.pose[6 * k + c];
  const double t2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
  double cb, cc;
  if (t2 < 1e-4) {
    cb = 0.5 - t2 / 24.0 + t2 * t2 / 720.0;
    cc = 1.0 / 6.0 - t2 / 120.0 + t2 * t2 / 5040.0;
  } else {
    const double t = sqrt(t2);
    cb = (1.0 - cos(t)) / t2;
    cc = (t - sin(t)) / (t2 * t);
  }
  const double x[3] = {w[1] * s[2] - w[2] * s[1], w[2] * s[0] - w[0] * s[2], w[0] * s[1] - w[1] * s[0]};
  const double xx[3] = {w[1] * x[2] - w[2] * x[1], w[2] * x[0] - w[0] * x[2], w[0] * x[1] - w[1] * x[0]};
  float* g = a.grad + 6 * (size_t)k;
  for (int c = 0; c < 3; ++c) g[c] += (float)(s[c] - cb * x[c] + cc * xx[c]);
  for (int c = 0; c < 3; ++c) g[3 + c] += (float)s[3 + c];
}

}  // namespace nfb
