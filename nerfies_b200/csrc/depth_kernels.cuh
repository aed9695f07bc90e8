// Per-frame depth maps: sensor depth resampled onto a capture's frames (nfb_depth_resample) and depth batches
// drawn alongside the rgb batches of a ray table (nfb_gather_depth).  Depth here is always the renderer's: the
// distance along the pixel centre's unit ray, in normalised scene units.
#pragma once

#include <cuda_runtime.h>

#include "camera_kernels.cuh"

namespace nfb {

__device__ __forceinline__ bool depth_valid(float z) { return isfinite(z) && z > 0.f; }

// Depth of ray order[(first + i) mod num_rays], the ray gather_rays_kernel draws for output i.
__global__ void __launch_bounds__(256) gather_depth_kernel(const nfb_ray_table t, long long first, long long count,
                                                           float* __restrict__ depth_out) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= count) return;
  const long long g = (first + i) % t.num_rays;
  long long r = g;
  if (t.order)
    r = t.order_is_64 ? __ldg(static_cast<const long long*>(t.order) + g) : __ldg(static_cast<const int*>(t.order) + g);
  depth_out[i] = __ldg(t.depth + r);
}

struct DepthResampleArgs {
  nfb_camera cam;            // the frame's camera at the output scale; image_size = (w, h) of the output
  int has_distortion;
  const float* src;          // (src_h, src_w) z-depth in sensor units; non-finite or <= 0: missing
  int src_h, src_w;
  double sx, sy;             // source pixels per output pixel (src_w / w, src_h / h)
  float factor;              // metric_scale * scene scale
  float* dst;                // (h, w) ray distance in scene units; NaN: missing
};

// One thread per output pixel.  The output pixel covers [x, x+1) x [y, y+1), i.e. [x sx, (x+1) sx) x
// [y sy, (y+1) sy) in source pixels; the source pixels whose centres fall in it are averaged over the valid
// ones.  When none does (upsampling) or none of those is valid, the source pixel containing the output
// centre is used if it is valid.  A missing pixel is never blended: the output is NaN when nothing valid is
// found.  The z-depth is turned into the distance along the pixel centre's unit ray d (camera_pixel_direction,
// distortion included): t = z / (d . a) with a the optical axis (row 2 of the world-to-camera rotation).
__global__ void __launch_bounds__(256) depth_resample_kernel(const DepthResampleArgs a) {
  const int w = a.cam.image_size[0], h = a.cam.image_size[1];
  const long long p = (long long)blockIdx.x * 256 + threadIdx.x;
  if (p >= (long long)w * h) return;
  const int x = (int)(p % w), y = (int)(p / w);
  // source centres j + 0.5 in [lo, hi): j in [ceil(lo - 0.5), ceil(hi - 0.5))
  const int j0 = max(0, (int)ceil(x * a.sx - 0.5)), j1 = min(a.src_w, (int)ceil((x + 1) * a.sx - 0.5));
  const int i0 = max(0, (int)ceil(y * a.sy - 0.5)), i1 = min(a.src_h, (int)ceil((y + 1) * a.sy - 0.5));
  double sum = 0.0;
  int n = 0;
  for (int i = i0; i < i1; ++i)
    for (int j = j0; j < j1; ++j) {
      const float z = __ldg(a.src + (size_t)i * a.src_w + j);
      if (depth_valid(z)) { sum += z; ++n; }
    }
  float z = NAN;
  if (n > 0) {
    z = (float)(sum / n);
  } else {
    const int jc = min(a.src_w - 1, (int)floor((x + 0.5) * a.sx)), ic = min(a.src_h - 1, (int)floor((y + 0.5) * a.sy));
    const float zc = __ldg(a.src + (size_t)ic * a.src_w + jc);
    if (depth_valid(zc)) z = zc;
  }
  float out = NAN;
  if (!isnan(z)) {
    float d[3];
    camera_pixel_direction(a.cam, a.has_distortion, (float)x + 0.5f, (float)y + 0.5f, d);
    const float cos_axis = d[0] * a.cam.orientation[6] + d[1] * a.cam.orientation[7] + d[2] * a.cam.orientation[8];
    const float t = z / cos_axis * a.factor;
    out = depth_valid(t) ? t : NAN;
  }
  a.dst[p] = out;
}

}  // namespace nfb
