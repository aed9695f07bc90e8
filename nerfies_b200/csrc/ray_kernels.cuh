// Per-ray kernels around the field evaluation: condition vectors, coarse
// sampling, volumetric rendering, hierarchical resampling.  All fp32, written
// in the reference's operation order; one warp per ray, data staged in shared
// memory so global accesses are coalesced 128-bit where the layout allows.
#pragma once
#include <math_constants.h>

#include "../../include/nerfies_b200.h"
#include "common.cuh"

namespace nfb {

// ---------------------------------------------------------------------------
// The per-ray condition vector of get_condition_inputs (models.py:186-228):
//   [warp glo code (G) | trunk (tc) | alpha (ac) | rgb: viewdir posenc (dv), appearance (ac), camera (cc)]
// The rgb condition repeats the appearance code iff it is the alpha condition (models.py:206-207).
// ---------------------------------------------------------------------------
struct CondLayout {
  int G, tc, ac, dv, cc;          // block widths (0: absent)
  int A, C;                       // appearance / camera table widths
  int stride;                     // floats per ray (1 when every block is absent)
  __host__ __device__ int rc() const { return dv + ac + cc; }
};

inline CondLayout cond_layout(const nfb_config& c) {
  CondLayout L{};
  L.G = c.warp_field_type != NFB_WARP_NONE ? c.num_warp_features : 0;
  L.A = c.num_appearance_features;
  L.C = c.num_camera_features;
  L.tc = (c.use_appearance_metadata && c.use_trunk_condition) ? L.A : 0;
  L.ac = (c.use_appearance_metadata && c.use_alpha_condition) ? L.A : 0;
  L.dv = c.use_viewdirs ? 3 + 6 * c.num_nerf_viewdir_freqs : 0;
  L.cc = c.use_camera_metadata ? L.C : 0;
  L.stride = L.G + L.tc + L.ac + L.rc();
  if (L.stride == 0) L.stride = 1;
  return L;
}

enum CondSource { kCondWarp, kCondApp, kCondViewdir, kCondCam, kCondPad };

// Where column q of the condition vector comes from; j = the column within that source.
__device__ __forceinline__ CondSource cond_source(const CondLayout& L, int q, int& j) {
  if (q < L.G) { j = q; return kCondWarp; }
  q -= L.G;
  if (q < L.tc) { j = q; return kCondApp; }
  q -= L.tc;
  if (q < L.ac) { j = q; return kCondApp; }
  q -= L.ac;
  if (q < L.dv) { j = q; return kCondViewdir; }
  q -= L.dv;
  if (q < L.ac) { j = q; return kCondApp; }
  q -= L.ac;
  j = q;
  return q < L.cc ? kCondCam : kCondPad;
}

// Embedding-table row of a ray (GloEncoder, glo.py:41-53): row 0 without ids, ids past the table clamp.
__device__ __forceinline__ size_t embed_row(const unsigned* ids, int ray, int n) {
  return min(ids ? ids[ray] : 0u, (unsigned)(n - 1));
}

struct CondArgs {
  const float* viewdirs;          // (B,3)
  const unsigned* warp_id;        // (B) or null
  const unsigned* app_id;         // (B) or null
  const unsigned* cam_id;         // (B) or null
  const float* warp_table;        // (n_warp, G)
  const float* app_table;         // (n_app, A)
  const float* cam_table;         // (n_cam, C)
  int n_warp, n_app, n_cam;
  CondLayout layout;
  float* cond;                    // (B, stride)
  int num_rays;
  int encoded;                    // metadata_encoded=True: the id pointers are (B, G|A|C) float embeddings
};

__global__ void ray_cond_kernel(const CondArgs a) {
  const CondLayout& L = a.layout;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)a.num_rays * L.stride) return;
  const int ray = (int)(idx / L.stride);
  int j;
  const CondSource src = cond_source(L, (int)(idx - (long long)ray * L.stride), j);
  // warping.py:186-187, models.py:198-199, 210-211: metadata_encoded passes the embeddings themselves
  auto embed = [&](const unsigned* ids, const float* table, int n, int width) {
    if (a.encoded && ids) return reinterpret_cast<const float*>(ids)[(size_t)ray * width + j];
    return table[embed_row(ids, ray, n) * width + j];
  };
  float v = 0.f;
  if (src == kCondWarp) {
    v = embed(a.warp_id, a.warp_table, a.n_warp, L.G);
  } else if (src == kCondApp) {
    v = embed(a.app_id, a.app_table, a.n_app, L.A);
  } else if (src == kCondCam) {
    v = embed(a.cam_id, a.cam_table, a.n_cam, L.C);
  } else if (src == kCondViewdir) {
    const float d[3] = {a.viewdirs[ray * 3 + 0], a.viewdirs[ray * 3 + 1], a.viewdirs[ray * 3 + 2]};
    v = (j < 3) ? d[j] : posenc_feature(d, j - 3);
  }
  a.cond[idx] = v;
}

// ---------------------------------------------------------------------------
// The per-ray terms of a NeRF level whose bottleneck the tensor-core program folds (TcFold,
// field_tc.cuh), from the condition vector, for the field pass that follows:
//   bias[ray, j] = c_r[j] + cond_rgb . W_r[W:, j]    (j < nr; zero up to cols)
//   alpha[ray]   = c_a + cond_alpha . w_a[W:]        (with an alpha condition)
// c_r = b_b W_r[:W] + b_r and c_a = b_a + b_b w_a[:W] come from fold_kernel.  fp64 sums of the exact
// fp32 products, rounded once.  One thread per output; consecutive threads write consecutive columns.
// ---------------------------------------------------------------------------
struct RayBiasArgs {
  const float* cond;              // (B, stride)
  int stride, num_rays;
  const float* w_rc;              // W_r[W:], rc rows of ldr
  int ldr, rc, rc_off, nr, cols;
  const float* c_r;               // (nr)
  const float* w_ac;              // w_a[W:], ac rows of lda (column 0)
  int lda, ac, ac_off;
  const float* c_a;               // (1)
  float* bias;                    // (B, cols)
  float* alpha;                   // (B)
};

__global__ void ray_bias_kernel(const RayBiasArgs a) {
  const int per = a.cols + (a.ac > 0);
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)a.num_rays * per) return;
  const long long ray = idx / per;
  const int j = (int)(idx - ray * per);
  const float* cond = a.cond + ray * a.stride;
  if (j < a.cols) {
    double v = 0.0;
    if (j < a.nr) {
      v = (double)a.c_r[j];
      for (int q = 0; q < a.rc; ++q)
        v = fma((double)cond[a.rc_off + q], (double)a.w_rc[(size_t)q * a.ldr + j], v);
    }
    a.bias[ray * a.cols + j] = (float)v;
  } else {
    double v = (double)a.c_a[0];
    for (int q = 0; q < a.ac; ++q) v = fma((double)cond[a.ac_off + q], (double)a.w_ac[(size_t)q * a.lda], v);
    a.alpha[ray] = (float)v;
  }
}

// ---------------------------------------------------------------------------
// modules.TimeEncoder (modules.py:297-322) per ray: annealed positional encoding
// of the timestamp, MLP(depth 6, width 64, skips (4,)) + `features`-wide output
// layer; writes (or, 'blend' encoder of TranslationField, warping.py:128-133,
// blends into) the warp-embedding block cond[:, 0:G].  fp32 FFMA, one CTA per
// kTimeRays rays, thread j owns output channel j.  Per-ray work (~26 K MAC) is
// negligible next to the per-sample field evaluation.
// ---------------------------------------------------------------------------
constexpr int kTimeRays = 8;
constexpr int kTimeThreads = 128;
constexpr int kTimeMaxIn = 40;     // 1 + 2 F, F <= 19

// Input k of the TimeEncoder at timestamp t (its input stage, shared by time_embed_kernel and the training
// tier's time_encode_kernel so that both see bitwise the same encoding): t itself, then per frequency f
// window[f] sin(2^f t) and window[f] sin(2^f t + pi/2) (modules.py:213-228 with C = 1).
__device__ __forceinline__ float time_encoding(float t, int k, const float* window) {
  if (k == 0) return t;
  const int f = (k - 1) >> 1, which = (k - 1) & 1;
  float ang = t * exp2f((float)f);
  if (which) ang = ang + kHalfPiF;
  return window[f] * sinf(ang);
}

struct TimeArgs {
  const float* params;           // packed dense buffer
  Net net;                       // hidden layers + output layer
  const float* time_f;           // (B) float timestamps, or null
  const unsigned* time_id;       // (B) ids used as timestamps ('blend': float(id)), or null
  int F;                         // metadata_encoder_num_freqs
  float window[20];              // cosine_easing_window(F, time_alpha)
  int blend;
  float time_alpha;
  float* cond;                   // (B, stride): block [0, G) is read (blend) / written
  int stride, G, num_rays;
};

__global__ void __launch_bounds__(kTimeThreads)
time_embed_kernel(const __grid_constant__ TimeArgs a) {
  __shared__ float xbuf[2][kTimeRays][kMaxWidth];
  __shared__ float in[kTimeRays][kTimeMaxIn];
  const int tid = threadIdx.x;
  const int ray0 = blockIdx.x * kTimeRays;
  const int din = 1 + 2 * a.F;
  for (int i = tid; i < kTimeRays * din; i += kTimeThreads) {
    const int r = i / din, k = i - r * din;
    const int ray = min(ray0 + r, a.num_rays - 1);
    const float t = a.time_f ? a.time_f[ray] : (float)a.time_id[ray];
    in[r][k] = time_encoding(t, k, a.window);
  }
  __syncthreads();
  int cur = 0;
  for (int s = 0; s < a.net.n_steps; ++s) {
    const Step& st = a.net.steps[s];
    const float* W = a.params + st.w_off;
    const float* src = xbuf[cur][0];
    float* dst = xbuf[cur ^ 1][0];
    for (int j = tid; j < st.n; j += kTimeThreads) {
      float acc[kTimeRays];
#pragma unroll
      for (int r = 0; r < kTimeRays; ++r) acc[r] = 0.f;
      for (int k = 0; k < st.k_x; ++k) {
        const float w = __ldg(W + (size_t)k * st.npad + j);
#pragma unroll
        for (int r = 0; r < kTimeRays; ++r) acc[r] = fmaf(src[r * kMaxWidth + k], w, acc[r]);
      }
      for (int k = 0; k < st.k_in; ++k) {
        const float w = __ldg(W + (size_t)(st.k_x + k) * st.npad + j);
#pragma unroll
        for (int r = 0; r < kTimeRays; ++r) acc[r] = fmaf(in[r][st.in_off + k], w, acc[r]);
      }
      const float b = __ldg(a.params + st.b_off + j);
#pragma unroll
      for (int r = 0; r < kTimeRays; ++r) dst[r * kMaxWidth + j] = apply_act(acc[r] + b, st.act);
    }
    __syncthreads();
    cur ^= 1;
  }
  for (int i = tid; i < kTimeRays * a.G; i += kTimeThreads) {
    const int r = i / a.G, q = i - r * a.G;
    const int ray = ray0 + r;
    if (ray >= a.num_rays) continue;
    float v = xbuf[cur][r][q];
    float* c = a.cond + (size_t)ray * a.stride + q;
    if (a.blend) v = (1.0f - a.time_alpha) * *c + a.time_alpha * v;     // warping.py:132-133
    *c = v;
  }
}

// ---------------------------------------------------------------------------
// sample_along_rays z_vals (model_utils.py:56-70).  z_lin/lower/upper are the
// per-model tables built on the host exactly as the reference builds them.
// ---------------------------------------------------------------------------
__global__ void coarse_z_kernel(const float* __restrict__ z_lin, const float* __restrict__ lower,
                                const float* __restrict__ upper, const float* __restrict__ t_rand,
                                float* __restrict__ z, int num_rays, int nc) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)num_rays * nc) return;
  const int i = (int)(idx % nc);
  if (t_rand) {
    z[idx] = lower[i] + (upper[i] - lower[i]) * t_rand[idx];
  } else {
    z[idx] = z_lin[i];
  }
}

// ---------------------------------------------------------------------------
// volumetric_rendering (model_utils.py:76-136) + compute_depth_map (:218-263).
// One warp per ray; the exclusive cumprod and the cumsum run sequentially on
// lane 0 (same order as the reference's scan), everything else is lane-parallel.
// ---------------------------------------------------------------------------
constexpr int kRaysPerBlock = 4;
constexpr int kMaxSamples = 1024;

struct CompositeArgs {
  const float4* samples;     // (B,S) r,g,b,sigma
  const float* z_vals;       // (B,S)
  const float* directions;   // (B,3)
  float* out;                // (B,6) rgb, depth, med_depth, acc
  float* weights;            // (B,S) or null
  int num_rays, S;
  int white_bg, sample_at_infinity;
};

__global__ void __launch_bounds__(32 * kRaysPerBlock)
composite_kernel(const CompositeArgs a) {
  extern __shared__ float sh[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ray = blockIdx.x * kRaysPerBlock + warp;
  if (ray >= a.num_rays) return;
  const int S = a.S;
  float* alpha = sh + warp * 3 * S;  // alpha -> weights
  float* zs = alpha + S;
  float* cum = zs + S;               // transmittance -> cumsum(weights)
  const float* zg = a.z_vals + (size_t)ray * S;
  const float4* sg = a.samples + (size_t)ray * S;
  const float dx = a.directions[ray * 3 + 0], dy = a.directions[ray * 3 + 1],
              dz = a.directions[ray * 3 + 2];
  const float dnorm = sqrtf(dx * dx + dy * dy + dz * dz);
  const float last = a.sample_at_infinity ? 1e10f : 1e-19f;
  for (int i = lane; i < S; i += 32) zs[i] = zg[i];
  __syncwarp();
  for (int i = lane; i < S; i += 32) {
    float dist = (i + 1 < S) ? (zs[i + 1] - zs[i]) : last;
    dist = dist * dnorm;
    // alpha = 1 - exp(-sigma*dist) (model_utils.py:108).  Evaluated as -expm1(-x):
    // the reference's float32 form loses all but ~12 bits when x is small (empty
    // space); expm1 returns the correctly rounded value of the same expression,
    // which is within the round-off band of any fp32 evaluation of 1 - exp(-x).
    alpha[i] = -expm1f(-sg[i].w * dist);
  }
  __syncwarp();
  if (lane == 0) {
    // accum_prod = [1, cumprod(1 - alpha[:-1] + eps)]  (model_utils.py:110-113)
    float t = 1.0f;
    for (int i = 0; i < S; ++i) {
      cum[i] = t;
      t = t * (1.0f - alpha[i] + 1e-10f);
    }
  }
  __syncwarp();
  float sr = 0.f, sg_ = 0.f, sb = 0.f, sd = 0.f, sa = 0.f, sa_nolast = 0.f;
  for (int i = lane; i < S; i += 32) {
    const float w = alpha[i] * cum[i];
    const float4 c = sg[i];
    sr += w * c.x; sg_ += w * c.y; sb += w * c.z;
    sd += w * zs[i];
    sa += w;
    if (i + 1 < S) sa_nolast += w;
    alpha[i] = w;
    if (a.weights) a.weights[(size_t)ray * S + i] = w;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sr += __shfl_xor_sync(0xffffffffu, sr, o);
    sg_ += __shfl_xor_sync(0xffffffffu, sg_, o);
    sb += __shfl_xor_sync(0xffffffffu, sb, o);
    sd += __shfl_xor_sync(0xffffffffu, sd, o);
    sa += __shfl_xor_sync(0xffffffffu, sa, o);
    sa_nolast += __shfl_xor_sync(0xffffffffu, sa_nolast, o);
  }
  __syncwarp();
  if (lane == 0) {
    // median depth: first sample whose cumulative weight reaches 0.5, else 0.
    float c = 0.f, med = 0.f;
    for (int i = 0; i < S; ++i) {
      c += alpha[i];
      if (c >= 0.5f) { med = zs[i]; break; }
    }
    float r = sr, g = sg_, b = sb;
    if (a.white_bg) {
      const float bg = 1.f - sa;
      r = r + bg; g = g + bg; b = b + bg;
    }
    float* o = a.out + (size_t)ray * 6;
    o[0] = r; o[1] = g; o[2] = b; o[3] = sd; o[4] = med;
    o[5] = a.sample_at_infinity ? sa_nolast : sa;
  }
}

// ---------------------------------------------------------------------------
// sample_pdf / piecewise_constant_pdf (model_utils.py:139-215) with the caller
// prep of models.py:353-357.  One warp per ray.
// ---------------------------------------------------------------------------
struct ResampleArgs {
  const float* z_coarse;   // (B,Nc)
  const float* w_coarse;   // (B,Nc)
  const float* u_rand;     // (B,Nf) or null
  const float* u_lin;      // (Nf) linspace(0,1,Nf)
  float* z_fine;           // (B,Nc+Nf) sorted
  // Optional, together: the new samples in draw order, and where each entry of z_fine came
  // from, as its index in concat(z_coarse, z_new) (gather_warped_kernel).
  float* z_new;            // (B,Nf) or null
  uint16_t* src;           // (B,Nc+Nf) or null
  int num_rays, nc, nf, npow2;
};

// One warp sorts keys[0, npow2) ascending (bitonic network); with kIdx, idx[] follows its keys.
template <bool kIdx>
__device__ __forceinline__ void bitonic_sort(float* keys, uint16_t* idx, int npow2, int lane) {
  for (int k = 2; k <= npow2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = lane; i < npow2; i += 32) {
        const int p = i ^ j;
        if (p > i) {
          const float x = keys[i], y = keys[p];
          const bool up = (i & k) == 0;
          if ((x > y) == up) {
            keys[i] = y; keys[p] = x;
            if constexpr (kIdx) { const uint16_t q = idx[i]; idx[i] = idx[p]; idx[p] = q; }
          }
        }
      }
      __syncwarp();
    }
  }
}

__global__ void __launch_bounds__(32 * kRaysPerBlock)
resample_kernel(const ResampleArgs a) {
  extern __shared__ float sh[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ray = blockIdx.x * kRaysPerBlock + warp;
  if (ray >= a.num_rays) return;
  const int nc = a.nc, nf = a.nf;
  const int nb = nc - 1;              // bins (= cdf entries), weights = nb - 1
  float* bins = sh + warp * (2 * nc + a.npow2);
  float* cdf = bins + nc;
  float* zs = cdf + nc;               // sort buffer, npow2 entries
  const float* zc = a.z_coarse + (size_t)ray * nc;
  const float* wc = a.w_coarse + (size_t)ray * nc;
  for (int i = lane; i < nc; i += 32) zs[i] = zc[i];
  __syncwarp();
  // z_vals_mid (models.py:353) and weights + eps (model_utils.py:156).
  for (int i = lane; i < nb; i += 32) bins[i] = .5f * (zs[i + 1] + zs[i]);
  for (int i = lane; i < nb - 1; i += 32) cdf[i + 1] = wc[i + 1] + 1e-5f;
  __syncwarp();
  if (lane == 0) {
    // weights.sum(), then cdf = [0, cumsum(weights / sum)] sequentially.
    float total = 0.f;
    for (int i = 1; i < nb; ++i) total += cdf[i];
    float c = 0.f;
    cdf[0] = 0.f;
    for (int i = 1; i < nb; ++i) {
      c += cdf[i] / total;
      cdf[i] = c;
    }
  }
  __syncwarp();
  for (int j = lane; j < nf; j += 32) {
    const float u = a.u_rand ? a.u_rand[(size_t)ray * nf + j] : a.u_lin[j];
    // count of cdf entries <= u  (mask = u >= cdf, model_utils.py:169).
    int lo = 0, hi = nb;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (cdf[mid] <= u) lo = mid + 1; else hi = mid;
    }
    const int idx = lo - 1;
    const int i0 = min(max(idx, 0), nb - 2);
    const int i1 = min(max(idx + 1, 1), nb - 1);
    const float c0 = cdf[i0], c1 = cdf[i1], b0 = bins[i0], b1 = bins[i1];
    float denom = c1 - c0;
    if (denom < 1e-5f) denom = 1.f;
    const float t = (u - c0) / denom;
    const float z = b0 + t * (b1 - b0);
    zs[nc + j] = z;
    if (a.z_new) a.z_new[(size_t)ray * nf + j] = z;
  }
  const int n = nc + nf;
  for (int i = n + lane; i < a.npow2; i += 32) zs[i] = CUDART_INF_F;
  // with `src`: the sort carries each key's index in concat(z_coarse, z_new) along; the swaps
  // depend on the keys alone, so z_fine is the same either way.  (Entries past n are the +inf
  // padding; index 0 keeps them in range should a non-finite key sort behind one.)
  uint16_t* si = a.src ? reinterpret_cast<uint16_t*>(sh + kRaysPerBlock * (2 * nc + a.npow2)) + warp * a.npow2
                       : nullptr;
  if (si)
    for (int i = lane; i < a.npow2; i += 32) si[i] = (uint16_t)(i < n ? i : 0);
  __syncwarp();
  // jnp.sort(concat([z_vals, z_samples])) (model_utils.py:213): bitonic network.
  if (si) bitonic_sort<true>(zs, si, a.npow2, lane);
  else bitonic_sort<false>(zs, nullptr, a.npow2, lane);
  float* out = a.z_fine + (size_t)ray * n;
  for (int i = lane; i < n; i += 32) out[i] = zs[i];
  if (si)
    for (int i = lane; i < n; i += 32) a.src[(size_t)ray * n + i] = si[i];
}

// ---------------------------------------------------------------------------
// The fine level's sample points from work already done (nfb_render_forward): the
// warped point of fine sample i of a ray is that of the coarse sample or of the new
// sample it was sorted from (ResampleArgs::src).  Both were warped from the same z
// bits by the same kernel and weights, so the result is what warping z_fine gives.
// One thread per fine sample.
// ---------------------------------------------------------------------------
struct GatherWarpedArgs {
  const float* warped_c;     // (B,Nc,3)  the coarse level's warped points
  const float* warped_new;   // (B,Nf,3)  the new samples' warped points, draw order
  const uint16_t* src;       // (B,Nc+Nf) index in concat(z_coarse, z_new)
  float* warped_fine;        // (B,Nc+Nf,3)
  int num_rays, nc, nf;
};

__global__ void gather_warped_kernel(const GatherWarpedArgs a) {
  const int n = a.nc + a.nf;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)a.num_rays * n) return;
  const long long ray = idx / n;
  const int s = a.src[idx];
  const float* p = s < a.nc ? a.warped_c + (ray * a.nc + s) * 3 : a.warped_new + (ray * a.nf + (s - a.nc)) * 3;
  float* o = a.warped_fine + idx * 3;
  o[0] = p[0]; o[1] = p[1]; o[2] = p[2];
}

}  // namespace nfb
