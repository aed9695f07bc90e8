// C ABI of nerfies_b200 (see include/nerfies_b200.h): handle, parameter
// packing, workspace and the launch sequence of NerfModel.__call__.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <string>
#include <vector>

#include "../../include/nerfies_b200.h"
#include "common.cuh"
#include "nfb_handle.h"
#include "field_simt.cuh"
#include "ray_kernels.cuh"
#include "camera_kernels.cuh"
#include "depth_kernels.cuh"
#include "pose_kernels.cuh"
#include "intrinsics_kernels.cuh"
#include "metrics_kernels.cuh"
#include "image_kernels.cuh"
#include "viz_kernels.cuh"
#include "capture_kernels.cuh"
#include "mesh_kernels.cuh"
#include "track_kernels.cuh"
#include "tc_common.cuh"
#include "tc_selftest.cuh"
#include "field_tc.cuh"

namespace {

using nfb::FieldProgram;
using nfb::Net;
using nfb::Step;

struct Builder {
  nfb_handle* h;
  long long off = 0;  // running float offset in the packed buffer

  long long alloc(long long n) {
    long long o = off;
    off += (n + 3) / 4 * 4;  // keep 16-byte alignment for cp.async
    return o;
  }

  // Adds one Dense layer made of `nparts` reference tensors side by side in N
  // (the SE(3) w and v heads are fused into one N=6 step).
  Step dense(const std::vector<std::string>& names, int k_x, int k_in, int in_off,
             const std::vector<int>& ns, int act, int src, int dst) {
    int n = 0;
    for (int v : ns) n += v;
    Step st{};
    st.k_x = k_x; st.k_in = k_in; st.in_off = in_off;
    st.n = n; st.npad = pad32(n);
    st.act = act; st.src = src; st.dst = dst;
    const int K = k_x + k_in;
    st.w_off = (int)alloc((long long)K * st.npad);
    st.b_off = (int)alloc(st.npad);
    int c = 0;
    for (size_t i = 0; i < names.size(); ++i) {
      h->specs.push_back({names[i] + "/kernel", K, ns[i], st.w_off, st.npad, c, 0});
      h->specs.push_back({names[i] + "/bias", 1, ns[i], st.b_off, st.npad, c, 0});
      c += ns[i];
    }
    return st;
  }
};

// Appends one step to `net`, whose step list is a fixed array: a network of more than kMaxSteps
// Dense layers (trunk, heads and branches together) is refused, never written past its end.
int push_step(Net& net, const Step& st, const std::string& name) {
  if (net.n_steps >= nfb::kMaxSteps)
    return fail("%s: too many layers (a network holds at most kMaxSteps = %d Dense layers)", name.c_str(),
                nfb::kMaxSteps);
  net.steps[net.n_steps++] = st;
  return 0;
}

int build_mlp(Builder& b, Net& net, const std::string& prefix, int depth, int width,
              unsigned skips, int in_dim, int in_off, int act, int first_src, int first_kx,
              int* cur_buf /* in: buffer holding X (if first_kx>0); out: buffer with result */) {
  // modules.MLP (modules.py:39-62): x = act(Dense([x, inputs] if i in skips else x)).
  int cur = *cur_buf;
  for (int i = 0; i < depth; ++i) {
    const bool skip = (skips >> i) & 1u;
    int k_x, k_in;
    if (i == 0) {
      if (skip) return fail("%s: a skip connection at layer 0 is not supported", prefix.c_str());
      k_x = first_kx; k_in = in_dim;
    } else {
      k_x = width; k_in = skip ? (first_kx + in_dim) : 0;
      if (skip && first_kx) return fail("%s: skip with a non-input first operand unsupported", prefix.c_str());
    }
    const int src = (i == 0) ? first_src : cur;
    int dst = (src == nfb::kB0) ? nfb::kB1 : nfb::kB0;
    if (push_step(net, b.dense({prefix + "/hidden_" + std::to_string(i)}, k_x, k_in, in_off, {width}, act, src, dst),
                  prefix))
      return -1;
    cur = dst;
  }
  *cur_buf = cur;
  return 0;
}

int build_programs(nfb_handle* h) {
  const nfb_config& c = h->cfg;
  Builder b{h};
  const bool use_warp = c.warp_field_type != NFB_WARP_NONE;
  const nfb::CondLayout& L = h->cond_layout = nfb::cond_layout(c);
  const int G = L.G, A = L.A, tc = L.tc, ac = L.ac, rc = L.rc();
  const int Dp = 3 + 6 * c.num_nerf_point_freqs;
  const int Dw = 3 + 6 * c.num_warp_freqs + G;
  if (Dp + tc + ac + rc > nfb::kMaxIn || (use_warp && Dw > nfb::kMaxIn))
    return fail("input feature block wider than %d", nfb::kMaxIn);
  auto check_width = [&](int w, const char* what) {
    if (w < 1 || w > nfb::kMaxWidth)
      return fail("%s=%d outside [1,%d]", what, w, nfb::kMaxWidth);
    return 0;
  };
  if (check_width(c.nerf_trunk_width, "nerf_trunk_width")) return -1;
  if (c.nerf_rgb_branch_depth > 0 && check_width(c.nerf_rgb_branch_width, "nerf_rgb_branch_width")) return -1;
  if (use_warp && check_width(c.warp_trunk_width, "warp_trunk_width")) return -1;
  if (c.alpha_channels != 1 || c.rgb_channels != 3)
    return fail("alpha_channels/rgb_channels must be 1/3 (volumetric_rendering assumes it)");
  if (c.nerf_trunk_depth < 1) return fail("nerf_trunk_depth must be >= 1");

  // Embedding tables come first in the parameter order (Flax names).
  Net warp{};
  if (use_warp) {
    // metadata encoder of the warp field (warping.py:109-123, 250-260)
    const int enc = c.warp_metadata_encoder;
    if (enc < NFB_WARP_ENC_GLO || enc > NFB_WARP_ENC_BLEND) return fail("bad warp_metadata_encoder");
    if (enc == NFB_WARP_ENC_BLEND && c.warp_field_type != NFB_WARP_TRANSLATION)
      return fail("Unknown metadata encoder type 'blend' for the SE(3) field (warping.py:258-260)");
    if (enc != NFB_WARP_ENC_TIME)
      h->specs.push_back({std::string(enc == NFB_WARP_ENC_GLO ? "warp_field/metadata_encoder" : "warp_field/glo_encoder") +
                          "/embed/embedding", c.num_warp_embeddings, G, 0, G, 0, 1});
    if (enc != NFB_WARP_ENC_GLO) {
      // modules.TimeEncoder (modules.py:297-322): depth 6, width 64, skips (4,), output = G features
      const int F = c.time_encoder_num_freqs;
      if (F < 0 || 1 + 2 * F > nfb::kTimeMaxIn) return fail("metadata_encoder_num_freqs=%d unsupported", F);
      const std::string root = enc == NFB_WARP_ENC_TIME ? "warp_field/metadata_encoder/mlp" : "warp_field/time_encoder/mlp";
      int tcur = nfb::kB0;
      Net tn{};
      if (build_mlp(b, tn, root, 6, 64, 1u << 4, 1 + 2 * F, 0, nfb::kRelu, nfb::kB0, 0, &tcur)) return -1;
      if (push_step(tn, b.dense({root + "/logit"}, 64, 0, 0, {G}, nfb::kNone, tcur, nfb::kOut0), root)) return -1;
      h->time_net = tn;
    }
    if (c.warp_field_type != NFB_WARP_SE3 && (c.warp_use_pivot || c.warp_use_translation))
      return fail("use_pivot / use_translation are SE3Field arguments (warping.py:242-243)");
    int cur = nfb::kB0;
    const bool se3 = c.warp_field_type == NFB_WARP_SE3;
    const std::string mlp_name = se3 ? "warp_field/trunk" : "warp_field/mlp";
    if (c.warp_trunk_depth < 1) return fail("warp trunk depth must be >= 1");
    if (build_mlp(b, warp, mlp_name, c.warp_trunk_depth, c.warp_trunk_width, c.warp_skips_mask,
                  Dw, 0, nfb::kRelu, nfb::kB0, 0, &cur)) return -1;
    if (se3) {
      // heads side by side in N: [w v (p) (t)] (warping.py:269-303)
      std::vector<std::string> names = {"warp_field/branches_w/logit", "warp_field/branches_v/logit"};
      std::vector<int> ns = {3, 3};
      if (c.warp_use_pivot) { names.push_back("warp_field/branches_p/logit"); ns.push_back(3); }
      if (c.warp_use_translation) { names.push_back("warp_field/branches_t/logit"); ns.push_back(3); }
      if (push_step(warp, b.dense(names, c.warp_trunk_width, 0, 0, ns, nfb::kNone, cur, nfb::kOut0), mlp_name))
        return -1;
    } else {
      if (push_step(warp, b.dense({"warp_field/mlp/logit"}, c.warp_trunk_width, 0, 0, {3}, nfb::kNone, cur,
                                  nfb::kOut0), mlp_name))
        return -1;
    }
  }
  if (c.use_appearance_metadata)
    h->specs.push_back({"appearance_encoder/embed/embedding", c.num_appearance_embeddings, A, 0, A, 0, 2});
  if (c.use_camera_metadata)
    h->specs.push_back({"camera_encoder/embed/embedding", c.num_camera_embeddings,
                        c.num_camera_features, 0, c.num_camera_features, 0, 3});

  const int levels = c.num_fine_samples > 0 ? 2 : 1;
  for (int lv = 0; lv < levels; ++lv) {
    const std::string root = lv == 0 ? "nerf_mlps_coarse" : "nerf_mlps_fine";
    Net nerf{};
    const int W = c.nerf_trunk_width;
    int cur = nfb::kB0;
    if (build_mlp(b, nerf, root + "/MLP_0", c.nerf_trunk_depth, W, c.nerf_skips_mask, Dp + tc, 0,
                  c.activation, nfb::kB0, 0, &cur)) return -1;
    const int P = cur;
    const int Q = (P == nfb::kB0) ? nfb::kB1 : nfb::kB0;
    const bool has_cond = ac > 0 || rc > 0;
    // Parameter order follows the Flax tree: MLP_0, bottleneck, MLP_1 (rgb), MLP_2 (alpha);
    // execution order is bottleneck, alpha, rgb (alpha must read the trunk output
    // before the rgb branch reuses that buffer).  Specs are re-sorted below.
    const size_t spec_mark = h->specs.size();
    if (has_cond && push_step(nerf, b.dense({root + "/bottleneck"}, W, 0, 0, {W}, nfb::kNone, P, Q), root))
      return -1;
    // alpha branch (depth 0: logit only), modules.py:152-157.
    const size_t alpha_mark = h->specs.size();
    if (push_step(nerf, ac > 0 ? b.dense({root + "/MLP_2/logit"}, W, ac, Dp + tc, {1}, nfb::kNone, Q, nfb::kOut0)
                               : b.dense({root + "/MLP_2/logit"}, W, 0, 0, {1}, nfb::kNone, P, nfb::kOut0),
                  root))
      return -1;
    const size_t rgb_mark = h->specs.size();
    // rgb branch, modules.py:159-164.
    int rsrc = (rc > 0) ? Q : P;
    int kx = W;
    int kin = rc, inoff = Dp + tc + ac;
    for (int i = 0; i < c.nerf_rgb_branch_depth; ++i) {
      const int dst = (rsrc == nfb::kB0) ? nfb::kB1 : nfb::kB0;
      if (push_step(nerf, b.dense({root + "/MLP_1/hidden_" + std::to_string(i)}, kx, kin, inoff,
                                  {c.nerf_rgb_branch_width}, c.activation, rsrc, dst), root))
        return -1;
      rsrc = dst; kx = c.nerf_rgb_branch_width; kin = 0;
    }
    if (push_step(nerf, b.dense({root + "/MLP_1/logit"}, kx, kin, inoff, {3}, nfb::kNone, rsrc, nfb::kOut1), root))
      return -1;
    // Re-order specs to the Flax order: bottleneck, MLP_1..., MLP_2.
    std::vector<ParamSpec> bott(h->specs.begin() + spec_mark, h->specs.begin() + alpha_mark);
    std::vector<ParamSpec> alpha(h->specs.begin() + alpha_mark, h->specs.begin() + rgb_mark);
    std::vector<ParamSpec> rgb(h->specs.begin() + rgb_mark, h->specs.end());
    h->specs.resize(spec_mark);
    h->specs.insert(h->specs.end(), bott.begin(), bott.end());
    h->specs.insert(h->specs.end(), rgb.begin(), rgb.end());
    h->specs.insert(h->specs.end(), alpha.begin(), alpha.end());

    FieldProgram& p = h->prog[lv];
    memset(&p, 0, sizeof(p));
    p.warp = warp;
    p.nerf = nerf;
    p.warp_type = c.warp_field_type;
    p.warp_pivot = use_warp && c.warp_use_pivot; p.warp_trans = use_warp && c.warp_use_translation;
    p.Fw = c.num_warp_freqs; p.G = G; p.Dw = Dw;
    p.Fp = c.num_nerf_point_freqs; p.Dp = Dp;
    p.tc = tc; p.ac = ac; p.rc = rc;
    p.cond_stride = L.stride;
    p.hidden_act = c.activation; p.sigma_act = c.sigma_activation;
    p.alpha_slot = nfb::kOut0; p.rgb_slot = nfb::kOut1;
  }
  if (levels == 1) h->prog[1] = h->prog[0];
  h->packed_floats = b.off;
  return 0;
}

// Host tables exactly as the reference builds them (float32 arithmetic).
void linspace01(int n, std::vector<float>& t) {
  t.resize(n);
  const double step = n > 1 ? 1.0 / (n - 1) : 0.0;
  for (int i = 0; i < n; ++i) t[i] = (float)(i * step);
  if (n > 1) t[n - 1] = 1.0f;
}

int upload(float** dst, const std::vector<float>& v) {
  NFB_CUDA(cudaMalloc(dst, std::max<size_t>(v.size(), 1) * sizeof(float)));
  if (!v.empty()) NFB_CUDA(cudaMemcpy(*dst, v.data(), v.size() * sizeof(float), cudaMemcpyHostToDevice));
  return 0;
}

int build_tables(nfb_handle* h) {
  const nfb_config& c = h->cfg;
  const int nc = c.num_coarse_samples;
  std::vector<float> t, z(nc), lower(nc), upper(nc), u;
  linspace01(nc, t);
  const float near_f = c.near_plane, far_f = c.far_plane;
  for (int i = 0; i < nc; ++i) {
    if (!c.use_linear_disparity) {
      // near * (1 - t) + far * t   (model_utils.py:58)
      volatile float a = near_f * (1.f - t[i]);
      volatile float bb = far_f * t[i];
      z[i] = a + bb;
    } else {
      // 1 / (1/near * (1 - t) + 1/far * t)   (model_utils.py:60)
      const float inv_near = (float)(1.0 / (double)near_f), inv_far = (float)(1.0 / (double)far_f);
      volatile float a = inv_near * (1.f - t[i]);
      volatile float bb = inv_far * t[i];
      volatile float s = a + bb;
      z[i] = 1.f / s;
    }
  }
  for (int i = 0; i < nc; ++i) {
    // mids/upper/lower of the stratified branch (model_utils.py:62-64).
    lower[i] = (i == 0) ? z[0] : .5f * (z[i] + z[i - 1]);
    upper[i] = (i == nc - 1) ? z[nc - 1] : .5f * (z[i + 1] + z[i]);
  }
  linspace01(std::max(c.num_fine_samples, 1), u);
  if (upload(&h->d_zlin, z) || upload(&h->d_lower, lower) || upload(&h->d_upper, upper) ||
      upload(&h->d_ulin, u))
    return -1;
  NFB_CUDA(cudaMalloc(&h->d_window, 64 * sizeof(float)));
  return 0;
}

// cosine_easing_window (modules.py:274-294) in float32: w[0..F).
void easing_window(float alpha, int F, float* w) {
  const float pi = 3.14159274101257324f;  // float32(np.pi)
  for (int k = 0; k < F; ++k) {
    float x = alpha - (float)k;
    x = fminf(fmaxf(x, 0.f), 1.f);
    volatile float arg = pi * x;
    arg = arg + pi;
    volatile float cv = cosf(arg);
    w[k] = 0.5f * (1.f + cv);
  }
}

int set_window(nfb_handle* h, float alpha, cudaStream_t stream) {
  if (h->cfg.warp_field_type == NFB_WARP_NONE) return 0;
  if (alpha == h->h_window_alpha) return 0;
  const int F = h->cfg.num_warp_freqs;
  if (F > 64) return fail("num_warp_freqs > 64");
  float w[64];
  easing_window(alpha, F, w);
  // Stream-ordered copy from pageable memory: the driver stages it before returning.
  NFB_CUDA(cudaMemcpyAsync(h->d_window, w, F * sizeof(float), cudaMemcpyHostToDevice, stream));
  h->h_window_alpha = alpha;
  return 0;
}

int launch_check(nfb_handle* h, const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("%s launch failed: %s", what, cudaGetErrorString(e));
  h->launches++;
  return 0;
}

// `time_encoder` false leaves the TimeEncoder's share of the warp block to the caller (the training tier runs
// it on a tape of its own: time_forward, train_api.cuh).
// With `warp_out` (B, G) the warp block alone is written there (nfb_warp_code; viewdirs may be null).
int run_cond(nfb_handle* h, int B, const float* viewdirs, const unsigned* warp_id,
             const unsigned* app_id, const unsigned* cam_id, cudaStream_t s, bool encoded = false,
             bool time_encoder = true, float* warp_out = nullptr) {
  const nfb_config& c = h->cfg;
  nfb::CondArgs a{};
  a.viewdirs = viewdirs; a.warp_id = warp_id; a.app_id = app_id; a.cam_id = cam_id;
  a.warp_table = h->d_warp_table; a.app_table = h->d_app_table; a.cam_table = h->d_cam_table;
  a.n_warp = c.num_warp_embeddings; a.n_app = c.num_appearance_embeddings; a.n_cam = c.num_camera_embeddings;
  a.layout = h->cond_layout; a.cond = h->d_cond; a.num_rays = B;
  a.encoded = encoded;
  if (warp_out) {
    nfb::CondLayout w{};
    w.G = h->cond_layout.G; w.A = h->cond_layout.A; w.C = h->cond_layout.C; w.stride = w.G;
    a.layout = w; a.cond = warp_out;
  }
  const nfb::CondLayout& L = a.layout;
  if (L.G + L.tc + L.ac + L.rc() == 0) return 0;
  const long long total = (long long)B * L.stride;
  const int enc = c.warp_field_type != NFB_WARP_NONE ? c.warp_metadata_encoder : NFB_WARP_ENC_GLO;
  if (enc == NFB_WARP_ENC_TIME && !encoded) a.warp_id = nullptr;   // `warp_id` carries float timestamps
  nfb::ray_cond_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(a);
  if (launch_check(h, "ray_cond_kernel")) return -1;
  if (enc != NFB_WARP_ENC_GLO && !encoded && warp_id && time_encoder) {
    // TimeEncoder on metadata['time'] ('time') or on float(id) ('blend', alpha = None)
    nfb::TimeArgs t{};
    t.params = h->d_packed; t.net = h->time_net;
    t.F = c.time_encoder_num_freqs;
    if (enc == NFB_WARP_ENC_TIME) t.time_f = reinterpret_cast<const float*>(warp_id);
    else t.time_id = warp_id;
    const float alpha = enc == NFB_WARP_ENC_TIME ? h->time_alpha : (float)t.F;   // modules.py:318-319
    easing_window(alpha, t.F, t.window);
    t.blend = enc == NFB_WARP_ENC_BLEND; t.time_alpha = h->time_alpha;
    t.cond = a.cond; t.stride = L.stride; t.G = L.G; t.num_rays = B;
    nfb::time_embed_kernel<<<(B + nfb::kTimeRays - 1) / nfb::kTimeRays, nfb::kTimeThreads, 0, s>>>(t);
    return launch_check(h, "time_embed_kernel");
  }
  return 0;
}

// Dynamic shared memory composite_kernel and resample_kernel are opted into (nfb_create).
constexpr int kRaySmemOptIn = 64 * 1024;
static_assert(nfb::kRaysPerBlock * 3 * nfb::kMaxSamples * sizeof(float) <= (size_t)kRaySmemOptIn,
              "composite_kernel's shared memory exceeds its opt-in at kMaxSamples");

// The fp16x3 kernel can finish a ray on chip (volumetric rendering fused into its rgb epilogue)
// when a ray's samples are whole 128-row tiles.
bool can_fuse_composite(const nfb_handle* h, int S) {
  return h->cfg.precision == NFB_PREC_FP16X3 && S % 128 == 0 && S <= nfb::kMaxSamples;
}

// Profiled launches (nfb_set_profiling) record the level's event pair around the field kernel.
// Warp passes and passes on given points are not timed here: with a warp field a level's field time
// spans its warp pass, the NeRF pass and whatever runs between them (prof_begin / prof_end).
int run_field(nfb_handle* h, int level, long long rows, int S, const float* origins,
              const float* directions, const float* z, float* samples, float* warped,
              bool use_warp, bool warp_only, cudaStream_t s, float* ray_out = nullptr,
              float* ray_weights = nullptr, const float* points = nullptr) {
  if (rows == 0) return 0;
  nfb::FieldArgs a{};
  a.ray_out = ray_out; a.ray_weights = ray_weights;
  a.white_bg = h->cfg.use_white_background; a.sample_at_infinity = h->cfg.use_sample_at_infinity;
  a.params = h->d_packed; a.origins = origins; a.directions = directions; a.z_vals = z;
  a.points = points;
  a.cond = h->d_cond; a.window = h->d_window; a.samples = samples; a.warped = warped;
  a.num_rows = rows; a.samples_per_ray = S; a.use_warp = use_warp; a.warp_only = warp_only;
  a.debug = h->debug_bits;
  const bool prof = h->profiling && !warp_only && !points;
  if (prof) NFB_CUDA(cudaEventRecord(h->ev[level][0], s));
  int rc;
  if (h->cfg.precision == NFB_PREC_FP32) {
    const long long tiles = (rows + nfb::kTM - 1) / nfb::kTM;
    nfb::field_simt_kernel<<<(unsigned)tiles, nfb::kSimtThreads, nfb::kSimtSmemBytes, s>>>(h->prog[level], a);
    rc = launch_check(h, "field_simt_kernel");
  } else {
    rc = nfb::tc::run_field_tc(h, level, a, s);
  }
  if (prof && rc == 0) {
    NFB_CUDA(cudaEventRecord(h->ev[level][1], s));
    h->ev_valid[level] = true;
  }
  return rc;
}

int prof_begin(nfb_handle* h, int level, cudaStream_t s) {
  if (h->profiling) NFB_CUDA(cudaEventRecord(h->ev[level][0], s));
  return 0;
}
int prof_end(nfb_handle* h, int level, cudaStream_t s) {
  if (!h->profiling) return 0;
  NFB_CUDA(cudaEventRecord(h->ev[level][1], s));
  h->ev_valid[level] = true;
  return 0;
}

// True when the samples are warped: then every level runs a warp pass (FieldArgs::warp_only) that
// writes the warped points, and the NeRF pass reads them (FieldArgs::points).  In the tensor-core
// kernel the warp MLP runs in 256-row tiles, the NeRF MLP in 128-row ones (field_tc.cuh).
bool warps(const nfb_handle* h, bool use_warp) {
  return use_warp && h->cfg.warp_field_type != NFB_WARP_NONE;
}

// The warp pass over the S samples of B rays at z (z = nullptr: free points, origins = the points).
int run_warp(nfb_handle* h, int level, long long B, int S, const float* origins, const float* directions,
             const float* z, float* warped, cudaStream_t s) {
  return run_field(h, level, B * S, S, origins, directions, z, nullptr, warped, true, true, s);
}

int run_composite(nfb_handle* h, int B, int S, const float* samples, const float* z,
                  const float* directions, float* out, float* weights, cudaStream_t s) {
  if (S > nfb::kMaxSamples) return fail("more than %d samples per ray", nfb::kMaxSamples);
  nfb::CompositeArgs a{};
  a.samples = reinterpret_cast<const float4*>(samples); a.z_vals = z; a.directions = directions;
  a.out = out; a.weights = weights; a.num_rays = B; a.S = S;
  a.white_bg = h->cfg.use_white_background; a.sample_at_infinity = h->cfg.use_sample_at_infinity;
  const int blocks = (B + nfb::kRaysPerBlock - 1) / nfb::kRaysPerBlock;
  const size_t smem = (size_t)nfb::kRaysPerBlock * 3 * S * sizeof(float);
  nfb::composite_kernel<<<blocks, 32 * nfb::kRaysPerBlock, smem, s>>>(a);
  return launch_check(h, "composite_kernel");
}

// `z_new` and `src` (both or neither): see ResampleArgs.
int run_resample(nfb_handle* h, int B, const float* zc, const float* wc, const float* u_rand,
                 float* zf, cudaStream_t s, float* z_new = nullptr, uint16_t* src = nullptr) {
  const nfb_config& c = h->cfg;
  nfb::ResampleArgs a{};
  a.z_coarse = zc; a.w_coarse = wc; a.u_rand = u_rand; a.u_lin = h->d_ulin; a.z_fine = zf;
  a.z_new = z_new; a.src = src;
  a.num_rays = B; a.nc = c.num_coarse_samples; a.nf = c.num_fine_samples;
  int p = 1;
  while (p < a.nc + a.nf) p <<= 1;
  a.npow2 = p;
  if (a.nc < 3) return fail("hierarchical sampling needs >= 3 coarse samples");
  const int blocks = (B + nfb::kRaysPerBlock - 1) / nfb::kRaysPerBlock;
  size_t smem = (size_t)nfb::kRaysPerBlock * (2 * a.nc + p) * sizeof(float);
  if (src) smem += (size_t)nfb::kRaysPerBlock * p * sizeof(uint16_t);
  // nfb_create admits Nc + Nf <= kMaxSamples: Nc < kMaxSamples and npow2 <= kMaxSamples
  static_assert(nfb::kRaysPerBlock * (3 * nfb::kMaxSamples * sizeof(float) + nfb::kMaxSamples * sizeof(uint16_t)) <=
                    (size_t)kRaySmemOptIn,
                "resample_kernel's shared memory exceeds its opt-in at kMaxSamples");
  nfb::resample_kernel<<<blocks, 32 * nfb::kRaysPerBlock, smem, s>>>(a);
  return launch_check(h, "resample_kernel");
}

// One level of nfb_render_forward: the field at the S samples of every ray, then volumetric
// rendering into `out` (and `weights`, if not null).  `warped` (nullable) receives the warped
// points; `points` (nullable) gives them instead of warping (FieldArgs::points).
int render_level(nfb_handle* h, int level, int B, int S, const float* origins, const float* directions,
                 const float* z, bool use_warp, float* out, float* weights, cudaStream_t s,
                 float* warped = nullptr, const float* points = nullptr) {
  const long long rows = (long long)B * S;
  if (can_fuse_composite(h, S))   // field + volumetric rendering in one kernel: 24 B per ray (+ the weights) leave the SM
    return run_field(h, level, rows, S, origins, directions, z, nullptr, warped, use_warp, false, s, out, weights,
                     points);
  if (run_field(h, level, rows, S, origins, directions, z, h->d_samples, warped, use_warp, false, s, nullptr, nullptr,
                points))
    return -1;
  return run_composite(h, B, S, h->d_samples, z, directions, out, weights, s);
}

// The coarse level of nfb_render_forward for a warped model: the warp pass writes the warped points
// into d_warped_c, where the NeRF pass and then the fine level (render_fine_reusing_warp) read them.
// Profiling times both launches as the level's field time.
int render_coarse_warped(nfb_handle* h, int B, const float* origins, const float* directions, float* out,
                         float* weights, cudaStream_t s) {
  const int nc = h->cfg.num_coarse_samples;
  if (prof_begin(h, 0, s) || run_warp(h, 0, B, nc, origins, directions, h->d_zc, h->d_warped_c, s) ||
      render_level(h, 0, B, nc, origins, directions, h->d_zc, true, out, weights, s, nullptr, h->d_warped_c))
    return -1;
  return prof_end(h, 0, s);
}

// The fine level of nfb_render_forward for a warped model.  Its Nc + Nf samples are the Nc coarse
// samples, whose warped points the coarse level kept in d_warped_c, and the Nf new ones: only those
// are warped (a warp pass in draw order), the two sets are gathered in z_fine's order, and the
// NeRF pass reads the gathered points.  A warped point depends on its z bits, its ray, the warp
// weights and the kernel alone, so this computes what warping all Nc + Nf samples computes.
// Profiling times the three launches as the level's field time.
int render_fine_reusing_warp(nfb_handle* h, int B, const float* origins, const float* directions,
                             const float* zf, float* out, float* weights, cudaStream_t s) {
  const nfb_config& c = h->cfg;
  const int nc = c.num_coarse_samples, nf = c.num_fine_samples, n = nc + nf;
  if (prof_begin(h, 1, s) || run_warp(h, 1, B, nf, origins, directions, h->d_znew, h->d_warped_new, s)) return -1;
  nfb::GatherWarpedArgs g{};
  g.warped_c = h->d_warped_c; g.warped_new = h->d_warped_new; g.src = h->d_src; g.warped_fine = h->d_warped_fine;
  g.num_rays = B; g.nc = nc; g.nf = nf;
  const long long total = (long long)B * n;
  nfb::gather_warped_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(g);
  if (launch_check(h, "gather_warped_kernel")) return -1;
  if (render_level(h, 1, B, n, origins, directions, zf, true, out, weights, s, nullptr, h->d_warped_fine)) return -1;
  return prof_end(h, 1, s);
}

// The tensor-core kernels never trap on a protocol error (see tc_common.cuh,
// mbar_wait): they raise a flag in mapped pinned host memory instead.  One int per
// process; every device's copy of the g_nfb_abort symbol points at it.
int* g_abort_host = nullptr;
unsigned long long g_abort_devices = 0;   // devices whose symbol has been set

int ensure_abort_flag() {
  int dev = 0;
  NFB_CUDA(cudaGetDevice(&dev));
  if (!g_abort_host) {
    NFB_CUDA(cudaHostAlloc(&g_abort_host, sizeof(int), cudaHostAllocMapped | cudaHostAllocPortable));
    *g_abort_host = 0;
  }
  if (dev < 64 && !(g_abort_devices >> dev & 1)) {
    int* dptr = nullptr;
    NFB_CUDA(cudaHostGetDevicePointer(&dptr, g_abort_host, 0));
    NFB_CUDA(cudaMemcpyToSymbol(nfb::tc::g_nfb_abort, &dptr, sizeof(dptr)));
    g_abort_devices |= 1ull << dev;
  }
  return 0;
}

int abort_check() {
  if (g_abort_host && *reinterpret_cast<volatile int*>(g_abort_host))
    return fail("a tensor-core kernel aborted: an mbarrier wait timed out (protocol error); its results are invalid "
                "and tensor-core launches are refused until nfb_reset_abort()");
  return 0;
}

// A handle's workspace (cond, z, samples, window table) is shared by its calls: work
// of consecutive calls must be ordered.  Calls on ONE stream are; when the caller
// switches streams the new stream first waits for the previous call's last kernel.
int enter_stream(nfb_handle* h, cudaStream_t s) {
  if (h->last_stream_valid && h->last_stream != s) {
    if (!h->ev_order) NFB_CUDA(cudaEventCreateWithFlags(&h->ev_order, cudaEventDisableTiming));
    NFB_CUDA(cudaEventRecord(h->ev_order, h->last_stream));
    NFB_CUDA(cudaStreamWaitEvent(s, h->ev_order, 0));
  }
  h->last_stream = s; h->last_stream_valid = true;
  return 0;
}

int check_call(nfb_handle* h, int B) {
  if (!h) return fail("null handle");
  if (abort_check()) return -1;
  if (!h->params_set) return fail("nfb_set_params has not been called");
  if (B < 0 || B > h->max_rays) return fail("num_rays=%d outside [0, max_rays=%d]", B, h->max_rays);
  return 0;
}

// Workspace of nfb_image_metrics: levels 1..4 of both images, then the fp64 partials of each
// scale's SSIM CTAs and of the level-0 downsample CTAs; every region 256-byte aligned.
struct MetricsPlan {
  int h[nfb::metrics::kScales], w[nfb::metrics::kScales];
  int tiles_x[nfb::metrics::kScales], tiles_y[nfb::metrics::kScales];
  long long level_off[nfb::metrics::kScales];   // bytes; X of level k, then Y (k >= 1)
  long long part_off[nfb::metrics::kScales];
  int pool_blocks;
  long long err_off, bytes;
};

int metrics_plan(int N, int height, int width, int C, MetricsPlan* p) {
  using namespace nfb::metrics;
  if (N < 1 || N > 65535) return fail("num_images=%d outside [1, 65535]", N);
  if (C < 1 || C > 4) return fail("channels=%d outside [1, 4]", C);
  if (height < kMinSize || width < kMinSize)
    return fail("MS-SSIM needs images of at least %dx%d (each of the %d scales must be >= %dx%d); got %dx%d",
                kMinSize, kMinSize, kScales, kTaps, kTaps, height, width);
  if ((height - kHalo + kTileH - 1) / kTileH > 65535) return fail("height=%d too large", height);
  auto align = [](long long b) { return (b + 255) / 256 * 256; };
  long long off = 0;
  for (int k = 0; k < kScales; ++k) {
    p->h[k] = k ? (p->h[k - 1] + 1) / 2 : height;
    p->w[k] = k ? (p->w[k - 1] + 1) / 2 : width;
    p->tiles_x[k] = (p->w[k] - kHalo + kTileW - 1) / kTileW;
    p->tiles_y[k] = (p->h[k] - kHalo + kTileH - 1) / kTileH;
    p->level_off[k] = off;
    if (k) off += 2 * align((long long)N * p->h[k] * p->w[k] * C * sizeof(float));
  }
  for (int k = 0; k < kScales; ++k) {
    p->part_off[k] = off;
    off += align((long long)N * C * p->tiles_x[k] * p->tiles_y[k] * 2 * sizeof(double));
  }
  p->pool_blocks = (int)(((long long)p->h[1] * p->w[1] + kThreads - 1) / kThreads);
  p->err_off = off;
  off += align((long long)N * p->pool_blocks * 3 * sizeof(double));
  p->bytes = off;
  return 0;
}

template <int C>
void launch_metrics(const MetricsPlan& p, int N, const float* image, const float* target,
                    const float* depth, const float* depth_target, char* ws, float* ms_ssim,
                    float* mse, float* depth_abs, cudaStream_t s) {
  using namespace nfb::metrics;
  float g[kTaps];                                      // _fspecial_gauss's kernel is the outer product of g
  double gs = 0.0;
  for (int t = 0; t < kTaps; ++t) gs += exp(-0.5 * (t - 5) * (t - 5) / (1.5 * 1.5));
  for (int t = 0; t < kTaps; ++t) g[t] = (float)(exp(-0.5 * (t - 5) * (t - 5) / (1.5 * 1.5)) / gs);
  const float* x = image;
  const float* y = target;
  for (int k = 0; k < kScales; ++k) {
    if (k < kScales - 1) {                             // level k + 1 (and, from level 0, MSE / depth)
      PoolArgs pa{};
      pa.x = x; pa.y = y; pa.h = p.h[k]; pa.w = p.w[k];
      pa.x_out = reinterpret_cast<float*>(ws + p.level_off[k + 1]);
      pa.y_out = pa.x_out + (long long)N * p.h[k + 1] * p.w[k + 1] * C;
      if (k == 0) {
        pa.err_part = reinterpret_cast<double*>(ws + p.err_off);
        pa.depth = depth; pa.depth_target = depth_target;
      }
      const long long blocks = ((long long)p.h[k + 1] * p.w[k + 1] + kThreads - 1) / kThreads;
      downsample_kernel<C><<<dim3((unsigned)blocks, N), kThreads, 0, s>>>(pa);
    }
    SsimArgs sa{};
    sa.x = x; sa.y = y; sa.h = p.h[k]; sa.w = p.w[k];
    sa.tiles_x = p.tiles_x[k]; sa.tiles_y = p.tiles_y[k];
    sa.part = reinterpret_cast<double*>(ws + p.part_off[k]);
    for (int t = 0; t < kTaps; ++t) sa.g[t] = g[t];
    ssim_level_kernel<C><<<dim3(sa.tiles_x, sa.tiles_y, N), kThreads, 0, s>>>(sa);
    if (k < kScales - 1) {
      x = reinterpret_cast<const float*>(ws + p.level_off[k + 1]);
      y = x + (long long)N * p.h[k + 1] * p.w[k + 1] * C;
    }
  }
  FinalArgs fa{};
  fa.C = C; fa.pool_blocks = p.pool_blocks;
  fa.values = (long long)p.h[0] * p.w[0] * C;
  for (int k = 0; k < kScales; ++k) {
    fa.tiles[k] = p.tiles_x[k] * p.tiles_y[k];
    fa.outputs[k] = (long long)(p.h[k] - kHalo) * (p.w[k] - kHalo);
    fa.part[k] = reinterpret_cast<const double*>(ws + p.part_off[k]);
  }
  fa.err_part = reinterpret_cast<const double*>(ws + p.err_off);
  fa.ms_ssim = ms_ssim; fa.mse = mse; fa.depth_abs = depth_abs;
  finalize_kernel<<<N, kThreads, 0, s>>>(fa);
}

// nfb_gather_rays, and with `pose` / `image` nfb_gather_rays_posed, and with `intrinsics`
// nfb_gather_rays_refined: one kernel, one pixel-to-ray path.
int gather_rays(const nfb_ray_table* table, long long first, long long count, float* origins, float* directions,
                float* pixels, float* rgb, int* appearance, int* camera, int* warp, float* time, const float* pose,
                int* image, const float* intrinsics, const int* group, int num_groups, void* stream) {
  if (!table) return fail("null ray table");
  const nfb_ray_table& t = *table;
  if (t.num_images < 1) return fail("ray table has %d images", t.num_images);
  if (t.num_rays < 1) return fail("ray table has %lld rays", t.num_rays);
  if (count < 0 || first < 0) return fail("negative ray range (first %lld, count %lld)", first, count);
  if (!t.cameras || !t.pixel_offsets) return fail("ray table needs cameras and pixel_offsets");
  if (rgb && !t.rgb) return fail("rgb requested but the ray table has none");
  if ((appearance && !t.appearance) || (camera && !t.camera) || (warp && !t.warp) || (time && !t.time))
    return fail("metadata requested but the ray table has none of that kind");
  if (intrinsics && (!group || num_groups < 1))
    return fail("intrinsics need a group map and num_groups >= 1 (got %d)", num_groups);
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail("no CUDA device: nerfies_b200 has no CPU path");
  if (count == 0) return 0;
  nfb::GatherArgs a{};
  a.t = t; a.first = first; a.count = count;
  a.origins = origins; a.directions = directions; a.pixels = pixels; a.rgb = rgb;
  a.appearance = appearance; a.camera = camera; a.warp = warp; a.time = time;
  a.pose = pose; a.image = image;
  a.intrinsics = intrinsics; a.group = group; a.num_groups = num_groups;
  nfb::gather_rays_kernel<<<(unsigned)((count + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("gather_rays_kernel launch failed: %s", cudaGetErrorString(e));
  return 0;
}
}  // namespace

extern "C" {

const char* nfb_last_error(void) { return g_error.c_str(); }
const char* nfb_version(void) { return "nerfies_b200 0.1 sm_90a"; }
long long nfb_kernel_launches(const nfb_handle* h) { return h ? h->launches : 0; }

static int launch_camera(const nfb_camera* cam, const float* pixels_in, long long first, long long count,
                         float* origins, float* directions, float* pixels_out, const float* intrinsics,
                         void* stream) {
  if (!cam) return fail("null argument");
  if (count < 0 || first < 0) return fail("negative pixel range");
  if (cam->image_size[0] < 1 || cam->image_size[1] < 1) return fail("image_size must be positive");
  if (!pixels_in && first + count > (long long)cam->image_size[0] * cam->image_size[1])
    return fail("pixel range [%lld, %lld) exceeds the %d x %d frame", first, first + count,
                cam->image_size[0], cam->image_size[1]);
  if (!(cam->focal_length != 0.f) || !(cam->pixel_aspect_ratio != 0.f)) return fail("focal_length and pixel_aspect_ratio must be non-zero");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail("no CUDA device: nerfies_b200 has no CPU path");
  if (count == 0) return 0;
  if (!directions) return fail("null argument");
  if ((reinterpret_cast<uintptr_t>(directions) | reinterpret_cast<uintptr_t>(origins)) & 15)
    return fail("origins / directions must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(pixels_out) & 7) return fail("pixels must be 8-byte aligned");
  nfb::CameraArgs a{};
  a.cam = *cam; a.pixels_in = pixels_in; a.first = first; a.count = count;
  a.origins = origins; a.directions = directions; a.pixels_out = pixels_out;
  a.has_distortion = nfb::camera_has_distortion(*cam);
  a.intrinsics = intrinsics;
  nfb::camera_rays_kernel<<<(unsigned)((count + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("camera_rays_kernel launch failed: %s", cudaGetErrorString(e));
  return 0;
}

int nfb_gather_rays(const nfb_ray_table* table, long long first, long long count, float* origins,
                    float* directions, float* pixels, float* rgb, int* appearance, int* camera, int* warp,
                    float* time, void* stream) {
  return gather_rays(table, first, count, origins, directions, pixels, rgb, appearance, camera, warp, time, nullptr,
                     nullptr, nullptr, nullptr, 0, stream);
}

int nfb_gather_rays_posed(const nfb_ray_table* table, long long first, long long count, const float* pose,
                          float* origins, float* directions, int* image, void* stream) {
  return gather_rays(table, first, count, origins, directions, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                     pose, image, nullptr, nullptr, 0, stream);
}

int nfb_gather_rays_refined(const nfb_ray_table* table, long long first, long long count, const float* pose,
                            const float* intrinsics, const int* group, int num_groups, float* origins,
                            float* directions, float* pixels, int* image, void* stream) {
  return gather_rays(table, first, count, origins, directions, pixels, nullptr, nullptr, nullptr, nullptr, nullptr,
                     pose, image, intrinsics, group, num_groups, stream);
}

int nfb_gather_depth(const nfb_ray_table* table, long long first, long long count, float* depth_out,
                     void* stream) {
  if (!table) return fail("null ray table");
  const nfb_ray_table& t = *table;
  if (t.num_rays < 1) return fail("ray table has %lld rays", t.num_rays);
  if (count < 0 || first < 0) return fail("negative ray range (first %lld, count %lld)", first, count);
  if (!t.depth) return fail("depth requested but the ray table has none");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail("no CUDA device: nerfies_b200 has no CPU path");
  if (count == 0) return 0;
  if (!depth_out) return fail("null argument");
  nfb::gather_depth_kernel<<<(unsigned)((count + 255) / 256), 256, 0, (cudaStream_t)stream>>>(t, first, count,
                                                                                             depth_out);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("gather_depth_kernel launch failed: %s", cudaGetErrorString(e));
  return 0;
}

long long nfb_pose_grad_workspace_size(int num_images, long long count) {
  if (num_images < 1 || count < 0) return -1;
  return std::max<long long>(1, (count + nfb::kPoseRays - 1) / nfb::kPoseRays) * num_images * 6 * (long long)sizeof(double);
}

int nfb_pose_grad(int num_images, const float* pose, const int* image, const float* directions,
                  const float* d_origins, const float* d_directions, long long count, float* grad, void* workspace,
                  long long workspace_bytes, void* stream) {
  if (num_images < 1) return fail("pose grad: num_images=%d must be >= 1", num_images);
  if (count < 0) return fail("pose grad: count=%lld must be >= 0", count);
  if (!grad) return fail("pose grad: null grad");
  if (count > 0 && (!image || !directions)) return fail("pose grad: null image / directions");
  if (!d_origins && !d_directions) return fail("pose grad: d_origins and d_directions are both null");
  const long long need = nfb_pose_grad_workspace_size(num_images, count);
  if (!workspace || workspace_bytes < need)
    return fail("pose grad: the workspace holds %lld bytes, %lld needed", workspace_bytes, need);
  if (count == 0) return 0;
  const int blocks = (int)((count + nfb::kPoseRays - 1) / nfb::kPoseRays);
  nfb::PoseGradArgs a{num_images, count, pose, image, directions, d_origins, d_directions,
                      static_cast<double*>(workspace), grad};
  cudaStream_t s = (cudaStream_t)stream;
  nfb::pose_partials_kernel<<<blocks, nfb::kPoseRays, 0, s>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("pose_partials_kernel launch failed: %s", cudaGetErrorString(e));
  nfb::pose_finish_kernel<<<(num_images + 127) / 128, 128, 0, s>>>(a, blocks);
  e = cudaGetLastError();
  if (e != cudaSuccess) return fail("pose_finish_kernel launch failed: %s", cudaGetErrorString(e));
  return 0;
}


int nfb_camera_rays(const nfb_camera* cam, long long first_pixel, long long count, float* origins,
                    float* directions, float* pixels, void* stream) {
  return launch_camera(cam, nullptr, first_pixel, count, origins, directions, pixels, nullptr, stream);
}

int nfb_pixels_to_rays(const nfb_camera* cam, const float* pixels, long long n, float* directions,
                       void* stream) {
  if (!pixels && n > 0) return fail("null argument");
  return launch_camera(cam, pixels, 0, n, nullptr, directions, nullptr, nullptr, stream);
}

int nfb_pixels_to_rays_refined(const nfb_camera* cam, const float* intrinsics, const float* pixels, long long n,
                               float* directions, void* stream) {
  if (!pixels && n > 0) return fail("null argument");
  return launch_camera(cam, pixels, 0, n, nullptr, directions, nullptr, intrinsics, stream);
}

long long nfb_intrinsics_grad_workspace_size(int num_groups, long long count) {
  if (num_groups < 1 || count < 0) return -1;
  return std::max<long long>(1, (count + nfb::kIntrinsicsRays - 1) / nfb::kIntrinsicsRays) * num_groups * 8 *
         (long long)sizeof(double);
}

int nfb_intrinsics_grad(const nfb_camera* cameras, int num_images, const float* pose, const float* intrinsics,
                        const int* group, int num_groups, unsigned parts, const int* image, const float* pixels,
                        const float* directions, const float* d_directions, long long count, float* grad,
                        void* workspace, long long workspace_bytes, void* stream) {
  if (num_images < 1) return fail("intrinsics grad: num_images=%d must be >= 1", num_images);
  if (num_groups < 1) return fail("intrinsics grad: num_groups=%d must be >= 1", num_groups);
  if (count < 0) return fail("intrinsics grad: count=%lld must be >= 0", count);
  if (parts & ~15u) return fail("intrinsics grad: unknown parts bits 0x%x", parts);
  if (!grad || !cameras || !group) return fail("intrinsics grad: null grad / cameras / group");
  if (count > 0 && (!image || !pixels || !directions || !d_directions))
    return fail("intrinsics grad: null image / pixels / directions / d_directions");
  const long long need = nfb_intrinsics_grad_workspace_size(num_groups, count);
  if (!workspace || workspace_bytes < need)
    return fail("intrinsics grad: the workspace holds %lld bytes, %lld needed", workspace_bytes, need);
  if (count == 0 || parts == 0) return 0;
  const int blocks = (int)((count + nfb::kIntrinsicsRays - 1) / nfb::kIntrinsicsRays);
  nfb::IntrinsicsGradArgs a{cameras, num_images, pose, intrinsics, group, num_groups, parts, image, pixels,
                            directions, d_directions, count, static_cast<double*>(workspace), grad};
  cudaStream_t s = (cudaStream_t)stream;
  nfb::intrinsics_partials_kernel<<<blocks, nfb::kIntrinsicsRays, 0, s>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("intrinsics_partials_kernel launch failed: %s", cudaGetErrorString(e));
  nfb::intrinsics_finish_kernel<<<(num_groups + 127) / 128, 128, 0, s>>>(a, blocks);
  e = cudaGetLastError();
  if (e != cudaSuccess) return fail("intrinsics_finish_kernel launch failed: %s", cudaGetErrorString(e));
  return 0;
}

long long nfb_image_metrics_workspace_size(int num_images, int height, int width, int channels) {
  MetricsPlan p;
  return metrics_plan(num_images, height, width, channels, &p) ? -1 : p.bytes;
}

int nfb_image_metrics(int num_images, int height, int width, int channels, const float* image,
                      const float* target, const float* depth, const float* depth_target, void* workspace,
                      long long workspace_bytes, float* ms_ssim, float* mse, float* depth_abs, void* stream) {
  MetricsPlan p;
  if (metrics_plan(num_images, height, width, channels, &p)) return -1;
  if (!image || !target) return fail("image and target must not be null");
  if ((depth == nullptr) != (depth_target == nullptr)) return fail("depth and depth_target are nullable only together");
  if (depth_abs && !depth) return fail("depth_abs needs depth and depth_target");
  if (!workspace || workspace_bytes < p.bytes)
    return fail("workspace of %lld bytes is smaller than the %lld bytes nfb_image_metrics_workspace_size returns",
                workspace ? workspace_bytes : 0ll, p.bytes);
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail("workspace must be 256-byte aligned");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail("no CUDA device: nerfies_b200 has no CPU path");
  char* ws = static_cast<char*>(workspace);
  cudaStream_t s = (cudaStream_t)stream;
  switch (channels) {
    case 1: launch_metrics<1>(p, num_images, image, target, depth, depth_target, ws, ms_ssim, mse, depth_abs, s); break;
    case 2: launch_metrics<2>(p, num_images, image, target, depth, depth_target, ws, ms_ssim, mse, depth_abs, s); break;
    case 3: launch_metrics<3>(p, num_images, image, target, depth, depth_target, ws, ms_ssim, mse, depth_abs, s); break;
    default: launch_metrics<4>(p, num_images, image, target, depth, depth_target, ws, ms_ssim, mse, depth_abs, s); break;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("image metrics launch failed: %s", cudaGetErrorString(e));
  return 0;
}

int nfb_image_quantize(const float* src, long long n, int bits, float scale, void* dst, void* stream) {
  if (bits != 8 && bits != 16) return fail("nfb_image_quantize: bits must be 8 or 16, got %d", bits);
  if (n < 0) return fail("nfb_image_quantize: negative count %lld", n);
  if (!(scale > 0.0f) || std::isinf(scale)) return fail("nfb_image_quantize: scale must be positive and finite");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail("no CUDA device: nerfies_b200 has no CPU path");
  if (n == 0) return 0;
  if (!src || !dst) return fail("null argument");
  if (reinterpret_cast<uintptr_t>(src) & 3) return fail("src must be 4-byte aligned");
  if (bits == 16 && (reinterpret_cast<uintptr_t>(dst) & 1)) return fail("a 16-bit dst must be 2-byte aligned");
  const bool aligned = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0;
  const long long vec = aligned ? n / (128 / bits) : 0;
  const long long threads = std::max(vec, n - vec * (128 / bits));
  const unsigned blocks = (unsigned)std::min<long long>((threads + nfb::image::kThreads - 1) / nfb::image::kThreads, 1 << 16);
  cudaStream_t s = (cudaStream_t)stream;
  if (bits == 8)
    nfb::image::image_quantize_kernel<unsigned char><<<blocks, nfb::image::kThreads, 0, s>>>(
        src, n, vec, scale, static_cast<unsigned char*>(dst));
  else
    nfb::image::image_quantize_kernel<unsigned short><<<blocks, nfb::image::kThreads, 0, s>>>(
        src, n, vec, scale, static_cast<unsigned short*>(dst));
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("image_quantize_kernel launch failed: %s", cudaGetErrorString(e));
  return 0;
}

static int device_sms(int* sms) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    return fail("no CUDA device: nerfies_b200 has no CPU path");
  return 0;
}

int nfb_frame_pyramid(const unsigned char* src, int height, int width, long long src_pitch, int num_levels,
                      const int* scales, unsigned char* const* dst, void* stream) {
  using namespace nfb::capture;
  if (num_levels < 1 || num_levels > kMaxLevels)
    return fail("nfb_frame_pyramid: num_levels=%d outside [1, %d]", num_levels, kMaxLevels);
  if (!src || !scales || !dst) return fail("null argument");
  PyramidArgs a{};
  a.src = src; a.src_pitch = src_pitch; a.height = height; a.width = width; a.num_levels = num_levels;
  int S = 0;
  for (int l = 0; l < num_levels; ++l) {
    const int s = scales[l];
    if (s < 1 || (s != 1 && s % 2)) return fail("nfb_frame_pyramid: scale %d is neither 1 nor even", s);
    if (!dst[l]) return fail("null argument");
    a.scale[l] = s; a.dst[l] = dst[l];
    S = std::max(S, s);
  }
  for (int l = 0; l < num_levels; ++l)
    if (S % a.scale[l]) return fail("nfb_frame_pyramid: scale %d does not divide the largest scale %d", a.scale[l], S);
  if (height < S || width < S || height % S || width % S)
    return fail("nfb_frame_pyramid: frame %d x %d is not a positive multiple of the largest scale %d", height, width, S);
  if (src_pitch < 3ll * width) return fail("nfb_frame_pyramid: src_pitch %lld is below 3 * width", src_pitch);
  a.max_scale = S;
  int sms = 0;
  if (device_sms(&sms)) return -1;
  const long long blocks = ((long long)(height / S) * (width / S) + 255) / 256;
  nfb::capture::frame_pyramid_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("frame_pyramid_kernel launch failed: %s", cudaGetErrorString(e));
  return 0;
}

long long nfb_blur_scores_workspace_size(int num_frames) {
  if (num_frames < 0) return fail("nfb_blur_scores: negative frame count %d", num_frames);
  return 16ll * num_frames;
}

int nfb_blur_scores(const unsigned char* frames, int num_frames, int height, int width, void* workspace,
                    long long workspace_bytes, double* scores, void* stream) {
  using namespace nfb::capture;
  if (num_frames < 0 || num_frames > 65535) return fail("nfb_blur_scores: num_frames=%d outside [0, 65535]", num_frames);
  if (height < 1 || width < 1) return fail("nfb_blur_scores: frame size %d x %d must be positive", height, width);
  if (num_frames == 0) return 0;
  if (!frames || !scores || !workspace) return fail("null argument");
  if (workspace_bytes < 16ll * num_frames)
    return fail("nfb_blur_scores: workspace of %lld bytes is smaller than the %lld bytes needed", workspace_bytes,
                16ll * num_frames);
  if ((reinterpret_cast<uintptr_t>(workspace) | reinterpret_cast<uintptr_t>(scores)) & 7)
    return fail("nfb_blur_scores: workspace and scores must be 8-byte aligned");
  int sms = 0;
  if (device_sms(&sms)) return -1;
  cudaStream_t s = (cudaStream_t)stream;
  BlurArgs a{};
  a.frames = frames; a.num_frames = num_frames; a.height = height; a.width = width;
  a.sums = static_cast<unsigned long long*>(workspace); a.scores = scores;
  cudaError_t e = cudaMemsetAsync(workspace, 0, 16ll * num_frames, s);
  if (e != cudaSuccess) return fail("nfb_blur_scores: memset failed: %s", cudaGetErrorString(e));
  const long long pixels = (long long)height * width;
  const long long per_frame = std::max(1ll, std::min((pixels + 2047) / 2048, std::max(1ll, 8ll * sms / num_frames)));
  blur_sums_kernel<<<dim3((unsigned)per_frame, num_frames), 256, 0, s>>>(a);
  blur_finalize_kernel<<<(num_frames + 127) / 128, 128, 0, s>>>(a);
  e = cudaGetLastError();
  if (e != cudaSuccess) return fail("blur score launch failed: %s", cudaGetErrorString(e));
  return 0;
}

int nfb_camera_project(const nfb_camera* cam, const float* points, long long n, float* pixels, void* stream) {
  if (!cam) return fail("null argument");
  if (n < 0) return fail("nfb_camera_project: negative point count %lld", n);
  int sms = 0;
  if (device_sms(&sms)) return -1;
  if (n == 0) return 0;
  if (!points || !pixels) return fail("null argument");
  nfb::camera_project_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(*cam, points, n, pixels);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("camera_project_kernel launch failed: %s", cudaGetErrorString(e));
  return 0;
}

int nfb_depth_resample(const nfb_camera* cam, const float* src, int src_h, int src_w, float factor, float* dst,
                       void* stream) {
  if (!cam) return fail("null argument");
  if (src_h < 1 || src_w < 1) return fail("nfb_depth_resample: source size %d x %d must be positive", src_h, src_w);
  if (cam->image_size[0] < 1 || cam->image_size[1] < 1) return fail("image_size must be positive");
  if (!(cam->focal_length != 0.f) || !(cam->pixel_aspect_ratio != 0.f))
    return fail("focal_length and pixel_aspect_ratio must be non-zero");
  if (!(factor > 0.f) || !std::isfinite(factor)) return fail("nfb_depth_resample: factor %g must be positive", factor);
  int sms = 0;
  if (device_sms(&sms)) return -1;
  if (!src || !dst) return fail("null argument");
  nfb::DepthResampleArgs a{};
  a.cam = *cam; a.has_distortion = nfb::camera_has_distortion(*cam);
  a.src = src; a.src_h = src_h; a.src_w = src_w;
  a.sx = (double)src_w / cam->image_size[0]; a.sy = (double)src_h / cam->image_size[1];
  a.factor = factor; a.dst = dst;
  const long long n = (long long)cam->image_size[0] * cam->image_size[1];
  nfb::depth_resample_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("depth_resample_kernel launch failed: %s", cudaGetErrorString(e));
  return 0;
}

// Workspace of nfb_near_far: the histograms, then the selection state, each 256-byte aligned.
static long long near_far_hist_bytes(int C) {
  using namespace nfb::capture;
  return ((long long)C * kRanks * kBins * sizeof(unsigned int) + 255) / 256 * 256;
}

long long nfb_near_far_workspace_size(int num_cameras) {
  if (num_cameras < 1 || num_cameras > 65535) return fail("nfb_near_far: num_cameras=%d outside [1, 65535]", num_cameras);
  return near_far_hist_bytes(num_cameras) + ((long long)num_cameras * sizeof(nfb::capture::NearFarState) + 255) / 256 * 256;
}

int nfb_near_far(const nfb_camera* cameras, int num_cameras, const double* points, long long num_points,
                 double q_near, double q_far, void* workspace, long long workspace_bytes, double* near,
                 double* far, long long* counts, void* stream) {
  using namespace nfb::capture;
  const long long need = nfb_near_far_workspace_size(num_cameras);
  if (need < 0) return -1;
  if (num_points < 0) return fail("nfb_near_far: negative point count %lld", num_points);
  if (!(q_near >= 0.0 && q_near <= 1.0 && q_far >= 0.0 && q_far <= 1.0))
    return fail("nfb_near_far: quantiles must lie in [0, 1]");
  if (!cameras || (num_points && !points) || !near || !far || !counts || !workspace) return fail("null argument");
  if (workspace_bytes < need)
    return fail("nfb_near_far: workspace of %lld bytes is smaller than the %lld bytes nfb_near_far_workspace_size returns",
                workspace_bytes, need);
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail("nfb_near_far: workspace must be 256-byte aligned");
  int sms = 0;
  if (device_sms(&sms)) return -1;
  cudaStream_t s = (cudaStream_t)stream;
  NearFarArgs a{};
  a.cameras = cameras; a.num_cameras = num_cameras; a.points = points; a.num_points = num_points;
  a.q[0] = q_near; a.q[1] = q_far;
  a.hist = static_cast<unsigned int*>(workspace);
  a.state = reinterpret_cast<NearFarState*>(static_cast<char*>(workspace) + near_far_hist_bytes(num_cameras));
  a.near = near; a.far = far; a.counts = counts;
  cudaError_t e = cudaMemsetAsync(a.hist, 0, near_far_hist_bytes(num_cameras), s);
  if (e != cudaSuccess) return fail("nfb_near_far: memset failed: %s", cudaGetErrorString(e));
  // Enough blocks per camera to fill the device twice over, each at least 256 points.
  const long long per_camera = std::max(1ll, std::min((num_points + 255) / 256, (2ll * 8 * sms + num_cameras - 1) / num_cameras));
  for (int pass = 0; pass < kPasses; ++pass) {
    near_far_hist_kernel<<<dim3((unsigned)per_camera, num_cameras), 256, 0, s>>>(a, pass);
    near_far_select_kernel<<<num_cameras, 32, 0, s>>>(a, pass);
  }
  e = cudaGetLastError();
  if (e != cudaSuccess) return fail("near/far launch failed: %s", cudaGetErrorString(e));
  return 0;
}

// Workspace of marching cubes: edge ids (3n + 1), triangle offsets (n + 1), the two int64 totals and
// CUB's scratch, each 256-byte aligned.
struct MeshPlan {
  long long n, ids_off, tris_off, totals_off, temp_off, temp_bytes, bytes;
};

static int mesh_plan(const char* fn, int nx, int ny, int nz, MeshPlan* p) {
  using nfb::mesh::kMaxSide;
  if (nx < 2 || ny < 2 || nz < 2 || nx > kMaxSide || ny > kMaxSide || nz > kMaxSide)
    return fail("%s: grid %d x %d x %d (nx, ny, nz): every side must lie in [2, %d]", fn, nx, ny, nz, kMaxSide);
  auto align = [](long long b) { return (b + 255) / 256 * 256; };
  p->n = (long long)nx * ny * nz;
  p->ids_off = 0;
  p->tris_off = align((3 * p->n + 1) * (long long)sizeof(unsigned));
  p->totals_off = p->tris_off + align((p->n + 1) * (long long)sizeof(unsigned));
  p->temp_off = p->totals_off + 256;
  size_t scan_edges = 0, scan_cubes = 0, reduce = 0;
  unsigned* u = nullptr;
  long long* ll = nullptr;
  if (cub::DeviceScan::ExclusiveSum(nullptr, scan_edges, u, u, 3 * p->n + 1) != cudaSuccess ||
      cub::DeviceScan::ExclusiveSum(nullptr, scan_cubes, u, u, p->n + 1) != cudaSuccess ||
      cub::DeviceReduce::Sum(nullptr, reduce, u, ll, p->n + 1) != cudaSuccess) {
    cudaGetLastError();
    return fail("%s: no CUDA device: nerfies_b200 has no CPU path", fn);
  }
  p->temp_bytes = align((long long)std::max(scan_edges, std::max(scan_cubes, reduce)));
  p->bytes = p->temp_off + p->temp_bytes;
  return 0;
}

static nfb::mesh::MeshArgs mesh_args(const float* grid, int nx, int ny, int nz, float level, void* workspace,
                                     const MeshPlan& p) {
  nfb::mesh::MeshArgs a{};
  char* ws = static_cast<char*>(workspace);
  a.grid = grid; a.nx = nx; a.ny = ny; a.nz = nz; a.n = p.n; a.level = level;
  a.edge_ids = reinterpret_cast<unsigned*>(ws + p.ids_off);
  a.tri_offsets = reinterpret_cast<unsigned*>(ws + p.tris_off);
  a.totals = reinterpret_cast<long long*>(ws + p.totals_off);
  return a;
}

static int mesh_check(const char* fn, const float* grid, void* workspace, long long workspace_bytes,
                      const MeshPlan& p) {
  if (!grid || !workspace) return fail("%s: null argument", fn);
  if (workspace_bytes < p.bytes)
    return fail("%s: workspace of %lld bytes is smaller than the %lld bytes nfb_marching_cubes_workspace_size returns",
                fn, workspace_bytes, p.bytes);
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail("%s: workspace must be 256-byte aligned", fn);
  if (reinterpret_cast<uintptr_t>(grid) & 3) return fail("%s: grid must be 4-byte aligned", fn);
  return 0;
}

long long nfb_marching_cubes_workspace_size(int nx, int ny, int nz) {
  MeshPlan p;
  return mesh_plan("nfb_marching_cubes_workspace_size", nx, ny, nz, &p) ? -1 : p.bytes;
}

int nfb_marching_cubes_count(const float* grid, int nx, int ny, int nz, float level, void* workspace,
                             long long workspace_bytes, long long* counts_out, void* stream) {
  using namespace nfb::mesh;
  const char* fn = "nfb_marching_cubes_count";
  MeshPlan p;
  if (mesh_plan(fn, nx, ny, nz, &p) || mesh_check(fn, grid, workspace, workspace_bytes, p)) return -1;
  if (!counts_out) return fail("%s: null argument", fn);
  cudaStream_t s = (cudaStream_t)stream;
  MeshArgs a = mesh_args(grid, nx, ny, nz, level, workspace, p);
  void* temp = static_cast<char*>(workspace) + p.temp_off;
  size_t temp_bytes = (size_t)p.temp_bytes;
  classify_kernel<<<(unsigned)((p.n + kThreads - 1) / kThreads), kThreads, 0, s>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cub::DeviceReduce::Sum(temp, temp_bytes, a.tri_offsets, a.totals + 1, p.n + 1, s);
  if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(temp, temp_bytes, a.edge_ids, a.edge_ids, 3 * p.n + 1, s);
  if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(temp, temp_bytes, a.tri_offsets, a.tri_offsets, p.n + 1, s);
  if (e == cudaSuccess) {
    finish_counts_kernel<<<1, 1, 0, s>>>(a, counts_out);
    e = cudaGetLastError();
  }
  if (e != cudaSuccess) return fail("%s: launch failed: %s", fn, cudaGetErrorString(e));
  return 0;
}

int nfb_marching_cubes(const float* grid, int nx, int ny, int nz, float level, const float* origin,
                       const float* spacing, void* workspace, long long workspace_bytes, float* vertices,
                       float* normals, int* faces, void* stream) {
  using namespace nfb::mesh;
  const char* fn = "nfb_marching_cubes";
  MeshPlan p;
  if (mesh_plan(fn, nx, ny, nz, &p) || mesh_check(fn, grid, workspace, workspace_bytes, p)) return -1;
  if (!origin || !spacing) return fail("%s: null argument", fn);
  cudaStream_t s = (cudaStream_t)stream;
  MeshArgs a = mesh_args(grid, nx, ny, nz, level, workspace, p);
  long long totals[2] = {0, 0};
  NFB_CUDA(cudaMemcpyAsync(totals, a.totals, sizeof(totals), cudaMemcpyDeviceToHost, s));
  NFB_CUDA(cudaStreamSynchronize(s));
  if (totals[0] > INT32_MAX || totals[1] > INT32_MAX)
    return fail("%s: %lld vertices and %lld faces: int32 indices hold at most %d", fn, totals[0], totals[1],
                INT32_MAX);
  if ((totals[0] && !vertices) || (totals[1] && !faces)) return fail("%s: null argument", fn);
  for (int d = 0; d < 3; ++d) { a.origin[d] = origin[d]; a.spacing[d] = spacing[d]; }
  a.vertices = vertices; a.normals = normals; a.faces = faces;
  if (totals[0]) vertex_kernel<<<(unsigned)((3 * p.n + kThreads - 1) / kThreads), kThreads, 0, s>>>(a);
  if (totals[1]) face_kernel<<<(unsigned)((p.n + kThreads - 1) / kThreads), kThreads, 0, s>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("%s: launch failed: %s", fn, cudaGetErrorString(e));
  return 0;
}

int nfb_marching_cubes_table(int* out) {
  using namespace nfb::mesh;
  if (out) {
    const int row = 1 + 3 * kMaxTriangles;
    for (int cs = 0; cs < 256; ++cs) {
      const int n = kCaseTable.count[cs];
      out[cs * row] = n;
      for (int i = 0; i < 3 * kMaxTriangles; ++i) out[cs * row + 1 + i] = i < 3 * n ? kCaseTable.edge[cs][i] : -1;
    }
  }
  return kMaxTriangles;
}

int nfb_colorize(const float* a, const float* b, int height, int width, int source, const double* table,
                 float cmin, float cmax, float d, int flags, void* workspace, double* out_f64,
                 unsigned char* out_u8, long long pitch, void* stream) {
  using namespace nfb::viz;
  if (source < NFB_VIZ_VALUE || source > NFB_VIZ_RGB) return fail("nfb_colorize: unknown source %d", source);
  if (height < 0 || width < 0) return fail("nfb_colorize: negative shape %d x %d", height, width);
  if (flags & ~(kInvert | kFrameMin | kFrameMax)) return fail("nfb_colorize: unknown flags 0x%x", flags);
  if ((long long)height * width == 0) return 0;
  if ((out_f64 == nullptr) == (out_u8 == nullptr)) return fail("nfb_colorize: pass exactly one of out_f64 and out_u8");
  if (source == NFB_VIZ_RGB && out_f64) return fail("nfb_colorize: the rgb source writes uint8 only");
  if (out_u8 && pitch < 3ll * width) return fail("nfb_colorize: pitch %lld is below 3 * width = %lld", pitch, 3ll * width);
  if ((long long)height * (3 * width / 16 + 2) >= (1ll << 31)) return fail("nfb_colorize: frame too large");
  const bool frame = flags & (kFrameMin | kFrameMax);
  if (source != NFB_VIZ_RGB && !(d > 0.0f)) return fail("nfb_colorize: d must be positive (it is a divisor or eps)");
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    return fail("no CUDA device: nerfies_b200 has no CPU path");
  const bool two = source == NFB_VIZ_ABS_ERROR || source == NFB_VIZ_SQ_ERROR;
  if (!a || (two && !b) || (source != NFB_VIZ_RGB && !table) || (frame && !workspace)) return fail("null argument");
  if (((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(workspace)) & 3) ||
      (reinterpret_cast<uintptr_t>(table) | reinterpret_cast<uintptr_t>(out_f64)) & 7)
    return fail("nfb_colorize: misaligned pointer");
  float* partials = static_cast<float*>(workspace);
  cudaStream_t s = (cudaStream_t)stream;
  switch (source) {
    case NFB_VIZ_VALUE: nfb::viz::launch<kValue>(a, b, height, width, table, cmin, cmax, d, flags, partials, out_f64, out_u8, pitch, sms, s); break;
    case NFB_VIZ_RECIPROCAL: nfb::viz::launch<kReciprocal>(a, b, height, width, table, cmin, cmax, d, flags, partials, out_f64, out_u8, pitch, sms, s); break;
    case NFB_VIZ_ABS_ERROR: nfb::viz::launch<kAbsError>(a, b, height, width, table, cmin, cmax, d, flags, partials, out_f64, out_u8, pitch, sms, s); break;
    case NFB_VIZ_SQ_ERROR: nfb::viz::launch<kSqError>(a, b, height, width, table, cmin, cmax, d, flags, partials, out_f64, out_u8, pitch, sms, s); break;
    default: nfb::viz::launch<kRgb>(a, b, height, width, table, cmin, cmax, d, flags & kInvert, partials, out_f64, out_u8, pitch, sms, s); break;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("colorize launch failed: %s", cudaGetErrorString(e));
  return 0;
}

int nfb_flow_colorize(const float* flow, const int* status, int height, int width, float max_flow, void* workspace,
                      unsigned char* out, long long pitch, void* stream) {
  using namespace nfb::viz;
  if (height < 0 || width < 0) return fail("nfb_flow_colorize: negative shape %d x %d", height, width);
  if ((long long)height * width == 0) return 0;
  if (!flow || !out) return fail("null argument");
  if (pitch < 3ll * width) return fail("nfb_flow_colorize: pitch %lld is below 3 * width = %lld", pitch, 3ll * width);
  const bool frame = !(max_flow > 0.f);
  if (frame && !workspace) return fail("nfb_flow_colorize: max_flow <= 0 takes the scale from the frame: null workspace");
  if ((reinterpret_cast<uintptr_t>(flow) | reinterpret_cast<uintptr_t>(workspace)) & 7 ||
      reinterpret_cast<uintptr_t>(status) & 3)
    return fail("nfb_flow_colorize: misaligned pointer");
  int sms = 0;
  if (device_sms(&sms)) return -1;
  cudaStream_t s = (cudaStream_t)stream;
  const long long n = (long long)height * width;
  const float2* f2 = reinterpret_cast<const float2*>(flow);
  double* partials = static_cast<double*>(workspace);
  if (frame) flow_max_kernel<<<kFlowMaxBlocks, kFlowThreads, 0, s>>>(f2, status, n, partials);
  const long long blocks = std::min<long long>((n + kFlowThreads - 1) / kFlowThreads, 4ll * sms);
  flow_colorize_kernel<<<(unsigned)blocks, kFlowThreads, 0, s>>>(f2, status, height, width, frame ? 0.0 : (double)max_flow,
                                                                 partials, out, pitch);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("flow colorize launch failed: %s", cudaGetErrorString(e));
  return 0;
}

int nfb_debug_provoke_timeout(nfb_handle* h, int enabled) {
  if (!h) return fail("null handle");
  h->debug_bits = enabled ? (h->debug_bits | nfb::kDebugTimeout) : (h->debug_bits & ~nfb::kDebugTimeout);
  return 0;
}

int nfb_debug_one_row_block(nfb_handle* h, int enabled) {
  if (!h) return fail("null handle");
  h->debug_bits = enabled ? (h->debug_bits | nfb::kDebugOneRowBlock) : (h->debug_bits & ~nfb::kDebugOneRowBlock);
  return 0;
}

int nfb_set_time_alpha(nfb_handle* h, float time_alpha) {
  if (!h) return fail("null handle");
  h->time_alpha = time_alpha;
  return 0;
}

int nfb_set_profiling(nfb_handle* h, int enabled) {
  if (!h) return fail("null handle");
  if (enabled && !h->ev[0][0]) {
    for (int l = 0; l < 2; ++l)
      for (int i = 0; i < 2; ++i) NFB_CUDA(cudaEventCreate(&h->ev[l][i]));
  }
  h->profiling = enabled != 0;
  h->ev_valid[0] = h->ev_valid[1] = false;
  return 0;
}

float nfb_field_time_ms(nfb_handle* h, int level) {
  if (!h || level < 0 || level > 1 || !h->ev_valid[level]) {
    fail("no profiled field launch for level %d", level);
    return -1.f;
  }
  if (cudaEventSynchronize(h->ev[level][1]) != cudaSuccess) { fail("cudaEventSynchronize failed"); return -1.f; }
  float ms = -1.f;
  if (cudaEventElapsedTime(&ms, h->ev[level][0], h->ev[level][1]) != cudaSuccess) { fail("cudaEventElapsedTime failed"); return -1.f; }
  return ms;
}

int nfb_check_abort(void* stream, int synchronize) {
  if (synchronize) NFB_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  return abort_check();
}

int nfb_reset_abort(void) {
  // only meaningful once every stream that ran a tensor-core launch has drained
  NFB_CUDA(cudaDeviceSynchronize());
  if (g_abort_host) *reinterpret_cast<volatile int*>(g_abort_host) = 0;
  return 0;
}

static int selftest_gemm(bool x3, int K, int N, const float* A, const float* W, float* C, int reps, long long* out,
                         cudaStream_t s) {
  using namespace nfb::tc;
  if (K < 1 || K > kSelfMaxKb * kBlockK || N < 1 || N > 256) return fail("selftest: K<=320, N<=256");
  if (reps < 1) return fail("selftest: reps must be >= 1");
  if (ensure_abort_flag() || abort_check()) return -1;
  const int nkb = (K + kBlockK - 1) / kBlockK;
  const int n_rows = (N + 15) / 16 * 16;
  std::vector<int> k_map(nkb * kBlockK, -1);
  for (int k = 0; k < K; ++k) k_map[k] = k;
  int* d_map = nullptr;
  uint8_t* d_w = nullptr;
  long long* d_out = nullptr;
  float* d_max = nullptr;
  NFB_CUDA(cudaMalloc(&d_map, k_map.size() * sizeof(int)));
  NFB_CUDA(cudaMalloc(&d_w, (size_t)nkb * (x3 ? 2 : 1) * n_rows * kRowBytes));
  NFB_CUDA(cudaMalloc(&d_out, 2 * sizeof(long long)));
  NFB_CUDA(cudaMalloc(&d_max, sizeof(float)));
  NFB_CUDA(cudaMemsetAsync(d_out, 0, 2 * sizeof(long long), s));
  NFB_CUDA(cudaMemsetAsync(d_max, 0, sizeof(float), s));
  NFB_CUDA(cudaMemcpyAsync(d_map, k_map.data(), k_map.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  const long long total = (long long)nkb * n_rows * kBlockK;
  float scale = 1.f;
  if (x3) {
    absmax_kernel<<<32, 256, 0, s>>>(W, (long long)K * N, d_max);
    pack_weight_x3_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(W, N, d_map, nkb, N, n_rows, d_max, d_w);
    float h_max = 0.f;
    NFB_CUDA(cudaMemcpyAsync(&h_max, d_max, sizeof(float), cudaMemcpyDeviceToHost, s));
    NFB_CUDA(cudaStreamSynchronize(s));
    scale = 1.f / x3_weight_scale(h_max) / (float)reps;
    NFB_CUDA(cudaFuncSetAttribute(tc_selftest_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSelfSmemBytes));
    tc_selftest_kernel<true><<<1, 128, kSelfSmemBytes, s>>>(A, K, d_w, nkb, n_rows, N, scale, reps, C, d_out);
  } else {
    pack_weight_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(W, N, d_map, nkb, N, n_rows,
                                                                      reinterpret_cast<__nv_bfloat16*>(d_w));
    NFB_CUDA(cudaFuncSetAttribute(tc_selftest_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSelfSmemBytes));
    tc_selftest_kernel<false><<<1, 128, kSelfSmemBytes, s>>>(A, K, d_w, nkb, n_rows, N, scale, reps, C, d_out);
  }
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  long long h_out[2] = {0, 0};
  if (e == cudaSuccess) e = cudaMemcpy(h_out, d_out, sizeof(h_out), cudaMemcpyDeviceToHost);
  cudaFree(d_map); cudaFree(d_w); cudaFree(d_out); cudaFree(d_max);
  if (e != cudaSuccess) return fail("selftest kernel failed: %s", cudaGetErrorString(e));
  if (out) { out[0] = h_out[0]; out[1] = h_out[1]; }
  return abort_check();
}

int nfb_selftest_gemm(int K, int N, const float* A, const float* W, float* C, void* stream) {
  return selftest_gemm(false, K, N, A, W, C, 1, nullptr, (cudaStream_t)stream);
}

int nfb_selftest_gemm3(int K, int N, const float* A, const float* W, float* C, int reps, long long* out,
                       void* stream) {
  return selftest_gemm(true, K, N, A, W, C, reps, out, (cudaStream_t)stream);
}

int nfb_create(const nfb_config* cfg, int max_rays, nfb_handle** out) {
  if (!cfg || !out) return fail("null argument");
  if (max_rays < 1) return fail("max_rays must be >= 1");
  if (cfg->num_coarse_samples < 2) return fail("num_coarse_samples must be >= 2");
  if (cfg->num_fine_samples < 0) return fail("num_fine_samples must be >= 0");
  // The fine level has Nc + Nf samples per ray: composite_kernel (and its adjoint) hold a ray's samples in
  // shared memory, up to kMaxSamples.  Within that bound resample_kernel's shared memory always fits its
  // 64 KiB opt-in (static_assert in run_resample).
  if (cfg->num_coarse_samples + cfg->num_fine_samples > nfb::kMaxSamples)
    return fail("num_coarse_samples + num_fine_samples = %d: more than %d samples per ray (kMaxSamples)",
                cfg->num_coarse_samples + cfg->num_fine_samples, nfb::kMaxSamples);
  if (cfg->num_fine_samples > 0 && cfg->num_coarse_samples < 3)
    return fail("hierarchical sampling needs >= 3 coarse samples (num_fine_samples > 0)");
  if (cfg->precision < NFB_PREC_FP32 || cfg->precision > NFB_PREC_FP16X3) return fail("bad precision");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail("no CUDA device: nerfies_b200 has no CPU path");
  nfb_handle* h = new nfb_handle();
  h->cfg = *cfg;
  h->max_rays = max_rays;
  auto bail = [&](int) { nfb_destroy(h); return -1; };
  if (cudaGetDevice(&h->device) != cudaSuccess) return bail(fail("cudaGetDevice failed"));
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, h->device) != cudaSuccess) return bail(fail("cudaGetDeviceProperties failed"));
  if (prop.major != 9) return bail(fail("device is sm_%d%d; this library is built for sm_90a only", prop.major, prop.minor));
  h->sm_count = prop.multiProcessorCount;
  if (ensure_abort_flag()) return bail(-1);
  if (build_programs(h)) return bail(-1);
  if (build_tables(h)) return bail(-1);
  const nfb_config& c = h->cfg;
  const int nc = c.num_coarse_samples, nfine = nc + c.num_fine_samples;
  auto dmalloc = [&](float** p, long long n) {
    return cudaMalloc(p, (size_t)std::max<long long>(n, 1) * sizeof(float)) == cudaSuccess ? 0
        : fail("cudaMalloc of %lld floats failed", n);
  };
  const long long B = max_rays;
  if (dmalloc(&h->d_packed, h->packed_floats) ||
      dmalloc(&h->d_warp_table, (long long)c.num_warp_embeddings * c.num_warp_features) ||
      dmalloc(&h->d_app_table, (long long)c.num_appearance_embeddings * c.num_appearance_features) ||
      dmalloc(&h->d_cam_table, (long long)c.num_camera_embeddings * c.num_camera_features) ||
      dmalloc(&h->d_cond, B * h->cond_layout.stride) || dmalloc(&h->d_zc, B * nc) ||
      dmalloc(&h->d_zf, B * nfine) || dmalloc(&h->d_wc, B * nc) ||
      dmalloc(&h->d_samples, B * nfine * 4) || dmalloc(&h->d_out_c, B * 6) ||
      dmalloc(&h->d_out_f, B * 6) || dmalloc(&h->d_in, B * 9))
    return bail(-1);
  if (cudaMalloc(&h->d_ids, (size_t)B * 3 * sizeof(unsigned)) != cudaSuccess) return bail(fail("cudaMalloc ids failed"));
  if (c.warp_field_type != NFB_WARP_NONE && dmalloc(&h->d_warped_c, B * nc * 3)) return bail(-1);   // warp pass
  if (c.warp_field_type != NFB_WARP_NONE && c.num_fine_samples > 0) {   // render_fine_reusing_warp
    const int nf = c.num_fine_samples;
    if (dmalloc(&h->d_warped_new, B * nf * 3) || dmalloc(&h->d_warped_fine, B * nfine * 3) ||
        dmalloc(&h->d_znew, B * nf))
      return bail(-1);
    if (cudaMalloc(&h->d_src, (size_t)B * nfine * sizeof(uint16_t)) != cudaSuccess)
      return bail(fail("cudaMalloc of %lld sample indices failed", B * nfine));
  }
  if (cudaMemset(h->d_packed, 0, (size_t)h->packed_floats * sizeof(float)) != cudaSuccess) return bail(fail("cudaMemset failed"));
  if (cudaFuncSetAttribute(nfb::field_simt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           nfb::kSimtSmemBytes) != cudaSuccess)
    return bail(fail("cannot reserve %d bytes of shared memory", nfb::kSimtSmemBytes));
  if (cudaFuncSetAttribute(nfb::composite_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           kRaySmemOptIn) != cudaSuccess ||
      cudaFuncSetAttribute(nfb::resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           kRaySmemOptIn) != cudaSuccess)
    return bail(fail("cannot reserve %d bytes of shared memory for the per-ray kernels", kRaySmemOptIn));
  if (c.precision != NFB_PREC_FP32 && nfb::tc::create_tc(h)) return bail(-1);
  *out = h;
  return 0;
}

void nfb_destroy(nfb_handle* h) {
  if (!h) return;
  nfb::tc::destroy_tc(h);
  float* bufs[] = {h->d_packed, h->d_warp_table, h->d_app_table, h->d_cam_table, h->d_zlin,
                   h->d_lower, h->d_upper, h->d_ulin, h->d_window, h->d_cond, h->d_zc, h->d_zf,
                   h->d_wc, h->d_samples, h->d_out_c, h->d_out_f, h->d_in, h->d_warped_c,
                   h->d_warped_new, h->d_warped_fine, h->d_znew};
  for (float* p : bufs) if (p) cudaFree(p);
  if (h->d_src) cudaFree(h->d_src);
  float* tbufs[] = {h->d_tape, h->d_gpacked, h->d_gwarp, h->d_gapp, h->d_gcam, h->d_dcond, h->d_tr_out, h->d_tr_w, h->d_loss,
                    h->d_ttape, reinterpret_cast<float*>(h->d_sel), h->d_time_tape, h->d_ray_pts, h->d_ntape};
  for (float* p : tbufs) if (p) cudaFree(p);
  if (h->d_ids) cudaFree(h->d_ids);
  if (h->d_invert) cudaFree(h->d_invert);
  if (h->d_track) cudaFree(h->d_track);
  for (int l = 0; l < 2; ++l)
    for (int i = 0; i < 2; ++i) if (h->ev[l][i]) cudaEventDestroy(h->ev[l][i]);
  if (h->h_in) cudaFreeHost(h->h_in);
  if (h->h_out) cudaFreeHost(h->h_out);
  if (h->h_ids) cudaFreeHost(h->h_ids);
  if (h->ev_order) cudaEventDestroy(h->ev_order);
  delete h;
}

int nfb_param_count(const nfb_handle* h) { return h ? (int)h->specs.size() : fail("null handle"); }

int nfb_param_info(const nfb_handle* h, int index, char* name, int name_capacity,
                   long long* rows, long long* cols) {
  if (!h) return fail("null handle");
  if (index < 0 || index >= (int)h->specs.size()) return fail("parameter index %d out of range", index);
  const ParamSpec& s = h->specs[index];
  if (name && name_capacity > 0) {
    strncpy(name, s.name.c_str(), name_capacity - 1);
    name[name_capacity - 1] = 0;
  }
  if (rows) *rows = s.rows;
  if (cols) *cols = s.cols;
  return 0;
}

int nfb_set_params(nfb_handle* h, const float* const* tensors, const long long* numels,
                   int count, void* stream) {
  if (!h || !tensors || !numels) return fail("null argument");
  if (count != (int)h->specs.size())
    return fail("expected %d parameter tensors, got %d", (int)h->specs.size(), count);
  cudaStream_t s = (cudaStream_t)stream;
  if (enter_stream(h, s)) return -1;
  for (int i = 0; i < count; ++i) {
    const ParamSpec& p = h->specs[i];
    if (numels[i] != p.rows * p.cols)
      return fail("parameter %d (%s): expected %lld x %lld = %lld elements, got %lld", i,
                  p.name.c_str(), p.rows, p.cols, p.rows * p.cols, numels[i]);
    if (!tensors[i]) return fail("parameter %d (%s) is null", i, p.name.c_str());
    float* base = p.table == 0 ? h->d_packed : p.table == 1 ? h->d_warp_table
                  : p.table == 2 ? h->d_app_table : h->d_cam_table;
    const long long n = p.rows * p.cols;
    if (n == 0) continue;
    pack_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(tensors[i], base + p.dst_off, p.rows,
                                                            p.cols, p.ld, p.c_off);
    if (launch_check(h, "pack_kernel")) return -1;
  }
  if (h->cfg.precision != NFB_PREC_FP32 && nfb::tc::pack_tc(h, s)) return -1;
  h->params_set = true;
  return 0;
}

int nfb_coarse_z_vals(nfb_handle* h, int B, const float* t_rand, float* z, void* stream) {
  if (check_call(h, B)) return -1;
  if (B == 0) return 0;
  if (enter_stream(h, (cudaStream_t)stream)) return -1;
  const int nc = h->cfg.num_coarse_samples;
  const long long total = (long long)B * nc;
  nfb::coarse_z_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      h->d_zlin, h->d_lower, h->d_upper, t_rand, z, B, nc);
  return launch_check(h, "coarse_z_kernel");
}

int nfb_sample_pdf(nfb_handle* h, int B, const float* z_coarse, const float* w_coarse,
                   const float* u_rand, float* z_fine, void* stream) {
  if (check_call(h, B)) return -1;
  if (h->cfg.num_fine_samples <= 0) return fail("model has no fine level");
  if (B == 0) return 0;
  if (enter_stream(h, (cudaStream_t)stream)) return -1;
  return run_resample(h, B, z_coarse, w_coarse, u_rand, z_fine, (cudaStream_t)stream);
}

int nfb_render_samples(nfb_handle* h, int level, int B, int S, const float* z_vals,
                       const float* origins, const float* directions, const float* viewdirs,
                       const unsigned* warp_id, const unsigned* app_id, const unsigned* cam_id,
                       float warp_alpha, unsigned flags, float* out, float* weights,
                       float* samples, float* warped_points, void* stream) {
  if (check_call(h, B)) return -1;
  if (level < 0 || level > 1 || (level == 1 && h->cfg.num_fine_samples <= 0)) return fail("bad level %d", level);
  const int smax = h->cfg.num_coarse_samples + h->cfg.num_fine_samples;
  if (S < 1 || (!samples && S > smax)) return fail("num_samples=%d exceeds the workspace (%d)", S, smax);
  if (B == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  if (enter_stream(h, s)) return -1;
  if (set_window(h, warp_alpha, s)) return -1;
  if (run_cond(h, B, viewdirs ? viewdirs : directions, warp_id, app_id, cam_id, s,
               (flags & NFB_FLAG_METADATA_ENCODED) != 0)) return -1;
  float* smp = samples ? samples : h->d_samples;
  const bool use_warp = !(flags & NFB_FLAG_NO_WARP);
  const long long rows = (long long)B * S;
  if (!warps(h, use_warp)) {
    if (run_field(h, level, rows, S, origins, directions, z_vals, smp, warped_points, use_warp, false, s)) return -1;
  } else {
    // The warp pass writes into the caller's warped_points or into the workspace (d_warped_fine
    // holds max_rays x (Nc + Nf) points, d_warped_c max_rays x Nc); a caller-sized S beyond it gets a
    // stream-ordered allocation for this call.
    float* pts = warped_points;
    float* tmp = nullptr;
    if (!pts) {
      const long long cap = (long long)h->max_rays * (h->d_warped_fine ? smax : h->cfg.num_coarse_samples);
      if (rows <= cap) {
        pts = h->d_warped_fine ? h->d_warped_fine : h->d_warped_c;
      } else {
        NFB_CUDA(cudaMallocAsync(&tmp, (size_t)rows * 3 * sizeof(float), s));
        pts = tmp;
      }
    }
    int rc = prof_begin(h, level, s);
    if (rc == 0) rc = run_warp(h, level, B, S, origins, directions, z_vals, pts, s);
    if (rc == 0) rc = run_field(h, level, rows, S, origins, directions, z_vals, smp, nullptr, true, false, s,
                                nullptr, nullptr, pts);
    if (rc == 0) rc = prof_end(h, level, s);
    if (tmp) NFB_CUDA(cudaFreeAsync(tmp, s));
    if (rc) return -1;
  }
  if (out) return run_composite(h, B, S, smp, z_vals, directions, out, weights, s);
  return 0;
}

int nfb_render_forward(nfb_handle* h, int B, const float* origins, const float* directions,
                       const float* viewdirs, const unsigned* warp_id, const unsigned* app_id,
                       const unsigned* cam_id, float warp_alpha, const float* t_rand,
                       const float* u_rand, unsigned flags, float* out_coarse, float* out_fine,
                       float* w_coarse, float* w_fine, float* z_fine, void* stream) {
  if (check_call(h, B)) return -1;
  if (B == 0) return 0;
  const nfb_config& c = h->cfg;
  cudaStream_t s = (cudaStream_t)stream;
  if (enter_stream(h, s)) return -1;
  const int nc = c.num_coarse_samples, nfine = nc + c.num_fine_samples;
  const bool use_warp = !(flags & NFB_FLAG_NO_WARP);
  const bool fine = c.num_fine_samples > 0 && !(flags & NFB_FLAG_COARSE_ONLY);
  if (set_window(h, warp_alpha, s)) return -1;
  if (run_cond(h, B, viewdirs ? viewdirs : directions, warp_id, app_id, cam_id, s,
               (flags & NFB_FLAG_METADATA_ENCODED) != 0)) return -1;
  // With a warp field the fine level warps only its new samples (render_fine_reusing_warp).
  const bool warp = warps(h, use_warp);
  // coarse level (models.py:332-349)
  if (nfb_coarse_z_vals(h, B, t_rand, h->d_zc, stream)) return -1;
  float* wc = w_coarse ? w_coarse : h->d_wc;
  float* oc = out_coarse ? out_coarse : h->d_out_c;
  if (warp ? render_coarse_warped(h, B, origins, directions, oc, wc, s)
           : render_level(h, 0, B, nc, origins, directions, h->d_zc, use_warp, oc, wc, s))
    return -1;
  if (!fine) return 0;
  // hierarchical resampling + fine level (models.py:352-370)
  float* zf = z_fine ? z_fine : h->d_zf;
  float* of = out_fine ? out_fine : h->d_out_f;
  if (warp) {
    if (run_resample(h, B, h->d_zc, wc, u_rand, zf, s, h->d_znew, h->d_src)) return -1;
    return render_fine_reusing_warp(h, B, origins, directions, zf, of, w_fine, s);
  }
  if (run_resample(h, B, h->d_zc, wc, u_rand, zf, s)) return -1;
  return render_level(h, 1, B, nfine, origins, directions, zf, use_warp, of, w_fine, s);
}

int nfb_render_forward_host(nfb_handle* h, int B, const float* origins, const float* directions,
                            const float* viewdirs, const unsigned* warp_id,
                            const unsigned* app_id, const unsigned* cam_id, float warp_alpha,
                            unsigned flags, float* out_coarse, float* out_fine, void* stream) {
  if (check_call(h, B)) return -1;
  if (flags & NFB_FLAG_METADATA_ENCODED)
    return fail("NFB_FLAG_METADATA_ENCODED is only supported by the device entry points");
  if (B == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  if (enter_stream(h, s)) return -1;
  const size_t mr = h->max_rays;
  // (each buffer on its own: a failed allocation leaves the others usable for the retry)
  if (!h->h_in) NFB_CUDA(cudaMallocHost(&h->h_in, mr * 9 * sizeof(float)));
  if (!h->h_out) NFB_CUDA(cudaMallocHost(&h->h_out, mr * 12 * sizeof(float)));
  if (!h->h_ids) NFB_CUDA(cudaMallocHost(&h->h_ids, mr * 3 * sizeof(unsigned)));
  const size_t n3 = (size_t)B * 3;
  memcpy(h->h_in, origins, n3 * sizeof(float));
  memcpy(h->h_in + mr * 3, directions, n3 * sizeof(float));
  if (viewdirs) memcpy(h->h_in + mr * 6, viewdirs, n3 * sizeof(float));
  const unsigned* ids[3] = {warp_id, app_id, cam_id};
  for (int i = 0; i < 3; ++i)
    if (ids[i]) memcpy(h->h_ids + mr * i, ids[i], (size_t)B * sizeof(unsigned));
  NFB_CUDA(cudaMemcpyAsync(h->d_in, h->h_in, n3 * sizeof(float), cudaMemcpyHostToDevice, s));
  NFB_CUDA(cudaMemcpyAsync(h->d_in + mr * 3, h->h_in + mr * 3, n3 * sizeof(float), cudaMemcpyHostToDevice, s));
  if (viewdirs)
    NFB_CUDA(cudaMemcpyAsync(h->d_in + mr * 6, h->h_in + mr * 6, n3 * sizeof(float), cudaMemcpyHostToDevice, s));
  for (int i = 0; i < 3; ++i)
    if (ids[i])
      NFB_CUDA(cudaMemcpyAsync(h->d_ids + mr * i, h->h_ids + mr * i, (size_t)B * sizeof(unsigned),
                               cudaMemcpyHostToDevice, s));
  if (nfb_render_forward(h, B, h->d_in, h->d_in + mr * 3, viewdirs ? h->d_in + mr * 6 : nullptr,
                         warp_id ? h->d_ids : nullptr, app_id ? h->d_ids + mr : nullptr,
                         cam_id ? h->d_ids + 2 * mr : nullptr, warp_alpha, nullptr, nullptr, flags,
                         h->d_out_c, h->d_out_f, nullptr, nullptr, nullptr, stream))
    return -1;
  const bool fine = h->cfg.num_fine_samples > 0 && !(flags & NFB_FLAG_COARSE_ONLY);
  if (out_coarse)
    NFB_CUDA(cudaMemcpyAsync(h->h_out, h->d_out_c, (size_t)B * 6 * sizeof(float), cudaMemcpyDeviceToHost, s));
  if (out_fine && fine)
    NFB_CUDA(cudaMemcpyAsync(h->h_out + mr * 6, h->d_out_f, (size_t)B * 6 * sizeof(float), cudaMemcpyDeviceToHost, s));
  NFB_CUDA(cudaStreamSynchronize(s));
  if (abort_check()) return -1;
  if (out_coarse) memcpy(out_coarse, h->h_out, (size_t)B * 6 * sizeof(float));
  if (out_fine && fine) memcpy(out_fine, h->h_out + mr * 6, (size_t)B * 6 * sizeof(float));
  return 0;
}

int nfb_warp_forward(nfb_handle* h, int P, const float* points, const unsigned* warp_id,
                     float warp_alpha, unsigned flags, float* warped, void* stream) {
  if (check_call(h, P)) return -1;
  if (h->cfg.warp_field_type == NFB_WARP_NONE) return fail("model has no warp field");
  if (P == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  if (enter_stream(h, s)) return -1;
  if (set_window(h, warp_alpha, s)) return -1;
  // Only the GLO block of the condition vector is read in warp-only mode; the
  // view-direction block is computed from `points` and ignored.
  if (run_cond(h, P, points, warp_id, nullptr, nullptr, s, (flags & NFB_FLAG_METADATA_ENCODED) != 0)) return -1;
  // Free points: rows = points, z = 0 (x = p + 0 * p = p exactly for finite p).
  return run_warp(h, 0, P, 1, points, points, nullptr, warped, s);
}

int nfb_warp_code(nfb_handle* h, int n, const unsigned* warp_id, float* code_out, void* stream) {
  if (check_call(h, n)) return -1;
  if (h->cfg.warp_field_type == NFB_WARP_NONE) return fail("warp code: the model has no warp field");
  if (n == 0) return 0;
  if (!warp_id || !code_out) return fail("warp code: warp_id / code_out is null");
  cudaStream_t s = (cudaStream_t)stream;
  if (enter_stream(h, s)) return -1;
  return run_cond(h, n, nullptr, warp_id, nullptr, nullptr, s, false, true, code_out);
}

int nfb_point_visibility(nfb_handle* h, int P, const float* points, const unsigned* warp_id,
                         const unsigned* appearance_id, const unsigned* camera_id, float warp_alpha,
                         unsigned flags, const nfb_camera* cam, float depth_tol, const int* invert_status,
                         float* pixels_out, float* depth_out, int* status_out, void* stream) {
  if (!h || !points || !cam || !pixels_out || !depth_out || !status_out) return fail("null argument");
  if (P < 0) return fail("P must be >= 0");
  if (check_call(h, std::min(P, h->max_rays))) return -1;
  const nfb_config& c = h->cfg;
  if (flags & NFB_FLAG_METADATA_ENCODED)
    return fail("point visibility: encoded metadata is not supported (pass ids or timestamps per point)");
  if (flags & ~NFB_FLAG_NO_WARP) return fail("point visibility: unsupported flags 0x%x (only NFB_FLAG_NO_WARP)", flags);
  if (!std::isfinite(depth_tol) || depth_tol < 0.f)
    return fail("point visibility: depth_tol=%g must be finite and >= 0", (double)depth_tol);
  if (cam->image_size[0] < 1 || cam->image_size[1] < 1)
    return fail("point visibility: image_size %d x %d must be positive", cam->image_size[0], cam->image_size[1]);
  if (!std::isfinite(cam->position[0]) || !std::isfinite(cam->position[1]) || !std::isfinite(cam->position[2]))
    return fail("point visibility: the camera position must be finite");
  if (warps(h, !(flags & NFB_FLAG_NO_WARP)) && !warp_id) return fail("point visibility: the warp field needs warp_id");
  if ((c.use_appearance_metadata && !appearance_id) || (c.use_camera_metadata && !camera_id))
    return fail("point visibility: the model reads appearance_id / camera_id; they must not be null");
  cudaStream_t s = (cudaStream_t)stream;
  if (enter_stream(h, s)) return -1;
  if (P == 0) return 0;
  const long long R = h->max_rays;
  if (!h->d_track && cudaMalloc(&h->d_track, (size_t)R * 6 * sizeof(float)) != cudaSuccess) {
    h->d_track = nullptr;
    return fail("point visibility: cannot allocate its %lld-byte ray workspace", R * 6 * (long long)sizeof(float));
  }
  const bool fine = c.num_fine_samples > 0;
  nfb::track::VisibilityArgs a{};
  a.cam = *cam; a.origins = h->d_track; a.directions = h->d_track + R * 3;
  a.render_out = fine ? h->d_out_f : h->d_out_c;
  a.near = c.near_plane; a.far = c.far_plane; a.depth_tol = depth_tol;
  // fixed work per chunk and nothing read back: every ray is rendered, OUTSIDE or not
  for (int p0 = 0; p0 < P; p0 += h->max_rays) {
    const int n = std::min(h->max_rays, P - p0);
    a.points = points + (size_t)p0 * 3; a.invert_status = invert_status ? invert_status + p0 : nullptr;
    a.pixels_out = pixels_out + (size_t)p0 * 2; a.depth_out = depth_out + (size_t)p0 * 2;
    a.status_out = status_out + p0; a.n = n;
    const unsigned blocks = (unsigned)((n + 255) / 256);
    nfb::track::visibility_rays_kernel<<<blocks, 256, 0, s>>>(a);
    if (launch_check(h, "visibility_rays_kernel")) return -1;
    if (nfb_render_forward(h, n, a.origins, a.directions, nullptr, warp_id ? warp_id + p0 : nullptr,
                           appearance_id ? appearance_id + p0 : nullptr, camera_id ? camera_id + p0 : nullptr,
                           warp_alpha, nullptr, nullptr, flags, h->d_out_c, fine ? h->d_out_f : nullptr, nullptr,
                           nullptr, nullptr, stream))
      return -1;
    nfb::track::visibility_classify_kernel<<<blocks, 256, 0, s>>>(a);
    if (launch_check(h, "visibility_classify_kernel")) return -1;
  }
  return 0;
}

}  // extern "C"

#include "train_api.cuh"
