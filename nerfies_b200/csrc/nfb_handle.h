// Internal definition of nfb_handle and small host helpers shared by the
// translation unit's parts (nfb_api.cu, field_tc.cuh).
#pragma once
#include <cuda_runtime.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/nerfies_b200.h"
#include "common.cuh"
#include "ray_kernels.cuh"
#include "tc_program.cuh"

namespace {

thread_local std::string g_error;

int fail(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_error = buf;
  return -1;
}

#define NFB_CUDA(expr)                                                        \
  do {                                                                        \
    cudaError_t e_ = (expr);                                                  \
    if (e_ != cudaSuccess)                                                    \
      return fail("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_),     \
                  __FILE__, __LINE__);                                        \
  } while (0)

struct ParamSpec {
  std::string name;
  long long rows, cols;
  // destination in the packed buffer: element (r, c) -> dst_off + r * ld + c_off + c
  long long dst_off;
  int ld, c_off;
  int table;  // 0 = packed dense buffer; 1/2/3 = warp/appearance/camera table
};

__global__ void pack_kernel(const float* __restrict__ src, float* __restrict__ dst,
                            long long rows, long long cols, int ld, int c_off) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * cols) return;
  const long long r = idx / cols, c = idx - r * cols;
  dst[r * ld + c_off + c] = src[idx];
}

int pad32(int n) { return (n + 31) / 32 * 32; }

}  // namespace

struct nfb_handle {
  nfb_config cfg;
  int max_rays = 0;
  int device = 0;
  nfb::FieldProgram prog[2];          // per level (coarse, fine)
  std::vector<ParamSpec> specs;
  long long packed_floats = 0;
  float* d_packed = nullptr;          // dense weights/biases (both levels + warp)
  float* d_warp_table = nullptr;
  float* d_app_table = nullptr;
  float* d_cam_table = nullptr;
  bool params_set = false;
  // per-model tables
  float *d_zlin = nullptr, *d_lower = nullptr, *d_upper = nullptr, *d_ulin = nullptr;
  float* d_window = nullptr;
  float h_window_alpha = NAN;
  // workspace
  float *d_cond = nullptr, *d_zc = nullptr, *d_zf = nullptr, *d_wc = nullptr;
  float* d_samples = nullptr;
  float *d_out_c = nullptr, *d_out_f = nullptr;
  // fine level on reused warped points (render_fine_reusing_warp): models with a warp field and
  // a fine level only
  float *d_warped_c = nullptr, *d_warped_new = nullptr, *d_warped_fine = nullptr, *d_znew = nullptr;
  uint16_t* d_src = nullptr;
  // device + pinned staging for the *_host entry point
  float *d_in = nullptr, *h_in = nullptr, *h_out = nullptr;
  unsigned *d_ids = nullptr, *h_ids = nullptr;
  long long launches = 0;
  bool profiling = false;
  cudaEvent_t ev[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};
  bool ev_valid[2] = {false, false};
  nfb::CondLayout cond_layout{};      // per-ray condition vectors (d_cond, d_dcond)
  int sm_count = 132;
  nfb::Net time_net{};                // TimeEncoder MLP ('time' / 'blend' warp metadata encoders)
  float time_alpha = 0.f;             // warp_extra['time_alpha'] (nfb_set_time_alpha)
  cudaStream_t last_stream = nullptr;  // stream of the previous call (see enter_stream)
  bool last_stream_valid = false;
  cudaEvent_t ev_order = nullptr;
  // training tier (train_api.cuh): tape + gradient buffers, allocated on first use
  float* d_tape = nullptr; long long tape_floats = 0;
  float *d_gpacked = nullptr, *d_gwarp = nullptr, *d_gapp = nullptr, *d_gcam = nullptr;
  float *d_dcond = nullptr, *d_tr_out = nullptr, *d_tr_w = nullptr, *d_loss = nullptr;
  float* d_ttape = nullptr; long long ttape_floats = 0;     // tangent tape (train_reg.cuh)
  float* d_ntape = nullptr; long long ntape_floats = 0;     // NeRF tangent tape (nfb_density_grad)
  float* d_time_tape = nullptr; long long time_tape_floats = 0;  // TimeEncoder tape, max_rays rows (time_forward)
  int* d_sel = nullptr; long long sel_cap = 0;              // selected tape rows (median-depth samples)
  float* d_ray_pts = nullptr; long long ray_pts_cap = 0;    // nfb_render_ray_vjp's point gradient (rows,3)
  void* d_invert = nullptr;           // nfb_warp_invert's per-point state, max_rays rows (allocated on first use)
  float* d_track = nullptr;           // nfb_point_visibility's rays (origins, directions), max_rays rows (first use)
  int train_precision = NFB_TRAIN_FP32;                     // the training GEMMs' kernel (launch_gemm)
  int debug_bits = 0;                 // FieldArgs::debug bits set through the test hook (abort-path test)
  // tensor-core path (precision != fp32)
  nfb::tc::TcProgram tcprog[2];
  unsigned char* d_wpack = nullptr;   // weight units, shared-memory image (bf16, or fp16 hi | lo)
  float* d_aux = nullptr;             // fp32 biases + alpha head
  long long wpack_bytes = 0, aux_floats = 0;
  // fold: simt_w_off is in d_fold, not d_packed
  struct TcPackJob { int level, step, chunk; int simt_w_off, ld, n, n0, k_total; bool fold; std::vector<int> k_map; };
  std::vector<TcPackJob> tc_jobs;
  struct TcAuxJob { int src_off, count, stride, dst_off; bool fold; };   // fold: src_off is in d_fold
  std::vector<TcAuxJob> tc_aux_jobs;
  // The bottleneck folded into the rgb branch (and, with an alpha condition, the alpha head), per level:
  // fold_kernel writes W_b W_r[:W] and b_b W_r[:W] + b_r (and W_b w_a[:W], b_a + b_b w_a[:W]) into d_fold at
  // every nfb_set_params; ray_bias_kernel adds the per-ray condition terms into d_ray_bias before each
  // tensor-core NeRF pass.
  nfb::tc::TcFold tc_fold[2];
  float* d_fold = nullptr;
  float* d_ray_bias = nullptr;        // (max_rays, 128 n_chunks) rgb bias, then (max_rays) alpha constants
};

