// Host side of the training tier: tape layout, the forward / backward launch
// sequence of one level, nfb_train_value_and_grad and nfb_adam_step
// (see train.cuh; included by nfb_api.cu after its helpers).
#pragma once
#include "train.cuh"
#include "train_reg.cuh"
#include "train_tc.cuh"
#include "warp_invert.cuh"

namespace {

using nfb::Net;
using nfb::Step;

// Step s reads the output of step producer[s] (or nothing when k_x == 0).
void net_producers(const Net& net, int* producer) {
  int writer[4] = {-1, -1, -1, -1};
  for (int s = 0; s < net.n_steps; ++s) {
    producer[s] = net.steps[s].k_x > 0 ? writer[net.steps[s].src] : -1;
    writer[net.steps[s].dst] = s;
  }
}

struct TapeLayout {
  long long rows = 0;
  // float offsets into the arena
  long long pts = 0, warped = 0, in_w = 0, in_n = 0, samples = 0, dwarped = 0, d_in_w = 0, d_in_n = 0;
  long long out_w[nfb::kMaxSteps], out_n[nfb::kMaxSteps], d_out_w[nfb::kMaxSteps], d_out_n[nfb::kMaxSteps];
  long long grad_begin = 0, grad_end = 0, total = 0;
  int ld_w = 0, ld_n = 0;
};

TapeLayout tape_layout(const nfb::FieldProgram& p, long long rows) {
  TapeLayout t;
  t.rows = rows;
  long long off = 0;
  auto take = [&](long long n) { long long o = off; off += (n + 63) / 64 * 64; return o; };
  t.ld_w = pad32(p.Dw);
  t.ld_n = pad32(p.Dp + p.tc + p.ac + p.rc);
  t.pts = take(rows * 3); t.warped = take(rows * 3);
  t.in_w = take(rows * t.ld_w); t.in_n = take(rows * t.ld_n);
  t.samples = take(rows * 4);
  for (int s = 0; s < p.warp.n_steps; ++s) t.out_w[s] = take(rows * p.warp.steps[s].npad);
  for (int s = 0; s < p.nerf.n_steps; ++s) t.out_n[s] = take(rows * p.nerf.steps[s].npad);
  t.grad_begin = off;
  t.dwarped = take(rows * 3);
  t.d_in_w = take(rows * t.ld_w); t.d_in_n = take(rows * t.ld_n);
  for (int s = 0; s < p.warp.n_steps; ++s) t.d_out_w[s] = take(rows * p.warp.steps[s].npad);
  for (int s = 0; s < p.nerf.n_steps; ++s) t.d_out_n[s] = take(rows * p.nerf.steps[s].npad);
  t.grad_end = off;
  t.total = off;
  return t;
}

// Rows per split of a weight-gradient GEMM (reduction over the rows of the batch; the partial tiles are
// atomicAdd-ed).  The output is tiny (<= 3 x 2 tiles of 128 x 128), so the split count sets the parallelism:
// aim at ~4 CTAs per resident slot (2 per SM) whatever the layer's width; a fixed 2048 rows left a 128-wide
// layer of a 131,072-row chunk with 64 CTAs for 132 SMs, 8192 rows measured 3x slower.
inline long long dw_split(const nfb_handle* h, long long M, int N, long long K) {
  const long long tiles = ((M + nfb::train::kT2 - 1) / nfb::train::kT2) * ((N + nfb::train::kT2 - 1) / nfb::train::kT2);
  const long long want = std::max<long long>(1, (8LL * h->sm_count) / tiles);   // splits
  long long per = (K + want - 1) / want;
  per = (per + 7) / 8 * 8;
  return std::min<long long>(4096, std::max<long long>(256, per));
}
// The same for tf32x3_gemm_kernel, which holds one CTA per SM (two 64 KB stages of shared memory): ~4 CTAs
// per SM, slices of whole k-blocks (32 rows).
inline long long dw_split_tf32x3(const nfb_handle* h, long long M, int N, long long K) {
  const long long tiles = ((M + nfb::train::kT2 - 1) / nfb::train::kT2) * ((N + nfb::train::kT2 - 1) / nfb::train::kT2);
  const long long want = std::max<long long>(1, (4LL * h->sm_count) / tiles);
  long long per = (K + want - 1) / want;
  per = (per + nfb::train::kTcBK - 1) / nfb::train::kTcBK * nfb::train::kTcBK;
  return std::min<long long>(8192, std::max<long long>(256, per));
}
// Rows per slice of a weight-gradient reduction in the handle's training precision.
inline long long dw_split_for(const nfb_handle* h, long long M, int N, long long K) {
  return h->train_precision == NFB_TRAIN_TF32X3 ? dw_split_tf32x3(h, M, N, K) : dw_split(h, M, N, K);
}
// kAKFast / kBNFast: see sgemm128_kernel (which functor index is contiguous in memory).  The handle's training
// precision picks the kernel: sgemm128_kernel (fp32) or tf32x3_gemm_kernel (train_tc.cuh).
template <bool kAKFast = true, bool kBNFast = true, class FA, class FB, class FC>
int launch_gemm(nfb_handle* h, long long M, int N, long long K, FA fa, FB fb, FC fc, long long k_split,
                cudaStream_t s, const char* what) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  const long long per = k_split > 0 ? k_split : K;
  dim3 grid((unsigned)((M + nfb::train::kT2 - 1) / nfb::train::kT2),
            (unsigned)((N + nfb::train::kT2 - 1) / nfb::train::kT2), (unsigned)((K + per - 1) / per));
  if (h->train_precision == NFB_TRAIN_TF32X3) {
    auto kernel = nfb::train::tf32x3_gemm_kernel<kAKFast, kBNFast, FA, FB, FC>;
    NFB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, nfb::train::kTcSmem));
    kernel<<<grid, 256, nfb::train::kTcSmem, s>>>(nfb::train::GemmShape{M, N, K}, fa, fb, fc, per);
  } else {
    nfb::train::sgemm128_kernel<kAKFast, kBNFast><<<grid, 256, 0, s>>>(nfb::train::GemmShape{M, N, K}, fa, fb, fc, per);
  }
  return launch_check(h, what);
}

int net_forward(nfb_handle* h, const Net& net, const float* in, int ld_in, const long long* out_off,
                float* arena, long long rows, cudaStream_t s) {
  int producer[nfb::kMaxSteps];
  net_producers(net, producer);
  for (int i = 0; i < net.n_steps; ++i) {
    const Step& st = net.steps[i];
    const float* x = producer[i] >= 0 ? arena + out_off[producer[i]] : in;
    const int ldx = producer[i] >= 0 ? net.steps[producer[i]].npad : ld_in;
    nfb::train::ConcatA a{x, ldx, st.k_x, in + st.in_off, ld_in};
    nfb::train::WeightB b{h->d_packed + st.w_off, st.npad};
    nfb::train::StoreBiasAct c{arena + out_off[i], st.npad, h->d_packed + st.b_off, st.act};
    if (launch_gemm(h, rows, st.n, st.k_x + st.k_in, a, b, c, 0, s, "sgemm (forward)")) return -1;
  }
  return 0;
}

int net_backward(nfb_handle* h, const Net& net, const float* in, float* d_in, int ld_in,
                 const long long* out_off, const long long* d_out_off, float* arena, long long rows,
                 cudaStream_t s) {
  int producer[nfb::kMaxSteps];
  net_producers(net, producer);
  for (int i = net.n_steps - 1; i >= 0; --i) {
    const Step& st = net.steps[i];
    const int K = st.k_x + st.k_in;
    nfb::train::DZ dz{arena + d_out_off[i], arena + out_off[i], st.npad, st.act};
    const float* x = producer[i] >= 0 ? arena + out_off[producer[i]] : in;
    const int ldx = producer[i] >= 0 ? net.steps[producer[i]].npad : ld_in;
    nfb::train::ConcatA a{x, ldx, st.k_x, in + st.in_off, ld_in};
    // dW += [X | IN]^T dZ   (reduction over the rows, split)
    if (launch_gemm<false, true>(h, K, st.n, rows, nfb::train::ConcatAT{a}, nfb::train::DZB{dz},
                                 nfb::train::AtomicAdd{h->d_gpacked + st.w_off, st.npad}, dw_split_for(h, K, st.n, rows), s, "sgemm (dW)")) return -1;
    // db += colsum(dZ)
    {
      dim3 grid((unsigned)((st.n + 31) / 32), (unsigned)std::min<long long>((rows + 255) / 256, 128));
      nfb::train::colsum_kernel<<<grid, 256, 0, s>>>(dz, rows, st.n, h->d_gpacked + st.b_off);
      if (launch_check(h, "colsum_kernel")) return -1;
    }
    // dX, dIN += dZ W^T; without d_in (an input that is not differentiated) dX only
    if (!d_in && producer[i] < 0) continue;
    float* dx = producer[i] >= 0 ? arena + d_out_off[producer[i]] : d_in;
    nfb::train::AccumSplit acc{dx, ldx, st.k_x, d_in ? d_in + st.in_off : nullptr, ld_in};
    if (launch_gemm<true, false>(h, rows, d_in ? K : st.k_x, st.n, dz,
                                 nfb::train::WeightBT{h->d_packed + st.w_off, st.npad}, acc, 0, s, "sgemm (dX)"))
      return -1;
  }
  return 0;
}

// ---- tangent tape (train_reg.cuh): three rows per selected point ----
struct TTapeLayout {
  long long trows = 0;
  long long in_t = 0, d_in_t = 0, total = 0;
  long long out_t[nfb::kMaxSteps], d_out_t[nfb::kMaxSteps];
};
TTapeLayout ttape_layout(const nfb::FieldProgram& p, long long sel_rows) {
  TTapeLayout t;
  t.trows = sel_rows * 3;
  long long off = 0;
  auto take = [&](long long n) { long long o = off; off += (n + 63) / 64 * 64; return o; };
  const int ld_w = pad32(p.Dw);
  t.in_t = take(t.trows * ld_w); t.d_in_t = take(t.trows * ld_w);
  for (int s = 0; s < p.warp.n_steps; ++s) { t.out_t[s] = take(t.trows * p.warp.steps[s].npad); t.d_out_t[s] = take(t.trows * p.warp.steps[s].npad); }
  t.total = off;
  return t;
}
// Grows the device buffer *buf of *cap elements to at least n elements (the contents are not kept).
template <class T>
int grow(T** buf, long long* cap, long long n, const char* what) {
  if (*cap >= n) return 0;
  if (*buf) cudaFree(*buf);
  *buf = nullptr; *cap = 0;
  if (cudaMalloc(buf, (size_t)n * sizeof(T)) != cudaSuccess)
    return fail("training: cannot allocate a %.2f GB %s", n * sizeof(T) * 1e-9, what);
  *cap = n;
  return 0;
}

// Tangent rows through the warp MLP: T_out = act'(Y_primal) * ([T_x | T_in] W).
int tnet_forward(nfb_handle* h, const Net& net, const float* tin, int ld_in, const long long* out_t,
                 const long long* out_primal, const float* arena, float* tarena, const int* sel, long long trows,
                 cudaStream_t s) {
  int producer[nfb::kMaxSteps];
  net_producers(net, producer);
  for (int i = 0; i < net.n_steps; ++i) {
    const Step& st = net.steps[i];
    const float* x = producer[i] >= 0 ? tarena + out_t[producer[i]] : tin;
    const int ldx = producer[i] >= 0 ? net.steps[producer[i]].npad : ld_in;
    nfb::train::ConcatA a{x, ldx, st.k_x, tin + st.in_off, ld_in};
    nfb::train::WeightB b{h->d_packed + st.w_off, st.npad};
    nfb::train::StoreMasked c{tarena + out_t[i], st.npad, arena + out_primal[i], sel, st.act};
    if (launch_gemm(h, trows, st.n, st.k_x + st.k_in, a, b, c, 0, s, "sgemm (tangent forward)")) return -1;
  }
  return 0;
}
// ... and backwards: weight gradients only (no bias; the masks are piecewise constant).
int tnet_backward(nfb_handle* h, const Net& net, const float* tin, float* d_tin, int ld_in, const long long* out_t,
                  const long long* d_out_t, const long long* out_primal, const float* arena, float* tarena,
                  const int* sel, long long trows, cudaStream_t s) {
  int producer[nfb::kMaxSteps];
  net_producers(net, producer);
  for (int i = net.n_steps - 1; i >= 0; --i) {
    const Step& st = net.steps[i];
    const int K = st.k_x + st.k_in;
    nfb::train::DZT dz{tarena + d_out_t[i], arena + out_primal[i], sel, st.npad, st.act};
    const float* x = producer[i] >= 0 ? tarena + out_t[producer[i]] : tin;
    const int ldx = producer[i] >= 0 ? net.steps[producer[i]].npad : ld_in;
    nfb::train::ConcatA a{x, ldx, st.k_x, tin + st.in_off, ld_in};
    if (launch_gemm<false, true>(h, K, st.n, trows, nfb::train::ConcatAT{a}, nfb::train::DZTB{dz},
                                 nfb::train::AtomicAdd{h->d_gpacked + st.w_off, st.npad}, dw_split_for(h, K, st.n, trows), s, "sgemm (tangent dW)")) return -1;
    if (i == 0 && st.k_x == 0) break;             // nothing upstream of the encoded input carries a parameter
    float* dx = producer[i] >= 0 ? tarena + d_out_t[producer[i]] : d_tin;
    nfb::train::AccumSplit acc{dx, ldx, st.k_x, d_tin + st.in_off, ld_in};
    if (launch_gemm<true, false>(h, trows, K, st.n, dz, nfb::train::WeightBT{h->d_packed + st.w_off, st.npad}, acc, 0, s,
                                 "sgemm (tangent dX)")) return -1;
  }
  return 0;
}

// Regularisers of one training step (training.py:138-147, 176-212, 246-257).
struct RegCfg {
  bool elastic = false; int reduce = 0, type = 0; float elastic_weight = 0.f;
  bool warp_reg = false; float warp_reg_weight = 0.f, warp_reg_alpha = -2.f, warp_reg_scale = 0.001f;
  int batch_rays = 1;             // rays of the whole local batch (the means are over it)
  float* stats = nullptr;         // device: nfb_train_value_and_grad_reg's loss_out layout
};

// The warp Jacobian's restriction: the tangent rows take the activation masks of a piecewise-linear MLP.
int check_relu_warp(const nfb::FieldProgram& p, const char* what) {
  for (int i = 0; i < p.warp.n_steps - 1; ++i)
    if (p.warp.steps[i].act != nfb::kRelu && p.warp.steps[i].act != nfb::kNone)
      return fail("%s: the warp MLP must use relu (piecewise-linear) activations", what);
  return 0;
}

// Jacobian (+ elastic loss and its adjoint when `with_grad`) at `sel_rows` tape rows of the warp tape in `A`.
int warp_jacobian_on_tape(nfb_handle* h, const nfb::FieldProgram& p, const TapeLayout& t, float* A, const int* sel,
                          long long sel_rows, const float* row_w, const RegCfg* reg, bool with_grad, float* jac_out,
                          cudaStream_t s) {
  using namespace nfb::train;
  if (check_relu_warp(p, "warp Jacobian")) return -1;
  const TTapeLayout tt = ttape_layout(p, sel_rows);
  if (grow(&h->d_ttape, &h->ttape_floats, tt.total, "tangent tape")) return -1;
  float* T = h->d_ttape;
  if (with_grad) NFB_CUDA(cudaMemsetAsync(T + tt.d_in_t, 0, (size_t)(tt.total - tt.d_in_t) * sizeof(float), s));
  const unsigned tblocks = (unsigned)((tt.trows + 127) / 128);
  EncodeTangentArgs e{A + t.pts, sel, h->d_window, T + tt.in_t, p.Fw, t.ld_w, sel_rows};
  encode_tangent_kernel<<<tblocks, 128, 0, s>>>(e);
  if (launch_check(h, "encode_tangent_kernel")) return -1;
  if (tnet_forward(h, p.warp, T + tt.in_t, t.ld_w, tt.out_t, t.out_w, A, T, sel, tt.trows, s)) return -1;
  const int hs = p.warp.n_steps - 1;
  JacArgs j{};
  j.head = A + t.out_w[hs]; j.ld = p.warp.steps[hs].npad; j.thead = T + tt.out_t[hs]; j.pts = A + t.pts;
  j.sel = sel; j.row_w = row_w; j.jac_out = jac_out; j.R = sel_rows;
  j.warp_type = p.warp_type; j.pivot = p.warp_pivot; j.trans = p.warp_trans;
  j.with_loss = reg != nullptr; j.loss_type = reg ? reg->type : 0;
  j.stats = reg ? reg->stats + kSlotElasticLoss : nullptr;
  if (with_grad) {
    j.d_head = A + t.d_out_w[hs]; j.d_thead = T + tt.d_out_t[hs];
    j.grad_scale = reg->elastic_weight / (float)reg->batch_rays;
  }
  jac_elastic_kernel<<<(unsigned)((sel_rows + 63) / 64), 64, 0, s>>>(j);
  if (launch_check(h, "jac_elastic_kernel")) return -1;
  if (with_grad &&
      tnet_backward(h, p.warp, T + tt.in_t, T + tt.d_in_t, t.ld_w, tt.out_t, tt.d_out_t, t.out_w, A, T, sel,
                    tt.trows, s))
    return -1;
  return 0;
}

// warp_field.apply on the t.rows rows of the tape: the encoded points (tape.pts, tape.in_w), the warp MLP
// (tape.out_w) and the tail (tape.warped).  The points are o + z d of the rays' S samples, or, with
// `points` not null, the rows of `points`; `cond` holds one condition vector per ray (per point).
int warp_forward(nfb_handle* h, const nfb::FieldProgram& p, const TapeLayout& t, const float* origins,
                 const float* directions, const float* z, int S, const float* points, const float* cond,
                 cudaStream_t s) {
  using namespace nfb::train;
  float* A = h->d_tape;
  const unsigned blocks = (unsigned)((t.rows + 127) / 128);
  EncodeArgs e{};
  e.origins = origins; e.directions = directions; e.z = z; e.pts_in = points; e.cond = cond; e.window = h->d_window;
  e.pts_out = A + t.pts; e.in = A + t.in_w; e.F = p.Fw; e.ld = t.ld_w; e.S = S;
  e.cond_stride = h->cond_layout.stride; e.cond_off = 0; e.n_cond = p.G; e.rows = t.rows;
  encode_kernel<<<blocks, 128, 0, s>>>(e);
  if (launch_check(h, "encode_kernel")) return -1;
  if (net_forward(h, p.warp, A + t.in_w, t.ld_w, t.out_w, A, t.rows, s)) return -1;
  const int hs = p.warp.n_steps - 1;
  WarpTailArgs w{A + t.out_w[hs], p.warp.steps[hs].npad, A + t.pts, A + t.warped, p.warp_type, p.warp_pivot,
                 p.warp_trans, t.rows};
  warp_tail_kernel<<<blocks, 128, 0, s>>>(w);
  return launch_check(h, "warp_tail_kernel");
}

// Adjoint of warp_forward: tape.dwarped -> the warp MLP's parameter gradients and, += per ray of S rows,
// the warp GLO block of `dcond`.
int warp_backward(nfb_handle* h, const nfb::FieldProgram& p, const TapeLayout& t, int S, float* dcond,
                  cudaStream_t s) {
  using namespace nfb::train;
  float* A = h->d_tape;
  const unsigned blocks = (unsigned)((t.rows + 127) / 128);
  const int hs = p.warp.n_steps - 1;
  WarpTailBwdArgs w{A + t.out_w[hs], p.warp.steps[hs].npad, A + t.pts, A + t.dwarped, A + t.d_out_w[hs],
                    p.warp_type, p.warp_pivot, p.warp_trans, t.rows};
  warp_tail_bwd_kernel<<<blocks, 128, 0, s>>>(w);
  if (launch_check(h, "warp_tail_bwd_kernel")) return -1;
  if (net_backward(h, p.warp, A + t.in_w, A + t.d_in_w, t.ld_w, t.out_w, t.d_out_w, A, t.rows, s)) return -1;
  EncodeBwdArgs e{};
  e.pts = A + t.pts; e.window = h->d_window; e.din = A + t.d_in_w; e.F = p.Fw; e.ld = t.ld_w; e.S = S;
  e.cond_stride = h->cond_layout.stride; e.cond_off = 0; e.n_cond = p.G; e.dpts = nullptr; e.dcond = dcond;
  e.rows = t.rows;
  encode_bwd_kernel<<<blocks, 128, 0, s>>>(e);
  return launch_check(h, "encode_bwd_kernel");
}

// ---- TimeEncoder tape ('time' / 'blend' warp metadata encoders): max_rays rows, one per ray or free point ----
struct TimeTapeLayout {
  long long in = 0, grad_begin = 0, total = 0;
  long long out[nfb::kMaxSteps], d_out[nfb::kMaxSteps];
  int ld = 0;
};
TimeTapeLayout time_tape_layout(const Net& net, int F, long long rows) {
  TimeTapeLayout t;
  long long off = 0;
  auto take = [&](long long n) { long long o = off; off += (n + 63) / 64 * 64; return o; };
  t.ld = pad32(1 + 2 * F);
  t.in = take(rows * t.ld);
  for (int s = 0; s < net.n_steps; ++s) t.out[s] = take(rows * net.steps[s].npad);
  t.grad_begin = off;
  for (int s = 0; s < net.n_steps; ++s) t.d_out[s] = take(rows * net.steps[s].npad);
  t.total = off;
  return t;
}

bool has_time_encoder(const nfb_handle* h) {
  return h->cfg.warp_field_type != NFB_WARP_NONE && h->cfg.warp_metadata_encoder != NFB_WARP_ENC_GLO;
}

// The TimeEncoder's share of the warp block of the condition vectors of `n` rays / points: its Dense layers
// through net_forward on the time tape, so that time_backward differentiates the activations used here.  The
// timestamps are `time_f` or, when it is null, float(`time_id`) (the 'blend' encoder and the background loss).
// Writes (or blends into the GLO rows already there) cond[:, 0:G], as time_embed_kernel does when rendering.
int time_forward(nfb_handle* h, int n, const float* time_f, const unsigned* time_id, cudaStream_t s) {
  using namespace nfb::train;
  if (!has_time_encoder(h)) return 0;
  const nfb_config& c = h->cfg;
  const Net& net = h->time_net;
  const TimeTapeLayout t = time_tape_layout(net, c.time_encoder_num_freqs, n);
  float* T = h->d_time_tape;
  const bool blend = c.warp_metadata_encoder == NFB_WARP_ENC_BLEND;
  TimeEncodeArgs e{};
  e.time_f = time_f; e.time_id = time_id;
  e.din = 1 + 2 * c.time_encoder_num_freqs; e.ld = t.ld; e.n = n; e.in = T + t.in;
  easing_window(blend ? (float)c.time_encoder_num_freqs : h->time_alpha, c.time_encoder_num_freqs, e.window);
  time_encode_kernel<<<(unsigned)(((long long)n * e.din + 255) / 256), 256, 0, s>>>(e);
  if (launch_check(h, "time_encode_kernel")) return -1;
  if (net_forward(h, net, T + t.in, t.ld, t.out, T, n, s)) return -1;
  const int last = net.n_steps - 1;
  TimeCondArgs w{T + t.out[last], net.steps[last].npad, h->d_cond, h->cond_layout.stride, h->cond_layout.G, n,
                 blend, h->time_alpha};
  time_cond_kernel<<<(unsigned)(((long long)n * w.G + 255) / 256), 256, 0, s>>>(w);
  return launch_check(h, "time_cond_kernel");
}

// Adjoint of time_forward: the condition-vector gradient of the same `n` rows -> the TimeEncoder's parameter
// gradients (d_gpacked).  time_alpha is a constant of the step.
int time_backward(nfb_handle* h, int n, const float* dcond, cudaStream_t s) {
  using namespace nfb::train;
  if (!has_time_encoder(h)) return 0;
  const nfb_config& c = h->cfg;
  const Net& net = h->time_net;
  const TimeTapeLayout t = time_tape_layout(net, c.time_encoder_num_freqs, n);
  float* T = h->d_time_tape;
  NFB_CUDA(cudaMemsetAsync(T + t.grad_begin, 0, (size_t)(t.total - t.grad_begin) * sizeof(float), s));
  const int last = net.n_steps - 1, G = h->cond_layout.G;
  const float scale = c.warp_metadata_encoder == NFB_WARP_ENC_BLEND ? h->time_alpha : 1.f;
  time_cond_bwd_kernel<<<(unsigned)(((long long)n * G + 255) / 256), 256, 0, s>>>(
      dcond, h->cond_layout.stride, G, scale, T + t.d_out[last], net.steps[last].npad, n);
  if (launch_check(h, "time_cond_bwd_kernel")) return -1;
  return net_backward(h, net, T + t.in, nullptr, t.ld, t.out, t.d_out, T, n, s);
}

// The condition vectors of `n` rays / points for the training tier (run_cond + time_forward).  `warp_id`
// holds float timestamps when `float_time` ('time' encoder on rays or Jacobian points), uint32 ids otherwise.
int train_cond(nfb_handle* h, int n, const float* viewdirs, const unsigned* warp_id, bool float_time,
               const unsigned* app_id, const unsigned* cam_id, cudaStream_t s) {
  if (has_time_encoder(h) && !warp_id)
    return fail("training: the 'time' / 'blend' warp metadata encoders need per-ray metadata (warp_id is null)");
  if (run_cond(h, n, viewdirs, warp_id, app_id, cam_id, s, false, false)) return -1;
  return time_forward(h, n, float_time ? reinterpret_cast<const float*>(warp_id) : nullptr,
                      float_time ? nullptr : warp_id, s);
}

// The taped forward of one level for `R` rays (rows = R * S) at the given z: warp field, encoding, NeRF MLP,
// raw -> samples, volumetric rendering into out6 (and weights, nullable).  *alpha_step / *rgb_step: the
// steps whose outputs hold the raw density and rgb.
int level_forward(nfb_handle* h, int level, int R, int S, const float* z, const float* origins,
                  const float* directions, const float* cond, bool use_warp, float* out6, float* weights,
                  cudaStream_t s, int* alpha_step_out, int* rgb_step_out) {
  using namespace nfb::train;
  const nfb::FieldProgram& p = h->prog[level];
  const long long rows = (long long)R * S;
  const TapeLayout t = tape_layout(p, rows);
  float* A = h->d_tape;
  const bool warp = use_warp && p.warp_type != 0;
  const unsigned blocks = (unsigned)((rows + 127) / 128);
  if (warp && warp_forward(h, p, t, origins, directions, z, S, nullptr, cond, s)) return -1;
  {
    EncodeArgs e{};
    e.origins = origins; e.directions = directions; e.z = z; e.cond = cond; e.window = nullptr;
    e.pts_in = warp ? A + t.warped : nullptr; e.pts_out = warp ? nullptr : A + t.warped;
    e.in = A + t.in_n; e.F = p.Fp; e.ld = t.ld_n; e.S = S;
    e.cond_stride = h->cond_layout.stride; e.cond_off = p.G; e.n_cond = p.tc + p.ac + p.rc; e.rows = rows;
    encode_kernel<<<blocks, 128, 0, s>>>(e);
    if (launch_check(h, "encode_kernel")) return -1;
  }
  if (net_forward(h, p.nerf, A + t.in_n, t.ld_n, t.out_n, A, rows, s)) return -1;
  // which steps hold the raw alpha / rgb (the last writers of the two output slots)
  int alpha_step = -1, rgb_step = -1;
  for (int i = 0; i < p.nerf.n_steps; ++i) {
    if (p.nerf.steps[i].dst == p.alpha_slot) alpha_step = i;
    if (p.nerf.steps[i].dst == p.rgb_slot) rgb_step = i;
  }
  if (alpha_step < 0 || rgb_step < 0) return fail("training: no alpha / rgb head in the program");
  const int ld_a = p.nerf.steps[alpha_step].npad, ld_rgb = p.nerf.steps[rgb_step].npad;
  raw_to_samples_kernel<<<blocks, 128, 0, s>>>(A + t.out_n[rgb_step], ld_rgb, A + t.out_n[alpha_step], ld_a,
                                               p.sigma_act, reinterpret_cast<float4*>(A + t.samples), rows);
  if (launch_check(h, "raw_to_samples_kernel")) return -1;
  *alpha_step_out = alpha_step;
  *rgb_step_out = rgb_step;
  return run_composite(h, R, S, A + t.samples, z, directions, out6, weights, s);
}

// The backward of one level for `R` rays (rows = R * S) on the tape that level_forward filled at the same z:
// composite_vjp_kernel seeded by the cotangents d_out (R,6) and d_weights (R,S) of the level's outputs, the
// regularisers of `reg` (on the level's `weights`), the NeRF MLP and its encoding, then the warp field, whose
// warped points also receive d_warped (R,S,3).  d_out, d_weights, d_warped and reg are nullable; `dcond` is the R
// rays' condition-vector gradient accumulator.
static_assert(nfb::train::composite_vjp_smem(nfb::kMaxSamples) <= 48 * 1024,
              "composite_vjp_kernel's shared memory exceeds the default 48 KiB at kMaxSamples");
int level_backward(nfb_handle* h, int level, int R, int S, const float* z, const float* directions, float* dcond,
                   bool use_warp, int alpha_step, int rgb_step, const float* d_out, const float* d_weights,
                   const float* d_warped, const float* weights, const RegCfg* reg, cudaStream_t s) {
  using namespace nfb::train;
  const nfb::FieldProgram& p = h->prog[level];
  const long long rows = (long long)R * S;
  const TapeLayout t = tape_layout(p, rows);
  float* A = h->d_tape;
  const bool warp = use_warp && p.warp_type != 0;
  const unsigned blocks = (unsigned)((rows + 127) / 128);
  NFB_CUDA(cudaMemsetAsync(A + t.grad_begin, 0, (size_t)(t.grad_end - t.grad_begin) * sizeof(float), s));
  {
    CompositeVjpArgs c{};
    c.samples = reinterpret_cast<const float4*>(A + t.samples); c.z = z; c.directions = directions;
    c.d_out = d_out; c.d_weights = d_weights;
    c.rgb_raw = A + t.out_n[rgb_step]; c.ld_rgb = p.nerf.steps[rgb_step].npad;
    c.alpha_raw = A + t.out_n[alpha_step]; c.ld_a = p.nerf.steps[alpha_step].npad;
    c.d_rgb_raw = A + t.d_out_n[rgb_step]; c.d_alpha_raw = A + t.d_out_n[alpha_step];
    c.num_rays = R; c.S = S;
    c.white_bg = h->cfg.use_white_background; c.sample_at_infinity = h->cfg.use_sample_at_infinity;
    c.sigma_act = p.sigma_act;
    const int nblk = (R + nfb::kRaysPerBlock - 1) / nfb::kRaysPerBlock;
    composite_vjp_kernel<<<nblk, 32 * nfb::kRaysPerBlock, composite_vjp_smem(S), s>>>(c);
    if (launch_check(h, "composite_vjp_kernel")) return -1;
  }
  const bool want_sel = reg && warp && ((reg->elastic && level == 0 && reg->reduce == 0) || reg->warp_reg);
  if (want_sel) {
    if (grow(&h->d_sel, &h->sel_cap, R, "median-depth row index")) return -1;
    depth_index_kernel<<<(unsigned)((R + 7) / 8), 256, 0, s>>>(weights, R, S, h->d_sel);
    if (launch_check(h, "depth_index_kernel")) return -1;
  }
  if (reg && reg->elastic && level == 0 && warp) {
    // training.py:176-193 (the coarse level only: training.py:242-244)
    const bool median = reg->reduce == 0;
    if (warp_jacobian_on_tape(h, p, t, A, median ? h->d_sel : nullptr, median ? R : rows, median ? nullptr : weights,
                              reg, true, nullptr, s))
      return -1;
  }
  if (net_backward(h, p.nerf, A + t.in_n, A + t.d_in_n, t.ld_n, t.out_n, t.d_out_n, A, rows, s)) return -1;
  {
    EncodeBwdArgs e{};
    e.pts = A + t.warped; e.window = nullptr; e.din = A + t.d_in_n; e.F = p.Fp; e.ld = t.ld_n; e.S = S;
    e.cond_stride = h->cond_layout.stride; e.cond_off = p.G; e.n_cond = p.tc + p.ac + p.rc;
    e.dpts = warp ? A + t.dwarped : nullptr; e.dcond = dcond; e.rows = rows;
    encode_bwd_kernel<<<blocks, 128, 0, s>>>(e);
    if (launch_check(h, "encode_bwd_kernel")) return -1;
  }
  if (!warp) return 0;
  // encode_bwd_kernel has set tape.dwarped; the warp-reg loss and d_warped add to it
  if (reg && reg->warp_reg) {
    // training.py:194-207: robust loss of |points - warped_points|^2 at the median-depth sample
    WarpMagArgs wm{A + t.pts, A + t.warped, h->d_sel, A + t.dwarped,
                   reg->stats + (level == 0 ? kSlotWarpRegCoarse : kSlotWarpRegFine),
                   reg->warp_reg_alpha, reg->warp_reg_scale, reg->warp_reg_weight / (float)reg->batch_rays, R};
    warp_mag_loss_kernel<<<(unsigned)((R + 127) / 128), 128, 0, s>>>(wm);
    if (launch_check(h, "warp_mag_loss_kernel")) return -1;
  }
  if (d_warped) {
    add_into_kernel<<<(unsigned)((rows * 3 + 255) / 256), 256, 0, s>>>(A + t.dwarped, d_warped, rows * 3);
    if (launch_check(h, "add_into_kernel")) return -1;
  }
  return warp_backward(h, p, t, S, dcond, s);
}

// The gradient accumulators of the packed parameters and of the three embedding tables, zeroed.
int zero_grads(nfb_handle* h, cudaStream_t s) {
  const nfb_config& c = h->cfg;
  NFB_CUDA(cudaMemsetAsync(h->d_gpacked, 0, (size_t)h->packed_floats * sizeof(float), s));
  NFB_CUDA(cudaMemsetAsync(h->d_gwarp, 0, (size_t)std::max(1, c.num_warp_embeddings * c.num_warp_features) * sizeof(float), s));
  NFB_CUDA(cudaMemsetAsync(h->d_gapp, 0, (size_t)std::max(1, c.num_appearance_embeddings * c.num_appearance_features) * sizeof(float), s));
  NFB_CUDA(cudaMemsetAsync(h->d_gcam, 0, (size_t)std::max(1, c.num_camera_embeddings * c.num_camera_features) * sizeof(float), s));
  return 0;
}

// `count` gradient tensors of `numels` elements: the order and sizes of nfb_param_info.
int check_grads(const nfb_handle* h, float* const* grads, const long long* numels, int count) {
  if (!grads || !numels) return fail("null gradient list");
  if (count != (int)h->specs.size()) return fail("expected %d gradient tensors, got %d", (int)h->specs.size(), count);
  for (int i = 0; i < count; ++i)
    if (numels[i] != h->specs[i].rows * h->specs[i].cols)
      return fail("gradient %d (%s): expected %lld elements", i, h->specs[i].name.c_str(), h->specs[i].rows * h->specs[i].cols);
  return 0;
}

// packed layouts -> the caller's tensors (+=), in the order of nfb_param_info
int unpack_grads(nfb_handle* h, float* const* grads, int count, cudaStream_t s) {
  for (int i = 0; i < count; ++i) {
    const ParamSpec& p = h->specs[i];
    const float* base = p.table == 0 ? h->d_gpacked : p.table == 1 ? h->d_gwarp : p.table == 2 ? h->d_gapp : h->d_gcam;
    const long long n = p.rows * p.cols;
    if (n == 0) continue;
    if (!grads[i]) return fail("gradient %d (%s) is null", i, p.name.c_str());
    nfb::train::unpack_grad_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(base + p.dst_off, grads[i], p.rows, p.cols, p.ld, p.c_off);
    if (launch_check(h, "unpack_grad_kernel")) return -1;
  }
  return 0;
}

// The adjoint of run_cond(encoded = true) for `n` rays: dcond -> the dense code gradients (+=), or row 0 of a
// table for a code the call did not pass.
int cond_vjp_encoded(nfb_handle* h, int n, const float* dcond, bool has_warp, bool has_app, bool has_cam,
                     float* d_warp, float* d_app, float* d_cam, cudaStream_t s) {
  nfb::train::CondVjpEncodedArgs a{};
  a.dcond = dcond; a.num_rays = n;
  a.has_warp = has_warp; a.has_app = has_app; a.has_cam = has_cam;
  a.d_warp = d_warp; a.d_app = d_app; a.d_cam = d_cam;
  // a 'time' encoder has no table: ray_cond_kernel's row-0 fallback reads memory no parameter owns
  a.d_warp_table = has_time_encoder(h) && h->cfg.warp_metadata_encoder == NFB_WARP_ENC_TIME ? nullptr : h->d_gwarp;
  a.d_app_table = h->d_gapp; a.d_cam_table = h->d_gcam;
  a.layout = h->cond_layout;
  const long long total = (long long)n * a.layout.stride;
  nfb::train::cond_vjp_encoded_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(a);
  return launch_check(h, "cond_vjp_encoded_kernel");
}

int train_prepare(nfb_handle* h, int chunk_rays) {
  const nfb_config& c = h->cfg;
  const int smax = c.num_coarse_samples + c.num_fine_samples;
  long long need = 0;
  for (int lv = 0; lv < 2; ++lv) need = std::max(need, tape_layout(h->prog[lv], (long long)chunk_rays * smax).total);
  if (h->tape_floats < need) {
    if (grow(&h->d_tape, &h->tape_floats, need, "tape")) return -1;
    NFB_CUDA(cudaMemset(h->d_tape, 0, (size_t)need * sizeof(float)));
  }
  if (!h->d_gpacked) {
    auto dm = [&](float** p, long long n) {
      return cudaMalloc(p, (size_t)std::max<long long>(n, 1) * sizeof(float)) == cudaSuccess ? 0
          : fail("training: cudaMalloc of %lld floats failed", n);
    };
    if (dm(&h->d_gpacked, h->packed_floats) ||
        dm(&h->d_gwarp, (long long)c.num_warp_embeddings * c.num_warp_features) ||
        dm(&h->d_gapp, (long long)c.num_appearance_embeddings * c.num_appearance_features) ||
        dm(&h->d_gcam, (long long)c.num_camera_embeddings * c.num_camera_features) ||
        dm(&h->d_dcond, (long long)h->max_rays * h->cond_layout.stride) ||
        // d_tr_out: a chunk's coarse outputs, fine outputs and photometric-loss cotangents, (R,6) each
        dm(&h->d_tr_out, (long long)h->max_rays * 18) || dm(&h->d_tr_w, (long long)h->max_rays * smax) ||
        dm(&h->d_loss, nfb::train::kLossSlots))
      return -1;
  }
  // the TimeEncoder's tape holds a whole batch: the batch's condition vectors are built before the chunk loop
  // and differentiated after it
  if (has_time_encoder(h) &&
      grow(&h->d_time_tape, &h->time_tape_floats,
           time_tape_layout(h->time_net, c.time_encoder_num_freqs, h->max_rays).total, "TimeEncoder tape"))
    return -1;
  return 0;
}

// Tape large enough for `rows` rows of either level (free points: one row per point).
int train_prepare_rows(nfb_handle* h, long long rows) {
  const int smax = h->cfg.num_coarse_samples + h->cfg.num_fine_samples;
  return train_prepare(h, (int)std::max<long long>(1, (rows + smax - 1) / smax));
}

// warp_field.apply on `n` free points (+ optional noise) on the tape of level 0: condition
// vectors per point, then warp_forward.  The points land in tape.pts, the warped points in tape.warped.
// `warp_id`: see train_cond; with `encoded`, the points' warp codes (n, G floats).
int warp_points_forward(nfb_handle* h, int n, const float* points, const float* noise, const unsigned* warp_id,
                        bool float_time, bool encoded, cudaStream_t s) {
  const nfb::FieldProgram& p = h->prog[0];
  const TapeLayout t = tape_layout(p, n);
  float* A = h->d_tape;
  nfb::train::add_noise_kernel<<<(unsigned)(((long long)n * 3 + 255) / 256), 256, 0, s>>>(points, noise, A + t.warped,
                                                                                        (long long)n * 3);
  if (launch_check(h, "add_noise_kernel")) return -1;
  // the "view direction" columns are unused here
  if (encoded ? run_cond(h, n, A + t.warped, warp_id, nullptr, nullptr, s, true, false)
              : train_cond(h, n, A + t.warped, warp_id, float_time, nullptr, nullptr, s))
    return -1;
  return warp_forward(h, p, t, nullptr, nullptr, nullptr, 1, A + t.warped, h->d_cond, s);
}

// Embedding gradients: the condition-vector gradients dcond of B rays, scattered into the tables' gradients
// (the adjoint of run_cond; time_backward is the TimeEncoder's).
int run_cond_bwd(nfb_handle* h, int B, const float* dcond, const unsigned* warp_id, const unsigned* app_id,
                 const unsigned* cam_id, cudaStream_t s) {
  const nfb_config& c = h->cfg;
  nfb::train::CondBwdArgs a{};
  a.dcond = dcond; a.num_rays = B;
  const int enc = has_time_encoder(h) ? c.warp_metadata_encoder : NFB_WARP_ENC_GLO;
  a.warp_scale = enc == NFB_WARP_ENC_GLO ? 1.f : enc == NFB_WARP_ENC_BLEND ? 1.f - h->time_alpha : 0.f;
  a.warp_id = enc == NFB_WARP_ENC_TIME ? nullptr : warp_id; a.app_id = app_id; a.cam_id = cam_id;
  a.d_warp_table = h->d_gwarp; a.d_app_table = h->d_gapp; a.d_cam_table = h->d_gcam;
  a.n_warp = c.num_warp_embeddings; a.n_app = c.num_appearance_embeddings; a.n_cam = c.num_camera_embeddings;
  a.layout = h->cond_layout;
  const long long total = (long long)B * a.layout.stride;
  nfb::train::cond_bwd_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(a);
  return launch_check(h, "cond_bwd_kernel");
}

// Adjoint of warp_points_forward, from the gradient of the warped points that the caller has seeded in
// tape.dwarped (after zeroing the tape's gradient region and h->d_dcond): the warp MLP's parameter gradients,
// then those of the codes: the tables' rows and the TimeEncoder's parameters or, with `encoded`, d_code
// (n, G; nullable).
int warp_points_backward(nfb_handle* h, int n, const unsigned* warp_id, bool encoded, float* d_code, cudaStream_t s) {
  const nfb::FieldProgram& p = h->prog[0];
  if (warp_backward(h, p, tape_layout(p, n), 1, h->d_dcond, s)) return -1;
  if (encoded) return cond_vjp_encoded(h, n, h->d_dcond, warp_id != nullptr, false, false, d_code, nullptr, nullptr, s);
  return run_cond_bwd(h, n, h->d_dcond, warp_id, nullptr, nullptr, s) || time_backward(h, n, h->d_dcond, s) ? -1 : 0;
}

// nfb_warp_invert's per-point state for max_rays points, carved from one allocation made on first use.
constexpr long long kInvertRowBytes = 4 * sizeof(double) + 25 * sizeof(float) + sizeof(int);   // 136
int invert_state(nfb_handle* h, nfb::train::InvertState* st) {
  const long long R = h->max_rays;
  if (!h->d_invert && cudaMalloc(&h->d_invert, (size_t)(R * kInvertRowBytes)) != cudaSuccess) {
    h->d_invert = nullptr;
    return fail("warp invert: cannot allocate its %lld-byte workspace", R * kInvertRowBytes);
  }
  char* b = static_cast<char*>(h->d_invert);
  auto take = [&](long long bytes) { char* p = b; b += bytes; return p; };
  st->dx = reinterpret_cast<double*>(take(R * 3 * sizeof(double)));
  st->rb = reinterpret_cast<double*>(take(R * sizeof(double)));
  st->cand = reinterpret_cast<float*>(take(R * 3 * sizeof(float)));
  st->jac = reinterpret_cast<float*>(take(R * 9 * sizeof(float)));
  st->xb = reinterpret_cast<float*>(take(R * 3 * sizeof(float)));
  st->jb = reinterpret_cast<float*>(take(R * 9 * sizeof(float)));
  st->lam = reinterpret_cast<float*>(take(R * sizeof(float)));
  st->status = reinterpret_cast<int*>(take(R * sizeof(int)));
  return 0;
}

// compute_background_loss (training.py:118-135) and its gradient, in chunks of max_rays points.
int train_background(nfb_handle* h, int P, const float* points, const unsigned* warp_ids, const float* noise,
                     float weight, cudaStream_t s) {
  using namespace nfb::train;
  const nfb::FieldProgram& p = h->prog[0];
  const int chunk = std::min(P, h->max_rays);
  if (train_prepare_rows(h, chunk)) return -1;
  for (int p0 = 0; p0 < P; p0 += chunk) {
    const int n = std::min(chunk, P - p0);
    const TapeLayout t = tape_layout(p, n);
    float* A = h->d_tape;
    // the ids are the timestamps of a 'time' encoder too: float(id) (training.py:120-131)
    if (warp_points_forward(h, n, points + (size_t)p0 * 3, noise ? noise + (size_t)p0 * 3 : nullptr, warp_ids + p0,
                            false, false, s))
      return -1;
    NFB_CUDA(cudaMemsetAsync(A + t.grad_begin, 0, (size_t)(t.grad_end - t.grad_begin) * sizeof(float), s));
    NFB_CUDA(cudaMemsetAsync(h->d_dcond, 0, (size_t)n * h->cond_layout.stride * sizeof(float), s));
    // alpha = -2, scale = 0.001: the defaults of compute_background_loss, which train_step does not override
    WarpMagArgs wm{A + t.pts, A + t.warped, nullptr, A + t.dwarped, h->d_loss + kSlotBackground, -2.0f, 0.001f,
                   weight / (float)P, n};
    warp_mag_loss_kernel<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(wm);
    if (launch_check(h, "warp_mag_loss_kernel") || warp_points_backward(h, n, warp_ids + p0, false, nullptr, s))
      return -1;
  }
  return 0;
}

}  // namespace

extern "C" {

int nfb_train_value_and_grad_reg(nfb_handle* h, int B, const float* origins, const float* directions,
                                 const float* viewdirs, const unsigned* warp_id, const unsigned* app_id,
                                 const unsigned* cam_id, float warp_alpha, const float* t_rand,
                                 const float* u_rand, unsigned flags, const float* rgb_target,
                                 int chunk_rays, const nfb_train_reg* reg, float* const* grads,
                                 const long long* numels, int count, float* loss_out, void* stream) {
  if (check_call(h, B)) return -1;
  if (!rgb_target || !grads || !numels || !loss_out) return fail("null argument");
  if (count != (int)h->specs.size()) return fail("expected %d gradient tensors, got %d", (int)h->specs.size(), count);
  if (flags & NFB_FLAG_METADATA_ENCODED) return fail("training with metadata_encoded=True is not supported");
  const nfb_config& c = h->cfg;
  if (check_grads(h, grads, numels, count)) return -1;
  cudaStream_t s = (cudaStream_t)stream;
  if (enter_stream(h, s)) return -1;
  if (B == 0) return 0;
  if (chunk_rays < 1) chunk_rays = 256;
  chunk_rays = std::min(chunk_rays, B);
  if (train_prepare(h, chunk_rays)) return -1;
  const int nc = c.num_coarse_samples, nfine = nc + c.num_fine_samples;
  const bool use_warp = !(flags & NFB_FLAG_NO_WARP);
  const bool fine = c.num_fine_samples > 0;
  if (set_window(h, warp_alpha, s)) return -1;
  if (zero_grads(h, s)) return -1;
  NFB_CUDA(cudaMemsetAsync(h->d_loss, 0, nfb::train::kLossSlots * sizeof(float), s));
  // condition vectors of the whole batch (per ray), their gradient accumulator
  const bool float_time = has_time_encoder(h) && c.warp_metadata_encoder == NFB_WARP_ENC_TIME;
  if (train_cond(h, B, viewdirs ? viewdirs : directions, warp_id, float_time, app_id, cam_id, s)) return -1;
  NFB_CUDA(cudaMemsetAsync(h->d_dcond, 0, (size_t)B * h->cond_layout.stride * sizeof(float), s));
  if (nfb_coarse_z_vals(h, B, t_rand, h->d_zc, stream)) return -1;
  const float scale = 1.f / ((float)B * 3.f);       // mean over the local batch (training.py:173)
  RegCfg rc_{};
  const RegCfg* rcfg = nullptr;
  if (reg && (reg->use_elastic_loss || reg->use_warp_reg_loss)) {
    if (!use_warp || h->prog[0].warp_type == 0)
      return fail("the elastic / warp-reg losses need a warp field (training.py:176-207)");
    if (reg->use_elastic_loss && (reg->elastic_loss_type < 0 || reg->elastic_loss_type > NFB_ELASTIC_LOG_DET))
      return fail("elastic_loss_type %d is not supported ('nr' differentiates an SVD with a repeated factor "
                  "and yields NaNs in the reference, training.py:59)", reg->elastic_loss_type);
    rc_.elastic = reg->use_elastic_loss != 0; rc_.reduce = reg->elastic_reduce_method; rc_.type = reg->elastic_loss_type;
    rc_.elastic_weight = reg->elastic_loss_weight;
    rc_.warp_reg = reg->use_warp_reg_loss != 0; rc_.warp_reg_weight = reg->warp_reg_loss_weight;
    rc_.warp_reg_alpha = reg->warp_reg_loss_alpha; rc_.warp_reg_scale = reg->warp_reg_loss_scale;
    rc_.batch_rays = B; rc_.stats = h->d_loss;
    rcfg = &rc_;
  }
  for (int r0 = 0; r0 < B; r0 += chunk_rays) {
    const int R = std::min(chunk_rays, B - r0);
    // the chunk's rays (the kernels index them from 0)
    const float* cond = h->d_cond + (size_t)r0 * h->cond_layout.stride;
    float* dcond = h->d_dcond + (size_t)r0 * h->cond_layout.stride;
    const float* o = origins + (size_t)r0 * 3;
    const float* d = directions + (size_t)r0 * 3;
    const float* tg = rgb_target + (size_t)r0 * 3;
    float* d_out = h->d_tr_out + 12 * (size_t)R;
    float* w = h->d_tr_w;
    // forward, photometric loss and backward of one level at z
    auto level = [&](int lv, int S, const float* z, float* out, int loss_slot) {
      int alpha_step = -1, rgb_step = -1;
      if (level_forward(h, lv, R, S, z, o, d, cond, use_warp, out, w, s, &alpha_step, &rgb_step)) return -1;
      nfb::train::photometric_loss_kernel<<<(unsigned)((R + 127) / 128), 128, 0, s>>>(out, tg, scale, R, d_out,
                                                                                     h->d_loss + loss_slot);
      if (launch_check(h, "photometric_loss_kernel")) return -1;
      return level_backward(h, lv, R, S, z, d, dcond, use_warp, alpha_step, rgb_step, d_out, nullptr, nullptr, w,
                            rcfg, s);
    };
    float* zc = h->d_zc + (size_t)r0 * nc;
    if (level(0, nc, zc, h->d_tr_out, nfb::train::kSlotRgbCoarse)) return -1;
    if (fine) {
      float* zf = h->d_zf + (size_t)r0 * nfine;
      if (run_resample(h, R, zc, w, u_rand ? u_rand + (size_t)r0 * c.num_fine_samples : nullptr, zf, s) ||
          level(1, nfine, zf, h->d_tr_out + 6 * (size_t)R, nfb::train::kSlotRgbFine))
        return -1;
    }
  }
  if (run_cond_bwd(h, B, h->d_dcond, warp_id, app_id, cam_id, s) || time_backward(h, B, h->d_dcond, s)) return -1;
  // background loss (training.py:118-135, 246-257): warp_field.apply on free points
  const int P = (reg && reg->use_background_loss) ? reg->num_background_points : 0;
  if (P > 0) {
    if (!use_warp || h->prog[0].warp_type == 0) return fail("the background loss needs a warp field");
    if (!reg->background_points || !reg->background_warp_ids) return fail("background points / warp ids are null");
    if (train_background(h, P, reg->background_points, reg->background_warp_ids, reg->background_noise,
                         reg->background_loss_weight, s))
      return -1;
  }
  {
    const long long jrows = (reg && reg->use_elastic_loss) ? (reg->elastic_reduce_method == 0 ? B : (long long)B * nc) : 1;
    nfb::train::finalize_stats_kernel<<<1, 32, 0, s>>>(h->d_loss, 1.f / (float)B, 1.f / (float)jrows, P > 0 ? 1.f / (float)P : 0.f);
    if (launch_check(h, "finalize_stats_kernel")) return -1;
  }
  if (unpack_grads(h, grads, count, s)) return -1;
  // without regularisers, loss_out holds the two rgb losses only
  const int slots = reg ? nfb::train::kLossSlots : nfb::train::kSlotRgbFine + 1;
  NFB_CUDA(cudaMemcpyAsync(loss_out, h->d_loss, slots * sizeof(float), cudaMemcpyDeviceToDevice, s));
  return 0;
}

int nfb_train_value_and_grad(nfb_handle* h, int B, const float* origins, const float* directions,
                             const float* viewdirs, const unsigned* warp_id, const unsigned* app_id,
                             const unsigned* cam_id, float warp_alpha, const float* t_rand,
                             const float* u_rand, unsigned flags, const float* rgb_target,
                             int chunk_rays, float* const* grads, const long long* numels, int count,
                             float* loss_out, void* stream) {
  return nfb_train_value_and_grad_reg(h, B, origins, directions, viewdirs, warp_id, app_id, cam_id, warp_alpha, t_rand,
                                      u_rand, flags, rgb_target, chunk_rays, nullptr, grads, numels, count, loss_out,
                                      stream);
}

int nfb_render_vjp(nfb_handle* h, int B, const float* origins, const float* directions, const float* viewdirs,
                   const unsigned* warp_id, const unsigned* app_id, const unsigned* cam_id, float warp_alpha,
                   unsigned flags, const float* z_coarse, const float* z_fine, const float* d_out_coarse,
                   const float* d_out_fine, const float* d_weights_coarse, const float* d_weights_fine,
                   const float* d_warped_coarse, const float* d_warped_fine, float* d_warp_code, float* d_app_code,
                   float* d_cam_code, int chunk_rays, float* const* grads, const long long* numels, int count,
                   void* stream) {
  if (check_call(h, B)) return -1;
  if (check_grads(h, grads, numels, count)) return -1;
  const nfb_config& c = h->cfg;
  const bool encoded = (flags & NFB_FLAG_METADATA_ENCODED) != 0;
  if (!encoded && (d_warp_code || d_app_code || d_cam_code))
    return fail("render VJP: code gradients need NFB_FLAG_METADATA_ENCODED");
  const bool use_warp = !(flags & NFB_FLAG_NO_WARP);
  const bool warp = use_warp && c.warp_field_type != NFB_WARP_NONE;
  const bool coarse = d_out_coarse || d_weights_coarse || d_warped_coarse;
  const bool fine = d_out_fine || d_weights_fine || d_warped_fine;
  if (fine && (c.num_fine_samples == 0 || (flags & NFB_FLAG_COARSE_ONLY)))
    return fail("render VJP: fine-level cotangents, but the call renders no fine level");
  if (!warp && (d_warped_coarse || d_warped_fine))
    return fail("render VJP: warped-point cotangents, but the call does not warp");
  cudaStream_t s = (cudaStream_t)stream;
  if (enter_stream(h, s)) return -1;
  if (B == 0) return 0;
  if (!origins || !directions) return fail("render VJP: origins / directions are null");
  if ((coarse && !z_coarse) || (fine && !z_fine)) return fail("render VJP: the z values of a level with cotangents are null");
  if (chunk_rays < 1) chunk_rays = 256;
  chunk_rays = std::min(chunk_rays, B);
  if (train_prepare(h, chunk_rays)) return -1;
  if (set_window(h, warp_alpha, s) || zero_grads(h, s)) return -1;
  // condition vectors of the whole batch (per ray), their gradient accumulator
  const float* vd = viewdirs ? viewdirs : directions;
  const bool time_enc = warp && !encoded && has_time_encoder(h);
  if (time_enc ? train_cond(h, B, vd, warp_id, c.warp_metadata_encoder == NFB_WARP_ENC_TIME, app_id, cam_id, s)
               : run_cond(h, B, vd, warp_id, app_id, cam_id, s, encoded, false))
    return -1;
  NFB_CUDA(cudaMemsetAsync(h->d_dcond, 0, (size_t)B * h->cond_layout.stride * sizeof(float), s));
  const int nc = c.num_coarse_samples, nfine = nc + c.num_fine_samples;
  auto at = [](const float* p, size_t off) { return p ? p + off : nullptr; };
  for (int r0 = 0; r0 < B; r0 += chunk_rays) {
    const int R = std::min(chunk_rays, B - r0);
    const float* cond = h->d_cond + (size_t)r0 * h->cond_layout.stride;
    float* dcond = h->d_dcond + (size_t)r0 * h->cond_layout.stride;
    const float* o = origins + (size_t)r0 * 3;
    const float* d = directions + (size_t)r0 * 3;
    // the taped forward of one level at z, then its backward from the caller's cotangents
    auto level = [&](int lv, int S, const float* z, const float* d_out, const float* d_weights, const float* d_warped) {
      int alpha_step = -1, rgb_step = -1;
      if (level_forward(h, lv, R, S, z, o, d, cond, use_warp, h->d_tr_out, nullptr, s, &alpha_step, &rgb_step))
        return -1;
      return level_backward(h, lv, R, S, z, d, dcond, use_warp, alpha_step, rgb_step, d_out, d_weights, d_warped,
                            nullptr, nullptr, s);
    };
    if (coarse && level(0, nc, z_coarse + (size_t)r0 * nc, at(d_out_coarse, (size_t)r0 * 6),
                        at(d_weights_coarse, (size_t)r0 * nc), at(d_warped_coarse, (size_t)r0 * nc * 3)))
      return -1;
    if (fine && level(1, nfine, z_fine + (size_t)r0 * nfine, at(d_out_fine, (size_t)r0 * 6),
                      at(d_weights_fine, (size_t)r0 * nfine), at(d_warped_fine, (size_t)r0 * nfine * 3)))
      return -1;
  }
  if (encoded) {
    if (cond_vjp_encoded(h, B, h->d_dcond, warp_id, app_id, cam_id, d_warp_code, d_app_code, d_cam_code, s)) return -1;
  } else if (run_cond_bwd(h, B, h->d_dcond, warp_id, app_id, cam_id, s) ||
             (time_enc && time_backward(h, B, h->d_dcond, s))) {
    return -1;
  }
  return unpack_grads(h, grads, count, s);
}

int nfb_warp_vjp(nfb_handle* h, int P, const float* points, const unsigned* warp_id, float warp_alpha,
                 unsigned flags, const float* d_warped, float* d_code, float* const* grads, const long long* numels,
                 int count, void* stream) {
  if (!h) return fail("null handle");
  if (P < 0) return fail("P must be >= 0");
  if (check_call(h, std::min(P, h->max_rays))) return -1;
  if (check_grads(h, grads, numels, count)) return -1;
  const nfb_config& c = h->cfg;
  if (h->prog[0].warp_type == 0) return fail("the model has no warp field");
  const bool encoded = (flags & NFB_FLAG_METADATA_ENCODED) != 0;
  if (d_code && !encoded) return fail("warp VJP: d_code needs NFB_FLAG_METADATA_ENCODED");
  cudaStream_t s = (cudaStream_t)stream;
  if (enter_stream(h, s)) return -1;
  if (P == 0) return 0;
  if (!points || !d_warped) return fail("warp VJP: points / d_warped are null");
  if (set_window(h, warp_alpha, s)) return -1;
  const int chunk = std::min(P, h->max_rays);
  if (train_prepare_rows(h, chunk) || zero_grads(h, s)) return -1;
  const nfb::FieldProgram& p = h->prog[0];
  const int G = h->cond_layout.G;
  for (int p0 = 0; p0 < P; p0 += chunk) {
    const int n = std::min(chunk, P - p0);
    const TapeLayout t = tape_layout(p, n);
    float* A = h->d_tape;
    // the chunk's ids, or with `encoded` its codes (G floats per point)
    const unsigned* ids = !warp_id ? nullptr
        : encoded ? reinterpret_cast<const unsigned*>(reinterpret_cast<const float*>(warp_id) + (size_t)p0 * G)
                  : warp_id + p0;
    if (warp_points_forward(h, n, points + (size_t)p0 * 3, nullptr, ids, c.warp_metadata_encoder == NFB_WARP_ENC_TIME,
                            encoded, s))
      return -1;
    NFB_CUDA(cudaMemsetAsync(A + t.grad_begin, 0, (size_t)(t.grad_end - t.grad_begin) * sizeof(float), s));
    NFB_CUDA(cudaMemsetAsync(h->d_dcond, 0, (size_t)n * h->cond_layout.stride * sizeof(float), s));
    NFB_CUDA(cudaMemcpyAsync(A + t.dwarped, d_warped + (size_t)p0 * 3, (size_t)n * 3 * sizeof(float),
                             cudaMemcpyDeviceToDevice, s));
    if (warp_points_backward(h, n, ids, encoded, d_code ? d_code + (size_t)p0 * G : nullptr, s)) return -1;
  }
  return unpack_grads(h, grads, count, s);
}

int nfb_warp_jacobian(nfb_handle* h, int P, const float* points, const unsigned* warp_id, float warp_alpha,
                      float* warped_out, float* jacobian_out, void* stream) {
  if (!h || !points || !jacobian_out) return fail("null argument");
  if (P < 0) return fail("P must be >= 0");
  if (check_call(h, std::min(P, h->max_rays))) return -1;
  const nfb_config& c = h->cfg;
  if (h->prog[0].warp_type == 0) return fail("the model has no warp field");
  cudaStream_t s = (cudaStream_t)stream;
  if (enter_stream(h, s)) return -1;
  if (P == 0) return 0;
  if (set_window(h, warp_alpha, s)) return -1;
  const int chunk = std::min(P, h->max_rays);
  if (train_prepare_rows(h, chunk)) return -1;
  for (int p0 = 0; p0 < P; p0 += chunk) {
    const int n = std::min(chunk, P - p0);
    if (warp_points_forward(h, n, points + (size_t)p0 * 3, nullptr, warp_id ? warp_id + p0 : nullptr,
                            c.warp_metadata_encoder == NFB_WARP_ENC_TIME, false, s))
      return -1;
    const nfb::FieldProgram& p = h->prog[0];
    const TapeLayout t = tape_layout(p, n);
    if (warped_out)
      NFB_CUDA(cudaMemcpyAsync(warped_out + (size_t)p0 * 3, h->d_tape + t.warped, (size_t)n * 3 * sizeof(float),
                               cudaMemcpyDeviceToDevice, s));
    if (warp_jacobian_on_tape(h, p, t, h->d_tape, nullptr, n, nullptr, nullptr, false, jacobian_out + (size_t)p0 * 9, s))
      return -1;
  }
  return 0;
}

int nfb_warp_invert(nfb_handle* h, int P, const float* targets, const float* init, const unsigned* warp_id,
                    float warp_alpha, int max_iters, float tol, float* points_out, float* residual_out,
                    float* jacobian_out, int* status_out, void* stream) {
  if (!h || !targets || !points_out || !residual_out) return fail("null argument");
  if (P < 0) return fail("P must be >= 0");
  if (check_call(h, std::min(P, h->max_rays))) return -1;
  const nfb_config& c = h->cfg;
  const nfb::FieldProgram& p = h->prog[0];
  if (p.warp_type == 0) return fail("the model has no warp field");
  if (check_relu_warp(p, "warp invert")) return -1;
  if (max_iters < 1 || max_iters > 64) return fail("warp invert: max_iters=%d outside [1, 64]", max_iters);
  if (!std::isfinite(tol) || !(tol > 0.f)) return fail("warp invert: tol=%g must be finite and > 0", (double)tol);
  cudaStream_t s = (cudaStream_t)stream;
  if (enter_stream(h, s)) return -1;
  if (P == 0) return 0;
  if (set_window(h, warp_alpha, s)) return -1;
  const int chunk = std::min(P, h->max_rays);
  nfb::train::InvertState st{};
  if (train_prepare_rows(h, chunk) || invert_state(h, &st)) return -1;
  const bool float_time = c.warp_metadata_encoder == NFB_WARP_ENC_TIME;
  for (int p0 = 0; p0 < P; p0 += chunk) {
    const int n = std::min(chunk, P - p0);
    const TapeLayout t = tape_layout(p, n);
    const unsigned* ids = warp_id ? warp_id + p0 : nullptr;
    const float* start = (init ? init : targets) + (size_t)p0 * 3;
    NFB_CUDA(cudaMemcpyAsync(st.cand, start, (size_t)n * 3 * sizeof(float), cudaMemcpyDeviceToDevice, s));
    nfb::train::InvertStepArgs a{};
    a.st = st; a.warped = h->d_tape + t.warped; a.target = targets + (size_t)p0 * 3; a.tol = tol; a.n = n;
    a.points_out = points_out + (size_t)p0 * 3; a.residual_out = residual_out + p0;
    a.jacobian_out = jacobian_out ? jacobian_out + (size_t)p0 * 9 : nullptr;
    a.status_out = status_out ? status_out + p0 : nullptr;
    // a fixed number of iterations, no readback: frozen points ride along unchanged
    for (int it = 0; it < max_iters; ++it) {
      if (warp_points_forward(h, n, st.cand, nullptr, ids, float_time, false, s) ||
          warp_jacobian_on_tape(h, p, t, h->d_tape, nullptr, n, nullptr, nullptr, false, st.jac, s))
        return -1;
      a.first = it == 0; a.last = it == max_iters - 1;
      nfb::train::warp_invert_step_kernel<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(a);
      if (launch_check(h, "warp_invert_step_kernel")) return -1;
    }
  }
  return 0;
}

int nfb_adam_step(float* params, const float* grads, float* m, float* v, long long n, float learning_rate,
                  float beta1, float beta2, float eps, long long step, void* stream) {
  if (!params || !grads || !m || !v) return fail("null argument");
  if (n <= 0) return 0;
  if (step < 1) return fail("adam: step counts from 1");
  const float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
  nfb::train::adam_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      params, grads, m, v, n, learning_rate, beta1, beta2, eps, bc1, bc2);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("adam_kernel launch failed: %s", cudaGetErrorString(e));
  return 0;
}

int nfb_set_train_precision(nfb_handle* h, int train_precision) {
  if (!h) return fail("null handle");
  if (train_precision != NFB_TRAIN_FP32 && train_precision != NFB_TRAIN_TF32X3)
    return fail("train precision %d is not NFB_TRAIN_FP32 (0) or NFB_TRAIN_TF32X3 (1)", train_precision);
  h->train_precision = train_precision;
  return 0;
}

int nfb_selftest_sgemm(int mode, long long rows, int n, int k_x, int k_in, int act, const float* x, int ldx,
                       const float* in, int ldin, const float* w, int ldw, const float* bias, float* y,
                       const float* dy, float* dx, float* din, float* dw, long long k_split,
                       long long* k_split_used, void* stream) {
  return nfb_selftest_train_gemm(NFB_TRAIN_FP32, mode, rows, n, k_x, k_in, act, x, ldx, in, ldin, w, ldw, bias, y,
                                 dy, dx, din, dw, k_split, k_split_used, stream);
}

// The three launches of net_forward / net_backward for one layer, with their functors.
int nfb_selftest_train_gemm(int train_precision, int mode, long long rows, int n, int k_x, int k_in, int act,
                            const float* x, int ldx, const float* in, int ldin, const float* w, int ldw,
                            const float* bias, float* y, const float* dy, float* dx, float* din, float* dw,
                            long long k_split, long long* k_split_used, void* stream) {
  using namespace nfb::train;
  const int K = k_x + k_in;
  if (rows < 1 || n < 1 || k_x < 0 || k_in < 0 || K < 1) return fail("selftest_sgemm: empty shape");
  if (ldx < k_x || ldin < k_in || ldw < n) return fail("selftest_sgemm: a leading dimension is below its width");
  if (act < nfb::kNone || act > nfb::kSoftplus) return fail("selftest_sgemm: bad activation %d", act);
  if (k_split < 0 || (k_split > 0 && mode != NFB_SGEMM_DW)) return fail("selftest_sgemm: k_split applies to dW only");
  if (!w || (mode != NFB_SGEMM_DX && ((k_x > 0 && !x) || (k_in > 0 && !in))))
    return fail("selftest_sgemm: null operand");
  // launch_gemm reads the SM count (dw_split) and counts launches in a handle; this call has none
  nfb_handle h;
  if (nfb_set_train_precision(&h, train_precision)) return -1;
  int dev = 0;
  NFB_CUDA(cudaGetDevice(&dev));
  NFB_CUDA(cudaDeviceGetAttribute(&h.sm_count, cudaDevAttrMultiProcessorCount, dev));
  cudaStream_t s = (cudaStream_t)stream;
  const ConcatA a{x, ldx, k_x, in, ldin};
  const DZ dz{dy, y, ldw, act};
  long long per = 0;
  int rc;
  if (mode == NFB_SGEMM_FORWARD) {
    if (!bias || !y) return fail("selftest_sgemm: null bias / y");
    rc = launch_gemm(&h, rows, n, K, a, WeightB{w, ldw}, StoreBiasAct{y, ldw, bias, act}, 0, s, "sgemm (forward)");
  } else if (mode == NFB_SGEMM_DX) {
    if (!y || !dy || (k_x > 0 && !dx) || (k_in > 0 && !din)) return fail("selftest_sgemm: null y / dy / dx / din");
    rc = launch_gemm<true, false>(&h, rows, K, n, dz, WeightBT{w, ldw}, AccumSplit{dx, ldx, k_x, din, ldin}, 0, s,
                                  "sgemm (dX)");
  } else if (mode == NFB_SGEMM_DW) {
    if (!y || !dy || !dw) return fail("selftest_sgemm: null y / dy / dw");
    per = k_split > 0 ? k_split : dw_split_for(&h, K, n, rows);
    rc = launch_gemm<false, true>(&h, K, n, rows, ConcatAT{a}, DZB{dz}, AtomicAdd{dw, ldw}, per, s, "sgemm (dW)");
  } else {
    return fail("selftest_sgemm: bad mode %d", mode);
  }
  if (k_split_used) *k_split_used = per;
  return rc;
}

}  // extern "C"
