// Training tier, part 2 (SURVEY §8(f) #2): the warp Jacobian and the regularisers of
// training.py:71-135, 176-212.
//
//   J = jax.jacfwd(warp)(x)            (warping.py:196-198, 385-387): forward mode through
//       the positional encoding, the warp MLP (TANGENT rows: three per point, one per input
//       direction, pushed through the same GEMM template with the ReLU masks of the primal
//       tape) and the SE(3) / translation tail (forward-mode numbers on the head outputs);
//   elastic loss  rho(sum log^2 svals(J)) etc. (training.py:71-115): 3x3 one-sided Jacobi
//       SVD per point, dL/dJ = U diag(.) V^T;
//   its gradient  - through the tangent head outputs: the tangent MLP backwards (weights only:
//       ReLU masks are piecewise constant, exactly what jax.grad of jacfwd gives), and
//                 - through the PRIMAL head outputs: second derivatives of the SE(3) tail by
//       nested forward-mode numbers, added to the primal head gradient;
//   warp-reg loss (training.py:194-207) and background loss (training.py:118-135): robust
//       losses of |warped - x|^2, adjoint = one vector added to d(warped).
#pragma once
#include "train.cuh"

namespace nfb {
namespace train {

// ---------------------------------------------------------------------------
// utils.general_loss_with_squared_residual (utils.py:264-331) and d loss / d squared_x.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void general_loss(float sq, float alpha, float scale, float& loss, float& dloss) {
  const float eps = 1.1920929e-07f;
  const float x = sq / (scale * scale);
  float l, dl;
  if (isinf(alpha) && alpha < 0.f) {
    l = -expm1f(-0.5f * x); dl = 0.5f * expf(-0.5f * x);
  } else if (alpha == 0.f) {
    l = log1pf(fminf(0.5f * x, 3e37f)); dl = 0.5f / (1.f + 0.5f * x);
  } else if (alpha == 2.f) {
    l = 0.5f * x; dl = 0.5f;
  } else if (isinf(alpha)) {
    l = expm1f(fminf(0.5f * x, 87.5f)); dl = 0.5f * x < 87.5f ? 0.5f * expf(0.5f * x) : 0.f;
  } else {
    const float b = fmaxf(eps, fabsf(alpha - 2.f));
    const float a = (alpha >= 0.f ? 1.f : -1.f) * fmaxf(eps, fabsf(alpha));
    const float base = x / b + 1.f;
    l = (b / a) * (powf(base, 0.5f * alpha) - 1.f);
    dl = 0.5f * powf(base, 0.5f * alpha - 1.f);
  }
  loss = scale * l;
  dloss = dl / scale;               // scale * dl / scale^2
}

// ---------------------------------------------------------------------------
// 3x3 SVD, one-sided Jacobi (Hestenes): A = U diag(s) V^T, s >= 0 in no particular
// order (every consumer is symmetric in the singular values).  A column of U that
// belongs to a vanishing singular value is left zero.
// ---------------------------------------------------------------------------
__device__ inline void svd3(const float A[3][3], float U[3][3], float s[3], float V[3][3]) {
  float G[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) { G[i][j] = A[i][j]; V[i][j] = i == j ? 1.f : 0.f; }
  for (int sweep = 0; sweep < 15; ++sweep) {
    float off = 0.f;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        float a = 0.f, b = 0.f, g = 0.f;
        for (int i = 0; i < 3; ++i) { a = fmaf(G[i][p], G[i][p], a); b = fmaf(G[i][q], G[i][q], b); g = fmaf(G[i][p], G[i][q], g); }
        if (fabsf(g) <= 1e-9f * sqrtf(a * b) || g == 0.f) continue;
        off = fmaxf(off, fabsf(g) / sqrtf(a * b));
        const float zeta = (b - a) / (2.f * g);
        const float t = (zeta >= 0.f ? 1.f : -1.f) / (fabsf(zeta) + sqrtf(1.f + zeta * zeta));
        const float c = 1.f / sqrtf(1.f + t * t), sn = c * t;
        for (int i = 0; i < 3; ++i) {
          const float gp = G[i][p], gq = G[i][q];
          G[i][p] = c * gp - sn * gq; G[i][q] = sn * gp + c * gq;
          const float vp = V[i][p], vq = V[i][q];
          V[i][p] = c * vp - sn * vq; V[i][q] = sn * vp + c * vq;
        }
      }
    if (off < 1e-7f) break;
  }
  for (int j = 0; j < 3; ++j) {
    float n = 0.f;
    for (int i = 0; i < 3; ++i) n = fmaf(G[i][j], G[i][j], n);
    n = sqrtf(n);
    s[j] = n;
    const float inv = n > 1e-30f ? 1.f / n : 0.f;
    for (int i = 0; i < 3; ++i) U[i][j] = G[i][j] * inv;
  }
}
__device__ __forceinline__ float det3(const float J[3][3]) {
  return J[0][0] * (J[1][1] * J[2][2] - J[1][2] * J[2][1]) - J[0][1] * (J[1][0] * J[2][2] - J[1][2] * J[2][0]) +
         J[0][2] * (J[1][0] * J[2][1] - J[1][1] * J[2][0]);
}
// cofactor matrix: d det / d J
__device__ __forceinline__ void cof3(const float J[3][3], float C[3][3]) {
  C[0][0] = J[1][1] * J[2][2] - J[1][2] * J[2][1]; C[0][1] = J[1][2] * J[2][0] - J[1][0] * J[2][2]; C[0][2] = J[1][0] * J[2][1] - J[1][1] * J[2][0];
  C[1][0] = J[0][2] * J[2][1] - J[0][1] * J[2][2]; C[1][1] = J[0][0] * J[2][2] - J[0][2] * J[2][0]; C[1][2] = J[0][1] * J[2][0] - J[0][0] * J[2][1];
  C[2][0] = J[0][1] * J[1][2] - J[0][2] * J[1][1]; C[2][1] = J[0][2] * J[1][0] - J[0][0] * J[1][2]; C[2][2] = J[0][0] * J[1][1] - J[0][1] * J[1][0];
}

enum ElasticType { kLogSvals = 0, kSvals = 1, kJtj = 2, kDiv = 3, kDet = 4, kLogDet = 5 };

// compute_elastic_loss (training.py:71-115): squared residual and its gradient w.r.t. J.
__device__ inline void elastic_sq(const float J[3][3], int type, float& sq, float dJ[3][3]) {
  const float eps = 1e-6f;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) dJ[i][j] = 0.f;
  if (type == kLogSvals || type == kSvals) {
    float U[3][3], s[3], V[3][3], g[3];
    svd3(J, U, s, V);
    sq = 0.f;
    for (int k = 0; k < 3; ++k) {
      if (type == kLogSvals) {
        const float l = logf(fmaxf(s[k], eps));
        sq += l * l;
        g[k] = s[k] > eps ? 2.f * l / s[k] : 0.f;          // jnp.maximum: zero gradient below eps
      } else {
        sq += (s[k] - 1.f) * (s[k] - 1.f);
        g[k] = 2.f * (s[k] - 1.f);
      }
    }
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j)
        dJ[i][j] = U[i][0] * g[0] * V[j][0] + U[i][1] * g[1] * V[j][1] + U[i][2] * g[2] * V[j][2];
  } else if (type == kJtj) {
    float E[3][3];
    sq = 0.f;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        E[i][j] = J[i][0] * J[j][0] + J[i][1] * J[j][1] + J[i][2] * J[j][2] - (i == j ? 1.f : 0.f);
        sq += E[i][j] * E[i][j];
      }
    sq *= 0.25f;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) dJ[i][j] = E[i][0] * J[0][j] + E[i][1] * J[1][j] + E[i][2] * J[2][j];
  } else if (type == kDiv) {
    const float div = J[0][0] + J[1][1] + J[2][2] - 3.f;          // utils.jacobian_to_div
    sq = div * div;
    for (int i = 0; i < 3; ++i) dJ[i][i] = 2.f * div;
  } else {
    const float det = det3(J);
    float C[3][3];
    cof3(J, C);
    float k;
    if (type == kDet) { sq = (det - 1.f) * (det - 1.f); k = 2.f * (det - 1.f); }
    else { const float l = logf(fmaxf(det, eps)); sq = l * l; k = det > eps ? 2.f * l / det : 0.f; }
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) dJ[i][j] = k * C[i][j];
  }
}

// ---------------------------------------------------------------------------
// Median-depth sample of every ray (model_utils.compute_depth_index, model_utils.py:218-245):
// first sample whose cumulative weight reaches 0.5 (0 when none does).  One warp per ray.
// ---------------------------------------------------------------------------
__global__ void depth_index_kernel(const float* __restrict__ weights, int num_rays, int S, int* __restrict__ sel) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ray = blockIdx.x * (blockDim.x >> 5) + warp;
  if (ray >= num_rays) return;
  float carry = 0.f;
  int found = -1;
  for (int i0 = 0; i0 < S && found < 0; i0 += 32) {
    const int i = i0 + lane;
    float c = i < S ? weights[(size_t)ray * S + i] : 0.f;
#pragma unroll
    for (int sh = 1; sh < 32; sh <<= 1) {
      const float t = __shfl_up_sync(0xffffffffu, c, sh);
      if (lane >= sh) c = c + t;
    }
    c = c + carry;
    const unsigned m = __ballot_sync(0xffffffffu, i < S && c >= 0.5f);
    if (m) found = i0 + __ffs(m) - 1;
    carry = __shfl_sync(0xffffffffu, c, 31);
  }
  if (lane == 0) sel[ray] = ray * S + (found < 0 ? 0 : found);
}

// ---------------------------------------------------------------------------
// Tangent of an encoded input: row r*3 + j = d enc(x) / d x_j of selected row r
// (annealed_sinusoidal_encode, modules.py:231-294: [x, w_f sin(2^f x), w_f sin(2^f x + pi/2)]);
// the metadata / condition columns do not depend on the point.  With `jac` the encoded point is
// itself a function of the input point u (the warped point y = W(u) of nfb_density_grad): row r*3 + j
// is then d enc(y) / d u_j = sum_c d enc / d y_c J_cj, J = jac[r] row-major (no sel).
// ---------------------------------------------------------------------------
struct EncodeTangentArgs {
  const float* pts; const int* sel; const float* window; float* tin;
  int F, ld; long long R;
  const float* jac;                // (R,9) input tangents, or null: the unit vectors e_j
};
__global__ void encode_tangent_kernel(const EncodeTangentArgs a) {
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= a.R * 3) return;
  const long long r = m / 3;
  const int j = (int)(m - r * 3);
  const long long row = a.sel ? a.sel[r] : r;
  float* o = a.tin + m * a.ld;
  for (int q = 0; q < a.ld; ++q) o[q] = 0.f;
  if (a.jac) {
    float x[3], t[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) { x[c] = a.pts[row * 3 + c]; t[c] = a.jac[r * 9 + c * 3 + j]; o[c] = t[c]; }
    for (int f = 0; f < a.F; ++f) {
      const float w = a.window ? a.window[f] : 1.f;
      const float s = exp2f((float)f);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float ang = x[c] * s;
        o[3 + f * 6 + c] = w * s * cosf(ang) * t[c];
        o[3 + f * 6 + 3 + c] = w * s * cosf(ang + kHalfPiF) * t[c];
      }
    }
    return;
  }
  const float xj = a.pts[row * 3 + j];
  o[j] = 1.f;
  for (int f = 0; f < a.F; ++f) {
    const float w = a.window ? a.window[f] : 1.f;
    const float s = exp2f((float)f);
    const float ang = xj * s;
    o[3 + f * 6 + j] = w * s * cosf(ang);
    o[3 + f * 6 + 3 + j] = w * s * cosf(ang + kHalfPiF);
  }
}

// GEMM functors of the tangent MLP: the activation mask comes from the PRIMAL tape row.
struct StoreMasked {               // Y_t = act'(Y_primal) * ([X_t | IN_t] W), no bias
  float* y; int ld; const float* y_primal; const int* sel; int act;
  __device__ void operator()(long long m, int n, float v) const {
    const long long row = sel ? sel[m / 3] : m / 3;
    y[m * ld + n] = v * act_grad_from_output(y_primal[row * ld + n], act);
  }
};
struct DZT {                       // dZ_t(m, n) = dY_t(m, n) * act'(Y_primal(row(m), n))
  const float* dy; const float* y_primal; const int* sel; int ld; int act;
  __device__ float operator()(long long m, long long n) const {
    const long long row = sel ? sel[m / 3] : m / 3;
    return dy[m * ld + n] * act_grad_from_output(y_primal[row * ld + n], act);
  }
};
struct DZTB {
  DZT z;
  __device__ float operator()(long long m, int n) const { return z(m, n); }
};

// ---------------------------------------------------------------------------
// The density and its gradient at free points (nfb_density_grad): sigma = act(raw) and
// d sigma / d x_j = act'(raw) * (tangent row r*3 + j of the raw density), the derivative taken as
// composite_vjp_kernel takes it (relu: 0 where raw <= 0).
// ---------------------------------------------------------------------------
struct DensityGradArgs {
  const float* raw; int ld;        // primal raw density, column 0 of the alpha head's tape rows
  const float* traw;               // its tangent rows r*3 + j (same ld)
  const float* pts;                // (R,3) the encoded (warped) points
  float* sigma;                    // (R) or null
  float* grad;                     // (R,3)
  float* warped;                   // (R,3) or null
  int sigma_act;
  long long R;
};
__global__ void density_grad_kernel(const DensityGradArgs a) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= a.R) return;
  const float raw = a.raw[r * a.ld];
  const float sigma = apply_act(raw, a.sigma_act);
  float dact;
  if (a.sigma_act == kSoftplus) dact = 1.f / (1.f + expf(-raw));
  else if (a.sigma_act == kRelu) dact = raw > 0.f ? 1.f : 0.f;
  else dact = act_grad_from_output(sigma, a.sigma_act);
  if (a.sigma) a.sigma[r] = sigma;
#pragma unroll
  for (int j = 0; j < 3; ++j) a.grad[r * 3 + j] = dact * a.traw[(r * 3 + j) * a.ld];
  if (a.warped)
#pragma unroll
    for (int c = 0; c < 3; ++c) a.warped[r * 3 + c] = a.pts[r * 3 + c];
}

// ---------------------------------------------------------------------------
// Jacobian of the warp at the selected rows, the elastic loss and its adjoint.
// ---------------------------------------------------------------------------
struct JacArgs {
  const float* head; int ld;       // primal head outputs (tape rows)
  const float* thead;              // tangent head outputs, row r*3 + j (same ld)
  const float* pts;                // (rows,3) primal points
  const int* sel;                  // selected tape rows or null (identity)
  const float* row_w;              // per selected tape row weight ('weight' reduce) or null
  float* d_head;                   // primal head gradient (+=) or null (forward only)
  float* d_thead;                  // tangent head gradient (=) or null
  float* jac_out;                  // (R,9) or null
  float* stats;                    // += [loss, residual, det, div, |curl|] sums, or null
  float grad_scale;                // elastic_loss_weight / batch rays
  int warp_type, pivot, trans, loss_type, with_loss;
  long long R;
};

// dh[q0 .. q0+3] += sum_ij G_ij d J_ij / d head_q  (second derivatives of the SE(3) tail)
template <int kQ0>
__device__ void se3_second_order(const float* h, const float Th[3][12], const float* x, int nh, bool pivot,
                                 bool trans, const float G[3][3], float* dh) {
  using In = Fwd<3, float>;
  using Out = Fwd<4, In>;
  Out in[12], xs[3], out[3];
  for (int q = 0; q < 12; ++q) {
    in[q] = Num<Out>::c(q < nh ? h[q] : 0.f);
    if (q < nh)
      for (int j = 0; j < 3; ++j) in[q].v.d[j] = Th[j][q];
    if (q >= kQ0 && q < kQ0 + 4 && q < nh) in[q].d[q - kQ0].v = 1.f;
  }
  for (int c = 0; c < 3; ++c) { xs[c] = Num<Out>::c(x[c]); xs[c].v.d[c] = 1.f; }
  se3_tail(in, xs, pivot, trans, out);
  for (int q = kQ0; q < kQ0 + 4 && q < nh; ++q) {
    float acc = 0.f;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) acc += G[i][j] * out[i].d[q - kQ0].d[j];
    dh[q] += acc;
  }
}

__global__ void __launch_bounds__(64) jac_elastic_kernel(const JacArgs a) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= a.R) return;
  const long long row = a.sel ? a.sel[r] : r;
  const int nh = a.warp_type == 2 ? 6 + (a.pivot ? 3 : 0) + (a.trans ? 3 : 0) : 3;
  float h[12], Th[3][12], x[3], J[3][3];
  for (int q = 0; q < 12; ++q) {
    h[q] = q < nh ? a.head[row * a.ld + q] : 0.f;
    for (int j = 0; j < 3; ++j) Th[j][q] = q < nh ? a.thead[(r * 3 + j) * a.ld + q] : 0.f;
  }
  for (int c = 0; c < 3; ++c) x[c] = a.pts[row * 3 + c];
  // J = d warp / d x: forward mode over the point, the head outputs carry their tangents Th
  if (a.warp_type == 2) {
    using S = Fwd<3, float>;
    S in[12], xs[3], out[3];
    for (int q = 0; q < 12; ++q) {
      in[q] = Num<S>::c(h[q]);
      for (int j = 0; j < 3; ++j) in[q].d[j] = Th[j][q];
    }
    for (int c = 0; c < 3; ++c) { xs[c] = Num<S>::c(x[c]); xs[c].d[c] = 1.f; }
    se3_tail(in, xs, a.pivot != 0, a.trans != 0, out);
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) J[i][j] = out[i].d[j];
  } else {
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) J[i][j] = (i == j ? 1.f : 0.f) + Th[j][i];      // warped = x + t(x)
  }
  if (a.jac_out)
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) a.jac_out[r * 9 + i * 3 + j] = J[i][j];
  if (!a.with_loss) return;
  float sq, dJ[3][3], loss, dl;
  elastic_sq(J, a.loss_type, sq, dJ);
  general_loss(sq, -2.0f, 0.03f, loss, dl);                       // training.py:113-114
  const float w = a.row_w ? a.row_w[row] : 1.f;
  if (a.stats) {
    atomicAdd(a.stats + 0, w * loss);
    atomicAdd(a.stats + 1, sqrtf(sq));
    atomicAdd(a.stats + 2, det3(J));
    atomicAdd(a.stats + 3, J[0][0] + J[1][1] + J[2][2] - 3.f);
    const float cx = J[2][1] - J[1][2], cy = J[0][2] - J[2][0], cz = J[1][0] - J[0][1];
    atomicAdd(a.stats + 4, sqrtf(cx * cx + cy * cy + cz * cz));
  }
  if (!a.d_thead) return;
  float G[3][3];
  const float k = a.grad_scale * w * dl;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) G[i][j] = k * dJ[i][j];
  if (a.warp_type != 2) {
    for (int j = 0; j < 3; ++j)
      for (int q = 0; q < 3; ++q) a.d_thead[(r * 3 + j) * a.ld + q] = G[q][j];     // J_qj = delta + Th[j][q]
    return;
  }
  Fwd<12, float> y[3];
  se3_head_jacobian(h, x, nh, a.pivot != 0, a.trans != 0, y);
  // J_ij = sum_q dy_i/dh_q Th[j][q] + dy_i/dx_j  ->  dL/dTh[j][q] = sum_i G_ij dy_i/dh_q
  for (int j = 0; j < 3; ++j)
    for (int q = 0; q < nh; ++q)
      a.d_thead[(r * 3 + j) * a.ld + q] = G[0][j] * y[0].d[q] + G[1][j] * y[1].d[q] + G[2][j] * y[2].d[q];
  float dh[12];
  for (int q = 0; q < 12; ++q) dh[q] = 0.f;
  se3_second_order<0>(h, Th, x, nh, a.pivot != 0, a.trans != 0, G, dh);
  se3_second_order<4>(h, Th, x, nh, a.pivot != 0, a.trans != 0, G, dh);
  if (nh > 8) se3_second_order<8>(h, Th, x, nh, a.pivot != 0, a.trans != 0, G, dh);
  for (int q = 0; q < nh; ++q) a.d_head[row * a.ld + q] += dh[q];
}

// ---------------------------------------------------------------------------
// Robust loss of |warped - x|^2 at selected rows; adjoint added to d(warped).
//   warp-reg (training.py:194-207): one row per ray (the median-depth sample);
//   background (training.py:118-135): every row (free points).
// ---------------------------------------------------------------------------
struct WarpMagArgs {
  const float* pts; const float* warped; const int* sel;
  float* dwarped;                // (rows,3): += at the selected rows, or null
  float* stats;                  // += [loss, sqrt(residual)] sums, or null
  float alpha, scale, grad_scale;
  long long R;
  float* dpts;                   // (rows,3): -= at the selected rows (the loss's direct term in x), or null
};
__global__ void warp_mag_loss_kernel(const WarpMagArgs a) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= a.R) return;
  const long long row = a.sel ? a.sel[r] : r;
  float d[3], sq = 0.f;
  for (int c = 0; c < 3; ++c) { d[c] = a.warped[row * 3 + c] - a.pts[row * 3 + c]; sq += d[c] * d[c]; }
  float loss, dl;
  general_loss(sq, a.alpha, a.scale, loss, dl);
  if (a.stats) {
    atomicAdd(a.stats + 0, loss);
    atomicAdd(a.stats + 1, sqrtf(sq));
  }
  if (a.dwarped)
    for (int c = 0; c < 3; ++c) a.dwarped[row * 3 + c] += a.grad_scale * dl * 2.f * d[c];
  if (a.dpts)
    for (int c = 0; c < 3; ++c) a.dpts[row * 3 + c] -= a.grad_scale * dl * 2.f * d[c];
}

__global__ void add_noise_kernel(const float* __restrict__ p, const float* __restrict__ noise, float* __restrict__ o,
                                 long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) o[i] = p[i] + (noise ? noise[i] : 0.f);
}

// Slots of nfb_train_value_and_grad_reg's loss_out (documented in include/nerfies_b200.h).
// jac_elastic_kernel writes five consecutive slots from kSlotElasticLoss, warp_mag_loss_kernel two.
enum LossSlot {
  kSlotRgbCoarse = 0, kSlotRgbFine = 1,
  kSlotElasticLoss = 2, kSlotElasticResidual = 3, kSlotJacDet = 4, kSlotJacDiv = 5, kSlotJacCurl = 6,
  kSlotWarpRegCoarse = 7, kSlotWarpRegResidualCoarse = 8, kSlotWarpRegFine = 9, kSlotWarpRegResidualFine = 10,
  kSlotBackground = 11, kSlotBackgroundResidual = 12,
  kSlotDepthCoarse = 13, kSlotDepthFine = 14, kSlotDepthCount = 15,
  kLossSlots = 16
};

// sums -> the means the reference reports (training.py:190-193, 201-206, 216-222, 254-257)
__global__ void finalize_stats_kernel(float* st, float inv_rays, float inv_jac_rows, float inv_bg) {
  if (threadIdx.x != 0) return;
  st[kSlotElasticLoss] *= inv_rays;     // sum over the samples, mean over the rays
  st[kSlotElasticResidual] *= inv_jac_rows;
  st[kSlotJacDet] *= inv_jac_rows; st[kSlotJacDiv] *= inv_jac_rows; st[kSlotJacCurl] *= inv_jac_rows;
  st[kSlotWarpRegCoarse] *= inv_rays; st[kSlotWarpRegResidualCoarse] *= inv_rays;
  st[kSlotWarpRegFine] *= inv_rays; st[kSlotWarpRegResidualFine] *= inv_rays;
  st[kSlotBackground] *= inv_bg; st[kSlotBackgroundResidual] *= inv_bg;
}

}  // namespace train
}  // namespace nfb
