// Inverse of the warp field at free points (nfb_warp_invert): the per-point update of a damped Newton
// solve of W(x) = y.  W and J come from the tape kernels (warp_points_forward, warp_jacobian_on_tape);
// this file holds only the update, one thread per point, in fp64 from their fp32 values.
#pragma once
#include <cuda_runtime.h>

#include "../../include/nerfies_b200.h"

namespace nfb {
namespace train {

// A step scale below this freezes the point as NFB_INVERT_STALLED (ten halvings of the Newton step).
constexpr double kInvertMinStep = 1.0 / 1024.0;
// A pivot at most this fraction of J's largest entry counts as zero: fp32 J carries ~6e-8 relative error
// per entry, so a smaller pivot is not told apart from a rank-deficient J.
constexpr double kInvertPivotTol = 1.0 / (1 << 20);

// Per-point state of one chunk: max_rays rows in the handle's workspace (see invert_state).
struct InvertState {
  double* dx;       // (n,3) Newton step from the best iterate
  double* rb;       // (n) residual of the best iterate (meaningless before the first iteration)
  float* cand;      // (n,3) the points the next forward pass evaluates
  float* jac;       // (n,9) J at the candidates (warp_jacobian_on_tape writes it)
  float* xb;        // (n,3) best iterate
  float* jb;        // (n,9) J at the best iterate
  float* lam;       // (n) step scale
  int* status;      // (n) NFB_INVERT_*; NFB_INVERT_MAX_ITERS while the point iterates
};

struct InvertStepArgs {
  InvertState st;
  const float* warped;   // (n,3) W at the candidates (tape.warped)
  const float* target;   // (n,3)
  double tol;
  int first, last;       // the chunk's first / last iteration
  float* points_out; float* residual_out; float* jacobian_out; int* status_out;   // written on `last`
  long long n;
};

// Solves A x = b in place (3x3 LU with partial pivoting); false when A is singular or not finite.
__device__ __forceinline__ bool lu_solve3(double A[3][3], double b[3]) {
  double scale = 0.0;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      if (!isfinite(A[i][j])) return false;
      scale = fmax(scale, fabs(A[i][j]));
    }
  if (!(scale > 0.0)) return false;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    // the pivot row, then a swap written as selects so that the arrays stay in registers
    int m = k;
    double best = fabs(A[k][k]);
#pragma unroll
    for (int r = k + 1; r < 3; ++r)
      if (fabs(A[r][k]) > best) { best = fabs(A[r][k]); m = r; }
#pragma unroll
    for (int r = k + 1; r < 3; ++r) {
      const bool sw = r == m;
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const double t = A[k][j];
        A[k][j] = sw ? A[r][j] : t;
        A[r][j] = sw ? t : A[r][j];
      }
      const double t = b[k];
      b[k] = sw ? b[r] : t;
      b[r] = sw ? t : b[r];
    }
    if (fabs(A[k][k]) <= kInvertPivotTol * scale) return false;
#pragma unroll
    for (int r = k + 1; r < 3; ++r) {
      const double f = A[r][k] / A[k][k];
#pragma unroll
      for (int j = k + 1; j < 3; ++j) A[r][j] -= f * A[k][j];
      b[r] -= f * b[k];
    }
  }
#pragma unroll
  for (int k = 2; k >= 0; --k) {
    double v = b[k];
#pragma unroll
    for (int j = k + 1; j < 3; ++j) v -= A[k][j] * b[j];
    b[k] = v / A[k][k];
  }
  return isfinite(b[0]) && isfinite(b[1]) && isfinite(b[2]);
}

// One iteration for every point of the chunk, after the forward pass and the Jacobian at the candidates.
//   accept a candidate whose residual is finite and below the best: converged at <= tol, else the Newton
//   step from it (singular J: frozen); otherwise halve the step from the best iterate (stalled below
//   kInvertMinStep).  A first candidate whose residual is not finite is frozen as NFB_INVERT_NONFINITE.
// A frozen point keeps its state; on the last iteration every point writes its outputs.
__global__ void __launch_bounds__(128) warp_invert_step_kernel(const InvertStepArgs a) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  const InvertState& s = a.st;
  int status = a.first ? NFB_INVERT_MAX_ITERS : s.status[i];
  if (status == NFB_INVERT_MAX_ITERS) {
    double res[3], r2 = 0.0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      res[c] = (double)a.target[i * 3 + c] - (double)a.warped[i * 3 + c];
      r2 += res[c] * res[c];
    }
    const double r = sqrt(r2);
    const bool better = isfinite(r) && (a.first || r < s.rb[i]);
    if (better || a.first) {
      // the candidate becomes the best iterate
#pragma unroll
      for (int c = 0; c < 3; ++c) s.xb[i * 3 + c] = s.cand[i * 3 + c];
#pragma unroll
      for (int q = 0; q < 9; ++q) s.jb[i * 9 + q] = s.jac[i * 9 + q];
      s.rb[i] = r;
    }
    if (!better) {
      if (a.first) {
        status = NFB_INVERT_NONFINITE;
      } else {
        const float lam = 0.5f * s.lam[i];
        s.lam[i] = lam;
        if ((double)lam < kInvertMinStep) {
          status = NFB_INVERT_STALLED;
        } else {
#pragma unroll
          for (int c = 0; c < 3; ++c)
            s.cand[i * 3 + c] = (float)((double)s.xb[i * 3 + c] + (double)lam * s.dx[i * 3 + c]);
        }
      }
    } else if (r <= a.tol) {
      status = NFB_INVERT_CONVERGED;
    } else {
      double A[3][3];
#pragma unroll
      for (int p = 0; p < 3; ++p)
#pragma unroll
        for (int q = 0; q < 3; ++q) A[p][q] = (double)s.jac[i * 9 + p * 3 + q];
      if (!lu_solve3(A, res)) {
        status = NFB_INVERT_SINGULAR;
      } else {
        s.lam[i] = 1.f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          s.dx[i * 3 + c] = res[c];
          s.cand[i * 3 + c] = (float)((double)s.cand[i * 3 + c] + res[c]);
        }
      }
    }
    s.status[i] = status;
  }
  if (!a.last) return;
#pragma unroll
  for (int c = 0; c < 3; ++c) a.points_out[i * 3 + c] = s.xb[i * 3 + c];
  a.residual_out[i] = (float)s.rb[i];
  if (a.jacobian_out)
#pragma unroll
    for (int q = 0; q < 9; ++q) a.jacobian_out[i * 9 + q] = s.jb[i * 9 + q];
  if (a.status_out) a.status_out[i] = status;
}

}  // namespace train
}  // namespace nfb
