"""The training GEMM in tf32x3 mode (tf32x3_gemm_kernel through launch_gemm, nfb_selftest_train_gemm)
against a float64 product, at the edges test_train_gemm_gpu.py checks the fp32 kernel at, plus the
k-block tails of the 32-wide tf32x3 staging and a dynamic-range case.

Bound, elementwise: |C - C_ref| <= c (|A||B| + |C_0|)_ij with
  c = 3.01 * 2^-22 + 1.01 * gamma_{3K+S+1},  gamma_n = n u / (1 - n u),  u = 2^-23,
K the reduction length, S the number of slices it is split into (1 for forward and dX) and C_0 the bias
or the pre-filled output.  Derivation: each operand value a is big + small + r with big = tf32(a),
small = tf32(a - big); tf32 keeps 11 significant bits, so |small| <= 2^-11 |a| and |r| <= 2^-11 |small|
<= 2^-22 |a|.  The kernel forms a_big b_big + a_big b_small + a_small b_big, which differs from a b by
a_small b_small + a_big r_b + r_a (b_big + b_small) + r_a r_b: at most 3.01 * 2^-22 |a||b|.  Every
tf32 x tf32 product is exact in fp32 (22 significant bits); the 3K products, C_0 and the S - 1 slice
partials are summed in fp32 (per k-block on the tensor cores, then across k-blocks, slices and C_0 with
fp32 adds), n terms in any order within gamma_{n-1} of their absolute sum, which is at most
1.01 (|A||B| + |C_0|).  u = 2^-23 rather than 2^-24 because the tensor cores' accumulation is not
specified as round-to-nearest.  A missing, doubled or misplaced term breaks the bound by orders of
magnitude; so does a scaled operand split, which the dynamic-range case (dZ rows at 1e-20 and 1e+20,
weights around 1e-4, where fp16 hi/lo halves underflow or overflow) would show.

The worst measured fraction of the bound per case goes to train_tf32x3_gemm_report.json in
NFB_REPORT_DIR (default: the system's temporary directory).
"""
import ctypes
import json
import os
import tempfile

import pytest
import torch

from tests.test_train_gemm_gpu import _layer, _ptr

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
FORWARD, DX, DW = 0, 1, 2
RELU, NONE = 1, 0
TF32X3 = 1
U = 2.0**-23
_REPORT = {}


@pytest.fixture(scope='module', autouse=True)
def _write_report():
  yield
  out_dir = os.environ.get('NFB_REPORT_DIR') or tempfile.gettempdir()
  os.makedirs(out_dir, exist_ok=True)
  with open(os.path.join(out_dir, 'train_tf32x3_gemm_report.json'), 'w') as f:
    json.dump(dict(worst_fraction_of_bound=max(_REPORT.values(), default=0.0), cases=_REPORT), f, indent=1)


def _c(K, S=1):
  n = 3 * K + S + 1
  return 3.01 * 2.0**-22 + 1.01 * n * U / (1 - n * U)


def _call(mode, rows, n, k_x, k_in, act, x, ldx, inp, ldin, w, ldw, bias, y, dy, dx, din, dw, k_split=0):
  from nerfies_b200 import _lib
  lib = _lib.load()
  used = ctypes.c_longlong(-1)
  _lib.check(lib.nfb_selftest_train_gemm(TF32X3, mode, rows, n, k_x, k_in, act, _ptr(x), ldx, _ptr(inp), ldin,
                                         _ptr(w), ldw, _ptr(bias), _ptr(y), _ptr(dy), _ptr(dx), _ptr(din),
                                         _ptr(dw), k_split, ctypes.byref(used), None))
  torch.cuda.synchronize()
  return used.value


def _check(got, ref, bound, what):
  got = got.cpu().double()
  err = (got - ref).abs()
  ok = err <= bound                         # NaN (an entry never written) fails
  if not bool(ok.all()):
    i = int((~ok).flatten().nonzero()[0])
    r, c = divmod(i, ref.shape[1])
    pytest.fail(f'{what}: {int((~ok).sum())} of {ok.numel()} entries outside the bound; first ({r}, {c}): '
                f'got {float(got[r, c]):.6e}, ref {float(ref[r, c]):.6e}, bound {float(bound[r, c]):.3e}')
  _REPORT[what] = float((err / bound.clamp_min(1e-300)).max())


# (rows, n, k_x, k_in, act) - GEMM M = rows, N = n, K = k_x + k_in
@pytest.mark.parametrize('rows,n,k_x,k_in,act', [
    (1, 1, 0, 1, RELU),           # M = N = K = 1
    (127, 3, 0, 7, NONE),         # K = 7 < one k8 step, the rgb head's N = 3
    (128, 128, 8, 0, RELU),       # exactly one tile, one k8 step
    (129, 129, 9, 0, NONE),       # one past the tile in M and N
    (4097, 256, 256, 51, RELU),   # the NeRF skip layer: 256 | 51 split, second tile across N
    (300, 307, 0, 51, RELU),      # N = 307: three tiles across, the first layer's K = 51
    (200, 64, 33, 0, RELU),       # K = 33: one k-block and a tail of one
    (200, 64, 0, 63, NONE),       # K = 63: one k-block and a tail of 31
])
def test_forward(rows, n, k_x, k_in, act):
  L = _layer(rows, n, k_x, k_in, seed=rows + 7 * n + k_x)
  K = k_x + k_in
  yd = torch.full((rows, L['ldw']), float('nan'), device=DEV)
  full = L['full_in'].to(DEV)
  inp = full[:, L['in_off']:] if k_in else None
  _call(FORWARD, rows, n, k_x, k_in, act, L['x'].to(DEV) if k_x else None, L['ldx'], inp, L['ldin'],
        L['w'].to(DEV), L['ldw'], L['b'].to(DEV), yd, None, None, None, None)
  w = L['w'][:, :n].double()
  z = L['a'] @ w + L['b'][:n].double()
  ref = torch.relu(z) if act == RELU else z
  bound = _c(K) * (L['a'].abs() @ w.abs() + L['b'][:n].double().abs())
  _check(yd[:, :n], ref, bound, f'forward rows={rows} n={n} K={k_x}|{k_in}')
  assert bool(torch.isnan(yd[:, n:]).all())
  if act == RELU and rows * n > 100:
    assert bool((yd[:, :n] == 0).any())


def _dx_case(rows, n, k_x, k_in, row_scale=None, w_scale=None):
  L = _layer(rows, n, k_x, k_in, seed=3 * rows + n + k_in)
  if w_scale is not None:
    L['w'] = L['w'] * w_scale
  if row_scale is not None:
    L['dy'] = L['dy'] * row_scale[:, None]
  g = torch.Generator().manual_seed(rows + n)
  dx0 = torch.randn(rows, L['ldx'], generator=g)
  din0 = torch.randn(rows, L['ldin'], generator=g)
  if row_scale is not None:
    dx0, din0 = dx0 * row_scale[:, None] * 1e-3, din0 * row_scale[:, None] * 1e-3
  dxd, dind = dx0.to(DEV), din0.to(DEV)
  _call(DX, rows, n, k_x, k_in, RELU, None, L['ldx'], None, L['ldin'], L['w'].to(DEV), L['ldw'], None,
        L['y'].to(DEV), L['dy'].to(DEV), dxd if k_x else None, dind[:, L['in_off']:] if k_in else None, None)
  dz = (L['dy'][:, :n] * (L['y'][:, :n] > 0)).double()
  wt = L['w'][:, :n].double().t()
  pre = torch.cat([dx0[:, :k_x], din0[:, L['in_off']:L['in_off'] + k_in]], 1).double()
  ref = pre + dz @ wt
  bound = _c(n) * (dz.abs() @ wt.abs() + pre.abs())
  got = torch.cat([dxd[:, :k_x], dind[:, L['in_off']:L['in_off'] + k_in]], 1)
  tag = ' dynamic range' if row_scale is not None else ''
  _check(got, ref, bound, f'dX rows={rows} n={n} K={k_x}|{k_in}{tag}')
  assert torch.equal(dxd[:, k_x:].cpu(), dx0[:, k_x:])
  assert torch.equal(dind[:, :L['in_off']].cpu(), din0[:, :L['in_off']])
  assert torch.equal(dind[:, L['in_off'] + k_in:].cpu(), din0[:, L['in_off'] + k_in:])


# (rows, n, k_x, k_in) - GEMM M = rows, N = k_x + k_in, K = n
@pytest.mark.parametrize('rows,n,k_x,k_in', [
    (1, 1, 0, 1),                 # M = N = K = 1
    (129, 7, 3, 0),               # N = 3, K = 7
    (300, 8, 120, 8),             # N = 128 split 120 | 8, K = 8
    (128, 9, 128, 1),             # N = 129 split 128 | 1, K = 9
    (127, 51, 0, 256),            # N = 256 all IN, K = 51
    (4097, 256, 256, 51),         # the skip layer's dX: N = 307 split 256 | 51, K = 256
    (300, 33, 64, 0),             # K = 33: a k-block tail of one
    (300, 63, 0, 64),             # K = 63: a k-block tail of 31
])
def test_dx_accumulates_into_both_blocks(rows, n, k_x, k_in):
  _dx_case(rows, n, k_x, k_in)


def _dw_case(rows, n, k_x, k_in, k_split, row_scale=None, w_scale=None):
  L = _layer(rows, n, k_x, k_in, seed=5 * rows + n + k_x)
  if row_scale is not None:
    L['dy'] = L['dy'] * row_scale[:, None]
  K = k_x + k_in
  g = torch.Generator().manual_seed(rows * 3 + n)
  dw0 = torch.randn(K, L['ldw'], generator=g)
  dwd = dw0.to(DEV)
  full = L['full_in'].to(DEV)
  split = rows - 1 if k_split < 0 else k_split
  used = _call(DW, rows, n, k_x, k_in, RELU, L['x'].to(DEV) if k_x else None, L['ldx'],
               full[:, L['in_off']:] if k_in else None, L['ldin'], L['w'].to(DEV), L['ldw'], None,
               L['y'].to(DEV), L['dy'].to(DEV), None, None, dwd, k_split=split)
  if split > 0:
    assert used == split
  else:
    assert used >= 256 and used % 32 == 0          # whole k-blocks of 32 rows
  S = (rows + used - 1) // used
  if rows >= 4097:
    assert S > 1, 'the shape is meant to split the reduction'
  dz = (L['dy'][:, :n] * (L['y'][:, :n] > 0)).double()
  a = L['a']
  ref = dw0[:, :n].double() + a.t() @ dz
  bound = _c(rows, S) * (a.t().abs() @ dz.abs() + dw0[:, :n].double().abs())
  tag = ' dynamic range' if row_scale is not None else ''
  _check(dwd[:, :n], ref, bound, f'dW rows={rows} n={n} K={k_x}|{k_in} k_split={used}{tag}')
  assert torch.equal(dwd[:, n:].cpu(), dw0[:, n:])


# (rows, n, k_x, k_in, k_split) - GEMM M = k_x + k_in, N = n, K = rows; k_split 0 = the tf32x3 split's choice,
# -1 = K - 1 (a slice length that is not a multiple of 32 and a last slice of one row)
@pytest.mark.parametrize('rows,n,k_x,k_in,k_split', [
    (1, 1, 0, 1, 0),              # M = N = K = 1
    (9, 3, 0, 127, 8),            # M = 127, K = 9 in slices of 8: a last slice of one row
    (51, 129, 128, 0, 0),         # M = 128, N = 129, K = 51 (one slice)
    (7, 128, 128, 1, 0),          # M = 129, K = 7
    (129, 256, 256, 51, 8),       # 17 slices of 8 rows each, the last ragged
    (307, 256, 256, 51, -1),      # slices of 306 rows
    (4097, 256, 256, 51, 256),    # 17 slices, the last of one row
    (4097, 307, 256, 51, 0),      # the tf32x3 split's choice at the skip layer's shape (several slices)
    (5120, 128, 128, 59, 0),      # a warp-trunk chunk of 40 rays x 128 samples
    (33, 64, 64, 0, 0),           # K = 33: a k-block tail of one
    (63, 64, 0, 64, 0),           # K = 63: a k-block tail of 31
])
def test_dw_split_reduction(rows, n, k_x, k_in, k_split):
  _dw_case(rows, n, k_x, k_in, k_split)


def _scales(rows):
  """dZ rows alternately at 1e-20 and 1e+20 (fp16's range is 6e-8 .. 6.5e4)."""
  return torch.where(torch.arange(rows) % 2 == 0, torch.tensor(1e-20), torch.tensor(1e20))


def test_dynamic_range_dx():
  _dx_case(300, 256, 256, 51, row_scale=_scales(300), w_scale=1e-4 * 256 ** 0.5)   # W ~ N(0, 1e-4^2)


def test_dynamic_range_dw():
  _dw_case(4097, 256, 256, 51, 0, row_scale=_scales(4097))


def test_dynamic_range_forward_weights():
  """Weights around 1e-4 (the warp heads' scale) on the forward."""
  rows, n, k_x, k_in = 500, 256, 256, 51
  L = _layer(rows, n, k_x, k_in, seed=11)
  L['w'] = L['w'] * 1e-4 * (k_x + k_in) ** 0.5
  yd = torch.full((rows, L['ldw']), float('nan'), device=DEV)
  full = L['full_in'].to(DEV)
  _call(FORWARD, rows, n, k_x, k_in, NONE, L['x'].to(DEV), L['ldx'], full[:, L['in_off']:], L['ldin'],
        L['w'].to(DEV), L['ldw'], L['b'].to(DEV) * 1e-4, yd, None, None, None, None)
  w = L['w'][:, :n].double()
  b = (L['b'][:n] * 1e-4).double()
  ref = L['a'] @ w + b
  _check(yd[:, :n], ref, _c(k_x + k_in) * (L['a'].abs() @ w.abs() + b.abs()), 'forward weights ~1e-4')


def test_rejects_bad_arguments():
  from nerfies_b200 import _lib
  lib = _lib.load()
  t = torch.zeros(64, device=DEV)
  p = _ptr(t)
  assert lib.nfb_selftest_train_gemm(TF32X3, FORWARD, 4, 4, 4, 0, RELU, p, 4, None, 0, p, 4, p, p, None, None,
                                     None, None, 8, None, None) != 0
  assert b'dW only' in lib.nfb_last_error()
  assert lib.nfb_selftest_train_gemm(TF32X3, 3, 4, 4, 4, 0, RELU, p, 4, None, 0, p, 4, p, p, p, p, None, p, 0,
                                     None, None) != 0
  assert b'bad mode' in lib.nfb_last_error()
