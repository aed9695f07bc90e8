"""The training tier's GEMM (sgemm128_kernel through launch_gemm, nfb_selftest_sgemm) against a
float64 product, at the edges of its 128 x 128 tiles, its k-steps of 8 and its split reduction.

The three launches of a Dense layer (train_api.cuh net_forward / net_backward) with their
production element functors:
  forward  y = act([X | IN] W + b)                       ConcatA  x WeightB  -> StoreBiasAct
  dX       dx, din += (dY * act'(Y)) W^T                 DZ       x WeightBT -> AccumSplit
  dW       dw += [X | IN]^T (dY * act'(Y)), split-K      ConcatAT x DZB      -> AtomicAdd

Bound, elementwise: |C - C_ref| <= 2 gamma_{K+1} (|A||B| + |C_0|)_ij with gamma_k = k u / (1 - k u),
u = 2^-24, K the reduction length and C_0 the bias or the pre-filled output.  It holds for any
split of the reduction and any order of the atomic additions; a missing, doubled or misplaced
term breaks it by orders of magnitude.
"""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
FORWARD, DX, DW = 0, 1, 2
RELU, NONE = 1, 0
U = 2.0**-24


def _gamma(k):
  return k * U / (1 - k * U)


def _ptr(t):
  return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _call(mode, rows, n, k_x, k_in, act, x, ldx, inp, ldin, w, ldw, bias, y, dy, dx, din, dw, k_split=0):
  from nerfies_b200 import _lib
  lib = _lib.load()
  used = ctypes.c_longlong(-1)
  _lib.check(lib.nfb_selftest_sgemm(mode, rows, n, k_x, k_in, act, _ptr(x), ldx, _ptr(inp), ldin, _ptr(w), ldw,
                                    _ptr(bias), _ptr(y), _ptr(dy), _ptr(dx), _ptr(din), _ptr(dw), k_split,
                                    ctypes.byref(used), None))
  torch.cuda.synchronize()
  return used.value


def _layer(rows, n, k_x, k_in, seed, in_off=5):
  """Operands in the tape's layout: X (rows, ldx), IN a column block at `in_off` of a wider
  input (the skip layers read the encoded input that way), W (K, ldw) with ldw = pad32(n)."""
  g = torch.Generator().manual_seed(seed)
  ldx, ldin, ldw = k_x + 3, in_off + k_in + 2, (n + 31) // 32 * 32
  x = torch.randn(rows, ldx, generator=g)
  full_in = torch.randn(rows, ldin, generator=g)
  w = torch.randn(k_x + k_in, ldw, generator=g) / (k_x + k_in) ** 0.5
  b = torch.randn(ldw, generator=g) * 0.1
  # Y of a relu layer: about half of the entries exact zeros (the mask of act')
  y = torch.relu(torch.randn(rows, ldw, generator=g))
  dy = torch.randn(rows, ldw, generator=g)
  a = torch.cat([x[:, :k_x], full_in[:, in_off:in_off + k_in]], 1).double()
  return dict(ldx=ldx, ldin=ldin, ldw=ldw, x=x, full_in=full_in, w=w, b=b, y=y, dy=dy, a=a, in_off=in_off)


def _check(got, ref, bound, what):
  got = got.cpu().double()
  err = (got - ref).abs()
  ok = err <= bound                         # NaN (an entry never written) fails
  if not bool(ok.all()):
    i = int((~ok).flatten().nonzero()[0])
    r, c = divmod(i, ref.shape[1])
    pytest.fail(f'{what}: {int((~ok).sum())} of {ok.numel()} entries outside the bound; first ({r}, {c}): '
                f'got {float(got[r, c]):.6e}, ref {float(ref[r, c]):.6e}, bound {float(bound[r, c]):.3e}')


# (rows, n, k_x, k_in, act) - GEMM M = rows, N = n, K = k_x + k_in
@pytest.mark.parametrize('rows,n,k_x,k_in,act', [
    (1, 1, 0, 1, RELU),           # M = N = K = 1
    (127, 3, 0, 7, NONE),         # K = 7 < one k-step, the rgb head's N = 3
    (128, 128, 8, 0, RELU),       # exactly one tile, one k-step
    (129, 129, 9, 0, NONE),       # one past the tile in M and N, one past the k-step
    (4097, 256, 256, 51, RELU),   # the NeRF skip layer: 256 | 51 split, second tile across N
    (300, 307, 0, 51, RELU),      # N = 307: three tiles across, the first layer's K = 51
])
def test_forward(rows, n, k_x, k_in, act):
  L = _layer(rows, n, k_x, k_in, seed=rows + 7 * n + k_x)
  K = k_x + k_in
  y = torch.full((rows, L['ldw']), float('nan'))
  yd = y.to(DEV)
  # IN is passed with its column offset folded into the pointer, as net_forward does
  full = L['full_in'].to(DEV)
  inp = full[:, L['in_off']:] if k_in else None
  _call(FORWARD, rows, n, k_x, k_in, act, L['x'].to(DEV) if k_x else None, L['ldx'], inp, L['ldin'],
        L['w'].to(DEV), L['ldw'], L['b'].to(DEV), yd, None, None, None, None)
  w = L['w'][:, :n].double()
  z = L['a'] @ w + L['b'][:n].double()
  ref = torch.relu(z) if act == RELU else z
  bound = 2 * _gamma(K + 1) * (L['a'].abs() @ w.abs() + L['b'][:n].double().abs())
  _check(yd[:, :n], ref, bound, f'forward rows={rows} n={n} K={k_x}|{k_in}')
  # the padding columns of the output are not written
  assert bool(torch.isnan(yd[:, n:]).all())
  if act == RELU and rows * n > 100:
    assert bool((yd[:, :n] == 0).any())


# (rows, n, k_x, k_in) - GEMM M = rows, N = k_x + k_in, K = n
@pytest.mark.parametrize('rows,n,k_x,k_in', [
    (1, 1, 0, 1),                 # M = N = K = 1
    (129, 7, 3, 0),               # N = 3, K = 7
    (300, 8, 120, 8),             # N = 128 split 120 | 8, K = 8
    (128, 9, 128, 1),             # N = 129 split 128 | 1, K = 9
    (127, 51, 0, 256),            # N = 256 all IN, K = 51
    (4097, 256, 256, 51),         # the skip layer's dX: N = 307 split 256 | 51, K = 256
])
def test_dx_accumulates_into_both_blocks(rows, n, k_x, k_in):
  L = _layer(rows, n, k_x, k_in, seed=3 * rows + n + k_in)
  g = torch.Generator().manual_seed(rows + n)
  dx0 = torch.randn(rows, L['ldx'], generator=g)
  din0 = torch.randn(rows, L['ldin'], generator=g)
  dxd, dind = dx0.to(DEV), din0.to(DEV)
  _call(DX, rows, n, k_x, k_in, RELU, None, L['ldx'], None, L['ldin'], L['w'].to(DEV), L['ldw'], None,
        L['y'].to(DEV), L['dy'].to(DEV), dxd if k_x else None, dind[:, L['in_off']:] if k_in else None, None)
  dz = (L['dy'][:, :n] * (L['y'][:, :n] > 0)).double()
  wt = L['w'][:, :n].double().t()
  prod, bprod = dz @ wt, dz.abs() @ wt.abs()
  pre = torch.cat([dx0[:, :k_x], din0[:, L['in_off']:L['in_off'] + k_in]], 1).double()
  ref = pre + prod
  bound = 2 * _gamma(n + 1) * (bprod + pre.abs())
  got = torch.cat([dxd[:, :k_x], dind[:, L['in_off']:L['in_off'] + k_in]], 1)
  _check(got, ref, bound, f'dX rows={rows} n={n} K={k_x}|{k_in}')
  # columns outside the two blocks keep their contents
  assert torch.equal(dxd[:, k_x:].cpu(), dx0[:, k_x:])
  assert torch.equal(dind[:, :L['in_off']].cpu(), din0[:, :L['in_off']])
  assert torch.equal(dind[:, L['in_off'] + k_in:].cpu(), din0[:, L['in_off'] + k_in:])


# (rows, n, k_x, k_in, k_split) - GEMM M = k_x + k_in, N = n, K = rows; k_split 0 = dw_split's choice,
# -1 = K - 1 (a slice length that is not a multiple of 8 and a last slice of one row)
@pytest.mark.parametrize('rows,n,k_x,k_in,k_split', [
    (1, 1, 0, 1, 0),              # M = N = K = 1
    (9, 3, 0, 127, 8),            # M = 127, K = 9 in slices of 8: a last slice of one row
    (51, 129, 128, 0, 0),         # M = 128, N = 129, K = 51 (dw_split: one slice)
    (7, 128, 128, 1, 0),          # M = 129, K = 7
    (129, 256, 256, 51, 8),       # 17 slices of one k-step each, the last ragged
    (307, 256, 256, 51, -1),      # slices of 306 rows
    (4097, 256, 256, 51, 256),    # 17 slices, the last of one row
    (4097, 307, 256, 51, 0),      # dw_split's choice at the skip layer's shape (several slices)
    (5120, 128, 128, 59, 0),      # a warp-trunk chunk of 40 rays x 128 samples
])
def test_dw_split_reduction(rows, n, k_x, k_in, k_split):
  L = _layer(rows, n, k_x, k_in, seed=5 * rows + n + k_x)
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
    assert used >= 256 and used % 8 == 0
  if rows >= 4097:
    assert (rows + used - 1) // used > 1, 'the shape is meant to split the reduction'
  dz = (L['dy'][:, :n] * (L['y'][:, :n] > 0)).double()
  a = L['a']
  ref = dw0[:, :n].double() + a.t() @ dz
  bound = 2 * _gamma(rows + 1) * (a.t().abs() @ dz.abs() + dw0[:, :n].double().abs())
  _check(dwd[:, :n], ref, bound, f'dW rows={rows} n={n} K={k_x}|{k_in} k_split={used}')
  assert torch.equal(dwd[:, n:].cpu(), dw0[:, n:])


def test_rejects_bad_arguments():
  from nerfies_b200 import _lib
  lib = _lib.load()
  t = torch.zeros(64, device=DEV)
  p = _ptr(t)
  assert lib.nfb_selftest_sgemm(FORWARD, 4, 4, 4, 0, RELU, p, 4, None, 0, p, 4, p, p, None, None, None, None, 8,
                                None, None) != 0
  assert b'dW only' in lib.nfb_last_error()
  assert lib.nfb_selftest_sgemm(DW, 4, 4, 4, 0, RELU, p, 2, None, 0, p, 4, None, p, p, None, None, p, 0,
                                None, None) != 0
  assert b'leading dimension' in lib.nfb_last_error()
  assert lib.nfb_selftest_sgemm(3, 4, 4, 4, 0, RELU, p, 4, None, 0, p, 4, p, p, p, p, None, p, 0, None, None) != 0
  assert b'bad mode' in lib.nfb_last_error()
