"""The training step's seed and regulariser kernels, and the adjoints between its MLPs and the rays and tables, on
their own, through their self-test entry points (nfb_selftest_composite_vjp, nfb_selftest_elastic,
nfb_selftest_depth_index, nfb_selftest_warp_mag_loss, nfb_selftest_encode_bwd, nfb_selftest_warp_tail_bwd,
nfb_selftest_ray_reduce, nfb_selftest_viewdir_vjp, nfb_selftest_cond_vjp),
against torch.autograd of the oracle's own functions in float64, element by element.

Each entry launches the production kernel with the production launch configuration and argument struct, so
the inputs can be designed: opaque walls, exact identities, rank-deficient Jacobians, crossings at lane and
chunk boundaries.  u = 2^-24.  Every bound is per element; none is relative to a tensor's maximum.

Composite adjoint (composite_vjp_kernel, the adjoint of O.volumetric_rendering on sigmoid(rgb_raw) and
act(alpha_raw)):
    |got - ref| <= 4 S u M + 3 band + floor
  * M is the same fp64 adjoint computed on absolute values: every cotangent term of d/dw_i by its magnitude,
    the transmittance T and the weights w as they are, the suffix sum sum_{k>i} |gw_k| w_k, and the activation
    derivatives that are formed from the output (1 - y^2, y (1 - y), y + 1) with their subtractions turned
    into additions.  One rounding per term per sample of the two scans gives S u; 4 covers the two roundings of
    each transmittance factor and those of the chain rule.
  * band is the conditioning of alpha when it is formed from fp32 sigma * dist: fp64 rerun with sigma * dist
    moved by 6 roundings (sigma, dist, |d| and their product) and alpha rounded to fp32 (1 - alpha is exact
    in fp32 only to 2^-25 absolute, which is 100 % behind a factor of 1e-7), and with each sigmoid(rgb_raw)
    moved by one rounding; the largest difference over two seeds (the `_moved` of test_render_vjp_gpu.py on
    these inputs).
  * floor covers fp32 underflow: S 2^-126 times the ray's cotangents, divided by the factor 1 - alpha + eps
    when the suffix sum is, so that transmittances that are subnormal or 0 in fp32 (several opaque samples in
    a row) are held to what fp32 can represent.
SVD and elastic gradients (svd3, elastic_sq, jac_elastic_kernel): max(floor, 3 x the fp64 band under
one-rounding moves of J), the floor derived per loss type from the fp32 rounding of s - 1, log s, det - 1 or
J J^T - I (_elastic_floor).  The band covers the conditioning of small singular values.  Each case also checks
that its bound constrains: at most 2^-6 of the point's largest gradient entry, or 4 x the point's fp32 floor
where the gradient itself is at that rounding.  For 'det' and 'log_det' the reference is dL/d det x cof(J)
(torch's det backward is 0 at an exactly singular J).  For rank-deficient J under 'svals' only the range-space
part of dJ is pinned, with the band taken on projected gradients (the kernel's choice for a vanishing singular
value is tested on its own: see test_svals_null_space).
SE(3) second order: the same with the band the larger of the one-rounding moves of (head, Th, x) and the fp32
oracle's distance from fp64 (theta - sin(theta) cancels at small theta in any fp32 evaluation), plus
(2^-16 + 8 u / theta^2) x the contraction of d_head and d_thead on absolute values (max_ij |dL/dJ_ij|
sum_ij |dJ_ij/dh_q|): 256 u for the rounding of the nested fp32 forward-mode tail, a few hundred operations
deep, and dL/dJ's own normwise 2^-20; 8 u / theta^2 for theta - sin(theta) and 1 - cos(theta), which fp32
keeps to u theta absolute against theta^3 / 6 and theta^2 / 2.  At theta = 1e-3 that term is about half of
d_head's own magnitude, so there only J and d_thead are pinned.
Median index: exact on dyadic weights (every summation order gives the same sums); on random weights a
disagreement only where the fp64 cumulative weight at either index lies within S u of 0.5.
Robust loss: the derivative to 32 u relative; the loss to max(16 u |ref|, 3 x the fp32 oracle's distance
from fp64) (the formula itself cancels at tiny residuals).
The adjoints between the MLPs and the rays / tables (nfb_selftest_encode_bwd, _warp_tail_bwd, _ray_reduce,
_viewdir_vjp, _cond_vjp): sums of n fp32 terms within gamma_{n + k} of their absolute sum, k the roundings each
term carries (a product, cosf's 2 ulp, the += onto a prefill); the encodings' adjoints against the fp64 derivative
at the fp32 angle the reference itself forms (2^f x exact, 2^f x + fl32(pi/2) rounded); the SE(3) tail's first
derivatives as its second derivatives above.  Each test states its bound.
Each case prints its worst error as a fraction of its bound.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import nerfies_oracle as O

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
U = 2.0**-24
TINY = 2.0**-126
ACT = {'relu': 1, 'elu': 2, 'leaky_relu': 3, 'tanh': 4, 'sigmoid': 5, 'softplus': 6}
NEGATIVE_SIGMA = ('elu', 'leaky_relu', 'tanh')
ELASTIC = {'log_svals': 0, 'svals': 1, 'jtj': 2, 'div': 3, 'det': 4, 'log_det': 5}


def _lib():
  from nerfies_b200 import _lib as L
  return L


def _ptr(t):
  return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _report(name, ratio):
  print(f'{name}: worst error / bound {ratio:.3g}')
  assert ratio <= 1.0, f'{name}: worst error / bound {ratio:.3g}'


def _ratio(got, ref, tol):
  err = (got.double() - ref).abs()
  assert not torch.isnan(got).any(), 'NaN in the kernel output'
  return float((err / tol.clamp_min(1e-300)).max()) if err.numel() else 0.0


# ---------------------------------------------------------------------------
# 1. composite_vjp_kernel
# ---------------------------------------------------------------------------
def _wall_raw(x, dist, act):
  """The raw density that makes sigma * dist = x (at least x) for the activation."""
  sigma = x / dist
  if act == 'softplus':
    return sigma + torch.log(-torch.expm1(-sigma))
  return sigma                                  # relu / elu / leaky_relu (sigmoid, tanh saturate at 1)


def _composite_inputs(R, S, regime, act, seed, inf):
  """(rgb_raw (R,S,3), alpha_raw (R,S), z (R,S), directions (R,3)), fp32 on the host."""
  g = torch.Generator().manual_seed(seed)
  z = torch.sort(0.02 + 0.81 * torch.rand(R, S, generator=g), -1).values
  dirs = torch.randn(R, 3, generator=g)
  rgb_raw = 2.0 * torch.randn(R, S, 3, generator=g)
  half = 4.0 + torch.randn(R, S, generator=g)
  dn = dirs.double().norm(dim=-1, keepdim=True)
  dist = torch.cat([z[:, 1:] - z[:, :-1], torch.full((R, 1), 1.0)], -1).double() * dn
  if regime == 'empty':
    raw = {'softplus': -30.0, 'sigmoid': -30.0, 'relu': -1.0}.get(act, -1e-20) * torch.ones(R, S)
    if act == 'relu':
      raw[:, ::3] = 0.0                         # relu at raw = 0 exactly: act' = 0
  elif regime in ('half', 'dup_z'):
    raw = half
    if regime == 'dup_z':
      # tied z (dist = 0) at lane boundaries and inside lanes, and a run of three equal values
      per = (S + 31) // 32
      for i in sorted({per - 1, 2 * per - 1, S // 3, S // 2, S // 2 + 1}):
        if 0 < i < S:
          z[:, i] = z[:, i - 1]
  elif regime in ('wall', 'opaque_run'):
    raw = half
    k0 = S // 5
    n = 1 if regime == 'wall' else 6
    for k in range(k0, min(S, k0 + n)):
      if k + 1 < S:
        raw[:, k] = _wall_raw(40.0, dist[:, k], act).float()
  else:
    raise ValueError(regime)
  if inf and act not in NEGATIVE_SIGMA:
    raw[:, -1] = raw[:, -1].abs()
  return rgb_raw, raw.float(), z, dirs


def _cotangent(R, S, which, seed):
  """d_out (R,6) and d_weights (R,S) (None where `which` leaves them out); med_depth's slot is random and
  must be ignored."""
  g = torch.Generator().manual_seed(seed)
  d_out = torch.randn(R, 6, generator=g)
  d_w = torch.randn(R, S, generator=g)
  keep = {'rgb': [0, 1, 2], 'depth': [3], 'acc': [5], 'all': [0, 1, 2, 3, 5]}.get(which, [])
  for c in (0, 1, 2, 3, 5):
    if c not in keep:
      d_out[:, c] = 0.0
  return (d_out if keep else None), (d_w if which in ('weights', 'all') else None)


def _run_composite(rgb_raw, alpha_raw, z, dirs, act, white, inf, d_out, d_w, ld_rgb, ld_a):
  """The kernel on padded layouts; checks that nothing outside the written columns changed."""
  R, S = z.shape
  rows = R * S
  rr = torch.full((rows, ld_rgb), float('nan'))
  rr[:, :3] = rgb_raw.reshape(rows, 3)
  ar = torch.full((rows, ld_a), float('nan'))
  ar[:, 0] = alpha_raw.reshape(rows)
  rr, ar = rr.to(DEV), ar.to(DEV)
  d_rgb = torch.full((rows, ld_rgb), float('nan'), device=DEV)
  d_a = torch.full((rows, ld_a), float('nan'), device=DEV)
  samples = torch.empty(rows, 4, device=DEV)
  L = _lib()
  dev = lambda t: None if t is None else t.contiguous().to(DEV)
  zd, dd, do, dw = dev(z), dev(dirs), dev(d_out), dev(d_w)
  L.check(L.load().nfb_selftest_composite_vjp(R, S, _ptr(rr), ld_rgb, _ptr(ar), ld_a, _ptr(zd), _ptr(dd), _ptr(do),
                                              _ptr(dw), int(white), int(inf), ACT[act], _ptr(samples), _ptr(d_rgb),
                                              _ptr(d_a), None))
  torch.cuda.synchronize()
  d_rgb, d_a = d_rgb.cpu(), d_a.cpu()
  assert torch.isnan(d_rgb[:, 3:]).all() and torch.isnan(d_a[:, 1:]).all(), 'write outside the output columns'
  return d_rgb[:, :3].reshape(R, S, 3), d_a[:, 0].reshape(R, S), samples.cpu()


def _dists(z, dirs, inf):
  last = 1e10 if inf else 1e-19
  return torch.cat([z[:, 1:] - z[:, :-1], torch.full_like(z[:, :1], last)], -1) * dirs.norm(dim=-1, keepdim=True)


def _composite_ref(rgb_raw, alpha_raw, z, dirs, act, white, inf, d_out, d_w, move_seed=None):
  """fp64 autograd of <cotangents, O.volumetric_rendering(sigmoid(rgb_raw), act(alpha_raw), ...)>, optionally
  with sigma * dist and sigmoid(rgb_raw) moved as an fp32 evaluation may move them (module docstring)."""
  rr = rgb_raw.double().clone()
  ar = alpha_raw.double().clone().requires_grad_(True)
  z, dirs = z.double(), dirs.double()
  sig_off = torch.zeros_like(ar)
  if move_seed is not None:
    g = torch.Generator().manual_seed(move_seed)
    rnd = lambda shape: 2 * torch.rand(shape, generator=g, dtype=torch.float64) - 1
    c = torch.sigmoid(rr)
    rr = rr + U * rnd(rr.shape) / (1 - c).clamp_min(1e-300)
    with torch.no_grad():
      sigma = O.activation_fn(act)(ar)
      dist = _dists(z, dirs, inf)
      x = sigma * dist
      xm = x * (1 + 6 * U * rnd(x.shape))
      a32 = (-torch.expm1(-xm)).float().double()
      x2 = torch.where(a32 < 1, -torch.log1p(-a32), torch.maximum(x, torch.full_like(x, 60.0)))
      sig_off = torch.where(dist > 0, (x2 - x) / torch.where(dist > 0, dist, torch.ones_like(dist)),
                            torch.zeros_like(x))
  rr = rr.requires_grad_(True)
  rgb = torch.sigmoid(rr)
  sigma = O.activation_fn(act)(ar) + sig_off
  out = O.volumetric_rendering(rgb, sigma, z, dirs, use_white_background=bool(white), sample_at_infinity=bool(inf))
  loss = 0.0
  if d_out is not None:
    do = d_out.double()
    loss = (out['rgb'] * do[:, :3]).sum() + (out['depth'] * do[:, 3]).sum() + (out['med_depth'] * do[:, 4]).sum() \
        + (out['acc'] * do[:, 5]).sum()
  if d_w is not None:
    loss = loss + (out['weights'] * d_w.double()).sum()
  loss.backward()
  zero = lambda t, gr: gr if gr is not None else torch.zeros_like(t)
  return zero(rr, rr.grad), zero(ar, ar.grad)


def _composite_bound(rgb_raw, alpha_raw, z, dirs, act, white, inf, d_out, d_w):
  """(M, floor) for d_rgb_raw (R,S,3) and d_alpha_raw (R,S): module docstring."""
  R, S = z.shape
  rr, ar, z, dirs = rgb_raw.double(), alpha_raw.double().clone().requires_grad_(True), z.double(), dirs.double()
  y = O.activation_fn(act)(ar)
  dact, = torch.autograd.grad(y.sum(), ar)
  y, ar = y.detach(), ar.detach()
  # the output-formed derivatives on absolute values (train.cuh act_grad_from_output)
  extra = {'tanh': y * y, 'sigmoid': y * y, 'elu': torch.where(y > 0, torch.zeros_like(y), y.abs() + 1)}
  dact_abs = dact.abs() + extra.get(act, torch.zeros_like(y))
  c = torch.sigmoid(rr)
  dist = _dists(z, dirs, inf)
  x = y * dist
  alpha = -torch.expm1(-x)
  f = 1 - alpha + 1e-10
  T = torch.cat([torch.ones_like(f[:, :1]), torch.cumprod(f[:, :-1], -1)], -1)
  w = (alpha * T).abs()                               # alpha < 0 where sigma < 0
  zero = torch.zeros(R, 6, dtype=torch.float64)
  do = d_out.double().abs() if d_out is not None else zero
  dw = d_w.double().abs() if d_w is not None else torch.zeros(R, S, dtype=torch.float64)
  g = do[:, :3]
  acc_on = torch.ones(S, dtype=torch.float64)
  if inf:
    acc_on[-1] = 0
  gw = (g[:, None, :] * c).sum(-1) + float(white) * g.sum(-1, keepdim=True) + do[:, 3:4] * z.abs() + \
      do[:, 5:6] * acc_on + dw
  suffix = lambda v: torch.flip(torch.cumsum(torch.flip(v, [-1]), -1), [-1]) - v
  tail = suffix(gw * w)
  # the fp64 oracle's own alpha = 1 - exp(-x) is exact only to 2^-53 absolute (a tiny alpha loses all its
  # digits there, where the kernel's expm1f keeps them): 2^-51 on every alpha
  ref_tail = 2.0**-51 * suffix(gw * T)
  G = g.sum(-1) + do[:, 3] * z.abs().max(-1).values + do[:, 5] + dw.max(-1).values
  under = (S * TINY * G)[:, None]
  bracket = gw * T + (tail + ref_tail + under) / f + under
  chain = dist * torch.exp(-x) * dact_abs
  m_alpha = chain * bracket
  floor_alpha = dist * dact_abs * TINY * bracket + 2.0**-149
  m_rgb = g[:, None, :] * w[..., None] * c * (1 + c)
  floor_rgb = g[:, None, :] * (S * TINY + 2.0**-51 * T[..., None] * c * (1 + c)) + 2.0**-149
  return m_rgb, floor_rgb, m_alpha, floor_alpha


def _check_composite(name, rgb_raw, alpha_raw, z, dirs, act, white, inf, d_out, d_w, ld_rgb=32, ld_a=32):
  S = z.shape[1]
  got_rgb, got_a, samples = _run_composite(rgb_raw, alpha_raw, z, dirs, act, white, inf, d_out, d_w, ld_rgb, ld_a)
  ref_rgb, ref_a = _composite_ref(rgb_raw, alpha_raw, z, dirs, act, white, inf, d_out, d_w)
  band_rgb, band_a = torch.zeros_like(ref_rgb), torch.zeros_like(ref_a)
  for seed in (1, 2):
    mr, ma = _composite_ref(rgb_raw, alpha_raw, z, dirs, act, white, inf, d_out, d_w, move_seed=seed)
    band_rgb = torch.maximum(band_rgb, (mr - ref_rgb).abs())
    band_a = torch.maximum(band_a, (ma - ref_a).abs())
  m_rgb, fl_rgb, m_a, fl_a = _composite_bound(rgb_raw, alpha_raw, z, dirs, act, white, inf, d_out, d_w)
  tol_rgb = 4 * S * U * m_rgb + 3 * band_rgb + fl_rgb
  tol_a = 4 * S * U * m_a + 3 * band_a + fl_a
  # raw_to_samples_kernel: sigmoid and the activation to a few roundings
  ref_s = torch.cat([torch.sigmoid(rgb_raw.double()), O.activation_fn(act)(alpha_raw.double())[..., None]], -1)
  s_err = float(((samples.reshape_as(ref_s).double() - ref_s).abs() / (8 * U * ref_s.abs() + 2.0**-149)).max())
  assert s_err <= 1.0, f'{name}: samples off by {s_err:.3g} of 8 u'
  r_rgb, r_a = _ratio(got_rgb, ref_rgb, tol_rgb), _ratio(got_a, ref_a, tol_a)
  _report(f'{name} d_rgb_raw', r_rgb)
  _report(f'{name} d_alpha_raw', r_a)
  return r_rgb, r_a


SHAPES = [1, 2, 31, 32, 33, 63, 65, 255, 257, 512, 1023, 1024]


@pytest.mark.parametrize('regime', ['half', 'wall'])
@pytest.mark.parametrize('S', SHAPES)
def test_composite_shapes(S, regime):
  """Every lane partition: trailing lanes that own nothing (S = 33: lanes 17-31), one sample per lane, S = 1;
  R = 7 rays leaves the last block of kRaysPerBlock = 4 short.  Tight strides at odd S, padded otherwise."""
  R = 7
  rgb_raw, raw, z, dirs = _composite_inputs(R, S, regime, 'softplus', seed=S, inf=True)
  d_out, d_w = _cotangent(R, S, 'all', seed=S + 1)
  tight = S % 2 == 1
  _check_composite(f'S={S} {regime}', rgb_raw, raw, z, dirs, 'softplus', S % 3 == 0, True, d_out, d_w,
                   ld_rgb=3 if tight else 32, ld_a=1 if tight else 32)


def _alpha32(raw, z, dirs, act, inf):
  sigma = O.activation_fn(act)(raw.float())
  return -torch.expm1(-sigma * _dists(z.float(), dirs.float(), inf))


@pytest.mark.parametrize('flags', [(0, 1), (1, 1), (0, 0), (1, 0)], ids=lambda f: f'white{f[0]}-inf{f[1]}')
@pytest.mark.parametrize('act', list(ACT))
@pytest.mark.parametrize('regime', ['empty', 'half', 'wall', 'opaque_run', 'dup_z'])
def test_composite_regimes(regime, act, flags):
  white, inf = flags
  if inf and act in NEGATIVE_SIGMA:
    pytest.skip('negative sigma times the 1e10 last distance is not finite in the reference either')
  R, S = 5, 65
  rgb_raw, raw, z, dirs = _composite_inputs(R, S, regime, act, seed=7, inf=inf)
  if regime in ('wall', 'opaque_run') and act in ('softplus', 'relu', 'elu', 'leaky_relu'):
    a = _alpha32(raw, z, dirs, act, inf)
    assert (a[:, S // 5] == 1.0).all(), 'the wall is not opaque in fp32'
    if regime == 'opaque_run':
      T = torch.cumprod(1 - a + 1e-10, -1)
      assert (T[:, S // 5 + 5] == 0).all(), 'the transmittance behind the run is not 0 in fp32'
  d_out, d_w = _cotangent(R, S, 'all', seed=11)
  _check_composite(f'{regime} {act} white={white} inf={inf}', rgb_raw, raw, z, dirs, act, white, inf, d_out, d_w)


@pytest.mark.parametrize('which', ['rgb', 'depth', 'acc', 'weights', 'all'])
def test_composite_cotangents(which):
  """One output's cotangent at a time, d_out or d_weights null."""
  R, S = 6, 257
  rgb_raw, raw, z, dirs = _composite_inputs(R, S, 'wall', 'softplus', seed=21, inf=True)
  d_out, d_w = _cotangent(R, S, which, seed=22)
  _check_composite(f'cotangent {which}', rgb_raw, raw, z, dirs, 'softplus', 1, True, d_out, d_w)


def test_composite_fullhd_fine_seed():
  """The fine level's seed of test_render_vjp_gpu.py's fullhd case with every cotangent: the fine MLP's raw rgb
  and density from the oracle in fp32 at the kernel's z_fine, through composite_vjp_kernel, against the fp64
  adjoint on the same raw inputs."""
  from tests import test_render_vjp_gpu as V
  c = V._gin_case('fullhd')
  cot = V._cotangents(c, V.OUTPUTS, seed=len(V.OUTPUTS))
  _, _, z = V._cuda_grads(c, cot)
  zf = z['fine'].float()
  with torch.no_grad():
    out = O.render_level(c.params, c.spec, 'fine', c.rays, zf, c.warp_alpha, dtype=torch.float32)
  rgb_raw, raw = out['raw_rgb'].float(), out['raw_alpha'][..., 0].float()
  g = cot['fine']
  B = zf.shape[0]
  d_out = torch.zeros(B, 6)
  d_out[:, :3], d_out[:, 3], d_out[:, 5] = g['rgb'].float(), g['depth'].float(), g['acc'].float()
  assert c.spec.sigma_activation == 'softplus'
  _check_composite('fullhd fine seed', rgb_raw, raw, zf, c.rays['directions'].float(), 'softplus',
                   c.spec.use_white_background, c.spec.use_sample_at_infinity, d_out, g['weights'].float(),
                   ld_rgb=32, ld_a=32)


# ---------------------------------------------------------------------------
# 2. jac_elastic_kernel: svd3 / elastic_sq (warp_type 1) and the SE(3) tail (warp_type 2)
# ---------------------------------------------------------------------------
def _rot(axis, angle):
  a = torch.tensor(axis, dtype=torch.float64)
  a = a / a.norm()
  K = O.skew(a)
  return torch.eye(3, dtype=torch.float64) + math.sin(angle) * K + (1 - math.cos(angle)) * (K @ K)


def _usv(s, seed):
  g = torch.Generator().manual_seed(seed)
  q1, _ = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
  q2, _ = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
  return q1 @ torch.diag(torch.tensor(s, dtype=torch.float64)) @ q2.T


def _designed():
  """Named 3x3 Jacobians (float64; the kernel sees I + fp32(J - I))."""
  I = torch.eye(3, dtype=torch.float64)
  R1 = _rot([1.0, -2.0, 0.5], 0.7)
  zero_col = _usv([1.2, 0.9, 0.6], 3)
  zero_col[:, 2] = 0
  rank1 = torch.zeros(3, 3, dtype=torch.float64)
  rank1[:, 0] = torch.tensor([0.6, -0.8, 0.5], dtype=torch.float64)
  return {
      'identity': I,
      'rotation': R1,
      'rotation_pi': _rot([0.0, 0.0, 1.0], math.pi),
      'reflection': R1 @ torch.diag(torch.tensor([1.0, 1.0, -1.0], dtype=torch.float64)),
      'diag_1_1_1+eps': torch.diag(torch.tensor([1.0, 1.0, 1.0 + 2.0**-20], dtype=torch.float64)),
      'diag_1_1_1+1e-4': torch.diag(torch.tensor([1.0, 1.0, 1.0 + 1e-4], dtype=torch.float64)),
      'repeated': _usv([2.0, 2.0, 0.5], 4),
      'repeated_3': _usv([1.5, 1.5, 1.5], 5),
      'nearly_repeated': _usv([1.5, 1.5 * (1 + 1e-5), 0.7], 6),
      'cond_1e3': _usv([1.0, 0.3, 1e-3], 7),
      'cond_1e6': _usv([2.0, 1e-2, 2e-6], 8),
      'zero_column': zero_col,
      'rank2': _usv([1.3, 0.8, 0.0], 9),
      'rank1': rank1,
      'rank1_rotated': _usv([1.1, 0.0, 0.0], 10),
      'below_clamp': _usv([1.0, 0.9, 1e-7], 11),
      'negative_det': _usv([1.0, 0.8, 0.5], 12) @ torch.diag(torch.tensor([1.0, 1.0, -1.0], dtype=torch.float64)),
  }


def _near_identity(n, scale, seed):
  g = torch.Generator().manual_seed(seed)
  return torch.eye(3, dtype=torch.float64) + scale * torch.randn(n, 3, 3, generator=g, dtype=torch.float64)


def _elastic_ref(J, loss_type, w, gs):
  """fp64 (loss, residual, dL/dJ) with L = sum gs w loss (O.compute_elastic_loss).  For 'det' and 'log_det' the
  gradient is dL/d det x cof(J): torch's det backward (and its forward mode) returns 0 at an exactly singular J,
  where the cofactor matrix is not 0.  det is affine in each entry, so cof_ij = det(J + E_ij) - det(J) exactly
  with the oracle's det, and dL/d det is autograd of the oracle's det residual (training.py:103-108) through
  O.general_loss_with_squared_residual, checked against compute_elastic_loss's own loss."""
  Jg = J.clone().requires_grad_(True)
  loss, res = O.compute_elastic_loss(Jg, loss_type=loss_type)
  if loss_type not in ('det', 'log_det'):
    dJ, = torch.autograd.grad((gs * w * loss).sum(), Jg)
    return loss.detach(), res.detach(), dJ
  d = torch.linalg.det(J).clone().requires_grad_(True)
  sq = (d - 1.0) ** 2 if loss_type == 'det' else torch.log(torch.clamp(d, min=1e-6)) ** 2
  l = O.general_loss_with_squared_residual(sq, alpha=-2.0, scale=0.03)
  assert torch.equal(l.detach(), loss.detach()), 'the det residual differs from compute_elastic_loss'
  dd, = torch.autograd.grad((gs * w * l).sum(), d)
  E = torch.eye(9, dtype=J.dtype).reshape(9, 3, 3)
  cof = (torch.linalg.det(J[:, None] + E[None]) - torch.linalg.det(J)[:, None]).reshape(-1, 3, 3)
  return loss.detach(), res.detach(), dd[:, None, None] * cof


def _run_elastic(R, warp_type, pivot, trans, loss_type, head, thead, ld, pts, sel, row_w, gs, d_head0):
  d_head = d_head0.clone().to(DEV) if d_head0 is not None else None
  jac = torch.full((R, 9), float('nan'), device=DEV)
  d_thead = torch.full((3 * R, ld), float('nan'), device=DEV)
  stats = torch.zeros(5, device=DEV)
  L = _lib()
  dev = lambda t: None if t is None else t.contiguous().to(DEV)
  h, th, p, s, rw = dev(head), dev(thead), dev(pts), dev(sel), dev(row_w)
  L.check(L.load().nfb_selftest_elastic(R, warp_type, pivot, trans, ELASTIC[loss_type], _ptr(h), _ptr(th), ld, _ptr(p),
                                        _ptr(s), _ptr(rw), gs, _ptr(jac), _ptr(d_head), _ptr(d_thead), _ptr(stats),
                                        None))
  torch.cuda.synchronize()
  return jac.cpu(), (d_head.cpu() if d_head is not None else None), d_thead.cpu(), stats.cpu()


def _dl(J, loss_type):
  """d general_loss / d sq at the point's squared residual (the robust loss of training.py:113-114)."""
  _, res = O.compute_elastic_loss(J, loss_type=loss_type)
  x = (res ** 2).clone().requires_grad_(True)
  dl, = torch.autograd.grad(O.general_loss_with_squared_residual(x, -2.0, 0.03).sum(), x)
  return x.detach(), dl


def _elastic_floor(J, loss_type, w, gs, ref):
  """Per element, what an fp32 evaluation of elastic_sq can be held to (module docstring):
    svd types: every singular value to 32 u s_max (one-sided Jacobi), which moves g_k = 2 log(s_k) / s_k
      ('log_svals') or 2 (s_k - 1) ('svals') by |g_k'| 32 u s_max, and U, V orthogonal to 2^-20, which moves dJ
      by 2^-20 sum |g_k|;
    'det', 'log_det': det to 12 u m^3 and each cofactor to 4 u m^2 (m = max |J_ij|): the rounding of (det - 1)
      or of log(det) / det times the cofactor, and the rounding of the cofactor times that factor;
    'jtj': E = J J^T - I to 4 u (|J| |J|^T + I) and E J to 3 u |E| |J|;  'div': trace - 3 to 4 u (|trace| + 3);
  all times gs w |dl|, plus 8 u |ref| for the products with gs, w, dl and dl's own conditioning on the error
  of sq (2 dsq / (sq + 4 scale^2) relative, dsq = sum |dsq/dJ| 32 u m)."""
  sq, dl = _dl(J, loss_type)
  k = (gs * w * dl.abs())[:, None, None]
  m = J.abs().flatten(1).max(-1).values[:, None, None]
  one = torch.ones_like(J)
  if loss_type in ('log_svals', 'svals'):
    s = torch.linalg.svdvals(J)
    ds = 32 * U * s[:, :1]
    if loss_type == 'log_svals':
      ok = s > 1e-6
      g = torch.where(ok, 2 * torch.log(s.clamp_min(1e-6)).abs() / s, torch.zeros_like(s))
      dg = torch.where(ok, 2 * (1 - torch.log(s.clamp_min(1e-6))).abs() / s.clamp_min(1e-6) ** 2, torch.zeros_like(s)) * ds
    else:
      g, dg = 2 * (s - 1).abs(), 2 * ds.expand_as(s)
    fl = (dg.sum(-1) + 2.0**-20 * g.sum(-1))[:, None, None] * one
  elif loss_type in ('det', 'log_det'):
    det = torch.linalg.det(J)[:, None, None]
    E = torch.eye(9, dtype=J.dtype).reshape(9, 3, 3)
    C = (torch.linalg.det(J[:, None] + E[None]) - det.reshape(-1, 1)).reshape(-1, 3, 3).abs()
    ddet, dC = 12 * U * m**3, 4 * U * m**2
    if loss_type == 'det':
      kp, dkp = 2 * (det - 1).abs(), 2 * ddet
    else:
      ok = det > 1e-6
      ld = torch.log(det.clamp_min(1e-6))
      kp = torch.where(ok, 2 * ld.abs() / det.clamp_min(1e-6), torch.zeros_like(det))
      dkp = torch.where(ok, 2 * (1 - ld).abs() / det.clamp_min(1e-6) ** 2 * ddet, torch.zeros_like(det))
    fl = dkp * C + kp * dC
  elif loss_type == 'jtj':
    Ja = J.abs()
    Ea = (J @ J.transpose(1, 2) - torch.eye(3, dtype=J.dtype)).abs()
    fl = 4 * U * (Ja @ Ja.transpose(1, 2) + torch.eye(3, dtype=J.dtype)) @ Ja + 3 * U * Ea @ Ja
  else:
    tr = J.diagonal(dim1=1, dim2=2).sum(-1)[:, None, None]
    fl = 2 * 4 * U * (tr.abs() + 3) * torch.eye(3, dtype=J.dtype).expand_as(J)
  dsq = (ref.abs() / k.clamp_min(1e-300)).flatten(1).sum(-1)[:, None, None] * 32 * U * m
  rel = 8 * U + 2 * dsq / (sq[:, None, None] + 4 * 0.03**2)
  return k * fl + rel * ref.abs()


def _range_projector(J):
  """Projector onto the range of J: the left singular vectors of the singular values above 1e-6 s_max."""
  Uf, s, _ = torch.linalg.svd(J)
  keep = (s > 1e-6 * s[:, :1]).double()
  return Uf @ torch.diag_embed(keep) @ Uf.transpose(1, 2)


def _moved_J(J, seed):
  """J moved by one rounding of each entry and of the point's largest entry (the latter moves the exact zeros of
  a rank-deficient J too)."""
  gm = torch.Generator().manual_seed(seed)
  r = lambda: 2 * torch.rand(J.shape, generator=gm, dtype=torch.float64) - 1
  big = J.abs().flatten(1).max(-1).values[:, None, None]
  return J * (1 + U * r()) + U * big * r()


def _elastic_case(name, Jd, loss_type, seed, project_null=False):
  """J = I + fp32(J - I) through warp_type 1 at R points; J, stats and d_thead against fp64."""
  R = Jd.shape[0]
  ld = 5
  th32 = (Jd - torch.eye(3, dtype=torch.float64)).float()          # Th[j][q] = J[q][j] - delta
  thead = torch.zeros(3 * R, ld)
  thead[:, :3] = th32.transpose(1, 2).reshape(3 * R, 3)
  J = (torch.eye(3) + th32).double()                               # the kernel's fp32 addition, exactly
  g = torch.Generator().manual_seed(seed)
  head = torch.randn(R, ld, generator=g)
  pts = torch.randn(R, 3, generator=g)
  w = torch.rand(R, generator=g, dtype=torch.float64) + 0.5
  gs = 0.37
  jac, _, d_thead, stats = _run_elastic(R, 1, 0, 0, loss_type, head, thead, ld, pts, None, w.float(), gs, None)
  assert torch.equal(jac.reshape(R, 3, 3).double(), J), f'{name}: J differs from I + Th^T'
  loss, res, dJ = _elastic_ref(J, loss_type, w.float().double(), gs)
  dJ_full = dJ
  got = d_thead.reshape(R, 3, ld)[:, :, :3].transpose(1, 2).double()   # got[r, q, j] = dL / dJ[q][j]
  P = torch.eye(3, dtype=torch.float64).expand_as(J)
  if project_null:
    P = _range_projector(J)
    got, dJ = P @ got, P @ dJ
  band = torch.zeros_like(dJ)
  for s in (1, 2, 3):
    Jm = _moved_J(J, 1000 + s)
    Pm = _range_projector(Jm) if project_null else P
    band = torch.maximum(band, (Pm @ _elastic_ref(Jm, loss_type, w.float().double(), gs)[2] - dJ).abs())
  floor = _elastic_floor(J, loss_type, w.float().double(), gs, dJ)
  tol = torch.maximum(floor, 3 * band) + 1e-300
  # the bound must constrain: at most 2^-6 of the point's largest gradient entry or 4 x the point's largest fp32
  # floor of _elastic_floor (where the gradient itself is at the rounding of J J^T - I, det - 1 or log s: J orthogonal,
  # det near 1), whichever is larger
  pmax = dJ.abs().flatten(1).max(-1).values[:, None, None]
  power = float((tol / torch.maximum(2.0**-6 * pmax, 4 * floor.flatten(1).max(-1).values[:, None, None]).clamp_min(1e-300)).max())
  print(f'{name} {loss_type}: bound / max(2^-6 x largest gradient entry, 4 x fp32 floor) {power:.3g}')
  assert power <= 1.0, f'{name} {loss_type}: the bound does not constrain the gradient ({power:.3g})'
  ratio = _ratio(got, dJ, tol)
  # stats: sum w loss, sum residual, sum det, sum div, sum |curl|
  ref_stats = torch.stack([(w.float().double() * loss).sum(), res.sum(), torch.linalg.det(J).sum(),
                           O.jacobian_to_div(J).sum(), O.jacobian_to_curl(J).norm(dim=-1).sum()])
  band_s = torch.zeros(5, dtype=torch.float64)
  for s in (1, 2, 3):
    Jm = _moved_J(J, 2000 + s)
    lm, rm, _ = _elastic_ref(Jm, loss_type, w.float().double(), gs)
    band_s[0] = max(band_s[0], float(((w.float().double() * lm).sum() - ref_stats[0]).abs()))
    band_s[1] = max(band_s[1], float((rm.sum() - ref_stats[1]).abs()))
  mag = torch.stack([(w.float().double() * loss).abs().sum(), res.abs().sum(), torch.ones(()) * R,
                     torch.ones(()) * R, O.jacobian_to_curl(J).norm(dim=-1).sum() + R])
  # sq to dsq = sum |dsq/dJ| 32 u m + 3 (32 u s_max)^2 (the square of the singular values' own error near a
  # residual of 0): the loss to |dl| dsq, the residual (its square root) to sqrt(dsq)
  sq, dl = _dl(J, loss_type)
  m = J.abs().flatten(1).max(-1).values
  smax = torch.linalg.svdvals(J)[:, 0]
  dsq = (dJ_full.abs().flatten(1).sum(-1) / (gs * w.float().double() * dl.abs()).clamp_min(1e-300)) * 32 * U * m \
      + 3 * (32 * U * smax) ** 2
  floor_s = torch.zeros(5, dtype=torch.float64)
  floor_s[0] = (w.float().double() * dl.abs() * dsq).sum()
  floor_s[1] = (dsq / (sq.sqrt() + dsq.sqrt())).sum()
  tol_s = 3 * band_s + 64 * U * mag * (R + 8) + floor_s + 1e-30
  ratio_s = _ratio(stats, ref_stats, tol_s)
  _report(f'{name} {loss_type} dJ', ratio)
  _report(f'{name} {loss_type} stats', ratio_s)


RANK_DEFICIENT = ('zero_column', 'rank2', 'rank1', 'rank1_rotated')


@pytest.mark.parametrize('loss_type', list(ELASTIC))
@pytest.mark.parametrize('name', list(_designed()))
def test_elastic_designed(name, loss_type):
  Jd = _designed()[name][None].repeat(3, 1, 1)
  _elastic_case(name, Jd, loss_type, seed=len(name), project_null=name in RANK_DEFICIENT and loss_type == 'svals')


@pytest.mark.parametrize('loss_type', list(ELASTIC))
@pytest.mark.parametrize('scale', [1e-4, 1e-2])
def test_elastic_near_identity(scale, loss_type):
  """A batch of J near I, at and above the scale of a freshly initialised warp."""
  _elastic_case(f'near I x{scale:g}', _near_identity(300, scale, seed=int(1 / scale)), loss_type, seed=5)


@pytest.mark.parametrize('name', ['zero_column', 'rank1'])
def test_svals_null_space(name):
  """'svals' at a singular value that is exactly 0 in fp32: svd3 leaves that column of U zero, so dJ drops the
  -2 u v^T term that jax's svdvals gradient has there (the gradient is not unique at s = 0).  dJ has no part
  in the left null space of J."""
  J = _designed()[name][None].repeat(2, 1, 1)
  R, ld = 2, 3
  th32 = (J - torch.eye(3, dtype=torch.float64)).float()
  thead = th32.transpose(1, 2).reshape(3 * R, 3).contiguous()
  Jk = (torch.eye(3) + th32).double()
  _, _, d_thead, _ = _run_elastic(R, 1, 0, 0, 'svals', torch.zeros(R, ld), thead, ld, torch.zeros(R, 3), None, None,
                                  1.0, None)
  got = d_thead.reshape(R, 3, ld).transpose(1, 2).double()
  Uf, s, _ = torch.linalg.svd(Jk)
  rank = {'zero_column': 2, 'rank1': 1}[name]
  assert (s[:, rank:] <= 1e-12 * s[:, :1]).all()
  null = Uf[:, :, rank:]
  leak = float((null.transpose(1, 2) @ got).abs().max())
  scale = float(got.abs().max())
  print(f'{name}: null-space part of dJ {leak:.3g} (dJ {scale:.3g})')
  assert scale > 0 and leak <= 2.0**-20 * scale


# ---- SE(3) tail ----
LAYOUTS = {'nh6': (0, 0), 'nh9_pivot': (1, 0), 'nh9_translation': (0, 1), 'nh12': (1, 1)}


def _se3_inputs(R, nh, theta, seed):
  g = torch.Generator().manual_seed(seed)
  axis = torch.randn(R, 3, generator=g)
  axis = axis / axis.norm(dim=-1, keepdim=True)
  head = torch.cat([theta * axis, 0.3 * torch.randn(R, 3, generator=g), 0.1 * torch.randn(R, nh - 6, generator=g)], -1)
  th = 0.05 * torch.randn(R, 3, nh, generator=g)
  th[:, :, :3] *= theta / 0.3 + 0.1                      # the axis' tangent at the axis' scale
  x = 0.5 * torch.randn(R, 3, generator=g)
  return head.float(), th.float(), x.float()


def _se3_ref(head, th, x, pivot, trans, loss_type, w, gs, dtype):
  """J = dy/dx + dy/dh Th^T of O.se3_tail, the elastic loss on it and its gradients w.r.t. the head (second
  order, through a double backward) and Th."""
  h = head.to(dtype).clone().requires_grad_(True)
  t = th.to(dtype).clone().requires_grad_(True)
  xx = x.to(dtype).clone().requires_grad_(True)
  k = 6
  pv = h[:, 6:9] if pivot else None
  k += 3 if pivot else 0
  tr = h[:, k:k + 3] if trans else None
  y = O.se3_tail(h[:, :3], h[:, 3:6], xx, pv, tr)
  Jx = torch.stack([torch.autograd.grad(y[:, i].sum(), xx, create_graph=True)[0] for i in range(3)], 1)
  Jh = torch.stack([torch.autograd.grad(y[:, i].sum(), h, create_graph=True)[0] for i in range(3)], 1)
  J = Jx + Jh @ t.transpose(1, 2)
  loss, _ = O.compute_elastic_loss(J, loss_type=loss_type)
  L = (gs * w.to(dtype) * loss).sum()
  dh, dt = torch.autograd.grad(L, (h, t), retain_graph=True)
  # the same contractions on absolute values, with G = dL/dJ at the point's largest |G| (the SVD's error in G is
  # normwise): max|G| sum_ij |dJ_ij / dh_q| and max|G| sum_i |dy_i / dh_q|
  G, = torch.autograd.grad(L, J, retain_graph=True)
  G = G.abs().flatten(1).max(-1).values[:, None, None].expand(-1, 3, 3)
  dJdh = torch.stack([torch.stack([torch.autograd.grad(J[:, i, j].sum(), h, retain_graph=True)[0]
                                   for j in range(3)], 1) for i in range(3)], 1)
  a_h = (G.abs()[..., None] * dJdh.abs()).sum((1, 2))
  a_t = (G.abs()[..., None] * Jh.abs()[:, :, None, :]).sum(1)
  return J.detach().double(), dh.double(), dt.double(), a_h.detach().double(), a_t.detach().double()


@pytest.mark.parametrize('theta', [1e-3, 0.3, 3.0])
@pytest.mark.parametrize('layout', list(LAYOUTS))
def test_se3_second_order(layout, theta):
  """J, d_thead and d_head (the second derivatives of the SE(3) tail) at every head layout, with sel and row_w
  (d_head += at the selected rows)."""
  pivot, trans = LAYOUTS[layout]
  nh = 6 + 3 * pivot + 3 * trans
  R, rows, ld = 70, 90, 16
  loss_type = 'log_svals'
  head_s, th, x_s = _se3_inputs(R, nh, theta, seed=nh + int(theta * 10))
  g = torch.Generator().manual_seed(3)
  sel = torch.randperm(rows, generator=g)[:R].int()
  head = torch.randn(rows, ld, generator=g)
  head[sel.long(), :nh] = head_s
  pts = torch.randn(rows, 3, generator=g)
  pts[sel.long()] = x_s
  row_w = torch.rand(rows, generator=g) + 0.5
  thead = torch.randn(3 * R, ld, generator=g)
  thead.reshape(R, 3, ld)[:, :, :nh] = th
  d_head0 = torch.randn(rows, ld, generator=g)
  gs = 0.8
  jac, d_head, d_thead, _ = _run_elastic(R, 2, pivot, trans, loss_type, head, thead, ld, pts, sel, row_w, gs, d_head0)
  w = row_w[sel.long()]
  J, dh, dt, a_h, a_t = _se3_ref(head_s, th, x_s, pivot, trans, loss_type, w, gs, torch.float64)
  # fp32 keeps theta - sin(theta) and 1 - cos(theta) to u theta absolute against theta^3 / 6 and theta^2 / 2
  k = (2.0**-16 + 8 * U / theta**2)
  a_h, a_t = k * a_h, k * a_t
  J32, dh32, dt32, _, _ = _se3_ref(head_s, th, x_s, pivot, trans, loss_type, w, gs, torch.float32)
  bJ, bh, bt = (J32 - J).abs(), (dh32 - dh).abs(), (dt32 - dt).abs()
  for s in (1, 2):
    gm = torch.Generator().manual_seed(100 + s)
    mv = lambda t: (t.double() * (1 + U * (2 * torch.rand(t.shape, generator=gm, dtype=torch.float64) - 1)))
    Jm, dhm, dtm, _, _ = _se3_ref(mv(head_s), mv(th), mv(x_s), pivot, trans, loss_type, w, gs, torch.float64)
    bJ, bh, bt = torch.maximum(bJ, (Jm - J).abs()), torch.maximum(bh, (dhm - dh).abs()), torch.maximum(bt, (dtm - dt).abs())
  pscale = lambda r: r.abs().flatten(1).max(-1).values.reshape(-1, *([1] * (r.dim() - 1)))
  gotJ = jac.reshape(R, 3, 3)
  got_dh = (d_head.double() - d_head0.double())[sel.long(), :nh]
  got_dt = d_thead.reshape(R, 3, ld)[:, :, :nh]
  ratios = {
      'J': _ratio(gotJ, J, torch.maximum(2.0**-20 * pscale(J), 3 * bJ)),
      'd_head': _ratio(got_dh, dh, torch.maximum(2.0**-20 * pscale(dh), 3 * bh) + a_h +
                       U * d_head[sel.long(), :nh].double().abs()),
      'd_thead': _ratio(got_dt, dt, torch.maximum(2.0**-20 * pscale(dt), 3 * bt) + a_t),
  }
  untouched = torch.ones(rows, dtype=torch.bool)
  untouched[sel.long()] = False
  assert torch.equal(d_head[untouched], d_head0[untouched]), 'd_head changed at a row that was not selected'
  assert torch.equal(d_head[:, nh:], d_head0[:, nh:]), 'd_head changed beyond the head outputs'
  for k, r in ratios.items():
    _report(f'{layout} theta={theta:g} {k}', r)


# ---------------------------------------------------------------------------
# 3. depth_index_kernel
# ---------------------------------------------------------------------------
def _run_depth(weights):
  R, S = weights.shape
  w = weights.float().contiguous().to(DEV)
  sel = torch.full((R,), -1, dtype=torch.int32, device=DEV)
  L = _lib()
  L.check(L.load().nfb_selftest_depth_index(R, S, _ptr(w), _ptr(sel), None))
  torch.cuda.synchronize()
  sel = sel.cpu().long()
  assert torch.equal(sel // S, torch.arange(R)), 'sel does not index the ray\'s own row'
  return sel - torch.arange(R) * S


def _dyadic_crossing(S, c, seed):
  """Dyadic weights whose cumulative sum reaches 0.5 exactly at index c (never when c is None)."""
  g = torch.Generator().manual_seed(seed)
  w = torch.randint(0, 3, (S,), generator=g).double() * 2.0**-13    # < 0.5 over 1024 samples
  if c is None:
    return w
  w[c] = 0.5 - w[:c].sum()
  return w


@pytest.mark.parametrize('R', [1, 7, 9])
@pytest.mark.parametrize('S', [1, 31, 32, 33, 1024])
def test_depth_index_dyadic(S, R):
  """Crossings at lane 0 and 31 of a chunk and in the first lane of the next through the carry, at the last
  sample, never; R not a multiple of the 8 warps of a block."""
  cands = [None, 0, 31, 32, 33, 63, 64, 95, 96, S - 1, 511, 512]
  rows = []
  for r in range(R):
    c = cands[(r * 5 + S) % len(cands)]
    if c is not None and c >= S:
      c = S - 1
    rows.append(_dyadic_crossing(S, c, seed=r))
  w = torch.stack(rows)
  if R == 9:
    w[-1] = 0.0                                       # a ray of zero weights
  got = _run_depth(w)
  ref = O.compute_depth_index(w)
  print(f'S={S} R={R}: indices {got.tolist()}')
  assert torch.equal(got, ref.long())


@pytest.mark.parametrize('S', [33, 257, 1024])
def test_depth_index_random(S):
  R = 301
  g = torch.Generator().manual_seed(S)
  w = (torch.rand(R, S, generator=g) * 2.0 / S * (0.5 + torch.rand(R, 1, generator=g))).float()
  got = _run_depth(w)
  ref = O.compute_depth_index(w.double()).long()
  cum = torch.cumsum(w.double(), -1)
  near = lambda i: (cum.gather(1, i[:, None])[:, 0] - 0.5).abs() <= S * U
  bad = (got != ref) & ~(near(got) | near(ref))
  assert not bad.any(), f'indices {torch.nonzero(bad)[:, 0].tolist()} differ away from the threshold'
  print(f'S={S}: {int((got != ref).sum())} of {R} indices differ, all within S u of 0.5')


# ---------------------------------------------------------------------------
# 4. warp_mag_loss_kernel (general_loss)
# ---------------------------------------------------------------------------
ALPHAS = [-math.inf, -2.0, 0.0, 1.0, 2.0, math.inf]


@pytest.mark.parametrize('use_sel', [False, True])
@pytest.mark.parametrize('alpha', ALPHAS, ids=lambda a: f'alpha={a:g}')
def test_warp_mag_loss(alpha, use_sel):
  """Residuals 0, 1e-12 scale^2, scale^2 and 1e3 scale^2 (the last crosses the 87.5 clamp of alpha = +inf);
  the loss and residual sums and d warped (+=)."""
  scale, gs = 0.03, 0.7
  g = torch.Generator().manual_seed(4)
  targets = torch.tensor([0.0, 1e-12, 1.0, 1e3], dtype=torch.float64) * scale**2
  R = len(targets)
  dirs = torch.randn(R, 3, generator=g, dtype=torch.float64)
  dirs = dirs / dirs.norm(dim=-1, keepdim=True)
  pts_r = torch.randn(R, 3, generator=g)
  pts_r[:2] = 0.0                                     # residuals 0 and 1e-12 scale^2 without cancellation
  warped_r = (pts_r.double() + dirs * targets.sqrt()[:, None]).float()
  rows = 11
  if use_sel:
    sel = torch.tensor([9, 2, 5, 0], dtype=torch.int32)
    pts, warped = torch.randn(rows, 3, generator=g), torch.randn(rows, 3, generator=g)
    pts[sel.long()], warped[sel.long()] = pts_r, warped_r
  else:
    sel, pts, warped = None, pts_r, warped_r
  dw0 = torch.randn(pts.shape[0], 3, generator=g)
  dwarped, stats = dw0.clone().to(DEV), torch.zeros(2, device=DEV)
  L = _lib()
  dev = lambda t: None if t is None else t.contiguous().to(DEV)
  p, wv, s = dev(pts), dev(warped), dev(sel)
  L.check(L.load().nfb_selftest_warp_mag_loss(R, _ptr(p), _ptr(wv), _ptr(s), alpha, scale, gs, _ptr(dwarped),
                                              _ptr(stats), None))
  torch.cuda.synchronize()
  dwarped, stats = dwarped.cpu(), stats.cpu()

  def ref(dtype):
    wr = warped_r.to(dtype).clone().requires_grad_(True)
    sq = ((wr - pts_r.to(dtype)) ** 2).sum(-1)
    loss = O.general_loss_with_squared_residual(sq, alpha, scale)
    dw, = torch.autograd.grad((gs * loss).sum(), wr)
    return loss.detach().double(), sq.detach().double(), dw.double()

  loss, sq, dw = ref(torch.float64)
  loss32 = ref(torch.float32)[0]
  got_dw = (dwarped - dw0)[sel.long()] if use_sel else dwarped - dw0
  tol_dw = 32 * U * dw.abs() + 4 * U * dw0[sel.long() if use_sel else slice(None)].abs().double() + 1e-30
  tol_loss = torch.maximum(16 * U * loss.abs(), 3 * (loss32 - loss).abs()).sum() + 1e-30
  r_dw = _ratio(got_dw, dw, tol_dw)
  r_loss = float((stats[0].double() - loss.sum()).abs() / tol_loss)
  r_res = float((stats[1].double() - sq.sqrt().sum()).abs() / (8 * U * sq.sqrt().sum() + 1e-30))
  if use_sel:
    rest = torch.ones(rows, dtype=torch.bool)
    rest[sel.long()] = False
    assert torch.equal(dwarped[rest], dw0[rest]), 'dwarped changed at a row that was not selected'
  _report(f'alpha={alpha:g} sel={use_sel} dwarped', r_dw)
  _report(f'alpha={alpha:g} sel={use_sel} loss sum', r_loss)
  _report(f'alpha={alpha:g} sel={use_sel} residual sum', r_res)


# ---------------------------------------------------------------------------
# 5. The adjoints between the MLPs and the rays / tables
# ---------------------------------------------------------------------------
def _posenc_ref(x, F, window, g, ld_off=0):
  """fp64 adjoint of the encoding [x | w_f sin(2^f x) | w_f sin(fl32(2^f x + fl32(pi/2)))] of x (rows,3) under the
  cotangent g (rows, >= 3 + 6F) (columns ld_off..): (the gradient, the sum of its terms' absolute values).  The
  shifted angle is rounded to fp32 as the reference's fp32 encoding rounds it (O.HALF_PI_F32); 2^f x is exact."""
  x = x.double()
  dx = g[:, ld_off:ld_off + 3].double().clone()
  mag = dx.abs()
  for f in range(F):
    s = 2.0**f
    w = 1.0 if window is None else float(window[f])
    ang = x * s
    ang2 = (x.float() * s + torch.tensor(O.HALF_PI_F32)).double()
    for gc, a in ((g[:, ld_off + 3 + 6 * f:ld_off + 6 + 6 * f], ang), (g[:, ld_off + 6 + 6 * f:ld_off + 9 + 6 * f], ang2)):
      t = gc.double() * w * s * torch.cos(a)
      dx += t
      mag += t.abs()
  return dx, mag


@pytest.mark.parametrize('windowed', [False, True])
@pytest.mark.parametrize('F,S', [(1, 1), (4, 33), (8, 128), (10, 512)])
def test_encode_bwd(F, S, windowed):
  """dpts and the per-ray dcond atomics of encode_bwd_kernel: F up to 10 (angles up to 2^9 |x|), a window with
  zero and fractional entries, cond columns with zero entries (skipped) and a prefilled dcond (+=).
  dpts: (2F + 10) u times the sum of its terms' absolute values (2F + 1 fused additions; cosf's 2 ulp and the
  products' roundings per term).  dcond: gamma_{S+1} times the sum of the absolute values of the S entries and
  the prefill."""
  R, n_cond, off, stride = 5, 13, 4, 21
  rows = R * S
  ld = 3 + 6 * F + n_cond + 2
  g = torch.Generator().manual_seed(F * 100 + S)
  pts = 2.0 * torch.randn(rows, 3, generator=g)
  din = torch.randn(rows, ld, generator=g)
  din[:, 3 + 6 * F:][torch.rand(rows, ld - 3 - 6 * F, generator=g) < 0.3] = 0.0
  din[:, -2:] = float('nan')                                # beyond the block: never read
  window = torch.from_numpy(O.cosine_easing_window(F, 0.55 * F + 0.3)) if windowed else None
  if windowed and F > 1:
    assert (window == 0).any() and ((window > 0) & (window < 1)).any()
  dcond0 = torch.randn(R, stride, generator=g)
  dpts = torch.full((rows, 3), float('nan'), device=DEV)
  dcond = dcond0.to(DEV)
  L = _lib()
  dev = lambda t: None if t is None else t.contiguous().to(DEV)
  pd, wd, dind = dev(pts), dev(window), dev(din)          # held until the kernel has run
  L.check(L.load().nfb_selftest_encode_bwd(rows, S, _ptr(pd), _ptr(wd), _ptr(dind), F, ld, stride, off, n_cond,
                                           _ptr(dpts), _ptr(dcond), None))
  torch.cuda.synchronize()
  ref, mag = _posenc_ref(pts, F, window, din)
  _report(f'encode_bwd F={F} S={S} window={windowed} dpts', _ratio(dpts.cpu(), ref, (2 * F + 10) * U * mag))
  blk = din[:, 3 + 6 * F:3 + 6 * F + n_cond].double().reshape(R, S, n_cond)
  ref_c = dcond0.double().clone()
  ref_c[:, off:off + n_cond] += blk.sum(1)
  tol_c = torch.zeros_like(ref_c)
  tol_c[:, off:off + n_cond] = 1.01 * (S + 1) * U * (blk.abs().sum(1) + dcond0[:, off:off + n_cond].double().abs())
  got_c = dcond.cpu()
  assert torch.equal(got_c[:, :off], dcond0[:, :off]) and torch.equal(got_c[:, off + n_cond:], dcond0[:, off + n_cond:])
  _report(f'encode_bwd F={F} S={S} dcond', _ratio(got_c, ref_c, tol_c))


def _tail_ref(head, x, warp_type, pivot, trans, dw, dtype):
  """(d head, d x) of <dw, O.se3_tail(...)> (or x + t) and the contractions sum_i |dw_i| |dy_i / d.|."""
  h = head.to(dtype).clone().requires_grad_(True)
  xx = x.to(dtype).clone().requires_grad_(True)
  if warp_type == 1:
    y = xx + h[:, :3]
  else:
    k = 6 + 3 * pivot
    y = O.se3_tail(h[:, :3], h[:, 3:6], xx, h[:, 6:9] if pivot else None, h[:, k:k + 3] if trans else None)
  jh = torch.stack([torch.autograd.grad(y[:, i].sum(), h, retain_graph=True)[0] for i in range(3)], 1)
  jx = torch.stack([torch.autograd.grad(y[:, i].sum(), xx, retain_graph=True)[0] for i in range(3)], 1)
  d = dw.to(dtype)
  return ((d[:, :, None] * jh).sum(1).double(), (d[:, :, None] * jx).sum(1).double(),
          (d.abs()[:, :, None] * jh.abs()).sum(1).double(), (d.abs()[:, :, None] * jx.abs()).sum(1).double())


@pytest.mark.parametrize('theta', [1e-3, 0.3, 3.0])
@pytest.mark.parametrize('layout', ['translation'] + list(LAYOUTS))
def test_warp_tail_adjoints(layout, theta):
  """warp_tail_bwd_kernel (dhead +=) and warp_tail_dx_kernel (dpts +=) at every head layout, into prefilled
  outputs.  Bound: 3 x the band (the fp32 oracle's distance from fp64 and fp64 under one-rounding moves of
  head and x), plus (2^-16 + 8 u / theta^2) x the contraction sum_i |dw_i| |dy_i / d.| (the nested fp32
  forward mode, and theta - sin(theta), 1 - cos(theta) kept to u theta absolute, as for the second order above;
  at theta = 1e-3 this term is about half of the w and v entries, which are then barely pinned), plus one
  rounding of the sum with the prefill.  The translation field's adjoints are the identity, to one rounding."""
  if layout == 'translation' and theta != 0.3:
    pytest.skip('the translation has no angle')
  warp_type, (pivot, trans) = (1, (0, 0)) if layout == 'translation' else (2, LAYOUTS[layout])
  nh = 3 if warp_type == 1 else 6 + 3 * pivot + 3 * trans
  rows, ld = 300, 16
  head_s, _, x = _se3_inputs(rows, max(nh, 6), theta, seed=nh + int(theta * 10) + 7)
  g = torch.Generator().manual_seed(5)
  head = torch.full((rows, ld), float('nan'))
  head[:, :nh] = head_s[:, :nh] if warp_type == 2 else 0.2 * torch.randn(rows, 3, generator=g)
  dw = torch.randn(rows, 3, generator=g)
  dh0, dx0 = torch.randn(rows, ld, generator=g), torch.randn(rows, 3, generator=g)
  dh, dx = dh0.to(DEV), dx0.to(DEV)
  L = _lib()
  hd_, xd, dwd = head.to(DEV), x.to(DEV), dw.to(DEV)
  L.check(L.load().nfb_selftest_warp_tail_bwd(rows, warp_type, pivot, trans, _ptr(hd_), ld, _ptr(xd), _ptr(dwd),
                                              _ptr(dh), _ptr(dx), None))
  torch.cuda.synchronize()
  dh, dx = dh.cpu(), dx.cpu()
  assert torch.equal(dh[:, nh:], dh0[:, nh:]), 'dhead changed beyond the head outputs'
  hs = head[:, :nh]
  rh, rx, ah, ax = _tail_ref(hs, x, warp_type, pivot, trans, dw, torch.float64)
  h32, x32, _, _ = _tail_ref(hs, x, warp_type, pivot, trans, dw, torch.float32)
  bh, bx = (h32 - rh).abs(), (x32 - rx).abs()
  for s in (1, 2):
    gm = torch.Generator().manual_seed(200 + s)
    mv = lambda t: t.double() * (1 + U * (2 * torch.rand(t.shape, generator=gm, dtype=torch.float64) - 1))
    mh, mx, _, _ = _tail_ref(mv(hs), mv(x), warp_type, pivot, trans, dw, torch.float64)
    bh, bx = torch.maximum(bh, (mh - rh).abs()), torch.maximum(bx, (mx - rx).abs())
  k = 0.0 if warp_type == 1 else 2.0**-16 + 8 * U / theta**2
  got_h, got_x = dh[:, :nh].double(), dx.double()
  ref_h, ref_x = dh0[:, :nh].double() + rh, dx0.double() + rx
  _report(f'warp tail {layout} theta={theta:g} dhead',
          _ratio(got_h, ref_h, 3 * bh + k * ah + U * ref_h.abs() + 2.0**-149))
  _report(f'warp tail {layout} theta={theta:g} dpts',
          _ratio(got_x, ref_x, 3 * bx + k * ax + U * ref_x.abs() + 2.0**-149))


@pytest.mark.parametrize('dnorm', [False, True])
@pytest.mark.parametrize('S', [1, 31, 32, 33, 512])
def test_ray_reduce(S, dnorm):
  """d_origins += sum_s g_s and d_directions += sum_s z_s g_s + d_dnorm d / |d| over R = 7 rays (a last block of
  kRaysPerBlock = 4 left short), twice into the same outputs (a coarse level of S samples, a fine one of
  S + 5), onto a prefill.  Bound: gamma_{S+S'+2} times the absolute sums and the prefill, plus 6 u |d_dnorm d / |d||
  per level (the norm's square root and the division)."""
  R = 7
  g = torch.Generator().manual_seed(S)
  dirs = torch.randn(R, 3, generator=g)
  o0, d0 = torch.randn(R, 3, generator=g), torch.randn(R, 3, generator=g)
  do, dd = o0.to(DEV), d0.to(DEV)
  ref_o, ref_d = o0.double().clone(), d0.double().clone()
  mag_o, mag_d = o0.double().abs(), d0.double().abs()
  L = _lib()
  n_terms = 0
  for lv, s_lv in enumerate((S, S + 5)):
    z = torch.sort(0.02 + 0.81 * torch.rand(R, s_lv, generator=g), -1).values
    gp = torch.randn(R, s_lv, 3, generator=g)
    gp[:, ::4] = 0.0
    dn = torch.randn(R, generator=g) if dnorm else None
    dev = lambda t: None if t is None else t.contiguous().to(DEV)
    gpd, zd, dirsd, dnd = dev(gp), dev(z), dev(dirs), dev(dn)
    L.check(L.load().nfb_selftest_ray_reduce(R, s_lv, _ptr(gpd), _ptr(zd), _ptr(dirsd), _ptr(dnd), _ptr(do), _ptr(dd),
                                             None))
    torch.cuda.synchronize()
    ref_o += gp.double().sum(1)
    mag_o += gp.double().abs().sum(1)
    zg = z.double()[..., None] * gp.double()
    ref_d += zg.sum(1)
    mag_d += zg.abs().sum(1)
    if dnorm:
      k = dn.double()[:, None] * dirs.double() / dirs.double().norm(dim=-1, keepdim=True)
      ref_d += k
      mag_d += 7 * k.abs()
    n_terms += s_lv + 1
  torch.cuda.synchronize()
  gam = 1.01 * (n_terms + 2) * U
  _report(f'ray_reduce S={S} d_dnorm={dnorm} d_origins', _ratio(do.cpu(), ref_o, gam * mag_o))
  _report(f'ray_reduce S={S} d_dnorm={dnorm} d_directions', _ratio(dd.cpu(), ref_d, gam * mag_d))


@pytest.mark.parametrize('accumulate', [0, 1])
def test_viewdir_vjp(accumulate):
  """The view-direction block's adjoint (F = 4, no window) at a block offset inside a wider dcond, = or +=
  a prefill.  Bound: as encode_bwd's dpts, plus one rounding of the prefill's sum."""
  R, F, off, stride = 133, 4, 11, 11 + 27 + 9
  g = torch.Generator().manual_seed(accumulate)
  vd = torch.randn(R, 3, generator=g)
  vd = vd / vd.norm(dim=-1, keepdim=True)
  dcond = torch.randn(R, stride, generator=g)
  out0 = torch.randn(R, 3, generator=g)
  out = out0.to(DEV)
  L = _lib()
  dcd, vdd = dcond.to(DEV), vd.to(DEV)
  L.check(L.load().nfb_selftest_viewdir_vjp(R, _ptr(dcd), stride, off, F, _ptr(vdd), _ptr(out), accumulate, None))
  torch.cuda.synchronize()
  ref, mag = _posenc_ref(vd, F, None, dcond, ld_off=off)
  if accumulate:
    ref, mag = ref + out0.double(), mag + out0.double().abs()
  _report(f'viewdir_vjp accumulate={accumulate}', _ratio(out.cpu(), ref, (2 * F + 11) * U * mag))


# ---- the condition vectors' adjoints (nfb_selftest_cond_vjp, on a handle's layout) ----
_COND_BASE = dict(num_coarse_samples=8, num_fine_samples=0, near=0.02, far=0.83, nerf_trunk_depth=2,
                  nerf_trunk_width=32, nerf_rgb_branch_width=16, num_nerf_point_freqs=2, use_warp=True,
                  warp_trunk_depth=2, warp_trunk_width=32, warp_skips=(), num_warp_embeddings=6,
                  use_appearance_metadata=True, num_appearance_embeddings=5, use_camera_metadata=True,
                  num_camera_embeddings=3, num_camera_features=4, use_trunk_condition=True,
                  use_alpha_condition=True)
COND_MODELS = {
    'glo': dict(warp_field_type='se3'),
    'blend': dict(warp_field_type='translation', warp_metadata_encoder_type='blend', metadata_encoder_num_freqs=2),
    'time': dict(warp_field_type='se3', warp_metadata_encoder_type='time', metadata_encoder_num_freqs=2),
}


def _cond_handle(kind):
  from tests.golden_util import model_from_spec, spec_to_dict, tree_to_device
  spec = O.OracleSpec(**{**_COND_BASE, **COND_MODELS[kind]})
  model = model_from_spec(spec_to_dict(spec), device=DEV)
  hd = model.handle()
  hd.set_params(tree_to_device(O.init_params(spec, 1), DEV))
  G, A, C = spec.num_warp_features, spec.num_appearance_features, spec.num_camera_features
  dv = 3 + 6 * spec.num_nerf_viewdir_freqs
  # [warp | trunk (A) | alpha (A) | rgb: viewdirs, appearance (A), camera]
  blocks = [('warp', 0, G), ('app', G, A), ('app', G + A, A), ('app', G + 2 * A + dv, A), ('cam', G + 3 * A + dv, C)]
  return spec, hd, blocks, G + 3 * A + dv + C


def _cond_call(hd, B, dcond, ids, encoded, has, dense, d_time):
  L = _lib()
  specs = hd.param_specs
  grads = [torch.zeros(r * c, device=DEV) for _, r, c in specs]
  gp = (ctypes.c_void_p * len(grads))(*[t.data_ptr() for t in grads])
  ne = (ctypes.c_longlong * len(grads))(*[t.numel() for t in grads])
  dev = lambda t: None if t is None else t.contiguous().to(DEV)
  dcd = dev(dcond)
  idd = [dev(ids.get(k)) for k in ('warp', 'app', 'cam')]      # held until the kernel has run
  L.check(L.load().nfb_selftest_cond_vjp(hd.h, B, _ptr(dcd), *[_ptr(t) for t in idd], encoded, has,
                                         *[_ptr(dense.get(k)) for k in ('warp', 'app', 'cam')], _ptr(d_time), gp, ne,
                                         len(grads), None))
  torch.cuda.synchronize()
  return {name: t.view(r, c).cpu() for t, (name, r, c) in zip(grads, specs)}


TABLES = {'warp': ('warp_field/metadata_encoder/embed/embedding', 'warp_field/glo_encoder/embed/embedding'),
          'app': ('appearance_encoder/embed/embedding',), 'cam': ('camera_encoder/embed/embedding',)}


def _table(grads, key):
  return next((grads[n] for n in TABLES[key] if n in grads), None)


@pytest.mark.parametrize('ids', ['spread', 'one_id', 'clamped'])
@pytest.mark.parametrize('case', ['glo', 'blend_0', 'blend_0.35', 'blend_1', 'time'])
def test_cond_bwd(case, ids):
  """cond_bwd_kernel's scatter-add into the tables: the appearance code's three blocks summed, the warp block
  scaled by 1 ('glo'), 1 - time_alpha ('blend') or not scattered ('time', no table), every ray on one id
  (atomic contention), ids at and past n - 1 (clamped to the last row); and time_cond_bwd_kernel's scale (1,
  or time_alpha under 'blend').  Bound: gamma_{n+1} times the absolute sum of the n entries a row receives
  (atomic additions in any order, each entry scaled by one rounding)."""
  kind, alpha = (case.split('_') + ['0'])[:2]
  spec, hd, blocks, stride = _cond_handle(kind)
  L = _lib()
  L.check(L.load().nfb_set_time_alpha(hd.h, float(alpha)))
  B = 300
  g = torch.Generator().manual_seed(len(case) + len(ids))
  dcond = torch.randn(B, stride, generator=g)
  dcond[torch.rand(B, stride, generator=g) < 0.2] = 0.0
  n = {'warp': spec.num_warp_embeddings, 'app': spec.num_appearance_embeddings, 'cam': spec.num_camera_embeddings}
  if ids == 'spread':
    idv = {k: torch.randint(0, v, (B,), generator=g) for k, v in n.items()}
  elif ids == 'one_id':
    idv = {k: torch.full((B,), v // 2, dtype=torch.long) for k, v in n.items()}
  else:
    idv = {k: torch.tensor([v - 1, v, v + 3, 2**31 + 5])[torch.randint(0, 4, (B,), generator=g)] for k, v in n.items()}
  ids32 = {k: torch.from_numpy(v.numpy().astype(np.uint32).view(np.int32)) for k, v in idv.items()}   # uint32 bits
  G = spec.num_warp_features
  d_time = torch.full((B, G), float('nan'), device=DEV) if kind != 'glo' else None
  grads = _cond_call(hd, B, dcond, ids32, 0, 0, {}, d_time)
  a32 = np.float32(alpha)                                   # time_alpha is an fp32 of the handle
  scale = {'glo': 1.0, 'blend': float(np.float32(1) - a32), 'time': 0.0}[kind]
  for key in ('warp', 'app', 'cam'):
    got = _table(grads, key)
    if got is None:
      assert key == 'warp' and kind == 'time'
      continue
    rows = idv[key].clamp(max=n[key] - 1)
    ref = torch.zeros(n[key], got.shape[1], dtype=torch.float64)
    mag = torch.zeros_like(ref)
    cnt = torch.zeros(n[key], 1, dtype=torch.float64)
    for name, off, w in blocks:
      if name != key:
        continue
      v = dcond[:, off:off + w].double() * (scale if key == 'warp' else 1.0)
      ref.index_add_(0, rows, v)
      mag.index_add_(0, rows, v.abs())
      cnt.index_add_(0, rows, torch.ones(B, 1, dtype=torch.float64))
    per = 3 if key == 'app' else 1
    _report(f'cond_bwd {case} ids={ids} {key}', _ratio(got, ref, 1.01 * (per * cnt + 2) * U * mag))
  if d_time is not None:
    ts = float(a32) if kind == 'blend' else 1.0
    ref = ts * dcond[:, :G].double()
    _report(f'time_cond_bwd {case}', _ratio(d_time.cpu(), ref, U * ref.abs()))


@pytest.mark.parametrize('dense', [False, True])
@pytest.mark.parametrize('has', range(8))
def test_cond_vjp_encoded(has, dense):
  """cond_vjp_encoded_kernel: each code the call passed (has: bits 1 warp, 2 appearance, 4 camera) gets its
  blocks' gradient in its dense output (+= a prefill; dropped with a null pointer), the appearance code the sum
  of its three blocks; a code it did not pass sends its blocks' sum over every ray to row 0 of its table.
  Bound: gamma_{n+2} times the absolute sum of the n entries (and the prefill)."""
  spec, hd, blocks, stride = _cond_handle('glo')
  B = 77
  g = torch.Generator().manual_seed(has)
  dcond = torch.randn(B, stride, generator=g)
  dcond[torch.rand(B, stride, generator=g) < 0.2] = 0.0
  widths = {'warp': spec.num_warp_features, 'app': spec.num_appearance_features, 'cam': spec.num_camera_features}
  bits = {'warp': 1, 'app': 2, 'cam': 4}
  pre = {k: torch.randn(B, w, generator=g) for k, w in widths.items()}
  out = {k: pre[k].to(DEV) for k in widths if dense}
  grads = _cond_call(hd, B, dcond, {}, 1, has, out, None)
  for key, w in widths.items():
    ref = torch.zeros(B, w, dtype=torch.float64)
    mag = torch.zeros_like(ref)
    for name, off, bw in blocks:
      if name == key:
        ref += dcond[:, off:off + bw].double()
        mag += dcond[:, off:off + bw].double().abs()
    table = _table(grads, key)
    if has & bits[key]:
      assert float(table.abs().sum()) == 0, f'{key}: a passed code sent a gradient to its table'
      if dense:
        r = ref + pre[key].double()
        _report(f'cond_vjp_encoded has={has} {key} dense', _ratio(out[key].cpu(), r, 4 * U * (mag + pre[key].double().abs())))
    else:
      if dense:
        assert torch.equal(out[key].cpu(), pre[key]), f'{key}: a code the call did not pass got a dense gradient'
      r0 = ref.sum(0)
      _report(f'cond_vjp_encoded has={has} {key} row 0', _ratio(table[0], r0, 1.01 * (3 * B + 2) * U * mag.sum(0)))
      assert float(table[1:].abs().sum()) == 0


def test_cond_vjp_rejects_bad_arguments():
  spec, hd, _, stride = _cond_handle('glo')
  L = _lib()
  lib = L.load()
  d = torch.zeros(4 * stride, device=DEV)
  n = len(hd.param_specs)
  grads = [torch.zeros(r * c, device=DEV) for _, r, c in hd.param_specs]
  gp = (ctypes.c_void_p * n)(*[t.data_ptr() for t in grads])
  ne = (ctypes.c_longlong * n)(*[t.numel() for t in grads])

  def call(B=4, dcond=_ptr(d), encoded=0, has=0, d_time=None, count=n):
    return lib.nfb_selftest_cond_vjp(hd.h, B, dcond, None, None, None, encoded, has, None, None, None, d_time, gp, ne,
                                     count, None)

  def refused(status, what):
    assert status != 0
    assert what in lib.nfb_last_error().decode(), lib.nfb_last_error()
  refused(call(B=-1), 'B=-1 must be >= 0')
  refused(call(dcond=None), 'null dcond')
  refused(call(encoded=2), 'encoded=2 is not 0 or 1')
  refused(call(has=1), 'with encoded only')
  refused(call(encoded=1, has=8), 'has_codes=8')
  refused(call(d_time=_ptr(d)), 'd_time needs a TimeEncoder')
  refused(call(count=n - 1), f'expected {n} gradient tensors')
