"""Volumetric rendering, median depth, resampling and their adjoints at the densities of a trained scene.

make_trained_like networks are soft everywhere (sigma * dist ~ 1e-2).  A trained scene has opaque surfaces
where alpha rounds to 1.0f, empty space where the weights are exactly 0, and delta-shaped weights that pile the
fine samples into one or two bins.  Those regimes are built here from a designed-density model: the default
NeRF architecture (trunk 8 x 256 with skip 4, bottleneck, rgb branch, MLP_2 alpha head) with weights that make
density and colour chosen piecewise-linear functions of the sample's z coordinate:

- hidden unit k of the first trunk layer is relu(x_z - knot_k); every later trunk layer and the bottleneck pass
  those units through (identity kernel rows, relu of a non-negative value is exact);
- sigma = relu(alpha_b + sum_k alpha_w[k] h_k), rgb = sigmoid(rgb_b + sum_k rgb_w[k] h_k); every other kernel
  entry (positional encoding, skip input, conditions) is 0.

Rays run along +z (with a small tilt), so a ray's origin places the profile relative to its samples.  Kernel
weights are 0 or 1 except in the alpha head, which the tensor-core kernels evaluate in fp32, so the fp16x3 split
is exact apart from the input coordinate's.  The reference is the oracle in fp64 on the z values the kernels
used; tolerances are TOL + 2 x the fp32 oracle's distance from fp64, as in test_parity_gpu.test_levels_vs_oracle.

The median depth is held to one rule in every mode: it is exactly one of the ray's z values - the first whose
fp64 cumulative sum of the kernel's own weights reaches 0.5, or any sample whose cumulative sum is within 1e-6
of 0.5 - or 0 when the ray's total weight is below 0.5 + 1e-6.
"""
import numpy as np
import pytest
import torch

from nerfies_b200 import _lib
from nerfies_b200.models import _prep_ids, _ptr, _stream
from oracle import nerfies_oracle as O
from tests.golden_util import flatten, med_depth_rule_ok, model_from_spec, rel_err, spec_to_dict, tree_to_device

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
TOL = 1e-4
GRAD_TOL = 2e-4
NEAR, FAR = 0.02, 0.83
SLAB_GAPS = 24


# ---------------------------------------------------------------------------
# The designed-density model and its rays
# ---------------------------------------------------------------------------
def _spec(nc, nf, **kw):
  return O.OracleSpec(num_coarse_samples=nc, num_fine_samples=nf, near=NEAR, far=FAR, num_nerf_point_freqs=8,
                      sigma_activation='relu', **kw)


def designed_params(spec, knots, alpha_w, alpha_b, rgb_w, rgb_b):
  """Parameters of `spec` (default NeRF architecture) with sigma and rgb piecewise linear in x_z (module doc).
  With a translation warp field its output layer is 0: the warp is the identity."""
  def zeros(t):
    return {k: zeros(v) for k, v in t.items()} if isinstance(t, dict) else torch.zeros_like(t)
  p = zeros(O.init_params(spec, 0))
  K = len(knots)
  assert K <= spec.nerf_rgb_branch_width and spec.nerf_trunk_width >= K
  u = torch.arange(K)
  for lv in ('coarse', 'fine')[:1 + (spec.num_fine_samples > 0)]:
    m = p[f'nerf_mlps_{lv}']
    t = m['MLP_0']
    t['hidden_0']['kernel'][2, u] = 1.0                       # the identity x_z column of the encoding
    t['hidden_0']['bias'][:K] = -torch.tensor(knots, dtype=torch.float32)
    for i in range(1, spec.nerf_trunk_depth):
      t[f'hidden_{i}']['kernel'][u, u] = 1.0                  # skip layers: the trunk rows come first
    if 'bottleneck' in m:
      m['bottleneck']['kernel'][u, u] = 1.0
    m['MLP_1']['hidden_0']['kernel'][u, u] = 1.0              # the bottleneck rows come first
    m['MLP_1']['logit']['kernel'][:K] = torch.tensor(rgb_w, dtype=torch.float32)
    m['MLP_1']['logit']['bias'][:] = torch.tensor(rgb_b, dtype=torch.float32)
    m['MLP_2']['logit']['kernel'][:K, 0] = torch.tensor(alpha_w, dtype=torch.float32)
    m['MLP_2']['logit']['bias'][:] = alpha_b
  return p


def _gap(S):
  """The coarse sample spacing in z (and in x_z for rays with d_z = 1)."""
  return (FAR - NEAR) / (S - 1)


def _rgb_w(K, seed):
  gen = torch.Generator().manual_seed(seed)
  return ((torch.rand(K, 3, generator=gen) * 2 - 1) * 20).tolist()


# Profiles around x_z = 0.5.  A negative bias makes sigma exactly 0 wherever the units' sum is 0 up to round-off.
def profile(regime, S):
  g = _gap(S)
  if regime == 'wall':
    # 0 before 0.5, a ramp over 0.1 gap, then sigma * gap = 64: alpha == 1.0f behind the wall
    A, e = 64.0 / g, 0.1 * g
    knots, aw = [0.5, 0.5 + e], [A / e, -A / e]
  elif regime == 'empty':
    knots, aw = [0.5], [0.0]
  elif regime == 'shell':
    # a hat of half-width 0.45 gap with sigma * gap = 8 at its centre: one sample holds almost all the weight.
    # (Its slopes of ~1e6 turn the units' round-off behind it into |sigma| ~ 1: the bias keeps that at 0.)
    P, h = 8.0 / g, 0.45 * g
    knots, aw = [0.5 - h, 0.5, 0.5 + h], [P / h, -2 * P / h, P / h]
    return dict(knots=knots, alpha_w=aw, alpha_b=-10.0, rgb_w=_rgb_w(3, 7), rgb_b=[0.3, -0.2, 0.1])
  elif regime == 'slab':
    # SLAB_GAPS + 1 samples: a trapezoid from 0.5 with ramps one gap wide, the sum of SLAB_GAPS hats spaced by
    # the gap, so sum_i (sigma_i + b) dist_i = P SLAB_GAPS gap |d| whatever the samples' offset; ln 2 at a
    # tilt of 0.05: total opacity 0.5
    n, b = SLAB_GAPS, 1e-2
    P = (np.log(2.0) / (g * np.sqrt(1 + 0.05**2)) + (n + 1) * b) / n
    knots, aw = [0.5, 0.5 + g, 0.5 + n * g, 0.5 + (n + 1) * g], [P / g, -P / g, -P / g, P / g]
    return dict(knots=knots, alpha_w=aw, alpha_b=-b, rgb_w=_rgb_w(4, 7), rgb_b=[0.3, -0.2, 0.1])
  else:
    raise ValueError(regime)
  return dict(knots=knots, alpha_w=aw, alpha_b=-1.0, rgb_w=_rgb_w(len(knots), 7), rgb_b=[0.3, -0.2, 0.1])


def make_rays(S, pos, tilt=1e-3, seed=0):
  """Rays along +z with direction (tx, ty, 1): coarse sample position pos[b] (an index, fractional between
  samples) of ray b sits at x_z = 0.5.  |(tx, ty)| = tilt[b] (or uniform in [0, tilt))."""
  B = len(pos)
  gen = torch.Generator().manual_seed(seed)
  pos = torch.as_tensor(pos, dtype=torch.float64)
  phi = torch.rand(B, generator=gen, dtype=torch.float64) * 2 * np.pi
  rho = (torch.as_tensor(tilt, dtype=torch.float64).expand(B) if np.ndim(tilt)
         else torch.rand(B, generator=gen, dtype=torch.float64) * tilt)
  t = NEAR + pos * _gap(S)
  oxy = torch.rand(B, 2, generator=gen, dtype=torch.float64) * 0.2 - 0.1
  origins = torch.stack([oxy[:, 0], oxy[:, 1], 0.5 - t], -1).float()
  directions = torch.stack([rho * torch.cos(phi), rho * torch.sin(phi), torch.ones(B, dtype=torch.float64)],
                           -1).float()
  md = {k: torch.zeros(B, 1, dtype=torch.int32) for k in ('warp', 'appearance', 'camera')}
  return {'origins': origins, 'directions': directions, 'metadata': md}


def _cpu(rays):
  return {k: ({a: b.cpu() for a, b in v.items()} if isinstance(v, dict) else v.cpu()) for k, v in rays.items()}


# ---------------------------------------------------------------------------
# The kernels through the C ABI
# ---------------------------------------------------------------------------
def _level(o6, w, z):
  return {'rgb': o6[:, :3].cpu(), 'depth': o6[:, 3].cpu(), 'med_depth': o6[:, 4].cpu(), 'acc': o6[:, 5].cpu(),
          'weights': w.cpu(), 'z_vals': z.cpu()}


def _ids(rays):
  return _prep_ids(rays['metadata']['warp'].to(DEV), DEV)


# (Every tensor handed to the C ABI is held by a name until the launches are synchronised: a temporary's memory
#  could be handed to the next allocation of the same call's arguments.)

def render_forward(model, params, rays, u_rand=None):
  """nfb_render_forward (the fp16x3 kernel finishes rays of whole 128-sample tiles on chip) -> per level."""
  B = rays['origins'].shape[0]
  hd = model.handle(B)
  hd.set_params(params)
  nc, nf = model.num_coarse_samples, model.num_fine_samples
  o, d = rays['origins'].to(DEV).contiguous(), rays['directions'].to(DEV).contiguous()
  out_c, w_c, z_c = (torch.empty(B, 6, device=DEV), torch.empty(B, nc, device=DEV),
                     torch.empty(B, nc, device=DEV))
  out_f = w_f = z_f = None
  if nf:
    out_f, w_f, z_f = (torch.empty(B, 6, device=DEV), torch.empty(B, nc + nf, device=DEV),
                       torch.empty(B, nc + nf, device=DEV))
  u = None if u_rand is None else u_rand.to(DEV).contiguous()
  ids = _ids(rays)
  _lib.check(hd.lib.nfb_render_forward(hd.h, B, _ptr(o), _ptr(d), None, _ptr(ids), None, None, 0.0, None,
                                       _ptr(u), 0, _ptr(out_c), _ptr(out_f), _ptr(w_c), _ptr(w_f), _ptr(z_f),
                                       _stream()))
  _lib.check(hd.lib.nfb_coarse_z_vals(hd.h, B, None, _ptr(z_c), _stream()))
  torch.cuda.synchronize()
  out = {'coarse': _level(out_c, w_c, z_c)}
  if nf:
    out['fine'] = _level(out_f, w_f, z_f)
  return out


def render_samples(model, params, level, rays, z):
  """nfb_render_samples: the field at z, then composite_kernel (every mode)."""
  B, S = z.shape
  hd = model.handle(B)
  hd.set_params(params)
  o, d = rays['origins'].to(DEV).contiguous(), rays['directions'].to(DEV).contiguous()
  zc = z.to(DEV).float().contiguous()
  out, w = torch.empty(B, 6, device=DEV), torch.empty(B, S, device=DEV)
  smp = torch.empty(B, S, 4, device=DEV)
  ids = _ids(rays)
  _lib.check(hd.lib.nfb_render_samples(hd.h, level, B, S, _ptr(zc), _ptr(o), _ptr(d), None, _ptr(ids),
                                       None, None, 0.0, 0, _ptr(out), _ptr(w), _ptr(smp), None, _stream()))
  torch.cuda.synchronize()
  return _level(out, w, zc)


# ---------------------------------------------------------------------------
# Checks
# ---------------------------------------------------------------------------
def assert_median(level, what):
  bad = ~med_depth_rule_ok(level['med_depth'], level['weights'], level['z_vals'])
  n = int(bad.sum())
  if n:
    b = int(bad.nonzero()[0])
    cum = torch.cumsum(level['weights'][b].double(), -1)
    j = int((cum >= 0.5).int().argmax())
    raise AssertionError(
        f'{what}: med_depth breaks the first-sample-reaching-0.5 rule on {n} of {bad.numel()} rays; ray {b}: '
        f'med_depth {float(level["med_depth"][b])!r}, z[{j}] = {float(level["z_vals"][b, j])!r}, cumulative '
        f'weight there {float(cum[j]) - 0.5:+.3e} from 0.5, total {float(cum[-1]) - 0.5:+.3e} from 0.5')


def assert_invariants(level, what, white_bg=False):
  for k in ('rgb', 'depth', 'acc', 'weights'):
    assert bool(torch.isfinite(level[k]).all()), f'{what}/{k} not finite'
  w = level['weights']
  assert float(w.min()) >= 0, what
  assert float(level['acc'].max()) <= 1 + 1e-5, what
  assert float(level['rgb'].min()) >= 0 and float(level['rgb'].max()) <= 1 + 1e-5, what
  z = level['z_vals']
  assert bool((z[:, 1:] >= z[:, :-1]).all()), f'{what}: z not sorted'
  assert_median(level, what)


def assert_vs_fp64(got, p, spec, level, rays, what):
  """rgb, depth, acc, weights against the oracle in fp64 on the kernel's z: TOL + 2 x the fp32 band."""
  z = got['z_vals']
  r64 = O.render_level(p, spec, level, rays, z, 0.0, dtype=torch.float64)
  r32 = O.render_level(p, spec, level, rays, z, 0.0)
  for k in ('rgb', 'depth', 'acc', 'weights'):
    band = rel_err(r32[k], r64[k])
    err = rel_err(got[k], r64[k])
    assert err < TOL + 2 * band, f'{what}/{k}: err vs fp64 {err:.3e}, fp32 band {band:.3e}'


def cdf_bound(w, z_mid, z):
  """Bound on pdf_cdf_residual of samples z drawn from coarse weights w (Nc,) over bins z_mid: three times the
  distance of resample_kernel's fp32 cdf (emulated) from fp64 (a sample sits between two fp32 knots), two fp32
  roundings of z times the bin's density, and where the reference's plateau rule applies (a bin of mass below
  1e-5, model_utils.py:176) the bin's mass: there the samples move linearly in u across the bin."""
  ww = w[1:-1].double() + 1e-5
  mass = ww / ww.sum()
  cdf = torch.cat([torch.zeros(1, dtype=torch.float64), torch.cumsum(mass, 0)])
  err = float((torch.from_numpy(_cdf_f32(w.numpy()).astype(np.float64)) - cdf).abs().max())
  j = (torch.searchsorted(z_mid.contiguous(), z.clamp(z_mid[0], z_mid[-1]).contiguous(), right=True) - 1)
  j = j.clamp(0, len(z_mid) - 2)
  density = mass[j] / (z_mid[j + 1] - z_mid[j])
  return (1e-6 + 3 * err + density * 2 * 2.0**-23 * z.abs()
          + torch.where(mass[j] < 1.1e-5, 1.1e-5, 0.0))


def assert_resampled(coarse, fine, u, what):
  """The fine level's new samples in CDF space against the kernel's own coarse weights (pdf_cdf_residual)."""
  zc, wc, zf = coarse['z_vals'].double(), coarse['weights'], fine['z_vals']
  z_mid = .5 * (zc[:, 1:] + zc[:, :-1])
  for b in range(zc.shape[0]):
    union = zf[b].tolist()
    for v in coarse['z_vals'][b].tolist():
      union.remove(min(union, key=lambda x: abs(x - v)))
    z_new = torch.tensor(sorted(union), dtype=torch.float64)
    ub = torch.sort(u[b].double()).values
    res = O.pdf_cdf_residual(z_mid[b:b + 1], wc[b:b + 1, 1:-1], z_new[None], ub[None])[0]
    bound = cdf_bound(wc[b], z_mid[b], z_new)
    assert bool((res <= bound).all()), (what, b, float((res - bound).max()))


# ---------------------------------------------------------------------------
# 1. Forward: opaque wall, empty ray, thin shell
# ---------------------------------------------------------------------------
def _sweep(regime, S, nf):
  """Ray positions of the profile: walls across lanes 31|32, tile 127|128 and, on the fine level, the fine
  tile boundary; shells centred on samples there."""
  idx = [5, 29, 30, 31, 32, 33, 62, 63, 95, 96, 110, 115, 120, S - 8]
  if S >= 256:
    idx += [124, 126, 127, 128, 129, 160, 191, 192, 220, 235, 245, 249]
  idx = sorted(i for i in set(idx) if i <= S - 7)
  if regime == 'wall':
    frac = np.linspace(0.3, 0.7, 17)
  elif regime == 'shell':
    frac = np.linspace(-0.1, 0.1, 5)
  else:
    frac = np.linspace(0.0, 0.9, 4)
  return [i + f for i in idx for f in frac]


# (Nc, Nf): fp16x3 fuses the composite of both levels for 128+128 and 256+256 and of neither for 64+32
SIZES = [(128, 128), (256, 256), (64, 32)]


@pytest.mark.parametrize('sizes', SIZES, ids=lambda s: f'{s[0]}+{s[1]}')
@pytest.mark.parametrize('regime', ['wall', 'empty', 'shell'])
@pytest.mark.parametrize('precision', ['fp32', 'fp16x3', 'bf16'])
def test_regimes_forward(precision, regime, sizes):
  nc, nf = sizes
  spec = _spec(nc, nf, use_white_background=regime == 'empty')
  p = designed_params(spec, **profile(regime, nc))
  rays = make_rays(nc, _sweep(regime, nc, nf), seed=nc)
  B = rays['origins'].shape[0]
  model = model_from_spec(spec_to_dict(spec), precision=precision, device=DEV, batch_size=B)
  pg = tree_to_device(p, DEV)
  fused = render_forward(model, pg, rays)
  u = torch.from_numpy(np.linspace(0., 1., nf, dtype=np.float32)).expand(B, -1)
  for lv, level in ((0, 'coarse'), (1, 'fine')):
    staged = render_samples(model, pg, lv, rays, fused[level]['z_vals'])
    for path, got in (('forward', fused[level]), ('staged', staged)):
      what = f'{precision} {regime} {nc}+{nf} {path} {level}'
      assert_invariants(got, what)
      if precision != 'bf16':
        assert_vs_fp64(got, p, spec, level, rays, what)
  assert_resampled(fused['coarse'], fused['fine'], u, f'{precision} {regime} {nc}+{nf}')

  c, f = fused['coarse'], fused['fine']
  if precision == 'bf16' and regime != 'empty':
    return
  if regime == 'empty':
    for lv in (c, f):
      for k in ('acc', 'depth', 'med_depth', 'weights'):
        assert bool((lv[k] == 0).all()), k
      assert bool((lv['rgb'] == 1).all())
  elif regime == 'wall':
    # the first opaque coarse sample is at the position the ray put it, and nothing leaks past the wall
    first = (c['weights'] > 0.5).int().argmax(-1)
    assert torch.equal(first, torch.tensor([int(s) + 1 for s in _sweep('wall', nc, nf)]))
    assert float((c['acc'] - 1).abs().max()) < 1e-6 and float((f['acc'] - 1).abs().max()) < 1e-6
    if nc % 128 == 0:
      # the new samples in front of the wall move it 0 to 0.2 Nf samples up the fine level: the sweep puts it
      # on each side of the fine level's tile boundaries
      fwall = (torch.cumsum(f['weights'].double(), -1) >= 0.5).int().argmax(-1)
      for edge in (128, 256)[:nc // 128]:
        assert bool(((fwall >= edge - 2) & (fwall < edge)).any()), (edge, fwall.unique())
        assert bool(((fwall >= edge) & (fwall < edge + 2)).any()), (edge, fwall.unique())
  elif regime == 'shell':
    wmax = c['weights'].max(-1).values
    assert float(wmax.min()) > 0.99
    # every new sample of the fine level lies in the shell sample's two bins
    zc = c['z_vals']
    i = c['weights'].argmax(-1)
    lo = zc.gather(1, (i - 1)[:, None]).double()
    hi = zc.gather(1, (i + 1)[:, None]).double()
    inside = (f['z_vals'] >= lo) & (f['z_vals'] <= hi)
    assert bool((inside.sum(-1) >= nf - 2).all())     # (u = 0 and u = 1 go to the ends of the grid)


def test_fine_level_with_an_identity_warp_reuses_tied_samples():
  """The warped model's fine level warps only its new samples and gathers the coarse ones by their index in
  the sorted union (ResampleArgs::src); behind a thin shell many new samples sit in one bin.  The identity warp
  makes the result the unwarped model's."""
  nc = nf = 128
  prof = profile('shell', nc)
  kw = dict(use_warp=True, warp_field_type='translation', num_warp_embeddings=1)
  spec_w, spec = _spec(nc, nf, **kw), _spec(nc, nf)
  rays = make_rays(nc, _sweep('shell', nc, nf), seed=3)
  B = rays['origins'].shape[0]
  for precision in ('fp32', 'fp16x3'):
    outs = []
    for s in (spec_w, spec):
      model = model_from_spec(spec_to_dict(s), precision=precision, device=DEV, batch_size=B)
      outs.append(render_forward(model, tree_to_device(designed_params(s, **prof), DEV), rays))
    for level in ('coarse', 'fine'):
      for k in ('rgb', 'depth', 'med_depth', 'acc', 'weights', 'z_vals'):
        assert torch.equal(outs[0][level][k], outs[1][level][k]), (precision, level, k)
    assert_invariants(outs[0]['fine'], f'{precision} warped fine')


# ---------------------------------------------------------------------------
# 2. Median depth at half opacity
# ---------------------------------------------------------------------------
def _slab_rays(S, n=3000, seed=11):
  """n rays through the slab, its last sample at any lane of any quarter and tile; tilts 0.05 * (1 +- 3.5e-3)
  move the total opacity over 0.5 +- ~3e-6."""
  gen = torch.Generator().manual_seed(seed)
  last = torch.randint(SLAB_GAPS + 2, S - 4, (n,), generator=gen)
  frac = 0.05 + 0.9 * torch.rand(n, generator=gen, dtype=torch.float64)
  pos = last.double() - SLAB_GAPS - 1 + frac      # the slab starts at pos: its last sample is `last`
  tilt = 0.05 * (1 + (torch.rand(n, generator=gen, dtype=torch.float64) * 2 - 1) * 3.5e-3)
  return make_rays(S, pos, tilt=tilt, seed=seed)


@pytest.mark.parametrize('path', ['forward', 'staged'])
@pytest.mark.parametrize('S', [128, 256])
@pytest.mark.parametrize('precision', ['fp32', 'fp16x3', 'bf16'])
def test_median_depth_at_half_opacity(precision, S, path):
  spec = _spec(S, 0)
  p = designed_params(spec, **profile('slab', S))
  rays = _slab_rays(S)
  B = rays['origins'].shape[0]
  model = model_from_spec(spec_to_dict(spec), precision=precision, device=DEV, batch_size=B)
  pg = tree_to_device(p, DEV)
  got = render_forward(model, pg, rays)['coarse']
  if path == 'staged':
    got = render_samples(model, pg, 0, rays, got['z_vals'])
  what = f'{precision} S={S} {path}'
  total = got['weights'].double().sum(-1)
  if precision != 'bf16':      # (bf16's densities move the total off 0.5)
    near = int(((total - 0.5).abs() <= 2.0**-22).sum())
    assert near >= 100, f'{what}: only {near} rays within 2^-22 of total weight 0.5'
  if precision != 'bf16':
    # exact zeros behind the slab, so the cumulative weight plateaus at the ray's total
    assert bool((got['weights'][:, -4:] == 0).all())
  assert_invariants(got, what)
  if precision != 'bf16':
    sub = slice(0, B, 10)
    assert_vs_fp64({k: v[sub] for k, v in got.items()}, p, spec, 'coarse',
                   {k: (v[sub] if torch.is_tensor(v) else {a: b[sub] for a, b in v.items()})
                    for k, v in rays.items()}, what)


# ---------------------------------------------------------------------------
# 3. nfb_sample_pdf on hand-built weights
# ---------------------------------------------------------------------------
def _cdf_f32(w):
  """resample_kernel's fp32 cdf (sequential sums, no fma) of coarse weights w (Nc,)."""
  x = (np.asarray(w, np.float32)[1:-1] + np.float32(1e-5)).astype(np.float32)
  total = np.float32(0)
  for v in x:
    total = np.float32(total + v)
  c, out = np.float32(0), [np.float32(0)]
  for v in x:
    c = np.float32(c + np.float32(v / total))
    out.append(c)
  return np.array(out, np.float32)


def _weights_with_last_cdf(nc, target, seed):
  """Coarse weights whose fp32 cdf ends exactly at `target`."""
  rng = np.random.default_rng(seed)
  for _ in range(20000):
    w = np.zeros(nc, np.float32)
    k = rng.integers(1, 6)
    w[rng.choice(np.arange(1, nc - 1), k, replace=False)] = rng.random(k).astype(np.float32)
    if _cdf_f32(w)[-1] == target:
      return w
  raise AssertionError(f'no weights found with a last cdf entry of {target!r}')


def _hand_weights(nc):
  one, below = np.float32(1.0), np.nextafter(np.float32(1.0), np.float32(0.0))   # 0.99999994
  rows = {'zeros': np.zeros(nc, np.float32)}
  d = np.zeros(nc, np.float32); d[1] = 1.0; rows['delta_first_bin'] = d
  d = np.zeros(nc, np.float32); d[nc - 2] = 1.0; rows['delta_last_bin'] = d
  d = np.zeros(nc, np.float32); d[nc // 3] = 0.7; d[nc // 3 + 5] = 0.3; rows['two_deltas'] = d
  rows['cdf_ends_at_1'] = _weights_with_last_cdf(nc, one, 1)
  rows['cdf_ends_below_1'] = _weights_with_last_cdf(nc, below, 2)
  return rows


@pytest.mark.parametrize('draws', ['linspace', 'stratified'])
@pytest.mark.parametrize('sizes', [(64, 64), (128, 128), (64, 32)], ids=lambda s: f'{s[0]}+{s[1]}')
def test_sample_pdf_on_hand_built_weights(sizes, draws):
  nc, nf = sizes
  spec = _spec(nc, nf)
  rows = _hand_weights(nc)
  names = list(rows)
  w = torch.from_numpy(np.stack([rows[k] for k in names]))
  B = w.shape[0]
  zc = O.coarse_z_vals(nc, NEAR, FAR, False)[None].expand(B, -1).contiguous()
  if draws == 'linspace':
    u, u_dev = torch.from_numpy(np.linspace(0., 1., nf, dtype=np.float32)).expand(B, -1), None
  else:
    gen = torch.Generator().manual_seed(5)
    u = torch.rand(B, nf, generator=gen)
    u[:, 0] = 0.0                                     # u = 0 and the largest u below 1
    u[:, 1] = float(np.nextafter(np.float32(1.0), np.float32(0.0)))
    u_dev = u.to(DEV).contiguous()
  model = model_from_spec(spec_to_dict(spec), device=DEV, batch_size=B)
  hd = model.handle(B)
  hd.set_params(tree_to_device(designed_params(spec, **profile('empty', nc)), DEV))
  zf = torch.empty(B, nc + nf, device=DEV)
  zc_dev, w_dev = zc.to(DEV), w.to(DEV).contiguous()
  _lib.check(hd.lib.nfb_sample_pdf(hd.h, B, _ptr(zc_dev), _ptr(w_dev), _ptr(u_dev), _ptr(zf), _stream()))
  torch.cuda.synchronize()
  zf = zf.cpu()
  assert bool(torch.isfinite(zf).all())
  assert bool((zf[:, 1:] >= zf[:, :-1]).all()), 'z_fine not sorted'
  for b, name in enumerate(names):
    # the bin of each new sample against the fp64 cdf, except where u is within 1e-6 of a cdf knot
    z_mid = .5 * (zc[b, 1:].double() + zc[b, :-1].double())
    ww = w[b, 1:-1].double() + 1e-5
    cdf = torch.cat([torch.zeros(1, dtype=torch.float64), torch.cumsum(ww / ww.sum(), 0)])
    union = zf[b].tolist()
    for v in zc[b].tolist():
      union.remove(min(union, key=lambda x: abs(x - v)))
    z_new = torch.tensor(sorted(union), dtype=torch.float64)
    us = torch.sort(u[b].double()).values
    j = (torch.searchsorted(cdf.contiguous(), us.contiguous(), right=True) - 1).clamp(0, nc - 3)
    clear = (us[:, None] - cdf[None]).abs().min(-1).values > 1e-6
    lo, hi = z_mid[j], z_mid[j + 1]
    eps = 1e-6 * (FAR - NEAR)
    inside = (z_new >= lo - eps) & (z_new <= hi + eps)
    assert bool((inside | ~clear).all()), (name, draws, int((~inside & clear).sum()))
    res = O.pdf_cdf_residual(z_mid[None], w[b:b + 1, 1:-1], z_new[None], us[None])[0]
    bound = cdf_bound(w[b], z_mid, z_new)
    assert bool((res <= bound).all()), (name, draws, float((res - bound).max()))
    if name == 'zeros':
      # uniform pdf: the new samples are the inverse of a straight cdf, bins spaced evenly
      zl = z_mid[0] + us * (z_mid[-1] - z_mid[0])
      assert float((z_new - zl).abs().max()) < 1e-5 * (FAR - NEAR), name


# ---------------------------------------------------------------------------
# 4. Backward at fixed z: composite_vjp_kernel seeded by the photometric loss and by given cotangents
# ---------------------------------------------------------------------------
def _grad_case(regime):
  S = 128
  spec = _spec(S, 0)
  p = designed_params(spec, **profile(regime, S))
  if regime == 'slab':
    pos = [i - SLAB_GAPS - 1 + f for i in (31, 60, 120) for f in np.linspace(0.05, 0.95, 5)]
    rays = make_rays(S, pos, tilt=0.05, seed=21)
  else:
    pos = [i + f for i in (30, 31, 64, 100) for f in (0.35, 0.5, 0.65)]
    rays = make_rays(S, pos, seed=21)
  return spec, p, rays


def _autograd64(spec, p, rays, loss_fn):
  p64 = {k: v.double().clone().requires_grad_(True) for k, v in flatten(p).items()}
  tree = {}
  for k, v in p64.items():
    node = tree
    for part in k.split('/')[:-1]:
      node = node.setdefault(part, {})
    node[k.split('/')[-1]] = v
  z = O.coarse_z_vals(spec.num_coarse_samples, NEAR, FAR, False)[None].expand(rays['origins'].shape[0], -1)
  out = O.render_level(tree, spec, 'coarse', rays, z, 0.0, dtype=torch.float64)
  loss = loss_fn(out)
  loss.backward()
  return float(loss), {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in p64.items()}


def _assert_grads(got, ref, what):
  for k, r in ref.items():
    a = got[k].cpu().double().reshape(r.shape)
    assert bool(torch.isfinite(a).all()), f'{what}: {k} not finite'
    err = float((a - r).abs().max()) / (float(r.abs().max()) + 1e-30)
    if float(r.abs().max()) == 0:
      assert float(a.abs().max()) == 0, f'{what}: {k} should be 0, max {float(a.abs().max()):.3e}'
    else:
      assert err < GRAD_TOL, f'{what}: {k} err {err:.3e}'


@pytest.mark.parametrize('regime', ['wall', 'empty', 'slab'])
def test_value_and_grad_at_extremes(regime):
  from nerfies_b200 import training
  spec, p, rays = _grad_case(regime)
  B = rays['origins'].shape[0]
  target = torch.rand(B, 3, generator=torch.Generator().manual_seed(4))
  loss64, ref = _autograd64(spec, p, rays, lambda o: ((o['rgb'] - target.double())**2).mean())
  model = model_from_spec(spec_to_dict(spec), device=DEV, batch_size=B)
  losses, grads = training.value_and_grad(model, tree_to_device(p, DEV), dict(_cpu(rays), rgb=target),
                                          {'alpha': 0.0}, chunk_rays=7)
  torch.cuda.synchronize()
  assert abs(float(losses['coarse']) - loss64) < 1e-5 * max(1.0, loss64)
  _assert_grads(flatten(training.grads_to_tree(model, grads)), ref, f'value_and_grad {regime}')


@pytest.mark.parametrize('train_precision', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('regime', ['wall', 'empty', 'slab'])
def test_apply_backward_at_extremes(regime, train_precision):
  spec, p, rays = _grad_case(regime)
  B, S = rays['origins'].shape[0], spec.num_coarse_samples
  gen = torch.Generator().manual_seed(9)
  cot = {'rgb': torch.randn(B, 3, generator=gen, dtype=torch.float64),
         'depth': torch.randn(B, generator=gen, dtype=torch.float64),
         'acc': torch.randn(B, generator=gen, dtype=torch.float64),
         'weights': torch.randn(B, S, generator=gen, dtype=torch.float64)}
  dot = lambda o: sum((o[k].double() * g.to(o[k].device)).sum() for k, g in cot.items())
  _, ref = _autograd64(spec, p, rays, dot)
  model = model_from_spec(spec_to_dict(spec), device=DEV, batch_size=B)
  model.train_precision = train_precision
  params = tree_to_device(p, DEV)
  leaves = flatten(params)
  for v in leaves.values():
    v.requires_grad_(True)
  out = model.apply({'params': params}, tree_to_device(rays, DEV), return_weights=True)
  dot(out['coarse']).backward()
  torch.cuda.synchronize()
  got = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaves.items()}
  _assert_grads(got, ref, f'apply backward {regime} {train_precision}')
