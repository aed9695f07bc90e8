"""Training tier at the gin model sizes: value_and_grad against torch.autograd on the oracle in
float64, every parameter tensor compared as max|a - r| / max|r|.

The golden fixtures of test_training_gpu.py have layers of at most 127 inputs and 64 outputs and
chunks of at most 240 rows, so there the training GEMM never runs a second 128-column tile, never
splits its weight-gradient reduction and the background loss never loops over chunks.  Here the
layers are 256 wide (skip layers K = 307, 283, 187), a chunk holds thousands of rows (every dW
reduction split many ways, the last slice ragged) and the background points span three chunks.

Tier A (coarse-only models, no resampling): each tensor within max(2e-4, 3 x band), the stated
tolerance of test_training_gpu.py widened only by the round-off band of the problem itself (the idea
of test_parity_gpu.py's _e2e_tol).  The band is the larger of the fp32 oracle's distance from fp64
and the distance fp64 runs move when the rays and the parameters move by fp32 round-off (see
_refs).
Tier B (both levels, the two benchmarked step configurations): the fine level resamples from the
kernel's own fp32 coarse weights (DESIGN.md §2), so the two-tier bound of test_training_gpu.py:
5e-3 for everything but nerf_mlps_fine, 2e-2 for it.

The error per tensor and case, beside both bands and its tolerance, goes to train_grad_report.json in
the directory NFB_REPORT_DIR names (default: the system's temporary directory), so that the run leaves
the source tree as it found it.
"""
import json
import os
import tempfile

import pytest
import torch

from oracle import nerfies_oracle as O
from tests.golden_util import flatten, model_from_spec, spec_to_dict, tree_to_device

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
TOL = 2e-4
_REPORT = []


@pytest.fixture(scope='module', autouse=True)
def _write_report():
  yield
  out_dir = os.environ.get('NFB_REPORT_DIR') or tempfile.gettempdir()
  os.makedirs(out_dir, exist_ok=True)
  with open(os.path.join(out_dir, 'train_grad_report.json'), 'w') as f:
    json.dump(_REPORT, f, indent=1)


# bench.py's workloads (gpu_quarterhd.gin, gpu_vrig_paper.gin, gpu_fullhd.gin model dimensions)
DIMS = {
    'quarterhd': dict(S=128, fp=8, fw=8, app=True, cam=False, alpha=8.0),
    'vrig': dict(S=128, fp=8, fw=6, app=False, cam=True, alpha=4.5),
    'fullhd': dict(S=256, fp=10, fw=8, app=True, cam=False, alpha=6.3),
}


def _spec(dims, fine):
  d = DIMS[dims]
  return O.OracleSpec(num_coarse_samples=d['S'], num_fine_samples=d['S'] if fine else 0, near=0.02, far=0.83,
                      num_nerf_point_freqs=d['fp'], num_warp_freqs=d['fw'], sigma_activation='softplus',
                      use_warp=True, warp_field_type='se3', use_appearance_metadata=d['app'],
                      use_camera_metadata=d['cam'], num_warp_embeddings=50,
                      num_appearance_embeddings=50 if d['app'] else 1, num_camera_embeddings=2 if d['cam'] else 1)


class Case:
  """One model, its trained-like parameters, rays, targets and (optionally) background points."""

  def __init__(self, dims, fine, num_rays, seed, background=0):
    self.dims, self.alpha = dims, DIMS[dims]['alpha']
    self.spec = _spec(dims, fine)
    self.params = O.make_trained_like(O.init_params(self.spec, seed), seed=seed + 1)
    self.rays = O.synthetic_rays(num_rays, self.spec, seed=seed + 2)
    gen = torch.Generator().manual_seed(seed + 3)
    self.target = torch.rand(num_rays, 3, generator=gen)
    self.bg = None
    if background:
      # noise of 0.05 rather than the default 0.001: a noise row applied to the wrong point moves the loss
      self.bg = dict(points=torch.rand(background, 3, generator=gen) * 0.6 - 0.3,
                     ids=torch.randint(0, self.spec.num_warp_embeddings, (background, 1), generator=gen),
                     noise=0.05 * torch.randn(background, 3, generator=gen))


def _oracle(c, dtype, sp=None, reg=None, rays=None, params=None):
  """Loss terms and parameter gradients of training.py:171-259 on the oracle in `dtype` (on `rays` and
  `params` instead of the case's when given).  z_fine comes from the oracle's own coarse weights in the same
  dtype and is a constant (lax.stop_gradient)."""
  reg = reg or {}
  rays = rays or c.rays
  p = {k: v.detach().clone() for k, v in flatten(O.tree_to(params or c.params, dtype)).items()}
  for v in p.values():
    v.requires_grad_(True)
  tree = {}
  for k, v in p.items():
    node = tree
    for part in k.split('/')[:-1]:
      node = node.setdefault(part, {})
    node[k.split('/')[-1]] = v
  with torch.no_grad():
    fwd = O.render_forward(tree, c.spec, rays, warp_alpha=c.alpha, dtype=dtype)
  parts, total = {}, 0.0
  for lv in ('coarse', 'fine') if c.spec.num_fine_samples else ('coarse',):
    out = O.render_level(tree, c.spec, lv, rays, fwd[lv]['z_vals'], c.alpha, dtype=dtype)
    parts['rgb_' + lv] = ((out['rgb'] - c.target.to(dtype))**2).mean()
    total = total + parts['rgb_' + lv]
    if reg.get('elastic') or reg.get('warp_reg'):
      r = O.level_regularisers(tree, c.spec, out, rays, c.alpha,
                               use_elastic_loss=reg.get('elastic', False) and lv == 'coarse',
                               elastic_reduce_method=reg.get('reduce', 'median'),
                               elastic_loss_type=reg.get('etype', 'log_svals'),
                               use_warp_reg_loss=reg.get('warp_reg', False),
                               warp_reg_loss_alpha=sp.warp_reg_loss_alpha, warp_reg_loss_scale=sp.warp_reg_loss_scale)
      if 'loss/elastic' in r:
        parts['elastic'] = r['loss/elastic']
        total = total + sp.elastic_loss_weight * r['loss/elastic']
      if 'loss/warp_reg' in r:
        parts['warp_reg_' + lv] = r['loss/warp_reg']
        total = total + sp.warp_reg_loss_weight * r['loss/warp_reg']
  if reg.get('background'):
    bg = c.bg
    l = O.compute_background_loss(tree, c.spec, bg['points'].to(dtype), bg['ids'], bg['noise'].to(dtype),
                                  c.alpha).mean()
    parts['background'] = l
    total = total + sp.background_loss_weight * l
  total.backward()
  grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)).double() for k, v in p.items()}
  return {k: float(v.detach()) for k, v in parts.items()}, grads


def _rel(a, r):
  return float((a - r).abs().max()) / (float(r.abs().max()) + 1e-30)


def _cuda(c, chunk_rays, sp=None, reg=None):
  from nerfies_b200 import training
  reg = reg or {}
  model = model_from_spec(spec_to_dict(c.spec), device=DEV)
  kw = {}
  if reg:
    bg = c.bg if reg.get('background') else None
    extra = dict(background_points=bg['points'], background_warp_ids=bg['ids'],
                 background_noise=bg['noise']) if bg else {}
    kw['reg'] = training.make_reg(model, sp, reg.get('elastic', False), reg.get('reduce', 'median'),
                                  reg.get('etype', 'log_svals'), bg is not None, reg.get('warp_reg', False), **extra)
  losses, grads = training.value_and_grad(model, tree_to_device(c.params, DEV), dict(c.rays, rgb=c.target),
                                          {'alpha': c.alpha}, chunk_rays=chunk_rays, **kw)
  torch.cuda.synchronize()
  got = flatten(training.grads_to_tree(model, grads))
  if reg.get('background'):
    # the chunk loop of train_background must run at least three times, the last chunk ragged
    max_rays = model.handle(0).max_rays
    assert c.bg['points'].shape[0] >= 2.5 * max_rays and c.bg['points'].shape[0] % max_rays
  return {k: float(v) for k, v in losses.items()}, {k: v.cpu().double() for k, v in got.items()}


_CASES = {}


def _tier_a_case(dims):
  """40 rays of a coarse-only model; the vrig one also carries 170 background points."""
  if dims not in _CASES:
    _CASES[dims] = Case(dims, False, 40, seed=100 + len(dims), background=170 if dims == 'vrig' else 0)
  return _CASES[dims]


_REFS = {}


def _rounded_inputs(c, seed):
  """float64 rays moved by up to one fp32 rounding (relative 2^-24) and parameters moved by up to 16:
  the typical backward error of the fp32 dot products of a 256-wide layer (sqrt(K) roundings) - an
  fp32 forward is an exact one with its weights moved about that much."""
  gen = torch.Generator().manual_seed(seed)
  move = lambda t, u: t.double() * (1 + u * (2 * torch.rand(t.shape, generator=gen, dtype=torch.float64) - 1))
  tree = lambda t: {k: tree(v) for k, v in t.items()} if isinstance(t, dict) else move(t, 16 * 2.0**-24)
  return (dict(c.rays, origins=move(c.rays['origins'], 2.0**-24), directions=move(c.rays['directions'], 2.0**-24)),
          tree(c.params))


def _refs(c, key, sp=None, reg=None):
  """(fp64 parts, fp64 grads, bands), cached per case.  Two round-off bands per tensor: the fp32
  oracle's distance from fp64, and how far fp64 runs move on _rounded_inputs.  The second is the
  conditioning of the loss itself: relu masks of pre-activations within round-off of zero can flip, the
  density head is steep and the encoding's top frequency is 2^7, so at the quarterhd size a different
  but equally valid fp32 rounding moves single gradients by 1e-3.  The fp32 oracle is one such
  rounding; the kernels are another (measured: nerf_mlps_coarse/MLP_0/hidden_0/kernel 1.1e-3 from
  fp64 with an fp32-oracle band of 3.2e-4, the same at every chunk size)."""
  if key not in _REFS:
    parts, g64 = _oracle(c, torch.float64, sp, reg)
    _, g32 = _oracle(c, torch.float32, sp, reg)
    bands = {k: dict(fp32_band=_rel(g32[k], g64[k]), rounding_band=0.0) for k in g64}
    for seed in (1, 2):
      rays, params = _rounded_inputs(c, seed)
      _, gr = _oracle(c, torch.float64, sp, reg, rays=rays, params=params)
      for k in g64:
        bands[k]['rounding_band'] = max(bands[k]['rounding_band'], _rel(gr[k], g64[k]))
    _REFS[key] = parts, g64, bands
  return _REFS[key]


def _compare(name, ref, bands, got, tol_of):
  bad = {}
  for k, r in ref.items():
    err = _rel(got[k].reshape(r.shape), r)
    tol = tol_of(k, bands[k])
    _REPORT.append(dict(case=name, tensor=k, err_vs_fp64=err, **bands[k], tol=tol))
    if not err <= tol:
      bad[k] = (err, tol)
  assert not bad, f'{name}: {bad}'


def _tier_a_tol(k, band):
  return max(TOL, 3.0 * max(band['fp32_band'], band['rounding_band']))


# ---------------------------------------------------------------------------
# Tier A: coarse-only models, photometric loss, every tensor at max(2e-4, 3 x round-off band)
# ---------------------------------------------------------------------------
@pytest.mark.parametrize('chunk', [40, 17])        # one chunk; 17 + 17 + 6
@pytest.mark.parametrize('dims', ['quarterhd', 'vrig', 'fullhd'])
def test_photometric_gradients_at_gin_sizes(dims, chunk):
  c = _tier_a_case(dims)
  parts, ref, band = _refs(c, (dims, 'photometric'))
  losses, got = _cuda(c, chunk)
  assert abs(losses['coarse'] - parts['rgb_coarse']) < 1e-5 * parts['rgb_coarse'], (losses['coarse'], parts)
  _compare(f'{dims} photometric chunk={chunk}', ref, band, got, _tier_a_tol)


_REG_SP = dict(learning_rate=1e-3, elastic_loss_weight=5.0, warp_reg_loss_weight=3.0, warp_reg_loss_alpha=-2.0,
               warp_reg_loss_scale=0.05, background_loss_weight=60.0)


@pytest.mark.parametrize('reg', [
    dict(elastic=True, reduce='weight', etype='log_svals'),     # vrig-trainstep's elastic loss
    dict(elastic=True, reduce='median', etype='svals'),
    dict(elastic=True, reduce='median', etype='det'),
    dict(warp_reg=True),
    dict(background=True),
], ids=lambda r: '-'.join(f'{k}={v}' for k, v in r.items()))
def test_regulariser_gradients_at_gin_sizes(reg):
  """vrig dimensions with each regulariser at a weight that dominates the warp field's gradient; 170
  background points against a 64-ray handle: chunks of 64, 64 and 42."""
  from nerfies_b200 import training
  sp = training.ScalarParams(**_REG_SP)
  c = _tier_a_case('vrig')
  key = '-'.join(f'{k}={v}' for k, v in reg.items())
  parts, ref, band = _refs(c, ('vrig', key), sp, reg)
  # the check must be able to fail: the regulariser moves the reference gradient of the warp field by far
  # more than the tolerance
  _, plain, _ = _refs(c, ('vrig', 'photometric'))
  moved = max(_rel(ref[k], plain[k]) for k in ref if k.startswith('warp_field/'))
  assert moved > 0.25, moved
  losses, got = _cuda(c, 17, sp, reg)
  assert abs(losses['coarse'] - parts['rgb_coarse']) < 1e-5 * parts['rgb_coarse']
  for k in ('elastic', 'warp_reg_coarse', 'background'):
    if k in parts:
      assert abs(losses[k] - parts[k]) < 2e-4 * max(abs(parts[k]), 1e-3), (k, losses[k], parts[k])
  _compare(f'vrig {key} chunk=17', ref, band, got, _tier_a_tol)


# ---------------------------------------------------------------------------
# Tier B: the two benchmarked step configurations, both levels, end to end
# ---------------------------------------------------------------------------
def _tier_b_tol(k, band):
  return 2e-2 if 'nerf_mlps_fine' in k else 5e-3


@pytest.mark.parametrize('workload', ['quarterhd-trainstep', 'vrig-trainstep'])
def test_benchmarked_step_end_to_end(workload):
  from nerfies_b200 import training
  if workload == 'quarterhd-trainstep':
    c = Case('quarterhd', True, 24, seed=200)
    sp, reg = None, {}
  else:
    c = Case('vrig', True, 24, seed=210, background=170)
    sp = training.ScalarParams(**_REG_SP)
    reg = dict(elastic=True, reduce='weight', etype='log_svals', background=True)
  parts, ref, band = _refs(c, (workload,), sp, reg)
  losses, got = _cuda(c, 24, sp, reg)
  assert abs(losses['coarse'] - parts['rgb_coarse']) < 1e-5 * parts['rgb_coarse']
  for k in ('elastic', 'background'):
    if k in parts:
      assert abs(losses[k] - parts[k]) < 2e-4 * max(abs(parts[k]), 1e-3), (k, losses[k], parts[k])
  _compare(f'{workload} both levels', ref, band, got, _tier_b_tol)
