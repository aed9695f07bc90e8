"""Training with the 'time' and 'blend' warp metadata encoders: the TimeEncoder's adjoint in the training step.

The TimeEncoder (modules.py:297-322) runs on a tape of its own through the training GEMMs; the gradient of the
condition vectors' warp block reaches its Dense layers ('time'), or is split between the GLO rows and the
TimeEncoder by (1 - time_alpha) and time_alpha ('blend').  Gradients are held to fp64 autograd on the oracle,
in both training precisions, with the tolerances of test_training_gpu.py (golden fixtures) and
test_training_scale_gpu.py (tier A at the gin sizes).  The oracle wrappers here forward time_alpha, which
those modules' helpers do not.

The last test checks the oracle's TimeEncoder regularisers against tests/golden/time_regularisers.npz (made by
oracle/make_golden_time_reg.py from the reference's own source) and needs no GPU.
"""
import dataclasses
import os
import types

import numpy as np
import pytest
import torch

from oracle import nerfies_oracle as O
from tests.golden_util import GOLDEN_DIR, Golden, flatten, model_from_spec, spec_to_dict, tree_to_device
from tests.test_training_scale_gpu import TOL, _rel, _rounded_inputs

gpu = pytest.mark.gpu
DEV = 'cuda:0'
PRECS = ['fp32', 'tf32x3']
NEW_KERNELS = ('time_encode_kernel', 'time_cond_kernel', 'time_cond_bwd_kernel')
_SP = dict(learning_rate=1e-3, elastic_loss_weight=5.0, warp_reg_loss_weight=3.0, warp_reg_loss_alpha=-2.0,
           warp_reg_loss_scale=0.05, background_loss_weight=60.0)


def _model(spec_dict, prec, **kw):
  m = model_from_spec(spec_dict, device=DEV, **kw)
  m.train_precision = prec
  return m


def _enc_prefix(spec):
  return 'warp_field/metadata_encoder/mlp/' if spec.warp_metadata_encoder_type == 'time' else 'warp_field/time_encoder/mlp/'


def _warp_meta(spec, rays):
  """What the warp field reads per ray: metadata['time'] ('time') or the warp ids (models.py:252-254)."""
  return rays['metadata']['time' if spec.warp_metadata_encoder_type == 'time' else 'warp']


def _level_reg(tree, spec, out, rays, warp_alpha, time_alpha, reg, sp, coarse):
  """level_regularisers (training.py:176-207) with the warp field's metadata and time_alpha forwarded."""
  res = {}
  weights = out['weights'].detach()                                   # lax.stop_gradient
  if reg.get('elastic') and coarse:
    B, S = weights.shape
    meta = _warp_meta(spec, rays)[:, None, :].expand(B, S, 1)
    pts = out['points']
    if reg.get('reduce', 'median') == 'median':
      idx = O.compute_depth_index(weights)
      pts = torch.gather(pts, 1, idx[:, None, None].expand(B, 1, 3))
      meta = meta[:, :1]
    jac = O.warp_jacobian(tree['warp_field'], spec, pts, meta, warp_alpha, time_alpha=time_alpha, create_graph=True)
    loss, _ = O.compute_elastic_loss(jac, loss_type=reg.get('etype', 'log_svals'))
    if reg.get('reduce', 'median') == 'weight':
      loss = weights * loss
    res['elastic'] = loss.sum(dim=-1).mean()
  if reg.get('warp_reg'):
    idx = O.compute_depth_index(weights)
    r = torch.gather(((out['points'] - out['warped_points'])**2).sum(dim=-1), 1, idx[:, None])
    res['warp_reg'] = O.general_loss_with_squared_residual(r, alpha=sp.warp_reg_loss_alpha,
                                                          scale=sp.warp_reg_loss_scale).mean()
  return res


def _oracle(c, dtype, rays=None, params=None, reg=None, sp=None, bg_ids=None):
  """(loss parts, parameter gradients) of training.py:171-259 on the oracle in `dtype`, time_alpha = c.time_alpha.
  Each level renders at the z of the oracle's own forward in the same dtype (a constant: lax.stop_gradient);
  `bg_ids` replaces the background points' ids as the TimeEncoder sees them."""
  reg = reg or {}
  rays = rays or c.rays
  p = {k: v.detach().clone() for k, v in flatten(O.tree_to(params or c.params, dtype)).items()}
  tree = {}
  for k, v in p.items():
    v.requires_grad_(True)
    node = tree
    for part in k.split('/')[:-1]:
      node = node.setdefault(part, {})
    node[k.split('/')[-1]] = v
  with torch.no_grad():
    fwd = O.render_forward(tree, c.spec, rays, warp_alpha=c.warp_alpha, dtype=dtype, time_alpha=c.time_alpha)
  parts, total = {}, 0.0
  for lv in ('coarse', 'fine') if c.spec.num_fine_samples else ('coarse',):
    out = O.render_level(tree, c.spec, lv, rays, fwd[lv]['z_vals'], c.warp_alpha, dtype=dtype,
                         time_alpha=c.time_alpha)
    parts['rgb_' + lv] = ((out['rgb'] - c.target.to(dtype))**2).mean()
    total = total + parts['rgb_' + lv]
    r = _level_reg(tree, c.spec, out, rays, c.warp_alpha, c.time_alpha, reg, sp, lv == 'coarse')
    if 'elastic' in r:
      parts['elastic'] = r['elastic']
      total = total + sp.elastic_loss_weight * r['elastic']
    if 'warp_reg' in r:
      parts['warp_reg_' + lv] = r['warp_reg']
      total = total + sp.warp_reg_loss_weight * r['warp_reg']
  if reg.get('background'):
    bg = c.bg
    l = O.compute_background_loss(tree, c.spec, bg['points'].to(dtype), bg['ids'] if bg_ids is None else bg_ids,
                                  bg['noise'].to(dtype), c.warp_alpha, time_alpha=c.time_alpha).mean()
    parts['background'] = l
    total = total + sp.background_loss_weight * l
  total.backward()
  grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)).double() for k, v in p.items()}
  return {k: float(v.detach()) for k, v in parts.items()}, grads


_REFS = {}


def _refs(c, key, reg=None, sp=None):
  """(fp64 parts, fp64 grads, bands), cached, with test_training_scale_gpu._refs's two round-off bands: the
  fp32 oracle's distance from fp64 and how far fp64 runs move on inputs moved by fp32 round-off."""
  if key not in _REFS:
    parts, g64 = _oracle(c, torch.float64, reg=reg, sp=sp)
    _, g32 = _oracle(c, torch.float32, reg=reg, sp=sp)
    bands = {k: _rel(g32[k], g64[k]) for k in g64}
    for seed in (1, 2):
      rays, params = _rounded_inputs(c, seed)
      _, gr = _oracle(c, torch.float64, rays=rays, params=params, reg=reg, sp=sp)
      for k in g64:
        bands[k] = max(bands[k], _rel(gr[k], g64[k]))
    _REFS[key] = parts, g64, bands
  return _REFS[key]


def _cuda(c, prec, chunk, reg=None, sp=None, model=None):
  from nerfies_b200 import training
  reg = reg or {}
  model = model or _model(spec_to_dict(c.spec), prec)
  kw = {}
  if reg:
    bg = c.bg if reg.get('background') else None
    extra = dict(background_points=bg['points'], background_warp_ids=bg['ids'],
                 background_noise=bg['noise']) if bg else {}
    kw['reg'] = training.make_reg(model, sp, reg.get('elastic', False), reg.get('reduce', 'median'),
                                  reg.get('etype', 'log_svals'), bg is not None, reg.get('warp_reg', False), **extra)
  losses, grads = training.value_and_grad(model, tree_to_device(c.params, DEV), dict(c.rays, rgb=c.target),
                                          c.warp_extra, chunk_rays=chunk, **kw)
  torch.cuda.synchronize()
  got = flatten(training.grads_to_tree(model, grads))
  return {k: float(v) for k, v in losses.items()}, {k: v.cpu().double() for k, v in got.items()}


def _errors(ref, got):
  return {k: _rel(got[k].reshape(r.shape), r) for k, r in ref.items()}


def _fixture(name, time_alpha='fixture', coarse_only=False):
  """A golden fixture ('time_small' / 'blend_small') as a case: its rays and parameters, a seeded target."""
  g = Golden(name)
  spec, params = g.spec, g.params
  if coarse_only:
    spec = dataclasses.replace(spec, num_fine_samples=0)
    params = {k: v for k, v in params.items() if k != 'nerf_mlps_fine'}
  ta = g.time_alpha if time_alpha == 'fixture' else time_alpha
  gen = torch.Generator().manual_seed(7)
  return types.SimpleNamespace(spec=spec, params=params, rays=g.rays, warp_alpha=g.warp_alpha, time_alpha=ta,
                               warp_extra={'alpha': g.warp_alpha, 'time_alpha': ta},
                               target=torch.rand(g.rays['origins'].shape[0], 3, generator=gen), bg=None)


def _two_tier(errs):
  """test_gradients_match_autograd_on_the_oracle's bound: the fine level resamples from the kernel's own fp32
  coarse weights, so 2e-2 for nerf_mlps_fine, 5e-3 for everything else."""
  return {k: e for k, e in errs.items() if e > (2e-2 if 'nerf_mlps_fine' in k else 5e-3)}


# ---------------------------------------------------------------------------
# Golden fixtures, both levels, with the fixture's time_alpha
# ---------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('name', ['time_small', 'blend_small'])
def test_fixture_gradients_match_autograd(name, prec):
  c = _fixture(name)
  parts, ref = _oracle(c, torch.float64)
  enc = [k for k in ref if k.startswith(_enc_prefix(c.spec))]
  # the TimeEncoder is really trained: every one of its tensors has a non-zero reference gradient
  assert len(enc) == 14 and all(float(ref[k].abs().max()) > 0 for k in enc), enc
  losses, got = _cuda(c, prec, 5)
  assert abs(losses['coarse'] - parts['rgb_coarse']) < 1e-5 * max(1.0, parts['rgb_coarse'])
  bad = _two_tier(_errors(ref, got))
  assert not bad, bad


@gpu
@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('name', ['time_small', 'blend_small'])
def test_fixture_gradients_on_the_oracle_z(name, prec):
  """Coarse-only: the kernels render at the oracle's z, so every tensor within TOL."""
  c = _fixture(name, coarse_only=True)
  parts, ref = _oracle(c, torch.float64)
  losses, got = _cuda(c, prec, 4)
  assert abs(losses['coarse'] - parts['rgb_coarse']) < 1e-5
  bad = {k: e for k, e in _errors(ref, got).items() if not e < TOL}
  assert not bad, bad


@gpu
@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('ta', [0.0, 0.35, 1.0])
def test_blend_time_alpha(ta, prec):
  """(1 - ta) glo(id) + ta TimeEncoder(float(id)): at ta = 0 the TimeEncoder gets exactly nothing, at 1 the
  GLO rows do."""
  c = _fixture('blend_small', time_alpha=ta)
  _, ref = _oracle(c, torch.float64)
  _, got = _cuda(c, prec, 3)
  bad = _two_tier(_errors(ref, got))
  assert not bad, bad
  glo = got['warp_field/glo_encoder/embed/embedding']
  enc = [got[k] for k in got if k.startswith('warp_field/time_encoder/')]
  if ta == 0.0:
    assert all(float(t.abs().max()) == 0.0 for t in enc)
    assert float(glo.abs().max()) > 0
  elif ta == 1.0:
    assert float(glo.abs().max()) == 0.0
    assert all(float(t.abs().max()) > 0 for t in enc)
  else:
    assert float(glo.abs().max()) > 0 and all(float(t.abs().max()) > 0 for t in enc)


@gpu
@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('ta', [0.0, 1.6, None], ids=['0', '1.6', 'None'])
def test_time_alpha(ta, prec):
  """The TimeEncoder's window at time_alpha 0 (the timestamp alone), 1.6 and None (= num_freqs)."""
  c = _fixture('time_small', time_alpha=ta)
  _, ref = _oracle(c, torch.float64)
  _, got = _cuda(c, prec, 4)
  bad = _two_tier(_errors(ref, got))
  assert not bad, bad


# ---------------------------------------------------------------------------
# vrig dimensions (256-wide SE(3) trunk) with the 'time' encoder: tier A
# ---------------------------------------------------------------------------
_VRIG = {}


def _vrig_time():
  """40 rays of a coarse-only vrig-sized model with a 3-frequency TimeEncoder at time_alpha 2.5, 170
  background points (against a 64-ray handle: chunks of 64, 64 and 42)."""
  if not _VRIG:
    spec = O.OracleSpec(num_coarse_samples=128, num_fine_samples=0, near=0.02, far=0.83, num_nerf_point_freqs=8,
                        num_warp_freqs=6, sigma_activation='softplus', use_warp=True, warp_field_type='se3',
                        use_appearance_metadata=False, use_camera_metadata=True, num_warp_embeddings=50,
                        num_appearance_embeddings=1, num_camera_embeddings=2,
                        warp_metadata_encoder_type='time', metadata_encoder_num_freqs=3)
    seed = 300
    gen = torch.Generator().manual_seed(seed + 3)
    rays = O.synthetic_rays(40, spec, seed=seed + 2)
    rays['metadata']['time'] = torch.rand(40, 1, generator=gen)
    bg = dict(points=torch.rand(170, 3, generator=gen) * 0.6 - 0.3,
              ids=torch.randint(1, spec.num_warp_embeddings, (170, 1), generator=gen),
              noise=0.05 * torch.randn(170, 3, generator=gen))
    _VRIG['c'] = types.SimpleNamespace(
        spec=spec, params=O.make_trained_like(O.init_params(spec, seed), seed=seed + 1), rays=rays, warp_alpha=4.5,
        time_alpha=2.5, warp_extra={'alpha': 4.5, 'time_alpha': 2.5}, target=torch.rand(40, 3, generator=gen), bg=bg)
  return _VRIG['c']


def _tier_a(errs, bands):
  return {k: (e, max(TOL, 3.0 * bands[k])) for k, e in errs.items() if not e <= max(TOL, 3.0 * bands[k])}


@gpu
@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('chunk', [40, 17])
def test_photometric_gradients_at_vrig_size(chunk, prec):
  c = _vrig_time()
  parts, ref, bands = _refs(c, 'photometric')
  losses, got = _cuda(c, prec, chunk)
  assert abs(losses['coarse'] - parts['rgb_coarse']) < 1e-5 * parts['rgb_coarse']
  bad = _tier_a(_errors(ref, got), bands)
  assert not bad, bad


@gpu
@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('reg', [
    dict(elastic=True, reduce='weight', etype='log_svals'),
    dict(elastic=True, reduce='median', etype='svals'),
    dict(warp_reg=True),
    dict(background=True),
], ids=lambda r: '-'.join(f'{k}={v}' for k, v in r.items()))
def test_regulariser_gradients_at_vrig_size(reg, prec):
  from nerfies_b200 import training
  sp = training.ScalarParams(**_SP)
  c = _vrig_time()
  key = '-'.join(f'{k}={v}' for k, v in reg.items())
  parts, ref, bands = _refs(c, key, reg, sp)
  _, plain, _ = _refs(c, 'photometric')
  moved = max(_rel(ref[k], plain[k]) for k in ref if k.startswith('warp_field/'))
  assert moved > 0.25, moved
  if reg.get('background'):
    # the ids are the TimeEncoder's timestamps as float(id): their float32 bit patterns would be another loss
    _, bits = _oracle(c, torch.float64, reg=reg, sp=sp, bg_ids=c.bg['ids'].to(torch.int32).view(torch.float32))
    wrong = max(_rel(bits[k], ref[k]) for k in ref if k.startswith(_enc_prefix(c.spec)))
    assert wrong > 0.25, wrong
  model = _model(spec_to_dict(c.spec), prec)
  if reg.get('background'):
    assert c.bg['points'].shape[0] >= 2.5 * model.handle(0).max_rays
  losses, got = _cuda(c, prec, 17, reg, sp, model=model)
  assert abs(losses['coarse'] - parts['rgb_coarse']) < 1e-5 * parts['rgb_coarse']
  for k in ('elastic', 'warp_reg_coarse', 'background'):
    if k in parts:
      assert abs(losses[k] - parts[k]) < 2e-4 * max(abs(parts[k]), 1e-3), (k, losses[k], parts[k])
  bad = _tier_a(_errors(ref, got), bands)
  assert not bad, bad


# ---------------------------------------------------------------------------
# Warp Jacobians
# ---------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('name', ['time_small', 'blend_small'])
def test_warp_jacobian(name, prec):
  """nfb_warp_jacobian through warp_field.apply(return_jacobian=True) and model.apply(return_warp_jacobian=True)
  against autograd on the oracle in float64; the embedding is a constant of jacfwd (warping.py:196-197)."""
  g = Golden(name)
  model = _model(g.spec_dict, prec)
  params = tree_to_device(g.params, DEV)
  extra = {'alpha': g.warp_alpha, 'time_alpha': g.time_alpha}
  gen = torch.Generator().manual_seed(5)
  P = 37
  pts = torch.rand(P, 3, generator=gen) * 0.6 - 0.3
  if g.spec.warp_metadata_encoder_type == 'time':
    meta = torch.rand(P, 1, generator=gen)
  else:
    meta = torch.randint(0, g.spec.num_warp_embeddings, (P, 1), generator=gen)
  p64 = O.tree_to(g.params, torch.float64)['warp_field']
  wf = model.create_warp_field(model, num_batch_dims=1)
  out = wf.apply({'params': params['warp_field']}, pts, meta, extra, return_jacobian=True)
  torch.cuda.synchronize()
  ref = O.warp_jacobian(p64, g.spec, pts.double(), meta, g.warp_alpha, time_alpha=g.time_alpha).detach()
  assert float((out['jacobian'].cpu().double() - ref).abs().max()) < 2e-5 * max(1.0, float(ref.abs().max()))
  o2 = model.apply({'params': params}, g.rays, warp_extra=extra, return_warp_jacobian=True, return_points=True)
  torch.cuda.synchronize()
  for lv in ('coarse', 'fine'):
    J = o2[lv]['warp_jacobian'].cpu()
    B, S = J.shape[:2]
    m = _warp_meta(g.spec, g.rays)[:, None, :].expand(B, S, 1).reshape(-1, 1)
    ref = O.warp_jacobian(p64, g.spec, o2[lv]['points'].cpu().double().reshape(-1, 3), m, g.warp_alpha,
                          time_alpha=g.time_alpha).detach().reshape(B, S, 3, 3)
    assert float((J.double() - ref).abs().max()) < 2e-5 * max(1.0, float(ref.abs().max())), lv


# ---------------------------------------------------------------------------
# train_step, isolation
# ---------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('prec', PRECS)
def test_train_step_with_time_alpha_schedule(prec):
  """A 'time' model trained with the time_alpha schedule of train.py (state.time_alpha = sched(step)): the loss
  falls and the TimeEncoder's tensors move."""
  from nerfies_b200 import schedules, training
  g = Golden('time_small')
  model = _model(g.spec_dict, prec)
  state = training.create_train_state(model, tree_to_device(g.params, DEV), warp_alpha=g.warp_alpha)
  before = {k: v.detach().clone() for k, v in flatten(state.optimizer.target['model']).items()}
  time_sched = schedules.from_config(('linear', 0.0, 3.0, 10))
  gen = torch.Generator().manual_seed(9)
  batch = dict(g.rays, rgb=torch.rand(g.rays['origins'].shape[0], 3, generator=gen))
  sp = training.ScalarParams(learning_rate=2e-3)
  first = last = None
  for step in range(10):
    state = dataclasses.replace(state, time_alpha=time_sched(step))
    state, stats, _ = training.train_step(model, step, state, batch, sp, chunk_rays=4)
    last = float(stats['coarse']['loss/total']) + float(stats['fine']['loss/total'])
    first = last if first is None else first
  assert last < 0.9 * first, (first, last)
  after = flatten(state.optimizer.target['model'])
  enc = [k for k in after if k.startswith('warp_field/metadata_encoder/mlp/')]
  assert len(enc) == 14
  assert all(not torch.equal(after[k], before[k]) for k in enc), [k for k in enc if torch.equal(after[k], before[k])]


def _kernel_names(fn):
  from torch.profiler import ProfilerActivity, profile
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    fn()
    torch.cuda.synchronize()
  return {e.name for e in prof.events()}


@gpu
def test_glo_model_launches_no_time_kernel():
  from nerfies_b200 import training
  g = Golden('se3_small')
  model = _model(g.spec_dict, 'fp32')
  params = tree_to_device(g.params, DEV)
  batch = dict(g.rays, rgb=torch.rand(g.rays['origins'].shape[0], 3))
  run = lambda m, p, b, extra: training.value_and_grad(m, p, b, extra, chunk_rays=5)
  run(model, params, batch, {'alpha': g.warp_alpha})
  names = _kernel_names(lambda: run(model, params, batch, {'alpha': g.warp_alpha}))
  assert not [n for n in names if any(k in n for k in NEW_KERNELS)]
  c = _fixture('time_small')
  tm = _model(Golden('time_small').spec_dict, 'fp32')
  tparams = tree_to_device(c.params, DEV)
  names = _kernel_names(lambda: run(tm, tparams, dict(c.rays, rgb=c.target), c.warp_extra))
  assert all(any(k in n for n in names) for k in NEW_KERNELS), sorted(n for n in names if 'time' in n)


@gpu
@pytest.mark.parametrize('name', ['time_small', 'blend_small'])
def test_training_leaves_the_render_bitwise_unchanged(name):
  c = _fixture(name)
  spec_dict = Golden(name).spec_dict
  params = tree_to_device(c.params, DEV)

  def render(model):
    out = model.apply({'params': params}, c.rays, warp_extra=c.warp_extra, return_weights=True)
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in flatten(out).items()}

  trained = _model(spec_dict, 'fp32')
  _cuda(c, 'fp32', 3, model=trained)
  got = render(trained)
  fresh = render(_model(spec_dict, 'fp32'))
  for k, v in fresh.items():
    assert torch.equal(got[k], v), k


# ---------------------------------------------------------------------------
# The oracle against the reference's own source (no GPU)
# ---------------------------------------------------------------------------
@pytest.mark.parametrize('name', ['time_small', 'blend_small'])
def test_oracle_time_regularisers_match_the_reference(name):
  """compute_background_loss with the ids as the TimeEncoder's timestamps, and warp_field.apply(...,
  return_jacobian=True), at a fractional time_alpha (oracle/make_golden_time_reg.py)."""
  Z = np.load(os.path.join(GOLDEN_DIR, 'time_regularisers.npz'))
  g = Golden(name)
  ta = float(Z[f'{name}/time_alpha'])
  assert ta != int(ta)
  p64 = O.tree_to(g.params, torch.float64)
  meta = torch.from_numpy(Z[f'jac/{name}/metadata'])
  meta = meta if meta.is_floating_point() else meta.long()
  pts = torch.from_numpy(Z[f'jac/{name}/points'])
  J = O.warp_jacobian(p64['warp_field'], g.spec, pts.double(), meta, g.warp_alpha, time_alpha=ta).detach()
  ref = Z[f'jac/{name}/jacobian']
  assert float(np.abs(J.numpy() - ref).max()) < 2e-6 * max(1.0, float(np.abs(ref).max()))
  warped = O.warp_field_apply(O.tree_to(g.params, torch.float32)['warp_field'], g.spec, pts, meta, g.warp_alpha,
                              time_alpha=ta)
  np.testing.assert_allclose(warped.numpy(), Z[f'jac/{name}/warped_points'], rtol=0, atol=2e-6)
  ids = torch.from_numpy(Z[f'bg/{name}/ids'].astype(np.int64))
  assert int(ids.max()) > 0
  loss = O.compute_background_loss(g.params, g.spec, torch.from_numpy(Z[f'bg/{name}/points']), ids,
                                   torch.from_numpy(Z[f'bg/{name}/noise']), g.warp_alpha, time_alpha=ta)
  np.testing.assert_allclose(loss.numpy(), Z[f'bg/{name}/loss'], rtol=2e-4, atol=1e-9)
