"""model.apply and warp_field.apply through torch.autograd (nfb_render_vjp, nfb_warp_vjp).

Each differentiable call is held to torch.autograd of the oracle in float64 on the z values the kernels used
(the fine level on the kernel's z_fine: resampling is a constant, and comparing on the oracle's own z would
measure the conditioning of resampling, DESIGN.md §2).  The loss is <cotangent, output> with random
cotangents on rgb, depth, acc, weights or warped_points alone and on all of them together; every parameter
tensor (and code) is held to the tier-A tolerance of test_training_scale_gpu.py, max(2e-4, 3 x band), the
band being the larger of the fp32 oracle's distance from fp64 and the distance fp64 moves when the rays and
parameters move by fp32 round-off.
"""
import ctypes

import pytest
import torch

from oracle import nerfies_oracle as O
from tests.golden_util import Golden, flatten, model_from_spec, spec_to_dict, tree_to_device

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
TOL = 2e-4
OUTPUTS = ('rgb', 'depth', 'acc', 'weights', 'warped_points')

# bench.py's workloads (gpu_quarterhd.gin, gpu_vrig_paper.gin, gpu_fullhd.gin model dimensions), two levels
DIMS = {
    'quarterhd': dict(S=128, fp=8, fw=8, app=True, cam=False, alpha=8.0),
    'vrig': dict(S=128, fp=8, fw=6, app=False, cam=True, alpha=4.5),
    'fullhd': dict(S=256, fp=10, fw=8, app=True, cam=False, alpha=6.3),
}


def _gin_spec(dims, fine=True):
  d = DIMS[dims]
  return O.OracleSpec(num_coarse_samples=d['S'], num_fine_samples=d['S'] if fine else 0, near=0.02, far=0.83,
                      num_nerf_point_freqs=d['fp'], num_warp_freqs=d['fw'], sigma_activation='softplus',
                      use_warp=True, warp_field_type='se3', use_appearance_metadata=d['app'],
                      use_camera_metadata=d['cam'], num_warp_embeddings=20,
                      num_appearance_embeddings=20 if d['app'] else 1, num_camera_embeddings=2 if d['cam'] else 1)


def _small_spec(**kw):
  base = dict(num_coarse_samples=32, num_fine_samples=32, near=0.02, far=0.83, nerf_trunk_depth=5,
              nerf_trunk_width=64, nerf_rgb_branch_width=32, num_nerf_point_freqs=5, num_warp_freqs=4,
              sigma_activation='softplus', use_warp=True, warp_field_type='se3', warp_trunk_depth=5,
              warp_trunk_width=64, use_appearance_metadata=True, use_camera_metadata=True,
              use_alpha_condition=True, num_warp_embeddings=6, num_appearance_embeddings=5,
              num_camera_embeddings=3)
  base.update(kw)
  return O.OracleSpec(**base)


class Case:
  """A model, its trained-like parameters and rays; `extra` holds the call's keyword arguments."""

  def __init__(self, spec, num_rays, seed, warp_alpha=4.0, time_alpha=None, params=None, rays=None,
               use_warp=True, encoded=False, stratified=False):
    self.spec, self.warp_alpha, self.time_alpha = spec, warp_alpha, time_alpha
    self.use_warp, self.encoded = use_warp, encoded
    self.params = params if params is not None else O.make_trained_like(O.init_params(spec, seed), seed=seed + 1)
    self.rays = rays if rays is not None else O.synthetic_rays(num_rays, spec, seed=seed + 2)
    B = self.rays['origins'].shape[0]
    gen = torch.Generator().manual_seed(seed + 3)
    if spec.warp_metadata_encoder_type == 'time' and 'time' not in self.rays['metadata']:
      self.rays['metadata']['time'] = torch.rand(B, 1, generator=gen)
    if encoded:
      # per-ray codes in place of the ids (models.py:198-213, warping.py:186-187)
      md = {'warp': torch.rand(B, spec.num_warp_features, generator=gen) * 0.05}
      if spec.use_appearance_metadata:
        md['appearance'] = torch.rand(B, spec.num_appearance_features, generator=gen) * 0.05
      if spec.use_camera_metadata:
        md['camera'] = torch.rand(B, spec.num_camera_features, generator=gen) * 0.05
      self.rays = dict(self.rays, metadata=md)
    self.t_rand = self.u_rand = None
    if stratified:
      self.t_rand = torch.rand(B, spec.num_coarse_samples, generator=gen)
      if spec.num_fine_samples:
        self.u_rand = torch.rand(B, spec.num_fine_samples, generator=gen)
    self.warp_extra = {'alpha': warp_alpha, 'time_alpha': time_alpha}


def _levels(spec):
  return ('coarse', 'fine') if spec.num_fine_samples else ('coarse',)


def _cotangents(c, which, seed):
  """Random cotangents of the outputs in `which`, per level, shaped like the outputs."""
  B = c.rays['origins'].shape[0]
  gen = torch.Generator().manual_seed(seed)
  out = {}
  for lv in _levels(c.spec):
    S = c.spec.num_coarse_samples + (c.spec.num_fine_samples if lv == 'fine' else 0)
    shapes = {'rgb': (B, 3), 'depth': (B,), 'acc': (B,), 'weights': (B, S), 'warped_points': (B, S, 3)}
    out[lv] = {k: torch.randn(*shapes[k], generator=gen, dtype=torch.float64) for k in which}
  return out


def _dot(outs, cot):
  total = 0.0
  for lv, d in cot.items():
    for k, g in d.items():
      total = total + (outs[lv][k].double() * g.to(outs[lv][k].device)).sum()
  return total


def _cuda_grads(c, cot, model=None, chunk=None, fast=False, warped=None):
  """Gradients of <cot, model.apply(...)> from loss.backward(): ({param name: grad}, {code: grad}, z per level);
  `warped` (a dict) receives each level's warped points."""
  model = model or model_from_spec(spec_to_dict(c.spec), device=DEV)
  if chunk:
    model.vjp_chunk_rays = chunk
  params = tree_to_device(c.params, DEV)
  leaves = flatten(params)
  for v in leaves.values():
    v.requires_grad_(True)
  rays = tree_to_device(c.rays, DEV)
  codes = {}
  if c.encoded:
    for k, v in rays['metadata'].items():
      codes[k] = v.clone().requires_grad_(True)
    rays = dict(rays, metadata=codes)
  kw = dict(t_rand=None if c.t_rand is None else c.t_rand.to(DEV),
            u_rand=None if c.u_rand is None else c.u_rand.to(DEV))
  out = model.apply({'params': params}, rays, warp_extra=c.warp_extra, use_warp=c.use_warp,
                    metadata_encoded=c.encoded, return_points=not fast, return_weights=True, **kw)
  _dot(out, cot).backward()
  torch.cuda.synchronize()
  grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)).cpu().double() for k, v in leaves.items()}
  cg = {k: v.grad.cpu().double() for k, v in codes.items() if v.grad is not None}
  z = {lv: out[lv]['z_vals'].detach().cpu() for lv in out} if not fast else None
  if warped is not None:
    warped.update({lv: out[lv]['warped_points'].detach().cpu() for lv in out})
  return grads, cg, z


def _oracle_grads(c, cot, z, dtype, rays=None, params=None):
  """fp64 (or fp32) autograd of <cot, O.render_level(...)> per level on the kernel's z."""
  rays = rays or c.rays
  p = {k: v.detach().clone().to(dtype).requires_grad_(True) for k, v in flatten(params or c.params).items()}
  tree = {}
  for k, v in p.items():
    node = tree
    for part in k.split('/')[:-1]:
      node = node.setdefault(part, {})
    node[k.split('/')[-1]] = v
  md = rays['metadata']
  codes = {}
  if c.encoded:
    codes = {k: v.detach().clone().to(dtype).requires_grad_(True) for k, v in md.items()}
    md = codes
  r = dict(rays, metadata=md)
  outs = {lv: O.render_level(tree, c.spec, lv, r, z[lv], c.warp_alpha, use_warp=c.use_warp, dtype=dtype,
                             metadata_encoded=c.encoded, time_alpha=c.time_alpha) for lv in z}
  _dot(outs, cot).backward()
  grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)).double() for k, v in p.items()}
  return grads, {k: v.grad.double() for k, v in codes.items() if v.grad is not None}


def _moved(c, seed):
  """Rays moved by up to one fp32 rounding and parameters by up to 16 (test_training_scale_gpu._rounded_inputs)."""
  gen = torch.Generator().manual_seed(seed)
  move = lambda t, u: t.double() * (1 + u * (2 * torch.rand(t.shape, generator=gen, dtype=torch.float64) - 1))
  tree = lambda t: {k: tree(v) for k, v in t.items()} if isinstance(t, dict) else move(t, 16 * 2.0**-24)
  return (dict(c.rays, origins=move(c.rays['origins'], 2.0**-24), directions=move(c.rays['directions'], 2.0**-24)),
          tree(c.params))


def _scale(ref):
  return max(float(v.abs().max()) for v in ref.values() if v.numel())


def _rel(a, r, floor):
  return float((a - r).abs().max()) / max(float(r.abs().max()), floor) if r.numel() else 0.0


def _check(name, c, cot, got, got_codes, z, wider=None):
  """wider(ref): {tensor: band} of a derived band of the tensor's own beside tier A's (of the float64
  reference gradients `ref`); such a tensor is also held within 3 x that band."""
  ref, ref_codes = _oracle_grads(c, cot, z, torch.float64)
  g32, c32 = _oracle_grads(c, cot, z, torch.float32)
  ref, g32 = {**ref, **ref_codes}, {**g32, **c32}
  moved = []
  for seed in (1, 2):
    mr, mp = _moved(c, seed)
    gm, cm = _oracle_grads(c, cot, z, torch.float64, rays=mr, params=mp)
    moved.append({**gm, **cm})
  got = {**got, **got_codes}
  # tensors the cotangent does not reach (e.g. the rgb branch under an acc cotangent) are compared with the
  # largest gradient of the call, scaled down
  floor = 1e-4 * _scale(ref)
  extra = wider(ref) if wider else {}
  bad, worst = {}, (0.0, None)
  for k, r in ref.items():
    band = max([_rel(g32[k], r, floor)] + [_rel(gm[k], r, floor) for gm in moved])
    err = _rel(got[k].reshape(r.shape), r, floor)
    tol = max(TOL, 3.0 * band, 3.0 * extra.get(k, 0.0))
    worst = max(worst, (err / tol, k, err, band), key=lambda t: t[0])
    if not err <= tol:
      bad[k] = (err, tol)
  print(f'{name}: worst error / tolerance {worst}')
  assert not bad, f'{name}: {bad}'


def _run(name, c, which, seed=0, wider=None, **kw):
  """wider(cot, z, ref): see _check."""
  cot = _cotangents(c, which, seed)
  got, got_codes, z = _cuda_grads(c, cot, **kw)
  _check(name, c, cot, got, got_codes, z, None if wider is None else lambda ref: wider(cot, z, ref))


# ---------------------------------------------------------------------------
# 1. against fp64 autograd on the oracle
# ---------------------------------------------------------------------------
_GIN = {}


def _gin_case(dims):
  if dims not in _GIN:
    _GIN[dims] = Case(_gin_spec(dims), 12, seed=300 + len(dims), warp_alpha=DIMS[dims]['alpha'])
  return _GIN[dims]


@pytest.mark.parametrize('which', [(k,) for k in OUTPUTS] + [OUTPUTS], ids=lambda w: '+'.join(w))
@pytest.mark.parametrize('dims', ['quarterhd', 'vrig', 'fullhd'])
def test_gin_dims_both_levels(dims, which):
  wider, pts = None, {}
  if dims == 'fullhd' and which == OUTPUTS:
    # The fine level's trunk is the one place where the fp32 forward's error, rather than the backward's, sets
    # the distance from fp64: the fine MLP reads its warped points through a 10-frequency encoding, so their
    # fp32 error (about 2e-7) moves its highest features by about 2^9 times that, and relu units of the trunk
    # whose pre-activations lie that close to 0 change sign.  Measured on an H100 80GB HBM3 at 700 W
    # (test_train_net_gpu.py::test_fullhd_fine_mlp): hidden_7's kernel is 1.42e-3 and its bias 1.09e-3 from
    # fp64 here; on this case's inputs and seed the fine MLP itself is within 3e-7 of fp64 and the seed's
    # amplification of its forward error within 2e-7, while fp64 itself moves by 1.42e-3 and 1.09e-3 when its
    # warped points are the kernel's fp32 ones, and by 6e-7 when every relu mask is held at its value on the
    # fp64 points: 17 trunk units change sign.  So the fine MLP's tensors are also held to 3 x that distance,
    # computed here on this call's warped points.
    from tests.test_train_net_gpu import fine_input_band
    wider = lambda cot, z, ref: fine_input_band(_gin_case(dims), cot, z, pts['fine'], ref)
  _run(f'{dims} {which}', _gin_case(dims), which, seed=len(which), wider=wider, warped=pts)


def _golden_case(name, **kw):
  g = Golden(name)
  return Case(g.spec, 0, seed=0, warp_alpha=g.warp_alpha, time_alpha=g.time_alpha if g.spec.use_warp else None,
              params=g.params, rays=g.rays, **kw)


_VARIANTS = {
    'coarse_only': lambda: Case(_small_spec(num_fine_samples=0), 24, seed=10),
    'translation': lambda: _golden_case('translation_small'),
    'time': lambda: _golden_case('time_small'),
    'blend': lambda: _golden_case('blend_small'),
    'call_no_warp': lambda: Case(_small_spec(), 24, seed=11, use_warp=False),
    'model_no_warp': lambda: Case(_small_spec(use_warp=False), 24, seed=12),
    'white_background': lambda: Case(_small_spec(use_white_background=True), 24, seed=13),
    'no_sample_at_infinity': lambda: Case(_small_spec(use_sample_at_infinity=False), 24, seed=14),
    'relu_sigma': lambda: Case(_small_spec(sigma_activation='relu'), 24, seed=15),
    'stratified': lambda: Case(_small_spec(), 24, seed=16, stratified=True),
    'encoded': lambda: Case(_small_spec(), 24, seed=17, encoded=True),
    'encoded_trunk_condition': lambda: Case(_small_spec(use_trunk_condition=True), 24, seed=18, encoded=True),
}


@pytest.mark.parametrize('variant', list(_VARIANTS))
def test_variants(variant):
  c = _VARIANTS[variant]()
  warps = c.spec.use_warp and c.use_warp
  _run(variant, c, OUTPUTS if warps else OUTPUTS[:4], seed=5)


def test_encoded_code_gradients_each():
  """metadata_encoded=True: every code gets the gradient of its own blocks; the appearance code feeds the alpha
  and (models.py:206-207) the rgb condition, so its gradient is their sum."""
  c = _VARIANTS['encoded']()
  cot = _cotangents(c, ('rgb', 'acc'), 9)
  got, codes, z = _cuda_grads(c, cot)
  assert set(codes) == {'warp', 'appearance', 'camera'}
  for k in codes:
    assert float(codes[k].abs().max()) > 0, k
  _check('encoded codes', c, cot, got, codes, z)


def test_fast_path_matches_staged_path():
  """Without return_points the forward is nfb_render_forward; its z_fine is saved for the backward."""
  c = Case(_small_spec(), 24, seed=20)
  cot = _cotangents(c, ('rgb', 'depth', 'acc', 'weights'), 3)
  staged, _, z = _cuda_grads(c, cot)
  fast, _, _ = _cuda_grads(c, cot, fast=True)
  for k in staged:
    assert _rel(fast[k], staged[k], 1e-4 * _scale(staged)) < 1e-5, k


# ---------------------------------------------------------------------------
# 2. against nfb_train_value_and_grad on coarse-only models
# ---------------------------------------------------------------------------
@pytest.mark.parametrize('dims', ['quarterhd', 'vrig'])
def test_mse_cotangent_equals_value_and_grad(dims):
  from nerfies_b200 import training
  c = Case(_gin_spec(dims, fine=False), 40, seed=40 + len(dims), warp_alpha=DIMS[dims]['alpha'])
  target = torch.rand(40, 3, generator=torch.Generator().manual_seed(5))
  model = model_from_spec(spec_to_dict(c.spec), device=DEV)
  params = tree_to_device(c.params, DEV)
  batch = dict(tree_to_device(c.rays, DEV), rgb=target.to(DEV))
  runs = []
  for _ in range(3):
    losses, g = training.value_and_grad(model, params, batch, c.warp_extra, chunk_rays=17)
    runs.append((float(losses['coarse']), {k: v.cpu().double() for k, v in
                                           flatten(training.grads_to_tree(model, g)).items()}))
  scale = _scale(runs[0][1])
  # the call's run-to-run noise (float atomicAdd order), relative to its largest gradient
  noise = max(float((runs[i][1][k] - runs[0][1][k]).abs().max()) for i in (1, 2) for k in runs[0][1]) / scale
  loss_noise = max(abs(runs[i][0] - runs[0][0]) for i in (1, 2))
  leaves = flatten(params)
  for v in leaves.values():
    v.requires_grad_(True)
  model.vjp_chunk_rays = 17
  out = model.apply({'params': params}, tree_to_device(c.rays, DEV), warp_extra=c.warp_extra)
  loss = ((out['coarse']['rgb'] - target.to(DEV))**2).mean()
  loss.backward()
  worst = max(float((leaves[k].grad.cpu().double() - r).abs().max()) for k, r in runs[0][1].items()) / scale
  dloss = abs(float(loss) - runs[0][0])
  print(f'{dims}: gradient {worst:.3e} (noise {noise:.3e}), loss {dloss:.3e} (noise {loss_noise:.3e}) '
        f'of {runs[0][0]:.6e}')
  assert noise > 0
  assert dloss <= 3 * loss_noise + 2e-7 * runs[0][0], (dloss, loss_noise)
  # Deviation from a plain 3 x noise (DESIGN.md §5.6): the cotangent comes from the render kernel's rgb,
  # value_and_grad's from the tape's, and the two fp32 forwards round differently.  Measured on an H100 80GB
  # HBM3: 7.1e-7 (noise 2.0e-7) at quarterhd and 1.2e-6 (noise 9.3e-8) at vrig of the largest gradient; the
  # losses agree within their noise.  Floor 1e-5, 20 x below tier A's 2e-4.
  assert worst <= max(3 * noise, 1e-5), (worst, noise)


# ---------------------------------------------------------------------------
# 3. chunking, training precision, render precision
# ---------------------------------------------------------------------------
def test_chunks_agree():
  c = Case(_small_spec(), 40, seed=50)
  cot = _cotangents(c, OUTPUTS, 7)
  g256, _, z = _cuda_grads(c, cot, chunk=256)
  g17, _, _ = _cuda_grads(c, cot, chunk=17)
  scale = _scale(g256)
  for k in g256:
    assert _rel(g17[k], g256[k], 1e-4 * scale) < 1e-5, k
  _check('chunk 17', c, cot, g17, {}, z)


@pytest.mark.parametrize('dims', ['quarterhd', 'vrig'])
def test_tf32x3(dims):
  c = _gin_case(dims)
  model = model_from_spec(spec_to_dict(c.spec), device=DEV)
  model.train_precision = 'tf32x3'
  cot = _cotangents(c, OUTPUTS, 11)
  got, codes, z = _cuda_grads(c, cot, model=model)
  _check(f'{dims} tf32x3', c, cot, got, codes, z)


def test_render_precision_does_not_matter_at_fixed_z():
  """Coarse-only with fixed draws: the z values are those of t_rand whatever the render kernel, and the VJP
  runs in the training precision, so the gradients agree up to atomicAdd order."""
  c = Case(_small_spec(num_fine_samples=0, num_coarse_samples=128), 24, seed=60, stratified=True)
  cot = _cotangents(c, ('rgb', 'depth', 'acc', 'weights'), 13)
  ref = None
  for prec in ('fp32', 'fp16x3', 'bf16'):
    model = model_from_spec(spec_to_dict(c.spec), precision=prec, device=DEV)
    g, _, _ = _cuda_grads(c, cot, model=model)
    if ref is None:
      ref = g
      continue
    for k in ref:
      assert _rel(g[k], ref[k], 1e-4 * _scale(ref)) < 1e-5, (prec, k)


# ---------------------------------------------------------------------------
# 4. no behaviour change
# ---------------------------------------------------------------------------
def _plain_call(model, params, rays, **kw):
  before = model.kernel_launches()
  out = model.apply({'params': params}, rays, warp_extra={'alpha': 4.0}, return_weights=True, **kw)
  torch.cuda.synchronize()
  return out, model.kernel_launches() - before


@pytest.mark.parametrize('return_points', [False, True])
def test_outputs_unchanged(return_points):
  c = Case(_small_spec(), 24, seed=70)
  model = model_from_spec(spec_to_dict(c.spec), device=DEV)
  params = tree_to_device(c.params, DEV)
  rays = tree_to_device(c.rays, DEV)
  ref, launches = _plain_call(model, params, rays, return_points=return_points)
  with torch.no_grad():
    grad_params = {k: v for k, v in flatten(tree_to_device(c.params, DEV)).items()}
  for v in grad_params.values():
    v.requires_grad_(True)
  tree = {}
  for k, v in grad_params.items():
    node = tree
    for part in k.split('/')[:-1]:
      node = node.setdefault(part, {})
    node[k.split('/')[-1]] = v
  with torch.no_grad():
    nograd, n2 = _plain_call(model, tree, rays, return_points=return_points)
  assert n2 == launches
  withgrad, _ = _plain_call(model, tree, rays, return_points=return_points)
  # rays that require grad, with no parameter that does: the plain call, as before
  grad_rays = dict(rays, origins=rays['origins'].clone().requires_grad_(True))
  raysgrad, n3 = _plain_call(model, params, grad_rays, return_points=return_points)
  assert n3 == launches
  for lv in ref:
    for k in ref[lv]:
      if k != 'points':
        assert raysgrad[lv][k].grad_fn is None, (lv, k)
        assert torch.equal(ref[lv][k], raysgrad[lv][k]), (lv, k)
      assert ref[lv][k].grad_fn is None and nograd[lv][k].grad_fn is None
      assert torch.equal(ref[lv][k], nograd[lv][k]), (lv, k)
      assert torch.equal(ref[lv][k], withgrad[lv][k].detach()), (lv, k)
    for k in ('rgb', 'depth', 'acc', 'weights'):
      assert withgrad[lv][k].grad_fn is not None, (lv, k)


def test_med_depth_has_no_gradient():
  """med_depth is piecewise constant in the parameters: its cotangent column is ignored, every gradient is 0."""
  c, model, params, rays = _grad_setup()
  out = model.apply({'params': params}, rays, warp_extra={'alpha': 4.0})
  (out['coarse']['med_depth'].sum() + out['fine']['med_depth'].sum()).backward()
  for k, v in flatten(params).items():
    assert v.grad is not None and not bool(v.grad.any()), k


# ---------------------------------------------------------------------------
# 5. refusals
# ---------------------------------------------------------------------------
def _grad_setup(spec_kw=None):
  c = Case(_small_spec(**(spec_kw or {})), 8, seed=80)
  model = model_from_spec(spec_to_dict(c.spec), device=DEV)
  params = tree_to_device(c.params, DEV)
  for v in flatten(params).values():
    v.requires_grad_(True)
  return c, model, params, tree_to_device(c.rays, DEV)


def test_refusals():
  c, model, params, rays = _grad_setup()
  with pytest.raises(NotImplementedError, match='Jacobian'):
    model.apply({'params': params}, rays, warp_extra={'alpha': 4.0}, return_warp_jacobian=True)
  for key in ('origins', 'directions', 'viewdirs'):
    r = dict(rays)
    r[key] = (rays['directions'] if key == 'viewdirs' else rays[key]).clone().requires_grad_(True)
    with pytest.raises(NotImplementedError, match='rays'):
      model.apply({'params': params}, r, warp_extra={'alpha': 4.0})
  out = model.apply({'params': params}, rays, warp_extra={'alpha': 4.0})
  leaf = params['nerf_mlps_coarse']['MLP_0']['hidden_0']['kernel']
  (g,) = torch.autograd.grad(out['coarse']['rgb'].sum(), leaf, create_graph=True)
  with pytest.raises(RuntimeError, match='once_differentiable|does not require grad|double backward'):
    g.sum().backward()
  wf = model.create_warp_field(model, 1)
  pts = torch.rand(10, 3, device=DEV)
  ids = torch.zeros(10, 1, dtype=torch.int32, device=DEV)
  with pytest.raises(NotImplementedError, match='Jacobian'):
    wf.apply({'params': params['warp_field']}, pts, ids, {'alpha': 4.0}, return_jacobian=True)
  with pytest.raises(NotImplementedError, match='points'):
    wf.apply({'params': params['warp_field']}, pts.clone().requires_grad_(True), ids, {'alpha': 4.0})


def test_abi_errors():
  from nerfies_b200 import _lib
  c, model, params, rays = _grad_setup()
  hd = model.handle(8)
  hd.set_params(params)
  lib = hd.lib
  n = len(hd.param_specs)
  numels = [r * k for _, r, k in hd.param_specs]
  flat = torch.zeros(sum(numels), device=DEV)
  ptrs, off = (ctypes.c_void_p * n)(), 0
  for i, k in enumerate(numels):
    ptrs[i] = flat.data_ptr() + 4 * off
    off += k
  nm = (ctypes.c_longlong * n)(*numels)
  o, d = rays['origins'].contiguous(), rays['directions'].contiguous()
  z = torch.rand(8, c.spec.num_coarse_samples, device=DEV).sort(-1).values
  g = torch.rand(8, 6, device=DEV)
  p = lambda t: ctypes.c_void_p(t.data_ptr())
  s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

  def vjp(B=8, o_=o, z_c=z, z_f=None, d_c=g, d_f=None, nm_=nm, count=n, flags=0, code=None):
    return lib.nfb_render_vjp(hd.h, B, p(o_) if o_ is not None else None, p(d), None, None, None, None, 4.0, flags,
                              p(z_c) if z_c is not None else None, p(z_f) if z_f is not None else None,
                              p(d_c) if d_c is not None else None, p(d_f) if d_f is not None else None,
                              None, None, None, None, p(code) if code is not None else None, None, None, 0, ptrs,
                              nm_, count, s)

  def err():
    return lib.nfb_last_error().decode()

  assert vjp() == 0
  assert vjp(o_=None) < 0 and 'null' in err()
  assert vjp(z_c=None) < 0 and 'null' in err()
  assert vjp(d_f=g) < 0 and 'z values' in err()                       # fine cotangents without z_fine
  assert vjp(count=n - 1) < 0 and 'expected' in err()
  bad = (ctypes.c_longlong * n)(*[k + 1 for k in numels])
  assert vjp(nm_=bad) < 0 and 'expected' in err()
  assert vjp(B=10**6) < 0 and 'max_rays' in err()
  assert vjp(code=g) < 0 and 'METADATA_ENCODED' in err()
  assert lib.nfb_render_vjp(None, 8, *[None] * 6, 0.0, 0, *[None] * 11, 0, ptrs, nm, n, s) < 0
  pts = torch.rand(8, 3, device=DEV)
  ids = torch.zeros(8, dtype=torch.int32, device=DEV)
  assert lib.nfb_warp_vjp(hd.h, 8, p(pts), p(ids), 4.0, 0, p(pts), None, ptrs, nm, n, s) == 0
  assert lib.nfb_warp_vjp(hd.h, 8, p(pts), p(ids), 4.0, 0, None, None, ptrs, nm, n, s) < 0 and 'null' in err()
  assert lib.nfb_warp_vjp(hd.h, 8, p(pts), p(ids), 4.0, 0, p(pts), None, None, nm, n, s) < 0
  assert lib.nfb_warp_vjp(hd.h, 8, p(pts), p(ids), 4.0, 0, p(pts), None, ptrs, nm, n - 1, s) < 0
  assert lib.nfb_warp_vjp(hd.h, -1, p(pts), p(ids), 4.0, 0, p(pts), None, ptrs, nm, n, s) < 0
  assert lib.nfb_warp_vjp(hd.h, 8, p(pts), p(ids), 4.0, 0, p(pts), p(pts), ptrs, nm, n, s) < 0
  torch.cuda.synchronize()
  del _lib


# ---------------------------------------------------------------------------
# warp_field.apply
# ---------------------------------------------------------------------------
@pytest.mark.parametrize('kind', ['se3', 'translation', 'time', 'blend', 'encoded'])
def test_warp_field_vjp(kind):
  if kind in ('translation', 'time', 'blend'):
    g = Golden(kind + '_small')
    spec, params = g.spec, g.params
  else:
    spec = _small_spec()
    params = O.make_trained_like(O.init_params(spec, 90), seed=91)
  ta = 0.7 if spec.warp_metadata_encoder_type != 'glo' else None
  P = 300
  gen = torch.Generator().manual_seed(92)
  pts = torch.rand(P, 3, generator=gen) * 0.6 - 0.3
  if kind == 'encoded':
    meta = torch.rand(P, spec.num_warp_features, generator=gen) * 0.05
  elif spec.warp_metadata_encoder_type == 'time':
    meta = torch.rand(P, 1, generator=gen)
  else:
    meta = torch.randint(0, spec.num_warp_embeddings, (P, 1), generator=gen, dtype=torch.int32)
  cot = torch.randn(P, 3, generator=gen, dtype=torch.float64)
  model = model_from_spec(spec_to_dict(spec), device=DEV, batch_size=128)     # 300 points: chunks of 128
  wp = tree_to_device(params['warp_field'], DEV)
  leaves = flatten(wp)
  for v in leaves.values():
    v.requires_grad_(True)
  m = meta.to(DEV)
  if kind == 'encoded':
    m = m.clone().requires_grad_(True)
  out = model.create_warp_field(model, 1).apply({'params': wp}, pts.to(DEV), m, {'alpha': 3.0, 'time_alpha': ta},
                                               metadata_encoded=kind == 'encoded')
  (out['warped_points'].double() * cot.to(DEV)).sum().backward()
  got = {k: v.grad.cpu().double() for k, v in leaves.items()}
  if kind == 'encoded':
    got['code'] = m.grad.cpu().double()

  def oracle(dtype):
    p = {k: v.detach().clone().to(dtype).requires_grad_(True) for k, v in flatten(params['warp_field']).items()}
    tree = {}
    for k, v in p.items():
      node = tree
      for part in k.split('/')[:-1]:
        node = node.setdefault(part, {})
      node[k.split('/')[-1]] = v
    md = meta.to(dtype).clone().requires_grad_(True) if kind == 'encoded' else meta
    w = O.warp_field_apply(tree, spec, pts.to(dtype), md, 3.0, metadata_encoded=kind == 'encoded', time_alpha=ta)
    (w.double() * cot).sum().backward()
    r = {k: (v.grad if v.grad is not None else torch.zeros_like(v)).double() for k, v in p.items()}
    if kind == 'encoded':
      r['code'] = md.grad.double()
    return r

  ref, r32 = oracle(torch.float64), oracle(torch.float32)
  floor = 1e-4 * _scale(ref)
  for k, r in ref.items():
    tol = max(TOL, 3 * _rel(r32[k], r, floor))
    assert _rel(got[k], r, floor) <= tol, (k, _rel(got[k], r, floor), tol)


# ---------------------------------------------------------------------------
# 6. test-time optimisation of an appearance code
# ---------------------------------------------------------------------------
def test_appearance_code_optimisation():
  """Render a small frame with appearance code a*, then fit a code from a0 with torch.optim.Adam through
  model.apply(metadata_encoded=True): the photometric loss falls by at least 10x."""
  spec = _small_spec(use_camera_metadata=False, num_appearance_features=8)
  c = Case(spec, 256, seed=100, encoded=True)
  model = model_from_spec(spec_to_dict(spec), device=DEV, batch_size=256)
  params = tree_to_device(c.params, DEV)
  rays = tree_to_device(c.rays, DEV)
  gen = torch.Generator().manual_seed(101)
  a_star = (torch.rand(1, spec.num_appearance_features, generator=gen) * 2 - 1).to(DEV)
  md = dict(rays['metadata'], appearance=a_star.expand(256, -1).contiguous())
  with torch.no_grad():
    target = model.apply({'params': params}, dict(rays, metadata=md), warp_extra={'alpha': 4.0},
                         metadata_encoded=True)['fine']['rgb']
  a = torch.zeros(1, spec.num_appearance_features, device=DEV, requires_grad=True)
  opt = torch.optim.Adam([a], lr=0.05)
  losses = []
  for _ in range(STEPS):
    opt.zero_grad()
    md = dict(rays['metadata'], appearance=a.expand(256, -1))
    out = model.apply({'params': params}, dict(rays, metadata=md), warp_extra={'alpha': 4.0}, metadata_encoded=True)
    loss = ((out['fine']['rgb'] - target)**2).mean()
    loss.backward()
    opt.step()
    losses.append(float(loss))
  reached = next((i for i, l in enumerate(losses) if l * 10 <= losses[0]), None)
  print(f'appearance code fit: loss {losses[0]:.3e} -> {losses[-1]:.3e}, 10x reached at step {reached}')
  assert losses[-1] * 10 <= losses[0], losses


# Measured on an H100 80GB HBM3: the loss first fell 10x at step 22 (1.70e-2 -> 7.6e-9 after 150 steps), so 150
# steps leave a margin of ~7x.
STEPS = 150
