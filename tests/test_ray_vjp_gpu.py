"""NerfModel.render_rays and nfb_render_ray_vjp: the renderer's adjoint with respect to the rays.

The gradients of <cot, outputs> with respect to origins, directions, viewdirs and (metadata_encoded=True) the
codes are held to torch.autograd of the oracle in float64 at the kernel's z values (O.render_level), under
test_render_vjp_gpu.py's tier-A rule: max(2e-4, 3 x band), the band being the larger of the fp32 oracle's
distance from fp64 and the distance fp64 moves when the rays and parameters move by fp32 round-off.  Errors
are relative to the largest element of each tensor, floored at 1e-4 of the call's largest ray gradient.
"""
import ctypes

import pytest
import torch

from oracle import nerfies_oracle as O
from tests.golden_util import flatten, model_from_spec, spec_to_dict, tree_to_device
from tests.test_render_vjp_gpu import (DIMS, OUTPUTS, TOL, Case, _cotangents, _dot, _gin_spec, _golden_case,
                                       _moved, _rel, _small_spec)

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
RAY_KEYS = ('origins', 'directions', 'viewdirs')


def _ray_case(c, viewdirs=False, nonunit=False, seed=0):
  """c with non-unit directions (|d| in [0.5, 2]) and / or a viewdirs key (unit, near the directions)."""
  gen = torch.Generator().manual_seed(seed + 77)
  B = c.rays['origins'].shape[0]
  rays = dict(c.rays)
  if nonunit:
    rays['directions'] = (rays['directions'] * (0.5 + 1.5 * torch.rand(B, 1, generator=gen))).float()
  if viewdirs:
    v = rays['directions'] + 0.3 * torch.randn(B, 3, generator=gen)
    rays['viewdirs'] = (v / torch.linalg.norm(v, dim=-1, keepdim=True)).float()
  c.rays = rays
  return c


def _d_out(cot, lv, B):
  d = cot.get(lv, {})
  if not any(k in d for k in ('rgb', 'depth', 'acc')):
    return None
  out = torch.zeros(B, 6, dtype=torch.float64)
  if 'rgb' in d:
    out[:, 0:3] = d['rgb']
  if 'depth' in d:
    out[:, 3] = d['depth']
  if 'acc' in d:
    out[:, 5] = d['acc']
  return out


def _abi_ray_vjp(model, c, cot, z, chunk=0, fill=0.0, outputs=RAY_KEYS, codes=True):
  """nfb_render_ray_vjp called directly (every cotangent, warped_points included) -> {name: grad}."""
  params = tree_to_device(c.params, DEV)
  rays = tree_to_device(c.rays, DEV)
  B = rays['origins'].shape[0]
  hd = model.handle(B)
  hd.set_params(params)
  model._set_time_alpha(hd, c.time_alpha)
  md = rays['metadata']
  ids = model._call_metadata(rays, B, c.encoded, c.use_warp and c.spec.use_warp)
  flags = (0 if c.use_warp else 1 << 1) | (4 if c.encoded else 0)
  f32 = lambda t: None if t is None else t.to(DEV, torch.float32).contiguous()
  cots = []
  for key in ('d_out', 'weights', 'warped_points'):
    for lv in ('coarse', 'fine'):
      if key == 'd_out':
        cots.append(f32(_d_out(cot, lv, B)))
      else:
        t = cot.get(lv, {}).get(key)
        cots.append(f32(t.reshape(B, -1) if t is not None else None))
  out = {}
  for k in outputs:
    if k == 'viewdirs' and 'viewdirs' not in rays:
      continue
    out[k] = torch.full((B, 3), fill, device=DEV)
  widths = {'warp': model.num_warp_features, 'appearance': model.num_appearance_features,
            'camera': model.num_camera_features}
  code_out = {k: torch.zeros(B, widths[k], device=DEV) for k in md} if (c.encoded and codes) else {}
  zs = [f32(z['coarse']), f32(z.get('fine'))]          # held until the call has read them
  p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
  rc = hd.lib.nfb_render_ray_vjp(
      hd.h, B, p(rays['origins'].contiguous()), p(rays['directions'].contiguous()),
      p(rays['viewdirs'].contiguous()) if 'viewdirs' in rays else None, *[p(t) for t in ids],
      float(c.warp_alpha), flags, p(zs[0]), p(zs[1]), *[p(t) for t in cots],
      p(out.get('origins')), p(out.get('directions')), p(out.get('viewdirs')), p(code_out.get('warp')),
      p(code_out.get('appearance')), p(code_out.get('camera')), chunk, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
  assert rc == 0, hd.lib.nfb_last_error().decode()
  torch.cuda.synchronize()
  return {**{k: v.cpu().double() for k, v in out.items()}, **{k: v.cpu().double() for k, v in code_out.items()}}


def _cuda_ray_grads(c, cot, model=None, chunk=None):
  """Gradients of <cot, render_rays(...)> from loss.backward() (through nfb_render_ray_vjp) and the z values; a
  warped_points cotangent goes through the ABI directly at the same z."""
  model = model or model_from_spec(spec_to_dict(c.spec), device=DEV)
  if chunk:
    model.vjp_chunk_rays = chunk
  params = tree_to_device(c.params, DEV)
  rays = tree_to_device(c.rays, DEV)
  leaves = {k: rays[k].clone().requires_grad_(True) for k in RAY_KEYS if k in rays}
  rays = dict(rays, **leaves)
  codes = {}
  if c.encoded:
    codes = {k: v.clone().requires_grad_(True) for k, v in rays['metadata'].items()}
    rays['metadata'] = codes
  kw = dict(t_rand=None if c.t_rand is None else c.t_rand.to(DEV),
            u_rand=None if c.u_rand is None else c.u_rand.to(DEV))
  out = model.render_rays({'params': params}, rays, warp_extra=c.warp_extra, metadata_encoded=c.encoded,
                          use_warp=c.use_warp, **kw)
  z = {lv: out[lv]['z_vals'].detach().cpu() for lv in out}
  if any('warped_points' in d for d in cot.values()):
    return _abi_ray_vjp(model, c, cot, z, chunk=chunk or 0), z
  _dot({lv: {k: v for k, v in out[lv].items()} for lv in out}, cot).backward()
  torch.cuda.synchronize()
  got = {k: v.grad.cpu().double() for k, v in {**leaves, **codes}.items() if v.grad is not None}
  return got, z


def _oracle_ray_grads(c, cot, z, dtype, rays=None, params=None):
  rays = rays or c.rays
  leaves = {k: rays[k].detach().clone().to(dtype).requires_grad_(True) for k in RAY_KEYS if k in rays}
  md = rays['metadata']
  codes = {}
  if c.encoded:
    codes = {k: v.detach().clone().to(dtype).requires_grad_(True) for k, v in md.items()}
    md = codes
  r = dict(rays, **leaves, metadata=md)
  p = O.tree_to(params if params is not None else c.params, dtype)
  outs = {lv: O.render_level(p, c.spec, lv, r, z[lv], c.warp_alpha, use_warp=c.use_warp, dtype=dtype,
                             metadata_encoded=c.encoded, time_alpha=c.time_alpha) for lv in z}
  _dot(outs, cot).backward()
  return {k: (v.grad if v.grad is not None else torch.zeros_like(v)).double() for k, v in {**leaves, **codes}.items()}


def _check(name, c, cot, got, z):
  ref = _oracle_ray_grads(c, cot, z, torch.float64)
  g32 = _oracle_ray_grads(c, cot, z, torch.float32)
  moved = []
  for seed in (1, 2):
    mr, mp = _moved(c, seed)
    moved.append(_oracle_ray_grads(c, cot, z, torch.float64, rays=mr, params=mp))
  floor = 1e-4 * max(float(v.abs().max()) for v in ref.values())
  bad, worst = {}, (0.0, None)
  for k, r in ref.items():
    assert k in got, (name, k, sorted(got))
    band = max([_rel(g32[k], r, floor)] + [_rel(m[k], r, floor) for m in moved])
    err = _rel(got[k].reshape(r.shape), r, floor)
    tol = max(TOL, 3.0 * band)
    worst = max(worst, (err / tol, k, err, band), key=lambda t: t[0])
    if not err <= tol:
      bad[k] = (err, tol)
  print(f'{name}: worst error / tolerance {worst}')
  assert not bad, f'{name}: {bad}'


def _run(name, c, which, seed=0, **kw):
  cot = _cotangents(c, which, seed)
  got, z = _cuda_ray_grads(c, cot, **kw)
  _check(name, c, cot, got, z)


# ---------------------------------------------------------------------------
# 1. against fp64 autograd on the oracle
# ---------------------------------------------------------------------------
_GIN = {}


def _gin_case(dims):
  if dims not in _GIN:
    c = Case(_gin_spec(dims), 12, seed=500 + len(dims), warp_alpha=DIMS[dims]['alpha'])
    _GIN[dims] = _ray_case(c, viewdirs=False, nonunit=True, seed=len(dims))
  return _GIN[dims]


@pytest.mark.parametrize('which', [(k,) for k in OUTPUTS] + [OUTPUTS], ids=lambda w: '+'.join(w))
@pytest.mark.parametrize('dims', ['quarterhd', 'vrig'])
def test_gin_dims(dims, which):
  _run(f'{dims} {which}', _gin_case(dims), which, seed=len(which))


@pytest.mark.parametrize('dims', ['quarterhd', 'vrig'])
def test_tf32x3(dims):
  c = _gin_case(dims)
  model = model_from_spec(spec_to_dict(c.spec), device=DEV)
  model.train_precision = 'tf32x3'
  _run(f'{dims} tf32x3', c, OUTPUTS, seed=11, model=model)


def _pivot_translation():
  return Case(_small_spec(warp_use_pivot=True, warp_use_translation=True), 24, seed=30)


_VARIANTS = {
    'se3': lambda: _ray_case(Case(_small_spec(), 24, seed=31), viewdirs=True, nonunit=True),
    'se3_pivot_translation': lambda: _ray_case(_pivot_translation(), viewdirs=True, nonunit=True),
    'translation': lambda: _ray_case(_golden_case('translation_small'), nonunit=True),
    'time': lambda: _ray_case(_golden_case('time_small'), viewdirs=True, nonunit=True),
    'call_no_warp': lambda: _ray_case(Case(_small_spec(), 24, seed=32, use_warp=False), nonunit=True),
    'model_no_warp': lambda: _ray_case(Case(_small_spec(use_warp=False), 24, seed=33), viewdirs=True, nonunit=True),
    'viewdirs_key': lambda: _ray_case(Case(_small_spec(), 24, seed=34), viewdirs=True),
    'no_viewdirs_key': lambda: _ray_case(Case(_small_spec(), 24, seed=35)),
    'unit_directions': lambda: Case(_small_spec(), 24, seed=36),
    'no_use_viewdirs': lambda: _ray_case(Case(_small_spec(use_viewdirs=False), 24, seed=37), viewdirs=True,
                                         nonunit=True),
    'white_background': lambda: _ray_case(Case(_small_spec(use_white_background=True), 24, seed=38), nonunit=True),
    'no_sample_at_infinity': lambda: _ray_case(Case(_small_spec(use_sample_at_infinity=False), 24, seed=39),
                                               nonunit=True),
    'relu_sigma': lambda: _ray_case(Case(_small_spec(sigma_activation='relu'), 24, seed=40), nonunit=True),
    'encoded': lambda: _ray_case(Case(_small_spec(), 24, seed=41, encoded=True), viewdirs=True, nonunit=True),
    'coarse_only': lambda: _ray_case(Case(_small_spec(num_fine_samples=0), 24, seed=43), nonunit=True),
    'stratified': lambda: _ray_case(Case(_small_spec(), 24, seed=44, stratified=True), nonunit=True),
}


@pytest.mark.parametrize('variant', list(_VARIANTS))
def test_variants(variant):
  c = _VARIANTS[variant]()
  warps = c.spec.use_warp and c.use_warp
  _run(variant, c, OUTPUTS if warps else OUTPUTS[:4], seed=5)


@pytest.mark.parametrize('which', [(k,) for k in OUTPUTS[:4]], ids=lambda w: w[0])
def test_encoded_each_cotangent(which):
  c = _VARIANTS['encoded']()
  _run(f'encoded {which}', c, which, seed=6)


# ---------------------------------------------------------------------------
# 2. an independent check: d_warped alone against the forward-mode warp Jacobian
# ---------------------------------------------------------------------------
@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('kind', ['se3', 'pivot_translation', 'translation'])
def test_warped_cotangent_equals_jacobian_transpose(kind, precision):
  """With only a d_warped cotangent, d_origins = sum_s J_s^T g_s and d_directions = sum_s z_s J_s^T g_s with
  J_s = nfb_warp_jacobian at x_s = o + z_s d (forward mode on the tangent tape).  Both sides are fp32 sums of
  the same S per-sample terms, reached by different arithmetic (reverse through the warp MLP's dX GEMMs vs
  its tangent GEMMs); the bound per element is 2e-4 of the sum of the terms' magnitudes,
  sum_s |J_s|^T |g_s| (and with z_s), the tier-A rule on the scale each element is formed at."""
  c = {'se3': lambda: Case(_small_spec(), 24, seed=60), 'pivot_translation': _pivot_translation,
       'translation': lambda: _golden_case('translation_small')}[kind]()
  c = _ray_case(c, nonunit=True, seed=61)
  model = model_from_spec(spec_to_dict(c.spec), device=DEV)
  model.train_precision = precision
  B = c.rays['origins'].shape[0]
  cot = {'coarse': {'warped_points': torch.randn(B, c.spec.num_coarse_samples, 3, dtype=torch.float64,
                                                  generator=torch.Generator().manual_seed(62))}}
  with torch.no_grad():
    out = model.render_rays({'params': tree_to_device(c.params, DEV)}, tree_to_device(c.rays, DEV),
                            warp_extra=c.warp_extra)
  z = {'coarse': out['coarse']['z_vals'].cpu()}
  got = _abi_ray_vjp(model, c, cot, z)
  rays = tree_to_device(c.rays, DEV)
  S = c.spec.num_coarse_samples
  zc = z['coarse'].to(DEV)
  pts = (rays['origins'][:, None, :] + zc[:, :, None] * rays['directions'][:, None, :]).reshape(-1, 3).contiguous()
  md = rays['metadata']
  meta = md['time'] if c.spec.warp_metadata_encoder_type == 'time' else md['warp']
  ids = meta.reshape(B, 1).expand(B, S).reshape(-1).contiguous()
  jac = torch.empty(B * S, 3, 3, device=DEV)
  hd = model.handle(B * S)
  hd.set_params(tree_to_device(c.params, DEV))
  p = lambda t: ctypes.c_void_p(t.data_ptr())
  assert hd.lib.nfb_warp_jacobian(hd.h, B * S, p(pts), p(ids), float(c.warp_alpha), None, p(jac),
                                  ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
  torch.cuda.synchronize()
  J = jac.cpu().double().reshape(B, S, 3, 3)
  g = cot['coarse']['warped_points']
  terms = torch.einsum('bsij,bsi->bsj', J, g)                 # J_s^T g_s
  mags = torch.einsum('bsij,bsi->bsj', J.abs(), g.abs())
  zz = z['coarse'].double()[:, :, None]
  for name, ref, mag in (('origins', terms.sum(1), mags.sum(1)),
                         ('directions', (zz * terms).sum(1), (zz.abs() * mags).sum(1))):
    err = (got[name] - ref).abs()
    ratio = float((err / (2e-4 * mag)).max())
    print(f'{kind} {precision} {name}: worst error / bound {ratio:.3f}')
    assert ratio <= 1.0, (name, ratio)


# ---------------------------------------------------------------------------
# 3. invariants
# ---------------------------------------------------------------------------
def test_chunks_agree_and_outputs_overwrite():
  c = _ray_case(Case(_small_spec(), 40, seed=70), viewdirs=True, nonunit=True)
  model = model_from_spec(spec_to_dict(c.spec), device=DEV)
  cot = _cotangents(c, OUTPUTS, 71)
  with torch.no_grad():
    out = model.render_rays({'params': tree_to_device(c.params, DEV)}, tree_to_device(c.rays, DEV),
                            warp_extra=c.warp_extra)
  z = {lv: out[lv]['z_vals'].cpu() for lv in out}
  runs = [_abi_ray_vjp(model, c, cot, z, chunk=40) for _ in range(2)]
  scale = max(float(v.abs().max()) for v in runs[0].values())
  noise = max(float((runs[1][k] - runs[0][k]).abs().max()) for k in runs[0]) / scale
  for chunk in (17, 40):
    g = _abi_ray_vjp(model, c, cot, z, chunk=chunk, fill=float('nan'))
    for k in runs[0]:
      d = float((g[k] - runs[0][k]).abs().max()) / scale
      assert d <= max(3 * noise, 1e-6), (chunk, k, d, noise)
  _check('chunk 17', c, cot, _abi_ray_vjp(model, c, cot, z, chunk=17, fill=1e30), z)


def test_no_weight_gradient_kernels():
  """The ray VJP forms no dW GEMM (AtomicAdd epilogue) and no bias column sum; render_rays leaves the
  parameters' .grad None and refuses parameters that require grad."""
  from torch.profiler import ProfilerActivity, profile
  c = _ray_case(Case(_small_spec(), 24, seed=80), viewdirs=True, nonunit=True)
  for prec in ('fp32', 'tf32x3'):
    model = model_from_spec(spec_to_dict(c.spec), device=DEV)
    model.train_precision = prec
    params = tree_to_device(c.params, DEV)
    rays = tree_to_device(c.rays, DEV)
    o = rays['origins'].clone().requires_grad_(True)
    out = model.render_rays({'params': params}, dict(rays, origins=o), warp_extra=c.warp_extra)
    loss = out['fine']['rgb'].sum() + out['coarse']['acc'].sum()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
      loss.backward()
      torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    assert any('ray_reduce_kernel' in n for n in names), prec
    assert any('gemm' in n for n in names), prec
    assert not any('colsum_kernel' in n for n in names), prec
    assert not any('gemm' in n and 'AtomicAdd' in n for n in names), prec
    assert o.grad is not None and bool(torch.isfinite(o.grad).all())
    for v in flatten(params).values():
      assert v.grad is None
    leaf = params['nerf_mlps_coarse']['MLP_0']['hidden_0']['kernel']
    leaf.requires_grad_(True)
    with pytest.raises(ValueError, match='requires grad'):
      model.render_rays({'params': params}, rays, warp_extra=c.warp_extra)


def test_apply_unchanged_by_render_rays():
  """model.apply and its parameter VJP on the same handle: the outputs bitwise, the gradients within their
  run-to-run noise (float atomicAdd order), before and after a render_rays call and its backward."""
  c = _ray_case(Case(_small_spec(), 24, seed=90), nonunit=True)
  model = model_from_spec(spec_to_dict(c.spec), device=DEV)
  rays = tree_to_device(c.rays, DEV)

  def apply_and_grads():
    params = tree_to_device(c.params, DEV)
    leaves = flatten(params)
    for v in leaves.values():
      v.requires_grad_(True)
    out = model.apply({'params': params}, rays, warp_extra=c.warp_extra, return_weights=True)
    (out['fine']['rgb'].sum() + out['coarse']['depth'].sum()).backward()
    torch.cuda.synchronize()
    return ({k: v.detach().clone() for lv in out for k, v in out[lv].items()},
            {k: v.grad.clone() for k, v in leaves.items()})

  out0, g0 = apply_and_grads()
  out1, g1 = apply_and_grads()
  d = rays['directions'].clone().requires_grad_(True)
  rr = model.render_rays({'params': tree_to_device(c.params, DEV)}, dict(rays, directions=d), warp_extra=c.warp_extra)
  rr['fine']['rgb'].sum().backward()
  out2, g2 = apply_and_grads()
  scale = max(float(v.abs().max()) for v in g0.values())
  noise = max(float((g1[k] - g0[k]).abs().max()) for k in g0) / scale
  for k in out0:
    assert torch.equal(out0[k], out2[k]), k
  for k in g0:
    assert float((g2[k] - g0[k]).abs().max()) / scale <= max(3 * noise, 1e-7), k


def test_render_rays_forward_equals_apply():
  c = _ray_case(Case(_small_spec(), 24, seed=95), viewdirs=True, nonunit=True)
  model = model_from_spec(spec_to_dict(c.spec), device=DEV)
  params = tree_to_device(c.params, DEV)
  rays = tree_to_device(c.rays, DEV)
  with torch.no_grad():
    ref = model.apply({'params': params}, rays, warp_extra=c.warp_extra, return_weights=True)
  got = model.render_rays({'params': params}, rays, warp_extra=c.warp_extra)
  for lv in ref:
    for k in ('rgb', 'depth', 'med_depth', 'acc', 'weights'):
      assert torch.equal(ref[lv][k], got[lv][k]), (lv, k)


def test_abi_errors():
  c = _ray_case(Case(_small_spec(), 8, seed=100), viewdirs=True)
  model = model_from_spec(spec_to_dict(c.spec), device=DEV)
  hd = model.handle(8)
  hd.set_params(tree_to_device(c.params, DEV))
  lib = hd.lib
  rays = tree_to_device(c.rays, DEV)
  o, d = rays['origins'].contiguous(), rays['directions'].contiguous()
  ids = model._call_metadata(rays, 8, False, True)
  z = torch.rand(8, c.spec.num_coarse_samples, device=DEV).sort(-1).values
  g = torch.rand(8, 6, device=DEV)
  out = torch.zeros(8, 3, device=DEV)
  wp = torch.rand(8, c.spec.num_coarse_samples, 3, device=DEV)
  p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
  s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

  def vjp(h=hd.h, B=8, flags=0, d_c=g, d_f=None, wp_c=None, d_o=out, d_v=None, v=None, code=None):
    return lib.nfb_render_ray_vjp(h, B, p(o), p(d), p(v), *[p(t) for t in ids], 4.0, flags, p(z), p(z), p(d_c),
                                  p(d_f), None, None, p(wp_c), None, p(d_o), None, p(d_v), p(code), None, None, 0, s)

  err = lambda: lib.nfb_last_error().decode()
  assert vjp() == 0
  assert vjp(h=None) < 0 and 'null' in err()
  assert vjp(d_o=None) < 0 and 'null' in err()
  assert vjp(code=torch.zeros(8, c.spec.num_warp_features, device=DEV)) < 0 and 'METADATA_ENCODED' in err()
  assert vjp(d_f=g, flags=1) < 0 and 'fine' in err()
  assert vjp(wp_c=wp, flags=2) < 0 and 'warp' in err()
  assert vjp(d_v=out) < 0 and 'viewdirs' in err()
  assert vjp(B=10**6) < 0 and 'max_rays' in err()
  assert vjp(B=0) == 0
  torch.cuda.synchronize()
