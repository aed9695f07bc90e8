"""CUDA path (through the C ABI) vs the golden fixtures recorded from the
reference's own source, and vs the oracle at larger sizes.

Tolerance: 1e-4 with the metric |a-b| / (|b| + 1e-2) per level (the north-star's
"1e-4 relative fp32"), asserted stage by stage because hierarchical resampling
is ill-conditioned in empty space (see tests/test_oracle_golden.py); resampling
is checked in CDF space; end to end the stated bound is 2e-3.
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import nerfies_oracle as O
from tests.golden_util import (CASES, Golden, med_depth_ok, model_from_spec,
                               rel_err, spec_to_dict, tree_to_device)

pytestmark = pytest.mark.gpu
TOL = 1e-4
TOL_E2E = 2e-3
_REPORT = []


@pytest.fixture(scope='module', autouse=True)
def _write_report():
  yield
  import json
  import os
  os.makedirs('gpurun_out', exist_ok=True)
  with open('gpurun_out/parity_report.json', 'w') as f:
    json.dump([dict(case=c, level=l, key=k, err_vs_fp64=e, fp32_band=b)
               for c, l, k, e, b in _REPORT], f, indent=1)
DEV = 'cuda:0'


def _render_level(model, params, level, rays, z, alpha, use_warp=True, time_alpha=0.0):
  """nfb_render_samples through the C ABI."""
  from nerfies_b200 import _lib
  from nerfies_b200.models import _prep_f32, _prep_ids, _ptr, _stream
  hd = model.handle(z.shape[0])
  hd.set_params(params)
  B, S = z.shape
  dev = model.device
  o = _prep_f32(rays['origins'], dev)
  d = _prep_f32(rays['directions'], dev)
  md = rays.get('metadata', {})
  ids = [_prep_ids(md.get(k), dev) for k in ('warp', 'appearance', 'camera')]
  if model.use_warp and model.warp_metadata_encoder_type == 'time':
    ids[0] = _prep_f32(md['time'], dev).reshape(-1)      # metadata['time'] (models.py:252-254)
  model._set_time_alpha(hd, time_alpha)
  zc = _prep_f32(z, dev)
  out = torch.empty(B, 6, device=dev)
  w = torch.empty(B, S, device=dev)
  smp = torch.empty(B, S, 4, device=dev)
  wp = torch.empty(B, S, 3, device=dev)
  flags = 0 if use_warp else _lib.FLAG_NO_WARP
  _lib.check(hd.lib.nfb_render_samples(
      hd.h, level, B, S, _ptr(zc), _ptr(o), _ptr(d), None, _ptr(ids[0]),
      _ptr(ids[1]), _ptr(ids[2]), float(alpha), flags, _ptr(out), _ptr(w),
      _ptr(smp), _ptr(wp), _stream()))
  torch.cuda.synchronize()
  return {'rgb': out[:, :3].cpu(), 'depth': out[:, 3].cpu(),
          'med_depth': out[:, 4].cpu(), 'acc': out[:, 5].cpu(),
          'weights': w.cpu(), 'warped_points': wp.cpu(), 'samples': smp.cpu()}


def _check_level(name, level, got, ref, z, use_warp):
  keys = ['rgb', 'depth', 'acc', 'weights']
  if use_warp:
    keys.append('warped_points')
  for k in keys:
    err = rel_err(got[k], ref[k])
    assert err < TOL, f'{name} {level}/{k}: rel err {err:.3e}'
  assert med_depth_ok(got['med_depth'], ref, z), f'{name} {level}/med_depth'


def _golden_model(g, precision):
  """The tensor-core modes cover relu MLPs up to 256 wide with encoded inputs and
  conditions of up to 64 columns; for other models they refuse loudly - skip those."""
  from nerfies_b200 import _lib
  model = model_from_spec(g.spec_dict, device=DEV, precision=precision)
  if precision != 'fp32':
    try:
      model.handle(64)
    except _lib.NfbError as e:
      assert 'use precision fp32' in str(e)
      pytest.skip(f'{g.name}: not a tensor-core shape ({e})')
  return model


@pytest.mark.parametrize('precision', ['fp32', 'fp16x3'])
@pytest.mark.parametrize('name', CASES)
def test_coarse_level_vs_reference_source(name, precision):
  g = Golden(name)
  model = _golden_model(g, precision)
  params = tree_to_device(g.params, DEV)
  z = g.out['coarse'].get('z_vals')
  if z is None:
    z, _ = O.sample_along_rays(g.rays['origins'], g.rays['directions'],
                               g.spec.num_coarse_samples, g.spec.near,
                               g.spec.far, g.spec.use_linear_disparity,
                               g.t_rand)
  got = _render_level(model, params, 0, g.rays, z, g.warp_alpha, time_alpha=g.time_alpha)
  _check_level(name, 'coarse', got, g.out['coarse'], z, g.spec.use_warp)


@pytest.mark.parametrize('precision', ['fp32', 'fp16x3'])
@pytest.mark.parametrize('name', CASES)
def test_fine_level_given_reference_z(name, precision):
  g = Golden(name)
  model = _golden_model(g, precision)
  params = tree_to_device(g.params, DEV)
  z = g.out['fine']['z_vals']
  got = _render_level(model, params, 1, g.rays, z, g.warp_alpha, time_alpha=g.time_alpha)
  _check_level(name, 'fine', got, g.out['fine'], z, g.spec.use_warp)


@pytest.mark.parametrize('name', CASES)
def test_coarse_z_and_resample(name):
  from nerfies_b200 import _lib
  from nerfies_b200.models import _ptr, _stream
  g = Golden(name)
  spec = g.spec
  model = model_from_spec(g.spec_dict, device=DEV)
  hd = model.handle(64)
  hd.set_params(tree_to_device(g.params, DEV))
  B = g.rays['origins'].shape[0]
  # sample_along_rays z_vals: bit-exact against the oracle's float32 table.
  t_rand = g.t_rand.to(DEV).contiguous() if g.t_rand is not None else None
  zc = torch.empty(B, spec.num_coarse_samples, device=DEV)
  _lib.check(hd.lib.nfb_coarse_z_vals(hd.h, B, _ptr(t_rand), _ptr(zc),
                                      _stream()))
  z_ref, _ = O.sample_along_rays(g.rays['origins'], g.rays['directions'],
                                 spec.num_coarse_samples, spec.near, spec.far,
                                 spec.use_linear_disparity, g.t_rand)
  if g.t_rand is None:
    assert torch.equal(zc.cpu(), z_ref.contiguous()), 'coarse z not bit-exact'
    assert torch.equal(zc.cpu(), g.out['coarse']['z_vals'])
  else:
    assert rel_err(zc.cpu(), z_ref) < 1e-6
  # sample_pdf on the reference's coarse weights.
  w = g.out['coarse']['weights'].to(DEV).contiguous()
  u_rand = g.u_rand.to(DEV).contiguous() if g.u_rand is not None else None
  zf = torch.empty(B, spec.num_coarse_samples + spec.num_fine_samples,
                   device=DEV)
  zc_in = z_ref.to(DEV).contiguous()
  _lib.check(hd.lib.nfb_sample_pdf(hd.h, B, _ptr(zc_in), _ptr(w), _ptr(u_rand),
                                   _ptr(zf), _stream()))
  torch.cuda.synchronize()
  zf = zf.cpu()
  ref = g.out['fine']['z_vals']
  assert bool((zf[:, 1:] >= zf[:, :-1]).all()), 'z_fine not sorted'
  assert float((zf - ref).abs().max()) < 2e-3 * (spec.far - spec.near)
  # CDF-space check of the new samples: remove the coarse z's from the union.
  z_mid = .5 * (z_ref[..., 1:] + z_ref[..., :-1])
  wts = g.out['coarse']['weights'][..., 1:-1]
  if g.u_rand is None:
    u = torch.from_numpy(np.linspace(0., 1., spec.num_fine_samples,
                                     dtype=np.float32)).expand(B, -1)
  else:
    u = g.u_rand
  for b in range(B):
    union = zf[b].tolist()
    for v in z_ref[b].tolist():
      union.remove(min(union, key=lambda x: abs(x - v)))
    z_new = torch.tensor(sorted(union))
    res = O.pdf_cdf_residual(z_mid[b:b + 1], wts[b:b + 1], z_new[None],
                             torch.sort(u[b:b + 1], -1).values)
    assert float(res.max()) < 5e-6, (name, b, float(res.max()))


_E2E_BAND = {}


def _e2e_tol(g, key, encoded=False):
  """End-to-end tolerance through the ill-conditioned inverse-CDF resampling.

  TOL_E2E, or three times the distance between the fixture (the reference's fp32 numpy
  run) and the oracle's fp64 shadow on the same inputs when that is larger: no
  fp32 implementation can agree with the fixture better than exact arithmetic
  does (e.g. 2.0e-3 on `acc` for encoded_small)."""
  ck = (g.name, encoded)
  if ck not in _E2E_BAND:
    rays = dict(g.rays, metadata=g.enc['metadata']) if encoded else g.rays
    ref = (g.enc['out'] if encoded else g.out)['fine']
    o64 = O.render_forward(g.params, g.spec, rays, warp_alpha=g.warp_alpha, metadata_encoded=encoded,
                           t_rand=g.t_rand, u_rand=g.u_rand, dtype=torch.float64,
                           time_alpha=g.time_alpha)['fine']
    _E2E_BAND[ck] = {k: rel_err(o64[k], ref[k]) for k in ('rgb', 'depth', 'acc')}
  return max(TOL_E2E, 3.0 * _E2E_BAND[ck][key])


@pytest.mark.parametrize('precision', ['fp32', 'fp16x3'])
@pytest.mark.parametrize('name', CASES)
def test_end_to_end_apply(name, precision):
  g = Golden(name)
  model = _golden_model(g, precision)
  params = tree_to_device(g.params, DEV)
  for return_points in (False, True):
    out = model.apply({'params': params}, g.rays,
                      warp_extra={'alpha': g.warp_alpha, 'time_alpha': g.time_alpha},
                      return_weights=True, return_points=return_points,
                      t_rand=g.t_rand, u_rand=g.u_rand)
    torch.cuda.synchronize()
    for k in ('rgb', 'depth', 'acc', 'weights'):
      assert rel_err(out['coarse'][k].cpu(), g.out['coarse'][k]) < TOL
    for k in ('rgb', 'depth', 'acc'):
      err = rel_err(out['fine'][k].cpu(), g.out['fine'][k])
      if not return_points:    # measured (not only bounded) end-to-end error per fixture -> the report
        _REPORT.append((f'{name}[{precision}] e2e vs fixture', 'fine', k, err, _e2e_tol(g, k)))
      assert err < _e2e_tol(g, k), f'{name} fine/{k}: {err:.3e} (tol {_e2e_tol(g, k):.1e})'
    if return_points:
      assert rel_err(out['coarse']['points'].cpu(),
                     g.out['coarse']['points']) < 1e-6
      assert out['fine']['points'].shape == g.out['fine']['points'].shape


@pytest.mark.parametrize('precision', ['fp32', 'fp16x3'])
@pytest.mark.parametrize('name', [c for c in CASES if c != 'nowarp_variants'])
def test_warp_forward(name, precision):
  g = Golden(name)
  model = _golden_model(g, precision)
  wf = model.create_warp_field(model, num_batch_dims=1)
  out = wf.apply({'params': tree_to_device(g.params, DEV)}, g.warp['points'],
                 g.warp['ids'], {'alpha': g.warp_alpha, 'time_alpha': g.time_alpha},
                 False, False)
  torch.cuda.synchronize()
  err = rel_err(out['warped_points'].cpu(), g.warp['warped_points'])
  assert err < TOL, f'{name}: {err:.3e}'
  # the reference call site passes the warp subtree only (training.py:127-131), and
  # metadata_encoded=True takes per-point embeddings (warping.py:186-187, 378)
  sub = {'params': tree_to_device(g.params, DEV)['warp_field']}
  out = wf.apply(sub, g.warp['points'], g.warp['enc_embed'],
                 {'alpha': g.warp_alpha, 'time_alpha': g.time_alpha}, False, True)
  torch.cuda.synchronize()
  err = rel_err(out['warped_points'].cpu(), g.warp['enc_warped_points'])
  assert err < TOL, f'{name} (metadata_encoded, warp subtree): {err:.3e}'
  # a changed warp subtree must take effect (no stale cached weights)
  import copy
  p2 = copy.deepcopy(g.params['warp_field'])
  head = 'branches_v' if g.spec.warp_field_type == 'se3' else 'mlp'
  p2[head]['logit']['bias'] = p2[head]['logit']['bias'] + 0.25
  out2 = wf.apply({'params': tree_to_device(p2, DEV)}, g.warp['points'], g.warp['enc_embed'],
                  {'alpha': g.warp_alpha, 'time_alpha': g.time_alpha}, False, True)
  torch.cuda.synchronize()
  assert float((out2['warped_points'] - out['warped_points']).abs().max()) > 1e-2


def test_metadata_encoded_apply():
  """metadata_encoded=True through model.apply (NFB_FLAG_METADATA_ENCODED): vs the
  reference source's encoded run, and bit-identical to the id path when the
  embeddings handed in are the GLO table rows."""
  g = Golden('encoded_small')
  model = model_from_spec(g.spec_dict, device=DEV)
  params = tree_to_device(g.params, DEV)
  rays = dict(g.rays, metadata=g.enc['metadata'])
  extra = {'alpha': g.warp_alpha, 'time_alpha': 0.0}
  for return_points in (False, True):
    out = model.apply({'params': params}, rays, warp_extra=extra, metadata_encoded=True,
                      return_weights=True, return_points=return_points)
    torch.cuda.synchronize()
    for k in ('rgb', 'depth', 'acc', 'weights'):
      err = rel_err(out['coarse'][k].cpu(), g.enc['out']['coarse'][k])
      assert err < TOL, f'encoded coarse/{k}: {err:.3e}'
    for k in ('rgb', 'depth', 'acc'):
      err = rel_err(out['fine'][k].cpu(), g.enc['out']['fine'][k])
      tol = _e2e_tol(g, k, encoded=True)
      assert err < tol, f'encoded fine/{k}: {err:.3e} (tol {tol:.1e})'
    if return_points:
      err = rel_err(out['coarse']['warped_points'].cpu(), g.enc['out']['coarse']['warped_points'])
      assert err < TOL, f'encoded warped points: {err:.3e}'
  p = g.params
  md = g.rays['metadata']
  emb = {'warp': p['warp_field']['metadata_encoder']['embed']['embedding'][md['warp'][:, 0].long()],
         'appearance': p['appearance_encoder']['embed']['embedding'][md['appearance'][:, 0].long()],
         'camera': p['camera_encoder']['embed']['embedding'][md['camera'][:, 0].long()]}
  a = model.apply({'params': params}, dict(g.rays, metadata=emb), warp_extra=extra, metadata_encoded=True)
  b = model.apply({'params': params}, g.rays, warp_extra=extra)
  torch.cuda.synchronize()
  for lv in ('coarse', 'fine'):
    for k in ('rgb', 'depth', 'acc'):
      assert torch.equal(a[lv][k], b[lv][k]), (lv, k)
  with pytest.raises(ValueError):
    model.apply({'params': params}, dict(g.rays, metadata={**emb, 'warp': emb['warp'][:, :3]}),
                warp_extra=extra, metadata_encoded=True)


def test_use_warp_false_override():
  g = Golden('se3_small')
  model = model_from_spec(g.spec_dict, device=DEV)
  params = tree_to_device(g.params, DEV)
  z = g.out['coarse']['z_vals']
  got = _render_level(model, params, 0, g.rays, z, g.warp_alpha,
                      use_warp=False)
  ref = O.render_level(g.params, g.spec, 'coarse', g.rays, z, g.warp_alpha,
                       use_warp=False)
  for k in ('rgb', 'depth', 'acc', 'weights'):
    assert rel_err(got[k], ref[k]) < TOL


# ---------------------------------------------------------------------------
# Oracle comparisons at larger sizes (gin-file dimensions).
# ---------------------------------------------------------------------------
def _oracle_case(spec, num_rays, seed, alpha, precision='fp32'):
  p = O.make_trained_like(O.init_params(spec, seed), seed=seed + 1)
  rays = O.synthetic_rays(num_rays, spec, seed=seed + 2)
  model = model_from_spec(spec_to_dict(spec), device=DEV, batch_size=num_rays,
                          precision=precision)
  return p, rays, model


# Both parity-holding modes: fp32 (CUDA cores) and fp16x3 (wgmma, three fp16 MMA
# chains per layer into one fp32 accumulator) must meet the same 1e-4 per stage.
@pytest.mark.parametrize('precision', ['fp32', 'fp16x3'])
@pytest.mark.parametrize('dims', ['quarterhd', 'vrig', 'fullhd_small'])
def test_levels_vs_oracle(dims, precision):
  if dims == 'quarterhd':
    spec = O.OracleSpec(num_coarse_samples=128, num_fine_samples=128,
                        near=0.02, far=0.83, num_nerf_point_freqs=8,
                        sigma_activation='softplus', use_warp=True,
                        use_appearance_metadata=True, num_warp_embeddings=200,
                        num_appearance_embeddings=200)
    n, alpha = 96, 8.0
  elif dims == 'vrig':
    spec = O.OracleSpec(num_coarse_samples=128, num_fine_samples=128,
                        near=0.02, far=0.83, num_nerf_point_freqs=8,
                        num_warp_freqs=6, sigma_activation='softplus',
                        use_warp=True, use_camera_metadata=True,
                        num_warp_embeddings=150, num_camera_embeddings=2)
    n, alpha = 80, 2.7
  else:
    spec = O.OracleSpec(num_coarse_samples=256, num_fine_samples=256,
                        near=0.02, far=0.83, num_nerf_point_freqs=10,
                        sigma_activation='softplus', use_warp=True,
                        use_appearance_metadata=True, num_warp_embeddings=50,
                        num_appearance_embeddings=50)
    n, alpha = 33, 8.0   # ragged: 33*256 rows is not a multiple of the tile
  p, rays, model = _oracle_case(spec, n, 5, alpha, precision)
  ref = O.render_forward(p, spec, rays, warp_alpha=alpha, return_points=True)
  pg = tree_to_device(p, DEV)
  # The truth is the fp64 shadow; the fp32 oracle's own distance from it is the
  # round-off band of the algorithm (e.g. 1 - exp(-x) in empty space), which the
  # CUDA result is allowed on top of the 1e-4 tolerance.
  for lv, level in ((0, 'coarse'), (1, 'fine')):
    z = ref[level]['z_vals']
    got = _render_level(model, pg, lv, rays, z, alpha)
    r64 = O.render_level(p, spec, level, rays, z, alpha, dtype=torch.float64)
    for k in ('rgb', 'depth', 'acc', 'weights', 'warped_points'):
      band = rel_err(ref[level][k], r64[k])
      err = rel_err(got[k], r64[k])
      _REPORT.append((f'{dims}[{precision}]', level, k, err, band))
      assert err < TOL + 2 * band, (
          f'{dims} {level}/{k}: err vs fp64 {err:.3e}, fp32 band {band:.3e}')
    assert med_depth_ok(got['med_depth'], ref[level], z)
  out = model.apply({'params': pg}, rays, warp_extra={'alpha': alpha})
  torch.cuda.synchronize()
  for k in ('rgb', 'depth', 'acc'):
    err = rel_err(out['fine'][k].cpu(), ref['fine'][k])
    assert err < TOL_E2E, f'{dims} e2e fine/{k}: {err:.3e}'
  mse = float(((out['fine']['rgb'].cpu() - ref['fine']['rgb'])**2).mean())
  assert -10 * np.log10(max(mse, 1e-20)) > 70, 'PSNR vs oracle below 70 dB'


# ---------------------------------------------------------------------------
# Size-independent properties at the benchmark's full size.
# ---------------------------------------------------------------------------
# (max-rel coarse, max-rel fine on the oracle's z, max-rel end to end, PSNR dB) per mode: the
# bounds bench.py states for the rays it times.
_MODE_BOUNDS = {'fp32': (1e-4, 1e-4, 2e-3, 70.0), 'fp16x3': (1e-4, 1e-4, 2e-3, 70.0),
                'bf16': (8e-2, 8e-2, 1.5e-1, 35.0)}


@pytest.mark.parametrize('precision', ['fp32', 'fp16x3', 'bf16'])
def test_full_size_properties(precision):
  spec = O.OracleSpec(num_coarse_samples=128, num_fine_samples=128, near=0.02,
                      far=0.83, num_nerf_point_freqs=8,
                      sigma_activation='softplus', use_warp=True,
                      use_appearance_metadata=True, num_warp_embeddings=200,
                      num_appearance_embeddings=200)
  B = 8192
  p, rays, model = _oracle_case(spec, B, 9, 8.0, precision)
  rays_cpu = rays
  pg = tree_to_device(p, DEV)
  rays = {'origins': rays['origins'].to(DEV),
          'directions': rays['directions'].to(DEV),
          'metadata': {k: v.to(DEV) for k, v in rays['metadata'].items()}}
  out = model.apply({'params': pg}, rays, warp_extra={'alpha': 8.0},
                    return_weights=True, return_points=True)
  out2 = model.apply({'params': pg}, rays, warp_extra={'alpha': 8.0},
                     return_weights=True)
  torch.cuda.synchronize()
  # determinism, and the staged path (field kernel -> composite_kernel) == the one-call entry
  # point: bit for bit, except in fp16x3 mode where the one-call path finishes the ray inside the
  # field kernel (warp-shuffle product / sum scans instead of composite_kernel's sequential
  # scans): same values up to fp32 re-association.
  out2b = model.apply({'params': pg}, rays, warp_extra={'alpha': 8.0}, return_weights=True)
  torch.cuda.synchronize()
  for lv in ('coarse', 'fine'):
    for k in ('rgb', 'depth', 'med_depth', 'acc', 'weights'):
      assert torch.equal(out2[lv][k], out2b[lv][k]), (lv, k)
      if precision != 'fp16x3':
        assert torch.equal(out[lv][k], out2[lv][k]), (lv, k)
      elif lv == 'coarse' and k != 'med_depth':
        # (the fine level of the two paths sees coarse weights that differ in the last bits, and
        #  inverse-CDF resampling amplifies that: compared on the coarse level)
        assert rel_err(out[lv][k].cpu(), out2[lv][k].cpu()) < 5e-6, (lv, k)
  # rays are independent: any sub-batch renders to the same bits.
  sub = slice(1000, 1777)
  rs = {'origins': rays['origins'][sub], 'directions': rays['directions'][sub],
        'metadata': {k: v[sub] for k, v in rays['metadata'].items()}}
  out3 = model.apply({'params': pg}, rs, warp_extra={'alpha': 8.0})
  for k in ('rgb', 'depth', 'med_depth', 'acc'):
    assert torch.equal(out3['fine'][k], out2['fine'][k][sub]), k
  f = out['fine']
  z = f['z_vals']
  assert bool((z[:, 1:] >= z[:, :-1]).all())
  assert float(z.min()) >= spec.near - 1e-6 and float(z.max()) <= spec.far + 1e-6
  w = f['weights']
  assert bool(torch.isfinite(w).all()) and float(w.min()) >= 0
  # with the sample at infinity the last alpha is 1: weights sum to one.
  assert float((w.sum(-1) - 1).abs().max()) < 1e-4
  assert float(f['acc'].min()) >= 0 and float(f['acc'].max()) <= 1 + 1e-5
  assert float(f['rgb'].min()) >= 0 and float(f['rgb'].max()) <= 1 + 1e-5
  # every coarse z survives in the sorted union (model_utils.py:213).
  zc = out['coarse']['z_vals']
  idx = torch.searchsorted(z.contiguous(), zc.contiguous())
  assert torch.equal(torch.gather(z, 1, idx.clamp(max=z.shape[1] - 1)), zc)
  # a sample of the 8192 rays against the oracle (every 64th ray: rays from every
  # part of the grid), in this mode's stated bounds.
  pick = torch.arange(0, B, 64)
  sub_cpu = {'origins': rays_cpu['origins'][pick], 'directions': rays_cpu['directions'][pick],
             'metadata': {k: v[pick] for k, v in rays_cpu['metadata'].items()}}
  ref = O.render_forward(p, spec, sub_cpu, warp_alpha=8.0, return_points=True)
  b_coarse, b_fz, b_e2e, b_psnr = _MODE_BOUNDS[precision]
  for k in ('rgb', 'depth', 'acc', 'weights'):
    err = rel_err(out['coarse'][k][pick.to(DEV)].cpu(), ref['coarse'][k])
    assert err < b_coarse, f'[{precision}] coarse/{k} of the full-size batch: {err:.3e}'
  for k in ('rgb', 'depth', 'acc'):
    err = rel_err(out['fine'][k][pick.to(DEV)].cpu(), ref['fine'][k])
    assert err < b_e2e, f'[{precision}] e2e fine/{k} of the full-size batch: {err:.3e}'
  mse = float(((out['fine']['rgb'][pick.to(DEV)].cpu() - ref['fine']['rgb'])**2).mean())
  assert -10 * np.log10(max(mse, 1e-20)) > b_psnr
  got = _render_level(model, pg, 1, sub_cpu, ref['fine']['z_vals'], 8.0)
  for k in ('rgb', 'depth', 'acc', 'weights', 'warped_points'):
    err = rel_err(got[k], ref['fine'][k])
    assert err < b_fz, f'[{precision}] fine/{k} on the oracle z: {err:.3e}'


def test_host_entry_point_matches_device_path():
  g = Golden('quarterhd_dims')
  model = model_from_spec(g.spec_dict, device=DEV)
  params = tree_to_device(g.params, DEV)
  dev_out = model.apply({'params': params}, g.rays,
                        warp_extra={'alpha': g.warp_alpha})
  host_rays = {'origins': g.rays['origins'].numpy(),
               'directions': g.rays['directions'].numpy(),
               'metadata': {k: v.numpy() for k, v in g.rays['metadata'].items()}}
  host_out = model.apply_host({'params': params}, host_rays,
                              warp_extra={'alpha': g.warp_alpha})
  for lv in ('coarse', 'fine'):
    for k in ('rgb', 'depth', 'med_depth', 'acc'):
      assert np.array_equal(host_out[lv][k], dev_out[lv][k].cpu().numpy())


def test_errors_are_loud():
  from nerfies_b200 import _lib
  g = Golden('se3_small')
  model = model_from_spec(g.spec_dict, device=DEV)
  hd = model.handle(16)
  with pytest.raises(_lib.NfbError, match='nfb_set_params'):
    _lib.check(hd.lib.nfb_coarse_z_vals(hd.h, 4, None, None, None))
  bad = dict(g.params)
  bad = {k: v for k, v in bad.items() if k != 'warp_field'}
  with pytest.raises(KeyError):
    hd.set_params(tree_to_device(bad, DEV))


# ---------------------------------------------------------------------------
# Tensor-core path (precision='bf16'): bf16 operands, fp32 accumulation.
# Checked two ways: tightly against the oracle run with the same operand
# rounding (wiring / layout / pipeline bugs), and loosely against the fp32
# reference (what bf16 costs; reported, see DESIGN.md).
# ---------------------------------------------------------------------------
# bf16 rounding decisions flip on ~1e-7 accumulation-order differences, so the
# comparison with the emulating oracle is statistical: the MEAN deviation must be
# far below bf16's own error (measured: 3e-5 vs 1.6e-3), the max bounded.
TOL_BF16_MEAN = 4e-4
TOL_BF16_MAX = 8e-2


def _bf16_case(dims):
  if dims == 'quarterhd':
    spec = O.OracleSpec(num_coarse_samples=128, num_fine_samples=128,
                        near=0.02, far=0.83, num_nerf_point_freqs=8,
                        sigma_activation='softplus', use_warp=True,
                        use_appearance_metadata=True, num_warp_embeddings=200,
                        num_appearance_embeddings=200)
    return spec, 70, 8.0       # 70*128 rows: ragged last tile pair
  if dims == 'vrig':
    spec = O.OracleSpec(num_coarse_samples=128, num_fine_samples=128,
                        near=0.02, far=0.83, num_nerf_point_freqs=8,
                        num_warp_freqs=6, sigma_activation='softplus',
                        use_warp=True, use_camera_metadata=True,
                        num_warp_embeddings=150, num_camera_embeddings=2)
    return spec, 64, 2.7
  if dims == 'test_local':
    spec = O.OracleSpec(num_coarse_samples=64, num_fine_samples=64, near=0.02,
                        far=0.83, num_nerf_point_freqs=10, num_warp_features=3,
                        sigma_activation='softplus', use_warp=True,
                        use_appearance_metadata=True, num_warp_embeddings=20,
                        num_appearance_embeddings=20)
    return spec, 37, 5.5
  spec = O.OracleSpec(num_coarse_samples=96, num_fine_samples=32, near=0.1,
                      far=1.5, num_nerf_point_freqs=10, sigma_activation='relu',
                      use_warp=False, use_white_background=True)
  return spec, 50, 0.0


@pytest.mark.parametrize('dims', ['quarterhd', 'vrig', 'test_local', 'nowarp'])
def test_bf16_levels_vs_bf16_oracle(dims):
  spec, n, alpha = _bf16_case(dims)
  p = O.make_trained_like(O.init_params(spec, 21), seed=22)
  rays = O.synthetic_rays(n, spec, seed=23)
  model = model_from_spec(spec_to_dict(spec), precision='bf16', device=DEV,
                          batch_size=n)
  pg = tree_to_device(p, DEV)
  ref32 = O.render_forward(p, spec, rays, warp_alpha=alpha, return_points=True)
  for lv, level in ((0, 'coarse'), (1, 'fine')):
    z = ref32[level]['z_vals']
    got = _render_level(model, pg, lv, rays, z, alpha)
    with O.bf16_operands():
      ref = O.render_level(p, spec, level, rays, z, alpha)
    keys = ['rgb', 'depth', 'acc', 'weights']
    if spec.use_warp:
      keys.append('warped_points')
    smp = torch.cat([ref['sample_rgb'], ref['sample_sigma'][..., None]], -1)
    mean_s = float((got['samples'] - smp).abs().mean())
    assert mean_s < TOL_BF16_MEAN, f'{dims} {level}/samples mean {mean_s:.3e}'
    for k in keys:
      err = rel_err(got[k], ref[k])
      mean = float((got[k] - ref[k]).abs().mean())
      e32 = rel_err(got[k], ref32[level][k])
      _REPORT.append((f'bf16:{dims}', level, k, err, e32))
      assert mean < TOL_BF16_MEAN, f'{dims} {level}/{k}: mean {mean:.3e}'
      assert err < TOL_BF16_MAX, f'{dims} {level}/{k}: max {err:.3e}'


def test_bf16_end_to_end_and_host_path():
  spec, n, alpha = _bf16_case('quarterhd')
  p = O.make_trained_like(O.init_params(spec, 31), seed=32)
  rays = O.synthetic_rays(300, spec, seed=33)
  model = model_from_spec(spec_to_dict(spec), precision='bf16', device=DEV,
                          batch_size=300)
  pg = tree_to_device(p, DEV)
  out = model.apply({'params': pg}, rays, warp_extra={'alpha': alpha},
                    return_weights=True)
  out2 = model.apply({'params': pg}, rays, warp_extra={'alpha': alpha},
                     return_weights=True)
  torch.cuda.synchronize()
  for lv in ('coarse', 'fine'):
    for k in ('rgb', 'depth', 'med_depth', 'acc', 'weights'):
      assert torch.equal(out[lv][k], out2[lv][k]), (lv, k)   # deterministic
  ref = O.render_forward(p, spec, rays, warp_alpha=alpha)
  mse = float(((out['fine']['rgb'].cpu() - ref['fine']['rgb'])**2).mean())
  psnr = -10 * np.log10(max(mse, 1e-20))
  _REPORT.append(('bf16:e2e', 'fine', 'psnr_db_vs_fp32_oracle', psnr, 0.0))
  assert psnr > 35, f'bf16 end-to-end PSNR vs fp32 oracle {psnr:.1f} dB'
  sub = slice(100, 171)
  rs = {'origins': rays['origins'][sub], 'directions': rays['directions'][sub],
        'metadata': {k: v[sub] for k, v in rays['metadata'].items()}}
  out3 = model.apply({'params': pg}, rs, warp_extra={'alpha': alpha})
  assert torch.equal(out3['fine']['rgb'], out['fine']['rgb'][sub])


def test_bf16_rejects_unsupported_models():
  from nerfies_b200 import _lib
  g = Golden('se3_small')
  # elu hidden layers: the tensor-core kernels implement relu only
  model = model_from_spec({**g.spec_dict, 'activation': 'elu'}, precision='bf16', device=DEV)
  with pytest.raises(_lib.NfbError, match='precision fp32'):
    model.handle(16)
