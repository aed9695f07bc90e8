"""The fp16x3 NeRF pass with the bottleneck folded into the rgb branch and the alpha head (field_tc.cuh:
build_tc_program, fold_kernel; ray_kernels.cuh: ray_bias_kernel), at the gin sizes (trunk 256 x 8, skip at
4, rgb branch 128), against the fp32 CUDA-core mode (which keeps the unfolded layers) and the fp64 oracle.
bf16, which keeps the bottleneck as a layer, runs the same cases.

* Conditions: appearance (rgb condition), appearance as the alpha condition too, camera metadata (vrig).
* Sample counts of 48 and 88 per ray on the staged path (nfb_render_samples): 128-row tiles span rays,
  so each accumulator row must take its own ray's bias.  End to end with 128 + 128 samples, where the
  fp16x3 kernel fuses the composite and a tile is one ray.
* Re-fold: new parameters on a handle that already rendered give what a fresh handle gives.
"""
import pytest
import torch

from oracle import nerfies_oracle as O
from tests.golden_util import model_from_spec, rel_err, spec_to_dict, tree_to_device

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
TOL = 1e-4                 # per level, fp16x3 (test_parity_gpu.test_levels_vs_oracle)
TOL_E2E = 2e-3
TOL_BF16_MEAN = 4e-4       # test_parity_gpu.test_bf16_levels_vs_bf16_oracle
TOL_BF16_MAX = 8e-2
TOL_BF16_E2E = 1.5e-1

GIN = dict(near=0.02, far=0.83, num_nerf_point_freqs=8, sigma_activation='softplus',
           use_warp=True, warp_field_type='se3', num_warp_embeddings=5)
CASES = {
    'appearance': dict(use_appearance_metadata=True, num_appearance_embeddings=6),
    'alpha_condition': dict(use_appearance_metadata=True, num_appearance_embeddings=6, use_alpha_condition=True,
                            use_rgb_condition=True),
    'vrig': dict(use_camera_metadata=True, num_camera_embeddings=3, num_warp_freqs=6),
}
KEYS = ('rgb', 'depth', 'acc', 'weights', 'sample_rgb', 'sample_sigma')


def _spec(name, nc, nf):
  return O.OracleSpec(**GIN, **CASES[name], num_coarse_samples=nc, num_fine_samples=nf)


def _params(spec, seed):
  return O.make_trained_like(O.init_params(spec, seed), seed=seed + 1)


def _model(spec, precision, batch):
  return model_from_spec(spec_to_dict(spec), device=DEV, precision=precision, batch_size=batch)


def _levels(model, params, rays, z_by_level, alpha):
  from tests.test_parity_gpu import _render_level
  out = {}
  for lv, z in z_by_level.items():
    got = _render_level(model, params, 0 if lv == 'coarse' else 1, rays, z, alpha)
    out[lv] = dict(got, sample_rgb=got['samples'][..., :3], sample_sigma=got['samples'][..., 3])
  return out


def _sigma_err(got, ref):
  return float((got.double() - ref.double()).abs().max()) / float(ref.double().abs().max())


def _err(k, got, ref):
  return _sigma_err(got, ref) if k == 'sample_sigma' else rel_err(got, ref)


@pytest.mark.parametrize('precision', ['fp16x3', 'bf16'])
@pytest.mark.parametrize('name', sorted(CASES))
def test_staged_levels_with_tiles_across_rays(name, precision):
  """48 and 88 samples per ray: every 128-row tile holds rows of two or three rays."""
  spec = _spec(name, 48, 40)
  seed = 300 + sorted(CASES).index(name)
  p = _params(spec, seed)
  rays = O.synthetic_rays(7, spec, seed=seed + 2)
  alpha = 4.5
  e2e = O.render_forward(p, spec, rays, warp_alpha=alpha, return_points=True)
  zs = {lv: e2e[lv]['z_vals'] for lv in e2e}
  pg = tree_to_device(p, DEV)
  got = _levels(_model(spec, precision, 7), pg, rays, zs, alpha)
  simt = _levels(_model(spec, 'fp32', 7), pg, rays, zs, alpha)
  for lv, z in zs.items():
    r32 = O.render_level(p, spec, lv, rays, z, alpha)
    if precision == 'bf16':
      # at least as close to fp32 as the oracle with bf16 operands is (up to a quarter)
      with O.bf16_operands():
        rb = O.render_level(p, spec, lv, rays, z, alpha)
      for k in KEYS:
        g = got[lv][k].cpu().double()
        scale = float(r32[k].double().abs().max()) if k == 'sample_sigma' else 1.0
        mean = float((g - r32[k].double()).abs().mean()) / scale
        band = float((rb[k].double() - r32[k].double()).abs().mean()) / scale
        assert mean < max(TOL_BF16_MEAN, 1.25 * band), f'{name} {lv}/{k}: mean {mean:.3e}, bf16 band {band:.3e}'
        assert _err(k, got[lv][k].cpu(), r32[k]) < TOL_BF16_MAX, f'{name} {lv}/{k}'
      continue
    r64 = O.render_level(p, spec, lv, rays, z, alpha, dtype=torch.float64)
    for k in KEYS:
      band = _err(k, r32[k], r64[k])
      err = _err(k, got[lv][k].cpu(), r64[k])
      assert err < TOL + 2 * band, f'{name} {lv}/{k}: err vs fp64 {err:.3e}, fp32 band {band:.3e}'
      err = _err(k, got[lv][k].cpu(), simt[lv][k].cpu())
      assert err < TOL + 2 * band, f'{name} {lv}/{k}: err vs fp32 mode {err:.3e}'


@pytest.mark.parametrize('precision', ['fp16x3', 'bf16'])
@pytest.mark.parametrize('name', sorted(CASES))
def test_end_to_end_at_128_samples(name, precision):
  """128 + 128 samples: the fused composite (fp16x3), a tile is one ray; staged and fused agree."""
  spec = _spec(name, 128, 128)
  seed = 310 + sorted(CASES).index(name)
  p = _params(spec, seed)
  rays = O.synthetic_rays(5, spec, seed=seed + 2)
  alpha = 4.5
  ref = O.render_forward(p, spec, rays, warp_alpha=alpha)
  pg = tree_to_device(p, DEV)
  model = _model(spec, precision, 5)
  out = model.apply({'params': pg}, rays, warp_extra={'alpha': alpha}, return_weights=True)
  simt = _model(spec, 'fp32', 5).apply({'params': pg}, rays, warp_extra={'alpha': alpha}, return_weights=True)
  torch.cuda.synchronize()
  tol = TOL_BF16_E2E if precision == 'bf16' else TOL_E2E
  for k in ('rgb', 'depth', 'acc'):
    assert rel_err(out['fine'][k].cpu(), ref['fine'][k]) < tol, f'{name} e2e fine/{k}'
    assert rel_err(out['fine'][k].cpu(), simt['fine'][k].cpu()) < tol, f'{name} e2e fine/{k} vs fp32 mode'
  if precision == 'fp16x3':
    staged = model.apply({'params': pg}, rays, warp_extra={'alpha': alpha}, return_weights=True,
                         return_points=True)
    torch.cuda.synchronize()
    for k in ('rgb', 'depth', 'acc', 'weights'):
      assert rel_err(out['coarse'][k].cpu(), staged['coarse'][k].cpu()) < 5e-6, f'{name} fused vs staged {k}'


@pytest.mark.parametrize('precision', ['fp16x3', 'bf16'])
@pytest.mark.parametrize('name', ['alpha_condition', 'vrig'])
def test_new_params_are_folded_again(name, precision):
  """Render, upload different weights to the same handle, render again: the result is bitwise what a
  fresh model with those weights renders (a stale fold would keep the first weights' bottleneck)."""
  spec = _spec(name, 48, 40)
  rays = O.synthetic_rays(6, spec, seed=320)
  z = {'coarse': O.sample_along_rays(rays['origins'], rays['directions'], 48, spec.near, spec.far,
                                     spec.use_linear_disparity)[0]}
  p1 = tree_to_device(_params(spec, 321), DEV)
  p2 = tree_to_device(_params(spec, 331), DEV)
  model = _model(spec, precision, 6)
  first = _levels(model, p1, rays, z, 4.5)['coarse']
  again = _levels(model, p2, rays, z, 4.5)['coarse']
  fresh = _levels(_model(spec, precision, 6), p2, rays, z, 4.5)['coarse']
  for k in KEYS:
    assert torch.equal(again[k], fresh[k]), f'{name} {k}: the handle kept a stale fold'
  assert not torch.equal(first['rgb'], again['rgb'])


def test_new_params_after_a_train_step_are_folded_again():
  """One training step changes every parameter; the next fp16x3 render uses the new bottleneck."""
  from nerfies_b200 import training
  spec = _spec('alpha_condition', 48, 0)
  rays = O.synthetic_rays(6, spec, seed=340)
  p = tree_to_device(_params(spec, 341), DEV)
  target = torch.rand(6, 3, generator=torch.Generator().manual_seed(342))
  model32 = _model(spec, 'fp32', 6)
  _, grads = training.value_and_grad(model32, p, dict(rays, rgb=target), {'alpha': 4.5}, chunk_rays=6)
  g = training.grads_to_tree(model32, grads)
  p2 = _step(p, g)
  z = {'coarse': O.sample_along_rays(rays['origins'], rays['directions'], 48, spec.near, spec.far,
                                     spec.use_linear_disparity)[0]}
  model = _model(spec, 'fp16x3', 6)
  _levels(model, p, rays, z, 4.5)
  again = _levels(model, p2, rays, z, 4.5)['coarse']
  fresh = _levels(_model(spec, 'fp16x3', 6), p2, rays, z, 4.5)['coarse']
  for k in KEYS:
    assert torch.equal(again[k], fresh[k]), k


def _step(p, g, lr=1e-1):
  if isinstance(p, dict):
    return {k: _step(v, g[k], lr) for k, v in p.items()}
  return p - lr * g.to(p.device).reshape(p.shape)
