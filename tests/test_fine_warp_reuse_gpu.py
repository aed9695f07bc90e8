"""The fine level of nfb_render_forward warps only its Nf new samples and reuses the coarse level's warped
points for the other Nc (render_fine_reusing_warp).  The staged path (return_points=True ->
nfb_render_samples) still warps every fine sample, so it is the yardstick here:

- model.apply against model.apply(..., return_points=True) with the same draws, every level output;
- the fine level alone: nfb_render_forward's fine outputs against nfb_render_samples(level 1) on the
  z_fine that nfb_render_forward returned, so both evaluate the field at the same samples.

fp32 and bf16 composite with composite_kernel on both paths and must agree bit for bit.  fp16x3 fuses the
composite into the field kernel when a level's samples are whole 128-row tiles and the staged path does
not; there the bounds of test_edge_cases_gpu.test_fused_composite_matches_the_staged_path apply, else
bit for bit as well.
"""
import pytest
import torch

from nerfies_b200 import _lib
from nerfies_b200.models import _prep_f32, _prep_ids, _ptr, _stream
from oracle import nerfies_oracle as O
from tests.golden_util import med_depth_rule_ok, model_from_spec, rel_err, spec_to_dict, tree_to_device

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ALPHA = 6.0
KEYS = ('rgb', 'depth', 'med_depth', 'acc', 'weights')

# name -> (OracleSpec overrides, rays, apply(use_warp=...))
CASES = {
    'se3_glo': (dict(), 300, True),
    'se3_pivot_translation': (dict(warp_use_pivot=True, warp_use_translation=True), 300, True),
    'translation': (dict(warp_field_type='translation'), 300, True),
    'time': (dict(warp_metadata_encoder_type='time', metadata_encoder_num_freqs=2), 300, True),
    'use_warp_false': (dict(), 300, False),
    # B * Nf = 37 * 64 is not a whole number of 128-row tiles: the warp-only pass ends on a tail tile
    'tail_tile': (dict(num_coarse_samples=64, num_fine_samples=64), 37, True),
    # Nc + Nf = 96 and Nc = 64: fp16x3 composites both levels with composite_kernel
    'staged_composite': (dict(num_coarse_samples=64, num_fine_samples=32), 300, True),
}


def _setup(case, precision, stratified):
  kw, B, use_warp = CASES[case]
  base = dict(num_coarse_samples=128, num_fine_samples=128, near=0.02, far=0.83, num_nerf_point_freqs=8,
              sigma_activation='softplus', use_warp=True, use_appearance_metadata=True,
              num_warp_embeddings=9, num_appearance_embeddings=9)
  spec = O.OracleSpec(**{**base, **kw})
  p = tree_to_device(O.make_trained_like(O.init_params(spec, 4)), DEV)
  model = model_from_spec(spec_to_dict(spec), precision=precision, device=DEV, batch_size=B)
  r = O.synthetic_rays(B, spec, seed=31)
  gen = torch.Generator().manual_seed(32)
  md = {k: v.to(DEV) for k, v in r['metadata'].items()}
  if spec.warp_metadata_encoder_type == 'time':
    md['time'] = torch.rand(B, 1, generator=gen).to(DEV)
  rays = {'origins': r['origins'].to(DEV), 'directions': r['directions'].to(DEV), 'metadata': md}
  draws = {}
  if stratified:
    draws = {'t_rand': torch.rand(B, spec.num_coarse_samples, generator=gen).to(DEV),
             'u_rand': torch.rand(B, spec.num_fine_samples, generator=gen).to(DEV)}
  return spec, model, {'params': p}, rays, draws, use_warp


def _fused(precision, S):
  return precision == 'fp16x3' and S % 128 == 0


def _assert_level(got, ref, fused, what, z):
  if not fused:
    for k in KEYS:
      assert torch.equal(got[k], ref[k]), f'{what}/{k}'
    return
  for k in ('rgb', 'depth', 'acc', 'weights'):
    assert rel_err(got[k].cpu(), ref[k].cpu()) < 5e-6, f'{what}/{k}'
  # median depth: the first sample whose cumulative weight reaches 0.5, on each path's own weights
  for lv in (got, ref):
    assert bool(med_depth_rule_ok(lv['med_depth'], lv['weights'], z).all()), f'{what}/med_depth'


@pytest.mark.parametrize('stratified', [False, True], ids=['deterministic', 'stratified'])
@pytest.mark.parametrize('case', sorted(CASES))
@pytest.mark.parametrize('precision', ['fp32', 'bf16', 'fp16x3'])
def test_apply_matches_the_staged_path(precision, case, stratified):
  spec, model, variables, rays, draws, use_warp = _setup(case, precision, stratified)
  kw = dict(warp_extra={'alpha': ALPHA, 'time_alpha': 1.0}, return_weights=True, use_warp=use_warp, **draws)
  out = model.apply(variables, rays, **kw)
  staged = model.apply(variables, rays, return_points=True, **kw)
  torch.cuda.synchronize()
  nc, nf = spec.num_coarse_samples, spec.num_fine_samples
  _assert_level(out['coarse'], staged['coarse'], _fused(precision, nc), 'coarse', staged['coarse']['z_vals'])
  if not _fused(precision, nc):
    # same coarse weights, so the same z_fine: the fine level must agree like the coarse one
    _assert_level(out['fine'], staged['fine'], _fused(precision, nc + nf), 'fine', staged['fine']['z_vals'])
  else:
    # the fused and staged coarse weights differ by re-association, and resampling moves z_fine with them
    # (the fine level on equal z_fine: test_fine_level_matches_render_samples)
    assert rel_err(out['fine']['rgb'].cpu(), staged['fine']['rgb'].cpu()) < 2e-3


@pytest.mark.parametrize('stratified', [False, True], ids=['deterministic', 'stratified'])
@pytest.mark.parametrize('case', sorted(CASES))
@pytest.mark.parametrize('precision', ['fp32', 'bf16', 'fp16x3'])
def test_fine_level_matches_render_samples(precision, case, stratified):
  spec, model, variables, rays, draws, use_warp = _setup(case, precision, stratified)
  model.apply(variables, rays, warp_extra={'alpha': ALPHA, 'time_alpha': 1.0})   # uploads the parameters
  B, nc, nf = rays['origins'].shape[0], spec.num_coarse_samples, spec.num_fine_samples
  n = nc + nf
  md = rays['metadata']
  warp_id = (_prep_f32(md['time'], DEV).reshape(-1) if spec.warp_metadata_encoder_type == 'time'
             else _prep_ids(md['warp'], DEV))
  app_id = _prep_ids(md['appearance'], DEV)
  flags = 0 if use_warp else _lib.FLAG_NO_WARP
  hd = model.handle(B)
  lib, h = hd.lib, hd.h
  o, d = rays['origins'].contiguous(), rays['directions'].contiguous()
  out_c, out_f = torch.empty(B, 6, device=DEV), torch.empty(B, 6, device=DEV)
  w_c, w_f = torch.empty(B, nc, device=DEV), torch.empty(B, n, device=DEV)
  z_f = torch.empty(B, n, device=DEV)
  _lib.check(lib.nfb_render_forward(h, B, _ptr(o), _ptr(d), None, _ptr(warp_id), _ptr(app_id), None, ALPHA,
                                    _ptr(draws.get('t_rand')), _ptr(draws.get('u_rand')), flags, _ptr(out_c),
                                    _ptr(out_f), _ptr(w_c), _ptr(w_f), _ptr(z_f), _stream()))
  out_s, w_s = torch.empty(B, 6, device=DEV), torch.empty(B, n, device=DEV)
  _lib.check(lib.nfb_render_samples(h, 1, B, n, _ptr(z_f), _ptr(o), _ptr(d), None, _ptr(warp_id), _ptr(app_id),
                                    None, ALPHA, flags, _ptr(out_s), _ptr(w_s), None, None, _stream()))
  torch.cuda.synchronize()
  level = lambda o6, w: {'rgb': o6[:, :3], 'depth': o6[:, 3], 'med_depth': o6[:, 4], 'acc': o6[:, 5], 'weights': w}
  _assert_level(level(out_f, w_f), level(out_s, w_s), _fused(precision, n), 'fine', z_f)
