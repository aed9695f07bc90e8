"""The render and training kernels across the model architectures ModelConfig accepts, against the
fp64 oracle, and the loud refusal of every configuration one step past a limit.

The field kernels interpret a layer list (nfb_api.cu: build_programs) that the tensor-core paths
translate again (field_tc.cuh: build_tc_program): widths off multiples of 32 and with a partial second
128-column N-chunk, rgb branches of depth 0, the trunk condition, conditions and encoded inputs of
exactly 64 columns, the 12-column SE(3) head, the deepest nets, every hidden and sigma activation and
the smallest and largest sample counts.  Each case has its own seeded parameters and a batch whose
rows do not fill the last 64-row (CUDA-core) or 128-row (tensor-core) tile.

Per case and precision:
* each level on the oracle's z: rgb, depth, acc, weights, per-sample rgb / sigma and warped points
  against render_level in fp64 (fp32 / fp16x3: TOL + 2 x the fp32 oracle's own distance from fp64, as
  test_parity_gpu.test_levels_vs_oracle; bf16: against the oracle with bf16 operands, mean / max);
* model.apply end to end against the fp32 oracle;
* the training step's gradients (fp32 and tf32x3) on a coarse-only variant against fp64 autograd, and
  the warp Jacobian against the oracle's in fp64.
A configuration the tensor-core paths cannot run is refused by them and still matches in fp32.
"""
import dataclasses

import numpy as np
import pytest
import torch

from oracle import nerfies_oracle as O
from tests.golden_util import (flatten, med_depth_ok, model_from_spec, rel_err,
                               spec_to_dict, tree_to_device)

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
TOL = 1e-4                 # per level, fp32 / fp16x3 (test_parity_gpu.test_levels_vs_oracle)
TOL_E2E = 2e-3             # end to end through resampling, fp32 / fp16x3
TOL_BF16_MEAN = 4e-4       # test_parity_gpu.test_bf16_levels_vs_bf16_oracle
TOL_BF16_MAX = 8e-2
TOL_BF16_E2E, PSNR_BF16 = 1.5e-1, 35.0   # test_parity_gpu._MODE_BOUNDS['bf16']
TOL_GRAD = 2e-4            # of each tensor's max |g| (test_training_gpu; tf32x3 is held to the same)
TOL_JAC = 2e-5

BASE = dict(num_coarse_samples=48, num_fine_samples=40, near=0.02, far=0.83,
            num_nerf_point_freqs=6, nerf_trunk_width=64, nerf_trunk_depth=4, nerf_skips=(2,),
            nerf_rgb_branch_width=32, sigma_activation='softplus')
SE3 = dict(use_warp=True, warp_field_type='se3', num_warp_embeddings=5, warp_trunk_width=32,
           warp_trunk_depth=3, warp_skips=(2,))
APP = dict(use_appearance_metadata=True, num_appearance_embeddings=6)


@dataclasses.dataclass(frozen=True)
class Case:
  spec: dict
  tc: bool = True          # the tensor-core paths (bf16, fp16x3) accept it
  rays: int = 7            # 7 x 48 and 7 x 88 rows: ragged for 64- and 128-row tiles
  alpha: float = 4.5


CASES = {
    # trunk 100 (one partial N-chunk, K-blocks with padding rows), rgb 72 over two layers
    'odd_widths': Case(dict(nerf_trunk_width=100, nerf_trunk_depth=3, nerf_skips=(2,),
                            nerf_rgb_branch_width=72, nerf_rgb_branch_depth=2, **SE3, **APP)),
    # trunk 200: a second N-chunk of 72 columns; rgb 129: one column into a second chunk
    'ragged_chunk': Case(dict(nerf_trunk_width=200, nerf_trunk_depth=5, nerf_skips=(1, 3),
                              nerf_rgb_branch_width=129)),
    'tiny': Case(dict(nerf_trunk_width=16, nerf_trunk_depth=1, nerf_skips=(), nerf_rgb_branch_width=1)),
    # no condition, no rgb branch: alpha and the rgb logit both read the trunk's last layer
    'rgb_depth0_nocond': Case(dict(nerf_rgb_branch_depth=0, use_viewdirs=False)),
    # Dp + tc = 51 + 13 = 64: the trunk condition fills the tensor-core input block
    'trunk_condition': Case(dict(num_nerf_point_freqs=8, use_trunk_condition=True,
                                 num_appearance_features=13, **APP)),
    # rc = 27 (viewdirs) + 8 (appearance) + 29 (camera) = 64, ac = 8
    'rgb_cond_64': Case(dict(num_nerf_point_freqs=8, use_alpha_condition=True, use_rgb_condition=True,
                             num_appearance_features=8, use_camera_metadata=True, num_camera_features=29,
                             num_camera_embeddings=3, **APP)),
    # warp 129 wide (128-row tiles, just past the 256-row limit), Dw = 51 + 13 = 64
    'warp_edges': Case(dict(SE3, warp_trunk_width=129, warp_trunk_depth=4, num_warp_freqs=8,
                            num_warp_features=13)),
    'se3_full_head': Case(dict(SE3, warp_use_pivot=True, warp_use_translation=True, warp_trunk_width=128,
                               warp_trunk_depth=6, warp_skips=(4,))),
    # 16 SIMT steps in the NeRF net (12 trunk, bottleneck, alpha, rgb, logit); 9 warp steps:
    # 9 + 15 = 24 tensor-core steps (alpha is folded)
    'deepest': Case(dict(nerf_trunk_depth=12, nerf_skips=(4, 8), warp_trunk_depth=8, **{
        k: v for k, v in SE3.items() if k != 'warp_trunk_depth'}, num_coarse_samples=128,
                         num_fine_samples=128), rays=5),
    # Nc + Nf = 1024 = kMaxSamples: the fused composite (fp16x3) and composite_kernel at their limit
    'samples_max': Case(dict(num_coarse_samples=384, num_fine_samples=640, nerf_trunk_depth=2, nerf_skips=()),
                        rays=3),
    'samples_min': Case(dict(num_coarse_samples=3, num_fine_samples=1)),
    'samples_min_coarse': Case(dict(num_coarse_samples=2, num_fine_samples=0)),
    # ---- one step past a tensor-core limit: refused there, still exact in fp32 ----
    'rc_65': Case(dict(num_nerf_point_freqs=8, use_alpha_condition=True, use_rgb_condition=True,
                       num_appearance_features=8, use_camera_metadata=True, num_camera_features=30,
                       num_camera_embeddings=3, **APP), tc=False),
    'trunk_condition_65': Case(dict(num_nerf_point_freqs=8, use_trunk_condition=True,
                                    num_appearance_features=14, **APP), tc=False),
    'warp_dw_65': Case(dict(SE3, num_warp_freqs=8, num_warp_features=14), tc=False),
    'tc_steps_25': Case(dict(nerf_trunk_depth=12, nerf_skips=(4, 8), warp_trunk_depth=9, **{
        k: v for k, v in SE3.items() if k != 'warp_trunk_depth'}), tc=False, rays=5),
    # rgb logit on [bottleneck | viewdirs]: a head reading the encoded inputs
    'rgb_depth0_cond': Case(dict(nerf_rgb_branch_depth=0), tc=False),
    # the fp32 input block at kMaxIn = 128: 63 (posenc) + 38 (trunk condition) + 27 (viewdirs)
    'input_128': Case(dict(num_nerf_point_freqs=10, use_trunk_condition=True, num_appearance_features=38,
                           **APP), tc=False),
}
# Densities that can be negative (elu, leaky_relu, tanh) give negative weights, for which hierarchical resampling
# has no distribution to draw from: such cases are compared on given z only, and without the sample at
# infinity (a negative density over a distance of 1e10 has no finite transmittance).
NEGATIVE_SIGMA = ('elu', 'leaky_relu', 'tanh')
for _act in ('elu', 'leaky_relu', 'tanh', 'sigmoid'):
  CASES[f'sigma_{_act}'] = Case(dict(sigma_activation=_act, use_alpha_condition=True,
                                     use_sample_at_infinity=_act not in NEGATIVE_SIGMA, **APP))
for _act in ('elu', 'leaky_relu', 'tanh', 'sigmoid', 'softplus'):
  CASES[f'hidden_{_act}'] = Case(dict(activation=_act, nerf_rgb_branch_depth=2, **SE3), tc=False)
PRECISIONS = ['fp32', 'fp16x3', 'bf16']


def _spec(case, **over):
  return O.OracleSpec(**{**BASE, **case.spec, **over})


def _model(spec, precision, batch):
  return model_from_spec(spec_to_dict(spec), device=DEV, precision=precision, batch_size=batch)


def _tc_model(name, precision, batch):
  """The model in `precision`; None (after checking the refusal) where the tensor cores refuse it."""
  from nerfies_b200 import _lib
  case = CASES[name]
  model = _model(_spec(case), precision, batch)
  if precision != 'fp32' and not case.tc:
    with pytest.raises(_lib.NfbError, match='use precision fp32'):
      model.handle(batch)
    return None
  return model


_REF = {}


def _reference(name):
  """Parameters, rays, and per level: the oracle's z, the fp32 oracle and the fp64 oracle on it."""
  if name not in _REF:
    case = CASES[name]
    spec = _spec(case)
    seed = 100 + sorted(CASES).index(name)
    p = O.make_trained_like(O.init_params(spec, seed), seed=seed + 1)
    rays = O.synthetic_rays(case.rays, spec, seed=seed + 2)
    levels = {}
    if spec.sigma_activation in NEGATIVE_SIGMA:
      z_c, _ = O.sample_along_rays(rays['origins'], rays['directions'], spec.num_coarse_samples,
                                   spec.near, spec.far, spec.use_linear_disparity)
      z_f, _ = O.sample_along_rays(rays['origins'], rays['directions'],
                                   spec.num_coarse_samples + spec.num_fine_samples, spec.near, spec.far,
                                   spec.use_linear_disparity)
      zs = {'coarse': z_c, 'fine': z_f}
      e2e = None
    else:
      e2e = O.render_forward(p, spec, rays, warp_alpha=case.alpha, return_points=True)
      zs = {lv: e2e[lv]['z_vals'] for lv in e2e}
    for lv in (['coarse', 'fine'] if spec.num_fine_samples > 0 else ['coarse']):
      z = zs[lv]
      r32 = O.render_level(p, spec, lv, rays, z, case.alpha)
      r64 = O.render_level(p, spec, lv, rays, z, case.alpha, dtype=torch.float64)
      levels[lv] = (z, r32, r64)
    _REF[name] = (spec, p, rays, levels, e2e)
  return _REF[name]


def _err(k, got, ref):
  """rel_err; the per-sample densities (pre-activation sums of up to a few hundred terms, magnitudes
  in the tens) are measured against the largest density of the case instead."""
  if k != 'sample_sigma':
    return rel_err(got, ref)
  return float((got.double() - ref.double()).abs().max()) / float(ref.double().abs().max())


def _mean(k, got, ref):
  d = float((got.double() - ref.double()).abs().mean())
  return d / float(ref.double().abs().max()) if k == 'sample_sigma' else d


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('name', sorted(CASES))
def test_levels_vs_oracle(name, precision):
  from tests.test_parity_gpu import _render_level
  case = CASES[name]
  model = _tc_model(name, precision, case.rays)
  if model is None:
    return
  spec, p, rays, levels, _ = _reference(name)
  pg = tree_to_device(p, DEV)
  keys = ['rgb', 'depth', 'acc', 'weights', 'sample_rgb', 'sample_sigma']
  keys += ['warped_points'] if spec.use_warp else []
  for lv, (z, r32, r64) in levels.items():
    got = _render_level(model, pg, 0 if lv == 'coarse' else 1, rays, z, case.alpha)
    got = dict(got, sample_rgb=got['samples'][..., :3], sample_sigma=got['samples'][..., 3])
    if precision == 'bf16':
      with O.bf16_operands():
        rb = O.render_level(p, spec, lv, rays, z, case.alpha)
      for k in keys:
        mean, err = _mean(k, got[k], rb[k]), _err(k, got[k], rb[k])
        # bf16 rounding decisions flip on accumulation-order differences, and steep density heads
        # (sigmoid, tanh) amplify a flip: the kernel must be at least twice as close to the bf16
        # emulation as bf16 itself is to fp32
        bound = max(TOL_BF16_MEAN, 0.5 * _mean(k, rb[k], r32[k]))
        assert mean < bound, f'{name} {lv}/{k}: mean {mean:.3e} (bound {bound:.1e})'
        assert err < TOL_BF16_MAX, f'{name} {lv}/{k}: max {err:.3e}'
      continue
    for k in keys:
      band = _err(k, r32[k], r64[k])
      err = _err(k, got[k], r64[k])
      assert err < TOL + 2 * band, f'{name}[{precision}] {lv}/{k}: err vs fp64 {err:.3e}, fp32 band {band:.3e}'
    if spec.sigma_activation not in NEGATIVE_SIGMA:
      assert med_depth_ok(got['med_depth'], r32, z), f'{name}[{precision}] {lv}/med_depth'


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('name', sorted(CASES))
def test_end_to_end_vs_oracle(name, precision):
  case = CASES[name]
  spec = _spec(case)
  if spec.sigma_activation in NEGATIVE_SIGMA:
    pytest.skip('negative densities: hierarchical resampling is undefined (levels checked on given z)')
  model = _tc_model(name, precision, case.rays)
  if model is None:
    return
  spec, p, rays, _, ref = _reference(name)
  pg = tree_to_device(p, DEV)
  out = model.apply({'params': pg}, rays, warp_extra={'alpha': case.alpha}, return_weights=True)
  torch.cuda.synchronize()
  last = 'fine' if spec.num_fine_samples > 0 else 'coarse'
  tol = TOL_BF16_E2E if precision == 'bf16' else TOL_E2E
  for k in ('rgb', 'depth', 'acc'):
    err = rel_err(out[last][k].cpu(), ref[last][k])
    assert err < tol, f'{name}[{precision}] e2e {last}/{k}: {err:.3e}'
  if precision == 'bf16':
    mse = float(((out[last]['rgb'].cpu() - ref[last]['rgb'])**2).mean())
    assert -10 * np.log10(max(mse, 1e-20)) > PSNR_BF16
  if precision == 'fp16x3' and spec.num_coarse_samples % 128 == 0:
    # the fused path (volumetric rendering in the field kernel's epilogue) against the staged one
    staged = model.apply({'params': pg}, rays, warp_extra={'alpha': case.alpha}, return_weights=True,
                         return_points=True)
    torch.cuda.synchronize()
    for k in ('rgb', 'depth', 'acc', 'weights'):
      err = rel_err(out['coarse'][k].cpu(), staged['coarse'][k].cpu())
      assert err < 5e-6, f'{name} fused vs staged coarse/{k}: {err:.3e}'


def _coarse_only(name):
  """The case's coarse-only variant: one level, no resampling between the oracle and the kernels."""
  spec, p, rays, _, _ = _reference(name)
  spec = dataclasses.replace(spec, num_fine_samples=0)
  p = {k: v for k, v in p.items() if k != 'nerf_mlps_fine'}
  return spec, p, rays


@pytest.mark.parametrize('train_precision', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('name', sorted(CASES))
def test_gradients_vs_autograd(name, train_precision):
  from nerfies_b200 import training
  case = CASES[name]
  spec, p, rays = _coarse_only(name)
  B = rays['origins'].shape[0]
  target = torch.rand(B, 3, generator=torch.Generator().manual_seed(7))
  p64 = O.tree_to(p, torch.float64)
  leaves = flatten(p64)
  for v in leaves.values():
    v.requires_grad_(True)
  out = O.render_forward(p64, spec, rays, warp_alpha=case.alpha, dtype=torch.float64)
  loss = ((out['coarse']['rgb'] - target.double())**2).mean()
  loss.backward()
  model = _model(spec, 'fp32', B)
  model.train_precision = train_precision
  losses, grads = training.value_and_grad(model, tree_to_device(p, DEV), dict(rays, rgb=target),
                                          {'alpha': case.alpha}, chunk_rays=B)
  torch.cuda.synchronize()
  loss = float(loss.detach())
  assert abs(float(losses['coarse']) - loss) < 1e-5 * max(1.0, loss)
  got = flatten(training.grads_to_tree(model, grads))
  for k, v in leaves.items():
    r = v.grad if v.grad is not None else torch.zeros_like(v)
    a = got[k].cpu().double().reshape(r.shape)
    err = float((a - r).abs().max()) / (float(r.abs().max()) + 1e-12)
    assert err < TOL_GRAD, f'{name}[{train_precision}] {k}: {err:.3e}'
  if spec.use_warp:
    gen = torch.Generator().manual_seed(8)
    pts = torch.rand(37, 3, generator=gen) * 0.6 - 0.3
    ids = torch.randint(0, spec.num_warp_embeddings, (37, 1), generator=gen)
    wf = model.create_warp_field(model, num_batch_dims=1)
    jo = wf.apply({'params': tree_to_device(p, DEV)['warp_field']}, pts, ids, {'alpha': case.alpha},
                  return_jacobian=True)
    torch.cuda.synchronize()
    ref = O.warp_jacobian(p64['warp_field'], spec, pts.double(), ids, case.alpha).detach()
    err = float((jo['jacobian'].cpu().double() - ref).abs().max())
    assert err < TOL_JAC * max(1.0, float(ref.abs().max())), f'{name} warp Jacobian: {err:.3e}'


def test_training_step_at_max_samples():
  """Both levels of a training step with Nc + Nf = kMaxSamples: the fine level's composite_vjp_kernel
  holds 1024 samples per ray in shared memory."""
  from nerfies_b200 import training
  spec, p, rays, _, ref = _reference('samples_max')
  assert spec.num_coarse_samples + spec.num_fine_samples == 1024
  B = rays['origins'].shape[0]
  target = torch.rand(B, 3, generator=torch.Generator().manual_seed(9))
  model = _model(spec, 'fp32', B)
  losses, grads = training.value_and_grad(model, tree_to_device(p, DEV), dict(rays, rgb=target),
                                          {'alpha': CASES['samples_max'].alpha}, chunk_rays=B)
  torch.cuda.synchronize()
  for lv in ('coarse', 'fine'):
    lref = float(((ref[lv]['rgb'] - target)**2).mean())
    assert abs(float(losses[lv]) - lref) < 2e-3 * max(1e-3, lref), (lv, float(losses[lv]), lref)
  assert bool(torch.isfinite(grads).all()) and float(grads.abs().max()) > 0


# ---------------------------------------------------------------------------
# One step past each limit: nfb_create refuses the model with a message naming the limit.
# ---------------------------------------------------------------------------
def _refused(spec_over, precision, match):
  from nerfies_b200 import _lib
  spec = O.OracleSpec(**{**BASE, **spec_over})
  model = _model(spec, precision, 8)
  with pytest.raises(_lib.NfbError, match=match):
    model.handle(8)


TC_LIMITS = {
    'rc_65': (CASES['rc_65'].spec, 'rgb condition wider than 64'),
    'trunk_condition_65': (CASES['trunk_condition_65'].spec, 'encoded inputs wider than 64'),
    'warp_dw_65': (CASES['warp_dw_65'].spec, 'encoded inputs wider than 64'),
    'tc_steps_25': (CASES['tc_steps_25'].spec, 'too many layers'),
    'hidden_elu': (CASES['hidden_elu'].spec, 'hidden activation other than relu'),
    'rgb_depth0_cond': (CASES['rgb_depth0_cond'].spec, 'head reading the encoded inputs'),
}


@pytest.mark.parametrize('precision', ['fp16x3', 'bf16'])
@pytest.mark.parametrize('limit', sorted(TC_LIMITS))
def test_tensor_core_limits_are_refused(limit, precision):
  over, match = TC_LIMITS[limit]
  _refused(over, precision, match)


def test_alpha_condition_past_64_is_refused_everywhere():
  """ac = 65 implies rc >= 65 (the appearance code conditions both heads) and an input block of at
  least 3 + 65 + 65 > kMaxIn columns: refused by every precision."""
  over = dict(num_nerf_point_freqs=0, use_viewdirs=False, use_alpha_condition=True, use_rgb_condition=True,
              num_appearance_features=65, **APP)
  _refused(over, 'fp16x3', 'condition wider than 64|wider than 128')
  _refused(over, 'fp32', 'input feature block wider than 128')


HOST_LIMITS = {
    # kMaxSteps = 16 per network: these wrote past the end of Net::steps
    'trunk14_rgb0': (dict(nerf_trunk_depth=14, nerf_skips=(4,), nerf_rgb_branch_depth=0), 'too many layers'),
    'trunk15_rgb0': (dict(nerf_trunk_depth=15, nerf_skips=(4,), nerf_rgb_branch_depth=0), 'too many layers'),
    'trunk16': (dict(nerf_trunk_depth=16, nerf_skips=(4,)), 'too many layers'),
    'warp16': (dict(SE3, warp_trunk_depth=16, warp_skips=(4,)), 'too many layers'),
    # fp32 input block of 129 columns: 63 + 39 + 27
    'input_129': (dict(num_nerf_point_freqs=10, use_trunk_condition=True, num_appearance_features=39, **APP),
                  'input feature block wider than 128'),
    # samples per ray: composite refuses S > kMaxSamples, resample_kernel's shared memory grows with S
    'samples_1025': (dict(num_coarse_samples=385, num_fine_samples=640), 'more than 1024 samples per ray'),
    'coarse_1025': (dict(num_coarse_samples=1025, num_fine_samples=0), 'more than 1024 samples per ray'),
    'resample_smem': (dict(num_coarse_samples=1000, num_fine_samples=1000), 'more than 1024 samples per ray'),
    'resample_nc2': (dict(num_coarse_samples=2, num_fine_samples=4), 'needs >= 3 coarse samples'),
}


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('limit', sorted(HOST_LIMITS))
def test_host_limits_are_refused(limit, precision):
  over, match = HOST_LIMITS[limit]
  _refused(over, precision, match)


def test_deepest_nets_are_accepted():
  """The step just inside kMaxSteps: a NeRF trunk of 13 with rgb depth 0 and viewdirs is 16 steps."""
  spec = O.OracleSpec(**{**BASE, 'nerf_trunk_depth': 13, 'nerf_skips': (4,), 'nerf_rgb_branch_depth': 0})
  _model(spec, 'fp32', 8).handle(8)
  spec = O.OracleSpec(**{**BASE, **SE3, 'warp_trunk_depth': 15, 'warp_skips': (4,)})
  _model(spec, 'fp32', 8).handle(8)
