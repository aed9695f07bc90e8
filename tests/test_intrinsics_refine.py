"""Camera intrinsics refinement on the host: the per-ray intrinsics adjoint restated in fp64 against torch.autograd
through camera.py's unrolled pixels_to_rays, intrinsics groups, the checkpoint round trip, refined cameras, and the
refusals of the drivers and of registration.  No GPU."""
import os

import numpy as np
import pytest
import torch

from nerfies_b200 import camera as camera_lib
from nerfies_b200 import checkpoints
from nerfies_b200 import configs
from nerfies_b200 import geometry
from nerfies_b200 import train as train_lib
from nerfies_b200 import training
from oracle import nerfies_oracle as O
from tests.golden_util import model_from_spec, spec_to_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
CAPTURE = os.path.join(GOLDEN, 'capture_small')
CASES = ['camera_pinhole', 'camera_distorted', 'camera_skew_distorted']


def load_fixture(name):
  z = np.load(os.path.join(GOLDEN, name + '.npz'))
  c = {k[4:]: z[k] for k in z.files if k.startswith('cam_')}
  cam = camera_lib.Camera(**{k: v for k, v in c.items()})
  return cam, z['pixels'].reshape(-1, 2)


# ---------------------------------------------------------------------------
# fp64 references: the rays of a refined, posed camera (autograd), and the adjoint the kernel computes
# ---------------------------------------------------------------------------
def refined_rays(cam, q, omega, pixels):
  """camera.py:225-269 in float64 torch for the camera refined by the delta q (8,) and rotated by omega (3,)
  about its centre (geometry.pose_rays): the ten Newton steps unrolled, differentiable in q and omega.  Also
  returns the Newton residual after the last step.  Undistortion always runs: with zero coefficients it is the
  identity, as the kernel's skipped undistortion is."""
  t = lambda v: torch.as_tensor(np.asarray(v, np.float64))
  px, py = t(pixels[:, 0]), t(pixels[:, 1])
  f0 = float(cam.focal_length)
  f = f0 * torch.exp(q[0])
  cx, cy = float(cam.principal_point[0]) + f0 * q[1], float(cam.principal_point[1]) + f0 * q[2]
  k1, k2, k3 = (float(cam.radial_distortion[j]) + q[3 + j] for j in range(3))
  p1, p2 = (float(cam.tangential_distortion[j]) + q[6 + j] for j in range(2))
  y0 = (py - cy) / (f * float(cam.pixel_aspect_ratio))
  x0 = (px - cx - y0 * float(cam.skew)) / f

  def residual(x, y):
    r = x * x + y * y
    d = 1.0 + r * (k1 + r * (k2 + k3 * r))
    fx = d * x + 2 * p1 * x * y + p2 * (r + 2 * x * x) - x0
    fy = d * y + 2 * p2 * x * y + p1 * (r + 2 * y * y) - y0
    d_r = k1 + r * (2.0 * k2 + 3.0 * k3 * r)
    d_x, d_y = 2.0 * x * d_r, 2.0 * y * d_r
    return (fx, fy, d + d_x * x + 2.0 * p1 * y + 6.0 * p2 * x, d_y * x + 2.0 * p1 * x + 2.0 * p2 * y,
            d_x * y + 2.0 * p2 * y + 2.0 * p1 * x, d + d_y * y + 2.0 * p2 * x + 6.0 * p1 * y)

  x, y = x0, y0
  for _ in range(10):
    fx, fy, fx_x, fx_y, fy_x, fy_y = residual(x, y)
    den = fy_x * fx_y - fx_x * fy_y
    x = x + (fx * fy_y - fy * fx_y) / den
    y = y + (fy * fx_x - fx * fy_x) / den
  fx, fy = residual(x, y)[:2]
  u = torch.stack([x, y, torch.ones_like(x)], -1)
  local = u / u.norm(dim=-1, keepdim=True)
  d = local @ t(cam.orientation)
  d = d / d.norm(dim=-1, keepdim=True)
  d = d @ geometry.rotvec_to_matrix(omega).T
  return d, torch.maximum(fx.abs(), fy.abs())


def host_adjoint(cam, q, omega, pixels, directions, g):
  """nfb_intrinsics_grad's per-ray adjoint restated in numpy fp64, summed over the rays (the file comment of
  csrc/intrinsics_kernels.cuh): pose undone, both normalisations, the undistortion at its fixed point by the
  implicit function theorem, then (x0, y0) to s and dc.  `directions` are the posed world directions."""
  q = np.asarray(q, np.float64)
  f0 = float(cam.focal_length)
  f = f0 * np.exp(q[0])
  fy = f * float(cam.pixel_aspect_ratio)
  cx, cy = float(cam.principal_point[0]) + f0 * q[1], float(cam.principal_point[1]) + f0 * q[2]
  k1, k2, k3 = (float(cam.radial_distortion[j]) + q[3 + j] for j in range(3))
  p1, p2 = (float(cam.tangential_distortion[j]) + q[6 + j] for j in range(2))
  sk = float(cam.skew)
  y0 = (pixels[:, 1] - cy) / fy
  x0 = (pixels[:, 0] - cx - y0 * sk) / f
  x, y = x0.copy(), y0.copy()
  jac = None
  for _ in range(11):   # ten steps, then the Jacobian at the result
    r = x * x + y * y
    d = 1 + r * (k1 + r * (k2 + k3 * r))
    fx = d * x + 2 * p1 * x * y + p2 * (r + 2 * x * x) - x0
    fyv = d * y + 2 * p2 * x * y + p1 * (r + 2 * y * y) - y0
    d_r = k1 + r * (2 * k2 + 3 * k3 * r)
    d_x, d_y = 2 * x * d_r, 2 * y * d_r
    jac = (d + d_x * x + 2 * p1 * y + 6 * p2 * x, d_y * x + 2 * p1 * x + 2 * p2 * y,
           d_x * y + 2 * p2 * y + 2 * p1 * x, d + d_y * y + 2 * p2 * x + 6 * p1 * y)
    if _ == 10:
      break
    den = jac[2] * jac[1] - jac[0] * jac[3]
    x, y = x + (fx * jac[3] - fyv * jac[1]) / den, y + (fyv * jac[0] - fx * jac[2]) / den
  R = geometry.rotvec_to_matrix(torch.as_tensor(omega, dtype=torch.float64)).numpy()
  gw, dw = g @ R, directions @ R                     # exp(omega)^T per row
  gp = gw - dw * (dw * gw).sum(1, keepdims=True)
  gl = gp @ cam.orientation.astype(np.float64).T     # R0 g'
  n = np.sqrt(x * x + y * y + 1)
  lg = (x * gl[:, 0] + y * gl[:, 1] + gl[:, 2]) / n
  gux, guy = (gl[:, 0] - x / n * lg) / n, (gl[:, 1] - y / n * lg) / n
  J0, J1, J2, J3 = jac
  det = J0 * J3 - J1 * J2
  gx0, gy0 = (J3 * gux - J2 * guy) / det, (J0 * guy - J1 * gux) / det
  r2, w = x * x + y * y, -(x * gx0 + y * gy0)
  gy0t = gy0 - gx0 * sk / f
  out = np.stack([-(x0 * gx0 + y0 * gy0t), -f0 * gx0 / f, -f0 * gy0t / fy, r2 * w, r2 * r2 * w, r2**3 * w,
                  -(2 * x * y * gx0 + (r2 + 2 * y * y) * gy0), -((r2 + 2 * x * x) * gx0 + 2 * x * y * gy0)], 1)
  return out.sum(0)


Q = np.array([0.03, 0.01, -0.015, 0.02, -0.01, 0.005, 0.0004, -0.0003])
OMEGA = np.array([0.02, -0.015, 0.01])


@pytest.mark.parametrize('name', CASES)
@pytest.mark.parametrize('at_zero', [False, True], ids=['delta', 'zero'])
def test_adjoint_matches_fp64_autograd(name, at_zero):
  """At converged pixels the implicit-function adjoint equals autograd through the unrolled Newton steps."""
  cam, pixels = load_fixture(name)
  pixels = pixels.astype(np.float64)
  q = torch.tensor(np.zeros(8) if at_zero else Q, dtype=torch.float64, requires_grad=True)
  omega = torch.tensor(np.zeros(3) if at_zero else OMEGA, dtype=torch.float64)
  d, res = refined_rays(cam, q, omega, pixels)
  converged = (res < 1e-13).numpy()
  assert converged.mean() > 0.9, converged.mean()
  g = np.random.default_rng(1).normal(size=(pixels.shape[0], 3)) * converged[:, None]
  (d * torch.as_tensor(g)).sum().backward()
  want = q.grad.numpy()
  got = host_adjoint(cam, q.detach().numpy(), omega.numpy(), pixels[converged], d.detach().numpy()[converged],
                     g[converged])
  # the adjoint takes the world normalisation at |R0^T l| = 1; the fixtures' float32 orientations are orthonormal
  # to about 1e-7, and that is the whole difference
  scale = np.abs(want).max()
  assert np.abs(got - want).max() <= 1e-6 * scale, (got, want)


def test_refined_camera():
  cam, _ = load_fixture('camera_distorted')
  same = geometry.refined_camera(cam, np.zeros(8))
  for k, v in cam.get_parameters().items():
    assert np.array_equal(getattr(same, k), v), k
  r = geometry.refined_camera(cam, Q)
  f0 = float(cam.focal_length)
  assert np.isclose(float(r.focal_length), f0 * np.exp(Q[0]), rtol=1e-7)
  assert np.allclose(r.principal_point, cam.principal_point + f0 * Q[1:3], rtol=1e-7)
  assert np.allclose(r.radial_distortion, cam.radial_distortion + Q[3:6], atol=1e-8)
  assert np.allclose(r.tangential_distortion, cam.tangential_distortion + Q[6:8], atol=1e-9)
  # the delta does not depend on the image scale
  a, b = geometry.refined_camera(cam.scale(0.5), Q), geometry.refined_camera(cam, Q).scale(0.5)
  assert np.isclose(float(a.focal_length), float(b.focal_length), rtol=1e-6)
  assert np.allclose(a.principal_point, b.principal_point, rtol=1e-6)


# ---------------------------------------------------------------------------
# groups, state and checkpoints
# ---------------------------------------------------------------------------
def _capture_cameras():
  ds = train_lib.driver_utils.make_datasource(configs.ExperimentConfig(), configs.ModelConfig(), CAPTURE)
  return ds, {i: ds.load_camera(i) for i in ds.train_ids}


def test_groups():
  _, cams = _capture_cameras()
  group, members = training.intrinsics_groups(list(cams.values()))
  # every camera of the small capture has its own principal point and aspect ratio
  assert group.tolist() == list(range(len(cams))) and members == [[k] for k in range(len(cams))]
  cam, _ = load_fixture('camera_distorted')
  other = cam.copy()
  other.position = other.position + 1
  moved_pp = cam.copy()
  moved_pp.principal_point = moved_pp.principal_point + 1
  group, members = training.intrinsics_groups([cam, other, moved_pp, cam, cam.scale(0.5)])
  assert group.tolist() == [0, 0, 1, 0, 2] and members == [[0, 1, 3], [2], [4]]


def _intrinsics(parts=('focal', 'radial')):
  cam, _ = load_fixture('camera_distorted')
  other = cam.copy()
  other.focal_length = np.array(80.0, np.float32)
  return training.CameraIntrinsics(['a', 'b', 'c'], [cam, other, cam], parts, 'cpu')


def test_state_round_trip(tmp_path):
  ci = _intrinsics()
  assert ci.group.tolist() == [0, 1, 0] and ci.group_items == [['a', 'c'], ['b']]
  assert ci.part_bits == 1 | 4
  ci.delta.copy_(torch.arange(16, dtype=torch.float32).reshape(2, 8) * 1e-3)
  ci.m.fill_(0.5)
  ci.v.fill_(0.25)
  ci.step = 7
  assert set(ci.item_delta()) == {'a', 'b', 'c'} and np.array_equal(ci.item_delta()['c'], ci.item_delta()['a'])
  state = training.model_utils.TrainState(training.model_utils.Optimizer({'model': {'w': np.zeros(2, np.float32)}}))
  state.camera_intrinsics = ci
  checkpoints.save_checkpoint(str(tmp_path), state, 3)
  saved = checkpoints.checkpoint_camera_poses(str(tmp_path), key='camera_intrinsics')
  assert checkpoints.checkpoint_camera_poses(str(tmp_path)) is None
  back = _intrinsics()
  back.load(saved)
  for a, b in ((ci.delta, back.delta), (ci.m, back.m), (ci.v, back.v)):
    assert torch.equal(a, b)
  assert back.step == 7
  other = training.CameraIntrinsics(['a', 'b', 'c'], [load_fixture('camera_distorted')[0]] * 3, ('focal',), 'cpu')
  with pytest.raises(ValueError, match='item groups'):
    other.load(saved)
  stats = ci.stats()
  assert np.isclose(float(stats['focal_change_pct']), 100 * (0.0 + 0.008) / 2)


def test_driver_refusals():
  tc = configs.TrainConfig(batch_size=8)
  assert tc.refine_camera_intrinsics == ()
  train_lib.check_camera_intrinsics(tc, None)
  with pytest.raises(ValueError, match='unknown camera intrinsics part'):
    train_lib.check_camera_intrinsics(configs.TrainConfig(batch_size=8, refine_camera_intrinsics=('focal', 'zoom')), None)
  ci = _intrinsics()
  saved = ci.state_dict()
  with pytest.raises(ValueError, match='refine_camera_intrinsics is empty'):
    train_lib.check_camera_intrinsics(tc, saved)
  on = configs.TrainConfig(batch_size=8, refine_camera_intrinsics=('focal',))
  cam, _ = load_fixture('camera_distorted')
  other = cam.copy()
  other.focal_length = np.array(80.0, np.float32)
  train_lib.check_camera_intrinsics(on, saved, {'a': cam, 'b': other, 'c': cam})
  with pytest.raises(ValueError, match='item groups'):
    train_lib.check_camera_intrinsics(on, saved, {'a': cam, 'b': cam, 'c': cam})
  with pytest.raises(ValueError, match='unknown camera intrinsics part'):
    training.CameraIntrinsics(['a'], [cam], ('skew',), 'cpu')


def test_gin_fields(tmp_path):
  configs.clear_config()
  try:
    configs.parse_config_files_and_bindings([], [
        "TrainConfig.refine_camera_intrinsics = ('focal', 'principal_point')",
        "TrainConfig.camera_intrinsics_lr_schedule = ('constant', 0.002)", 'TrainConfig.batch_size = 8'])
    tc = configs.TrainConfig()
    assert tc.refine_camera_intrinsics == ('focal', 'principal_point')
    assert training.ScalarParams(learning_rate=1.0).camera_intrinsics_learning_rate == 0.0
  finally:
    configs.clear_config()


# ---------------------------------------------------------------------------
# registration
# ---------------------------------------------------------------------------
def _model(**kw):
  spec = O.OracleSpec(num_coarse_samples=8, num_fine_samples=8, near=0.02, far=0.83, nerf_trunk_depth=2,
                      nerf_trunk_width=16, **kw)
  return model_from_spec(spec_to_dict(spec), device='cpu')


def test_registration_refusals():
  """The intrinsics parts are registration's `intrinsics`, accepted on any model, alone or with `optimize`
  groups; as `optimize` entries they stay unknown, with a pointer to `intrinsics`."""
  plain = _model()
  assert geometry.check_registration(plain, ['pose'], 10, 16, intrinsics=['focal']) == ('pose',)
  assert geometry.check_registration(plain, [], 1, 1, intrinsics=list(geometry.INTRINSICS_PARTS)) == ()
  with pytest.raises(ValueError, match=r"unknown optimize entry 'focal'.*intrinsics="):
    geometry.check_registration(plain, ['pose', 'focal'], 10, 16)
  for bad in ('zoom', 'skew', 'pose'):
    with pytest.raises(ValueError, match='unknown intrinsics part'):
      geometry.check_registration(plain, ['pose'], 10, 16, intrinsics=[bad])
  with pytest.raises(ValueError, match='empty'):
    geometry.check_registration(plain, [], 10, 16, intrinsics=[])
  with pytest.raises(ValueError, match='appearance'):
    geometry.check_registration(plain, ['appearance'], 10, 16, intrinsics=['focal'])


def test_driver_refusals_come_before_any_gpu_work(tmp_path):
  """register_camera refuses an unknown --intrinsics part before any GPU work; the known ones get past the
  refusals (to the missing checkpoint)."""
  from tests.test_register_camera import _Source, _register
  from nerfies_b200 import register_camera
  _Source(tmp_path / 'cap')
  for kw, msg in ((dict(item='a', optimize=['pose'], intrinsics=['zoom']), 'unknown intrinsics part'),
                  (dict(item='a', optimize=['pose'], intrinsics=['focal', 'skew']), 'unknown intrinsics part'),
                  (dict(item='a', optimize=['pose', 'radial']), 'unknown optimize')):
    with pytest.raises(ValueError, match=msg):
      _register(tmp_path, **kw)
  for kw in (dict(item='a', optimize=['pose'], intrinsics=['focal', 'principal_point', 'radial', 'tangential']),
             dict(item='b', optimize=[], intrinsics=['focal'])):
    with pytest.raises(FileNotFoundError, match='no checkpoints'):
      _register(tmp_path, **kw)
  args = register_camera.make_parser().parse_args(['--base_folder', str(tmp_path), '--item', 'a'])
  assert args.intrinsics == ''
  args = register_camera.make_parser().parse_args(['--base_folder', str(tmp_path), '--intrinsics', 'focal,radial',
                                                   '--lr_focal', '0.01'])
  assert args.intrinsics == 'focal,radial' and args.lr_focal == 0.01
  assert args.lr_principal_point == geometry.DEFAULT_LRS['principal_point']
