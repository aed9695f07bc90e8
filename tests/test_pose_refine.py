"""Training-camera pose refinement without a GPU: the per-image pose gradient's formula (what nfb_pose_grad
computes) against torch.autograd of geometry.pose_rays in float64, the poses' checkpoint round trip, the
driver's refusals and the TrainConfig fields."""
import numpy as np
import pytest
import torch

from nerfies_b200 import checkpoints
from nerfies_b200 import configs
from nerfies_b200 import geometry
from nerfies_b200 import model_utils
from nerfies_b200 import train
from nerfies_b200 import training


def _left_jacobian_t(w, s):
  """J_l(w)^T s with the series of pose_kernels.cuh below |w|^2 = 1e-4."""
  t2 = float((w * w).sum())
  if t2 < 1e-4:
    b, c = 0.5 - t2 / 24 + t2 * t2 / 720, 1 / 6 - t2 / 120 + t2 * t2 / 5040
  else:
    t = np.sqrt(t2)
    b, c = (1 - np.cos(t)) / t2, (t - np.sin(t)) / (t2 * t)
  x = torch.linalg.cross(w, s)
  return s - b * x + c * torch.linalg.cross(w, x)


@pytest.mark.parametrize('omega_norm', [0.0, 3e-3, 0.5])
def test_pose_gradient_formula_matches_autograd(omega_norm):
  gen = torch.Generator().manual_seed(int(omega_norm * 1000) + 1)
  dt = torch.float64
  n = 50
  local = torch.nn.functional.normalize(torch.randn(n, 3, generator=gen, dtype=dt), dim=1)
  q, _ = torch.linalg.qr(torch.randn(3, 3, generator=gen, dtype=dt))
  p0 = torch.randn(3, generator=gen, dtype=dt)
  axis = torch.nn.functional.normalize(torch.randn(3, generator=gen, dtype=dt), dim=0)
  omega = (axis * omega_norm).requires_grad_(True)
  v = (0.01 * torch.randn(3, generator=gen, dtype=dt)).requires_grad_(True)
  g_o = torch.randn(n, 3, generator=gen, dtype=dt)
  g_d = torch.randn(n, 3, generator=gen, dtype=dt)
  o, d = geometry.pose_rays(local, q, p0, omega, v)
  ((o * g_o).sum() + (d * g_d).sum()).backward()
  want = torch.cat([omega.grad, v.grad])
  got = torch.cat([_left_jacobian_t(omega.detach(), torch.linalg.cross(d.detach(), g_d).sum(0)), g_o.sum(0)])
  assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max()), (got, want)


def _state_with_poses(items):
  state = model_utils.TrainState(model_utils.Optimizer({'model': {'w': torch.arange(4.0)}}))
  poses = training.CameraPoses(items, 'cpu')
  poses.pose.copy_(torch.randn(len(items), 6))
  poses.m.copy_(torch.randn(len(items), 6))
  poses.v.copy_(torch.rand(len(items), 6))
  poses.step = 7
  state.camera_poses = poses
  return state, poses


def test_checkpoint_round_trip_with_poses(tmp_path):
  items = ['left_000', 'right_001', 'left_003']
  state, poses = _state_with_poses(items)
  checkpoints.save_checkpoint(str(tmp_path), state, 7)
  restored = checkpoints.restore_checkpoint(str(tmp_path), state)
  assert restored.camera_poses is not None
  again = training.CameraPoses(list(reversed(items)), 'cpu')
  again.load(restored.camera_poses)
  for k, item in enumerate(again.item_ids):
    i = items.index(item)
    for a, b in ((again.pose, poses.pose), (again.m, poses.m), (again.v, poses.v)):
      assert torch.equal(a[k], b[i])
  assert again.step == 7
  assert checkpoints.checkpoint_camera_poses(str(tmp_path))['items'].keys() == set(items)


def test_checkpoint_without_poses_restores_as_before(tmp_path):
  state = model_utils.TrainState(model_utils.Optimizer({'model': {'w': torch.arange(4.0)}}))
  checkpoints.save_checkpoint(str(tmp_path), state, 3)
  assert 'camera_poses' not in checkpoints.msgpack_restore((tmp_path / 'checkpoint_3').read_bytes())
  assert checkpoints.restore_checkpoint(str(tmp_path), state).camera_poses is None
  assert checkpoints.checkpoint_camera_poses(str(tmp_path)) is None
  assert checkpoints.checkpoint_camera_poses(str(tmp_path / 'none')) is None


def test_refusals(tmp_path):
  items = ['a', 'b']
  state, _ = _state_with_poses(items)
  checkpoints.save_checkpoint(str(tmp_path), state, 5)
  saved = checkpoints.checkpoint_camera_poses(str(tmp_path))
  off = configs.TrainConfig(batch_size=4)
  on = configs.TrainConfig(batch_size=4, refine_camera_poses=True)
  with pytest.raises(ValueError, match='refine_camera_poses is off'):
    train.check_camera_poses(off, saved)
  with pytest.raises(ValueError, match='camera poses of items'):
    train.check_camera_poses(on, saved, ['a', 'c'])
  with pytest.raises(ValueError, match='camera poses of items'):
    training.CameraPoses(['a'], 'cpu').load(saved)
  train.check_camera_poses(on, saved, ['b', 'a'])
  train.check_camera_poses(off, None, ['a'])


def test_train_config_from_gin():
  configs.clear_config()
  try:
    configs.parse_config('\n'.join([
        'TrainConfig.batch_size = 8',
        'TrainConfig.refine_camera_poses = True',
        "TrainConfig.camera_pose_lr_schedule = ('constant', 0.002)",
    ]))
    tc = configs.TrainConfig()
    assert tc.refine_camera_poses is True
    assert tuple(tc.camera_pose_lr_schedule) == ('constant', 0.002)
  finally:
    configs.clear_config()
  tc = configs.TrainConfig(batch_size=8)
  assert tc.refine_camera_poses is False
  assert tc.camera_pose_lr_schedule['type'] == 'exponential'


def test_flatten_stats_reports_the_poses():
  stats = {'coarse': {'loss/rgb': 1.0}, 'camera_poses': {'rotation_deg': 0.5, 'translation': 0.01}}
  out = train.flatten_stats(stats)
  assert out['camera_poses/rotation_deg'] == 0.5 and out['camera_poses/translation'] == 0.01
