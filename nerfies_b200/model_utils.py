"""The caller-visible pieces of nerfies/model_utils.py that are not kernels."""
import dataclasses
from typing import Any


@dataclasses.dataclass
class Optimizer:
  """Stand-in for flax.optim.Optimizer: callers read `.target` only
  (evaluation.py:86 reads state.optimizer.target['model'])."""
  target: Any


@dataclasses.dataclass
class TrainState:
  """model_utils.TrainState (model_utils.py:25-33)."""
  optimizer: Optimizer
  warp_alpha: float = 0.0
  time_alpha: float = 0.0
  # training.CameraPoses while refining the training cameras; a restored checkpoint's saved poses
  # ({'step', 'items': {item_id: {'pose', 'grad_ema', 'grad_sq_ema'}}}); or None
  camera_poses: Any = None
  # training.CameraIntrinsics while refining the training cameras' intrinsics; a restored checkpoint's saved
  # deltas ({'step', 'groups': {group: {'items', 'delta', 'grad_ema', 'grad_sq_ema'}}}); or None
  camera_intrinsics: Any = None

  @property
  def warp_extra(self):
    return {'alpha': self.warp_alpha, 'time_alpha': self.time_alpha}
