"""nerfies_b200: Hopper-native (sm_90a) render hot path of google/nerfies.

Public surface (mirrors the reference's, SURVEY.md §8b):
  nerfies_b200.configs     ModelConfig / TrainConfig / EvalConfig + gin subset
  nerfies_b200.models      construct_nerf, NerfModel.apply, WarpField.apply
  nerfies_b200.evaluation  render_image
  nerfies_b200.model_utils TrainState
  nerfies_b200.training    train_step (value_and_grad + gradient all-reduce + Adam)
  nerfies_b200.datasets    NerfiesDataSource: a capture on the GPU, train.py / eval.py batches
  nerfies_b200.schedules   the annealing schedules of train.py
  nerfies_b200.train       python -m nerfies_b200.train: the training driver (train.py:100-326)
  nerfies_b200.eval        python -m nerfies_b200.eval: the evaluation driver (eval.py:225-419)
The arithmetic lives in libnerfies_b200.so (include/nerfies_b200.h); there is no
CPU or PyTorch fallback.
"""
from nerfies_b200 import configs  # noqa: F401
from nerfies_b200 import models  # noqa: F401
from nerfies_b200 import model_utils  # noqa: F401
from nerfies_b200 import evaluation  # noqa: F401
from nerfies_b200 import camera  # noqa: F401
from nerfies_b200 import checkpoints  # noqa: F401
from nerfies_b200 import training  # noqa: F401
from nerfies_b200 import datasets  # noqa: F401
from nerfies_b200 import schedules  # noqa: F401
from nerfies_b200.models import construct_nerf, NerfModel  # noqa: F401

__version__ = '0.1'
