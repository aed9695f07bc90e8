"""What `nerfies_b200.train` and `nerfies_b200.eval` share: the flags of the reference's drivers
(train.py:43-50, eval.py:46-52), the experiment directory layout (train.py:117-122,
eval.py:243-262), the data source of a run (train.py:159-174) and the scalar log.

Scalars go to `<exp_dir>/summaries/{train,eval}.jsonl`, one JSON object per line
({'step': s, '<tag>': value, ...}); the reference writes TensorBoard event files, and TensorBoard
is not a dependency of this package.
"""
import argparse
import json
import os
import pathlib

import torch
import torch.distributed as dist

from nerfies_b200 import configs
from nerfies_b200 import datasets


def make_parser(prog, default_precision):
  """--base_folder --data_dir --gin_configs --gin_bindings with the reference's names and meaning,
  plus this package's --precision (render kernels), --train_precision and --max_steps."""
  p = argparse.ArgumentParser(prog=prog)
  p.add_argument('--base_folder', required=True, help='where to store ckpts and logs')
  p.add_argument('--data_dir', default=None, help='input data directory.')
  p.add_argument('--gin_configs', action='append', default=[], help='Gin config files.')
  p.add_argument('--gin_bindings', action='append', default=[], help='Gin parameter bindings.')
  p.add_argument('--precision', default=default_precision, choices=('fp32', 'bf16', 'fp16x3'),
                 help='render kernels (models.construct_nerf)')
  p.add_argument('--train_precision', default='fp32', choices=('fp32', 'tf32x3'),
                 help='training GEMMs (models.construct_nerf)')
  p.add_argument('--max_steps', type=int, default=None, help='overrides TrainConfig.max_steps')
  return p


def parse_configs(gin_configs, gin_bindings):
  """Parses the gin files and bindings (train.py:107-110) and returns their text, which is what
  the run writes to `<exp_dir>/config.gin`."""
  configs.clear_config()
  configs.parse_config_files_and_bindings(gin_configs, gin_bindings, skip_unknown=True)
  parts = []
  for path in gin_configs:
    with open(path) as f:
      parts.append(f'# {path}\n{f.read().rstrip()}\n')
  if gin_bindings:
    parts.append('# bindings\n' + '\n'.join(gin_bindings) + '\n')
  return '\n'.join(parts)


def experiment_dirs(base_folder, subname=None):
  """{'exp', 'summaries', 'checkpoints', 'renders'} paths of a run (train.py:117-122)."""
  exp_dir = pathlib.Path(base_folder)
  if subname:
    exp_dir = exp_dir / subname
  return {'exp': exp_dir, 'summaries': exp_dir / 'summaries', 'checkpoints': exp_dir / 'checkpoints',
          'renders': exp_dir / 'renders'}


def make_datasource(exp_config, model_config, data_dir):
  """train.py:159-174 / eval.py:277-292."""
  spec = exp_config.datasource_spec
  if spec is None:
    if data_dir is None:
      raise ValueError('--data_dir is required when ExperimentConfig.datasource_spec is not set')
    spec = {'type': exp_config.datasource_type, 'data_dir': data_dir}
  return datasets.from_config(
      spec, image_scale=exp_config.image_scale,
      use_appearance_id=model_config.use_appearance_metadata,
      use_camera_id=model_config.use_camera_metadata, use_warp_id=model_config.use_warp,
      use_time=model_config.warp_metadata_encoder_type == 'time',
      random_seed=exp_config.random_seed, **exp_config.datasource_kwargs)


class ScalarWriter:
  """Appends {'step': step, **scalars} as one JSON line per call; every line is flushed."""

  def __init__(self, path):
    self.path = pathlib.Path(path)
    self.path.parent.mkdir(parents=True, exist_ok=True)
    self._file = open(self.path, 'a')

  def write(self, step, scalars):
    self._file.write(json.dumps({'step': int(step), **{k: float(v) for k, v in scalars.items()}}) + '\n')
    self._file.flush()

  def close(self):
    self._file.close()


def read_scalars(path):
  """The records a ScalarWriter wrote."""
  with open(path) as f:
    return [json.loads(line) for line in f if line.strip()]


def init_distributed():
  """One process per GPU.  Under torchrun (RANK / WORLD_SIZE / LOCAL_RANK set) joins the NCCL group
  unless the caller already did; returns (rank, world_size, whether this call created the group)."""
  if dist.is_available() and dist.is_initialized():
    return dist.get_rank(), dist.get_world_size(), False
  world = int(os.environ.get('WORLD_SIZE', '1'))
  if world == 1:
    return 0, 1, False
  rank, local = int(os.environ['RANK']), int(os.environ.get('LOCAL_RANK', os.environ['RANK']))
  torch.cuda.set_device(local)
  dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', local))
  return rank, world, True
