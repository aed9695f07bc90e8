"""The training driver: the loop of the reference's train.py:100-326 over this package's CUDA path.

  python -m nerfies_b200.train --base_folder EXP --data_dir CAPTURE --gin_configs configs/x.gin
  torchrun --nproc_per_node=N -m nerfies_b200.train ...        # one process per GPU

Gin files in; `<exp_dir>/config.gin`, `<exp_dir>/checkpoints/checkpoint_<step>` (flax layout, with
Adam's moments) and `<exp_dir>/summaries/train.jsonl` out.  The scalars the reference sends to
TensorBoard (train.py:56-81) are appended to that file as one JSON object per logging step, with
the reference's tags (`loss/total/coarse`, `params/learning_rate`, ...); TensorBoard is not
installed with this package and is out of scope, as are the embedding histograms
(train.py:84-97).  Reading a scalar is the only host synchronisation in the loop and happens on a
logging or printing step only.

Where this differs from the reference, on purpose:
  * Resuming.  The reference zips range(init_step, ...) with a FRESH iterator (train.py:274), so a
    resumed run replays the shuffled order from its head.  Here the iterators start at the batch
    step `init_step` would have drawn in an uninterrupted run (`first_batch`), and the per-step
    random key is a function of (random_seed, rank, step), so a run stopped at a checkpoint and
    started again ends with the parameters and Adam moments of an uninterrupted run.
  * The random key.  `training.train_step` seeds the stratified draws and the background loss's
    ids and noise from the key it is given and returns it unchanged; the reference splits its key
    every step (training.py:163).  The driver passes a new key per step instead.
"""
import sys
import time

import torch

from nerfies_b200 import checkpoints
from nerfies_b200 import configs
from nerfies_b200 import datasets
from nerfies_b200 import driver_utils
from nerfies_b200 import models
from nerfies_b200 import schedules
from nerfies_b200 import training


def step_key(random_seed, rank, step):
  """The key of one rank's training step: distinct per step and per rank (train.py:270-271),
  and a function of the step alone so that a resumed run draws what it would have drawn."""
  return ((int(random_seed) * 1000003 + int(rank)) * 1000003 + int(step)) % (2**62)


def flatten_stats(stats):
  """train_step's stats under the tags of train.py:71-78: '<key>/<branch>' and 'loss/background'."""
  out = {}
  for branch in ('coarse', 'fine'):
    for key, value in stats.get(branch, {}).items():
      out[f'{key}/{branch}'] = value
  if 'background_loss' in stats:
    out['loss/background'] = stats['background_loss']
  return out


def train(exp_config, model_config, train_config, base_folder, data_dir=None, precision='fp32',
          train_precision='fp32', config_str='', datasource=None, log=print):
  """Trains to `train_config.max_steps` (resuming from the newest checkpoint of the experiment)
  and returns the final TrainState.  `datasource` replaces the one built from the configs."""
  rank, world, own_group = driver_utils.init_distributed()
  try:
    return _train(exp_config, model_config, train_config, base_folder, data_dir, precision,
                  train_precision, config_str, datasource, log, rank, world)
  finally:
    if own_group:
      torch.distributed.destroy_process_group()


def _train(exp_config, model_config, train_config, base_folder, data_dir, precision, train_precision,
           config_str, datasource, log, rank, world):
  dirs = driver_utils.experiment_dirs(base_folder, exp_config.subname)
  writer = None
  if rank == 0:                                                      # train.py:125-141
    for key in ('exp', 'summaries', 'checkpoints'):
      dirs[key].mkdir(parents=True, exist_ok=True)
    (dirs['exp'] / 'config.gin').write_text(config_str)
    writer = driver_utils.ScalarWriter(dirs['summaries'] / 'train.jsonl')
  if train_config.batch_size % world != 0:
    raise ValueError('Batch size must be divisible by the number of devices.')

  if datasource is None:
    datasource = driver_utils.make_datasource(exp_config, model_config, data_dir)
  learning_rate_sched = schedules.from_config(train_config.lr_schedule)          # train.py:199-203
  warp_alpha_sched = schedules.from_config(train_config.warp_alpha_schedule)
  time_alpha_sched = schedules.from_config(train_config.time_alpha_schedule)
  elastic_loss_weight_sched = schedules.from_config(train_config.elastic_loss_weight_schedule)

  model, params = models.construct_nerf(                                         # train.py:205-217
      step_key(exp_config.random_seed, 0, 0), model_config, batch_size=train_config.batch_size // world,
      appearance_ids=datasource.appearance_ids, camera_ids=datasource.camera_ids,
      warp_ids=datasource.warp_ids, near=datasource.near, far=datasource.far,
      use_warp_jacobian=train_config.use_elastic_loss, use_weights=train_config.use_elastic_loss,
      precision=precision, train_precision=train_precision)
  state = training.create_train_state(model, params, warp_alpha=warp_alpha_sched(0),
                                      time_alpha=time_alpha_sched(0))
  restored = checkpoints.restore_checkpoint(str(dirs['checkpoints']), state, device=model.device)
  if restored is not state:                                                      # train.py:232-233
    state.optimizer.load(restored)
    model.invalidate_params()
  init_step = state.optimizer.step + 1

  first_batch = init_step - 1
  train_iter = datasource.create_iterator(                                       # train.py:175-183
      datasource.train_ids, flatten=True, shuffle=True, batch_size=train_config.batch_size,
      shuffle_buffer_size=train_config.shuffle_buffer_size, first_batch=first_batch)
  points_iter = None
  if train_config.use_background_loss:                                           # train.py:185-197
    points = datasource.load_points(shuffle=True)
    points_batch_size = min(len(points), world * train_config.background_points_batch_size)
    points_batch_size -= points_batch_size % world
    points_iter = datasets.iterator_from_dataset(points, batch_size=points_batch_size,
                                                 first_batch=first_batch)

  scalar_params = training.ScalarParams(                                         # train.py:225-231
      learning_rate=learning_rate_sched(0), elastic_loss_weight=elastic_loss_weight_sched(0),
      warp_reg_loss_weight=train_config.warp_reg_loss_weight,
      warp_reg_loss_alpha=train_config.warp_reg_loss_alpha,
      warp_reg_loss_scale=train_config.warp_reg_loss_scale,
      background_loss_weight=train_config.background_loss_weight)

  def save(step):
    if rank == 0:
      checkpoints.save_checkpoint(str(dirs['checkpoints']), state, step, keep=2)   # training.py:46-53

  log(f'Starting training at step {init_step} of {train_config.max_steps} on {world} GPU(s)')
  mark = torch.cuda.Event(enable_timing=True)
  mark.record()
  mark_step, mark_wall = init_step - 1, time.time()
  step = init_step - 1
  for step, batch in zip(range(init_step, train_config.max_steps + 1), train_iter):   # train.py:274-322
    if points_iter is not None:
      batch['background_points'] = next(points_iter)
    scalar_params.learning_rate = learning_rate_sched(step)
    scalar_params.elastic_loss_weight = elastic_loss_weight_sched(step)
    state.warp_alpha = warp_alpha_sched(step)
    state.time_alpha = time_alpha_sched(step)
    state, stats, _ = training.train_step(
        model, step_key(exp_config.random_seed, rank, step), state, batch, scalar_params,
        use_elastic_loss=train_config.use_elastic_loss,
        elastic_reduce_method=train_config.elastic_reduce_method,
        elastic_loss_type=train_config.elastic_loss_type,
        use_background_loss=train_config.use_background_loss,
        use_warp_reg_loss=train_config.use_warp_reg_loss)

    if step % train_config.print_every == 0 and rank == 0:
      log(f'step={step}, warp_alpha={state.warp_alpha:.04f}, time_alpha={state.time_alpha:.04f}, '
          f'{(step - mark_step) / max(time.time() - mark_wall, 1e-9):.2f} steps/s (host clock)')
      for branch in ('coarse', 'fine'):
        if branch in stats:
          log(f'\t{branch} metrics: ' + ', '.join(f'{k}={float(v):.04f}' for k, v in stats[branch].items()))
    if step % train_config.save_every == 0:
      save(step)
    if step % train_config.log_every == 0 and rank == 0:
      now = torch.cuda.Event(enable_timing=True)
      now.record()
      scalars = {'params/learning_rate': scalar_params.learning_rate,            # train.py:64-68
                 'params/warp_alpha': state.warp_alpha, 'params/time_alpha': state.time_alpha,
                 'params/elastic_loss/weight': scalar_params.elastic_loss_weight}
      scalars.update({k: float(v) for k, v in flatten_stats(stats).items()})     # the synchronisation
      now.synchronize()
      scalars['time/steps_per_sec'] = (step - mark_step) * 1000.0 / max(mark.elapsed_time(now), 1e-6)
      writer.write(step, scalars)
      mark, mark_step, mark_wall = now, step, time.time()

  if step >= init_step and train_config.max_steps % train_config.save_every != 0:   # train.py:321-322
    save(step)
  torch.cuda.synchronize(model.device)
  if writer is not None:
    writer.close()
  return state


def main(argv=None):
  args = driver_utils.make_parser('nerfies_b200.train', 'fp32').parse_args(argv)
  config_str = driver_utils.parse_configs(args.gin_configs, args.gin_bindings)
  exp_config = configs.ExperimentConfig()                                        # train.py:113-115
  model_config = configs.ModelConfig()
  train_config = configs.TrainConfig()
  if args.max_steps is not None:
    train_config.max_steps = args.max_steps
  train(exp_config, model_config, train_config, args.base_folder, args.data_dir,
        precision=args.precision, train_precision=args.train_precision, config_str=config_str)
  return 0


if __name__ == '__main__':
  sys.exit(main())
