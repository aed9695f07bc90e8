"""The evaluation driver: the loop of the reference's eval.py:225-419 over this package's CUDA path.

  python -m nerfies_b200.eval --base_folder EXP --data_dir CAPTURE --gin_configs configs/x.gin

Polls `<exp_dir>/checkpoints` for a step it has not rendered; for each of the val / train / test
sets renders the chosen items with `evaluation.render_frame`, scores them with
`evaluation.compute_metrics` and appends the means to `<exp_dir>/summaries/eval.jsonl` as
`metrics-eval/{mse,psnr,ssim}/{tag}` (eval.py:205-214).  With `EvalConfig.save_output`,
`rgb_<id>.png` (8 bit) and `depth_expected_<id>.png`, `depth_median_<id>.png` (16 bit, depth / 1000
as image_utils.save_depth) go to `<exp_dir>/renders/<step, 8 digits>/<tag>/` (eval.py:97-109, 166).
With `--save_viz`, each frame also writes the colour-mapped images of eval.py:87-109, 129-132
(`visualization.colorize_uint8`, magma): `depth_expected_viz_`, `depth_median_viz_` (the reference's
two files), and the images the reference sends to TensorBoard, `disparity_expected_viz_`,
`disparity_median_viz_`, `acc_viz_` and, for items with a target, `rgb_abs_error_viz_` and
`rgb_sq_error_viz_<id>.png`.
Frames are quantised on the device (`nfb_image_quantize`), copied to pinned host memory without
blocking, and PNG-encoded by a worker thread while the next frame renders; every worker is joined
before `evaluate` returns.

Not written: TensorBoard images and scalars (TensorBoard is not a dependency; the scalars are in
eval.jsonl).  The colour tables are OpenCV's (see `visualization`).  Test cameras are rendered and saved but not scored, as in the reference.  Frames
smaller than 161 pixels on a side have no MS-SSIM: `ssim` is left out for them, with one notice.
"""
import concurrent.futures
import functools
import os
import shutil
import sys
import time

import numpy as np
import torch

from nerfies_b200 import checkpoints
from nerfies_b200 import configs
from nerfies_b200 import driver_utils
from nerfies_b200 import evaluation
from nerfies_b200 import model_utils
from nerfies_b200 import models
from nerfies_b200 import visualization


def strided_subset(sequence, count):
  """The items eval.py:295-299 picks: every (len // count)-th item, at least every item, so
  possibly more than `count`; the whole sequence when `count` is 0 or None."""
  sequence = list(sequence)
  if not count:
    return sequence
  return sequence[::max(1, len(sequence) // count)]


def checkpoint_steps(checkpoint_dir, prefix='checkpoint_'):
  """Steps of the `checkpoint_<step>` files of a directory, ascending; [] when it does not exist."""
  try:
    names = os.listdir(str(checkpoint_dir))
  except FileNotFoundError:
    return []
  steps = [checkpoints._step_of(name, prefix) for name in names]
  return sorted(int(s) for s in steps if s is not None)


def next_checkpoint_step(checkpoint_dir, last_step):
  """The newest step if it is newer than `last_step`, else None (eval.py:358-370: the reference
  restores the latest checkpoint and skips it when `step <= last_step`)."""
  steps = checkpoint_steps(checkpoint_dir)
  return steps[-1] if steps and steps[-1] > last_step else None


def choose_test_metadata(datasource, step):
  """One metadata choice per checkpoint for the test cameras (eval.py:170-194: drawn from
  PRNGKey(step), the same for every frame).  Indices into the source's id lists, which is what
  this package's batches carry; numpy's generator, not jax's."""
  rs = np.random.RandomState(step)
  metadata = {}
  if datasource.use_appearance_id:
    metadata['appearance'] = int(rs.randint(len(datasource.appearance_ids)))
  if datasource.use_warp_id:
    metadata['warp'] = int(rs.randint(len(datasource.warp_ids)))
  if datasource.use_camera_id:
    metadata['camera'] = int(rs.randint(len(datasource.camera_ids)))
  if datasource.use_time:
    metadata['time'] = float(rs.uniform(0.0, 1.0))
  return metadata


def viz_images(render, rgb_target, near, far):
  """The colour-mapped images of eval.py:87-96, 129-132 as uint8 device images, by file stem."""
  viz = visualization.colorize_uint8
  images = {'depth_expected_viz': viz(render['depth'], near, far, invert=True),
            'depth_median_viz': viz(render['med_depth'], near, far, invert=True),
            'disparity_expected_viz': viz(render['depth'], source='reciprocal'),
            'disparity_median_viz': viz(render['med_depth'], source='reciprocal'),
            'acc_viz': viz(render['acc'], 0.0, 1.0)}
  if rgb_target is not None:
    images['rgb_abs_error_viz'] = viz(rgb_target, 0, 1, source='abs_error', target=render['rgb'])
    images['rgb_sq_error_viz'] = viz(rgb_target, 0, 1, source='sq_error', target=render['rgb'])
  return images


def render_and_score(model, params, camera, warp_extra, metadata, rgb_target, viz_range=None):
  """One frame on the GPU: ({file stem: uint8 / uint16 device image}, {metric: 0-d device tensor}).
  The images are what eval.py:99-108 saves, plus `viz_images` when `viz_range` is the scene's
  (near, far); the metrics eval.py:118-125's, without `ssim` for frames MS-SSIM cannot take."""
  render = evaluation.render_frame(model, params, camera, warp_extra, metadata)
  images = {'rgb': evaluation.image_to_uint8(render['rgb']),
            'depth_expected': evaluation.depth_to_uint16(render['depth']),
            'depth_median': evaluation.depth_to_uint16(render['med_depth'])}
  if viz_range is not None:
    images.update(viz_images(render, rgb_target, *viz_range))
  metrics = {}
  if rgb_target is not None:
    if min(rgb_target.shape[:2]) >= evaluation.MIN_METRICS_SIZE:
      out = evaluation.compute_metrics(render['rgb'], rgb_target)
      metrics = {k: out[k] for k in ('mse', 'psnr', 'ssim')}
    else:   # nfb_image_metrics takes no frame this small; eval.py:120-121 as written, on the device
      mse = ((render['rgb'] - rgb_target)**2).mean()
      metrics = {'mse': mse, 'psnr': evaluation.compute_psnr(mse)}
  return images, metrics


def _host_copy(image):
  """Starts the copy of a device image to pinned host memory; returns a callable that waits for it
  and gives the numpy array.  Host arrays (a stand-in renderer's) pass through."""
  if not torch.is_tensor(image):
    return lambda: np.asarray(image)
  if not image.is_cuda:
    return image.numpy
  host = torch.empty(image.shape, dtype=image.dtype, pin_memory=True)
  host.copy_(image, non_blocking=True)
  done = torch.cuda.Event()
  done.record(torch.cuda.current_stream(image.device))

  def wait():
    done.synchronize()
    return host.numpy()
  return wait


def write_png(path, array):
  """8-bit RGB / 16-bit grey PNG with cv2, which `datasets.decode_image` reads back."""
  import cv2
  array = np.ascontiguousarray(array)
  if array.ndim == 3:
    array = array[:, :, ::-1]                                                    # RGB -> BGR
  ok, buf = cv2.imencode('.png', array)
  if not ok:
    raise IOError(f'could not encode {path}')
  with open(path, 'wb') as f:
    f.write(buf.tobytes())


def process_items(tag, items, step, model, params, warp_extra, save_dir, writer, pool, frame_fn, log):
  """eval.py:155-214 for one tag.  `items`: (item_id, camera, metadata, rgb target or None)."""
  save_dir = save_dir / f'{step:08d}' / tag if save_dir else None
  if save_dir:
    save_dir.mkdir(parents=True, exist_ok=True)
  meters, pending, noticed = {}, [], False
  for i, (item_id, camera, metadata, rgb_target) in enumerate(items):
    log(f'[{tag}:{i + 1}/{len(items)}] Processing {item_id}')
    item_id = str(item_id).replace('/', '_')
    images, metrics = frame_fn(model, params, camera, warp_extra, metadata, rgb_target)
    if rgb_target is not None and 'ssim' not in metrics and not noticed:
      log(f'\t{tag}: frames below {evaluation.MIN_METRICS_SIZE} pixels on a side have no MS-SSIM; ssim is not logged')
      noticed = True
    for key, value in metrics.items():
      meters.setdefault(key, []).append(value)
    if save_dir:
      for stem, image in images.items():
        wait = _host_copy(image)
        pending.append(pool.submit(lambda w=wait, p=save_dir / f'{stem}_{item_id}.png': write_png(p, w())))
  for future in pending:
    future.result()
  if meters and writer is not None:                                              # eval.py:210-214
    writer.write(step, {f'metrics-eval/{k}/{tag}': sum(float(v) for v in vs) / len(vs)
                        for k, vs in meters.items()})


def delete_old_renders(render_dir, max_renders):
  """eval.py:217-222."""
  paths = sorted(p for p in render_dir.iterdir() if p.is_dir())
  for path in paths[:-max_renders] if max_renders else []:
    shutil.rmtree(path)


def evaluate(exp_config, model_config, train_config, eval_config, base_folder, data_dir=None,
             precision='fp16x3', poll_seconds=10.0, datasource=None, construct_fn=models.construct_nerf,
             frame_fn=render_and_score, log=print, save_viz=False):
  """Renders and scores checkpoints until `eval_once` is set or step `max_steps` has been rendered.
  Returns the list of steps handled.  `datasource`, `construct_fn` and `frame_fn` replace the data
  source, the model constructor and the renderer (tests run the loop without a GPU that way).
  `save_viz` passes `viz_range=(near, far)` to `frame_fn`, which then adds the colour-mapped images."""
  rank, world, own_group = driver_utils.init_distributed()
  pool = concurrent.futures.ThreadPoolExecutor(max_workers=2)
  writer = None
  try:
    dirs = driver_utils.experiment_dirs(base_folder, exp_config.subname)
    if rank == 0:
      for key in ('exp', 'summaries', 'renders'):
        dirs[key].mkdir(parents=True, exist_ok=True)
      writer = driver_utils.ScalarWriter(dirs['summaries'] / 'eval.jsonl')
    if datasource is None:
      datasource = driver_utils.make_datasource(exp_config, model_config, data_dir)
    if save_viz:
      frame_fn = functools.partial(frame_fn, viz_range=(datasource.near, datasource.far))

    def items_of(ids):                                                           # eval.py:297-300
      return [(i, datasource.load_camera(i), item['metadata'], item['rgb'])
              for i in ids for item in [datasource.get_item(i)]]
    sets = [('val', items_of(strided_subset(datasource.val_ids, eval_config.num_val_eval))),
            ('train', items_of(strided_subset(datasource.train_ids, eval_config.num_train_eval)))]
    test_cameras = datasource.load_test_cameras(count=eval_config.num_test_eval)   # eval.py:302-309

    model, params = construct_fn(                                                # eval.py:311-323
        0, model_config, batch_size=eval_config.chunk, appearance_ids=datasource.appearance_ids,
        camera_ids=datasource.camera_ids, warp_ids=datasource.warp_ids, near=datasource.near,
        far=datasource.far, use_warp_jacobian=False, use_weights=False, precision=precision)
    init_state = model_utils.TrainState(model_utils.Optimizer({'model': params}))
    device = getattr(model, 'device', 'cpu')

    handled, last_step = [], 0
    while True:                                                                  # eval.py:358-415
      step = next_checkpoint_step(dirs['checkpoints'], last_step)
      if step is None:
        log(f'No new checkpoints (last rendered step {last_step}).')
        time.sleep(poll_seconds)
        continue
      state = checkpoints.restore_checkpoint(str(dirs['checkpoints']), init_state, step=step, device=device)
      save_dir = dirs['renders'] if eval_config.save_output and rank == 0 else None
      todo = list(sets)
      if test_cameras:
        md = choose_test_metadata(datasource, step)
        todo.append(('test', [(f'{k:03d}', cam, md, None) for k, cam in enumerate(test_cameras)]))
      for tag, items in todo:
        process_items(tag, items, step, model, state.optimizer.target['model'], state.warp_extra,
                      save_dir, writer, pool, frame_fn, log)
      if save_dir:
        delete_old_renders(dirs['renders'], eval_config.max_render_checkpoints)
      handled.append(step)
      if eval_config.eval_once or step >= train_config.max_steps:
        return handled
      last_step = step
  finally:
    pool.shutdown(wait=True)
    if writer is not None:
      writer.close()
    if own_group:
      torch.distributed.destroy_process_group()


def main(argv=None, poll_seconds=10.0):
  parser = driver_utils.make_parser('nerfies_b200.eval', 'fp16x3')
  parser.add_argument('--eval_once', action='store_true', help='sets EvalConfig.eval_once')
  parser.add_argument('--save_viz', action='store_true',
                      help='also write the colour-mapped depth, disparity, accumulation and error images')
  args = parser.parse_args(argv)
  driver_utils.parse_configs(args.gin_configs, args.gin_bindings)
  exp_config = configs.ExperimentConfig()                                        # eval.py:238-241
  model_config = configs.ModelConfig(use_stratified_sampling=False)
  train_config = configs.TrainConfig()
  eval_config = configs.EvalConfig()
  if args.max_steps is not None:
    train_config.max_steps = args.max_steps
  if args.eval_once:
    eval_config.eval_once = True
  evaluate(exp_config, model_config, train_config, eval_config, args.base_folder, args.data_dir,
           precision=args.precision, poll_seconds=poll_seconds, save_viz=args.save_viz)
  return 0


if __name__ == '__main__':
  sys.exit(main())
