"""The video driver: the last three cells of the reference's notebooks/Nerfies_Render_Video.ipynb
("Load cameras", "Render video frames", "Show rendered video") over this package's CUDA path.

  python -m nerfies_b200.render_video --base_folder EXP --data_dir CAPTURE --gin_configs configs/x.gin \\
      [--camera_path camera-paths/orbit-mild] [--fps 30] [--step N] [--metadata appearance=3 ...] [--normals]

Loads every camera of `<data_dir>/<camera_path>` in sorted order, restores the checkpoint of
`--step` (default: the newest) as `eval.evaluate` does, and renders each camera with
`evaluation.render_frame`.  Each frame is the notebook's
image_to_uint8(concatenate([rgb, colorize(median depth, near, far, invert=True)], axis=1)), made on
the device by `visualization.video_frame`, copied to pinned host memory without blocking and
handed to one worker thread, which writes `frame_<i:05d>.png` and appends the frame to `video.mp4`
(OpenCV, mp4v, `--fps`) in order while the next frame renders.  The video's sides are even, as 4:2:0
video needs: an odd last row or column of the frame is repeated in it (the PNGs are exact).  Output:
`<exp_dir>/videos/<camera path name>/<step, 8 digits>/`; not under `renders/`, whose oldest entries
eval deletes.  With `--normals`, each frame's normal map at the same median depth (eval.normal_image:
colours in the camera's frame, black where a ray meets no surface) also goes to `normals_<i:05d>.png` and
`normals.mp4` in that directory.

Metadata: every input the model reads is 0 ('appearance', 'warp', 'camera' ids) or 0.0 ('time'),
the notebook's zeros, unless `--metadata key=value` sets it.  The notebook builds no 'camera' id,
so it cannot render a vrig model; here it is 0 as well.

Deliberate difference: the model is built with `ModelConfig(use_stratified_sampling=False)`, as
eval.py does.  The notebook leaves stratified sampling on, which jitters the samples of every frame
and makes the video flicker.

Multi-GPU: under torchrun every rank renders its slab of each frame and rank 0 writes the files.
"""
import concurrent.futures
import pathlib
import sys

import numpy as np
import torch

from nerfies_b200 import checkpoints
from nerfies_b200 import configs
from nerfies_b200 import driver_utils
from nerfies_b200 import eval as eval_lib
from nerfies_b200 import evaluation
from nerfies_b200 import model_utils
from nerfies_b200 import models
from nerfies_b200 import visualization


def default_metadata(datasource, overrides=()):
  """{key: 0 / 0.0} for every metadata input the model reads, updated by 'key=value' strings."""
  metadata = {}
  for key, used in (('appearance', datasource.use_appearance_id), ('warp', datasource.use_warp_id),
                    ('camera', datasource.use_camera_id), ('time', datasource.use_time)):
    if used:
      metadata[key] = 0.0 if key == 'time' else 0
  for item in overrides:
    key, sep, value = item.partition('=')
    if not sep or key not in metadata:
      raise ValueError(f'--metadata {item!r}: expected key=value with key one of {sorted(metadata)} '
                       '(the metadata this model reads)')
    metadata[key] = float(value) if key == 'time' else int(value)
  return metadata


def render_video_frame(model, params, camera, warp_extra, metadata, near, far, normals=False):
  """One video frame on the device: uint8 (h, 2w, 3), rgb | colour-mapped median depth; with `normals`,
  the pair (frame, the normal map at the same median depth, uint8 (h, w, 3): eval.normal_image)."""
  render = evaluation.render_frame(model, params, camera, warp_extra, metadata)
  frame = visualization.video_frame(render['rgb'], render['med_depth'], near, far)
  if not normals:
    return frame
  return frame, eval_lib.normal_image(model, params, camera, warp_extra, metadata, render['med_depth'])


class _VideoSink:
  """<stem>_<i>.png files and one mp4, written in the order frames arrive."""

  def __init__(self, out_dir, fps, stem='frame', video='video.mp4'):
    self.out_dir, self.fps, self.writer, self.count = out_dir, fps, None, 0
    self.stem, self.video = stem, video

  def write(self, frame):
    import cv2
    eval_lib.write_png(self.out_dir / f'{self.stem}_{self.count:05d}.png', frame)
    h, w = frame.shape[:2]
    # 4:2:0 video needs even sides: an odd last row / column is repeated (the encoder would drop it)
    bgr = np.pad(frame[:, :, ::-1], ((0, h % 2), (0, w % 2), (0, 0)), mode='edge')
    if self.writer is None:
      self.writer = cv2.VideoWriter(str(self.out_dir / self.video), cv2.VideoWriter_fourcc(*'mp4v'), self.fps,
                                    (bgr.shape[1], bgr.shape[0]))
      if not self.writer.isOpened():
        raise IOError(f'could not open {self.out_dir / self.video} for writing')
    self.writer.write(np.ascontiguousarray(bgr))
    self.count += 1

  def close(self):
    if self.writer is not None:
      self.writer.release()


def render_video(exp_config, model_config, base_folder, data_dir=None, camera_path='camera-paths/orbit-mild',
                 fps=30.0, step=None, metadata=(), precision='fp16x3', datasource=None,
                 construct_fn=models.construct_nerf, frame_fn=render_video_frame, log=print, normals=False):
  """Renders the camera path; returns the output directory.  `datasource`, `construct_fn` and
  `frame_fn` replace the data source, the model constructor and the frame renderer (tests run the
  loop without a GPU that way).  With `normals`, frame_fn is called with normals=True and returns
  (frame, normal map)."""
  rank, world, own_group = driver_utils.init_distributed()
  pool = concurrent.futures.ThreadPoolExecutor(max_workers=1)          # one worker: frames stay in order
  sink = normal_sink = None
  try:
    dirs = driver_utils.experiment_dirs(base_folder, exp_config.subname)
    if datasource is None:
      datasource = driver_utils.make_datasource(exp_config, model_config, data_dir)
    camera_dir = pathlib.Path(datasource.data_dir) / camera_path
    paths = datasource.glob_cameras(camera_dir)
    if not paths:
      raise FileNotFoundError(f'no cameras in {camera_dir}')
    cameras = [datasource.load_camera(p) for p in paths]
    steps = eval_lib.checkpoint_steps(dirs['checkpoints'])
    if step is None:
      if not steps:
        raise FileNotFoundError(f'no checkpoints in {dirs["checkpoints"]}')
      step = steps[-1]
    elif step not in steps:
      raise FileNotFoundError(f'no checkpoint of step {step} in {dirs["checkpoints"]} (steps: {steps})')
    md = default_metadata(datasource, metadata)

    model, params = construct_fn(                                                # as eval.evaluate
        0, model_config, batch_size=configs.EvalConfig().chunk, appearance_ids=datasource.appearance_ids,
        camera_ids=datasource.camera_ids, warp_ids=datasource.warp_ids, near=datasource.near,
        far=datasource.far, use_warp_jacobian=False, use_weights=False, precision=precision)
    init_state = model_utils.TrainState(model_utils.Optimizer({'model': params}))
    state = checkpoints.restore_checkpoint(str(dirs['checkpoints']), init_state, step=step,
                                           device=getattr(model, 'device', 'cpu'))
    out_dir = dirs['exp'] / 'videos' / pathlib.Path(camera_path).name / f'{step:08d}'
    if rank == 0:
      out_dir.mkdir(parents=True, exist_ok=True)
      sink = _VideoSink(out_dir, fps)
      if normals:
        normal_sink = _VideoSink(out_dir, fps, 'normals', 'normals.mp4')
    pending = []
    for i, camera in enumerate(cameras):
      log(f'Rendering frame {i + 1}/{len(cameras)}')
      frame = frame_fn(model, state.optimizer.target['model'], camera, state.warp_extra, md, datasource.near,
                       datasource.far, **({'normals': True} if normals else {}))
      frame, normal_frame = frame if normals else (frame, None)
      if sink is not None:
        wait = eval_lib._host_copy(frame)
        pending.append(pool.submit(lambda w=wait: sink.write(w())))
      if normal_sink is not None:
        wait = eval_lib._host_copy(normal_frame)
        pending.append(pool.submit(lambda w=wait: normal_sink.write(w())))
    for future in pending:
      future.result()
    return out_dir
  finally:
    pool.shutdown(wait=True)
    for s in (sink, normal_sink):
      if s is not None:
        s.close()
    if own_group:
      torch.distributed.destroy_process_group()


def main(argv=None):
  parser = driver_utils.make_parser('nerfies_b200.render_video', 'fp16x3')
  parser.add_argument('--camera_path', default='camera-paths/orbit-mild',
                      help='directory of camera files, relative to --data_dir')
  parser.add_argument('--fps', type=float, default=30.0, help='frame rate of video.mp4')
  parser.add_argument('--step', type=int, default=None, help='checkpoint step (default: the newest)')
  parser.add_argument('--metadata', action='append', default=[], metavar='KEY=VALUE',
                      help="metadata of every frame, e.g. appearance=3 or time=0.5 (default 0)")
  parser.add_argument('--normals', action='store_true',
                      help='also write normals_<i>.png and normals.mp4, the surface normals at the median depth')
  args = parser.parse_args(argv)
  driver_utils.parse_configs(args.gin_configs, args.gin_bindings)
  exp_config = configs.ExperimentConfig()
  model_config = configs.ModelConfig(use_stratified_sampling=False)
  out_dir = render_video(exp_config, model_config, args.base_folder, args.data_dir, camera_path=args.camera_path,
                         fps=args.fps, step=args.step, metadata=args.metadata, precision=args.precision,
                         normals=args.normals)
  print(f'Wrote {out_dir}')
  return 0


if __name__ == '__main__':
  sys.exit(main())
