"""Time nfb_colorize and the video driver on the GPU.

  python tools/bench_viz.py [--frames N] [--out results/bench_viz.json]

1. colorize_uint8 at 1080 x 1920: the value source with given bounds (one launch) and the
   reciprocal source with bounds from the frame (range pass + colour pass), timed with CUDA events
   over 200 launches after 20 of warm-up.  GB/s is over the algorithmic bytes: 4 B read and 3 B
   written per pixel, plus 4 B read per pixel by the range pass.
2. The video driver's wall time per frame against `render_frame`'s render_ms, for a random-init
   model of gpu_quarterhd.gin's size at 1080 x 1920 cameras: the PNG and mp4 encoding runs in a
   worker thread and should not add to the time per frame.
Prints one JSON object with the card's name and power limit.
"""
import argparse
import json
import os
import pathlib
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, W = 1080, 1920


def card():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
  except (OSError, subprocess.SubprocessError, IndexError):
    out = torch.cuda.get_device_name(0)
  return out


def time_colorize(fn, iters=200, warmup=20):
  for _ in range(warmup):
    fn()
  start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  for _ in range(iters):
    fn()
  end.record()
  end.synchronize()
  return start.elapsed_time(end) / iters


def bench_kernels():
  from nerfies_b200 import visualization as viz
  dev = torch.device('cuda', 0)
  g = torch.Generator(device=dev).manual_seed(0)
  depth = torch.rand(H, W, device=dev, generator=g) * 3 + 0.05
  out = torch.empty(H, W, 3, dtype=torch.uint8, device=dev)
  n = H * W
  res = {}
  for name, fn, nbytes in (
      ('value_given', lambda: viz.colorize_uint8(depth, 0.1, 2.5, invert=True, out=out), 7 * n),
      ('reciprocal_frame', lambda: viz.colorize_uint8(depth, source='reciprocal', out=out), 11 * n)):
    ms = time_colorize(fn)
    res[name] = {'us': ms * 1e3, 'GB/s': nbytes / (ms * 1e-3) / 1e9, 'bytes': nbytes}
  return res


class _Source:
  use_appearance_id = use_warp_id = True
  use_camera_id = use_time = False
  appearance_ids = warp_ids = tuple(range(8))
  camera_ids = ()
  near, far = 0.1, 2.5

  def __init__(self, data_dir, cameras):
    self.data_dir, self.cameras = data_dir, cameras

  def glob_cameras(self, path):
    return list(range(len(self.cameras)))

  def load_camera(self, i):
    return self.cameras[i]


def bench_video(frames):
  from nerfies_b200 import camera as camera_lib, checkpoints, configs, evaluation, model_utils, models
  from nerfies_b200 import render_video
  configs.clear_config()
  configs.parse_config_files_and_bindings([os.path.join(ROOT, 'tests', 'golden', 'gin', 'gpu_quarterhd.gin')],
                                          [], skip_unknown=True)
  model_config = configs.ModelConfig(use_stratified_sampling=False)
  cams = []
  for i in range(frames):
    a = 0.2 * i
    rot = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]], np.float32)
    cams.append(camera_lib.Camera(orientation=rot, position=(-rot[2] * 1.0).astype(np.float32), focal_length=1500.0,
                                  principal_point=[W / 2, H / 2], image_size=[W, H]))
  with tempfile.TemporaryDirectory() as tmp:
    source = _Source(tmp, cams)
    model, params = models.construct_nerf(0, model_config, 8192, source.appearance_ids, (), source.warp_ids,
                                          near=source.near, far=source.far, precision='fp16x3')
    checkpoints.save_checkpoint(os.path.join(tmp, 'checkpoints'),
                                model_utils.TrainState(model_utils.Optimizer({'model': params})), 1)
    construct = lambda *a, **kw: (model, params)
    render_ms = []
    for cam in cams[:2] + cams:                                                  # 2 warm-up frames
      t = {}
      evaluation.render_frame(model, params, cam, {'alpha': 0.0, 'time_alpha': 0.0}, {'appearance': 0, 'warp': 0},
                              timings=t)
      render_ms.append(t['render_ms'] + t['gather_ms'])
    render_video.render_video(configs.ExperimentConfig(), model_config, tmp, camera_path='warm', datasource=_Source(
        tmp, cams[:2]), construct_fn=construct, log=lambda s: None)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    render_video.render_video(configs.ExperimentConfig(), model_config, tmp, camera_path='path', datasource=source,
                              construct_fn=construct, log=lambda s: None)
    wall = (time.perf_counter() - t0) * 1e3
    written = sorted(os.listdir(pathlib.Path(tmp) / 'videos' / 'path' / '00000001'))
  assert len(written) == frames + 1, written
  return {'frames': frames, 'wall_ms_per_frame': wall / frames,
          'render_frame_ms_mean': float(np.mean(render_ms[2:])), 'render_frame_ms': render_ms[2:]}


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--frames', type=int, default=6)
  p.add_argument('--out', default=None)
  args = p.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_viz needs a CUDA device')
  torch.cuda.set_device(0)
  res = {'card': card(), 'colorize_uint8_1080x1920': bench_kernels(), 'video_1080x1920': bench_video(args.frames)}
  line = json.dumps(res)
  print(line)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
      f.write(line + '\n')


if __name__ == '__main__':
  main()
