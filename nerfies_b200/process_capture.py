"""python -m nerfies_b200.process_capture: a COLMAP reconstruction to a Nerfies capture.

The reference's capture notebook (notebooks/Nerfies_Capture_Processing.ipynb) as two commands,
because COLMAP runs between them:

  images   "Resize images into different scales": every PNG of --frames_dir, cropped to a
           multiple of the largest scale, written at each scale to <data_dir>/rgb/<s>x/.
  scene    "Load COLMAP scene" through "Save test cameras": reads <colmap_dir>/*.bin, drops the
           frames the blur filter selects, and writes scene.json, dataset.json, metadata.json,
           camera/<id>.json, camera-paths/orbit-mild/<i>.json and points.npy (the track-filtered
           COLMAP points in world coordinates, which TrainConfig.use_background_loss reads).

The flags are the notebook's @param values; its other literals are constants of
nerfies_b200.capture.  PNGs are decoded on host threads, each frame is uploaded once, and PNGs
are encoded on a worker thread while the GPU works on the next frame.
"""
import argparse
import concurrent.futures
import json
import pathlib
import sys

import numpy as np
import torch

from nerfies_b200 import capture
from nerfies_b200 import colmap
from nerfies_b200 import datasets

MIN_TRACK_LENGTH = 5
ORBIT_PATH = 'orbit-mild'
BLUR_BATCH = 8


def _scales(text):
  try:
    return capture.check_scales(int(s) for s in text.split(','))
  except ValueError as e:
    raise argparse.ArgumentTypeError(str(e)) from None


def _positive_float(text):
  v = float(text)
  if not v > 0:
    raise argparse.ArgumentTypeError(f'{text} is not positive')
  return v


def _positive_int(text):
  v = int(text)
  if v < 1:
    raise argparse.ArgumentTypeError(f'{text} is not a positive integer')
  return v


def make_parser():
  p = argparse.ArgumentParser(prog='python -m nerfies_b200.process_capture')
  sub = p.add_subparsers(dest='command', required=True)
  im = sub.add_parser('images', help='write the image pyramid of every frame')
  im.add_argument('--frames_dir', required=True, help='directory of the extracted frames (*.png)')
  im.add_argument('--data_dir', required=True, help='capture directory; frames go to rgb/<s>x/')
  im.add_argument('--image_scales', type=_scales, default=[1, 2, 4, 8],
                  help='comma-separated scales, each 1 or even (default 1,2,4,8)')
  sc = sub.add_parser('scene', help='write the capture files from a COLMAP model')
  sc.add_argument('--data_dir', required=True, help='capture directory holding rgb/1x/')
  sc.add_argument('--colmap_dir', required=True, help='COLMAP model directory (cameras.bin, images.bin, points3D.bin)')
  sc.add_argument('--colmap_image_scale', type=_positive_float, default=4,
                  help='the scale of the frames COLMAP was run on')
  sc.add_argument('--blur_filter_perc', type=float, default=95.0,
                  help='drop the frames whose blur score is at or above this percentile (0: none)')
  sc.add_argument('--orbit_frames', type=_positive_int, default=100)
  sc.add_argument('--orbit_radius', type=float, default=0.75)
  sc.add_argument('--orbit_x_scale', type=float, default=0.75)
  sc.add_argument('--orbit_y_scale', type=float, default=0.75)
  for s in (im, sc):
    s.add_argument('--device', default='cuda', help='CUDA device')
  return p


def _write_png(path, array):
  from nerfies_b200.eval import write_png
  path.parent.mkdir(parents=True, exist_ok=True)
  write_png(str(path), array)


def run_images(frames_dir, data_dir, scales, device):
  frames = sorted(pathlib.Path(frames_dir).glob('*.png'))
  if not frames:
    raise FileNotFoundError(f'no *.png frames in {frames_dir}')
  rgb_dir = pathlib.Path(data_dir) / 'rgb'
  with concurrent.futures.ThreadPoolExecutor() as decode, \
      concurrent.futures.ThreadPoolExecutor(max_workers=1) as encode:
    pending = []
    for path, image in zip(frames, decode.map(datasets.decode_image, frames)):
      levels = capture.downsample_frames(torch.from_numpy(image).to(device), scales)
      host = {s: t.cpu().numpy() for s, t in levels.items()}
      pending += [encode.submit(_write_png, rgb_dir / f'{s}x' / f'{path.stem}.png', a) for s, a in host.items()]
    for f in pending:
      f.result()
  return [p.stem for p in frames]


def _blur_scores(data_dir, item_ids, device):
  paths = [pathlib.Path(data_dir) / 'rgb' / '1x' / f'{i}.png' for i in item_ids]
  scores = []
  with concurrent.futures.ThreadPoolExecutor() as decode:
    images = decode.map(datasets.decode_image, paths)
    batch = []
    for path, image in zip(paths, images):
      if batch and batch[0].shape != image.shape:
        raise ValueError(f'{path} is {image.shape[1]}x{image.shape[0]}, other frames are '
                         f'{batch[0].shape[1]}x{batch[0].shape[0]}')
      batch.append(image)
      if len(batch) == BLUR_BATCH:
        scores.append(capture.blur_scores(torch.from_numpy(np.stack(batch)).to(device)).cpu())
        batch = []
    if batch:
      scores.append(capture.blur_scores(torch.from_numpy(np.stack(batch)).to(device)).cpu())
  return torch.cat(scores).numpy()


def run_scene(args):
  data_dir = pathlib.Path(args.data_dir)
  device = torch.device(args.device)
  cameras, points = colmap.load_scene(args.colmap_dir, MIN_TRACK_LENGTH)
  if args.colmap_image_scale != 1:
    cameras = {k: c.scale(args.colmap_image_scale) for k, c in cameras.items()}
  registered = sorted(cameras)
  scores = _blur_scores(data_dir, registered, device)
  removed = capture.blur_filter(registered, scores, args.blur_filter_perc)
  print(f'Filtering {len(removed)} IDs: {removed}')
  for i in removed:
    cameras.pop(i)
  item_ids = sorted(cameras)
  if not item_ids:
    raise ValueError('the blur filter removed every frame')
  camera_list = [cameras[i] for i in item_ids]
  near, far, _ = capture.estimate_near_far(item_ids, camera_list, points, device)
  scene = capture.scene_info(points, camera_list, near, far)
  dataset, metadata = capture.split_and_metadata(item_ids)
  orbit = capture.orbit_camera_path(camera_list, args.orbit_frames, args.orbit_radius, args.orbit_x_scale,
                                    args.orbit_y_scale)

  def dump(path, blob):
    path.parent.mkdir(parents=True, exist_ok=True)
    with open(path, 'w') as f:
      json.dump(blob, f, indent=2)

  dump(data_dir / 'scene.json', scene)
  dump(data_dir / 'dataset.json', dataset)
  dump(data_dir / 'metadata.json', metadata)
  for i in item_ids:
    dump(data_dir / 'camera' / f'{i}.json', cameras[i].to_json())
  for k, c in enumerate(orbit):
    dump(data_dir / 'camera-paths' / ORBIT_PATH / f'{k:06d}.json', c.to_json())
  np.save(data_dir / 'points.npy', points)
  print(f'near {near:.4f} far {far:.4f} (unscaled); {len(item_ids)} items; wrote {data_dir}')
  return {'removed': removed, 'scores': dict(zip(registered, scores.tolist())), 'near': near, 'far': far}


def main(argv=None):
  args = make_parser().parse_args(argv)
  if args.command == 'images':
    run_images(args.frames_dir, args.data_dir, args.image_scales, torch.device(args.device))
  else:
    run_scene(args)
  return 0


if __name__ == '__main__':
  sys.exit(main())
