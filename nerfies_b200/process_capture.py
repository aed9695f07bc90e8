"""python -m nerfies_b200.process_capture: a COLMAP reconstruction to a Nerfies capture.

The reference's capture notebook (notebooks/Nerfies_Capture_Processing.ipynb) as two commands,
because COLMAP runs between them:

  images   "Resize images into different scales": every PNG of --frames_dir, cropped to a
           multiple of the largest scale, written at each scale to <data_dir>/rgb/<s>x/.
  scene    "Load COLMAP scene" through "Save test cameras": reads <colmap_dir>/*.bin, drops the
           frames the blur filter selects, and writes scene.json, dataset.json, metadata.json,
           camera/<id>.json, camera-paths/orbit-mild/<i>.json and points.npy (the track-filtered
           COLMAP points in world coordinates, which TrainConfig.use_background_loss reads).
  depth    per-frame sensor depth (--depth_dir: <id>.npy metric z-depth maps at any resolution, e.g.
           a phone's LiDAR) to depth/<s>x/<id>.npy for every scale under rgb/: float32 maps of the
           frame's size holding the distance along each pixel centre's unit ray in scene units (the
           renderer's depth), NaN where nothing was measured.  Sensor units become COLMAP units by
           --depth_scale, or by the median ratio of the COLMAP points' camera depth to the sensor depth
           at their pixels.  Run after `scene`.

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
  dp = sub.add_parser('depth', help='write depth/<s>x/ from per-frame sensor depth maps')
  dp.add_argument('--data_dir', required=True, help='capture directory (after `scene`)')
  dp.add_argument('--depth_dir', required=True,
                  help='directory of <id>.npy sensor z-depth maps (distance along the optical axis), any resolution')
  dp.add_argument('--depth_scale', type=_positive_float, default=None,
                  help='sensor units -> COLMAP world units (default: estimated from points.npy)')
  dp.add_argument('--allow_missing', action='store_true',
                  help='skip the items without a depth map (no file is written for them)')
  for s in (im, sc, dp):
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


def _png_size(path):
  """(h, w) of a PNG from its header."""
  with open(path, 'rb') as f:
    head = f.read(24)
  if head[:8] != b'\x89PNG\r\n\x1a\n':
    raise ValueError(f'{path} is not a PNG')
  w, h = (int.from_bytes(head[o:o + 4], 'big') for o in (16, 20))
  return h, w


def _load_sensor_depth(path):
  depth = np.load(path)
  if depth.ndim != 2 or not np.issubdtype(depth.dtype, np.floating):
    raise ValueError(f'{path}: a sensor depth map is a 2-D float array, not {depth.dtype} {depth.shape}')
  return depth


def run_depth(args, log=print):
  """`depth`: checks everything on the host first (ids, map files and shapes, scene.json, scales, each frame's
  size against its scaled camera, points), so a refusal writes nothing; then one nfb_depth_resample launch per
  item and scale.  Returns {'metric_scale', 'pairs', 'iqr',
  'written': [paths], 'missing': [ids]}."""
  data_dir, raw_dir = pathlib.Path(args.data_dir), pathlib.Path(args.depth_dir)
  for name in ('scene.json', 'dataset.json'):
    if not (data_dir / name).exists():
      raise FileNotFoundError(f'{data_dir / name} is missing: run `process_capture scene` first')
  scene = json.loads((data_dir / 'scene.json').read_text())
  ids = [str(i) for i in json.loads((data_dir / 'dataset.json').read_text())['ids']]
  missing = [i for i in ids if not (raw_dir / f'{i}.npy').exists()]
  if missing and not args.allow_missing:
    raise FileNotFoundError(f'{len(missing)} item(s) have no depth map in {raw_dir}: {missing[:10]} '
                            '(--allow_missing skips them)')
  ids = [i for i in ids if i not in missing]
  if not ids:
    raise FileNotFoundError(f'no item of {data_dir / "dataset.json"} has a depth map in {raw_dir}')
  sensors = {i: _load_sensor_depth(raw_dir / f'{i}.npy') for i in ids}
  scales = sorted(int(p.name[:-1]) for p in (data_dir / 'rgb').glob('*x')
                  if p.is_dir() and p.name[:-1].isdigit()) if (data_dir / 'rgb').is_dir() else []
  if not scales:
    raise FileNotFoundError(f'{data_dir / "rgb"} holds no <s>x/ directory')
  cameras = {i: datasets.camera_lib.Camera.from_json(data_dir / 'camera' / f'{i}.json') for i in ids}
  frames = []                 # (item, scale, camera at that scale) of every map to write
  for i in ids:
    for s in scales:
      png = data_dir / 'rgb' / f'{s}x' / f'{i}.png'
      if not png.exists():
        continue
      cam = cameras[i].scale(1.0 / s)
      if cam.image_shape != _png_size(png):
        raise ValueError(f'{png} is {_png_size(png)} (h, w) but its camera scaled by 1/{s} gives {cam.image_shape}')
      frames.append((i, s, cam))
  points = None
  if args.depth_scale is None:
    if not (data_dir / 'points.npy').exists():
      raise FileNotFoundError(f'{data_dir / "points.npy"} is missing: pass --depth_scale')
    points = np.load(data_dir / 'points.npy')
  device = torch.device(args.device)
  pairs, iqr = 0, None
  if points is None:
    metric_scale = float(args.depth_scale)
  else:
    metric_scale, pairs, iqr = capture.estimate_depth_scale(
        [capture.depth_scale_pairs(points, cameras[i], sensors[i], device) for i in ids])
    log(f'metric scale {metric_scale:.6g} from {pairs} point/depth pairs (interquartile range {iqr:.3g})')
  factor = metric_scale * float(scene['scale'])
  written = []
  for i, s, cam in frames:
    out = data_dir / 'depth' / f'{s}x' / f'{i}.npy'
    out.parent.mkdir(parents=True, exist_ok=True)
    np.save(out, capture.resample_depth(sensors[i], cam, factor, device))
    written.append(out)
  log(f'wrote {len(written)} depth maps for {len(ids)} items at scales {scales}'
      + (f'; {len(missing)} items without a map: {missing[:10]}' if missing else ''))
  return {'metric_scale': metric_scale, 'pairs': pairs, 'iqr': iqr, 'written': written, 'missing': missing}


def main(argv=None):
  args = make_parser().parse_args(argv)
  if args.command == 'images':
    run_images(args.frames_dir, args.data_dir, args.image_scales, torch.device(args.device))
  elif args.command == 'depth':
    run_depth(args)
  else:
    run_scene(args)
  return 0


if __name__ == '__main__':
  sys.exit(main())
