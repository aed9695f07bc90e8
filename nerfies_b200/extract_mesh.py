"""The mesh driver: a trained model's surface as a PLY file.

  python -m nerfies_b200.extract_mesh --base_folder EXP --data_dir CAPTURE --gin_configs X.gin \\
      [--step N] [--resolution 256] [--threshold SIGMA] [--bbox x0 y0 z0 x1 y1 z1] \\
      [--canonical] [--metadata warp=3 ...] [--level fine|coarse] [--colors] [--world_coords] \\
      [--track [--frames V ...]]

Restores the checkpoint of `--step` (default: the newest) and its warp_extra as render_video does,
evaluates the density of `--level`'s NeRF MLP on a grid over the box (geometry.density_grid) and
extracts the surface {sigma > threshold} by marching cubes (geometry.marching_cubes).

- Space: by default the observation space of the frame the metadata names (frame 0 unless
  `--metadata` says otherwise: the shape render_video shows); `--canonical` gives the template
  (no warp).  A model without a warp field has only the template.
- Box, in the scene's normalised coordinates: `--bbox`, else scene.json's `bbox` (written by
  process_capture) normalised by its `center` and `scale`, else the extent of points.npy
  (normalised as datasets.load_points does) grown by 10 % of the extent on every side.
- Resolution: grid points along the box's longest side; the other sides get as many points as
  cubic voxels need to cover the box (the box grows to a whole number of voxels).
- Threshold: by default ln 2 * num_coarse_samples / (far - near), the density at which one coarse
  sample step of the model is half opaque; it does not depend on the grid resolution.
- Output: `<exp_dir>/meshes/<step, 8 digits>/<canonical | warp_<id> | time_<t>>.ply`, binary PLY
  with normals (and colours with `--colors`: each vertex's colour seen along -normal).  With
  `--world_coords` the vertices are mapped back to the capture's world frame (x / scale + center).
- `--track [--frames V ...]`: the template mesh (as `--canonical`, written as `canonical.ply`) carried
  into every frame with one topology: each vertex is the inverse of the frame's warp at the template
  vertex (geometry.track_surface; tolerance TRACK_TOL_VOXELS of the voxel size, TRACK_MAX_ITERS
  Newton iterations), warm-started from its solution in the previous frame where that converged.
  Frames are `--frames` (warp ids as `--metadata warp=` takes them, or timestamps with the 'time'
  encoder), by default every training frame's in increasing order.  Output in
  `meshes/<step>/track/`: `canonical.ply`, one PLY per frame (named as the frame's own mesh would be)
  with the canonical faces and the tracked normals, and `track.npz` with `frames`, `faces (F, 3)`,
  `vertices (T, V, 3)`, `residual (T, V)` (|W(x) - template vertex|, normalised scene units) and
  `status (T, V)` (uint8, nfb_warp_invert's NFB_INVERT_*).

One process, one GPU.
"""
import json
import math
import pathlib
import sys

import numpy as np
import torch

from nerfies_b200 import _lib
from nerfies_b200 import checkpoints
from nerfies_b200 import configs
from nerfies_b200 import driver_utils
from nerfies_b200 import eval as eval_lib
from nerfies_b200 import geometry
from nerfies_b200 import model_utils
from nerfies_b200 import models
from nerfies_b200.render_video import default_metadata

MAX_SIDE = 1024
POINTS_PADDING = 0.1
TRACK_TOL_VOXELS = 1e-2
TRACK_MAX_ITERS = 16


def scene_box(data_dir, bbox=None):
  """The box ((x0, y0, z0), (x1, y1, z1)) float64 in normalised scene coordinates (see the module
  docstring for the order of the sources)."""
  if bbox is not None:
    box = np.asarray(bbox, np.float64).reshape(2, 3)
    if not np.all(np.isfinite(box)) or not np.all(box[1] > box[0]):
      raise ValueError(f'--bbox {list(np.ravel(bbox))}: expected x0 y0 z0 x1 y1 z1 with x1 > x0, y1 > y0, z1 > z0')
    return box
  data_dir = pathlib.Path(data_dir)
  with open(data_dir / 'scene.json') as f:
    scene = json.load(f)
  center, scale = np.asarray(scene['center'], np.float64), float(scene['scale'])
  if 'bbox' in scene:
    return (np.asarray(scene['bbox'], np.float64).reshape(2, 3) - center) * scale
  if (data_dir / 'points.npy').exists():
    points = ((np.load(data_dir / 'points.npy') - center) * scale).astype(np.float32)
    if len(points):
      lo, hi = points.min(0).astype(np.float64), points.max(0).astype(np.float64)
      pad = POINTS_PADDING * np.maximum(hi - lo, 1e-6)
      return np.stack([lo - pad, hi + pad])
  raise ValueError(f'no box for the mesh: pass --bbox, or give {data_dir / "scene.json"} a bbox '
                   f'(process_capture writes one), or provide {data_dir / "points.npy"}')


def grid_for_box(box, resolution):
  """(grid box, shape (nz, ny, nx)): `resolution` points along the longest side, cubic voxels, the
  box grown at its upper end to a whole number of voxels on every axis."""
  if not 2 <= resolution <= MAX_SIDE:
    raise ValueError(f'--resolution {resolution}: must lie in [2, {MAX_SIDE}]')
  box = np.asarray(box, np.float64)
  extent = box[1] - box[0]
  voxel = extent.max() / (resolution - 1)
  n = [min(MAX_SIDE, max(2, int(math.ceil(e / voxel - 1e-9)) + 1)) for e in extent]
  hi = box[0] + (np.array(n) - 1) * voxel
  return np.stack([box[0], hi]), (n[2], n[1], n[0])


def default_threshold(num_coarse_samples, near, far):
  """ln 2 * Nc / (far - near): sigma whose coarse step (far - near) / Nc has opacity 1/2."""
  return math.log(2.0) * num_coarse_samples / (far - near)


def mesh_name(canonical, metadata):
  if canonical:
    return 'canonical'
  if 'warp' in metadata:
    return f'warp_{metadata["warp"]}'
  if 'time' in metadata:
    return f'time_{metadata["time"]:g}'
  return 'canonical'


def check_track(canonical, metadata, model_config):
  """Refuses --track with what it contradicts: raises ValueError."""
  if canonical:
    raise ValueError('--track carries the template into every frame; it does not take --canonical')
  for item in metadata:
    if item.partition('=')[0] in ('warp', 'time'):
      raise ValueError(f'--metadata {item!r}: --track visits the frames of --frames, not one frame of --metadata')
  if not model_config.use_warp:
    raise ValueError('--track needs a model with a warp field (ModelConfig.use_warp)')


def track_frames(datasource, model_config, frames=None):
  """The frames --track visits, as the model reads them: `frames` (strings or numbers), else the
  training frames in increasing order: the warp ids (their index among the training warp ids, as
  --metadata warp= takes them) or, with the 'time' encoder, the timestamps."""
  time = model_config.warp_metadata_encoder_type == 'time'
  if frames:
    return [float(f) if time else int(f) for f in frames]
  if time:
    found = sorted({float(datasource.get_time(i)) for i in datasource.train_ids}) if datasource.use_time else []
  else:
    found = list(range(len(datasource.warp_ids)))
  if not found:
    raise ValueError('--track: the datasource exposes no frames; pass --frames')
  return found


def extract_mesh(exp_config, model_config, base_folder, data_dir=None, step=None, resolution=256, threshold=None,
                 bbox=None, canonical=False, metadata=(), level='fine', colors=False, world_coords=False,
                 precision='fp16x3', datasource=None, construct_fn=models.construct_nerf, log=print, track=False,
                 frames=None):
  """Writes the mesh; returns the PLY's path (with `track`, the path of track.npz)."""
  if level not in geometry.LEVELS:
    raise ValueError(f"--level must be 'coarse' or 'fine', got {level!r}")
  if track:
    check_track(canonical, metadata, model_config)
  elif frames:
    raise ValueError('--frames chooses the frames of --track; without --track use --metadata')
  dirs = driver_utils.experiment_dirs(base_folder, exp_config.subname)
  if datasource is None:
    datasource = driver_utils.make_datasource(exp_config, model_config, data_dir)
  box, shape = grid_for_box(scene_box(datasource.data_dir, bbox), resolution)
  if threshold is None:
    threshold = default_threshold(model_config.num_coarse_samples, datasource.near, datasource.far)
  steps = eval_lib.checkpoint_steps(dirs['checkpoints'])
  if step is None:
    if not steps:
      raise FileNotFoundError(f'no checkpoints in {dirs["checkpoints"]}')
    step = steps[-1]
  elif step not in steps:
    raise FileNotFoundError(f'no checkpoint of step {step} in {dirs["checkpoints"]} (steps: {steps})')
  md = default_metadata(datasource, metadata)
  canonical = canonical or not model_config.use_warp
  if track:
    frame_list = track_frames(datasource, model_config, frames)
    canonical = True

  model, params = construct_fn(                                                   # as render_video
      0, model_config, batch_size=configs.EvalConfig().chunk, appearance_ids=datasource.appearance_ids,
      camera_ids=datasource.camera_ids, warp_ids=datasource.warp_ids, near=datasource.near,
      far=datasource.far, use_warp_jacobian=False, use_weights=False, precision=precision)
  init_state = model_utils.TrainState(model_utils.Optimizer({'model': params}))
  state = checkpoints.restore_checkpoint(str(dirs['checkpoints']), init_state, step=step,
                                         device=getattr(model, 'device', 'cpu'))
  params = state.optimizer.target['model']
  log(f'Density grid {shape[2]} x {shape[1]} x {shape[0]} over {box.tolist()} (level {level}, '
      f'{"canonical" if canonical else "observation space"})')
  grid = geometry.density_grid(model, params, box, shape, state.warp_extra, md, use_warp=not canonical, level=level)
  vertices, faces, normals, axes = geometry.marching_cubes(grid, threshold, box, return_axes=True)
  log(f'Marching cubes at sigma {threshold:g}: {len(vertices)} vertices, {len(faces)} faces')
  rgb = None
  if colors:
    rgb = geometry.vertex_colors(model, params, vertices, normals, state.warp_extra, md, use_warp=not canonical,
                                 level=level, axes=axes)
  to_world = lambda v: v
  if world_coords:
    center, scale = np.asarray(datasource.scene_center, np.float64), float(datasource.scene_scale)
    to_world = lambda v: (v.double() / scale + torch.as_tensor(center, device=v.device)).float()
  out_dir = dirs['exp'] / 'meshes' / f'{step:08d}'
  if track:
    out_dir = out_dir / 'track'
  out_dir.mkdir(parents=True, exist_ok=True)
  path = out_dir / f'{mesh_name(canonical, md)}.ply'
  geometry.write_ply(path, to_world(vertices), faces, normals, rgb)
  if not track:
    return path
  return track_mesh(model, params, state.warp_extra, md, vertices, faces, normals, axes, frame_list,
                    TRACK_TOL_VOXELS * float(geometry.grid_spacing(box, shape)[0]), out_dir, to_world,
                    level=level, colors=colors, time=model_config.warp_metadata_encoder_type == 'time', log=log)


def track_mesh(model, params, warp_extra, metadata, vertices, faces, normals, axes, frames, tol, out_dir, to_world,
               level='fine', colors=False, time=False, log=print):
  """The template mesh in each of `frames` (see the module docstring): one PLY per frame and track.npz
  in out_dir; returns the path of track.npz."""
  key = 'time' if time else 'warp'
  tracked, residual, status = [], [], []
  converged = None
  for f in frames:
    md = dict(metadata, **{key: f})
    init = None if converged is None else torch.where(converged[:, None], tracked_v, vertices)
    t = geometry.track_surface(model, params, vertices, normals, warp_extra, md, init=init, tol=tol,
                               max_iters=TRACK_MAX_ITERS)
    tracked_v = t['vertices']
    converged = t['status'] == _lib.INVERT_STATUS['converged']
    rgb = None
    if colors:
      rgb = geometry.vertex_colors(model, params, tracked_v, t['normals'], warp_extra, md, use_warp=True,
                                   level=level, axes=axes)
    name = mesh_name(False, {key: f})
    geometry.write_ply(out_dir / f'{name}.ply', to_world(tracked_v), faces, t['normals'], rgb)
    tracked.append(to_world(tracked_v).cpu().numpy())
    residual.append(t['residual'].cpu().numpy())
    status.append(t['status'].cpu().numpy().astype(np.uint8))
    finite = residual[-1][np.isfinite(residual[-1])]
    log(f'{name}: {int(converged.sum())} of {len(tracked_v)} vertices converged, worst residual '
        f'{float(finite.max()) if len(finite) else float("nan"):.3g}, {t["folded"]} folded (det J <= 0)')
  path = out_dir / 'track.npz'
  np.savez(path, frames=np.asarray(frames, np.float32 if time else np.int64),
           faces=faces.cpu().numpy().astype(np.int32), vertices=np.stack(tracked).astype(np.float32),
           residual=np.stack(residual).astype(np.float32), status=np.stack(status))
  return path


def make_parser():
  parser = driver_utils.make_parser('nerfies_b200.extract_mesh', 'fp16x3')
  parser.add_argument('--step', type=int, default=None, help='checkpoint step (default: the newest)')
  parser.add_argument('--resolution', type=int, default=256, help='grid points along the box\'s longest side')
  parser.add_argument('--threshold', type=float, default=None,
                      help='density level of the surface (default: ln 2 * num_coarse_samples / (far - near))')
  parser.add_argument('--bbox', type=float, nargs=6, default=None, metavar=('X0', 'Y0', 'Z0', 'X1', 'Y1', 'Z1'),
                      help='box in normalised scene coordinates (default: scene.json, then points.npy)')
  parser.add_argument('--canonical', action='store_true', help='the template shape (no warp)')
  parser.add_argument('--metadata', action='append', default=[], metavar='KEY=VALUE',
                      help='metadata of the frame, e.g. warp=3 or time=0.5 (default 0)')
  parser.add_argument('--level', default='fine', choices=('fine', 'coarse'), help='NeRF MLP whose density is used')
  parser.add_argument('--colors', action='store_true', help='vertex colours seen along -normal')
  parser.add_argument('--world_coords', action='store_true', help='vertices in the capture\'s world frame')
  parser.add_argument('--track', action='store_true',
                      help='the template mesh carried into every frame with one topology (meshes/<step>/track/)')
  parser.add_argument('--frames', nargs='+', default=None, metavar='V',
                      help='with --track: warp ids (timestamps with the \'time\' encoder); default: the training frames')
  return parser


def main(argv=None):
  args = make_parser().parse_args(argv)
  driver_utils.parse_configs(args.gin_configs, args.gin_bindings)
  exp_config = configs.ExperimentConfig()
  model_config = configs.ModelConfig(use_stratified_sampling=False)
  path = extract_mesh(exp_config, model_config, args.base_folder, args.data_dir, step=args.step,
                      resolution=args.resolution, threshold=args.threshold,
                      bbox=None if args.bbox is None else np.reshape(args.bbox, (2, 3)), canonical=args.canonical,
                      metadata=args.metadata, level=args.level, colors=args.colors,
                      world_coords=args.world_coords, precision=args.precision, track=args.track,
                      frames=args.frames)
  print(f'Wrote {path}')
  return 0


if __name__ == '__main__':
  sys.exit(main())
