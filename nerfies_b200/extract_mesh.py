"""The mesh driver: a trained model's surface as a PLY file.

  python -m nerfies_b200.extract_mesh --base_folder EXP --data_dir CAPTURE --gin_configs X.gin \\
      [--step N] [--resolution 256] [--threshold SIGMA] [--bbox x0 y0 z0 x1 y1 z1] \\
      [--canonical] [--metadata warp=3 ...] [--level fine|coarse] [--colors] [--world_coords]

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

One process, one GPU.
"""
import json
import math
import pathlib
import sys

import numpy as np
import torch

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


def extract_mesh(exp_config, model_config, base_folder, data_dir=None, step=None, resolution=256, threshold=None,
                 bbox=None, canonical=False, metadata=(), level='fine', colors=False, world_coords=False,
                 precision='fp16x3', datasource=None, construct_fn=models.construct_nerf, log=print):
  """Writes the mesh; returns the PLY's path."""
  if level not in geometry.LEVELS:
    raise ValueError(f"--level must be 'coarse' or 'fine', got {level!r}")
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
  if world_coords:
    center, scale = np.asarray(datasource.scene_center, np.float64), float(datasource.scene_scale)
    vertices = (vertices.double() / scale + torch.as_tensor(center, device=vertices.device)).float()
  out_dir = dirs['exp'] / 'meshes' / f'{step:08d}'
  out_dir.mkdir(parents=True, exist_ok=True)
  path = out_dir / f'{mesh_name(canonical, md)}.ply'
  geometry.write_ply(path, vertices, faces, normals, rgb)
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
                      world_coords=args.world_coords, precision=args.precision)
  print(f'Wrote {path}')
  return 0


if __name__ == '__main__':
  sys.exit(main())
