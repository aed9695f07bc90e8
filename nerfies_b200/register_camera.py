"""The camera registration driver: where was a photo taken?  Fits a camera pose, and the photo's codes, to
the photo with the model held fixed (geometry.register_camera, iNeRF-style).

  python -m nerfies_b200.register_camera --base_folder EXP --data_dir CAPTURE --gin_configs X.gin \\
      (--item ITEM | --image PNG) [--init_camera JSON] [--optimize pose,appearance] \\
      [--intrinsics focal,principal_point,radial,tangential] [--steps 200] \\
      [--batch_rays 1024] [--lr_rotation R] [--lr_position P] [--lr_appearance A] [--lr_camera C] \\
      [--lr_warp W] [--lr_focal F] [--lr_principal_point C] [--lr_radial K] [--lr_tangential T] [--lr_decay D] [--seed S] [--step N] [--metadata key=value ...] [--name NAME]

Restores the checkpoint of `--step` (default: the newest) and its warp_extra as render_video does.  The target
is `--item`'s rgb at the experiment's scale or `--image`, which must have the camera's size.  The starting
camera is `--init_camera` (a camera JSON at the capture's original scale, scaled as datasource.load_camera
scales an item's camera) or the item's own camera.  The codes start from the item's metadata (with
`--image`: zeros) and `--metadata key=value` overrides, as render_video reads them.  `--optimize` names the
groups fitted: pose, appearance, camera, warp ('warp' needs a 'glo' warp encoder).  `--intrinsics` names the
camera intrinsics parts fitted as well: focal, principal_point, radial, tangential (an intrinsics delta,
geometry.refined_camera; 'radial' and 'tangential' also fit a camera without distortion, starting from 0).

Output in `<exp_dir>/registrations/<step, 8 digits>/<name>/` (name: the item, or the image's stem):
  camera.json     the registered camera at the capture's original scale (drops in beside camera/*.json), with
                  the fitted intrinsics;
  codes.npz       the fitted codes, (1, width) each, the ids they started from, and a fitted intrinsics delta;
  log.jsonl       per logged step: step, loss, psnr (of the batch), rotation_deg (|omega|), translation (|v|),
                  focal_change_pct, principal_point_px;
  rgb_before.png / rgb_after.png   the frame rendered at the starting / registered camera and codes;
  summary.json    the full-frame PSNR before and after, and the final pose change.
Every refusal (unknown item, --optimize entry or --intrinsics part, a group the model cannot fit, an image of the wrong size,
steps or batch_rays below 1) comes before any GPU work.  One process, one GPU.
"""
import json
import pathlib
import sys

import numpy as np

from nerfies_b200 import camera as camera_lib
from nerfies_b200 import checkpoints
from nerfies_b200 import configs
from nerfies_b200 import datasets
from nerfies_b200 import driver_utils
from nerfies_b200 import eval as eval_lib
from nerfies_b200 import geometry
from nerfies_b200 import model_utils
from nerfies_b200 import models
from nerfies_b200 import render_video


def original_scale_camera(datasource, camera, template):
  """`camera` (the experiment's scale, centred and scaled into the scene) at the capture's original scale:
  load_camera undone, with `template`'s (the unscaled JSON's) intrinsics and image size."""
  out = template.copy()
  out.orientation = camera.orientation.copy()
  position = camera.position.astype(np.float64) / datasource.scene_scale + datasource.scene_center
  out.position = position.astype(np.float32)
  return out


def check_inputs(datasource, model_config, item=None, image=None, init_camera=None, optimize=('pose',), steps=1,
                 batch_rays=1, metadata=(), intrinsics=()):
  """Refuses what cannot be registered, before any GPU work: raises ValueError.  Returns (name, target rgb
  uint8 (h, w, 3) on the host, starting camera, its unscaled template, metadata)."""
  if (item is None) == (image is None):
    raise ValueError('pass one of --item (a capture item) and --image (a PNG)')
  optimize = geometry.check_registration(model_config, optimize, steps, batch_rays, intrinsics)
  if item is not None:
    if item not in set(datasource.all_ids):
      raise ValueError(f"unknown item {item!r}: not among the capture's train and val items")
    rgb = datasets.decode_image(datasource.get_rgb_path(item))
    md = datasource._item_metadata(item)
    name = str(item)
  else:
    rgb = datasets.decode_image(image)
    md = {}
    name = pathlib.Path(image).stem
  md = dict(render_video.default_metadata(datasource), **md)
  given = render_video.default_metadata(datasource, metadata)
  md.update({k: given[k] for k in (m.partition('=')[0] for m in metadata)})
  if init_camera is not None:
    template = camera_lib.Camera.from_json(init_camera)
    camera = datasource.load_camera(pathlib.Path(init_camera))
  elif item is not None:
    template = camera_lib.Camera.from_json(datasource.camera_dir / f'{item}{datasource.camera_ext}')
    camera = datasource.load_camera(item)
  else:
    raise ValueError('--image needs --init_camera (there is no item camera to start from)')
  if tuple(rgb.shape[:2]) != camera.image_shape:
    raise ValueError(f'the target is {rgb.shape[1]} x {rgb.shape[0]} pixels but the camera is '
                     f'{camera.image_shape[1]} x {camera.image_shape[0]}')
  return name, optimize, rgb, camera, template, md


def register(exp_config, model_config, base_folder, data_dir=None, item=None, image=None, init_camera=None,
             optimize=('pose', 'appearance'), steps=200, batch_rays=1024, lrs=None, lr_decay=1.0, seed=0, step=None,
             metadata=(), name=None, precision='fp32', train_precision='fp32', datasource=None, construct_fn=models.construct_nerf,
             log=print, intrinsics=()):
  """Registers the target; returns the output directory."""
  import torch
  dirs = driver_utils.experiment_dirs(base_folder, exp_config.subname)
  if datasource is None:
    datasource = driver_utils.make_datasource(exp_config, model_config, data_dir)
  out_name, optimize, rgb, camera, template, md = check_inputs(
      datasource, model_config, item, image, init_camera, optimize, steps, batch_rays, metadata, intrinsics)
  steps_found = eval_lib.checkpoint_steps(dirs['checkpoints'])
  if step is None:
    if not steps_found:
      raise FileNotFoundError(f'no checkpoints in {dirs["checkpoints"]}')
    step = steps_found[-1]
  elif step not in steps_found:
    raise FileNotFoundError(f'no checkpoint of step {step} in {dirs["checkpoints"]} (steps: {steps_found})')
  model, params = construct_fn(                                                   # as render_video
      0, model_config, batch_size=configs.EvalConfig().chunk, appearance_ids=datasource.appearance_ids,
      camera_ids=datasource.camera_ids, warp_ids=datasource.warp_ids, near=datasource.near,
      far=datasource.far, use_warp_jacobian=False, use_weights=False, precision=precision,
      train_precision=train_precision)
  init_state = model_utils.TrainState(model_utils.Optimizer({'model': params}))
  state = checkpoints.restore_checkpoint(str(dirs['checkpoints']), init_state, step=step, device=model.device)
  params = state.optimizer.target['model']
  extra = state.warp_extra
  target = torch.from_numpy(rgb.astype(np.float32) / np.float32(255.0)).to(model.device)
  codes0 = geometry.registration_codes(model, params, md, extra)
  before = geometry.render_camera(model, params, camera, extra, codes0)
  log(f'Registering {out_name} ({", ".join(tuple(optimize) + tuple(intrinsics))}), {steps} steps of {batch_rays} rays')
  registered, fitted, history = geometry.register_camera(model, params, camera, target, extra, md, optimize=optimize,
                                                         steps=steps, batch_rays=batch_rays, lrs=lrs, seed=seed,
                                                         lr_decay=lr_decay, intrinsics=intrinsics)
  delta = fitted.pop('intrinsics', None)
  codes1 = dict(codes0, **fitted)
  after = geometry.render_camera(model, params, registered, extra, codes1)
  psnr = lambda a: float(-10.0 * torch.log10(((a - target)**2).mean()))
  out_dir = dirs['exp'] / 'registrations' / f'{step:08d}' / (name or out_name)
  out_dir.mkdir(parents=True, exist_ok=True)
  with open(out_dir / 'camera.json', 'w') as f:
    out_camera = original_scale_camera(datasource, registered, template)
    if delta is not None:   # the delta does not depend on the image scale
      out_camera = geometry.refined_camera(out_camera, delta)
    json.dump(out_camera.to_json(), f, indent=2)
  np.savez(out_dir / 'codes.npz', **{k: v.cpu().numpy() for k, v in codes1.items()},
           **({} if delta is None else {'intrinsics': delta.cpu().numpy()}),
           **{f'start_{k}': np.asarray(v) for k, v in md.items()})
  with open(out_dir / 'log.jsonl', 'w') as f:
    for h in history:
      f.write(json.dumps(h) + '\n')
  to_u8 = lambda a: (a.clamp(0, 1) * 255.0 + 0.5).to(torch.uint8).cpu().numpy()
  eval_lib.write_png(out_dir / 'rgb_before.png', to_u8(before))
  eval_lib.write_png(out_dir / 'rgb_after.png', to_u8(after))
  summary = {'psnr_before': psnr(before), 'psnr_after': psnr(after), 'rotation_deg': history[-1]['rotation_deg'],
             'translation': history[-1]['translation'], 'steps': int(steps), 'optimize': list(optimize)}
  if delta is not None:
    q = delta.double().cpu().reshape(8)
    summary.update({'intrinsics': list(intrinsics), 'focal_change_pct': 100.0 * float(np.expm1(float(q[0]))),
                    'principal_point_px': float(camera.focal_length) * float(q[1:3].norm())})
  with open(out_dir / 'summary.json', 'w') as f:
    json.dump(summary, f, indent=2)
  log(f'{out_name}: full-frame PSNR {summary["psnr_before"]:.2f} -> {summary["psnr_after"]:.2f} dB, '
      f'rotation {summary["rotation_deg"]:.4f} deg, translation {summary["translation"]:.5f}')
  return out_dir


def make_parser():
  parser = driver_utils.make_parser('nerfies_b200.register_camera', 'fp32')
  parser.add_argument('--item', default=None, help="a capture item: its rgb at the experiment's scale is the target")
  parser.add_argument('--image', default=None, help="a PNG of the camera's size to register")
  parser.add_argument('--init_camera', default=None, help='the starting camera JSON (default: the item\'s camera)')
  parser.add_argument('--optimize', default='pose,appearance',
                      help='comma-separated groups to fit: pose, appearance, camera, warp')
  parser.add_argument('--intrinsics', default='',
                      help='comma-separated camera intrinsics parts to fit as well: focal, principal_point, radial, '
                      'tangential (default: none)')
  parser.add_argument('--steps', type=int, default=200)
  parser.add_argument('--batch_rays', type=int, default=1024)
  for k, v in geometry.DEFAULT_LRS.items():
    parser.add_argument(f'--lr_{k}', type=float, default=v, help=f'Adam learning rate of the {k} group')
  parser.add_argument('--lr_decay', type=float, default=1.0,
                      help='each learning rate decays exponentially to this fraction of itself at the last step')
  parser.add_argument('--seed', type=int, default=0, help='the pixel batches\' generator seed')
  parser.add_argument('--step', type=int, default=None, help='checkpoint step (default: the newest)')
  parser.add_argument('--metadata', nargs='*', default=(), metavar='KEY=VALUE',
                      help='override the starting metadata ids (or time)')
  parser.add_argument('--name', default=None, help='output directory name (default: the item or image stem)')
  return parser


def main(argv=None):
  args = make_parser().parse_args(argv)
  driver_utils.parse_configs(args.gin_configs, args.gin_bindings)
  exp_config = configs.ExperimentConfig()
  model_config = configs.ModelConfig(use_stratified_sampling=False)
  lrs = {k: getattr(args, f'lr_{k}') for k in geometry.DEFAULT_LRS}
  out = register(exp_config, model_config, args.base_folder, args.data_dir, item=args.item, image=args.image,
                 init_camera=args.init_camera, optimize=[s for s in args.optimize.split(',') if s],
                 intrinsics=[s for s in args.intrinsics.split(',') if s],
                 steps=args.steps, batch_rays=args.batch_rays, lrs=lrs, lr_decay=args.lr_decay, seed=args.seed,
                 step=args.step, metadata=args.metadata, name=args.name, precision=args.precision,
                 train_precision=args.train_precision)
  print(f'Wrote {out}')
  return 0


if __name__ == '__main__':
  sys.exit(main())
