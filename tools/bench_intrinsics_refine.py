"""Times training.train_step with the training cameras' refinement off, poses only, and poses plus intrinsics, the
kernels the intrinsics refinement adds, and the registration step with and without 'focal'; prints one JSON document.

  python tools/bench_intrinsics_refine.py [--runs R] [--warmup W]

For the quarterhd-trainstep and vrig-trainstep workloads (bench.py's model configuration and batch, one GPU,
fp32 training precision, trained-like weights), `off`, `poses` and `poses_intrinsics` steps alternate in one
process after W warm-up steps of each, R of each timed with CUDA events on the current stream.  `poses` is
bench_pose_refine's `on` (64 images); `poses_intrinsics` adds the intrinsics gradient (nfb_intrinsics_grad over
two groups of 32 images, all four parts) at the tail of the flat gradient and the deltas' Adam step.  The batch
is the same in all three and carries 'image' and 'pixels'.
The kernels, each over 200 launches at the workload's batch size on a 64-image table of 480 x 270 frames:
nfb_gather_rays_posed, nfb_gather_rays_refined (poses and two groups' deltas) and nfb_intrinsics_grad.
The registration step: geometry.register_camera of a 480 x 270 camera with 1024-ray batches, optimize 'pose'
against 'pose' with intrinsics 'focal', (time of 25 steps - time of 5 steps) / 20 on the host clock around synchronised work.
Reported: median, min and max, and the card's name, power limit and maximum SM clock (nvidia-smi, read-only).
"""
import argparse
import ctypes
import json
import os
import statistics
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.bench_pose_refine import NUM_IMAGES, _table, _time  # noqa: E402
from tools.bench_train_precision import _card, _setup  # noqa: E402

SIZE = (480, 270)


def _stats(xs):
  return {'median': statistics.median(xs), 'min': min(xs), 'max': max(xs)}


def _cameras():
  """bench_pose_refine's table cameras, the second half with another focal length: two intrinsics groups."""
  from nerfies_b200 import camera as camera_lib
  return [camera_lib.Camera(orientation=np.eye(3), position=[0.0, 0.0, -0.45 - 0.001 * k],
                            focal_length=400.0 if k < NUM_IMAGES // 2 else 420.0,
                            principal_point=[SIZE[0] / 2, SIZE[1] / 2], image_size=list(SIZE))
          for k in range(NUM_IMAGES)]


def _step(c, poses, intrinsics, ev):
  from nerfies_b200 import training
  c['state'].camera_poses = poses
  c['state'].camera_intrinsics = intrinsics
  ev[0].record()
  training.train_step(c['model'], 0, c['state'], c['batch'], c['sp'], chunk_rays=c['chunk'], **c['kw'])
  ev[1].record()


def _kernels(B, dev, intrinsics):
  from nerfies_b200 import _lib
  from nerfies_b200.models import _ptr, _stream
  lib = _lib.load()
  table = _table(dev)
  t = table.table()
  pose = (torch.randn(NUM_IMAGES, 6, device=dev) * 0.01).contiguous()
  delta = (torch.randn(2, 8, device=dev) * 1e-3).contiguous()
  o, d = torch.empty(B, 3, device=dev), torch.empty(B, 3, device=dev)
  pixels = torch.empty(B, 2, device=dev)
  image = torch.empty(B, dtype=torch.int32, device=dev)
  g_d = torch.randn(B, 3, device=dev)
  grad = torch.zeros(2, 8, device=dev)
  ws = torch.empty(int(lib.nfb_intrinsics_grad_workspace_size(2, B)), dtype=torch.uint8, device=dev)
  group = intrinsics.group
  posed = lambda: _lib.check(lib.nfb_gather_rays_posed(ctypes.byref(t), 1000, B, _ptr(pose), _ptr(o), _ptr(d),
                                                       _ptr(image), _stream()))
  refined = lambda: _lib.check(lib.nfb_gather_rays_refined(ctypes.byref(t), 1000, B, _ptr(pose), _ptr(delta),
                                                           _ptr(group), 2, _ptr(o), _ptr(d), _ptr(pixels),
                                                           _ptr(image), _stream()))
  igrad = lambda: _lib.check(lib.nfb_intrinsics_grad(_ptr(intrinsics.cameras), NUM_IMAGES, _ptr(pose), _ptr(delta),
                                                     _ptr(group), 2, 15, _ptr(image), _ptr(pixels), _ptr(d),
                                                     _ptr(g_d), B, _ptr(grad), _ptr(ws), ws.numel(), _stream()))
  return {'gather_rays_posed_ms': _time(posed), 'gather_rays_refined_ms': _time(refined),
          'intrinsics_grad_ms': _time(igrad)}


def _registration(c, dev):
  from nerfies_b200 import geometry
  cam = _cameras()[0]
  params = c['state'].optimizer.target['model']
  md = {k: int(v.reshape(-1)[0]) for k, v in c['batch']['metadata'].items()}
  image = torch.rand(SIZE[1], SIZE[0], 3, generator=torch.Generator().manual_seed(4)).to(dev)
  extra = c['state'].warp_extra
  out = {}
  for name, intrinsics in (('pose', ()), ('pose_focal', ('focal',))):
    wall = {}
    for steps in (5, 25, 5, 25):
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      geometry.register_camera(c['model'], params, cam, image, extra, md, optimize=('pose',), intrinsics=intrinsics,
                               steps=steps, batch_rays=1024)
      torch.cuda.synchronize()
      wall[steps] = time.perf_counter() - t0   # the second of each: warmed up
    out[f'register_step_{name}_ms'] = (wall[25] - wall[5]) / 20 * 1e3
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--runs', type=int, default=10)
  ap.add_argument('--warmup', type=int, default=2)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_intrinsics_refine needs a CUDA device')
  if args.runs < 3:
    raise SystemExit('--runs must be at least 3')
  from nerfies_b200 import training
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  results = []
  for name in ('quarterhd-trainstep', 'vrig-trainstep'):
    c = _setup(name, 'fp32', dev)
    B = c['B']
    g = torch.Generator().manual_seed(3)
    c['batch']['image'] = torch.randint(0, NUM_IMAGES, (B,), generator=g).to(device=dev, dtype=torch.int32)
    c['batch']['pixels'] = (torch.rand(B, 2, generator=g) * torch.tensor(SIZE, dtype=torch.float32)).to(dev)
    poses = training.CameraPoses([str(k) for k in range(NUM_IMAGES)], dev)
    intrinsics = training.CameraIntrinsics([str(k) for k in range(NUM_IMAGES)], _cameras(),
                                           ('focal', 'principal_point', 'radial', 'tangential'), dev)
    ms = {'off_ms': [], 'poses_ms': [], 'poses_intrinsics_ms': []}
    for k in range(args.warmup + args.runs):
      for key, p, q in (('off_ms', None, None), ('poses_ms', poses, None), ('poses_intrinsics_ms', poses, intrinsics)):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        _step(c, p, q, ev)
        ev[1].synchronize()
        if k >= args.warmup:
          ms[key].append(ev[0].elapsed_time(ev[1]))
    c['state'].camera_poses = c['state'].camera_intrinsics = None
    med = {k: statistics.median(v) for k, v in ms.items()}
    res = {'workload': name, 'rays': B, **{k: _stats(v) for k, v in ms.items()},
           'poses_over_off': med['poses_ms'] / med['off_ms'],
           'poses_intrinsics_over_poses': med['poses_intrinsics_ms'] / med['poses_ms'],
           **_kernels(B, dev, intrinsics)}
    if name == 'quarterhd-trainstep':
      res.update(_registration(c, dev))
    results.append(res)
    print(json.dumps(res), file=sys.stderr)
    del c
    torch.cuda.empty_cache()
  print(json.dumps({'card': _card(), 'runs': args.runs, 'warmup': args.warmup, 'results': results}, indent=1))


if __name__ == '__main__':
  main()
