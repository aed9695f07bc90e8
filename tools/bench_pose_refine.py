"""Times training.train_step with the training cameras' pose refinement off and on, and the two kernels the
refinement adds, then prints one JSON document.

  python tools/bench_pose_refine.py [--runs R] [--warmup W]

For the quarterhd-trainstep and vrig-trainstep workloads (bench.py's model configuration and batch, one GPU,
fp32 training precision, trained-like weights), `off` and `on` steps alternate in one process after W warm-up
steps of each, R of each timed with CUDA events on the current stream.  `on` adds the ray gradients to the
step (nfb_train_value_and_grad_rays), the per-image pose gradient (nfb_pose_grad over 64 images) at the tail
of the flat gradient, and the poses' Adam step.  The batch is the same in both; `on` carries 'image'.
The kernels, each over 200 launches at the workload's batch size: nfb_gather_rays_posed on a 64-image table of
480 x 270 frames (against nfb_gather_rays of the same rays), and nfb_pose_grad.
Reported: median, min and max, and the card's name, power limit and maximum SM clock (nvidia-smi, read-only).
"""
import argparse
import json
import os
import statistics
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.bench_train_precision import _card, _setup  # noqa: E402

NUM_IMAGES = 64


def _stats(xs):
  return {'median': statistics.median(xs), 'min': min(xs), 'max': max(xs)}


def _step(c, poses, ev):
  from nerfies_b200 import training
  c['state'].camera_poses = poses
  ev[0].record()
  training.train_step(c['model'], 0, c['state'], c['batch'], c['sp'], chunk_rays=c['chunk'], **c['kw'])
  ev[1].record()


def _table(dev):
  from nerfies_b200 import camera as camera_lib
  from nerfies_b200 import datasets
  size = (480, 270)
  cams = [camera_lib.Camera(orientation=np.eye(3), position=[0.0, 0.0, -0.45 - 0.001 * k], focal_length=400.0,
                            principal_point=[size[0] / 2, size[1] / 2], image_size=list(size))
          for k in range(NUM_IMAGES)]
  images = [np.zeros((size[1], size[0], 3), np.uint8) for _ in cams]
  order = np.random.default_rng(0).permutation(NUM_IMAGES * size[0] * size[1])
  return datasets.DeviceRayTable(datasets.RayTable(images, cams, {}), dev, order)


def _time(fn, n=200):
  fn()
  e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
  e[0].record()
  for _ in range(n):
    fn()
  e[1].record()
  e[1].synchronize()
  return e[0].elapsed_time(e[1]) / n


def _kernels(B, dev):
  import ctypes
  from nerfies_b200 import _lib
  from nerfies_b200.models import _ptr, _stream
  lib = _lib.load()
  table = _table(dev)
  t = table.table()
  pose = (torch.randn(NUM_IMAGES, 6, device=dev) * 0.01).contiguous()
  o, d = torch.empty(B, 3, device=dev), torch.empty(B, 3, device=dev)
  image = torch.empty(B, dtype=torch.int32, device=dev)
  g_o, g_d = torch.randn(B, 3, device=dev), torch.randn(B, 3, device=dev)
  grad = torch.zeros(NUM_IMAGES, 6, device=dev)
  ws = torch.empty(int(lib.nfb_pose_grad_workspace_size(NUM_IMAGES, B)), dtype=torch.uint8, device=dev)
  plain = lambda: _lib.check(lib.nfb_gather_rays(ctypes.byref(t), 1000, B, _ptr(o), _ptr(d), None, None, None, None,
                                                 None, None, _stream()))
  posed = lambda: _lib.check(lib.nfb_gather_rays_posed(ctypes.byref(t), 1000, B, _ptr(pose), _ptr(o), _ptr(d),
                                                       _ptr(image), _stream()))
  pgrad = lambda: _lib.check(lib.nfb_pose_grad(NUM_IMAGES, _ptr(pose), _ptr(image), _ptr(d), _ptr(g_o), _ptr(g_d), B,
                                               _ptr(grad), _ptr(ws), ws.numel(), _stream()))
  return {'gather_rays_ms': _time(plain), 'gather_rays_posed_ms': _time(posed), 'pose_grad_ms': _time(pgrad)}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--runs', type=int, default=10)
  ap.add_argument('--warmup', type=int, default=2)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_pose_refine needs a CUDA device')
  if args.runs < 3:
    raise SystemExit('--runs must be at least 3')
  from nerfies_b200 import training
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  results = []
  for name in ('quarterhd-trainstep', 'vrig-trainstep'):
    c = _setup(name, 'fp32', dev)
    B = c['B']
    c['batch']['image'] = torch.randint(0, NUM_IMAGES, (B,), generator=torch.Generator().manual_seed(3)).to(
        device=dev, dtype=torch.int32)
    poses = training.CameraPoses([str(k) for k in range(NUM_IMAGES)], dev)
    ms = {'off_ms': [], 'on_ms': []}
    for k in range(args.warmup + args.runs):
      for key, p in (('off_ms', None), ('on_ms', poses)):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        _step(c, p, ev)
        ev[1].synchronize()
        if k >= args.warmup:
          ms[key].append(ev[0].elapsed_time(ev[1]))
    c['state'].camera_poses = None
    res = {'workload': name, 'rays': B, **{k: _stats(v) for k, v in ms.items()},
           'on_over_off': statistics.median(ms['on_ms']) / statistics.median(ms['off_ms']), **_kernels(B, dev)}
    results.append(res)
    print(json.dumps(res), file=sys.stderr)
    del c
    torch.cuda.empty_cache()
  print(json.dumps({'card': _card(), 'runs': args.runs, 'warmup': args.warmup, 'results': results}, indent=1))


if __name__ == '__main__':
  main()
