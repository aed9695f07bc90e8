"""Times training.train_step with the depth loss off and on, and nfb_gather_depth, then prints one JSON document.

  python tools/bench_depth_loss.py [--runs R] [--warmup W]

For the quarterhd-trainstep and vrig-trainstep workloads (bench.py's model configuration and batch, one GPU,
fp32 training precision, trained-like weights), `off` and `on` steps alternate in one process after W warm-up
steps of each, R of each timed with CUDA events on the current stream.  The batch is the same in both; `on` adds
use_depth_loss with a depth target on every ray but every seventh (NaN), which costs one count launch for the
batch and one seed launch per level.  nfb_gather_depth is timed over 200 launches at the workload's batch size
on a 64-image table of 480 x 270 frames, against nfb_gather_rays of the same rays.
Reported: median, min and max, and the card's name, power limit and maximum SM clock (nvidia-smi, read-only).
"""
import argparse
import ctypes
import json
import os
import statistics
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.bench_pose_refine import _time  # noqa: E402
from tools.bench_train_precision import _card, _setup  # noqa: E402

NUM_IMAGES = 64


def _stats(xs):
  return {'median': statistics.median(xs), 'min': min(xs), 'max': max(xs)}


def _step(c, on, ev):
  from nerfies_b200 import training
  ev[0].record()
  training.train_step(c['model'], 0, c['state'], c['batch'], c['sp'], chunk_rays=c['chunk'], use_depth_loss=on,
                      **c['kw'])
  ev[1].record()


def _gather(B, dev):
  from nerfies_b200 import _lib
  from nerfies_b200 import camera as camera_lib
  from nerfies_b200 import datasets
  from nerfies_b200.models import _ptr, _stream
  size = (480, 270)
  cams = [camera_lib.Camera(orientation=np.eye(3), position=[0.0, 0.0, -0.45 - 0.001 * k], focal_length=400.0,
                            principal_point=[size[0] / 2, size[1] / 2], image_size=list(size))
          for k in range(NUM_IMAGES)]
  images = [np.zeros((size[1], size[0], 3), np.uint8) for _ in cams]
  depths = [np.full((size[1], size[0]), 1.0, np.float32) for _ in cams]
  order = np.random.default_rng(0).permutation(NUM_IMAGES * size[0] * size[1])
  table = datasets.DeviceRayTable(datasets.RayTable(images, cams, {}, depths), dev, order)
  lib = _lib.load()
  t = table.table()
  o, d, rgb = (torch.empty(B, 3, device=dev) for _ in range(3))
  depth = torch.empty(B, device=dev)
  rays = lambda: _lib.check(lib.nfb_gather_rays(ctypes.byref(t), 1000, B, _ptr(o), _ptr(d), None, _ptr(rgb), None,
                                                None, None, None, _stream()))
  dep = lambda: _lib.check(lib.nfb_gather_depth(ctypes.byref(t), 1000, B, _ptr(depth), _stream()))
  return {'gather_rays_ms': _time(rays), 'gather_depth_ms': _time(dep), 'table_depth_bytes': 4 * table.num_rays}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--runs', type=int, default=10)
  ap.add_argument('--warmup', type=int, default=2)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_depth_loss needs a CUDA device')
  if args.runs < 3:
    raise SystemExit('--runs must be at least 3')
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  results = []
  for name in ('quarterhd-trainstep', 'vrig-trainstep'):
    c = _setup(name, 'fp32', dev)
    B = c['B']
    gen = torch.Generator().manual_seed(5)
    target = 0.2 + 0.6 * torch.rand(B, 1, generator=gen)
    target[::7] = float('nan')
    c['batch']['depth'] = target.to(dev)
    c['sp'].depth_loss_weight = 0.1
    ms = {'off_ms': [], 'on_ms': []}
    for k in range(args.warmup + args.runs):
      for key, on in (('off_ms', False), ('on_ms', True)):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        _step(c, on, ev)
        ev[1].synchronize()
        if k >= args.warmup:
          ms[key].append(ev[0].elapsed_time(ev[1]))
    res = {'workload': name, 'rays': B, **{k: _stats(v) for k, v in ms.items()},
           'on_over_off': statistics.median(ms['on_ms']) / statistics.median(ms['off_ms']), **_gather(B, dev)}
    results.append(res)
    print(json.dumps(res), file=sys.stderr)
    del c
    torch.cuda.empty_cache()
  print(json.dumps({'card': _card(), 'runs': args.runs, 'warmup': args.warmup, 'results': results}, indent=1))


if __name__ == '__main__':
  main()
