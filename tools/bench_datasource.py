"""Measures the preloaded data path of nerfies_b200.datasets on a synthetic capture and prints one
JSON line.

The capture (seeded, `--items` items of `--width` x `--height`, default 400 x 480x270: the scale of
gpu_quarterhd) is written under `--out`.  Reported: the load time split into decode (PNG decode in a
thread pool, cameras, metadata), permutation (the reference's rng.permutation(num_rays) on the host)
and upload (uint8 rgb, cameras, offsets, metadata and the order, ending in a synchronise); the device
bytes the ray table holds; and the device time per nfb_gather_rays batch at 6144 and 6144 / 8 rays
(every output requested) from CUDA events over `--launches` launches after warm-up, queued in
windows behind a device-side sleep so that host launch overhead is not what is timed.  The card's name
and power limit are read in the same run.

    python tools/bench_datasource.py [--out DIR] [--items 400] [--width 480] [--height 270]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from nerfies_b200 import _lib  # noqa: E402
from nerfies_b200 import datasets  # noqa: E402

WINDOW = 250                 # launches queued behind one sleep
SLEEP_CYCLES = 40_000_000    # ~20 ms at 2 GHz: longer than enqueueing a window


def _power_limit():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    return float(out.splitlines()[0])
  except Exception:
    return None


def write_capture(root, items, width, height, seed=0):
  import cv2
  rng = np.random.RandomState(seed)
  ids = [f'{k:06d}' for k in range(items)]
  for sub in ('camera', 'rgb/1x'):
    os.makedirs(os.path.join(root, sub), exist_ok=True)
  yy, xx = np.mgrid[0:height, 0:width]
  for k, item in enumerate(ids):
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    cam = {'orientation': q.tolist(), 'position': (rng.normal(size=3) * 0.3).tolist(),
           'focal_length': 0.9 * width, 'principal_point': [width / 2, height / 2], 'skew': 0.0,
           'pixel_aspect_ratio': 1.0, 'radial_distortion': [0.05, -0.08, 0.02],
           'tangential_distortion': [1e-3, -5e-4], 'image_size': [width, height]}
    with open(os.path.join(root, 'camera', item + '.json'), 'w') as f:
      json.dump(cam, f)
    base = np.stack([xx * 255 // width, yy * 255 // height, np.full_like(xx, k % 256)], -1)
    image = (base + rng.randint(0, 16, size=base.shape)).clip(0, 255).astype(np.uint8)
    cv2.imwrite(os.path.join(root, 'rgb', '1x', item + '.png'), image)
  with open(os.path.join(root, 'metadata.json'), 'w') as f:
    json.dump({i: {'appearance_id': k, 'camera_id': 0, 'warp_id': k} for k, i in enumerate(ids)}, f)
  with open(os.path.join(root, 'dataset.json'), 'w') as f:
    json.dump({'train_ids': ids, 'val_ids': []}, f)
  with open(os.path.join(root, 'scene.json'), 'w') as f:
    json.dump({'center': [0.0, 0.0, 0.0], 'scale': 1.0, 'near': 0.1, 'far': 2.0}, f)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--out', default=None)
  ap.add_argument('--items', type=int, default=400)
  ap.add_argument('--width', type=int, default=480)
  ap.add_argument('--height', type=int, default=270)
  ap.add_argument('--launches', type=int, default=2000)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_datasource needs a CUDA device')
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  root = os.path.join(args.out or tempfile.mkdtemp(), 'capture')
  write_capture(root, args.items, args.width, args.height)
  ds = datasets.NerfiesDataSource(root, image_scale=1, use_appearance_id=True, use_warp_id=True,
                                  random_seed=0, device=dev)
  torch.zeros(1, device=dev)
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  host = ds.ray_table(ds.train_ids)
  t1 = time.perf_counter()
  order = ds.rng.permutation(host.num_rays)
  t2 = time.perf_counter()
  table = datasets.DeviceRayTable(host, dev, order)
  torch.cuda.synchronize()
  t3 = time.perf_counter()
  lib, t = _lib.load(), table.table()
  stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
  per_batch = {}
  for rays in (6144, 6144 // 8):
    # preallocated outputs, so that the events time the kernel and not the allocator
    out = table.gather(0, rays)
    ptrs = [ctypes.c_void_p(out[k].data_ptr()) for k in ('origins', 'directions', 'pixels', 'rgb')] + [
        ctypes.c_void_p(out['metadata'][k].data_ptr()) if k in out['metadata'] else None
        for k in ('appearance', 'camera', 'warp', 'time')]

    def launch(first):
      _lib.check(lib.nfb_gather_rays(ctypes.byref(t), first, rays, *ptrs, stream))

    first = 0
    for _ in range(50):
      launch(first)
      first += rays
    total_ms = 0.0
    for _ in range(args.launches // WINDOW):
      # A kernel takes less time than its launch from Python: queue a window of launches behind a
      # device-side sleep so that the events time the kernels back to back, not the host.
      torch.cuda.synchronize()
      torch.cuda._sleep(SLEEP_CYCLES)
      ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
      ev[0].record()
      for _ in range(WINDOW):
        launch(first)
        first += rays
      ev[1].record()
      torch.cuda.synchronize()
      total_ms += ev[0].elapsed_time(ev[1])
    per_batch[str(rays)] = round(total_ms / (args.launches // WINDOW * WINDOW) * 1e3, 2)
  print(json.dumps({
      'kernel': 'nfb_gather_rays', 'items': args.items, 'image': [args.height, args.width],
      'num_rays': host.num_rays, 'load_s': {'decode': round(t1 - t0, 3), 'permutation': round(t2 - t1, 3),
                                            'upload': round(t3 - t2, 3)},
      'device_MB': round(table.nbytes() / 1e6, 1), 'order_dtype': str(table.order.dtype),
      'us_per_batch': per_batch, 'launches': args.launches,
      'gpu': torch.cuda.get_device_name(dev), 'power_limit_w': _power_limit()}))


if __name__ == '__main__':
  main()
