"""Times capture processing on the GPU against the notebook's host code.

  python tools/bench_capture.py [--frames 40] [--cameras 800] [--points 200000]

1. pyramid (1,2,4,8) and blur score of one 1080p frame already on the device (CUDA events over
   many launches), against cv2.resize and cvtColor + Laplacian + var on the host;
2. near/far for C cameras x P points (one nfb_near_far call, device-synchronised), against the
   notebook's numpy loop over the cameras;
3. a capture's frames through `images` and the blur scores of `scene`, split into PNG decode (host
   threads), device work (upload, kernels, download) and PNG encode (one worker thread).
Prints one JSON line.  Needs a CUDA device.
"""
import argparse
import concurrent.futures
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nerfies_b200 import camera as camera_lib  # noqa: E402
from nerfies_b200 import capture  # noqa: E402
from nerfies_b200 import datasets  # noqa: E402
from nerfies_b200.eval import write_png  # noqa: E402


def event_ms(fn, reps):
  for _ in range(3):
    fn()
  start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  for _ in range(reps):
    fn()
  end.record()
  torch.cuda.synchronize()
  return start.elapsed_time(end) / reps


def host_ms(fn, reps):
  fn()
  t = time.perf_counter()
  for _ in range(reps):
    fn()
  return (time.perf_counter() - t) * 1e3 / reps


def numpy_near_far(cam, pts):
  local = np.matmul(cam.orientation, (pts - cam.position).T).T
  x, y = local[:, 0] / local[:, 2], local[:, 1] / local[:, 2]
  r2 = x ** 2 + y ** 2
  rd, td = cam.radial_distortion, cam.tangential_distortion
  d = 1.0 + r2 * (rd[0] + r2 * (rd[1] + rd[2] * r2))
  xd = x * d + 2.0 * td[0] * x * y + td[1] * (r2 + 2.0 * x ** 2)
  yd = y * d + 2.0 * td[1] * x * y + td[0] * (r2 + 2.0 * y ** 2)
  px = cam.focal_length * xd + cam.skew * yd + cam.principal_point[0]
  py = cam.focal_length * cam.pixel_aspect_ratio * yd + cam.principal_point[1]
  depths = local[:, 2][(px >= 0) & (px <= cam.image_size_x) & (py >= 0) & (py <= cam.image_size_y)]
  depths = depths[depths > 0]
  return np.quantile(depths, 0.001), np.quantile(depths, 0.999)


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--frames', type=int, default=40)
  p.add_argument('--cameras', type=int, default=800)
  p.add_argument('--points', type=int, default=200_000)
  args = p.parse_args()
  import cv2
  dev = torch.device('cuda', 0)
  props = torch.cuda.get_device_properties(dev)
  out = {'gpu': props.name}
  try:
    import subprocess
    out['power_limit'] = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'],
                                        capture_output=True, text=True).stdout.strip()
  except OSError:
    out['power_limit'] = 'unknown'
  rng = np.random.RandomState(0)

  frame = rng.randint(0, 256, size=(1080, 1920, 3), dtype=np.uint8)
  d = torch.from_numpy(frame).to(dev)
  out['pyramid_1080p_gpu_us'] = 1e3 * event_ms(lambda: capture.downsample_frames(d, [1, 2, 4, 8]), 200)
  out['blur_1080p_gpu_us'] = 1e3 * event_ms(lambda: capture.blur_scores(d[None]), 200)
  out['pyramid_1080p_cv2_us'] = 1e3 * host_ms(
      lambda: [cv2.resize(frame, (1920 // s, 1080 // s), cv2.INTER_AREA) for s in (2, 4, 8)], 20)
  out['blur_1080p_cv2_us'] = 1e3 * host_ms(
      lambda: cv2.Laplacian(cv2.cvtColor(frame, cv2.COLOR_RGB2GRAY), cv2.CV_64F).var(), 20)

  cams = []
  for k in range(args.cameras):
    a = 2 * np.pi * k / args.cameras
    pos = np.array([3 * np.cos(a), 0.2 * np.sin(3 * a), 3 * np.sin(a)])
    z = -pos / np.linalg.norm(pos)
    x = np.cross([0, -1, 0], z)
    x /= np.linalg.norm(x)
    cams.append(camera_lib.Camera(np.stack([x, np.cross(z, x), z]), pos, 1500.0, [960.0, 540.0], [1920, 1080],
                                  radial_distortion=[0.01, -0.02, 0.0], tangential_distortion=[1e-3, -2e-3]))
  pts = rng.normal(size=(args.points, 3)) * 0.8
  capture.near_far_per_camera(cams, pts, dev)
  torch.cuda.synchronize()
  times = []
  for _ in range(5):
    t = time.perf_counter()
    near_i, far_i, counts = capture.near_far_per_camera(cams, pts, dev)
    times.append((time.perf_counter() - t) * 1e3)
  out['near_far_gpu_ms'] = min(times)
  out['near_far_gpu_ms_median'] = float(np.median(times))
  t = time.perf_counter()
  ref = [numpy_near_far(c, pts) for c in cams]
  out['near_far_numpy_ms'] = (time.perf_counter() - t) * 1e3
  out['near_far_max_rel_diff'] = float(max(abs(a - r[0]) / r[0] for a, r in zip(near_i, ref)))

  with tempfile.TemporaryDirectory() as tmp:
    from scipy import ndimage
    base = ndimage.gaussian_filter(rng.uniform(0, 255, size=(1080, 1920, 3)), (3, 3, 0))
    paths = []
    for i in range(args.frames):
      paths.append(os.path.join(tmp, f'{i:06d}.png'))
      cv2.imwrite(paths[-1], np.roll(base, 7 * i, axis=1).astype(np.uint8))
    t0 = time.perf_counter()
    with concurrent.futures.ThreadPoolExecutor() as pool:
      images = list(pool.map(datasets.decode_image, paths))
    t1 = time.perf_counter()
    levels = []
    for im in images:
      lv = capture.downsample_frames(torch.from_numpy(im).to(dev), [1, 2, 4, 8])
      levels.append({s: v.cpu().numpy() for s, v in lv.items()})
    scores = torch.cat([capture.blur_scores(torch.from_numpy(np.stack(images[i:i + 8])).to(dev)).cpu()
                        for i in range(0, len(images), 8)])
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    os.makedirs(os.path.join(tmp, 'out'))
    with concurrent.futures.ThreadPoolExecutor(max_workers=1) as pool:
      list(pool.map(lambda a: write_png(os.path.join(tmp, 'out', f'{a[0]}_{a[1]}.png'), a[2]),
                    [(i, s, v) for i, lv in enumerate(levels) for s, v in lv.items()]))
    t3 = time.perf_counter()
    out.update({'capture_frames': args.frames, 'png_decode_ms': (t1 - t0) * 1e3, 'device_ms': (t2 - t1) * 1e3,
                'png_encode_ms': (t3 - t2) * 1e3, 'blur_scores_finite': bool(torch.isfinite(scores).all())})
  print(json.dumps(out))


if __name__ == '__main__':
  main()
