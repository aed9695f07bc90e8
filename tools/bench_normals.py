"""Times nfb_density_grad (geometry.density_gradient) and the normal map of a 1080p frame; prints one JSON document.

  python tools/bench_normals.py [--runs R] [--warmup W] [--points P]

For the quarterhd, vrig and fullhd model dimensions (bench.py's model_config and trained-like weights, the
handle's max_rays = 65536), in both training precisions (fp32 and tf32x3): P free points (default 262144) in
the scene's box, warped, at the fine level; W warm-up calls, then R calls timed with CUDA events on the current
stream; points per second from the median.
The 1080p normal map on the fullhd model (fp32 training precision; the frame rendered in fp16x3 as eval.py
renders it): render_frame's time, and the time geometry.normal_map adds at its median depth (only pixels with
a surface are evaluated; their count is reported) and with a surface at every pixel (depth 0.4 everywhere).
Also reported: the card's name, power limit and maximum SM clock (nvidia-smi, read-only).
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

from bench import FAR, N_IDS, NEAR, WORKLOADS, model_config, trained_like  # noqa: E402
from tools.bench_train_precision import _card  # noqa: E402

DIMS = {'quarterhd': 'quarterhd-train', 'vrig': 'vrig-train', 'fullhd': 'fullhd-train'}
MAX_RAYS = 65536


def _model(dims, train_precision, precision, dev):
  import nerfies_b200 as nb
  wl = WORKLOADS[DIMS[dims]]
  model, params = nb.construct_nerf(0, model_config(wl), MAX_RAYS, range(N_IDS), range(2), range(N_IDS), NEAR, FAR,
                                    precision=precision, device=dev, train_precision=train_precision)
  cpu = lambda t: ({k: cpu(v) for k, v in t.items()} if isinstance(t, dict) else t.cpu())
  gpu = lambda t: ({k: gpu(v) for k, v in t.items()} if isinstance(t, dict) else t.to(dev))
  return model, gpu(trained_like(cpu(params), seed=1)), wl


def _metadata(wl):
  md = {'warp': 3}
  if wl['app']:
    md['appearance'] = 5
  if wl['cam']:
    md['camera'] = 1
  return md


def _time(fn, runs, warmup):
  for _ in range(warmup):
    fn()
  ms = []
  for _ in range(runs):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    fn()
    ev[1].record()
    ev[1].synchronize()
    ms.append(ev[0].elapsed_time(ev[1]))
  return {'median': statistics.median(ms), 'min': min(ms), 'max': max(ms)}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--runs', type=int, default=5)
  ap.add_argument('--warmup', type=int, default=2)
  ap.add_argument('--points', type=int, default=262144)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_normals needs a CUDA device')
  from nerfies_b200 import camera as camera_lib
  from nerfies_b200 import evaluation, geometry
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  pts = ((torch.rand(args.points, 3, generator=torch.Generator().manual_seed(0)) - 0.5) * 0.6).to(dev)
  results = []
  for dims in DIMS:
    for mode in ('fp32', 'tf32x3'):
      model, params, wl = _model(dims, mode, 'fp32', dev)
      extra, md = {'alpha': float(wl['fw'])}, _metadata(wl)
      t = _time(lambda: geometry.density_gradient(model, params, pts, extra, md), args.runs, args.warmup)
      res = {'dims': dims, 'train_precision': mode, 'points': args.points, 'ms': t,
             'points_per_s': args.points / (t['median'] * 1e-3)}
      results.append(res)
      print(json.dumps(res), file=sys.stderr)
      del model, params
      torch.cuda.empty_cache()

  model, params, wl = _model('fullhd', 'fp32', 'fp16x3', dev)
  extra, md = {'alpha': float(wl['fw'])}, _metadata(wl)
  cam = camera_lib.Camera(orientation=np.eye(3), position=[0.0, 0.0, -0.45], focal_length=1400.0,
                          principal_point=[960.0, 540.0], image_size=[1920, 1080])
  render = evaluation.render_frame(model, params, cam, extra, md)
  med = render['med_depth']
  frame = {'render_frame_ms': _time(lambda: evaluation.render_frame(model, params, cam, extra, md), args.runs,
                                    args.warmup),
           'surface_pixels': int((med > 0).sum()),
           'normal_map_ms': _time(lambda: geometry.normal_map(model, params, cam, med, extra, md), args.runs,
                                  args.warmup),
           'normal_map_all_pixels_ms': _time(
               lambda: geometry.normal_map(model, params, cam, torch.full_like(med, 0.4), extra, md), args.runs,
               args.warmup)}
  frame['all_pixels_points_per_s'] = 1920 * 1080 / (frame['normal_map_all_pixels_ms']['median'] * 1e-3)
  print(json.dumps({'card': _card(), 'runs': args.runs, 'warmup': args.warmup, 'density_grad': results,
                    'fullhd_1080p': frame}, indent=1))


if __name__ == '__main__':
  main()
