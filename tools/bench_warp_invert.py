"""Warp inversion cost (nfb_warp_invert), beside the per-frame surface extraction it replaces.

  python tools/bench_warp_invert.py [--points 1000000 3500000] [--iters 4 8 16] [--side 256]

Model: bench.py's north-star model (gpu_quarterhd.gin dimensions, SE(3) warp) with
oracle.make_trained_like weights, on a handle of the mesh driver's size (EvalConfig().chunk points
per chunk).  Targets are uniform in [-0.5, 0.5]^3; 3.5 M is about the vertex count of the 256^3
bench mesh.  For each training precision (fp32, tf32x3), point count and max_iters:
geometry.invert_warp of frame 1 from init = NULL, timed with CUDA events around one call after a
warm-up call, and the fraction of points that converged (tol 1e-2 of the 256^3 grid's voxel, as the
driver's --track uses).  Beside them, from the same run: one frame's density grid (fp16x3, fine
level, observation space) and marching cubes at --side^3, which is what a per-frame extraction
costs.

Prints one JSON document with the card's name, power limit and maximum SM clock (read-only query).
"""
import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch  # noqa: E402

from bench import FAR, N_IDS, NEAR, WORKLOADS, model_config  # noqa: E402
from tools.bench_mesh import BOX, _timed  # noqa: E402
from tools.bench_train_precision import _card  # noqa: E402


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--points', type=int, nargs='+', default=[1_000_000, 3_500_000])
  ap.add_argument('--iters', type=int, nargs='+', default=[4, 8, 16])
  ap.add_argument('--side', type=int, default=256)
  args = ap.parse_args()
  import nerfies_b200 as nb
  from nerfies_b200 import _lib, configs, geometry
  from oracle import nerfies_oracle as O
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  wl = WORKLOADS['northstar']
  model, params = nb.construct_nerf(0, model_config(wl), configs.EvalConfig().chunk, range(N_IDS), range(2),
                                    range(N_IDS), NEAR, FAR, precision='fp16x3', device=dev)
  cpu = lambda t: {k: cpu(v) for k, v in t.items()} if isinstance(t, dict) else t.cpu()
  gpu = lambda t: {k: gpu(v) for k, v in t.items()} if isinstance(t, dict) else t.to(dev)
  params = gpu(O.make_trained_like(cpu(params), seed=1))
  extra, md = {'alpha': float(wl['fw']), 'time_alpha': 0.0}, {'warp': 1, 'appearance': 0}
  N = args.side
  voxel = (BOX[1][0] - BOX[0][0]) / (N - 1)
  tol = 1e-2 * voxel
  result = {'card': _card(), 'model': 'north-star (gpu_quarterhd.gin dims)', 'max_rays': model.handle().max_rays,
            'tol': tol, 'invert': []}
  gen = torch.Generator(device=dev).manual_seed(0)
  converged = _lib.INVERT_STATUS['converged']
  for prec in ('fp32', 'tf32x3'):
    model.train_precision = prec
    geometry.invert_warp(model, params, torch.zeros(1024, 3, device=dev), extra, md, max_iters=2, tol=tol)
    for P in args.points:
      y = torch.rand(P, 3, device=dev, generator=gen) - 0.5
      for k in args.iters:
        fn = lambda: geometry.invert_warp(model, params, y, extra, md, max_iters=k, tol=tol)
        fn()
        ms, out = _timed(fn, 1)
        status = out['status']
        row = {'train_precision': prec, 'points': P, 'max_iters': k, 'ms': round(ms, 2),
               'points_per_s': P / ms * 1e3, 'converged_fraction': float((status == converged).float().mean()),
               'status_counts': torch.bincount(status.long(), minlength=5).tolist()}
        result['invert'].append(row)
        print(json.dumps(row), file=sys.stderr)
      del y, out
      torch.cuda.empty_cache()
  shape = (N, N, N)
  grid_fn = lambda: geometry.density_grid(model, params, BOX, shape, extra, md)
  grid_fn()
  grid_ms, grid = _timed(grid_fn, 1)
  level = float(grid.median())
  mc_fn = lambda: geometry.marching_cubes(grid, level, BOX)
  mc_fn()
  mc_ms, (v, f, _) = _timed(mc_fn, 3)
  result['frame_extraction'] = {'side': N, 'density_grid_ms': round(grid_ms, 2), 'marching_cubes_ms': round(mc_ms, 3),
                                'vertices': len(v), 'faces': len(f)}
  print(json.dumps(result, indent=1))


if __name__ == '__main__':
  main()
