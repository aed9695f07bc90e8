"""Surface extraction cost: the density grid and marching cubes, timed separately.

  python tools/bench_mesh.py [--sizes 256 512] [--iters 5] [--precision fp16x3]

Model: bench.py's north-star model (gpu_quarterhd.gin dimensions, SE(3) warp, 128 + 128 samples)
with oracle.make_trained_like weights.  For each cubic grid of side N over [-0.5, 0.5]^3:

1. geometry.density_grid of the fine level in frame 0's observation space (warp + NeRF MLP per
   point), CUDA events around whole calls after one warm-up call: ms and points per second;
2. geometry.marching_cubes of that grid at its median density (a dense surface, so the emit passes
   do real work), CUDA events around --iters calls after warm-up.  Each call includes the host
   synchronisation that reads the counts and the output allocations.  Achieved bytes per second
   count what the passes must move as designed: 72 bytes per grid point (grid read by the classify
   pass; 12 + 4 bytes of flags and counts written; the int64 reduction's read; both scans' reads and
   writes; the vertex and face passes' reads of ids and offsets) plus 24 per vertex (position and
   normal) and 24 per face (its indices written, the three ids read), against HBM3's 3.35 TB/s.

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
from tools.bench_train_precision import _card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
BOX = ((-0.5, -0.5, -0.5), (0.5, 0.5, 0.5))


def mc_bytes(n, V, F):
  return 72 * n + 24 * V + 24 * F


def _timed(fn, iters):
  start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  for _ in range(iters):
    out = fn()
  end.record()
  end.synchronize()
  return start.elapsed_time(end) / iters, out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--sizes', type=int, nargs='+', default=[256, 512])
  ap.add_argument('--iters', type=int, default=5)
  ap.add_argument('--precision', default='fp16x3', choices=['fp32', 'bf16', 'fp16x3'])
  args = ap.parse_args()
  import nerfies_b200 as nb
  from nerfies_b200 import configs, geometry
  from oracle import nerfies_oracle as O
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  wl = WORKLOADS['northstar']
  model, params = nb.construct_nerf(0, model_config(wl), configs.EvalConfig().chunk, range(N_IDS), range(2),
                                    range(N_IDS), NEAR, FAR, precision=args.precision, device=dev)
  cpu = lambda t: {k: cpu(v) for k, v in t.items()} if isinstance(t, dict) else t.cpu()
  gpu = lambda t: {k: gpu(v) for k, v in t.items()} if isinstance(t, dict) else t.to(dev)
  params = gpu(O.make_trained_like(cpu(params), seed=1))
  extra, md = {'alpha': float(wl['fw']), 'time_alpha': 0.0}, {'warp': 0, 'appearance': 0}
  result = {'card': _card(), 'precision': args.precision, 'model': 'north-star (gpu_quarterhd.gin dims)',
            'hbm_bytes_per_s': HBM_BYTES_PER_S, 'sizes': []}
  for N in args.sizes:
    shape = (N, N, N)
    grid_fn = lambda: geometry.density_grid(model, params, BOX, shape, extra, md)
    grid_fn()
    grid_ms, grid = _timed(grid_fn, 1 if N >= 512 else 2)
    level = float(grid.median())
    mc_fn = lambda: geometry.marching_cubes(grid, level, BOX)
    mc_fn()
    mc_ms, (v, f, _) = _timed(mc_fn, args.iters)
    n = N**3
    moved = mc_bytes(n, len(v), len(f))
    row = {'side': N, 'points': n, 'density_grid_ms': round(grid_ms, 2),
           'density_grid_points_per_s': n / grid_ms * 1e3, 'level': level, 'vertices': len(v), 'faces': len(f),
           'marching_cubes_ms': round(mc_ms, 3), 'marching_cubes_bytes': moved,
           'marching_cubes_bytes_per_s': moved / mc_ms * 1e3,
           'marching_cubes_share_of_hbm': moved / mc_ms * 1e3 / HBM_BYTES_PER_S,
           'marching_cubes_share_of_total': mc_ms / (mc_ms + grid_ms)}
    result['sizes'].append(row)
    print(json.dumps(row), file=sys.stderr)
    del grid, v, f
    torch.cuda.empty_cache()
  print(json.dumps(result, indent=1))


if __name__ == '__main__':
  main()
