"""Where the fine level's time goes, and what warping each ray's samples only once can save.

  python tools/bench_fine_warp.py [--points P] [--iters N] [--steps K]

1. Warp only: nfb_warp_forward (the warp MLP and the SE(3) tail of field_wg_kernel, nothing of the NeRF
   MLP) on P free points of bench.py's north-star model, timed with CUDA events over N launches after
   warm-up.  The per-point cost times B * Nc (the coarse samples the fine level would otherwise warp
   again) bounds what reusing the coarse level's warped points can save per step.
2. Per-pass kernel times of one north-star step (model.apply, deterministic path) from torch.profiler,
   averaged over K profiled steps, in launch order.  The kernels after resample_kernel are the fine
   level: the warp-only pass over the new samples, the gather of the warped points and the NeRF pass.

Prints one JSON document with the card's name, power limit and maximum SM clock (read-only query).
"""
import argparse
import json
import os
import statistics
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch  # noqa: E402

from bench import FAR, N_IDS, NEAR, WORKLOADS, model_config, synthetic_rays, trained_like  # noqa: E402
from tools.bench_train_precision import _card  # noqa: E402

WORKLOAD = 'northstar'


def _model(dev, batch, precision):
  import nerfies_b200 as nb
  wl = WORKLOADS[WORKLOAD]
  model, params = nb.construct_nerf(0, model_config(wl), batch, range(N_IDS), range(2), range(N_IDS),
                                    NEAR, FAR, precision=precision, device=dev)
  cpu = lambda t: ({k: cpu(v) for k, v in t.items()} if isinstance(t, dict) else t.cpu())
  gpu = lambda t: ({k: gpu(v) for k, v in t.items()} if isinstance(t, dict) else t.to(dev))
  return model, {'params': gpu(trained_like(cpu(params), seed=1))}


def warp_only(dev, P, iters, precision):
  """Events around N back-to-back nfb_warp_forward launches on P points: ms per launch, ns per point."""
  from nerfies_b200 import _lib
  from nerfies_b200.models import _ptr, _stream
  wl = WORKLOADS[WORKLOAD]
  model, variables = _model(dev, P, precision)
  g = torch.Generator().manual_seed(5)
  pts = (torch.rand(P, 3, generator=g) - 0.5).to(dev)
  ids = torch.randint(0, N_IDS, (P, 1), generator=g, dtype=torch.int32).to(dev)
  extra = {'alpha': float(wl['fw'])}
  wf = model.create_warp_field(model, 1)
  out = wf.apply(variables, pts, ids, extra)['warped_points']          # uploads the parameters
  hd = model.handle(P)
  ids_u = ids.reshape(-1).contiguous()

  def launch():
    _lib.check(hd.lib.nfb_warp_forward(hd.h, P, _ptr(pts), _ptr(ids_u), extra['alpha'], 0, _ptr(out),
                                       _stream()))

  for _ in range(5):
    launch()
  torch.cuda.synchronize()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(iters):
    launch()
  b.record()
  b.synchronize()
  ms = a.elapsed_time(b) / iters
  B, nc = wl['rays'], wl['nc']
  del model, variables, hd
  torch.cuda.empty_cache()
  return {'points': P, 'launches': iters, 'ms_per_launch': ms, 'ns_per_point': ms * 1e6 / P,
          'bound_ms_per_step': ms / P * B * nc,
          'bound_note': f'per-point warp cost x B*Nc = {B} x {nc} coarse samples the fine level re-warps'}


def step_profile(dev, steps, precision):
  """torch.profiler kernel times of `steps` north-star forwards, grouped by launch index within a step."""
  from torch.profiler import ProfilerActivity, profile
  wl = WORKLOADS[WORKLOAD]
  B = wl['rays']
  model, variables = _model(dev, B, precision)
  rays_host = synthetic_rays(B, 1000, wl)
  rays = {'origins': rays_host['origins'].to(dev), 'directions': rays_host['directions'].to(dev),
          'metadata': {k: v.to(dev) for k, v in rays_host['metadata'].items()}}
  extra = {'alpha': float(wl['fw']), 'time_alpha': 0.0}
  for _ in range(3):
    model.apply(variables, rays, warp_extra=extra)
  torch.cuda.synchronize()
  launches0 = model.kernel_launches()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(steps):
      model.apply(variables, rays, warp_extra=extra)
    torch.cuda.synchronize()
  per_step = (model.kernel_launches() - launches0) // steps
  ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and not e.name.startswith('Memset') and not e.name.startswith('Memcpy')),
              key=lambda e: e.time_range.start)
  if per_step <= 0 or len(ev) != per_step * steps:
    raise SystemExit(f'expected {per_step} kernels per step, the profile has {len(ev)} for {steps} steps')
  passes = []
  for i in range(per_step):
    ks = ev[i::per_step]
    name = ks[0].name.split('(')[0]
    passes.append({'kernel': name[5:] if name.startswith('void ') else name,
                   'ms': statistics.mean(k.time_range.elapsed_us() for k in ks) / 1e3})
  names = [p['kernel'] for p in passes]
  fine = passes[names.index('nfb::resample_kernel') + 1:] if 'nfb::resample_kernel' in names else []
  return {'rays': B, 'profiled_steps': steps, 'kernels_per_step': per_step, 'passes': passes,
          'fine_level_ms': sum(p['ms'] for p in fine)}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--points', type=int, default=1 << 20)
  ap.add_argument('--iters', type=int, default=50)
  ap.add_argument('--steps', type=int, default=3)
  ap.add_argument('--precision', default='fp16x3', choices=['fp16x3', 'bf16', 'fp32'])
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_fine_warp needs a CUDA device')
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  result = {'card': _card(), 'workload': WORKLOAD, 'precision': args.precision,
            'warp_only': warp_only(dev, args.points, args.iters, args.precision),
            'step': step_profile(dev, args.steps, args.precision)}
  print(json.dumps(result, indent=1))


if __name__ == '__main__':
  main()
