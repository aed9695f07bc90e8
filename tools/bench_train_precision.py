"""Times training.train_step in both training precisions (NerfModel.train_precision 'fp32' and 'tf32x3')
on bench.py's quarterhd-trainstep and vrig-trainstep inputs, and prints one JSON document.

  python tools/bench_train_precision.py [--runs R] [--warmup W] [--workloads quarterhd-trainstep,vrig-trainstep]

The inputs are bench.py's (WORKLOADS, model_config, trained_like, synthetic_rays, the same seeds, chunk
sizes and regularisers as `bench.py --workload ...-trainstep`).  Per workload:
  * value_and_grad_ms: median and range over R steps per mode, the modes alternating step by step in one
    process, after W warm-up steps each (CUDA events, train_step's own timings);
  * kernel time per GEMM role (forward / dX / dW, told apart by the epilogue functor in the kernel name)
    from one more step per mode under torch.profiler, a run of its own;
  * achieved TFLOP/s per role: 2 x the MACs of the photometric loss's GEMMs (bench.py's forward FLOP per
    ray-sample x the ray-samples of both levels, the same for dX and dW) over that role's kernel time.
    The tangent GEMMs of the elastic loss and the background loss's warp GEMMs are timed but not counted,
    so vrig's rates are lower bounds;
  * the largest relative gradient difference between the modes (max |g_tf32x3 - g_fp32| / max |g_fp32| over
    every parameter tensor) at the first step's parameters;
  * the card's name, power limit and maximum SM clock (nvidia-smi, read-only query).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch  # noqa: E402

from bench import FAR, N_IDS, NEAR, WORKLOADS, model_config, synthetic_rays, trained_like  # noqa: E402

MODES = ('fp32', 'tf32x3')
ROLES = {'StoreBiasAct': 'forward', 'StoreMasked': 'forward', 'AccumSplit': 'dX', 'AtomicAdd': 'dW'}


def _card():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader',
                          '-i', '0'], capture_output=True, text=True, timeout=30).stdout.strip()
    name, power, clock = [s.strip() for s in out.splitlines()[0].split(',')]
    return {'name': name, 'power_limit': power, 'max_sm_clock': clock}
  except Exception as e:  # pylint: disable=broad-except
    return {'error': repr(e)}


def _setup(name, mode, dev):
  """bench.py measure_train_step's inputs on one GPU, in training precision `mode`."""
  import nerfies_b200 as nb
  from nerfies_b200 import training
  wl = WORKLOADS[name]
  B = wl['rays']
  model, params = nb.construct_nerf(0, model_config(wl), B, range(N_IDS), range(2), range(N_IDS), NEAR, FAR,
                                    precision='fp32', device=dev, train_precision=mode)
  cpu = lambda t: ({k: cpu(v) for k, v in t.items()} if isinstance(t, dict) else t.cpu())
  gpu = lambda t: ({k: gpu(v) for k, v in t.items()} if isinstance(t, dict) else t.to(dev))
  state = training.create_train_state(model, gpu(trained_like(cpu(params), seed=1)), warp_alpha=float(wl['fw']))
  rays = synthetic_rays(B, 1000, wl)
  g = torch.Generator().manual_seed(77)
  batch = {'origins': rays['origins'].to(dev), 'directions': rays['directions'].to(dev),
           'metadata': {k: v.to(dev) for k, v in rays['metadata'].items()},
           'rgb': torch.rand(B, 3, generator=g).to(dev)}
  sp = training.ScalarParams(learning_rate=1e-3)
  chunk, kw = 1024, {}
  if wl.get('reg'):
    sp = training.ScalarParams(learning_rate=1e-3, elastic_loss_weight=0.001, background_loss_weight=1.0)
    batch['background_points'] = (torch.rand(B, 3, generator=g) * 0.6 - 0.3).to(dev)
    kw = dict(use_elastic_loss=True, elastic_reduce_method='weight', use_background_loss=True)
    chunk = 512
  return dict(wl=wl, B=B, model=model, state=state, batch=batch, sp=sp, chunk=chunk, kw=kw)


def _grads(c):
  """value_and_grad at the current parameters, the regularisers as train_step sets them (fixed draws)."""
  from nerfies_b200 import training
  reg = None
  if c['kw']:
    pts = c['batch']['background_points']
    g = torch.Generator().manual_seed(5)
    reg = training.make_reg(c['model'], c['sp'], True, 'weight', 'log_svals', True, False, background_points=pts,
                            background_warp_ids=torch.randint(0, N_IDS, (pts.shape[0],), generator=g),
                            background_noise=c['sp'].background_noise_std * torch.randn(pts.shape[0], 3, generator=g))
  c['model'].invalidate_params()
  _, grads = training.value_and_grad(c['model'], c['state'].optimizer.target['model'], c['batch'],
                                     c['state'].warp_extra, rngs={'coarse': 0, 'fine': 0}, chunk_rays=c['chunk'],
                                     reg=reg)
  torch.cuda.synchronize()
  return grads


def _grad_diff(cs):
  from nerfies_b200 import training
  ref = training.grads_to_tree(cs['fp32']['model'], _grads(cs['fp32']))
  got = training.grads_to_tree(cs['tf32x3']['model'], _grads(cs['tf32x3']))
  worst, where = 0.0, None

  def walk(r, g, path):
    nonlocal worst, where
    if isinstance(r, dict):
      for k in r:
        walk(r[k], g[k], path + (k,))
      return
    d = float((g.double() - r.double()).abs().max()) / (float(r.double().abs().max()) + 1e-30)
    if d > worst:
      worst, where = d, '/'.join(path)

  walk(ref, got, ())
  return {'max_rel_diff': worst, 'tensor': where}


def _step(c, timings=None):
  from nerfies_b200 import training
  c['state'], stats, _ = training.train_step(c['model'], 0, c['state'], c['batch'], c['sp'], chunk_rays=c['chunk'],
                                             timings=timings, **c['kw'])
  return float(stats['fine']['loss/total'])


def _profile(c):
  """Kernel time (ms) per GEMM role, and of everything else, in one train_step."""
  from torch.profiler import ProfilerActivity, profile
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    _step(c)
    torch.cuda.synchronize()
  out = {'forward': 0.0, 'dX': 0.0, 'dW': 0.0, 'other': 0.0}
  kernels = set()
  for e in prof.events():
    if e.device_type != torch.autograd.DeviceType.CUDA:
      continue
    t = e.device_time_total / 1e3
    role = 'other'
    if 'gemm' in e.name:
      kernels.add(e.name.split('<')[0].split()[-1])
      role = next((r for f, r in ROLES.items() if f in e.name), 'other')
    out[role] += t
  return {k: round(v, 3) for k, v in out.items()}, sorted(kernels)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--runs', type=int, default=5)
  ap.add_argument('--warmup', type=int, default=2)
  ap.add_argument('--workloads', default='quarterhd-trainstep,vrig-trainstep')
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_train_precision needs a CUDA device')
  if args.runs < 3:
    raise SystemExit('--runs must be at least 3')
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  result = {'card': _card(), 'runs': args.runs, 'warmup': args.warmup, 'workloads': {}}
  for name in args.workloads.split(','):
    cs = {m: _setup(name, m, dev) for m in MODES}
    res = {'grad_diff_first_step': _grad_diff(cs)}
    for m in MODES:
      for _ in range(args.warmup):
        _step(cs[m])
    torch.cuda.synchronize()
    ms = {m: [] for m in MODES}
    loss = {m: [] for m in MODES}
    for _ in range(args.runs):
      for m in MODES:
        t = {}
        loss[m].append(_step(cs[m], timings=t))
        ms[m].append(t['value_and_grad_ms'])
    c = cs['fp32']
    rows = c['B'] * (2 * c['wl']['nc'] + c['wl']['nf'])          # ray-samples of both levels
    flop = rows * c['wl']['flop']                                  # per role: forward, dX, dW
    for m in MODES:
      roles, kernels = _profile(cs[m])
      res[m] = {
          'value_and_grad_ms': {'median': statistics.median(ms[m]), 'min': min(ms[m]), 'max': max(ms[m]),
                                'all': [round(x, 2) for x in ms[m]]},
          'gemm_kernel_ms': roles, 'gemm_kernels': kernels,
          'tflops_photometric': {r: round(flop / (roles[r] * 1e-3) / 1e12, 1) if roles[r] else None
                                 for r in ('forward', 'dX', 'dW')},
          'loss_first_last': [loss[m][0], loss[m][-1]],
      }
    res['speedup_median'] = res['fp32']['value_and_grad_ms']['median'] / res['tf32x3']['value_and_grad_ms']['median']
    res['ranges_apart'] = res['tf32x3']['value_and_grad_ms']['max'] < res['fp32']['value_and_grad_ms']['min']
    res['gemm_flop_per_role'] = flop
    result['workloads'][name] = res
    del cs
    torch.cuda.empty_cache()
  print(json.dumps(result, indent=1))


if __name__ == '__main__':
  main()
