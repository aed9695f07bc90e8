"""Times loss.backward() through model.apply against the training step's value_and_grad, on bench.py's
quarterhd-trainstep inputs, and prints one JSON document.

  python tools/bench_render_vjp.py [--runs R] [--warmup W]

Measured, alternating R times after W warm-up calls each, with CUDA events on the current stream:
  value_and_grad: training.value_and_grad (photometric loss, fp32 training GEMMs);
  apply_backward: model.apply of the fp16x3 render kernels with the parameters requiring grad, torch's
    mean((rgb - target)^2) of both levels, and backward() (nfb_render_vjp, fp32 training GEMMs).
Then one call of each under torch.profiler: the device time of composite_vjp_kernel, which seeds both
backwards, and of photometric_loss_kernel, which writes its cotangents in the training step.  Reported: median,
min and max of each, and the card's name, power limit and maximum SM clock (nvidia-smi, read-only query).
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

WORKLOAD = 'quarterhd-trainstep'


def _setup(dev):
  import nerfies_b200 as nb
  wl = WORKLOADS[WORKLOAD]
  B = wl['rays']
  cfg = model_config(wl)
  cpu = lambda t: ({k: cpu(v) for k, v in t.items()} if isinstance(t, dict) else t.cpu())
  gpu = lambda t: ({k: gpu(v) for k, v in t.items()} if isinstance(t, dict) else t.to(dev))
  models, params = {}, None
  for prec in ('fp32', 'fp16x3'):
    models[prec], p = nb.construct_nerf(0, cfg, B, range(N_IDS), range(2), range(N_IDS), NEAR, FAR,
                                        precision=prec, device=dev)
    params = params or gpu(trained_like(cpu(p), seed=1))
  rays = synthetic_rays(B, 1000, wl)
  g = torch.Generator().manual_seed(77)
  batch = {'origins': rays['origins'].to(dev), 'directions': rays['directions'].to(dev),
           'metadata': {k: v.to(dev) for k, v in rays['metadata'].items()},
           'rgb': torch.rand(B, 3, generator=g).to(dev)}
  grad_params = {}

  def leaves(t, out):
    return {k: leaves(v, out) for k, v in t.items()} if isinstance(t, dict) else out.setdefault(
        id(t), t.detach().clone().requires_grad_(True))
  grad_tree = leaves(params, grad_params)
  return dict(models=models, params=params, grad_tree=grad_tree, grad_leaves=list(grad_params.values()),
              batch=batch, warp_extra={'alpha': float(wl['fw']), 'time_alpha': 0.0})


def _value_and_grad(c):
  from nerfies_b200 import training
  training.value_and_grad(c['models']['fp32'], c['params'], c['batch'], c['warp_extra'], chunk_rays=512)


def _apply_backward(c):
  for t in c['grad_leaves']:
    t.grad = None
  model = c['models']['fp16x3']
  model.vjp_chunk_rays = 512
  out = model.apply({'params': c['grad_tree']}, c['batch'], warp_extra=c['warp_extra'])
  tgt = c['batch']['rgb']
  loss = ((out['coarse']['rgb'] - tgt)**2).mean() + ((out['fine']['rgb'] - tgt)**2).mean()
  loss.backward()


def _timed(fn, c):
  ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
  ev[0].record()
  fn(c)
  ev[1].record()
  ev[1].synchronize()
  return ev[0].elapsed_time(ev[1])


def _stats(xs):
  return {'median': statistics.median(xs), 'min': min(xs), 'max': max(xs), 'all': [round(x, 2) for x in xs]}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--runs', type=int, default=5)
  ap.add_argument('--warmup', type=int, default=2)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_render_vjp needs a CUDA device')
  if args.runs < 3:
    raise SystemExit('--runs must be at least 3')
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  c = _setup(dev)
  fns = {'value_and_grad_ms': _value_and_grad, 'apply_backward_ms': _apply_backward}
  for fn in fns.values():
    for _ in range(args.warmup):
      fn(c)
  ms = {k: [] for k in fns}
  for _ in range(args.runs):
    for k, fn in fns.items():
      ms[k].append(_timed(fn, c))
  result = {'card': _card(), 'workload': WORKLOAD, 'rays': WORKLOADS[WORKLOAD]['rays'], 'runs': args.runs,
            'warmup': args.warmup, **{k: _stats(v) for k, v in ms.items()}}
  result['apply_backward_minus_value_and_grad_ms_median'] = (result['apply_backward_ms']['median'] -
                                                             result['value_and_grad_ms']['median'])
  kernels = {}
  for key, fn in fns.items():
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
      fn(c)
      torch.cuda.synchronize()
    for e in prof.key_averages():
      for name in ('composite_vjp_kernel', 'photometric_loss_kernel'):
        if name in e.key:
          k = kernels.setdefault(key, {}).setdefault(name, {'calls': 0, 'device_ms': 0.0})
          k['calls'] += e.count
          k['device_ms'] += e.device_time_total / 1000.0
  result['kernels'] = kernels
  print(json.dumps(result, indent=1))


if __name__ == '__main__':
  main()
