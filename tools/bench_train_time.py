"""Times what the 'time' warp metadata encoder adds to a training step: training.value_and_grad of bench.py's
vrig-trainstep inputs for the same model with the 'glo' and with the 'time' encoder, in both training
precisions, and prints one JSON document.

  python tools/bench_train_time.py [--runs R] [--warmup W]

Per training precision the two encoders' models live in one process and their steps alternate, after W
warm-up steps each; value_and_grad_ms is train_step's own CUDA-event timing.  The 'time' model is the 'glo'
model with the TimeEncoder (modules.py:297-322, the reference's default of one frequency) in place of the
GLO table, fed metadata['time'] in [0, 1) and time_alpha = 1; its background points' ids are its timestamps.
Reported: the median, min and max of each, the median overhead of 'time' over 'glo', and the card's name,
power limit and maximum SM clock (nvidia-smi, read-only query).
"""
import argparse
import dataclasses
import json
import os
import statistics
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch  # noqa: E402

from bench import FAR, N_IDS, NEAR, WORKLOADS, model_config, synthetic_rays, trained_like  # noqa: E402
from tools.bench_train_precision import _card  # noqa: E402

WORKLOAD = 'vrig-trainstep'
ENCODERS = ('glo', 'time')


def _setup(encoder, prec, dev):
  """bench.py measure_train_step's vrig-trainstep inputs on one GPU, with warp metadata encoder `encoder`."""
  import nerfies_b200 as nb
  from nerfies_b200 import training
  wl = WORKLOADS[WORKLOAD]
  B = wl['rays']
  cfg = dataclasses.replace(model_config(wl), warp_metadata_encoder_type=encoder)
  model, params = nb.construct_nerf(0, cfg, B, range(N_IDS), range(2), range(N_IDS), NEAR, FAR,
                                    precision='fp32', device=dev, train_precision=prec)
  cpu = lambda t: ({k: cpu(v) for k, v in t.items()} if isinstance(t, dict) else t.cpu())
  gpu = lambda t: ({k: gpu(v) for k, v in t.items()} if isinstance(t, dict) else t.to(dev))
  state = training.create_train_state(model, gpu(trained_like(cpu(params), seed=1)), warp_alpha=float(wl['fw']),
                                      time_alpha=1.0)
  rays = synthetic_rays(B, 1000, wl)
  g = torch.Generator().manual_seed(77)
  md = {k: v.to(dev) for k, v in rays['metadata'].items()}
  md['time'] = torch.rand(B, 1, generator=g).to(dev)
  batch = {'origins': rays['origins'].to(dev), 'directions': rays['directions'].to(dev), 'metadata': md,
           'rgb': torch.rand(B, 3, generator=g).to(dev),
           'background_points': (torch.rand(B, 3, generator=g) * 0.6 - 0.3).to(dev)}
  sp = training.ScalarParams(learning_rate=1e-3, elastic_loss_weight=0.001, background_loss_weight=1.0)
  kw = dict(use_elastic_loss=True, elastic_reduce_method='weight', use_background_loss=True)
  return dict(model=model, state=state, batch=batch, sp=sp, kw=kw)


def _step(c, timings):
  from nerfies_b200 import training
  c['state'], _, _ = training.train_step(c['model'], 0, c['state'], c['batch'], c['sp'], chunk_rays=512,
                                         timings=timings, **c['kw'])


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--runs', type=int, default=5)
  ap.add_argument('--warmup', type=int, default=2)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_train_time needs a CUDA device')
  if args.runs < 3:
    raise SystemExit('--runs must be at least 3')
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  result = {'card': _card(), 'workload': WORKLOAD, 'runs': args.runs, 'warmup': args.warmup, 'precisions': {}}
  for prec in ('fp32', 'tf32x3'):
    cs = {e: _setup(e, prec, dev) for e in ENCODERS}
    for e in ENCODERS:
      for _ in range(args.warmup):
        _step(cs[e], {})
    ms = {e: [] for e in ENCODERS}
    for _ in range(args.runs):
      for e in ENCODERS:
        t = {}
        _step(cs[e], t)
        ms[e].append(t['value_and_grad_ms'])
    res = {e: {'value_and_grad_ms': {'median': statistics.median(ms[e]), 'min': min(ms[e]), 'max': max(ms[e]),
                                     'all': [round(x, 2) for x in ms[e]]}} for e in ENCODERS}
    med = {e: res[e]['value_and_grad_ms']['median'] for e in ENCODERS}
    res['time_overhead_pct_median'] = 100.0 * (med['time'] - med['glo']) / med['glo']
    result['precisions'][prec] = res
    del cs
    torch.cuda.empty_cache()
  print(json.dumps(result, indent=1))


if __name__ == '__main__':
  main()
