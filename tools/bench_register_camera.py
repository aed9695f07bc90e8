"""Times one camera-registration step (geometry.register_camera's work per step) at the gin model
dimensions and prints one JSON document.

  python tools/bench_register_camera.py [--runs R] [--warmup W]

For quarterhd and vrig dims (bench.py's model configuration, trained-like weights), R = 1024 and 4096 rays
and both training precisions (fp32, tf32x3), with CUDA events on the current stream, alternating R runs after W
warm-up calls:
  forward_ms:  NerfModel.render_rays of the rays a pose gives (nfb_render_forward, fp32 render kernels);
  backward_ms: loss.backward() of the rgb loss of both levels (nfb_render_ray_vjp: per chunk and level the
               taped forward, then the backward without weight gradients), plus the pose chain;
  step_ms:     the two and the Adam update: one registration step;
  value_and_grad_ms: training.value_and_grad at the same rays (the parameter gradients' backward).
Then one backward under torch.profiler, its device time split into the taped forward (the forward GEMMs,
StoreBiasAct, and the encode / warp tail / raw-to-samples kernels) and the ray backward (everything else).
Reported: median, min and max, and the card's name, power limit and maximum SM clock (nvidia-smi, read-only).
"""
import argparse
import json
import os
import statistics
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch  # noqa: E402

from bench import FAR, N_IDS, NEAR, WORKLOADS, model_config, trained_like  # noqa: E402
from tools.bench_train_precision import _card  # noqa: E402

DIMS = {'quarterhd': 'quarterhd-train', 'vrig': 'vrig-train'}
TAPED_FORWARD = ('StoreBiasAct', 'encode_kernel', 'warp_tail_kernel', 'raw_to_samples_kernel', 'composite_kernel',
                 'ray_cond_kernel')


def _setup(dims, dev):
  import nerfies_b200 as nb
  wl = WORKLOADS[DIMS[dims]]
  cfg = model_config(wl)
  model, p = nb.construct_nerf(0, cfg, 4096, range(N_IDS), range(2), range(N_IDS), NEAR, FAR, precision='fp32',
                               device=dev)
  cpu = lambda t: ({k: cpu(v) for k, v in t.items()} if isinstance(t, dict) else t.cpu())
  gpu = lambda t: ({k: gpu(v) for k, v in t.items()} if isinstance(t, dict) else t.to(dev))
  params = gpu(trained_like(cpu(p), seed=1))
  model.vjp_chunk_rays = 1024
  g = torch.Generator().manual_seed(5)
  d = torch.randn(4096, 3, generator=g)
  local = (d / d.norm(dim=-1, keepdim=True)).to(dev)
  md = {'warp': 1}
  if wl['app']:
    md['appearance'] = 2
  if wl['cam']:
    md['camera'] = 1
  return dict(model=model, params=params, local=local, md=md, target=torch.rand(4096, 3, generator=g).to(dev),
              extra={'alpha': float(wl['fw']), 'time_alpha': 0.0})


def _step_parts(c, R):
  """(rays, loss-closure) for one registration step of R rays, pose and appearance as register_camera does."""
  from nerfies_b200 import geometry
  model, dev = c['model'], c['model'].device
  omega = torch.full((3,), 1e-3, device=dev, requires_grad=True)
  offset = torch.full((3,), 1e-3, device=dev, requires_grad=True)
  codes = {k: v.requires_grad_(k == 'appearance') for k, v in
           geometry.registration_codes(model, c['params'], c['md'], c['extra']).items()}
  opt = torch.optim.Adam([omega, offset] + [v for v in codes.values() if v.requires_grad], lr=1e-3)
  return omega, offset, codes, opt


def _forward(c, R, state):
  from nerfies_b200 import geometry
  omega, offset, codes, _ = state
  model = c['model']
  o, d = geometry.pose_rays(c['local'][:R], torch.eye(3, device=model.device), torch.zeros(3, device=model.device),
                            omega, offset)
  out = model.render_rays({'params': c['params']}, {'origins': o, 'directions': d,
                                                    'metadata': {k: v.expand(R, -1) for k, v in codes.items()}},
                          warp_extra=c['extra'], metadata_encoded=True)
  return geometry.photometric_loss(out, c['target'][:R])


def _run_step(c, R, state, ev=None):
  opt = state[3]
  if ev:
    ev[0].record()
  loss = _forward(c, R, state)
  if ev:
    ev[1].record()
  opt.zero_grad()
  loss.backward()
  if ev:
    ev[2].record()
  opt.step()
  if ev:
    ev[3].record()


def _value_and_grad(c, R):
  from nerfies_b200 import training
  model = c['model']
  batch = {'origins': c['local'][:R] * 0 + 0.01, 'directions': c['local'][:R], 'rgb': c['target'][:R],
           'metadata': {k: torch.full((R, 1), v, dtype=torch.int32, device=model.device) for k, v in c['md'].items()}}
  training.value_and_grad(model, c['params'], batch, c['extra'], chunk_rays=1024)


def _stats(xs):
  return {'median': statistics.median(xs), 'min': min(xs), 'max': max(xs)}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--runs', type=int, default=5)
  ap.add_argument('--warmup', type=int, default=2)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_register_camera needs a CUDA device')
  if args.runs < 3:
    raise SystemExit('--runs must be at least 3')
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  results = []
  for dims in DIMS:
    c = _setup(dims, dev)
    for prec in ('fp32', 'tf32x3'):
      c['model'].train_precision = prec
      for R in (1024, 4096):
        state = _step_parts(c, R)
        for _ in range(args.warmup):
          _run_step(c, R, state)
          _value_and_grad(c, R)
        ms = {'forward_ms': [], 'backward_ms': [], 'step_ms': [], 'value_and_grad_ms': []}
        for _ in range(args.runs):
          ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
          _run_step(c, R, state, ev)
          ev[3].synchronize()
          ms['forward_ms'].append(ev[0].elapsed_time(ev[1]))
          ms['backward_ms'].append(ev[1].elapsed_time(ev[2]))
          ms['step_ms'].append(ev[0].elapsed_time(ev[3]))
          e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
          e[0].record()
          _value_and_grad(c, R)
          e[1].record()
          e[1].synchronize()
          ms['value_and_grad_ms'].append(e[0].elapsed_time(e[1]))
        torch.cuda.synchronize()
        loss = _forward(c, R, state)
        state[3].zero_grad()
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
          loss.backward()
          torch.cuda.synchronize()
        split = {'taped_forward_device_ms': 0.0, 'ray_backward_device_ms': 0.0}
        for e in prof.key_averages():
          if e.device_time_total <= 0:
            continue
          t = e.device_time_total / 1000.0
          if any(k in e.key for k in TAPED_FORWARD):
            split['taped_forward_device_ms'] += t
          else:
            split['ray_backward_device_ms'] += t
        results.append({'dims': dims, 'train_precision': prec, 'rays': R, **{k: _stats(v) for k, v in ms.items()},
                        **{k: round(v, 3) for k, v in split.items()}})
        print(json.dumps(results[-1]), file=sys.stderr)
  print(json.dumps({'card': _card(), 'runs': args.runs, 'warmup': args.warmup, 'results': results}, indent=1))


if __name__ == '__main__':
  main()
