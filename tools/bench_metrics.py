"""Times nfb_image_metrics (MS-SSIM + MSE + depth error of eval.py:process_batch) on one and on
eight 1080x1920x3 frames with CUDA events and prints one JSON line.

Algorithmic bytes: both images read once plus the MS-SSIM pyramid (levels 1-4 of both images
written once and read once).  The floor is those bytes over the data-sheet HBM3 bandwidth of the
H100 SXM (3.35 TB/s), a bound, not a measured rate.  The card's name and power limit are read in
the same run."""
import ctypes
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from nerfies_b200 import _lib  # noqa: E402

H, W, C = 1080, 1920, 3
CALLS, WARMUP = 200, 20
DATASHEET_TBPS = 3.35


def _power_limit():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    return float(out.splitlines()[0])
  except Exception:
    return None


def _algorithmic_bytes(n):
  b = 2 * n * H * W * C * 4
  h, w = H, W
  for _ in range(4):
    h, w = (h + 1) // 2, (w + 1) // 2
    b += 2 * 2 * n * h * w * C * 4
  return b


def main():
  if not torch.cuda.is_available():
    raise SystemExit('bench_metrics needs a CUDA device')
  lib = _lib.load()
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
  p = lambda t: ctypes.c_void_p(t.data_ptr())
  gen = torch.Generator(device=dev).manual_seed(0)
  results = {}
  for n in (1, 8):
    target = torch.rand(n, H, W, C, device=dev, generator=gen)
    image = (target + 0.03 * torch.randn(n, H, W, C, device=dev, generator=gen)).clamp_(0, 1)
    depth = torch.rand(n, H, W, device=dev, generator=gen) + 1.0
    depth_t = depth + 0.1 * torch.randn(n, H, W, device=dev, generator=gen)
    size = lib.nfb_image_metrics_workspace_size(n, H, W, C)
    ws = torch.empty(size, dtype=torch.uint8, device=dev)
    out = torch.empty(3, n, device=dev)

    def call():
      _lib.check(lib.nfb_image_metrics(n, H, W, C, p(image), p(target), p(depth), p(depth_t), p(ws), size,
                                       p(out[0]), p(out[1]), p(out[2]), stream))

    for _ in range(WARMUP):
      call()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(CALLS):
      call()
    ev[1].record()
    torch.cuda.synchronize()
    ms = ev[0].elapsed_time(ev[1]) / CALLS
    nbytes = _algorithmic_bytes(n)
    results[f'N{n}'] = {'ms_per_call': round(ms, 4), 'ms_per_frame': round(ms / n, 4),
                        'algorithmic_MB': round(nbytes / 1e6, 2), 'effective_GB_per_s': round(nbytes / ms / 1e6, 1),
                        'datasheet_floor_ms': round(nbytes / (DATASHEET_TBPS * 1e12) * 1e3, 4),
                        'ms_ssim_mean': float(out[0].mean())}
  print(json.dumps({'kernel': 'nfb_image_metrics', 'shape': [H, W, C], 'calls': CALLS,
                    'gpu': torch.cuda.get_device_name(dev), 'power_limit_w': _power_limit(),
                    'results': results}))


if __name__ == '__main__':
  main()
