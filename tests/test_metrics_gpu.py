"""nfb_image_metrics (MS-SSIM, MSE, depth error of eval.py:process_batch) on the GPU against the
float64 numpy oracle (tests/metrics_oracle.py): |d ms_ssim| <= 1e-5, mse and depth_abs <= 1e-6
relative; the measured maxima are printed."""
import ctypes

import numpy as np
import pytest
import torch

from nerfies_b200 import _lib, evaluation
from tests import metrics_oracle as M

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
SSIM_TOL, REL_TOL = 1e-5, 1e-6
_worst = {'ssim': 0.0, 'mse': 0.0, 'depth': 0.0}


def _smooth(rng, h, w, c):
  yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
  f = rng.uniform(0.005, 0.05, (2, c))
  ph = rng.uniform(0, 6.3, (2, c))
  return (0.5 + 0.2 * np.sin(xx[..., None] * f[0] + ph[0]) * np.cos(yy[..., None] * f[1] + ph[1]))


def _pair(kind, rng, h, w, c):
  """(image, target) float32 of one kind of input."""
  if kind == 'noise':
    x, y = rng.random((h, w, c)), rng.random((h, w, c))
  elif kind == 'smooth':
    y = _smooth(rng, h, w, c)
    x = y + rng.normal(0, 0.03, y.shape)
  elif kind == 'constant':
    x, y = np.full((h, w, c), rng.uniform(0.1, 0.9)), np.full((h, w, c), rng.uniform(0.1, 0.9))
  elif kind == 'identical':
    x = y = _smooth(rng, h, w, c) + rng.normal(0, 0.05, (h, w, c))
  elif kind == 'anti':
    y = rng.random((h, w, c))
    x = 1.0 - y
  return x.astype(np.float32), y.astype(np.float32)


def _depth(rng, n, h, w):
  d = rng.uniform(0.5, 3.0, (n, h, w)).astype(np.float32)
  t = (d + rng.normal(0, 0.1, d.shape)).astype(np.float32)
  t[rng.random(t.shape) < 0.2] = np.nan
  return d, t


def _metrics(x, y, depth=None, depth_target=None):
  """Raw C-ABI call on host arrays; returns host (ms_ssim, mse, depth_abs)."""
  lib = _lib.load()
  n, h, w, c = x.shape
  tx, ty = torch.from_numpy(x).to(DEV), torch.from_numpy(y).to(DEV)
  td = tt = None
  if depth is not None:
    td, tt = torch.from_numpy(depth).to(DEV), torch.from_numpy(depth_target).to(DEV)
  size = lib.nfb_image_metrics_workspace_size(n, h, w, c)
  ws = torch.empty(size, dtype=torch.uint8, device=DEV)
  out = torch.full((3, n), -7.0, device=DEV)
  p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
  _lib.check(lib.nfb_image_metrics(n, h, w, c, p(tx), p(ty), p(td), p(tt), p(ws), size, p(out[0]), p(out[1]),
                                   p(out[2]) if td is not None else None,
                                   ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
  torch.cuda.synchronize()
  return out.cpu().numpy()


CASES = [  # (N, h, w, c, kinds (one per image), depth)
    (1, 161, 161, 3, ['noise'], False),
    (4, 161, 161, 1, ['smooth', 'noise', 'constant', 'anti'], True),
    (1, 177, 181, 3, ['smooth'], True),
    (4, 177, 181, 3, ['noise', 'smooth', 'smooth', 'constant'], False),
    (1, 177, 181, 1, ['noise'], False),
    (1, 270, 480, 3, ['smooth'], True),
    (4, 270, 480, 1, ['smooth', 'noise', 'smooth', 'noise'], True),
    (1, 1080, 1920, 3, ['smooth'], True),
    (1, 200, 200, 3, ['constant'], False),
]


@pytest.mark.parametrize('case', CASES, ids=lambda c: f'{c[0]}x{c[1]}x{c[2]}x{c[3]}-{"-".join(c[4])}')
def test_metrics_match_fp64_oracle(case):
  n, h, w, c, kinds, with_depth = case
  rng = np.random.default_rng(h * 7 + w + c + n)
  pairs = [_pair(k, rng, h, w, c) for k in kinds]
  x, y = np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])
  d = t = None
  if with_depth:
    d, t = _depth(rng, n, h, w)
  got = _metrics(x, y, d, t)
  want_ssim, want_mse = M.ms_ssim(y, x), M.mse(x, y)
  err_ssim = float(np.abs(got[0] - want_ssim).max())
  err_mse = float((np.abs(got[1] - want_mse) / want_mse).max())
  msg = f'ms_ssim {got[0]} vs {want_ssim}'
  print(f'\n{case}: max |d ms_ssim| {err_ssim:.2e}, max rel d mse {err_mse:.2e}', end='')
  _worst['ssim'] = max(_worst['ssim'], err_ssim)
  _worst['mse'] = max(_worst['mse'], err_mse)
  assert err_ssim <= SSIM_TOL, msg
  assert err_mse <= REL_TOL
  for i, k in enumerate(kinds):
    if k == 'anti':
      assert want_ssim[i] == 0.0 and got[0][i] == 0.0
  if with_depth:
    want_d = M.depth_abs(d, t)
    err_d = float((np.abs(got[2] - want_d) / want_d).max())
    print(f', max rel d depth_abs {err_d:.2e}', end='')
    _worst['depth'] = max(_worst['depth'], err_d)
    assert err_d <= REL_TOL
  print(f'  (worst so far: {_worst})', end='')


def test_identical_images_give_exactly_one():
  rng = np.random.default_rng(5)
  x = np.stack([_pair('identical', rng, 177, 181, 3)[0] for _ in range(2)])
  got = _metrics(x, x.copy())
  assert (got[0] == 1.0).all(), got[0]
  assert (got[1] == 0.0).all()


def test_too_small_is_a_loud_error():
  lib = _lib.load()
  for h, w in ((160, 200), (200, 160)):
    a = torch.zeros(1, h, w, 3, device=DEV)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    assert lib.nfb_image_metrics(1, h, w, 3, p(a), p(a), None, None, p(ws), 1 << 20, p(ws), None, None, None) < 0
    assert b'161' in lib.nfb_last_error()
    with pytest.raises(ValueError, match='161'):
      evaluation.compute_multiscale_ssim(a[0], a[0])
    with pytest.raises(ValueError, match='161'):
      evaluation.compute_metrics(a, a)


def test_two_calls_are_bit_identical():
  rng = np.random.default_rng(9)
  x, y = _pair('smooth', rng, 1080, 1920, 3)
  d, t = _depth(rng, 1, 1080, 1920)
  first = _metrics(x[None], y[None], d, t)
  second = _metrics(x[None], y[None], d, t)
  assert first.tobytes() == second.tobytes()


def test_nan_depth_targets():
  rng = np.random.default_rng(11)
  x, y = _pair('smooth', rng, 170, 190, 3)
  d, t = _depth(rng, 2, 170, 190)
  t[1] = np.nan
  got = _metrics(np.stack([x, x]), np.stack([y, y]), d, t)
  assert np.isfinite(got[2][0]) and np.isnan(got[2][1])
  assert abs(got[2][0] - M.depth_abs(d[0], t[0])) <= REL_TOL * M.depth_abs(d[0], t[0])


def test_python_mirror_shapes_and_values():
  rng = np.random.default_rng(13)
  x, y = _pair('smooth', rng, 180, 200, 3)
  gx, gy = torch.from_numpy(x).to(DEV), torch.from_numpy(y).to(DEV)
  s = evaluation.compute_multiscale_ssim(gy, gx)
  assert s.shape == () and s.is_cuda
  assert abs(float(s) - float(M.ms_ssim(y, x))) <= SSIM_TOL
  sb = evaluation.compute_multiscale_ssim(torch.stack([gy, gx]), torch.stack([gx, gx]))
  assert sb.shape == (2,) and float(sb[1]) == 1.0
  with pytest.raises(ValueError, match='no CPU path'):
    evaluation.compute_multiscale_ssim(gx, gy.cpu())


def test_compute_metrics_end_to_end_on_a_rendered_frame():
  """render_frame of a small fp16x3 model on a 176x176 camera, then compute_metrics on the device
  == the oracle on host copies of the same tensors (eval.py:118-140)."""
  import nerfies_b200 as nb
  from oracle import nerfies_oracle as O
  cfg = nb.configs.ModelConfig(use_stratified_sampling=False, use_warp=True, warp_field_type='se3',
                               use_appearance_metadata=True, num_coarse_samples=32, num_fine_samples=32,
                               num_nerf_point_freqs=8, sigma_activation='softplus')
  model, params = nb.construct_nerf(0, cfg, 8192, range(10), [0], range(10), near=0.02, far=0.83,
                                    precision='fp16x3', device=DEV)
  cpu = lambda t: ({k: cpu(v) for k, v in t.items()} if isinstance(t, dict) else t.cpu())
  dev = lambda t: ({k: dev(v) for k, v in t.items()} if isinstance(t, dict) else t.to(DEV))
  params = dev(O.make_trained_like(cpu(params), seed=4))
  R = np.array([[np.cos(0.3), 0, np.sin(0.3)], [0, 1, 0], [-np.sin(0.3), 0, np.cos(0.3)]], np.float32)
  cam = nb.camera.Camera(orientation=R, position=[0.1, -0.05, -0.4], focal_length=150.0,
                         principal_point=[88.0, 88.0], image_size=[176, 176])
  frame = evaluation.render_frame(model, params, cam, {'alpha': 6.5, 'time_alpha': 0.0},
                                  {'warp': 3, 'appearance': 7}, max_rays=8192)
  rng = np.random.default_rng(17)
  target = torch.from_numpy(_smooth(rng, 176, 176, 3).astype(np.float32)).to(DEV)
  depth_target = (frame['med_depth'] + 0.05).unsqueeze(-1).contiguous()
  depth_target[::7, ::5] = float('nan')
  out = evaluation.compute_metrics(frame['rgb'], target, frame['med_depth'], depth_target)
  assert set(out) == {'mse', 'psnr', 'ssim', 'depth_abs'}
  rgb, tgt = frame['rgb'].cpu().numpy(), target.cpu().numpy()
  assert abs(float(out['ssim']) - float(M.ms_ssim(tgt, rgb))) <= SSIM_TOL
  want_mse = float(M.mse(rgb, tgt))
  assert abs(float(out['mse']) - want_mse) <= REL_TOL * want_mse
  assert abs(float(out['psnr']) - (-10 * np.log10(want_mse))) <= 1e-4
  want_d = float(M.depth_abs(frame['med_depth'].cpu().numpy(), depth_target.cpu().numpy()))
  assert abs(float(out['depth_abs']) - want_d) <= REL_TOL * want_d
