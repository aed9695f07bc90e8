"""Depth supervision on the GPU: sensor depth onto a capture's frames (process_capture depth, nfb_depth_resample)
against the numpy camera on a synthetic plane, the metric-scale estimate, depth batches (nfb_gather_depth), the
depth loss's parameter and ray gradients against fp64 autograd of the oracle, its off path, the drivers and
its effect on a few training steps."""
import ctypes
import os
import shutil

import numpy as np
import pytest
import torch

from nerfies_b200 import _lib
from nerfies_b200 import datasets
from nerfies_b200 import process_capture
from nerfies_b200 import training
from nerfies_b200.models import _ptr, _stream
from oracle import nerfies_oracle as O
from tests import depth_oracle as D
from tests.golden_util import Golden, flatten, model_from_spec, tree_to_device

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAPTURE = os.path.join(ROOT, 'tests', 'golden', 'capture_small')
IDS = ['left_000', 'left_003', 'right_001', 'left_007', 'right_004', 'right_009']
SCENE_SCALE = 0.7           # capture_small/scene.json
METRIC = 2.5                # sensor units -> world units of the synthetic maps
TOL = 2e-4


def _capture_with_sensor(tmp_path, src_hw, holes=True):
  """A copy of capture_small and a directory of synthetic sensor maps of the plane at (h, w) = src_hw."""
  data = tmp_path / 'capture'
  shutil.copytree(CAPTURE, data)
  raw = tmp_path / 'raw'
  raw.mkdir()
  maps = {}
  for k, i in enumerate(IDS):
    m = D.sensor_map(D.load_camera(CAPTURE, i), *src_hw, METRIC).astype(np.float32)
    if holes:   # missing measurements: a block of zeros, NaNs, a negative and an infinite value
      h, w = m.shape
      m[h // 3:h // 3 + max(1, h // 6), w // 4:w // 4 + max(1, w // 5)] = 0.0
      m[k % h, ::7] = np.nan
      m[-1, -1], m[0, -1] = -1.0, np.inf
    np.save(raw / f'{i}.npy', m)
    maps[i] = m
  return data, raw, maps


@pytest.mark.parametrize('src_hw', [(27, 48), (54, 96), (18, 32)], ids=['equal', 'finer_2x', 'coarser_1.5x'])
def test_conversion_matches_the_numpy_camera(tmp_path, src_hw):
  data, raw, maps = _capture_with_sensor(tmp_path, src_hw)
  out = process_capture.run_depth(process_capture.make_parser().parse_args(
      ['depth', '--data_dir', str(data), '--depth_dir', str(raw), '--depth_scale', str(METRIC)]), log=print)
  assert out['metric_scale'] == METRIC and len(out['written']) == len(IDS)
  worst, checked = 0.0, 0
  for i in IDS:
    got = np.load(data / 'depth' / '2x' / f'{i}.npy')
    cam = D.scaled(D.load_camera(CAPTURE, i), 2)
    assert got.dtype == np.float32 and got.shape == (27, 48)
    want = D.resample_rule(cam, maps[i].astype(np.float64), METRIC * SCENE_SCALE)
    assert np.array_equal(np.isnan(got), np.isnan(want)), i
    ok = ~np.isnan(want)
    if ok.any():
      worst = max(worst, float(np.max(np.abs(got[ok] - want[ok]) / want[ok])))
    # every resolution: inside the analytic range of the plane's depth over the widened footprint, converted with
    # the output centre's ray (the conversion is the kernel's own, checked against the camera above)
    lo, hi = D.footprint_z_range(D.load_camera(CAPTURE, i), src_hw, got.shape)
    cos_axis = D.C.camera_to_rays(cam)['directions'].astype(np.float64) @ cam['orientation'][2].astype(np.float64)
    chk = ~np.isnan(got) & ~np.isnan(lo)
    checked += int(chk.sum())
    lo_t, hi_t = lo / cos_axis * SCENE_SCALE, hi / cos_axis * SCENE_SCALE
    assert np.all(got[chk] >= lo_t[chk] * (1 - 1e-5)) and np.all(got[chk] <= hi_t[chk] * (1 + 1e-5)), i
    if src_hw == (27, 48) and float(cam['skew']) == 0.0:
      # the same pixel centres: the analytic ray distance to the plane, scaled into the scene.  Camera.scale keeps
      # the skew, so a skewed camera's 2x frame is not its 1x frame resampled: those cameras are left out here
      t, _ = D.ray_distance(D.load_camera(CAPTURE, i), D.C.get_pixel_centers(cam) * 2)
      assert np.allclose(got[ok], t[ok] * SCENE_SCALE, rtol=2e-5, atol=0), i
  print(f'{src_hw}: worst relative error {worst:.2e}; {checked} pixels inside the analytic range')
  assert worst < 2e-5 and checked > 500
  # right_009 does not see the plane: every pixel stays missing
  assert np.isnan(np.load(data / 'depth' / '2x' / 'right_009.npy')).all()


def test_metric_scale_is_estimated_from_the_points(tmp_path):
  data, raw, _ = _capture_with_sensor(tmp_path, (54, 96), holes=False)
  np.save(data / 'points.npy', D.plane_points(CAPTURE, IDS, 200))
  out = process_capture.run_depth(process_capture.make_parser().parse_args(
      ['depth', '--data_dir', str(data), '--depth_dir', str(raw)]), log=print)
  print(f"metric scale {out['metric_scale']!r} from {out['pairs']} pairs, IQR {out['iqr']:.2e}")
  assert out['pairs'] >= 100
  assert abs(out['metric_scale'] / METRIC - 1) < 1e-4
  # too few pairs: refused, asking for --depth_scale
  np.save(data / 'points.npy', D.plane_points(CAPTURE, IDS, 200)[:5])
  with pytest.raises(ValueError, match='--depth_scale'):
    process_capture.run_depth(process_capture.make_parser().parse_args(
        ['depth', '--data_dir', str(data), '--depth_dir', str(raw)]), log=print)


# ---------------------------------------------------------------------------
# depth batches
# ---------------------------------------------------------------------------
def _host_table(seed=0):
  """Three items of different sizes; the middle one has no depth map."""
  rng = np.random.RandomState(seed)
  cams, images, depths = [], [], []
  from nerfies_b200 import camera as camera_lib
  for k, (w, h) in enumerate(((7, 5), (6, 4), (9, 3))):
    cams.append(camera_lib.Camera(orientation=np.eye(3), position=np.zeros(3), focal_length=10.0,
                                  principal_point=np.array([w / 2, h / 2]), image_size=np.array([w, h])))
    images.append(rng.randint(0, 256, (h, w, 3), dtype=np.uint8))
    d = rng.uniform(0.1, 2.0, (h, w)).astype(np.float32)
    d[0, 0] = np.nan
    depths.append(None if k == 1 else d)
  return datasets.RayTable(images, cams, {}, depths)


def test_gather_depth_follows_the_ray_order():
  host = _host_table()
  n = host.num_rays
  flat = np.concatenate([np.full(h * w, np.nan, np.float32) if d is None else d.reshape(-1)
                         for (h, w), d in zip(host.shapes, host.depths)])
  rgb = np.concatenate([im.reshape(-1, 3) for im in host.images]).astype(np.float32) / np.float32(255)
  order = np.random.RandomState(3).permutation(n)
  table = datasets.DeviceRayTable(host, DEV, order)
  assert table.nbytes() - datasets.DeviceRayTable(datasets.RayTable(host.images, host.cameras, {}), DEV,
                                                  order).nbytes() == 4 * n
  for first, count in ((0, n), (n - 5, 13), (2 * n + 3, 40)):       # the repeat boundary, a second lap
    b = table.gather(first, count)
    idx = order[(first + np.arange(count)) % n]
    assert b['depth'].shape == (count, 1)
    np.testing.assert_array_equal(b['depth'].cpu().numpy()[:, 0], flat[idx])
    np.testing.assert_array_equal(b['rgb'].cpu().numpy(), rgb[idx])     # ray i of both batches is one ray
  # rank 1 of 2 from batch 3 on: the per-rank slice of the reference's batches
  it = datasets._ray_iterator(table, 8, True, 1, 2, first_batch=3)
  for step in range(3, 6):
    b = next(it)
    idx = order[(step * 8 + 4 + np.arange(4)) % n]
    np.testing.assert_array_equal(b['depth'].cpu().numpy()[:, 0], flat[idx])
  # an item: (h, w, 1), NaN where there is no map
  item = table.item(1)
  assert item['depth'].shape == (4, 6, 1) and torch.isnan(item['depth']).all()
  # without depth the batches carry none
  assert 'depth' not in datasets.DeviceRayTable(datasets.RayTable(host.images, host.cameras, {}), DEV).gather(0, 4)


# ---------------------------------------------------------------------------
# the depth loss in the training step
# ---------------------------------------------------------------------------
SP = training.ScalarParams(learning_rate=1e-3, depth_loss_weight=0.7)


def _coarse_only(name):
  g = Golden(name)
  sd = dict(g.spec_dict, num_fine_samples=0)
  spec = O.OracleSpec(**{**sd, 'nerf_skips': tuple(sd['nerf_skips']), 'warp_skips': tuple(sd['warp_skips'])})
  params = {k: v for k, v in g.params.items() if k != 'nerf_mlps_fine'}
  return g, sd, spec, params


def _targets(depth, seed, invalid):
  """Depth targets near the rendered depth (both signs of the error) with `invalid` rays without one."""
  gen = torch.Generator().manual_seed(seed)
  t = depth.detach().double().cpu() + 0.2 * (torch.rand(depth.shape[0], generator=gen, dtype=torch.float64) - 0.5)
  t = t.clamp_min(1e-3).float()
  if invalid == 'all':
    t[:] = float('nan')
    t[::3] = 0.0
  elif invalid:
    t[::4] = float('nan')
    t[1::9] = 0.0
    t[2::11] = -1.0
    t[3::13] = float('inf')
  return t


def _oracle_depth_loss(depth, target):
  ok = torch.isfinite(target) & (target > 0)
  n = int(ok.sum())
  if n == 0:
    return depth.sum() * 0.0
  return (depth[ok] - target[ok].to(depth.dtype)).abs().sum() / n


def _oracle(spec, params, rays, rgb, target, alpha, zc, dtype, ray_grads=False, zf=None, fine_out=None):
  """rgb MSE + weight * L1 depth of the coarse level at the given z and, with `zf`, plus the same terms of the
  fine level at zf (a constant), by autograd in `dtype`.  Returns the coarse level's losses; `fine_out` (a dict)
  receives the fine level's as 'rgb' and 'depth'."""
  p = {k: v.detach().clone().requires_grad_(True) for k, v in flatten(O.tree_to(params, dtype)).items()}
  tree = {}
  for k, v in p.items():
    node = tree
    for part in k.split('/')[:-1]:
      node = node.setdefault(part, {})
    node[k.split('/')[-1]] = v
  r = dict(rays)
  if ray_grads:
    r['origins'] = rays['origins'].to(dtype).clone().requires_grad_(True)
    r['directions'] = rays['directions'].to(dtype).clone().requires_grad_(True)
  out = O.render_level(tree, spec, 'coarse', r, zc, alpha, dtype=dtype)
  rgb_loss = ((out['rgb'] - rgb.to(dtype))**2).mean()
  depth_loss = _oracle_depth_loss(out['depth'], target)
  total = rgb_loss + SP.depth_loss_weight * depth_loss
  if zf is not None:
    fine = O.render_level(tree, spec, 'fine', r, zf, alpha, dtype=dtype)
    fine_rgb, fine_depth = ((fine['rgb'] - rgb.to(dtype))**2).mean(), _oracle_depth_loss(fine['depth'], target)
    total = total + fine_rgb + SP.depth_loss_weight * fine_depth
    if fine_out is not None:
      fine_out.update(rgb=float(fine_rgb), depth=float(fine_depth))
  total.backward()
  grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)).double() for k, v in p.items()}
  rays_g = (r['origins'].grad.double(), r['directions'].grad.double()) if ray_grads else None
  return float(rgb_loss), float(depth_loss), grads, rays_g, out['depth'].detach()


def _gpu(model, params, batch, alpha, g, depth_on=True, weight=None, ray_grads=False, chunk_rays=5):
  sp = training.ScalarParams(learning_rate=1e-3, depth_loss_weight=SP.depth_loss_weight if weight is None else weight)
  reg = training.make_reg(model, sp, use_depth_loss=depth_on, depth_target=batch['depth'] if depth_on else None)
  d = tuple(torch.empty(batch['origins'].shape[0], 3, device=DEV) for _ in range(2)) if ray_grads else None
  loss = torch.zeros(16, device=DEV)
  losses, grads = training.value_and_grad(model, params, batch, {'alpha': alpha}, chunk_rays=chunk_rays,
                                          t_rand=g.t_rand, u_rand=g.u_rand, reg=reg, ray_grads=d)
  torch.cuda.synchronize()
  return losses, grads, d


def _z(spec, params, g):
  with torch.no_grad():
    return O.render_forward(O.tree_to(params, torch.float64), spec, g.rays, warp_alpha=g.warp_alpha,
                            dtype=torch.float64, t_rand=g.t_rand)['coarse']


@pytest.mark.parametrize('name', ['se3_small', 'translation_small', 'nowarp_variants', 'time_small'])
@pytest.mark.parametrize('invalid', [False, True], ids=['all_valid', 'some_invalid'])
def test_depth_loss_gradients_match_fp64_autograd(name, invalid):
  """Coarse-only golden models (no resampling: the GPU and the oracle share every z); each parameter tensor
  within max(2e-4, 3 x the fp32 oracle's distance from fp64) of its largest entry, as the ray-gradient tests."""
  g, sd, spec, params = _coarse_only(name)
  torch.manual_seed(11)
  B = g.rays['origins'].shape[0]
  rgb = torch.rand(B, 3)
  fwd = _z(spec, params, g)
  target = _targets(fwd['depth'], 5, invalid)
  lr, ld, ref, _, _ = _oracle(spec, params, g.rays, rgb, target, g.warp_alpha, fwd['z_vals'], torch.float64)
  _, _, r32, _, _ = _oracle(spec, params, g.rays, rgb, target, g.warp_alpha, fwd['z_vals'], torch.float32)
  model = model_from_spec(sd, device=DEV)
  losses, grads, _ = _gpu(model, tree_to_device(params, DEV), dict(g.rays, rgb=rgb, depth=target[:, None]),
                          g.warp_alpha, g)
  assert abs(float(losses['coarse']) - lr) < 1e-5 * max(1.0, lr)
  assert abs(float(losses['depth_coarse']) - ld) < 1e-5 * max(1.0, ld), (float(losses['depth_coarse']), ld)
  ok = torch.isfinite(target) & (target > 0)
  assert float(losses['depth_count']) == int(ok.sum())
  assert float(losses['depth_fine']) == 0.0           # coarse-only: no fine level
  got = flatten(training.grads_to_tree(model, grads))
  for k, r in ref.items():
    scale = float(r.abs().max()) + 1e-30
    band = float((r32[k] - r).abs().max()) / scale
    err = float((got[k].cpu().double().reshape(r.shape) - r).abs().max()) / scale
    assert err <= max(TOL, 3 * band), (k, err, band)


@pytest.mark.parametrize('name', ['se3_small', 'nowarp_variants'])
def test_depth_loss_gradients_with_a_fine_level(name):
  """Both levels: the fine level on the z_fine the kernels resampled (resampling is a constant; comparing on the
  oracle's own z_fine would measure the conditioning of the inverse CDF).  z_fine comes from the fp32 render of
  the same rays and draws, whose coarse weights are the training step's, so the fine loss the step reports must
  equal the oracle's on it.  Each parameter tensor within max(2e-4, 3 x the fp32 oracle's distance from fp64)."""
  g = Golden(name)
  spec = O.OracleSpec(**{**g.spec_dict, 'nerf_skips': tuple(g.spec_dict['nerf_skips']),
                         'warp_skips': tuple(g.spec_dict['warp_skips'])})
  assert spec.num_fine_samples > 0
  torch.manual_seed(15)
  B = g.rays['origins'].shape[0]
  rgb = torch.rand(B, 3)
  model = model_from_spec(g.spec_dict, device=DEV)
  params = tree_to_device(g.params, DEV)
  kw = {k: None if v is None else torch.as_tensor(v).to(DEV) for k, v in (('t_rand', g.t_rand), ('u_rand', g.u_rand))}
  with torch.no_grad():
    out = model.apply({'params': params}, tree_to_device(g.rays, DEV), warp_extra={'alpha': g.warp_alpha},
                      return_points=True, **kw)
  zc, zf = (out[lv]['z_vals'].detach().cpu().double() for lv in ('coarse', 'fine'))
  target = _targets(out['fine']['depth'].cpu(), 9, True)
  fine = {}
  _, ldc, ref, _, _ = _oracle(spec, g.params, g.rays, rgb, target, g.warp_alpha, zc, torch.float64, zf=zf,
                              fine_out=fine)
  lf, ldf = fine['rgb'], fine['depth']
  _, _, r32, _, _ = _oracle(spec, g.params, g.rays, rgb, target, g.warp_alpha, zc, torch.float32, zf=zf)
  losses, grads, _ = _gpu(model, params, dict(g.rays, rgb=rgb, depth=target[:, None]), g.warp_alpha, g)
  print(f"{name}: fine rgb {float(losses['fine']):.9g} vs {lf:.9g}, fine depth {float(losses['depth_fine']):.9g} vs "
        f"{ldf:.9g}, coarse depth {float(losses['depth_coarse']):.9g} vs {ldc:.9g}")
  assert abs(float(losses['fine']) - lf) < 1e-5 * max(1.0, lf)
  assert abs(float(losses['depth_fine']) - ldf) < 1e-5 * max(1.0, ldf)
  assert abs(float(losses['depth_coarse']) - ldc) < 1e-5 * max(1.0, ldc)
  got = flatten(training.grads_to_tree(model, grads))
  for k, r in ref.items():
    scale = float(r.abs().max()) + 1e-30
    band = float((r32[k] - r).abs().max()) / scale
    err = float((got[k].cpu().double().reshape(r.shape) - r).abs().max()) / scale
    print(f'  {k}: error {err:.2e}, band {band:.2e}')
    assert err <= max(TOL, 3 * band), (k, err, band)


def test_depth_loss_gradients_at_a_gin_size():
  """quarterhd dims (256-wide layers, 128 samples), 40 rays of a coarse-only model, some invalid targets."""
  from tests.test_training_scale_gpu import Case
  from tests.golden_util import spec_to_dict
  c = Case('quarterhd', False, 40, seed=21)
  fwd = O.render_forward(O.tree_to(c.params, torch.float64), c.spec, c.rays, warp_alpha=c.alpha, dtype=torch.float64)
  zc = fwd['coarse']['z_vals'].detach()
  target = _targets(fwd['coarse']['depth'], 6, True)
  lr, ld, ref, _, _ = _oracle(c.spec, c.params, c.rays, c.target, target, c.alpha, zc, torch.float64)
  _, _, r32, _, _ = _oracle(c.spec, c.params, c.rays, c.target, target, c.alpha, zc, torch.float32)
  model = model_from_spec(spec_to_dict(c.spec), device=DEV)
  reg = training.make_reg(model, SP, use_depth_loss=True, depth_target=target)
  losses, grads = training.value_and_grad(model, tree_to_device(c.params, DEV),
                                          dict(c.rays, rgb=c.target, depth=target[:, None]), {'alpha': c.alpha},
                                          chunk_rays=16, reg=reg)
  torch.cuda.synchronize()
  assert abs(float(losses['depth_coarse']) - ld) < 1e-5 * max(1.0, ld)
  got = flatten(training.grads_to_tree(model, grads))
  for k, r in ref.items():
    scale = float(r.abs().max()) + 1e-30
    band = float((r32[k] - r).abs().max()) / scale
    err = float((got[k].cpu().double().reshape(r.shape) - r).abs().max()) / scale
    assert err <= max(TOL, 3 * band), (k, err, band)


@pytest.mark.parametrize('name', ['se3_small', 'nowarp_variants'])
def test_depth_loss_ray_gradients_match_fp64_autograd(name):
  g, sd, spec, params = _coarse_only(name)
  torch.manual_seed(12)
  B = g.rays['origins'].shape[0]
  rgb = torch.rand(B, 3)
  fwd = _z(spec, params, g)
  target = _targets(fwd['depth'], 7, True)
  _, _, _, ref, _ = _oracle(spec, params, g.rays, rgb, target, g.warp_alpha, fwd['z_vals'], torch.float64, True)
  _, _, _, r32, _ = _oracle(spec, params, g.rays, rgb, target, g.warp_alpha, fwd['z_vals'], torch.float32, True)
  model = model_from_spec(sd, device=DEV)
  _, _, (d_o, d_d) = _gpu(model, tree_to_device(params, DEV), dict(g.rays, rgb=rgb, depth=target[:, None]),
                          g.warp_alpha, g, ray_grads=True)
  for got, want, w32, what in ((d_o, ref[0], r32[0], 'origins'), (d_d, ref[1], r32[1], 'directions')):
    scale = float(want.abs().max())
    band = float((w32 - want).abs().max()) / scale
    err = float((got.cpu().double() - want).abs().max()) / scale
    print(f'{name} {what}: error {err:.3e}, band {band:.3e}')
    assert err <= max(TOL, 3 * band), (what, err, band)
  # the depth term reaches the rays: without it they move
  _, _, (o0, d0) = _gpu(model, tree_to_device(params, DEV), dict(g.rays, rgb=rgb, depth=target[:, None]),
                        g.warp_alpha, g, depth_on=False, ray_grads=True)
  assert float((o0 - d_o).abs().max()) > 1e-3 * float(d_o.abs().max())


def _raw_call(model, batch, g, depth_struct):
  """nfb_train_value_and_grad_reg alone (value_and_grad has set the parameters): (launches, loss_out, grads)."""
  hd = model.handle(batch['origins'].shape[0])
  numels = [r * c for _, r, c in hd.param_specs]
  flat = torch.zeros(sum(numels), device=DEV)
  ptrs, off = (ctypes.c_void_p * len(numels))(), 0
  for i, k in enumerate(numels):
    ptrs[i], off = flat.data_ptr() + 4 * off, off + k
  loss = torch.full((16,), -1.0, device=DEV)
  o, d = (batch[k].to(DEV).contiguous() for k in ('origins', 'directions'))
  wid = batch['metadata']['warp'].to(DEV, torch.int32).reshape(-1).contiguous() if model.use_warp else None
  aid = batch['metadata'].get('appearance')
  aid = None if aid is None or not model.use_appearance_metadata else aid.to(DEV, torch.int32).reshape(-1).contiguous()
  tr, ur = (None if x is None else torch.as_tensor(x).to(DEV).float().contiguous() for x in (g.t_rand, g.u_rand))
  with torch.cuda.device(DEV):
    n0 = model.kernel_launches()
    _lib.check(hd.lib.nfb_train_value_and_grad_reg(
        hd.h, o.shape[0], _ptr(o), _ptr(d), None, _ptr(wid), _ptr(aid), None, float(g.warp_alpha), _ptr(tr),
        _ptr(ur), 0, _ptr(batch['rgb'].to(DEV).contiguous()), 5, ctypes.byref(depth_struct), ptrs,
        (ctypes.c_longlong * len(numels))(*numels), len(numels), _ptr(loss), _stream()))
    n = model.kernel_launches() - n0
  torch.cuda.synchronize()
  return n, loss.cpu(), flat.clone()


def test_off_path_and_all_invalid_batch():
  """use_depth_loss = 0 with a depth target: the launches of a call without one, outputs within the spread of
  two plain calls (the dW sums use float atomics) and loss_out[13:16] = 0.  An all-invalid batch: the gradients
  of the depth-off call within that spread, and the depth slots exactly 0."""
  g = Golden('se3_small')
  torch.manual_seed(13)
  B = g.rays['origins'].shape[0]
  model = model_from_spec(g.spec_dict, device=DEV)
  params = tree_to_device(g.params, DEV)
  rgb = torch.rand(B, 3)
  fwd = _z(O.OracleSpec(**{**g.spec_dict, 'nerf_skips': tuple(g.spec_dict['nerf_skips']),
                           'warp_skips': tuple(g.spec_dict['warp_skips'])}), g.params, g)
  batch = dict(g.rays, rgb=rgb, depth=_targets(fwd['depth'], 8, False)[:, None])
  training.value_and_grad(model, params, batch, {'alpha': g.warp_alpha}, chunk_rays=5, t_rand=g.t_rand,
                          u_rand=g.u_rand)       # sets the parameters on the handle
  target = batch['depth'].to(DEV).reshape(-1).contiguous()
  none = _lib.TrainReg()
  off = _lib.TrainReg(depth_loss_weight=0.7, depth_target=target.data_ptr())          # use_depth_loss = 0
  on = _lib.TrainReg(use_depth_loss=1, depth_loss_weight=0.7, depth_target=target.data_ptr())
  invalid = torch.full_like(target, float('nan'))
  invalid[::2] = 0.0
  all_invalid = _lib.TrainReg(use_depth_loss=1, depth_loss_weight=0.7, depth_target=invalid.data_ptr())
  n0, l0, g0 = _raw_call(model, batch, g, none)
  n1, l1, g1 = _raw_call(model, batch, g, none)
  n2, l2, g2 = _raw_call(model, batch, g, off)
  n3, l3, g3 = _raw_call(model, batch, g, on)
  n4, l4, g4 = _raw_call(model, batch, g, all_invalid)
  assert n0 == n1 == n2, (n0, n1, n2)
  fine = g.spec_dict['num_fine_samples'] > 0
  chunks = -(-B // 5)
  # one count launch, one seed launch per level and tape chunk
  assert n3 == n4 == n0 + 1 + (2 if fine else 1) * chunks, (n0, n3, n4)
  spread = float((g0 - g1).abs().max())
  scale = float(g0.abs().max())
  for other in (g2, g4):
    assert float((g0 - other).abs().max()) <= max(4 * spread, 1e-6 * scale), (float((g0 - other).abs().max()), spread)
  assert float((g0 - g3).abs().max()) > 1e-3 * scale         # the depth term moves the gradient
  for l in (l0, l2, l4):
    assert (l[13:16] == 0).all(), l
  assert (l4[:2] - l0[:2]).abs().max() <= max(4 * float((l0[:2] - l1[:2]).abs().max()), 1e-6)
  assert l3[13] > 0 and l3[15] == B and (l3[14] > 0) == fine
  assert torch.isfinite(g4).all()


def test_depth_loss_lowers_the_depth_error():
  """From one seed and the same batch, K steps with the depth loss end with a lower batch depth error than K
  steps without it."""
  from nerfies_b200 import model_utils
  g = Golden('se3_small')
  B = g.rays['origins'].shape[0]
  torch.manual_seed(14)
  rgb = torch.rand(B, 3)
  spec = O.OracleSpec(**{**g.spec_dict, 'nerf_skips': tuple(g.spec_dict['nerf_skips']),
                         'warp_skips': tuple(g.spec_dict['warp_skips'])})
  depth = _z(spec, g.params, g)['depth'].float()
  target = (depth + 0.15).clamp_min(1e-3)[:, None]
  batch = dict(g.rays, rgb=rgb, depth=target)
  errors = {}
  for on in (False, True):
    model = model_from_spec(g.spec_dict, device=DEV)
    state = training.create_train_state(model, tree_to_device(g.params, DEV), warp_alpha=g.warp_alpha)
    sp = training.ScalarParams(learning_rate=3e-3, depth_loss_weight=1.0)
    for _ in range(30):
      state, stats, _ = training.train_step(model, 5, state, batch, sp, use_depth_loss=on)
    measure = training.make_reg(model, training.ScalarParams(learning_rate=0.0), use_depth_loss=True,
                                depth_target=target)
    losses, _ = training.value_and_grad(model, state.optimizer.target['model'], batch, state.warp_extra,
                                        rngs={'coarse': 5, 'fine': 5}, reg=measure)
    errors[on] = float(losses['depth_coarse']) + float(losses['depth_fine'])
    if on:
      assert 'loss/depth' in stats['coarse']
  print(errors)
  assert errors[True] < 0.8 * errors[False], errors


# ---------------------------------------------------------------------------
# the drivers
# ---------------------------------------------------------------------------
@pytest.fixture
def _clean_gin():
  from nerfies_b200 import configs
  configs.clear_config()
  yield
  configs.clear_config()


def test_train_then_eval_with_depth(tmp_path, _clean_gin):
  from nerfies_b200 import driver_utils, eval as eval_lib, train as train_lib
  from tests.test_drivers_gpu import GIN
  data, raw, _ = _capture_with_sensor(tmp_path, (18, 32))
  process_capture.run_depth(process_capture.make_parser().parse_args(
      ['depth', '--data_dir', str(data), '--depth_dir', str(raw), '--depth_scale', str(METRIC)]), log=print)
  gin = tmp_path / 'depth.gin'
  gin.write_text(GIN + "ExperimentConfig.datasource_kwargs = {'use_depth': True}\n"
                 'TrainConfig.use_depth_loss = True\n'
                 "TrainConfig.depth_loss_weight_schedule = ('constant', 0.1)\n"
                 'TrainConfig.max_steps = 30\n')
  base = tmp_path / 'exp'
  argv = ['--base_folder', str(base), '--data_dir', str(data), '--gin_configs', str(gin), '--precision', 'fp32']
  assert train_lib.main(argv) == 0
  records = driver_utils.read_scalars(base / 'summaries' / 'train.jsonl')
  last = records[-1]
  assert last['loss/depth/coarse'] > 0 and last['loss/depth/fine'] > 0
  assert last['params/depth_loss/weight'] == pytest.approx(0.1)
  assert last['loss/total/coarse'] > last['loss/rgb/coarse']
  assert eval_lib.main(argv + ['--eval_once', '--save_viz'], poll_seconds=0.0) == 0
  ev = {}
  for record in driver_utils.read_scalars(base / 'summaries' / 'eval.jsonl'):
    ev.update(record)
  assert np.isfinite(ev['metrics-eval/depth_abs/val']) and np.isfinite(ev['metrics-eval/depth_abs/train'])
  renders = base / 'renders' / '00000030'
  for tag in ('val', 'train'):
    names = set(os.listdir(renders / tag))
    for stem in ('depth_target_viz', 'depth_median_error_viz', 'depth_expected_error_viz'):
      assert any(n.startswith(stem + '_') for n in names), (tag, stem)
  # the depth loss without depth in the data source: refused before step 1
  gin_off = tmp_path / 'nodepth.gin'
  gin_off.write_text(gin.read_text().replace("ExperimentConfig.datasource_kwargs = {'use_depth': True}\n", ''))
  base2 = tmp_path / 'exp2'
  with pytest.raises(ValueError, match='datasource_kwargs'):
    train_lib.main(['--base_folder', str(base2), '--data_dir', str(data), '--gin_configs', str(gin_off),
                    '--precision', 'fp32'])
  assert not (base2 / 'checkpoints').exists() or not os.listdir(base2 / 'checkpoints')
