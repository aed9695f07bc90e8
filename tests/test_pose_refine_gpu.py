"""Training-camera pose refinement on the GPU: the training step's ray gradients (nfb_train_value_and_grad_rays)
against the plain step and against fp64 autograd of the oracle, posed ray batches (nfb_gather_rays_posed), the
per-image pose gradient (nfb_pose_grad) against fp64, recovery of perturbed cameras, and the drivers."""
import ctypes
import os

import numpy as np
import pytest
import torch

from nerfies_b200 import _lib
from nerfies_b200 import camera as camera_lib
from nerfies_b200 import datasets
from nerfies_b200 import geometry
from nerfies_b200 import training
from nerfies_b200.models import _ptr, _stream
from oracle import nerfies_oracle as O
from tests.golden_util import Golden, model_from_spec, tree_to_device

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAPTURE = os.path.join(ROOT, 'tests', 'golden', 'capture_small')
TOL = 2e-4
SP = training.ScalarParams(learning_rate=1e-3, elastic_loss_weight=5.0, warp_reg_loss_weight=3.0,
                           warp_reg_loss_alpha=-2.0, warp_reg_loss_scale=0.05)


def _coarse_only(name):
  """A golden case as a coarse-only model: no resampling, so the GPU and the oracle share every z."""
  g = Golden(name)
  sd = dict(g.spec_dict, num_fine_samples=0)
  spec = O.OracleSpec(**{**sd, 'nerf_skips': tuple(sd['nerf_skips']), 'warp_skips': tuple(sd['warp_skips'])})
  params = {k: v for k, v in g.params.items() if k != 'nerf_mlps_fine'}
  return g, sd, spec, params


def _reg(model, elastic, warp_reg):
  if not (elastic or warp_reg):
    return None
  return training.make_reg(model, SP, use_elastic_loss=elastic, elastic_reduce_method='median',
                           use_warp_reg_loss=warp_reg)


def _gpu(model, params, batch, g, reg, rays, sd=None):
  d = tuple(torch.empty(batch['origins'].shape[0], 3, device=DEV) for _ in range(2)) if rays else None
  losses, grads = training.value_and_grad(model, params, batch, {'alpha': g.warp_alpha}, chunk_rays=5,
                                          t_rand=g.t_rand, u_rand=g.u_rand, reg=reg, ray_grads=d)
  torch.cuda.synchronize()
  return losses, grads, d


@pytest.mark.parametrize('regs', [(False, False), (True, True)], ids=['plain', 'elastic+warp_reg'])
def test_ray_outputs_change_nothing_else(regs):
  """Null ray outputs: the launches of nfb_train_value_and_grad_reg.  With or without them, the losses and
  parameter gradients agree within the spread of two plain calls (the dW sums use float atomics)."""
  g = Golden('se3_small')
  torch.manual_seed(3)
  model = model_from_spec(g.spec_dict, device=DEV)
  params = tree_to_device(g.params, DEV)
  batch = dict(g.rays, rgb=torch.rand(g.rays['origins'].shape[0], 3))
  runs = []
  for rays in (False, False, True):
    runs.append(_gpu(model, params, batch, g, _reg(model, *regs), rays))
  # the launches of the two entries alone (value_and_grad has set the parameters), with null ray outputs and
  # with them
  hd = model.handle(batch['origins'].shape[0])
  reg = _reg(model, *regs)
  numels = [r * c for _, r, c in hd.param_specs]
  flat = torch.zeros(sum(numels), device=DEV)
  ptrs, off = (ctypes.c_void_p * len(numels))(), 0
  for i, k in enumerate(numels):
    ptrs[i], off = flat.data_ptr() + 4 * off, off + k
  loss = torch.zeros(16, device=DEV)
  o, d = (batch[k].to(DEV).contiguous() for k in ('origins', 'directions'))
  wid = batch['metadata']['warp'].to(DEV, torch.int32).reshape(-1).contiguous()
  aid = batch['metadata'].get('appearance')
  aid = None if aid is None or not model.use_appearance_metadata else aid.to(DEV, torch.int32).reshape(-1).contiguous()
  tr, ur = (None if x is None else torch.as_tensor(x).to(DEV).float().contiguous() for x in (g.t_rand, g.u_rand))
  d_o, d_d = torch.empty_like(o), torch.empty_like(d)
  args = (hd.h, o.shape[0], _ptr(o), _ptr(d), None, _ptr(wid), _ptr(aid), None, float(g.warp_alpha), _ptr(tr),
          _ptr(ur), 0, _ptr(batch['rgb'].to(DEV).contiguous()), 5, ctypes.byref(reg[0]) if reg else None, ptrs,
          (ctypes.c_longlong * len(numels))(*numels), len(numels), _ptr(loss))
  counts = []
  with torch.cuda.device(DEV):
    for fn, extra in ((hd.lib.nfb_train_value_and_grad_reg, ()), (hd.lib.nfb_train_value_and_grad_rays, (None, None)),
                      (hd.lib.nfb_train_value_and_grad_rays, (_ptr(d_o), _ptr(d_d)))):
      n0 = model.kernel_launches()
      _lib.check(fn(*args, *extra, _stream()))
      counts.append(model.kernel_launches() - n0)
  torch.cuda.synchronize()
  assert counts[0] == counts[1] < counts[2], counts
  (l0, g0, _), (l1, g1, _), (l2, g2, _) = runs
  spread = float((g0 - g1).abs().max())
  scale = float(g0.abs().max())
  assert float((g0 - g2).abs().max()) <= max(4 * spread, 1e-6 * scale), (float((g0 - g2).abs().max()), spread)
  for k in l0:
    assert abs(float(l0[k]) - float(l2[k])) <= max(4 * abs(float(l0[k]) - float(l1[k])), 1e-6 * abs(float(l0[k]))), k


def _oracle_ray_grads(spec, params, rays, target, zc, warp_alpha, elastic, warp_reg, dtype):
  o = rays['origins'].to(dtype).clone().requires_grad_(True)
  d = rays['directions'].to(dtype).clone().requires_grad_(True)
  r = dict(rays, origins=o, directions=d)
  p = O.tree_to(params, dtype)
  out = O.render_level(p, spec, 'coarse', r, zc, warp_alpha, dtype=dtype)
  loss = ((out['rgb'] - target.to(dtype))**2).mean()
  if warp_reg:
    reg = O.level_regularisers(p, spec, out, r, warp_alpha, use_warp_reg_loss=True,
                               warp_reg_loss_alpha=SP.warp_reg_loss_alpha, warp_reg_loss_scale=SP.warp_reg_loss_scale)
    loss = loss + SP.warp_reg_loss_weight * reg['loss/warp_reg']
  if elastic:
    # the elastic loss's Jacobian at points held constant (stop_gradient)
    held = dict(out, points=out['points'].detach())
    reg = O.level_regularisers(p, spec, held, r, warp_alpha, use_elastic_loss=True, elastic_reduce_method='median')
    loss = loss + SP.elastic_loss_weight * reg['loss/elastic']
  loss.backward()
  return o.grad.double(), d.grad.double()


@pytest.mark.parametrize('name,elastic,warp_reg', [
    ('se3_small', False, False), ('se3_small', True, True), ('se3_small', False, True),
    ('translation_small', True, True), ('time_small', False, False), ('nowarp_variants', False, False),
])
def test_ray_gradients_match_fp64_autograd(name, elastic, warp_reg):
  """Per ray, against torch.autograd in float64 of the oracle at the step's z (coarse-only models); tier A:
  max(2e-4, 3 x the fp32 oracle's distance from fp64) of the largest component."""
  g, sd, spec, params = _coarse_only(name)
  torch.manual_seed(7)
  B = g.rays['origins'].shape[0]
  target = torch.rand(B, 3)
  model = model_from_spec(sd, device=DEV)
  with torch.no_grad():
    zc = O.render_forward(O.tree_to(params, torch.float64), spec, g.rays, warp_alpha=g.warp_alpha,
                          dtype=torch.float64, t_rand=g.t_rand)['coarse']['z_vals']
  _, _, (d_o, d_d) = _gpu(model, tree_to_device(params, DEV), dict(g.rays, rgb=target), g,
                          _reg(model, elastic, warp_reg), True)
  ref = _oracle_ray_grads(spec, params, g.rays, target, zc, g.warp_alpha, elastic, warp_reg, torch.float64)
  r32 = _oracle_ray_grads(spec, params, g.rays, target, zc, g.warp_alpha, elastic, warp_reg, torch.float32)
  for got, want, w32, what in ((d_o, ref[0], r32[0], 'origins'), (d_d, ref[1], r32[1], 'directions')):
    scale = float(want.abs().max())
    band = float((w32 - want).abs().max()) / scale
    err = float((got.cpu().double() - want).abs().max()) / scale
    print(f'{name} {what}: error {err:.3e}, band {band:.3e}')
    assert err <= max(TOL, 3 * band), (what, err, band)


# ---------------------------------------------------------------------------
# a ray table in memory: cameras around a model, the model's renders as the targets
# ---------------------------------------------------------------------------
def _cameras(n, size=(40, 30)):
  cams = []
  for k in range(n):
    a = 2 * np.pi * k / n
    # looking at the origin from 0.45 away, tilted by up to 15 degrees
    R = geometry.rotvec_to_matrix(torch.tensor([0.25 * np.sin(a), 0.25 * np.cos(a), 0.0], dtype=torch.float64)).numpy()
    pos = -R.T @ np.array([0.0, 0.0, 0.45])
    cams.append(camera_lib.Camera(orientation=R, position=pos, focal_length=0.9 * size[0],
                                  principal_point=[size[0] / 2, size[1] / 2], image_size=list(size)))
  return cams


def _setup_scene(seed, n=6):
  from tests.test_render_vjp_gpu import _small_spec
  from tests.golden_util import spec_to_dict
  spec = _small_spec(use_camera_metadata=False, num_appearance_features=8, num_appearance_embeddings=4,
                     num_coarse_samples=64, num_fine_samples=0)
  params = tree_to_device(O.make_trained_like(O.init_params(spec, seed), seed=seed + 1), DEV)
  model = model_from_spec(spec_to_dict(spec), device=DEV, batch_size=2048)
  cams = _cameras(n)
  md = {'warp': np.array([1] * n, np.int32), 'appearance': np.array([2] * n, np.int32)}
  images = []
  for cam in cams:
    rays = camera_lib.camera_to_rays(cam, DEV)
    h, w = cam.image_shape
    meta = {k: torch.full((h * w, 1), int(v[0]), dtype=torch.int32, device=DEV) for k, v in md.items()}
    with torch.no_grad():
      out = model.apply({'params': params}, {'origins': rays['origins'].reshape(-1, 3),
                                             'directions': rays['directions'].reshape(-1, 3), 'metadata': meta},
                        warp_extra={'alpha': 4.0})
    rgb = out['coarse']['rgb'].reshape(h, w, 3).clamp(0, 1)
    images.append((rgb * 255).round().to(torch.uint8).cpu().numpy())
  table = datasets.DeviceRayTable(datasets.RayTable(images, cams, md), DEV)
  return spec, params, model, cams, table


def test_posed_gather():
  _, _, _, cams, table = _setup_scene(300, n=3)
  count, first = 1600, 1000          # the rays of all three 40 x 30 frames
  plain = table.gather(first, count, order=False)
  zero = table.gather(first, count, order=False, poses=torch.zeros(3, 6, device=DEV))
  assert torch.equal(plain['origins'], zero['origins']) and torch.equal(plain['directions'], zero['directions'])
  assert torch.equal(plain['rgb'], zero['rgb']) and torch.equal(plain['pixels'], zero['pixels'])
  rays = torch.arange(first, first + count, dtype=torch.int64)
  want = torch.searchsorted(torch.from_numpy(table.offsets), rays, right=True) - 1
  assert torch.equal(zero['image'].cpu().long(), want)
  gen = torch.Generator().manual_seed(1)
  pose = torch.cat([torch.randn(3, 3, generator=gen) * 0.05, torch.randn(3, 3, generator=gen) * 0.02], 1)
  moved = table.gather(first, count, order=False, poses=pose.to(DEV))
  for k in range(3):
    sel = want == k
    R0 = torch.tensor(cams[k].orientation)
    local = plain['directions'].cpu()[sel] @ R0.T
    o, d = geometry.pose_rays(local, R0, torch.tensor(cams[k].position), pose[k, :3], pose[k, 3:])
    assert float((moved['directions'].cpu()[sel] - d).abs().max()) < 2e-6
    assert float((moved['origins'].cpu()[sel] - o).abs().max()) < 2e-6


def _pose_grad(image, directions, d_o, d_d, pose, n):
  lib = _lib.load()
  ws = torch.empty(int(lib.nfb_pose_grad_workspace_size(n, image.numel())), dtype=torch.uint8, device=DEV)
  out = torch.zeros(n, 6, device=DEV)
  _lib.check(lib.nfb_pose_grad(n, _ptr(pose), _ptr(image), _ptr(directions), _ptr(d_o), _ptr(d_d), image.numel(),
                               _ptr(out), _ptr(ws), ws.numel(), _stream()))
  return out


def test_pose_gradient_matches_fp64_and_is_repeatable():
  """(N,6) pose gradients through pose_rays -> the oracle against the GPU's, tier A; a fourth image without a
  ray gets 0; two calls give the same bits."""
  spec, params, model, cams, table = _setup_scene(310, n=3)
  gen = torch.Generator().manual_seed(2)
  pose = torch.cat([torch.randn(3, 3, generator=gen) * 0.02, torch.randn(3, 3, generator=gen) * 0.01], 1)
  pose4 = torch.cat([pose, torch.zeros(1, 6)]).to(DEV).contiguous()
  B = 600
  batch = table.gather(50, B, order=False, poses=pose4[:3].contiguous())
  plain = table.gather(50, B, order=False)
  batch['rgb'] = torch.rand(B, 3, generator=gen).to(DEV)
  t_rand = torch.rand(B, spec.num_coarse_samples, generator=gen)
  d_o, d_d = torch.empty(B, 3, device=DEV), torch.empty(B, 3, device=DEV)
  p = params
  training.value_and_grad(model, p, batch, {'alpha': 4.0}, chunk_rays=256, t_rand=t_rand, ray_grads=(d_o, d_d))
  got = _pose_grad(batch['image'], batch['directions'], d_o, d_d, pose4, 4)
  again = _pose_grad(batch['image'], batch['directions'], d_o, d_d, pose4, 4)
  torch.cuda.synchronize()
  assert torch.equal(got, again)
  assert torch.equal(got[3], torch.zeros(6, device=DEV))
  img = batch['image'].cpu().long()
  with torch.no_grad():
    zc = O.render_forward(O.tree_to(_flat_cpu(p), torch.float64), spec,
                          {'origins': batch['origins'].cpu(), 'directions': batch['directions'].cpu(),
                           'metadata': {k: v.cpu() for k, v in batch['metadata'].items()}},
                          warp_alpha=4.0, dtype=torch.float64, t_rand=t_rand)['coarse']['z_vals']

  def oracle(dtype):
    w = pose.to(dtype).clone().requires_grad_(True)
    d0 = plain['directions'].cpu().to(dtype)
    o0 = plain['origins'].cpu().to(dtype)
    os_, ds_ = [], []
    for k in range(3):
      R = geometry.rotvec_to_matrix(w[k, :3])
      ds_.append(d0 @ R.T)
      os_.append(o0 + w[k, 3:])
    onehot = torch.nn.functional.one_hot(img, 3).to(dtype)[:, :, None]
    o = (torch.stack(os_, 1) * onehot).sum(1)
    d = (torch.stack(ds_, 1) * onehot).sum(1)
    rays = {'origins': o, 'directions': d, 'metadata': {k: v.cpu() for k, v in batch['metadata'].items()}}
    out = O.render_level(O.tree_to(_flat_cpu(p), dtype), spec, 'coarse', rays, zc, 4.0, dtype=dtype)
    ((out['rgb'] - batch['rgb'].cpu().to(dtype))**2).mean().backward()
    return w.grad.double()

  ref, r32 = oracle(torch.float64), oracle(torch.float32)
  scale = float(ref.abs().max())
  band = float((r32 - ref).abs().max()) / scale
  err = float((got[:3].cpu().double() - ref).abs().max()) / scale
  print(f'pose gradient: error {err:.3e}, band {band:.3e}')
  assert err <= max(TOL, 3 * band), (err, band)


def _flat_cpu(t):
  return {k: _flat_cpu(v) for k, v in t.items()} if isinstance(t, dict) else t.detach().cpu()


def _rotation_error_deg(a, b):
  R = a.orientation.astype(np.float64) @ b.orientation.astype(np.float64).T
  return float(np.degrees(np.arccos(np.clip((np.trace(R) - 1) / 2, -1, 1))))


def test_perturbed_cameras_are_recovered():
  """Six cameras around a trained-like model, targets its renders; each camera perturbed by 1.5 deg and 1.5% of
  the scene; training with the parameters' learning rate at 0 and the poses free."""
  spec, params, model, cams, table = _setup_scene(320)
  n = len(cams)
  rng = np.random.default_rng(5)
  truth = []
  for k in range(n):
    axis, direction = rng.normal(size=3), rng.normal(size=3)
    truth.append(np.concatenate([axis / np.linalg.norm(axis) * np.radians(1.5),
                                 direction / np.linalg.norm(direction) * 0.015 * (spec.far - spec.near) / 0.81]))
  # the table's cameras are the perturbed ones: the pose that undoes the perturbation is the one to find
  perturbed = [geometry.posed_camera(c, torch.tensor(t[:3]), torch.tensor(t[3:])) for c, t in zip(cams, truth)]
  images = [table.rgb[3 * int(table.offsets[k]):3 * int(table.offsets[k + 1])].reshape(*cams[k].image_shape, 3).cpu()
            .numpy() for k in range(n)]
  table = datasets.DeviceRayTable(datasets.RayTable(images, perturbed, {
      'warp': np.array([1] * n, np.int32), 'appearance': np.array([2] * n, np.int32)}), DEV,
      order=np.random.default_rng(6).permutation(int(table.offsets[-1])))
  state = training.create_train_state(model, params, warp_alpha=4.0)
  state.camera_poses = training.CameraPoses([str(k) for k in range(n)], DEV)
  sp = training.ScalarParams(learning_rate=0.0)

  def errors():
    pose = state.camera_poses.pose.detach().cpu().double()
    cams1 = [geometry.posed_camera(c, pose[k, :3], pose[k, 3:]) for k, c in enumerate(perturbed)]
    return ([_rotation_error_deg(c1, c) for c1, c in zip(cams1, cams)],
            [float(np.linalg.norm(c1.position.astype(np.float64) - c.position)) for c1, c in zip(cams1, cams)])

  rot0, pos0 = errors()
  psnr = []
  for step in range(STEPS):
    sp.camera_pose_learning_rate = 3e-3 * 0.05**(step / STEPS)
    batch = table.gather(step * 1024, 1024, poses=state.camera_poses.pose)
    state, stats, _ = training.train_step(model, step, state, batch, sp)
    if step in (0, STEPS - 1):
      psnr.append(float(stats['coarse']['metric/psnr']))
  rot1, pos1 = errors()
  print('rotation (deg):', [f'{a:.3f} -> {b:.4f}' for a, b in zip(rot0, rot1)])
  print('position:', [f'{a:.4f} -> {b:.5f}' for a, b in zip(pos0, pos1)])
  print(f'batch PSNR {psnr[0]:.2f} -> {psnr[1]:.2f} dB')
  # Measured on an H100 80GB HBM3 at 700 W, 400 steps: rotation 1.5 -> at most 0.015 deg, position 0.015 -> at
  # most 5e-5, batch PSNR 34.8 -> 59.0 dB: far inside the 5x asked here.
  assert all(b * 5 <= a for a, b in zip(rot0, rot1)) and all(b * 5 <= a for a, b in zip(pos0, pos1))
  assert psnr[1] > psnr[0]


STEPS = 400


# ---------------------------------------------------------------------------
# the drivers on the small capture
# ---------------------------------------------------------------------------
@pytest.fixture
def _clean_gin():
  from nerfies_b200 import configs
  configs.clear_config()
  yield
  configs.clear_config()


def _gin(tmp_path):
  from tests.test_drivers_gpu import GIN
  path = tmp_path / 'test.gin'
  path.write_text(GIN + 'ModelConfig.use_stratified_sampling = False\nTrainConfig.refine_camera_poses = True\n'
                  "TrainConfig.camera_pose_lr_schedule = ('constant', 0.001)\n")
  return str(path)


def test_drivers_refine_save_resume_and_eval(tmp_path, _clean_gin):
  from nerfies_b200 import checkpoints, driver_utils, eval as eval_lib, train as train_lib
  from tests.test_drivers_gpu import _argv
  gin = _gin(tmp_path)
  bases = {k: tmp_path / k for k in ('whole', 'again', 'resumed')}
  for k in ('whole', 'again'):
    assert train_lib.main(_argv(bases[k], gin)) == 0
  assert train_lib.main(_argv(bases['resumed'], gin, '--max_steps', '30')) == 0
  assert train_lib.main(_argv(bases['resumed'], gin)) == 0
  saved = {k: checkpoints.restore_checkpoint(str(b / 'checkpoints'), device='cpu').camera_poses
           for k, b in bases.items()}
  items = sorted(saved['whole']['items'])
  assert len(items) == 4
  flat = lambda s, key: np.concatenate([np.asarray(s['items'][i][key], np.float64) for i in items])
  for key in ('pose', 'grad_ema', 'grad_sq_ema'):
    noise = np.linalg.norm(flat(saved['whole'], key) - flat(saved['again'], key))
    dist = np.linalg.norm(flat(saved['whole'], key) - flat(saved['resumed'], key))
    print(f'{key}: two uninterrupted runs {noise:.3e}, resumed {dist:.3e}, |x| {np.linalg.norm(flat(saved["whole"], key)):.3e}')
    assert dist <= 10 * noise + 1e-6 * np.linalg.norm(flat(saved['whole'], key)), key
  assert np.linalg.norm(flat(saved['whole'], 'pose')) > 0
  records = driver_utils.read_scalars(bases['whole'] / 'summaries' / 'train.jsonl')
  assert records[-1]['camera_poses/rotation_deg'] > 0 and records[-1]['camera_poses/translation'] > 0
  for step in ('00000030', '00000060'):
    files = sorted(os.listdir(bases['whole'] / 'cameras' / step))
    assert files == [f'{i}.json' for i in items]
  cam = camera_lib.Camera.from_json(bases['whole'] / 'cameras' / '00000060' / f'{items[0]}.json')
  orig = camera_lib.Camera.from_json(os.path.join(CAPTURE, 'camera', f'{items[0]}.json'))
  assert np.array_equal(cam.image_size, orig.image_size)
  assert 0 < float(np.abs(cam.position - orig.position).max()) < 0.1 * float(np.abs(orig.position).max() + 1)
  # flag off on a checkpoint with poses: refused before any GPU work
  with open(gin) as f:
    off = f.read().replace('TrainConfig.refine_camera_poses = True', 'TrainConfig.refine_camera_poses = False')
  (tmp_path / 'off.gin').write_text(off)
  with pytest.raises(ValueError, match='refine_camera_poses is off'):
    train_lib.main(_argv(bases['whole'], str(tmp_path / 'off.gin'), '--max_steps', '61'))
  # eval renders train items from the refined cameras
  lines = []
  assert eval_lib.evaluate(*_eval_configs(gin), str(bases['whole']), CAPTURE, precision='fp32', poll_seconds=0.0,
                           log=lines.append) == [60]
  assert any('refined camera poses' in l for l in lines)
  assert os.listdir(bases['whole'] / 'renders' / '00000060' / 'train')


def _eval_configs(gin):
  from nerfies_b200 import configs
  configs.clear_config()
  configs.parse_config_files_and_bindings([gin], ['EvalConfig.eval_once = True'])
  return configs.ExperimentConfig(), configs.ModelConfig(), configs.TrainConfig(), configs.EvalConfig()


def _two_rank_worker(rank, world, port, tmp, gin):
  import sys
  os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                    LOCAL_RANK=str(rank))
  sys.path.insert(0, ROOT)
  from nerfies_b200 import configs, driver_utils, train as train_lib
  text = driver_utils.parse_configs([gin], ['TrainConfig.max_steps = 10', 'TrainConfig.save_every = 5'])
  state = train_lib.train(configs.ExperimentConfig(), configs.ModelConfig(), configs.TrainConfig(),
                          os.path.join(tmp, 'exp'), CAPTURE, config_str=text, log=lambda s: None)
  torch.save(state.camera_poses.pose.cpu(), os.path.join(tmp, f'poses{rank}.pt'))


def test_two_ranks_end_with_equal_poses(tmp_path, _clean_gin):
  if torch.cuda.device_count() < 2:
    pytest.skip('needs 2 GPUs')
  import torch.multiprocessing as mp
  port = 29700 + os.getpid() % 1500
  mp.spawn(_two_rank_worker, args=(2, port, str(tmp_path), _gin(tmp_path)), nprocs=2, join=True)
  poses = [torch.load(tmp_path / f'poses{r}.pt') for r in range(2)]
  assert torch.equal(poses[0], poses[1]) and float(poses[0].abs().max()) > 0
