"""Camera intrinsics refinement on the GPU: refined ray batches (nfb_gather_rays_refined, nfb_pixels_to_rays_refined)
against the plain ones bit for bit and against fp64 rays, the per-group intrinsics gradient (nfb_intrinsics_grad)
against fp64 autograd of the oracle, recovery of a perturbed group and of a registered photo's focal length, and
the drivers."""
import ctypes
import json
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
from tests.golden_util import model_from_spec, spec_to_dict, tree_to_device
from tests.test_intrinsics_refine import refined_rays
from tests.test_pose_refine_gpu import _cameras, _eval_configs, _flat_cpu

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAPTURE = os.path.join(ROOT, 'tests', 'golden', 'capture_small')
TOL = 2e-4
ALL = ('focal', 'principal_point', 'radial', 'tangential')


def _kinds(cams):
  """Distorted, pinhole and skewed-distorted intrinsics on cameras 0, 1, 2 (mod 3)."""
  out = []
  for k, c in enumerate(cams):
    c = c.copy()
    if k % 3 != 1:
      c.radial_distortion = np.array([0.05, -0.08, 0.02], np.float32)
      c.tangential_distortion = np.array([0.001, -0.0005], np.float32)
    if k % 3 == 2:
      c.skew = np.array(0.7, np.float32)
      c.pixel_aspect_ratio = np.array(1.005, np.float32)
    out.append(c)
  return out


def _spec_model(seed, batch_size=2048):
  from tests.test_render_vjp_gpu import _small_spec
  spec = _small_spec(use_camera_metadata=False, num_appearance_features=8, num_appearance_embeddings=4,
                     num_coarse_samples=64, num_fine_samples=0)
  params = tree_to_device(O.make_trained_like(O.init_params(spec, seed), seed=seed + 1), DEV)
  return spec, params, model_from_spec(spec_to_dict(spec), device=DEV, batch_size=batch_size)


def _render(model, params, cam, md):
  rays = camera_lib.camera_to_rays(cam, DEV)
  h, w = cam.image_shape
  meta = {k: torch.full((h * w, 1), int(v[0]), dtype=torch.int32, device=DEV) for k, v in md.items()}
  with torch.no_grad():
    out = model.apply({'params': params}, {'origins': rays['origins'].reshape(-1, 3),
                                           'directions': rays['directions'].reshape(-1, 3), 'metadata': meta},
                      warp_extra={'alpha': 4.0})
  return (out['coarse']['rgb'].reshape(h, w, 3).clamp(0, 1) * 255).round().to(torch.uint8).cpu().numpy()


def _table(cams, images=None, order=None):
  n = len(cams)
  md = {'warp': np.array([1] * n, np.int32), 'appearance': np.array([2] * n, np.int32)}
  if images is None:
    rng = np.random.default_rng(0)
    images = [rng.integers(0, 256, size=(*c.image_shape, 3), dtype=np.uint8) for c in cams]
  return datasets.DeviceRayTable(datasets.RayTable(images, cams, md), DEV, order=order), md


def _deltas(g, scale, seed):
  gen = torch.Generator().manual_seed(seed)
  q = torch.randn(g, 8, generator=gen) * torch.tensor([0.03, 0.01, 0.01, 0.02, 0.01, 0.005, 4e-4, 4e-4]) * scale
  return q.to(DEV).contiguous()


# ---------------------------------------------------------------------------
# refined rays
# ---------------------------------------------------------------------------
def test_zero_deltas_reproduce_the_rays_bit_for_bit():
  cams = _kinds(_cameras(3))
  table, _ = _table(cams)
  n = int(table.offsets[-1])
  group = torch.tensor([0, 1, 0], dtype=torch.int32, device=DEV)
  zero = torch.zeros(2, 8, device=DEV)
  plain = table.gather(0, n, order=False)
  refined = table.gather(0, n, order=False, intrinsics=(zero, group))
  for k in ('origins', 'directions', 'pixels', 'rgb'):
    assert torch.equal(plain[k], refined[k]), k
  pose = torch.cat([torch.randn(3, 3) * 0.05, torch.randn(3, 3) * 0.02], 1).to(DEV).contiguous()
  posed = table.gather(0, n, order=False, poses=pose)
  both = table.gather(0, n, order=False, poses=pose, intrinsics=(zero, group))
  for k in ('origins', 'directions', 'image'):
    assert torch.equal(posed[k], both[k]), k
  # the posed entry point itself, and the refined one returning pixels
  lib = _lib.load()
  t = table.table()
  outs = [torch.empty(n, 3, device=DEV) for _ in range(4)]
  pix = torch.empty(n, 2, device=DEV)
  with torch.cuda.device(DEV):
    _lib.check(lib.nfb_gather_rays_posed(ctypes.byref(t), 0, n, _ptr(pose), _ptr(outs[0]), _ptr(outs[1]), None,
                                         _stream()))
    _lib.check(lib.nfb_gather_rays_refined(ctypes.byref(t), 0, n, _ptr(pose), _ptr(zero), _ptr(group), 2,
                                           _ptr(outs[2]), _ptr(outs[3]), _ptr(pix), None, _stream()))
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[2]) and torch.equal(outs[1], outs[3])
  order_free = table.gather(0, n, order=False)
  assert torch.equal(pix, order_free['pixels'])
  # registration's pixels -> rays
  for cam in cams:
    px = camera_lib.camera_to_rays(cam, DEV)['pixels'].reshape(-1, 2).contiguous()
    want = cam.pixels_to_rays(px)
    for q in (None, torch.zeros(8, device=DEV)):
      got = torch.empty_like(want)
      _lib.check(lib.nfb_pixels_to_rays_refined(ctypes.byref(cam._struct()), _ptr(q), _ptr(px), px.shape[0],
                                                _ptr(got), _stream()))
      torch.cuda.synchronize()
      assert torch.equal(got, want)


def test_refined_rays_match_fp64():
  cams = _kinds(_cameras(3))
  table, _ = _table(cams)
  n = int(table.offsets[-1])
  group = torch.tensor([1, 0, 1], dtype=torch.int32, device=DEV)
  q = _deltas(2, 1.0, 3)
  pose = torch.cat([torch.randn(3, 3) * 0.05, torch.randn(3, 3) * 0.02], 1).to(DEV).contiguous()
  for p in (None, pose):
    got = table.gather(0, n, order=False, poses=p, intrinsics=(q, group))
    for k, cam in enumerate(cams):
      sel = slice(int(table.offsets[k]), int(table.offsets[k + 1]))
      omega = torch.zeros(3, dtype=torch.float64) if p is None else p[k, :3].cpu().double()
      want, res = refined_rays(cam, q[int(group[k])].cpu().double(), omega, got['pixels'][sel].cpu().double().numpy())
      err = float((got['directions'][sel].cpu().double() - want).abs().max())
      assert err < 5e-6, (k, err)
      shift = 0.0 if p is None else p[k, 3:].cpu()
      assert torch.equal(got['origins'][sel].cpu(), (torch.as_tensor(cam.position) + shift).expand(want.shape[0], 3))


# ---------------------------------------------------------------------------
# the intrinsics gradient
# ---------------------------------------------------------------------------
def _intrinsics_grad(cams_dev, n_images, pose, q, group, parts, batch, d_d):
  lib = _lib.load()
  g, count = q.shape[0], batch['image'].numel()
  ws = torch.empty(int(lib.nfb_intrinsics_grad_workspace_size(g, count)), dtype=torch.uint8, device=DEV)
  out = torch.zeros(g, 8, device=DEV)
  bits = sum(_lib.INTRINSICS_PARTS[p] for p in parts)
  _lib.check(lib.nfb_intrinsics_grad(_ptr(cams_dev), n_images, _ptr(pose), _ptr(q), _ptr(group), g, bits,
                                     _ptr(batch['image']), _ptr(batch['pixels']), _ptr(batch['directions']),
                                     _ptr(d_d), count, _ptr(out), _ptr(ws), ws.numel(), _stream()))
  torch.cuda.synchronize()
  return out


@pytest.mark.parametrize('posed', [False, True], ids=['no_pose', 'pose'])
def test_intrinsics_gradient_matches_fp64_and_is_repeatable(posed):
  """(G,8) gradients through the refined (and posed) rays -> the oracle against the GPU's, tier A.  Three images
  (distorted, pinhole, skewed) in groups [0, 2, 0] of three: group 1 has no ray and gets 0.  Each part alone
  gives exactly its entries of the full gradient and zero elsewhere; two calls give the same bits."""
  spec, params, model = _spec_model(410)
  cams = _kinds(_cameras(3))
  table, _ = _table(cams)
  group = torch.tensor([0, 2, 0], dtype=torch.int32, device=DEV)
  q = _deltas(3, 1.0, 4)
  gen = torch.Generator().manual_seed(2)
  pose = (torch.cat([torch.randn(3, 3, generator=gen) * 0.02, torch.randn(3, 3, generator=gen) * 0.01], 1)
          .to(DEV).contiguous() if posed else None)
  B = 900
  batch = table.gather(0, B * 4, poses=pose, intrinsics=(q, group))
  batch = {k: (v[::4].contiguous() if torch.is_tensor(v) else {kk: vv[::4].contiguous() for kk, vv in v.items()})
           for k, v in batch.items()}
  batch['rgb'] = torch.rand(B, 3, generator=gen).to(DEV)
  t_rand = torch.rand(B, spec.num_coarse_samples, generator=gen)
  d_o, d_d = torch.empty(B, 3, device=DEV), torch.empty(B, 3, device=DEV)
  training.value_and_grad(model, params, batch, {'alpha': 4.0}, chunk_rays=256, t_rand=t_rand, ray_grads=(d_o, d_d))
  ci = training.CameraIntrinsics([str(k) for k in range(3)], cams, ALL, DEV)
  got = _intrinsics_grad(ci.cameras, 3, pose, q, group, ALL, batch, d_d)
  again = _intrinsics_grad(ci.cameras, 3, pose, q, group, ALL, batch, d_d)
  assert torch.equal(got, again)
  assert torch.equal(got[1], torch.zeros(8, device=DEV))
  for part in ALL:
    alone = _intrinsics_grad(ci.cameras, 3, pose, q, group, (part,), batch, d_d)
    mask = torch.zeros(8, dtype=torch.bool, device=DEV)
    mask[list(_lib.INTRINSICS_ENTRIES[part])] = True
    assert torch.equal(alone[:, mask], got[:, mask]) and not alone[:, ~mask].any(), part
  img = batch['image'].cpu().long()
  px = batch['pixels'].cpu().double().numpy()
  md = {k: v.cpu() for k, v in batch['metadata'].items()}
  with torch.no_grad():
    zc = O.render_forward(O.tree_to(_flat_cpu(params), torch.float64), spec,
                          {'origins': batch['origins'].cpu(), 'directions': batch['directions'].cpu(), 'metadata': md},
                          warp_alpha=4.0, dtype=torch.float64, t_rand=t_rand)['coarse']['z_vals']

  def oracle(dtype):
    qq = q.cpu().double().clone().requires_grad_(True)
    ds = []
    for k, cam in enumerate(cams):
      omega = torch.zeros(3, dtype=torch.float64) if pose is None else pose[k, :3].cpu().double()
      ds.append(refined_rays(cam, qq[int(group[k])], omega, px)[0])
    onehot = torch.nn.functional.one_hot(img, 3).double()[:, :, None]
    d = (torch.stack(ds, 1) * onehot).sum(1).to(dtype)
    rays = {'origins': batch['origins'].cpu().to(dtype), 'directions': d, 'metadata': md}
    out = O.render_level(O.tree_to(_flat_cpu(params), dtype), spec, 'coarse', rays, zc, 4.0, dtype=dtype)
    ((out['rgb'] - batch['rgb'].cpu().to(dtype))**2).mean().backward()
    return qq.grad.double()

  ref, r32 = oracle(torch.float64), oracle(torch.float32)
  scale = float(ref.abs().max())
  band = float((r32 - ref).abs().max()) / scale
  err = float((got.cpu().double() - ref).abs().max()) / scale
  print(f'intrinsics gradient ({"pose" if posed else "no pose"}): error {err:.3e}, band {band:.3e}')
  assert err <= max(TOL, 3 * band), (err, band)


# ---------------------------------------------------------------------------
# recovery
# ---------------------------------------------------------------------------
STEPS = 400


def test_perturbed_group_is_recovered():
  """Six cameras sharing one group's intrinsics around a trained-like model, targets its renders; the group
  perturbed by 3% in focal, 1.5 px in principal point and 0.02 in k1; intrinsics-only training, the model
  (learning rate 0) and the poses (not refined) held."""
  spec, params, model = _spec_model(420)
  size = (80, 60)
  cams = []
  for c in _cameras(6, size=size):
    c.radial_distortion = np.array([0.03, 0.0, 0.0], np.float32)
    cams.append(c)
  md = {'warp': np.array([1] * 6, np.int32), 'appearance': np.array([2] * 6, np.int32)}
  images = [_render(model, params, c, md) for c in cams]
  shift = 1.5 / np.sqrt(2) / float(cams[0].focal_length)   # 1.5 px
  truth = np.array([np.log(1.03), shift, -shift, 0.02, 0, 0, 0, 0])
  perturbed = [geometry.refined_camera(c, truth) for c in cams]
  n = int(sum(h * w for h, w in (c.image_shape for c in cams)))
  table, _ = _table(perturbed, images, order=np.random.default_rng(6).permutation(n))
  state = training.create_train_state(model, params, warp_alpha=4.0)
  ci = training.CameraIntrinsics([str(k) for k in range(6)], perturbed, ('focal', 'principal_point', 'radial'), DEV)
  assert ci.delta.shape == (1, 8)
  state.camera_intrinsics = ci
  sp = training.ScalarParams(learning_rate=0.0)

  def errors():
    c1 = geometry.refined_camera(perturbed[0], ci.delta[0])
    return (abs(float(c1.focal_length) / float(cams[0].focal_length) - 1),
            float(np.linalg.norm(c1.principal_point.astype(np.float64) - cams[0].principal_point)),
            abs(float(c1.radial_distortion[0]) - float(cams[0].radial_distortion[0])))

  e0 = errors()
  psnr = []
  for step in range(STEPS):
    sp.camera_intrinsics_learning_rate = 3e-3 * 0.02**(step / STEPS)
    batch = table.gather(step * 1024, 1024, intrinsics=(ci.delta, ci.group))
    state, stats, _ = training.train_step(model, step, state, batch, sp)
    if step in (0, STEPS - 1):
      psnr.append(float(stats['coarse']['metric/psnr']))
  e1 = errors()
  print(f'focal {100 * e0[0]:.3f}% -> {100 * e1[0]:.4f}%, principal point {e0[1]:.3f} -> {e1[1]:.4f} px, '
        f'k1 {e0[2]:.4f} -> {e1[2]:.5f}, batch PSNR {psnr[0]:.2f} -> {psnr[1]:.2f} dB')
  print('stats:', {k: float(v) for k, v in stats['camera_intrinsics'].items()})
  assert torch.equal(ci.delta[0, 6:], torch.zeros(2, device=DEV))   # tangential not fitted: exactly 0
  assert all(b * 5 <= a for a, b in zip(e0, e1)), (e0, e1)
  assert psnr[1] > psnr[0]


def test_registration_recovers_focal():
  """A photo rendered from a camera; registration starts from the camera with a focal 5% off and fits
  the pose and the focal length."""
  spec, params, model = _spec_model(430)
  cam = _cameras(6, size=(80, 60))[1]
  md = {'warp': np.array([1], np.int32), 'appearance': np.array([2], np.int32)}
  image = torch.from_numpy(_render(model, params, cam, md).astype(np.float32) / 255.0)
  start = cam.copy()
  start.focal_length = np.array(float(cam.focal_length) * 1.05, np.float32)
  got, codes, history = geometry.register_camera(model, params, start, image, {'alpha': 4.0},
                                                 {'warp': 1, 'appearance': 2}, optimize=('pose',), intrinsics=('focal',),
                                                 steps=300, batch_rays=1024, lr_decay=0.05)
  err = abs(float(got.focal_length) / float(cam.focal_length) - 1)
  R = got.orientation.astype(np.float64) @ cam.orientation.astype(np.float64).T
  rot_deg = float(np.degrees(np.arccos(np.clip((np.trace(R) - 1) / 2, -1, 1))))
  print(f'focal error 5% -> {100 * err:.4f}%, rotation {rot_deg:.4f} deg, '
        f'loss {history[0]["loss"]:.3e} -> {history[-1]["loss"]:.3e}, last logged focal change '
        f'{history[-1]["focal_change_pct"]:.3f}%')
  assert codes['intrinsics'].shape == (1, 8) and float(codes['intrinsics'][0, 1:].abs().max()) == 0.0
  assert err * 5 <= 0.05 and history[-1]['loss'] < history[0]['loss']


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
  path.write_text(GIN + 'ModelConfig.use_stratified_sampling = False\n'
                  "TrainConfig.refine_camera_intrinsics = ('focal', 'radial')\n"
                  "TrainConfig.camera_intrinsics_lr_schedule = ('constant', 0.001)\n")
  return str(path)


def test_drivers_refine_save_resume_eval_and_register(tmp_path, _clean_gin):
  from nerfies_b200 import checkpoints, configs, driver_utils, eval as eval_lib, register_camera, train as train_lib
  from tests.test_drivers_gpu import _argv
  gin = _gin(tmp_path)
  bases = {k: tmp_path / k for k in ('whole', 'again', 'resumed')}
  for k in ('whole', 'again'):
    assert train_lib.main(_argv(bases[k], gin)) == 0
  assert train_lib.main(_argv(bases['resumed'], gin, '--max_steps', '30')) == 0
  assert train_lib.main(_argv(bases['resumed'], gin)) == 0
  saved = {k: checkpoints.restore_checkpoint(str(b / 'checkpoints'), device='cpu').camera_intrinsics
           for k, b in bases.items()}
  groups = sorted(saved['whole']['groups'].values(), key=lambda g: g['items'])
  assert len(groups) == 4 and all(len(g['items']) == 1 for g in groups)   # one group per image here
  flat = lambda s, key: np.concatenate([np.asarray(g[key], np.float64) for g in
                                        sorted(s['groups'].values(), key=lambda g: g['items'])])
  for key in ('delta', 'grad_ema', 'grad_sq_ema'):
    noise = np.linalg.norm(flat(saved['whole'], key) - flat(saved['again'], key))
    dist = np.linalg.norm(flat(saved['whole'], key) - flat(saved['resumed'], key))
    print(f'{key}: two uninterrupted runs {noise:.3e}, resumed {dist:.3e}, |x| {np.linalg.norm(flat(saved["whole"], key)):.3e}')
    assert dist <= 10 * noise + 1e-6 * np.linalg.norm(flat(saved['whole'], key)), key
  delta = flat(saved['whole'], 'delta').reshape(-1, 8)
  assert np.abs(delta[:, 0]).max() > 0 and np.abs(delta[:, 3:6]).max() > 0
  assert not delta[:, 1:3].any() and not delta[:, 6:8].any()      # principal point and tangential not fitted
  records = driver_utils.read_scalars(bases['whole'] / 'summaries' / 'train.jsonl')
  assert records[-1]['camera_intrinsics/focal_change_pct'] > 0
  item = groups[0]['items'][0]
  cam = camera_lib.Camera.from_json(bases['whole'] / 'cameras' / '00000060' / f'{item}.json')
  orig = camera_lib.Camera.from_json(os.path.join(CAPTURE, 'camera', f'{item}.json'))
  assert np.array_equal(cam.image_size, orig.image_size)
  assert np.isclose(float(cam.focal_length), float(orig.focal_length) * np.exp(float(groups[0]['delta'][0])),
                    rtol=1e-6) and cam.focal_length != orig.focal_length
  # refinement off on a checkpoint with intrinsics: refused before any GPU work
  with open(gin) as f:
    off = f.read().replace("TrainConfig.refine_camera_intrinsics = ('focal', 'radial')", '')
  (tmp_path / 'off.gin').write_text(off)
  with pytest.raises(ValueError, match='refine_camera_intrinsics is empty'):
    train_lib.main(_argv(bases['whole'], str(tmp_path / 'off.gin'), '--max_steps', '61'))
  # eval renders the train items from the refined cameras
  lines = []
  assert eval_lib.evaluate(*_eval_configs(gin), str(bases['whole']), CAPTURE, precision='fp32', poll_seconds=0.0,
                           log=lines.append) == [60]
  assert any('refined camera intrinsics' in l for l in lines)
  assert os.listdir(bases['whole'] / 'renders' / '00000060' / 'train')
  # register an item with pose and focal
  configs.clear_config()
  argv = ['--base_folder', str(bases['whole']), '--data_dir', CAPTURE, '--gin_configs', gin, '--item', item,
          '--steps', '20', '--batch_rays', '256', '--optimize', 'pose', '--intrinsics', 'focal']
  assert register_camera.main(argv) == 0
  out = bases['whole'] / 'registrations' / '00000060' / item
  reg = camera_lib.Camera.from_json(out / 'camera.json')
  q = np.load(out / 'codes.npz')['intrinsics'].reshape(8)
  assert np.isclose(float(reg.focal_length), float(orig.focal_length) * np.exp(q[0]), rtol=1e-6)
  log = [json.loads(l) for l in (out / 'log.jsonl').read_text().splitlines()]
  assert len(log) == 20 and 'focal_change_pct' in log[-1]
  summary = json.loads((out / 'summary.json').read_text())
  assert 'focal_change_pct' in summary


def _two_rank_worker(rank, world, port, tmp, gin):
  import sys
  os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                    LOCAL_RANK=str(rank))
  sys.path.insert(0, ROOT)
  from nerfies_b200 import configs, driver_utils, train as train_lib
  text = driver_utils.parse_configs([gin], ['TrainConfig.max_steps = 10', 'TrainConfig.save_every = 5'])
  state = train_lib.train(configs.ExperimentConfig(), configs.ModelConfig(), configs.TrainConfig(),
                          os.path.join(tmp, 'exp'), CAPTURE, config_str=text, log=lambda s: None)
  torch.save(state.camera_intrinsics.delta.cpu(), os.path.join(tmp, f'delta{rank}.pt'))


def test_two_ranks_end_with_equal_deltas(tmp_path, _clean_gin):
  if torch.cuda.device_count() < 2:
    pytest.skip('needs 2 GPUs')
  import torch.multiprocessing as mp
  port = 29700 + os.getpid() % 1500
  mp.spawn(_two_rank_worker, args=(2, port, str(tmp_path), _gin(tmp_path)), nprocs=2, join=True)
  deltas = [torch.load(tmp_path / f'delta{r}.pt') for r in range(2)]
  assert torch.equal(deltas[0], deltas[1]) and float(deltas[0].abs().max()) > 0
