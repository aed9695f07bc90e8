"""geometry.register_camera on the GPU: the pose chain's gradient against fp64 autograd through the oracle, and
convergence on a frame the model rendered itself."""
import numpy as np
import pytest
import torch

from nerfies_b200 import camera as camera_lib
from nerfies_b200 import geometry
from oracle import nerfies_oracle as O
from tests.golden_util import model_from_spec, spec_to_dict, tree_to_device
from tests.test_mesh_gpu import CAPTURE, checkpoint  # noqa: F401  (the trained-like checkpoint fixture)
from tests.test_render_vjp_gpu import TOL, _small_spec

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _setup(seed, size=(48, 36)):
  # coarse only: the loss sums the levels' rgb errors, and a self-rendered target of one level is not the
  # other level's image, so with two levels the true pose would not be the loss's minimum
  spec = _small_spec(use_camera_metadata=False, num_appearance_features=8, num_appearance_embeddings=4,
                     num_coarse_samples=64, num_fine_samples=0)
  params = O.make_trained_like(O.init_params(spec, seed), seed=seed + 1)
  model = model_from_spec(spec_to_dict(spec), device=DEV, batch_size=2048)
  # a camera 0.5 in front of the scene box's centre, looking along +z
  cam = camera_lib.Camera(orientation=np.eye(3), position=[0.0, 0.0, -0.45], focal_length=0.9 * size[0],
                          principal_point=[size[0] / 2, size[1] / 2], image_size=list(size))
  return spec, params, model, cam


def _frame(model, params, cam, md, warp_extra):
  rays = camera_lib.camera_to_rays(cam, DEV)
  h, w = cam.image_shape
  B = h * w
  meta = {k: torch.full((B, 1), v, dtype=torch.int32, device=DEV) for k, v in md.items()}
  with torch.no_grad():
    out = model.apply({'params': tree_to_device(params, DEV)}, {'origins': rays['origins'].reshape(-1, 3),
                                                                 'directions': rays['directions'].reshape(-1, 3),
                                                                 'metadata': meta}, warp_extra=warp_extra)
  return out['coarse']['rgb'].reshape(h, w, 3)


def _psnr(a, b):
  return float(-10 * torch.log10(((a - b)**2).mean()))


def test_pose_gradient_against_fp64():
  """d loss / d (omega, v) of one registration step (pose_rays -> render_rays -> photometric_loss) against
  torch.autograd in float64 of the same pose formula through the oracle at the kernel's z, on the same
  pixel batch; tier A: max(2e-4, 3 x the fp32 oracle's distance from fp64) of the largest component."""
  spec, params, model, cam = _setup(200)
  md = {'warp': 1, 'appearance': 2}
  gen = torch.Generator().manual_seed(3)
  B = 256
  local = camera_lib.camera_to_rays(cam.copy(), DEV)['directions'].reshape(-1, 3)
  idx = torch.randint(0, local.shape[0], (B,), generator=gen).to(DEV)
  target = torch.rand(B, 3, generator=gen).to(DEV)
  omega0 = torch.tensor([0.01, -0.02, 0.015])
  v0 = torch.tensor([0.005, 0.01, -0.008])
  meta = {k: torch.full((B, 1), v, dtype=torch.int32) for k, v in md.items()}
  omega = omega0.to(DEV).requires_grad_(True)
  v = v0.to(DEV).requires_grad_(True)
  R0, p0 = torch.tensor(cam.orientation, device=DEV), torch.tensor(cam.position, device=DEV)
  o, d = geometry.pose_rays(local[idx], R0, p0, omega, v)
  out = model.render_rays({'params': tree_to_device(params, DEV)},
                          {'origins': o, 'directions': d, 'metadata': tree_to_device(meta, DEV)},
                          warp_extra={'alpha': 4.0})
  geometry.photometric_loss(out, target).backward()
  got = torch.cat([omega.grad, v.grad]).cpu().double()
  z = {lv: out[lv]['z_vals'].cpu() for lv in out}

  def oracle(dtype):
    w_ = omega0.to(dtype).requires_grad_(True)
    v_ = v0.to(dtype).requires_grad_(True)
    oo, dd = geometry.pose_rays(local[idx].cpu().to(dtype), R0.cpu().to(dtype), p0.cpu().to(dtype), w_, v_)
    r = {'origins': oo, 'directions': dd, 'metadata': meta}
    p = O.tree_to(params, dtype)
    outs = {lv: O.render_level(p, spec, lv, r, z[lv], 4.0, dtype=dtype) for lv in z}
    geometry.photometric_loss(outs, target.cpu().to(dtype)).backward()
    return torch.cat([w_.grad, v_.grad]).double()

  ref, r32 = oracle(torch.float64), oracle(torch.float32)
  scale = float(ref.abs().max())
  band = float((r32 - ref).abs().max()) / scale
  err = float((got - ref).abs().max()) / scale
  print(f'pose gradient: error {err:.3e}, band {band:.3e}, ref {ref.tolist()}')
  assert err <= max(TOL, 3 * band), (err, band)


def _rotation_error_deg(a, b):
  R = a.orientation.astype(np.float64) @ b.orientation.astype(np.float64).T
  return float(np.degrees(np.arccos(np.clip((np.trace(R) - 1) / 2, -1, 1))))


def test_converges_from_a_perturbed_pose():
  spec, params, model, cam = _setup(210)
  md = {'warp': 1, 'appearance': 2}
  extra = {'alpha': 4.0}
  image = _frame(model, params, cam, md, extra)
  rng = np.random.default_rng(4)
  axis = rng.normal(size=3)
  omega = axis / np.linalg.norm(axis) * np.radians(1.5)
  direction = rng.normal(size=3)
  offset = direction / np.linalg.norm(direction) * 0.015 * (spec.far - spec.near) / 0.81
  start = geometry.posed_camera(cam, torch.tensor(omega), torch.tensor(offset))
  rot0, pos0 = _rotation_error_deg(start, cam), float(np.linalg.norm(start.position - cam.position))
  psnr0 = _psnr(_frame(model, params, start, md, extra), image)
  got, _, hist = geometry.register_camera(model, tree_to_device(params, DEV), start, image, extra, md,
                                          optimize=('pose',), steps=STEPS, batch_rays=1024, seed=5, lr_decay=0.1)
  rot1, pos1 = _rotation_error_deg(got, cam), float(np.linalg.norm(got.position - cam.position))
  psnr1 = _psnr(_frame(model, params, got, md, extra), image)
  print(f'pose: rotation {rot0:.4f} -> {rot1:.5f} deg, position {pos0:.5f} -> {pos1:.6f}, '
        f'PSNR {psnr0:.2f} -> {psnr1:.2f} dB, loss {hist[0]["loss"]:.3e} -> {hist[-1]["loss"]:.3e}')
  # Measured on an H100 80GB HBM3 at 700 W: rotation 1.5 -> 0.00000 deg, position 0.0150 -> 0.000000, PSNR 34.2 ->
  # 139.3 dB in 300 steps: far inside the 10x asked here.
  assert rot1 * 10 <= rot0 and pos1 * 10 <= pos0 and psnr1 > psnr0


def test_converges_from_a_wrong_appearance_row():
  spec, params, model, cam = _setup(220)
  extra = {'alpha': 4.0}
  image = _frame(model, params, cam, {'warp': 1, 'appearance': 2}, extra)
  wrong = {'warp': 1, 'appearance': 0}
  psnr0 = _psnr(_frame(model, params, cam, wrong, extra), image)
  p = tree_to_device(params, DEV)
  true_code = p['appearance_encoder']['embed']['embedding'][2]
  start_code = p['appearance_encoder']['embed']['embedding'][0]
  got, codes, hist = geometry.register_camera(model, p, cam, image, extra, wrong, optimize=('pose', 'appearance'),
                                              steps=STEPS, batch_rays=1024, seed=6, lr_decay=0.1)
  rot1, pos1 = _rotation_error_deg(got, cam), float(np.linalg.norm(got.position - cam.position))
  code_err0 = float((start_code - true_code).norm())
  code_err1 = float((codes['appearance'][0] - true_code).norm())
  # the registered frame with the fitted code (metadata_encoded)
  rays = camera_lib.camera_to_rays(got, DEV)
  n = rays['origins'].numel() // 3
  md = {'warp': p['warp_field']['metadata_encoder']['embed']['embedding'][1:2].expand(n, -1),
        'appearance': codes['appearance'].expand(n, -1)}
  with torch.no_grad():
    out = model.apply({'params': p}, {'origins': rays['origins'].reshape(-1, 3),
                                      'directions': rays['directions'].reshape(-1, 3), 'metadata': md},
                      warp_extra=extra, metadata_encoded=True)
  psnr1 = _psnr(out['coarse']['rgb'].reshape(image.shape), image)
  print(f'appearance: code error {code_err0:.4f} -> {code_err1:.4f}, PSNR {psnr0:.2f} -> {psnr1:.2f} dB, pose '
        f'drift {rot1:.5f} deg / {pos1:.6f}, loss {hist[0]["loss"]:.3e} -> {hist[-1]["loss"]:.3e}')
  # Measured on an H100 80GB HBM3 at 700 W: PSNR 42.1 -> 83.8 dB, loss 5.7e-5 -> 4.4e-9, pose drift 0.00000 deg /
  # 2.1e-5, code error 0.056 -> 0.0064 (the code's directions that barely change the colour stay loose, so the
  # code itself is not held to 10x).  Bounds: a 20 dB gain, a 1000x loss drop, drift below 0.01 deg / 1e-4.
  assert psnr1 >= psnr0 + 20 and hist[-1]['loss'] * 1000 <= hist[0]['loss']
  assert rot1 <= 0.01 and pos1 <= 1e-4


STEPS = 300


@pytest.mark.parametrize('enc', ['time', 'blend'])
def test_warp_code_of_a_fixed_time_renders_as_the_ids(enc):
  """nfb_warp_code: the encoded warp code of a time ('time') or id ('blend') renders bitwise as the ids do."""
  spec = _small_spec(use_camera_metadata=False, num_fine_samples=0, warp_field_type='translation',
                     warp_metadata_encoder_type=enc)
  params = tree_to_device(O.make_trained_like(O.init_params(spec, 240), seed=241), DEV)
  model = model_from_spec(spec_to_dict(spec), device=DEV, batch_size=2048)
  cam = _setup(240)[3]
  md = {'time': 0.3, 'appearance': 1} if enc == 'time' else {'warp': 2, 'appearance': 1}
  extra = {'alpha': 4.0, 'time_alpha': 0.6}
  codes = geometry.registration_codes(model, params, md, extra)
  got = geometry.render_camera(model, params, cam, extra, codes)
  rays = camera_lib.camera_to_rays(cam, DEV)
  n = rays['origins'].numel() // 3
  meta = {'appearance': torch.full((n, 1), 1, dtype=torch.int32, device=DEV)}
  meta.update({'time': torch.full((n, 1), 0.3, device=DEV)} if enc == 'time' else
              {'warp': torch.full((n, 1), 2, dtype=torch.int32, device=DEV)})
  with torch.no_grad():
    ref = model.apply({'params': params}, {'origins': rays['origins'].reshape(-1, 3),
                                           'directions': rays['directions'].reshape(-1, 3), 'metadata': meta},
                      warp_extra=extra)['coarse']['rgb'].reshape(got.shape)
  assert torch.equal(got, ref)


def test_time_encoder_pose_and_appearance():
  """A 'time' warp encoder: the pose and the appearance code are fitted with the warp code held at the
  TimeEncoder's output for the frame's time."""
  spec = _small_spec(use_camera_metadata=False, num_appearance_features=8, num_appearance_embeddings=4,
                     num_coarse_samples=64, num_fine_samples=0, warp_metadata_encoder_type='time')
  params = tree_to_device(O.make_trained_like(O.init_params(spec, 250), seed=251), DEV)
  model = model_from_spec(spec_to_dict(spec), device=DEV, batch_size=2048)
  cam = _setup(250)[3]
  extra = {'alpha': 4.0, 'time_alpha': 1.0}
  true_md, start_md = {'time': 0.25, 'appearance': 2}, {'time': 0.25, 'appearance': 0}
  image = geometry.render_camera(model, params, cam, extra, geometry.registration_codes(model, params, true_md, extra))
  start = geometry.posed_camera(cam, torch.tensor([0.0, np.radians(1.0), 0.0]), torch.tensor([0.005, 0.0, 0.0]))
  psnr0 = _psnr(geometry.render_camera(model, params, start, extra,
                                       geometry.registration_codes(model, params, start_md, extra)), image)
  got, codes, hist = geometry.register_camera(model, params, start, image, extra, start_md,
                                              optimize=('pose', 'appearance'), steps=STEPS, batch_rays=1024, seed=7,
                                              lr_decay=0.1)
  psnr1 = _psnr(geometry.render_camera(model, params, got, extra,
                                       dict(geometry.registration_codes(model, params, start_md, extra), **codes)),
                image)
  rot1, pos1 = _rotation_error_deg(got, cam), float(np.linalg.norm(got.position - cam.position))
  print(f'time encoder: PSNR {psnr0:.2f} -> {psnr1:.2f} dB, rotation 1.0 -> {rot1:.5f} deg, position 0.005 -> '
        f'{pos1:.6f}, loss {hist[0]["loss"]:.3e} -> {hist[-1]["loss"]:.3e}')
  assert psnr1 >= psnr0 + 10 and rot1 * 10 <= 1.0 and pos1 * 10 <= 0.005


def test_driver_end_to_end(checkpoint):  # noqa: F811
  import json
  from nerfies_b200 import configs, datasets, register_camera
  base, gin, model, params, source = checkpoint
  item = source.train_ids[0]
  argv = ['--base_folder', str(base), '--data_dir', CAPTURE, '--gin_configs', gin, '--item', item,
          '--steps', '40', '--batch_rays', '256', '--optimize', 'pose,appearance']
  configs.clear_config()
  assert register_camera.main(argv) == 0
  out = base / 'registrations' / '00000007' / item
  for f in ('camera.json', 'codes.npz', 'log.jsonl', 'rgb_before.png', 'rgb_after.png', 'summary.json'):
    assert (out / f).exists(), f
  cam = camera_lib.Camera.from_json(out / 'camera.json')
  orig = camera_lib.Camera.from_json(source.camera_dir / f'{item}{source.camera_ext}')
  # the capture's original scale: same intrinsics and size as the item's own JSON, a pose near it
  assert np.array_equal(cam.image_size, orig.image_size) and cam.focal_length == orig.focal_length
  reloaded = source.load_camera(out / 'camera.json')
  assert reloaded.image_shape == source.load_camera(item).image_shape
  log = [json.loads(l) for l in (out / 'log.jsonl').read_text().splitlines()]
  assert len(log) == 40 and log[-1]['loss'] < log[0]['loss']
  codes = dict(np.load(out / 'codes.npz'))
  assert codes['appearance'].shape == (1, model.num_appearance_features)
  summary = json.loads((out / 'summary.json').read_text())
  rgb = datasets.decode_image(out / 'rgb_after.png')
  assert rgb.shape[:2] == source.load_camera(item).image_shape
  print(f'driver: loss {log[0]["loss"]:.3e} -> {log[-1]["loss"]:.3e}, PSNR {summary["psnr_before"]:.2f} -> '
        f'{summary["psnr_after"]:.2f}')
  configs.clear_config()
  with pytest.raises(ValueError, match='unknown item'):
    register_camera.main([a if a != item else 'nope' for a in argv])
  configs.clear_config()
