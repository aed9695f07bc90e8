"""Camera registration's host logic, without a device: the torch Rodrigues formula against scipy, the pose
parametrisation against the registered Camera it reports, and the refusals."""
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from nerfies_b200 import camera as camera_lib
from nerfies_b200 import geometry
from oracle import nerfies_oracle as O
from tests.golden_util import model_from_spec, spec_to_dict


@pytest.mark.parametrize('angle', [1e-8, 1e-6, 1e-4, 5e-3, 1e-2, 0.1, 0.5, 1.0, 2.0, 3.0, np.pi - 1e-3])
def test_rodrigues_matches_scipy(angle):
  rng = np.random.default_rng(int(angle * 1e6) % 1000)
  for _ in range(8):
    axis = rng.normal(size=3)
    w = axis / np.linalg.norm(axis) * angle
    ref = Rotation.from_rotvec(w).as_matrix()
    got32 = geometry.rotvec_to_matrix(torch.tensor(w, dtype=torch.float32)).double().numpy()
    got64 = geometry.rotvec_to_matrix(torch.tensor(w, dtype=torch.float64)).numpy()
    # fp32: a few roundings of entries of magnitude <= 1; fp64: the series' remainder and roundings
    assert np.abs(got32 - ref).max() <= 5e-7, angle
    assert np.abs(got64 - ref).max() <= 1e-14, angle


def test_rodrigues_gradient_at_zero():
  w = torch.zeros(3, dtype=torch.float64, requires_grad=True)
  R = geometry.rotvec_to_matrix(w)
  (g,) = torch.autograd.grad((R * torch.arange(9.0, dtype=torch.float64).reshape(3, 3)).sum(), w)
  # d exp([w]x) / dw at 0 is the skew generator: d R_ij / dw_k = -eps_ijk
  M = torch.arange(9.0, dtype=torch.float64).reshape(3, 3)
  ref = torch.tensor([M[2, 1] - M[1, 2], M[0, 2] - M[2, 0], M[1, 0] - M[0, 1]], dtype=torch.float64)
  assert torch.allclose(g, ref)


def test_pose_rays_match_posed_camera():
  rng = np.random.default_rng(3)
  R0 = Rotation.from_rotvec(rng.normal(size=3)).as_matrix()
  cam = camera_lib.Camera(orientation=R0, position=[0.1, -0.2, 0.3], focal_length=50.0,
                          principal_point=[16, 12], image_size=[32, 24])
  omega = torch.tensor([0.02, -0.01, 0.03], dtype=torch.float64)
  offset = torch.tensor([0.01, 0.02, -0.03], dtype=torch.float64)
  local = torch.tensor(rng.normal(size=(10, 3)))
  local = local / local.norm(dim=-1, keepdim=True)
  o, d = geometry.pose_rays(local, torch.tensor(cam.orientation, dtype=torch.float64),
                            torch.tensor(cam.position, dtype=torch.float64), omega, offset)
  posed = geometry.posed_camera(cam, omega, offset)
  # Camera convention: world direction = orientation^T local
  ref = local.numpy() @ posed.orientation.astype(np.float64)
  assert np.abs(d.numpy() - ref).max() < 1e-6
  assert np.abs(o.numpy() - posed.position[None].astype(np.float64)).max() < 1e-7
  assert np.abs(posed.orientation.astype(np.float64) @ posed.orientation.T.astype(np.float64) - np.eye(3)).max() < 1e-6


def _model(**kw):
  spec = O.OracleSpec(num_coarse_samples=8, num_fine_samples=8, near=0.02, far=0.83, nerf_trunk_depth=2,
                      nerf_trunk_width=16, **kw)
  return model_from_spec(spec_to_dict(spec), device='cpu')


def test_refusals():
  plain = _model()
  assert geometry.check_registration(plain, ['pose'], 10, 16) == ('pose',)
  with pytest.raises(ValueError, match='unknown optimize'):
    geometry.check_registration(plain, ['pose', 'focal'], 10, 16)
  with pytest.raises(ValueError, match='empty'):
    geometry.check_registration(plain, [], 10, 16)
  with pytest.raises(ValueError, match='appearance'):
    geometry.check_registration(plain, ['appearance'], 10, 16)
  with pytest.raises(ValueError, match='camera metadata'):
    geometry.check_registration(plain, ['camera'], 10, 16)
  with pytest.raises(ValueError, match='no warp field'):
    geometry.check_registration(plain, ['warp'], 10, 16)
  with pytest.raises(ValueError, match='steps'):
    geometry.check_registration(plain, ['pose'], 0, 16)
  with pytest.raises(ValueError, match='batch_rays'):
    geometry.check_registration(plain, ['pose'], 10, 0)
  timed = _model(use_warp=True, warp_metadata_encoder_type='time', use_appearance_metadata=True)
  with pytest.raises(ValueError, match='function of time'):
    geometry.check_registration(timed, ['warp'], 10, 16)
  assert geometry.check_registration(timed, ['pose', 'appearance'], 10, 16) == ('pose', 'appearance')
  assert geometry.check_registration(timed, ['pose'], 10, 16) == ('pose',)
  glo = _model(use_warp=True, use_appearance_metadata=True)
  assert geometry.check_registration(glo, ('pose', 'appearance', 'warp'), 1, 1) == ('pose', 'appearance', 'warp')


def test_unknown_embedding_row_is_refused():
  model = _model(use_warp=True, use_appearance_metadata=True, num_warp_embeddings=3, num_appearance_embeddings=2)
  params = O.init_params(O.OracleSpec(num_coarse_samples=8, num_fine_samples=8, nerf_trunk_depth=2,
                                      nerf_trunk_width=16, use_warp=True, use_appearance_metadata=True,
                                      num_warp_embeddings=3, num_appearance_embeddings=2), 0)
  codes = geometry.registration_codes(model, params, {'warp': 2, 'appearance': 1})
  assert codes['warp'].shape == (1, 8) and torch.equal(codes['appearance'][0],
                                                       params['appearance_encoder']['embed']['embedding'][1])
  for md, msg in (({'warp': 3, 'appearance': 0}, "'warp'"), ({'warp': 0, 'appearance': 2}, "'appearance'"),
                  ({'warp': -1, 'appearance': 0}, "'warp'")):
    with pytest.raises(ValueError, match=msg):
      geometry.registration_codes(model, params, md)
  with pytest.raises(KeyError, match='appearance'):
    geometry.registration_codes(model, params, {'warp': 0})


# ---- the driver ------------------------------------------------------------------------------------------
class _Source:
  """The datasource attributes the driver reads before any GPU work: items a (40 x 30) and b."""

  use_appearance_id, use_warp_id, use_camera_id, use_time = True, True, False, False
  camera_ext = '.json'

  def __init__(self, root):
    import cv2
    self.root = root
    self.camera_dir = root / 'camera'
    self.camera_dir.mkdir(parents=True, exist_ok=True)
    self.all_ids = ['a', 'b']
    cam = camera_lib.Camera(np.eye(3), np.zeros(3), 50.0, (20.0, 15.0), (40, 30))
    for i in self.all_ids:
      (self.camera_dir / f'{i}.json').write_text(__import__('json').dumps(cam.to_json()))
      cv2.imwrite(str(root / f'{i}.png'), np.zeros((30, 40, 3), np.uint8))
    cv2.imwrite(str(root / 'small.png'), np.zeros((20, 40, 3), np.uint8))

  def get_rgb_path(self, item):
    return self.root / f'{item}.png'

  def _item_metadata(self, item):
    return {'appearance': self.all_ids.index(item), 'warp': 1}

  def load_camera(self, item):
    path = item if not isinstance(item, str) else self.camera_dir / f'{item}.json'
    return camera_lib.Camera.from_json(path)


def _register(tmp_path, **kw):
  from nerfies_b200 import configs, register_camera
  mc = kw.pop('model_config', configs.ModelConfig(use_warp=True, use_appearance_metadata=True))
  return register_camera.register(configs.ExperimentConfig(), mc, str(tmp_path), datasource=_Source(tmp_path / 'cap'),
                                  log=lambda s: None, **kw)


def test_driver_refusals_come_before_any_gpu_work(tmp_path):
  from nerfies_b200 import configs
  cap = tmp_path / 'cap'
  _Source(cap)
  timed = configs.ModelConfig(use_warp=True, warp_metadata_encoder_type='time', use_appearance_metadata=True)
  for kw, exc, msg in (
      (dict(item='x'), ValueError, "'x'"),
      (dict(), ValueError, 'one of --item'),
      (dict(item='a', image=str(cap / 'a.png')), ValueError, 'one of --item'),
      (dict(item='a', optimize=['pose', 'focal']), ValueError, 'unknown optimize'),
      (dict(item='a', optimize=['appearance'], model_config=configs.ModelConfig(use_warp=True)), ValueError,
       'no appearance'),
      (dict(item='a', optimize=['warp'], model_config=configs.ModelConfig()), ValueError, 'no warp field'),
      (dict(item='a', optimize=['warp'], model_config=timed), ValueError, 'function of time'),
      (dict(image=str(cap / 'small.png'), init_camera=str(cap / 'camera' / 'a.json')), ValueError, '40 x 20'),
      (dict(image=str(cap / 'a.png')), ValueError, '--init_camera'),
      (dict(item='a', steps=0), ValueError, 'steps'),
      (dict(item='a', batch_rays=0), ValueError, 'batch_rays'),
      (dict(item='a', metadata=['camera=1']), ValueError, '--metadata')):
    with pytest.raises(exc, match=msg):
      _register(tmp_path, **kw)
  # past the refusals: the missing checkpoint
  for kw in (dict(item='b'), dict(image=str(cap / 'a.png'), init_camera=str(cap / 'camera' / 'b.json')),
             dict(item='a', optimize=['pose', 'appearance'], model_config=timed, metadata=['appearance=1'])):
    with pytest.raises(FileNotFoundError, match='no checkpoints'):
      _register(tmp_path, **kw)


def test_driver_parser_defaults():
  from nerfies_b200 import register_camera
  args = register_camera.make_parser().parse_args(['--base_folder', '/x', '--item', 'a'])
  assert (args.item, args.image, args.init_camera, args.optimize, args.steps, args.batch_rays, args.seed,
          args.lr_decay) == ('a', None, None, 'pose,appearance', 200, 1024, 0, 1.0)
  assert args.lr_rotation == geometry.DEFAULT_LRS['rotation']
