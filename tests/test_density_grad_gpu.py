"""nfb_density_grad (geometry.density_gradient): the density of a level's NeRF MLP and its gradient with respect
to free points through the warp field, and what is built on it: geometry.normal_map,
visualization.normals_to_color and the drivers' normal outputs.

The gradient is held to torch.autograd of the oracle in float64 (O.warp_field_apply, O.nerf_mlp on the warped
point with O.get_condition_inputs, then sigma's activation) under the rule of test_ray_vjp_gpu.py: the largest
error, relative to the largest element of the reference, is at most max(2e-4, 3 x band), the band being the fp32
oracle's distance from fp64 on the same scale.  An analytic scene (sigma = relu(k (a.y - c)) behind a constant
rigid warp) pins the frames and the sign of the normals exactly.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import nerfies_oracle as O
from tests.golden_util import model_from_spec, spec_to_dict, tree_to_device
from tests.test_mesh import read_ply
from tests.test_render_vjp_gpu import DIMS, TOL, Case, _gin_spec, _golden_case, _small_spec

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAPTURE = os.path.join(ROOT, 'tests', 'golden', 'capture_small')


def _p(t):
  return None if t is None else ctypes.c_void_p(t.data_ptr())


def _points(spec, P, seed):
  """P points inside the scene's sampling range and per-point metadata (ids, a timestamp for 'time')."""
  gen = torch.Generator().manual_seed(seed)
  r = O.synthetic_rays(P, spec, seed=seed)
  z = spec.near + (spec.far - spec.near) * torch.rand(P, 1, generator=gen)
  md = dict(r['metadata'])
  if spec.use_warp and spec.warp_metadata_encoder_type == 'time':
    md['time'] = torch.rand(P, 1, generator=gen)
  return (r['origins'] + z * r['directions']).float(), md


def _oracle(c, pts, md, level, dtype, use_warp):
  """(sigma, grad_x sigma, warped points) of the oracle in `dtype`."""
  spec = c.spec
  p = O.tree_to(c.params, dtype)
  x = pts.to(dtype).clone().requires_grad_(True)
  y = x[:, None, :]
  if use_warp and spec.use_warp:
    meta = md['time'] if spec.warp_metadata_encoder_type == 'time' else md['warp']
    y = O.warp_field_apply(p['warp_field'], spec, y, meta[:, None, :], c.warp_alpha, False, c.time_alpha)
  P = pts.shape[0]
  viewdirs = torch.zeros(P, 3, dtype=dtype)
  viewdirs[:, 2] = 1.0
  tc, ac, rc = O.get_condition_inputs(p, spec, viewdirs, md)
  raw = O.nerf_mlp(p[f'nerf_mlps_{level}'], spec, O.sinusoidal_encode(y, spec.num_nerf_point_freqs), tc, ac, rc)
  sigma = O.activation_fn(spec.sigma_activation)(raw['alpha'][..., 0])[:, 0]
  (g,) = torch.autograd.grad(sigma.sum(), x)
  return sigma.detach().double(), g.double(), y.detach()[:, 0].double()


def _model(c, precision='fp32', batch=64):
  model = model_from_spec(spec_to_dict(c.spec), device=DEV, batch_size=batch)
  model.train_precision = precision
  return model


def _abi(model, c, pts, md, level, use_warp=True, flags=None):
  """nfb_density_grad called directly with per-point metadata -> (rc, sigma, grad, warped)."""
  spec = c.spec
  hd = model.handle()
  hd.set_params(tree_to_device(c.params, DEV))
  model._set_time_alpha(hd, c.time_alpha)
  P = pts.shape[0]
  x = pts.to(DEV).contiguous()
  time = spec.use_warp and spec.warp_metadata_encoder_type == 'time'
  wid = (md['time'].float() if time else md['warp'].int()).reshape(-1).to(DEV).contiguous()
  aid = md['appearance'].int().reshape(-1).to(DEV).contiguous() if spec.use_appearance_metadata else None
  if flags is None:
    flags = 0 if use_warp else 2
  out = [torch.full((P,), float('nan'), device=DEV), torch.full((P, 3), float('nan'), device=DEV),
         torch.full((P, 3), float('nan'), device=DEV)]
  rc = hd.lib.nfb_density_grad(hd.h, {'coarse': 0, 'fine': 1}[level], P, _p(x), _p(wid), _p(aid), float(c.warp_alpha),
                               flags, *[_p(t) for t in out], ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
  torch.cuda.synchronize()
  return rc, [t.cpu().double() for t in out]


def _rel(a, ref):
  return float((a - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)


def _check(name, c, level, use_warp=True, precision='fp32', P=300, batch=128, seed=0):
  model = _model(c, precision, batch)
  pts, md = _points(c.spec, P, seed)
  rc, (sigma, grad, warped) = _abi(model, c, pts, md, level, use_warp)
  assert rc == 0, model.handle().lib.nfb_last_error().decode()
  s64, g64, y64 = _oracle(c, pts, md, level, torch.float64, use_warp)
  s32, g32, y32 = _oracle(c, pts, md, level, torch.float32, use_warp)
  err, band = _rel(grad, g64), _rel(g32, g64)
  serr, sband = _rel(sigma, s64), _rel(s32, s64)
  print(f'{name} {level} {precision}: |grad| max {float(g64.abs().max()):.3g}, err {err:.2e} (band {band:.2e}); '
        f'sigma err {serr:.2e} (band {sband:.2e})')
  assert float(g64.abs().max()) > 0, 'the case has no gradient to check'
  assert err <= max(TOL, 3 * band), (name, level, err, band)
  assert serr <= max(TOL, 3 * sband), (name, level, serr, sband)
  assert _rel(warped, y64) <= max(1e-5, 3 * _rel(y32, y64)), name


_CASES = {
    'model_no_warp': lambda: Case(_small_spec(use_warp=False), 4, seed=1),
    'se3_alpha_condition': lambda: Case(_small_spec(), 4, seed=2),
    'se3_pivot': lambda: Case(_small_spec(warp_use_pivot=True), 4, seed=3),
    'se3_translation': lambda: Case(_small_spec(warp_use_translation=True), 4, seed=4),
    'se3_pivot_translation': lambda: Case(_small_spec(warp_use_pivot=True, warp_use_translation=True), 4, seed=5),
    'translation': lambda: _golden_case('translation_small'),
    'time': lambda: _golden_case('time_small'),
    'blend': lambda: _golden_case('blend_small'),
    'relu_sigma': lambda: Case(_small_spec(sigma_activation='relu'), 4, seed=6),
    'elu_hidden': lambda: Case(_small_spec(activation='elu'), 4, seed=7),
    'trunk_condition': lambda: Case(_small_spec(use_trunk_condition=True, use_alpha_condition=False), 4, seed=8),
}


@pytest.mark.parametrize('level', ['coarse', 'fine'])
@pytest.mark.parametrize('case', list(_CASES))
def test_gradient_vs_fp64(case, level):
  c = _CASES[case]()
  _check(case, c, level)


@pytest.mark.parametrize('level', ['coarse', 'fine'])
def test_call_without_warp(level):
  """NFB_FLAG_NO_WARP: the canonical field, J = I."""
  _check('call_no_warp', Case(_small_spec(), 4, seed=9), level, use_warp=False)


def test_coarse_only_model():
  c = Case(_small_spec(num_fine_samples=0), 4, seed=10)
  _check('coarse_only', c, 'coarse')
  rc, _ = _abi(_model(c), c, *_points(c.spec, 8, 0), 'fine')
  assert rc < 0


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('dims', ['quarterhd', 'vrig'])
def test_gin_dims(dims, precision):
  c = Case(_gin_spec(dims), 4, seed=20 + len(dims), warp_alpha=DIMS[dims]['alpha'])
  for level in ('coarse', 'fine'):
    _check(dims, c, level, precision=precision)


def test_chunks_agree():
  """300 points in chunks of 128 (two full chunks and a ragged one) give what one chunk of 300 gives."""
  c = Case(_small_spec(), 4, seed=11)
  pts, md = _points(c.spec, 300, 3)
  _, a = _abi(_model(c, batch=128), c, pts, md, 'fine')
  _, b = _abi(_model(c, batch=300), c, pts, md, 'fine')
  for x, y in zip(a, b):
    assert torch.equal(x, y)


def test_sigma_equals_density_grid():
  from nerfies_b200 import geometry
  c = Case(_small_spec(), 4, seed=12)
  model = _model(c, batch=64)
  params = tree_to_device(c.params, DEV)
  md = {'warp': 2, 'appearance': 1, 'camera': 0}
  extra = {'alpha': c.warp_alpha}
  box, shape = ((-0.4, -0.3, -0.35), (0.35, 0.4, 0.3)), (5, 6, 7)
  sp = geometry.grid_spacing(box, shape)
  axis = [np.float32(box[0][d]) + np.arange(n, dtype=np.float32) * sp[d] for d, n in enumerate(shape[::-1])]
  k, j, i = np.meshgrid(axis[2], axis[1], axis[0], indexing='ij')
  points = torch.from_numpy(np.stack([i, j, k], -1).reshape(-1, 3).astype(np.float32)).to(DEV)
  for use_warp in (True, False):
    for level in ('coarse', 'fine'):
      grid = geometry.density_grid(model, params, box, shape, extra, md, use_warp=use_warp, level=level)
      got = geometry.density_gradient(model, params, points, extra, md, use_warp=use_warp, level=level)
      assert got['sigma'].grad_fn is None and got['gradient'].grad_fn is None
      err = _rel(got['sigma'].double().cpu(), grid.reshape(-1).double().cpu())
      print(f'warp={use_warp} {level}: sigma vs density_grid {err:.2e}')
      assert err < 1e-5


def test_refusals():
  c = Case(_small_spec(), 4, seed=13)
  model = _model(c, batch=8)
  hd = model.handle()
  hd.set_params(tree_to_device(c.params, DEV))
  lib = hd.lib
  x = torch.rand(8, 3, device=DEV)
  g = torch.empty(8, 3, device=DEV)
  ids = torch.zeros(8, dtype=torch.int32, device=DEV)
  s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

  def call(h=hd.h, level=1, P=8, pts=x, flags=0, grad=g):
    return lib.nfb_density_grad(h, level, P, _p(pts), _p(ids), None, 4.0, flags, None, _p(grad), None, s)

  def err():
    return lib.nfb_last_error().decode()

  assert call() == 0
  assert call(P=0) == 0
  assert call(h=None) < 0 and 'null' in err()
  assert call(pts=None) < 0 and 'null' in err()
  assert call(grad=None) < 0 and 'grad_out' in err()
  assert call(P=-1) < 0 and 'P=-1' in err()
  assert call(level=2) < 0 and 'level 2' in err()
  assert call(flags=4) < 0 and 'METADATA_ENCODED' in err()
  assert call(flags=1) < 0 and 'flags' in err()
  assert call(flags=2) == 0
  fresh = _model(c, batch=8)
  assert lib.nfb_density_grad(fresh.handle().h, 1, 8, _p(x), _p(ids), None, 4.0, 0, None, _p(g), None, s) < 0
  assert 'nfb_set_params' in err()
  coarse = Case(_small_spec(num_fine_samples=0), 4, seed=14)
  cm = _model(coarse, batch=8)
  ch = cm.handle()
  ch.set_params(tree_to_device(coarse.params, DEV))
  assert lib.nfb_density_grad(ch.h, 1, 8, _p(x), _p(ids), None, 4.0, 0, None, _p(g), None, s) < 0
  assert 'coarse-only' in err()
  torch.cuda.synchronize()


# ---------------------------------------------------------------------------
# the analytic scene: sigma = relu(k (a.y - c)), y = R x + t (the SE(3) head biases alone)
# ---------------------------------------------------------------------------
K, C_PLANE, OFFSET = 50.0, 0.1, 10.0
A = np.array([0.48, -0.6, 0.64])                # unit
W0, V0 = [0.3, -0.2, 0.4], [0.1, 0.05, -0.1]


def _analytic():
  spec = O.OracleSpec(num_coarse_samples=64, num_fine_samples=64, near=0.1, far=3.0, nerf_trunk_depth=5,
                      nerf_trunk_width=64, nerf_rgb_branch_width=32, num_nerf_point_freqs=4, num_warp_freqs=2,
                      sigma_activation='relu', use_warp=True, warp_field_type='se3', warp_trunk_depth=3,
                      warp_trunk_width=32, num_warp_embeddings=2)
  zero = lambda t: {k: zero(v) for k, v in t.items()} if isinstance(t, dict) else torch.zeros_like(t)
  p = zero(O.init_params(spec))
  p['warp_field']['branches_w']['logit']['bias'] = torch.tensor(W0)
  p['warp_field']['branches_v']['logit']['bias'] = torch.tensor(V0)
  for lv in ('coarse', 'fine'):
    m = p[f'nerf_mlps_{lv}']
    m['MLP_0']['hidden_0']['kernel'][0:3, 0] = torch.tensor(A, dtype=torch.float32)
    m['MLP_0']['hidden_0']['bias'][0] = OFFSET           # a.y + OFFSET > 0 in the scene: relu passes it on
    for i in range(1, spec.nerf_trunk_depth):
      m['MLP_0'][f'hidden_{i}']['kernel'][0, 0] = 1.0
    m['MLP_2']['logit']['kernel'][0, 0] = K
    m['MLP_2']['logit']['bias'][0] = -K * (OFFSET + C_PLANE)
  c = Case(spec, 4, seed=0, params=p)
  # y = R x + t in fp64, from the oracle's SE(3) tail
  w, v = torch.tensor([W0], dtype=torch.float64), torch.tensor([V0], dtype=torch.float64)
  basis = torch.cat([torch.zeros(1, 3), torch.eye(3)]).double()
  y = O.se3_tail(w.expand(4, 3), v.expand(4, 3), basis)
  t = y[0].numpy()
  R = (y[1:] - y[0]).numpy().T
  return c, R, t


def _look_at_camera(axis, position, size=(32, 24), focal=30.0):
  from nerfies_b200 import camera as camera_lib
  z = axis / np.linalg.norm(axis)
  up = np.array([0.0, 0.0, 1.0]) if abs(z[2]) < 0.9 else np.array([1.0, 0.0, 0.0])
  x = np.cross(up, z)
  x /= np.linalg.norm(x)
  y = np.cross(z, x)
  return camera_lib.Camera(np.stack([x, y, z]), position, focal, (size[0] / 2, size[1] / 2), size)


def test_analytic_scene():
  from nerfies_b200 import evaluation, geometry, visualization
  c, R, t = _analytic()
  model = _model(c, batch=256)
  params = tree_to_device(c.params, DEV)
  extra, md = {'alpha': c.warp_alpha}, {'warp': 0}
  u = R.T @ A                                  # the plane u.x = c' in the observation space
  cp = C_PLANE - A @ t
  n_expect = -u / np.linalg.norm(u)
  # free points on both sides
  gen = torch.Generator().manual_seed(0)
  pts = (torch.rand(500, 3, generator=gen) - 0.5) * 2.0
  side = pts.double().numpy() @ u - cp
  got = geometry.density_gradient(model, params, pts, extra, md)
  g = got['gradient'].double().cpu().numpy()
  inside, outside = side > 1e-3, side < -1e-3
  np.testing.assert_allclose(g[inside], np.broadcast_to(K * u, g[inside].shape), rtol=0, atol=1e-5 * K)
  assert np.all(g[outside] == 0)
  np.testing.assert_allclose(got['sigma'].cpu().numpy()[inside], K * side[inside], rtol=1e-4, atol=1e-3)
  np.testing.assert_allclose(got['warped_points'].double().cpu().numpy(), pts.double().numpy() @ R.T + t, atol=1e-5)

  q = u * cp / (u @ u)                         # a point on the plane
  # a camera looking straight at the plane: every pixel sees it, facing the camera
  cam = _look_at_camera(u, q - 1.5 * u / np.linalg.norm(u))
  render = evaluation.render_frame(model, params, cam, extra, md)
  nm = geometry.normal_map(model, params, cam, render['med_depth'], extra, md)
  assert bool(nm['valid'].all())
  err = float((nm['normals'].double().cpu() - torch.from_numpy(n_expect)).abs().max())
  print(f'facing camera: normal error {err:.2e}')
  assert err < 1e-5
  color = visualization.normals_to_color(nm['normals'], nm['valid'], cam).cpu().numpy().astype(int)
  assert np.all(np.abs(color - np.array([127.5, 127.5, 255])) <= 1), np.unique(color.reshape(-1, 3), axis=0)

  # a camera looking along the plane from its empty side: rays that reach the plane before far are valid
  along = np.cross(u, [1.0, 0.0, 0.0])
  pos = q - 0.3 * u / np.linalg.norm(u)
  cam = _look_at_camera(along, pos, size=(40, 30), focal=12.0)
  render = evaluation.render_frame(model, params, cam, extra, md)
  nm = geometry.normal_map(model, params, cam, render['med_depth'], extra, md)
  from nerfies_b200 import camera as camera_lib
  rays = camera_lib.camera_to_rays(cam, DEV)
  d = rays['directions'].double().cpu().numpy()
  o = rays['origins'].double().cpu().numpy()
  ud = d @ u
  s_hit = np.where(ud > 0, (cp - o @ u) / np.where(ud > 0, ud, 1.0), np.inf)
  valid = nm['valid'].cpu().numpy()
  sure_hit = s_hit < c.spec.far - 0.3
  sure_miss = s_hit > c.spec.far + 0.05
  assert sure_hit.any() and sure_miss.any()
  assert np.all(valid[sure_hit]) and not np.any(valid[sure_miss])
  normals = nm['normals'].double().cpu().numpy()
  assert np.abs(normals[valid] - n_expect).max() < 1e-5
  assert np.all(normals[~valid] == 0)
  color = visualization.normals_to_color(nm['normals'], nm['valid'], cam).cpu().numpy()
  assert np.all(color[~valid] == 0)


# ---------------------------------------------------------------------------
# the drivers on the small capture
# ---------------------------------------------------------------------------
GIN = """
ExperimentConfig.image_scale = 2
ModelConfig.num_coarse_samples = 16
ModelConfig.num_fine_samples = 16
ModelConfig.use_warp = True
ModelConfig.warp_field_type = 'se3'
ModelConfig.use_appearance_metadata = True
ModelConfig.num_nerf_point_freqs = 2
ModelConfig.num_warp_freqs = 2
TrainConfig.batch_size = 512
TrainConfig.max_steps = 7
EvalConfig.num_val_eval = None
EvalConfig.num_train_eval = 1
EvalConfig.num_test_eval = 1
"""


@pytest.fixture(scope='module')
def checkpoint(tmp_path_factory):
  """A checkpoint of trained-like random parameters for the small capture."""
  from nerfies_b200 import checkpoints, configs, driver_utils, model_utils, models
  tmp = tmp_path_factory.mktemp('normals_drivers')
  gin = tmp / 'test.gin'
  gin.write_text(GIN)
  configs.clear_config()
  configs.parse_config_files_and_bindings([str(gin)])
  model_config = configs.ModelConfig(use_stratified_sampling=False)
  source = driver_utils.make_datasource(configs.ExperimentConfig(), model_config, CAPTURE)
  model, params = models.construct_nerf(0, model_config, 4096, source.appearance_ids, source.camera_ids,
                                        source.warp_ids, near=source.near, far=source.far, precision='fp32')
  cpu = lambda t: {k: cpu(v) for k, v in t.items()} if isinstance(t, dict) else t.detach().cpu()
  params = O.make_trained_like(cpu(params), seed=5)
  state = model_utils.TrainState(model_utils.Optimizer({'model': params}), warp_alpha=3.0)
  checkpoints.save_checkpoint(str(tmp / 'exp' / 'checkpoints'), state, 7)
  configs.clear_config()
  yield tmp / 'exp', str(gin), model, tree_to_device(params, DEV), source
  configs.clear_config()


def _argv(base, gin, *more):
  return ['--base_folder', str(base), '--data_dir', CAPTURE, '--gin_configs', gin, '--precision', 'fp32', *more]


def _expected_normals(model, params, camera, extra, md):
  from nerfies_b200 import evaluation, geometry, visualization
  render = evaluation.render_frame(model, params, camera, extra, md)
  nm = geometry.normal_map(model, params, camera, render['med_depth'], extra, md)
  return visualization.normals_to_color(nm['normals'], nm['valid'], camera).cpu().numpy(), nm, render


def test_eval_save_normals(checkpoint):
  from nerfies_b200 import configs, datasets, eval as eval_lib
  base, gin, model, params, source = checkpoint
  configs.clear_config()
  assert eval_lib.main(_argv(base, gin, '--eval_once', '--save_normals'), poll_seconds=0.0) == 0
  out = base / 'renders' / '00000007'
  extra = {'alpha': 3.0, 'time_alpha': 0.0}
  assert 'normals_000.png' in os.listdir(out / 'test')
  for item_id in source.val_ids:
    got = datasets.decode_image(out / 'val' / f'normals_{item_id}.png')
    item = source.get_item(item_id)
    want, nm, render = _expected_normals(model, params, source.load_camera(item_id), extra, item['metadata'])
    assert got.shape == tuple(render['rgb'].shape)
    np.testing.assert_array_equal(got, want)
    invalid = ~nm['valid'].cpu().numpy()
    assert np.all(got[invalid] == 0)
    print(f'{item_id}: {int((~invalid).sum())} of {invalid.size} pixels have a normal')
  configs.clear_config()


def test_render_video_normals(checkpoint):
  import cv2
  from nerfies_b200 import configs, datasets, render_video
  base, gin, model, params, source = checkpoint
  configs.clear_config()
  assert render_video.main(_argv(base, gin, '--camera_path', 'camera-paths/orbit-extreme', '--normals')) == 0
  out = base / 'videos' / 'orbit-extreme' / '00000007'
  assert sorted(os.listdir(out)) == ['frame_00000.png', 'frame_00001.png', 'frame_00002.png', 'normals.mp4',
                                     'normals_00000.png', 'normals_00001.png', 'normals_00002.png', 'video.mp4']
  paths = source.glob_cameras(os.path.join(CAPTURE, 'camera-paths', 'orbit-extreme'))
  extra = {'alpha': 3.0, 'time_alpha': 0.0}
  for i, path in enumerate(paths):
    got = datasets.decode_image(out / f'normals_{i:05d}.png')
    want, nm, _ = _expected_normals(model, params, source.load_camera(path), extra, {'appearance': 0, 'warp': 0})
    assert got.shape == (27, 48, 3)
    np.testing.assert_array_equal(got, want)
    assert np.all(got[~nm['valid'].cpu().numpy()] == 0)
  video = cv2.VideoCapture(str(out / 'normals.mp4'))
  count = 0
  while video.read()[0]:
    count += 1
  assert count == 3
  configs.clear_config()


def test_extract_mesh_analytic_normals(checkpoint):
  from nerfies_b200 import configs, extract_mesh, geometry
  base, gin, model, params, source = checkpoint
  box, shape = extract_mesh.grid_for_box(extract_mesh.scene_box(CAPTURE), 48)
  md = {'appearance': 0, 'warp': 0}
  extra = {'alpha': 3.0, 'time_alpha': 0.0}
  level = float(geometry.density_grid(model, params, box, shape, extra, md).median())
  argv = _argv(base, gin, '--resolution', '48', '--threshold', repr(level))
  path = base / 'meshes' / '00000007' / 'warp_0.ply'
  configs.clear_config()
  assert extract_mesh.main(argv) == 0
  grid_mesh = read_ply(path)
  configs.clear_config()
  assert extract_mesh.main(argv + ['--analytic_normals', '--colors']) == 0
  mesh = read_ply(path)
  np.testing.assert_array_equal(mesh['vertices'], grid_mesh['vertices'])
  np.testing.assert_array_equal(mesh['faces'], grid_mesh['faces'])
  n, ng = mesh['normals'].astype(np.float64), grid_mesh['normals'].astype(np.float64)
  assert len(n) > 100
  assert np.abs(np.linalg.norm(n, axis=-1) - 1).max() < 1e-5
  agree = float(np.mean((n * ng).sum(-1) > 0))
  print(f'{len(n)} vertices; analytic and grid normals agree in sign on {agree:.1%}')
  assert agree >= 0.9
  # and the density falls along them: sigma one step of 1e-3 outside below sigma one step inside
  v = torch.from_numpy(mesh['vertices']).to(DEV)
  step = 1e-3 * torch.from_numpy(n.astype(np.float32)).to(DEV)
  out = geometry.density_gradient(model, params, v + step, extra, md)['sigma']
  inside = geometry.density_gradient(model, params, v - step, extra, md)['sigma']
  falls = float((out < inside).float().mean())
  print(f'sigma falls along the analytic normal at {falls:.1%} of the vertices')
  assert falls >= 0.99
  # the same normals from the library
  want, kept = extract_mesh.analytic_normals(model, params, torch.from_numpy(mesh['vertices']).to(DEV),
                                             torch.from_numpy(ng.astype(np.float32)).to(DEV), extra, md, True,
                                             'fine')
  np.testing.assert_array_equal(n.astype(np.float32), want.cpu().numpy())
  configs.clear_config()
