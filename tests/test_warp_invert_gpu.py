"""Inverting the warp field (nfb_warp_invert, geometry.invert_warp / track_surface) and the mesh driver's --track.

- Rigid warps (SE(3) and translation fields whose heads are a constant) against the closed form in fp64.
- make_trained_like warps at the quarterhd and vrig fixture sizes with each metadata encoder, in both training
  precisions, against the fp64 oracle's warp at the returned points; with the head scaled so that
  ||J - I|| < 1/2 on the sampled box, nearly every point converges.
- A designed piecewise-linear translation warp with a flat and a folded region: failures are reported.
- Determinism across calls, chunk sizes and iteration counts; argument errors.
- A plane under a rigid warp, and the driver end to end on the small capture.
"""
import ctypes
import dataclasses

import numpy as np
import pytest
import torch

from oracle import nerfies_oracle as O
from tests.golden_util import Golden, model_from_spec, spec_to_dict, tree_to_device
from tests.test_mesh import read_ply
from tests.test_mesh_gpu import CAPTURE, checkpoint  # noqa: F401  (the trained-like checkpoint fixture)
from tests.test_render_extremes_gpu import designed_params

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
PRECS = ['fp32', 'tf32x3']
CONVERGED, MAX_ITERS, SINGULAR, STALLED, NONFINITE = range(5)
# The kernels' fp32 warp against the fp64 oracle's at the same point, in scene units (|x| <= 0.5).
W_BAND = 1e-5


def _model(spec, prec='fp32', batch_size=256):
  m = model_from_spec(spec_to_dict(spec), device=DEV, batch_size=batch_size)
  m.train_precision = prec
  return m


def _zero(t):
  return {k: _zero(v) for k, v in t.items()} if isinstance(t, dict) else torch.zeros_like(t)


def _points(P, seed, lo=-0.3, hi=0.3):
  gen = torch.Generator().manual_seed(seed)
  return torch.rand(P, 3, generator=gen) * (hi - lo) + lo


def _oracle_warp(params, spec, points, md, alpha, time_alpha=None):
  """fp64 warp_field_apply at `points` (P,3) for the scalar metadata md."""
  P = points.shape[0]
  if spec.warp_metadata_encoder_type == 'time':
    meta = torch.full((P, 1), float(md['time']), dtype=torch.float64)
  else:
    meta = torch.full((P, 1), int(md['warp']), dtype=torch.int64)
  p64 = O.tree_to(params, torch.float64)['warp_field']
  return O.warp_field_apply(p64, spec, points.double(), meta, alpha, time_alpha=time_alpha).detach()


def _invert(model, params, targets, md, extra, **kw):
  from nerfies_b200 import geometry
  out = geometry.invert_warp(model, tree_to_device(params, DEV), targets.to(DEV), extra, md, **kw)
  torch.cuda.synchronize()
  return {k: v.cpu() for k, v in out.items()}


# ---------------------------------------------------------------------------
# 1. Rigid warps: closed form
# ---------------------------------------------------------------------------
SCREW_W, SCREW_V = [0.3, -0.5, 0.2], [0.1, 0.05, -0.2]
PIVOT, TRANS = [0.05, -0.02, 0.04], [-0.03, 0.06, 0.01]


def _f64(v):
  return torch.tensor(v, dtype=torch.float32).double()


def _rigid(warp_type, pivot=False, trans=False):
  """A spec whose warp is W(x) = R x + t exactly (head kernels 0, head biases the motion) and (R, t) in fp64."""
  spec = O.OracleSpec(num_coarse_samples=8, num_fine_samples=0, near=0.02, far=0.83, nerf_trunk_depth=2,
                      nerf_trunk_width=32, nerf_rgb_branch_width=16, use_appearance_metadata=False, use_warp=True,
                      warp_field_type=warp_type, warp_trunk_depth=3, warp_trunk_width=32, num_warp_embeddings=3,
                      warp_use_pivot=pivot, warp_use_translation=trans)
  params = O.make_trained_like(O.init_params(spec, 1), seed=2)
  R, t = _rigid_heads(params['warp_field'], pivot, trans)
  return spec, params, R, t


def _rigid_heads(wf, pivot, trans):
  """Sets the heads of the warp field `wf` (in place) to a constant motion; returns its (R, t) in fp64."""
  if 'mlp' in wf:
    wf['mlp']['logit']['kernel'].zero_()
    wf['mlp']['logit']['bias'][:] = torch.tensor(TRANS)
    R, t = torch.eye(3, dtype=torch.float64), _f64(TRANS)
  else:
    for name, v in (('w', SCREW_W), ('v', SCREW_V), ('p', PIVOT), ('t', TRANS)):
      if f'branches_{name}' in wf:
        wf[f'branches_{name}']['logit']['kernel'].zero_()
        wf[f'branches_{name}']['logit']['bias'][:] = torch.tensor(v)
    w, v = _f64(SCREW_W), _f64(SCREW_V)
    theta = torch.linalg.norm(w)
    R, t = O.exp_se3(torch.cat([w / theta, v / theta]), theta)
    if pivot:
      t = t + R @ _f64(PIVOT) - _f64(PIVOT)
    if trans:
      t = t + _f64(TRANS)
  return R, t


@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('case', ['se3', 'se3-pivot', 'se3-translation', 'se3-pivot-translation', 'translation'])
def test_rigid_warps_match_the_closed_form(case, prec):
  spec, params, R, t = _rigid(case.split('-')[0], 'pivot' in case, 'translation' in case[3:])
  model = _model(spec, prec)
  y = _points(300, 1)
  tol = 1e-5
  out = _invert(model, params, y, {'warp': 1}, {'alpha': 3.0}, max_iters=3, tol=tol, return_jacobian=True)
  want = ((y.double() - t) @ R)                                 # R^T (y - t), row vectors
  err = (out['points'].double() - want).norm(dim=-1)
  print(f'{case} {prec}: max |x - R^T(y - t)| {float(err.max()):.2e}, max residual {float(out["residual"].max()):.2e}')
  assert bool((out['status'] == CONVERGED).all()), out['status'].unique()
  assert float(out['residual'].max()) <= tol
  assert float(err.max()) <= tol + W_BAND
  assert float((out['jacobian'].double() - R).abs().max()) < 1e-6


# ---------------------------------------------------------------------------
# 2. Nonlinear warps against the fp64 oracle
# ---------------------------------------------------------------------------
def _nonlinear(name):
  """(spec, make_trained_like params, metadata, warp_extra) at a fixture's size with one encoder."""
  if name == 'quarterhd-glo':
    spec = Golden('quarterhd_dims').spec
    md, extra = {'warp': 3}, {'alpha': 8.0}
  elif name == 'quarterhd-blend':
    spec = dataclasses.replace(Golden('quarterhd_dims').spec, warp_field_type='translation',
                               warp_metadata_encoder_type='blend', num_warp_embeddings=20)
    md, extra = {'warp': 7}, {'alpha': 8.0, 'time_alpha': 0.4}
  else:                                                       # vrig: 256-wide SE(3) trunk, 'time' encoder
    spec = O.OracleSpec(num_coarse_samples=128, num_fine_samples=0, near=0.02, far=0.83, num_nerf_point_freqs=8,
                        num_warp_freqs=6, sigma_activation='softplus', use_warp=True, warp_field_type='se3',
                        warp_trunk_width=256, use_appearance_metadata=False, use_camera_metadata=True,
                        num_warp_embeddings=50, num_camera_embeddings=2, warp_metadata_encoder_type='time',
                        metadata_encoder_num_freqs=3)
    md, extra = {'time': 0.37}, {'alpha': 4.5, 'time_alpha': 2.5}
  params = O.make_trained_like(O.init_params(spec, 11), seed=12)
  return spec, params, md, extra


def _scale_head(params, s):
  """The warp field's output layer (SE(3) branches or translation head) times s."""
  def rec(t, path):
    if isinstance(t, dict):
      return {k: rec(v, path + (k,)) for k, v in t.items()}
    head = len(path) == 4 and path[0] == 'warp_field' and path[2] == 'logit' and (
        path[1] == 'mlp' or path[1].startswith('branches_'))
    return t * s if head else t
  return rec(params, ())


def _jacobian(model, params, points, md, extra):
  from nerfies_b200 import geometry
  wf = model.create_warp_field(model, num_batch_dims=1)
  P = points.shape[0]
  meta = geometry._warp_ids(model, md, P).reshape(P, 1)
  out = wf.apply({'params': tree_to_device(params, DEV)['warp_field']}, points.to(DEV), meta, extra,
                 return_jacobian=True)
  return out['jacobian'].cpu().double()


def _dist_from_identity(J):
  return float(torch.linalg.matrix_norm(J - torch.eye(3, dtype=J.dtype), ord=2).max())


@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('name', ['quarterhd-glo', 'quarterhd-blend', 'vrig-time'])
def test_nonlinear_warps_against_the_oracle(name, prec):
  spec, params, md, extra = _nonlinear(name)
  model = _model(spec, prec)
  tol = 1e-5
  box = _points(4096, 5)
  # ||J - I|| is close to linear in the head's scale: aim at 0.35
  s, d = 1.0, _dist_from_identity(_jacobian(model, params, box, md, extra))
  for _ in range(3):
    s *= 0.35 / d
    scaled = _scale_head(params, s)
    d = _dist_from_identity(_jacobian(model, scaled, box, md, extra))
    if 0.25 < d < 0.45:
      break
  assert d < 0.5, d
  y = _points(3000, 6, -0.25, 0.25)
  for what, p in (('trained-like', params), (f'head x {s:.3g}', scaled)):
    out = _invert(model, p, y, md, extra, max_iters=16, tol=tol)
    conv = out['status'] == CONVERGED
    ref = _oracle_warp(p, spec, out['points'], md, extra['alpha'], extra.get('time_alpha'))
    res64 = (ref - y.double()).norm(dim=-1)
    moved = float((out['points'] - y).norm(dim=-1).max())
    print(f'{name} {prec} {what} (|J - I| <= {d:.3f}): {int(conv.sum())}/{len(y)} converged, max |x - y| '
          f'{moved:.3g}, max fp64 residual of the converged {float(res64[conv].max()):.2e}')
    assert float(res64[conv].max()) <= tol + W_BAND
    assert float((out['residual'].double() - res64).abs().max()) <= W_BAND
    assert float(conv.double().mean()) >= 0.999, out['status'].bincount()


# ---------------------------------------------------------------------------
# 3. Failure is reported, never hidden
# ---------------------------------------------------------------------------
# At warp_alpha = 0 the warp's encoding is the point itself: a translation field whose first layer holds
# relu(u - knot_k) of u = x_0 and whose output is t_0 = sum_k c_k h_k moves x_0 to g(u) = u + t_0:
#   u < -0.1: g = u;   -0.1 .. 0: slope -1 (a fold);   0 .. 0.3: slope 1;   u > 0.3: g = 0.1 (flat).
# So targets with y_0 > 0.1 have no preimage and those with y_0 in (-0.2, -0.1) have three.
KNOTS, SLOPES = [-0.1, 0.0, 0.3], [-2.0, 2.0, -1.0]


def _designed_translation():
  spec = O.OracleSpec(num_coarse_samples=8, num_fine_samples=0, near=0.02, far=0.83, nerf_trunk_depth=2,
                      nerf_trunk_width=32, nerf_rgb_branch_width=16, use_appearance_metadata=False, use_warp=True,
                      warp_field_type='translation', warp_trunk_depth=2, warp_trunk_width=32, num_warp_embeddings=2)
  params = O.init_params(spec, 3)
  mlp = params['warp_field']['mlp'] = _zero(params['warp_field']['mlp'])
  K = len(KNOTS)
  u = torch.arange(K)
  mlp['hidden_0']['kernel'][0, u] = 1.0
  mlp['hidden_0']['bias'][:K] = -torch.tensor(KNOTS)
  mlp['hidden_1']['kernel'][u, u] = 1.0
  mlp['logit']['kernel'][u, 0] = torch.tensor(SLOPES)
  return spec, params


def _g(u):
  return u + sum(c * np.maximum(u - k, 0.0) for k, c in zip(KNOTS, SLOPES))


@pytest.mark.parametrize('prec', PRECS)
def test_failures_are_reported(prec):
  spec, params = _designed_translation()
  model = _model(spec, prec)
  tol = 1e-5
  y = _points(4000, 9, -0.4, 0.4)
  y[:8, 0] = torch.tensor([0.1 + 10 * tol, 0.15, 0.35, -0.15, -0.12, -0.18, 0.05, -0.3])
  extra = {'alpha': 0.0}
  out = _invert(model, params, y, {'warp': 1}, extra, max_iters=16, tol=tol)
  x = out['points'].double()
  np.testing.assert_allclose(_g(x[:, 0].numpy()) - x[:, 0].numpy(),
                             (_oracle_warp(params, spec, x, {'warp': 1}, 0.0) - x)[:, 0].numpy(), atol=1e-7)
  res64 = (_oracle_warp(params, spec, x, {'warp': 1}, 0.0) - y.double()).norm(dim=-1)
  status = out['status']
  none = y[:, 0] >= 0.1 + 10 * tol
  counts = {k: int((status == v).sum()) for k, v in (('converged', CONVERGED), ('max_iters', MAX_ITERS),
                                                      ('singular', SINGULAR), ('stalled', STALLED))}
  print(f'{prec}: {counts}; without a preimage: {int(none.sum())}, statuses {status[none].unique().tolist()}')
  assert not bool((status[none] == CONVERGED).any())
  assert int((status[none] == SINGULAR).sum()) + int((status[none] == STALLED).sum()) > 0
  assert float((out['residual'].double() - res64).abs().max()) <= W_BAND
  conv = status == CONVERGED
  assert float(res64[conv].max()) <= tol + W_BAND
  # the frozen non-converged points hold a residual at least the distance to the range of g
  assert float((res64[none] - (y[none, 0].double() - 0.1)).min()) >= -W_BAND
  # a start with no finite residual
  bad = y[:4].clone()
  init = bad.clone()
  init[1, 2] = float('nan')
  init[3, 0] = float('inf')
  out = _invert(model, params, bad, {'warp': 1}, extra, init=init, max_iters=4, tol=tol)
  assert out['status'][1] == NONFINITE and out['status'][3] == NONFINITE
  assert not torch.isfinite(out['residual'][[1, 3]]).any()


# ---------------------------------------------------------------------------
# 4. Determinism, chunking, iteration counts, arguments
# ---------------------------------------------------------------------------
def _small():
  spec, params, md, extra = _nonlinear('quarterhd-glo')
  spec = dataclasses.replace(spec, warp_trunk_width=64, nerf_trunk_width=64, num_coarse_samples=16,
                             num_fine_samples=0)
  params = O.make_trained_like(O.init_params(spec, 4), seed=5)
  return spec, params, md, extra


@pytest.mark.parametrize('prec', PRECS)
def test_determinism_and_chunking(prec):
  spec, params, md, extra = _small()
  model = _model(spec, prec, batch_size=64)
  R = model.handle().max_rays
  assert R == 64
  P = int(2.5 * R)
  y = _points(P, 13)
  init = y + 0.01 * torch.randn(P, 3, generator=torch.Generator().manual_seed(1))
  kw = dict(max_iters=6, tol=1e-5, return_jacobian=True)
  full = _invert(model, params, y, md, extra, init=init, **kw)
  again = _invert(model, params, y, md, extra, init=init, **kw)
  for k in full:
    assert torch.equal(full[k], again[k]), k
  for n in (1, R - 1, R + 1, P):
    part = _invert(model, params, y[:n], md, extra, init=init[:n], **kw)
    for k in full:
      assert torch.equal(part[k], full[k][:n]), (n, k)
  # a converged point is frozen: 2k iterations give the k-iteration result bitwise
  k4 = _invert(model, params, y, md, extra, max_iters=4, tol=1e-5, return_jacobian=True)
  k8 = _invert(model, params, y, md, extra, max_iters=8, tol=1e-5, return_jacobian=True)
  conv = k4['status'] == CONVERGED
  print(f'{prec}: statuses after 4 iterations {k4["status"].bincount(minlength=5).tolist()}, after 8 '
        f'{k8["status"].bincount(minlength=5).tolist()}')
  assert 0 < int(conv.sum())
  for k in k4:
    assert torch.equal(k4[k][conv], k8[k][conv]), k


def test_argument_errors():
  from nerfies_b200 import geometry
  spec, params, md, extra = _small()
  model = _model(spec, batch_size=64)
  geometry.invert_warp(model, tree_to_device(params, DEV), torch.zeros(0, 3), extra, md)       # P = 0: a no-op
  hd = model.handle()
  lib = hd.lib
  y = torch.zeros(5, 3, device=DEV)
  o3, o1 = torch.empty(5, 3, device=DEV), torch.empty(5, device=DEV)
  ids = torch.ones(5, dtype=torch.int32, device=DEV)
  p = lambda t: ctypes.c_void_p(t.data_ptr())

  def call(P=5, targets=p(y), iters=8, tol=1e-5, pts=p(o3), res=p(o1)):
    return lib.nfb_warp_invert(hd.h, P, targets, None, p(ids), 0.0, iters, tol, pts, res, None, None, None)

  assert call(P=0) == 0
  for kw, msg in ((dict(targets=None), b'null'), (dict(pts=None), b'null'), (dict(res=None), b'null'),
                  (dict(P=-1), b'P must be'),
                  (dict(iters=0), b'max_iters'), (dict(iters=65), b'max_iters'), (dict(tol=0.0), b'tol'),
                  (dict(tol=-1.0), b'tol'), (dict(tol=float('nan')), b'tol'), (dict(tol=float('inf')), b'tol')):
    assert call(**kw) != 0, kw
    assert msg in lib.nfb_last_error(), (kw, lib.nfb_last_error())
  with pytest.raises(ValueError, match='targets'):
    geometry.invert_warp(model, tree_to_device(params, DEV), torch.zeros(4, 2), extra, md)
  with pytest.raises(ValueError, match='init'):
    geometry.invert_warp(model, tree_to_device(params, DEV), torch.zeros(4, 3), extra, md, init=torch.zeros(3, 3))
  # no warp field: refused by the library and by the wrapper
  flat = dataclasses.replace(spec, use_warp=False)
  nowarp = _model(flat, batch_size=64)
  hn = nowarp.handle()
  hn.set_params(tree_to_device({k: v for k, v in params.items() if k != 'warp_field'}, DEV))
  assert lib.nfb_warp_invert(hn.h, 5, p(y), None, None, 0.0, 8, 1e-5, p(o3), p(o1), None, None, None) != 0
  assert b'no warp field' in lib.nfb_last_error()
  with pytest.raises(ValueError, match='warp field'):
    geometry.invert_warp(nowarp, params, y, extra, md)


# ---------------------------------------------------------------------------
# 5. A plane carried by a rigid warp
# ---------------------------------------------------------------------------
@pytest.mark.parametrize('prec', PRECS)
def test_tracked_plane(prec):
  from nerfies_b200 import geometry
  spec = O.OracleSpec(num_coarse_samples=16, num_fine_samples=0, near=0.02, far=0.83, num_nerf_point_freqs=8,
                      sigma_activation='relu', use_appearance_metadata=False, use_warp=True, warp_field_type='se3',
                      num_warp_embeddings=3, warp_use_pivot=True)
  # sigma = 10 relu(x_z + 0.21): the surface {sigma > 1} is the plane z = -0.11, outward normal -z
  params = designed_params(spec, knots=[-0.21], alpha_w=[10.0], alpha_b=0.0, rgb_w=[[1.0, 0.0, 0.0]],
                           rgb_b=[0.0, 0.0, 0.0])
  R, t = _rigid_heads(params['warp_field'], pivot=True, trans=False)
  model = _model(spec, prec, batch_size=256)
  dp = tree_to_device(params, DEV)
  box = ((-0.3, -0.3, -0.3), (0.3, 0.3, 0.3))
  md, extra = {'warp': 2}, {'alpha': 3.0}
  grid = geometry.density_grid(model, dp, box, (13, 13, 13), extra, md, use_warp=False, level='coarse')
  v, f, n = geometry.marching_cubes(grid, 1.0, box)
  assert len(v) > 100 and float((v[:, 2] + 0.11).abs().max()) < 1e-5
  tol = 1e-5
  out = geometry.track_surface(model, dp, v, n, extra, md, tol=tol)
  assert bool((out['status'] == CONVERGED).all()) and out['folded'] == 0
  x = out['vertices'].cpu().double()
  assert float((x - (v.cpu().double() - t) @ R).norm(dim=-1).max()) <= tol + W_BAND
  # on the moved plane: (R x + t)_z = -0.11
  dist = (x @ R.T + t)[:, 2] + 0.11
  want_n = n.cpu().double() @ R                                  # R^T n, row vectors
  print(f'{prec}: {len(v)} vertices, max distance from the moved plane {float(dist.abs().max()):.2e}, max normal '
        f'error {float((out["normals"].cpu().double() - want_n).abs().max()):.2e}')
  assert float(dist.abs().max()) <= tol + 2e-5
  assert float((out['normals'].cpu().double() - want_n).abs().max()) <= 1e-5
  assert out['vertices'].shape == v.shape and f.shape[1] == 3


# ---------------------------------------------------------------------------
# 6. The driver end to end
# ---------------------------------------------------------------------------
def test_extract_mesh_track_end_to_end(checkpoint):  # noqa: F811
  from nerfies_b200 import configs, extract_mesh, geometry
  base, gin, model, params, source = checkpoint
  box, shape = extract_mesh.grid_for_box(extract_mesh.scene_box(CAPTURE), 32)
  canon = geometry.density_grid(model, params, box, shape, {'alpha': 3.0}, {'appearance': 0, 'warp': 0},
                                use_warp=False)
  level = float(canon.median())
  argv = ['--base_folder', str(base), '--data_dir', CAPTURE, '--gin_configs', gin, '--precision', 'fp32',
          '--resolution', '32', '--threshold', repr(level), '--track']
  configs.clear_config()
  assert extract_mesh.main(argv + ['--colors']) == 0
  out = base / 'meshes' / '00000007' / 'track'
  can = read_ply(out / 'canonical.ply')
  cv, cf, cn = geometry.marching_cubes(canon, level, box)
  np.testing.assert_array_equal(can['vertices'], cv.cpu().numpy())
  np.testing.assert_array_equal(can['faces'], cf.cpu().numpy())
  npz = dict(np.load(out / 'track.npz'))
  frames = list(range(len(source.warp_ids)))
  T, V, F = len(frames), len(cv), len(cf)
  assert F > 50 and npz['frames'].tolist() == frames
  assert npz['faces'].shape == (F, 3) and np.array_equal(npz['faces'], can['faces'])
  assert npz['vertices'].shape == (T, V, 3) and npz['vertices'].dtype == np.float32
  assert npz['residual'].shape == (T, V) and npz['status'].shape == (T, V) and npz['status'].dtype == np.uint8
  for i, fr in enumerate(frames):
    ply = read_ply(out / f'warp_{fr}.ply')
    assert np.array_equal(ply['faces'], can['faces']) and len(ply['vertices']) == V
    np.testing.assert_array_equal(ply['vertices'], npz['vertices'][i])
    assert ply['colors'].shape == (V, 3) and ply['normals'].shape == (V, 3)
  conv = npz['status'] == CONVERGED
  print(f'{T} frames x {V} vertices: {conv.mean():.4%} converged, max residual {npz["residual"][conv].max():.2e}')
  assert conv.mean() > 0.99
  tol = extract_mesh.TRACK_TOL_VOXELS * float(geometry.grid_spacing(box, shape)[0])
  assert npz['residual'][conv].max() <= tol
  # the first frame from the template, as geometry.track_surface gives it
  first = geometry.track_surface(model, params, cv, cn, {'alpha': 3.0}, {'appearance': 0, 'warp': 0}, tol=tol)
  np.testing.assert_array_equal(npz['vertices'][0], first['vertices'].cpu().numpy())
  # chosen frames, world coordinates
  configs.clear_config()
  assert extract_mesh.main(argv + ['--frames', '2', '1', '--world_coords']) == 0
  world = dict(np.load(out / 'track.npz'))
  assert world['frames'].tolist() == [2, 1] and world['vertices'].shape == (2, V, 3)
  # frame 2 starts from the template here and from frame 1's solution above: the same root within 2 tol
  both = (world['status'][0] == CONVERGED) & (npz['status'][2] == CONVERGED)
  assert both.mean() > 0.99
  np.testing.assert_allclose(world['vertices'][0][both],
                             npz['vertices'][2][both] / source.scene_scale + source.scene_center,
                             rtol=0, atol=2 * tol / source.scene_scale + 1e-5)
  np.testing.assert_allclose(read_ply(out / 'canonical.ply')['vertices'],
                             cv.cpu().numpy() / source.scene_scale + source.scene_center, rtol=0, atol=1e-5)
  # the refusals
  for extra_args, msg in ((['--canonical'], '--canonical'), (['--metadata', 'warp=1'], '--frames')):
    configs.clear_config()
    with pytest.raises(ValueError, match=msg):
      extract_mesh.main(argv + extra_args)
  configs.clear_config()
