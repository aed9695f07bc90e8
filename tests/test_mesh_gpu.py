"""Marching cubes, the density grid and the mesh driver on the GPU.

Analytic grids check the mesh's topology (closed, oriented, Euler characteristic), its vertices
against the documented interpolation evaluated with torch, and its geometry on a sphere.  The
density grid and vertex colours are checked against the fp64 oracle at the same points, and the
driver end to end on the small capture."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from oracle import nerfies_oracle as O
from tests.golden_util import Golden, model_from_spec, rel_err, tree_to_device
from tests.test_mesh import read_ply

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAPTURE = os.path.join(ROOT, 'tests', 'golden', 'capture_small')


def _box(shape):
  """The box of a grid with unit spacing: point [k, j, i] at (i, j, k)."""
  nz, ny, nx = shape
  return ((0.0, 0.0, 0.0), (nx - 1.0, ny - 1.0, nz - 1.0))


def _coords(shape):
  nz, ny, nx = shape
  k, j, i = torch.meshgrid(*(torch.arange(n, device=DEV, dtype=torch.float64) for n in shape), indexing='ij')
  return i, j, k


def _sphere(shape, center, r):
  i, j, k = _coords(shape)
  return (r - torch.sqrt((i - center[0])**2 + (j - center[1])**2 + (k - center[2])**2)).float().contiguous()


def _mc(grid, level=0.0, bbox=None):
  from nerfies_b200 import geometry
  return geometry.marching_cubes(grid, level, bbox or _box(grid.shape))


def _edge_check(faces, num_vertices, allowed=None):
  """Directed edges of the faces: each at most once, and each with its reverse (closed and
  consistently oriented), except edges `allowed(a, b)` accepts.  Returns the number of edges."""
  f = (faces.cpu().numpy() if torch.is_tensor(faces) else np.asarray(faces)).astype(np.int64)
  assert f.size == 0 or (f.min() >= 0 and f.max() < num_vertices)
  a = f.reshape(-1)
  b = np.roll(f, -1, axis=1).reshape(-1)
  key, rev = a * num_vertices + b, b * num_vertices + a
  assert len(np.unique(key)) == len(key), 'a directed edge appears twice'
  lonely = ~np.isin(rev, key)
  if allowed is None:
    assert not lonely.any(), f'{int(lonely.sum())} edges without their reverse'
  else:
    assert allowed(a[lonely], b[lonely]).all(), 'open edges away from the box'
  return len(key) // 2


def _closed(vertices, faces):
  E = _edge_check(faces, len(vertices))
  return len(vertices) - E + len(faces)          # Euler characteristic


def _crossings(grid, level):
  inside = grid > level
  return sum(int((inside.narrow(d, 1, inside.shape[d] - 1) != inside.narrow(d, 0, inside.shape[d] - 1)).sum())
             for d in (2, 1, 0))


def _expected_vertices(grid, level, bbox):
  """The documented interpolation, in torch float32, in the library's order (axis, linear index)."""
  from nerfies_b200 import geometry
  shape = grid.shape
  sp = torch.tensor(geometry.grid_spacing(bbox, shape), device=DEV)
  org = torch.tensor(np.asarray(bbox[0], np.float32), device=DEV)
  out = []
  for axis, d in ((0, 2), (1, 1), (2, 0)):                 # x-edges run along dim 2 of (nz, ny, nx)
    v0 = grid.narrow(d, 0, shape[d] - 1)
    v1 = grid.narrow(d, 1, shape[d] - 1)
    cross = (v0 > level) != (v1 > level)
    k, j, i = torch.nonzero(cross, as_tuple=True)
    a, b = v0[cross], v1[cross]
    t = (level - a) / (b - a)
    t = torch.where(torch.isnan(a) | torch.isnan(b), torch.full_like(t, 0.5), t)
    idx = [i, j, k]
    xyz = []
    for c in range(3):
      x0 = org[c] + idx[c].float() * sp[c]
      if c == axis:
        x1 = org[c] + (idx[c] + 1).float() * sp[c]
        x0 = x0 + t * (x1 - x0)
      xyz.append(x0)
    out.append(torch.stack(xyz, -1))
  return torch.cat(out)


SHAPES = [(41, 45, 47), (33, 60, 29), (64, 64, 64)]


@pytest.mark.parametrize('shape', SHAPES)
def test_sphere_is_closed_and_matches_the_interpolation(shape):
  c = [(n - 1) / 2 + 0.3 for n in shape[::-1]]
  r = min(shape) / 2 - 3.1
  grid = _sphere(shape, c, r)
  bbox = ((-1.0, 0.5, 2.0), (-1.0 + 0.5 * (shape[2] - 1), 0.5 + 0.25 * (shape[1] - 1), 2.0 + 0.75 * (shape[0] - 1)))
  v, f, n = _mc(grid, 0.0, bbox)
  assert _closed(v, f) == 2
  assert len(v) == _crossings(grid, 0.0)
  want = _expected_vertices(grid, 0.0, bbox)
  err = float((v - want).abs().max())
  scale = float(want.abs().max())
  print(f'{shape}: {len(v)} vertices, {len(f)} faces, max |vertex - torch| {err:.3e}')
  assert err <= 2 * scale * np.finfo(np.float32).eps


def test_sphere_geometry():
  shape, r = (61, 63, 59), 24.0
  c = (29.25, 31.5, 30.125)
  v, f, n = _mc(_sphere(shape, c, r))
  assert _closed(v, f) == 2
  vd, fd = v.double(), f.long()
  p0, p1, p2 = vd[fd[:, 0]], vd[fd[:, 1]], vd[fd[:, 2]]
  volume = float((p0 * torch.cross(p1, p2, dim=-1)).sum() / 6)
  exact = 4 / 3 * math.pi * r**3
  radial = vd - torch.tensor(c, device=DEV, dtype=torch.float64)
  dist = radial.norm(dim=-1)
  cosang = (n.double() * radial).sum(-1) / dist / n.double().norm(dim=-1)
  angle = float(torch.rad2deg(torch.acos(cosang.clamp(-1, 1))).max())
  print(f'volume {volume:.2f} vs {exact:.2f} ({volume / exact - 1:+.3%}), radial error '
        f'{float((dist - r).abs().max()):.4f} voxel, normals within {angle:.3f} degrees of radial')
  assert volume > 0 and abs(volume / exact - 1) < 0.01
  assert float((dist - r).abs().max()) < 0.05
  assert angle < 2.0
  assert torch.allclose(n.norm(dim=-1), torch.ones(len(n), device=DEV), atol=1e-5)


def test_torus_and_two_spheres():
  shape = (31, 71, 69)
  i, j, k = _coords(shape)
  x, y, z = i - 34.0, j - 35.2, k - 15.1
  torus = (6.0**2 - ((torch.sqrt(x * x + y * y) - 20.0)**2 + z * z)).float().contiguous()
  v, f, _ = _mc(torus)
  assert _closed(v, f) == 0
  two = torch.maximum(_sphere(shape, (20.0, 35.0, 15.0), 10.0), _sphere(shape, (48.3, 35.0, 15.0), 12.0))
  v, f, _ = _mc(two.contiguous())
  assert _closed(v, f) == 4


def test_random_field_is_closed_and_oriented():
  """Uniform noise with an outside border: every ambiguous face configuration occurs many times."""
  g = torch.Generator(device=DEV).manual_seed(0)
  grid = torch.rand(37, 42, 51, device=DEV, generator=g)
  grid[0], grid[-1], grid[:, 0], grid[:, -1], grid[:, :, 0], grid[:, :, -1] = 0, 0, 0, 0, 0, 0
  v, f, n = _mc(grid, 0.5)
  _edge_check(f, len(v))
  assert len(v) == _crossings(grid, 0.5)
  inside = grid > 0.5
  a, b = inside[:, :-1, :-1], inside[:, 1:, 1:]
  diag = (a & b & ~inside[:, 1:, :-1] & ~inside[:, :-1, 1:]) | (~a & ~b & inside[:, 1:, :-1] & inside[:, :-1, 1:])
  assert int(diag.sum()) > 1000                       # ambiguous z-faces
  # determinism: a second call is bitwise equal
  v2, f2, n2 = _mc(grid, 0.5)
  assert torch.equal(v, v2) and torch.equal(f, f2) and torch.equal(n, n2)


def test_degenerate_grids():
  shape = (9, 10, 11)
  for fill in (0.0, 1.0):                             # all outside, all inside: nothing crosses
    v, f, n = _mc(torch.full(shape, fill, device=DEV), 0.5)
    assert v.shape == (0, 3) and f.shape == (0, 3) and n.shape == (0, 3)
  # ties: value == level is outside
  grid = torch.zeros(shape, device=DEV)
  grid[3:6, 3:7, 4:8] = 1.0
  grid[4, 4, 5] = 0.5
  for level in (0.5, 0.0, 1.0):
    v, f, _ = _mc(grid, level)
    assert len(v) == _crossings(grid, level)
    if len(f):
      _closed(v, f)
  v, f, _ = _mc(grid, 1.0)
  assert len(v) == 0                                  # nothing is > 1
  v, f, _ = _mc(grid, 0.0)
  assert _closed(v, f) == 2                            # the box, with the tie point inside
  # NaN cells are outside: the mesh stays closed and finite
  sphere = _sphere((25, 27, 29), (14.0, 13.0, 12.0), 9.0)
  sphere[12, 13, 14] = float('nan')                   # the centre
  sphere[12, 13, 22] = float('nan')                   # on the surface
  sphere[2, 2, 2] = float('nan')                      # outside
  v, f, n = _mc(sphere)
  _edge_check(f, len(v))
  assert torch.isfinite(v).all() and torch.isfinite(n).all()
  assert len(v) == _crossings(sphere, 0.0)
  want = _expected_vertices(sphere, 0.0, _box(sphere.shape))
  assert float((v - want).abs().max()) <= 1e-5


def test_bad_arguments():
  from nerfies_b200 import _lib, geometry
  lib = _lib.load()
  with pytest.raises(ValueError, match='>= 2'):
    geometry.marching_cubes(torch.zeros(1, 4, 4, device=DEV), 0.0, ((0, 0, 0), (1, 1, 1)))
  with pytest.raises(ValueError, match='float32'):
    geometry.marching_cubes(torch.zeros(4, 4, 4, device=DEV, dtype=torch.float64), 0.0, ((0, 0, 0), (1, 1, 1)))
  with pytest.raises(ValueError, match='CUDA'):
    geometry.marching_cubes(torch.zeros(4, 4, 4), 0.0, ((0, 0, 0), (1, 1, 1)))
  with pytest.raises(ValueError, match='contiguous'):
    geometry.marching_cubes(torch.zeros(4, 4, 8, device=DEV)[..., ::2], 0.0, ((0, 0, 0), (1, 1, 1)))
  with pytest.raises(_lib.NfbError, match=r'\[2, 1024\]'):
    geometry.marching_cubes(torch.zeros(2, 2, 1025, device=DEV), 0.0, ((0, 0, 0), (1, 1, 1)))
  assert lib.nfb_marching_cubes_workspace_size(1, 4, 4) < 0 and b'[2, 1024]' in lib.nfb_last_error()
  need = lib.nfb_marching_cubes_workspace_size(4, 4, 4)
  assert need >= 16 * 64
  ws = torch.empty(need, dtype=torch.uint8, device=DEV)
  counts = torch.empty(4, dtype=torch.int64, device=DEV)
  grid = torch.zeros(4, 4, 4, device=DEV)
  p = lambda t: ctypes.c_void_p(t.data_ptr())
  assert lib.nfb_marching_cubes_count(None, 4, 4, 4, 0.0, p(ws), need, p(counts), None) != 0
  assert b'null' in lib.nfb_last_error()
  assert lib.nfb_marching_cubes_count(p(grid), 4, 4, 4, 0.0, p(ws), need - 1, p(counts), None) != 0
  assert b'workspace' in lib.nfb_last_error()
  assert lib.nfb_marching_cubes_count(p(grid), 4, 4, 4, 0.0, p(ws), need, None, None) != 0
  f3 = (ctypes.c_float * 3)(0, 0, 0)
  assert lib.nfb_marching_cubes(p(grid), 4, 4, 4, 0.0, None, f3, p(ws), need, None, None, None, None) != 0
  assert b'null' in lib.nfb_last_error()


# ---- density grid and vertex colours against the oracle -----------------------------------------------
FIXTURES = ['se3_small', 'translation_small', 'time_small', 'alpha_cond_init']
BOX = ((-0.37, -0.29, -0.44), (0.41, 0.33, 0.28))
SHAPE = (5, 7, 9)                                     # (nz, ny, nx): 35 rows, 8 per call


def _fixture_model(name, precision):
  from nerfies_b200 import _lib
  g = Golden(name)
  model = model_from_spec(g.spec_dict, precision=precision, device=DEV, batch_size=8)
  try:
    model.handle()
  except _lib.NfbError as e:
    assert 'use precision fp32' in str(e)
    pytest.skip(f'{name}: not a tensor-core shape ({e})')
  md = {k: (float(v[0, 0]) if k == 'time' else int(v[0, 0])) for k, v in g.rays['metadata'].items()}
  extra = {'alpha': g.warp_alpha, 'time_alpha': g.time_alpha}
  return g, model, md, extra


def _oracle_points(g, points, directions, md, use_warp, level):
  P = points.shape[0]
  rays = {'origins': points.cpu(), 'directions': directions.cpu(),
          'metadata': {k: torch.full((P, 1), v, dtype=torch.float32 if k == 'time' else torch.int32)
                       for k, v in md.items()}}
  return O.render_level(g.params, g.spec, level, rays, torch.zeros(P, 1), g.warp_alpha, use_warp=use_warp,
                        dtype=torch.float64, time_alpha=g.time_alpha)


@pytest.mark.parametrize('precision', ['fp32', 'fp16x3'])
@pytest.mark.parametrize('name', FIXTURES)
def test_density_grid_vs_oracle(name, precision):
  from nerfies_b200 import geometry
  g, model, md, extra = _fixture_model(name, precision)
  params = tree_to_device(g.params, DEV)
  sp = geometry.grid_spacing(BOX, SHAPE)
  axis = [np.float32(BOX[0][d]) + np.arange(n, dtype=np.float32) * sp[d] for d, n in enumerate(SHAPE[::-1])]
  k, j, i = np.meshgrid(axis[2], axis[1], axis[0], indexing='ij')
  points = torch.from_numpy(np.stack([i, j, k], -1).reshape(-1, 3).astype(np.float32))
  dirs = torch.tensor([[1.0, 0.0, 0.0]]).expand(len(points), 3)
  for use_warp in (False, True):
    for level in ('coarse', 'fine'):
      got = geometry.density_grid(model, params, BOX, SHAPE, extra, md, use_warp=use_warp, level=level)
      assert got.shape == SHAPE
      ref = _oracle_points(g, points, dirs, md, use_warp, level)['sample_sigma'].reshape(SHAPE)
      err = rel_err(got.cpu(), ref)
      print(f'{name} {precision} warp={use_warp} {level}: sigma in [{float(ref.min()):.3g}, {float(ref.max()):.3g}], '
            f'rel err {err:.2e}')
      assert err < 1e-4, (use_warp, level)


@pytest.mark.parametrize('precision', ['fp32', 'fp16x3'])
@pytest.mark.parametrize('name', ['se3_small', 'time_small'])
def test_vertex_colors_vs_oracle(name, precision):
  from nerfies_b200 import geometry
  g, model, md, extra = _fixture_model(name, precision)
  params = tree_to_device(g.params, DEV)
  gen = torch.Generator().manual_seed(3)
  V = 21                                              # three calls of 8 rays
  verts = (torch.rand(V, 3, generator=gen) - 0.5) * 0.6
  normals = torch.nn.functional.normalize(torch.randn(V, 3, generator=gen), dim=-1)
  normals[4] = 0.0
  axes = torch.zeros(V, dtype=torch.uint8)
  axes[4] = 2
  for use_warp in (True, False):
    got = geometry.vertex_colors(model, params, verts.to(DEV), normals.to(DEV), extra, md, use_warp=use_warp,
                                 level='fine', axes=axes.to(DEV))
    dirs = -normals
    dirs[4] = torch.tensor([0.0, 0.0, 1.0])
    ref = _oracle_points(g, verts, dirs, md, use_warp, 'fine')['sample_rgb'][:, 0]
    err = rel_err(got.cpu(), ref)
    print(f'{name} {precision} warp={use_warp}: rgb rel err {err:.2e}')
    assert err < 1e-4
  with pytest.raises(ValueError, match='axes'):
    geometry.vertex_colors(model, params, verts.to(DEV), normals.to(DEV), extra, md)


# ---- the driver end to end ------------------------------------------------------------------------
GIN = """
ExperimentConfig.image_scale = 2
ModelConfig.num_coarse_samples = 16
ModelConfig.num_fine_samples = 16
ModelConfig.use_warp = True
ModelConfig.warp_field_type = 'se3'
ModelConfig.use_appearance_metadata = True
"""


@pytest.fixture(scope='module')
def checkpoint(tmp_path_factory):
  """A checkpoint of trained-like random parameters for the small capture."""
  from nerfies_b200 import checkpoints, configs, driver_utils, model_utils, models
  tmp = tmp_path_factory.mktemp('mesh_driver')
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


def _on_box_face(box, shape, vertices):
  """(a, b) -> both vertices on one face plane of the grid's box (where the mesh may be open)."""
  from nerfies_b200 import geometry
  sp = geometry.grid_spacing(box, shape)
  lo = np.asarray(box[0], np.float32)
  hi = np.array([np.float32(lo[d]) + np.float32(shape[::-1][d] - 1) * sp[d] for d in range(3)], np.float32)
  v = vertices

  def allowed(a, b):
    ok = np.zeros(len(a), bool)
    for d in range(3):
      for plane in (lo[d], hi[d]):
        ok |= (v[a, d] == plane) & (v[b, d] == plane)
    return ok
  return allowed


def test_extract_mesh_end_to_end(checkpoint):
  from nerfies_b200 import configs, evaluation, extract_mesh, geometry
  base, gin, model, params, source = checkpoint
  box, shape = extract_mesh.grid_for_box(extract_mesh.scene_box(CAPTURE), 48)
  md = {'appearance': 0, 'warp': 0}
  extra = {'alpha': 3.0, 'time_alpha': 0.0}
  grid = geometry.density_grid(model, params, box, shape, extra, md)
  level = float(grid.median())
  argv = ['--base_folder', str(base), '--data_dir', CAPTURE, '--gin_configs', gin, '--precision', 'fp32',
          '--resolution', '48', '--colors', '--threshold', repr(level)]
  assert extract_mesh.main(argv) == 0
  path = base / 'meshes' / '00000007' / 'warp_0.ply'
  got = read_ply(path)
  v, f, n, axes = geometry.marching_cubes(grid, level, box, return_axes=True)
  colors = evaluation.image_to_uint8(geometry.vertex_colors(model, params, v, n, extra, md, axes=axes))
  assert len(f) > 100
  for k, want in (('vertices', v), ('faces', f), ('normals', n), ('colors', colors)):
    np.testing.assert_array_equal(got[k], want.cpu().numpy(), err_msg=k)
  vh = got['vertices']
  _edge_check(got['faces'], len(vh), _on_box_face(box, shape, vh))
  assert np.all(vh >= np.float32(box[0]) - 1e-6) and np.all(vh <= box[1] + 1e-5)
  print(f'median threshold {level:.4g}: {len(vh)} vertices, {len(got["faces"])} faces')

  # world frame: x / scale + center
  configs.clear_config()
  assert extract_mesh.main(argv + ['--world_coords', '--canonical']) == 0
  world = read_ply(base / 'meshes' / '00000007' / 'canonical.ply')['vertices'].astype(np.float64)
  wbox = box / source.scene_scale + np.asarray(source.scene_center)
  assert len(world) and np.all(world >= wbox[0] - 1e-5) and np.all(world <= wbox[1] + 1e-5)
  canon = geometry.density_grid(model, params, box, shape, extra, md, use_warp=False)
  cv, _, _ = geometry.marching_cubes(canon, level, box)
  np.testing.assert_allclose(world, (cv.double().cpu().numpy() / source.scene_scale + source.scene_center),
                             rtol=0, atol=1e-5)

  # the default threshold: a valid file, possibly empty
  configs.clear_config()
  assert extract_mesh.main(argv[:-2] + ['--level', 'coarse', '--resolution', '24']) == 0
  default = read_ply(base / 'meshes' / '00000007' / 'warp_0.ply')
  print(f'default threshold {extract_mesh.default_threshold(16, source.near, source.far):.4g}: '
        f'{len(default["vertices"])} vertices')
  _edge_check(default['faces'], len(default['vertices']),
              _on_box_face(*extract_mesh.grid_for_box(extract_mesh.scene_box(CAPTURE), 24), default['vertices']))
