"""Marching cubes without a GPU: the case table against its rule, the PLY writer, and the mesh
driver's box, grid, threshold and argument handling."""
import ctypes
import json
import math

import numpy as np
import pytest

from nerfies_b200 import _lib, extract_mesh, geometry

# ---- the case table --------------------------------------------------------------------------------
# Restated from include/nerfies_b200.h: corner c at (c & 1, c >> 1 & 1, c >> 2 & 1); edge
# 4 * axis + u + 2 v along `axis` from the corner whose other two coordinates (lower axis first) are
# (u, v).


def _corner(c):
  return np.array([c & 1, (c >> 1) & 1, (c >> 2) & 1])


def _edge(c0, c1):
  axis = int(np.flatnonzero(_corner(c0) != _corner(c1))[0])
  lo = _corner(c0 & c1)
  others = [d for d in range(3) if d != axis]
  return 4 * axis + int(lo[others[0]]) + 2 * int(lo[others[1]])


def _edge_corners(e):
  axis, others = e // 4, [d for d in range(3) if d != e // 4]
  p = np.zeros(3, int)
  p[others[0]], p[others[1]] = e & 1, (e >> 1) & 1
  c0 = int(p[0] + 2 * p[1] + 4 * p[2])
  return c0, c0 | (1 << axis)


def _faces():
  """Six faces, each its four corners counter-clockwise seen from outside, found by angle."""
  faces = []
  for axis in range(3):
    for side in (0, 1):
      n = np.zeros(3)
      n[axis] = 1 if side else -1
      u = np.zeros(3)
      u[(axis + 1) % 3] = 1
      v = np.cross(n, u)
      corners = [c for c in range(8) if _corner(c)[axis] == side]
      ang = [math.atan2((_corner(c) - 0.5) @ v, (_corner(c) - 0.5) @ u) for c in corners]
      faces.append([corners[i] for i in np.argsort(ang)])
  return faces


FACES = _faces()


def face_segments(case, face, join_ambiguous=False):
  """The rule: each run of consecutive inside corners, walked counter-clockwise from outside, gives
  the segment (entry edge, exit edge).  join_ambiguous: on a face with two inside corners on a
  diagonal, join them instead (the other resolution, which the rule forbids)."""
  inside = [bool(case >> c & 1) for c in face]
  ring = list(face)
  if join_ambiguous and inside in ([True, False, True, False], [False, True, False, True]):
    # joined: the segments cut off the two outside corners, directed as entries -> exits
    entries = [_edge(ring[q], ring[(q + 1) % 4]) for q in range(4) if not inside[q] and inside[(q + 1) % 4]]
    exits = [_edge(ring[q], ring[(q + 1) % 4]) for q in range(4) if inside[q] and not inside[(q + 1) % 4]]
    return {(entries[0], exits[1]), (entries[1], exits[0])}
  segs = set()
  for q in range(4):
    if not inside[q] and inside[(q + 1) % 4]:
      r = (q + 1) % 4
      while inside[r]:
        r = (r + 1) % 4
      segs.add((_edge(ring[q], ring[(q + 1) % 4]), _edge(ring[(r - 1) % 4], ring[r])))
  return segs


def _face_edges(face):
  return {_edge(face[q], face[(q + 1) % 4]) for q in range(4)}


def table_errors(table, rule=face_segments):
  """Every violation of the rule by an (256, 1 + 3 M) table, as strings."""
  errors = []
  for case in range(256):
    n = table[case, 0]
    tris = table[case, 1:1 + 3 * n].reshape(n, 3)
    crossing = {e for e in range(12) if (case >> _edge_corners(e)[0] & 1) != (case >> _edge_corners(e)[1] & 1)}
    if set(tris.ravel().tolist()) != crossing:
      errors.append(f'case {case}: edges {sorted(set(tris.ravel().tolist()))} != crossing {sorted(crossing)}')
    directed = [(int(t[i]), int(t[(i + 1) % 3])) for t in tris for i in range(3)]
    if len(set(directed)) != len(directed):
      errors.append(f'case {case}: a directed edge appears twice')
    boundary = {d for d in directed if d[::-1] not in directed}
    in_face = {d for d in directed if d not in boundary and any(
        d[0] in _face_edges(f) and d[1] in _face_edges(f) for f in FACES)}
    if in_face:
      errors.append(f'case {case}: interior edges {sorted(in_face)} lie in a cube face')
    for fi, face in enumerate(FACES):
      fe = _face_edges(face)
      on_face = {d for d in boundary if d[0] in fe and d[1] in fe}
      if on_face != rule(case, face):
        errors.append(f'case {case} face {fi}: boundary {sorted(on_face)} != rule {sorted(rule(case, face))}')
    on_some_face = {d for d in boundary if any(d[0] in _face_edges(f) and d[1] in _face_edges(f) for f in FACES)}
    if on_some_face != boundary:
      errors.append(f'case {case}: boundary segments off every face {sorted(boundary - on_some_face)}')
  return errors


def library_table():
  lib = _lib.load()
  m = lib.nfb_marching_cubes_table(None)
  buf = (ctypes.c_int * (256 * (1 + 3 * m)))()
  assert lib.nfb_marching_cubes_table(buf) == m
  return np.array(buf).reshape(256, 1 + 3 * m)


def test_case_table_follows_the_rule():
  table = library_table()
  assert table[0, 0] == 0 and table[255, 0] == 0
  assert table_errors(table) == []
  # padding after each case's triangles
  for case in range(256):
    assert np.all(table[case, 1 + 3 * table[case, 0]:] == -1)
  print(f'max triangles per case: {table.shape[1] // 3}, counts {np.bincount(table[:, 0]).tolist()}')


def test_joining_an_ambiguous_face_fails_the_check():
  """Case 9 (corners 0 and 3 inside, on a diagonal of the z = 0 face): the rule cuts off each corner,
  two triangles.  Joined across that face instead, the same six edges form one tube loop."""
  table = library_table().copy()
  assert table[9, 0] == 2
  joined = [11, 1, 4, 8, 0, 5]                     # the loop 0 -> 5 -> 11 -> 1 -> 4 -> 8, fanned from 11
  row = [4] + [e for i in range(1, 5) for e in (joined[0], joined[i], joined[i + 1])]
  wide = np.full((256, max(table.shape[1], len(row))), -1)
  wide[:, :table.shape[1]] = table
  wide[9, :len(row)] = row
  errors = table_errors(wide)
  assert errors and all(e.startswith('case 9 face 4') for e in errors), errors
  # and it is exactly what the other resolution of that face would give
  rule = lambda case, face: face_segments(case, face, join_ambiguous=(case == 9 and face == FACES[4]))
  assert [e for e in table_errors(wide, rule) if e.startswith('case 9')] == []


def test_table_needs_no_device():
  assert _lib.load().nfb_marching_cubes_table(None) == library_table()[:, 0].max()


# ---- PLY --------------------------------------------------------------------------------------------
def read_ply(path):
  """{'vertices', 'faces'[, 'normals'][, 'colors']} of a binary little-endian PLY, with numpy."""
  data = open(path, 'rb').read()
  end = data.index(b'end_header\n') + len(b'end_header\n')
  lines = data[:end].decode('ascii').split('\n')
  assert lines[:2] == ['ply', 'format binary_little_endian 1.0']
  nv = nf = 0
  cols = []
  for line in lines[2:]:
    w = line.split()
    if w[:2] == ['element', 'vertex']:
      nv = int(w[2])
    elif w[:2] == ['element', 'face']:
      nf = int(w[2])
    elif w[:1] == ['property'] and w[1] != 'list':
      cols.append((w[2], {'float': '<f4', 'uchar': 'u1'}[w[1]]))
    elif w[:1] == ['property']:
      assert w[1:] == ['list', 'uchar', 'int', 'vertex_indices']
  rows = np.frombuffer(data, np.dtype(cols), nv, end)
  tri = np.frombuffer(data, np.dtype([('n', 'u1'), ('i', '<i4', (3,))]), nf, end + rows.nbytes)
  assert np.all(tri['n'] == 3) and end + rows.nbytes + tri.nbytes == len(data)
  out = {'vertices': np.stack([rows[k] for k in 'xyz'], -1).reshape(nv, 3), 'faces': tri['i'].reshape(nf, 3)}
  names = rows.dtype.names or ()
  if 'nx' in names:
    out['normals'] = np.stack([rows[k] for k in ('nx', 'ny', 'nz')], -1).reshape(nv, 3)
  if 'red' in names:
    out['colors'] = np.stack([rows[k] for k in ('red', 'green', 'blue')], -1).reshape(nv, 3)
  return out


def test_ply_round_trip(tmp_path):
  rng = np.random.default_rng(0)
  v = rng.standard_normal((7, 3)).astype(np.float32)
  n = rng.standard_normal((7, 3)).astype(np.float32)
  c = rng.integers(0, 256, (7, 3)).astype(np.uint8)
  f = rng.integers(0, 7, (5, 3)).astype(np.int32)
  geometry.write_ply(tmp_path / 'a.ply', v, f, n, c)
  got = read_ply(tmp_path / 'a.ply')
  for k, want in (('vertices', v), ('faces', f), ('normals', n), ('colors', c)):
    np.testing.assert_array_equal(got[k], want, err_msg=k)
  geometry.write_ply(tmp_path / 'b.ply', v, f)
  assert set(read_ply(tmp_path / 'b.ply')) == {'vertices', 'faces'}
  head = open(tmp_path / 'a.ply', 'rb').read(400).split(b'end_header')[0].decode()
  assert 'property float nx' in head and 'property uchar red' in head and 'element face 5' in head


def test_empty_ply(tmp_path):
  geometry.write_ply(tmp_path / 'e.ply', np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32),
                     np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint8))
  got = read_ply(tmp_path / 'e.ply')
  assert got['vertices'].shape == (0, 3) and got['faces'].shape == (0, 3) and got['colors'].shape == (0, 3)


def test_ply_rejects_bad_shapes(tmp_path):
  with pytest.raises(ValueError, match='normals'):
    geometry.write_ply(tmp_path / 'x.ply', np.zeros((2, 3), np.float32), np.zeros((0, 3), np.int32),
                       np.zeros((3, 3), np.float32))
  with pytest.raises(ValueError, match='faces'):
    geometry.write_ply(tmp_path / 'x.ply', np.zeros((2, 3), np.float32), np.zeros((4,), np.int32))


# ---- driver logic -----------------------------------------------------------------------------------
def _capture(tmp_path, scene, points=None):
  tmp_path.mkdir(parents=True, exist_ok=True)
  (tmp_path / 'scene.json').write_text(json.dumps(scene))
  if points is not None:
    np.save(tmp_path / 'points.npy', points)
  return tmp_path


def test_box_from_scene_json(tmp_path):
  d = _capture(tmp_path, {'center': [1.0, 2.0, 3.0], 'scale': 0.5, 'near': 0.1, 'far': 2.0,
                          'bbox': [[-1.0, 0.0, 1.0], [3.0, 6.0, 4.0]]}, np.zeros((4, 3)))
  np.testing.assert_allclose(extract_mesh.scene_box(d), [[-1.0, -1.0, -1.0], [1.0, 2.0, 0.5]])


def test_box_from_points(tmp_path):
  points = np.array([[0.0, 0.0, 0.0], [2.0, 4.0, 1.0], [1.0, 1.0, 0.5]])
  d = _capture(tmp_path, {'center': [1.0, 0.0, 0.0], 'scale': 2.0, 'near': 0.1, 'far': 2.0}, points)
  lo, hi = np.array([-2.0, 0.0, 0.0]), np.array([2.0, 8.0, 2.0])           # (p - center) * scale
  np.testing.assert_allclose(extract_mesh.scene_box(d), [lo - 0.1 * (hi - lo), hi + 0.1 * (hi - lo)], rtol=1e-6)


def test_box_explicit_and_missing(tmp_path):
  d = _capture(tmp_path / 'none', {'center': [0, 0, 0], 'scale': 1.0, 'near': 0.1, 'far': 2.0})
  box = extract_mesh.scene_box(d, [[0, 0, 0], [1, 2, 3]])
  np.testing.assert_array_equal(box, [[0, 0, 0], [1, 2, 3]])
  with pytest.raises(ValueError, match='no box'):
    extract_mesh.scene_box(d)
  with pytest.raises(ValueError, match='--bbox'):
    extract_mesh.scene_box(d, [[0, 0, 0], [1, -2, 3]])


def test_box_of_the_small_capture():
  """tests/golden/capture_small's scene.json has no bbox: the box comes from its points."""
  import os
  d = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'capture_small')
  scene = json.load(open(os.path.join(d, 'scene.json')))
  pts = (np.load(os.path.join(d, 'points.npy')) - scene['center']) * scene['scale']
  box = extract_mesh.scene_box(d)
  assert np.all(box[0] < pts.min(0)) and np.all(box[1] > pts.max(0))


def test_grid_has_cubic_voxels():
  box, shape = extract_mesh.grid_for_box([[0.0, -1.0, 0.5], [2.0, 0.3, 1.2]], 65)
  assert shape == (24, 43, 65)                                               # (nz, ny, nx)
  spacing = geometry.grid_spacing(box, shape)
  assert np.all(spacing == spacing[0]) and spacing[0] == np.float32(2.0 / 64)
  assert np.all(box[1] >= [2.0, 0.3, 1.2]) and np.all(box[1] - [2.0, 0.3, 1.2] < 2.0 / 64)
  assert extract_mesh.grid_for_box([[0, 0, 0], [1, 1e-6, 1]], 8)[1] == (8, 2, 8)
  for bad in (1, 1025):
    with pytest.raises(ValueError, match='resolution'):
      extract_mesh.grid_for_box([[0, 0, 0], [1, 1, 1]], bad)


def test_default_threshold():
  assert extract_mesh.default_threshold(64, 0.5, 2.5) == pytest.approx(math.log(2) * 32)
  # one coarse step at that density is half opaque
  sigma, step = extract_mesh.default_threshold(16, 0.05, 2.5), (2.5 - 0.05) / 16
  assert 1 - math.exp(-sigma * step) == pytest.approx(0.5)


def test_mesh_names():
  assert extract_mesh.mesh_name(True, {'warp': 3}) == 'canonical'
  assert extract_mesh.mesh_name(False, {'warp': 3, 'appearance': 1}) == 'warp_3'
  assert extract_mesh.mesh_name(False, {'time': 0.5}) == 'time_0.5'


def test_flags():
  args = extract_mesh.make_parser().parse_args(
      ['--base_folder', '/x', '--bbox', '0', '0', '0', '1', '1', '1', '--resolution', '48', '--canonical', '--colors',
       '--world_coords', '--level', 'coarse', '--threshold', '2.5', '--metadata', 'warp=2'])
  assert (args.bbox, args.resolution, args.canonical, args.colors, args.world_coords, args.level, args.threshold,
          args.metadata) == ([0, 0, 0, 1, 1, 1], 48, True, True, True, 'coarse', 2.5, ['warp=2'])
  for bad in (['--level', 'medium'], ['--bbox', '0', '1'], ['--resolution', 'x']):
    with pytest.raises(SystemExit):
      extract_mesh.make_parser().parse_args(['--base_folder', '/x'] + bad)


def test_driver_refuses_bad_arguments_before_any_gpu_work(tmp_path):
  from nerfies_b200 import configs

  class Source:
    data_dir = _capture(tmp_path / 'cap', {'center': [0, 0, 0], 'scale': 1.0, 'near': 0.1, 'far': 2.0})
    near, far = 0.1, 2.0

  run = lambda **kw: extract_mesh.extract_mesh(configs.ExperimentConfig(), configs.ModelConfig(), str(tmp_path),
                                               datasource=Source(), log=lambda s: None, **kw)
  with pytest.raises(ValueError, match='no box'):
    run()
  with pytest.raises(ValueError, match='resolution'):
    run(bbox=[[0, 0, 0], [1, 1, 1]], resolution=1)
  with pytest.raises(ValueError, match='level'):
    run(bbox=[[0, 0, 0], [1, 1, 1]], level='medium')
  with pytest.raises(FileNotFoundError, match='no checkpoints'):
    run(bbox=[[0, 0, 0], [1, 1, 1]])
