"""Host side of capture processing (nerfies_b200.colmap / capture / process_capture) against the
capture the reference's notebook wrote for tests/golden/colmap_small (oracle/make_golden_capture.py):
the COLMAP reader, the split, metadata, scene box and orbit path, the JSON layouts and the CLI's
argument errors; and the numpy statement of the pixel steps (tests/capture_oracle.py) against cv2."""
import json
import os
import pathlib

import numpy as np
import pytest

from nerfies_b200 import capture
from nerfies_b200 import colmap
from nerfies_b200 import process_capture
from tests import capture_oracle

GOLDEN = pathlib.Path(__file__).resolve().parent / 'golden'
SMALL = GOLDEN / 'colmap_small'
EXPECTED = SMALL / 'expected'


@pytest.fixture(scope='module')
def ref():
  return dict(np.load(GOLDEN / 'capture_process.npz'))


@pytest.fixture(scope='module')
def scene():
  cameras, points = colmap.load_scene(SMALL / 'sparse' / '0', process_capture.MIN_TRACK_LENGTH)
  return {k: c.scale(4) for k, c in cameras.items()}, points


def _json(path):
  with open(path) as f:
    return json.load(f)


def _assert_camera_json(got, want):
  assert sorted(got) == sorted(want)
  for k in want:
    np.testing.assert_array_equal(np.float32(got[k]), np.float32(want[k]), err_msg=k)


def test_reader_matches_the_notebook(scene, ref):
  cameras, points = scene
  assert sorted(cameras) == sorted(ref['blur_ids'].tolist())
  assert '000016' not in cameras                        # the unregistered frame
  np.testing.assert_array_equal(points, ref['points'])   # track-filtered, file order
  for item in ref['item_ids']:
    _assert_camera_json(cameras[str(item)].to_json(), _json(EXPECTED / 'camera' / f'{item}.json'))


def test_track_filter_counts_distinct_images(tmp_path):
  all_points, _ = colmap.read_points3d(SMALL / 'sparse' / '0' / 'points3D.bin')
  kept, _ = colmap.read_points3d(SMALL / 'sparse' / '0' / 'points3D.bin', 5)
  assert 0 < len(kept) < len(all_points)


def test_unsupported_camera_model(tmp_path):
  import struct
  path = tmp_path / 'cameras.bin'
  path.write_bytes(struct.pack('<Q', 1) + struct.pack('<IiQQ', 1, 6, 10, 10) + struct.pack('<12d', *[1.0] * 12))
  with pytest.raises(ValueError, match='FULL_OPENCV'):
    colmap.read_cameras(path)
  for model_id, n in ((0, 3), (1, 4), (2, 4), (3, 5)):
    path.write_bytes(struct.pack('<Q', 1) + struct.pack('<IiQQ', 1, model_id, 10, 8) +
                     struct.pack(f'<{n}d', *range(2, 2 + n)))
    cam = colmap.read_cameras(path)[1]
    image = colmap.ColmapImage(1, np.array([1.0, 0, 0, 0]), np.zeros(3), 1, 'a.png')
    c = colmap.convert_camera(cam, image)
    assert float(c.focal_length) == 2.0 and c.tangential_distortion.tolist() == [0.0, 0.0]
    assert float(c.radial_distortion[2]) == 0.0


def test_split_and_metadata(ref):
  dataset, metadata = capture.split_and_metadata(ref['item_ids'].tolist())
  assert dataset == _json(EXPECTED / 'dataset.json')
  assert metadata == _json(EXPECTED / 'metadata.json')
  big, meta = capture.split_and_metadata([f'{i:04d}' for i in range(45)])
  assert big['val_ids'] == ['0000', '0020', '0040'] and meta['0020']['warp_id'] == 19


def test_blur_filter_drops_the_sharpest(ref):
  ids = ref['blur_ids'].tolist()
  assert capture.blur_filter(ids, ref['blur_scores'], 95.0) == ref['removed_ids'].tolist()
  assert ref['blur_scores'][ids.index(ref['removed_ids'][0])] == ref['blur_scores'].max()
  assert capture.blur_filter(ids, ref['blur_scores'], 0.0) == []


def test_scene_info_given_near_far(scene, ref):
  cameras, points = scene
  cams = [cameras[str(i)] for i in ref['item_ids']]
  got = capture.scene_info(points, cams, float(ref['near']), float(ref['far']))
  want = _json(EXPECTED / 'scene.json')
  assert sorted(got) == sorted(want)
  for k in want:
    np.testing.assert_allclose(got[k], want[k], rtol=1e-12, err_msg=k)
  # the notebook's combination of the per-camera planes
  assert np.quantile(ref['near_i'], 0.001) / 0.8 == pytest.approx(float(ref['near']), rel=1e-15)
  assert np.quantile(ref['far_i'], 0.999) * 1.2 == pytest.approx(float(ref['far']), rel=1e-15)


def test_orbit_path(scene, ref):
  cameras, _ = scene
  cams = [cameras[str(i)] for i in ref['item_ids']]
  path = capture.orbit_camera_path(cams, 100, 0.75, 0.75, 0.75)
  files = sorted((EXPECTED / 'camera-paths' / 'orbit-mild').iterdir())
  assert [f.name for f in files] == [f'{i:06d}.json' for i in range(100)]
  np.testing.assert_allclose(capture.triangulate_rays([c.position for c in cams], [c.optical_axis for c in cams]),
                             ref['look_at'], rtol=1e-6, atol=1e-6)
  for cam, f in zip(path, files):
    got, want = cam.to_json(), _json(f)
    assert sorted(got) == sorted(want)
    for k in want:
      np.testing.assert_allclose(np.float32(got[k]), np.float32(want[k]), rtol=2e-6, atol=2e-6, err_msg=f'{f.name} {k}')


def test_look_at_errors(scene):
  cam = next(iter(scene[0].values()))
  with pytest.raises(ValueError, match='too close'):
    cam.look_at(np.zeros(3), np.zeros(3), np.array([0, 1, 0]))
  with pytest.raises(ValueError, match='parallel'):
    cam.look_at(np.zeros(3), np.array([0, 0, 1.0]), np.array([0, 0, 1.0]))


def test_points_to_local_points(scene):
  cam = next(iter(scene[0].values()))
  p = np.array([[0.1, 0.2, 0.3], [1, -1, 2]], np.float32)
  np.testing.assert_array_equal(cam.points_to_local_points(p), np.matmul(cam.orientation, (p - cam.position).T).T)


def test_filter_outlier_points_box(ref, scene):
  _, points = scene
  inl = capture.filter_outlier_points(points)
  lo, hi = np.quantile(points, 0.025, axis=0), np.quantile(points, 0.975, axis=0)
  assert ((inl >= lo) & (inl <= hi)).all() and len(inl) < len(points)


@pytest.mark.parametrize('argv, message', [
    (['images', '--frames_dir', 'a', '--data_dir', 'b', '--image_scales', '1,3'], 'scale 3'),
    (['images', '--frames_dir', 'a', '--data_dir', 'b', '--image_scales', '4,6'], 'does not divide'),
    (['images', '--data_dir', 'b'], '--frames_dir'),
    (['scene', '--data_dir', 'b'], '--colmap_dir'),
    (['scene', '--data_dir', 'b', '--colmap_dir', 'c', '--colmap_image_scale', '0'], 'not positive'),
    (['scene', '--data_dir', 'b', '--colmap_dir', 'c', '--orbit_frames', '0'], 'not a positive'),
    (['frames'], 'invalid choice'),
])
def test_cli_argument_errors(argv, message, capsys):
  with pytest.raises(SystemExit) as e:
    process_capture.make_parser().parse_args(argv)
  assert e.value.code == 2
  assert message in capsys.readouterr().err


def test_cli_defaults_are_the_notebooks():
  a = process_capture.make_parser().parse_args(['scene', '--data_dir', 'd', '--colmap_dir', 'c'])
  assert (a.colmap_image_scale, a.blur_filter_perc, a.orbit_frames, a.orbit_radius, a.orbit_x_scale,
          a.orbit_y_scale) == (4, 95.0, 100, 0.75, 0.75, 0.75)
  a = process_capture.make_parser().parse_args(['images', '--frames_dir', 'f', '--data_dir', 'd'])
  assert a.image_scales == [1, 2, 4, 8]


def test_oracle_pyramid_equals_cv2():
  cv2 = pytest.importorskip('cv2')
  rng = np.random.RandomState(0)
  for scale in (2, 4, 6, 8, 16):
    for h, w in ((48, 96), (96, 144)):
      image = rng.randint(0, 256, size=(h, w, 3), dtype=np.uint8)
      want = cv2.resize(image, (w // scale, h // scale), cv2.INTER_AREA)   # the notebook's call
      np.testing.assert_array_equal(capture_oracle.downsample(image, scale), want)


def test_oracle_pyramid_equals_expected_pngs():
  from nerfies_b200 import datasets
  for name in ('000000', '000016'):
    frame = capture_oracle.make_divisible(datasets.decode_image(SMALL / 'frames' / f'{name}.png'), 8)
    for s in (1, 2, 4, 8):
      np.testing.assert_array_equal(capture_oracle.downsample(frame, s),
                                    datasets.decode_image(EXPECTED / 'rgb' / f'{s}x' / f'{name}.png'))


def test_oracle_grey_equals_cv2_for_every_rgb_triple():
  cv2 = pytest.importorskip('cv2')
  v = np.arange(1 << 24, dtype=np.uint32)
  rgb = np.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
  np.testing.assert_array_equal(capture_oracle.grey(rgb), cv2.cvtColor(rgb, cv2.COLOR_RGB2GRAY))


def test_oracle_blur_score_equals_cv2(ref):
  cv2 = pytest.importorskip('cv2')
  from nerfies_b200 import datasets
  rng = np.random.RandomState(1)
  for h, w in ((1, 7), (2, 2), (37, 53)):
    image = rng.randint(0, 256, size=(h, w, 3), dtype=np.uint8)
    g = cv2.cvtColor(image, cv2.COLOR_RGB2GRAY)
    np.testing.assert_array_equal(capture_oracle.laplacian(g), cv2.Laplacian(g, cv2.CV_64F))
  for item, score in zip(ref['blur_ids'], ref['blur_scores']):
    image = datasets.decode_image(EXPECTED / 'rgb' / '1x' / f'{item}.png')
    assert capture_oracle.blur_score(image) == pytest.approx(score, rel=1e-12)
