"""Capture processing on the GPU against the capture the reference's notebook wrote
(tests/golden/colmap_small, tests/golden/capture_process.npz) and against numpy: pyramid pixels,
blur scores, per-camera near/far planes, Camera.project, and `images` + `scene` end to end, followed
by loading and training on the result."""
import json
import pathlib

import numpy as np
import pytest
import torch

from nerfies_b200 import camera as camera_lib
from nerfies_b200 import capture
from nerfies_b200 import colmap
from nerfies_b200 import datasets
from nerfies_b200 import process_capture
from tests import capture_oracle

pytestmark = pytest.mark.gpu
ROOT = pathlib.Path(__file__).resolve().parent.parent
GOLDEN = ROOT / 'tests' / 'golden'
SMALL = GOLDEN / 'colmap_small'
EXPECTED = SMALL / 'expected'
DEV = torch.device('cuda', 0)


@pytest.fixture(scope='module')
def ref():
  return dict(np.load(GOLDEN / 'capture_process.npz'))


def _d(a):
  return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def test_pyramid_equals_the_notebooks_pngs():
  for f in sorted((SMALL / 'frames').glob('*.png')):
    levels = capture.downsample_frames(_d(datasets.decode_image(f)), [1, 2, 4, 8])
    for s, t in levels.items():
      np.testing.assert_array_equal(t.cpu().numpy(), datasets.decode_image(EXPECTED / 'rgb' / f'{s}x' / f.name),
                                    err_msg=f'{f.name} {s}x')


def test_pyramid_of_a_1080p_frame_equals_the_oracle():
  rng = np.random.RandomState(3)
  frame = rng.randint(0, 256, size=(1085, 1923, 3), dtype=np.uint8)
  for scales in ([1, 2, 4, 8], [8, 2], [1], [16, 4, 2, 1], [6, 2]):
    levels = capture.downsample_frames(_d(frame), scales)
    cropped = capture_oracle.make_divisible(frame, max(scales))
    assert sorted(levels) == sorted(scales)
    for s, t in levels.items():
      np.testing.assert_array_equal(t.cpu().numpy(), capture_oracle.downsample(cropped, s), err_msg=f'{scales} {s}')
  # a non-contiguous view (a crop of a wider frame) reads through its row pitch
  wide = _d(frame)[:, 3:3 + 1600]
  np.testing.assert_array_equal(capture.downsample_frames(wide, [4])[4].cpu().numpy(),
                                capture_oracle.downsample(frame[:1084, 3:1603], 4))


def test_pyramid_refusals():
  frame = torch.zeros(16, 16, 3, dtype=torch.uint8, device=DEV)
  for scales, msg in (([3], 'scale 3'), ([4, 6], 'does not divide'), ([32], 'smaller')):
    with pytest.raises(ValueError, match=msg):
      capture.downsample_frames(frame, scales)
  with pytest.raises(ValueError, match='uint8'):
    capture.downsample_frames(frame.float(), [2])


def test_blur_scores_equal_the_notebook(ref):
  ids = ref['blur_ids'].tolist()
  frames = np.stack([datasets.decode_image(EXPECTED / 'rgb' / '1x' / f'{i}.png') for i in ids])
  got = capture.blur_scores(_d(frames)).cpu().numpy()
  np.testing.assert_allclose(got, ref['blur_scores'], rtol=1e-12, atol=0)
  rng = np.random.RandomState(5)
  for shape in ((3, 1080, 1920), (2, 1, 9), (1, 2, 2), (5, 33, 47)):
    frames = rng.randint(0, 256, size=shape + (3,), dtype=np.uint8)
    got = capture.blur_scores(_d(frames)).cpu().numpy()
    want = [capture_oracle.blur_score(f) for f in frames]
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=0, err_msg=str(shape))


def _scene():
  cameras, points = colmap.load_scene(SMALL / 'sparse' / '0', process_capture.MIN_TRACK_LENGTH)
  return {k: c.scale(4) for k, c in cameras.items()}, points


def test_near_far_per_camera_equals_the_notebook(ref):
  cameras, points = _scene()
  cams = [cameras[str(i)] for i in ref['item_ids']]
  near_i, far_i, counts = capture.near_far_per_camera(cams, capture.scene_points(points, cams), DEV)
  np.testing.assert_array_equal(counts, ref['counts'])
  np.testing.assert_allclose(near_i, ref['near_i'], rtol=1e-12, atol=0)
  np.testing.assert_allclose(far_i, ref['far_i'], rtol=1e-12, atol=0)
  near, far, _ = capture.estimate_near_far([str(i) for i in ref['item_ids']], cams, points, DEV)
  assert near == pytest.approx(float(ref['near']), rel=1e-12)
  assert far == pytest.approx(float(ref['far']), rel=1e-12)


def _numpy_near_far(cam, pts):
  c = {k: np.asarray(v) for k, v in cam.get_parameters().items()}
  local = np.matmul(c['orientation'], (pts - c['position']).T).T
  with np.errstate(divide='ignore', invalid='ignore'):
    x, y = local[:, 0] / local[:, 2], local[:, 1] / local[:, 2]
    r2 = x ** 2 + y ** 2
    rd, td = c['radial_distortion'], c['tangential_distortion']
    d = 1.0 + r2 * (rd[0] + r2 * (rd[1] + rd[2] * r2))
    xy = x * y
    xd = x * d + 2.0 * td[0] * xy + td[1] * (r2 + 2.0 * x ** 2)
    yd = y * d + 2.0 * td[1] * xy + td[0] * (r2 + 2.0 * y ** 2)
    px = c['focal_length'] * xd + c['skew'] * yd + c['principal_point'][0]
    py = c['focal_length'] * c['pixel_aspect_ratio'] * yd + c['principal_point'][1]
    inside = (px >= 0) & (px <= cam.image_size_x) & (py >= 0) & (py <= cam.image_size_y)
  depths = local[:, 2][inside]
  depths = depths[depths > 0]
  if len(depths) == 0:
    return np.nan, np.nan, 0
  return np.quantile(depths, 0.001), np.quantile(depths, 0.999), len(depths)


def test_near_far_synthetic_against_numpy():
  rng = np.random.RandomState(11)
  w, h = 640, 480
  cams = []
  for k in range(64):
    a = 2 * np.pi * k / 64
    pos = np.array([3 * np.cos(a), 0.2 * np.sin(3 * a), 3 * np.sin(a)])
    z = -pos / np.linalg.norm(pos)
    x = np.cross([0, -1, 0], z); x /= np.linalg.norm(x)
    cams.append(camera_lib.Camera(np.stack([x, np.cross(z, x), z]), pos, 500.0 + k, [w / 2 + 1.5, h / 2 - 2.5],
                                  [w, h], skew=0.01 * (k % 3), pixel_aspect_ratio=1.0 + 0.001 * k,
                                  radial_distortion=[0.01, -0.02, 0.003], tangential_distortion=[1e-3, -2e-3]))
  # camera 5 looks away from every point
  c5 = cams[5]
  cams[5] = camera_lib.Camera(-c5.orientation, c5.position * 10, 500.0, [w / 2, h / 2], [w, h])
  pts = rng.normal(size=(300_000, 3)) * 0.8
  pts[:1000] *= 5                                        # many behind some camera
  # camera 63: a pinhole at the origin; points landing exactly on its frame edges count (inclusive bound)
  cams[63] = camera_lib.Camera(np.eye(3), np.zeros(3), 100.0, [50.0, 40.0], [100, 80])
  pts[1000:1004] = [[-1.0, 0.0, 2.0], [1.0, 0.8, 2.0], [1.0, -0.8, 4.0], [1.0001, 0.0, 2.0]]
  want = [_numpy_near_far(c, pts) for c in cams]
  near_i, far_i, counts = capture.near_far_per_camera(cams, pts, DEV)
  assert counts[5] == 0 and np.isnan(near_i[5]) and np.isnan(far_i[5])
  np.testing.assert_array_equal(counts, [n for _, _, n in want])
  np.testing.assert_allclose(near_i, [v for v, _, _ in want], rtol=1e-12, atol=0)
  np.testing.assert_allclose(far_i, [v for _, v, _ in want], rtol=1e-12, atol=0)
  ids = [f'item{k}' for k in range(64)]
  with pytest.raises(ValueError, match='item5'):
    capture.estimate_near_far(ids, cams, pts, DEV)
  _, _, c63 = capture.near_far_per_camera(cams[63:], pts[1000:1004], DEV)
  assert c63.tolist() == [3]
  _, _, none = capture.near_far_per_camera(cams[:2], np.zeros((0, 3)), DEV)
  assert none.tolist() == [0, 0]


@pytest.mark.parametrize('name', ['camera_distorted', 'camera_pinhole', 'camera_skew_distorted'])
def test_camera_project_equals_the_reference(name):
  z = np.load(GOLDEN / f'{name}.npz')
  cam = {k[4:]: z[k] for k in z.files if k.startswith('cam_')}
  c = camera_lib.Camera(**cam)
  pts = cam['position'] + z['directions'].reshape(-1, 3)[::7] * np.float32(1.5)
  got = c.project(_d(pts.astype(np.float32))).cpu().numpy()
  want = z['projected']
  ulp = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
  assert ulp.max() == 0, f'{name}: {int(ulp.max())} ulp, {int((ulp > 0).sum())} of {ulp.size} values differ'


def _j(p):
  with open(p) as f:
    return json.load(f)


def test_end_to_end_reproduces_the_notebook(tmp_path, ref):
  data = tmp_path / 'capture'
  assert process_capture.main(['images', '--frames_dir', str(SMALL / 'frames'), '--data_dir', str(data)]) == 0
  result = process_capture.run_scene(process_capture.make_parser().parse_args(
      ['scene', '--data_dir', str(data), '--colmap_dir', str(SMALL / 'sparse' / '0')]))
  assert result['removed'] == ref['removed_ids'].tolist()
  for s in (1, 2, 4, 8):
    names = sorted(p.name for p in (EXPECTED / 'rgb' / f'{s}x').iterdir())
    assert sorted(p.name for p in (data / 'rgb' / f'{s}x').iterdir()) == names
    for n in names:
      np.testing.assert_array_equal(datasets.decode_image(data / 'rgb' / f'{s}x' / n),
                                    datasets.decode_image(EXPECTED / 'rgb' / f'{s}x' / n))
  assert _j(data / 'dataset.json') == _j(EXPECTED / 'dataset.json')
  assert _j(data / 'metadata.json') == _j(EXPECTED / 'metadata.json')
  got, want = _j(data / 'scene.json'), _j(EXPECTED / 'scene.json')
  assert sorted(got) == sorted(want)
  for k in want:
    np.testing.assert_allclose(got[k], want[k], rtol=1e-9, err_msg=k)
  for sub in ('camera', 'camera-paths/orbit-mild'):
    files = sorted(p.name for p in (EXPECTED / sub).iterdir())
    assert sorted(p.name for p in (data / sub).iterdir()) == files
    for n in files:
      g, w = _j(data / sub / n), _j(EXPECTED / sub / n)
      assert sorted(g) == sorted(w)
      for k in w:
        if sub == 'camera':
          np.testing.assert_array_equal(np.float32(g[k]), np.float32(w[k]), err_msg=f'{n} {k}')
        else:   # look_at cameras: float64 in the notebook, float32 here
          np.testing.assert_allclose(np.float32(g[k]), np.float32(w[k]), rtol=2e-6, atol=2e-6, err_msg=f'{n} {k}')
  np.testing.assert_array_equal(np.load(data / 'points.npy'), ref['points'])

  source = datasets.from_config({'type': 'nerfies', 'data_dir': str(data)}, image_scale=4, device=DEV,
                                use_appearance_id=True, use_warp_id=True, random_seed=0)
  batch = next(source.create_iterator(source.train_ids, batch_size=64, flatten=True, shuffle=True))
  assert batch['rgb'].shape == (64, 3) and batch['origins'].is_cuda
  assert source.load_points().shape == (len(ref['points']), 3)

  from nerfies_b200 import train as train_lib
  gin = tmp_path / 'bg.gin'
  base = (ROOT / 'tests' / 'golden' / 'gin' / 'test_local.gin').read_text()
  gin.write_text(base + '\nTrainConfig.use_background_loss = True\nTrainConfig.batch_size = 256\n')
  assert train_lib.main(['--base_folder', str(tmp_path / 'exp'), '--data_dir', str(data), '--gin_configs', str(gin),
                         '--max_steps', '2']) == 0
  assert (tmp_path / 'exp' / 'summaries' / 'train.jsonl').exists()
