"""Depth supervision on the host: the depth maps of a data source, the config fields, the refusals of
`process_capture depth` before any GPU work, the metric-scale estimate's statistics and the drivers' depth
plumbing."""
import os
import shutil
import types

import numpy as np
import pytest

from nerfies_b200 import capture
from nerfies_b200 import configs
from nerfies_b200 import datasets
from nerfies_b200 import process_capture

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
CAPTURE = os.path.join(GOLDEN, 'capture_small')
IDS = ['left_000', 'left_003', 'right_001', 'left_007', 'right_004', 'right_009']


@pytest.fixture
def data(tmp_path):
  d = tmp_path / 'capture'
  shutil.copytree(CAPTURE, d)
  return d


def _source(data_dir, **kw):
  return datasets.from_config({'type': 'nerfies', 'data_dir': str(data_dir)}, image_scale=2, device='cpu',
                              use_depth=True, **kw)


def test_load_depth_marks_missing_values_and_absent_files(data):
  (data / 'depth' / '2x').mkdir(parents=True)
  m = np.linspace(0.5, 2.0, 27 * 48, dtype=np.float32).reshape(27, 48)
  m[0, :4] = [0.0, -1.0, np.inf, np.nan]
  np.save(data / 'depth' / '2x' / 'left_000.npy', m.astype(np.float64))   # any float dtype is read
  ds = _source(data)
  got = ds.load_depth('left_000')
  assert got.dtype == np.float32 and got.shape == (27, 48)
  assert np.isnan(got[0, :4]).all()
  np.testing.assert_array_equal(got[1:], m[1:])
  assert ds.load_depth('left_003') is None
  item = ds.get_item('left_000')
  assert tuple(item['depth'].shape) == (27, 48, 1)
  assert 'depth' not in ds.get_item('left_003')
  host = ds.ray_table(['left_000', 'left_003'])
  assert host.depths[1] is None and host.depths[0].shape == (27, 48)
  # no map for any item: a table without depth
  assert ds.ray_table(['left_003', 'right_001']).depths is None
  # use_depth off: no map is read
  plain = datasets.from_config({'type': 'nerfies', 'data_dir': str(data)}, image_scale=2, device='cpu')
  assert 'depth' not in plain.get_item('left_000') and plain.ray_table(['left_000']).depths is None


def test_depth_map_refusals(data):
  (data / 'depth' / '2x').mkdir(parents=True)
  np.save(data / 'depth' / '2x' / 'left_000.npy', np.ones((27, 47), np.float32))
  ds = _source(data)
  with pytest.raises(ValueError, match='depth map'):
    ds.get_item('left_000')
  with pytest.raises(ValueError, match='depth map'):
    ds.ray_table(['left_000'])
  np.save(data / 'depth' / '2x' / 'left_000.npy', np.ones((27, 48, 1), np.float32))
  with pytest.raises(ValueError, match='2-D float'):
    ds.load_depth('left_000')
  np.save(data / 'depth' / '2x' / 'left_000.npy', np.ones((27, 48), np.int32))
  with pytest.raises(ValueError, match='2-D float'):
    ds.load_depth('left_000')
  with pytest.raises(NotImplementedError, match='use_relative_depth'):
    _source(data, use_relative_depth=True)


def test_config_fields_parse_from_gin():
  configs.clear_config()
  try:
    t = configs.TrainConfig(batch_size=8)
    assert t.use_depth_loss is False and t.depth_loss_weight_schedule == ('constant', 0.0)
    configs.parse_config("TrainConfig.batch_size = 8\nTrainConfig.use_depth_loss = True\n"
                         "TrainConfig.depth_loss_weight_schedule = ('constant', 0.05)\n"
                         "ExperimentConfig.datasource_kwargs = {'use_depth': True}\n")
    t = configs.TrainConfig()
    assert t.use_depth_loss is True and t.depth_loss_weight_schedule == ('constant', 0.05)
    assert configs.ExperimentConfig().datasource_kwargs == {'use_depth': True}
  finally:
    configs.clear_config()


def _no_gpu(monkeypatch):
  def boom(*a, **k):
    raise AssertionError('GPU work started before the inputs were checked')
  monkeypatch.setattr(capture, 'resample_depth', boom)
  monkeypatch.setattr(capture, 'depth_scale_pairs', boom)


def _run(data, raw, *more):
  args = process_capture.make_parser().parse_args(
      ['depth', '--data_dir', str(data), '--depth_dir', str(raw), '--device', 'cpu', *more])
  return process_capture.run_depth(args, log=lambda *_: None)


def _raw(tmp_path, ids=IDS, shape=(27, 48), dtype=np.float32):
  raw = tmp_path / 'raw'
  raw.mkdir(exist_ok=True)
  for i in ids:
    np.save(raw / f'{i}.npy', np.ones(shape, dtype))
  return raw


def test_process_capture_depth_refusals_come_before_gpu_work(tmp_path, data, monkeypatch):
  _no_gpu(monkeypatch)
  raw = _raw(tmp_path, IDS[:-1])
  with pytest.raises(FileNotFoundError, match='right_009.*--allow_missing'):
    _run(data, raw, '--depth_scale', '2')
  np.save(raw / 'right_009.npy', np.ones((3, 4, 2), np.float32))
  with pytest.raises(ValueError, match='2-D float'):
    _run(data, raw, '--depth_scale', '2')
  np.save(raw / 'right_009.npy', np.ones((3, 4), np.uint16))
  with pytest.raises(ValueError, match='2-D float'):
    _run(data, raw, '--depth_scale', '2')
  np.save(raw / 'right_009.npy', np.ones((3, 4), np.float32))
  os.remove(data / 'scene.json')
  with pytest.raises(FileNotFoundError, match='scene.json'):
    _run(data, raw, '--depth_scale', '2')
  shutil.copy(os.path.join(CAPTURE, 'scene.json'), data / 'scene.json')
  os.remove(data / 'points.npy')
  with pytest.raises(FileNotFoundError, match='--depth_scale'):
    _run(data, raw)
  with pytest.raises(SystemExit):      # the scale must be positive
    _run(data, raw, '--depth_scale', '0')


def _write_png(path, rgb):
  """An 8-bit RGB PNG with the standard library alone."""
  import struct
  import zlib
  h, w, _ = rgb.shape
  chunk = lambda kind, data: (struct.pack('>I', len(data)) + kind + data +
                              struct.pack('>I', zlib.crc32(kind + data) & 0xffffffff))
  raw = b''.join(b'\x00' + rgb[y].tobytes() for y in range(h))
  path.write_bytes(b'\x89PNG\r\n\x1a\n' + chunk(b'IHDR', struct.pack('>IIBBBBB', w, h, 8, 2, 0, 0, 0)) +
                   chunk(b'IDAT', zlib.compress(raw)) + chunk(b'IEND', b''))


def test_a_frame_size_mismatch_is_refused_before_anything_is_written(tmp_path, data, monkeypatch):
  _no_gpu(monkeypatch)
  raw = _raw(tmp_path)
  _write_png(data / 'rgb' / '2x' / 'right_009.png', np.zeros((26, 48, 3), np.uint8))   # the last item
  with pytest.raises(ValueError, match='right_009.png is \\(26, 48\\)'):
    _run(data, raw, '--depth_scale', '2')
  assert not (data / 'depth').exists()


def test_allow_missing_skips_items(tmp_path, data, monkeypatch):
  raw = _raw(tmp_path, IDS[:2])
  calls = []
  monkeypatch.setattr(capture, 'resample_depth',
                      lambda sensor, cam, factor, device: calls.append((cam.image_shape, factor)) or
                      np.zeros(cam.image_shape, np.float32))
  out = _run(data, raw, '--depth_scale', '2', '--allow_missing')
  assert out['missing'] == IDS[2:]
  assert sorted(os.listdir(data / 'depth' / '2x')) == sorted(f'{i}.npy' for i in IDS[:2])
  assert calls == [((27, 48), 2 * 0.7)] * 2


def test_estimate_depth_scale_statistics_and_refusal():
  rng = np.random.RandomState(0)
  z = rng.uniform(1, 3, 101)
  pairs = [(z[:50], z[:50] / 1.7), (z[50:], z[50:] / 1.7)]
  scale, n, iqr = capture.estimate_depth_scale(pairs)
  assert n == 101 and abs(scale - 1.7) < 1e-12 and iqr < 1e-12
  noisy = [(z, z / (1.7 * (1 + 0.01 * rng.randn(101))))]
  scale, n, iqr = capture.estimate_depth_scale(noisy)
  assert abs(scale / 1.7 - 1) < 0.01 and 0 < iqr < 0.1
  with pytest.raises(ValueError, match='--depth_scale'):
    capture.estimate_depth_scale([(z[:10], z[:10])])
  with pytest.raises(ValueError, match='--depth_scale'):
    capture.estimate_depth_scale([])


def test_train_refuses_the_depth_loss_without_depth(data):
  from nerfies_b200 import train as train_lib
  t = types.SimpleNamespace(use_depth_loss=True)
  plain = datasets.from_config({'type': 'nerfies', 'data_dir': str(data)}, image_scale=2, device='cpu')
  with pytest.raises(ValueError, match='datasource_kwargs'):
    train_lib.check_depth(t, plain)
  with pytest.raises(ValueError, match='process_capture depth'):
    train_lib.check_depth(t, _source(data))
  (data / 'depth' / '2x').mkdir(parents=True)
  np.save(data / 'depth' / '2x' / f'{_source(data).train_ids[0]}.npy', np.ones((27, 48), np.float32))
  train_lib.check_depth(t, _source(data))
  train_lib.check_depth(types.SimpleNamespace(use_depth_loss=False), plain)


def test_eval_passes_depth_targets_to_the_frame_function():
  from nerfies_b200 import eval as eval_lib
  seen = []

  def frame_fn(model, params, camera, warp_extra, metadata, rgb_target, **kw):
    seen.append(kw)
    return {}, {'mse': 1.0, **({'depth_abs': 0.5} if 'depth_target' in kw else {})}

  class Writer:
    def __init__(self):
      self.rows = []

    def write(self, step, scalars):
      self.rows.append(scalars)

  w = Writer()
  items = [('a', None, {}, 0.0, 'DEPTH'), ('b', None, {}, 0.0)]
  eval_lib.process_items('val', items, 1, None, None, None, None, w, None, frame_fn, log=lambda *_: None)
  assert seen == [{'depth_target': 'DEPTH'}, {}]
  assert w.rows == [{'metrics-eval/mse/val': 1.0, 'metrics-eval/depth_abs/val': 0.5}]
  # an item without a single measurement (NaN depth_abs) drops out of the tag's depth mean
  w.rows = []
  frame_nan = lambda *a, **kw: ({}, {'mse': 1.0, **({'depth_abs': kw['depth_target']} if 'depth_target' in kw else {})})
  eval_lib.process_items('val', [('a', None, {}, 0.0, float('nan')), ('b', None, {}, 0.0, 0.25)], 1, None, None, None,
                         None, w, None, frame_nan, log=lambda *_: None)
  assert w.rows == [{'metrics-eval/mse/val': 1.0, 'metrics-eval/depth_abs/val': 0.25}]
  # refined train items keep their depth
  out = eval_lib.refined_items(items, None, None)
  assert out[0][4] == 'DEPTH' and len(out[1]) == 4
