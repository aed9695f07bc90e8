"""The colour maps without a GPU: the numpy statement of colorize (tests/viz_oracle.py) against the
fixture recorded from the reference's own source, OpenCV's turbo table against the reference's,
and the video and eval drivers' loops over stand-ins."""
import os

import numpy as np
import pytest

from nerfies_b200 import checkpoints, configs, datasets, model_utils, visualization
from nerfies_b200 import eval as eval_lib
from nerfies_b200 import render_video
from tests import viz_oracle

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'viz_turbo.npz')


@pytest.fixture(scope='module')
def golden():
  return dict(np.load(GOLDEN))


def _cases(g):
  """(fixture key, values, colorize keyword arguments) of every colorize call the fixture records."""
  near, far = float(g['near']), float(g['far'])
  values = viz_oracle.source_values
  cases = []
  for inv in (0, 1):
    cases += [(f'unit_given_inv{inv}', g['unit'], dict(cmin=0.0, cmax=1.0, invert=bool(inv))),
              (f'unit_int_inv{inv}', g['unit'], dict(cmin=0, cmax=1, invert=bool(inv))),
              (f'finite_frame_inv{inv}', g['finite'], dict(invert=bool(inv))),
              (f'finite_min_inv{inv}', g['finite'], dict(cmax=0.75, invert=bool(inv)))]
  return cases + [
      ('unit_frame_inv0', g['unit'], {}), ('flat_frame_inv0', g['flat'], {}),
      ('depth_viz', g['depth'], dict(cmin=near, cmax=far, invert=True)),
      ('disp_viz', values(g['depth'], 'reciprocal'), {}),
      ('disp_positive_viz', values(g['positive_depth'], 'reciprocal'), {}),
      ('acc_viz', g['acc'], dict(cmin=0.0, cmax=1.0)),
      ('abs_error_viz', values(g['target'], 'abs_error', g['rgb']), dict(cmin=0, cmax=1)),
      ('sq_error_viz', values(g['target'], 'sq_error', g['rgb']), dict(cmin=0, cmax=1))]


def test_oracle_equals_the_reference_bit_for_bit(golden):
  for key, values, kw in _cases(golden):
    got = viz_oracle.colorize(values, golden['table'], **kw)
    np.testing.assert_array_equal(got, golden[key], err_msg=key)                 # NaN == NaN here
    np.testing.assert_array_equal(viz_oracle.to_uint8(got), golden[key + '_u8'], err_msg=key)
  assert np.isnan(golden['unit_frame_inv0']).all() and (golden['disp_viz_u8'][0, 0] == 0).all()
  frame = viz_oracle.video_frame(golden['video_rgb'], golden['depth'], golden['table'], float(golden['near']),
                                 float(golden['far']))
  np.testing.assert_array_equal(frame, golden['video_frame'])


def test_opencv_turbo_is_the_reference_table_rounded_to_8_bits(golden):
  np.testing.assert_array_equal(visualization.get_colormap('turbo'), np.round(255 * golden['table']) / 255)
  assert visualization.get_colormap('magma').shape == (256, 3)
  with pytest.raises(ValueError, match='unknown colour map'):
    visualization.get_colormap('no_such_map')
  with pytest.raises(ValueError, match=r'\(256, 3\)'):
    visualization.get_colormap(np.zeros((255, 3)))


def test_float32_and_float64_products_quantise_alike():
  """The video frame's rgb half: concatenate promotes rgb to float64 before the product with 255.
  For every float32 in [1/512, 1] that product truncates to the same integer as the float32 product
  (below 1/512 both are under 0.5, above 1 both clip to 255)."""
  lo, hi = np.float32(1 / 512).view(np.int32), np.float32(1).view(np.int32)
  for start in range(lo, hi + 1, 1 << 24):
    v = np.arange(start, min(start + (1 << 24), hi + 1), dtype=np.int32).view(np.float32)
    assert np.array_equal((v * np.float32(255)).astype(np.uint8), (v.astype(np.float64) * 255).astype(np.uint8))


def test_no_cpu_path():
  import torch
  with pytest.raises(ValueError, match='CUDA'):
    visualization.colorize(torch.zeros(4, 4))
  with pytest.raises(ValueError, match='CUDA'):
    visualization.colorize_uint8(np.zeros((4, 4), np.float32))


# ---- the drivers' loops over stand-ins ------------------------------------------------------------
class _Source:
  use_appearance_id = use_warp_id = use_camera_id = use_time = True
  appearance_ids = warp_ids = camera_ids = (0, 1, 2)
  near, far = 0.1, 2.0
  train_ids = ['t0', 't1']
  val_ids = ['v0']

  def __init__(self, data_dir):
    self.data_dir = data_dir

  glob_cameras = datasets.NerfiesDataSource.glob_cameras
  camera_ext = '.json'

  def load_camera(self, path):
    return str(path)

  def get_item(self, item_id):
    return {'rgb': np.full((4, 6, 3), 0.5, np.float32), 'metadata': {}}

  def load_test_cameras(self, count=None):
    return ['camera:test0']


def _save(base, *steps):
  for step in steps:
    state = model_utils.TrainState(model_utils.Optimizer({'model': {'w': np.full((1,), step, np.float32)}}))
    checkpoints.save_checkpoint(str(base / 'checkpoints'), state, step)


def _construct(key, config, **kw):
  return object(), {'w': np.zeros((1,), np.float32)}


def test_video_loop_over_stand_ins(tmp_path):
  data = tmp_path / 'capture'
  (data / 'camera-paths' / 'orbit').mkdir(parents=True)
  for name in ('002', '000', '001', '003'):
    (data / 'camera-paths' / 'orbit' / f'{name}.json').write_text('{}')
  base = tmp_path / 'exp'
  _save(base, 30, 60)
  (base / 'renders' / '00000060').mkdir(parents=True)
  calls = []

  def frame(model, params, camera, warp_extra, metadata, near, far):
    step = int(params['w'][0])
    calls.append((camera, dict(metadata), near, far))
    index = int(os.path.basename(camera)[:3])
    return np.full((2, 6, 3), [index, step, 7], np.uint8)

  run = lambda **kw: render_video.render_video(
      configs.ExperimentConfig(), configs.ModelConfig(), str(base), camera_path='camera-paths/orbit',
      datasource=_Source(data), construct_fn=_construct, frame_fn=frame, log=lambda s: None, **kw)
  out = run()
  assert out == base / 'videos' / 'orbit' / '00000060'                           # the newest step
  assert sorted(os.listdir(out)) == [f'frame_{i:05d}.png' for i in range(4)] + ['video.mp4']
  for i in range(4):                                                             # sorted camera order
    np.testing.assert_array_equal(datasets.decode_image(out / f'frame_{i:05d}.png')[0, 0], [i, 60, 7])
  assert calls[0][1:] == ({'appearance': 0, 'warp': 0, 'camera': 0, 'time': 0.0}, 0.1, 2.0)
  assert os.listdir(base / 'renders') == ['00000060']                            # renders/ untouched
  import cv2
  video = cv2.VideoCapture(str(out / 'video.mp4'))
  count = 0
  while video.read()[0]:
    count += 1
  assert count == 4

  calls.clear()
  out = run(step=30, metadata=['appearance=2', 'time=0.25'])
  assert out == base / 'videos' / 'orbit' / '00000030'
  assert calls[0][1] == {'appearance': 2, 'warp': 0, 'camera': 0, 'time': 0.25}
  np.testing.assert_array_equal(datasets.decode_image(out / 'frame_00003.png')[0, 0], [3, 30, 7])
  with pytest.raises(FileNotFoundError, match='step 45'):
    run(step=45)
  with pytest.raises(ValueError, match='key=value'):
    run(metadata=['bogus=1'])


def test_video_flags():
  parser_args = ['--base_folder', '/x', '--camera_path', 'camera-paths/a', '--fps', '24', '--step', '5',
                 '--metadata', 'warp=1', '--metadata', 'appearance=2']
  seen = {}
  original = render_video.render_video
  try:
    render_video.render_video = lambda *a, **kw: seen.update(kw) or '/x/out'
    assert render_video.main(parser_args) == 0
  finally:
    render_video.render_video = original
  assert (seen['camera_path'], seen['fps'], seen['step'], seen['metadata']) == (
      'camera-paths/a', 24.0, 5, ['warp=1', 'appearance=2'])


def test_eval_save_viz_over_stand_ins(tmp_path):
  base = tmp_path / 'exp'
  _save(base, 60)
  seen = []

  def frame(model, params, camera, warp_extra, metadata, rgb_target, viz_range=None):
    seen.append(viz_range)
    images = {'rgb': np.zeros((4, 6, 3), np.uint8), 'depth_expected': np.zeros((4, 6), np.uint16),
              'depth_median': np.zeros((4, 6), np.uint16)}
    if viz_range is not None:
      stems = ['depth_expected_viz', 'depth_median_viz', 'disparity_expected_viz', 'disparity_median_viz', 'acc_viz']
      if rgb_target is not None:
        stems += ['rgb_abs_error_viz', 'rgb_sq_error_viz']
      images.update({s: np.full((4, 6, 3), 9, np.uint8) for s in stems})
    return images, {}

  ev = configs.EvalConfig(eval_once=True, num_val_eval=None, num_train_eval=1, num_test_eval=1)
  assert eval_lib.evaluate(configs.ExperimentConfig(), configs.ModelConfig(), configs.TrainConfig(batch_size=8, max_steps=60), ev,
                           str(base), datasource=_Source(tmp_path), construct_fn=_construct, frame_fn=frame,
                           poll_seconds=0.0, log=lambda s: None, save_viz=True) == [60]
  assert set(seen) == {(0.1, 2.0)}
  out = base / 'renders' / '00000060'
  base_stems = ['rgb', 'depth_expected', 'depth_median', 'depth_expected_viz', 'depth_median_viz',
                'disparity_expected_viz', 'disparity_median_viz', 'acc_viz']
  assert sorted(os.listdir(out / 'val')) == sorted(f'{s}_v0.png' for s in base_stems + ['rgb_abs_error_viz',
                                                                                        'rgb_sq_error_viz'])
  assert sorted(os.listdir(out / 'test')) == sorted(f'{s}_000.png' for s in base_stems)   # no target: no error maps
