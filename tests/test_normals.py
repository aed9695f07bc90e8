"""The drivers' normal outputs without a GPU: the flags, the refusals that come before any GPU work, and the
video loop's normal frames over stand-ins (tests/test_visualization.py's)."""
import os

import numpy as np
import pytest

from nerfies_b200 import configs, datasets
from nerfies_b200 import eval as eval_lib
from nerfies_b200 import extract_mesh, render_video
from tests.test_visualization import _construct, _save, _Source


def test_eval_refuses_save_normals_without_saved_output(tmp_path):
  ev = configs.EvalConfig(save_output=False, eval_once=True)

  def construct(*a, **kw):
    raise AssertionError('no model is built before the refusal')
  with pytest.raises(ValueError, match='save_normals.*save_output'):
    eval_lib.evaluate(configs.ExperimentConfig(), configs.ModelConfig(), configs.TrainConfig(batch_size=8), ev,
                      str(tmp_path / 'exp'), datasource=_Source(str(tmp_path)), construct_fn=construct,
                      poll_seconds=0.0, log=lambda s: None, save_normals=True)
  assert not (tmp_path / 'exp').exists()


def test_eval_passes_normals_to_the_frame_function(tmp_path):
  base = tmp_path / 'exp'
  _save(base, 5)
  seen = []

  def frame(model, params, camera, warp_extra, metadata, rgb_target, normals=False):
    seen.append(normals)
    images = {'rgb': np.zeros((4, 6, 3), np.uint8)}
    if normals:
      images['normals'] = np.full((4, 6, 3), 9, np.uint8)
    return images, {}
  ev = configs.EvalConfig(eval_once=True, num_val_eval=None, num_train_eval=1, num_test_eval=1)
  train = configs.TrainConfig(batch_size=8, max_steps=5)
  assert eval_lib.evaluate(configs.ExperimentConfig(), configs.ModelConfig(), train, ev, str(base),
                           datasource=_Source(str(tmp_path)), construct_fn=_construct, frame_fn=frame,
                           poll_seconds=0.0, log=lambda s: None, save_normals=True) == [5]
  assert seen and all(seen)
  np.testing.assert_array_equal(datasets.decode_image(base / 'renders' / '00000005' / 'val' / 'normals_v0.png'),
                                np.full((4, 6, 3), 9, np.uint8))


def test_video_loop_writes_normal_frames(tmp_path):
  data = tmp_path / 'capture'
  (data / 'camera-paths' / 'orbit').mkdir(parents=True)
  for name in ('000', '001'):
    (data / 'camera-paths' / 'orbit' / f'{name}.json').write_text('{}')
  base = tmp_path / 'exp'
  _save(base, 3)

  def frame(model, params, camera, warp_extra, metadata, near, far, normals=False):
    index = int(os.path.basename(camera)[:3])
    rgb = np.full((2, 6, 3), [index, 1, 7], np.uint8)
    return (rgb, np.full((2, 3, 3), [index, 2, 8], np.uint8)) if normals else rgb

  run = lambda **kw: render_video.render_video(
      configs.ExperimentConfig(), configs.ModelConfig(), str(base), camera_path='camera-paths/orbit',
      datasource=_Source(data), construct_fn=_construct, frame_fn=frame, log=lambda s: None, **kw)
  out = run(normals=True)
  assert sorted(os.listdir(out)) == ['frame_00000.png', 'frame_00001.png', 'normals.mp4', 'normals_00000.png',
                                     'normals_00001.png', 'video.mp4']
  for i in range(2):
    np.testing.assert_array_equal(datasets.decode_image(out / f'normals_{i:05d}.png')[0, 0], [i, 2, 8])
    np.testing.assert_array_equal(datasets.decode_image(out / f'frame_{i:05d}.png')[0, 0], [i, 1, 7])
  for f in os.listdir(out):
    os.remove(out / f)
  out = run()                                                  # without the flag: today's files only
  assert sorted(os.listdir(out)) == ['frame_00000.png', 'frame_00001.png', 'video.mp4']


def _flag_seen(module, fn_name, argv, key):
  seen = {}
  original = getattr(module, fn_name)
  try:
    setattr(module, fn_name, lambda *a, **kw: seen.update(kw) or '/x/out')
    assert module.main(argv) == 0
  finally:
    setattr(module, fn_name, original)
    configs.clear_config()
  return seen[key]


def test_flags():
  base = ['--base_folder', '/x', '--gin_bindings', 'TrainConfig.batch_size = 8']
  assert _flag_seen(eval_lib, 'evaluate', base + ['--save_normals'], 'save_normals') is True
  assert _flag_seen(eval_lib, 'evaluate', base, 'save_normals') is False
  assert _flag_seen(render_video, 'render_video', base + ['--normals'], 'normals') is True
  assert _flag_seen(render_video, 'render_video', base, 'normals') is False
  assert _flag_seen(extract_mesh, 'extract_mesh', base + ['--analytic_normals'], 'analytic') is True
  assert _flag_seen(extract_mesh, 'extract_mesh', base, 'analytic') is False
