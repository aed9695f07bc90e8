"""The mesh driver's --track logic that needs no GPU: its refusals, the frames it visits and its flags."""
import json

import pytest

from nerfies_b200 import configs
from nerfies_b200 import extract_mesh


class _Source:
  """The datasource attributes the driver reads before any GPU work."""

  def __init__(self, data_dir, warp_ids=(), times=None):
    data_dir.mkdir(parents=True, exist_ok=True)
    (data_dir / 'scene.json').write_text(json.dumps({'center': [0, 0, 0], 'scale': 1.0, 'near': 0.1, 'far': 2.0}))
    self.data_dir = data_dir
    self.near, self.far = 0.1, 2.0
    self.warp_ids = tuple(warp_ids)
    self.use_time = times is not None
    self.train_ids = list(times) if times else []
    self._times = dict(times or {})

  def get_time(self, item_id):
    return self._times[item_id]


def _run(tmp_path, model_config, **kw):
  return extract_mesh.extract_mesh(configs.ExperimentConfig(), model_config, str(tmp_path),
                                   datasource=_Source(tmp_path / 'cap'), bbox=[[0, 0, 0], [1, 1, 1]],
                                   log=lambda s: None, track=True, **kw)


def test_track_refusals_come_before_any_gpu_work(tmp_path):
  warp = configs.ModelConfig(use_warp=True)
  with pytest.raises(ValueError, match='--canonical'):
    _run(tmp_path, warp, canonical=True)
  for item in ('warp=1', 'time=0.5'):
    with pytest.raises(ValueError, match='--frames'):
      _run(tmp_path, warp, metadata=[item])
  with pytest.raises(ValueError, match='warp field'):
    _run(tmp_path, configs.ModelConfig(use_warp=False))
  with pytest.raises(ValueError, match='--frames'):
    extract_mesh.extract_mesh(configs.ExperimentConfig(), warp, str(tmp_path), datasource=_Source(tmp_path / 'cap'),
                              frames=['1'], log=lambda s: None)
  # other metadata is the frames' own (appearance for the colours): past the refusals, to the missing checkpoint
  with pytest.raises(FileNotFoundError, match='no checkpoints'):
    _run(tmp_path, warp, metadata=['appearance=1'])


def test_track_frames(tmp_path):
  glo = configs.ModelConfig(use_warp=True)
  source = _Source(tmp_path / 'a', warp_ids=(10, 11, 20, 21))
  # the training frames as the model reads them: the index among the training warp ids
  assert extract_mesh.track_frames(source, glo) == [0, 1, 2, 3]
  assert extract_mesh.track_frames(source, glo, ['3', '1']) == [3, 1]
  with pytest.raises(ValueError):
    extract_mesh.track_frames(source, glo, ['0.5'])
  time = configs.ModelConfig(use_warp=True, warp_metadata_encoder_type='time')
  timed = _Source(tmp_path / 'b', times={'a': 0.5, 'b': -1.0, 'c': 0.5, 'd': 1.0})
  assert extract_mesh.track_frames(timed, time) == [-1.0, 0.5, 1.0]
  assert extract_mesh.track_frames(timed, time, ['0.25']) == [0.25]
  for cfg, empty in ((glo, _Source(tmp_path / 'c')), (time, _Source(tmp_path / 'd', times={}))):
    with pytest.raises(ValueError, match='pass --frames'):
      extract_mesh.track_frames(empty, cfg)


def test_track_flags():
  parse = lambda extra: extract_mesh.make_parser().parse_args(['--base_folder', '/x'] + extra)
  args = parse(['--track', '--frames', '2', '0', '5'])
  assert args.track and args.frames == ['2', '0', '5']
  args = parse([])
  assert not args.track and args.frames is None
  assert extract_mesh.TRACK_MAX_ITERS == 16 and extract_mesh.TRACK_TOL_VOXELS == 1e-2
