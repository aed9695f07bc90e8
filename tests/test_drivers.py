"""Host logic of the train / eval drivers, without a GPU: flags, gin files into the config
dataclasses, the experiment layout, eval's choice of items, checkpoint polling, the scalar log,
the eval loop over stand-ins for the data source, model and renderer, Adam's moments through a
checkpoint, and the numpy statement of the image conversions on hand-computed values."""
import os

import numpy as np
import pytest
import torch

from nerfies_b200 import checkpoints, configs, datasets, driver_utils, model_utils, training
from nerfies_b200 import eval as eval_lib
from nerfies_b200 import train as train_lib
from tests import image_oracle

GIN = """
include 'base.gin'
ExperimentConfig.image_scale = 2
ExperimentConfig.subname = 'run_a'
ModelConfig.num_coarse_samples = %samples
TrainConfig.batch_size = 512
TrainConfig.max_steps = 60
TrainConfig.lr_schedule = {'type': 'constant', 'value': 0.001}
EvalConfig.num_val_eval = None
"""
BASE_GIN = """
samples = 16
ModelConfig.use_warp = True
ModelConfig.warp_field_type = 'se3'
ModelConfig.sigma_activation = @nn.softplus
EvalConfig.chunk = 4096
"""


@pytest.fixture(autouse=True)
def _clean_gin():
  configs.clear_config()
  yield
  configs.clear_config()


def test_flags_have_the_reference_names():
  args = driver_utils.make_parser('train', 'fp32').parse_args(
      ['--base_folder', '/x', '--data_dir', '/d', '--gin_configs', 'a.gin', '--gin_configs', 'b.gin',
       '--gin_bindings', 'TrainConfig.batch_size = 8', '--max_steps', '7', '--train_precision', 'tf32x3'])
  assert (args.base_folder, args.data_dir, args.gin_configs) == ('/x', '/d', ['a.gin', 'b.gin'])
  assert args.gin_bindings == ['TrainConfig.batch_size = 8'] and args.max_steps == 7
  assert (args.precision, args.train_precision) == ('fp32', 'tf32x3')
  with pytest.raises(SystemExit):
    driver_utils.make_parser('train', 'fp32').parse_args(['--data_dir', '/d'])        # no --base_folder
  with pytest.raises(SystemExit):
    driver_utils.make_parser('train', 'fp32').parse_args(['--base_folder', '/x', '--precision', 'fp8'])


def test_gin_files_resolve_into_the_config_dataclasses(tmp_path):
  (tmp_path / 'base.gin').write_text(BASE_GIN)
  (tmp_path / 'test.gin').write_text(GIN)
  text = driver_utils.parse_configs([str(tmp_path / 'test.gin')], ['TrainConfig.save_every = 30'])
  exp, model, train = configs.ExperimentConfig(), configs.ModelConfig(use_stratified_sampling=False), configs.TrainConfig()
  ev = configs.EvalConfig()
  assert (exp.image_scale, exp.subname) == (2, 'run_a')
  assert (model.num_coarse_samples, model.use_warp, model.sigma_activation) == (16, True, 'softplus')
  assert not model.use_stratified_sampling
  assert (train.batch_size, train.max_steps, train.save_every) == (512, 60, 30)
  assert (ev.chunk, ev.num_val_eval, ev.num_train_eval) == (4096, None, 10)
  assert 'ExperimentConfig.image_scale = 2' in text and 'TrainConfig.save_every = 30' in text
  # a second parse starts clean: bindings of the first do not leak into it
  driver_utils.parse_configs([], ['TrainConfig.batch_size = 4'])
  assert configs.TrainConfig().max_steps == 1000000


def test_experiment_layout(tmp_path):
  d = driver_utils.experiment_dirs(tmp_path, 'run_a')
  assert d['exp'] == tmp_path / 'run_a' and d['checkpoints'] == tmp_path / 'run_a' / 'checkpoints'
  assert d['summaries'] == tmp_path / 'run_a' / 'summaries' and d['renders'] == tmp_path / 'run_a' / 'renders'
  assert driver_utils.experiment_dirs(tmp_path)['exp'] == tmp_path


@pytest.mark.parametrize('count, want', [
    (0, list('abcdefg')), (None, list('abcdefg')), (1, ['a']), (2, ['a', 'd', 'g']), (3, ['a', 'c', 'e', 'g']),
    (4, list('abcdefg')), (7, list('abcdefg')), (20, list('abcdefg'))])
def test_eval_item_selection(count, want):
  assert eval_lib.strided_subset(list('abcdefg'), count) == want
  assert eval_lib.strided_subset([], count) == []


def test_checkpoint_polling_order(tmp_path):
  ckpt = tmp_path / 'checkpoints'
  assert eval_lib.checkpoint_steps(ckpt) == [] and eval_lib.next_checkpoint_step(ckpt, 0) is None
  ckpt.mkdir()
  assert eval_lib.next_checkpoint_step(ckpt, 0) is None
  for name in ('checkpoint_900', 'checkpoint_10000', 'checkpoint_30', 'checkpoint_30.tmp', 'notes.txt'):
    (ckpt / name).write_bytes(b'')
  assert eval_lib.checkpoint_steps(ckpt) == [30, 900, 10000]                    # numeric, not lexical
  assert eval_lib.next_checkpoint_step(ckpt, 0) == 10000
  assert eval_lib.next_checkpoint_step(ckpt, 900) == 10000
  assert eval_lib.next_checkpoint_step(ckpt, 10000) is None


def test_scalar_writer_appends_json_lines(tmp_path):
  path = tmp_path / 'summaries' / 'train.jsonl'
  w = driver_utils.ScalarWriter(path)
  w.write(5, {'loss/total/coarse': torch.tensor(0.25), 'params/learning_rate': 1e-3})
  w.close()
  w = driver_utils.ScalarWriter(path)                                            # a resumed run appends
  w.write(10, {'loss/total/coarse': np.float32(0.125)})
  w.close()
  assert driver_utils.read_scalars(path) == [
      {'step': 5, 'loss/total/coarse': 0.25, 'params/learning_rate': 1e-3}, {'step': 10, 'loss/total/coarse': 0.125}]


def test_train_helpers():
  keys = {train_lib.step_key(12345, r, s) for r in range(2) for s in range(1, 50)}
  assert len(keys) == 98 and all(0 <= k < 2**62 for k in keys)
  stats = {'coarse': {'loss/total': 1.0}, 'fine': {'loss/total': 2.0, 'metric/psnr': 3.0}, 'background_loss': 4.0}
  assert train_lib.flatten_stats(stats) == {'loss/total/coarse': 1.0, 'loss/total/fine': 2.0,
                                            'metric/psnr/fine': 3.0, 'loss/background': 4.0}


def test_first_batch_starts_the_stream_there():
  starts = lambda first: [s for s, _ in zip(datasets._batch_starts(100, 8, True, first), range(3))]
  assert starts(0) == [(0, 8), (8, 8), (16, 8)] and starts(30) == [(240, 8), (248, 8), (256, 8)]


# ---- Adam's moments through a checkpoint -------------------------------------------------------
def _adam(seed):
  g = torch.Generator().manual_seed(seed)
  flat = torch.randn(10, generator=g)
  target = {'model': {'a': {'kernel': flat[0:6].view(2, 3), 'bias': flat[6:9].view(3)}, 'e': {'embedding': flat[9:10].view(1, 1)}}}
  opt = training.AdamOptimizer(target, flat, [('a/kernel', 0, 6), ('a/bias', 6, 3), ('e/embedding', 9, 1)])
  opt.m.copy_(torch.randn(10, generator=g))
  opt.v.copy_(torch.rand(10, generator=g))
  return opt


def test_checkpoint_carries_adam_moments(tmp_path):
  """A checkpoint of a training state holds Adam's moments in flax's layout, and loading it into a
  fresh optimizer gives back parameters, moments and the step count bit for bit."""
  src = _adam(1)
  state = model_utils.TrainState(src, warp_alpha=2.5, time_alpha=0.5)
  checkpoints.save_checkpoint(str(tmp_path), state, 30)
  back = checkpoints.restore_checkpoint(str(tmp_path), state)
  leaf = back.param_states['model']['a']['kernel']
  assert set(leaf) == {'grad_ema', 'grad_sq_ema'} and leaf['grad_ema'].shape == (2, 3)
  dst = _adam(2)
  dst.load(back)
  assert dst.step == 30
  for name in ('flat', 'm', 'v'):
    assert torch.equal(getattr(dst, name), getattr(src, name)), name
  # a checkpoint without moments (a state that never trained) cannot be resumed from
  plain = model_utils.TrainState(model_utils.Optimizer(src.target))
  checkpoints.save_checkpoint(str(tmp_path / 'plain'), plain, 5)
  with pytest.raises(ValueError, match='no Adam moments'):
    _adam(3).load(checkpoints.restore_checkpoint(str(tmp_path / 'plain')))


# ---- the eval loop over stand-ins ---------------------------------------------------------------
class _Source:
  use_appearance_id = use_warp_id = True
  use_camera_id = use_time = False
  appearance_ids = warp_ids = (0, 1, 2)
  camera_ids = ()
  near, far = 0.1, 2.0
  train_ids = ['t0', 't1', 't2', 't3']
  val_ids = ['v0', 'v1']

  def load_camera(self, item_id):
    return f'camera:{item_id}'

  def get_item(self, item_id):
    return {'rgb': np.full((4, 6, 3), 0.5, np.float32), 'metadata': {'warp': 1, 'appearance': 2}}

  def load_test_cameras(self, count=None):
    return ['camera:test0']


def _frame(model, params, camera, warp_extra, metadata, rgb_target):
  """Stand-in renderer: images that encode the checkpoint's parameter, metrics that depend on it."""
  value = int(np.asarray(params['w']).reshape(-1)[0])
  rgb = np.zeros((4, 6, 3), np.uint8)
  rgb[..., 0], rgb[..., 1], rgb[..., 2] = value, 7, 200
  images = {'rgb': rgb, 'depth_expected': np.full((4, 6), 1000 + value, np.uint16),
            'depth_median': np.full((4, 6), 65535, np.uint16)}
  metrics = {} if rgb_target is None else {'mse': 0.01 * value, 'psnr': float(value)}
  return images, metrics


def test_eval_loop_over_stand_ins(tmp_path):
  base = tmp_path / 'exp'
  ckpt = str(base / 'checkpoints')
  for step in (30, 60):
    state = model_utils.TrainState(model_utils.Optimizer({'model': {'w': np.full((1,), step, np.float32)}}), warp_alpha=1.5)
    checkpoints.save_checkpoint(ckpt, state, step)
  exp = configs.ExperimentConfig()
  train = configs.TrainConfig(batch_size=8, max_steps=60)
  ev = configs.EvalConfig(eval_once=False, num_val_eval=None, num_train_eval=2, num_test_eval=1, max_render_checkpoints=1)
  construct = lambda key, config, **kw: (object(), {'w': np.zeros((1,), np.float32)})
  lines = []
  handled = eval_lib.evaluate(exp, configs.ModelConfig(), train, ev, str(base), datasource=_Source(),
                              construct_fn=construct, frame_fn=_frame, poll_seconds=0.0, log=lines.append)
  assert handled == [60]                       # the newest checkpoint; it is the last step, so the loop ends
  records = driver_utils.read_scalars(base / 'summaries' / 'eval.jsonl')
  assert records == [{'step': 60, 'metrics-eval/mse/val': pytest.approx(0.6), 'metrics-eval/psnr/val': 60.0},
                     {'step': 60, 'metrics-eval/mse/train': pytest.approx(0.6), 'metrics-eval/psnr/train': 60.0}]
  out = base / 'renders' / '00000060'
  assert sorted(os.listdir(out)) == ['test', 'train', 'val']
  assert sorted(os.listdir(out / 'val')) == sorted(f'{stem}_{i}.png' for i in ('v0', 'v1')
                                                   for stem in ('rgb', 'depth_expected', 'depth_median'))
  assert sorted(os.listdir(out / 'train')) == sorted(f'{stem}_{i}.png' for i in ('t0', 't2')
                                                     for stem in ('rgb', 'depth_expected', 'depth_median'))
  assert sorted(os.listdir(out / 'test')) == ['depth_expected_000.png', 'depth_median_000.png', 'rgb_000.png']
  rgb = datasets.decode_image(out / 'val' / 'rgb_v1.png')
  assert rgb.shape == (4, 6, 3) and (rgb == np.array([60, 7, 200], np.uint8)).all()        # RGB order kept
  import cv2
  depth = cv2.imread(str(out / 'test' / 'depth_expected_000.png'), cv2.IMREAD_UNCHANGED)
  assert depth.dtype == np.uint16 and (depth == 1060).all()
  assert sum('no MS-SSIM' in line for line in lines) == 2                        # one notice per scored set

  # eval_once handles the newest checkpoint and returns even when it is not the last step; only
  # max_render_checkpoints render directories are kept
  train90 = configs.TrainConfig(batch_size=8, max_steps=90)
  ev_once = configs.EvalConfig(eval_once=True, num_val_eval=1, num_train_eval=1, num_test_eval=1, max_render_checkpoints=1)
  checkpoints.save_checkpoint(ckpt, model_utils.TrainState(model_utils.Optimizer({'model': {'w': np.full((1,), 75, np.float32)}})), 75)
  assert eval_lib.evaluate(exp, configs.ModelConfig(), train90, ev_once, str(base), datasource=_Source(),
                           construct_fn=construct, frame_fn=_frame, poll_seconds=0.0, log=lines.append) == [75]
  assert os.listdir(base / 'renders') == ['00000075']


# ---- the image conversions, stated with numpy, on hand-computed values ---------------------------
def test_image_conversions_on_hand_computed_values():
  f = lambda *v: np.array(v, np.float32)
  below_one = np.nextafter(np.float32(1), np.float32(0))
  # 0.999 * 255 = 254.745 -> 254: the cast truncates; 254.9999 / 255 likewise
  assert image_oracle.image_to_uint8(f(0.0, 1.0, 0.999, below_one, 0.5, 1 / 255, -0.0)).tolist() == [0, 255, 254, 254, 127, 1, 0]
  assert image_oracle.image_to_uint8(f(-1e-9, -3.0, 1.0000001, 2.0, 1e30)).tolist() == [0, 0, 255, 255, 255]
  assert image_oracle.image_to_uint8(f(np.nan, -np.nan, np.inf, -np.inf)).tolist() == [0, 0, 255, 0]
  assert image_oracle.image_to_uint8(f(1e-45, 0.00392, 0.00393)).tolist() == [0, 0, 1]    # 0.9996 -> 0, 1.00215 -> 1
  assert image_oracle.image_to_uint16(f(0.0, 1.0, 0.999, below_one, 0.5, -0.0)).tolist() == [0, 65535, 65469, 65534, 32767, 0]
  assert image_oracle.image_to_uint16(f(-1e-9, -3.0, 1.0000001, 2.0)).tolist() == [0, 0, 65535, 65535]
  assert image_oracle.image_to_uint16(f(np.nan, -np.nan, np.inf, -np.inf)).tolist() == [0, 0, 65535, 0]
  # save_depth: depth / 1000 in float32, then the 16-bit conversion: 1.0 -> 65.535 -> 65
  assert image_oracle.depth_to_uint16(f(0.0, 1.0, 500.0, 999.99, 1000.0, 2000.0, -1.0, np.nan, np.inf)).tolist() == [
      0, 65, 32767, 65534, 65535, 65535, 0, 0, 65535]
  assert image_oracle.image_to_uint8(image_oracle.SPECIALS).dtype == np.uint8


def test_quantize_entry_point_rejects_bad_arguments():
  import ctypes
  from nerfies_b200 import _lib
  lib = _lib.load()
  p = ctypes.c_void_p(256)
  assert lib.nfb_image_quantize(p, 16, 12, 1.0, p, None) != 0 and b'bits' in lib.nfb_last_error()
  assert lib.nfb_image_quantize(p, -1, 8, 1.0, p, None) != 0 and b'negative' in lib.nfb_last_error()
  for scale in (0.0, -1.0, float('nan'), float('inf')):
    assert lib.nfb_image_quantize(p, 16, 8, scale, p, None) != 0 and b'scale' in lib.nfb_last_error()
  if not torch.cuda.is_available():
    assert lib.nfb_image_quantize(p, 16, 8, 1.0, p, None) != 0 and b'no CUDA device' in lib.nfb_last_error()


def test_model_takes_the_empty_id_lists_of_a_data_source():
  """A data source gives () for metadata that is switched off (`camera_ids` without camera
  metadata); the model's configuration must not need a largest id of it."""
  from nerfies_b200 import models
  c = configs.ModelConfig(use_warp=True)
  model = models.NerfModel(
      num_coarse_samples=8, num_fine_samples=8, use_viewdirs=True, near=0.1, far=1.0, noise_std=None,
      nerf_trunk_depth=c.nerf_trunk_depth, nerf_trunk_width=c.nerf_trunk_width,
      nerf_rgb_branch_depth=c.nerf_rgb_branch_depth, nerf_rgb_branch_width=c.nerf_rgb_branch_width,
      use_alpha_condition=False, use_rgb_condition=False, activation='relu', sigma_activation='relu',
      nerf_skips=c.nerf_skips, alpha_channels=1, rgb_channels=3, use_stratified_sampling=False,
      use_white_background=False, use_sample_at_infinity=True, num_nerf_point_freqs=10, num_nerf_viewdir_freqs=4,
      use_linear_disparity=False, use_warp_jacobian=False, use_weights=False, use_appearance_metadata=False,
      use_camera_metadata=False, use_warp=True, appearance_ids=(), camera_ids=(), warp_ids=(3, 5),
      num_appearance_features=8, num_camera_features=2, num_warp_freqs=8, num_warp_features=8,
      warp_field_type='se3', warp_metadata_encoder_type='glo', warp_kwargs={}, precision='fp32', batch_size=8,
      device='cpu', train_precision='fp32')
  cfg = model.nfb_config()
  assert (cfg.num_warp_embeddings, cfg.num_appearance_embeddings, cfg.num_camera_embeddings) == (6, 1, 1)
