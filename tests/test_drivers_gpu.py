"""The train and eval drivers end to end on the small capture (tests/golden/capture_small: four
train and two val items of 27 x 48 pixels under rgb/2x, three test cameras): train, checkpoint,
resume, restore in a second model, render, save and score."""
import os
import sys

import cv2
import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAPTURE = os.path.join(ROOT, 'tests', 'golden', 'capture_small')

GIN = """
ExperimentConfig.image_scale = 2
ExperimentConfig.random_seed = 7
ModelConfig.num_coarse_samples = 16
ModelConfig.num_fine_samples = 16
ModelConfig.use_warp = True
ModelConfig.warp_field_type = 'se3'
ModelConfig.use_appearance_metadata = True
TrainConfig.batch_size = 512
TrainConfig.max_steps = 60
TrainConfig.save_every = 30
TrainConfig.log_every = 1
TrainConfig.print_every = 20
TrainConfig.lr_schedule = {'type': 'exponential', 'initial_value': 0.001, 'final_value': 0.0001, 'num_steps': 60}
TrainConfig.warp_alpha_schedule = {'type': 'linear', 'initial_value': 0.0, 'final_value': 4.0, 'num_steps': 40}
EvalConfig.num_val_eval = None
EvalConfig.num_train_eval = 1
EvalConfig.num_test_eval = 1
"""


@pytest.fixture(autouse=True)
def _clean_gin():
  from nerfies_b200 import configs
  configs.clear_config()
  yield
  configs.clear_config()


def _gin(tmp_path, extra=''):
  path = tmp_path / 'test.gin'
  path.write_text(GIN + extra)
  return str(path)


def _argv(base, gin, *more):
  return ['--base_folder', str(base), '--data_dir', CAPTURE, '--gin_configs', gin, '--precision', 'fp32', *more]


def _restore(base, step=None):
  from nerfies_b200 import checkpoints
  return checkpoints.restore_checkpoint(str(base / 'checkpoints'), step=step, device='cuda:0')


def _leaves(tree, prefix=''):
  for k, v in sorted(tree.items()):
    if isinstance(v, dict):
      yield from _leaves(v, f'{prefix}{k}/')
    else:
      yield prefix + k, v


def test_train_then_eval_end_to_end(tmp_path):
  from nerfies_b200 import configs, datasets, driver_utils, evaluation, models
  from nerfies_b200 import eval as eval_lib, train as train_lib
  gin, base = _gin(tmp_path), tmp_path / 'exp'
  assert train_lib.main(_argv(base, gin)) == 0
  assert sorted(os.listdir(base / 'checkpoints')) == ['checkpoint_30', 'checkpoint_60']
  assert 'TrainConfig.batch_size = 512' in (base / 'config.gin').read_text()
  records = driver_utils.read_scalars(base / 'summaries' / 'train.jsonl')
  assert [r['step'] for r in records] == list(range(1, 61))
  want = {'step', 'params/learning_rate', 'params/warp_alpha', 'params/time_alpha', 'params/elastic_loss/weight',
          'time/steps_per_sec'} | {f'{k}/{lv}' for k in ('loss/rgb', 'loss/total', 'metric/psnr') for lv in ('coarse', 'fine')}
  for r in records:
    assert set(r) == want and all(np.isfinite(v) for v in r.values()), r
  assert records[0]['params/warp_alpha'] == pytest.approx(0.1) and records[-1]['params/warp_alpha'] == 4.0
  assert records[-1]['params/learning_rate'] == pytest.approx(1e-4)
  total = [r['loss/total/coarse'] + r['loss/total/fine'] for r in records]
  first, last = float(np.mean(total[:10])), float(np.mean(total[-10:]))
  print(f'loss/total (coarse + fine): mean of steps 1-10 {first:.5f}, of steps 51-60 {last:.5f}')
  assert last < first

  assert eval_lib.main(_argv(base, gin, '--eval_once'), poll_seconds=0.0) == 0
  out = base / 'renders' / '00000060'
  assert sorted(os.listdir(out)) == ['test', 'train', 'val']
  assert sorted(os.listdir(out / 'test')) == ['depth_expected_000.png', 'depth_median_000.png', 'rgb_000.png']

  # a second model, built and restored here, renders what the driver saved and scored
  configs.clear_config()
  configs.parse_config_files_and_bindings([gin])
  exp_config, model_config = configs.ExperimentConfig(), configs.ModelConfig(use_stratified_sampling=False)
  source = driver_utils.make_datasource(exp_config, model_config, CAPTURE)
  assert source.val_ids == ['right_009', 'right_001']
  model, _ = models.construct_nerf(1, model_config, 4096, source.appearance_ids, source.camera_ids, source.warp_ids,
                                   near=source.near, far=source.far, precision='fp32')
  state = _restore(base)
  assert state.step == 60 and state.warp_alpha == 4.0
  psnrs = []
  for item_id in source.val_ids:
    item, camera = source.get_item(item_id), source.load_camera(item_id)
    render = evaluation.render_frame(model, state.optimizer.target['model'], camera, state.warp_extra, item['metadata'])
    want_rgb = evaluation.image_to_uint8(render['rgb']).cpu().numpy()
    got_rgb = datasets.decode_image(out / 'val' / f'rgb_{item_id}.png')
    assert got_rgb.shape == tuple(item['rgb'].shape) == (27, 48, 3)
    np.testing.assert_array_equal(got_rgb, want_rgb)
    for stem, key in (('depth_expected', 'depth'), ('depth_median', 'med_depth')):
      got = cv2.imread(str(out / 'val' / f'{stem}_{item_id}.png'), cv2.IMREAD_UNCHANGED)
      assert got.dtype == np.uint16
      np.testing.assert_array_equal(got, evaluation.depth_to_uint16(render[key]).cpu().numpy())
    psnrs.append(float(evaluation.compute_psnr(((render['rgb'] - item['rgb'])**2).mean())))
  scalars = driver_utils.read_scalars(base / 'summaries' / 'eval.jsonl')
  assert [set(r) - {'step'} for r in scalars] == [{f'metrics-eval/{k}/{tag}' for k in ('mse', 'psnr')}
                                                   for tag in ('val', 'train')]       # 27 x 48: no MS-SSIM
  assert scalars[0]['step'] == 60 and scalars[0]['metrics-eval/psnr/val'] == pytest.approx(np.mean(psnrs), rel=1e-6)


def test_resume_is_exact(tmp_path):
  """30 steps, stop, start again to step 60 == 60 uninterrupted steps: step counting, the position of
  the data stream after a resume and the step the schedules see.  The training step sums dW, db and
  the embedding gradients with float atomicAdd, whose order changes from run to run, so two identical
  runs already differ in the last bits and bitwise equality is not available: the resumed run must
  be as close to an uninterrupted run as a second uninterrupted run is (within 10 x their relative
  L2 distance), and its loss follows the uninterrupted run's step by step."""
  from nerfies_b200 import driver_utils, train as train_lib
  gin = _gin(tmp_path, 'ModelConfig.use_stratified_sampling = False\n')
  bases = {k: tmp_path / k for k in ('whole', 'again', 'resumed')}
  for k in ('whole', 'again'):
    assert train_lib.main(_argv(bases[k], gin)) == 0
  assert train_lib.main(_argv(bases['resumed'], gin, '--max_steps', '30')) == 0
  assert os.listdir(bases['resumed'] / 'checkpoints') == ['checkpoint_30']
  at_30 = _restore(bases['resumed'])
  assert train_lib.main(_argv(bases['resumed'], gin)) == 0
  assert sorted(os.listdir(bases['resumed'] / 'checkpoints')) == ['checkpoint_30', 'checkpoint_60']

  logs = {k: driver_utils.read_scalars(b / 'summaries' / 'train.jsonl') for k, b in bases.items()}
  assert [r['step'] for r in logs['resumed']] == list(range(1, 61))              # 1..30, then 31..60 appended
  for a, b in zip(logs['whole'], logs['resumed']):
    for key in ('params/learning_rate', 'params/warp_alpha', 'params/time_alpha'):
      assert a[key] == b[key], (a['step'], key)                                  # the schedules saw the same step
    # the same batch at the same step: a stream replayed from its head would give another loss
    assert b['loss/total/fine'] == pytest.approx(a['loss/total/fine'], rel=1e-2), a['step']
  assert logs['whole'][30]['loss/total/fine'] != pytest.approx(logs['whole'][0]['loss/total/fine'], rel=1e-3)

  final = {k: _restore(b) for k, b in bases.items()}
  assert all(s.step == 60 for s in final.values()) and at_30.step == 30
  trees = lambda s: {**dict(_leaves(s.optimizer.target, 'target/')), **dict(_leaves(s.param_states, 'moments/'))}
  whole, again, resumed = (trees(final[k]) for k in ('whole', 'again', 'resumed'))
  assert set(whole) == set(resumed) and any(k.endswith('grad_sq_ema') for k in whole)
  # single leaves with small entries (biases, the warp heads) drift apart by more than their own size
  # within 60 Adam steps, so the distance is taken over all parameters, and over all moments, at once
  for part in ('target/', 'moments/'):
    names = [n for n in whole if n.startswith(part)]
    flat = lambda t: torch.cat([t[n].reshape(-1).double() for n in names])
    noise = float((flat(whole) - flat(again)).norm() / flat(whole).norm())
    dist = float((flat(whole) - flat(resumed)).norm() / flat(whole).norm())
    print(f'{part} relative L2 distance: two uninterrupted runs {noise:.3e}, resumed vs uninterrupted {dist:.3e}')
    assert dist <= 10 * noise + 1e-6, (part, dist, noise)


def test_regulariser_config_runs(tmp_path):
  from nerfies_b200 import driver_utils, eval as eval_lib, train as train_lib
  gin = _gin(tmp_path, """
ModelConfig.warp_metadata_encoder_type = 'time'
TrainConfig.max_steps = 5
TrainConfig.use_elastic_loss = True
TrainConfig.elastic_loss_weight_schedule = ('constant', 0.001)
TrainConfig.use_background_loss = True
TrainConfig.background_loss_weight = 1.0
TrainConfig.background_points_batch_size = 64
TrainConfig.use_warp_reg_loss = True
TrainConfig.warp_reg_loss_weight = 0.001
TrainConfig.time_alpha_schedule = ('constant', 2.0)
""")
  base = tmp_path / 'exp'
  assert train_lib.main(_argv(base, gin)) == 0
  records = driver_utils.read_scalars(base / 'summaries' / 'train.jsonl')
  assert [r['step'] for r in records] == [1, 2, 3, 4, 5]
  want = {'loss/rgb/coarse', 'loss/rgb/fine', 'loss/total/coarse', 'loss/total/fine', 'metric/psnr/coarse',
          'metric/psnr/fine', 'loss/elastic/coarse', 'residual/elastic/coarse', 'metric/jacobian_det/coarse',
          'metric/jacobian_div/coarse', 'metric/jacobian_curl/coarse', 'loss/warp_reg/coarse', 'loss/warp_reg/fine',
          'residual/warp_reg/coarse', 'residual/warp_reg/fine', 'loss/background'}
  for r in records:
    assert want <= set(r) and all(np.isfinite(v) for v in r.values()), r
    assert r['params/time_alpha'] == 2.0 and r['params/elastic_loss/weight'] == pytest.approx(0.001)
  assert os.listdir(base / 'checkpoints') == ['checkpoint_5']                    # 5 % save_every != 0: saved at the end
  # the 'time' encoder's float metadata reaches the renderer through the eval driver
  assert eval_lib.main(_argv(base, gin, '--eval_once'), poll_seconds=0.0) == 0
  assert len(os.listdir(base / 'renders' / '00000005' / 'val')) == 6


def test_render_frame_takes_the_time_encoders_float_metadata():
  """render_frame passes metadata['time'] as float32: the frame equals model.apply on the frame's
  rays with that timestamp, and differs from the frame at another timestamp."""
  from nerfies_b200 import camera as camera_lib, configs, evaluation, models
  dev = torch.device('cuda', 0)
  cfg = configs.ModelConfig(use_stratified_sampling=False, use_warp=True, warp_field_type='se3',
                            warp_metadata_encoder_type='time', num_coarse_samples=16, num_fine_samples=16)
  model, params = models.construct_nerf(3, cfg, 2048, [], [], range(4), near=0.02, far=0.83, precision='fp32', device=dev)
  # warp heads start at U[0, 1e-4): scale them up so that the timestamp moves the image
  for branch in ('branches_w', 'branches_v'):
    params['warp_field'][branch]['logit']['kernel'] *= 3e3
  cam = camera_lib.Camera(orientation=np.eye(3, dtype=np.float32), position=[0.0, 0.0, -0.4], focal_length=40.0,
                          principal_point=[24.0, 13.5], image_size=[48, 27])
  extra = {'alpha': 4.0, 'time_alpha': 4.0}
  frame = evaluation.render_frame(model, params, cam, extra, {'time': 0.6})
  rays = camera_lib.camera_to_rays(cam, dev)
  flat = {'origins': rays['origins'].reshape(-1, 3), 'directions': rays['directions'].reshape(-1, 3),
          'metadata': {'time': torch.full((27 * 48, 1), 0.6, device=dev)}}
  want = model.apply({'params': params}, flat, warp_extra=extra)['fine']['rgb'].reshape(27, 48, 3)
  assert torch.equal(frame['rgb'], want)
  other = evaluation.render_frame(model, params, cam, extra, {'time': 0.0})
  assert not torch.equal(frame['rgb'], other['rgb'])


def test_frames_large_enough_are_scored_with_ms_ssim():
  from nerfies_b200 import camera as camera_lib, configs, evaluation, models, eval as eval_lib
  dev = torch.device('cuda', 0)
  cfg = configs.ModelConfig(use_stratified_sampling=False, num_coarse_samples=8, num_fine_samples=8)
  model, params = models.construct_nerf(3, cfg, 4096, [], [], [], near=0.02, far=0.83, precision='fp32', device=dev)
  cam = camera_lib.Camera(orientation=np.eye(3, dtype=np.float32), position=[0.0, 0.0, -0.4], focal_length=150.0,
                          principal_point=[88.0, 84.0], image_size=[176, 168])
  target = torch.rand(168, 176, 3, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
  images, metrics = eval_lib.render_and_score(model, params, cam, {'alpha': 0.0, 'time_alpha': 0.0}, {}, target)
  render = evaluation.render_frame(model, params, cam, {'alpha': 0.0, 'time_alpha': 0.0}, {})
  want = evaluation.compute_metrics(render['rgb'], target)
  assert set(metrics) == {'mse', 'psnr', 'ssim'}
  for k in metrics:
    assert torch.equal(metrics[k], want[k]), k
  assert images['rgb'].shape == (168, 176, 3) and images['depth_median'].dtype == torch.uint16


def _two_rank_worker(rank, world, port, tmp, gin):
  os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                    LOCAL_RANK=str(rank))
  sys.path.insert(0, ROOT)
  from nerfies_b200 import configs, driver_utils, train as train_lib
  text = driver_utils.parse_configs([gin], ['TrainConfig.max_steps = 10', 'TrainConfig.save_every = 5'])
  state = train_lib.train(configs.ExperimentConfig(), configs.ModelConfig(), configs.TrainConfig(),
                          os.path.join(tmp, 'exp'), CAPTURE, config_str=text, log=lambda s: None)
  torch.save(state.optimizer.flat.cpu(), os.path.join(tmp, f'flat{rank}.pt'))


def test_two_ranks_end_with_equal_parameters(tmp_path):
  if torch.cuda.device_count() < 2:
    pytest.skip('needs 2 GPUs')
  port = 29700 + os.getpid() % 1500
  mp.spawn(_two_rank_worker, args=(2, port, str(tmp_path), _gin(tmp_path)), nprocs=2, join=True)
  flat = [torch.load(tmp_path / f'flat{r}.pt') for r in range(2)]
  assert torch.equal(flat[0], flat[1])
  assert sorted(os.listdir(tmp_path / 'exp' / 'checkpoints')) == ['checkpoint_10', 'checkpoint_5']
  assert len(os.listdir(tmp_path / 'exp' / 'summaries')) == 1                    # rank 0's train.jsonl only
