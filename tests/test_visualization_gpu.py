"""nfb_colorize against the reference's recorded outputs (tests/golden/viz_turbo.npz) and the numpy
statement of colorize (tests/viz_oracle.py): exact equality for every source, given and frame
bounds, invert, special values, odd shapes and unaligned column offsets; determinism and CUDA-graph
capture; the video frame; and the video and eval drivers end to end on the small capture."""
import os

import numpy as np
import pytest
import torch

from tests import viz_oracle

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'viz_turbo.npz')
CAPTURE = os.path.join(ROOT, 'tests', 'golden', 'capture_small')
DEV = torch.device('cuda', 0)


@pytest.fixture(scope='module')
def golden():
  return dict(np.load(GOLDEN))


def _d(a):
  return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def test_kernel_equals_the_reference(golden):
  from nerfies_b200 import visualization as viz
  g, table = golden, golden['table']
  near, far = float(g['near']), float(g['far'])
  cases = [('depth_viz', g['depth'], dict(cmin=near, cmax=far, invert=True)),
           ('disp_viz', g['depth'], dict(source='reciprocal')),
           ('disp_positive_viz', g['positive_depth'], dict(source='reciprocal')),
           ('acc_viz', g['acc'], dict(cmin=0.0, cmax=1.0)),
           ('abs_error_viz', g['target'], dict(cmin=0, cmax=1, source='abs_error', target=_d(g['rgb']))),
           ('sq_error_viz', g['target'], dict(cmin=0, cmax=1, source='sq_error', target=_d(g['rgb']))),
           ('unit_frame_inv0', g['unit'], {}), ('flat_frame_inv0', g['flat'], {})]
  for inv in (0, 1):
    cases += [(f'unit_given_inv{inv}', g['unit'], dict(cmin=0.0, cmax=1.0, invert=bool(inv))),
              (f'unit_int_inv{inv}', g['unit'], dict(cmin=0, cmax=1, invert=bool(inv))),
              (f'finite_frame_inv{inv}', g['finite'], dict(invert=bool(inv))),
              (f'finite_min_inv{inv}', g['finite'], dict(cmax=0.75, invert=bool(inv)))]
  for key, values, kw in cases:
    np.testing.assert_array_equal(viz.colorize(_d(values), cmap=table, **kw).cpu().numpy(), g[key], err_msg=key)
    np.testing.assert_array_equal(viz.colorize_uint8(_d(values), cmap=table, **kw).cpu().numpy(), g[key + '_u8'],
                                  err_msg=key)
  frame = viz.video_frame(_d(g['video_rgb']), _d(g['depth']), near, far, cmap=table)
  np.testing.assert_array_equal(frame.cpu().numpy(), g['video_frame'])


def _values(shape, seed, source):
  """Random values with the special ones spread in: values of x around [0, 1] for 'value'; depths
  (with zeros) for 'reciprocal'; (h, w, 3) images for the error sources."""
  rng = np.random.RandomState(seed)
  if source in ('abs_error', 'sq_error'):
    a = rng.uniform(-0.2, 1.2, shape + (3,)).astype(np.float32)
    b = rng.uniform(0, 1, shape + (3,)).astype(np.float32)
    b.reshape(-1)[:7] = a.reshape(-1)[:7]
    return a, b
  x = rng.uniform(-0.1, 1.1, shape).astype(np.float32)
  edges = (rng.randint(0, 256, x.size // 3) / 255.0).astype(np.float32)
  x.reshape(-1)[:len(edges)] = np.nextafter(edges, np.float32(rng.choice([-1, 2])))
  special = np.array([0, -0.0, 1, np.inf, -np.inf, np.nan, 1 + 2**-23, -2**-24], np.float32)
  flat = x.reshape(-1)
  picks = rng.choice(flat.size, min(flat.size, 16), replace=False)
  flat[picks] = special[np.arange(len(picks)) % len(special)]
  rng.shuffle(flat)
  if source == 'reciprocal':
    x = np.abs(x) * 3
    x.reshape(-1)[picks[:2]] = 0.0
  return x, None


SHAPES = [(1, 1), (27, 48), (5, 37), (13, 101), (1080, 1920)]


@pytest.mark.parametrize('source', ['value', 'reciprocal', 'abs_error', 'sq_error'])
@pytest.mark.parametrize('shape', SHAPES)
def test_every_source_equals_the_oracle(source, shape):
  from nerfies_b200 import visualization as viz
  a, b = _values(shape, sum(shape) + len(source), source)
  table = np.random.RandomState(3).uniform(0, 1, (256, 3))
  fa = np.where(np.isfinite(a), a, np.float32(0.5)) if b is None else a          # frame bounds without NaN
  target = None if b is None else _d(b)
  for bounds in ((0.0, 1.0), (0, 1), (0.25, 0.7), (None, None), (0.1, None), (None, 0.9)):
    for invert in (False, True):
      for arr in (a, fa):
        want = viz_oracle.colorize(viz_oracle.source_values(arr, source, b), table, *bounds, invert=invert)
        got = viz.colorize_uint8(_d(arr), *bounds, cmap=table, invert=invert, source=source, target=target)
        np.testing.assert_array_equal(got.cpu().numpy(), viz_oracle.to_uint8(want), err_msg=f'{bounds} {invert}')
        if shape != (1080, 1920):
          got64 = viz.colorize(_d(arr), *bounds, cmap=table, invert=invert, source=source, target=target)
          np.testing.assert_array_equal(got64.cpu().numpy(), want, err_msg=f'{bounds} {invert}')


@pytest.mark.parametrize('shape', [(1, 1), (27, 48), (7, 33), (1080, 1920)])
@pytest.mark.parametrize('column', [0, 1, 5, 16])
def test_uint8_into_a_column_range(shape, column):
  """Rows of any pitch and column offsets that break 16-byte alignment; bytes around the window
  stay untouched."""
  from nerfies_b200 import visualization as viz
  a, _ = _values(shape, 7, 'value')
  a = np.where(np.isnan(a), np.float32(0.5), a)                                  # a frame min, not NaN
  h, w = shape
  canvas = torch.full((h, w + column + 3, 3), 77, dtype=torch.uint8, device=DEV)
  viz.colorize_uint8(_d(a), None, 0.8, cmap='turbo', invert=True, out=canvas[:, column:column + w])
  want = viz_oracle.to_uint8(viz_oracle.colorize(a, viz.get_colormap('turbo'), None, 0.8, invert=True))
  got = canvas.cpu().numpy()
  np.testing.assert_array_equal(got[:, column:column + w], want)
  assert (got[:, :column] == 77).all() and (got[:, column + w:] == 77).all()


def test_repeatable_and_capturable_in_a_cuda_graph():
  from nerfies_b200 import visualization as viz
  a, _ = _values((270, 480), 5, 'reciprocal')
  x = _d(a)
  first = viz.colorize_uint8(x, source='reciprocal', cmap='magma')
  assert torch.equal(first, viz.colorize_uint8(x, source='reciprocal', cmap='magma'))
  out = torch.empty_like(first)
  stream = torch.cuda.Stream()
  stream.wait_stream(torch.cuda.current_stream())
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.stream(stream):
    viz.colorize_uint8(x, source='reciprocal', cmap='magma', out=out)           # warm-up outside the capture
    with torch.cuda.graph(graph, stream=stream):
      viz.colorize_uint8(x, source='reciprocal', cmap='magma', out=out)
  torch.cuda.current_stream().wait_stream(stream)
  out.zero_()
  x.mul_(2)                                                                      # the graph reads the new values
  graph.replay()
  torch.cuda.synchronize()
  assert torch.equal(out, viz.colorize_uint8(x, source='reciprocal', cmap='magma'))


@pytest.mark.parametrize('shape', [(1, 1), (27, 48), (9, 31), (1080, 1920)])
def test_video_frame_equals_the_notebook(shape):
  from nerfies_b200 import evaluation, visualization as viz
  rng = np.random.RandomState(shape[1])
  rgb = rng.uniform(-0.05, 1.05, shape + (3,)).astype(np.float32)
  edges = (np.arange(256) / 255.0).astype(np.float32)
  ends = np.concatenate([edges, np.nextafter(edges, np.float32(0)), np.nextafter(edges, np.float32(1)),
                         np.float32([np.nan, np.inf, -np.inf])])
  rgb.reshape(-1)[:min(rgb.size, len(ends))] = ends[:rgb.size]
  depth = rng.uniform(0.0, 3.0, shape).astype(np.float32)
  table = viz.get_colormap('magma')
  frame = viz.video_frame(_d(rgb), _d(depth), 0.1, 2.5)
  np.testing.assert_array_equal(frame.cpu().numpy(), viz_oracle.video_frame(rgb, depth, table, 0.1, 2.5))
  # the float32 product of nfb_image_quantize gives the same rgb half
  np.testing.assert_array_equal(frame[:, :shape[1]].cpu().numpy(), evaluation.image_to_uint8(_d(rgb)).cpu().numpy())


def test_bad_arguments_are_refused():
  from nerfies_b200 import visualization as viz
  x = torch.zeros(4, 6, device=DEV)
  with pytest.raises(ValueError, match='source'):
    viz.colorize(x, source='log')
  with pytest.raises(ValueError, match='float32'):
    viz.colorize(x.double())
  with pytest.raises(ValueError, match='empty'):
    viz.colorize(x[:0])
  with pytest.raises(ValueError, match='out must be'):
    viz.colorize_uint8(x, 0, 1, out=torch.empty(4, 6, 4, dtype=torch.uint8, device=DEV)[..., :3])
  with pytest.raises(ValueError, match='error maps'):
    viz.colorize(torch.zeros(4, 6, 3, device=DEV), 0, 1, source='abs_error', target=torch.zeros(4, 5, 3, device=DEV))
  assert viz.colorize(x[:0], 0.0, 1.0).shape == (0, 6, 3)


# ---- the drivers end to end on the small capture ---------------------------------------------------
GIN = """
ExperimentConfig.image_scale = 2
ModelConfig.num_coarse_samples = 16
ModelConfig.num_fine_samples = 16
ModelConfig.use_warp = True
ModelConfig.warp_field_type = 'se3'
ModelConfig.use_appearance_metadata = True
TrainConfig.batch_size = 256
TrainConfig.max_steps = 4
TrainConfig.save_every = 4
EvalConfig.num_val_eval = None
EvalConfig.num_train_eval = 1
EvalConfig.num_test_eval = 1
"""


@pytest.fixture(scope='module')
def trained(tmp_path_factory):
  from nerfies_b200 import configs, train as train_lib
  tmp = tmp_path_factory.mktemp('viz_drivers')
  gin = tmp / 'test.gin'
  gin.write_text(GIN)
  base = tmp / 'exp'
  configs.clear_config()
  assert train_lib.main(['--base_folder', str(base), '--data_dir', CAPTURE, '--gin_configs', str(gin),
                         '--precision', 'fp32']) == 0
  yield base, str(gin)
  configs.clear_config()


def _model_and_state(base, gin):
  from nerfies_b200 import checkpoints, configs, driver_utils, models
  configs.clear_config()
  configs.parse_config_files_and_bindings([gin])
  model_config = configs.ModelConfig(use_stratified_sampling=False)
  source = driver_utils.make_datasource(configs.ExperimentConfig(), model_config, CAPTURE)
  model, _ = models.construct_nerf(1, model_config, 4096, source.appearance_ids, source.camera_ids, source.warp_ids,
                                   near=source.near, far=source.far, precision='fp32')
  state = checkpoints.restore_checkpoint(str(base / 'checkpoints'), device='cuda:0')
  return source, model, state


def test_render_video_end_to_end(trained):
  import cv2
  from nerfies_b200 import datasets, evaluation, render_video, visualization
  base, gin = trained
  assert render_video.main(['--base_folder', str(base), '--data_dir', CAPTURE, '--gin_configs', gin,
                            '--precision', 'fp32', '--camera_path', 'camera-paths/orbit-extreme']) == 0
  out = base / 'videos' / 'orbit-extreme' / '00000004'
  assert sorted(os.listdir(out)) == ['frame_00000.png', 'frame_00001.png', 'frame_00002.png', 'video.mp4']
  source, model, state = _model_and_state(base, gin)
  table = visualization.get_colormap('magma')
  paths = source.glob_cameras(os.path.join(CAPTURE, 'camera-paths', 'orbit-extreme'))
  for i, path in enumerate(paths):
    got = datasets.decode_image(out / f'frame_{i:05d}.png')
    assert got.shape == (27, 96, 3)
    render = evaluation.render_frame(model, state.optimizer.target['model'], source.load_camera(path),
                                     state.warp_extra, {'appearance': 0, 'warp': 0})
    want = viz_oracle.video_frame(render['rgb'].cpu().numpy(), render['med_depth'].cpu().numpy(), table,
                                  source.near, source.far)
    np.testing.assert_array_equal(got, want)
  video = cv2.VideoCapture(str(out / 'video.mp4'))
  frames = []
  while True:
    ok, frame = video.read()
    if not ok:
      break
    frames.append(frame)
  assert len(frames) == 3 and all(f.shape == (28, 96, 3) for f in frames)     # 27 rows + the repeated last one


def test_eval_save_viz_end_to_end(trained):
  from nerfies_b200 import datasets, evaluation, eval as eval_lib, visualization as viz
  base, gin = trained
  assert eval_lib.main(['--base_folder', str(base), '--data_dir', CAPTURE, '--gin_configs', gin, '--precision',
                        'fp32', '--eval_once', '--save_viz'], poll_seconds=0.0) == 0
  out = base / 'renders' / '00000004'
  stems = ['rgb', 'depth_expected', 'depth_median', 'depth_expected_viz', 'depth_median_viz',
           'disparity_expected_viz', 'disparity_median_viz', 'acc_viz']
  assert sorted(os.listdir(out / 'test')) == sorted(f'{s}_000.png' for s in stems)
  source, model, state = _model_and_state(base, gin)
  table = viz.get_colormap('magma')
  for item_id in source.val_ids:
    assert sorted(os.listdir(out / 'val')) == sorted(f'{s}_{i}.png' for i in source.val_ids
                                                     for s in stems + ['rgb_abs_error_viz', 'rgb_sq_error_viz'])
    item = source.get_item(item_id)
    render = evaluation.render_frame(model, state.optimizer.target['model'], source.load_camera(item_id),
                                     state.warp_extra, item['metadata'])
    r = {k: v.cpu().numpy() for k, v in render.items()}
    target = item['rgb'].cpu().numpy()
    want = {'depth_expected_viz': viz_oracle.colorize(r['depth'], table, source.near, source.far, invert=True),
            'depth_median_viz': viz_oracle.colorize(r['med_depth'], table, source.near, source.far, invert=True),
            'disparity_expected_viz': viz_oracle.colorize(viz_oracle.source_values(r['depth'], 'reciprocal'), table),
            'disparity_median_viz': viz_oracle.colorize(viz_oracle.source_values(r['med_depth'], 'reciprocal'),
                                                        table),
            'acc_viz': viz_oracle.colorize(r['acc'], table, 0.0, 1.0),
            'rgb_abs_error_viz': viz_oracle.colorize(viz_oracle.source_values(target, 'abs_error', r['rgb']),
                                                     table, 0, 1),
            'rgb_sq_error_viz': viz_oracle.colorize(viz_oracle.source_values(target, 'sq_error', r['rgb']),
                                                    table, 0, 1)}
    for stem, image in want.items():
      np.testing.assert_array_equal(datasets.decode_image(out / 'val' / f'{stem}_{item_id}.png'),
                                    viz_oracle.to_uint8(image), err_msg=stem)
