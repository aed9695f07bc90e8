"""nfb_gather_rays through nerfies_b200.datasets on the GPU, against batches recorded from the
reference's own preloaded iterator (tests/golden/datasource_small.npz, oracle/make_golden_data.py)
and against the per-item composition of camera.camera_to_rays and load_rgb."""
import ctypes
import json
import os
import shutil

import numpy as np
import pytest
import torch

from nerfies_b200 import _lib
from nerfies_b200 import camera as camera_lib
from nerfies_b200 import datasets
from nerfies_b200 import schedules

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
CAPTURE = os.path.join(GOLDEN, 'capture_small')
TOL = 2e-6      # tests/test_camera.py: directions against the reference's float32 numpy
CONFIGS = {
    'A': (dict(use_appearance_id=True, use_camera_id=True, use_warp_id=True, use_time=True, random_seed=12345),
          1000, 7, 16, 5),
    'B': (dict(use_warp_id=True, random_seed=777, train_stride=2), 700, 5, 24, 4),
}


@pytest.fixture(scope='module')
def ref():
  return np.load(os.path.join(GOLDEN, 'datasource_small.npz'))


def make(kwargs, data_dir=CAPTURE):
  return datasets.from_config({'type': 'nerfies', 'data_dir': data_dir}, image_scale=2, device=DEV, **kwargs)


def frame_rays(ds, ids):
  """camera_to_rays + load_rgb of each item, flattened and concatenated in item order."""
  cat = lambda key: torch.cat([r[key].reshape(-1, r[key].shape[-1]) for r in rays])
  rays = [dict(camera_lib.camera_to_rays(ds.load_camera(i), DEV), rgb=ds.load_rgb(i)) for i in ids]
  return {k: cat(k) for k in ('origins', 'directions', 'pixels', 'rgb')}


@pytest.mark.parametrize('name', sorted(CONFIGS))
def test_training_batches_match_reference(ref, name):
  kwargs, B, steps, pb, psteps = CONFIGS[name]
  ds = make(kwargs)
  it = ds.create_iterator(ds.train_ids, batch_size=B, flatten=True, shuffle=True)
  num_rays = 27 * 48 * len(ds.train_ids)
  assert num_rays % B and steps * B > num_rays          # the run crosses the epoch boundary
  order = np.random.RandomState(kwargs['random_seed']).permutation(num_rays)
  frames = frame_rays(ds, ds.train_ids)
  for s in range(steps):
    got = next(it)
    p = f'{name}/batch/{s}/'
    for k in ('rgb', 'origins', 'pixels'):
      assert torch.equal(got[k].cpu(), torch.from_numpy(ref[p + k])), (s, k)
    d = got['directions'].cpu().numpy()
    assert np.abs(d - ref[p + 'directions']).max() <= TOL, s
    idx = torch.from_numpy(order[(s * B + np.arange(B)) % num_rays]).to(DEV)
    for k in ('directions', 'rgb', 'pixels', 'origins'):
      assert torch.equal(got[k], frames[k][idx]), (s, k)
    keys = [k[len(p + 'metadata/'):] for k in ref.files if k.startswith(p + 'metadata/')]
    assert sorted(got['metadata']) == sorted(keys)
    for k in keys:
      want = ref[p + 'metadata/' + k]
      want = want.astype(np.float32) if k == 'time' else want.astype(np.int32)
      assert got['metadata'][k].shape == (B, 1)
      assert np.array_equal(got['metadata'][k].cpu().numpy(), want), (s, k)
  points = ds.load_points(shuffle=True)
  assert torch.equal(points.cpu(), torch.from_numpy(ref[f'{name}/points']))
  pit = datasets.iterator_from_dataset(points, batch_size=pb)
  for s in range(psteps):
    assert torch.equal(next(pit).cpu(), torch.from_numpy(ref[f'{name}/points_batch/{s}'])), s


@pytest.mark.parametrize('name', sorted(CONFIGS))
def test_eval_items_match_reference(ref, name):
  ds = make(CONFIGS[name][0])
  it = ds.create_iterator(ds.val_ids, batch_size=0)
  for item in ds.val_ids:
    got = next(it)
    p = f'{name}/val/{item}/'
    for k in ('rgb', 'origins', 'pixels'):
      assert torch.equal(got[k].cpu(), torch.from_numpy(ref[p + k])), (item, k)
    assert np.abs(got['directions'].cpu().numpy() - ref[p + 'directions']).max() <= TOL
    for k, v in got['metadata'].items():
      want = ref[p + 'metadata/' + k]
      assert np.array_equal(v.cpu().numpy(), want.astype(v.cpu().numpy().dtype)), (item, k)
  assert torch.equal(next(it)['rgb'], ds.load_rgb(ds.val_ids[0]))    # repeat=True starts over


@pytest.mark.parametrize('world_size', [2, 3])
def test_rank_slices_concatenate_to_the_batch(world_size):
  kwargs, B = dict(CONFIGS['A'][0]), 1002
  whole = make(kwargs).create_iterator(['left_000', 'left_003', 'left_007'], batch_size=B, flatten=True,
                                       shuffle=True, rank=0, world_size=1)
  ranks = [make(kwargs).create_iterator(['left_000', 'left_003', 'left_007'], batch_size=B, flatten=True,
                                        shuffle=True, rank=r, world_size=world_size) for r in range(world_size)]
  pts = make(kwargs).load_points()
  pwhole = datasets.iterator_from_dataset(pts, batch_size=36, rank=0, world_size=1)
  pranks = [datasets.iterator_from_dataset(pts, batch_size=36, rank=r, world_size=world_size)
            for r in range(world_size)]
  for _ in range(5):                      # 3 * 1296 rays: the 4th batch wraps
    w = next(whole)
    parts = [next(r) for r in ranks]
    for k in ('origins', 'directions', 'pixels', 'rgb'):
      assert torch.equal(torch.cat([p[k] for p in parts]), w[k]), k
    for k in w['metadata']:
      assert torch.equal(torch.cat([p['metadata'][k] for p in parts]), w['metadata'][k]), k
    assert torch.equal(torch.cat([next(r) for r in pranks]), next(pwhole))


def test_mixed_image_sizes_in_a_writable_copy(tmp_path):
  import cv2
  data = tmp_path / 'capture'
  # contents only: the checkout may be read-only, and copytree's default (copy2) would carry its
  # file modes into the copy that this test rewrites
  shutil.copytree(CAPTURE, data, copy_function=shutil.copyfile)
  for d, _, _ in os.walk(data):
    os.chmod(d, 0o755)
  with open(data / 'camera' / 'left_003.json') as f:
    cam = json.load(f)
  cam['image_size'] = [80, 62]
  cam['principal_point'] = [41.0, 30.5]
  with open(data / 'camera' / 'left_003.json', 'w') as f:
    json.dump(cam, f)
  rng = np.random.RandomState(3)
  cv2.imwrite(str(data / 'rgb' / '2x' / 'left_003.png'), rng.randint(0, 256, (31, 40, 3)).astype(np.uint8))
  ds = make(dict(use_warp_id=True, use_appearance_id=True, random_seed=5), data_dir=data)
  ids = ['left_000', 'left_003', 'right_004']
  frames = frame_rays(ds, ids)
  n = frames['rgb'].shape[0]
  assert n == 27 * 48 * 2 + 31 * 40
  it = ds.create_iterator(ids, batch_size=512, flatten=True, shuffle=False)
  for s in range(8):
    got = next(it)
    idx = torch.from_numpy((s * 512 + np.arange(512)) % n).to(DEV)
    for k in frames:
      assert torch.equal(got[k], frames[k][idx]), (s, k)
  items = ds.create_iterator(ids, batch_size=0, repeat=False)
  for i, x in zip(ids, items):
    r = camera_lib.camera_to_rays(ds.load_camera(i), DEV)
    assert torch.equal(x['rgb'], ds.load_rgb(i))
    for k in r:
      assert torch.equal(x[k], r[k]), (i, k)


def test_next_does_not_synchronise():
  ds = make(CONFIGS['A'][0])
  it = ds.create_iterator(ds.train_ids, batch_size=4096, flatten=True, shuffle=True)
  pit = datasets.iterator_from_dataset(ds.load_points(shuffle=True), batch_size=32)
  next(it), next(pit)
  torch.cuda.synchronize()
  torch.cuda.set_sync_debug_mode('error')
  try:
    for _ in range(4):
      batch = next(it)
      batch['background_points'] = next(pit)
  finally:
    torch.cuda.set_sync_debug_mode(0)
  torch.cuda.synchronize()
  assert batch['rgb'].shape == (4096, 3)


def test_abi_errors_without_a_launch():
  lib = _lib.load()
  torch.cuda.synchronize()
  out = torch.empty(16, 3, device=DEV)
  cam = camera_lib.Camera.from_json(os.path.join(CAPTURE, 'camera', 'left_000.json')).scale(0.5)
  cams = torch.frombuffer(bytearray(bytes(cam._struct())), dtype=torch.uint8).to(DEV)
  offs = torch.tensor([0, 27 * 48], dtype=torch.int64, device=DEV)
  t = _lib.NfbRayTable(num_images=1, cameras=cams.data_ptr(), pixel_offsets=offs.data_ptr(), num_rays=27 * 48)
  stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
  p = ctypes.c_void_p(out.data_ptr())
  none = [None] * 6

  def call(table, first, count, rgb=None):
    return lib.nfb_gather_rays(table, first, count, None, p, None, rgb, *none[:4], stream)

  assert call(None, 0, 4) != 0 and b'null' in lib.nfb_last_error()
  empty = _lib.NfbRayTable.from_buffer_copy(t)
  empty.num_rays = 0
  assert call(ctypes.byref(empty), 0, 4) != 0 and b'rays' in lib.nfb_last_error()
  assert call(ctypes.byref(t), 0, -1) != 0 and b'negative' in lib.nfb_last_error()
  assert call(ctypes.byref(t), 0, 4, rgb=p) != 0 and b'rgb' in lib.nfb_last_error()
  assert call(ctypes.byref(t), 0, 16) == 0
  torch.cuda.synchronize()
  assert torch.equal(out, camera_lib.camera_to_rays(cam, DEV, 0, 16)['directions'])


def test_train_step_fed_by_the_iterator(ref):
  import nerfies_b200 as nb
  from nerfies_b200 import configs, training
  ds = make(CONFIGS['A'][0])
  tc = configs.TrainConfig(batch_size=1000, use_background_loss=True, background_loss_weight=1.0)
  it = ds.create_iterator(ds.train_ids, batch_size=tc.batch_size, flatten=True, shuffle=True)
  points_iter = datasets.iterator_from_dataset(ds.load_points(shuffle=True), batch_size=16)
  lr, warp_alpha = schedules.from_config(tc.lr_schedule), schedules.from_config(tc.warp_alpha_schedule)
  cfg = configs.ModelConfig(num_coarse_samples=16, num_fine_samples=16, nerf_trunk_depth=4, nerf_trunk_width=64,
                            nerf_skips=(2,), nerf_rgb_branch_width=32, num_nerf_point_freqs=6,
                            use_appearance_metadata=True, use_warp=True, warp_field_type='se3')
  model, params = nb.construct_nerf(0, cfg, tc.batch_size, ds.appearance_ids, ds.camera_ids, ds.warp_ids,
                                    ds.near, ds.far, device=DEV, precision='fp32')
  clone = lambda t: {k: clone(v) for k, v in t.items()} if isinstance(t, dict) else torch.as_tensor(t).clone()

  def step(state, s, batch):
    state.warp_alpha = warp_alpha(s)
    sp = training.ScalarParams(learning_rate=lr(s), background_loss_weight=tc.background_loss_weight)
    return training.train_step(model, s, state, batch, sp, use_background_loss=True)

  state = training.create_train_state(model, clone(params))
  firsts = None
  for s in range(1, 4):
    batch = next(it)
    batch['background_points'] = next(points_iter)
    state, stats, _ = step(state, s, batch)
    vals = {lv: float(stats[lv]['loss/total']) for lv in ('coarse', 'fine')}
    assert all(np.isfinite(v) for v in vals.values()) and np.isfinite(float(stats['background_loss']))
    firsts = firsts or vals
  p = 'A/batch/0/'
  batch = {k: torch.from_numpy(ref[p + k]).to(DEV) for k in ('origins', 'directions', 'pixels', 'rgb')}
  batch['metadata'] = {k: torch.from_numpy(ref[p + 'metadata/' + k].astype(np.int32)).to(DEV)
                       for k in ('appearance', 'warp')}
  batch['background_points'] = torch.from_numpy(ref['A/points_batch/0']).to(DEV)
  _, stats, _ = step(training.create_train_state(model, clone(params)), 1, batch)
  for lv, v in firsts.items():
    assert abs(float(stats[lv]['loss/total']) - v) <= 1e-4 * abs(v), lv
