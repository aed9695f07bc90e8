"""CPU side of nerfies_b200.datasets / schedules against fixtures recorded from the reference's
own nerfies/datasets and nerfies/schedules.py (oracle/make_golden_data.py): ids, metadata,
cameras, image decoding, the rng draw order, schedules and the error cases."""
import json
import os
import shutil

import numpy as np
import pytest
import torch

from nerfies_b200 import datasets
from nerfies_b200 import schedules

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
CAPTURE = os.path.join(GOLDEN, 'capture_small')
CONFIGS = {
    'A': dict(use_appearance_id=True, use_camera_id=True, use_warp_id=True, use_time=True, random_seed=12345),
    'B': dict(use_warp_id=True, random_seed=777, train_stride=2),
}


@pytest.fixture(scope='module')
def ref():
  return np.load(os.path.join(GOLDEN, 'datasource_small.npz'))


def make(name, data_dir=CAPTURE, **kw):
  return datasets.from_config({'type': 'nerfies', 'data_dir': data_dir}, image_scale=2, device='cpu',
                              **{**CONFIGS[name], **kw})


@pytest.mark.parametrize('name', sorted(CONFIGS))
def test_ids_and_scene(ref, name):
  ds = make(name)
  for key in ('train_ids', 'val_ids', 'all_ids'):
    assert list(getattr(ds, key)) == ref[f'{name}/{key}'].tolist(), key
  for key in ('appearance_ids', 'camera_ids', 'warp_ids', 'time_ids'):
    assert getattr(ds, key) == tuple(ref[f'{name}/{key}'].tolist()), key
  assert [ds.near, ds.far] == ref[f'{name}/near_far'].tolist()
  assert ds.has_metadata


@pytest.mark.parametrize('name', sorted(CONFIGS))
def test_cameras_scaled_and_centred(ref, name):
  ds = make(name)
  for item in ds.train_ids:
    got = ds.load_camera(item).get_parameters()
    for k, v in got.items():
      want = ref[f'{name}/camera/{item}/{k}']
      if k == 'position':          # float64 in the reference until camera_to_rays rebuilds the Camera
        want = want.astype(np.float32)
      assert v.dtype == want.dtype and np.array_equal(v, want), (item, k)


def test_item_metadata_and_time(ref):
  ds = make('A')
  batch = {k: ref[f'A/batch/0/metadata/{k}'] for k in ('appearance', 'camera', 'warp', 'time')}
  # every (appearance, camera, warp, time) tuple of a batch is one of the train items'
  items = {tuple(ds._item_metadata(i)[k] for k in ('appearance', 'camera', 'warp', 'time'))
           for i in ds.train_ids}
  rows = set(zip(*[batch[k][:, 0].tolist() for k in ('appearance', 'camera', 'warp', 'time')]))
  assert rows <= items and len(rows) == len(items)
  # the item without a time_id falls back to its warp id: 21 / max(train time ids) * 2 - 1
  assert ds.get_time('right_009') == ref['A/val/right_009/metadata/time'][0, 0, 0]
  table = ds.ray_table(ds.train_ids)
  assert table.metadata['time'].dtype == np.float32
  assert np.array_equal(table.metadata['time'],
                        np.array([ds.get_time(i) for i in ds.train_ids]).astype(np.float32))


def test_decode_matches_reference_rgb(ref):
  for key in ref.files:
    if key.startswith('rgb/'):
      img = datasets.decode_image(os.path.join(CAPTURE, 'rgb', '2x', key[4:] + '.png'))
      assert img.dtype == np.uint8
      got = img.astype(np.float32) / np.float32(255.0)
      assert np.array_equal(got, ref[key]), key


def test_pil_fallback_same_bytes(monkeypatch):
  path = os.path.join(CAPTURE, 'rgb', '2x', 'left_000.png')
  a = datasets.decode_image(path)
  monkeypatch.setattr(datasets, 'cv2', None)
  assert np.array_equal(datasets.decode_image(path), a)


@pytest.mark.parametrize('name', sorted(CONFIGS))
def test_rng_draw_order(ref, name, monkeypatch):
  """create_iterator draws permutation(num_rays) (used only with shuffle), then load_points draws
  permutation(len(points)), then the val iterator draws again: the reference's order."""
  uploads = []
  monkeypatch.setattr(datasets, '_upload', lambda host, device, order: uploads.append((host, order)))
  ds = make(name)
  ds.create_iterator(ds.train_ids, flatten=True, shuffle=True, batch_size=8)
  points = ds.load_points(shuffle=True)
  assert np.array_equal(points.numpy(), ref[f'{name}/points'])
  ds.create_iterator(ds.val_ids, batch_size=0)             # unshuffled: still draws
  assert np.array_equal(ds.rng.randint(0, 2**31 - 1, size=4), ref[f'{name}/rng_after'])
  (train, order), (val, val_order) = uploads
  assert val_order is None
  expect = np.random.RandomState(CONFIGS[name]['random_seed']).permutation(train.num_rays)
  assert np.array_equal(order, expect)
  assert train.num_rays == 27 * 48 * len(ds.train_ids)
  assert list(train.offsets) == [27 * 48 * k for k in range(len(ds.train_ids) + 1)]


def test_batch_rays_are_table_rays(ref):
  """The fixture's first batch, traced back through the drawn order to the host table: rgb
  bitwise equal to u8 / 255 of the ray's pixel and the pixel centre of its row-major index."""
  ds = make('A')
  host = ds.ray_table(ds.train_ids)
  order = np.random.RandomState(12345).permutation(host.num_rays)[:1000]
  k = np.searchsorted(host.offsets, order, side='right') - 1
  p = order - host.offsets[k]
  rgb = np.stack([host.images[kk].reshape(-1, 3)[pp] for kk, pp in zip(k, p)]).astype(np.float32) / np.float32(255)
  assert np.array_equal(rgb, ref['A/batch/0/rgb'])
  pixels = np.stack([p % 48 + 0.5, p // 48 + 0.5], -1).astype(np.float32)
  assert np.array_equal(pixels, ref['A/batch/0/pixels'])


def test_schedules_match_reference():
  z = np.load(os.path.join(GOLDEN, 'schedules.npz'))
  steps = [int(s) for s in z['steps']]
  names = [k[len('value/'):] for k in z.files if k.startswith('value/')]
  assert len(names) == 9
  for name in names:
    sched = schedules.from_config(json.loads(str(z['spec/' + name])))
    got = np.array([sched(s) for s in steps])
    want = z['value/' + name]
    np.testing.assert_allclose(got, want, rtol=1e-6, atol=0, err_msg=name)
    assert all(float(np.float32(v)) == v for v in got), name


def test_schedules_accept_train_config():
  from nerfies_b200 import configs
  tc = configs.TrainConfig(batch_size=1024)
  for spec in (tc.lr_schedule, tc.warp_alpha_schedule, tc.time_alpha_schedule, tc.elastic_loss_weight_schedule):
    assert isinstance(schedules.from_config(spec)(0), float)
  assert schedules.from_config(tc.warp_alpha_schedule)(40000) == 4.0
  with pytest.raises(ValueError):
    schedules.from_config(('nope', 1))
  with pytest.raises(ValueError):
    schedules.from_config(3.0)


def test_errors(tmp_path):
  with pytest.raises(NotImplementedError, match='lazy'):
    make('A', preload=False).create_iterator(['left_000'], batch_size=8, flatten=True)
  with pytest.raises(NotImplementedError):
    make('A').create_iterator(['left_000'], batch_size=8, shuffle=True)
  with pytest.raises(ValueError, match='divisible'):
    make('A').create_iterator(['left_000'], batch_size=10, flatten=True, rank=0, world_size=3)
  with pytest.raises(NotImplementedError):
    make('A').get_item('left_000', scale_factor=0.5)
  # a missing image
  broken = tmp_path / 'capture'
  shutil.copytree(CAPTURE, broken)
  os.remove(broken / 'rgb' / '2x' / 'left_000.png')
  with pytest.raises(FileNotFoundError):
    make('A', data_dir=broken).ray_table(['left_000'])
  # an image whose shape differs from its scaled camera's
  import cv2
  cv2.imwrite(str(broken / 'rgb' / '2x' / 'left_000.png'), np.zeros((27, 47, 3), np.uint8))
  with pytest.raises(ValueError, match="left_000"):
    make('A', data_dir=broken).ray_table(['left_003', 'left_000'])
  with pytest.raises(ValueError, match='Unknown datasource'):
    datasets.from_config({'type': 'blender', 'data_dir': CAPTURE}, image_scale=2)


def test_test_cameras():
  ds = make('A')
  cams = ds.load_test_cameras()
  assert len(cams) == 3 and cams[0].image_shape == (27, 48)
  assert len(ds.load_test_cameras(count=1)) == 1
  assert len(ds.create_cameras_dataset(cams)) == 3


def test_item_batches_without_flatten_need_a_device():
  ds = make('A')
  with pytest.raises(ValueError, match='CUDA'):
    ds.create_iterator(ds.val_ids, batch_size=0)
  with pytest.raises(ValueError, match='CUDA'):
    datasets.iterator_from_dataset(torch.zeros(4, 3), batch_size=2)
