"""Generate tests/golden/capture_small/, tests/golden/datasource_small.npz and
tests/golden/schedules.npz by executing the reference's own data and schedule code.

TEST INFRASTRUCTURE.  Authoring container only (needs /root/reference):

    python oracle/make_golden_data.py

1. Writes a small seeded Nerfies capture: six items whose cameras are 96x54 at full resolution
   (distorted, skewed + distorted and pinhole), rgb under rgb/2x/ (48x27 PNGs, so image_scale=2
   runs Camera.scale(0.5)), non-contiguous appearance / camera / warp / time ids (one item has no
   time_id: the warp_id fallback), a val split, a scene centre and scale, points.npy and three
   test cameras under camera-paths/orbit-extreme/.
2. Runs the reference's unmodified nerfies/datasets/{core,nerfies}.py on it (tf.data, flax and
   imageio are the numpy stand-ins of oracle/jaxshim) for two configurations and records: the id
   tuples, near / far, each train item's scaled and centred camera, every item's float32 rgb,
   a run of create_iterator(train_ids, flatten=True, shuffle=True) batches that crosses the epoch
   boundary, load_points(shuffle=True) drawn after it and its iterator_from_dataset batches, and
   the batch_size=0 items of val_ids.
3. Evaluates the reference's nerfies/schedules.py for every schedule type, including
   defaults.gin's DEFAULT_LR_SCHEDULE and TrainConfig's default warp-alpha schedule.
"""
import collections
import collections.abc
import json
import os
import shutil
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
REFERENCE = os.environ.get('NERFIES_REFERENCE', '/root/reference')
sys.path.insert(0, os.path.join(HERE, 'jaxshim'))
sys.path.insert(0, REFERENCE)
sys.path.insert(0, REPO)
# schedules.from_config tests `collections.Mapping`, which Python 3.10 moved to collections.abc.
collections.Mapping = collections.abc.Mapping

# The shim's additions for these modules live in files of their own, installed here.
import tensorflow  # noqa: E402  (oracle/jaxshim)
from tensorflow import data_api  # noqa: E402
from jax import numpy as jnp  # noqa: E402  (oracle/jaxshim)
data_api.install(tensorflow)
jnp.searchsorted = jnp._wrap(np.searchsorted)      # schedules.PiecewiseSchedule

from nerfies import datasets as ref_datasets  # noqa: E402  (the reference)
from nerfies import schedules as ref_schedules  # noqa: E402  (the reference)
from oracle import camera_oracle as C  # noqa: E402

GOLDEN = os.path.join(REPO, 'tests', 'golden')
CAPTURE = os.path.join(GOLDEN, 'capture_small')

ITEMS = ['left_000', 'left_003', 'right_001', 'left_007', 'right_004', 'right_009']
KINDS = ['distorted', 'skew', 'pinhole', 'distorted', 'skew', 'pinhole']
APPEARANCE = [3, 7, 3, 12, 7, 12]
CAMERA = [0, 2, 2, 5, 0, 5]
WARP = [10, 11, 11, 20, 21, 21]   # val items share a train item's warp id
TIME = [0, 4, 9, 13, 20, None]          # None: no time_id, the reader falls back to warp_id
TRAIN = ['left_003', 'left_000', 'right_004', 'left_007']
VAL = ['right_009', 'right_001']

CONFIGS = {
    'A': dict(kwargs=dict(use_appearance_id=True, use_camera_id=True, use_warp_id=True, use_time=True,
                          random_seed=12345), batch_size=1000, batches=7, points_batch=16, point_batches=5),
    'B': dict(kwargs=dict(use_appearance_id=False, use_camera_id=False, use_warp_id=True, use_time=False,
                          random_seed=777, train_stride=2), batch_size=700, batches=5, points_batch=24,
              point_batches=4),
}

SCHEDULES = {
    'constant': ('constant', 0.3),
    'linear_warp_alpha': {'type': 'linear', 'initial_value': 0.0, 'final_value': 8.0, 'num_steps': 80000},
    'linear_zero_steps': ('linear', 1.0, 0.5, 0),
    'exponential_default_lr': {'type': 'exponential', 'initial_value': 0.001, 'final_value': 0.0001,
                               'num_steps': 1000000},
    'exponential_eps': ('exponential', 0.5, 0.0, 5000),
    'cosine_easing': ('cosine_easing', 0.01, 1e-8, 100000),
    'step': {'type': 'step', 'initial_value': 0.1, 'decay_interval': 1000, 'decay_factor': 0.5,
             'max_decays': 4},
    'piecewise_elastic': {'type': 'piecewise', 'schedules': [
        (50000, ('constant', 0.01)), (100000, ('cosine_easing', 0.01, 1e-8, 100000))]},
    'delayed_lr': {'type': 'delayed', 'delay_steps': 2500, 'delay_mult': 0.01,
                   'base_schedule': {'type': 'exponential', 'initial_value': 0.001,
                                     'final_value': 0.0001, 'num_steps': 1000000}},
}
STEPS = [0, 1, 2, 7, 100, 999, 1000, 1001, 2499, 2500, 4000, 4999, 5000, 10000, 49999, 50000,
         50001, 79999, 80000, 100000, 149999, 150000, 500000, 999999, 1000000, 1200000]


def write_capture():
  if os.path.exists(CAPTURE):
    shutil.rmtree(CAPTURE)
  for sub in ('camera', 'rgb/2x', 'camera-paths/orbit-extreme'):
    os.makedirs(os.path.join(CAPTURE, sub))
  rng = np.random.RandomState(2024)
  metadata = {}
  for k, (item, kind) in enumerate(zip(ITEMS, KINDS)):
    cam = C.synthetic_camera(seed=40 + k, width=96, height=54, distortion=kind != 'pinhole',
                             skew=0.6 if kind == 'skew' else 0.0)
    with open(os.path.join(CAPTURE, 'camera', item + '.json'), 'w') as f:
      json.dump({name: np.asarray(v).tolist() for name, v in cam.items()}, f, indent=1)
    image = rng.randint(0, 256, size=(27, 48, 3)).astype(np.uint8)
    assert cv2.imwrite(os.path.join(CAPTURE, 'rgb', '2x', item + '.png'), image)
    metadata[item] = {'appearance_id': APPEARANCE[k], 'camera_id': CAMERA[k], 'warp_id': WARP[k]}
    if TIME[k] is not None:
      metadata[item]['time_id'] = TIME[k]
  for k in range(3):
    cam = C.synthetic_camera(seed=90 + k, width=96, height=54, distortion=False)
    with open(os.path.join(CAPTURE, 'camera-paths', 'orbit-extreme', f'{k:06d}.json'), 'w') as f:
      json.dump({name: np.asarray(v).tolist() for name, v in cam.items()}, f, indent=1)
  with open(os.path.join(CAPTURE, 'metadata.json'), 'w') as f:
    json.dump(metadata, f, indent=1)
  with open(os.path.join(CAPTURE, 'dataset.json'), 'w') as f:
    json.dump({'count': len(ITEMS), 'num_exemplars': len(TRAIN), 'ids': ITEMS, 'train_ids': TRAIN,
               'val_ids': VAL}, f, indent=1)
  with open(os.path.join(CAPTURE, 'scene.json'), 'w') as f:
    json.dump({'scale': 0.7, 'center': [0.1, -0.2, 0.3], 'near': 0.05, 'far': 2.5}, f, indent=1)
  np.save(os.path.join(CAPTURE, 'points.npy'), rng.normal(size=(50, 3)))


def record_datasource():
  out = {}
  for name, cfg in CONFIGS.items():
    ds = ref_datasets.from_config({'type': 'nerfies', 'data_dir': CAPTURE}, image_scale=2, **cfg['kwargs'])
    p = name + '/'
    for key in ('train_ids', 'val_ids', 'all_ids', 'appearance_ids', 'camera_ids', 'warp_ids', 'time_ids'):
      out[p + key] = np.array(list(getattr(ds, key)))
    out[p + 'near_far'] = np.array([ds.near, ds.far])
    for item in ds.train_ids:
      for k, v in ds.load_camera(item).get_parameters().items():
        out[p + f'camera/{item}/{k}'] = np.asarray(v)
    it = ds.create_iterator(ds.train_ids, flatten=True, shuffle=True, batch_size=cfg['batch_size'])
    for s in range(cfg['batches']):
      batch = next(it)
      for k, v in batch.items():
        if k == 'metadata':
          for mk, mv in v.items():
            out[p + f'batch/{s}/metadata/{mk}'] = mv[0]
        else:
          out[p + f'batch/{s}/{k}'] = v[0]
    points = ds.load_points(shuffle=True)
    out[p + 'points'] = points
    pit = ref_datasets.iterator_from_dataset(
        ref_datasets.tf.data.Dataset.from_tensor_slices(points), batch_size=cfg['points_batch'])
    for s in range(cfg['point_batches']):
      out[p + f'points_batch/{s}'] = next(pit)[0]
    vit = ds.create_iterator(ds.val_ids, batch_size=0)
    for item in ds.val_ids:
      x = next(vit)
      for k, v in x.items():
        if k == 'metadata':
          for mk, mv in v.items():
            out[p + f'val/{item}/metadata/{mk}'] = np.asarray(mv)
        else:
          out[p + f'val/{item}/{k}'] = np.asarray(v)
    out[p + 'rng_after'] = ds.rng.randint(0, 2**31 - 1, size=4)
  ds = ref_datasets.from_config({'type': 'nerfies', 'data_dir': CAPTURE}, image_scale=2)
  for item in ITEMS:
    out['rgb/' + item] = ds.load_rgb(item)
  np.savez_compressed(os.path.join(GOLDEN, 'datasource_small.npz'), **out)
  print('datasource_small.npz:', len(out), 'arrays')


def record_schedules():
  out = {'steps': np.array(STEPS, np.int64)}
  for name, spec in SCHEDULES.items():
    sched = ref_schedules.from_config(spec)
    out['value/' + name] = np.array([float(sched(s)) for s in STEPS], np.float64)
    out['spec/' + name] = np.array(json.dumps(spec))
  np.savez_compressed(os.path.join(GOLDEN, 'schedules.npz'), **out)
  print('schedules.npz:', len(SCHEDULES), 'schedules x', len(STEPS), 'steps')


if __name__ == '__main__':
  write_capture()
  record_datasource()
  record_schedules()
