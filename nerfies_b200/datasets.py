"""Nerfies captures on the GPU: drop-in for `from nerfies import datasets`.

Covers the reference's default data path (nerfies/datasets/core.py, nerfies/datasets/nerfies.py):
the preloaded iterator of train.py (flattened, shuffled rays) and eval.py (whole items), the
background points of train.py:187-197 and the test-camera rays of eval.py, without TensorFlow.

A capture is decoded once on the host and uploaded once as uint8 RGB (3 B per ray) with one
`nfb_camera` and the metadata indices per item (the "ray table", include/nerfies_b200.h).  Every
batch afterwards is one `nfb_gather_rays` launch on the current stream, which computes origins,
directions, pixel centres, rgb and metadata of the requested rays from that table: no host work,
no host<->device copy and no synchronisation per step.

The ray order is the reference's: `create_iterator` draws `self.rng.permutation(num_rays)` on
every call (core.py:425), shuffled or not, and the shuffled order is stored on the device (int32,
or int64 past 2^31 rays).  Batch s of rank r of W is the rays [s * B + r * B / W, + B / W) of the
repeated order (repeat() before batch(), then prepare_tf_data's per-device split), so a run draws
the batches the reference draws for the same `random_seed`.

Not covered (NotImplementedError): the lazy tf.data path (`preload=False`, whose shuffle buffers
have no order to reproduce), `shuffle_pixels`, `get_item(scale_factor != 1)`, depth, and
`flatten=False` with `shuffle=True`.
"""
import concurrent.futures
import ctypes
import itertools
import json
import os
import pathlib

import numpy as np
import torch

from nerfies_b200 import _lib
from nerfies_b200 import camera as camera_lib

try:
  import cv2
except ImportError:  # PIL gives the same bytes for 8-bit PNGs
  cv2 = None

_METADATA_KEYS = ('appearance', 'camera', 'warp', 'time')


def decode_image(path):
  """uint8 (h, w, 3) RGB of an image file, as datasets/nerfies.py:57-63 decodes it
  (cv2.imdecode(IMREAD_COLOR) then BGR -> RGB); PIL's convert('RGB') without cv2."""
  with open(path, 'rb') as f:
    raw = f.read()
  if cv2 is not None:
    image = cv2.imdecode(np.frombuffer(raw, np.uint8), cv2.IMREAD_COLOR)
    if image is None:
      raise ValueError(f'{path}: not a decodable image')
    return np.ascontiguousarray(image[:, :, ::-1])
  import io
  from PIL import Image
  return np.asarray(Image.open(io.BytesIO(raw)).convert('RGB'))


def _parallel_map(fn, items):
  with concurrent.futures.ThreadPoolExecutor() as pool:
    return list(pool.map(fn, items))


def _dist_rank_world(rank, world_size):
  if rank is None or world_size is None:
    import torch.distributed as dist
    on = dist.is_available() and dist.is_initialized()
    rank = (dist.get_rank() if on else 0) if rank is None else rank
    world_size = (dist.get_world_size() if on else 1) if world_size is None else world_size
  if not 0 <= rank < world_size:
    raise ValueError(f'rank {rank} is not in [0, {world_size})')
  return rank, world_size


def _rank_slice(batch_size, rank, world_size):
  """(offset, count) of a rank's share of a batch (prepare_tf_data's contiguous split)."""
  if batch_size % world_size != 0:
    raise ValueError('Batch size must be divisible by the number of devices.')
  per = batch_size // world_size
  return rank * per, per


def _batch_starts(total, batch_size, repeat, first_batch=0):
  """(start, size) of each batch of a dataset of `total` elements from batch `first_batch` on:
  repeat() then batch(), or batch() alone, which ends with a partial batch."""
  for step in itertools.count(first_batch):
    start = step * batch_size
    if not repeat and start >= total:
      return
    yield start, batch_size if repeat else min(batch_size, total - start)


class RayTable:
  """A capture's items on the host: uint8 rgb, cameras, pixel offsets and metadata."""

  def __init__(self, images, cameras, metadata):
    self.shapes = [img.shape[:2] for img in images]
    sizes = [h * w for h, w in self.shapes]
    self.offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    self.num_rays = int(self.offsets[-1])
    self.images = images
    self.cameras = cameras
    self.metadata = metadata            # {key: (num_images,) int32 | float32}


class DeviceRayTable:
  """The ray table uploaded once to `device`; `gather` is one nfb_gather_rays launch."""

  def __init__(self, host, device, order=None):
    device = torch.device(device)
    if device.type != 'cuda':
      raise ValueError(f'the ray table lives on a CUDA device, not {device}: nerfies_b200 has no CPU path')
    self.device = device
    self.num_rays = host.num_rays
    self.shapes = host.shapes
    self.offsets = host.offsets
    n = len(host.cameras)
    self.rgb = torch.empty(host.num_rays * 3, dtype=torch.uint8, device=device)
    for img, o in zip(host.images, host.offsets):
      self.rgb[3 * o:3 * o + img.size].copy_(torch.from_numpy(img.reshape(-1)))
    structs = (_lib.NfbCamera * n)(*[c._struct() for c in host.cameras])
    self.cameras = torch.frombuffer(bytearray(bytes(structs)), dtype=torch.uint8).to(device)
    self.pixel_offsets = torch.from_numpy(host.offsets).to(device)
    self.metadata = {k: torch.from_numpy(v).to(device) for k, v in host.metadata.items()}
    self.order = None if order is None else self._upload_order(order)
    self._struct = None

  def _upload_order(self, order):
    dtype = np.int32 if self.num_rays < 2**31 else np.int64
    return torch.from_numpy(np.ascontiguousarray(order, dtype)).to(self.device)

  def table(self):
    if self._struct is None:
      t = _lib.NfbRayTable()
      t.num_images = len(self.shapes)
      t.cameras = self.cameras.data_ptr()
      t.pixel_offsets = self.pixel_offsets.data_ptr()
      t.rgb = self.rgb.data_ptr()
      for k, v in self.metadata.items():
        setattr(t, k, v.data_ptr())
      t.order = None if self.order is None else self.order.data_ptr()
      t.order_is_64 = int(self.order is not None and self.order.dtype == torch.int64)
      t.num_rays = self.num_rays
      self._struct = t
    return self._struct

  def nbytes(self):
    ts = [self.rgb, self.cameras, self.pixel_offsets, self.order, *self.metadata.values()]
    return sum(t.numel() * t.element_size() for t in ts if t is not None)

  def gather(self, first, count, order=True):
    """Rays [first, first + count) of the (repeated) order; `order=False`: identity order."""
    dev = self.device
    f32 = dict(dtype=torch.float32, device=dev)
    out = {'origins': torch.empty(count, 3, **f32), 'directions': torch.empty(count, 3, **f32),
           'pixels': torch.empty(count, 2, **f32), 'rgb': torch.empty(count, 3, **f32),
           'metadata': {k: torch.empty(count, 1, dtype=v.dtype, device=dev) for k, v in self.metadata.items()}}
    t = self.table()
    if not order and self.order is not None:
      t = _lib.NfbRayTable.from_buffer_copy(t)
      t.order = None
    md = out['metadata']
    ptr = lambda x: None if x is None else ctypes.c_void_p(x.data_ptr())
    with torch.cuda.device(dev):
      _lib.check(_lib.load().nfb_gather_rays(
          ctypes.byref(t), int(first), int(count), ptr(out['origins']), ptr(out['directions']),
          ptr(out['pixels']), ptr(out['rgb']), *[ptr(md.get(k)) for k in _METADATA_KEYS],
          ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return out

  def item(self, k):
    """Item k as (h, w, ·) tensors; metadata (h, w, 1) (eval.py:297-300, batch_size=0)."""
    h, w = self.shapes[k]
    out = self.gather(int(self.offsets[k]), h * w, order=False)
    shape = lambda x: x.reshape(h, w, -1)
    return {'rgb': shape(out['rgb']), 'origins': shape(out['origins']),
            'directions': shape(out['directions']), 'pixels': shape(out['pixels']),
            'metadata': {key: shape(v) for key, v in out['metadata'].items()}}


def _upload(host, device, order):
  return DeviceRayTable(host, device, order)


class NerfiesDataSource:
  """A Nerfies capture directory (datasets/nerfies.py:81-193 with core.DataSource)."""

  def __init__(self, data_dir, image_scale, shuffle_pixels=False, camera_type='json',
               test_camera_trajectory='orbit-extreme', use_appearance_id=False, use_camera_id=False,
               use_warp_id=False, use_depth=False, use_relative_depth=False, use_time=False,
               random_seed=0, train_stride=1, val_stride=1, preload=True, device=None, **_):
    if shuffle_pixels:
      raise NotImplementedError('shuffle_pixels belongs to the lazy tf.data path, which is not implemented')
    if use_depth or use_relative_depth:
      raise NotImplementedError('NerfiesDataSource has no depth (the reference defines no load_depth)')
    if camera_type != 'json':
      raise ValueError(f'Unknown camera type {camera_type!r}.')
    self.data_dir = pathlib.Path(data_dir)
    with open(self.data_dir / 'dataset.json') as f:
      ids = json.load(f)
    self._train_ids = [str(i) for i in ids['train_ids']]
    self._val_ids = [str(i) for i in ids['val_ids']]
    with open(self.data_dir / 'scene.json') as f:
      scene = json.load(f)
    self.scene_center = np.array(scene['center'])
    self.scene_scale = scene['scale']
    self._near, self._far = scene['near'], scene['far']
    self.metadata_dict = None
    if (self.data_dir / 'metadata.json').exists():
      with open(self.data_dir / 'metadata.json') as f:
        self.metadata_dict = json.load(f)
    self.image_scale = image_scale
    self.shuffle_pixels = shuffle_pixels
    self.camera_type = camera_type
    self.test_camera_trajectory = test_camera_trajectory
    self.rgb_dir = self.data_dir / 'rgb' / f'{image_scale}x'
    self.camera_dir = self.data_dir / 'camera'
    self.use_appearance_id, self.use_camera_id = use_appearance_id, use_camera_id
    self.use_warp_id, self.use_time = use_warp_id, use_time
    self.use_depth = False
    self.train_stride, self.val_stride = train_stride, val_stride
    self.rng = np.random.RandomState(random_seed)
    self.preload = preload
    self._device = device
    self._id_cache = {}

  @property
  def device(self):
    if self._device is None:
      self._device = torch.device('cuda', torch.cuda.current_device())
    return torch.device(self._device)

  # ---- ids (core.py:227-315) ----
  train_ids = property(lambda self: self._train_ids[::self.train_stride])
  val_ids = property(lambda self: self._val_ids[::self.val_stride])
  all_ids = property(lambda self: sorted(itertools.chain(self.train_ids, self.val_ids)))
  near = property(lambda self: self._near)
  far = property(lambda self: self._far)
  has_metadata = property(lambda self: self.use_appearance_id or self.use_warp_id or self.use_camera_id)
  camera_ext = '.json'

  def _metadata_value(self, item_id, key):
    entry = self.metadata_dict[item_id]
    if key == 'time_id' and key not in entry:
      key = 'warp_id'          # datasets/nerfies.py:188-193: older captures
    return entry[key]

  def get_appearance_id(self, item_id):
    return self._metadata_value(item_id, 'appearance_id')

  def get_camera_id(self, item_id):
    return self._metadata_value(item_id, 'camera_id')

  def get_warp_id(self, item_id):
    return self._metadata_value(item_id, 'warp_id')

  def get_time_id(self, item_id):
    return self._metadata_value(item_id, 'time_id')

  def _ids(self, key, enabled):
    """Sorted distinct ids of the train items (core.py:276-303)."""
    if not enabled:
      return tuple()
    if key not in self._id_cache:
      self._id_cache[key] = tuple(sorted({self._metadata_value(i, key) for i in self.train_ids}))
    return self._id_cache[key]

  appearance_ids = property(lambda self: self._ids('appearance_id', self.use_appearance_id))
  camera_ids = property(lambda self: self._ids('camera_id', self.use_camera_id))
  warp_ids = property(lambda self: self._ids('warp_id', self.use_warp_id))
  time_ids = property(lambda self: self._ids('time_id', self.use_time))

  def get_time(self, item_id):
    return (self.get_time_id(item_id) / max(self.time_ids)) * 2.0 - 1.0

  def _item_metadata(self, item_id):
    md = {}
    if self.use_appearance_id:
      md['appearance'] = self.appearance_ids.index(self.get_appearance_id(item_id))
    if self.use_camera_id:
      md['camera'] = self.camera_ids.index(self.get_camera_id(item_id))
    if self.use_warp_id:
      md['warp'] = self.warp_ids.index(self.get_warp_id(item_id))
    if self.use_time:
      md['time'] = self.get_time(item_id)
    return md

  # ---- items ----
  def get_rgb_path(self, item_id):
    return self.rgb_dir / f'{item_id}.png'

  def load_rgb(self, item_id):
    """float32 (h, w, 3) on the device: u8 / 255 (datasets/nerfies.py:62)."""
    rgb = decode_image(self.get_rgb_path(item_id)).astype(np.float32) / np.float32(255.0)
    return torch.from_numpy(rgb).to(self.device)

  def load_camera(self, item_id, scale_factor=1.0):
    """The item's camera (or the camera file `item_id` when it is a path), scaled to the images
    and centred and scaled into the scene (core.py:78-107, in float64 then float32)."""
    if isinstance(item_id, (pathlib.PurePath, os.PathLike)):
      path = pathlib.Path(item_id)
    else:
      path = self.camera_dir / f'{item_id}{self.camera_ext}'
    if path.suffix != '.json':
      raise ValueError('File must have extension .pb or .json.')
    camera = camera_lib.Camera.from_json(path)
    scale = scale_factor / self.image_scale
    if scale != 1.0:
      camera = camera.scale(scale)
    position = (camera.position.astype(np.float64) - self.scene_center) * self.scene_scale
    camera.position = position.astype(np.float32)
    return camera

  def get_item(self, item_id, scale_factor=1.0):
    """{'camera_params', 'rgb' (device float32), 'metadata'} (core.py:567-619)."""
    if scale_factor != 1.0:
      raise NotImplementedError('get_item(scale_factor != 1) needs image_utils.rescale_image, '
                                'which is not implemented')
    camera = self.load_camera(item_id)
    return {'camera_params': camera.get_parameters(), 'rgb': self.load_rgb(item_id),
            'metadata': self._item_metadata(item_id)}

  def load_points(self, shuffle=False):
    """Background points (N, 3) float32 on the device, centred and scaled into the scene; with
    `shuffle`, permuted by a draw from `self.rng` (datasets/nerfies.py:167-177)."""
    points = np.load(self.data_dir / 'points.npy')
    points = ((points - self.scene_center) * self.scene_scale).astype(np.float32)
    if shuffle:
      points = points[self.rng.permutation(len(points))]
    return torch.from_numpy(np.ascontiguousarray(points)).to(self.device)

  def glob_cameras(self, path):
    return sorted(pathlib.Path(path).glob(f'*{self.camera_ext}'))

  def load_test_cameras(self, count=None):
    camera_dir = self.data_dir / 'camera-paths' / self.test_camera_trajectory
    if not camera_dir.exists():
      return []
    paths = self.glob_cameras(camera_dir)
    if count is not None:
      paths = paths[::max(1, len(paths) // count)]
    return _parallel_map(self.load_camera, paths)

  # ---- the preloaded ray table ----
  def ray_table(self, item_ids):
    """Decodes the items (in a thread pool) into a host RayTable; checks each image against its
    camera's image_shape."""
    item_ids = list(item_ids)
    if not item_ids:
      raise ValueError('no items')
    images = _parallel_map(lambda i: decode_image(self.get_rgb_path(i)), item_ids)
    cameras = _parallel_map(self.load_camera, item_ids)
    for item_id, img, cam in zip(item_ids, images, cameras):
      if img.shape[:2] != cam.image_shape:
        raise ValueError(f'item {item_id!r}: image {self.get_rgb_path(item_id)} is {img.shape[:2]} (h, w) but '
                         f'its camera scaled by 1/{self.image_scale} gives {cam.image_shape}')
    mds = [self._item_metadata(i) for i in item_ids]
    metadata = {k: np.array([md[k] for md in mds], np.float32 if k == 'time' else np.int32)
                for k in _METADATA_KEYS if k in mds[0]}
    return RayTable(images, cameras, metadata)

  def create_iterator(self, item_ids, batch_size, repeat=True, flatten=False, shuffle=False,
                      prefetch_size=0, shuffle_buffer_size=1000000, devices=None, rank=None,
                      world_size=None, first_batch=0):
    """The batches of core.py:352-372 with preload (see the module docstring).  With
    `batch_size=0`, whole items as (h, w, ·) tensors; otherwise dicts of rank `rank`'s
    batch_size / world_size rays ('metadata' values (b, 1)).  `prefetch_size`,
    `shuffle_buffer_size` and `devices` are accepted for the reference's signature: batches are
    made on this source's device, in order on the current stream, when next() is called.
    `first_batch` (flattened rays only) starts the stream at that batch, at no cost: a resumed
    run continues where the interrupted one stopped instead of replaying the order's head."""
    del prefetch_size, shuffle_buffer_size, devices
    if not self.preload:
      raise NotImplementedError('preload=False is the lazy tf.data path with shuffle buffers; it has no '
                                'reproducible order and is not implemented')
    if shuffle and not flatten:
      raise NotImplementedError('shuffle without flatten: the reference permutes items with a permutation '
                                'of the rays (core.py:425-440)')
    rank, world_size = _dist_rank_world(rank, world_size)
    if batch_size > 0:
      _rank_slice(batch_size, rank, world_size)
    host = self.ray_table(item_ids)
    order = self.rng.permutation(host.num_rays)      # core.py:425: drawn on every call
    table = _upload(host, self.device, order if shuffle else None)
    if first_batch and not (flatten and batch_size > 0):
      raise NotImplementedError('first_batch is for batches of flattened rays')
    if batch_size <= 0:
      return _item_iterator(table, repeat)
    if flatten:
      return _ray_iterator(table, batch_size, repeat, rank, world_size, first_batch)
    return _item_batch_iterator(table, batch_size, repeat, rank, world_size)

  def create_cameras_dataset(self, cameras, flatten=False, shuffle=False):
    """The rays of each test camera (or camera file), made by camera.camera_to_rays on this
    source's device when iterated.  This is the numpy Camera's arithmetic (camera.py), which the
    kernel reproduces, not tf_camera.py's TensorFlow arithmetic that core.py:321-350 uses."""
    if flatten or shuffle:
      raise NotImplementedError('create_cameras_dataset yields whole frames only')
    if cameras and isinstance(cameras[0], (str, pathlib.PurePath, os.PathLike)):
      cameras = _parallel_map(self.load_camera, [pathlib.Path(c) for c in cameras])
    return CamerasDataset(cameras, self.device)


class CamerasDataset:
  """Re-iterable: camera_to_rays of each camera, (h, w, ·) tensors."""

  def __init__(self, cameras, device):
    self.cameras, self.device = list(cameras), device

  def __len__(self):
    return len(self.cameras)

  def __iter__(self):
    for cam in self.cameras:
      yield camera_lib.camera_to_rays(cam, self.device)


def _item_iterator(table, repeat):
  while True:
    for k in range(len(table.shapes)):
      yield table.item(k)
    if not repeat:
      return


def _ray_iterator(table, batch_size, repeat, rank, world_size, first_batch=0):
  for start, size in _batch_starts(table.num_rays, batch_size, repeat, first_batch):
    offset, count = _rank_slice(size, rank, world_size)
    yield table.gather(start + offset, count)


def _item_batch_iterator(table, batch_size, repeat, rank, world_size):
  """flatten=False, batch_size > 0: batches of whole items, stacked (items of one size)."""
  n = len(table.shapes)
  for start, size in _batch_starts(n, batch_size, repeat):
    offset, count = _rank_slice(size, rank, world_size)
    items = [table.item((start + offset + j) % n) for j in range(count)]
    stack = lambda *xs: torch.stack(xs)
    yield {k: stack(*[it[k] for it in items]) for k in ('rgb', 'origins', 'directions', 'pixels')} | {
        'metadata': {k: stack(*[it['metadata'][k] for it in items]) for k in items[0]['metadata']}}


def iterator_from_dataset(dataset, batch_size, repeat=True, prefetch_size=0, devices=None, rank=None,
                          world_size=None, first_batch=0):
  """Batches of a device tensor along its first axis (train.py:187-197's background points), with
  core.py:131-160's repeat-then-batch semantics and rank `rank`'s contiguous slice of each batch;
  a batch is at most two device-to-device copies.  With `batch_size=0`, the elements of
  `dataset` one by one (eval.py's test cameras: `create_cameras_dataset`).  `first_batch` starts
  the batches of a tensor at that batch (see `create_iterator`)."""
  del prefetch_size, devices
  if first_batch and batch_size <= 0:
    raise NotImplementedError('first_batch is for batches of a tensor')
  if batch_size <= 0:
    return _elements(dataset, repeat)
  if not torch.is_tensor(dataset) or not dataset.is_cuda:
    raise ValueError('iterator_from_dataset batches a CUDA tensor (e.g. load_points())')
  rank, world_size = _dist_rank_world(rank, world_size)
  _rank_slice(batch_size, rank, world_size)
  return _tensor_batches(dataset, batch_size, repeat, rank, world_size, first_batch)


def _elements(dataset, repeat):
  while True:
    yield from dataset
    if not repeat:
      return


def _tensor_batches(points, batch_size, repeat, rank, world_size, first_batch=0):
  n = points.shape[0]
  for start, size in _batch_starts(n, batch_size, repeat, first_batch):
    offset, count = _rank_slice(size, rank, world_size)
    out = torch.empty((count,) + tuple(points.shape[1:]), dtype=points.dtype, device=points.device)
    done, src = 0, (start + offset) % n
    while done < count:
      m = min(count - done, n - src)
      out[done:done + m].copy_(points[src:src + m])
      done, src = done + m, 0
    yield out


def from_config(spec, **kwargs):
  """A data source from a {'type': 'nerfies', 'data_dir': ...} spec (datasets/__init__.py)."""
  spec = dict(spec)
  ds_type = spec.pop('type')
  if ds_type == 'nerfies':
    return NerfiesDataSource(**spec, **kwargs)
  raise ValueError(f'Unknown datasource type {ds_type!r}')
