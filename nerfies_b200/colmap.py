"""COLMAP sparse models on the host: cameras.bin, images.bin and points3D.bin.

Read from COLMAP's documented binary layout (little-endian):
  cameras.bin   u64 count; per camera: u32 camera_id, i32 model_id, u64 width, u64 height,
                f64 params[n(model)]
  images.bin    u64 count; per image: u32 image_id, f64 qvec[4] (w, x, y, z), f64 tvec[3],
                u32 camera_id, NUL-terminated name, u64 num_points2D, then per 2D point
                f64 x, f64 y, i64 point3D_id
  points3D.bin  u64 count; per point: u64 point3D_id, f64 xyz[3], u8 rgb[3], f64 error,
                u64 track_length, then per track element u32 image_id, u32 point2D_idx

`load_scene` turns a model into what the capture notebook's SceneManager.from_pycolmap holds:
one nerfies_b200.Camera per registered image, keyed by the image name up to its first '.', and
the points whose tracks see at least `min_track_length` distinct images, in file order.
"""
import dataclasses
import os
import struct

import numpy as np

from nerfies_b200.camera import Camera

# model_id -> (name, parameter names).  Missing coefficients are zero in `convert_camera`.
CAMERA_MODELS = {
    0: ('SIMPLE_PINHOLE', ('f', 'cx', 'cy')),
    1: ('PINHOLE', ('fx', 'fy', 'cx', 'cy')),
    2: ('SIMPLE_RADIAL', ('f', 'cx', 'cy', 'k1')),
    3: ('RADIAL', ('f', 'cx', 'cy', 'k1', 'k2')),
    4: ('OPENCV', ('fx', 'fy', 'cx', 'cy', 'k1', 'k2', 'p1', 'p2')),
}
# Parameter counts of COLMAP's other models, so that an unsupported one is named, not misparsed.
_OTHER_MODELS = {5: ('OPENCV_FISHEYE', 8), 6: ('FULL_OPENCV', 12), 7: ('FOV', 5),
                 8: ('SIMPLE_RADIAL_FISHEYE', 4), 9: ('RADIAL_FISHEYE', 5), 10: ('THIN_PRISM_FISHEYE', 12)}


@dataclasses.dataclass
class ColmapCamera:
  camera_id: int
  model: str
  width: int
  height: int
  params: dict


@dataclasses.dataclass
class ColmapImage:
  image_id: int
  qvec: np.ndarray        # (w, x, y, z)
  tvec: np.ndarray
  camera_id: int
  name: str


class _Reader:
  def __init__(self, path):
    with open(path, 'rb') as f:
      self.data = f.read()
    self.path = path
    self.pos = 0

  def read(self, fmt):
    size = struct.calcsize('<' + fmt)
    if self.pos + size > len(self.data):
      raise ValueError(f'{self.path}: truncated at byte {self.pos}')
    out = struct.unpack_from('<' + fmt, self.data, self.pos)
    self.pos += size
    return out

  def cstring(self):
    end = self.data.find(b'\0', self.pos)
    if end < 0:
      raise ValueError(f'{self.path}: unterminated image name at byte {self.pos}')
    out = self.data[self.pos:end].decode('utf-8')
    self.pos = end + 1
    return out


def read_cameras(path):
  r = _Reader(path)
  cameras = {}
  for _ in range(r.read('Q')[0]):
    camera_id, model_id, width, height = r.read('IiQQ')
    if model_id not in CAMERA_MODELS:
      name, _ = _OTHER_MODELS.get(model_id, (f'model id {model_id}', 0))
      raise ValueError(f'COLMAP camera {camera_id} uses the {name} model; supported models are '
                       f'{", ".join(n for n, _ in CAMERA_MODELS.values())}')
    name, keys = CAMERA_MODELS[model_id]
    params = dict(zip(keys, r.read('d' * len(keys))))
    cameras[camera_id] = ColmapCamera(camera_id, name, width, height, params)
  return cameras


def read_images(path):
  r = _Reader(path)
  images = {}
  for _ in range(r.read('Q')[0]):
    image_id = r.read('I')[0]
    qvec = np.array(r.read('dddd'))
    tvec = np.array(r.read('ddd'))
    camera_id = r.read('I')[0]
    name = r.cstring()
    n2d = r.read('Q')[0]
    r.pos += 24 * n2d                   # the 2D observations are not needed here
    if r.pos > len(r.data):
      raise ValueError(f'{path}: truncated in image {image_id}')
    images[image_id] = ColmapImage(image_id, qvec, tvec, camera_id, name)
  return images


def read_points3d(path, min_track_length=0):
  """(xyz (n, 3) float64, point ids (n,) uint64) of the points whose track holds at least
  `min_track_length` distinct image ids, in file order."""
  r = _Reader(path)
  xyz, ids = [], []
  for _ in range(r.read('Q')[0]):
    point_id = r.read('Q')[0]
    p = r.read('ddd')
    r.read('BBBd')                      # colour and reprojection error
    track_length = r.read('Q')[0]
    track = r.read('I' * (2 * track_length))
    if len(set(track[0::2])) >= min_track_length:
      xyz.append(p)
      ids.append(point_id)
  return np.array(xyz, np.float64).reshape(-1, 3), np.array(ids, np.uint64)


def qvec_to_rotation(q):
  """Rotation matrix of the quaternion (w, x, y, z)."""
  w, x, y, z = q
  return np.eye(3) + 2 * np.array([
      [-y * y - z * z, x * y - z * w, x * z + y * w],
      [x * y + z * w, -x * x - z * z, y * z - x * w],
      [x * z - y * w, y * z + x * w, -x * x - y * y]])


def convert_camera(colmap_camera, image):
  """A nerfies_b200.Camera as the notebook's convert_colmap_camera builds it: world-to-camera
  rotation R, position -(t @ R), focal fx, pixel aspect ratio 1 and k3 = 0."""
  p = colmap_camera.params
  rotation = qvec_to_rotation(image.qvec)
  fx = p.get('fx', p.get('f'))
  return Camera(orientation=rotation, position=-(image.tvec @ rotation), focal_length=fx,
                pixel_aspect_ratio=fx / fx, principal_point=np.array([p['cx'], p['cy']]),
                radial_distortion=np.array([p.get('k1', 0.0), p.get('k2', 0.0), 0.0]),
                tangential_distortion=np.array([p.get('p1', 0.0), p.get('p2', 0.0)]), skew=0.0,
                image_size=np.array([colmap_camera.width, colmap_camera.height]))


def item_id(image_name):
  """The notebook's item id of a COLMAP image: its name up to the first '.'."""
  return image_name.split('.')[0]


def load_scene(model_dir, min_track_length=5):
  """({item id: Camera}, track-filtered points (n, 3) float64) of a COLMAP model directory."""
  model_dir = str(model_dir)
  cameras = read_cameras(os.path.join(model_dir, 'cameras.bin'))
  images = read_images(os.path.join(model_dir, 'images.bin'))
  points, _ = read_points3d(os.path.join(model_dir, 'points3D.bin'), min_track_length)
  result = {}
  for image in images.values():
    if image.camera_id not in cameras:
      raise ValueError(f'image {image.name!r} refers to camera {image.camera_id}, which cameras.bin lacks')
    result[item_id(image.name)] = convert_camera(cameras[image.camera_id], image)
  return result, points
