"""Camera geometry on the evaluation path: rays of a frame generated on the GPU.

Mirror of the part of `nerfies.camera.Camera` (nerfies/camera.py:108-341) and of
`datasets/core.py:50-75 camera_to_rays` that `eval.py` uses per rendered frame:
same constructor arguments, JSON layout, property names and error behaviour;
`pixels_to_rays` / `camera_to_rays` run `camera_rays_kernel` through the C ABI
(`nfb_camera_rays`, `nfb_pixels_to_rays`) and return torch tensors on the device
instead of numpy arrays.  There is no CPU path.
"""
import copy
import ctypes
import json

import numpy as np
import torch

from nerfies_b200 import _lib


def _ptr(t):
  return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream(device):
  return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


_FIELDS = ('orientation', 'position', 'focal_length', 'principal_point', 'skew', 'pixel_aspect_ratio',
           'radial_distortion', 'tangential_distortion', 'image_size')


class Camera:
  """Camera geometry with the field names, JSON layout and derived properties of
  nerfies.camera.Camera (camera.py:108-223); the ray math itself runs on the GPU."""

  def __init__(self, orientation, position, focal_length, principal_point, image_size, skew=0.0,
               pixel_aspect_ratio=1.0, radial_distortion=None, tangential_distortion=None,
               dtype=np.float32):
    if dtype != np.float32:
      raise ValueError('nerfies_b200.Camera computes in float32 like the reference default')
    values = dict(orientation=orientation, position=position, focal_length=focal_length,
                  principal_point=principal_point, skew=skew, pixel_aspect_ratio=pixel_aspect_ratio,
                  radial_distortion=np.zeros(3) if radial_distortion is None else radial_distortion,
                  tangential_distortion=np.zeros(2) if tangential_distortion is None else tangential_distortion)
    for name, value in values.items():
      setattr(self, name, np.array(value, np.float32))
    self.image_size = np.array(image_size, np.uint32)   # (width, height), camera.py:136
    self.dtype = dtype
    if self.orientation.shape != (3, 3) or self.position.shape != (3,):
      raise ValueError('orientation must be (3,3) and position (3,)')

  # ---- JSON (same keys as camera.py:139-180, including the legacy 'tangential') ----
  @classmethod
  def from_json(cls, path):
    with open(str(path), 'r') as fp:
      blob = json.load(fp)
    if 'tangential' in blob:
      blob['tangential_distortion'] = blob['tangential']
    return cls(**{name: np.asarray(blob[name]) for name in _FIELDS})

  def get_parameters(self):
    return {name: getattr(self, name) for name in _FIELDS}

  def to_json(self):
    return {name: np.asarray(value).tolist() for name, value in self.get_parameters().items()}

  # ---- derived quantities (names of camera.py:182-223) ----
  scale_factor_x = property(lambda self: self.focal_length)
  scale_factor_y = property(lambda self: self.focal_length * self.pixel_aspect_ratio)
  principal_point_x = property(lambda self: self.principal_point[0])
  principal_point_y = property(lambda self: self.principal_point[1])
  has_tangential_distortion = property(lambda self: bool(np.any(self.tangential_distortion != 0.0)))
  has_radial_distortion = property(lambda self: bool(np.any(self.radial_distortion != 0.0)))
  image_size_x = property(lambda self: self.image_size[0])
  image_size_y = property(lambda self: self.image_size[1])
  image_shape = property(lambda self: (int(self.image_size[1]), int(self.image_size[0])))
  optical_axis = property(lambda self: self.orientation[2, :])
  translation = property(lambda self: -np.matmul(self.orientation, self.position))

  def copy(self):
    return copy.deepcopy(self)

  def scale(self, scale):
    """A camera for the image resized by `scale` (camera.py:323-341)."""
    if scale <= 0:
      raise ValueError('scale needs to be positive.')
    params = {k: np.copy(v) for k, v in self.get_parameters().items()}
    params['focal_length'] = self.focal_length * scale
    params['principal_point'] = self.principal_point * scale
    params['image_size'] = np.array([int(round(float(n) * scale)) for n in self.image_size])
    return Camera(**params)

  def points_to_local_points(self, points):
    """World points (..., 3) in the camera frame, on the host (camera.py:279-282)."""
    points = np.asarray(points)
    return np.matmul(self.orientation, (points - self.position).reshape(-1, 3).T).T.reshape(points.shape)

  def look_at(self, position, look_at, up, eps=1e-6):
    """A copy of the camera at `position` looking at `look_at` with `up` along the image's -y
    (camera.py:342-387).  The rotation is computed in float64 and stored as float32."""
    position = np.asarray(position, np.float64)
    optical_axis = np.asarray(look_at, np.float64) - position
    norm = np.linalg.norm(optical_axis)
    if norm < eps:
      raise ValueError('The camera center and look at position are too close.')
    optical_axis /= norm
    right_vector = np.cross(optical_axis, up)
    norm = np.linalg.norm(right_vector)
    if norm < eps:
      raise ValueError('The up-vector is parallel to the optical axis.')
    right_vector /= norm
    camera_rotation = np.identity(3)
    camera_rotation[0, :] = right_vector
    camera_rotation[1, :] = np.cross(optical_axis, right_vector)
    camera_rotation[2, :] = optical_axis
    look_at_camera = self.copy()
    look_at_camera.position = position.astype(np.float32)
    look_at_camera.orientation = camera_rotation.astype(np.float32)
    return look_at_camera

  # ---- the C-ABI view ----
  def _struct(self):
    c = _lib.NfbCamera()
    c.orientation[:] = [float(v) for v in self.orientation.reshape(-1)]
    c.position[:] = [float(v) for v in self.position]
    c.focal_length = float(self.focal_length)
    c.principal_point[:] = [float(v) for v in self.principal_point]
    c.skew = float(self.skew)
    c.pixel_aspect_ratio = float(self.pixel_aspect_ratio)
    c.radial_distortion[:] = [float(v) for v in self.radial_distortion]
    c.tangential_distortion[:] = [float(v) for v in self.tangential_distortion]
    c.image_size[:] = [int(self.image_size[0]), int(self.image_size[1])]
    return c

  # ---- GPU paths ----
  def pixels_to_rays(self, pixels):
    """Unit world-space ray directions of float32 pixel positions (..., 2) on a CUDA device.

    Replaces Camera.pixels_to_rays (camera.py:244-269); same argument checks."""
    if not torch.is_tensor(pixels):
      raise TypeError('pixels must be a torch tensor on a CUDA device')
    if pixels.shape[-1] != 2:
      raise ValueError('The last dimension of pixels must be 2.')
    if pixels.dtype != torch.float32:
      raise ValueError(f'pixels dtype ({pixels.dtype!r}) must match camera dtype (float32)')
    if not pixels.is_cuda:
      raise ValueError('pixels must live on a CUDA device: nerfies_b200 has no CPU path')
    lib = _lib.load()
    batch_shape = pixels.shape[:-1]
    flat = pixels.reshape(-1, 2).contiguous()
    out = torch.empty(flat.shape[0], 3, dtype=torch.float32, device=pixels.device)
    with torch.cuda.device(pixels.device):
      _lib.check(lib.nfb_pixels_to_rays(ctypes.byref(self._struct()), _ptr(flat), flat.shape[0],
                                        _ptr(out), _stream(pixels.device)))
    return out.reshape(*batch_shape, 3)

  def project(self, points):
    """Pixel positions (..., 2) of float32 world points (..., 3) on a CUDA device
    (camera.py:283-315), in float32 arithmetic as the reference's numpy computes it."""
    if not torch.is_tensor(points):
      raise TypeError('points must be a torch tensor on a CUDA device')
    if points.shape[-1] != 3:
      raise ValueError('The last dimension of points must be 3.')
    if points.dtype != torch.float32:
      raise ValueError(f'points dtype ({points.dtype!r}) must match camera dtype (float32)')
    if not points.is_cuda:
      raise ValueError('points must live on a CUDA device: nerfies_b200 has no CPU path')
    lib = _lib.load()
    batch_shape = points.shape[:-1]
    flat = points.reshape(-1, 3).contiguous()
    out = torch.empty(flat.shape[0], 2, dtype=torch.float32, device=points.device)
    with torch.cuda.device(points.device):
      _lib.check(lib.nfb_camera_project(ctypes.byref(self._struct()), _ptr(flat), flat.shape[0], _ptr(out),
                                        _stream(points.device)))
    return out.reshape(*batch_shape, 2)

  def get_pixel_centers(self, device):
    """Pixel centres (H, W, 2) on `device` (camera.py:317-321)."""
    return camera_to_rays(self, device)['pixels']


def camera_to_rays(camera, device, first_pixel=0, count=None):
  """Rays of a frame, generated on the GPU (datasets/core.py:50-75).

  Returns {'origins', 'directions', 'pixels'}: (H, W, 3|3|2) float32 tensors on
  `device` - or (count, ·) for a row-major pixel sub-range (one rank's slice of a
  frame, one render_image chunk)."""
  device = torch.device(device)
  if device.type != 'cuda':
    raise ValueError('camera_to_rays needs a CUDA device: nerfies_b200 has no CPU path')
  lib = _lib.load()
  h, w = camera.image_shape
  whole = count is None and first_pixel == 0
  n = h * w - first_pixel if count is None else int(count)
  origins = torch.empty(n, 3, dtype=torch.float32, device=device)
  directions = torch.empty(n, 3, dtype=torch.float32, device=device)
  pixels = torch.empty(n, 2, dtype=torch.float32, device=device)
  with torch.cuda.device(device):
    _lib.check(lib.nfb_camera_rays(ctypes.byref(camera._struct()), int(first_pixel), n, _ptr(origins),
                                   _ptr(directions), _ptr(pixels), _stream(device)))
  if whole:
    return {'origins': origins.reshape(h, w, 3), 'directions': directions.reshape(h, w, 3),
            'pixels': pixels.reshape(h, w, 2)}
  return {'origins': origins, 'directions': directions, 'pixels': pixels}
