"""visualization.colorize (visualization.py:177-219) on the GPU, and the render-video notebook's
frame (Nerfies_Render_Video.ipynb, "Show rendered video"), through `nfb_colorize`.

`colorize` returns what the reference returns, float64 (..., 3), value for value for the same
table.  `colorize_uint8` is the same followed by image_utils.image_to_uint8 in one launch (two when a
bound comes from the frame), without a float64 image in between; it can write into a column range
of a wider frame.  `source` selects what is mapped: the array ('value'), its reciprocal
('reciprocal', eval.py:94-95's disparity), or the per-pixel error sum of two (h, w, 3) images
('abs_error', 'sq_error', eval.py:129-132).  Bounds are Python numbers, as eval.py passes them:
with both given, max(cmax - cmin, eps) is taken in float64 on the host; a bound left None is the
frame's min / max, found on the device (NaN if the frame holds a NaN, as np.min), and the
subtraction is then float32, as numpy does it with a float32 scalar.

Colour tables: matplotlib is not a dependency, so `get_colormap` takes OpenCV's 256-entry tables
(cv2.applyColorMap over 0..255, BGR -> RGB, / 255).  Each entry is within 0.5 / 255 of matplotlib's,
so a uint8 pixel is at most one level from the reference's.  OpenCV's turbo equals
round(255 * the reference's turbo table) / 255 (checked in tests/test_visualization.py); magma and
the others could not be compared with matplotlib.  A caller's own (256, 3) table is taken as given.

`flow_to_color` colour-codes optical flow (track_pixels' dense flow) with the Baker et al. wheel.
"""
import ctypes
import functools

import numpy as np
import torch

from nerfies_b200 import _lib

SOURCES = {'value': 0, 'reciprocal': 1, 'abs_error': 2, 'sq_error': 3}
_RGB = 4
_INVERT, _FRAME_MIN, _FRAME_MAX = 1, 2, 4
_WORKSPACE_FLOATS = 512              # NFB_VIZ_WORKSPACE_BYTES / 4
_device_tables = {}


@functools.lru_cache(maxsize=32)
def _opencv_table(name):
  import cv2
  code = getattr(cv2, 'COLORMAP_' + name.upper(), None)
  if code is None:
    names = sorted(k[len('COLORMAP_'):].lower() for k in dir(cv2) if k.startswith('COLORMAP_'))
    raise ValueError(f'unknown colour map {name!r}; OpenCV has {names}')
  bgr = cv2.applyColorMap(np.arange(256, dtype=np.uint8).reshape(256, 1), code)
  table = bgr[:, 0, ::-1].astype(np.float64) / 255.0
  table.setflags(write=False)
  return table


def get_colormap(name):
  """(256, 3) float64 RGB table of OpenCV's colour map `name` ('magma', 'turbo', 'viridis', ...), or
  the caller's own (256, 3) table."""
  if isinstance(name, str):
    return _opencv_table(name)
  table = np.asarray(name, np.float64)
  if table.shape != (256, 3):
    raise ValueError(f'a colour table must be (256, 3), got {table.shape}')
  return table


def _table_on(cmap, device):
  """The table as a device tensor; named tables are uploaded once per device."""
  if not isinstance(cmap, str):
    return torch.as_tensor(np.ascontiguousarray(get_colormap(cmap)), device=device)
  key = (cmap, device)
  if key not in _device_tables:
    _device_tables[key] = torch.as_tensor(get_colormap(cmap).copy(), device=device)
  return _device_tables[key]


def _check(name, t):
  if not torch.is_tensor(t) or not t.is_cuda:
    raise ValueError(f'{name} must be a torch tensor on a CUDA device: nerfies_b200 has no CPU path')
  if t.dtype != torch.float32:
    raise ValueError(f'{name} must be float32, got {t.dtype}')
  return t.contiguous()


def _launch(array, target, source, cmin, cmax, cmap, eps, invert, out_f64, out_u8, height, width, pitch):
  flags = _INVERT if invert else 0
  if cmin is None or cmax is None:
    if array.numel() == 0:
      raise ValueError('the range of an empty frame is undefined (np.min raises for it)')
    flags |= (_FRAME_MIN if cmin is None else 0) | (_FRAME_MAX if cmax is None else 0)
    d = eps
  else:
    d = max(cmax - cmin, eps)          # Python numbers: float64, as numpy with two Python floats
  dev = array.device
  ptr = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
  with torch.cuda.device(dev):
    table = _table_on(cmap, dev) if source != _RGB else None
    workspace = torch.empty(_WORKSPACE_FLOATS, dtype=torch.float32, device=dev) if flags & (_FRAME_MIN | _FRAME_MAX) else None
    _lib.check(_lib.load().nfb_colorize(
        ptr(array), ptr(target), height, width, source, ptr(table),
        float(cmin or 0.0), float(cmax or 0.0), float(d), flags, ptr(workspace), ptr(out_f64), ptr(out_u8),
        pitch, ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))


def _inputs(array, source, target):
  """(array, target, value shape) for a source."""
  if source not in SOURCES:
    raise ValueError(f'unknown source {source!r}; one of {sorted(SOURCES)}')
  array = _check('array', array)
  if SOURCES[source] < 2:
    if target is not None:
      raise ValueError(f'source {source!r} takes no target')
    return array, None, tuple(array.shape)
  target = _check('target', target)
  if array.shape != target.shape or array.dim() < 1 or array.shape[-1] != 3:
    raise ValueError(f'error maps take two (..., 3) images of one shape, got {tuple(array.shape)} and '
                     f'{tuple(target.shape)}')
  if target.device != array.device:
    raise ValueError('array and target must be on one device')
  return array, target, tuple(array.shape[:-1])


def colorize(array, cmin=None, cmax=None, cmap='magma', eps=1e-6, invert=False, source='value', target=None):
  """visualization.colorize: CUDA float32 in, CUDA float64 (..., 3) out.  With an error source,
  `array` and `target` are the two (..., 3) images."""
  array, target, shape = _inputs(array, source, target)
  out = torch.empty(shape + (3,), dtype=torch.float64, device=array.device)
  n = out.numel() // 3
  _launch(array, target, SOURCES[source], cmin, cmax, cmap, eps, invert, out, None, 1 if n else 0, n, 0)
  return out


def colorize_uint8(array, cmin=None, cmax=None, cmap='magma', eps=1e-6, invert=False, source='value', target=None,
                   out=None):
  """image_to_uint8(colorize(...)) in one pass: torch.uint8 (..., 3).  `out`, if given, is an
  (h, w, 3) uint8 view with rows of any stride and packed pixels (a column range of a wider frame,
  such as frame[:, w:]); the values are (h, w) and `out` is returned."""
  array, target, shape = _inputs(array, source, target)
  if out is None:
    out = torch.empty(shape + (3,), dtype=torch.uint8, device=array.device)
    height, width = (1, out.numel() // 3) if len(shape) < 2 else (int(np.prod(shape[:-1])), shape[-1])
    pitch = 3 * width
  else:
    if (not torch.is_tensor(out) or out.dtype != torch.uint8 or out.device != array.device or
        tuple(out.shape) != shape + (3,) or len(shape) != 2 or out.stride()[1:] != (3, 1)):
      raise ValueError(f'out must be a uint8 (h, w, 3) view on {array.device} with packed pixels for values of '
                       f'shape (h, w) = {shape}')
    (height, width), pitch = shape, out.stride(0)
  _launch(array, target, SOURCES[source], cmin, cmax, cmap, eps, invert, None, out, height, width, pitch)
  return out


def video_frame(rgb, depth, near, far, cmap='magma'):
  """The render-video notebook's frame, image_to_uint8(np.concatenate([rgb, colorize(depth, near,
  far, invert=True)], axis=1)): torch.uint8 (h, 2w, 3) from rgb (h, w, 3) and depth (h, w), in two
  launches.  concatenate promotes rgb to float64, so its product with 255 is float64 here too."""
  rgb = _check('rgb', rgb)
  h, w = tuple(depth.shape)
  if tuple(rgb.shape) != (h, w, 3):
    raise ValueError(f'rgb {tuple(rgb.shape)} and depth {tuple(depth.shape)} are not one frame')
  frame = torch.empty((h, 2 * w, 3), dtype=torch.uint8, device=rgb.device)
  _launch(rgb, None, _RGB, 0.0, 1.0, None, 1.0, False, None, frame, h, w, frame.stride(0))
  colorize_uint8(depth, near, far, cmap, invert=True, out=frame[:, w:])
  return frame


def normals_to_color(normals, valid, camera):
  """A normal map (geometry.normal_map's world-frame (h, w, 3) normals and (h, w) valid mask) as a
  torch.uint8 (h, w, 3) image: each normal in the camera's frame (n_c = camera.orientation @ n; x right,
  y down, z forward) coloured RGB = (n_c * (1, -1, -1) + 1) / 2, so a surface facing the camera is
  (0.5, 0.5, 1) and one facing up is green; invalid pixels are black.  Quantised by nfb_image_quantize."""
  normals = _check('normals', normals)
  if normals.dim() != 3 or normals.shape[-1] != 3:
    raise ValueError(f'normals must be (h, w, 3), got {tuple(normals.shape)}')
  if not torch.is_tensor(valid) or valid.device != normals.device or tuple(valid.shape) != tuple(normals.shape[:2]):
    raise ValueError(f'valid must be an (h, w) = {tuple(normals.shape[:2])} tensor on {normals.device}')
  from nerfies_b200 import evaluation
  dev = normals.device
  rot = torch.as_tensor(np.asarray(camera.orientation, np.float32), device=dev)
  flip = torch.tensor([1.0, -1.0, -1.0], device=dev)
  rgb = (normals @ rot.T * flip + 1.0) * 0.5
  rgb = torch.where(valid.bool()[..., None], rgb, 0.0)
  return evaluation.image_to_uint8(rgb.contiguous())


def flow_to_color(flow, status=None, max_flow=None):
  """Optical flow (h, w, 2) float32 on a CUDA device in the colour coding of Baker et al. (IJCV 2011),
  torch.uint8 (h, w, 3) on the same device (nfb_flow_colorize).  `status` (h, w) (_lib.TRACK_STATUS
  codes) blacks out every pixel that is not 'visible'; the flow is divided by `max_flow`, or, when it is
  None or <= 0, by the largest magnitude among the visible pixels."""
  flow = _check('flow', flow)
  if flow.dim() != 3 or flow.shape[-1] != 2:
    raise ValueError(f'flow must be (h, w, 2), got {tuple(flow.shape)}')
  h, w = int(flow.shape[0]), int(flow.shape[1])
  if status is not None:
    if not torch.is_tensor(status) or status.device != flow.device or tuple(status.shape) != (h, w):
      raise ValueError(f'status must be an (h, w) = ({h}, {w}) tensor on {flow.device}')
    status = status.to(torch.int32).contiguous()
  out = torch.empty(h, w, 3, dtype=torch.uint8, device=flow.device)
  scale = float(max_flow) if max_flow is not None and max_flow > 0 else 0.0
  ptr = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
  with torch.cuda.device(flow.device):
    workspace = torch.empty(_WORKSPACE_FLOATS, dtype=torch.float32, device=flow.device) if scale == 0.0 else None
    _lib.check(_lib.load().nfb_flow_colorize(ptr(flow), ptr(status), h, w, scale, ptr(workspace), ptr(out), 3 * w,
                                             ctypes.c_void_p(torch.cuda.current_stream(flow.device).cuda_stream)))
  return out
