"""Capture processing: from frames and a COLMAP model to the files a Nerfies capture holds.

The steps of the reference's capture notebook (notebooks/Nerfies_Capture_Processing.ipynb) from
"Resize images into different scales" through "Save test cameras", as library calls.  The
per-pixel and per-point work runs on the GPU (include/nerfies_b200.h, "capture processing"):
  downsample_frames    the image pyramid of one frame            nfb_frame_pyramid
  blur_scores          variance of the Laplacian per frame       nfb_blur_scores
  estimate_near_far    per-camera depth quantiles                nfb_near_far
  resample_depth       a sensor depth map onto one frame         nfb_depth_resample
  depth_scale_pairs    points projected into a frame             nfb_camera_project
The rest is host arithmetic on a handful of values per camera:
  blur_filter, filter_outlier_points, scene_info, orbit_camera_path, split_and_metadata,
  estimate_depth_scale.
DESIGN.md §5.5d lists what each step reproduces, including where the notebook's code and its
comments disagree.
"""
import bisect
import ctypes
import math

import numpy as np
import torch

from nerfies_b200 import _lib

VAL_STRIDE = 20              # dataset.json: val_ids = ids[::20]
INLIER_FRACTION = 0.95       # filter_outlier_points(points, 0.95)
NEAR_QUANTILE, FAR_QUANTILE = 0.001, 0.999
NEAR_MARGIN, FAR_MARGIN = 0.8, 1.2
ORBIT_Z_OFFSET = -0.1


def _ptr(t):
  return ctypes.c_void_p(t.data_ptr())


def _stream(device):
  return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _cuda_u8_frames(frames, ndim):
  if not torch.is_tensor(frames) or not frames.is_cuda:
    raise ValueError('frames must be a torch tensor on a CUDA device: nerfies_b200 has no CPU path')
  if frames.dtype != torch.uint8 or frames.dim() != ndim or frames.shape[-1] != 3:
    raise ValueError(f'frames must be uint8 RGB of {ndim} dimensions (..., height, width, 3), got '
                     f'{frames.dtype} {tuple(frames.shape)}')


def check_scales(scales):
  scales = [int(s) for s in scales]
  if not scales:
    raise ValueError('at least one image scale is needed')
  for s in scales:
    if s != 1 and (s < 2 or s % 2):
      raise ValueError(f'image scale {s} is not supported: scales must be 1 or even')
  top = max(scales)
  for s in scales:
    if top % s:
      raise ValueError(f'image scale {s} does not divide the largest scale {top}')
  return scales


def downsample_frames(frame, scales):
  """The notebook's pyramid of one (H, W, 3) uint8 frame on a CUDA device: the frame cropped to a
  multiple of max(scales) (make_divisible), then each scale; scale s > 1 is what the notebook's
  cv2.resize call computes (bilinear, see DESIGN.md §5.5d).  Returns {scale: (H/s, W/s, 3) uint8}."""
  scales = check_scales(scales)
  _cuda_u8_frames(frame, 3)
  if frame.stride(2) != 1 or frame.stride(1) != 3:
    frame = frame.contiguous()
  top = max(scales)
  h, w = frame.shape[0] - frame.shape[0] % top, frame.shape[1] - frame.shape[1] % top
  if h == 0 or w == 0:
    raise ValueError(f'frame {tuple(frame.shape[:2])} is smaller than the largest scale {top}')
  levels = {s: torch.empty(h // s, w // s, 3, dtype=torch.uint8, device=frame.device) for s in scales}
  order = list(levels)
  lib = _lib.load()
  with torch.cuda.device(frame.device):
    _lib.check(lib.nfb_frame_pyramid(
        _ptr(frame), h, w, frame.stride(0), len(order), (ctypes.c_int * len(order))(*order),
        (ctypes.c_void_p * len(order))(*[levels[s].data_ptr() for s in order]), _stream(frame.device)))
  return levels


def blur_scores(frames):
  """cv2.Laplacian(cv2.cvtColor(rgb, COLOR_RGB2GRAY), CV_64F).var() of each frame of an
  (N, H, W, 3) uint8 CUDA tensor, as an (N,) float64 CUDA tensor."""
  _cuda_u8_frames(frames, 4)
  frames = frames.contiguous()
  n, h, w = frames.shape[:3]
  lib = _lib.load()
  scores = torch.empty(n, dtype=torch.float64, device=frames.device)
  workspace = torch.empty(max(1, int(lib.nfb_blur_scores_workspace_size(n))), dtype=torch.uint8,
                          device=frames.device)
  with torch.cuda.device(frames.device):
    _lib.check(lib.nfb_blur_scores(_ptr(frames), n, h, w, _ptr(workspace), workspace.numel(), _ptr(scores),
                                   _stream(frames.device)))
  return scores


def blur_filter(item_ids, scores, blur_filter_perc):
  """The ids the notebook's "Filter blurry frames" cell removes, sharpest last: those whose score is
  >= np.percentile(scores, blur_filter_perc).  A high variance of the Laplacian is a SHARP frame, so
  the default 95 drops the sharpest 5 %; the notebook does exactly this.  No ids when perc <= 0."""
  if blur_filter_perc <= 0.0:
    return []
  scores = np.asarray(scores, np.float64)
  thres = np.percentile(scores, blur_filter_perc)
  inds = np.where(scores >= thres)[0]
  inds = inds[np.argsort([scores[i] for i in inds])]
  return [item_ids[i] for i in inds]


def filter_outlier_points(points, inner_percentile=INLIER_FRACTION):
  """Points inside the per-axis [(1 - p) / 2, 1 - (1 - p) / 2] quantile box (numpy 'linear')."""
  outer = 1.0 - inner_percentile
  lower = outer / 2.0
  upper = 1.0 - lower
  centers_min = np.quantile(points, lower, axis=0)
  centers_max = np.quantile(points, upper, axis=0)
  too_near = np.any(points < centers_min[None, :], axis=1)
  too_far = np.any(points > centers_max[None, :], axis=1)
  return points[~(too_near | too_far)]


def scene_points(points, cameras):
  """The notebook's point set for near/far and the scene box: the inlier points, then the camera
  positions (float32, promoted to float64)."""
  positions = np.stack([c.position for c in cameras])
  return np.concatenate([filter_outlier_points(np.asarray(points, np.float64)), positions], axis=0)


def _camera_table(cameras, device):
  structs = (_lib.NfbCamera * len(cameras))(*[c._struct() for c in cameras])
  raw = np.frombuffer(bytes(structs), np.uint8)
  return torch.from_numpy(raw.copy()).to(device)


def near_far_per_camera(cameras, points, device):
  """(near (C,), far (C,), counts (C,)) of each camera as the notebook's
  estimate_near_far_for_image computes them, for the float64 points (P, 3) given as they are (no
  outlier filter here).  One device call for all cameras; near and far are NaN where a camera
  sees no point."""
  device = torch.device(device)
  if device.type != 'cuda':
    raise ValueError('near_far_per_camera needs a CUDA device: nerfies_b200 has no CPU path')
  if not cameras:
    raise ValueError('no cameras')
  lib = _lib.load()
  pts = torch.as_tensor(np.ascontiguousarray(points, np.float64)).reshape(-1, 3).to(device)
  table = _camera_table(cameras, device)
  c = len(cameras)
  nbytes = int(lib.nfb_near_far_workspace_size(c))
  if nbytes < 0:
    raise _lib.NfbError(lib.nfb_last_error().decode())
  workspace = torch.empty(nbytes, dtype=torch.uint8, device=device)
  near = torch.empty(c, dtype=torch.float64, device=device)
  far = torch.empty(c, dtype=torch.float64, device=device)
  counts = torch.empty(c, dtype=torch.int64, device=device)
  with torch.cuda.device(device):
    _lib.check(lib.nfb_near_far(_ptr(table), c, _ptr(pts), pts.shape[0], NEAR_QUANTILE, FAR_QUANTILE,
                                _ptr(workspace), nbytes, _ptr(near), _ptr(far), _ptr(counts), _stream(device)))
  return near.cpu().numpy(), far.cpu().numpy(), counts.cpu().numpy()


def estimate_near_far(item_ids, cameras, points, device):
  """The notebook's near/far planes: per camera, the 0.001 and 0.999 depth quantiles of the inlier
  points and camera positions it sees; then near = quantile(near_i, 0.001) / 0.8 and
  far = quantile(far_i, 0.999) * 1.2.  Returns (near, far, {'near', 'far', 'counts'} per camera).
  A camera that sees no point raises ValueError naming its item."""
  near_i, far_i, counts = near_far_per_camera(cameras, scene_points(points, cameras), device)
  empty = [item_ids[i] for i in np.where(counts == 0)[0]]
  if empty:
    raise ValueError(f'no point projects into the frame of item(s) {", ".join(map(str, empty))}: '
                     'their near/far planes are undefined')
  near = np.quantile(near_i, NEAR_QUANTILE) / NEAR_MARGIN
  far = np.quantile(far_i, FAR_QUANTILE) * FAR_MARGIN
  return float(near), float(far), {'near': near_i, 'far': far_i, 'counts': counts}


def scene_info(points, cameras, near, far):
  """scene.json: the centre and scale of the bounding box of the inlier points and camera
  positions, and the near / far planes in the scaled scene."""
  allp = scene_points(points, cameras)
  bbox_corners = np.stack([allp.min(axis=0), allp.max(axis=0)])
  scene_center = np.mean(bbox_corners, axis=0)
  scene_scale = 1.0 / np.sqrt(np.sum((bbox_corners[1] - bbox_corners[0]) ** 2))
  return {'scale': float(scene_scale), 'center': scene_center.tolist(), 'bbox': bbox_corners.tolist(),
          'near': float(near * scene_scale), 'far': float(far * scene_scale)}


def triangulate_rays(origins, directions):
  """Least-squares intersection of rays (unit weights): the x minimising the summed squared
  distance to every line, sum_i (I - d_i d_i^T) x = sum_i (I - d_i d_i^T) o_i with unit d_i.  This
  is the formula of tensorflow_graphics.geometry.representation.ray.triangulate, which the notebook
  calls with endpoints o_i + d_i in float32."""
  origins = np.asarray(origins, np.float32)
  endpoints = origins + np.asarray(directions, np.float32)
  d = (endpoints - origins).astype(np.float64)
  d /= np.linalg.norm(d, axis=-1, keepdims=True)
  proj = np.eye(3)[None] - d[:, :, None] * d[:, None, :]
  return np.linalg.solve(proj.sum(0), np.einsum('nij,nj->i', proj, origins.astype(np.float64)))


def orbit_camera_path(cameras, num_frames=100, radius=0.75, x_scale=0.75, y_scale=0.75,
                      z_offset=ORBIT_Z_OFFSET):
  """The notebook's 'orbit-mild' path: cameras[0] copied to num_frames positions on an ellipse
  around the mean camera position, each looking at the point nearest every optical axis, with up
  the negated mean of the orientations' second columns."""
  origins = np.array([c.position for c in cameras])
  directions = np.array([c.optical_axis for c in cameras])
  look_at = triangulate_rays(origins, directions)
  avg_position = np.mean(origins, axis=0)
  up = -np.mean([c.orientation[..., 1] for c in cameras], axis=0)
  bounding_size = np.linalg.norm(origins.max(axis=0) - origins.min(axis=0)) / 2
  xs, ys = x_scale * bounding_size, y_scale * bounding_size
  path = []
  for angle in np.linspace(0, 2 * math.pi, num=num_frames):
    position = avg_position + np.array([np.cos(angle) * radius * xs, np.sin(angle) * radius * ys, z_offset])
    path.append(cameras[0].look_at(position, look_at, up))
  return path


def split_and_metadata(item_ids):
  """(dataset.json, metadata.json) of the notebook: every 20th sorted id is a val id; a val item
  takes the warp / appearance id of the train id it would be inserted before."""
  all_ids = sorted(item_ids)
  val_ids = all_ids[::VAL_STRIDE]
  train_ids = sorted(set(all_ids) - set(val_ids))
  dataset = {'count': len(all_ids), 'num_exemplars': len(train_ids), 'ids': all_ids, 'train_ids': train_ids,
             'val_ids': val_ids}
  metadata = {}
  for i, image_id in enumerate(train_ids):
    metadata[image_id] = {'warp_id': i, 'appearance_id': i, 'camera_id': 0}
  for image_id in val_ids:
    i = bisect.bisect_left(train_ids, image_id)
    metadata[image_id] = {'warp_id': i, 'appearance_id': i, 'camera_id': 0}
  return dataset, metadata


# ---- per-frame depth maps (process_capture depth) ----
MIN_DEPTH_SCALE_PAIRS = 32   # fewer (point, sensor depth) pairs than this: ask for --depth_scale


def resample_depth(sensor, camera, factor, device):
  """A sensor depth map onto one frame (nfb_depth_resample): `sensor` (src_h, src_w) float z-depth in sensor
  units (non-finite or <= 0 = missing), `camera` the frame's camera at the output scale, `factor` =
  metric_scale * scene scale.  Returns float32 (h, w) numpy on the host: the distance along each pixel
  centre's unit ray in scene units, NaN where nothing was measured."""
  src = torch.from_numpy(np.ascontiguousarray(sensor, np.float32)).to(device)
  h, w = camera.image_shape
  out = torch.empty(h, w, dtype=torch.float32, device=device)
  lib = _lib.load()
  with torch.cuda.device(device):
    _lib.check(lib.nfb_depth_resample(ctypes.byref(camera._struct()), _ptr(src), src.shape[0], src.shape[1],
                                      float(factor), _ptr(out), _stream(device)))
  return out.cpu().numpy()


def depth_scale_pairs(points, camera, sensor, device):
  """(camera z of each point, sensor depth at its pixel) for the points (N, 3) in world units that project
  inside the frame of `camera` (its capture camera, any scale; nfb_camera_project) in front of it and land
  where the four sensor pixels around them are all valid.  The sensor depth is interpolated bilinearly in
  inverse depth, which is exact on a plane seen by a pinhole.  Two float64 vectors."""
  pts = np.asarray(points, np.float32).reshape(-1, 3)
  if not len(pts):
    return np.zeros(0), np.zeros(0)
  pixels = camera.project(torch.from_numpy(pts).to(device)).cpu().double().numpy()
  z = (pts.astype(np.float64) - camera.position.astype(np.float64)) @ camera.orientation[2].astype(np.float64)
  w, h = (int(v) for v in camera.image_size)
  sh, sw = sensor.shape
  # sensor pixel coordinates, with the pixel centres at integers
  u = pixels[:, 0] * (sw / w) - 0.5
  v = pixels[:, 1] * (sh / h) - 0.5
  ok = (z > 0) & np.isfinite(u) & np.isfinite(v) & (u >= 0) & (v >= 0) & (u <= sw - 1) & (v <= sh - 1)
  u, v, z = u[ok], v[ok], z[ok]
  j0 = np.minimum(np.floor(u).astype(np.int64), max(sw - 2, 0))
  i0 = np.minimum(np.floor(v).astype(np.int64), max(sh - 2, 0))
  j1, i1 = np.minimum(j0 + 1, sw - 1), np.minimum(i0 + 1, sh - 1)
  fu, fv = u - j0, v - i0
  s = np.asarray(sensor, np.float64)
  corners = [s[i0, j0], s[i0, j1], s[i1, j0], s[i1, j1]]
  valid = np.all([np.isfinite(c) & (c > 0) for c in corners], axis=0)
  with np.errstate(divide='ignore', invalid='ignore'):
    inv = [1.0 / c for c in corners]
    inv_d = ((1 - fv) * ((1 - fu) * inv[0] + fu * inv[1]) + fv * ((1 - fu) * inv[2] + fu * inv[3]))
    depth = 1.0 / inv_d
  valid &= np.isfinite(depth) & (depth > 0)
  return z[valid], depth[valid]


def estimate_depth_scale(pairs, min_pairs=MIN_DEPTH_SCALE_PAIRS):
  """metric_scale (sensor units -> world units) from the (camera z, sensor depth) pairs of every frame: the
  median of z / sensor depth.  Returns (scale, number of pairs, interquartile range of the ratios); raises
  ValueError with fewer than `min_pairs` pairs."""
  z = np.concatenate([p[0] for p in pairs]) if pairs else np.zeros(0)
  d = np.concatenate([p[1] for p in pairs]) if pairs else np.zeros(0)
  if len(z) < min_pairs:
    raise ValueError(f'only {len(z)} COLMAP points meet a sensor depth (at least {min_pairs} are needed to '
                     'estimate the metric scale): pass --depth_scale')
  ratio = z / d
  q1, med, q3 = np.percentile(ratio, [25, 50, 75])
  return float(med), len(ratio), float(q3 - q1)
