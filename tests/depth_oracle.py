"""Synthetic sensor depth for the depth tests: one world plane seen by the cameras of a capture, in float64
through the numpy reference camera (oracle/camera_oracle.py), and the resampling rule of nfb_depth_resample
restated in numpy.

TEST INFRASTRUCTURE: imported by tests/test_depth*.py only.
"""
import json
import math
import pathlib

import numpy as np

from oracle import camera_oracle as C

# The world plane n . X = c (COLMAP world units) of every synthetic map: the rays of each capture_small camera
# that meet it in front of the camera see it; the others measure nothing.
PLANE_N = np.array([0.6, -0.48, 0.64]) / np.linalg.norm([0.6, -0.48, 0.64])
PLANE_C = 1.1
# the sensor's range in world units: farther (grazing) measurements are missing, as past a LiDAR's range
Z_MAX = 8.0


def load_camera(capture, item_id):
  """The item's capture camera (1x, world units) as an oracle camera dict."""
  j = json.loads((pathlib.Path(capture) / 'camera' / f'{item_id}.json').read_text())
  return C.make_camera(j['orientation'], j['position'], j['focal_length'], j['principal_point'], j['image_size'],
                       j['skew'], j['pixel_aspect_ratio'], j['radial_distortion'], j['tangential_distortion'])


def ray_distance(cam, pixels):
  """Distance along the unit ray of `cam` (1x) at float pixel positions (..., 2) to the plane, in world units;
  NaN where the ray does not meet the plane in front of the camera.  Also returns the rays' unit directions."""
  d = C.pixels_to_rays(cam, np.asarray(pixels, np.float32)).astype(np.float64)
  o = cam['position'].astype(np.float64)
  den = d @ PLANE_N
  with np.errstate(divide='ignore', invalid='ignore'):
    t = (PLANE_C - o @ PLANE_N) / den
  t = np.where(np.isfinite(t) & (t > 0), t, np.nan)
  return t, d


def sensor_map(cam, src_h, src_w, metric_scale):
  """A (src_h, src_w) z-depth map in sensor units of the plane: the sensor shares the camera's view, its pixel
  centres are at 1x positions ((j + 0.5) W / src_w, (i + 0.5) H / src_h).  Missing pixels are 0."""
  w1, h1 = int(cam['image_size'][0]), int(cam['image_size'][1])
  jj, ii = np.meshgrid(np.arange(src_w) + 0.5, np.arange(src_h) + 0.5)
  px = np.stack([jj * (w1 / src_w), ii * (h1 / src_h)], axis=-1)
  t, d = ray_distance(cam, px)
  z = t * (d @ cam['orientation'][2].astype(np.float64))
  return np.where(np.isfinite(z) & (z < Z_MAX), z / metric_scale, 0.0)


def valid(z):
  return np.isfinite(z) & (z > 0)


def resample_rule(cam_s, src, factor):
  """nfb_depth_resample restated in float64: cam_s the frame's oracle camera at the output scale."""
  w, h = int(cam_s['image_size'][0]), int(cam_s['image_size'][1])
  src_h, src_w = src.shape
  sx, sy = src_w / w, src_h / h
  ok = valid(src)
  zs = np.full((h, w), np.nan)
  for y in range(h):
    i0, i1 = max(0, math.ceil(y * sy - 0.5)), min(src_h, math.ceil((y + 1) * sy - 0.5))
    for x in range(w):
      j0, j1 = max(0, math.ceil(x * sx - 0.5)), min(src_w, math.ceil((x + 1) * sx - 0.5))
      block, m = src[i0:i1, j0:j1], ok[i0:i1, j0:j1]
      if m.any():
        zs[y, x] = block[m].mean()
      else:
        ic, jc = min(src_h - 1, math.floor((y + 0.5) * sy)), min(src_w - 1, math.floor((x + 0.5) * sx))
        if ok[ic, jc]:
          zs[y, x] = src[ic, jc]
  d = C.camera_to_rays(cam_s)['directions'].astype(np.float64)
  cos_axis = d @ cam_s['orientation'][2].astype(np.float64)
  return zs / cos_axis * factor


def scaled(cam, s):
  """The oracle camera for the image resized by 1 / s (Camera.scale)."""
  out = dict(cam)
  out['focal_length'] = np.float32(cam['focal_length'] / np.float32(s))
  out['principal_point'] = (cam['principal_point'] / np.float32(s)).astype(np.float32)
  out['image_size'] = np.array([int(round(float(n) / s)) for n in cam['image_size']], np.uint32)
  return out


def plane_points(capture, item_ids, per_camera, seed=0):
  """World points on the plane (float32 (N, 3)): the plane points of random pixel rays of each camera."""
  rng = np.random.RandomState(seed)
  pts = []
  for i in item_ids:
    cam = load_camera(capture, i)
    w1, h1 = int(cam['image_size'][0]), int(cam['image_size'][1])
    px = np.stack([rng.uniform(2, w1 - 2, per_camera), rng.uniform(2, h1 - 2, per_camera)], axis=-1)
    t, d = ray_distance(cam, px)
    keep = np.isfinite(t) & (t < Z_MAX)
    pts.append(cam['position'].astype(np.float64) + t[keep, None] * d[keep])
  return np.concatenate(pts).astype(np.float32)


def footprint_z_range(cam, src_hw, out_hw, n=9):
  """Per output pixel of an (h, w) = out_hw frame, the least and greatest analytic z-depth (world units) of the
  plane over the pixel's footprint widened by half a source pixel on each side, in the 1x frame of `cam`, from an
  n x n grid that includes the corners.  The resampler's value must lie in that range: a mean over the source
  centres inside the footprint is a convex combination of values there, and the source pixel containing the
  output centre has its centre within half a source pixel of it.  This holds for any correct footprint rule and
  needs no restatement of the kernel's.  NaN where the region is not all seen within the sensor's range."""
  w1, h1 = int(cam['image_size'][0]), int(cam['image_size'][1])
  (src_h, src_w), (h, w) = src_hw, out_hw
  hx, hy = 0.5 * w1 / src_w, 0.5 * h1 / src_h
  x0 = np.clip(np.arange(w) * (w1 / w) - hx, 0, w1)
  x1 = np.clip((np.arange(w) + 1) * (w1 / w) + hx, 0, w1)
  y0 = np.clip(np.arange(h) * (h1 / h) - hy, 0, h1)
  y1 = np.clip((np.arange(h) + 1) * (h1 / h) + hy, 0, h1)
  f = np.linspace(0, 1, n)
  xs = x0[:, None] + f[None, :] * (x1 - x0)[:, None]            # (w, n)
  ys = y0[:, None] + f[None, :] * (y1 - y0)[:, None]            # (h, n)
  px = np.broadcast_to(xs[None, :, None, :], (h, w, n, n))
  py = np.broadcast_to(ys[:, None, :, None], (h, w, n, n))
  t, d = ray_distance(cam, np.stack([px, py], axis=-1).reshape(-1, 2))
  z = (t * (d @ cam['orientation'][2].astype(np.float64))).reshape(h, w, n * n)
  z = np.where(z < Z_MAX, z, np.nan)
  return z.min(axis=-1), z.max(axis=-1)
