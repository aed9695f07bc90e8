"""numpy statement of the reference's visualization.colorize (visualization.py:177-219),
image_utils.image_to_uint8 (image_utils.py:114-121) and the render-video notebook's frame, written
from their definitions with every precision explicit (numpy 2, NEP 50): the yardstick of
nfb_colorize.  tests/golden/viz_turbo.npz, recorded from the reference's own source, pins it."""
import numpy as np

f32 = np.float32


def source_values(a, source='value', b=None):
  """The float32 value colorize maps: a, 1 / a, or eval.py:129-132's error sums ((e0 + e1) + e2)."""
  a = np.asarray(a, f32)
  with np.errstate(divide='ignore', invalid='ignore'):
    if source == 'value':
      return a
    if source == 'reciprocal':
      return (f32(1) / a).astype(f32)
    d = a - np.asarray(b, f32)
    e = np.abs(d) if source == 'abs_error' else d * d
    return (e[..., 0] + e[..., 1]) + e[..., 2]


def colorize(values, table, cmin=None, cmax=None, eps=1e-6, invert=False):
  """float64 (..., 3).  Bounds are Python numbers or None (the frame's min / max, float32)."""
  v = np.asarray(values, f32)
  table = np.asarray(table, np.float64)
  with np.errstate(invalid='ignore', over='ignore'):
    if cmin is not None and cmax is not None:
      lo, d = f32(cmin), f32(max(cmax - cmin, eps))                 # float64 subtraction, then float32
    else:
      lo = f32(np.min(v)) if cmin is None else f32(cmin)
      hi = f32(np.max(v)) if cmax is None else f32(cmax)
      diff = f32(hi - lo)
      d = f32(eps) if f32(eps) > diff else diff
    x = ((v - lo) / d).astype(f32)
    y = (f32(1) - x) if invert else x
    t = (y * f32(255)).astype(f32)
    a = np.floor(t)
    f = (t - a).astype(f32).astype(np.float64)
    ia = np.where(np.isnan(a), 0, np.clip(np.nan_to_num(a), 0, 255)).astype(np.int64)
    ib = np.minimum(ia + 1, 255)
    out = table[ia] + (table[ib] - table[ia]) * f[..., None]
  out[x > 1] = 0.0 if invert else 1.0
  out[x < 0] = 1.0 if invert else 0.0
  return out


def to_uint8(image):
  """image_to_uint8 of a float64 image: float64 product, clip, truncation; NaN -> 0."""
  with np.errstate(invalid='ignore'):
    return (np.asarray(image, np.float64) * 255).clip(0.0, 255).astype(np.uint8)


def video_frame(rgb, depth, table, near, far):
  """image_to_uint8(np.concatenate([rgb, colorize(depth, near, far, invert=True)], axis=1))."""
  return to_uint8(np.concatenate([np.asarray(rgb, f32).astype(np.float64),
                                  colorize(depth, table, near, far, invert=True)], axis=1))
