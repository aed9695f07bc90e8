"""Generate tests/golden/viz_turbo.npz by executing the reference's own visualization.colorize.

TEST INFRASTRUCTURE.  Authoring container only (needs /root/reference):

    python oracle/make_golden_viz.py

nerfies/visualization.py is imported unmodified.  Its matplotlib imports get import-only stubs:
the turbo table is a literal of that file and its path through colorize never calls matplotlib.
image_utils.image_to_uint8 runs on the jaxshim.  The fixture stores the turbo table, inputs with
the special values of every stage (0, 1, the k/255 bin edges and their neighbours, values just
outside [0, 1], +-inf, NaN, depth 0 under the reciprocal) and colorize's float64 outputs, each
with its uint8 conversion, for:
  * given bounds (Python floats: fp64 subtraction; ints) and bounds from the frame (fp32),
    invert off and on;
  * eval.py:87-96's depth, disparity and accumulation images;
  * eval.py:129-132's rgb error maps;
  * the render-video notebook's frame, image_to_uint8(concatenate([rgb, depth_viz], 1)), whose rgb
    half holds every bin edge k / 255 and its float32 neighbours.
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
REFERENCE = os.environ.get('NERFIES_REFERENCE', '/root/reference')
sys.path.insert(0, os.path.join(HERE, 'jaxshim'))
sys.path.insert(0, REFERENCE)


def _stub_matplotlib():
  mpl, cm, colors = (types.ModuleType(n) for n in ('matplotlib', 'matplotlib.cm', 'matplotlib.colors'))

  def unavailable(*args, **kwargs):
    raise RuntimeError('matplotlib is not installed: only the turbo table is available')
  cm.get_cmap = unavailable
  colors.LinearSegmentedColormap = types.SimpleNamespace(from_list=unavailable)
  mpl.cm, mpl.colors = cm, colors
  sys.modules.update({'matplotlib': mpl, 'matplotlib.cm': cm, 'matplotlib.colors': colors})


_stub_matplotlib()
from nerfies import image_utils  # noqa: E402  (the reference)
from nerfies import visualization as viz  # noqa: E402  (the reference)

H, W = 27, 48
NEAR, FAR = 0.1, 2.5          # Python floats, as eval.py passes datasource.near / far


def _specials():
  """Values of x = (v - 0) / 1 at every stage boundary of colorize."""
  f32 = np.float32
  k = np.arange(256, dtype=np.float64)
  edges = (k / 255.0).astype(f32)
  v = [edges, np.nextafter(edges, f32(-1)), np.nextafter(edges, f32(2)),
       f32([0.0, -0.0, 1.0, 0.5, 1e-7, 1e-30, 1e-45, -1e-45, 1.0 - 2**-24, 1.0 + 2**-23, -2**-24, 1.5, -0.5,
            1e30, -1e30, np.inf, -np.inf, np.nan])]
  return np.concatenate(v).astype(f32)


def _frame(values, rng, lo, hi):
  """An (H, W) float32 frame: `values` first, uniform draws in [lo, hi) after them."""
  out = rng.uniform(lo, hi, H * W).astype(np.float32)
  out[:len(values)] = values
  return out.reshape(H, W)


def main():
  rng = np.random.RandomState(11)
  table = np.asarray(viz.get_colormap('turbo'), np.float64)
  colorize = lambda a, **kw: viz.colorize(a, cmap='turbo', **kw)
  to_u8 = image_utils.image_to_uint8
  specials = _specials()
  out = {'table': table, 'near': np.float64(NEAR), 'far': np.float64(FAR)}

  # x in and around [0, 1] with every special value; given bounds as Python floats and as ints
  unit = _frame(specials, rng, -0.1, 1.1)
  out['unit'] = unit
  for name, kw in {'unit_given': dict(cmin=0.0, cmax=1.0), 'unit_int': dict(cmin=0, cmax=1)}.items():
    for inv in (False, True):
      out[f'{name}_inv{int(inv)}'] = colorize(unit, invert=inv, **kw)
  # bounds from the frame: finite values, and the frame with its NaN (every colour NaN -> 0)
  finite = np.where(np.isfinite(unit), unit, np.float32(0.25)).astype(np.float32)
  out['finite'] = finite
  for inv in (False, True):
    out[f'finite_frame_inv{int(inv)}'] = colorize(finite, invert=inv)
    out[f'finite_min_inv{int(inv)}'] = colorize(finite, cmax=0.75, invert=inv)     # one bound from the frame
  out['unit_frame_inv0'] = colorize(unit)
  # a flat frame: cmax - cmin = 0 < eps
  out['flat'] = np.full((3, 5), 0.3, np.float32)
  out['flat_frame_inv0'] = colorize(out['flat'])

  # eval.py:87-96 on a depth frame with zeros and values outside [near, far]
  depth = _frame((NEAR + specials[np.isfinite(specials)] * (FAR - NEAR)).astype(np.float32), rng, 0.0, 3.0)
  depth[0, :4] = [0.0, -0.0, NEAR, FAR]
  acc = _frame(specials, rng, 0.0, 1.0)
  out.update(depth=depth, acc=acc)
  out['depth_viz'] = colorize(depth, cmin=NEAR, cmax=FAR, invert=True)
  out['disp_viz'] = colorize(1.0 / depth)                                        # inf at depth 0: NaN -> black
  positive = np.abs(depth) + np.float32(0.05)
  out['positive_depth'] = positive
  out['disp_positive_viz'] = colorize(1.0 / positive)
  out['acc_viz'] = colorize(acc, cmin=0.0, cmax=1.0)

  # eval.py:129-132
  rgb = rng.uniform(0, 1, (H, W, 3)).astype(np.float32)
  target = np.clip(rgb + rng.normal(0, 0.3, (H, W, 3)), 0, 1).astype(np.float32)
  target[0, 0] = rgb[0, 0]
  out.update(rgb=rgb, target=target)
  out['abs_error_viz'] = colorize(abs(target - rgb).sum(axis=-1), cmin=0, cmax=1)
  out['sq_error_viz'] = colorize(((target - rgb)**2).sum(axis=-1), cmin=0, cmax=1)

  # the render-video notebook's frame (concatenate promotes rgb to float64 before the product)
  video_rgb = rgb.copy()
  edges = (np.arange(256) / 255.0).astype(np.float32)
  near_edges = np.concatenate([edges, np.nextafter(edges, np.float32(0)), np.nextafter(edges, np.float32(1))])
  video_rgb.reshape(-1)[:len(near_edges)] = near_edges
  out['video_rgb'] = video_rgb
  out['video_frame'] = to_u8(np.concatenate([video_rgb, colorize(depth, cmin=NEAR, cmax=FAR, invert=True)], axis=1))

  for key in [k for k in out if k.endswith('_viz') or '_inv' in k]:
    out[key + '_u8'] = to_u8(out[key])
  path = os.path.join(REPO, 'tests', 'golden', 'viz_turbo.npz')
  np.savez_compressed(path, **out)
  print(path, len(out), 'arrays')


if __name__ == '__main__':
  main()
