"""Generate tests/golden/colmap_small and tests/golden/capture_process.npz by running the capture
notebook's own cells.

TEST INFRASTRUCTURE.  Authoring container only (needs the reference checkout):

    python oracle/make_golden_capture.py

1. Synthesises a small scene: 17 frames of 84 x 68 pixels (not multiples of 8), each a smooth
   texture under its own Gaussian blur; 16 of them registered by an OPENCV camera (k1, k2, p1, p2)
   at 4x; points in a box, outliers beyond it, and tracks both shorter and longer than 5 images.
2. Writes the COLMAP model as sparse/0/{cameras,images,points3D}.bin (COLMAP's binary layout).
3. Executes the notebook's cells from notebooks/Nerfies_Capture_Processing.ipynb, read at
   generation time, from "Resize images into different scales" through "Save test cameras", with
   the shell lines dropped, the reference's third_party/pycolmap and nerfies.camera, the numpy
   shims of oracle/jaxshim, plotly, matplotlib and mediapipe (unused: use_face is False) stubbed, and tensorflow_graphics'
   ray.triangulate restated below.
4. Asserts that no projected point lies within 1e-6 px of a frame edge, so that the frustum test
   does not depend on the last bit of the projection.
"""
import json
import os
import pathlib
import shutil
import struct
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
REFERENCE = os.environ.get('NERFIES_REFERENCE', '/root/reference')
OUT = os.path.join(REPO, 'tests', 'golden', 'colmap_small')

W1, H1 = 84, 68              # 1x frame size; cropped to 80 x 64 by make_divisible(., 8)
COLMAP_SCALE = 4
NUM_FRAMES = 17              # frame 16 is not registered


def quat_from_rotation(R):
  w = 0.5 * np.sqrt(max(1e-12, 1.0 + np.trace(R)))
  return np.array([w, (R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w)])


def rotation_from_quat(q):
  w, x, y, z = q / np.linalg.norm(q)
  return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                   [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                   [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def synthesize(rng):
  from scipy import ndimage
  frames = []
  for i in range(NUM_FRAMES):
    noise = rng.uniform(0, 255, size=(H1, W1, 3))
    smooth = ndimage.gaussian_filter(noise, sigma=(2.0, 2.0, 0))
    smooth = (smooth - smooth.mean()) * 4 + 128
    blurred = ndimage.gaussian_filter(smooth, sigma=(0.4 + 0.13 * i, 0.4 + 0.13 * i, 0))
    frames.append(np.clip(np.round(blurred), 0, 255).astype(np.uint8))
  # poses: on an arc at distance ~4 looking at the origin (world-to-camera rotations)
  poses = []
  for i in range(NUM_FRAMES - 1):
    a = -0.5 + i / (NUM_FRAMES - 2)
    c = np.array([4 * np.sin(a), 0.3 * np.cos(3 * a), -4 * np.cos(a)]) + rng.normal(size=3) * 0.05
    z = -c / np.linalg.norm(c)
    x = np.cross([0, -1, 0], z); x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = rotation_from_quat(quat_from_rotation(np.stack([x, y, z])))
    q = quat_from_rotation(R)
    R = rotation_from_quat(q)
    poses.append((q, -R @ c))
  inliers = rng.uniform(-1, 1, size=(600, 3)) * np.array([1.0, 0.8, 1.0])
  outliers = rng.normal(size=(24, 3)) * 6
  points = np.concatenate([inliers, outliers])[rng.permutation(624)]
  return frames, poses, points


def write_model(model_dir, poses, points, rng):
  os.makedirs(model_dir, exist_ok=True)
  # COLMAP sees the 4x frames, which make_divisible cropped before downsampling
  w, h = (W1 - W1 % 8) // COLMAP_SCALE, (H1 - H1 % 8) // COLMAP_SCALE
  params = [18.0, 18.3, w / 2 + 0.3, h / 2 - 0.2, 0.04, -0.03, 1.5e-3, -8e-4]   # fx fy cx cy k1 k2 p1 p2
  with open(os.path.join(model_dir, 'cameras.bin'), 'wb') as f:
    f.write(struct.pack('<Q', 1))
    f.write(struct.pack('<IiQQ', 1, 4, w, h) + struct.pack('<8d', *params))
  image_ids = [10 + 3 * i for i in range(len(poses))]                 # COLMAP ids are arbitrary
  order = rng.permutation(len(poses))
  with open(os.path.join(model_dir, 'images.bin'), 'wb') as f:
    f.write(struct.pack('<Q', len(poses)))
    for i in order:
      q, t = poses[i]
      f.write(struct.pack('<I4d3dI', image_ids[i], *q, *t, 1))
      f.write(f'{i:06d}.png'.encode() + b'\0')
      f.write(struct.pack('<Q', 2) + struct.pack('<ddq', 1.0, 2.0, -1) + struct.pack('<ddq', 3.0, 4.0, -1))
  lengths = []
  with open(os.path.join(model_dir, 'points3D.bin'), 'wb') as f:
    f.write(struct.pack('<Q', len(points)))
    for k, p in enumerate(points):
      n = int(rng.randint(2, 9))                                        # distinct images in the track
      ids = list(rng.choice(image_ids, size=n, replace=False))
      ids += ids[:int(rng.randint(0, 3))]                               # repeated images count once
      lengths.append(n)
      f.write(struct.pack('<Q3d3Bd', 1000 + 7 * k, *p, 1, 2, 3, 0.5))
      f.write(struct.pack('<Q', len(ids)) + b''.join(struct.pack('<II', i, j) for j, i in enumerate(ids)))
  return np.array(lengths)


def ray_triangulate(startpoints, endpoints, weights):
  """tensorflow_graphics.geometry.representation.ray.triangulate: the least-squares point of
  weighted lines, solving sum_i w_i (I - d_i d_i^T) x = sum_i w_i (I - d_i d_i^T) s_i with
  d_i = normalize(e_i - s_i)."""
  s = np.asarray(startpoints, np.float64)
  d = np.asarray(endpoints, np.float64) - s
  d /= np.linalg.norm(d, axis=-1, keepdims=True)
  proj = np.eye(3) - d[..., :, None] * d[..., None, :]
  wp = np.asarray(weights)[..., None, None] * proj
  b = np.einsum('...nij,...nj->...i', wp, s)
  return np.linalg.solve(wp.sum(-3), b[..., None])[..., 0].astype(np.float32)


def install_stubs():
  sys.path.insert(0, os.path.join(HERE, 'jaxshim'))
  sys.path.insert(0, REFERENCE)
  sys.path.insert(0, os.path.join(REFERENCE, 'third_party', 'pycolmap'))
  # pycolmap defines INVALID_POINT3D = np.uint64(-1), which numpy 2 rejects: give it the wrapped value.
  import scipy.optimize  # noqa: F401  (pycolmap's import, made before the patch)
  uint64 = np.uint64
  np.uint64 = lambda v=0: uint64(v % (1 << 64)) if isinstance(v, int) else uint64(v)
  import pycolmap  # noqa: F401
  np.uint64 = uint64
  from PIL import Image
  imageio = types.ModuleType('imageio')
  imageio.imread = lambda f: np.asarray(Image.open(f))
  sys.modules['imageio'] = imageio
  anything = type('Anything', (), {'__getattr__': lambda self, k: self, '__call__': lambda self, *a, **k: self})()
  for name in ('plotly', 'plotly.graph_objs', 'plotly.offline', 'matplotlib', 'matplotlib.pyplot', 'mediapipe'):
    m = types.ModuleType(name)
    m.__getattr__ = lambda k: anything
    sys.modules[name] = m
  for name in ('tensorflow_graphics', 'tensorflow_graphics.geometry', 'tensorflow_graphics.geometry.representation',
               'tensorflow_graphics.geometry.representation.ray'):
    sys.modules[name] = types.ModuleType(name)
  sys.modules['tensorflow_graphics.geometry.representation.ray'].triangulate = ray_triangulate


def notebook_cells():
  nb = json.load(open(os.path.join(REFERENCE, 'notebooks', 'Nerfies_Capture_Processing.ipynb')))
  cells = [''.join(c['source']) for c in nb['cells'] if c['cell_type'] == 'code']
  first = next(i for i, c in enumerate(cells) if 'Resize images into different scales' in c)
  last = next(i for i, c in enumerate(cells) if 'Save test cameras' in c)
  keep = []
  for c in cells[first:last + 1]:
    if 'Example frame' in c:
      continue
    if any(k in c for k in ('Extract features', 'Match features', '# @title Reconstruction', 'Verify that SfM')):
      continue
    keep.append('\n'.join(line for line in c.split('\n') if not line.lstrip().startswith('!')))
  return keep


def main():
  rng = np.random.RandomState(20261017)
  frames, poses, points = synthesize(rng)
  if os.path.exists(OUT):
    shutil.rmtree(OUT)
  import cv2
  os.makedirs(os.path.join(OUT, 'frames'))
  for i, f in enumerate(frames):
    cv2.imwrite(os.path.join(OUT, 'frames', f'{i:06d}.png'), f[:, :, ::-1])
  write_model(os.path.join(OUT, 'sparse', '0'), poses, points, rng)

  install_stubs()
  work = pathlib.Path(tempfile.mkdtemp())
  cwd = os.getcwd()
  os.chdir(work)
  try:
    shutil.copytree(os.path.join(OUT, 'frames'), 'rgb-raw')
    root = work / 'capture'
    g = {'__name__': '__notebook__', 'Path': pathlib.Path, 'root_dir': root, 'rgb_dir': work / 'rgb',
         'tmp_rgb_raw_dir': 'rgb-raw', 'colmap_dir': work / 'colmap', 'colmap_image_scale': COLMAP_SCALE}
    os.makedirs(work / 'colmap' / 'sparse')
    shutil.copytree(os.path.join(OUT, 'sparse', '0'), work / 'colmap' / 'sparse' / '0')
    root.mkdir()
    for cell in notebook_cells():
      exec(compile(cell, '<notebook>', 'exec'), g)
    # edge margin of every projection the near/far step made
    sm = g['new_scene_manager']
    pts = np.concatenate([g['filter_outlier_points'](sm.points, 0.95), sm.camera_positions])
    counts, per_near, per_far = [], [], []
    for item in sm.image_ids:
      cam = sm.camera_dict[item]
      px = cam.project(pts)
      margin = np.nanmin(np.abs(np.concatenate([px[:, 0], px[:, 0] - cam.image_size_x, px[:, 1],
                                             px[:, 1] - cam.image_size_y])))
      assert margin > 1e-6, (item, margin)
      near, far = g['estimate_near_far_for_image'](sm, item)
      d = cam.points_to_local_points(pts)[..., 2]
      inside = (px[:, 0] >= 0) & (px[:, 0] <= cam.image_size_x) & (px[:, 1] >= 0) & (px[:, 1] <= cam.image_size_y)
      counts.append(int(((d > 0) & inside).sum()))
      per_near.append(near)
      per_far.append(far)
    expected = pathlib.Path(OUT) / 'expected'
    shutil.copytree(root, expected)
    shutil.copytree(work / 'rgb', expected / 'rgb')
    blur_ids = sorted(g['scene_manager'].image_ids + list(g['blur_filter_image_ids']))
    np.savez_compressed(
        os.path.join(REPO, 'tests', 'golden', 'capture_process.npz'),
        blur_ids=np.array(blur_ids), blur_scores=np.asarray(g['blur_scores'], np.float64),
        removed_ids=np.array(g['blur_filter_image_ids']), item_ids=np.array(sm.image_ids),
        near_i=np.array(per_near), far_i=np.array(per_far), counts=np.array(counts),
        near=np.float64(g['near']), far=np.float64(g['far']), points=np.asarray(sm.points, np.float64),
        look_at=np.asarray(g['look_at'], np.float64))
    print('removed', list(g['blur_filter_image_ids']), 'near', g['near'], 'far', g['far'], 'counts', counts)
  finally:
    os.chdir(cwd)
    shutil.rmtree(work)


if __name__ == '__main__':
  main()
