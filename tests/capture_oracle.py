"""numpy statement of the capture notebook's pixel steps (DESIGN.md §5.5d), held to cv2 in
tests/test_capture.py and used as the reference of the GPU kernels."""
import numpy as np


def make_divisible(image, divisor):
  h, w = image.shape[:2]
  return image[:h - h % divisor, :w - w % divisor]


def downsample(image, scale):
  """cv2.resize(image, (w // s, h // s)) with its default INTER_LINEAR, uint8, s = 1 or even."""
  if scale == 1:
    return image
  o = scale // 2 - 1
  a = image[o::scale, o::scale].astype(np.int32)
  b = image[o::scale, o + 1::scale].astype(np.int32)
  c = image[o + 1::scale, o::scale].astype(np.int32)
  d = image[o + 1::scale, o + 1::scale].astype(np.int32)
  return ((a + b + c + d + 2) >> 2).astype(np.uint8)


def grey(rgb):
  """cv2.cvtColor(rgb, COLOR_RGB2GRAY) for uint8: 15-bit fixed point."""
  rgb = rgb.astype(np.int64)
  return ((9798 * rgb[..., 0] + 19235 * rgb[..., 1] + 3735 * rgb[..., 2] + 16384) >> 15).astype(np.uint8)


def laplacian(g):
  """cv2.Laplacian(g, CV_64F) (ksize 1, BORDER_REFLECT_101) as int64."""
  p = np.pad(g.astype(np.int64), 1, mode='reflect')
  return p[:-2, 1:-1] + p[2:, 1:-1] + p[1:-1, :-2] + p[1:-1, 2:] - 4 * p[1:-1, 1:-1]


def blur_score(rgb):
  return float(laplacian(grey(rgb)).astype(np.float64).var())
