"""numpy statement of the reference's image conversions, written from their definitions
(image_utils.py:114-131, 172-174): the yardstick of nfb_image_quantize."""
import numpy as np

# products that land just below an integer (the cast truncates), the ends of the range, values
# outside it and the non-finite values
SPECIALS = np.array([0.0, -0.0, 1.0, np.nextafter(np.float32(0), np.float32(1)), np.nextafter(np.float32(0), np.float32(-1)),
                     np.nextafter(np.float32(1), np.float32(0)), np.nextafter(np.float32(1), np.float32(2)),
                     0.999, 0.5, 1.0 / 255.0, 254.0 / 255.0, 0.00392, 0.99999, -1e-9, -3.0, 2.0, 1e30, -1e30,
                     np.nan, -np.nan, np.inf, -np.inf], np.float32)


def image_to_uint8(image):
  assert image.dtype == np.float32
  with np.errstate(invalid='ignore'):
    return (image * 255).clip(0.0, 255).astype(np.uint8)


def image_to_uint16(image):
  assert image.dtype == np.float32
  with np.errstate(invalid='ignore'):
    return (image * 65535).clip(0.0, 65535).astype(np.uint16)


def depth_to_uint16(depth):
  """save_depth: image_to_uint16(depth / 1000.0)."""
  assert depth.dtype == np.float32
  return image_to_uint16(depth / 1000.0)
