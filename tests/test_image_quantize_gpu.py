"""nfb_image_quantize against the numpy statement of image_utils.image_to_uint8 / image_to_uint16 /
save_depth (tests/image_oracle.py): exact equality, on the vector path, on pointers that break
16-byte alignment, and for n = 0 and n = 1."""
import ctypes

import numpy as np
import pytest
import torch

from tests import image_oracle

pytestmark = pytest.mark.gpu


def _values(n, seed):
  rng = np.random.RandomState(seed)
  x = rng.uniform(-0.25, 1.25, n).astype(np.float32)
  k = rng.randint(0, 65536, n // 4)                      # products that land on and next to integers
  x[:n // 4] = (k / 65535.0).astype(np.float32)
  x[n // 4:n // 2] = (rng.randint(0, 256, n // 2 - n // 4) / 255.0).astype(np.float32)
  s = image_oracle.SPECIALS
  x[-len(s):] = s                                        # in the scalar tail
  x[1000:1000 + len(s)] = s                              # in the vector body
  return x


@pytest.mark.parametrize('bits', [8, 16])
def test_image_quantize_equals_numpy(bits):
  from nerfies_b200 import evaluation
  n = 2**20 + 3
  x = _values(n, bits)
  dev = torch.device('cuda', 0)
  xd = torch.from_numpy(x).to(dev)
  fn, oracle = ((evaluation.image_to_uint8, image_oracle.image_to_uint8) if bits == 8
                else (evaluation.image_to_uint16, image_oracle.image_to_uint16))
  out = fn(xd)
  assert out.dtype == (torch.uint8 if bits == 8 else torch.uint16) and out.shape == xd.shape
  np.testing.assert_array_equal(out.cpu().numpy(), oracle(x))
  # shapes are kept; n = 0 and n = 1
  assert fn(xd[:12].reshape(2, 2, 3)).shape == (2, 2, 3)
  assert fn(xd[:0]).numel() == 0
  for v in (0.999, float('nan'), 2.0):
    one = np.array([v], np.float32)
    np.testing.assert_array_equal(fn(torch.from_numpy(one).to(dev)).cpu().numpy(), oracle(one))
  if bits == 16:
    d = (x * 1500.0).astype(np.float32)
    np.testing.assert_array_equal(evaluation.depth_to_uint16(torch.from_numpy(d).to(dev)).cpu().numpy(),
                                  image_oracle.depth_to_uint16(d))


@pytest.mark.parametrize('bits', [8, 16])
@pytest.mark.parametrize('src_off, dst_off', [(1, 0), (0, 1), (3, 5), (2, 2)])
def test_image_quantize_on_unaligned_pointers(bits, src_off, dst_off):
  """Offsets in elements: src at 4 * src_off bytes, dst at dst_off * (bits / 8) bytes past a
  16-byte boundary.  The bytes around the output must stay untouched."""
  from nerfies_b200 import _lib
  lib = _lib.load()
  n = 4099
  x = _values(n + 8, 3)
  dev = torch.device('cuda', 0)
  src = torch.from_numpy(x).to(dev)
  dtype, np_dtype = (torch.uint8, np.uint8) if bits == 8 else (torch.uint16, np.uint16)
  dst = torch.from_numpy(np.full(n + 16, 77, np_dtype)).to(dev)
  _lib.check(lib.nfb_image_quantize(
      ctypes.c_void_p(src.data_ptr() + 4 * src_off), n, bits, 1.0,
      ctypes.c_void_p(dst.data_ptr() + dst_off * (bits // 8)), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
  got = dst.cpu().numpy()
  oracle = image_oracle.image_to_uint8 if bits == 8 else image_oracle.image_to_uint16
  np.testing.assert_array_equal(got[dst_off:dst_off + n], oracle(x[src_off:src_off + n]))
  assert (got[:dst_off] == 77).all() and (got[dst_off + n:] == 77).all()
  assert dst.dtype == dtype
