"""The train_precision argument is checked on the host: models.construct_nerf / NerfModel accept 'fp32'
(the default) and 'tf32x3', independently of the render `precision`, and reject anything else with a
ValueError; the C entry points reject an unknown NFB_TRAIN_* value before touching a device."""
import pytest

import nerfies_b200 as nb
from nerfies_b200 import _lib


def _construct(**kw):
  cfg = nb.configs.ModelConfig(num_coarse_samples=8, num_fine_samples=8, use_warp=True, warp_field_type='se3')
  return nb.construct_nerf(0, cfg, 16, range(3), range(2), range(5), near=0.02, far=0.83, device='cpu', **kw)[0]


def test_default_is_fp32_and_independent_of_precision():
  assert _construct().train_precision == 'fp32'
  m = _construct(precision='bf16', train_precision='tf32x3')
  assert (m.precision, m.train_precision) == ('bf16', 'tf32x3')
  m.train_precision = 'fp32'
  assert (m.precision, m.train_precision) == ('bf16', 'fp32')


@pytest.mark.parametrize('bad', ['tf32', 'bf16', 'fp16x3', 'TF32X3', None, 1])
def test_unknown_train_precision_raises(bad):
  with pytest.raises(ValueError, match='train_precision'):
    _construct(train_precision=bad)
  m = _construct()
  with pytest.raises(ValueError, match='train_precision'):
    m.train_precision = bad
  assert m.train_precision == 'fp32'


def test_c_entry_points_reject_bad_values():
  lib = _lib.load()
  assert _lib.TRAIN_PRECISIONS == {'fp32': 0, 'tf32x3': 1}
  assert lib.nfb_set_train_precision(None, 1) != 0
  assert b'null handle' in lib.nfb_last_error()
  p = 16  # never dereferenced: the precision is checked first
  for bad in (-1, 2):
    assert lib.nfb_selftest_train_gemm(bad, 0, 4, 4, 4, 0, 1, p, 4, None, 0, p, 4, p, p, None, None, None, None, 0,
                                       None, None) != 0
    assert b'train precision' in lib.nfb_last_error()
