"""Per-frame metrics of eval.py:process_batch without a GPU: the MS-SSIM oracle pinned by
closed-form known answers, compute_psnr, the Python argument checks and the C ABI's workspace
query (the library loads without a device)."""
import ctypes
import math

import numpy as np
import pytest
import torch

from nerfies_b200 import _lib, evaluation
from tests import metrics_oracle as M

C1, C2 = 0.01 ** 2, 0.03 ** 2


def _noise(seed, shape):
  return np.random.default_rng(seed).random(shape, dtype=np.float32)


@pytest.mark.parametrize('dtype', [np.float64, np.float32])
def test_identical_images_give_exactly_one(dtype):
  x = _noise(0, (2, 177, 181, 3))
  np.testing.assert_array_equal(M.ms_ssim(x, x, dtype), np.ones(2))


def test_constant_images_closed_form():
  # cs = 1 at every scale, so only the scale-4 luminance remains, raised to its power factor.
  a, b = 0.3, 0.7
  want = ((2 * a * b + C1) / (a * a + b * b + C1)) ** 0.1333
  assert abs(want - 0.95789516) < 1e-8
  got = M.ms_ssim(np.full((165, 170, 3), a), np.full((165, 170, 3), b))
  assert abs(float(got) - want) < 1e-12


def test_fp32_tf_order_loses_accuracy_on_flat_images():
  """In float32, cs of a flat region is F(xy) - F(x)F(y) over c2 = 9e-4: TF's own operation order
  lands ~1e-4 from the exact value (the reason the kernel shifts each tile first)."""
  got = float(M.ms_ssim(np.full((165, 170, 1), 0.3), np.full((165, 170, 1), 0.7), np.float32))
  assert 1e-5 < abs(got - 0.9578951635219879) < 1e-3


def test_gaussian_is_separable():
  g1 = M.gauss_1d()
  np.testing.assert_allclose(M.fspecial_gauss(), np.outer(g1, g1), rtol=0, atol=1e-15)
  assert abs(g1.sum() - 1.0) < 1e-15 and abs(g1[5] - 0.26601172) < 1e-8   # cv2.getGaussianKernel(11, 1.5)


def test_level_sizes_of_odd_shapes():
  assert M.level_sizes(177, 181) == [(177, 181), (89, 91), (45, 46), (23, 23), (12, 12)]
  assert M.level_sizes(161, 161)[-1] == (11, 11)
  assert M.level_sizes(160, 200)[-1] == (10, 13)


def test_symmetric_pad_repeats_the_edge():
  x = np.arange(3 * 3, dtype=np.float64).reshape(1, 3, 3, 1)
  y = M.downsample(x)[0, ..., 0]
  np.testing.assert_array_equal(y, [[2.0, 3.5], [6.5, 8.0]])


def test_anti_correlated_images_give_zero():
  x = _noise(1, (177, 181, 3))
  _, cs = M.ssim_per_channel(x.astype(np.float64), 1.0 - x.astype(np.float64),
                             lambda v: M.filter_separable(v, M.gauss_1d()))
  assert (cs < 0).all()
  assert M.ms_ssim(x, 1.0 - x) == 0.0


def test_fp32_variant_tracks_fp64_on_noise():
  x, y = _noise(2, (161, 163, 3)), _noise(3, (161, 163, 3))
  y = 0.5 * x + 0.5 * y
  assert abs(float(M.ms_ssim(x, y, np.float32)) - float(M.ms_ssim(x, y))) < 1e-5


def test_oracle_size_check():
  for h, w in ((160, 200), (200, 160)):
    with pytest.raises(ValueError, match='161'):
      M.ms_ssim(np.zeros((h, w, 3)), np.zeros((h, w, 3)))


def test_mse_and_depth_abs_oracle():
  x, y = _noise(4, (2, 4, 5, 3)), _noise(5, (2, 4, 5, 3))
  np.testing.assert_allclose(M.mse(x, y), ((x.astype(np.float64) - y) ** 2).reshape(2, -1).mean(1))
  d = np.array([[1.0, 2.0], [3.0, 4.0]])
  t = np.array([[1.5, np.nan], [2.0, np.nan]])[..., None]
  assert M.depth_abs(d, t) == pytest.approx(0.75)
  assert np.isnan(M.depth_abs(d, np.full((2, 2, 1), np.nan)))


def test_compute_psnr_closed_form():
  # utils.py:103: -10 log(mse) / log(10)
  assert evaluation.compute_psnr(0.01) == pytest.approx(20.0, abs=1e-12)
  t = evaluation.compute_psnr(torch.tensor([1e-3, 0.25]))
  np.testing.assert_allclose(t.numpy(), [30.0, -10 * math.log10(0.25)], rtol=1e-6)


def test_python_argument_checks_fire_before_the_device():
  a = torch.zeros(170, 170, 3)
  with pytest.raises(ValueError, match='no CPU path'):
    evaluation.compute_multiscale_ssim(a, a)
  with pytest.raises(ValueError, match='differ'):
    evaluation.compute_multiscale_ssim(a, torch.zeros(170, 171, 3))
  with pytest.raises(ValueError, match='float32'):
    evaluation.compute_multiscale_ssim(a.double(), a.double())
  with pytest.raises(ValueError, match='161'):
    evaluation.compute_metrics(torch.zeros(160, 200, 3), torch.zeros(160, 200, 3))
  with pytest.raises(ValueError, match='channels'):
    evaluation.compute_multiscale_ssim(torch.zeros(170, 170, 5), torch.zeros(170, 170, 5))
  with pytest.raises(ValueError):
    evaluation.compute_multiscale_ssim(np.zeros((170, 170, 3), np.float32), a)


def test_workspace_size_query():
  lib = _lib.load()
  n, h, w, c = 2, 177, 181, 3
  size = lib.nfb_image_metrics_workspace_size(n, h, w, c)
  levels = M.level_sizes(h, w)
  pyramid = sum(2 * n * hh * ww * c * 4 for hh, ww in levels[1:])
  assert size >= pyramid and size % 256 == 0
  assert lib.nfb_image_metrics_workspace_size(1, 1080, 1920, 3) > size
  for args, msg in (((1, 160, 200, 3), b'161'), ((1, 200, 160, 3), b'161'), ((1, 200, 200, 0), b'channels'),
                    ((1, 200, 200, 5), b'channels'), ((0, 200, 200, 3), b'num_images')):
    assert lib.nfb_image_metrics_workspace_size(*args) < 0, args
    assert msg in lib.nfb_last_error(), (args, lib.nfb_last_error())


def test_c_abi_errors_without_a_device():
  lib = _lib.load()
  p = ctypes.c_void_p
  ws = lib.nfb_image_metrics_workspace_size(1, 200, 200, 3)
  assert lib.nfb_image_metrics(1, 160, 200, 3, p(256), p(256), None, None, p(256), ws,
                               None, None, None, None) < 0
  assert b'161' in lib.nfb_last_error()
  assert lib.nfb_image_metrics(1, 200, 200, 3, None, p(256), None, None, p(256), ws, None, None, None, None) < 0
  assert b'null' in lib.nfb_last_error()
  assert lib.nfb_image_metrics(1, 200, 200, 3, p(256), p(256), None, None, p(256), ws - 1,
                               None, None, None, None) < 0
  assert b'workspace' in lib.nfb_last_error()
