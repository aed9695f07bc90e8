"""wgmma plumbing self-test: GMMA descriptors / 128-byte swizzle / accumulator
fragment layout against a torch fp64 reference of the same op (bf16-rounded
operands, fp32 accumulation)."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('K,N', [(64, 16), (64, 256), (51, 128), (128, 128),
                                 (256, 256), (320, 256), (187, 128), (283, 6),
                                 (256, 1)])
def test_selftest_gemm(K, N):
  from nerfies_b200 import _lib
  lib = _lib.load()
  g = torch.Generator().manual_seed(K * 1000 + N)
  A = torch.randn(128, K, generator=g).cuda()
  W = (torch.randn(K, N, generator=g) * 0.1).cuda()
  C = torch.full((128, N), float('nan'), device='cuda')
  _lib.check(lib.nfb_selftest_gemm(K, N, ctypes.c_void_p(A.data_ptr()),
                                   ctypes.c_void_p(W.data_ptr()),
                                   ctypes.c_void_p(C.data_ptr()), None))
  ref = A.bfloat16().double() @ W.bfloat16().double()
  err = float((C.double() - ref).abs().max())
  scale = float(ref.abs().max()) + 1e-6
  assert err / scale < 1e-5, f'K={K} N={N}: max abs err {err:.3e} (scale {scale:.2f})'


@pytest.mark.parametrize('K,N', [(64, 128), (128, 128), (256, 128), (192, 256), (187, 64), (256, 16), (200, 12)])
def test_selftest_gemm_fp16x3(K, N):
  """The three fp16 chains of the fp16x3 field kernel against an fp64 product of the
  fp32 values."""
  from nerfies_b200 import _lib
  lib = _lib.load()
  g = torch.Generator().manual_seed(K * 1000 + N + 13)
  A = torch.randn(128, K, generator=g).cuda()
  W = (torch.randn(K, N, generator=g) * 0.1).cuda()
  C = torch.full((128, N), float('nan'), device='cuda')
  out = (ctypes.c_longlong * 2)()
  _lib.check(lib.nfb_selftest_gemm3(K, N, ctypes.c_void_p(A.data_ptr()), ctypes.c_void_p(W.data_ptr()),
                                    ctypes.c_void_p(C.data_ptr()), 1, out, None))
  ref = A.double() @ W.double()
  err = float((C.double() - ref).abs().max())
  scale = float(ref.abs().max()) + 1e-6
  assert err / scale < 2e-6, f'K={K} N={N}: max abs err {err:.3e} (scale {scale:.2f})'
  assert out[1] == ((K + 63) // 64) * 12 and out[0] > 0
