"""The C-ABI library loads without a GPU and exports every symbol the header
declares; with no device, handle creation fails loudly (no CPU fallback)."""
import ctypes
import os
import re

from nerfies_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
  text = open(os.path.join(REPO, 'include', 'nerfies_b200.h')).read()
  text = re.sub(r'/\*.*?\*/', '', text, flags=re.S)
  return sorted(set(re.findall(r'\b(nfb_[a-z_0-9]+)\s*\(', text)))


def test_header_and_binding_agree():
  assert _header_symbols() == sorted(_lib.SYMBOLS)


def test_library_exports_every_declared_symbol():
  lib = _lib.load()
  for name in _header_symbols():
    assert hasattr(lib, name), f'{name} not exported'
  assert lib.nfb_version().decode().startswith('nerfies_b200')


def test_config_struct_matches_header():
  text = open(os.path.join(REPO, 'include', 'nerfies_b200.h')).read()
  body = re.search(r'typedef struct nfb_config \{(.*?)\} nfb_config;', text,
                   re.S).group(1)
  body = re.sub(r'/\*.*?\*/', '', body, flags=re.S)
  names = []
  for decl in body.split(';'):
    decl = decl.strip()
    if not decl:
      continue
    decl = re.sub(r'^(unsigned|int|float)\s+', '', decl)
    names += [n.strip() for n in decl.split(',')]
  assert names == [f[0] for f in _lib.NfbConfig._fields_]


def test_no_device_is_a_loud_error():
  import torch
  if torch.cuda.is_available():
    return
  lib = _lib.load()
  cfg = _lib.NfbConfig()
  cfg.num_coarse_samples = 8
  h = ctypes.c_void_p()
  assert lib.nfb_create(ctypes.byref(cfg), 4, ctypes.byref(h)) != 0
  assert b'no CUDA device' in lib.nfb_last_error()


def test_camera_struct_matches_header():
  text = open(os.path.join(REPO, 'include', 'nerfies_b200.h')).read()
  body = re.search(r'typedef struct nfb_camera \{(.*?)\} nfb_camera;', text, re.S).group(1)
  body = re.sub(r'/\*.*?\*/', '', body, flags=re.S)
  fields = []
  for decl in body.split(';'):
    decl = decl.strip()
    if not decl:
      continue
    m = re.match(r'(int|float)\s+([a-z_]+)(?:\[(\d+)\])?$', decl)
    assert m, decl
    fields.append((m.group(2), m.group(1), int(m.group(3) or 1)))
  got = []
  for name, ctype in _lib.NfbCamera._fields_:
    n = getattr(ctype, '_length_', 1)
    base = ctype._type_ if n > 1 or hasattr(ctype, '_length_') else ctype
    got.append((name, 'float' if base is ctypes.c_float else 'int', n))
  assert fields == got
  assert ctypes.sizeof(_lib.NfbCamera) == 4 * sum(n for _, _, n in fields)


def test_camera_entry_points_fail_loudly_without_a_device():
  import torch
  if torch.cuda.is_available():
    return
  lib = _lib.load()
  cam = _lib.NfbCamera()
  cam.focal_length = 100.0
  cam.pixel_aspect_ratio = 1.0
  cam.image_size[:] = [4, 4]
  assert lib.nfb_camera_rays(ctypes.byref(cam), 0, 16, None, ctypes.c_void_p(16), None, None) != 0
  assert b'no CUDA device' in lib.nfb_last_error()
  assert lib.nfb_camera_rays(ctypes.byref(cam), 10, 16, None, ctypes.c_void_p(16), None, None) != 0
  assert b'exceeds' in lib.nfb_last_error()


def test_selftest_entries_refuse_bad_arguments():
  """The training kernels' self-test entries refuse bad arguments before touching a device (every call here
  is refused, so the fake pointers are never read)."""
  lib = _lib.load()
  p = ctypes.c_void_p(256)

  def refused(status, what):
    assert status != 0
    assert what in lib.nfb_last_error().decode(), lib.nfb_last_error()

  def vjp(R=4, S=8, ld_rgb=3, ld_a=1, act=6, rgb=p, d_rgb=p, samples=p):
    return lib.nfb_selftest_composite_vjp(R, S, rgb, ld_rgb, p, ld_a, p, p, None, None, 0, 1, act, samples, d_rgb, p,
                                          None)
  refused(vjp(S=1025), 'S=1025 outside [1, 1024]')
  refused(vjp(S=0), 'S=0 outside')
  refused(vjp(R=-1), 'R=-1 must be >= 0')
  refused(vjp(ld_rgb=2), 'leading dimension is below its width')
  refused(vjp(ld_a=0), 'leading dimension is below its width')
  refused(vjp(act=7), 'bad activation 7')
  refused(vjp(act=-1), 'bad activation -1')
  refused(vjp(rgb=None), 'null input or output')
  refused(vjp(d_rgb=None), 'null input or output')
  refused(vjp(samples=ctypes.c_void_p(264)), 'not 16-byte aligned')

  def elastic(R=4, warp_type=2, pivot=0, trans=0, loss_type=0, ld=6, head=p, jac=p, d_head=p, d_thead=p, stats=p):
    return lib.nfb_selftest_elastic(R, warp_type, pivot, trans, loss_type, head, p, ld, p, None, None, 1.0, jac,
                                    d_head, d_thead, stats, None)
  refused(elastic(R=-2), 'R=-2 must be >= 0')
  refused(elastic(warp_type=0), 'warp_type 0 is not 1 or 2')
  refused(elastic(warp_type=1, pivot=1), 'belong to warp_type 2')
  refused(elastic(trans=2), 'belong to warp_type 2')
  refused(elastic(loss_type=6), 'unknown loss type 6')
  refused(elastic(loss_type=-1), 'unknown loss type -1')
  refused(elastic(pivot=1, trans=1, ld=11), 'ld=11 is below the 12 head outputs')
  refused(elastic(warp_type=1, ld=2), 'ld=2 is below the 3 head outputs')
  refused(elastic(head=None), 'null head / thead / pts')
  refused(elastic(jac=None, d_thead=None, stats=None), 'no output')
  refused(elastic(d_head=None), 'needs d_head with d_thead')

  refused(lib.nfb_selftest_depth_index(4, 1025, p, p, None), 'S=1025 outside [1, 1024]')
  refused(lib.nfb_selftest_depth_index(-1, 8, p, p, None), 'R=-1 must be >= 0')
  refused(lib.nfb_selftest_depth_index(4, 8, p, None, None), 'null weights / sel')

  def mag(R=4, alpha=-2.0, scale=0.03, pts=p, stats=p):
    return lib.nfb_selftest_warp_mag_loss(R, pts, p, None, alpha, scale, 1.0, None, stats, None)
  refused(mag(R=-1), 'R=-1 must be >= 0')
  refused(mag(alpha=float('nan')), 'alpha is NaN')
  refused(mag(scale=0.0), 'must be finite and > 0')
  refused(mag(scale=float('inf')), 'must be finite and > 0')
  refused(mag(stats=None), 'null pts / warped / stats')
  refused(mag(pts=None), 'null pts / warped / stats')

  # the layer walker's entries take a handle; the rest of their refusals are in test_train_net_gpu.py
  n = ctypes.c_int()
  steps = (ctypes.c_int * 112)()
  refused(lib.nfb_selftest_net_steps(None, 0, 1, ctypes.byref(n), steps), 'selftest_net_steps: null handle')
  refused(lib.nfb_selftest_net(None, 0, 1, 4, p, 64, p, None, 0, 0, None, None, 0, None), 'selftest_net: null handle')
  refused(lib.nfb_selftest_cond_vjp(None, 4, p, None, None, None, 0, 0, None, None, None, None, None, None, 0, None),
          'null handle')

  def enc(rows=4, S=2, F=2, ld=20, stride=8, off=0, n_cond=4, din=p, dpts=p, dcond=p):
    return lib.nfb_selftest_encode_bwd(rows, S, p, None, din, F, ld, stride, off, n_cond, dpts, dcond, None)
  refused(enc(rows=-1), 'rows=-1 must be >= 0')
  refused(enc(S=0), 'S=0 must be >= 1')
  refused(enc(F=-1), 'negative F')
  refused(enc(ld=18), 'ld=18 is below 3 + 6 F + n_cond')
  refused(enc(stride=3), 'cond_stride is below')
  refused(enc(din=None), 'null din')
  refused(enc(dpts=None, dcond=None), 'no output')

  def tail(rows=4, warp_type=2, pivot=0, trans=0, ld=6, head=p, dhead=p, dpts=p):
    return lib.nfb_selftest_warp_tail_bwd(rows, warp_type, pivot, trans, head, ld, p, p, dhead, dpts, None)
  refused(tail(rows=-1), 'rows=-1 must be >= 0')
  refused(tail(warp_type=0), 'warp_type 0 is not 1 or 2')
  refused(tail(warp_type=1, trans=1), 'belong to warp_type 2')
  refused(tail(pivot=1, trans=1, ld=11), 'ld=11 is below the 12 head outputs')
  refused(tail(head=None), 'null input, or no output')
  refused(tail(dhead=None, dpts=None), 'null input, or no output')

  def reduce(R=4, S=8, dpts=p, d_o=p, d_d=p):
    return lib.nfb_selftest_ray_reduce(R, S, dpts, p, p, None, d_o, d_d, None)
  refused(reduce(R=-1), 'R=-1 must be >= 0')
  refused(reduce(S=1025), 'S=1025 outside [1, 1024]')
  refused(reduce(dpts=None), 'null input, or no output')
  refused(reduce(d_o=None, d_d=None), 'null input, or no output')

  def viewdir(R=4, stride=27, off=0, F=4, acc=0, out=p):
    return lib.nfb_selftest_viewdir_vjp(R, p, stride, off, F, p, out, acc, None)
  refused(viewdir(R=-1), 'R=-1 must be >= 0')
  refused(viewdir(stride=28, off=2), 'stride is below off + 3 + 6 F')
  refused(viewdir(acc=2), 'accumulate=2 is not 0 or 1')
  refused(viewdir(out=None), 'null dcond / viewdirs / out')
