"""ctypes binding of libnerfies_b200.so (C ABI: include/nerfies_b200.h).

There is no CPU path: importing this module without the built library, or
creating a handle without a CUDA device, raises.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# NFB_LIB_PATH: override of the library path (to compare two builds of the kernels).
LIB_PATH = os.environ.get('NFB_LIB_PATH') or os.path.join(_HERE, 'libnerfies_b200.so')

# Every symbol include/nerfies_b200.h declares (checked by tests/test_abi.py).
SYMBOLS = [
    'nfb_create', 'nfb_destroy', 'nfb_param_count', 'nfb_param_info',
    'nfb_set_params', 'nfb_render_forward', 'nfb_render_forward_host',
    'nfb_render_samples', 'nfb_sample_pdf', 'nfb_coarse_z_vals',
    'nfb_warp_forward', 'nfb_kernel_launches', 'nfb_last_error', 'nfb_version',
    'nfb_set_profiling', 'nfb_field_time_ms', 'nfb_selftest_gemm',
    'nfb_camera_rays', 'nfb_pixels_to_rays', 'nfb_selftest_gemm3',
    'nfb_debug_provoke_timeout', 'nfb_set_time_alpha', 'nfb_train_value_and_grad', 'nfb_adam_step',
    'nfb_train_value_and_grad_reg', 'nfb_warp_jacobian', 'nfb_check_abort', 'nfb_reset_abort',
    'nfb_image_metrics_workspace_size', 'nfb_image_metrics', 'nfb_gather_rays', 'nfb_selftest_sgemm',
    'nfb_set_train_precision', 'nfb_selftest_train_gemm', 'nfb_debug_one_row_block',
    'nfb_image_quantize', 'nfb_render_vjp', 'nfb_warp_vjp', 'nfb_colorize',
    'nfb_frame_pyramid', 'nfb_blur_scores_workspace_size', 'nfb_blur_scores', 'nfb_camera_project',
    'nfb_near_far_workspace_size', 'nfb_near_far', 'nfb_marching_cubes_workspace_size',
    'nfb_marching_cubes_count', 'nfb_marching_cubes', 'nfb_marching_cubes_table', 'nfb_warp_invert',
]

class TrainReg(ctypes.Structure):
  """nfb_train_reg (include/nerfies_b200.h)."""
  _fields_ = [('use_elastic_loss', ctypes.c_int), ('elastic_reduce_method', ctypes.c_int),
              ('elastic_loss_type', ctypes.c_int), ('elastic_loss_weight', ctypes.c_float),
              ('use_warp_reg_loss', ctypes.c_int), ('warp_reg_loss_weight', ctypes.c_float),
              ('warp_reg_loss_alpha', ctypes.c_float), ('warp_reg_loss_scale', ctypes.c_float),
              ('use_background_loss', ctypes.c_int), ('num_background_points', ctypes.c_int),
              ('background_points', ctypes.c_void_p), ('background_warp_ids', ctypes.c_void_p),
              ('background_noise', ctypes.c_void_p), ('background_loss_weight', ctypes.c_float)]


ELASTIC_TYPES = {'log_svals': 0, 'svals': 1, 'jtj': 2, 'div': 3, 'det': 4, 'log_det': 5}
ELASTIC_REDUCE = {'median': 0, 'weight': 1}
ACTIVATIONS = {'none': 0, 'relu': 1, 'elu': 2, 'leaky_relu': 3, 'tanh': 4,
               'sigmoid': 5, 'softplus': 6}
WARP_TYPES = {None: 0, 'none': 0, 'translation': 1, 'se3': 2}
WARP_ENCODERS = {'glo': 0, 'time': 1, 'blend': 2}
PRECISIONS = {'fp32': 0, 'bf16': 1, 'fp16x3': 2}
TRAIN_PRECISIONS = {'fp32': 0, 'tf32x3': 1}
FLAG_COARSE_ONLY = 1
FLAG_NO_WARP = 2
FLAG_METADATA_ENCODED = 4
# nfb_warp_invert's per-point status (NFB_INVERT_*)
INVERT_STATUS = {'converged': 0, 'max_iters': 1, 'singular': 2, 'stalled': 3, 'nonfinite': 4}


class NfbConfig(ctypes.Structure):
  """struct nfb_config - field order must match the header."""
  _fields_ = [
      ('num_coarse_samples', ctypes.c_int),
      ('num_fine_samples', ctypes.c_int),
      ('num_nerf_point_freqs', ctypes.c_int),
      ('num_nerf_viewdir_freqs', ctypes.c_int),
      ('num_warp_freqs', ctypes.c_int),
      ('nerf_trunk_depth', ctypes.c_int),
      ('nerf_trunk_width', ctypes.c_int),
      ('nerf_rgb_branch_depth', ctypes.c_int),
      ('nerf_rgb_branch_width', ctypes.c_int),
      ('nerf_skips_mask', ctypes.c_uint),
      ('alpha_channels', ctypes.c_int),
      ('rgb_channels', ctypes.c_int),
      ('warp_field_type', ctypes.c_int),
      ('warp_trunk_depth', ctypes.c_int),
      ('warp_trunk_width', ctypes.c_int),
      ('warp_skips_mask', ctypes.c_uint),
      ('num_warp_features', ctypes.c_int),
      ('num_appearance_features', ctypes.c_int),
      ('num_camera_features', ctypes.c_int),
      ('num_warp_embeddings', ctypes.c_int),
      ('num_appearance_embeddings', ctypes.c_int),
      ('num_camera_embeddings', ctypes.c_int),
      ('use_viewdirs', ctypes.c_int),
      ('use_appearance_metadata', ctypes.c_int),
      ('use_camera_metadata', ctypes.c_int),
      ('use_trunk_condition', ctypes.c_int),
      ('use_alpha_condition', ctypes.c_int),
      ('use_rgb_condition', ctypes.c_int),
      ('activation', ctypes.c_int),
      ('sigma_activation', ctypes.c_int),
      ('use_white_background', ctypes.c_int),
      ('use_linear_disparity', ctypes.c_int),
      ('use_sample_at_infinity', ctypes.c_int),
      ('near_plane', ctypes.c_float),
      ('far_plane', ctypes.c_float),
      ('precision', ctypes.c_int),
      ('warp_metadata_encoder', ctypes.c_int),
      ('time_encoder_num_freqs', ctypes.c_int),
      ('warp_use_pivot', ctypes.c_int),
      ('warp_use_translation', ctypes.c_int),
  ]


class NfbCamera(ctypes.Structure):
  """struct nfb_camera - field order must match the header."""
  _fields_ = [
      ('orientation', ctypes.c_float * 9),
      ('position', ctypes.c_float * 3),
      ('focal_length', ctypes.c_float),
      ('principal_point', ctypes.c_float * 2),
      ('skew', ctypes.c_float),
      ('pixel_aspect_ratio', ctypes.c_float),
      ('radial_distortion', ctypes.c_float * 3),
      ('tangential_distortion', ctypes.c_float * 2),
      ('image_size', ctypes.c_int * 2),
  ]


class NfbRayTable(ctypes.Structure):
  """struct nfb_ray_table - field order must match the header."""
  _fields_ = [
      ('num_images', ctypes.c_int),
      ('cameras', ctypes.c_void_p),
      ('pixel_offsets', ctypes.c_void_p),
      ('rgb', ctypes.c_void_p),
      ('appearance', ctypes.c_void_p),
      ('camera', ctypes.c_void_p),
      ('warp', ctypes.c_void_p),
      ('time', ctypes.c_void_p),
      ('order', ctypes.c_void_p),
      ('order_is_64', ctypes.c_int),
      ('num_rays', ctypes.c_longlong),
  ]


class NfbError(RuntimeError):
  pass


_lib = None


def load():
  """Loads the shared library (once).  Raises if it has not been built."""
  global _lib
  if _lib is not None:
    return _lib
  if not os.path.exists(LIB_PATH):
    raise ImportError(
        f'{LIB_PATH} is missing: build it with `python -c "import '
        '__graft_entry__ as g; g.build()"` (nvcc, sm_90a). nerfies_b200 has '
        'no CPU or PyTorch fallback.')
  lib = ctypes.CDLL(LIB_PATH)
  vp, ci, cf, cu = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_uint
  lib.nfb_create.argtypes = [ctypes.POINTER(NfbConfig), ci, ctypes.POINTER(vp)]
  lib.nfb_create.restype = ci
  lib.nfb_destroy.argtypes = [vp]
  lib.nfb_destroy.restype = None
  lib.nfb_param_count.argtypes = [vp]
  lib.nfb_param_count.restype = ci
  lib.nfb_param_info.argtypes = [vp, ci, ctypes.c_char_p, ci,
                                 ctypes.POINTER(ctypes.c_longlong),
                                 ctypes.POINTER(ctypes.c_longlong)]
  lib.nfb_param_info.restype = ci
  lib.nfb_set_params.argtypes = [vp, ctypes.POINTER(vp),
                                 ctypes.POINTER(ctypes.c_longlong), ci, vp]
  lib.nfb_set_params.restype = ci
  lib.nfb_render_forward.argtypes = [vp, ci] + [vp] * 6 + [cf, vp, vp, cu
                                                           ] + [vp] * 6
  lib.nfb_render_forward.restype = ci
  lib.nfb_render_forward_host.argtypes = [vp, ci] + [vp] * 6 + [cf, cu, vp, vp,
                                                                vp]
  lib.nfb_render_forward_host.restype = ci
  lib.nfb_render_samples.argtypes = [vp, ci, ci, ci] + [vp] * 7 + [cf, cu
                                                                   ] + [vp] * 5
  lib.nfb_render_samples.restype = ci
  lib.nfb_sample_pdf.argtypes = [vp, ci, vp, vp, vp, vp, vp]
  lib.nfb_sample_pdf.restype = ci
  lib.nfb_coarse_z_vals.argtypes = [vp, ci, vp, vp, vp]
  lib.nfb_coarse_z_vals.restype = ci
  lib.nfb_warp_forward.argtypes = [vp, ci, vp, vp, cf, cu, vp, vp]
  lib.nfb_train_value_and_grad.argtypes = [vp, ci] + [vp] * 6 + [cf, vp, vp, cu, vp, ci, ctypes.POINTER(vp),
                                           ctypes.POINTER(ctypes.c_longlong), ci, vp, vp]
  lib.nfb_train_value_and_grad.restype = ci
  lib.nfb_train_value_and_grad_reg.argtypes = [vp, ci] + [vp] * 6 + [cf, vp, vp, cu, vp, ci, vp, ctypes.POINTER(vp),
                                               ctypes.POINTER(ctypes.c_longlong), ci, vp, vp]
  lib.nfb_train_value_and_grad_reg.restype = ci
  lib.nfb_render_vjp.argtypes = [vp, ci] + [vp] * 6 + [cf, cu] + [vp] * 11 + [ci, ctypes.POINTER(vp),
                                                                              ctypes.POINTER(ctypes.c_longlong), ci, vp]
  lib.nfb_render_vjp.restype = ci
  lib.nfb_warp_vjp.argtypes = [vp, ci, vp, vp, cf, cu, vp, vp, ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_longlong),
                               ci, vp]
  lib.nfb_warp_vjp.restype = ci
  lib.nfb_warp_jacobian.argtypes = [vp, ci, vp, vp, cf, vp, vp, vp]
  lib.nfb_warp_jacobian.restype = ci
  lib.nfb_warp_invert.argtypes = [vp, ci, vp, vp, vp, cf, ci, cf, vp, vp, vp, vp, vp]
  lib.nfb_warp_invert.restype = ci
  lib.nfb_check_abort.argtypes = [vp, ci]
  lib.nfb_check_abort.restype = ci
  lib.nfb_reset_abort.argtypes = []
  lib.nfb_reset_abort.restype = ci
  lib.nfb_adam_step.argtypes = [vp, vp, vp, vp, ctypes.c_longlong, cf, cf, cf, cf, ctypes.c_longlong, vp]
  lib.nfb_adam_step.restype = ci
  lib.nfb_set_time_alpha.argtypes = [vp, cf]
  lib.nfb_set_time_alpha.restype = ci
  lib.nfb_warp_forward.restype = ci
  lib.nfb_kernel_launches.argtypes = [vp]
  lib.nfb_kernel_launches.restype = ctypes.c_longlong
  lib.nfb_set_profiling.argtypes = [vp, ci]
  lib.nfb_set_profiling.restype = ci
  lib.nfb_field_time_ms.argtypes = [vp, ci]
  lib.nfb_field_time_ms.restype = cf
  lib.nfb_selftest_gemm.argtypes = [ci, ci, vp, vp, vp, vp]
  lib.nfb_selftest_gemm.restype = ci
  ll = ctypes.c_longlong
  lib.nfb_camera_rays.argtypes = [ctypes.POINTER(NfbCamera), ll, ll, vp, vp, vp, vp]
  lib.nfb_camera_rays.restype = ci
  lib.nfb_pixels_to_rays.argtypes = [ctypes.POINTER(NfbCamera), vp, ll, vp, vp]
  lib.nfb_pixels_to_rays.restype = ci
  lib.nfb_gather_rays.argtypes = [ctypes.POINTER(NfbRayTable), ll, ll] + [vp] * 9
  lib.nfb_gather_rays.restype = ci
  lib.nfb_image_metrics_workspace_size.argtypes = [ci, ci, ci, ci]
  lib.nfb_image_metrics_workspace_size.restype = ll
  lib.nfb_image_metrics.argtypes = [ci, ci, ci, ci, vp, vp, vp, vp, vp, ll, vp, vp, vp, vp]
  lib.nfb_image_metrics.restype = ci
  lib.nfb_image_quantize.argtypes = [vp, ll, ci, cf, vp, vp]
  lib.nfb_image_quantize.restype = ci
  lib.nfb_colorize.argtypes = [vp, vp, ci, ci, ci, vp, cf, cf, cf, ci, vp, vp, vp, ll, vp]
  lib.nfb_colorize.restype = ci
  lib.nfb_frame_pyramid.argtypes = [vp, ci, ci, ll, ci, ctypes.POINTER(ci), ctypes.POINTER(vp), vp]
  lib.nfb_frame_pyramid.restype = ci
  lib.nfb_blur_scores_workspace_size.argtypes = [ci]
  lib.nfb_blur_scores_workspace_size.restype = ll
  lib.nfb_blur_scores.argtypes = [vp, ci, ci, ci, vp, ll, vp, vp]
  lib.nfb_blur_scores.restype = ci
  lib.nfb_camera_project.argtypes = [ctypes.POINTER(NfbCamera), vp, ll, vp, vp]
  lib.nfb_camera_project.restype = ci
  lib.nfb_near_far_workspace_size.argtypes = [ci]
  lib.nfb_near_far_workspace_size.restype = ll
  lib.nfb_near_far.argtypes = [vp, ci, vp, ll, ctypes.c_double, ctypes.c_double, vp, ll, vp, vp, vp, vp]
  lib.nfb_near_far.restype = ci
  lib.nfb_marching_cubes_workspace_size.argtypes = [ci, ci, ci]
  lib.nfb_marching_cubes_workspace_size.restype = ll
  lib.nfb_marching_cubes_count.argtypes = [vp, ci, ci, ci, cf, vp, ll, vp, vp]
  lib.nfb_marching_cubes_count.restype = ci
  lib.nfb_marching_cubes.argtypes = [vp, ci, ci, ci, cf, ctypes.POINTER(cf), ctypes.POINTER(cf), vp, ll, vp, vp,
                                     vp, vp]
  lib.nfb_marching_cubes.restype = ci
  lib.nfb_marching_cubes_table.argtypes = [ctypes.POINTER(ci)]
  lib.nfb_marching_cubes_table.restype = ci
  lib.nfb_selftest_gemm3.argtypes =[ci, ci, vp, vp, vp, ci, vp, vp]
  lib.nfb_selftest_gemm3.restype = ci
  lib.nfb_selftest_sgemm.argtypes = [ci, ll, ci, ci, ci, ci, vp, ci, vp, ci, vp, ci] + [vp] * 6 + [
      ll, ctypes.POINTER(ll), vp]
  lib.nfb_selftest_sgemm.restype = ci
  lib.nfb_selftest_train_gemm.argtypes = [ci] + lib.nfb_selftest_sgemm.argtypes
  lib.nfb_selftest_train_gemm.restype = ci
  lib.nfb_set_train_precision.argtypes = [vp, ci]
  lib.nfb_set_train_precision.restype = ci
  lib.nfb_debug_provoke_timeout.argtypes = [vp, ci]
  lib.nfb_debug_provoke_timeout.restype = ci
  lib.nfb_debug_one_row_block.argtypes = [vp, ci]
  lib.nfb_debug_one_row_block.restype = ci
  lib.nfb_last_error.argtypes = []
  lib.nfb_last_error.restype = ctypes.c_char_p
  lib.nfb_version.argtypes = []
  lib.nfb_version.restype = ctypes.c_char_p
  _lib = lib
  return lib


def check(status):
  if status != 0:
    raise NfbError(load().nfb_last_error().decode())
