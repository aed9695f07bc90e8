"""Mirror of nerfies/evaluation.py: render_image, plus the model_fn factory
that eval.py builds with jax.pmap (eval.py:330-348), plus a whole-frame renderer.

Multi-GPU: one process per GPU (torch.distributed, NCCL).  `device_count` is
the number of shards a chunk is split into, exactly as in the reference
(utils.shard, utils.py:334-338); each rank renders shard `rank` and the shards
are exchanged with ONE all_gather per chunk of the packed 24 B/ray/level result
(the reference's lax.all_gather, eval.py:339, moves the same values as 4 arrays
per level).  With device_count == 1 there is no collective.

`render_frame` is the GPU-native form of the same job (eval.py:330-353 +
datasets/core.py:50-75): every rank generates the rays of its contiguous slab of
the frame on the GPU (camera_rays_kernel), renders it in large launches, and the
frame is assembled with a single all_gather of 24 B/ray at the end - instead of
h*w/chunk host round trips with a collective each.

`compute_metrics`, `compute_multiscale_ssim` and `compute_psnr` are the per-frame
metrics of eval.py:process_batch (eval.py:58-62, 120-122, 140; utils.py:94-103),
computed on the device by the library's metrics kernels (`nfb_image_metrics`).

`image_to_uint8`, `image_to_uint16` and `depth_to_uint16` are image_utils.py:114-131, 172-174 on
the device (`nfb_image_quantize`): a frame leaves the GPU as the 8- / 16-bit image that is saved.
"""
import ctypes
import math
import time

import torch
import torch.distributed as dist

from nerfies_b200 import _lib

MIN_METRICS_SIZE = 161   # MS-SSIM: each of the 5 scales (161 -> 81 -> 41 -> 21 -> 11) >= 11x11

_TREE_TYPES = (dict,)
_KEYS = (('rgb', slice(0, 3)), ('depth', 3), ('med_depth', 4), ('acc', 5))


def _tree_map(fn, tree):
  if isinstance(tree, dict):
    return {k: _tree_map(fn, v) for k, v in tree.items()}
  return fn(tree)


def shard(xs, device_count):
  """utils.shard (utils.py:334-338)."""
  return _tree_map(lambda x: x.reshape((device_count, -1) + tuple(x.shape[1:])), xs)


def unshard(x, padding=0):
  """utils.unshard (utils.py:346-351)."""
  y = x.reshape((x.shape[0] * x.shape[1],) + tuple(x.shape[2:]))
  return y[:-padding] if padding > 0 else y


def _dist_info():
  distributed = dist.is_available() and dist.is_initialized()
  return (dist.get_world_size() if distributed else 1,
          dist.get_rank() if distributed else 0)


def _unpack(packed):
  """(..., 6) -> {'rgb' (...,3), 'depth', 'med_depth', 'acc' (...)} (views)."""
  return {k: packed[..., i] for k, i in _KEYS}


def make_model_fn(model, **apply_kwargs):
  """The `_model_fn` + pmap + all_gather of eval.py:330-348 as a plain callable
  with the same signature: model_fn(key_0, key_1, params, rays_dict, warp_extra)
  where every leaf of rays_dict has a leading shard axis (device_count, n, ...).
  Returns every shard's output stacked on axis 0, like lax.all_gather."""
  simple = not apply_kwargs      # extra outputs (weights, points) take the per-key path

  def model_fn(key_0, key_1, params, rays_dict, warp_extra):
    n_shards = rays_dict['origins'].shape[0]
    world, rank = _dist_info()
    if world > 1 and n_shards != world:
      raise ValueError(f'device_count={n_shards} must equal the world size '
                       f'{world}')
    mine = range(n_shards) if world == 1 else [rank]
    outs = []
    for s in mine:
      rays = _tree_map(lambda x: x[s], rays_dict)
      outs.append(model.apply({'params': params}, rays, warp_extra=warp_extra,
                              rngs={'coarse': key_0, 'fine': key_1},
                              mutable=False, _packed=simple, **apply_kwargs))
    if simple:
      levels = list(outs[0])
      if world == 1:
        return {lv: _unpack(torch.stack([o[lv] for o in outs], 0)) for lv in levels}
      # one collective per chunk: (levels, n, 6) from every rank
      mine_packed = torch.stack([outs[0][lv] for lv in levels], 0).contiguous()
      buf = torch.empty((world * len(levels),) + tuple(mine_packed.shape[1:]),
                        device=mine_packed.device, dtype=mine_packed.dtype)
      dist.all_gather_into_tensor(buf, mine_packed)
      buf = buf.reshape((world, len(levels)) + tuple(mine_packed.shape[1:]))
      return {lv: _unpack(buf[:, i]) for i, lv in enumerate(levels)}
    if world == 1:
      return {lv: {k: torch.stack([o[lv][k] for o in outs], 0)
                   for k in outs[0][lv]} for lv in outs[0]}
    gathered = {}
    for lv, ret in outs[0].items():
      gathered[lv] = {}
      for k, v in ret.items():
        v = v.contiguous()
        buf = torch.empty((world * v.shape[0],) + tuple(v.shape[1:]),
                          device=v.device, dtype=v.dtype)
        dist.all_gather_into_tensor(buf, v)
        gathered[lv][k] = buf.reshape((world,) + tuple(v.shape))
    return gathered

  return model_fn


def render_image(state, rays_dict, model_fn, device_count, rng, chunk=8192,
                 default_ret_key=None):
  """Render all the pixels of an image (evaluation.py:28-101): same arguments,
  chunking, edge padding to a multiple of device_count, and output pytree
  {rgb (h,w,3), depth, med_depth, acc (h,w)}."""
  h, w = rays_dict['origins'].shape[:2]
  rays_dict = _tree_map(lambda x: torch.as_tensor(x).reshape((h * w, -1)),
                        rays_dict)
  num_rays = h * w
  key_0 = key_1 = rng  # keys are unused on the deterministic eval path.
  ret_maps = []
  start_time = time.time()
  num_batches = int(math.ceil(num_rays / chunk))
  for batch_idx in range(num_batches):
    ray_idx = batch_idx * chunk
    chunk_rays = _tree_map(lambda x: x[ray_idx:ray_idx + chunk], rays_dict)
    num_chunk_rays = chunk_rays['origins'].shape[0]
    remainder = num_chunk_rays % device_count
    if remainder != 0:
      padding = device_count - remainder
      # jnp.pad(..., mode='edge'): repeat the last ray.
      chunk_rays = _tree_map(
          lambda x: torch.cat([x, x[-1:].expand(padding, *x.shape[1:])], 0),
          chunk_rays)
    else:
      padding = 0
    chunk_rays = shard(chunk_rays, device_count)
    model_out = model_fn(key_0, key_1, state.optimizer.target['model'],
                         chunk_rays, state.warp_extra)
    if not default_ret_key:
      ret_key = 'fine' if 'fine' in model_out else 'coarse'
    else:
      ret_key = default_ret_key
    ret_map = {k: unshard(v, padding) for k, v in model_out[ret_key].items()}
    ret_maps.append(ret_map)
  out = {}
  for key in ret_maps[0]:
    value = torch.cat([m[key] for m in ret_maps], dim=0)
    out[key] = value.reshape((h, w) + tuple(value.shape[1:]))
  render_image.last_seconds = time.time() - start_time
  return out


def render_frame(model, params, camera, warp_extra, metadata=None, max_rays=65536,
                 default_ret_key=None, timings=None):
  """One full frame from a Camera, GPU-native (eval.py:330-353 without the host
  loop): rank r renders pixels [r * n, (r + 1) * n) of the row-major frame,
  n = ceil(h * w / world); rays come from camera_rays_kernel on the device
  (datasets/core.py:50-75), the slab is rendered in launches of up to `max_rays`
  rays, and ONE all_gather of the packed (n, 6) result assembles the frame on
  every rank (padding rays past the end repeat the last pixel, like the
  reference's edge padding, and are dropped).

  metadata: {'warp': id, 'appearance': id, 'camera': id, 'time': t} scalars applied to every
  ray (eval.py:344-348 renders one camera with one metadata id per frame).
  timings (optional dict) receives {'render_ms', 'gather_ms'} measured with CUDA
  events on the current stream.  Returns {rgb (h,w,3), depth, med_depth, acc}."""
  from nerfies_b200 import camera as camera_lib
  world, rank = _dist_info()
  dev = model.device
  h, w = camera.image_shape
  total = h * w
  per = -(-total // world)
  first = rank * per
  count = max(0, min(per, total - first))
  md = metadata or {}
  ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)] if timings is not None else None
  if ev:
    ev[0].record()
  packed = torch.empty(per, 6, device=dev)
  levels_key = None
  done = 0
  while done < count:
    n = min(max_rays, count - done)
    rays = camera_lib.camera_to_rays(camera, dev, first_pixel=first + done, count=n)
    rays_dict = {'origins': rays['origins'], 'directions': rays['directions'],
                 # ids are int32; 'time' (the TimeEncoder's input, models.py:252-254) is float32
                 'metadata': {k: (torch.full((n, 1), float(v), dtype=torch.float32, device=dev) if k == 'time'
                                  else torch.full((n, 1), int(v), dtype=torch.int32, device=dev))
                              for k, v in md.items()}}
    out = model.apply({'params': params}, rays_dict, warp_extra=warp_extra, _packed=True)
    if levels_key is None:
      levels_key = default_ret_key or ('fine' if 'fine' in out else 'coarse')
    packed[done:done + n] = out[levels_key]
    done += n
  if count < per:
    # edge padding (this rank's slab runs past the frame): repeat the last pixel's result
    fill = packed[count - 1:count] if count > 0 else torch.zeros(1, 6, device=dev)
    packed[count:] = fill
  if ev:
    ev[1].record()
  if world > 1:
    buf = torch.empty(world * per, 6, device=dev)
    dist.all_gather_into_tensor(buf, packed)
  else:
    buf = packed
  if ev:
    ev[2].record()
    ev[2].synchronize()
    timings['render_ms'] = ev[0].elapsed_time(ev[1])
    timings['gather_ms'] = ev[1].elapsed_time(ev[2])
  frame = buf[:total]
  return {k: frame[:, i].reshape((h, w) + ((3,) if k == 'rgb' else ()))
          for k, i in _KEYS}


def _check_images(a, b, what):
  for t in (a, b):
    if not torch.is_tensor(t):
      raise ValueError(f'{what} must be torch tensors on a CUDA device')
  if a.shape != b.shape:
    raise ValueError(f'{what}: shapes {tuple(a.shape)} and {tuple(b.shape)} differ')
  if a.dim() not in (3, 4):
    raise ValueError(f'{what}: expected (h, w, c) or (N, h, w, c) images, got {tuple(a.shape)}')
  if a.dtype != torch.float32 or b.dtype != torch.float32:
    raise ValueError(f'{what}: dtype must be float32, got {a.dtype} and {b.dtype}')
  h, w, c = a.shape[-3:]
  if h < MIN_METRICS_SIZE or w < MIN_METRICS_SIZE:
    raise ValueError(f'{what}: MS-SSIM needs images of at least {MIN_METRICS_SIZE}x{MIN_METRICS_SIZE} '
                     f'(each of its 5 scales must be >= 11x11); got {h}x{w}')
  if not 1 <= c <= 4:
    raise ValueError(f'{what}: {c} channels; 1 to 4 are supported')
  if not (a.is_cuda and b.is_cuda) or a.device != b.device:
    raise ValueError(f'{what} must live on one CUDA device: nerfies_b200 has no CPU path')


def _image_metrics(image, target, depth=None, depth_target=None):
  """One nfb_image_metrics call on (N, h, w, c) images; returns (ms_ssim, mse, depth_abs), (N,)."""
  n, h, w, c = image.shape
  dev = image.device
  lib = _lib.load()
  ws_bytes = lib.nfb_image_metrics_workspace_size(n, h, w, c)
  if ws_bytes < 0:
    raise ValueError(lib.nfb_last_error().decode())
  image, target = image.contiguous(), target.contiguous()
  if depth is not None:
    depth, depth_target = depth.contiguous(), depth_target.contiguous()
  out = torch.empty(3, n, dtype=torch.float32, device=dev)
  ptr = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
  with torch.cuda.device(dev):
    workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    _lib.check(lib.nfb_image_metrics(
        n, h, w, c, ptr(image), ptr(target), ptr(depth), ptr(depth_target), ptr(workspace), ws_bytes,
        ptr(out[0]), ptr(out[1]), ptr(out[2]) if depth is not None else None,
        ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
  return out[0], out[1], (out[2] if depth is not None else None)


def _image_quantize(image, bits, scale):
  """One nfb_image_quantize call; the result has the image's shape."""
  if not torch.is_tensor(image) or not image.is_cuda:
    raise ValueError('the image must be a torch tensor on a CUDA device: nerfies_b200 has no CPU path')
  if image.dtype != torch.float32:
    raise ValueError(f'Input image should be float32 but is of type {image.dtype}')
  image = image.contiguous()
  out = torch.empty(image.shape, dtype=torch.uint8 if bits == 8 else torch.uint16, device=image.device)
  with torch.cuda.device(image.device):
    _lib.check(_lib.load().nfb_image_quantize(
        ctypes.c_void_p(image.data_ptr()), image.numel(), bits, float(scale), ctypes.c_void_p(out.data_ptr()),
        ctypes.c_void_p(torch.cuda.current_stream(image.device).cuda_stream)))
  return out


def image_to_uint8(image):
  """image_utils.image_to_uint8 (image_utils.py:114-121) on the device:
  (image * 255).clip(0, 255).astype(uint8), value for value.  CUDA float32 in, torch.uint8 out."""
  return _image_quantize(image, 8, 1.0)


def image_to_uint16(image):
  """image_utils.image_to_uint16 (image_utils.py:124-131) on the device; torch.uint16 out."""
  return _image_quantize(image, 16, 1.0)


def depth_to_uint16(depth):
  """What image_utils.save_depth writes (image_utils.py:172-174): image_to_uint16(depth / 1000.0)."""
  return _image_quantize(depth, 16, 1000.0)


def compute_multiscale_ssim(image1, image2):
  """eval.py:58-62: tf.image.ssim_multiscale(image1, image2, max_val=1.0) with TF's defaults, on
  the GPU.  image1, image2: CUDA float32 (h, w, c) or (N, h, w, c), h, w >= 161, c in 1..4.
  Returns a 0-d or (N,) tensor on the device (the mean over channels, like TF)."""
  _check_images(image1, image2, 'compute_multiscale_ssim')
  batched = image1.dim() == 4
  a, b = (image1, image2) if batched else (image1[None], image2[None])
  ssim = _image_metrics(a, b)[0]
  return ssim if batched else ssim[0]


def compute_psnr(mse):
  """utils.py:94-103: PSNR of a mean squared error for pixel values in [0, 1]."""
  if torch.is_tensor(mse):
    return -10. * torch.log(mse) / math.log(10.)
  return -10. * math.log(mse) / math.log(10.)


def compute_metrics(rgb, rgb_target, depth_med=None, depth_target=None):
  """The `out` dict of eval.py:process_batch (eval.py:118-140) from ONE library call:
  {'mse', 'psnr', 'ssim'} and, with depth, 'depth_abs'.

  rgb, rgb_target: CUDA float32 (h, w, c) or (N, h, w, c) (render_frame's 'rgb' and
  batch['rgb']); depth_med (h, w) / (N, h, w) and depth_target of the same shape or with a
  trailing 1 (datasets/core.py:610).  Values are 0-d tensors, or (N,) for a batch; per image.

  depth_abs = nanmean(|depth_target[..., 0] - depth_med|) per pixel.  This deviates from the
  reference on purpose: eval.py:140 subtracts the (h, w) depth_med from the (h, w, 1)
  depth_target, a broadcast that raises for a non-square frame and, for a square one, averages
  the (h, w, w) array of unrelated pairs."""
  _check_images(rgb, rgb_target, 'compute_metrics')
  if (depth_med is None) != (depth_target is None):
    raise ValueError('compute_metrics: pass both depth_med and depth_target, or neither')
  batched = rgb.dim() == 4
  image, target = (rgb, rgb_target) if batched else (rgb[None], rgb_target[None])
  depth = dtarget = None
  if depth_med is not None:
    shape = tuple(image.shape[:3])
    for name, t in (('depth_med', depth_med), ('depth_target', depth_target)):
      if not torch.is_tensor(t) or t.dtype != torch.float32 or t.device != rgb.device:
        raise ValueError(f'compute_metrics: {name} must be a float32 tensor on {rgb.device}')
    if tuple(depth_med.shape) not in (shape, shape[1:]) or (tuple(depth_med.shape) == shape[1:]) == batched:
      raise ValueError(f'compute_metrics: depth_med shape {tuple(depth_med.shape)} does not match rgb '
                       f'{tuple(rgb.shape)}')
    if depth_target.shape[-1:] == (1,) and depth_target.dim() == depth_med.dim() + 1:
      depth_target = depth_target[..., 0]
    if depth_target.shape != depth_med.shape:
      raise ValueError(f'compute_metrics: depth_target shape {tuple(depth_target.shape)} does not match '
                       f'depth_med {tuple(depth_med.shape)}')
    depth, dtarget = depth_med.reshape(shape), depth_target.reshape(shape)
  ssim, mse, depth_abs = _image_metrics(image, target, depth, dtarget)
  out = {'mse': mse, 'psnr': compute_psnr(mse), 'ssim': ssim}
  if depth_abs is not None:
    out['depth_abs'] = depth_abs
  return out if batched else {k: v[0] for k, v in out.items()}
