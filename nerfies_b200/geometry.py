"""A trained model's surface as a triangle mesh: the density on a 3D grid through the render
kernels, marching cubes in CUDA (include/nerfies_b200.h, nfb_marching_cubes*), vertex colours and
a binary PLY writer; the inverse of the warp field (nfb_warp_invert), which carries the template mesh
into a frame with its topology; and pixels followed from one frame into others through the warp field
with a visibility test (nfb_point_visibility, track_pixels).  No reference analogue: the reference
renders images only.

Grids are (nz, ny, nx) float32 on the device, x fastest; a box ((x0, y0, z0), (x1, y1, z1)) holds the
grid's first and last points on each axis, so value [k, j, i] lies at box[0] + (i, j, k) * spacing with
spacing = (box[1] - box[0]) / (shape - 1).  Each grid point is float32(box[0]) + float32(index) *
float32(spacing), each operation rounded once: the same points marching cubes places its vertices
between.
"""
import ctypes

import numpy as np
import torch

from nerfies_b200 import _lib
from nerfies_b200 import evaluation
from nerfies_b200.models import _ptr, _stream

LEVELS = {'coarse': 0, 'fine': 1}


def grid_spacing(bbox, shape):
  """float32 (3,) spacing (x, y, z) of a grid of `shape` (nz, ny, nx) spanning `bbox`."""
  lo, hi = (np.asarray(b, np.float64) for b in bbox)
  n = np.array(shape[::-1], np.float64)
  return ((hi - lo) / (n - 1)).astype(np.float32)


def _check_box(bbox, shape):
  if len(shape) != 3 or any(int(s) < 2 for s in shape):
    raise ValueError(f'grid shape {tuple(shape)}: expected (nz, ny, nx) with every side >= 2')
  lo, hi = (np.asarray(b, np.float64) for b in bbox)
  if lo.shape != (3,) or hi.shape != (3,) or not np.all(hi > lo) or not np.all(np.isfinite(lo) & np.isfinite(hi)):
    raise ValueError(f'bbox {bbox}: expected ((x0, y0, z0), (x1, y1, z1)) with x1 > x0, y1 > y0, z1 > z0')


def _axis_points(lo, spacing, n, dev):
  """float32(lo) + float32(i) * float32(spacing) for i < n, each operation rounded once."""
  return (torch.arange(n, device=dev, dtype=torch.float32) * float(spacing)) + float(np.float32(lo))


def _metadata_ids(model, metadata, n):
  """(warp_id, app_id, cam_id) device tensors of n rays from scalar metadata, as models.apply reads them."""
  md = metadata or {}
  return (_warp_ids(model, md, n), _ids(model, md, 'appearance', model.use_appearance_metadata, n),
          _ids(model, md, 'camera', model.use_camera_metadata, n))


def _ids(model, md, key, used, n):
  if not used:
    return None
  if key not in md:
    raise KeyError(f"metadata['{key}'] is required by this model")
  return torch.full((n,), int(md[key]), dtype=torch.int32, device=model.device)


def _warp_ids(model, md, n):
  """The warp metadata of n rays or points: float timestamps with the 'time' encoder, ids otherwise."""
  if model.use_warp and model.warp_metadata_encoder_type == 'time':
    if 'time' not in md:
      raise KeyError("metadata['time'] is required by this model")
    return torch.full((n,), float(md['time']), dtype=torch.float32, device=model.device)
  return _ids(model, md, 'warp', model.use_warp, n)


def _prepare(model, params, warp_extra, use_warp, level):
  if level not in LEVELS:
    raise ValueError(f"level must be 'coarse' or 'fine', got {level!r}")
  if level == 'fine' and model.num_fine_samples <= 0:
    raise ValueError("level='fine': this model has no fine level")
  hd = model.handle()
  hd.set_params(params)
  warp_extra = warp_extra or {}
  model._set_time_alpha(hd, warp_extra.get('time_alpha'))
  flags = 0 if (use_warp and model.use_warp) else _lib.FLAG_NO_WARP
  return hd, float(warp_extra.get('alpha', 0.0)), flags, LEVELS[level]


def density_grid(model, params, bbox, shape, warp_extra=None, metadata=None, use_warp=True, level='fine'):
  """The density sigma of `level`'s NeRF MLP at every point of a (nz, ny, nx) grid over `bbox`:
  with use_warp, of the frame the metadata names (its observation space, warped into the template
  by the warp field); without, of the canonical template.

  Each (k, j) row of the grid is one ray along +x from its first point with z values i * spacing_x,
  rendered by nfb_render_samples with the per-sample outputs only.  Calls are chunked to at most the
  handle's max_rays rows and its warped-point workspace, so no call allocates."""
  _check_box(bbox, shape)
  nz, ny, nx = (int(s) for s in shape)
  hd, alpha, flags, lv = _prepare(model, params, warp_extra, use_warp, level)
  dev = model.device
  sx, sy, sz = (float(s) for s in grid_spacing(bbox, shape))
  lo = bbox[0]
  lines = nz * ny
  per_call = hd.max_rays
  if flags != _lib.FLAG_NO_WARP and model.use_warp:
    smax = model.num_coarse_samples + model.num_fine_samples if model.num_fine_samples > 0 else model.num_coarse_samples
    per_call = min(per_call, max(1, hd.max_rays * smax // nx))
  per_call = min(per_call, lines)
  y = _axis_points(lo[1], sy, ny, dev)
  z = _axis_points(lo[2], sz, nz, dev)
  z_row = _axis_points(0.0, sx, nx, dev)
  warp_id, app_id, cam_id = _metadata_ids(model, metadata, per_call)
  grid = torch.empty(nz, ny, nx, device=dev)
  flat = grid.view(lines, nx)
  z_vals = z_row.expand(per_call, nx).contiguous()
  directions = torch.zeros(per_call, 3, device=dev)
  directions[:, 0] = 1.0
  samples = torch.empty(per_call, nx, 4, device=dev)
  x0 = float(np.float32(lo[0]))
  with torch.cuda.device(dev):
    for first in range(0, lines, per_call):
      B = min(per_call, lines - first)
      rows = torch.arange(first, first + B, device=dev)
      origins = torch.stack([torch.full((B,), x0, device=dev), y[rows % ny], z[rows // ny]], -1).contiguous()
      _lib.check(hd.lib.nfb_render_samples(
          hd.h, lv, B, nx, _ptr(z_vals), _ptr(origins), _ptr(directions), None, _ptr(warp_id), _ptr(app_id),
          _ptr(cam_id), alpha, flags, None, None, _ptr(samples), None, _stream()))
      flat[first:first + B] = samples[:B, :, 3]
  return grid


def vertex_colors(model, params, vertices, normals, warp_extra=None, metadata=None, use_warp=True,
                  level='fine', axes=None):
  """float32 (V, 3) colour of each vertex: sigmoid(rgb) of `level`'s NeRF MLP at the vertex, seen
  along -normal (one ray per vertex, one sample at z = 0, from the vertex toward the inside).  A
  vertex whose normal is zero looks along its edge's axis, which `axes` ((V,) 0 | 1 | 2, as
  marching_cubes(..., return_axes=True) gives) must then provide."""
  if vertices.dim() != 2 or vertices.shape[-1] != 3 or normals.shape != vertices.shape:
    raise ValueError(f'vertices and normals must both be (V, 3), got {tuple(vertices.shape)} and '
                     f'{tuple(normals.shape)}')
  hd, alpha, flags, lv = _prepare(model, params, warp_extra, use_warp, level)
  dev = model.device
  V = vertices.shape[0]
  colors = torch.empty(V, 3, device=dev)
  if V == 0:
    return colors
  directions = -normals.to(device=dev, dtype=torch.float32)
  zero = (normals == 0).all(-1)
  if bool(zero.any()):
    if axes is None:
      raise ValueError('vertex_colors: some normals are zero; pass the vertices\' edge axes (axes=...)')
    directions[zero] = torch.nn.functional.one_hot(axes.to(dev)[zero].long(), 3).float()
  origins = vertices.to(device=dev, dtype=torch.float32).contiguous()
  directions = directions.contiguous()
  per_call = min(hd.max_rays, V)
  z_vals = torch.zeros(per_call, 1, device=dev)
  samples = torch.empty(per_call, 1, 4, device=dev)
  warp_id, app_id, cam_id = _metadata_ids(model, metadata, per_call)
  with torch.cuda.device(dev):
    for first in range(0, V, per_call):
      B = min(per_call, V - first)
      _lib.check(hd.lib.nfb_render_samples(
          hd.h, lv, B, 1, _ptr(z_vals), _ptr(origins[first:]), _ptr(directions[first:]), None, _ptr(warp_id),
          _ptr(app_id), _ptr(cam_id), alpha, flags, None, None, _ptr(samples), None, _stream()))
      colors[first:first + B] = samples[:B, 0, :3]
  return colors


def density_gradient(model, params, points, warp_extra=None, metadata=None, use_warp=True, level='fine'):
  """The density sigma of `level`'s NeRF MLP at free points (P, 3) and its gradient with respect to the
  points (nfb_density_grad): with use_warp, of the frame the metadata names (grad_x sigma(W(x)) =
  J_W(x)^T grad_y sigma(y), y = W(x)); without, of the canonical template.  Forward mode through the warp
  field and the NeRF trunk in the model's training precision (fp32 or tf32x3); a relu's derivative at 0
  is 0.  Metadata as density_grid: 'warp' (or 'time') and 'appearance' where the model reads them; the
  camera code and view directions do not reach sigma.
  Returns {'sigma' (P,), 'gradient' (P, 3), 'warped_points' (P, 3) (the points themselves without a
  warp)}, plain float32 tensors on the model's device: parameters that require grad give them no
  grad_fn, and nothing is differentiated through them."""
  hd, alpha, flags, lv = _prepare(model, params, warp_extra, use_warp, level)
  dev = model.device
  points = _f32(points, dev, 3, 'density_gradient: points')
  P = points.shape[0]
  md = metadata or {}
  warp_id = _warp_ids(model, md, P) if flags != _lib.FLAG_NO_WARP else None
  app_id = _ids(model, md, 'appearance', model.use_appearance_metadata, P)
  out = {'sigma': torch.empty(P, device=dev), 'gradient': torch.empty(P, 3, device=dev),
         'warped_points': torch.empty(P, 3, device=dev)}
  if P == 0:
    return out
  with torch.cuda.device(dev):
    _lib.check(hd.lib.nfb_density_grad(hd.h, lv, P, _ptr(points), _ptr(warp_id), _ptr(app_id), alpha, flags,
                                       _ptr(out['sigma']), _ptr(out['gradient']), _ptr(out['warped_points']),
                                       _stream()))
  return out


def normal_map(model, params, camera, depth, warp_extra=None, metadata=None, level='fine'):
  """World-frame surface normals of a frame: at each pixel's point x = o + depth * d (the rays of
  `camera`), n = -grad sigma / |grad sigma| of `level`'s NeRF MLP in the frame the metadata names
  (density_gradient).  `depth` (H, W) is render_frame's 'med_depth', whose 0 marks a ray with no
  surface.  A pixel is valid where depth > 0 and the gradient is finite and nonzero; invalid pixels
  get 0.  Returns {'normals' (H, W, 3), 'valid' (H, W) bool} on the model's device."""
  from nerfies_b200 import camera as camera_lib
  dev = model.device
  h, w = camera.image_shape
  depth = torch.as_tensor(depth).to(device=dev, dtype=torch.float32)
  if tuple(depth.shape) != (h, w):
    raise ValueError(f'normal_map: depth must be the frame\'s (H, W) = ({h}, {w}), got {tuple(depth.shape)}')
  rays = camera_lib.camera_to_rays(camera, dev)
  hit = (depth > 0).reshape(-1)
  points = (rays['origins'] + depth[..., None] * rays['directions']).reshape(-1, 3)[hit]
  grad = density_gradient(model, params, points, warp_extra, metadata, use_warp=True, level=level)['gradient']
  norm = grad.norm(dim=-1)
  ok = torch.isfinite(grad).all(-1) & torch.isfinite(norm) & (norm > 0)
  normals = torch.zeros(h * w, 3, device=dev)
  valid = torch.zeros(h * w, dtype=torch.bool, device=dev)
  normals[hit] = torch.where(ok[:, None], -grad / torch.where(ok, norm, 1.0)[:, None], 0.0)
  valid[hit] = ok
  return {'normals': normals.reshape(h, w, 3), 'valid': valid.reshape(h, w)}


def invert_warp(model, params, targets, warp_extra=None, metadata=None, init=None, max_iters=16, tol=1e-5,
                return_jacobian=False):
  """The points x of the frame the metadata names whose warp W(x) is `targets` (P, 3) template points
  (nfb_warp_invert: damped Newton on the warp field and its Jacobian, from `init` or the targets).
  Returns {'points' (P, 3), 'residual' (P,) |W(points) - targets|, 'status' (P,) int32
  (_lib.INVERT_STATUS)[, 'jacobian' (P, 3, 3) J at points]}, all on the model's device.  Only points
  whose status is converged are within `tol` of a preimage; the others hold the best iterate found."""
  if not model.use_warp:
    raise ValueError('invert_warp: the model has no warp field')
  dev = model.device
  targets = torch.as_tensor(targets).to(device=dev, dtype=torch.float32).contiguous()
  if targets.dim() != 2 or targets.shape[-1] != 3:
    raise ValueError(f'invert_warp: targets must be (P, 3), got {tuple(targets.shape)}')
  P = targets.shape[0]
  if init is not None:
    init = torch.as_tensor(init).to(device=dev, dtype=torch.float32).contiguous()
    if init.shape != targets.shape:
      raise ValueError(f'invert_warp: init must be {tuple(targets.shape)}, got {tuple(init.shape)}')
  hd, alpha, _, _ = _prepare(model, params, warp_extra, True, 'coarse')
  warp_id = _warp_ids(model, metadata or {}, P)
  out = {'points': torch.empty(P, 3, device=dev), 'residual': torch.empty(P, device=dev),
         'status': torch.empty(P, dtype=torch.int32, device=dev)}
  jac = torch.empty(P, 3, 3, device=dev) if return_jacobian else None
  if P == 0:
    return dict(out, jacobian=jac) if return_jacobian else out
  with torch.cuda.device(dev):
    _lib.check(hd.lib.nfb_warp_invert(hd.h, P, _ptr(targets), _ptr(init), _ptr(warp_id), alpha, int(max_iters),
                                      float(tol), _ptr(out['points']), _ptr(out['residual']), _ptr(jac),
                                      _ptr(out['status']), _stream()))
  if return_jacobian:
    out['jacobian'] = jac
  return out


def track_surface(model, params, vertices, normals, warp_extra, metadata, init=None, tol=1e-5, max_iters=16):
  """A template mesh's vertices (V, 3) and outward normals carried into the frame the metadata names:
  the vertices are invert_warp's points, the normals normalize(J^T n), the gradient direction of
  sigma_template(W(x)) (zero where n is).  Where det J <= 0 the warp folds locally and the faces'
  winding flips there; such vertices are counted ('folded'), not repaired.
  Returns {'vertices', 'normals', 'residual', 'status', 'folded' (int)}."""
  if vertices.dim() != 2 or vertices.shape[-1] != 3 or normals.shape != vertices.shape:
    raise ValueError(f'vertices and normals must both be (V, 3), got {tuple(vertices.shape)} and '
                     f'{tuple(normals.shape)}')
  inv = invert_warp(model, params, vertices, warp_extra, metadata, init=init, max_iters=max_iters, tol=tol,
                    return_jacobian=True)
  J = inv['jacobian']
  n = normals.to(device=J.device, dtype=torch.float32)
  moved = torch.nn.functional.normalize((J.transpose(1, 2) @ n.unsqueeze(-1)).squeeze(-1), dim=-1)
  folded = int((torch.linalg.det(J.double()) <= 0).sum()) if len(J) else 0
  return {'vertices': inv['points'], 'normals': moved, 'residual': inv['residual'], 'status': inv['status'],
          'folded': folded}


def default_depth_tol(model):
  """One coarse sample step, (far - near) / num_coarse_samples: the depth band of point_visibility."""
  return (model.far - model.near) / model.num_coarse_samples


def _f32(t, dev, shape_last, what):
  t = torch.as_tensor(t).to(device=dev, dtype=torch.float32).contiguous()
  if t.dim() != 2 or t.shape[-1] != shape_last:
    raise ValueError(f'{what} must be (N, {shape_last}), got {tuple(t.shape)}')
  return t


def point_visibility(model, params, points, warp_extra, metadata, camera, depth_tol=None, invert_status=None):
  """Whether `camera` sees the observation-space points (P, 3) of the frame the metadata names
  (nfb_point_visibility): each point's projection, its distance from the camera and the median depth of
  the deterministic render of the ray from the camera through it.  depth_tol defaults to
  default_depth_tol; invert_status (P,) int32 (invert_warp's 'status') marks points whose inversion did
  not converge as unresolved.  Returns {'pixels' (P, 2), 'depth' (P, 2) (dist, med), 'status' (P,) int32
  (_lib.TRACK_STATUS)}, all on the model's device."""
  dev = model.device
  points = _f32(points, dev, 3, 'point_visibility: points')
  P = points.shape[0]
  if invert_status is not None:
    invert_status = torch.as_tensor(invert_status).to(device=dev, dtype=torch.int32).contiguous()
    if invert_status.shape != (P,):
      raise ValueError(f'point_visibility: invert_status must be ({P},), got {tuple(invert_status.shape)}')
  depth_tol = default_depth_tol(model) if depth_tol is None else float(depth_tol)
  hd, alpha, flags, _ = _prepare(model, params, warp_extra, True, 'coarse')
  warp_id, app_id, cam_id = _metadata_ids(model, metadata, P)
  out = {'pixels': torch.empty(P, 2, device=dev), 'depth': torch.empty(P, 2, device=dev),
         'status': torch.empty(P, dtype=torch.int32, device=dev)}
  if P == 0:
    return out
  with torch.cuda.device(dev):
    _lib.check(hd.lib.nfb_point_visibility(
        hd.h, P, _ptr(points), _ptr(warp_id), _ptr(app_id), _ptr(cam_id), alpha, flags,
        ctypes.byref(camera._struct()), depth_tol, _ptr(invert_status), _ptr(out['pixels']), _ptr(out['depth']),
        _ptr(out['status']), _stream()))
  return out


def pixel_grid(camera, stride, device):
  """Every `stride`-th pixel centre of the frame, (ceil(h / stride) * ceil(w / stride), 2) float32, x
  fastest."""
  if int(stride) < 1:
    raise ValueError(f'stride must be >= 1, got {stride}')
  h, w = camera.image_shape
  y = torch.arange(0, h, int(stride), device=device, dtype=torch.float32) + 0.5
  x = torch.arange(0, w, int(stride), device=device, dtype=torch.float32) + 0.5
  return torch.stack(torch.meshgrid(x, y, indexing='xy'), -1).reshape(-1, 2)


def _ray_metadata(metadata, n, dev):
  """rays_dict['metadata'] of n rays from scalar metadata, as evaluation.render_frame builds it."""
  return {k: (torch.full((n, 1), float(v), dtype=torch.float32, device=dev) if k == 'time'
              else torch.full((n, 1), int(v), dtype=torch.int32, device=dev)) for k, v in (metadata or {}).items()}


def source_points(model, params, camera, warp_extra, metadata, pixels=None, stride=1):
  """The surface points seen at pixels of the frame the camera and metadata name: `pixels` (Q, 2), or
  every `stride`-th pixel centre (pixel_grid).  Each pixel's ray (nfb_pixels_to_rays) is rendered on
  the deterministic path and its point is o + med * d, with med the median depth of the last level:
  the depth point_visibility measures, so a pixel tracked into its own frame is visible by
  construction (the expected depth blends foreground and background at silhouettes).
  Returns {'pixels' (Q, 2), 'points' (Q, 3) observation space, 'template' (Q, 3) (nfb_warp_forward of
  the points; the points themselves without a warp field), 'has_surface' (Q,) bool (med > 0)}."""
  dev = model.device
  pixels = pixel_grid(camera, stride, dev) if pixels is None else _f32(pixels, dev, 2, 'source_points: pixels')
  Q = pixels.shape[0]
  directions = camera.pixels_to_rays(pixels) if Q else torch.empty(0, 3, device=dev)
  origin = torch.as_tensor(camera.position, dtype=torch.float32, device=dev)
  med = torch.empty(Q, device=dev)
  per_call = model.handle().max_rays
  level = 'fine' if model.num_fine_samples > 0 else 'coarse'
  with torch.no_grad():
    for first in range(0, Q, per_call):
      n = min(per_call, Q - first)
      rays = {'origins': origin.expand(n, 3).contiguous(), 'directions': directions[first:first + n],
              'metadata': _ray_metadata(metadata, n, dev)}
      out = model.apply({'params': params}, rays, warp_extra=warp_extra, _packed=True)
      med[first:first + n] = out[level][:, 4]
  points = (origin + med[:, None] * directions).contiguous()
  template = points.clone()
  if model.use_warp and Q:
    hd, alpha, _, _ = _prepare(model, params, warp_extra, True, 'coarse')
    warp_id = _warp_ids(model, metadata or {}, min(Q, hd.max_rays))
    with torch.cuda.device(dev):
      for first in range(0, Q, hd.max_rays):
        n = min(hd.max_rays, Q - first)
        _lib.check(hd.lib.nfb_warp_forward(hd.h, n, _ptr(points[first:]), _ptr(warp_id), alpha, 0,
                                           _ptr(template[first:]), _stream()))
  return {'pixels': pixels, 'points': points, 'template': template, 'has_surface': med > 0}


def track_points(model, params, template_points, warp_extra, metadata, camera, init=None, max_iters=16, tol=1e-5,
                 depth_tol=None):
  """Template points (Q, 3) placed in the frame the camera and metadata name and tested for visibility
  there: invert_warp (skipped without a warp field, where the template is the observation space), then
  point_visibility with the inversion's status.  Returns {'points' (Q, 3), 'pixels' (Q, 2), 'residual'
  (Q,) (zero without a warp field), 'status' (Q,) int32 (_lib.TRACK_STATUS), 'depth' (Q, 2),
  'invert_status' (Q,) int32 or None}."""
  dev = model.device
  template_points = _f32(template_points, dev, 3, 'track_points: template_points')
  if model.use_warp:
    inv = invert_warp(model, params, template_points, warp_extra, metadata, init=init, max_iters=max_iters, tol=tol)
    points, residual, inv_status = inv['points'], inv['residual'], inv['status']
  else:
    points, residual, inv_status = template_points, torch.zeros(len(template_points), device=dev), None
  vis = point_visibility(model, params, points, warp_extra, metadata, camera, depth_tol, inv_status)
  return {'points': points, 'pixels': vis['pixels'], 'residual': residual, 'status': vis['status'],
          'depth': vis['depth'], 'invert_status': inv_status}


def track_pixels(model, params, warp_extra, source, targets, pixels=None, stride=1, max_iters=16, tol=1e-5,
                 depth_tol=None):
  """Pixels of a source frame followed into each target frame; `source` and each target are (camera,
  metadata) pairs.  The source's surface points and their template points are computed once
  (source_points); each target is then track_points, its inversion warm-started from the previous
  target's solution where that converged and from the source point elsewhere.  Source pixels without a
  surface (median depth 0) get the status 'no_surface' in every target.
  Returns {'source_pixels' (Q, 2), 'source_points' (Q, 3), 'has_surface' (Q,), and stacked over the T
  targets 'pixels' (T, Q, 2), 'points' (T, Q, 3), 'residual' (T, Q), 'status' (T, Q) int32, 'depth'
  (T, Q, 2)}, on the model's device."""
  src_camera, src_md = source
  src = source_points(model, params, src_camera, warp_extra, src_md, pixels, stride)
  no_surface = ~src['has_surface']
  keys = ('pixels', 'points', 'residual', 'status', 'depth')
  rows = {k: [] for k in keys}
  prev, converged = None, None
  for camera, md in targets:
    init = src['points'] if converged is None else torch.where(converged[:, None], prev, src['points'])
    t = track_points(model, params, src['template'], warp_extra, md, camera, init=init, max_iters=max_iters, tol=tol,
                     depth_tol=depth_tol)
    t['status'] = torch.where(no_surface, _lib.TRACK_STATUS['no_surface'], t['status']).to(torch.int32)
    if t['invert_status'] is not None:
      prev, converged = t['points'], t['invert_status'] == _lib.INVERT_STATUS['converged']
    for k in keys:
      rows[k].append(t[k])
  Q = len(src['pixels'])
  empty = {'pixels': (Q, 2), 'points': (Q, 3), 'residual': (Q,), 'status': (Q,), 'depth': (Q, 2)}
  out = {k: torch.stack(v) if v else torch.empty((0,) + empty[k], device=model.device,
                                                 dtype=torch.int32 if k == 'status' else torch.float32)
         for k, v in rows.items()}
  return dict(out, source_pixels=src['pixels'], source_points=src['points'], has_surface=src['has_surface'])


def marching_cubes(grid, level, bbox, return_axes=False):
  """Surface {grid > level} of a (nz, ny, nx) float32 CUDA grid over `bbox` (nfb_marching_cubes):
  vertices (V, 3) float32, faces (F, 3) int32 (counter-clockwise seen from outside) and outward unit
  normals (V, 3) float32 (zero where the gradient is), all on the grid's device.  With return_axes,
  also each vertex's edge axis (V,) uint8."""
  if not torch.is_tensor(grid) or grid.device.type != 'cuda':
    raise ValueError('marching_cubes: grid must be a CUDA tensor')
  if grid.dtype != torch.float32:
    raise ValueError(f'marching_cubes: grid must be float32, got {grid.dtype}')
  if grid.dim() != 3:
    raise ValueError(f'marching_cubes: grid must be (nz, ny, nx), got shape {tuple(grid.shape)}')
  if not grid.is_contiguous():
    raise ValueError('marching_cubes: grid must be contiguous')
  _check_box(bbox, grid.shape)
  nz, ny, nx = grid.shape
  lib = _lib.load()
  dev = grid.device
  spacing = grid_spacing(bbox, grid.shape)
  origin = np.asarray(bbox[0], np.float32)
  f3 = lambda a: (ctypes.c_float * 3)(*[float(v) for v in a])
  with torch.cuda.device(dev):
    need = lib.nfb_marching_cubes_workspace_size(nx, ny, nz)
    if need < 0:
      raise _lib.NfbError(lib.nfb_last_error().decode())
    workspace = torch.empty(need, dtype=torch.uint8, device=dev)
    counts = torch.empty(4, dtype=torch.int64, device=dev)
    _lib.check(lib.nfb_marching_cubes_count(_ptr(grid), nx, ny, nz, float(level), _ptr(workspace), need,
                                            _ptr(counts), _stream()))
    V, F, y_first, z_first = counts.tolist()
    if V > 2**31 - 1 or F > 2**31 - 1:
      raise ValueError(f'marching_cubes: {V} vertices and {F} faces do not fit int32 indices')
    vertices = torch.empty(V, 3, device=dev)
    normals = torch.empty(V, 3, device=dev)
    faces = torch.empty(F, 3, dtype=torch.int32, device=dev)
    _lib.check(lib.nfb_marching_cubes(_ptr(grid), nx, ny, nz, float(level), f3(origin), f3(spacing),
                                      _ptr(workspace), need, _ptr(vertices), _ptr(normals), _ptr(faces),
                                      _stream()))
  if not return_axes:
    return vertices, faces, normals
  axes = torch.zeros(V, dtype=torch.uint8, device=dev)
  axes[y_first:z_first] = 1
  axes[z_first:] = 2
  return vertices, faces, normals, axes


def write_ply(path, vertices, faces, normals=None, colors=None):
  """Binary little-endian PLY: vertices `float x y z`, then `float nx ny nz` with normals and
  `uchar red green blue` with colors (uint8, or a float32 CUDA tensor in [0, 1] that
  evaluation.image_to_uint8 quantizes);
  faces `list uchar int vertex_indices`.  An empty mesh is a valid file."""
  v = _host(vertices, np.float32, 'vertices')
  f = _host(faces, np.int32, 'faces')
  cols = [('x', '<f4'), ('y', '<f4'), ('z', '<f4')]
  parts = [v]
  if normals is not None:
    n = _host(normals, np.float32, 'normals')
    if n.shape != v.shape:
      raise ValueError(f'normals must be {v.shape}, got {n.shape}')
    cols += [('nx', '<f4'), ('ny', '<f4'), ('nz', '<f4')]
    parts.append(n)
  if colors is not None:
    if tuple(colors.shape) != v.shape:
      raise ValueError(f'colors must be {v.shape}, got {tuple(colors.shape)}')
    if colors.dtype in (np.uint8, torch.uint8):
      c = _host(colors, np.uint8, 'colors')
    else:
      c = evaluation.image_to_uint8(colors).cpu().numpy()
    cols += [('red', 'u1'), ('green', 'u1'), ('blue', 'u1')]
    parts.append(c)
  rows = np.empty(len(v), dtype=np.dtype(cols))
  k = 0
  for p in parts:
    for i in range(3):
      rows[cols[k][0]] = p[:, i]
      k += 1
  tri = np.empty(len(f), dtype=np.dtype([('n', 'u1'), ('i', '<i4', (3,))]))
  tri['n'] = 3
  tri['i'] = f
  header = ['ply', 'format binary_little_endian 1.0', f'element vertex {len(v)}']
  header += [f'property {"float" if t == "<f4" else "uchar"} {name}' for name, t in cols]
  header += [f'element face {len(f)}', 'property list uchar int vertex_indices', 'end_header']
  with open(path, 'wb') as out:
    out.write(('\n'.join(header) + '\n').encode('ascii'))
    out.write(rows.tobytes())
    out.write(tri.tobytes())


def _host(t, dtype, what):
  a = t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)
  a = np.ascontiguousarray(a.reshape(-1, 3) if a.size == 0 else a, dtype=dtype)
  if a.ndim != 2 or a.shape[1] != 3:
    raise ValueError(f'{what} must be (N, 3), got {a.shape}')
  return a



# ---------------------------------------------------------------------------
# Camera registration (iNeRF-style): fit a camera pose, and the photo's codes, to a photo by gradient descent
# on the photometric loss through NerfModel.render_rays (nfb_render_ray_vjp).
# ---------------------------------------------------------------------------
OPTIMIZE = ('pose', 'appearance', 'camera', 'warp')
# the camera intrinsics parts a registration can also fit (register_camera's `intrinsics`, kept apart from
# `optimize`): 'focal', 'principal_point', 'radial', 'tangential'
INTRINSICS_PARTS = tuple(_lib.INTRINSICS_PARTS)
# the intrinsics parts' rates are for the entries of the delta (refined_camera): the focal log-scale, the
# principal point in focal lengths and the distortion coefficients
DEFAULT_LRS = {'rotation': 2e-3, 'position': 2e-3, 'appearance': 1e-2, 'camera': 1e-2, 'warp': 1e-2,
               'focal': 1e-3, 'principal_point': 1e-4, 'radial': 1e-3, 'tangential': 1e-4}


def _skew(w):
  z = torch.zeros((), dtype=w.dtype, device=w.device)
  return torch.stack([torch.stack([z, -w[2], w[1]]), torch.stack([w[2], z, -w[0]]),
                      torch.stack([-w[1], w[0], z])])


def rotvec_to_matrix(w):
  """exp([w]x) of a (3,) rotation vector (Rodrigues, differentiable, in w's dtype):
  I + sin(t)/t K + 2 sin^2(t/2)/t^2 K^2 with t = |w|, K = [w]x; below t^2 = 1e-4 both factors are their
  Taylor series to t^4 (the remainder is below fp32 rounding), so w = 0 has a gradient."""
  t2 = (w * w).sum()
  small = t2 < 1e-4
  t = torch.sqrt(torch.where(small, torch.ones_like(t2), t2))
  a = torch.where(small, 1 - t2 / 6 + t2 * t2 / 120, torch.sin(t) / t)
  h = torch.sin(t / 2)
  b = torch.where(small, 0.5 - t2 / 24 + t2 * t2 / 720, 2 * h * h / (t * t))
  K = _skew(w)
  return torch.eye(3, dtype=w.dtype, device=w.device) + a * K + b * (K @ K)


def pose_rays(local, orientation, position, omega, offset):
  """Rays of camera-frame unit directions `local` (N,3) under the pose (omega, offset) applied to a camera
  with world-to-camera rotation `orientation` (R0) and centre `position` (p0): a rotation by omega about
  the camera centre in the world frame and a move of the centre by offset.
    directions = exp(omega) R0^T local,  origins = p0 + offset."""
  R = rotvec_to_matrix(omega)
  directions = (local @ orientation) @ R.T
  origins = (position + offset).expand_as(directions)
  return origins, directions


def posed_camera(camera, omega, offset):
  """The Camera of pose_rays: orientation R0 exp(omega)^T, position p0 + offset (float64, stored float32)."""
  R = rotvec_to_matrix(torch.as_tensor(omega, dtype=torch.float64).detach().cpu()).numpy()
  out = camera.copy()
  out.orientation = (camera.orientation.astype(np.float64) @ R.T).astype(np.float32)
  out.position = (camera.position.astype(np.float64) +
                  np.asarray(torch.as_tensor(offset).detach().cpu(), np.float64)).astype(np.float32)
  return out


def refined_camera(camera, delta):
  """The Camera of an intrinsics delta q = (s, dcx, dcy, dk1, dk2, dk3, dp1, dp2) (nfb_gather_rays_refined):
  focal f0 exp(s), principal point c0 + f0 dc, radial k0 + dk, tangential p0 + dp (float64, stored float32).
  The delta does not depend on the image scale: a camera scaled by Camera.scale and then refined is the
  refined camera scaled."""
  q = np.asarray(torch.as_tensor(delta).detach().cpu(), np.float64).reshape(8)
  f0 = float(camera.focal_length)
  out = camera.copy()
  out.focal_length = np.array(f0 * np.exp(q[0]), np.float32)
  out.principal_point = (camera.principal_point.astype(np.float64) + f0 * q[1:3]).astype(np.float32)
  out.radial_distortion = (camera.radial_distortion.astype(np.float64) + q[3:6]).astype(np.float32)
  out.tangential_distortion = (camera.tangential_distortion.astype(np.float64) + q[6:8]).astype(np.float32)
  return out


class _RefinedDirections(torch.autograd.Function):
  """Camera-frame directions of pixel positions under an intrinsics delta: forward nfb_pixels_to_rays_refined
  of the identity-pose camera, backward nfb_intrinsics_grad with one image and one group."""

  @staticmethod
  def forward(ctx, delta, pixels, camera, parts):
    lib = _lib.load()
    dev = pixels.device
    delta = delta.detach().to(torch.float32).contiguous()
    out = torch.empty(pixels.shape[0], 3, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
      _lib.check(lib.nfb_pixels_to_rays_refined(ctypes.byref(camera._struct()), _ptr(delta), _ptr(pixels),
                                                pixels.shape[0], _ptr(out), _stream()))
    ctx.save_for_backward(delta, pixels, out)
    ctx.camera, ctx.parts = camera, parts
    return out

  @staticmethod
  def backward(ctx, grad_out):
    delta, pixels, out = ctx.saved_tensors
    lib = _lib.load()
    dev, n = pixels.device, pixels.shape[0]
    cams = torch.frombuffer(bytearray(bytes(ctx.camera._struct())), dtype=torch.uint8).to(dev)
    zeros = torch.zeros(n, dtype=torch.int32, device=dev)
    grad = torch.zeros(8, dtype=torch.float32, device=dev)
    ws = torch.empty(int(lib.nfb_intrinsics_grad_workspace_size(1, n)), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
      _lib.check(lib.nfb_intrinsics_grad(_ptr(cams), 1, None, _ptr(delta), _ptr(zeros), 1, ctx.parts, _ptr(zeros),
                                         _ptr(pixels), _ptr(out), _ptr(grad_out.to(torch.float32).contiguous()), n,
                                         _ptr(grad), _ptr(ws), ws.numel(), _stream()))
    return grad, None, None, None


def refined_directions(camera, delta, pixels, parts):
  """Unit directions (N,3) in `camera`'s frame of float32 pixel positions (N,2) on the device, with the camera
  refined by the (8,) delta (refined_camera); differentiable in `delta` for the entries of `parts` (names of
  _lib.INTRINSICS_PARTS) and no others."""
  ident = camera.copy()
  ident.orientation = np.eye(3, dtype=np.float32)
  ident.position = np.zeros(3, np.float32)
  bits = sum(_lib.INTRINSICS_PARTS[p] for p in parts)
  return _RefinedDirections.apply(delta, pixels.reshape(-1, 2).to(torch.float32).contiguous(), ident, bits)


def photometric_loss(out, target):
  """training.py's rgb loss: the mean squared error of each level's rgb, summed over the levels."""
  return sum(((lv['rgb'] - target)**2).mean() for lv in out.values())


def registration_codes(model, params, metadata, warp_extra=None):
  """The codes a registration starts from, as (1, width) float32 tensors on the model's device: the
  embedding rows `metadata` names ({'appearance': id, 'camera': id, 'warp': id}) and, with a 'time' /
  'blend' warp encoder, the warp code of metadata['time'] / metadata['warp'] at warp_extra's time_alpha
  (nfb_warp_code: the TimeEncoder's output, or its blend with the GLO row).  An id outside its table
  raises ValueError."""
  metadata = metadata or {}
  codes = {}

  def row(key, table):
    node = params
    for part in table + ('embed', 'embedding'):
      node = node[part]
    i = int(metadata[key])
    if not 0 <= i < node.shape[0]:
      raise ValueError(f"metadata['{key}'] = {i}: outside the {node.shape[0]} rows of its embedding table")
    return node[i:i + 1].detach().to(device=model.device, dtype=torch.float32).clone()

  enc = model.warp_metadata_encoder_type
  for key, used in (('warp', model.use_warp), ('appearance', model.use_appearance_metadata),
                    ('camera', model.use_camera_metadata)):
    need = 'time' if key == 'warp' and used and enc == 'time' else key
    if used and need not in metadata:
      raise KeyError(f"metadata['{need}'] is required by this model")
  if model.use_warp:
    if enc == 'glo':
      codes['warp'] = row('warp', ('warp_field', 'metadata_encoder'))
    else:
      if enc == 'blend':
        row('warp', ('warp_field', 'glo_encoder'))                  # the id's range
        wid = torch.tensor([int(metadata['warp'])], dtype=torch.int32, device=model.device)
      else:
        wid = torch.tensor([float(metadata['time'])], dtype=torch.float32, device=model.device)
      hd = model.handle()
      hd.set_params(params)
      model._set_time_alpha(hd, (warp_extra or {}).get('time_alpha'))
      code = torch.empty(1, model.num_warp_features, device=model.device)
      with torch.cuda.device(model.device):
        _lib.check(hd.lib.nfb_warp_code(hd.h, 1, _ptr(wid), _ptr(code), _stream()))
      codes['warp'] = code
  if model.use_appearance_metadata:
    codes['appearance'] = row('appearance', ('appearance_encoder',))
  if model.use_camera_metadata:
    codes['camera'] = row('camera', ('camera_encoder',))
  return codes


def check_registration(model, optimize, steps, batch_rays, intrinsics=()):
  """Refuses what cannot be registered: raises ValueError.  Returns the optimised groups as a tuple.
  `intrinsics` names the camera intrinsics parts to fit (INTRINSICS_PARTS); they are not `optimize` entries."""
  optimize = tuple(optimize)
  for k in optimize:
    if k not in OPTIMIZE:
      hint = (f'; the camera intrinsics {INTRINSICS_PARTS} are fitted through intrinsics= (--intrinsics)'
              if k in INTRINSICS_PARTS else '')
      raise ValueError(f'unknown optimize entry {k!r}: expected some of {OPTIMIZE}{hint}')
  for k in intrinsics:
    if k not in INTRINSICS_PARTS:
      raise ValueError(f'unknown intrinsics part {k!r}: expected some of {INTRINSICS_PARTS}')
  if not optimize and not tuple(intrinsics):
    raise ValueError('optimize is empty: nothing to fit')
  if 'appearance' in optimize and not model.use_appearance_metadata:
    raise ValueError("optimize 'appearance': the model has no appearance metadata")
  if 'camera' in optimize and not model.use_camera_metadata:
    raise ValueError("optimize 'camera': the model has no camera metadata")
  time_enc = model.use_warp and model.warp_metadata_encoder_type != 'glo'
  if 'warp' in optimize and (not model.use_warp or time_enc):
    raise ValueError("optimize 'warp': the model has no warp field" if not model.use_warp else
                     f"optimize 'warp': the '{model.warp_metadata_encoder_type}' encoder's code is a function of "
                     'time, not a free code')
  if int(steps) < 1:
    raise ValueError(f'steps={steps}: must be >= 1')
  if int(batch_rays) < 1:
    raise ValueError(f'batch_rays={batch_rays}: must be >= 1')
  return optimize


def register_camera(model, params, camera, image, warp_extra=None, codes=None, optimize=('pose', 'appearance'),
                    steps=200, batch_rays=1024, lrs=None, seed=0, log_every=1, lr_decay=1.0, intrinsics=()):
  """Fits `camera`'s pose (and the photo's codes) to `image` (H, W, 3) float in [0, 1], the model held fixed.

  The pose is a rotation vector omega about the camera centre (world frame) and a centre offset v
  (pose_rays), both starting at 0; the codes start from the embedding rows `codes` names
  ({'appearance': id, 'camera': id, 'warp': id, or 'time': t with a 'time' warp encoder;
  registration_codes), and with a 'time' / 'blend' warp encoder the warp code stays that of the fixed time.  Each
  step draws `batch_rays` pixels uniformly from a device generator seeded with `seed`, renders them with
  deterministic sampling (as eval.py) through NerfModel.render_rays and takes one Adam step on
  photometric_loss, with the learning rate of each group in `lrs` ('rotation', 'position',
  'appearance', 'camera', 'warp', 'focal', 'principal_point', 'radial', 'tangential'; DEFAULT_LRS otherwise).
  With lr_decay < 1 each rate decays
  exponentially from its value at the first step to lr_decay times it at the last.  The camera-frame directions come from
  Camera's own ray kernel on an identity-pose copy, so distortion is the kernel's.  The parts `intrinsics`
  names (some of 'focal', 'principal_point', 'radial', 'tangential') fit an intrinsics delta (refined_camera)
  starting at 0:
  the batch's directions then come from refined_directions each step; 'radial' and 'tangential' also fit a
  camera without distortion.

  Returns (camera, codes, history): the registered Camera, the fitted codes {'appearance': (1, A), ...}
  (with an intrinsics part also 'intrinsics', the (1, 8) delta, which the returned camera already applies)
  and one dict per logged step (step, loss, psnr of the batch's fine (else coarse) level, rotation_deg
  |omega| in degrees, translation |v|, focal_change_pct 100 (exp(s) - 1), principal_point_px |f0 dc| at the
  camera's scale), before that step's update."""
  from nerfies_b200 import camera as camera_lib
  optimize = check_registration(model, optimize, steps, batch_rays, intrinsics)
  lrs = dict(DEFAULT_LRS, **(lrs or {}))
  dev = model.device
  h, w = camera.image_shape
  image = torch.as_tensor(image).to(device=dev, dtype=torch.float32)
  if tuple(image.shape) != (h, w, 3):
    raise ValueError(f'image shape {tuple(image.shape)} does not match the camera\'s {h} x {w} x 3')
  ident = camera.copy()
  ident.orientation = np.eye(3, dtype=np.float32)
  ident.position = np.zeros(3, np.float32)
  ident_rays = camera_lib.camera_to_rays(ident, dev)
  local = ident_rays['directions'].reshape(-1, 3)
  pixels = ident_rays['pixels'].reshape(-1, 2)
  intr_parts = tuple(intrinsics)
  # the delta's entries by part, each fitted (at its own rate) or held at 0
  pieces = {k: torch.zeros(len(_lib.INTRINSICS_ENTRIES[k]), device=dev, requires_grad=k in intr_parts)
            for k in INTRINSICS_PARTS}
  delta = lambda: torch.cat([pieces[k] for k in INTRINSICS_PARTS])
  target = image.reshape(-1, 3)
  R0 = torch.as_tensor(camera.orientation, device=dev)
  p0 = torch.as_tensor(camera.position, device=dev)
  encoded = any(k in optimize for k in ('appearance', 'camera', 'warp'))
  md = dict(codes or {})
  if encoded:
    start = registration_codes(model, params, md, warp_extra)
  else:
    start = {}
  fit = {k: v.clone().requires_grad_(k in optimize) for k, v in start.items()}
  omega = torch.zeros(3, device=dev, requires_grad='pose' in optimize)
  offset = torch.zeros(3, device=dev, requires_grad='pose' in optimize)
  groups = []
  if 'pose' in optimize:
    groups += [{'params': [omega], 'lr': lrs['rotation']}, {'params': [offset], 'lr': lrs['position']}]
  groups += [{'params': [fit[k]], 'lr': lrs[k]} for k in fit if k in optimize]
  groups += [{'params': [pieces[k]], 'lr': lrs[k]} for k in intr_parts]
  opt = torch.optim.Adam(groups)
  base_lrs = [g['lr'] for g in groups]
  gen = torch.Generator(device=dev)
  gen.manual_seed(int(seed))
  history = []
  n = h * w
  for step in range(int(steps)):
    idx = torch.randint(0, n, (int(batch_rays),), device=dev, generator=gen)
    loc = refined_directions(camera, delta(), pixels[idx], intr_parts) if intr_parts else local[idx]
    origins, directions = pose_rays(loc, R0, p0, omega, offset)
    if encoded:
      metadata = {k: v.expand(len(idx), -1) for k, v in fit.items()}
    else:
      metadata = {k: torch.full((len(idx), 1), v, device=dev,
                                dtype=torch.float32 if k == 'time' else torch.int32) for k, v in md.items()}
    opt.zero_grad()
    out = model.render_rays({'params': params}, {'origins': origins, 'directions': directions, 'metadata': metadata},
                            warp_extra=warp_extra, metadata_encoded=encoded)
    loss = photometric_loss(out, target[idx])
    loss.backward()
    if step % max(1, int(log_every)) == 0 or step == int(steps) - 1:
      last = out['fine'] if 'fine' in out else out['coarse']
      mse = float(((last['rgb'].detach() - target[idx])**2).mean())
      history.append({'step': step, 'loss': float(loss), 'psnr': float(-10.0 * np.log10(max(mse, 1e-30))),
                      'rotation_deg': float(torch.linalg.norm(omega.detach())) * 180.0 / np.pi,
                      'translation': float(torch.linalg.norm(offset.detach())),
                      'focal_change_pct': 100.0 * float(torch.expm1(pieces['focal'].detach()[0])),
                      'principal_point_px': float(camera.focal_length) * float(torch.linalg.norm(
                          pieces['principal_point'].detach()))})
    opt.step()
    for g, lr in zip(opt.param_groups, base_lrs):
      g['lr'] = lr * float(lr_decay)**((step + 1) / max(1, int(steps) - 1))
  out_codes = {k: v.detach() for k, v in fit.items()}
  registered = posed_camera(camera, omega, offset)
  if intr_parts:
    out_codes['intrinsics'] = delta().detach().reshape(1, 8)
    registered = refined_camera(registered, out_codes['intrinsics'])
  return registered, out_codes, history


def render_camera(model, params, camera, warp_extra, codes, chunk=None):
  """The (H, W, 3) rgb of `camera`'s frame (the fine level, else the coarse one) with the per-frame codes
  `codes` ({'warp': (1, G), 'appearance': (1, A), 'camera': (1, C)}, registration_codes) passed encoded,
  deterministic sampling, in chunks of `chunk` rays (default: the model's batch size)."""
  from nerfies_b200 import camera as camera_lib
  rays = camera_lib.camera_to_rays(camera, model.device)
  h, w = camera.image_shape
  o, d = rays['origins'].reshape(-1, 3), rays['directions'].reshape(-1, 3)
  chunk = int(chunk or model.batch_size)
  out = []
  with torch.no_grad():
    for i in range(0, o.shape[0], chunk):
      n = min(chunk, o.shape[0] - i)
      md = {k: v.expand(n, -1) for k, v in codes.items()}
      lv = model.apply({'params': params}, {'origins': o[i:i + n], 'directions': d[i:i + n], 'metadata': md},
                       warp_extra=warp_extra, metadata_encoded=True)
      out.append((lv['fine'] if 'fine' in lv else lv['coarse'])['rgb'])
  return torch.cat(out).reshape(h, w, 3)
