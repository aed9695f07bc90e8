"""A trained model's surface as a triangle mesh: the density on a 3D grid through the render
kernels, marching cubes in CUDA (include/nerfies_b200.h, nfb_marching_cubes*), vertex colours and
a binary PLY writer; the inverse of the warp field (nfb_warp_invert), which carries the template mesh
into a frame with its topology.  No reference analogue: the reference renders images only.

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

