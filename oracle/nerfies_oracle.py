"""CPU oracle for the per-ray render hot path of google/nerfies (NerfModel.__call__).

TEST INFRASTRUCTURE ONLY.  This file restates, on the CPU in PyTorch (fp32 by
default, fp64 as an error-attribution shadow), the algorithm of the reference
hot path.  Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s
`cpu_baseline` / `--impl reference` legs may import it; the product package
`nerfies_b200` never does (it fails loudly when its CUDA library is missing).

PINNING STATUS.  The reference ships no tests, golden vectors or fixtures, and
its third-party arithmetic back end (jax==0.2.20 / flax==0.3.4,
requirements.txt:2,6) is not installable in this image.  The oracle is pinned
two ways instead (see oracle/README.md):
  1. closed-form known-answer tests derived from the cited source lines
     (tests/test_oracle_kat.py);
  2. golden vectors produced by executing the reference's OWN Python source
     (/root/reference/nerfies/{models,model_utils,modules,warping,rigid_body,
     glo}.py, unmodified) on top of a numpy stand-in for the jax/flax API
     (oracle/jaxshim, generator oracle/make_golden.py, fixtures tests/golden/).
     The algorithm is the reference's; only the array primitives (matmul, sin,
     exp, sort, cumprod) are numpy's instead of XLA's.
Parity against a real JAX/XLA run remains unverified ("parity unpinned" at the
XLA boundary).

All citations are file:line in /root/reference/nerfies/.
Parameter pytrees use the Flax names of SURVEY.md §8a R12, Dense kernels are
(in, out) and applied as x @ kernel + bias.
"""
from __future__ import annotations

import dataclasses
import math
from typing import Any, Dict, Optional, Sequence, Tuple

import numpy as np
import torch

Tensor = torch.Tensor


# --------------------------------------------------------------------------
# Model description (mirrors NerfModel attributes, models.py:76-120).
# --------------------------------------------------------------------------
@dataclasses.dataclass
class OracleSpec:
  """The subset of NerfModel attributes that shape the forward pass."""
  num_coarse_samples: int = 64
  num_fine_samples: int = 128
  near: float = 0.0
  far: float = 1.0
  use_viewdirs: bool = True
  nerf_trunk_depth: int = 8
  nerf_trunk_width: int = 256
  nerf_rgb_branch_depth: int = 1
  nerf_rgb_branch_width: int = 128
  nerf_skips: Tuple[int, ...] = (4,)
  alpha_channels: int = 1
  rgb_channels: int = 3
  num_nerf_point_freqs: int = 10
  num_nerf_viewdir_freqs: int = 4
  activation: str = 'relu'
  sigma_activation: str = 'relu'
  use_white_background: bool = False
  use_linear_disparity: bool = False
  use_sample_at_infinity: bool = True
  use_appearance_metadata: bool = False
  use_camera_metadata: bool = False
  use_warp: bool = False
  use_trunk_condition: bool = False
  use_alpha_condition: bool = False
  use_rgb_condition: bool = False
  num_appearance_features: int = 8
  num_camera_features: int = 2
  num_warp_features: int = 8
  num_warp_freqs: int = 8
  num_appearance_embeddings: int = 1
  num_camera_embeddings: int = 1
  num_warp_embeddings: int = 1
  warp_field_type: str = 'se3'
  # SE3Field defaults (warping.py:224-227).
  warp_trunk_depth: int = 6
  warp_trunk_width: int = 128
  warp_skips: Tuple[int, ...] = (4,)
  # metadata encoder of the warp field (warping.py:109-123, 250-260): 'glo',
  # 'time' (modules.TimeEncoder on metadata['time']) or, TranslationField only,
  # 'blend'; warp_kwargs['metadata_encoder_num_freqs'] (warping.py:84, 233).
  warp_metadata_encoder_type: str = 'glo'
  metadata_encoder_num_freqs: int = 1
  # SE3Field(use_pivot=..., use_translation=...) (warping.py:242-243).
  warp_use_pivot: bool = False
  warp_use_translation: bool = False


_ACTIVATIONS = {
    'relu': torch.relu,
    'elu': torch.nn.functional.elu,
    'leaky_relu': lambda x: torch.nn.functional.leaky_relu(x, 0.01),
    'tanh': torch.tanh,
    'sigmoid': torch.sigmoid,
    # jax.nn.softplus(x) = logaddexp(x, 0).
    'softplus': lambda x: torch.logaddexp(x, torch.zeros_like(x)),
}


def activation_fn(name: str):
  return _ACTIVATIONS[name]


# --------------------------------------------------------------------------
# R1  sample_along_rays  (model_utils.py:36-73)
# --------------------------------------------------------------------------
def coarse_z_vals(num_samples: int, near: float, far: float,
                  use_linear_disparity: bool,
                  dtype=torch.float32) -> Tensor:
  """z_vals for one ray, non-stratified (model_utils.py:56-60)."""
  # jnp.linspace(0., 1., n) is float32; numpy's float32 linspace is the
  # correctly rounded i/(n-1).
  t = torch.from_numpy(np.linspace(0., 1., num_samples, dtype=np.float32))
  t = t.to(dtype)
  if not use_linear_disparity:
    return near * (1. - t) + far * t
  return 1. / (1. / near * (1. - t) + 1. / far * t)


def sample_along_rays(origins: Tensor, directions: Tensor, num_samples: int,
                      near: float, far: float, use_linear_disparity: bool,
                      t_rand: Optional[Tensor] = None):
  """model_utils.py:36-73.  `t_rand` (B, Nc) stands in for random.uniform
  (model_utils.py:65); None = the non-stratified branch (:67-70)."""
  dtype = origins.dtype
  z = coarse_z_vals(num_samples, near, far, use_linear_disparity, dtype)
  batch = origins.shape[0]
  if t_rand is not None:
    mids = .5 * (z[1:] + z[:-1])
    upper = torch.cat([mids, z[-1:]], -1)
    lower = torch.cat([z[:1], mids], -1)
    z = lower + (upper - lower) * t_rand.to(dtype)
  else:
    z = z[None, :].expand(batch, num_samples)
  points = origins[:, None, :] + z[:, :, None] * directions[:, None, :]
  return z, points


# --------------------------------------------------------------------------
# R3 / R6  Sinusoidal encoders  (modules.py:172-294)
# --------------------------------------------------------------------------
HALF_PI_F32 = float(np.float32(np.pi / 2))  # jnp.pi / 2 added to f32 arrays


def cosine_easing_window(num_bands: int, alpha: float) -> np.ndarray:
  """modules.py:274-294, evaluated in float32 like jnp would."""
  bands = np.linspace(0.0, num_bands - 1.0, num_bands, dtype=np.float32)
  x = np.clip(np.float32(alpha) - bands, np.float32(0.0), np.float32(1.0))
  pi = np.float32(np.pi)
  return (np.float32(0.5) * (np.float32(1.0) + np.cos(pi * x + pi))).astype(
      np.float32)


def sinusoidal_encode(x: Tensor, num_freqs: int,
                      window: Optional[Tensor] = None) -> Tensor:
  """SinusoidalEncoder.__call__ (modules.py:201-228), optionally windowed as in
  AnnealedSinusoidalEncoder.__call__ (modules.py:240-272).

  x: (..., C).  Output (..., C + 2*F*C): identity, then for each frequency a
  block of C sines followed by a block of C "cosines" sin(a + fl32(pi/2)).
  """
  if num_freqs == 0:
    return x
  dtype = x.dtype
  freqs = 2.0 ** torch.linspace(0, num_freqs - 1.0, num_freqs,
                                dtype=torch.float64)
  freqs = freqs.to(dtype)  # exact powers of two.
  angles = x[..., None, :] * freqs[:, None]  # (..., F, C)
  if dtype == torch.float32:
    half_pi = torch.tensor(HALF_PI_F32, dtype=dtype)
  else:
    half_pi = torch.tensor(math.pi / 2, dtype=dtype)
  feats = torch.stack((angles, angles + half_pi), dim=-2)  # (..., F, 2, C)
  feats = torch.sin(feats)
  if window is not None:
    feats = window.to(dtype)[:, None, None] * feats
  feats = feats.reshape(*x.shape[:-1], -1)
  return torch.cat([x, feats], dim=-1)


# --------------------------------------------------------------------------
# MLP  (modules.py:26-62)
# --------------------------------------------------------------------------
# When set, dense() rounds both operands to bfloat16 and accumulates in fp32:
# the arithmetic of the tensor-core path (NFB_PREC_BF16), so that its wiring can
# be checked at a tolerance far below bf16's own 4e-3 rounding.
_BF16_OPERANDS = False


class bf16_operands:
  """Context manager: emulate bf16-operand / fp32-accumulate Dense layers."""

  def __enter__(self):
    global _BF16_OPERANDS
    self._old = _BF16_OPERANDS
    _BF16_OPERANDS = True

  def __exit__(self, *exc):
    global _BF16_OPERANDS
    _BF16_OPERANDS = self._old


def dense(p: Dict[str, Tensor], x: Tensor, exact: bool = False) -> Tensor:
  k = p['kernel'].to(x.dtype)
  if _BF16_OPERANDS and not exact:
    x = x.bfloat16().to(x.dtype)
    k = k.bfloat16().to(k.dtype)
  return x @ k + p['bias'].to(x.dtype)


def mlp(params: Dict[str, Any], x: Tensor, depth: int, skips: Sequence[int],
        hidden_activation: str = 'relu', has_logit: bool = False) -> Tensor:
  """modules.py:39-62.  Skip concat order is [x, inputs] (:47-48); the hidden
  activation follows every hidden layer; the logit layer has identity output
  activation by default (:34)."""
  act = activation_fn(hidden_activation)
  inputs = x
  for i in range(depth):
    if i in skips:
      x = torch.cat([x, inputs], dim=-1)
    x = act(dense(params[f'hidden_{i}'], x))
  if has_logit:
    x = dense(params['logit'], x)
  return x


# --------------------------------------------------------------------------
# R5  rigid_body.py
# --------------------------------------------------------------------------
def skew(w: Tensor) -> Tensor:
  """rigid_body.py:21-36 batched: (...,3) -> (...,3,3)."""
  z = torch.zeros_like(w[..., 0])
  return torch.stack([
      torch.stack([z, -w[..., 2], w[..., 1]], -1),
      torch.stack([w[..., 2], z, -w[..., 0]], -1),
      torch.stack([-w[..., 1], w[..., 0], z], -1),
  ], -2)


def exp_so3(w: Tensor, theta: Tensor) -> Tensor:
  """rigid_body.py:54-68."""
  W = skew(w)
  eye = torch.eye(3, dtype=w.dtype)
  th = theta[..., None, None]
  return eye + torch.sin(th) * W + (1.0 - torch.cos(th)) * (W @ W)


def exp_se3(S: Tensor, theta: Tensor) -> Tuple[Tensor, Tensor]:
  """rigid_body.py:71-89.  Returns (R, p) of the homogeneous transform."""
  w, v = S[..., :3], S[..., 3:]
  W = skew(w)
  R = exp_so3(w, theta)
  eye = torch.eye(3, dtype=S.dtype)
  th = theta[..., None, None]
  M = th * eye + (1.0 - torch.cos(th)) * W + (th - torch.sin(th)) * (W @ W)
  p = (M @ v[..., None])[..., 0]
  return R, p


# --------------------------------------------------------------------------
# R3-R5  SE3Field  (warping.py:202-389)
# --------------------------------------------------------------------------
# TimeEncoder defaults (modules.py:301-304): not configurable through the model.
TIME_ENCODER_DEPTH, TIME_ENCODER_WIDTH, TIME_ENCODER_SKIPS = 6, 64, (4,)


def time_encode(params: Dict[str, Any], num_freqs: int, time: Tensor,
                alpha: Optional[float], dtype) -> Tensor:
  """modules.TimeEncoder.__call__ (modules.py:317-322): annealed positional
  encoding of the (..., 1) timestamp, then MLP(depth 6, width 64, skips (4,))
  with a `features`-wide output layer.  alpha None -> num_freqs."""
  if alpha is None:
    alpha = num_freqs
  window = torch.from_numpy(cosine_easing_window(num_freqs, alpha))
  enc = sinusoidal_encode(time.to(dtype), num_freqs, window)
  return mlp(params['mlp'], enc, TIME_ENCODER_DEPTH, TIME_ENCODER_SKIPS, 'relu',
             has_logit=True)


def se3_field_warp(params: Dict[str, Any], spec: OracleSpec, points: Tensor,
                   metadata_embed: Tensor, alpha: float) -> Tensor:
  """SE3Field.warp (warping.py:322-353) for (..., 3) points with a matching
  (..., G) metadata embedding."""
  window = torch.from_numpy(cosine_easing_window(spec.num_warp_freqs, alpha))
  points_embed = sinusoidal_encode(points, spec.num_warp_freqs, window)
  inputs = torch.cat([points_embed, metadata_embed.to(points.dtype)], dim=-1)
  trunk_output = mlp(params['trunk'], inputs, spec.warp_trunk_depth,
                     spec.warp_skips, 'relu')
  w = dense(params['branches_w']['logit'], trunk_output)
  v = dense(params['branches_v']['logit'], trunk_output)
  pivot = (dense(params['branches_p']['logit'], trunk_output)
           if spec.warp_use_pivot else None)
  translation = (dense(params['branches_t']['logit'], trunk_output)
                 if spec.warp_use_translation else None)
  return se3_tail(w, v, points, pivot, translation)


def se3_tail(w: Tensor, v: Tensor, points: Tensor, pivot: Optional[Tensor] = None,
             translation: Optional[Tensor] = None) -> Tensor:
  """SE3Field.warp after its branch MLPs (warping.py:330-353): the screw axis
  (w, v) scaled by theta = |w|, the optional pivot and translation heads."""
  theta = torch.linalg.norm(w, dim=-1)
  w = w / theta[..., None]
  v = v / theta[..., None]
  R, p = exp_se3(torch.cat([w, v], dim=-1), theta)
  # from_homogenous(transform @ to_homogenous(x)) (rigid_body.py:92-97); the
  # homogeneous coordinate is exactly 1.
  warped = points
  if pivot is not None:                                 # warping.py:339-342
    warped = warped + pivot
  warped = (R @ warped[..., None])[..., 0] + p
  warped = warped / torch.ones_like(warped[..., :1])
  if pivot is not None:                                 # warping.py:347-348
    warped = warped - pivot
  if translation is not None:                           # warping.py:350-352
    warped = warped + translation
  return warped


def translation_field_warp(params, spec, points, metadata_embed, alpha):
  """TranslationField.warp (warping.py:149-158)."""
  window = torch.from_numpy(cosine_easing_window(spec.num_warp_freqs, alpha))
  points_embed = sinusoidal_encode(points, spec.num_warp_freqs, window)
  inputs = torch.cat([points_embed, metadata_embed.to(points.dtype)], dim=-1)
  translation = mlp(params['mlp'], inputs, spec.warp_trunk_depth,
                    spec.warp_skips, 'relu', has_logit=True)
  return points + translation


def glo_encode(params: Dict[str, Any], ids: Tensor) -> Tensor:
  """GloEncoder.__call__ (glo.py:41-53)."""
  if ids.shape[-1] == 1:
    ids = ids[..., 0]
  return params['embed']['embedding'][ids.long()]


def encode_warp_metadata(params, spec: OracleSpec, metadata: Tensor,
                         time_alpha: Optional[float], dtype) -> Tensor:
  """encode_metadata of TranslationField (warping.py:125-141) / SE3Field
  (warping.py:309-320)."""
  kind = spec.warp_metadata_encoder_type
  F = spec.metadata_encoder_num_freqs
  if kind == 'glo':
    return glo_encode(params['metadata_encoder'], metadata)
  if kind == 'time':
    return time_encode(params['metadata_encoder'], F, metadata, time_alpha, dtype)
  if kind == 'blend' and spec.warp_field_type == 'translation':
    glo_embed = glo_encode(params['glo_encoder'], metadata).to(dtype)
    # self.time_encoder(metadata): the integer ids themselves, alpha=None
    time_embed = time_encode(params['time_encoder'], F, metadata.to(dtype), None, dtype)
    return (1.0 - time_alpha) * glo_embed + time_alpha * time_embed
  raise ValueError(f'Unknown metadata encoder type {kind!r}')


def warp_field_apply(params, spec: OracleSpec, points: Tensor,
                     metadata: Tensor, alpha: float,
                     metadata_encoded: bool = False,
                     time_alpha: Optional[float] = None) -> Tensor:
  """SE3Field.__call__ / TranslationField.__call__ without the Jacobian
  (warping.py:355-389, 160-199)."""
  if metadata_encoded:
    embed = metadata
  else:
    embed = encode_warp_metadata(params, spec, metadata, time_alpha, points.dtype)
  if spec.warp_field_type == 'se3':
    return se3_field_warp(params, spec, points, embed, alpha)
  if spec.warp_field_type == 'translation':
    return translation_field_warp(params, spec, points, embed, alpha)
  raise ValueError(f'Unknown warp field type: {spec.warp_field_type!r}')


# --------------------------------------------------------------------------
# R7  NerfMLP  (modules.py:65-169)
# --------------------------------------------------------------------------
def nerf_mlp(params: Dict[str, Any], spec: OracleSpec, x: Tensor,
             trunk_condition: Optional[Tensor],
             alpha_condition: Optional[Tensor],
             rgb_condition: Optional[Tensor]) -> Dict[str, Tensor]:
  """x: (B, S, Dp); conditions (B, C) broadcast over samples (:114-122)."""
  B, S, _ = x.shape

  def bc(c):
    return c[:, None, :].expand(B, S, c.shape[-1]).to(x.dtype)

  trunk_input = x
  if trunk_condition is not None:
    trunk_input = torch.cat([x, bc(trunk_condition)], dim=-1)
  h = mlp(params['MLP_0'], trunk_input, spec.nerf_trunk_depth,
          spec.nerf_skips, spec.activation)
  bottleneck = None
  if alpha_condition is not None or rgb_condition is not None:
    bottleneck = dense(params['bottleneck'], h)
  if alpha_condition is not None:
    alpha_input = torch.cat([bottleneck, bc(alpha_condition)], dim=-1)
  else:
    alpha_input = h
  if alpha_condition is None:
    # (the tensor-core path evaluates this Dense(1) on CUDA cores: fp32 activations,
    #  bf16-rounded weights, fp32 accumulation)
    pl = params['MLP_2']['logit']
    if _BF16_OPERANDS:
      pl = {'kernel': pl['kernel'].bfloat16().to(pl['kernel'].dtype), 'bias': pl['bias']}
    alpha = dense(pl, alpha_input, exact=True)
  else:
    alpha = mlp(params['MLP_2'], alpha_input, 0, (), spec.activation,
                has_logit=True)
  if rgb_condition is not None:
    rgb_input = torch.cat([bottleneck, bc(rgb_condition)], dim=-1)
  else:
    rgb_input = h
  rgb = mlp(params['MLP_1'], rgb_input, spec.nerf_rgb_branch_depth, (),
            spec.activation, has_logit=True)
  return {'rgb': rgb, 'alpha': alpha}


# --------------------------------------------------------------------------
# R9  volumetric_rendering  (model_utils.py:76-136, 218-263)
# --------------------------------------------------------------------------
def volumetric_rendering(rgb: Tensor, sigma: Tensor, z_vals: Tensor,
                         dirs: Tensor, use_white_background: bool,
                         sample_at_infinity: bool = True,
                         eps: float = 1e-10) -> Dict[str, Tensor]:
  dtype = rgb.dtype
  last_sample_z = 1e10 if sample_at_infinity else 1e-19
  dists = torch.cat([
      z_vals[..., 1:] - z_vals[..., :-1],
      torch.full_like(z_vals[..., :1], last_sample_z)], -1)
  dists = dists * torch.linalg.norm(dirs[..., None, :], dim=-1)
  alpha = 1.0 - torch.exp(-sigma * dists)
  accum_prod = torch.cat([
      torch.ones_like(alpha[..., :1]),
      torch.cumprod(1.0 - alpha[..., :-1] + eps, dim=-1)], dim=-1)
  weights = alpha * accum_prod
  out_rgb = (weights[..., None] * rgb).sum(dim=-2)
  exp_depth = (weights * z_vals).sum(dim=-1)
  # compute_depth_map (model_utils.py:248-263) via the opaqueness mask
  # (:218-239): first sample where cumsum(weights) >= 0.5.
  cum = torch.cumsum(weights, dim=-1)
  opaque = cum >= torch.tensor(0.5, dtype=dtype)
  padded = torch.cat([torch.zeros_like(opaque[..., :1]), opaque[..., :-1]], -1)
  mask = torch.logical_xor(opaque, padded).to(dtype)
  med_depth = (mask * z_vals).sum(dim=-1)
  acc = weights.sum(dim=-1)
  if use_white_background:
    out_rgb = out_rgb + (1. - acc[..., None])
  if sample_at_infinity:
    acc = weights[..., :-1].sum(dim=-1)
  return {'rgb': out_rgb, 'depth': exp_depth, 'med_depth': med_depth,
          'acc': acc, 'weights': weights}


# --------------------------------------------------------------------------
# R10  piecewise_constant_pdf / sample_pdf  (model_utils.py:139-215)
# --------------------------------------------------------------------------
def piecewise_constant_pdf(bins: Tensor, weights: Tensor, num_samples: int,
                           u_rand: Optional[Tensor] = None) -> Tensor:
  """Line-by-line restatement incl. the mask/minmax inversion (:169-179)."""
  dtype = bins.dtype
  eps = 1e-5
  weights = weights + eps
  pdf = weights / weights.sum(dim=-1, keepdim=True)
  cdf = torch.cumsum(pdf, dim=-1)
  cdf = torch.cat([torch.zeros_like(cdf[..., :1]), cdf], dim=-1)
  if u_rand is not None:
    u = u_rand.to(dtype)
  else:
    u = torch.from_numpy(
        np.linspace(0., 1., num_samples, dtype=np.float32)).to(dtype)
    u = u.expand(*cdf.shape[:-1], num_samples)
  mask = u[..., None, :] >= cdf[..., :, None]

  def minmax(x):
    x0 = torch.where(mask, x[..., None], x[..., :1, None]).max(dim=-2).values
    x1 = torch.where(~mask, x[..., None], x[..., -1:, None]).min(dim=-2).values
    x0 = torch.minimum(x0, x[..., -2:-1])
    x1 = torch.maximum(x1, x[..., 1:2])
    return x0, x1

  bins_g0, bins_g1 = minmax(bins)
  cdf_g0, cdf_g1 = minmax(cdf)
  denom = cdf_g1 - cdf_g0
  denom = torch.where(denom < eps, torch.ones_like(denom), denom)
  t = (u - cdf_g0) / denom
  return bins_g0 + t * (bins_g1 - bins_g0)


def sample_pdf(bins, weights, origins, directions, z_vals, num_samples,
               u_rand=None):
  """model_utils.py:190-215."""
  z_samples = piecewise_constant_pdf(bins, weights, num_samples, u_rand)
  z = torch.sort(torch.cat([z_vals, z_samples], dim=-1), dim=-1).values
  points = origins[..., None, :] + z[..., None] * directions[..., None, :]
  return z, points


# --------------------------------------------------------------------------
# R2 / R11  NerfModel  (models.py:186-375)
# --------------------------------------------------------------------------
def get_condition_inputs(params, spec: OracleSpec, viewdirs: Tensor,
                         metadata: Dict[str, Tensor],
                         metadata_encoded: bool = False):
  """models.py:186-228, including the `use_alpha_condition` guard on the rgb
  append (:206-207)."""
  trunk_c, alpha_c, rgb_c = [], [], []
  if spec.use_viewdirs:
    rgb_c.append(sinusoidal_encode(viewdirs, spec.num_nerf_viewdir_freqs))
  if spec.use_appearance_metadata:
    if metadata_encoded:
      code = metadata['appearance']
    else:
      code = glo_encode(params['appearance_encoder'], metadata['appearance'])
    code = code.to(viewdirs.dtype)
    if spec.use_trunk_condition:
      trunk_c.append(code)
    if spec.use_alpha_condition:
      alpha_c.append(code)
    if spec.use_alpha_condition:
      rgb_c.append(code)
  if spec.use_camera_metadata:
    if metadata_encoded:
      code = metadata['camera']
    else:
      code = glo_encode(params['camera_encoder'], metadata['camera'])
    rgb_c.append(code.to(viewdirs.dtype))
  cat = lambda xs: torch.cat(xs, dim=-1) if xs else None
  return cat(trunk_c), cat(alpha_c), cat(rgb_c)


def render_samples(params, spec: OracleSpec, level: str, points, z_vals,
                   directions, viewdirs, metadata, warp_alpha, use_warp=True,
                   metadata_encoded=False, return_points=False,
                   time_alpha=None):
  """models.py:230-287.  noise_regularize (model_utils.py:266-282) is a no-op
  whenever it can run: with noise_std > 0 and stratified sampling the reference
  indexes the NerfMLP's output DICT as an array (models.py:272-275 hands
  {'rgb','alpha'} to raw[..., 3:4]) and raises, so there is no behaviour to restate."""
  trunk_c, alpha_c, rgb_c = get_condition_inputs(
      params, spec, viewdirs, metadata, metadata_encoded)
  out = {}
  if return_points:
    out['points'] = points
  if use_warp:
    # models.py:252-254
    warp_meta = (metadata['time'] if spec.warp_metadata_encoder_type == 'time'
                 else metadata['warp'])
    if metadata_encoded:
      warp_meta = warp_meta[:, None, :].expand(*points.shape[:2],
                                                spec.num_warp_features)
    else:
      warp_meta = warp_meta[:, None, :].expand(*points.shape[:2], 1)
    points = warp_field_apply(params['warp_field'], spec, points, warp_meta,
                              warp_alpha, metadata_encoded, time_alpha)
    if return_points:
      out['warped_points'] = points
  points_embed = sinusoidal_encode(points, spec.num_nerf_point_freqs)
  raw = nerf_mlp(params[f'nerf_mlps_{level}'], spec, points_embed, trunk_c,
                 alpha_c, rgb_c)
  rgb = torch.sigmoid(raw['rgb'])
  sigma = activation_fn(spec.sigma_activation)(raw['alpha'][..., 0])
  out['raw_rgb'] = raw['rgb']
  out['raw_alpha'] = raw['alpha']
  out['sample_rgb'] = rgb
  out['sample_sigma'] = sigma
  out.update(volumetric_rendering(
      rgb, sigma, z_vals, directions,
      use_white_background=spec.use_white_background,
      sample_at_infinity=spec.use_sample_at_infinity))
  return out


def render_forward(params, spec: OracleSpec, rays_dict: Dict[str, Any],
                   warp_alpha: float = 0.0, use_warp: bool = True,
                   metadata_encoded: bool = False, return_points: bool = False,
                   t_rand: Optional[Tensor] = None,
                   u_rand: Optional[Tensor] = None,
                   dtype=torch.float32, time_alpha: Optional[float] = None
                   ) -> Dict[str, Dict[str, Tensor]]:
  """NerfModel.__call__ (models.py:289-375), deterministic unless the caller
  supplies the uniform draws `t_rand` (B,Nc) / `u_rand` (B,Nf) that stand in
  for jax.random.  Always returns weights plus per-sample diagnostics."""
  use_warp = spec.use_warp and use_warp
  origins = rays_dict['origins'].to(dtype)
  directions = rays_dict['directions'].to(dtype)
  metadata = rays_dict.get('metadata', {})
  viewdirs = rays_dict.get('viewdirs', rays_dict['directions']).to(dtype)
  params = tree_to(params, dtype)

  z_vals, points = sample_along_rays(
      origins, directions, spec.num_coarse_samples, spec.near, spec.far,
      spec.use_linear_disparity, t_rand)
  coarse = render_samples(params, spec, 'coarse', points, z_vals, directions,
                          viewdirs, metadata, warp_alpha, use_warp,
                          metadata_encoded, return_points, time_alpha)
  coarse['z_vals'] = z_vals
  out = {'coarse': coarse}
  if spec.num_fine_samples > 0:
    z_mid = .5 * (z_vals[..., 1:] + z_vals[..., :-1])
    z_fine, points = sample_pdf(z_mid, coarse['weights'][..., 1:-1], origins,
                                directions, z_vals, spec.num_fine_samples,
                                u_rand)
    fine = render_samples(params, spec, 'fine', points, z_fine, directions,
                          viewdirs, metadata, warp_alpha, use_warp,
                          metadata_encoded, return_points, time_alpha)
    fine['z_vals'] = z_fine
    out['fine'] = fine
  return out


def render_level(params, spec: OracleSpec, level: str,
                 rays_dict: Dict[str, Any], z_vals: Tensor,
                 warp_alpha: float = 0.0, use_warp: bool = True,
                 dtype=torch.float32, metadata_encoded: bool = False,
                 time_alpha: Optional[float] = None) -> Dict[str, Tensor]:
  """One level of NerfModel.__call__ for caller-supplied z_vals: points =
  o + z d (model_utils.py:72-73 / :214-215) then render_samples
  (models.py:230-287).  Used to test the levels in isolation."""
  use_warp = spec.use_warp and use_warp
  origins = rays_dict['origins'].to(dtype)
  directions = rays_dict['directions'].to(dtype)
  viewdirs = rays_dict.get('viewdirs', rays_dict['directions']).to(dtype)
  z_vals = z_vals.to(dtype)
  points = origins[:, None, :] + z_vals[:, :, None] * directions[:, None, :]
  out = render_samples(tree_to(params, dtype), spec, level, points, z_vals,
                       directions, viewdirs, rays_dict.get('metadata', {}),
                       warp_alpha, use_warp, metadata_encoded, True, time_alpha)
  out['z_vals'] = z_vals
  return out


def pdf_cdf_residual(bins: Tensor, weights: Tensor, z_samples: Tensor,
                     u: Tensor) -> Tensor:
  """|F(z) - u| where F is the piecewise-linear CDF of model_utils.py:153-158
  evaluated in float64 - a conditioning-free check of inverse-CDF samples
  (position errors in near-empty bins are amplified by 1/pdf, CDF errors are
  not).  bins (B,n), weights (B,n-1), z_samples/u (B,Nf)."""
  b = bins.double()
  w = weights.double() + 1e-5
  pdf = w / w.sum(-1, keepdim=True)
  cdf = torch.cat([torch.zeros_like(pdf[..., :1]), torch.cumsum(pdf, -1)], -1)
  z = z_samples.double().clamp(b[..., :1], b[..., -1:])
  idx = torch.searchsorted(b.contiguous(), z.contiguous(), right=True) - 1
  idx = idx.clamp(0, b.shape[-1] - 2)
  b0 = torch.gather(b, -1, idx)
  b1 = torch.gather(b, -1, idx + 1)
  c0 = torch.gather(cdf, -1, idx)
  c1 = torch.gather(cdf, -1, idx + 1)
  t = (z - b0) / (b1 - b0).clamp_min(1e-30)
  return (c0 + t * (c1 - c0) - u.double()).abs()


# --------------------------------------------------------------------------
# SURVEY 8(f) #2: warp Jacobian, elastic / warp-reg / background regularisers
# --------------------------------------------------------------------------
def warp_jacobian(params, spec: OracleSpec, points: Tensor, metadata: Tensor,
                  alpha: float, time_alpha: Optional[float] = None,
                  create_graph: bool = False) -> Tensor:
  """jax.jacfwd(self.warp, argnums=0)(points, metadata_embed, extra)
  (warping.py:196-198, 385-387), vmapped over the batch dimensions by
  model_utils.vmap_module (warping.py:46-57): J[..., i, j] = d warped_i / d point_j.
  `points` (..., 3), `metadata` (..., 1) ids.  Differentiable w.r.t. the
  parameters when create_graph=True (double backward through autograd)."""
  shape = points.shape[:-1]
  pts = points.reshape(-1, 3).detach().clone().requires_grad_(True)
  meta = metadata.reshape(-1, metadata.shape[-1])
  embed = encode_warp_metadata(params, spec, meta, time_alpha, pts.dtype)
  warp = se3_field_warp if spec.warp_field_type == 'se3' else translation_field_warp
  warped = warp(params, spec, pts, embed, alpha)
  rows = []
  for i in range(3):
    g, = torch.autograd.grad(warped[:, i].sum(), pts, create_graph=create_graph,
                             retain_graph=True)
    rows.append(g)
  return torch.stack(rows, dim=-2).reshape(*shape, 3, 3)


def log1p_safe(x: Tensor) -> Tensor:
  """utils.py:244-246."""
  return torch.log1p(torch.clamp(x, max=3e37))


def expm1_safe(x: Tensor) -> Tensor:
  """utils.py:254-256."""
  return torch.expm1(torch.clamp(x, max=87.5))


def general_loss_with_squared_residual(squared_x: Tensor, alpha: float,
                                       scale: float) -> Tensor:
  """utils.py:264-331 (Barron's general robust loss on a squared residual)."""
  eps = float(np.finfo(np.float32).eps)
  x = squared_x / (scale ** 2)
  if alpha == -math.inf:
    loss = -torch.expm1(-0.5 * x)
  elif alpha == 0:
    loss = log1p_safe(0.5 * x)
  elif alpha == 2:
    loss = 0.5 * x
  elif alpha == math.inf:
    loss = expm1_safe(0.5 * x)
  else:
    beta_safe = max(eps, abs(alpha - 2.0))
    alpha_safe = (1.0 if alpha >= 0 else -1.0) * max(eps, abs(alpha))
    loss = (beta_safe / alpha_safe) * (torch.pow(x / beta_safe + 1.0, 0.5 * alpha) - 1.0)
  return scale * loss


def jacobian_to_curl(jacobian: Tensor) -> Tensor:
  """utils.py:71-84."""
  return torch.stack([jacobian[..., 2, 1] - jacobian[..., 1, 2],
                      jacobian[..., 0, 2] - jacobian[..., 2, 0],
                      jacobian[..., 1, 0] - jacobian[..., 0, 1]], dim=-1)


def jacobian_to_div(jacobian: Tensor) -> Tensor:
  """utils.py:87-91: trace(J) - 3."""
  return jacobian[..., 0, 0] + jacobian[..., 1, 1] + jacobian[..., 2, 2] - 3.0


def nearest_rotation_svd(matrix: Tensor, eps: float = 1e-6) -> Tensor:
  """training.py:57-68."""
  u, _, vh = torch.linalg.svd(matrix + eps, full_matrices=False)
  det = torch.linalg.det(u @ vh)
  m = torch.diag_embed(torch.stack([torch.ones_like(det), torch.ones_like(det), det], dim=-1))
  return u @ m @ vh


def compute_elastic_loss(jacobian: Tensor, eps: float = 1e-6,
                         loss_type: str = 'log_svals') -> Tuple[Tensor, Tensor]:
  """training.py:71-115, batched over the leading dimensions (the reference vmaps it
  twice, training.py:180).  Returns (loss, residual)."""
  if loss_type == 'log_svals':
    svals = torch.linalg.svdvals(jacobian)
    log_svals = torch.log(torch.clamp(svals, min=eps))
    sq_residual = torch.sum(log_svals ** 2, dim=-1)
  elif loss_type == 'svals':
    svals = torch.linalg.svdvals(jacobian)
    sq_residual = torch.sum((svals - 1.0) ** 2, dim=-1)
  elif loss_type == 'jtj':
    jtj = jacobian @ jacobian.transpose(-1, -2)
    sq_residual = ((jtj - torch.eye(3, dtype=jacobian.dtype)) ** 2).sum(dim=(-1, -2)) / 4.0
  elif loss_type == 'div':
    sq_residual = jacobian_to_div(jacobian) ** 2
  elif loss_type == 'det':
    sq_residual = (torch.linalg.det(jacobian) - 1.0) ** 2
  elif loss_type == 'log_det':
    sq_residual = torch.log(torch.clamp(torch.linalg.det(jacobian), min=eps)) ** 2
  elif loss_type == 'nr':
    rot = nearest_rotation_svd(jacobian)
    sq_residual = torch.sum((jacobian - rot) ** 2, dim=(-1, -2))
  else:
    raise NotImplementedError(f'Unknown elastic loss type {loss_type!r}')
  residual = torch.sqrt(sq_residual)
  loss = general_loss_with_squared_residual(sq_residual, alpha=-2.0, scale=0.03)
  return loss, residual


def compute_opaqueness_mask(weights: Tensor, depth_threshold: float = 0.5) -> Tensor:
  """model_utils.py:218-239."""
  opaqueness = torch.cumsum(weights, dim=-1) >= depth_threshold
  padded = torch.cat([torch.zeros_like(opaqueness[..., :1]), opaqueness[..., :-1]], dim=-1)
  return torch.logical_xor(opaqueness, padded)


def compute_depth_index(weights: Tensor, depth_threshold: float = 0.5) -> Tensor:
  """model_utils.py:242-245: argmax of the mask (0 when the ray never reaches the threshold)."""
  return torch.argmax(compute_opaqueness_mask(weights, depth_threshold).to(torch.int32), dim=-1)


def compute_background_loss(params, spec: OracleSpec, points: Tensor, metadata: Tensor,
                            point_noise: Tensor, warp_alpha: float, alpha: float = -2.0,
                            scale: float = 0.001, time_alpha: Optional[float] = None) -> Tensor:
  """training.py:118-135 with the random draws supplied by the caller: `metadata` (P,1)
  = random.choice(key, warp_ids), `point_noise` (P,3) = noise_std * random.normal."""
  pts = points + point_noise
  warped = warp_field_apply(params['warp_field'], spec, pts, metadata, warp_alpha,
                            False, time_alpha)
  sq_residual = torch.sum((warped - pts) ** 2, dim=-1)
  return general_loss_with_squared_residual(sq_residual, alpha=alpha, scale=scale)


def level_regularisers(params, spec: OracleSpec, out: Dict[str, Tensor], rays_dict,
                       warp_alpha: float, use_elastic_loss: bool = False,
                       elastic_reduce_method: str = 'median', elastic_loss_type: str = 'log_svals',
                       use_warp_reg_loss: bool = False, warp_reg_loss_alpha: float = -2.0,
                       warp_reg_loss_scale: float = 0.001, create_graph: bool = True
                       ) -> Dict[str, Tensor]:
  """The regulariser terms of _compute_loss_and_stats (training.py:171-212) for one level's
  `out` (render_level(..., return_points) output: 'points', 'warped_points', 'weights')."""
  res = {}
  weights = out['weights'].detach()                               # lax.stop_gradient
  if use_elastic_loss:
    B, S = weights.shape
    meta = rays_dict['metadata']['warp'][:, None, :].expand(B, S, 1)
    pts = out['points']
    if elastic_reduce_method == 'median':
      idx = compute_depth_index(weights)                          # training.py:184-188
      pts = torch.gather(pts, 1, idx[:, None, None].expand(B, 1, 3))
      meta = meta[:, :1]
    jac = warp_jacobian(params['warp_field'], spec, pts, meta, warp_alpha, create_graph=create_graph)
    loss, residual = compute_elastic_loss(jac, loss_type=elastic_loss_type)
    if elastic_reduce_method == 'weight':
      loss = weights * loss
    res['loss/elastic'] = loss.sum(dim=-1).mean()
    res['residual/elastic'] = residual.mean()
    res['jacobian'] = jac
  if use_warp_reg_loss:
    idx = compute_depth_index(weights)
    warp_mag = ((out['points'] - out['warped_points']) ** 2).sum(dim=-1)
    r = torch.gather(warp_mag, 1, idx[:, None])
    res['loss/warp_reg'] = general_loss_with_squared_residual(
        r, alpha=warp_reg_loss_alpha, scale=warp_reg_loss_scale).mean()
    res['residual/warp_reg'] = torch.sqrt(r).mean()
  return res


# --------------------------------------------------------------------------
# R12  parameter construction with the reference initialisers
# --------------------------------------------------------------------------
def tree_to(tree, dtype):
  if isinstance(tree, dict):
    return {k: tree_to(v, dtype) for k, v in tree.items()}
  if torch.is_tensor(tree) and tree.is_floating_point():
    return tree.to(dtype)
  return tree


def _glorot(gen, fan_in, fan_out):
  a = math.sqrt(6.0 / (fan_in + fan_out))
  return (torch.rand(fan_in, fan_out, generator=gen) * 2 - 1) * a


def _uniform(gen, shape, scale):
  return torch.rand(*shape, generator=gen) * scale


def _dense_init(gen, fan_in, fan_out, kind='glorot', scale=None):
  if kind == 'glorot':
    k = _glorot(gen, fan_in, fan_out)
  else:
    k = _uniform(gen, (fan_in, fan_out), scale)
  return {'kernel': k, 'bias': torch.zeros(fan_out)}


def _mlp_init(gen, in_dim, depth, width, skips, out_channels=0,
              out_kind='glorot', out_scale=None):
  p = {}
  d = in_dim
  for i in range(depth):
    if i in skips:
      d = d + in_dim
    p[f'hidden_{i}'] = _dense_init(gen, d, width)
    d = width
  if out_channels > 0:
    p['logit'] = _dense_init(gen, d, out_channels, out_kind, out_scale)
  return p


def cond_dims(spec: OracleSpec):
  """(trunk, alpha, rgb) condition widths per models.py:186-228."""
  t = a = r = 0
  if spec.use_viewdirs:
    r += 3 + 6 * spec.num_nerf_viewdir_freqs
  if spec.use_appearance_metadata:
    if spec.use_trunk_condition:
      t += spec.num_appearance_features
    if spec.use_alpha_condition:
      a += spec.num_appearance_features
      r += spec.num_appearance_features
  if spec.use_camera_metadata:
    r += spec.num_camera_features
  return t, a, r


def init_params(spec: OracleSpec, seed: int = 0) -> Dict[str, Any]:
  """Random parameters with the reference's initialisers (SURVEY §8a R12):
  glorot-uniform Dense kernels, zero biases, warp heads U[0,1e-4), embeddings
  U[0,0.05).  (Not bit-identical to jax.random - only the distributions.)"""
  gen = torch.Generator().manual_seed(seed)
  params = {}
  if spec.use_warp:
    dw = 3 + 6 * spec.num_warp_freqs + spec.num_warp_features
    glo = lambda: {'embed': {'embedding': _uniform(
        gen, (spec.num_warp_embeddings, spec.num_warp_features), 0.05)}}
    tenc = lambda: {'mlp': _mlp_init(
        gen, 1 + 2 * spec.metadata_encoder_num_freqs, TIME_ENCODER_DEPTH,
        TIME_ENCODER_WIDTH, TIME_ENCODER_SKIPS, spec.num_warp_features,
        'uniform', 0.05)}
    if spec.warp_metadata_encoder_type == 'glo':
      wf = {'metadata_encoder': glo()}
    elif spec.warp_metadata_encoder_type == 'time':
      wf = {'metadata_encoder': tenc()}
    else:
      wf = {'glo_encoder': glo(), 'time_encoder': tenc()}
    if spec.warp_field_type == 'se3':
      wf['trunk'] = _mlp_init(gen, dw, spec.warp_trunk_depth,
                              spec.warp_trunk_width, spec.warp_skips)
      wf['branches_w'] = {'logit': _dense_init(
          gen, spec.warp_trunk_width, 3, 'uniform', 1e-4)}
      wf['branches_v'] = {'logit': _dense_init(
          gen, spec.warp_trunk_width, 3, 'uniform', 1e-4)}
      if spec.warp_use_pivot:
        wf['branches_p'] = {'logit': _dense_init(
            gen, spec.warp_trunk_width, 3, 'uniform', 1e-4)}
      if spec.warp_use_translation:
        wf['branches_t'] = {'logit': _dense_init(
            gen, spec.warp_trunk_width, 3, 'uniform', 1e-4)}
    else:
      wf['mlp'] = _mlp_init(gen, dw, spec.warp_trunk_depth,
                            spec.warp_trunk_width, spec.warp_skips, 3,
                            'uniform', 1e-4)
    params['warp_field'] = wf
  if spec.use_appearance_metadata:
    params['appearance_encoder'] = {'embed': {'embedding': _uniform(
        gen, (spec.num_appearance_embeddings, spec.num_appearance_features),
        0.05)}}
  if spec.use_camera_metadata:
    params['camera_encoder'] = {'embed': {'embedding': _uniform(
        gen, (spec.num_camera_embeddings, spec.num_camera_features), 0.05)}}
  tc, ac, rc = cond_dims(spec)
  dp = 3 + 6 * spec.num_nerf_point_freqs
  levels = ['coarse'] + (['fine'] if spec.num_fine_samples > 0 else [])
  for level in levels:
    m = {}
    m['MLP_0'] = _mlp_init(gen, dp + tc, spec.nerf_trunk_depth,
                           spec.nerf_trunk_width, spec.nerf_skips)
    w = spec.nerf_trunk_width
    if ac or rc:
      m['bottleneck'] = _dense_init(gen, w, w)
    m['MLP_1'] = _mlp_init(gen, w + rc, spec.nerf_rgb_branch_depth,
                           spec.nerf_rgb_branch_width, (), spec.rgb_channels)
    m['MLP_2'] = _mlp_init(gen, w + ac, 0, 128, (), spec.alpha_channels)
    params[f'nerf_mlps_{level}'] = m
  return params


def make_trained_like(params, scale: float = 3.0, bias_std: float = 0.1,
                      seed: int = 1):
  """A second, non-degenerate weight set (SURVEY §8d): hidden kernels x scale^
  (1/depth-ish) and non-zero biases so sigma/alpha/the resampled PDF vary."""
  gen = torch.Generator().manual_seed(seed)

  def rec(t, path):
    if isinstance(t, dict):
      return {k: rec(v, path + (k,)) for k, v in t.items()}
    if 'warp_field' in path and path[-2] == 'logit':
      # keep the warp small but non-trivial: rotation/translation ~1e-2.
      if path[-1] == 'kernel':
        return (torch.rand(t.shape, generator=gen) * 2 - 1) * 2e-3
      return (torch.rand(t.shape, generator=gen) * 2 - 1) * 1e-2
    if path[-1] == 'kernel':
      if path[-2] == 'logit' and 'MLP_2' in path:
        return t * (4.0 * scale)  # density head: make sigma vary strongly.
      if path[-2] == 'logit':
        return t * scale
      return t * 1.3
    if path[-1] == 'bias':
      return torch.randn(t.shape, generator=gen) * bias_std
    return t

  return rec(params, ())


def synthetic_rays(num_rays: int, spec: OracleSpec, seed: int = 0):
  """Seeded synthetic inputs of SURVEY.md §8(d)."""
  gen = torch.Generator().manual_seed(seed)
  origins = torch.rand(num_rays, 3, generator=gen) - 0.5
  d = torch.randn(num_rays, 3, generator=gen)
  directions = d / torch.linalg.norm(d, dim=-1, keepdim=True)
  md = {
      'warp': torch.randint(0, spec.num_warp_embeddings, (num_rays, 1),
                            generator=gen, dtype=torch.int32),
      'appearance': torch.randint(0, spec.num_appearance_embeddings,
                                  (num_rays, 1), generator=gen,
                                  dtype=torch.int32),
      'camera': torch.randint(0, spec.num_camera_embeddings, (num_rays, 1),
                              generator=gen, dtype=torch.int32),
  }
  return {'origins': origins, 'directions': directions, 'metadata': md}
