"""Configuration surface of the reference (nerfies/configs.py:35-212).

Same dataclasses, same field names and defaults, so the reference's gin files
parse unchanged.  `gin-config` is not available here, so `parse_config_files_and_bindings`
implements the subset of the gin language those files use: `include`, macros
(`name = value`, `%name`), `Class.field = value` bindings with Python literals,
and `@nn.relu`-style references to the activations registered at
configs.py:27-32.  Activations are carried as strings ('relu', 'softplus', ...).
"""
import ast
import dataclasses
import os
import re
from typing import Any, Mapping, Optional, Tuple

ScheduleDef = Any

# gin.config.external_configurable(nn.<act>, module='flax.nn')  (configs.py:27-32)
ACTIVATIONS = ('elu', 'relu', 'leaky_relu', 'tanh', 'sigmoid', 'softplus')
REQUIRED = object()

_BINDINGS = {}   # 'ModelConfig.field' -> value; filled by the parser


def activation_name(act) -> str:
  """Accepts 'relu' or a callable named relu (jax.nn.relu / torch.relu ...)."""
  if isinstance(act, str):
    name = act
  else:
    name = getattr(act, '__name__', None) or str(act)
  name = name.split('.')[-1]
  if name not in ACTIVATIONS:
    raise ValueError(f'unsupported activation {act!r}; the reference registers '
                     f'{ACTIVATIONS} (configs.py:27-32)')
  return name


def _configurable(cls):
  """gin.configurable(): constructor defaults are overridden by bindings."""
  orig_init = cls.__init__
  field_names = {f.name for f in dataclasses.fields(cls)}

  def __init__(self, *args, **kwargs):
    prefix = cls.__name__ + '.'
    for key, value in _BINDINGS.items():
      if key.startswith(prefix):
        field = key[len(prefix):]
        if field not in field_names:
          raise ValueError(f'gin binding for unknown field {key}')
        kwargs.setdefault(field, value)
    orig_init(self, *args, **kwargs)
    for f in dataclasses.fields(cls):
      if getattr(self, f.name) is REQUIRED:
        raise ValueError(f'{cls.__name__}.{f.name} is required (gin.REQUIRED)')

  cls.__init__ = __init__
  return cls


@_configurable
@dataclasses.dataclass
class ModelConfig:
  """Parameters for the model (configs.py:37-105)."""
  use_linear_disparity: bool = False
  use_white_background: bool = False
  use_stratified_sampling: bool = True
  use_sample_at_infinity: bool = True
  noise_std: Optional[float] = None
  nerf_trunk_depth: int = 8
  nerf_trunk_width: int = 256
  nerf_rgb_branch_depth: int = 1
  nerf_rgb_branch_width: int = 128
  activation: Any = 'relu'
  sigma_activation: Any = 'relu'
  nerf_skips: Tuple[int, ...] = (4,)
  alpha_channels: int = 1
  rgb_channels: int = 3
  num_nerf_point_freqs: int = 10
  num_nerf_viewdir_freqs: int = 4
  num_coarse_samples: int = 64
  num_fine_samples: int = 128
  use_viewdirs: bool = True
  use_trunk_condition: bool = False
  use_alpha_condition: bool = False
  use_rgb_condition: bool = False
  use_appearance_metadata: bool = False
  appearance_metadata_dims: int = 8
  use_camera_metadata: bool = False
  camera_metadata_dims: int = 2
  use_warp: bool = False
  num_warp_freqs: int = 8
  num_warp_features: int = 8
  warp_field_type: str = 'translation'
  warp_metadata_encoder_type: str = 'glo'
  warp_kwargs: Mapping[str, Any] = dataclasses.field(default_factory=dict)


@_configurable
@dataclasses.dataclass
class ExperimentConfig:
  """configs.py:108-124."""
  subname: Optional[str] = None
  image_scale: int = 4
  random_seed: int = 12345
  datasource_type: str = 'nerfies'
  datasource_spec: Optional[Mapping[str, Any]] = None
  datasource_kwargs: Mapping[str, Any] = dataclasses.field(default_factory=dict)


@_configurable
@dataclasses.dataclass
class TrainConfig:
  """configs.py:127-190."""
  batch_size: Any = REQUIRED
  lr_schedule: ScheduleDef = dataclasses.field(default_factory=lambda: {
      'type': 'exponential', 'initial_value': 0.001, 'final_value': 0.0001,
      'num_steps': 1000000})
  max_steps: int = 1000000
  warp_alpha_schedule: ScheduleDef = dataclasses.field(default_factory=lambda: {
      'type': 'linear', 'initial_value': 0.0, 'final_value': 8.0,
      'num_steps': 80000})
  time_alpha_schedule: ScheduleDef = ('constant', 0.0)
  use_elastic_loss: bool = False
  elastic_loss_weight_schedule: ScheduleDef = ('constant', 0.0)
  elastic_reduce_method: str = 'weight'
  elastic_loss_type: str = 'log_svals'
  use_background_loss: bool = False
  background_loss_weight: float = 0.0
  background_points_batch_size: int = 16384
  use_warp_reg_loss: bool = False
  warp_reg_loss_weight: float = 0.0
  warp_reg_loss_alpha: float = -2.0
  warp_reg_loss_scale: float = 0.001
  shuffle_buffer_size: int = 5000000
  # Refine the training cameras' poses jointly with the model (training.CameraPoses): a rotation about each
  # camera centre and a move of the centre per train item, starting at zero.
  refine_camera_poses: bool = False
  # One Adam learning rate for the rotation (radians) and the translation (scene units), which are comparable
  # in a normalised scene.  The default is a guess that nobody has tuned.
  camera_pose_lr_schedule: ScheduleDef = dataclasses.field(default_factory=lambda: {
      'type': 'exponential', 'initial_value': 1e-3, 'final_value': 1e-5, 'num_steps': 1000000})
  # Refine the training cameras' intrinsics jointly with the model (training.CameraIntrinsics): the parts named
  # here, some of 'focal', 'principal_point', 'radial' and 'tangential', of one delta per group of train items
  # whose capture intrinsics are all equal, starting at zero.  Works with or without refine_camera_poses, but
  # a group's principal-point shift is nearly a rotation of each of its cameras about its centre: with both
  # on, 'principal_point' and the poses are close to degenerate.
  refine_camera_intrinsics: Tuple[str, ...] = ()
  # One Adam learning rate for the focal log-scale, the principal point (in focal lengths) and the distortion
  # coefficients.  The default is a guess that nobody has tuned.
  camera_intrinsics_lr_schedule: ScheduleDef = dataclasses.field(default_factory=lambda: {
      'type': 'exponential', 'initial_value': 1e-4, 'final_value': 1e-6, 'num_steps': 1000000})
  # Supervise the expected depth of both levels with the per-frame depth maps of the capture (L1 over the rays
  # with a measurement).  Needs ExperimentConfig.datasource_kwargs = {'use_depth': True} and depth/<s>x/ maps
  # (process_capture depth).
  use_depth_loss: bool = False
  # The weight of the depth loss; its scale is that of scene units against the photometric loss's squared
  # colours.  The default leaves the loss at no effect until a schedule is chosen.
  depth_loss_weight_schedule: ScheduleDef = ('constant', 0.0)
  save_every: int = 10000
  log_every: int = 500
  histogram_every: int = 5000
  print_every: int = 25


@_configurable
@dataclasses.dataclass
class EvalConfig:
  """configs.py:193-212."""
  eval_once: bool = False
  save_output: bool = True
  chunk: int = 8192
  max_render_checkpoints: int = 3
  num_val_eval: Optional[int] = 10
  num_train_eval: Optional[int] = 10
  num_test_eval: Optional[int] = 10


# ---------------------------------------------------------------------------
# gin subset
# ---------------------------------------------------------------------------
class _Ref:
  """'@nn.softplus' / '@flax.nn.relu' configurable reference."""

  def __init__(self, name):
    self.name = name


def _strip_comment(line):
  out, quote = [], None
  for ch in line:
    if quote:
      if ch == quote:
        quote = None
    elif ch in '\'"':
      quote = ch
    elif ch == '#':
      break
    out.append(ch)
  return ''.join(out).rstrip()


def _logical_statements(text):
  """Joins lines until brackets balance (gin values may span lines)."""
  buf, depth = [], 0
  for raw in text.splitlines():
    line = _strip_comment(raw)
    if not line.strip() and depth == 0:
      continue
    buf.append(line)
    depth += sum(line.count(c) for c in '([{') - sum(
        line.count(c) for c in ')]}')
    if depth <= 0:
      yield ' '.join(s.strip() for s in buf)
      buf, depth = [], 0
  if buf:
    raise ValueError('gin: unbalanced brackets in ' + ' '.join(buf))


_MACRO = re.compile(r'%([A-Za-z_][A-Za-z0-9_./]*)')
_REFERENCE = re.compile(r'@([A-Za-z_][A-Za-z0-9_./]*)(\(\))?')


def _evaluate(expr, macros, _stack=()):
  """Evaluates a gin value.  `macros` maps names to UNEVALUATED expressions:
  gin resolves %macros lazily, so a later file may override a macro that an
  earlier include already used (gpu_vrig_paper.gin:25 vs defaults.gin:19,29)."""
  placeholders = {}

  def sub_macro(m):
    name = m.group(1)
    if name not in macros:
      raise ValueError(f'gin: undefined macro %{name}')
    if name in _stack:
      raise ValueError(f'gin: recursive macro %{name}')
    key = f'__gin_{len(placeholders)}__'
    placeholders[key] = _evaluate(macros[name], macros, _stack + (name,))
    return repr(key)

  def sub_ref(m):
    key = f'__gin_{len(placeholders)}__'
    placeholders[key] = _Ref(m.group(1))
    return repr(key)

  expr = _MACRO.sub(sub_macro, expr)
  expr = _REFERENCE.sub(sub_ref, expr)
  value = ast.literal_eval(expr)

  def restore(v):
    if isinstance(v, str) and v in placeholders:
      return placeholders[v]
    if isinstance(v, dict):
      return {restore(k): restore(x) for k, x in v.items()}
    if isinstance(v, (list, tuple)):
      return type(v)(restore(x) for x in v)
    return v

  return restore(value)


def _resolve_refs(v):
  if isinstance(v, _Ref):
    return activation_name(v.name)
  if isinstance(v, dict):
    return {k: _resolve_refs(x) for k, x in v.items()}
  if isinstance(v, (list, tuple)):
    return type(v)(_resolve_refs(x) for x in v)
  return v


def _parse_text(text, macros, bindings, search_dirs, skip_unknown):
  known = {'ModelConfig', 'ExperimentConfig', 'TrainConfig', 'EvalConfig'}
  for stmt in _logical_statements(text):
    if stmt.startswith('include '):
      rel = ast.literal_eval(stmt[len('include '):].strip())
      for d in search_dirs:
        # the reference's files use both 'x.gin' and 'configs/x.gin'.
        for cand in (os.path.join(d, rel), os.path.join(d, os.path.basename(rel))):
          if os.path.exists(cand):
            with open(cand) as f:
              _parse_text(f.read(), macros, bindings,
                          [os.path.dirname(cand)] + search_dirs, skip_unknown)
            break
        else:
          continue
        break
      else:
        raise FileNotFoundError(f'gin include {rel!r} not found')
      continue
    if stmt.startswith('import '):
      continue
    if '=' not in stmt:
      raise ValueError(f'gin: cannot parse {stmt!r}')
    lhs, rhs = stmt.split('=', 1)
    lhs = lhs.strip()
    value = rhs.strip()
    if '.' in lhs:
      scope = lhs.split('.')[-2].split('/')[-1]
      field = lhs.split('.')[-1]
      if scope not in known:
        if skip_unknown:
          continue
        raise ValueError(f'gin: unknown configurable {scope!r}')
      bindings[f'{scope}.{field}'] = value
    else:
      macros[lhs] = value


def _resolve(macros, parsed):
  return {k: _resolve_refs(_evaluate(v, macros)) for k, v in parsed.items()}


def parse_config_files_and_bindings(config_files=None, bindings=None,
                                    skip_unknown=True):
  """gin.parse_config_files_and_bindings for the subset described above
  (train.py:107-110, eval.py:232-235)."""
  macros, parsed = {}, {}
  for path in config_files or []:
    with open(path) as f:
      _parse_text(f.read(), macros, parsed, [os.path.dirname(path) or '.'],
                  skip_unknown)
  if bindings:
    if isinstance(bindings, str):
      bindings = [bindings]
    _parse_text('\n'.join(bindings), macros, parsed, ['.'], skip_unknown)
  parsed = _resolve(macros, parsed)
  _BINDINGS.update(parsed)
  return dict(parsed)


def parse_config(text, skip_unknown=True):
  """gin.parse_config on a string."""
  macros, parsed = {}, {}
  _parse_text(text, macros, parsed, ['.'], skip_unknown)
  parsed = _resolve(macros, parsed)
  _BINDINGS.update(parsed)
  return dict(parsed)


def clear_config():
  _BINDINGS.clear()
