"""Annealing schedules of train.py (the learning rate, warp_alpha, time_alpha and the elastic
loss weight), evaluated on the host.

Drop-in for `from nerfies import schedules` (nerfies/schedules.py:25-200): the same spec formats
- a tuple / list `('type', *args)`, a mapping `{'type': ..., **kwargs}` or a Schedule - and the
same schedule types.  `configs.TrainConfig`'s schedule fields are accepted as they are.

A schedule returns a Python float holding a float32 value.  The steps the reference evaluates
with jnp (the `minimum` / `clip` / `sin` / `searchsorted` terms) are computed in float32 here,
the ones it evaluates on Python floats in float64, so the values agree with the reference to the
last float32 bit or two (tests/test_datasource.py holds them to 1e-6 relative).
"""
import abc
import collections.abc
import math

import numpy as np

_f32 = np.float32


def _out(value):
  return float(_f32(value))


def _ratio(step, num_steps):
  """jnp.minimum(step / num_steps, 1.0): the quotient is rounded to float32."""
  return min(_f32(step / num_steps), _f32(1.0))


class Schedule(abc.ABC):
  """A value per training step; calling the schedule is `get`."""

  @abc.abstractmethod
  def get(self, step):
    """The value at `step` (a Python float)."""

  def __call__(self, step):
    return self.get(step)


class ConstantSchedule(Schedule):
  """`value` at every step."""

  def __init__(self, value):
    self.value = value

  def get(self, step):
    return _out(self.value)


class LinearSchedule(Schedule):
  """`initial_value` to `final_value` over `num_steps`, then constant."""

  def __init__(self, initial_value, final_value, num_steps):
    self.initial_value, self.final_value, self.num_steps = initial_value, final_value, num_steps

  def get(self, step):
    if self.num_steps == 0:
      return _out(self.final_value)
    a = _ratio(step, self.num_steps)
    return _out((_f32(1.0) - a) * _f32(self.initial_value) + a * _f32(self.final_value))


class ExponentialSchedule(Schedule):
  """Geometric decay from `initial_value` to max(`final_value`, eps) over `num_steps`."""

  def __init__(self, initial_value, final_value, num_steps, eps=1e-10):
    if initial_value <= final_value:
      raise ValueError('Final value must be less than initial value.')
    self.initial_value, self.final_value, self.num_steps, self.eps = (
        initial_value, final_value, num_steps, eps)

  def get(self, step):
    if step >= self.num_steps:
      return _out(self.final_value)
    ratio = max(self.final_value, self.eps) / self.initial_value
    return _out(self.initial_value * ratio**(step / (self.num_steps - 1)))


class CosineEasingSchedule(Schedule):
  """Half a cosine from `initial_value` to `final_value` over `num_steps`."""

  def __init__(self, initial_value, final_value, num_steps):
    self.initial_value, self.final_value, self.num_steps = initial_value, final_value, num_steps

  def get(self, step):
    x = min(max(_ratio(step, self.num_steps), _f32(0.0)), _f32(1.0))
    phase = _f32(math.pi) * x + _f32(math.pi)
    return _out(self.initial_value + (self.final_value - self.initial_value) * 0.5 * (1 + math.cos(phase)))


class StepSchedule(Schedule):
  """`initial_value * decay_factor**k` after k whole `decay_interval`s, up to `max_decays`."""

  def __init__(self, initial_value, decay_interval, decay_factor, max_decays, final_value=None):
    self.initial_value, self.decay_interval, self.decay_factor, self.max_decays = (
        initial_value, decay_interval, decay_factor, max_decays)
    self.final_value = (initial_value * decay_factor**max_decays if final_value is None
                        else final_value)

  def get(self, step):
    k = step // self.decay_interval
    if k >= self.max_decays:
      return _out(self.final_value)
    return _out(self.initial_value * self.decay_factor**k)


class PiecewiseSchedule(Schedule):
  """[(num_steps, schedule), ...]: each schedule runs for its steps, restarted at 0."""

  def __init__(self, schedules):
    schedules = list(schedules)
    self.schedules = [from_config(spec) for _, spec in schedules]
    # starts of the 2nd, 3rd, ... pieces (int32, as jnp.cumsum of Python ints)
    self.milestones = np.cumsum(np.array([n for n, _ in schedules], np.int32))[:-1]

  def get(self, step):
    k = int(np.searchsorted(self.milestones, step, side='right'))
    start = int(self.milestones[k - 1]) if k >= 1 else 0
    return self.schedules[k].get(step - start)


class DelayedSchedule(Schedule):
  """`base_schedule` scaled by a factor that rises from `delay_mult` to 1 as
  sin(pi/2 * t) over the first `delay_steps` steps."""

  def __init__(self, base_schedule, delay_steps, delay_mult):
    self.base_schedule = from_config(base_schedule)
    self.delay_steps, self.delay_mult = delay_steps, delay_mult

  def get(self, step):
    t = min(max(_f32(step / self.delay_steps), _f32(0.0)), _f32(1.0))
    rise = np.sin(_f32(0.5 * math.pi) * t, dtype=np.float32)
    factor = _f32(self.delay_mult) + _f32(1 - self.delay_mult) * rise
    return _out(factor * _f32(self.base_schedule(step)))


SCHEDULE_MAP = {
    'constant': ConstantSchedule,
    'linear': LinearSchedule,
    'exponential': ExponentialSchedule,
    'cosine_easing': CosineEasingSchedule,
    'step': StepSchedule,
    'piecewise': PiecewiseSchedule,
    'delayed': DelayedSchedule,
}


def _make(kind, args=(), kwargs=None):
  if kind not in SCHEDULE_MAP:
    raise ValueError(f'Unknown schedule type {kind!r}; known: {sorted(SCHEDULE_MAP)}')
  return SCHEDULE_MAP[kind](*args, **(kwargs or {}))


def from_tuple(spec):
  kind, *args = spec
  return _make(kind, args)


def from_dict(spec):
  spec = dict(spec)
  return _make(spec.pop('type'), kwargs=spec)


def from_config(spec):
  """A Schedule from a Schedule, a ('type', *args) tuple / list or a {'type': ...} mapping."""
  if isinstance(spec, Schedule):
    return spec
  if isinstance(spec, (tuple, list)):
    return from_tuple(spec)
  if isinstance(spec, collections.abc.Mapping):
    return from_dict(spec)
  raise ValueError(f'Unknown type {type(spec)}.')
