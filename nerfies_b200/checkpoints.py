"""Reading (and writing) the reference's training checkpoints (SURVEY §8(f) row 4).

The reference saves `flax.training.checkpoints.save_checkpoint(path, state, step)`
(nerfies/training.py:46-53) and `eval.py:364` / `train.py:232` restore it.  flax
(`flax==0.3.4`, requirements.txt:2) is a third-party dependency that is absent
from /root/reference and cannot be installed here, so its published on-disk
format is restated (flax/serialization.py, flax/training/checkpoints.py of the
0.3 line) - "parity unpinned" against a file written by real flax:

  * a checkpoint is one file `<dir>/checkpoint_<step>`; restore picks the one with
    the largest step (natural sort of the numeric suffix);
  * the bytes are msgpack of the state dict of the pytree.  Leaves use msgpack
    extension types: 1 = ndarray, packed as msgpack((shape, dtype.name, raw C-order
    bytes)); 2 = native complex (two doubles); 3 = numpy scalar (same layout as 1).
    Arrays above 2^30 bytes are split: {'__msgpack_chunked_array__': True,
    'shape': (...), 'chunks': {'0': ndarray, '1': ...}};
  * TrainState (model_utils.py:25-33) serialises as {'optimizer': {'target': {...},
    'state': {'step': i, 'param_states': {...}}}, 'warp_alpha': a, 'time_alpha': t};
    `target` is {'model': params} with the Flax parameter names this package uses
    natively (`warp_field/trunk/hidden_0/kernel`, ...), Dense kernels (in, out).

Pure host code: no kernel, no device work except the final `.to(device)`.
"""
import os
import re

import msgpack
import numpy as np
import torch

from nerfies_b200 import model_utils

_EXT_NDARRAY, _EXT_COMPLEX, _EXT_NPSCALAR = 1, 2, 3
_MAX_CHUNK_BYTES = 2**30


# ------------------------------------------------------------------ msgpack <-> pytree
def _ndarray_from_bytes(data):
  shape, dtype_name, buffer = msgpack.unpackb(data, raw=True)
  dtype_name = dtype_name.decode() if isinstance(dtype_name, bytes) else dtype_name
  return np.frombuffer(buffer, dtype=np.dtype(dtype_name)).reshape(tuple(shape)).copy()


def _ext_hook(code, data):
  if code == _EXT_NDARRAY:
    return _ndarray_from_bytes(data)
  if code == _EXT_NPSCALAR:
    return _ndarray_from_bytes(data)[()]
  if code == _EXT_COMPLEX:
    re_, im = msgpack.unpackb(data)
    return complex(re_, im)
  return msgpack.ExtType(code, data)


def _unchunk(tree):
  if isinstance(tree, dict):
    if tree.get('__msgpack_chunked_array__'):
      chunks = tree['chunks']
      flat = np.concatenate([np.asarray(chunks[str(i)]).reshape(-1) for i in range(len(chunks))])
      shape = tree['shape']
      if isinstance(shape, dict):      # flax writes _tuple_to_dict(shape): {'0': d0, '1': d1, ...}
        shape = [shape[str(i)] for i in range(len(shape))]
      return flat.reshape(tuple(int(d) for d in shape))
    return {k: _unchunk(v) for k, v in tree.items()}
  return tree


def msgpack_restore(encoded):
  """bytes -> nested dict of numpy arrays / python scalars (flax.serialization.msgpack_restore)."""
  tree = msgpack.unpackb(encoded, ext_hook=_ext_hook, raw=False, strict_map_key=False)
  return _unchunk(tree)


def _pack_ndarray(a):
  a = np.asarray(a)          # (ascontiguousarray would turn 0-d scalars into shape (1,))
  return msgpack.packb((a.shape, a.dtype.name, a.tobytes()), use_bin_type=True)


def _default(obj):
  if torch.is_tensor(obj):
    obj = obj.detach().cpu().numpy()
  if isinstance(obj, np.ndarray):
    return msgpack.ExtType(_EXT_NDARRAY, _pack_ndarray(obj))
  if isinstance(obj, np.generic):
    return msgpack.ExtType(_EXT_NPSCALAR, _pack_ndarray(np.asarray(obj)))
  if isinstance(obj, complex):
    return msgpack.ExtType(_EXT_COMPLEX, msgpack.packb((obj.real, obj.imag)))
  raise TypeError(f'cannot serialise {type(obj)!r}')


def _chunk(tree):
  if isinstance(tree, dict):
    return {k: _chunk(v) for k, v in tree.items()}
  if torch.is_tensor(tree):
    tree = tree.detach().cpu().numpy()
  if isinstance(tree, np.ndarray) and tree.nbytes > _MAX_CHUNK_BYTES:
    flat = tree.reshape(-1)
    per = max(1, _MAX_CHUNK_BYTES // tree.dtype.itemsize)
    chunks = {str(i): flat[s:s + per] for i, s in enumerate(range(0, flat.size, per))}
    # flax (serialization._chunk): the shape travels as _tuple_to_dict(shape), like `chunks`
    return {'__msgpack_chunked_array__': True,
            'shape': {str(i): int(d) for i, d in enumerate(tree.shape)}, 'chunks': chunks}
  return tree


def msgpack_serialize(tree):
  """Nested dict of arrays -> bytes in the layout flax.serialization.msgpack_serialize writes."""
  return msgpack.packb(_chunk(tree), default=_default, strict_types=True, use_bin_type=True)


# ------------------------------------------------------------------ checkpoint directory
def _step_of(name, prefix):
  m = re.fullmatch(re.escape(prefix) + r'(\d+(?:\.\d+)?)', name)
  return float(m.group(1)) if m else None


def latest_checkpoint(ckpt_dir, prefix='checkpoint_'):
  """Path of the checkpoint with the largest step in `ckpt_dir`, or None."""
  if not os.path.isdir(ckpt_dir):
    return None
  best = None
  for name in os.listdir(ckpt_dir):
    step = _step_of(name, prefix)
    if step is not None and (best is None or step > best[0]):
      best = (step, name)
  return os.path.join(ckpt_dir, best[1]) if best else None


def _to_torch(tree, device):
  if isinstance(tree, dict):
    return {k: _to_torch(v, device) for k, v in tree.items()}
  a = np.asarray(tree)
  if a.dtype == np.float64:
    a = a.astype(np.float32)
  return torch.from_numpy(np.ascontiguousarray(a)).to(device)


def restore_checkpoint(ckpt_dir, target=None, step=None, prefix='checkpoint_', device='cpu'):
  """flax.training.checkpoints.restore_checkpoint for the reference's TrainState.

  Returns `target` unchanged when the directory holds no checkpoint (the reference's
  behaviour for a fresh run); otherwise a `model_utils.TrainState` whose
  `optimizer.target['model']` is the parameter pytree (torch tensors on `device`,
  Flax names) and which carries `warp_alpha`, `time_alpha` and `.step`."""
  if os.path.isfile(ckpt_dir):
    path = ckpt_dir
  elif step is not None:
    path = os.path.join(ckpt_dir, f'{prefix}{step}')
    if not os.path.exists(path):
      raise ValueError(f'Matching checkpoint not found: {path}')
  else:
    path = latest_checkpoint(ckpt_dir, prefix)
    if path is None:
      return target
  with open(path, 'rb') as fp:
    state_dict = msgpack_restore(fp.read())
  try:
    opt = state_dict['optimizer']
    params = opt['target']
  except (KeyError, TypeError) as e:
    raise ValueError(f'{path} is not a nerfies TrainState checkpoint (missing {e})') from e
  if target is not None:
    _check_same_structure(target.optimizer.target, params, 'optimizer/target')
  state = model_utils.TrainState(
      model_utils.Optimizer(_to_torch(params, device)),
      warp_alpha=float(np.asarray(state_dict.get('warp_alpha', 0.0)).reshape(-1)[0]),
      time_alpha=float(np.asarray(state_dict.get('time_alpha', 0.0)).reshape(-1)[0]))
  state.step = int(np.asarray(opt.get('state', {}).get('step', 0)).reshape(-1)[0])
  # Adam's moments, {'model': {...: {'grad_ema', 'grad_sq_ema'}}}: what a resumed run needs
  state.param_states = _to_torch(opt.get('state', {}).get('param_states') or {}, device)
  return state


def _check_same_structure(want, got, where):
  """from_state_dict's structural check: same keys, same leaf shapes."""
  if isinstance(want, dict):
    if not isinstance(got, dict) or set(want) != set(got):
      raise ValueError(f'checkpoint structure mismatch at {where}: expected keys {sorted(want)}, '
                       f'found {sorted(got) if isinstance(got, dict) else type(got).__name__}')
    for k in want:
      _check_same_structure(want[k], got[k], f'{where}/{k}')
  else:
    ws, gs = tuple(want.shape), tuple(np.asarray(got).shape)
    if ws != gs:
      raise ValueError(f'checkpoint shape mismatch at {where}: expected {ws}, found {gs}')


def save_checkpoint(ckpt_dir, state, step, prefix='checkpoint_', keep=2):
  """Writes `state` in the reference's layout (training.py:46-53); keeps the newest `keep` files.
  An optimizer that has `param_states` (training.AdamOptimizer) gets its moments written where flax
  writes them, so that a run can resume; the plain `model_utils.Optimizer` has none."""
  os.makedirs(ckpt_dir, exist_ok=True)
  tree = {
      'optimizer': {'target': state.optimizer.target,
                    'state': {'step': np.asarray(step, np.int32),
                              'param_states': getattr(state.optimizer, 'param_states', {})}},
      'warp_alpha': np.asarray(state.warp_alpha, np.float32),
      'time_alpha': np.asarray(state.time_alpha, np.float32),
  }
  path = os.path.join(ckpt_dir, f'{prefix}{step}')
  tmp = path + '.tmp'
  with open(tmp, 'wb') as fp:
    fp.write(msgpack_serialize(tree))
  os.replace(tmp, path)
  steps = sorted((s, n) for n in os.listdir(ckpt_dir) if (s := _step_of(n, prefix)) is not None)
  for _, name in steps[:-keep] if keep else []:
    os.remove(os.path.join(ckpt_dir, name))
  return path
