"""What nerfies/datasets/core.py needs of TensorFlow to import and run its preloaded path:
TensorSpec and dtypes for its signatures, and an in-memory tf.data.Dataset with
from_tensor_slices / repeat / batch / iteration.

TEST INFRASTRUCTURE: oracle/make_golden_data.py calls `install(tensorflow)` before it imports
the reference's datasets package, which adds these names to the file-IO stub's namespace."""
import types

import numpy as np


class DType:
  def __init__(self, np_dtype):
    self.as_numpy_dtype = np_dtype


float32, uint32, int32, string = DType(np.float32), DType(np.uint32), DType(np.int32), DType(object)


class TensorSpec:
  def __init__(self, shape=None, dtype=None):
    self.shape, self.dtype = shape, dtype


class Tensor(np.ndarray):
  """An eager tensor: numpy with the `_numpy()` accessor prepare_tf_data calls."""

  def _numpy(self):
    return np.asarray(self)


def _tree(f, t):
  return {k: _tree(f, v) for k, v in t.items()} if isinstance(t, dict) else f(t)


class Dataset:
  """Dataset.from_tensor_slices(tree) -> .repeat() -> .batch(n): batches of consecutive
  elements, across the epoch boundary when repeated; the last batch is partial otherwise."""

  def __init__(self, tree, repeat=False, batch=0):
    self._tree, self._repeat, self._batch = tree, repeat, batch
    leaves = []
    _tree(leaves.append, tree)
    self._n = len(leaves[0]) if leaves else 0

  @staticmethod
  def from_tensor_slices(tree):
    return Dataset(_tree(np.asarray, tree))

  def repeat(self):
    return Dataset(self._tree, True, self._batch)

  def batch(self, n):
    return Dataset(self._tree, self._repeat, n)

  def __iter__(self):
    step = self._batch or 1
    start = 0
    while self._repeat or start < self._n:
      idx = np.arange(start, start + step)
      if not self._repeat:
        idx = idx[idx < self._n]
      idx = idx % self._n
      take = (lambda x: x[idx]) if self._batch else (lambda x: x[idx[0]])
      yield _tree(lambda x: np.asarray(take(x)).view(Tensor), self._tree)
      start += step


def install(tf):
  """Adds the names above to the `tensorflow` stand-in module `tf`."""
  tf.float32, tf.uint32, tf.int32, tf.string = float32, uint32, int32, string
  tf.dtypes = types.SimpleNamespace(as_dtype=lambda d: d if isinstance(d, DType) else DType(d),
                                    float32=float32, uint32=uint32, int32=int32)
  tf.TensorSpec = TensorSpec
  tf.data = types.SimpleNamespace(Dataset=Dataset, experimental=types.SimpleNamespace(AUTOTUNE=-1))
