"""flax.jax_utils for nerfies/datasets/core.py (single device: nothing to replicate or prefetch)."""


def replicate(tree, devices=None):
  return tree


def prefetch_to_device(iterator, size, devices=None):
  return iterator
