"""tensorflow.python.data.util.nest: imported by nerfies/datasets/core.py, used only by its lazy
tf.data path, which oracle/make_golden_data.py does not run."""
