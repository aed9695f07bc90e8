"""tf.experimental.numpy: nerfies/tf_camera.py only needs it to import (annotations)."""
import numpy  # noqa: F401
