from . import data  # noqa: F401
