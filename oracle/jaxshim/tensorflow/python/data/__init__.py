from . import util  # noqa: F401
