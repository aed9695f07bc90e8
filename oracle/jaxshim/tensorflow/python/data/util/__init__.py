from . import nest  # noqa: F401
