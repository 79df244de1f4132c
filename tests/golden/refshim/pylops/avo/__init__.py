from . import poststack  # noqa: F401
