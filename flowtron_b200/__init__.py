"""flowtron_b200 — H100-native (sm_90a) implementation of the Flowtron AR-flow hot path."""
from . import _lib  # noqa: F401
