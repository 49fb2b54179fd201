"""rnc — H100-native kernels (librnc.so) and host-side drivers for RAFT-NCUP's per-iteration hot path."""
from . import native  # noqa: F401
