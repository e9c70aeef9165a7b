"""g2pc — host layer of the H100-native 3DGS-to-PC hot path (ctypes over libg2pc.so)."""
from . import config  # noqa: F401
