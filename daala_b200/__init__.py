"""daala_b200 -- H100-native (sm_90a) per-block encode hot path of xiph/daala.

The product is the CUDA library `libdaala_b200.so` (C ABI: include/daala_b200.h);
this package is the thin Python host side: ctypes bindings (`_native`), frame
geometry + device-buffer plumbing (`frame`), synthetic content (`synth`).
PyTorch is used only for device memory, streams and torch.distributed.
"""
from . import _native  # noqa: F401

__all__ = ["_native"]
__version__ = "0.1"
