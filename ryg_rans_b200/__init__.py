"""ryg_rans_b200 -- GPU-native (H100) interleaved rANS coder behind ryg_rans's API surface.

The product is the C-ABI shared library ``librans_b200.so`` (CUDA kernels for sm_90a
+ C++ host code, sources in ``csrc/``, interface in ``include/rans_b200.h``).  This
Python package is only plumbing for tests and benchmarks: it builds the library
in-tree with nvcc and exposes it through ctypes.  There is NO CPU fallback: if the
library is missing or no GPU is visible, calls fail loudly.
"""
from .build import build, LIB_PATH  # noqa: F401
from .api import (  # noqa: F401
    Lib, Context, Model, RansError, SymbolStats,
    CODER_WORD, CODER_BYTE, CODER_ALIAS, CODER_RANS64, MEM_HOST, MEM_DEVICE, LANES,
    load,
)

__all__ = ["build", "load", "Lib", "Context", "Model", "RansError", "SymbolStats",
           "CODER_WORD", "CODER_BYTE", "CODER_ALIAS", "CODER_RANS64", "MEM_HOST", "MEM_DEVICE", "LANES", "LIB_PATH"]
