"""scanner_b200 -- H100-native implementation of Scanner's decode -> evaluate -> save hot path.

Layers (see DESIGN.md):
  include/scn_kernels.h + scanner_b200/csrc   hand-written sm_90a kernels behind a C ABI
  include/scanner/...   + scanner_b200/csrc/engine   C++ host pipeline with Scanner's
                                                     REGISTER_OP / REGISTER_KERNEL plugin API
  scanner_b200/*.py     thin Python surface (ctypes over the C ABI; scannerpy-shaped graph API)

There is no CPU fallback: importing works anywhere, but every op raises if the CUDA library is
missing or no device is present.
"""
from . import cabi  # noqa: F401
from . import types  # noqa: F401
from .client import (CacheMode, Client, ColumnType, DeviceHandle, DeviceType, FilesStream, NamedStream,  # noqa: F401
                     NamedVideoStream, NullElement, PerfParams, ScannerException, SliceList)
from .pyops import Kernel, KernelConfig, register_python_op  # noqa: F401
from .types import BlobType, FrameType  # noqa: F401

__all__ = ["cabi", "Client", "DeviceType", "PerfParams", "NamedStream", "NamedVideoStream", "CacheMode",
           "ScannerException", "SliceList", "NullElement", "FilesStream", "ColumnType", "DeviceHandle", "BlobType", "register_python_op", "Kernel", "KernelConfig", "FrameType", "types"]
