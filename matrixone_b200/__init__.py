"""matrixone_b200 -- H100 (sm_90a) batch operators and vector-distance kernels behind MatrixOne's cgo C-ABI.

The product is the shared library `libmo_b200.so` (include/mo_b200.h); this package is its Python harness:
  capi      ctypes prototypes of every exported symbol
  vector    host mirror of vector.Vector / nulls bitmap / varlena cells / XCall argument blocks
  ops       the reference-facing operator calls (Q6 / Q1 / aggregates / brute-force & IVF search) over the C-ABI
  datagen   numpy twin of the device-side synthetic column generators
There is no CPU implementation in here: without the built library and a CUDA device every call raises.
"""
from . import capi  # noqa: F401
from .capi import MoError, load_library  # noqa: F401

__all__ = ["capi", "MoError", "load_library"]
