"""databend_b200 — H100-native replacement for Databend's in-memory vectorised execution hot
path, behind the reference's operator interface.  Compute lives in libdbx (CUDA, sm_90a)
reached through the C-ABI in include/dbx.h; there is no CPU fallback."""
from . import abi  # noqa: F401
from .block import Column, DataBlock  # noqa: F401
