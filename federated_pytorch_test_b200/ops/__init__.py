"""Operators: ``functional`` (dispatch + ATen oracle) and ``cuda_ops`` (sm_90a kernels)."""
from . import functional

__all__ = ["functional"]
