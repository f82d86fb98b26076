"""Optimizers: ``LBFGSNew`` (reference-compatible) and the fused block Adam and SGD."""
from .block_sgd import BlockSGD
from .lbfgsnew import LBFGSNew

__all__ = ["BlockSGD", "LBFGSNew"]
