"""trino_b200 — H100-native (sm_90a) implementation of Trino's columnar operator hot path.

The product is trino_b200/libtrino_gpu.so (hand-written CUDA behind the C ABI of include/trino_gpu.h);
this package is the thin host-side mirror of the reference's Operator/OperatorFactory interface.
"""
from . import abi  # noqa: F401
from .page import Block, DictionaryBlock, Page, RunLengthEncodedBlock  # noqa: F401

__all__ = ["abi", "Block", "DictionaryBlock", "RunLengthEncodedBlock", "Page"]
