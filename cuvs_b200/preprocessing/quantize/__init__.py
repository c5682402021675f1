"""Quantizers — mirrors python/cuvs/cuvs/preprocessing/quantize: ``scalar`` (float rows to int8 codes and back) and
``binary`` (float rows to packed bits)."""
from . import binary, scalar  # noqa: F401

__all__ = ["binary", "scalar"]
