"""Preprocessing — mirrors python/cuvs/cuvs/preprocessing: the scalar and binary quantizers."""
from . import quantize  # noqa: F401
