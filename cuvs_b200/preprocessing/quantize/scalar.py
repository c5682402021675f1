"""Scalar quantizer — same surface as python/cuvs/cuvs/preprocessing/quantize/scalar/scalar.pyx (QuantizerParams, Quantizer,
train, transform, inverse_transform): float32 / float16 / float64 rows to int8 codes over a trained [min, max] range, and back.
Inputs are torch tensors or numpy arrays in host or device memory; results are torch tensors on the input's device."""
from __future__ import annotations

import ctypes as C

import torch

from ..._capi import DL, as_tensor, check, lib
from ...common.resources import auto_sync_resources
from ._common import empty_like_rows


class _ParamsC(C.Structure):  # include/cuvs/preprocessing/quantize/scalar.h: struct cuvsScalarQuantizerParams
    _fields_ = [("quantile", C.c_float)]


class _QuantizerC(C.Structure):  # cuvsScalarQuantizer
    _fields_ = [("min_", C.c_double), ("max_", C.c_double)]


class QuantizerParams:
    """quantile: the share of values kept inside [min, max], in (0, 1] (default 0.99); the rest are clipped."""

    def __init__(self, *, quantile=None):
        self._p = C.POINTER(_ParamsC)()
        check(lib.cuvsScalarQuantizerParamsCreate(C.byref(self._p)))
        if quantile is not None:
            self._p.contents.quantile = quantile

    def __del__(self):
        try:
            lib.cuvsScalarQuantizerParamsDestroy(self._p)
        except Exception:
            pass

    @property
    def quantile(self):
        return self._p.contents.quantile


class Quantizer:
    def __init__(self):
        self._p = C.POINTER(_QuantizerC)()
        check(lib.cuvsScalarQuantizerCreate(C.byref(self._p)))

    def __del__(self):
        try:
            if self._p:
                lib.cuvsScalarQuantizerDestroy(self._p)
                self._p = None
        except Exception:
            pass

    @property
    def min(self):
        return self._p.contents.min_

    @property
    def max(self):
        return self._p.contents.max_

    def __repr__(self):
        return f"scalar.Quantizer(min={self.min}, max={self.max})"


@auto_sync_resources
def train(params, dataset, resources=None):
    """A Quantizer whose [min, max] holds the central `params.quantile` share of a sample of `dataset`'s values."""
    x = as_tensor(dataset)
    q = Quantizer()
    check(lib.cuvsScalarQuantizerTrain(resources.get_c_obj(), params._p, DL(x).ptr, q._p))
    return q


@auto_sync_resources
def transform(quantizer, dataset, output=None, resources=None):
    """int8 codes of `dataset` (same shape); `output`, when given, receives them."""
    x = as_tensor(dataset)
    if output is None:
        output = empty_like_rows(x, tuple(x.shape), torch.int8)
    check(lib.cuvsScalarQuantizerTransform(resources.get_c_obj(), quantizer._p, DL(x).ptr, DL(as_tensor(output)).ptr))
    return output


@auto_sync_resources
def inverse_transform(quantizer, dataset, output=None, resources=None):
    """The values int8 codes stand for, float32 unless `output` (float32, float16 or float64) is given."""
    x = as_tensor(dataset)
    if output is None:
        output = empty_like_rows(x, tuple(x.shape), torch.float32)
    check(lib.cuvsScalarQuantizerInverseTransform(resources.get_c_obj(), quantizer._p, DL(x).ptr, DL(as_tensor(output)).ptr))
    return output
