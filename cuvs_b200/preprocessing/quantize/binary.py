"""Binary quantizer — the surface of python/cuvs/cuvs/preprocessing/quantize/binary/binary.pyx (transform), plus the C ABI's
trained thresholds (QuantizerParams, Quantizer, train, and transform's ``quantizer=``).  Bit j % 8 of byte j // 8 of a row is
set when column j exceeds its threshold: numpy's ``packbits(x > t, axis=1, bitorder="little")``.  Inputs are torch tensors or
numpy arrays in host or device memory; results are uint8 torch tensors on the input's device."""
from __future__ import annotations

import ctypes as C

import torch

from ..._capi import DL, as_tensor, check, index_handle, lib
from ...common.resources import auto_sync_resources
from ._common import empty_like_rows

_THRESHOLDS = {"zero": 0, "mean": 1, "sampling_median": 2}


class _ParamsC(C.Structure):  # include/cuvs/preprocessing/quantize/binary.h: struct cuvsBinaryQuantizerParams
    _fields_ = [("threshold", C.c_int), ("sampling_ratio", C.c_float)]


class QuantizerParams:
    """threshold: "zero", "mean" (default: each column's mean) or "sampling_median" (each column's median over a sample of
    `sampling_ratio` of the rows, default 0.1)."""

    def __init__(self, *, threshold="mean", sampling_ratio=None):
        if threshold not in _THRESHOLDS:
            raise ValueError(f"threshold must be one of {sorted(_THRESHOLDS)}, got {threshold!r}")
        self._p = C.POINTER(_ParamsC)()
        check(lib.cuvsBinaryQuantizerParamsCreate(C.byref(self._p)))
        self._p.contents.threshold = _THRESHOLDS[threshold]
        if sampling_ratio is not None:
            self._p.contents.sampling_ratio = sampling_ratio

    def __del__(self):
        try:
            lib.cuvsBinaryQuantizerParamsDestroy(self._p)
        except Exception:
            pass

    @property
    def threshold(self):
        return {v: k for k, v in _THRESHOLDS.items()}[self._p.contents.threshold]

    @property
    def sampling_ratio(self):
        return self._p.contents.sampling_ratio


class Quantizer:
    def __init__(self):
        self._p = C.POINTER(index_handle)()
        check(lib.cuvsBinaryQuantizerCreate(C.byref(self._p)))

    def __del__(self):
        try:
            if self._p:
                lib.cuvsBinaryQuantizerDestroy(self._p)
                self._p = None
        except Exception:
            pass

    def __repr__(self):
        return "binary.Quantizer()"


@auto_sync_resources
def train(params, dataset, resources=None):
    """A Quantizer holding `dataset`'s per-column thresholds (none for "zero")."""
    x = as_tensor(dataset)
    q = Quantizer()
    check(lib.cuvsBinaryQuantizerTrain(resources.get_c_obj(), params._p, DL(x).ptr, q._p))
    return q


@auto_sync_resources
def transform(dataset, output=None, quantizer=None, resources=None):
    """uint8 [n, ceil(dim / 8)] bits of `dataset` against 0, or against `quantizer`'s thresholds.  A given `output` may be wider
    or longer: its extra bytes are zeroed and its extra rows left as they are."""
    x = as_tensor(dataset)
    if output is None:
        output = empty_like_rows(x, (x.shape[0], (x.shape[1] + 7) // 8), torch.uint8)
    o = DL(as_tensor(output))
    if quantizer is None:
        check(lib.cuvsBinaryQuantizerTransform(resources.get_c_obj(), DL(x).ptr, o.ptr))
    else:
        check(lib.cuvsBinaryQuantizerTransformWithParams(resources.get_c_obj(), quantizer._p, DL(x).ptr, o.ptr))
    return output
