"""The scalar and binary quantizers in NumPy (DESIGN.md "Quantizers"), value for value.

Scalar: a quantile range [min_, max_] taken from the sorted values (`quantile_positions` gives the ranks), the code of x is
-128 at or below lo (and for NaN), 127 at or above hi, else lroundf(float32(scale * x + offset)) with the product and the sum
rounded separately in float64 (as NumPy does); the inverse maps code c to T((c - offset) / scale).  Binary: bit j % 8 of byte
j // 8 is x_j > t_j in the rows' type, packed LSB first; the thresholds are zero, the column mean, or the column median of a
row sample of odd size `median_sample_size`.  The row draw itself is the library's own, so `scalar_train` and the median are
stated only for samples that are the whole dataset.
"""
from __future__ import annotations

import math

import numpy as np

SCALAR_SAMPLE_VALUES = 1_000_000


def scalar_sample_rows(n, d):
    """R = min(n, max(1, floor(1e6 / d))): the rows the scalar quantizer samples."""
    return min(n, max(1, SCALAR_SAMPLE_VALUES // d))


def quantile_positions(S, quantile):
    """(rank of min_, rank of max_) among S sorted values: p = ceil((0.5 + 0.5 q) S) - 1 in float64, min at S - 1 - p.
    `quantile` is taken as the float32 the params struct holds."""
    q = float(np.float32(quantile))
    p = math.ceil((0.5 + 0.5 * q) * S) - 1
    return S - 1 - p, p


def scalar_train(x, quantile):
    """(min_, max_) as Python floats for a dataset whose sample is the whole of it."""
    x = np.asarray(x)
    n, d = x.shape
    assert scalar_sample_rows(n, d) == n, "the restatement covers whole-dataset samples only"
    v = np.sort(x.ravel())
    lo, hi = quantile_positions(v.size, quantile)
    return float(v[lo]), float(v[hi])


def scalar_map(min_, max_, dtype):
    """(lo, hi in dtype, scale, offset): lo = T(min_), hi = T(max_); scale = 255 / (hi - lo) if hi > lo else 1;
    offset = -128 - lo * scale."""
    with np.errstate(over="ignore"):
        lo, hi = np.array(min_, np.float64).astype(dtype), np.array(max_, np.float64).astype(dtype)
    l, h = float(lo), float(hi)
    scale = 255.0 / (h - l) if h > l else 1.0
    offset = -128.0 - l * scale
    return lo, hi, scale, offset


def lroundf(f):
    """C lroundf of float32 values: round half away from zero (exact in float64)."""
    f = np.asarray(f, np.float32).astype(np.float64)
    return (np.sign(f) * np.floor(np.abs(f) + 0.5)).astype(np.int64)


def scalar_transform(x, min_, max_):
    x = np.asarray(x)
    lo, hi, scale, offset = scalar_map(min_, max_, x.dtype)
    y = np.multiply(scale, x.astype(np.float64))
    y = np.add(y, offset)
    with np.errstate(invalid="ignore", over="ignore"):
        mid = lroundf(y.astype(np.float32))
        below = ~(x > lo)  # at or below lo, and NaN
        above = x >= hi
    out = np.where(below, -128, np.where(above, 127, np.where(below | above, 0, mid)))
    return out.astype(np.int8)


def scalar_inverse(codes, min_, max_, dtype=np.float32):
    _, _, scale, offset = scalar_map(min_, max_, dtype)
    table = ((np.arange(-128, 128, dtype=np.float64) - offset) / scale).astype(dtype)
    return table[np.asarray(codes, np.int8).astype(np.int64) + 128]


def median_sample_size(n, ratio):
    """s = max(2 * ceil(floor(n * ratio) / 2), 2) - 1 with n * ratio a float32 product; odd and at most n."""
    m = int(np.float32(n) * np.float32(ratio))
    s = max((m + 1) // 2 * 2, 2) - 1
    if s > n:
        s = n if n % 2 else n - 1
    return s


def thresholds(x, kind, sampling_ratio=0.1):
    """Per-column thresholds in x's type: None for "zero", the mean (exact where the float64 sums are), or the median of a
    sample that is every row ("sampling_median" with an odd n whose sample size is n)."""
    x = np.asarray(x)
    n = x.shape[0]
    if kind == "zero":
        return None
    if kind == "mean":
        return (x.astype(np.float64).sum(0) / n).astype(x.dtype)
    assert kind == "sampling_median"
    s = median_sample_size(n, sampling_ratio)
    assert s == n, "the restatement covers whole-dataset samples only"
    return np.sort(x, axis=0)[(s - 1) // 2]


def pack(x, t=None):
    """uint8 [n, ceil(d / 8)]: bit j % 8 of byte j // 8 set iff x_j > t_j (t = 0), LSB first."""
    x = np.asarray(x)
    t = np.zeros(x.shape[1], x.dtype) if t is None else np.asarray(t, x.dtype)
    with np.errstate(invalid="ignore"):
        return np.packbits(x > t[None, :], axis=1, bitorder="little")
