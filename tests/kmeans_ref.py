"""float64 model of k-means' assignment, cost and Lloyd update, and the error bound of the fixed-point centroid sums.

The GPU's labels are held to the oracle's fp32 expanded-L2 argmin (`oracle.kmeans_assign`); everything else — costs, updated
centres — is held to the float64 values computed here from differences, so an error in the kernels' arithmetic cannot hide in
a reference that makes the same error.
"""
import math

import numpy as np


def _chunks(n, width, budget=1 << 24):
    step = max(1, budget // max(1, width))
    for r0 in range(0, n, step):
        yield r0, min(n, r0 + step)


def assign(x, c):
    """argmin_j ||x_i - c_j||^2 in float64 from differences; ties go to the smaller j (np.argmin keeps the first)."""
    x, c = np.asarray(x, np.float64), np.asarray(c, np.float64)
    labels = np.empty(x.shape[0], np.int64)
    for r0, r1 in _chunks(x.shape[0], c.shape[0] * x.shape[1]):
        d = ((x[r0:r1, None, :] - c[None, :, :]) ** 2).sum(-1)
        labels[r0:r1] = d.argmin(1)
    return labels


def point_costs(x, c, labels):
    """||x_i - c_{labels_i}||^2 in float64, from differences."""
    x, c = np.asarray(x, np.float64), np.asarray(c, np.float64)
    labels = np.asarray(labels, np.int64)
    out = np.empty(x.shape[0], np.float64)
    for r0, r1 in _chunks(x.shape[0], x.shape[1]):
        out[r0:r1] = ((x[r0:r1] - c[labels[r0:r1]]) ** 2).sum(1)
    return out


def cost(x, c, labels, weights=None, normalize_weight=False, sqrt=False):
    """sum_i w_i * ||x_i - c_{labels_i}||^2 in float64 (sqrt: sum_i w_i * ||x_i - c_{labels_i}||).  normalize_weight rescales the
    weights to sum to n first, w_i * n / sum(w), as the reference's predict does; without weights every w_i is 1."""
    d = point_costs(x, c, labels)
    if sqrt:
        d = np.sqrt(d)
    if weights is None:
        return float(d.sum())
    w = np.asarray(weights, np.float64)
    if normalize_weight:
        w = w * (x.shape[0] / w.sum())
    return float((w * d).sum())


def lloyd_update(x, labels, c_old):
    """One Lloyd update in extended precision: the mean of each cluster's members; a cluster without members keeps its old
    centre.  Returns (centres as np.longdouble, member counts)."""
    x = np.asarray(x, np.float32)
    labels = np.asarray(labels, np.int64)
    k, d = c_old.shape
    counts = np.bincount(labels, minlength=k)
    order = np.argsort(labels, kind="stable")
    xs = x[order].astype(np.longdouble)
    new = np.asarray(c_old, np.float32).astype(np.longdouble)
    live = np.flatnonzero(counts)
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])[live]
    sums = np.add.reduceat(xs, starts, axis=0) if len(live) else np.zeros((0, d), np.longdouble)
    new[live] = sums / counts[live, None].astype(np.longdouble)
    return new, counts


def fixed_quantum(x, n=None):
    """The unit of the fixed-point centroid sums (ivf_common.cuh fixed_scale): 2^(ex + nb - 62), where max|x| < 2^ex (frexp of
    the largest magnitude) and n < 2^nb, n the number of summed rows (default: the rows of x).  Each term is rounded to a
    whole unit, so a cluster's mean is within quantum / 2 of the exact mean before it is rounded to fp32."""
    x = np.asarray(x, np.float32)
    n = x.shape[0] if n is None else n
    m = float(np.abs(x).max()) if x.size else 0.0
    ex = math.frexp(m)[1]
    nb = max(int(n), 1).bit_length()
    return math.ldexp(1.0, max(ex + nb - 62, -1000))


def update_bound(gpu_centres, ref_centres, quantum):
    """Per-coordinate bar of a fixed-point Lloyd update against lloyd_update: quantum / 2 from the rounded terms, half an fp32
    ulp of the centre from the final cast, and 2^-50 |centre| for the two double roundings (int64 -> double, the division)."""
    g = np.asarray(gpu_centres, np.float32)
    r = np.asarray(ref_centres, np.longdouble)
    ulp = np.maximum(np.spacing(np.abs(g)), np.spacing(np.abs(r.astype(np.float32))))
    return quantum / 2 + 0.5 * ulp.astype(np.longdouble) + np.abs(r) * np.longdouble(2.0 ** -50)


def relative_cost_bar(d):
    """Relative error allowed for a cost summed from fp32 squared differences of d components: max(1e-6, d * 2^-24)."""
    return max(1e-6, d * 2.0 ** -24)
