"""The exact-integer IVF-Flat search of tests/ivf_int_ref.py against the oracle's, at widths where the oracle's fp32 sums are
exact (every partial sum below 2^24), so that the GPU tests may hold 8-bit searches at wider rows to it."""
import numpy as np
import pytest

import oracle
from tests.ivf_int_ref import int_ivf_search
from tests.ivf_oracle import assert_same_answer, certain_probes


def _lists(dtype, n, d, n_lists, seed):
    rng = np.random.default_rng(seed)
    lo, hi = (-128, 128) if dtype == np.int8 else (0, 256)
    centers = rng.uniform(lo / 2, hi / 2, (n_lists, d)) if dtype == np.int8 else rng.uniform(60, 200, (n_lists, d))
    x = np.clip(np.rint(centers[rng.integers(0, n_lists, n)] + 12 * rng.standard_normal((n, d))), lo, hi - 1)
    x[n // 2:] = x[:n - n // 2]  # exact duplicates: ties in every metric
    q = np.clip(np.rint(centers[rng.integers(0, n_lists, 40)] + 12 * rng.standard_normal((40, d))), lo, hi - 1)
    lab = np.argmin(((x[:, None, :] - centers[None]) ** 2).sum(-1), axis=1)
    order = np.argsort(lab, kind="stable")
    offsets = np.concatenate([[0], np.cumsum(np.bincount(lab, minlength=n_lists))])
    ids = (order * 7 + 3).astype(np.int64)  # ids unrelated to list positions
    return centers.astype(np.float32), offsets, x[order].astype(dtype), ids, q.astype(dtype)


@pytest.mark.parametrize("metric", ["sqeuclidean", "euclidean", "inner_product"])
@pytest.mark.parametrize("dtype,d", [(np.uint8, 64), (np.int8, 33), (np.int8, 128)])
def test_int_reference_equals_the_oracle(dtype, d, metric):
    centers, offsets, rows, ids, qs = _lists(dtype, 3000, d, 12, 5 + d)
    n_probes = 4
    sure = certain_probes(centers, qs.astype(np.float32), n_probes, metric)
    assert sure.mean() >= 0.5
    for k in (1, 10, 100, 1500):
        got = int_ivf_search(centers, offsets, rows, ids, qs, n_probes, k, metric)
        rd, ri = oracle.ivf_flat_search(centers, offsets, rows.astype(np.float32), ids, qs.astype(np.float32), n_probes, k, metric)
        assert_same_answer(got[0][sure], got[1][sure], rd[sure], ri[sure])
