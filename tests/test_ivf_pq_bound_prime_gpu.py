"""The pruning-bound pre-pass of the code-streaming IVF-PQ scan (scan_pq.cu: pq_bound_prime_kernel).

Before the scan, every query's bound is lowered to a sound value taken from the first rows of its nearest list, so that no
work item starts without a bound.  The bound only drops rows that cannot be among the query's k best, so a search with it
must return what the search without any bound (CUVS_B200_PQ_NO_BOUND=1, which also skips the pre-pass) returns, byte for
byte, and what the oracle finds in the same lists."""
import numpy as np
import pytest
import torch

import oracle
from tests.ivf_oracle import check_rows, pq_search
from tests.util import clustered, launches

pytestmark = pytest.mark.gpu

N_PROBES = 8
LUTS = {"f16": np.float16, "f32": np.float32}  # one pass (bf16 residual) / two passes (hi + lo residual planes)


def _search(monkeypatch, index, qs, k, lut, bound, n_probes=N_PROBES):
    from cuvs_b200.neighbors import ivf_pq
    monkeypatch.setenv("CUVS_B200_PQ_PATH", "stream")
    for name in ("CUVS_B200_PQ_GROUP", "CUVS_B200_PQ_CAP"):
        monkeypatch.delenv(name, raising=False)
    if bound:
        monkeypatch.delenv("CUVS_B200_PQ_NO_BOUND", raising=False)
    else:
        monkeypatch.setenv("CUVS_B200_PQ_NO_BOUND", "1")
    q = torch.from_numpy(qs).cuda()
    l0 = launches()
    d, i = ivf_pq.search(ivf_pq.SearchParams(n_probes=n_probes, lut_dtype=LUTS[lut]), index, q, k)
    torch.cuda.synchronize()
    return d.cpu().numpy(), i.cpu().numpy(), launches() - l0


def _primed_equals_unbounded(monkeypatch, index, qs, k, lut, n_probes=N_PROBES, copies_of=None):
    """-> the primed search.  It launches one kernel more than the unbounded one (the pre-pass) and returns the same
    distances and, unless `copies_of` (the rows by id) is given, the same ids; with it, an id may instead be an exact copy of
    the other one: which of several tied copies survives the scan's own published bound depends on the order of its items."""
    d, i, n = _search(monkeypatch, index, qs, k, lut, True, n_probes)
    d0, i0, n0 = _search(monkeypatch, index, qs, k, lut, False, n_probes)
    assert n == n0 + 1
    np.testing.assert_array_equal(d, d0)
    if copies_of is None:
        np.testing.assert_array_equal(i, i0)
    else:
        diff = i != i0
        assert (copies_of[i[diff]] == copies_of[i0[diff]]).all()
    return d, i


@pytest.fixture(scope="module", params=["sqeuclidean", "inner_product", "cosine"])
def metric_index(request):
    from cuvs_b200.neighbors import ivf_pq
    metric = request.param
    ds, centers = clustered(30000, 128, 71, n_centers=48)
    qs, _ = clustered(600, 128, 72, centers=centers)
    index = ivf_pq.build(ivf_pq.IndexParams(n_lists=48, pq_dim=64, metric=metric, kmeans_n_iters=10), torch.from_numpy(ds).cuda())
    assert index.streamed
    return metric, ds, qs, index


@pytest.mark.parametrize("lut", ["f16", "f32"])
@pytest.mark.parametrize("k", [1, 10, 20, 32])
def test_primed_search_equals_unbounded_and_matches_oracle(monkeypatch, metric_index, k, lut):
    metric, ds, qs, index = metric_index
    d, i = _primed_equals_unbounded(monkeypatch, index, qs, k, lut)
    check_rows(i, len(ds))
    rd, ri = pq_search(index, qs, N_PROBES, k, metric)
    # the bar of the other tensor-core paths against the fp32 LUT sums; one pass rounds the residual to bf16
    eps, floor = (3e-3, 0.99) if lut == "f32" else (2e-2, 0.97)
    assert oracle.recall_with_ties(i, d, ri, rd, eps=eps) >= floor


@pytest.mark.parametrize("lut", ["f16", "f32"])
@pytest.mark.parametrize("k", [1, 20])
def test_prepass_bound_is_finite_and_above_the_kth_distance(monkeypatch, metric_index, k, lut):
    """The bounds as the pre-pass leaves them (before the scan lowers them further): a finite bound for nearly every query (its
    nearest list has well over k rows), never below the query's final k-th distance (inner product: the library returns
    -distance)."""
    import ctypes as C
    from cuvs_b200._capi import lib
    metric, _, qs, index = metric_index
    lib.cuvsB200IvfPqPrimedBounds.restype = C.c_int64
    lib.cuvsB200IvfPqPrimedBounds.argtypes = [C.POINTER(C.c_float), C.c_int64]
    lib.cuvsB200IvfPqKeepPrimedBounds(1)
    try:
        d, _, _ = _search(monkeypatch, index, qs, k, lut, True)
        bounds = np.zeros(len(qs), np.float32)
        n = lib.cuvsB200IvfPqPrimedBounds(bounds.ctypes.data_as(C.POINTER(C.c_float)), len(bounds))
    finally:
        lib.cuvsB200IvfPqKeepPrimedBounds(0)
    assert n == len(qs)
    kth = -d[:, k - 1] if metric == "inner_product" else d[:, k - 1]
    finite = bounds < 1e38
    assert finite.mean() >= 0.95
    assert (bounds[finite] >= kth[finite]).all()


@pytest.fixture(scope="module")
def dup_index():
    """Every vector 8 times: the copies share a list and a code, so their scores tie exactly, also at the k-th place."""
    from cuvs_b200.neighbors import ivf_pq
    base, centers = clustered(3000, 128, 81, n_centers=24)
    ds = np.repeat(base, 8, axis=0)[np.random.default_rng(82).permutation(8 * len(base))]
    qs, _ = clustered(400, 128, 83, centers=centers)
    index = ivf_pq.build(ivf_pq.IndexParams(n_lists=24, pq_dim=64, kmeans_n_iters=10), torch.from_numpy(ds).cuda())
    assert index.streamed
    return ds, qs, index


@pytest.mark.parametrize("lut", ["f16", "f32"])
@pytest.mark.parametrize("k", [10, 20, 32])
def test_tied_copies_at_the_kth_place(monkeypatch, dup_index, k, lut):
    ds, qs, index = dup_index
    d, i = _primed_equals_unbounded(monkeypatch, index, qs, k, lut, copies_of=ds)
    assert np.mean([len(np.unique(r)) < k for r in d]) > 0.5  # the copies really tie inside the results
    rd, ri = pq_search(index, qs, N_PROBES, k)
    assert oracle.recall_with_ties(i, d, ri, rd, eps=2e-2) >= 0.97


@pytest.fixture(scope="module")
def short_lists_index():
    """Lists of 1, 2, 3, 5, 19, 128, 129 and 300 rows beside long ones: a nearest list with fewer than k rows (no bound from
    it), with one tile only, or with a partly filled last tile (padding rows)."""
    from cuvs_b200.neighbors import ivf_pq
    dim, n_lists = 64, 16
    train, _ = clustered(8000, dim, 91, n_centers=n_lists, sigma=0.05)
    index = ivf_pq.build(ivf_pq.IndexParams(n_lists=n_lists, pq_dim=32, kmeans_n_iters=10, add_data_on_build=False),
                         torch.from_numpy(train).cuda())
    centers = index.centers.cpu().numpy()[:, :dim]
    sep = min(np.linalg.norm(centers[a] - centers[b]) for a in range(n_lists) for b in range(a))
    sigma = 0.1 * sep / np.sqrt(dim)
    sizes = [1, 2, 3, 5, 19, 128, 129, 300, 1500, 2000, 700, 1000, 900, 1200, 800, 600]
    rng = np.random.default_rng(92)
    lab = np.concatenate([np.full(s, j) for j, s in enumerate(sizes)])
    rows = (centers[lab] + sigma * rng.standard_normal((len(lab), dim))).astype(np.float32)
    rows = rows[rng.permutation(len(rows))]
    ivf_pq.extend(index, torch.from_numpy(rows).cuda(), torch.arange(len(rows), dtype=torch.int64).cuda())
    assert index.streamed
    # most queries sit in the short lists, so their nearest list is one of them
    qs = (centers[rng.integers(0, 8, 512)] + sigma * rng.standard_normal((512, dim))).astype(np.float32)
    return rows, qs, index, sizes


@pytest.mark.parametrize("lut", ["f16", "f32"])
@pytest.mark.parametrize("k", [1, 10, 20, 32])
def test_short_nearest_lists(monkeypatch, short_lists_index, k, lut):
    rows, qs, index, sizes = short_lists_index
    assert sorted(index.list_sizes.cpu().numpy().tolist()) == sorted(sizes)
    d, i = _primed_equals_unbounded(monkeypatch, index, qs, k, lut, n_probes=4)
    check_rows(i, len(rows))
    rd, ri = pq_search(index, qs, 4, k)
    eps, floor = (3e-3, 0.99) if lut == "f32" else (2e-2, 0.97)
    assert oracle.recall_with_ties(i, d, ri, rd, eps=eps) >= floor


def test_zero_queries(monkeypatch, metric_index):
    _, _, qs, index = metric_index
    d, i, _ = _search(monkeypatch, index, qs[:0], 10, "f16", True)
    assert d.shape == (0, 10) and i.shape == (0, 10)
