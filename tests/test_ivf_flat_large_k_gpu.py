"""IVF-Flat search with 64 < k <= 2048.

k > 64 runs the fine scan with the store epilogue: every (query, probe, list row) score goes to a dense per-pair segment, the
segmented select keeps each pair's kc2 = min(2k, 2048) best, and the probes are merged and re-scored exactly as on the k <= 64
path.  Checked against the oracle's IVF-Flat search (and its exact kNN for the cosine metric, with every list probed), against
the k = 64 search of the same index (prefix), with a bitset filter that leaves most pairs with fewer than kc2 kept rows, for
the fill of missing slots, for invariance under a forced workspace split, for the k limit, and through the multi-GPU search.

Agreement with the oracle at k = 2048, where the re-score sees only the 2048 best bf16 scores (no slack), is asserted at >= 0.99
(>= 0.999 for k <= 1024).  Measured on an H100 80GB HBM3 (700 W power limit) for the 30k x 128 L2 index below:
recall_with_ties 1.0000 at k = 2048, with 99.69 % of the result slots holding the oracle's id (the rest are distance ties);
every case with k <= 1024 matched the oracle's ids in all slots.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from tests.ivf_oracle import I64_MAX, check_rows, flat_search
from tests.util import clustered, uniform

pytestmark = pytest.mark.gpu

FLT_MAX = np.finfo(np.float32).max
N_LISTS = 64
N_PROBES = 32  # ~15k probed rows per query: more than 2k for every k below
_INDEX = {}


def _mod():
    from cuvs_b200.neighbors import ivf_flat
    return ivf_flat


def _data(d):
    n = 30000 if d <= 128 else 20000
    ds, centers = clustered(n, d, 31 + d, n_centers=32)
    qs, _ = clustered(100, d, 32 + d, centers=centers)
    return ds, qs


def _index(metric, d=128):
    """One index per (metric, dim), built once for the module."""
    key = (metric, d)
    if key not in _INDEX:
        m = _mod()
        ds, qs = _data(d)
        _INDEX[key] = (m.build(m.IndexParams(n_lists=N_LISTS, metric=metric, kmeans_n_iters=10), torch.from_numpy(ds).cuda()), ds, qs)
    return _INDEX[key]


def _search(index, qs, n_probes, k, **kw):
    m = _mod()
    d, i = m.search(m.SearchParams(n_probes=n_probes), index, torch.from_numpy(qs).cuda(), k, **kw)
    return d.cpu().numpy(), i.cpu().numpy()


def _timed_count(name, fn):
    """Runs fn with the library's section timers on; returns how many `name` sections it ran."""
    from cuvs_b200._capi import lib
    lib.cuvsB200TimingTotalMs.restype = C.c_double
    lib.cuvsB200TimingReset()
    lib.cuvsB200TimingEnable(1)
    try:
        out = fn()
        torch.cuda.synchronize()
    finally:
        lib.cuvsB200TimingEnable(0)
    cnt = C.c_int(0)
    lib.cuvsB200TimingTotalMs(name, C.byref(cnt))
    return out, cnt.value


CASES = [("sqeuclidean", 128, k) for k in (65, 100, 128, 129, 256, 257, 1023, 1024, 2048)]
CASES += [(metric, 128, k) for metric in ("inner_product", "cosine", "euclidean") for k in (100, 1024)]
CASES += [("sqeuclidean", 256, k) for k in (100, 1024)]  # Kp = 256: the streamed-A scan kernel (KB = 0)


@pytest.mark.parametrize("metric,d,k", CASES)
def test_large_k_matches_oracle(metric, d, k):
    index, ds, qs = _index(metric, d)
    if metric == "cosine":
        # the oracle's IVF search has no cosine metric: probe every list, which makes the search exact, and compare with
        # the oracle's exact kNN
        dist, idx = _search(index, qs, N_LISTS, k)
        rd, ri = oracle.knn(ds, qs, k, metric)
        floor = 1.0
    else:
        dist, idx = _search(index, qs, N_PROBES, k)
        rd, ri = flat_search(index, ds, qs, N_PROBES, k, metric)
        floor = N_PROBES / N_LISTS
    assert idx.shape == (len(qs), k)
    assert (idx != I64_MAX).all(), "the probed lists hold more than k rows"
    check_rows(idx)
    rec = oracle.recall_with_ties(idx, dist, ri, rd, eps=1e-3)
    assert rec >= (0.999 if k <= 1024 else 0.99), rec
    # against exact ground truth: the reference test-suite's recall floor n_probes / n_lists
    gd, gi = oracle.knn(ds, qs, k, metric)
    assert oracle.recall(idx, gi) >= min(0.999, floor) - 1e-3


@pytest.mark.parametrize("metric", ["sqeuclidean", "inner_product"])
def test_first_64_of_k100_are_at_least_as_good_as_k64(metric):
    """The k = 100 search re-scores at least the k = 64 search's true top 64 in the same arithmetic: its j-th distance is never
    worse, and almost always equal.  Uniform data over many small lists, where a query's 64 nearest rows are spread over
    several lists; tests/test_ivf_mid_k_gpu.py checks the same on clustered data, where most of them sit in one list and the
    k = 64 search depends on its certificate sending such queries to the store path."""
    m = _mod()
    ds = uniform(30000, 32, 17)
    qs = uniform(200, 32, 18)
    index = m.build(m.IndexParams(n_lists=256, metric=metric, kmeans_n_iters=10), torch.from_numpy(ds).cuda())
    d64, _ = _search(index, qs, 64, 64)
    d100, _ = _search(index, qs, 64, 100)
    head = d100[:, :64]
    if metric == "inner_product":
        assert (head >= d64).all()
    else:
        assert (head <= d64).all()
    assert (head == d64).mean() >= 0.999


def test_bitset_filter_never_returns_a_filtered_row():
    """About 5 % of the rows are kept, so most (query, probe) pairs hold fewer kept rows than the kc2 = 400 the segmented select
    takes from them, and the select's output includes rows that the filter hid (their score is +inf).  None of them may come
    back, and the result is the oracle's search over the kept rows only."""
    from cuvs_b200.neighbors import filters
    index, ds, qs = _index("sqeuclidean")
    n, k = len(ds), 200
    keep = np.random.default_rng(5).random(n) < 0.05
    bits = np.packbits(np.concatenate([keep, np.zeros((-n) % 32, bool)]), bitorder="little").view(np.uint32)
    dist, idx = _search(index, qs, N_PROBES, k, filter=filters.from_bitset(torch.from_numpy(bits.view(np.int32)).cuda()))
    valid = idx != I64_MAX
    assert keep[idx[valid]].all(), "a filtered-out row was returned"
    check_rows(idx)
    sizes = index.list_sizes.cpu().numpy().astype(np.int64)
    ids_f = [i[keep[i]] for i in (index.list_indices(l).cpu().numpy() for l in range(index.n_lists))]
    offsets = np.concatenate([[0], np.cumsum([len(i) for i in ids_f])])
    all_ids = np.concatenate(ids_f)
    assert sizes.sum() == n
    rd, ri = oracle.ivf_flat_search(index.centers.cpu().numpy(), offsets, ds[all_ids], all_ids, qs, N_PROBES, k, "sqeuclidean")
    assert (valid == (ri != I64_MAX)).all(), "the number of results differs from the oracle's"
    assert oracle.recall_with_ties(idx, dist, ri, rd, eps=1e-3) >= 0.999


@pytest.mark.parametrize("metric", ["sqeuclidean", "inner_product"])
def test_missing_slots_are_filled(metric):
    """One probe over lists of a few rows: the slots past the list's rows hold INT64_MAX and FLT_MAX (-FLT_MAX for inner
    product), as on the k <= 64 path."""
    m = _mod()
    ds = uniform(64, 8, 9)
    index = m.build(m.IndexParams(n_lists=16, metric=metric, kmeans_n_iters=5), torch.from_numpy(ds).cuda())
    dist, idx = _search(index, ds[:4], 1, 100)
    missing = idx == I64_MAX
    assert missing[:, int(index.list_sizes.to(torch.int64).max()):].all()
    assert (dist[missing] == (-FLT_MAX if metric == "inner_product" else FLT_MAX)).all()
    assert (~missing).sum(axis=1).min() >= 1
    check_rows(idx)
    if metric == "sqeuclidean":
        assert (idx[:, 0] == np.arange(4)).all()


def test_workspace_split_gives_identical_results(monkeypatch):
    """A 1 MiB workspace budget splits the 100 queries into many batches; neighbours and distances are bit-identical."""
    index, ds, qs = _index("sqeuclidean")
    (d0, i0), n0 = _timed_count(b"ivf_flat_scan", lambda: _search(index, qs, N_PROBES, 256))
    monkeypatch.setenv("CUVS_B200_FLAT_LARGE_K_BUDGET_MB", "1")
    (d1, i1), n1 = _timed_count(b"ivf_flat_scan", lambda: _search(index, qs, N_PROBES, 256))
    assert n0 == 1 and n1 >= 3, (n0, n1)
    np.testing.assert_array_equal(i1, i0)
    np.testing.assert_array_equal(d1, d0)


def test_k_above_2048_is_refused():
    index, ds, qs = _index("sqeuclidean")
    with pytest.raises(Exception, match="2048"):
        _search(index, qs[:4], N_PROBES, 2049)


class _MgIndexParams(C.Structure):
    _fields_ = [("base_params", C.c_void_p), ("mode", C.c_int)]


class _MgSearchParams(C.Structure):
    _fields_ = [("base_params", C.c_void_p), ("search_mode", C.c_int), ("merge_mode", C.c_int), ("n_rows_per_batch", C.c_int64)]


@pytest.mark.parametrize("mode", [0, 1])  # CUVS_NEIGHBORS_MG_REPLICATED = 0, CUVS_NEIGHBORS_MG_SHARDED = 1
def test_multi_gpu_ivf_flat_k100_matches_exact_knn(mode):
    """cuvsMultiGpuIvfFlatSearch at k = 100 with every list probed: exact search on the visible devices."""
    from cuvs_b200._capi import DL, check, lib
    from cuvs_b200.neighbors.ivf_flat import _IndexParamsC, _SearchParamsC
    ds, centers = clustered(30000, 64, 21, n_centers=32)
    qs, _ = clustered(300, 64, 22, centers=centers)
    k = 100
    res = C.c_void_p()
    check(lib.cuvsMultiGpuResourcesCreate(C.byref(res)))
    ip = C.POINTER(_MgIndexParams)()
    sp = C.POINTER(_MgSearchParams)()
    check(lib.cuvsMultiGpuIvfFlatIndexParamsCreate(C.byref(ip)))
    check(lib.cuvsMultiGpuIvfFlatSearchParamsCreate(C.byref(sp)))
    ip.contents.mode = mode
    base = C.cast(ip.contents.base_params, C.POINTER(_IndexParamsC)).contents
    base.n_lists, base.kmeans_n_iters = 64, 10
    C.cast(sp.contents.base_params, C.POINTER(_SearchParamsC)).contents.n_probes = 64
    index = C.c_void_p()
    check(lib.cuvsMultiGpuIvfFlatIndexCreate(C.byref(index)))
    t_ds, t_q = torch.from_numpy(ds), torch.from_numpy(qs)
    nb = torch.empty((300, k), dtype=torch.int64)
    dd = torch.empty((300, k), dtype=torch.float32)
    d_ds, d_q, d_nb, d_dd = DL(t_ds), DL(t_q), DL(nb), DL(dd)
    check(lib.cuvsMultiGpuIvfFlatBuild(res, ip, d_ds.ptr, index))
    check(lib.cuvsMultiGpuIvfFlatSearch(res, sp, index, d_q.ptr, d_nb.ptr, d_dd.ptr))
    gd, gi = oracle.knn(ds, qs, k)
    assert oracle.recall_with_ties(nb.numpy(), dd.numpy(), gi, gd, eps=1e-3) >= 0.999
    check_rows(nb.numpy())
    check(lib.cuvsMultiGpuIvfFlatIndexDestroy(index))
    check(lib.cuvsMultiGpuIvfFlatSearchParamsDestroy(sp))
    check(lib.cuvsMultiGpuIvfFlatIndexParamsDestroy(ip))
    check(lib.cuvsMultiGpuResourcesDestroy(res))
