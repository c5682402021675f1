"""IVF-Flat search with 32 < k <= 64, against the oracle.

A search that keeps a fixed number of candidates per column half of each (query, probed list) pair before the exact re-score
loses true neighbours as soon as more of them than that sit in one half of one list, which is the common case on clustered
data: a query's 64 nearest rows then mostly live in the list of its own cluster.  These tests put the neighbours there on
purpose (fewer data centres than lists, few probes) and compare every k in 33..64 with the oracle's IVF-Flat search over the
same lists, for each metric, on uniform data over many small lists as well, with a bitset filter, and against the k = 100
search of the same index.  The IVF-PQ searches at these k are part of tests/test_ivf_pq_code_shapes_gpu.py."""
import numpy as np
import pytest
import torch

import oracle
from tests.ivf_oracle import I64_MAX, check_rows, flat_search
from tests.util import clustered, uniform

pytestmark = pytest.mark.gpu

KS = [33, 48, 64]
_INDEX = {}


def _mod():
    from cuvs_b200.neighbors import ivf_flat
    return ivf_flat


def _index(data, metric):
    """clustered: 30k x 128 around 16 centres, 64 lists, probed 8 at a time.  uniform: 30k x 32 over 256 lists."""
    key = (data, metric)
    if key not in _INDEX:
        m = _mod()
        if data == "clustered":
            ds, centers = clustered(30000, 128, 41, n_centers=16)
            qs, _ = clustered(300, 128, 42, centers=centers)
            n_lists, n_probes = 64, 8
        else:
            ds, qs = uniform(30000, 32, 43), uniform(300, 32, 44)
            n_lists, n_probes = 256, 32
        index = m.build(m.IndexParams(n_lists=n_lists, metric=metric, kmeans_n_iters=10), torch.from_numpy(ds).cuda())
        _INDEX[key] = (index, ds, qs, n_probes)
    return _INDEX[key]


def _search(index, qs, n_probes, k, **kw):
    m = _mod()
    d, i = m.search(m.SearchParams(n_probes=n_probes), index, torch.from_numpy(qs).cuda(), k, **kw)
    return d.cpu().numpy(), i.cpu().numpy()


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("metric", ["sqeuclidean", "inner_product", "euclidean"])
@pytest.mark.parametrize("data", ["clustered", "uniform"])
def test_search_matches_oracle(data, metric, k):
    index, ds, qs, n_probes = _index(data, metric)
    dist, idx = _search(index, qs, n_probes, k)
    rd, ri = flat_search(index, ds, qs, n_probes, k, metric)
    check_rows(idx)
    assert (idx != I64_MAX).all()
    rec = oracle.recall_with_ties(idx, dist, ri, rd, eps=1e-3)
    assert rec >= 0.999, rec
    same = (idx == ri).mean()
    assert same >= 0.995, f"only {same:.4f} of result slots agree with the oracle"


@pytest.mark.parametrize("k", KS)
def test_cosine_with_every_list_probed_is_exact(k):
    """The oracle's IVF search has no cosine metric: probing every list makes the search exact, so compare with its kNN."""
    index, ds, qs, _ = _index("clustered", "cosine")
    dist, idx = _search(index, qs, index.n_lists, k)
    rd, ri = oracle.knn(ds, qs, k, "cosine")
    check_rows(idx)
    assert oracle.recall_with_ties(idx, dist, ri, rd, eps=1e-3) >= 0.999


def test_bitset_filter_at_k64():
    """40 % of the rows kept: the answer is the oracle's search over the kept rows, and no filtered row comes back."""
    from cuvs_b200.neighbors import filters
    index, ds, qs, n_probes = _index("clustered", "sqeuclidean")
    n = len(ds)
    keep = np.random.default_rng(45).random(n) < 0.4
    bits = np.packbits(np.concatenate([keep, np.zeros((-n) % 32, bool)]), bitorder="little").view(np.uint32)
    dist, idx = _search(index, qs, n_probes, 64, filter=filters.from_bitset(torch.from_numpy(bits.view(np.int32)).cuda()))
    valid = idx != I64_MAX
    assert keep[idx[valid]].all(), "a filtered-out row was returned"
    check_rows(idx)
    rd, ri = flat_search(index, ds, qs, n_probes, 64, "sqeuclidean", keep)
    assert (valid == (ri != I64_MAX)).all(), "the number of results differs from the oracle's"
    assert oracle.recall_with_ties(idx, dist, ri, rd, eps=1e-3) >= 0.999
    assert (idx == ri).mean() >= 0.995


@pytest.mark.parametrize("metric", ["sqeuclidean", "inner_product"])
def test_first_64_of_k100_equal_k64_on_clustered_data(metric):
    """The k = 100 search re-scores a superset of the k = 64 search's candidates in the same arithmetic: its first 64 distances
    are never worse and, when the k = 64 search keeps every true neighbour, equal; ids agree wherever no tie makes the order
    arbitrary."""
    index, ds, qs, n_probes = _index("clustered", metric)
    d64, i64 = _search(index, qs, n_probes, 64)
    d100, i100 = _search(index, qs, n_probes, 100)
    head, ihead = d100[:, :64], i100[:, :64]
    if metric == "inner_product":
        assert (head >= d64).all()
    else:
        assert (head <= d64).all()
    assert (head == d64).mean() >= 0.999, (head == d64).mean()
    tied = np.zeros(d64.shape, bool)
    tied[:, 1:] |= d64[:, 1:] == d64[:, :-1]
    tied[:, :-1] |= d64[:, :-1] == d64[:, 1:]
    tied[:, -1] = True  # the 64th entry may tie with the 65th, which only the k = 100 search sees
    ok = (head == d64) & ~tied
    assert (ihead[ok] == i64[ok]).all()
