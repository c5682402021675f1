"""GPU parity: cuvsIvfFlat{Build,Search,Extend,Serialize} through the C ABI vs the oracle.

Mirrors cpp/tests/neighbors/ann_ivf_flat.cuh (recall >= n_probes/n_lists floor, eps 1e-3) and
python/cuvs/cuvs/tests/test_ivf_flat.py, plus an element-wise check: with the library's own centres
and list membership fed to the oracle's IVF search, ids must agree except at distance ties."""
import numpy as np
import pytest
import torch

import oracle
from tests.ivf_oracle import flat_lists, flat_search
from tests.util import clustered, launches, uniform

pytestmark = pytest.mark.gpu


def _mod():
    from cuvs_b200.neighbors import ivf_flat
    return ivf_flat


@pytest.mark.parametrize("n,d,n_lists,n_probes,k,metric", [
    (20000, 128, 64, 8, 10, "sqeuclidean"), (20000, 96, 100, 100, 10, "sqeuclidean"), (8000, 64, 32, 6, 16, "euclidean"),
    (10000, 33, 50, 10, 5, "inner_product"), (30000, 128, 128, 16, 32, "sqeuclidean"), (6000, 16, 20, 5, 1, "sqeuclidean"),
    (12000, 256, 40, 8, 10, "sqeuclidean")])
def test_search_matches_oracle(n, d, n_lists, n_probes, k, metric):
    m = _mod()
    ds, centers = clustered(n, d, 5, n_centers=max(8, n_lists // 2))
    qs, _ = clustered(300, d, 6, centers=centers)
    l0 = launches()
    index = m.build(m.IndexParams(n_lists=n_lists, metric=metric, kmeans_n_iters=10), torch.from_numpy(ds).cuda())
    assert len(index) == n and index.n_lists == n_lists and index.dim == d
    dist, idx = m.search(m.SearchParams(n_probes=n_probes), index, torch.from_numpy(qs).cuda(), k)
    assert launches() > l0
    dist, idx = dist.cpu().numpy(), idx.cpu().numpy()
    _, ids = flat_lists(index)
    assert index.list_sizes.cpu().numpy().sum() == n and sorted(ids.tolist()) == list(range(n))
    rd, ri = flat_search(index, ds, qs, n_probes, k, metric)
    # element-wise: same id, or an equal-distance tie (ann_utils.cuh:257-289)
    assert oracle.recall_with_ties(idx, dist, ri, rd, eps=1e-3) >= 0.999
    same = (idx == ri).mean()
    assert same >= 0.995, f"only {same:.4f} of result slots agree with the oracle"
    # against exact ground truth: recall floor of the reference test-suite
    gd, gi = oracle.knn(ds, qs, k, metric)
    rec = oracle.recall(idx, gi)
    assert rec >= min(0.999, n_probes / n_lists) - 1e-3, rec
    if n_probes == n_lists:  # exhaustive probing == exact search
        assert rec >= 0.9999


def test_balanced_lists_and_recall_on_clustered_data():
    m = _mod()
    ds, centers = clustered(50000, 128, 1)
    qs, _ = clustered(500, 128, 2, centers=centers)
    index = m.build(m.IndexParams(n_lists=256, kmeans_n_iters=20), torch.from_numpy(ds).cuda())
    sizes = index.list_sizes.cpu().numpy()
    assert sizes.min() > 0 and sizes.max() <= 8 * sizes.mean()
    _, idx = m.search(m.SearchParams(n_probes=32), index, torch.from_numpy(qs).cuda(), 10)
    _, gi = oracle.knn(ds, qs, 10)
    assert oracle.recall(idx.cpu().numpy(), gi) >= 0.95


def test_extend_with_ids_and_save_load(tmp_path):
    m = _mod()
    ds, centers = clustered(12000, 64, 3, n_centers=40)
    qs, _ = clustered(100, 64, 4, centers=centers)
    index = m.build(m.IndexParams(n_lists=40, add_data_on_build=False), torch.from_numpy(ds).cuda())
    assert len(index) == 0
    ids = np.arange(12000, dtype=np.int64) * 7 + 3
    m.extend(index, torch.from_numpy(ds[:5000]).cuda(), torch.from_numpy(ids[:5000]).cuda())
    m.extend(index, torch.from_numpy(ds[5000:]), torch.from_numpy(ids[5000:]))  # host inputs
    assert len(index) == 12000
    d1, i1 = m.search(m.SearchParams(n_probes=40), index, torch.from_numpy(qs).cuda(), 10)
    _, gi = oracle.knn(ds, qs, 10)
    assert oracle.recall(i1.cpu().numpy(), ids[gi]) >= 0.9999
    m.save(str(tmp_path / "flat.idx"), index)
    again = m.load(str(tmp_path / "flat.idx"))
    d2, i2 = m.search(m.SearchParams(n_probes=40), again, torch.from_numpy(qs).cuda(), 10)
    assert torch.equal(i1, i2) and torch.equal(d1, d2)


def test_out_of_bounds_record_when_probed_lists_are_small():
    m = _mod()
    ds = uniform(64, 8, 9)
    index = m.build(m.IndexParams(n_lists=16, kmeans_n_iters=5), torch.from_numpy(ds).cuda())
    d, i = m.search(m.SearchParams(n_probes=1), index, torch.from_numpy(ds[:4]).cuda(), 32)
    i = i.cpu().numpy()
    assert (i == np.iinfo(np.int64).max).any()  # kOutOfBoundsRecord (ivf_common.cuh:25-31)
    assert (i[:, 0] == np.arange(4)).all()


def test_bitset_prefilter_equals_search_over_the_kept_rows():
    """cuvsFilter{BITSET} (bit = 1 keeps, ids are source ids): same answer as the oracle searching lists from which the
    filtered rows were removed; no filtered id is ever returned (cpp/tests/neighbors/ann_ivf_flat.cuh filter cases)."""
    from cuvs_b200.neighbors import filters
    m = _mod()
    ds, centers = clustered(12000, 64, 5, n_centers=16)
    qs, _ = clustered(200, 64, 6, centers=centers)
    index = m.build(m.IndexParams(n_lists=32, kmeans_n_iters=10), torch.from_numpy(ds).cuda())
    keep = np.random.default_rng(9).random(12000) < 0.4
    bits = np.packbits(np.concatenate([keep, np.zeros((-len(keep)) % 32, bool)]), bitorder="little").view(np.uint32)
    dist, idx = m.search(m.SearchParams(n_probes=8), index, torch.from_numpy(qs).cuda(), 10,
                         filter=filters.from_bitset(torch.from_numpy(bits.view(np.int32)).cuda()))
    dist, idx = dist.cpu().numpy(), idx.cpu().numpy()
    valid = idx != np.iinfo(np.int64).max
    assert keep[idx[valid]].all(), "a filtered-out row was returned"
    rd, ri = flat_search(index, ds, qs, 8, 10, "sqeuclidean", keep)
    assert oracle.recall_with_ties(idx, dist, ri, rd, eps=1e-3) >= 0.999


_FUSED_CACHE = {}


@pytest.mark.parametrize("n_probes", [20, 32, 48, 64])
@pytest.mark.parametrize("nq", [37, 1000])
def test_fused_coarse_search_equals_the_dense_one(n_probes, nq, monkeypatch):
    """n_lists >= 4096 takes the fused coarse search (ivf_common.cu: per-(centre range, column half) lists of 32 kept in the scan
    epilogue + a ranked merge, certificate for n_probes > 32) instead of the dense [nq, n_lists] score block + select_k.
    Same scores, same (score, id) order => the probe lists, hence the search results, are identical.  Also vs the oracle."""
    m = _mod()
    n, d, n_lists, k = 120000, 64, 4096, 10
    if "index" not in _FUSED_CACHE:
        ds, centers = clustered(n, d, 21, n_centers=3000)
        _FUSED_CACHE.update(ds=ds, centers=centers,
                            index=m.build(m.IndexParams(n_lists=n_lists, kmeans_n_iters=4), torch.from_numpy(ds).cuda()))
    ds, centers, index = _FUSED_CACHE["ds"], _FUSED_CACHE["centers"], _FUSED_CACHE["index"]
    qs, _ = clustered(nq, d, 22, centers=centers)
    q = torch.from_numpy(qs).cuda()
    monkeypatch.setenv("CUVS_B200_COARSE_FUSED", "0")
    d0, i0 = m.search(m.SearchParams(n_probes=n_probes), index, q, k)
    l0 = launches()
    monkeypatch.setenv("CUVS_B200_COARSE_FUSED", "1")
    d1, i1 = m.search(m.SearchParams(n_probes=n_probes), index, q, k)
    assert launches() > l0
    d0, i0, d1, i1 = d0.cpu().numpy(), i0.cpu().numpy(), d1.cpu().numpy(), i1.cpu().numpy()
    np.testing.assert_array_equal(i1, i0)
    np.testing.assert_array_equal(d1, d0)
    rd, ri = flat_search(index, ds, qs[:64], n_probes, k, "sqeuclidean")
    assert oracle.recall_with_ties(i1[:64], d1[:64], ri, rd, eps=1e-3) >= 0.999
