"""Every index at the embedding widths users run (384 ... 4096), against the oracle.

The width decides which code runs: the scan engine keeps the query tile in shared memory at padded widths 64 and 128,
streams its k-blocks from 192 to 2048, and above 2048 brute force answers on its exact SIMT path while the IVF and k-means
builds refuse the width.  CAGRA's walk fits fewer warps per CTA as the width grows, and the IVF-PQ LUT outgrows shared
memory (the LUT kernel then keeps it in global memory).  The widths below sit at those edges (129, 255 / 256 / 257,
2047 / 2048 / 2049) and at common embedding sizes; row and query counts leave partial 128-row tiles.  Every fixture is
generated from a seed here."""
import functools

import numpy as np
import pytest
import torch

import oracle
from tests.cagra_cosine_ref import cagra_cosine_search
from tests.ivf_oracle import check_rows, flat_search, pq_search
from tests.ivf_pq_codes import index_codes, unpack_codes
from tests.util import clustered, last_flagged, uniform

pytestmark = pytest.mark.gpu

TC_WIDTHS = (129, 192, 255, 256, 257, 384, 512, 768, 1000, 1024, 1536, 2047, 2048)
WIDE_WIDTHS = (2049, 3072, 4096)  # past the tensor-core kernels' 2048 padded columns
METRICS = ("sqeuclidean", "inner_product", "cosine")


def _rows(d):
    """(rows, queries) of a width: the oracle's CPU work stays bounded at d >= 1024."""
    return (10001, 257) if d < 1024 else (10001, 200)


def _np(d, i):
    return d.cpu().numpy(), i.cpu().numpy().astype(np.int64)


def _bitset(keep):
    from cuvs_b200.neighbors import filters
    keep = np.asarray(keep, bool)
    bits = np.packbits(np.concatenate([keep, np.zeros((-len(keep)) % 32, bool)]), bitorder="little").view(np.int32)
    return filters.from_bitset(torch.from_numpy(bits.copy()).cuda())


# ------------------------------------------------------------------------------------------------------------ brute force
@functools.lru_cache(maxsize=4)
def _bf_case(d, metric):
    """(rows, queries, index, the oracle's 100 best): the oracle orders ties by id, so its k best are a prefix of these."""
    from cuvs_b200.neighbors import brute_force
    n, nq = _rows(d)
    ds, qs = uniform(n, d, 1000 + d), uniform(nq, d, 2000 + d)
    index = brute_force.build(torch.from_numpy(ds).cuda(), metric=metric)
    return ds, qs, index, oracle.knn(ds, qs, 100, metric)


@pytest.mark.parametrize("k", [1, 10, 48, 64, 100])
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", TC_WIDTHS + WIDE_WIDTHS)
def test_brute_force_equals_oracle(d, metric, k):
    from cuvs_b200.neighbors import brute_force
    ds, qs, index, (rd, ri) = _bf_case(d, metric)
    dist, idx = _np(*brute_force.search(index, torch.from_numpy(qs).cuda(), k))
    rd, ri = rd[:, :k], ri[:, :k]
    assert (idx == ri).all(), f"{(idx != ri).sum()} index mismatches"
    np.testing.assert_array_equal(dist, rd)
    if d <= 2048 and k <= 64:  # the tensor-core candidates carry the result, not the exact fallback
        nq = len(qs)
        bound = max(1, nq // 100) if k <= 24 else nq // 20  # (the bars of test_brute_force_gpu.py)
        assert last_flagged() <= bound, f"{last_flagged()} of {nq} queries fell back to the exact path"


def test_brute_force_bitset_at_1536():
    from cuvs_b200.neighbors import brute_force
    ds, qs, index, _ = _bf_case(1536, "sqeuclidean")
    keep = np.random.default_rng(15).random(len(ds)) < 0.4
    dist, idx = _np(*brute_force.search(index, torch.from_numpy(qs).cuda(), 10, prefilter=_bitset(keep)))
    kept = np.flatnonzero(keep)
    rd, ri = oracle.knn(ds[kept], qs, 10)
    np.testing.assert_array_equal(idx, kept[ri])
    np.testing.assert_array_equal(dist, rd)


# ----------------------------------------------------------------------------------------------- certificate error budget
def _family(name, n, d, seed):
    rng = np.random.default_rng(seed)
    if name == "uniform":
        return rng.uniform(-1, 1, (n, d)).astype(np.float32)
    if name == "uint8":  # descriptors: no cancellation in the products
        return rng.integers(0, 256, (n, d)).astype(np.float32)
    x, _ = clustered(n, d, seed, n_centers=20)  # post-ReLU embeddings
    return np.maximum(x, 0)


@pytest.mark.parametrize("family", ["uniform", "uint8", "relu"])
@pytest.mark.parametrize("d", TC_WIDTHS)
def test_candidate_error_budget(d, family):
    """The certificate's eps (eps_rel(Kp) (|q|^2 + max|x|^2), brute_force.cu) must stay 4x above the worst error of the
    tensor-core scores at every width, on data with and without cancellation (the margin test_brute_force_gpu.py asks at
    d = 128).  eps_rel = max(2^-15, 2^-16 + Kp 2^-24): the split-bf16 products plus the fp32 accumulation of Kp products."""
    from cuvs_b200._capi import DL, check, lib
    from cuvs_b200.common import Resources
    from cuvs_b200.neighbors import brute_force
    ds, qs = _family(family, 10001, d, 31 + d), _family(family, 256, d, 32 + d)
    index = brute_force.build(torch.from_numpy(ds).cuda())
    res = Resources()
    q = torch.from_numpy(qs).cuda()
    pos = torch.zeros(len(qs), 16, dtype=torch.uint32, device="cuda")
    sc = torch.zeros(len(qs), 16, dtype=torch.float32, device="cuda")
    check(lib.cuvsB200BruteForceCandidates(res.get_c_obj(), index._p, DL(q).ptr, DL(pos).ptr, DL(sc).ptr))
    pos = pos.cpu().numpy().astype(np.int64)
    s = sc.cpu().numpy().astype(np.float64)
    q64 = qs.astype(np.float64)
    qn = (q64 ** 2).sum(1)
    approx = qn[:, None] + 2 * s
    exact = ((q64[:, None, :] - ds[pos].astype(np.float64)) ** 2).sum(-1)
    xn_max = (ds.astype(np.float64) ** 2).sum(1).max()
    rel = np.abs(approx - exact) / (qn[:, None] + xn_max)
    kp = -(-d // 64) * 64
    eps_rel = max(2.0 ** -15, 2.0 ** -16 + kp * 2.0 ** -24)
    print(f"\nbudget d={d} family={family}: worst relative error {rel.max():.3e}, eps_rel {eps_rel:.3e}")
    assert rel.max() <= eps_rel / 4, f"observed relative error {rel.max():.3e}"


# -------------------------------------------------------------------------------------------------------------- IVF-Flat
FLAT_WIDTHS = (256, 257, 512, 768, 1024, 1536, 2047, 2048)
FLAT_LISTS, FLAT_PROBES = 64, 8


@functools.lru_cache(maxsize=3)
def _flat_case(d, metric):
    m = _ivf_flat()
    n, nq = _rows(d)
    ds, centers = clustered(n, d, 5 + d, n_centers=FLAT_LISTS // 2)
    qs, _ = clustered(nq, d, 6 + d, centers=centers)
    index = m.build(m.IndexParams(n_lists=FLAT_LISTS, metric=metric, kmeans_n_iters=10), torch.from_numpy(ds).cuda())
    # the oracle's IVF search has no cosine metric: a cosine search probes every list, which makes it exact
    ref = oracle.knn(ds, qs, 100, metric) if metric == "cosine" else flat_search(index, ds, qs, FLAT_PROBES, 100, metric)
    return ds, qs, index, ref


def _ivf_flat():
    from cuvs_b200.neighbors import ivf_flat
    return ivf_flat


@pytest.mark.parametrize("k", [10, 48, 100])
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", FLAT_WIDTHS)
def test_ivf_flat_matches_oracle(d, metric, k):
    """The bars of test_ivf_flat_gpu.py::test_search_matches_oracle, against the oracle over the index's own lists (cosine:
    every list probed, against the oracle's exact kNN)."""
    m = _ivf_flat()
    ds, qs, index, (rd, ri) = _flat_case(d, metric)
    n_probes = FLAT_LISTS if metric == "cosine" else FLAT_PROBES
    dist, idx = _np(*m.search(m.SearchParams(n_probes=n_probes), index, torch.from_numpy(qs).cuda(), k))
    rd, ri = rd[:, :k], ri[:, :k]
    check_rows(idx, len(ds))
    assert oracle.recall_with_ties(idx, dist, ri, rd, eps=1e-3) >= 0.999
    same = (idx == ri).mean()
    assert same >= 0.995, f"only {same:.4f} of result slots agree with the oracle"


@pytest.mark.parametrize("d", FLAT_WIDTHS)
def test_ivf_flat_all_lists_probed_is_exact(d):
    """Every list probed: the oracle's exact kNN, up to neighbours at a distance tie (eps 1e-3, relative).  Past d = 128 a
    plain id recall of 0.9999 does not hold: the scan's bf16 candidate cut is not certified (DESIGN.md §4), and it drops
    about one of 2500 slots for a row whose distance is within 1e-3 of the k-th."""
    m = _ivf_flat()
    ds, qs, index, _ = _flat_case(d, "sqeuclidean")
    dist, idx = _np(*m.search(m.SearchParams(n_probes=FLAT_LISTS), index, torch.from_numpy(qs).cuda(), 10))
    gd, gi = oracle.knn(ds, qs, 10)
    assert oracle.recall_with_ties(idx, dist, gi, gd, eps=1e-3) >= 0.9999
    assert oracle.recall(idx, gi) >= 0.999


def test_ivf_flat_extend_save_load_at_1536(tmp_path):
    m = _ivf_flat()
    ds, qs, full, _ = _flat_case(1536, "sqeuclidean")
    index = m.build(m.IndexParams(n_lists=FLAT_LISTS, kmeans_n_iters=10, add_data_on_build=False), torch.from_numpy(ds).cuda())
    m.extend(index, torch.from_numpy(ds[:4000]).cuda(), torch.arange(4000, dtype=torch.int64).cuda())
    m.extend(index, torch.from_numpy(ds[4000:]).cuda(), torch.arange(4000, len(ds), dtype=torch.int64).cuda())
    assert len(index) == len(ds)
    sp, q = m.SearchParams(n_probes=FLAT_PROBES), torch.from_numpy(qs).cuda()
    d1, i1 = m.search(sp, index, q, 48)
    m.save(str(tmp_path / "flat.idx"), index)
    again = m.load(str(tmp_path / "flat.idx"))
    d2, i2 = m.search(sp, again, q, 48)
    assert torch.equal(i1, i2) and torch.equal(d1, d2)
    rd, ri = flat_search(index, ds, qs, FLAT_PROBES, 48, "sqeuclidean")
    assert oracle.recall_with_ties(i1.cpu().numpy(), d1.cpu().numpy(), ri, rd, eps=1e-3) >= 0.999


def test_ivf_flat_refuses_2049():
    from cuvs_b200._capi import CuvsError
    m = _ivf_flat()
    with pytest.raises(CuvsError, match="2048"):
        m.build(m.IndexParams(n_lists=8), torch.from_numpy(uniform(1000, 2049, 3)).cuda())


# ---------------------------------------------------------------------------------------------------------------- IVF-PQ
PQ_WIDTHS = (256, 512, 768, 1024, 1536, 2048)
PQ_LISTS, PQ_PROBES = 32, 8
# name: (pq_dim as a function of d (0 = the library's choice, d / 2 from 128 up), codebook kind, pq_bits, conservative)
PQ_SHAPES = {
    "auto_sub8": (lambda d: 0, "subspace", 8, False),
    "auto_cl5_cons": (lambda d: 0, "cluster", 5, True),
    "q4_sub5_cons": (lambda d: d // 4, "subspace", 5, True),
    "q4_cl8": (lambda d: d // 4, "cluster", 8, False),
}
LUTS = {"f32": np.float32, "f16": np.float16, "fp8": np.uint8}


def _ivf_pq():
    from cuvs_b200.neighbors import ivf_pq
    return ivf_pq


@functools.lru_cache(maxsize=2)
def _pq_case(d, shape):
    m = _ivf_pq()
    pq_dim, kind, bits, cons = PQ_SHAPES[shape]
    n, nq = _rows(d)
    ds, qs = uniform(n, d, 1234 + d, 0.1, 2.0), uniform(nq, d, 4321 + d, 0.1, 2.0)
    index = m.build(m.IndexParams(n_lists=PQ_LISTS, kmeans_n_iters=10, kmeans_trainset_fraction=1.0, pq_dim=pq_dim(d),
                                  codebook_kind=kind, pq_bits=bits, conservative_memory_allocation=cons),
                    torch.from_numpy(ds).cuda())
    assert index.dim == d and len(index) == n and index.pq_bits == bits
    assert index.pq_dim == (pq_dim(d) or d // 2)
    return ds, qs, index


@functools.lru_cache(maxsize=4)
def _pq_oracle(d, shape, lut):
    ds, qs, index = _pq_case(d, shape)
    return pq_search(index, qs, PQ_PROBES, 100, lut=lut, per_cluster=PQ_SHAPES[shape][1] == "cluster")


def _pq_search(monkeypatch, index, qs, k, path, lut="f32"):
    m = _ivf_pq()
    monkeypatch.setenv("CUVS_B200_PQ_PATH", path)
    return _np(*m.search(m.SearchParams(n_probes=PQ_PROBES, lut_dtype=LUTS[lut]), index, torch.from_numpy(qs).cuda(), k))


@pytest.mark.parametrize("lut", list(LUTS))
@pytest.mark.parametrize("shape", list(PQ_SHAPES))
@pytest.mark.parametrize("d", PQ_WIDTHS)
def test_ivf_pq_lut_scan_matches_oracle(monkeypatch, d, shape, lut):
    """Every index the build accepts also searches with every LUT dtype and k (a LUT too large for shared memory is kept in
    global memory), to the bars of test_ivf_pq_code_shapes_gpu.py::test_lut_scan_matches_oracle."""
    ds, qs, index = _pq_case(d, shape)
    rd_all, ri_all = _pq_oracle(d, shape, lut)
    for k in (10, 32, 48, 100):
        dist, idx = _pq_search(monkeypatch, index, qs, k, "lut", lut)
        rd, ri = rd_all[:, :k], ri_all[:, :k]
        check_rows(idx, len(ds))
        assert oracle.recall_with_ties(idx, dist, ri, rd, eps=1e-5) >= 0.999, k
        same = idx == ri
        assert (same | (np.abs(dist - rd) <= 1e-5 * np.maximum(1.0, np.abs(rd)))).mean() >= 0.99, k
        np.testing.assert_allclose(dist[same], rd[same], rtol=1e-5, atol=1e-5)
        if lut == "f32":  # the LUT kernel sums fp32 entries in the oracle's order
            np.testing.assert_array_equal(dist[same], rd[same])


@pytest.mark.parametrize("shape", list(PQ_SHAPES))
@pytest.mark.parametrize("d", PQ_WIDTHS)
def test_ivf_pq_default_path_matches_oracle(monkeypatch, d, shape):
    """Without a path override the search picks its own scan (decoded rows, or the LUT kernel on a conservative index and for
    k > 32): the bars of test_tensor_core_request_matches_oracle and test_store_path_k100_matches_oracle."""
    ds, qs, index = _pq_case(d, shape)
    rd_all, ri_all = _pq_oracle(d, shape, "f32")
    for k in (10, 32, 48, 100):
        dist, idx = _pq_search(monkeypatch, index, qs, k, "tc")
        check_rows(idx, len(ds))
        assert oracle.recall_with_ties(idx, dist, ri_all[:, :k], rd_all[:, :k], eps=2e-3) >= 0.995, k


def test_ivf_pq_transform_at_1536():
    """transform() of the first rows gives their list and their stored codes; each code is the codebook entry nearest to the
    row's rotated residual (float64, up to a near-tie), as test_transform_equals_stored_codes_and_nearest_entries checks."""
    m = _ivf_pq()
    for shape in ("auto_sub8", "q4_cl8"):
        ds, qs, index = _pq_case(1536, shape)
        nt = 256
        labels, packed = m.transform(index, torch.from_numpy(ds[:nt]).cuda())
        labels = labels.cpu().numpy().astype(np.int64)
        codes = unpack_codes(packed.cpu().numpy(), index.pq_dim, index.pq_bits)
        offs, stored, ids = index_codes(index)
        pos = np.empty(len(ds), np.int64)
        pos[ids] = np.arange(len(ds))
        rows = pos[np.arange(nt)]
        assert (np.searchsorted(offs, rows, side="right") - 1 == labels).all(), "transform's labels are not the rows' lists"
        assert (codes == stored[rows]).all(), "transform's codes are not the stored codes"
        rot = index.rotation_matrix.cpu().numpy().astype(np.float64)
        cr = index.centers_rot.cpu().numpy().astype(np.float64)
        pq = index.pq_centers.cpu().numpy().astype(np.float64)  # [books, pq_len, 2^bits]
        pq_dim, pq_len = index.pq_dim, index.pq_len
        resid = (ds[:nt].astype(np.float64) @ rot.T - cr[labels]).reshape(nt, pq_dim, pq_len)
        for r in range(nt):
            books = pq[labels[r]][None] if PQ_SHAPES[shape][1] == "cluster" else pq  # [pq_dim | 1, pq_len, 2^bits]
            err = ((resid[r][:, :, None] - books) ** 2).sum(1)  # [pq_dim, 2^bits]
            chosen = err[np.arange(pq_dim), codes[r]]
            assert (chosen <= err.min(1) + 1e-4 * np.maximum(1.0, err.min(1))).all(), f"row {r}: a code is not the nearest entry"


def test_ivf_pq_refuses_2049():
    from cuvs_b200._capi import CuvsError
    m = _ivf_pq()
    with pytest.raises(CuvsError, match="2048"):
        m.build(m.IndexParams(n_lists=8), torch.from_numpy(uniform(1000, 2049, 3)).cuda())


# --------------------------------------------------------------------------------------------------------------- k-means
KM_WIDTHS = (256, 257, 768, 1024, 2047, 2048)
KM_CLUSTERS = 100


def _km():
    from cuvs_b200.cluster import kmeans
    return kmeans


def _sq_dist64(x, c):
    x, c = x.astype(np.float64), c.astype(np.float64)
    return np.maximum((x * x).sum(1)[:, None] + (c * c).sum(1)[None, :] - 2.0 * (x @ c.T), 0.0)


@pytest.mark.parametrize("d", KM_WIDTHS)
def test_kmeans_predict_and_cost(d):
    """Labels equal the float64 argmin except between centroids whose float64 distances are within the tie tolerance
    2^-15 (|x|^2 + max|c|^2) (the split-bf16 assignment's budget); the cost is the float64 sum."""
    km = _km()
    x, c = uniform(10001, d, 3 + d), uniform(KM_CLUSTERS, d, 4 + d)
    labels, inertia = km.predict(km.KMeansParams(n_clusters=KM_CLUSTERS), torch.from_numpy(x).cuda(), torch.from_numpy(c).cuda())
    labels = labels.cpu().numpy().astype(np.int64)
    dd = _sq_dist64(x, c)
    best = dd.argmin(1)
    rows = np.arange(len(x))
    tol = 2.0 ** -15 * ((x.astype(np.float64) ** 2).sum(1) + (c.astype(np.float64) ** 2).sum(1).max())
    gap = dd[rows, labels] - dd[rows, best]
    assert (gap <= tol).all(), f"{(gap > tol).sum()} labels are not a near-tie of the float64 argmin"
    assert (labels != best).mean() < 1e-3
    cost64 = dd[rows, best].sum()
    assert inertia == pytest.approx(cost64, rel=1e-4)
    assert km.cluster_cost(torch.from_numpy(x).cuda(), torch.from_numpy(c).cuda()) == pytest.approx(cost64, rel=1e-4)


@pytest.mark.parametrize("d", KM_WIDTHS)
def test_kmeans_fit_from_given_centroids_is_one_lloyd_step(d):
    km = _km()
    x, centers = clustered(10001, d, 9 + d, n_centers=20)
    c0 = centers + 0.01 * np.random.default_rng(d).standard_normal(centers.shape).astype(np.float32)
    cent, _, _ = km.fit(km.KMeansParams(n_clusters=20, init_method="array", max_iter=1), torch.from_numpy(x).cuda(),
                        centroids=torch.from_numpy(c0.copy()).cuda())
    lab = _sq_dist64(x, c0).argmin(1)
    expect = np.stack([x[lab == j].astype(np.float64).mean(0) if (lab == j).any() else c0[j] for j in range(20)])
    np.testing.assert_allclose(cent.cpu().numpy(), expect, rtol=1e-4, atol=1e-4)


def test_kmeans_refuses_2049():
    from cuvs_b200._capi import CuvsError
    km = _km()
    x = torch.from_numpy(uniform(1000, 2049, 3)).cuda()
    with pytest.raises(CuvsError, match="2048"):
        km.fit(km.KMeansParams(n_clusters=4, max_iter=2), x)
    with pytest.raises(CuvsError, match="2048"):
        km.predict(km.KMeansParams(n_clusters=4), x, x[:4].contiguous())


# ----------------------------------------------------------------------------------------------------------------- CAGRA
CAGRA_N, CAGRA_DEGREE = 5001, 32


@functools.lru_cache(maxsize=2)
def _cagra_data(d):
    """Rows and queries of a rank-8 manifold in d dims, and an exact kNN graph over the rows (float64 distances)."""
    rng = np.random.default_rng(50 + d)
    a = (rng.standard_normal((8, d)) / np.sqrt(8)).astype(np.float32)
    ds = (rng.standard_normal((CAGRA_N, 8)).astype(np.float32) @ a + 0.05 * rng.standard_normal((CAGRA_N, d)).astype(np.float32))
    qs = (rng.standard_normal((200, 8)).astype(np.float32) @ a + 0.05 * rng.standard_normal((200, d)).astype(np.float32))
    return ds, qs


@functools.lru_cache(maxsize=2)
def _cagra_graph(d, metric="sqeuclidean"):
    ds, _ = _cagra_data(d)
    x = ds.astype(np.float64)
    if metric == "cosine":
        x = x / np.linalg.norm(x, axis=1, keepdims=True)
        score = -(x @ x.T)
    else:
        n2 = (x * x).sum(1)
        score = n2[None, :] - 2.0 * (x @ x.T)
    np.fill_diagonal(score, np.inf)
    return np.argsort(score, axis=1, kind="stable")[:, :CAGRA_DEGREE].astype(np.uint32)


def _cagra():
    from cuvs_b200.neighbors import cagra
    return cagra


def _cagra_index(d, metric="sqeuclidean"):
    ds, _ = _cagra_data(d)
    return _cagra().from_graph(torch.from_numpy(_cagra_graph(d, metric).astype(np.int64)).cuda(), torch.from_numpy(ds).cuda(),
                               metric=metric)


@pytest.mark.parametrize("d", [256, 384, 1024, 1536, 2048])
def test_cagra_single_cta_matches_oracle(d):
    """The criteria of test_cagra_search_space_gpu.py::test_single_cta_matches_oracle."""
    m = _cagra()
    ds, qs = _cagra_data(d)
    dist, idx = _np(*m.search(m.SearchParams(itopk_size=64, algo="single_cta"), _cagra_index(d), torch.from_numpy(qs).cuda(), 10))
    rd, ri, _ = oracle.cagra_search(_cagra_graph(d), ds, qs, 10, itopk=64)
    ri = ri.astype(np.int64)
    assert oracle.recall_with_ties(idx, dist, ri, rd, eps=1e-4) >= 0.999
    same = idx == ri
    assert same.mean() >= 0.99
    np.testing.assert_allclose(dist[same], rd[same], rtol=1e-5, atol=1e-5)


def _check_exact_result(ds, qs, dist, idx, k):
    assert all(len(set(r.tolist())) == k for r in idx), "duplicate ids"
    assert (idx >= 0).all() and (idx < len(ds)).all(), "id out of range"
    assert (np.diff(dist, axis=1) >= 0).all(), "distances not sorted"
    np.testing.assert_allclose(dist, ((ds[idx].astype(np.float64) - qs[:, None, :]) ** 2).sum(-1), rtol=1e-5, atol=1e-5)


def test_cagra_multi_cta_and_fp16_walk_at_1536():
    """The multi-CTA walk: unique, sorted, exact distances, recall at least the single-CTA walk's minus 0.02.  The fp16 walk:
    distances are the fp32 re-rank of its results, sorted and unique."""
    m = _cagra()
    d = 1536
    ds, qs = _cagra_data(d)
    _, gi = oracle.knn(ds, qs, 10)
    q = torch.from_numpy(qs).cuda()
    _, i_single = _np(*m.search(m.SearchParams(itopk_size=64, algo="single_cta"), _cagra_index(d), q, 10))
    dist, idx = _np(*m.search(m.SearchParams(itopk_size=64, search_width=4, algo="multi_cta"), _cagra_index(d), q[:32], 10))
    _check_exact_result(ds, qs[:32], dist, idx, 10)
    assert oracle.recall(idx, gi[:32]) >= oracle.recall(i_single[:32], gi[:32]) - 0.02
    index = _cagra_index(d)
    index.set_walk_precision(16)
    dist, idx = _np(*m.search(m.SearchParams(itopk_size=128, algo="single_cta"), index, q, 10))
    _check_exact_result(ds, qs, dist, idx, 10)
    assert oracle.recall(idx, gi) >= oracle.recall(i_single, gi) - 0.02


def test_cagra_cosine_at_1024():
    m = _cagra()
    d = 1024
    ds, qs = _cagra_data(d)
    dist, idx = _np(*m.search(m.SearchParams(itopk_size=64, algo="single_cta"), _cagra_index(d, "cosine"),
                              torch.from_numpy(qs).cuda(), 10))
    rd, ri, _ = cagra_cosine_search(_cagra_graph(d, "cosine"), ds, qs, 10, itopk=64)
    ri = ri.astype(np.int64)
    assert oracle.recall_with_ties(idx, dist, ri, rd, eps=1e-4) >= 0.999
    same = idx == ri
    assert same.mean() >= 0.99
    np.testing.assert_allclose(dist[same], rd[same], rtol=0, atol=1e-4)


def test_cagra_build_at_768():
    """build (graph from the library's own IVF-PQ kNN at this width) and search, with the recall floor of
    test_cagra_gpu.py::test_build_search_save_load."""
    m = _cagra()
    rng = np.random.default_rng(768)
    a = (rng.standard_normal((8, 768)) / np.sqrt(8)).astype(np.float32)
    ds = (rng.standard_normal((10001, 8)).astype(np.float32) @ a + 0.05 * rng.standard_normal((10001, 768)).astype(np.float32))
    qs = (rng.standard_normal((257, 8)).astype(np.float32) @ a + 0.05 * rng.standard_normal((257, 768)).astype(np.float32))
    index = m.build(m.IndexParams(graph_degree=32), torch.from_numpy(ds).cuda())
    _, idx = _np(*m.search(m.SearchParams(itopk_size=64), index, torch.from_numpy(qs).cuda(), 10))
    _, gi = oracle.knn(ds, qs, 10)
    assert oracle.recall(idx, gi) >= 0.95


# --------------------------------------------------------------------------------------------- refine, pairwise distance
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("n_cand", [257, 2048])
@pytest.mark.parametrize("d", [1536, 2048, 3072])
def test_refine_equals_exact_rerank(d, n_cand, metric):
    """The bars of test_ivf_pq_large_k_gpu.py::test_refine_many_candidates_equals_exact_rerank."""
    from cuvs_b200.neighbors import refine
    rng = np.random.default_rng(d + n_cand)
    ds = rng.standard_normal((20000, d)).astype(np.float32)
    qs = rng.standard_normal((33, d)).astype(np.float32)
    cand = np.stack([rng.choice(len(ds), n_cand, replace=False) for _ in range(len(qs))]).astype(np.int64)
    k = 100

    def run(c):
        out = refine(torch.from_numpy(ds).cuda(), torch.from_numpy(qs).cuda(), torch.from_numpy(c).cuda(), k=k, metric=metric)
        return out[0].cpu().numpy(), out[1].cpu().numpy()

    dist, idx = run(cand)
    ex = np.empty(cand.shape)
    for r in range(len(qs)):  # float64, one query at a time
        q, sub = qs[r].astype(np.float64), ds[cand[r]].astype(np.float64)
        if metric == "sqeuclidean":
            ex[r] = ((sub - q) ** 2).sum(1)
        elif metric == "inner_product":
            ex[r] = -(sub @ q)
        else:
            ex[r] = 1 - (sub @ q) / (np.linalg.norm(q) * np.linalg.norm(sub, axis=1))
    order = np.argsort(ex, axis=1, kind="stable")[:, :k]
    ri, rd = np.take_along_axis(cand, order, 1), np.take_along_axis(ex, order, 1)
    # an id may differ from the float64 re-rank only at an fp32 near-tie: its own float64 distance is the slot's to 1e-5
    pos = {(r, c): j for r in range(len(qs)) for j, c in enumerate(cand[r])}
    got = np.array([[ex[r, pos[(r, c)]] for c in row] for r, row in enumerate(idx)])
    np.testing.assert_allclose(got, rd, rtol=1e-5, atol=1e-5)
    assert (idx == ri).mean() >= 0.99
    if metric == "inner_product":
        rd = -rd
    np.testing.assert_allclose(dist, rd, rtol=1e-4, atol=1e-4)
    if n_cand > 256:  # bit-identical to the one-warp path on the same 256 real candidates
        c2 = cand.copy()
        c2[:, 256:] = -1
        db, ib = run(c2)
        dw, iw = run(np.ascontiguousarray(cand[:, :256]))
        assert (ib == iw).all() and (db.view(np.uint32) == dw.view(np.uint32)).all()


@pytest.mark.parametrize("metric,code", [("sqeuclidean", 0), ("euclidean", 1), ("inner_product", 6), ("cosine", 2)])
@pytest.mark.parametrize("d", [1536, 2048, 3072])
def test_pairwise_distance(d, metric, code):
    """cuvsPairwiseDistance vs float64 to the tolerance of test_mg_gpu.py::test_pairwise_distance, plus the fp32 rounding of a
    d-term dot product, 2^-22 |x| |y| (which the inner product, near 0 where x and y are near orthogonal, shows)."""
    import ctypes as C
    from cuvs_b200._capi import DL, check, lib
    from cuvs_b200.common import Resources
    x, y = uniform(257, d, 1 + d), uniform(129, d, 2 + d)
    out = torch.empty((257, 129), dtype=torch.float32, device="cuda")
    res = Resources()
    xg, yg = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    dx, dy, do = DL(xg), DL(yg), DL(out)
    check(lib.cuvsPairwiseDistance(res.get_c_obj(), dx.ptr, dy.ptr, do.ptr, C.c_int(code), C.c_float(2.0)))
    res.sync()
    x64, y64 = x.astype(np.float64), y.astype(np.float64)
    dot = x64 @ y64.T
    sq = (x64 ** 2).sum(1)[:, None] + (y64 ** 2).sum(1)[None, :] - 2 * dot
    ref = {"sqeuclidean": sq, "euclidean": np.sqrt(np.maximum(sq, 0)), "inner_product": dot,
           "cosine": 1 - dot / np.sqrt((x64 ** 2).sum(1)[:, None] * (y64 ** 2).sum(1)[None, :])}[metric]
    nx, ny = np.sqrt((x64 ** 2).sum(1)), np.sqrt((y64 ** 2).sum(1))
    got = out.cpu().numpy()
    tol = 2e-5 + 2e-5 * np.abs(ref) + (2.0 ** -22 * nx[:, None] * ny[None, :] if metric == "inner_product" else 0.0)
    bad = np.abs(got - ref) > tol
    assert not bad.any(), f"{bad.sum()} of {bad.size} distances off, worst {np.abs(got - ref)[bad].max():.3e}"
