"""IVF-PQ search with 64 < k <= 2048 and cuvsRefine with 257..2048 candidates.

k > 64 writes every (query, probe, list row) score to a dense per-pair segment (store epilogue of the code-stream scan, store
mode of the LUT kernel), selects each pair's k best with the segmented select_k and merges the probes as the k <= 64 path
does.  Checked against the oracle's IVF-PQ search (any k; n_probes follows the reference's var_k rule
max(n_probes, min(n_lists, k)), ann_ivf_pq.cuh:1161-1171), against the k = 64 search of the same index (prefix
consistency), and for invariance under a forced workspace split and forced work-item widths."""
import numpy as np
import pytest
import torch

import oracle
from tests.ivf_oracle import check_rows, pq_search
from tests.util import clustered, uniform

pytestmark = pytest.mark.gpu

KS = [65, 100, 128, 129, 256, 257, 1023, 2048]


def _mod():
    from cuvs_b200.neighbors import ivf_pq
    return ivf_pq


def _search(monkeypatch, index, qs, n_probes, k, path, lut="f32", **env):
    m = _mod()
    monkeypatch.setenv("CUVS_B200_PQ_PATH", path)
    for key, v in env.items():
        monkeypatch.setenv(key, str(v))
    kw = {"lut_dtype": {"f32": np.float32, "f16": np.float16, "fp8": np.uint8}[lut]}
    d, i = m.search(m.SearchParams(n_probes=n_probes, **kw), index, torch.from_numpy(qs).cuda(), k)
    for key in env:
        monkeypatch.delenv(key)
    return d.cpu().numpy(), i.cpu().numpy()


def _probes(n_lists, k, base=8):
    return max(base, min(n_lists, k))


def _check_prefix(d64, i64, dk, ik):
    """The first 64 columns of a k > 64 search equal the k = 64 search: distances to 1e-6 relative, ids where not tied."""
    np.testing.assert_allclose(dk[:, :64], d64, rtol=1e-6, atol=1e-6)
    tied = np.zeros_like(d64, dtype=bool)
    tied[:, 1:] |= d64[:, 1:] == d64[:, :-1]
    tied[:, :-1] |= d64[:, :-1] == d64[:, 1:]
    tied[:, -1] = True  # the 64th entry may tie with the 65th, which only the k > 64 search sees
    assert (ik[:, :64][~tied] == i64[~tied]).all()


@pytest.fixture(scope="module")
def stream_index():
    """dim 64, pq_dim 32, pq_len 2, 8 bits, per-subspace codebooks: served by the code-stream scan."""
    m = _mod()
    ds = uniform(4096, 64, 1234, 0.1, 2.0)
    qs = uniform(256, 64, 4321, 0.1, 2.0)
    index = m.build(m.IndexParams(n_lists=32, pq_dim=32, pq_bits=8, kmeans_n_iters=20), torch.from_numpy(ds).cuda())
    assert index.streamed
    return ds, qs, index


@pytest.mark.parametrize("k", KS)
def test_lut_store_matches_oracle(monkeypatch, stream_index, k):
    ds, qs, index = stream_index
    p = _probes(32, k)
    d, i = _search(monkeypatch, index, qs, p, k, "lut")
    rd, ri = pq_search(index, qs, p, k, "sqeuclidean")
    check_rows(i, len(ds))
    assert oracle.recall_with_ties(i, d, ri, rd, eps=1e-5) >= 0.999
    same = i == ri
    assert same.mean() >= 0.99
    np.testing.assert_allclose(d[same], rd[same], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("lut", ["f32", "f16"])
def test_stream_store_matches_oracle(monkeypatch, stream_index, k, lut):
    ds, qs, index = stream_index
    p = _probes(32, k)
    d, i = _search(monkeypatch, index, qs, p, k, "stream", lut=lut)
    rd, ri = pq_search(index, qs, p, k, "sqeuclidean", lut=lut)
    check_rows(i, len(ds))
    if lut == "f32":
        assert oracle.recall_with_ties(i, d, ri, rd, eps=2e-3) >= 0.99
    else:
        assert oracle.recall_with_ties(i, d, ri, rd, eps=1e-2) >= 0.975


@pytest.mark.parametrize("path,lut", [("stream", "f32"), ("stream", "f16"), ("lut", "f32")])
@pytest.mark.parametrize("k", [65, 256])
def test_prefix_equals_k64_search(monkeypatch, stream_index, path, lut, k):
    ds, qs, index = stream_index
    d64, i64 = _search(monkeypatch, index, qs, 32, 64, path, lut=lut)
    dk, ik = _search(monkeypatch, index, qs, 32, k, path, lut=lut)
    _check_prefix(d64, i64, dk, ik)


@pytest.mark.parametrize("metric", ["inner_product", "cosine", "euclidean"])
@pytest.mark.parametrize("shape", ["stream", "per_cluster", "pq_bits5"])
def test_metrics_and_index_shapes(monkeypatch, metric, shape):
    """Every metric on each class of index shape: the k = 100 search extends the k = 64 search of the same index."""
    m = _mod()
    ds, centers = clustered(8000, 64, 3, n_centers=40)
    qs, _ = clustered(128, 64, 4, centers=centers)
    kw = {"stream": dict(pq_dim=32), "per_cluster": dict(pq_dim=32, codebook_kind="cluster"), "pq_bits5": dict(pq_dim=32, pq_bits=5)}[shape]
    index = m.build(m.IndexParams(n_lists=40, metric=metric, kmeans_n_iters=10, **kw), torch.from_numpy(ds).cuda())
    assert index.streamed == (shape == "stream")
    for path in (["stream", "lut"] if shape == "stream" else ["lut"]):  # k > 64 serves these shapes with the LUT kernel
        d64, i64 = _search(monkeypatch, index, qs, 40, 64, path)
        dk, ik = _search(monkeypatch, index, qs, 40, 100, path)
        check_rows(ik, len(ds))
        _check_prefix(d64, i64, dk, ik)
        if metric == "inner_product" and shape == "stream" and path == "lut":
            rd, ri = pq_search(index, qs, 40, 100, metric)
            assert oracle.recall_with_ties(ik, dk, ri, rd, eps=1e-5) >= 0.999


@pytest.mark.parametrize("k", [128, 129])
@pytest.mark.parametrize("path", ["stream", "lut"])
def test_reference_special_cases_recall_floor(monkeypatch, k, path):
    """ann_ivf_pq.cuh:1220-1245: 10 000 x 16, 500 queries, n_lists 100, n_probes 100, k 128 / 129, the recall floor of
    test_reference_recall_floor."""
    m = _mod()
    ds = uniform(10000, 16, 1234, 0.1, 2.0)
    qs = uniform(500, 16, 4321, 0.1, 2.0)
    index = m.build(m.IndexParams(n_lists=100, kmeans_trainset_fraction=1.0), torch.from_numpy(ds).cuda())
    d, i = _search(monkeypatch, index, qs, 100, k, path)
    gd, gi = oracle.knn(ds, qs, k)
    check_rows(i, len(ds))
    assert oracle.recall_with_ties(i, d, gi, gd, eps=1e-4 * 4) >= 0.86


@pytest.mark.parametrize("path,lut", [("stream", "f32"), ("stream", "f16"), ("lut", "f32")])
def test_split_batches_and_group_widths_are_invariant(monkeypatch, stream_index, path, lut):
    ds, qs, index = stream_index
    d0, i0 = _search(monkeypatch, index, qs, 32, 300, path, lut=lut)
    # 1 MiB holds the workspace of a few queries only: the batch runs in many pieces
    d1, i1 = _search(monkeypatch, index, qs, 32, 300, path, lut=lut, CUVS_B200_PQ_LARGE_K_BUDGET_MB=1)
    assert (i0 == i1).all() and (d0 == d1).all()
    if path == "stream":
        for g in (32, 64, 128):
            dg, ig = _search(monkeypatch, index, qs, 32, 300, path, lut=lut, CUVS_B200_PQ_GROUP=g)
            assert (i0 == ig).all() and (d0 == dg).all()


@pytest.mark.parametrize("path", ["stream", "lut"])
def test_fewer_probed_rows_than_k_fill_like_k64(monkeypatch, path):
    m = _mod()
    ds = uniform(1024, 64, 7, 0.1, 2.0)
    qs = uniform(64, 64, 8, 0.1, 2.0)
    index = m.build(m.IndexParams(n_lists=128, pq_dim=32), torch.from_numpy(ds).cuda())
    sizes = index.list_sizes.cpu().numpy()
    assert sizes.max() < 64
    d64, i64 = _search(monkeypatch, index, qs, 1, 64, path)
    dk, ik = _search(monkeypatch, index, qs, 1, 200, path)
    _check_prefix(d64, i64, dk, ik)
    # the k = 64 search already shows the fill (one list holds < 64 rows); the k = 200 search continues it
    fill_i, fill_d = i64[:, -1], d64[:, -1]
    assert (fill_i == np.iinfo(np.int64).max).all()
    assert (ik[:, 64:] == fill_i[:, None]).all() and (dk[:, 64:] == fill_d[:, None]).all()


def test_k_above_2048_is_a_clean_error(monkeypatch, stream_index):
    ds, qs, index = stream_index
    with pytest.raises(Exception, match="2048"):
        _search(monkeypatch, index, qs[:4], 32, 2049, "stream")
    d, i = _search(monkeypatch, index, qs[:4], 32, 10, "stream")  # the library is still usable
    assert (i[:, 0] >= 0).all()


# ---------------------------------------------------------------------------------------------------------------- refine
def _refine(ds, qs, cand, k, metric):
    from cuvs_b200.neighbors import refine
    d, i = refine(torch.from_numpy(ds).cuda(), torch.from_numpy(qs).cuda(), torch.from_numpy(cand).cuda(), k=k, metric=metric)
    return d.cpu().numpy(), i.cpu().numpy()


@pytest.mark.parametrize("metric", ["sqeuclidean", "inner_product", "cosine"])
@pytest.mark.parametrize("n_cand", [257, 512, 2048])
def test_refine_many_candidates_equals_exact_rerank(metric, n_cand):
    """The one-CTA-per-query path (> 256 candidates) scores and ranks exactly like the one-warp path: a candidate list whose
    first 256 entries are real and the rest invalid (-1) gives bit-identical ids and distances to the 256-column list."""
    rng = np.random.default_rng(n_cand)
    ds = rng.standard_normal((20000, 96)).astype(np.float32)
    qs = rng.standard_normal((300, 96)).astype(np.float32)
    cand = np.stack([rng.choice(len(ds), n_cand, replace=False) for _ in range(len(qs))]).astype(np.int64)
    k = 100
    d, i = _refine(ds, qs, cand, k, metric)
    # exact re-rank in float64: same ids (ties aside) and distances to fp32 rounding
    x, q = ds.astype(np.float64), qs.astype(np.float64)
    sub = x[cand]
    if metric == "sqeuclidean":
        ex = ((q[:, None, :] - sub) ** 2).sum(-1)
    elif metric == "inner_product":
        ex = -(q[:, None, :] * sub).sum(-1)
    else:
        ex = 1 - (q[:, None, :] * sub).sum(-1) / (np.linalg.norm(q, axis=1)[:, None] * np.linalg.norm(sub, axis=2))
    order = np.argsort(ex, axis=1, kind="stable")[:, :k]
    ri = np.take_along_axis(cand, order, 1)
    rd = np.take_along_axis(ex, order, 1)
    if metric == "inner_product":
        rd = -rd
    assert (i == ri).mean() >= 0.999
    np.testing.assert_allclose(d, rd, rtol=1e-4, atol=1e-4)
    # bit-identical to the one-warp path on the same 256 real candidates
    c2 = cand.copy()
    c2[:, 256:] = -1
    db, ib = _refine(ds, qs, c2, k, metric)
    dw, iw = _refine(ds, qs, np.ascontiguousarray(cand[:, :256]), k, metric)
    assert (ib == iw).all() and (db.view(np.uint32) == dw.view(np.uint32)).all()


def test_refine_invalid_candidates_fill_like_the_warp_path():
    rng = np.random.default_rng(3)
    ds = rng.standard_normal((5000, 32)).astype(np.float32)
    qs = rng.standard_normal((50, 32)).astype(np.float32)
    cand = np.full((50, 600), -1, np.int64)
    cand[:, :40] = rng.integers(0, len(ds), (50, 40))
    d, i = _refine(ds, qs, cand, 100, "sqeuclidean")
    dw, iw = _refine(ds, qs, np.ascontiguousarray(cand[:, :200]), 100, "sqeuclidean")
    assert (i == iw).all() and (d.view(np.uint32) == dw.view(np.uint32)).all()


def test_ivf_pq_then_refine_beats_plain_search(monkeypatch):
    m = _mod()
    ds, centers = clustered(50000, 64, 11, n_centers=100)
    qs, _ = clustered(200, 64, 12, centers=centers)
    index = m.build(m.IndexParams(n_lists=100, pq_dim=32, kmeans_n_iters=10), torch.from_numpy(ds).cuda())
    gd, gi = oracle.knn(ds, qs, 100)
    d100, i100 = _search(monkeypatch, index, qs, 20, 100, "auto")
    d400, i400 = _search(monkeypatch, index, qs, 20, 400, "auto")
    rd, ri = _refine(ds, qs, i400, 100, "sqeuclidean")
    assert oracle.recall(ri, gi) > oracle.recall(i100, gi)
