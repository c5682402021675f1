"""IVF-PQ with the cosine metric (CosineExpanded) through the C ABI.

Reference semantics (cpp/src/neighbors/ivf_pq/ivf_pq_build.cuh:159-174, :1336-1348; ivf_pq_search.cuh:101-107, :545-549,
:1020-1025): unit training rows and unit centres, residuals R x/|x| - c_rot[label], probes ranked by -q.c, and the fine
score 1 - q^.(c + y) with q^ the unit rotated query.  The library's own quantizers, codes and list membership are read back
through the getters and fed to the oracle's LUT-sum search with the unit rotated queries (tests/ivf_pq_cosine_ref.py).  Every
fine-scan kernel must reproduce it.  Recall floors follow cpp/tests/neighbors/ann_ivf_pq.cuh:1105-1122 (the L2
floor x 0.94, x 0.70 for the 8-bit LUT)."""
import os

import numpy as np
import pytest
import torch

import oracle
from tests.ivf_oracle import pq_search
from tests.ivf_pq_codes import index_codes
from tests.util import clustered, uniform

pytestmark = pytest.mark.gpu


def _mod():
    from cuvs_b200.neighbors import ivf_pq
    return ivf_pq


def mixed_norm(n, d, seed, n_centers=64, centers=None):
    """Clustered rows times a seeded log-uniform factor in [0.1, 10]: cosine and inner-product rankings differ."""
    x, centers = clustered(n, d, seed, n_centers=n_centers, centers=centers)
    f = np.exp(np.random.default_rng(seed + 1000).uniform(np.log(0.1), np.log(10.0), n)).astype(np.float32)
    return (x * f[:, None]).astype(np.float32), centers


def _by_id(index):
    """-> (ids, list label, codes) of every stored row, ordered by id: with the default ids, the order of the dataset."""
    offs, codes, ids = index_codes(index)
    labels = np.searchsorted(offs, np.arange(len(ids)), side="right") - 1
    order = np.argsort(ids, kind="stable")
    return ids[order], labels[order], codes[order]


def _oracle(index, qs, n_probes, k, lut="f32", dist="f32"):
    return pq_search(index, qs, n_probes, k, "cosine", lut, dist)


def _search(index, qs, n_probes, k, path, **kw):
    m = _mod()
    os.environ["CUVS_B200_PQ_PATH"] = path
    try:
        d, i = m.search(m.SearchParams(n_probes=n_probes, **kw), index, torch.as_tensor(qs).cuda(), k)
    finally:
        del os.environ["CUVS_B200_PQ_PATH"]
    return d.cpu().numpy(), i.cpu().numpy()


_LUT = {"f32": np.float32, "f16": np.float16, "fp8": np.uint8}


# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def stream_shape():
    """20k x 128 mixed-norm rows, pq_dim 64 (pq_len 2, 8-bit codes): the code-streaming scan's shape."""
    m = _mod()
    ds, centers = mixed_norm(20000, 128, 21)
    qs, _ = mixed_norm(512, 128, 22, centers=centers)
    index = m.build(m.IndexParams(n_lists=64, pq_dim=64, metric="cosine", kmeans_n_iters=10), torch.from_numpy(ds).cuda())
    return ds, qs, index


def test_quantiser_shape(stream_shape):
    m = _mod()
    ds, qs, index = stream_shape
    c = index.centers.cpu().numpy().astype(np.float64)
    np.testing.assert_allclose(np.linalg.norm(c, axis=1), 1.0, rtol=0, atol=1e-5)
    # stored codes are transform() of the same rows
    ids, lab, codes = _by_id(index)
    assert (ids == np.arange(len(ds))).all()
    tlab, tcodes = m.transform(index, torch.from_numpy(ds).cuda())
    assert (tcodes.cpu().numpy() == codes).all()
    assert (tlab.cpu().numpy().astype(np.int64) == lab).all()
    # the same scan path as an inner-product index of the same shape
    ip = m.build(m.IndexParams(n_lists=64, pq_dim=64, metric="inner_product", kmeans_n_iters=10), torch.from_numpy(ds).cuda())
    assert index.streamed and index._info()[0] == ip._info()[0]


# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def small_index():
    m = _mod()
    ds, centers = mixed_norm(4096, 64, 31, n_centers=32)
    qs, _ = mixed_norm(1024, 64, 32, centers=centers)
    index = m.build(m.IndexParams(n_lists=32, pq_dim=32, pq_bits=8, metric="cosine", kmeans_n_iters=20), torch.from_numpy(ds).cuda())
    return ds, qs, index


def _matched_by_id(i, d, ri, rd):
    """-> (fraction of returned ids that the oracle also returns for that query, |d - rd| of each such id)."""
    hit, diff = 0, []
    for a, da, b, db in zip(i, d, ri, rd):
        ref = {int(x): float(y) for x, y in zip(b, db)}
        for x, y in zip(a, da):
            if int(x) in ref:
                hit += 1
                diff.append(abs(float(y) - ref[int(x)]))
    return hit / i.size, np.asarray(diff)


@pytest.mark.parametrize("lut,dist,tol", [("f32", "f32", 1e-5), ("f16", "f32", 1e-5), ("fp8", "f32", 1e-5), ("f16", "f16", 2e-2)])
def test_lut_scan_matches_oracle(small_index, lut, dist, tol):
    """Ids are compared per query as sets and distances per id: the fp16 and fp_8bit LUT entries make exact ties common, and
    the kernel and the oracle order tied rows differently (row position against id)."""
    ds, qs, index = small_index
    d, i = _search(index, qs, 8, 32, "lut", lut_dtype=_LUT[lut], internal_distance_dtype=_LUT[dist])
    rd, ri = _oracle(index, qs, 8, 32, lut, dist)
    assert oracle.recall_with_ties(i, d, ri, rd, eps=max(tol, 1e-5)) >= 0.999
    if dist == "f32":
        same, diff = _matched_by_id(i, d, ri, rd)
        assert same >= 0.99
        # the kernel rounds q.c before subtracting it where the oracle fuses it (fmaf): an fp32 ulp apart, which can move a
        # reduced-precision LUT entry across a rounding boundary in rare rows
        assert (diff <= tol).mean() >= (1.0 if lut == "f32" else 0.999)
        assert diff.max() <= {"f32": tol, "f16": 1e-4, "fp8": 1e-2}[lut]


@pytest.mark.parametrize("path,k", [("tc", 32), ("stream", 32), ("stream", 64)])
def test_tensor_core_paths_match_oracle(small_index, path, k):
    """"tc" with 1024 queries x 8 probes over 32 lists probes densely and is served from the decoded-row cache; "stream" forces
    the code-streaming scan, which also serves k = 64."""
    ds, qs, index = small_index
    assert index.streamed and index.has_decoded_rows
    d, i = _search(index, qs, 8, k, path)
    rd, ri = _oracle(index, qs, 8, k)
    assert oracle.recall_with_ties(i, d, ri, rd, eps=2e-3) >= 0.995
    same = i == ri
    np.testing.assert_allclose(d[same], rd[same], rtol=2e-3, atol=2e-3)
    assert all(len(set(r.tolist())) == k for r in i) and (i >= 0).all() and (i < len(ds)).all()


@pytest.mark.parametrize("path,lut,floor", [("lut", "f32", 0.86 * 0.94), ("tc", "f32", 0.86 * 0.94), ("lut", "f16", 0.84 * 0.94),
                                            ("lut", "fp8", 0.84 * 0.70), ("tc", "fp8", 0.84 * 0.70)])
def test_reference_recall_floor(path, lut, floor):
    """ann_ivf_pq.cuh:26-43 defaults (4096 x 64, 1024 queries, k 32, n_lists 32, pq_dim auto, trainset fraction 1.0, n_probes 20),
    cosine ground truth, floors scaled as enum_variety_cosine (:1105-1122)."""
    m = _mod()
    ds = uniform(4096, 64, 1234, 0.1, 2.0)
    qs = uniform(1024, 64, 4321, 0.1, 2.0)
    index = m.build(m.IndexParams(n_lists=32, kmeans_trainset_fraction=1.0, metric="cosine"), torch.from_numpy(ds).cuda())
    d, i = _search(index, qs, 20, 32, path, lut_dtype=_LUT[lut])
    gd, gi = oracle.knn(ds, qs, 32, metric="cosine")
    assert oracle.recall_with_ties(i, d, gi, gd, eps=4e-4) >= floor


@pytest.mark.parametrize("path,tol", [("lut", 1e-5), ("stream", 1e-4)])
def test_query_scale_invariance(stream_shape, path, tol):
    """q and 7.3 q are the same cosine query.  The fp32 LUT path agrees to 1e-5; the code-streaming scan splits the unit query
    into two bf16 planes, whose last bits can differ between q^ and (7.3 q)^, so it agrees to 1e-4."""
    ds, qs, index = stream_shape
    d1, i1 = _search(index, qs, 16, 10, path)
    d2, i2 = _search(index, (qs * np.float32(7.3)).astype(np.float32), 16, 10, path)
    assert (i1 == i2).mean() >= 0.999
    np.testing.assert_allclose(d2, d1, rtol=0, atol=tol)


@pytest.mark.parametrize("path", ["lut", "stream", "tc"])
def test_zero_rows_and_zero_query(path):
    """A zero row scales to the zero vector: its cosine distance to anything is 1, and nothing turns into NaN or Inf."""
    m = _mod()
    ds, centers = mixed_norm(6000, 64, 41, n_centers=16)
    ds[::50] = 0.0
    qs, _ = mixed_norm(64, 64, 42, centers=centers)
    qs[0] = 0.0
    qs[1] = ds[50]  # a zero row of the data as the query
    qs = np.concatenate([qs] * 5)  # 320 queries x 8 probes over 16 lists: dense enough for the decoded-row cache ("tc")
    index = m.build(m.IndexParams(n_lists=16, pq_dim=32, metric="cosine", kmeans_n_iters=10), torch.from_numpy(ds).cuda())
    d, i = _search(index, qs, 8, 10, path)
    assert np.isfinite(d).all() and (i >= 0).all() and (i < len(ds)).all()
    assert (d[[0, 1, 64, 65]] == 1.0).all()
    rd, ri = _oracle(index, qs[:64], 8, 10)
    assert np.isfinite(rd).all() and (rd[:2] == 1.0).all()


def test_extend_in_chunks_equals_build_with_data():
    m = _mod()
    ds, _ = mixed_norm(12000, 128, 51)
    params = dict(n_lists=32, pq_dim=64, metric="cosine", kmeans_n_iters=10)
    full = m.build(m.IndexParams(**params), torch.from_numpy(ds).cuda())
    empty = m.build(m.IndexParams(add_data_on_build=False, **params), torch.from_numpy(ds).cuda())
    assert len(empty) == 0
    ids = np.arange(len(ds), dtype=np.int64)
    m.extend(empty, torch.from_numpy(ds[:5000]).cuda(), torch.from_numpy(ids[:5000]).cuda())
    m.extend(empty, torch.from_numpy(ds[5000:]).cuda(), torch.from_numpy(ids[5000:]).cuda())
    assert len(empty) == len(ds)
    assert np.array_equal(full.list_sizes.cpu().numpy(), empty.list_sizes.cpu().numpy())
    for a, b in zip(index_codes(full), index_codes(empty)):
        assert np.array_equal(a, b)


def test_save_load_roundtrip(tmp_path, stream_shape):
    m = _mod()
    ds, qs, index = stream_shape
    path = str(tmp_path / "cos.idx")
    m.save(path, index)
    records = []
    with open(path, "rb") as f:
        size = os.fstat(f.fileno()).st_size
        while f.tell() < size:
            records.append(np.lib.format.read_array(f, allow_pickle=False))
    assert int(records[0]) == 4 and int(records[6]) == 2  # serialization version, metric = CosineExpanded
    again = m.load(path)
    for path_ in ("lut", "stream"):
        d1, i1 = _search(index, qs, 16, 10, path_)
        d2, i2 = _search(again, qs, 16, 10, path_)
        assert np.array_equal(i1, i2) and np.array_equal(d1, d2)


def test_build_is_deterministic():
    m = _mod()
    ds = torch.from_numpy(mixed_norm(30000, 128, 61)[0]).cuda()
    out = []
    for _ in range(2):
        index = m.build(m.IndexParams(n_lists=64, pq_dim=64, metric="cosine", kmeans_n_iters=10), ds)
        out.append((index.centers.cpu().numpy().copy(), index.pq_centers.cpu().numpy().copy()) + index_codes(index))
    for a, b in zip(*out):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("dtype", [np.float16, np.int8])
def test_narrow_dtypes_match_the_widened_fp32_index(dtype):
    """fp16 / int8 inputs are widened to fp32 on ingestion: the cosine index equals the one built from the widened values, and
    so do the search results (the distances are plain cosine distances, not rescaled by the int8 divisor)."""
    m = _mod()
    x, centers = mixed_norm(8000, 64, 71, n_centers=16)
    q, _ = mixed_norm(200, 64, 72, centers=centers)
    if dtype == np.int8:
        s = 100.0 / np.abs(x).max()
        x, q = np.clip(np.rint(x * s), -127, 127).astype(np.int8), np.clip(np.rint(q * s), -127, 127).astype(np.int8)
    else:
        x, q = x.astype(np.float16), q.astype(np.float16)
    params = m.IndexParams(n_lists=16, pq_dim=32, metric="cosine", kmeans_n_iters=10)
    narrow = m.build(params, torch.from_numpy(x).cuda())
    wide = m.build(params, torch.from_numpy(x.astype(np.float32)).cuda())
    assert np.array_equal(narrow.centers.cpu().numpy(), wide.centers.cpu().numpy())
    assert np.array_equal(narrow.pq_centers.cpu().numpy(), wide.pq_centers.cpu().numpy())
    for a, b in zip(index_codes(narrow), index_codes(wide)):
        assert np.array_equal(a, b)
    d1, i1 = _search(narrow, q, 8, 10, "auto")
    d2, i2 = _search(wide, q.astype(np.float32), 8, 10, "auto")
    # int8 rounding makes duplicate rows, whose exact ties the scan may keep in either order
    assert np.array_equal(d1, d2) and oracle.recall_with_ties(i1, d1, i2, d2, eps=0.0) == 1.0
    assert d1.max() <= 2.5  # cosine distances in [0, 2] up to PQ error


def test_refine_reaches_recall():
    from cuvs_b200.neighbors import refine
    m = _mod()
    ds, centers = mixed_norm(100000, 128, 81, n_centers=256)
    qs, _ = mixed_norm(500, 128, 82, centers=centers)
    dsg, qsg = torch.from_numpy(ds).cuda(), torch.from_numpy(qs).cuda()
    index = m.build(m.IndexParams(n_lists=256, pq_dim=64, metric="cosine", kmeans_n_iters=10), dsg)
    _, cand = _search(index, qs, 32, 40, "auto")
    rd, ri = refine(dsg, qsg, torch.from_numpy(cand).cuda(), k=10, metric="cosine")
    gd, gi = oracle.knn(ds, qs, 10, metric="cosine")
    assert oracle.recall(ri.cpu().numpy(), gi) >= 0.95
