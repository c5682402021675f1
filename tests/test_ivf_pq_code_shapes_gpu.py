"""IVF-PQ indexes without a code stream (pq_bits 4-7, per-cluster codebooks, pq_dim outside {32, 64}, pq_len != 2), against
the oracle.

Each index is built by the library; its own quantizers, list membership and codes (list_data, unpacked by
tests/ivf_pq_codes.py) are fed to the oracle's LUT-sum search with the index's pq_bits and codebook kind, and every search
path has to reproduce it:
  * the LUT kernel with fp32 / fp16 / fp_8bit<5> LUTs and fp32 / fp16 accumulation (the bars of
    test_ivf_pq_gpu.py::test_lut_scan_matches_oracle);
  * a tensor-core request at k 10, 32, 48 and 64 (the bar of test_tensor_core_path_matches_lut_semantics);
  * the k = 100 store path;
  * inner product and cosine on a per-cluster index and on a pq_len 3 index with rot_dim > dim.
Codes are also checked directly: transform() equals the stored codes, each is the nearest codebook entry of its rotated
residual, and extend, save / load, build_precomputed and conservative_memory_allocation do not change them or the search
output.  The recall floors of the reference's enum_variety cases (cpp/tests/neighbors/ann_ivf_pq.cuh:979-1013, defaults
:26-43) close the file."""
import numpy as np
import pytest
import torch

import oracle
from tests.ivf_oracle import check_rows, pq_search
from tests.ivf_pq_codes import index_codes, unpack_codes
from tests.util import uniform

pytestmark = pytest.mark.gpu

# name: (dim, build parameters)
SHAPES = {
    "bits4": (64, dict(pq_dim=32, pq_bits=4)),
    "bits5": (64, dict(pq_dim=32, pq_bits=5)),
    "bits6": (64, dict(pq_dim=32, pq_bits=6)),
    "bits7": (64, dict(pq_dim=32, pq_bits=7)),
    "cluster8": (64, dict(pq_dim=32, pq_bits=8, codebook_kind="cluster")),
    "cluster5": (64, dict(pq_dim=32, pq_bits=5, codebook_kind="cluster")),
    "cluster4": (64, dict(pq_dim=32, pq_bits=4, codebook_kind="cluster")),
    "d96_len4": (96, dict(pq_dim=24, pq_bits=6)),             # pq_dim % 16 != 0: the LUT kernel's unaligned code loads
    "d100_len3": (100, dict(pq_dim=34, pq_bits=8)),           # rot_dim 102 > dim
    "random_rotation": (64, dict(pq_dim=32, pq_bits=8, force_random_rotation=True)),
}
for _d in (1, 2, 3, 4, 5, 8, 15, 16, 17):  # the reference's small_dims / small_dims_per_cluster, pq_dim chosen by the library
    SHAPES[f"small{_d}"] = (_d, dict())
    SHAPES[f"small{_d}_cluster"] = (_d, dict(codebook_kind="cluster"))
MAIN = [s for s in SHAPES if not s.startswith("small")]

N, NQ, N_LISTS, N_PROBES = 4096, 256, 32, 8
_CACHE = {}


def _mod():
    from cuvs_b200.neighbors import ivf_pq
    return ivf_pq


def _params(shape, **kw):
    m = _mod()
    return m.IndexParams(n_lists=N_LISTS, kmeans_n_iters=10, kmeans_trainset_fraction=1.0, **{**SHAPES[shape][1], **kw})


def _data(shape):
    dim = SHAPES[shape][0]
    return uniform(N, dim, 1234 + dim, 0.1, 2.0), uniform(NQ, dim, 4321 + dim, 0.1, 2.0)


def _built(shape, metric="sqeuclidean"):
    """One index per (shape, metric), built once for the module."""
    key = (shape, metric)
    if key not in _CACHE:
        ds, qs = _data(shape)
        _CACHE[key] = (ds, qs, _mod().build(_params(shape, metric=metric), torch.from_numpy(ds).cuda()))
    return _CACHE[key]


def _per_cluster(shape):
    return SHAPES[shape][1].get("codebook_kind") == "cluster"


def _oracle(index, shape, qs, n_probes, k, metric="sqeuclidean", lut="f32", dist="f32"):
    return pq_search(index, qs, n_probes, k, metric, lut, dist, per_cluster=_per_cluster(shape))


def _search(monkeypatch, index, qs, n_probes, k, path, lut="f32", dist="f32"):
    m = _mod()
    monkeypatch.setenv("CUVS_B200_PQ_PATH", path)
    kw = {"lut_dtype": {"f32": np.float32, "f16": np.float16, "fp8": np.uint8}[lut],
          "internal_distance_dtype": {"f32": np.float32, "f16": np.float16}[dist]}
    d, i = m.search(m.SearchParams(n_probes=n_probes, **kw), index, torch.from_numpy(qs).cuda(), k)
    return d.cpu().numpy(), i.cpu().numpy()


def test_shapes_are_built_as_asked():
    """Every shape above builds (none is refused) and none of them is served by the code stream but random_rotation."""
    for shape in SHAPES:
        ds, qs, index = _built(shape)
        dim, kw = SHAPES[shape]
        assert index.dim == dim and len(index) == N
        assert index.pq_bits == kw.get("pq_bits", 8)
        if "pq_dim" in kw:
            assert index.pq_dim == kw["pq_dim"]
        assert index.pq_len == -(-dim // index.pq_dim)
        assert index.streamed == (shape == "random_rotation"), shape
        rot = index.rotation_matrix.cpu().numpy()
        assert rot.shape == (index.pq_dim * index.pq_len, dim)
        np.testing.assert_allclose(rot.T.astype(np.float64) @ rot, np.eye(dim), atol=1e-5)  # orthonormal columns
        n_books = N_LISTS if _per_cluster(shape) else index.pq_dim
        assert tuple(index.pq_centers.shape) == (n_books, index.pq_len, 1 << index.pq_bits)


@pytest.mark.parametrize("lut,dist,tol", [("f32", "f32", 1e-5), ("f16", "f32", 1e-5), ("fp8", "f32", 1e-5), ("f16", "f16", 2e-2)])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_lut_scan_matches_oracle(monkeypatch, shape, lut, dist, tol):
    ds, qs, index = _built(shape)
    d, i = _search(monkeypatch, index, qs, N_PROBES, 32, "lut", lut, dist)
    rd, ri = _oracle(index, shape, qs, N_PROBES, 32, lut=lut, dist=dist)
    check_rows(i, N)
    assert oracle.recall_with_ties(i, d, ri, rd, eps=tol) >= 0.999
    if dist == "f32":
        same = i == ri
        # (dims 1-5 hold many rows with equal codes in one list: a slot also agrees when its distance equals the oracle's)
        agree = same | (np.abs(d - rd) <= tol * np.maximum(1.0, np.abs(rd)))
        assert agree.mean() >= 0.99
        np.testing.assert_allclose(d[same], rd[same], rtol=tol, atol=tol)


@pytest.mark.parametrize("k", [10, 32, 48, 64])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_tensor_core_request_matches_oracle(monkeypatch, shape, k):
    ds, qs, index = _built(shape)
    d, i = _search(monkeypatch, index, qs, N_PROBES, k, "tc")
    rd, ri = _oracle(index, shape, qs, N_PROBES, k)
    check_rows(i, N)
    assert oracle.recall_with_ties(i, d, ri, rd, eps=2e-3) >= 0.995


@pytest.mark.parametrize("path", ["lut", "tc"])
@pytest.mark.parametrize("shape", MAIN)
def test_store_path_k100_matches_oracle(monkeypatch, shape, path):
    ds, qs, index = _built(shape)
    d, i = _search(monkeypatch, index, qs, N_PROBES, 100, path)
    rd, ri = _oracle(index, shape, qs, N_PROBES, 100)
    check_rows(i, N)
    if path == "lut" or not index.streamed:  # the LUT kernel's store mode
        assert oracle.recall_with_ties(i, d, ri, rd, eps=1e-5) >= 0.999
    else:  # the code stream's store epilogue (the bar of test_ivf_pq_large_k_gpu.py::test_stream_store_matches_oracle)
        assert oracle.recall_with_ties(i, d, ri, rd, eps=2e-3) >= 0.99


@pytest.mark.parametrize("path", ["lut", "tc"])
@pytest.mark.parametrize("metric", ["inner_product", "cosine"])
@pytest.mark.parametrize("shape", ["cluster8", "d100_len3"])
def test_other_metrics_match_oracle(monkeypatch, shape, metric, path):
    ds, qs, index = _built(shape, metric)
    for k in (10, 64):
        d, i = _search(monkeypatch, index, qs, N_PROBES, k, path)
        rd, ri = _oracle(index, shape, qs, N_PROBES, k, metric)
        check_rows(i, N)
        if path == "lut":
            assert oracle.recall_with_ties(i, d, ri, rd, eps=1e-5) >= 0.999
        else:  # (the decoded rows of an inner-product index hold c + y rounded to bf16: the bar of test_other_metrics)
            assert oracle.recall_with_ties(i, d, ri, rd, eps=3e-3) >= 0.99


@pytest.mark.parametrize("shape", list(SHAPES))
def test_transform_equals_stored_codes_and_nearest_entries(shape):
    """transform() of the first rows gives their list and their stored codes; each code is the codebook entry nearest to the
    row's rotated residual (float64, up to a near-tie)."""
    m = _mod()
    ds, qs, index = _built(shape)
    labels, packed = m.transform(index, torch.from_numpy(ds[:512]).cuda())
    labels = labels.cpu().numpy().astype(np.int64)
    codes = unpack_codes(packed.cpu().numpy(), index.pq_dim, index.pq_bits)
    offs, stored, ids = index_codes(index)
    pos = np.empty(N, np.int64)
    pos[ids] = np.arange(N)
    rows = pos[np.arange(512)]
    assert (np.searchsorted(offs, rows, side="right") - 1 == labels).all(), "transform's labels are not the rows' lists"
    assert (codes == stored[rows]).all(), "transform's codes are not the stored codes"
    rot = index.rotation_matrix.cpu().numpy().astype(np.float64)
    cr = index.centers_rot.cpu().numpy().astype(np.float64)
    pq = index.pq_centers.cpu().numpy().astype(np.float64)                  # [books, pq_len, 2^bits]
    pq_dim, pq_len = index.pq_dim, index.pq_len
    resid = (ds[:512].astype(np.float64) @ rot.T - cr[labels]).reshape(512, pq_dim, pq_len)
    books = pq[labels][:, None].repeat(pq_dim, 1) if _per_cluster(shape) else pq[None].repeat(512, 0)
    err = ((resid[:, :, :, None] - books) ** 2).sum(2)                       # [512, pq_dim, 2^bits]
    chosen = np.take_along_axis(err, codes[:, :, None].astype(np.int64), 2)[..., 0]
    assert (chosen <= err.min(2) + 1e-4 * np.maximum(1.0, err.min(2))).all(), "a code is not its subspace's nearest entry"


@pytest.mark.parametrize("shape", MAIN)
def test_extend_in_two_chunks_equals_build(shape):
    m = _mod()
    ds, qs, index = _built(shape)
    empty = m.build(_params(shape, add_data_on_build=False), torch.from_numpy(ds).cuda())
    m.extend(empty, torch.from_numpy(ds[:1500]).cuda(), None)
    m.extend(empty, torch.from_numpy(ds[1500:]).cuda(), None)
    assert torch.equal(empty.pq_centers, index.pq_centers) and torch.equal(empty.centers, index.centers)
    o0, c0, i0 = index_codes(index)
    o1, c1, i1 = index_codes(empty)
    assert (o0 == o1).all() and (i0 == i1).all() and (c0 == c1).all()


@pytest.mark.parametrize("shape", MAIN)
def test_save_load_gives_identical_search(monkeypatch, tmp_path, shape):
    m = _mod()
    ds, qs, index = _built(shape)
    m.save(str(tmp_path / "pq.idx"), index)
    again = m.load(str(tmp_path / "pq.idx"))
    for path, k in (("lut", 32), ("tc", 10), ("tc", 64), ("lut", 100)):
        d0, i0 = _search(monkeypatch, index, qs, N_PROBES, k, path)
        d1, i1 = _search(monkeypatch, again, qs, N_PROBES, k, path)
        assert (i0 == i1).all() and (d0 == d1).all(), (path, k)


@pytest.mark.parametrize("shape", ["cluster8", "cluster5", "cluster4", "small17_cluster"])
def test_build_precomputed_per_cluster_gives_the_same_codes(shape):
    m = _mod()
    ds, qs, index = _built(shape)
    pre = m.build_precomputed(_params(shape), index.dim, index.pq_centers, index.centers, index.centers_rot, index.rotation_matrix)
    m.extend(pre, torch.from_numpy(ds).cuda(), None)
    o0, c0, i0 = index_codes(index)
    o1, c1, i1 = index_codes(pre)
    assert (o0 == o1).all() and (i0 == i1).all() and (c0 == c1).all()


@pytest.mark.parametrize("shape", ["bits5", "cluster8", "d96_len4", "random_rotation"])
def test_conservative_index_serves_a_tensor_core_request_with_the_lut_kernel(monkeypatch, shape):
    """conservative_memory_allocation keeps neither decoded rows nor a code stream: a tc request gives the LUT kernel's output,
    which is that of the same index built without it."""
    m = _mod()
    ds, qs, index = _built(shape)
    cons = m.build(_params(shape, conservative_memory_allocation=True), torch.from_numpy(ds).cuda())
    assert not cons.streamed and not cons.has_decoded_rows
    for k in (10, 48, 64):
        d0, i0 = _search(monkeypatch, cons, qs, N_PROBES, k, "tc")
        d1, i1 = _search(monkeypatch, cons, qs, N_PROBES, k, "lut")
        d2, i2 = _search(monkeypatch, index, qs, N_PROBES, k, "lut")
        assert (i0 == i1).all() and (d0 == d1).all()
        assert (i0 == i2).all() and (d0 == d2).all()


@pytest.mark.parametrize("path", ["lut", "tc"])
@pytest.mark.parametrize("kind,pq_bits,floor", [("cluster", 4, 0.79), ("cluster", 5, 0.83), ("subspace", 6, 0.84),
                                                ("subspace", 7, 0.85), ("cluster", 8, 0.86)])
def test_enum_variety_recall_floor(monkeypatch, kind, pq_bits, floor, path):
    """ann_ivf_pq.cuh:26-43 defaults (4096 x 64, 1024 queries, k 32, n_lists 32, n_probes 20, pq_dim auto = 64, trainset
    fraction 1.0) with the enum_variety floors, against exact ground truth as eval_neighbours counts it."""
    m = _mod()
    ds = uniform(4096, 64, 1234, 0.1, 2.0)
    qs = uniform(1024, 64, 4321, 0.1, 2.0)
    index = m.build(m.IndexParams(n_lists=32, kmeans_trainset_fraction=1.0, pq_bits=pq_bits, codebook_kind=kind),
                    torch.from_numpy(ds).cuda())
    assert index.pq_dim == 64 and index.pq_bits == pq_bits
    d, i = _search(monkeypatch, index, qs, 20, 32, path)
    gd, gi = oracle.knn(ds, qs, 32)
    rec = oracle.recall_with_ties(i, d, gi, gd, eps=1e-4 * 4)
    assert rec >= floor, rec
