"""GPU parity: cuvsIvfPq{Build,BuildPrecomputed,Search,Extend,Transform,Serialize} via the C ABI vs the oracle.

Element-wise: the library's own quantizers (centres, rotation, codebooks), list membership and codes are
read back through the reference's getter API and fed to the oracle's LUT-sum search
(oracle_ivf_pq_search); the LUT-scan kernel must reproduce it (fp32 LUT: same ids except at ties,
distances to 1e-5), the decoded-tile tensor-core path within PQ-noise-free tolerance 2e-3.
Recall floors follow cpp/tests/neighbors/ann_ivf_pq.cuh:978-1064 (>= 0.86 at pq_bits 8, defaults
4096 x 64, 1024 queries, k 32, n_lists 32)."""
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


def _search(index, qs, n_probes, k, path, **kw):
    m = _mod()
    os.environ["CUVS_B200_PQ_PATH"] = path
    d, i = m.search(m.SearchParams(n_probes=n_probes, **kw), index, torch.from_numpy(qs).cuda(), k)
    return d.cpu().numpy(), i.cpu().numpy()


@pytest.fixture(scope="module")
def small_index():
    m = _mod()
    ds = uniform(4096, 64, 1234, 0.1, 2.0)  # ann_ivf_pq.cuh:150-168 distribution
    qs = uniform(1024, 64, 4321, 0.1, 2.0)
    index = m.build(m.IndexParams(n_lists=32, pq_dim=32, pq_bits=8, kmeans_n_iters=20), torch.from_numpy(ds).cuda())
    return ds, qs, index


def test_index_shapes_and_packing(small_index):
    ds, qs, index = small_index
    assert (index.n_lists, index.dim, index.pq_dim, index.pq_len, index.pq_bits, len(index)) == (32, 64, 32, 2, 8, 4096)
    assert tuple(index.pq_centers.shape) == (32, 2, 256) and tuple(index.centers_padded.shape) == (32, 72)
    cp = index.centers_padded.cpu().numpy()
    np.testing.assert_allclose(cp[:, 64], (cp[:, :64] ** 2).sum(1), rtol=1e-5)  # |c|^2 column (ivf_pq_index.cu:78-80)
    offs, codes, ids = index_codes(index)
    assert sorted(ids.tolist()) == list(range(4096)) and codes.shape == (4096, 32)
    # codes really are the nearest codebook entries of the rotated residuals (transform == what is stored)
    m = _mod()
    labels, tcodes = m.transform(index, torch.from_numpy(ds[:512]).cuda())
    pos = {int(i): j for j, i in enumerate(ids)}
    stored = codes[[pos[i] for i in range(512)]]
    assert (tcodes.cpu().numpy() == stored).all()


@pytest.mark.parametrize("lut,dist,tol", [("f32", "f32", 1e-5), ("f16", "f32", 1e-5), ("fp8", "f32", 1e-5), ("f16", "f16", 2e-2)])
def test_lut_scan_matches_oracle(small_index, lut, dist, tol):
    ds, qs, index = small_index
    kw = {"lut_dtype": {"f32": np.float32, "f16": np.float16, "fp8": np.uint8}[lut],
          "internal_distance_dtype": {"f32": np.float32, "f16": np.float16}[dist]}
    d, i = _search(index, qs, 8, 32, "lut", **kw)
    rd, ri = pq_search(index, qs, 8, 32, "sqeuclidean", lut, dist)
    assert oracle.recall_with_ties(i, d, ri, rd, eps=max(tol, 1e-5)) >= 0.999
    if dist == "f32":
        same = i == ri
        assert same.mean() >= 0.99
        np.testing.assert_allclose(d[same], rd[same], rtol=tol, atol=tol)


def test_tensor_core_path_matches_lut_semantics(small_index):
    ds, qs, index = small_index
    d, i = _search(index, qs, 8, 32, "tc")
    rd, ri = pq_search(index, qs, 8, 32, "sqeuclidean")
    assert oracle.recall_with_ties(i, d, ri, rd, eps=2e-3) >= 0.995
    same = i == ri
    assert same.mean() >= 0.97
    np.testing.assert_allclose(d[same], rd[same], rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("path", ["lut", "tc"])
def test_reference_recall_floor(path):
    """ann_ivf_pq.cuh:26-43 defaults (4096 x 64, 1024 queries, k 32, n_lists 32, pq_dim auto = 64, trainset
    fraction 1.0, n_probes 20) with the :978-1064 floor for pq_bits = 8, evaluated like eval_neighbours
    (id match or distance within eps)."""
    m = _mod()
    ds = uniform(4096, 64, 1234, 0.1, 2.0)
    qs = uniform(1024, 64, 4321, 0.1, 2.0)
    index = m.build(m.IndexParams(n_lists=32, kmeans_trainset_fraction=1.0), torch.from_numpy(ds).cuda())
    assert index.pq_dim == 64 and index.pq_len == 1
    d, i = _search(index, qs, 20, 32, path)
    gd, gi = oracle.knn(ds, qs, 32)
    assert oracle.recall_with_ties(i, d, gi, gd, eps=1e-4 * 4) >= 0.86


@pytest.mark.parametrize("metric,path", [("inner_product", "lut"), ("inner_product", "tc"), ("euclidean", "tc")])
def test_other_metrics(metric, path):
    m = _mod()
    ds, centers = clustered(20000, 96, 3, n_centers=64)
    qs, _ = clustered(200, 96, 4, centers=centers)
    index = m.build(m.IndexParams(n_lists=64, pq_dim=48, metric=metric, kmeans_n_iters=10), torch.from_numpy(ds).cuda())
    d, i = _search(index, qs, 16, 10, path)
    rd, ri = pq_search(index, qs, 16, 10, metric)
    assert oracle.recall_with_ties(i, d, ri, rd, eps=3e-3) >= 0.99


def test_build_precomputed_extend_save_load(tmp_path, small_index):
    m = _mod()
    ds, qs, index = small_index
    params = m.IndexParams(n_lists=32, pq_dim=32, pq_bits=8)
    pre = m.build_precomputed(params, 64, index.pq_centers, index.centers, index.centers_rot, index.rotation_matrix)
    assert len(pre) == 0
    ids = np.arange(4096, dtype=np.int64) + 100
    m.extend(pre, torch.from_numpy(ds[:2000]).cuda(), torch.from_numpy(ids[:2000]).cuda())
    m.extend(pre, torch.from_numpy(ds[2000:]).cuda(), torch.from_numpy(ids[2000:]).cuda())
    assert len(pre) == 4096
    d1, i1 = _search(pre, qs[:100], 8, 10, "lut")
    d0, i0 = _search(index, qs[:100], 8, 10, "lut")
    assert ((i1 - 100) == i0).mean() >= 0.999  # same quantizers, same codes -> same answers
    m.save(str(tmp_path / "pq.idx"), pre)
    again = m.load(str(tmp_path / "pq.idx"))
    d2, i2 = _search(again, qs[:100], 8, 10, "lut")
    assert (i1 == i2).all() and (d1 == d2).all()


def test_refine_restores_exact_order(small_index):
    from cuvs_b200.neighbors import refine
    ds, qs, index = small_index
    d, i = _search(index, qs, 32, 32, "tc")
    rd, ri = refine(torch.from_numpy(ds).cuda(), torch.from_numpy(qs).cuda(), torch.from_numpy(i).cuda(), k=10)
    rd, ri = rd.cpu().numpy(), ri.cpu().numpy()
    # refined distances are the exact fp32 distances of the returned ids, sorted
    exact = ((qs[:, None, :] - ds[ri]) ** 2).sum(-1)
    np.testing.assert_allclose(rd, exact, rtol=1e-5, atol=1e-5)
    assert (np.diff(rd, axis=1) >= 0).all()
    gd, gi = oracle.knn(ds, qs, 10)
    assert oracle.recall(ri, gi) >= 0.95


def test_massive_ties_take_the_merge_fallback():
    """Thousands of exact duplicates: every candidate of every probe ties at the pruning bound, so the per-query merge
    cannot filter (more survivors than its buffer) and must fall back to its k-round selection; still k distinct ids,
    all at the same distance, and a far-away row never shows up."""
    m = _mod()
    rng = np.random.default_rng(3)
    base = rng.standard_normal(64).astype(np.float32)
    ds = np.tile(base, (6000, 1))
    ds[-1] += 50.0                                     # one outlier
    qs = np.tile(base, (7, 1)) + 0.01
    os.environ["CUVS_B200_PQ_PATH"] = "tc"
    index = m.build(m.IndexParams(n_lists=4, pq_dim=32, kmeans_n_iters=5), torch.from_numpy(ds).cuda())
    d, i = m.search(m.SearchParams(n_probes=4), index, torch.from_numpy(qs).cuda(), 10)
    d, i = d.cpu().numpy(), i.cpu().numpy()
    assert all(len(set(r.tolist())) == 10 for r in i) and (i >= 0).all() and (i < 5999).all()
    assert np.allclose(d, d[:, :1], rtol=0, atol=1e-3 * max(1.0, float(np.abs(d).max())))


def test_wide_vectors_take_the_streamed_scan():
    """dim 192 > 128: rot_dim = 192 -> the scan streams the query k-blocks next to the list k-blocks; same LUT semantics."""
    m = _mod()
    ds = uniform(6000, 192, 11, 0.1, 2.0)
    qs = uniform(200, 192, 12, 0.1, 2.0)
    index = m.build(m.IndexParams(n_lists=16, pq_dim=96, kmeans_n_iters=10, kmeans_trainset_fraction=1.0), torch.from_numpy(ds).cuda())
    assert index.pq_len == 2
    d, i = _search(index, qs, 8, 10, "tc")
    rd, ri = pq_search(index, qs, 8, 10, "sqeuclidean")
    assert oracle.recall_with_ties(i, d, ri, rd, eps=2e-3) >= 0.99
    gd, gi = oracle.knn(ds, qs, 10)
    assert oracle.recall(i, gi) >= 0.6  # iid-uniform 192-d data, 8 of 16 lists, 2 dims per code: PQ noise, not the scan


# ---------------------------------------------------------------------------------------------------------------
# The reduced-precision request (lut_dtype f16 / u8) is what bench.py times: a ONE-pass tensor-core scan whose query-side
# residual is rounded to bf16 (8-bit significand) where the reference rounds the LUT entries to fp16 / fp_8bit<5>.  These
# tests pin that path against the oracle's LUT search run with the matching lut_dtype, BEFORE any refine:
#   * recall_with_ties (eval_neighbours, ann_utils.cuh:257-289) at eps = 1e-2 relative: bf16 rounding of r perturbs
#     |r - y|^2 by <= 2 |r - y| |r| 2^-9 ~ 4e-3 |r - y|^2 when |r| ~ |r - y| (the fp16 LUT's own error is ~2^-11 per entry,
#     fp_8bit<5>'s ~2^-4: ours sits between the two);
#   * the reference's own acceptance floors for reduced LUTs against EXACT ground truth
#     (cpp/tests/neighbors/ann_ivf_pq.cuh:978-1064: min_recall 0.84-0.86 at pq_bits 8, fp16 / fp8 LUT variants).
@pytest.mark.parametrize("metric", ["sqeuclidean", "inner_product"])
@pytest.mark.parametrize("lut", ["f16", "fp8"])
@pytest.mark.parametrize("dim,pq_dim", [(128, 64), (192, 96)])
def test_one_pass_scan_matches_reduced_lut_oracle(metric, lut, dim, pq_dim):
    m = _mod()
    ds, centers = clustered(30000, dim, 5, n_centers=48)
    qs, _ = clustered(256, dim, 6, centers=centers)
    index = m.build(m.IndexParams(n_lists=48, pq_dim=pq_dim, metric=metric, kmeans_n_iters=10), torch.from_numpy(ds).cuda())
    kw = {"lut_dtype": {"f16": np.float16, "fp8": np.uint8}[lut]}
    d, i = _search(index, qs, 12, 10, "tc", **kw)
    # against the oracle's LUT search with the SAME reduced lut_dtype.  fp16 LUT entries carry ~2^-11 relative error: eps 1e-2.
    # fp_8bit<5> entries carry ~2^-4 (signed variant for inner product: 2^-3) and the 64 entries of a score add up, so the
    # reference's own fp8 answer sits several percent away from the exact LUT sum; ours (bf16 residual, exact codebook) is the
    # more accurate of the two and is compared at the fp8 format's error scale.
    rd, ri = pq_search(index, qs, 12, 10, metric, lut, "f32")
    # (floor 0.975, not 0.99: the clustered test data has ~1000 near-equidistant neighbours per point, so a 0.5 % score error
    # flips ranks across the k-th position, and a flipped row only counts when its distance lands within eps of a true one;
    # the k-means build is not bit-reproducible either, so the figure moves by ~0.5 % between runs)
    assert oracle.recall_with_ties(i, d, ri, rd, eps=1e-2 if lut == "f16" else 8e-2) >= 0.975
    # ... and against the fp32-LUT answer it is at least as close as the reference's reduced LUTs are allowed to be
    fd, fi = pq_search(index, qs, 12, 10, metric, "f32", "f32")
    assert oracle.recall_with_ties(i, d, fi, fd, eps=1e-2) >= 0.975
    same = i == fi
    assert same.mean() >= (0.9 if metric == "sqeuclidean" else 0.75)  # (inner-product scores of ~150 with near-ties: ranks swap)
    np.testing.assert_allclose(d[same], fd[same], rtol=2e-2, atol=2e-2)


@pytest.mark.parametrize("lut", ["f16", "fp8"])
def test_one_pass_scan_reference_recall_floor(lut):
    """ann_ivf_pq.cuh:26-43 defaults with the fp16 / fp8 LUT variants of :978-1064 (floor 0.84-0.86), exact ground truth."""
    m = _mod()
    ds = uniform(4096, 64, 1234, 0.1, 2.0)
    qs = uniform(1024, 64, 4321, 0.1, 2.0)
    index = m.build(m.IndexParams(n_lists=32, kmeans_trainset_fraction=1.0), torch.from_numpy(ds).cuda())
    d, i = _search(index, qs, 20, 32, "tc", lut_dtype={"f16": np.float16, "fp8": np.uint8}[lut])
    gd, gi = oracle.knn(ds, qs, 32)
    assert oracle.recall_with_ties(i, d, gi, gd, eps=4e-4) >= 0.84


# ---------------------------------------------------------------------------------------------------------------
# The code-streaming scan (scan_pq.cu) serves pq_bits 8 / pq_len 2 / pq_dim 32|64 indexes.  Every work-item width
# (32 / 64 / 128 probing queries as the MMA's N side), both operand depths (rot_dim 64 -> one k-block, 128 -> two), both
# candidate-list sizes (k <= 16 -> 16 slots, k <= 32 -> 32) and both pass counts are pinned to the oracle's LUT search.
@pytest.fixture(scope="module")
def stream_index_128():
    m = _mod()
    ds, centers = clustered(40000, 128, 15, n_centers=64)
    qs, _ = clustered(512, 128, 16, centers=centers)
    index = m.build(m.IndexParams(n_lists=64, pq_dim=64, kmeans_n_iters=10), torch.from_numpy(ds).cuda())
    return ds, qs, index


@pytest.mark.parametrize("group", [32, 64, 128])
@pytest.mark.parametrize("which,k,lut", [("d64", 10, "f16"), ("d64", 32, "f16"), ("d128", 10, "f16"), ("d128", 32, "f32"), ("d128", 10, "f32")])
def test_streamed_scan_all_shapes(small_index, stream_index_128, group, which, k, lut):
    ds, qs, index = small_index if which == "d64" else stream_index_128
    assert index.streamed, "pq_bits 8 / pq_len 2 / pq_dim 32|64 must be served by the code-streaming scan"
    os.environ["CUVS_B200_PQ_GROUP"] = str(group)
    try:
        kw = {} if lut == "f32" else {"lut_dtype": np.float16}
        d, i = _search(index, qs, 8, k, "stream", **kw)
    finally:
        del os.environ["CUVS_B200_PQ_GROUP"]
    rd, ri = pq_search(index, qs, 8, k, "sqeuclidean", lut, "f32")
    eps = 2e-3 if lut == "f32" else 1e-2
    assert oracle.recall_with_ties(i, d, ri, rd, eps=eps) >= (0.99 if lut == "f32" else 0.975)
    # returned ids are unique per query and really belong to the probed lists' rows (no padding rows, no garbage)
    assert all(len(set(r.tolist())) == k for r in i) and (i >= 0).all() and (i < len(ds)).all()


@pytest.mark.parametrize("k", [40, 64])
def test_streamed_scan_k_up_to_64(stream_index_128, k):
    """k in 33..64 (refine_ratio x k candidate generation): 64 kept entries per (query, probe), 128-entry buffers, 32-query work
    items — same answers as the reference-formulation LUT kernel and the oracle."""
    ds, qs, index = stream_index_128
    assert index.streamed
    d, i = _search(index, qs, 8, k, "stream", lut_dtype=np.float16)
    rd, ri = pq_search(index, qs, 8, k, "sqeuclidean", "f16", "f32")
    assert oracle.recall_with_ties(i, d, ri, rd, eps=1e-2) >= 0.975
    assert all(len(set(r.tolist())) == k for r in i) and (i >= 0).all() and (i < len(ds)).all()
    d2, i2 = _search(index, qs, 8, k, "lut", lut_dtype=np.float16)
    same = np.mean([len(set(a) & set(b)) / float(k) for a, b in zip(i, i2)])
    assert same >= 0.97, same
    # the 2-pass scan (fp32 LUT semantics) through the same wide buffers
    d3, i3 = _search(index, qs, 8, k, "stream")
    rd3, ri3 = pq_search(index, qs, 8, k, "sqeuclidean", "f32", "f32")
    assert oracle.recall_with_ties(i3, d3, ri3, rd3, eps=2e-3) >= 0.99


def test_streamed_index_keeps_no_decoded_rows():
    """Beyond the decoded-row budget (here: 0) the code stream is the whole index: codes + half-norms + ids per vector."""
    m = _mod()
    ds, centers = clustered(40000, 128, 15, n_centers=64)
    os.environ["CUVS_B200_PQ_DECODED_BUDGET_MB"] = "0"
    try:
        index = m.build(m.IndexParams(n_lists=64, pq_dim=64, kmeans_n_iters=10), torch.from_numpy(ds).cuda())
    finally:
        del os.environ["CUVS_B200_PQ_DECODED_BUDGET_MB"]
    assert index.streamed
    # code stream (68 B) + ids (8 B) per vector, padded lists, + quantizers: well under the 256 B/vector of decoded rows
    assert index.device_bytes < len(ds) * 200


def test_small_index_dense_batch_takes_the_decoded_row_cache(stream_index_128):
    """A small index also caches decoded rows; a batch with >= 128 probing queries per list is served from them, a sparse one
    from the code stream: both must agree with each other (same arithmetic: bf16 residual x bf16 codebook rows)."""
    ds, qs, index = stream_index_128
    assert index.streamed and index.device_bytes > len(ds) * 256   # the cache is there
    q = np.concatenate([qs] * 4)[:1100]                             # 1100 queries x 8 probes / 64 lists = 137 per list: dense
    d_dense, i_dense = _search(index, q, 8, 10, "auto", lut_dtype=np.float16)
    d_str, i_str = _search(index, q, 8, 10, "stream", lut_dtype=np.float16)
    same = np.mean([len(set(a) & set(b)) / 10.0 for a, b in zip(i_dense, i_str)])
    assert same >= 0.995, same
    rd, ri = pq_search(index, q, 8, 10, "sqeuclidean", "f16", "f32")
    assert oracle.recall_with_ties(i_dense, d_dense, ri, rd, eps=1e-2) >= 0.975


def test_streamed_scan_empty_and_tiny_lists():
    """n_lists close to n: lists of 0..3 rows, every tile almost entirely padding; probes of empty lists are dropped."""
    m = _mod()
    ds = uniform(300, 64, 5, -1, 1)
    qs = uniform(40, 64, 6, -1, 1)
    index = m.build(m.IndexParams(n_lists=128, pq_dim=32, kmeans_n_iters=4, kmeans_trainset_fraction=1.0), torch.from_numpy(ds).cuda())
    assert index.streamed
    d, i = _search(index, qs, 128, 10, "stream", lut_dtype=np.float16)
    rd, ri = pq_search(index, qs, 128, 10, "sqeuclidean", "f16", "f32")
    assert oracle.recall_with_ties(i, d, ri, rd, eps=1e-2) >= 0.99


def test_streamed_scan_is_invariant_to_the_work_item_width(stream_index_128):
    """The per-(query, probe) candidate lists are exact top-KC selections, so the final answer cannot depend on how many probing
    queries share a work item: 32-, 64- and 128-wide items must return the same neighbours (a lost candidate shows up here
    long before it moves a recall number)."""
    ds, qs, index = stream_index_128
    res = {}
    for g in (32, 64, 128):
        os.environ["CUVS_B200_PQ_GROUP"] = str(g)
        try:
            res[g] = _search(index, qs, 8, 10, "stream", lut_dtype=np.float16)
        finally:
            del os.environ["CUVS_B200_PQ_GROUP"]
    for g in (64, 128):
        same = (res[g][1] == res[32][1]).mean()
        assert same >= 0.999, (g, same)
        np.testing.assert_allclose(res[g][0], res[32][0], rtol=1e-5, atol=1e-5)


def test_build_and_search_are_identical_from_run_to_run():
    """Coarse centres and PQ codebooks are trained with fixed-point sums: two builds from the same data hold the same quantizers
    and return the same neighbours and distances to the bit."""
    m = _mod()
    ds = torch.from_numpy(uniform(30000, 64, 77, 0.1, 2.0)).cuda()
    qs = torch.from_numpy(uniform(500, 64, 78, 0.1, 2.0)).cuda()
    out = []
    for _ in range(2):
        index = m.build(m.IndexParams(n_lists=64, pq_dim=32, pq_bits=8, kmeans_n_iters=10), ds)
        d, i = m.search(m.SearchParams(n_probes=16), index, qs, 10)
        out.append((index.centers.clone(), index.pq_centers.clone(), d.clone(), i.clone()))
    for a, b in zip(*out):
        assert torch.equal(a, b)
