"""The IVF coarse search never waits for the host (ivf_common.cu: coarse_select_fused).

With n_lists >= 4096 the coarse search keeps 16 candidates per (query, centre range, column half) and merges them under a
certificate; the queries whose certificate fails are packed on the device and take the dense scan + select_k, in launches
sized for a batch in which every query is flagged.  So an IVF-PQ search, and the refine behind it, can be captured in a
CUDA graph, and the flagged queries' probes are those of the dense path (CUVS_B200_COARSE_FUSED=0)."""
import os

import numpy as np
import pytest
import torch

from cuvs_b200.common.resources import Resources
from cuvs_b200.neighbors import ivf_flat, ivf_pq
from cuvs_b200.neighbors.refine import refine

pytestmark = pytest.mark.gpu

N_LISTS = 4096
PER_LIST = 32
BLOB_LISTS = 512  # for a 1000-query batch the fused scan splits the 4096 centres into 8 ranges of 512: range 0 is the blob


@pytest.fixture(scope="module")
def crowded():
    """Rows [0, 512 * 32) lie in one tight blob and the rest around the origin.  k-means starts from evenly spaced training
    rows, so most of centres 0..511 start, and stay, in the blob: most of a blob query's nearest centres lie in the first
    centre range, more of them than one range's two candidate lists of 16 can hold, and its certificate fails."""
    rng = np.random.default_rng(31)
    d = 64
    n = N_LISTS * PER_LIST
    p = np.zeros(d, np.float32)
    p[0] = 6.0
    blob = BLOB_LISTS * PER_LIST
    ds = rng.standard_normal((n, d)).astype(np.float32)
    ds[:blob] = p + 0.05 * rng.standard_normal((blob, d)).astype(np.float32)
    qs = rng.standard_normal((1000, d)).astype(np.float32)
    qs[:500] = p + 0.05 * rng.standard_normal((500, d)).astype(np.float32)
    return torch.from_numpy(ds).cuda(), torch.from_numpy(qs).cuda()


@pytest.fixture(scope="module")
def pq_index(crowded):
    ds, _ = crowded
    return ivf_pq.build(ivf_pq.IndexParams(n_lists=N_LISTS, pq_dim=32, kmeans_n_iters=4), ds)


def _crowded_queries(centers, qs, n_probes):
    """queries with more than 32 of their n_probes nearest centres (fp32) in the first range: more than its two lists of 16
    hold, so one of them is full of the query's n_probes best and the fused certificate cannot hold"""
    c = centers.float()
    dist = (c * c).sum(1)[None, :] - 2.0 * qs @ c.t()
    top = dist.topk(n_probes, dim=1, largest=False).indices
    return int(((top < BLOB_LISTS).sum(dim=1) > 32).sum().item())


def _with_env(name, value, fn):
    old = os.environ.get(name)
    os.environ[name] = value
    try:
        return fn()
    finally:
        if old is None:
            del os.environ[name]
        else:
            os.environ[name] = old


def test_search_and_refine_capture_in_a_cuda_graph(crowded, pq_index):
    """Capture fails on any host round trip (a stream synchronise is illegal while the stream captures).  The shapes take the
    fused coarse path (4096 lists) and the code-stream scan with its bound pre-pass (8-bit codes, pq_len 2, k <= 32, fewer
    than 128 queries per list on average).  The replay equals the eager calls bit for bit."""
    ds, qs = crowded
    assert pq_index.streamed
    nq, kc, k = qs.shape[0], 20, 10
    sp = ivf_pq.SearchParams(n_probes=64, lut_dtype=np.float16)
    assert nq * 64 < 128 * N_LISTS
    outs = [torch.empty((nq, kc), dtype=torch.int64, device="cuda"), torch.empty((nq, kc), dtype=torch.float32, device="cuda"),
            torch.empty((nq, k), dtype=torch.int64, device="cuda"), torch.empty((nq, k), dtype=torch.float32, device="cuda")]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        res = Resources()

        def run():
            ivf_pq.search(sp, pq_index, qs, kc, neighbors=outs[0], distances=outs[1], resources=res)
            refine(ds, qs, outs[0], indices=outs[2], distances=outs[3], resources=res)

        run()
        res.sync()
        eager = [t.clone() for t in outs]
        for t in outs:
            t.fill_(-7)
        res.sync()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            run()
    torch.cuda.synchronize()
    assert all(bool((t == -7).all()) for t in outs), "capture ran the search instead of recording it"
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(outs, eager):
        assert torch.equal(a, b)
    del graph


def test_flagged_queries_get_the_dense_probes(crowded, pq_index):
    ds, qs = crowded
    n_probes = 64
    assert _crowded_queries(pq_index.centers, qs, n_probes) >= 100
    sp = ivf_pq.SearchParams(n_probes=n_probes)

    def pq_search():
        d, i = ivf_pq.search(sp, pq_index, qs, 20)
        return d.cpu().numpy(), i.cpu().numpy()

    d1, i1 = pq_search()
    d0, i0 = _with_env("CUVS_B200_COARSE_FUSED", "0", pq_search)
    np.testing.assert_array_equal(i1, i0)
    np.testing.assert_array_equal(d1, d0)

    # IVF-Flat shares the coarse search; at k = 256 a query returns most of its probed lists' rows
    flat = ivf_flat.build(ivf_flat.IndexParams(n_lists=N_LISTS, kmeans_n_iters=4), ds)
    assert _crowded_queries(flat.centers, qs, n_probes) >= 100
    fsp = ivf_flat.SearchParams(n_probes=n_probes)
    for k in (10, 256):
        def flat_search():
            d, i = ivf_flat.search(fsp, flat, qs, k)
            return d.cpu().numpy(), i.cpu().numpy()

        d1, i1 = flat_search()
        d0, i0 = _with_env("CUVS_B200_COARSE_FUSED", "0", flat_search)
        np.testing.assert_array_equal(i1, i0)
        np.testing.assert_array_equal(d1, d0)


def test_large_batch_needs_no_dense_score_block():
    """The flagged queries' dense fallback runs in passes of bounded size: a 3M-query batch at 8192 lists (one batch: one
    probe per query) would need 98 GB for the dense [queries, centres] scores, more than the device has, and it searches in
    one piece, with the same results as small batches."""
    rng = np.random.default_rng(41)
    d, n_lists = 32, 8192
    ds = torch.from_numpy(rng.standard_normal((n_lists * 24, d)).astype(np.float32)).cuda()
    index = ivf_pq.build(ivf_pq.IndexParams(n_lists=n_lists, pq_dim=16, kmeans_n_iters=2), ds)
    nq = 3_000_000
    qs = torch.randn((nq, d), generator=torch.Generator(device="cuda").manual_seed(42), device="cuda")
    assert nq * n_lists * 4 > torch.cuda.get_device_properties(0).total_memory
    sp = ivf_pq.SearchParams(n_probes=1)
    d_all, i_all = ivf_pq.search(sp, index, qs, 1)
    for s0 in (0, nq - 1000):
        d_part, i_part = ivf_pq.search(sp, index, qs[s0:s0 + 1000], 1)
        assert torch.equal(i_part, i_all[s0:s0 + 1000]) and torch.equal(d_part, d_all[s0:s0 + 1000])
