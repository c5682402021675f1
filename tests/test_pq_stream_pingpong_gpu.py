"""The code-streaming IVF-PQ scan's ping-pong consumer (scan_pq.cu, 64-query work items, one pass).

The two MMA warpgroups own alternate 128-row tiles of the running tile sequence, and each keeps its own per-query thresholds
and candidate buffers.  A warpgroup's buffer holds only rows of its own earlier tiles, but the other warpgroup's buffer may
already hold rows of later tiles, which lose exact ties.  So a row must survive a tie with the other warpgroup's threshold,
and the read-out ranks the union of both buffers.  The 32-query items keep the rows-on-M consumer with one buffer per query,
so with exact per-(query, probe) selections both must return the same neighbours and distances, ties included.
"""
import numpy as np
import pytest
import torch

from tests.util import clustered

pytestmark = pytest.mark.gpu


def _search(monkeypatch, index, qs, k, group, n_probes, bound=True, cap=None):
    from cuvs_b200.neighbors import ivf_pq
    monkeypatch.setenv("CUVS_B200_PQ_PATH", "stream")
    monkeypatch.setenv("CUVS_B200_PQ_GROUP", str(group))
    if bound:
        monkeypatch.delenv("CUVS_B200_PQ_NO_BOUND", raising=False)
    else:
        monkeypatch.setenv("CUVS_B200_PQ_NO_BOUND", "1")
    if cap is None:
        monkeypatch.delenv("CUVS_B200_PQ_CAP", raising=False)
    else:
        monkeypatch.setenv("CUVS_B200_PQ_CAP", str(cap))
    d, i = ivf_pq.search(ivf_pq.SearchParams(n_probes=n_probes, lut_dtype=np.float16), index, torch.from_numpy(qs).cuda(), k)
    return d.cpu().numpy(), i.cpu().numpy()


def _assert_same(a, b, ds=None):
    """Identical neighbours and distances.  With `ds`, a neighbour may instead be an exact copy of the other one: the pruning
    bound drops a row whose score equals another item's published k-th best, and which copy that is depends on the order in
    which the items of one query run (rows-on-M kernels alike)."""
    (da, ia), (db, ib) = a, b
    np.testing.assert_array_equal(da, db)
    if ds is None:
        np.testing.assert_array_equal(ia, ib)
    else:
        diff = ia != ib
        assert (ds[ia[diff]] == ds[ib[diff]]).all()


@pytest.fixture(scope="module")
def dup_index():
    """Every vector 16 times, shuffled: the copies share a list and a code, so their scores are bit-equal, and they are
    spread over the list's ~10 tiles, i.e. over both warpgroups.  (Not more: when more than k copies of the k-th score fall
    into ONE tile and that tile overflows a buffer, the re-test after compaction drops some of them whatever their
    positions, in every consumer of this kernel, so no two consumers need agree on which copies are returned.)"""
    from cuvs_b200.neighbors import ivf_pq
    base, centers = clustered(2500, 128, 41, n_centers=32)
    ds = np.repeat(base, 16, axis=0)[np.random.default_rng(42).permutation(16 * len(base))]
    qs, _ = clustered(512, 128, 43, centers=centers)
    index = ivf_pq.build(ivf_pq.IndexParams(n_lists=32, pq_dim=64, kmeans_n_iters=10), torch.from_numpy(ds).cuda())
    assert index.streamed
    return ds, qs, index


@pytest.mark.parametrize("bound", [True, False])
@pytest.mark.parametrize("k", [10, 32])
def test_exact_ties_match_the_rows_on_m_consumer(monkeypatch, dup_index, k, bound):
    ds, qs, index = dup_index
    ref = _search(monkeypatch, index, qs, k, 32, 8, bound)
    # the copies really tie: most queries see one score several times among their k results
    assert np.mean([len(np.unique(r)) < k for r in ref[0]]) > 0.5
    _assert_same(_search(monkeypatch, index, qs, k, 64, 8, bound), ref, ds if bound else None)


N_TILES = 6


def _tie_layout(kc):
    """Rows of one 6-tile list, by kind: 0 = a copy of v, 1 = near v (closer than any other distinct row), 2 = mid, 3 = far.
    Tiles 0 and 1 (warpgroups 0 and 1): mid rows, which set both warpgroups' thresholds.  Tile 2 (warpgroup 0): one copy of v
    and 127 near rows, all hits, so its buffers overflow and are compacted round after round.  Tile 3 (warpgroup 1): kc - 1
    copies among far rows, which miss.  Tile 4 (warpgroup 0): far rows.  Tile 5 (warpgroup 1): copies only.  Without the
    pruning bound kth = KC = kc, so a (query, probe) pair's top kth is tile 2's copy and tile 3's, all at v's score.
    Warpgroup 1, with little to filter, reaches kth entries at that score with tile 5's copies while warpgroup 0 is still
    re-testing tile 2's overflow: its threshold then equals the score of tile 2's copy, and a strict `t > thr[other]` loses
    that copy."""
    kind = np.full(128 * N_TILES, 2)
    kind[256:384] = 1
    kind[300] = 0
    kind[384:512] = 3
    kind[384 + 4 * np.arange(kc - 1)] = 0
    kind[512:640] = 3
    kind[640:] = 0
    return kind


@pytest.fixture(scope="module", params=[16, 32], ids=["KC16", "KC32"])
def tie_index(request):
    from cuvs_b200.neighbors import ivf_pq
    kc = request.param
    dim, n_lists, n = 128, 8, 128 * N_TILES
    train, _ = clustered(8000, dim, 61, n_centers=n_lists)
    index = ivf_pq.build(ivf_pq.IndexParams(n_lists=n_lists, pq_dim=64, kmeans_n_iters=10, add_data_on_build=False),
                         torch.from_numpy(train).cuda())
    centers = index.centers.cpu().numpy()[:, :dim]
    sep = min(np.linalg.norm(centers[a] - centers[b]) for a in range(n_lists) for b in range(a))
    sigma = min(0.25, 0.1 * sep / np.sqrt(dim))
    rng = np.random.default_rng(62)
    kind = _tie_layout(kc)
    spread = np.array([0.0, 1.5, 2.2, 3.0])[kind][:, None] * sigma  # distance of each kind of row from v, in sigma
    blocks, qs = [], []
    for lab in range(n_lists):  # block `lab`: row i is meant for row i of list `lab`; id = n lab + i
        v = centers[lab] + sigma * rng.standard_normal(dim)
        blocks.append((v + spread * rng.standard_normal((n, dim))).astype(np.float32))
        qs.append(v + 0.05 * sigma * rng.standard_normal((64, dim)))
    qs = np.concatenate(qs).astype(np.float32)
    # one extend per tile, so that every row lands in its tile (the order inside one extend's share of a list is not pinned)
    for t in range(N_TILES):
        rows = np.concatenate([b[128 * t:128 * (t + 1)] for b in blocks])
        ids = np.concatenate([n * lab + 128 * t + np.arange(128) for lab in range(n_lists)])
        ivf_pq.extend(index, torch.from_numpy(rows).cuda(), torch.from_numpy(ids).cuda())
    assert index.streamed
    expect = []
    for lab in range(n_lists):
        order = index.list_indices(lab).cpu().numpy()
        assert len(order) == n and ((order - n * lab) // 128 == np.arange(n) // 128).all()
        expect.append([i for i in order if kind[i - n * lab] == 0])  # v's copies in list order: tile 2's, then tile 3's
    return kc, qs, index, np.array(expect)


def test_ties_with_later_rows_of_the_other_warpgroup(monkeypatch, tie_index):
    """Group 64 returns exactly the earliest copies, as group 32 does (no pruning bound, small buffers: many overflows)."""
    kc, qs, index, v_ids = tie_index
    k = 10 if kc == 16 else 32
    expect = v_ids[np.arange(len(qs)) // 64, :k]  # query j probes list j // 64 only
    for group in (32, 64):
        d, i = _search(monkeypatch, index, qs, k, group, 1, bound=False, cap=kc + 8)
        assert (d == d[:, :1]).all()  # every returned row is a copy of v
        np.testing.assert_array_equal(i, expect)


def test_candidate_cap_is_per_warpgroup(monkeypatch, capfd, tie_index):
    """CUVS_B200_PQ_CAP sets each warpgroup's buffer: the launch reports the cap, and shared memory grows by two buffer sets
    of 64 queries x cap entries.  The smallest cap (KC + 8) and the largest that still leaves two code stages give the same
    answer."""
    kc, qs, index, _ = tie_index
    k = 10 if kc == 16 else 32
    monkeypatch.setenv("CUVS_B200_PQ_DEBUG", "1")
    res, fixed = [], set()
    for cap in (kc + 8, 53):
        capfd.readouterr()
        res.append(_search(monkeypatch, index, qs, k, 64, 1, bound=False, cap=cap))
        line = [ln for ln in capfd.readouterr().err.splitlines() if ln.startswith("[pq_stream_scan] NQ=64 ")][-1]
        f = dict(kv.split("=") for kv in line.split()[1:] if "=" in kv)
        assert int(f["cap"]) == cap and int(f["KC"]) == kc and int(f["PASSES"]) == 1 and int(f["cstages"]) >= 2
        fixed.add(int(f["smem"]) - int(f["cstages"]) * int(f["blk"]) - 2 * 64 * cap * 8)
    assert len(fixed) == 1  # the rest of the layout does not depend on the cap
    _assert_same(res[1], res[0])


@pytest.fixture(scope="module")
def odd_lists_index():
    """Lists of 1, 2, 3, 5, 128, 129, 130 and 257 rows between long ones: items of one, two and three tiles shift which
    warpgroup takes an item's first tile, and a one-tile item leaves one warpgroup without a tile."""
    from cuvs_b200.neighbors import ivf_pq
    dim, n_lists = 64, 16
    train, _ = clustered(8000, dim, 51, n_centers=n_lists, sigma=0.05)
    index = ivf_pq.build(ivf_pq.IndexParams(n_lists=n_lists, pq_dim=32, kmeans_n_iters=10, add_data_on_build=False),
                         torch.from_numpy(train).cuda())
    centers = index.centers.cpu().numpy()[:, :dim]
    # rows and queries stay well inside their centre's cell: noise of norm ~ 1/10 of the closest two centres' distance
    sep = min(np.linalg.norm(centers[a] - centers[b]) for a in range(n_lists) for b in range(a))
    sigma = 0.1 * sep / np.sqrt(dim)
    sizes = [1, 3, 129, 700, 1, 3, 129, 1000, 257, 2, 130, 1500, 1, 128, 384, 5]
    rng = np.random.default_rng(52)
    lab = np.concatenate([np.full(s, j) for j, s in enumerate(sizes)])
    rows = (centers[lab] + sigma * rng.standard_normal((len(lab), dim))).astype(np.float32)
    src = np.arange(0, len(lab) - 1, 7)
    src = src[lab[src] == lab[src + 1]]
    rows[src + 1] = rows[src]  # exact copies inside a list: ties
    rows = rows[rng.permutation(len(rows))]
    ivf_pq.extend(index, torch.from_numpy(rows).cuda(), torch.arange(len(rows), dtype=torch.int64).cuda())
    assert index.streamed
    qs = (centers[rng.integers(0, n_lists, 512)] + sigma * rng.standard_normal((512, dim))).astype(np.float32)
    return rows, qs, index, sizes


@pytest.mark.parametrize("bound", [True, False])
@pytest.mark.parametrize("k", [10, 32])
def test_odd_and_one_tile_items_match_the_rows_on_m_consumer(monkeypatch, odd_lists_index, k, bound):
    rows, qs, index, sizes = odd_lists_index
    assert sorted(index.list_sizes.cpu().numpy().tolist()) == sorted(sizes)
    ref = _search(monkeypatch, index, qs, k, 32, 8, bound)
    d, i = _search(monkeypatch, index, qs, k, 64, 8, bound)
    assert all(len(set(r.tolist())) == k for r in i) and (i >= 0).all() and (i < len(rows)).all()
    _assert_same((d, i), ref, rows if bound else None)
