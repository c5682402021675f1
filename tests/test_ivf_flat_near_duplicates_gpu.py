"""IVF-Flat against the oracle on near-duplicate rows.

The fine scan ranks a pair's rows by a one-pass bf16 score of residuals, bf16(q - c) . bf16(x - c), and only the best few
(kc2) reach the exact fp32 re-score.  Where many rows sit within that score's error of a query's k-th neighbour, the bf16
ranking alone would drop true neighbours; the search has to notice (its certificate) and score those queries exactly.  These
families put many rows there:

  * `dups<R>`: 300 clustered base rows (8 centres ~ N(0, 1), sigma 0.25), each repeated R times with N(0, eps^2) jitter
    (eps 1e-3; `e4`: 1e-4).  Queries are base rows plus N(0, 0.1^2), every fourth one a base row itself.
  * `ladder`: per query, 300 rows at squared distances 1 + i * 2e-6 (i < 300, in shuffled order), far below the bf16 score's
    error, so the k-th boundary of every k <= 300 falls inside the ladder.
  * `dups48` shifted by 10 and by 100 in every component.
  * `u8`: uint8 rows, half of the copies exact and half one step away in three components: integer distances tie exactly.

Every index takes the generating centres as its lists (set_centers, then extend), so that list membership does not depend on
k-means.  Results are held to the oracle with assert_same_answer: distances bit for bit, ids outside the last tie group."""
import numpy as np
import pytest
import torch

import oracle
from tests.ivf_oracle import assert_same_answer, certain_probes, check_rows, flat_search
from tests.util import clustered, last_flagged

pytestmark = pytest.mark.gpu

D, NQ, N_BASE = 128, 64, 300
KS = [1, 10, 32, 48, 64, 100, 256, 1024, 2048]
FAMILIES = ["dups48", "dups128", "dups128e4", "ladder", "dups48_shift10", "dups48_shift100", "u8"]
# every list probed, except on dups48 / dups128 (4 of 8 lists, on the queries whose probe set is certain)
N_PROBES = {"dups48": 4, "dups128": 4}
BIG_NQ = 600

_DATA = {}


def _dups(reps, eps, shift=0.0, nq=NQ, seed=81):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((8, D)).astype(np.float32)
    base, _ = clustered(N_BASE, D, seed + 1, centers=centers)
    x = np.repeat(base, reps, axis=0) + eps * rng.standard_normal((N_BASE * reps, D))
    pick = rng.choice(N_BASE, nq, replace=nq > N_BASE)
    qs = base[pick] + 0.1 * rng.standard_normal((nq, D))
    qs[::4] = base[pick[::4]]
    f = lambda a: (a + shift).astype(np.float32)  # noqa: E731
    return f(x), f(qs), f(centers)


def _ladder(seed=85, n_q=40, rungs=300):
    """Query j sits at 4 N(0, 1); its rows at q_j + sqrt(1 + i 2e-6) u_ij with unit u_ij = 0.7 v_j + 0.71 g_ij (normalised),
    so the list centre (their mean) lies ~0.7 from the query and ~0.7 from every row: the bf16 score's error is ~1e-4, the
    rungs 2e-6 apart."""
    rng = np.random.default_rng(seed)
    qs = 4.0 * rng.standard_normal((n_q, D))
    v = rng.standard_normal((n_q, 1, D))
    v /= np.linalg.norm(v, axis=2, keepdims=True)
    g = rng.standard_normal((n_q, rungs, D))
    g /= np.linalg.norm(g, axis=2, keepdims=True)
    u = 0.7 * v + 0.71 * g
    u /= np.linalg.norm(u, axis=2, keepdims=True)
    r = np.sqrt(1.0 + 2e-6 * np.arange(rungs))
    rows = qs[:, None, :] + r[None, :, None] * u
    rows = rows[:, rng.permutation(rungs)]
    return rows.reshape(-1, D).astype(np.float32), qs.astype(np.float32), rows.mean(1).astype(np.float32)


def _u8(seed=87, reps=64):
    rng = np.random.default_rng(seed)
    centers = rng.uniform(100.0, 150.0, (8, D))
    base = np.clip(np.rint(centers[rng.integers(0, 8, N_BASE)] + 3.0 * rng.standard_normal((N_BASE, D))), 0, 255)
    x = np.repeat(base, reps, axis=0)
    moved = rng.random(len(x)) < 0.5
    for j in range(3):
        col = rng.integers(0, D, len(x))
        x[np.arange(len(x)), col] += np.where(moved, rng.choice([-1.0, 1.0], len(x)), 0.0)
    pick = rng.choice(N_BASE, NQ, replace=False)
    qs = base[pick].copy()
    noisy = np.arange(NQ) % 4 != 0
    qs[noisy] += rng.integers(-2, 3, (noisy.sum(), D))
    return np.clip(x, 0, 255).astype(np.uint8), np.clip(qs, 0, 255).astype(np.uint8), centers.astype(np.float32)


def family(name):
    """-> (rows, queries, list centres), seeded."""
    if name not in _DATA:
        if name == "ladder":
            _DATA[name] = _ladder()
        elif name == "u8":
            _DATA[name] = _u8()
        else:
            reps = 128 if name.startswith("dups128") else 48
            eps = 1e-4 if name.endswith("e4") else 1e-3
            shift = float(name.split("_shift")[1]) if "_shift" in name else 0.0
            _DATA[name] = _dups(reps, eps, shift)
    return _DATA[name]


def _f32(x):
    return np.asarray(x, np.float32)


def _mod():
    from cuvs_b200.neighbors import ivf_flat
    return ivf_flat


def _build(name, metric, chunks=1):
    """The family's rows in lists around its centres, added by `chunks` extend calls (device and host input in turn)."""
    m = _mod()
    ds, _, centers = family(name)
    index = m.build(m.IndexParams(n_lists=len(centers), metric=metric, add_data_on_build=False), torch.from_numpy(ds).cuda())
    m.set_centers(index, torch.from_numpy(centers).cuda())
    for j, part in enumerate(np.array_split(ds, chunks)):
        m.extend(index, torch.from_numpy(part).cuda() if j % 2 == 0 else torch.from_numpy(part), None)
    assert len(index) == len(ds)
    return index


_INDEX = {}


def _index(name, metric):
    if (name, metric) not in _INDEX:
        _INDEX[(name, metric)] = _build(name, metric)
    return _INDEX[(name, metric)]


def _n_probes(name):
    return N_PROBES.get(name, len(family(name)[2]))


def _search(index, qs, n_probes, k, **kw):
    m = _mod()
    d, i = m.search(m.SearchParams(n_probes=n_probes), index, torch.from_numpy(qs).cuda(), k, **kw)
    return d.cpu().numpy(), i.cpu().numpy()


_ORACLE = {}


def _oracle(name, metric, k):
    """The oracle's answer over the index's lists (cosine, with every list probed: its exact kNN), taken once at the
    largest k."""
    if (name, metric) not in _ORACLE:
        ds, qs, _ = family(name)
        kmax = min(max(KS), len(ds))
        if metric == "cosine":
            assert _n_probes(name) == len(family(name)[2])
            _ORACLE[(name, metric)] = oracle.knn(_f32(ds), _f32(qs), kmax, "cosine")
        else:
            _ORACLE[(name, metric)] = flat_search(_index(name, metric), _f32(ds), _f32(qs), _n_probes(name), kmax, metric)
    rd, ri = _ORACLE[(name, metric)]
    return rd[:, :k], ri[:, :k]


def _sure(name, metric, index=None):
    _, qs, _ = family(name)
    index = index or _index(name, metric)
    sure = certain_probes(index.centers.cpu().numpy(), _f32(qs), _n_probes(name), metric)
    assert sure.mean() >= 0.5, f"only {sure.sum()} of {len(sure)} queries have a certain probe set"
    return sure


def _check(name, metric, k):
    index = _index(name, metric)
    _, qs, _ = family(name)
    dist, idx = _search(index, qs, _n_probes(name), k)
    rd, ri = _oracle(name, metric, k)
    sure = _sure(name, metric)
    assert_same_answer(dist[sure], idx[sure], rd[sure], ri[sure])
    return last_flagged()


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("name", FAMILIES)
def test_sqeuclidean_every_k_regime(name, k):
    """k <= 32: fused lists of 16 / 32 per column half, kc2 = 32; 33..64: kc2 = 2k; > 64: the store path, kc2 = min(2k, 2048)."""
    _check(name, "sqeuclidean", k)


@pytest.mark.parametrize("k", [1, 10, 48, 256, 2048])
@pytest.mark.parametrize("metric", ["euclidean", "inner_product", "cosine"])
@pytest.mark.parametrize("name", ["dups128", "ladder", "dups48_shift10", "u8"])
def test_other_metrics(name, metric, k):
    if metric == "cosine" and _n_probes(name) < len(family(name)[2]):
        pytest.skip("the oracle's IVF search has no cosine: compared with its kNN with every list probed")
    _check(name, metric, k)


@pytest.mark.parametrize("k", [10, 48, 256])
@pytest.mark.parametrize("name", ["dups128", "ladder", "u8"])
def test_bitset_filter(name, k):
    """About half the rows kept: the oracle's search over the kept rows."""
    from cuvs_b200.neighbors import filters
    ds, qs, _ = family(name)
    index = _index(name, "sqeuclidean")
    n = len(ds)
    keep = np.random.default_rng(88).random(n) < 0.5
    bits = np.packbits(np.concatenate([keep, np.zeros((-n) % 32, bool)]), bitorder="little").view(np.uint32)
    dist, idx = _search(index, qs, _n_probes(name), k, filter=filters.from_bitset(torch.from_numpy(bits.view(np.int32)).cuda()))
    valid = idx != np.iinfo(np.int64).max
    assert keep[idx[valid]].all(), "a filtered-out row was returned"
    rd, ri = flat_search(index, _f32(ds), _f32(qs), _n_probes(name), k, "sqeuclidean", keep)
    sure = _sure(name, "sqeuclidean")
    assert_same_answer(dist[sure], idx[sure], rd[sure], ri[sure])


@pytest.mark.parametrize("name", ["dups128", "ladder"])
def test_filled_by_two_extends(name):
    ds, qs, _ = family(name)
    index = _build(name, "sqeuclidean", chunks=2)
    sure = _sure(name, "sqeuclidean", index)
    for k in (10, 64, 256):
        dist, idx = _search(index, qs, _n_probes(name), k)
        rd, ri = flat_search(index, _f32(ds), _f32(qs), _n_probes(name), k, "sqeuclidean")
        assert_same_answer(dist[sure], idx[sure], rd[sure], ri[sure])


@pytest.mark.parametrize("k", [10, 100, 256])
def test_query_batch_split(k, monkeypatch):
    """600 queries on dups128 with every list probed; at k > 64 a 1 MiB workspace budget splits them into batches of a few
    queries, each with its own certificate and fallback."""
    ds, _, centers = family("dups128")
    _, qs, _ = _dups(128, 1e-3, nq=BIG_NQ)
    monkeypatch.setenv("CUVS_B200_FLAT_LARGE_K_BUDGET_MB", "1")
    index = _index("dups128", "sqeuclidean")
    dist, idx = _search(index, qs, len(centers), k)
    rd, ri = flat_search(index, ds, qs, len(centers), k, "sqeuclidean")
    assert_same_answer(dist, idx, rd, ri)
    check_rows(idx, len(ds))


# ---------------------------------------------------------------------------------------------------------------- certificate
@pytest.mark.parametrize("name,k", [("dups128", 10), ("dups128", 48), ("dups128", 2048), ("ladder", 10), ("ladder", 48),
                                    ("ladder", 100)])
def test_certificate_flags_the_adversarial_families(name, k):
    """Cases where the bf16 ranking alone loses neighbours: the certificate has to send queries to the exact fallback.  (At
    k = 256 the 512 candidates of a query hold its whole ladder or several whole groups of copies, and nothing is lost.)"""
    flagged = _check(name, "sqeuclidean", k)
    assert flagged >= NQ // 4, f"only {flagged} of the queries were flagged"


def _control_shapes():
    yield "shift0", 30000, 128, 32, 8, 10, 72, 73, 74, "sqeuclidean"  # tests/test_far_from_origin_gpu.py's control
    # tests/test_ivf_flat_gpu.py::test_search_matches_oracle
    for n, d, n_lists, n_probes, k, metric in [(20000, 128, 64, 8, 10, "sqeuclidean"), (8000, 64, 32, 6, 16, "euclidean"),
                                               (10000, 33, 50, 10, 5, "inner_product"), (30000, 128, 128, 16, 32, "sqeuclidean"),
                                               (12000, 256, 40, 8, 10, "sqeuclidean"), (20000, 128, 64, 8, 256, "sqeuclidean")]:
        yield f"{n}x{d}", n, d, n_lists, n_probes, k, None, 5, 6, metric


@pytest.mark.parametrize("case", list(_control_shapes()), ids=lambda c: f"{c[0]}-k{c[5]}-{c[9]}")
def test_certificate_flags_few_queries_on_ordinary_data(case):
    """Clustered data without duplicates: the bound must be tight enough that almost every query keeps its bf16 candidates."""
    _, n, d, n_lists, n_probes, k, center_seed, ds_seed, q_seed, metric = case
    m = _mod()
    if center_seed is None:
        ds, centers = clustered(n, d, ds_seed, n_centers=max(8, n_lists // 2))
    else:
        centers = np.random.default_rng(center_seed).standard_normal((n_lists, d)).astype(np.float32)
        ds, _ = clustered(n, d, ds_seed, centers=centers)
    qs, _ = clustered(300, d, q_seed, centers=centers)
    index = m.build(m.IndexParams(n_lists=n_lists, metric=metric, kmeans_n_iters=10), torch.from_numpy(ds).cuda())
    dist, idx = _search(index, qs, n_probes, k)
    flagged = last_flagged()
    assert flagged <= 0.05 * len(qs), f"{flagged} of {len(qs)} queries flagged"
    rd, ri = flat_search(index, ds, qs, n_probes, k, metric)
    sure = certain_probes(index.centers.cpu().numpy(), qs, n_probes, metric)
    assert_same_answer(dist[sure], idx[sure], rd[sure], ri[sure])


def _ordinary():
    """Clustered data without duplicates, k-means lists (the shape of tests/test_ivf_flat_gpu.py)."""
    if "ordinary" not in _DATA:
        ds, centers = clustered(20000, D, 5, n_centers=32)
        qs, _ = clustered(NQ, D, 6, centers=centers)
        _DATA["ordinary"] = (ds, qs, None)
    return _DATA["ordinary"]


@pytest.mark.parametrize("k", [10, 48])
@pytest.mark.parametrize("metric", ["sqeuclidean", "inner_product", "cosine"])
@pytest.mark.parametrize("name", ["ordinary", "dups128", "ladder", "dups48_shift100", "u8"])
def test_candidate_error_budget(name, metric, k):
    """The budget of each merged candidate's own pair must dominate its observed |approx - exact|: by 4x, and by 2x where rows
    nearly repeat the query (dups128 in L2 and cosine; on an H100 its worst candidate reached 0.39 of the budget, the other
    families 0.24).  Doubling the budget to keep 4x there too flagged 27 instead of 0 of the 10k bench queries at k = 10."""
    err, ratio = budget_ratio(name, metric, k)
    bar = 0.5 if name == "dups128" and metric != "inner_product" else 0.25
    assert ratio.max() <= bar, f"observed error {err.max():.3e} is {ratio.max():.2f} of the budget"


def budget_ratio(name, metric, k):
    """-> (|approx - exact|, that over the budget of the candidate's own pair) of every merged candidate of a search with 2
    probes, [nq, kc2] (0 in empty slots).
    Approximate distances are in the scan's units: |q - x|^2, 2 (1 - cos) for cosine, -q.x for inner product."""
    import ctypes as C
    from cuvs_b200._capi import DL, check, lib
    from cuvs_b200.common import Resources
    if name == "ordinary":
        ds, qs, _ = _ordinary()
        m = _mod()
        index = m.build(m.IndexParams(n_lists=64, metric=metric, kmeans_n_iters=10), torch.from_numpy(ds).cuda())
    else:
        ds, qs, _ = family(name)
        index = _index(name, metric)
    q = torch.from_numpy(_f32(qs)).cuda()
    kc2 = max(32, 2 * k)
    ids = torch.zeros(len(qs), kc2, dtype=torch.int64, device="cuda")
    dist = torch.zeros(len(qs), kc2, dtype=torch.float32, device="cuda")
    bound = torch.zeros(len(qs), kc2, dtype=torch.float32, device="cuda")
    res = Resources()
    check(lib.cuvsB200IvfFlatCandidates(res.get_c_obj(), index._p, C.c_uint32(2), C.c_int(k), DL(q).ptr, DL(ids).ptr, DL(dist).ptr,
                                        DL(bound).ptr))
    ids, approx, bound = ids.cpu().numpy(), dist.cpu().numpy().astype(np.float64), bound.cpu().numpy().astype(np.float64)
    valid = ids != np.iinfo(np.int64).max
    assert valid[:, :k].all()
    x = np.asarray(ds, np.float64)[np.where(valid, ids, 0)]
    qq = np.asarray(qs, np.float64)[:, None, :]
    if metric == "sqeuclidean":
        exact = ((qq - x) ** 2).sum(-1)
    elif metric == "inner_product":
        exact = -(qq * x).sum(-1)
    else:
        exact = 2.0 * (1.0 - (qq * x).sum(-1) / (np.linalg.norm(qq, axis=-1) * np.linalg.norm(x, axis=-1)))
    err = np.where(valid, np.abs(approx - exact), 0.0)
    return err, np.where(valid, err / bound, 0.0)
