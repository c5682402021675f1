"""Search on data far from the origin, against the oracle.

The tensor-core scans rank rows by the expanded form |x|^2/2 - q.x with the products taken in bf16.  Their error follows the
size of the vectors, not the distances: on data far from the origin, or made of tight clusters far apart, the expanded form
cancels almost everything and what is left is bf16 rounding.  Every other suite draws its data near the origin, so these
tests move it away:

  * `clustered` (32 centres ~ N(0, 1), sigma 0.25) shifted by 0 (the control), 3, 10, 100, -50 in every component, or by a
    per-dimension vector uniform(0, 50);
  * tight clusters far apart: the centres times 10 and times 30, sigma 0.25 (subtracting the global mean does not help these);
  * uint8 rows 200 +- 10 through the narrow-dtype path.

IVF-Flat and brute force return exact fp32 distances, so they are held to the oracle bit for bit (assert_same_answer).  IVF-Flat
is compared on queries whose probe set is certain (certain_probes); the families whose probes are ambiguous at this scale are
probed exhaustively.  Its far-apart indexes take the generating centres as their lists (set_centers, then extend): k-means
started from 32 strided rows leaves some of those clusters without a centre and puts two of them in one list, whose rows then
lie far from their centre, which is a question of k-means quality, not of the scan.  IVF-PQ is held to the oracle's LUT
search at the bar each path meets near the origin (tests/test_ivf_pq_gpu.py)."""
import os

import numpy as np
import pytest
import torch

import oracle
from tests.ivf_oracle import assert_same_answer, certain_probes, check_rows, flat_search, pq_search
from tests.util import clustered, last_flagged

pytestmark = pytest.mark.gpu

N, D, NQ, N_CENTERS, N_LISTS = 30000, 128, 300, 32, 32
SHIFTS = {"shift0": 0.0, "shift3": 3.0, "shift10": 10.0, "shift100": 100.0, "shift-50": -50.0}
FAMILIES = list(SHIFTS) + ["perdim", "apart10", "apart30", "u8"]
# probes of 32 lists: 8 where the centre gaps are wide enough for most probe sets to be certain, every list otherwise
N_PROBES = {"shift0": 8, "shift3": 8, "apart10": 8, "apart30": 8}
FLT_MAX = np.finfo(np.float32).max

_DATA = {}
_CENTERS = {}  # the generating centres of the far-apart families


def family(name):
    """-> (rows [N, D], queries [NQ, D]), seeded: float32, uint8 for "u8"."""
    if name not in _DATA:
        if name == "u8":
            rng = np.random.default_rng(71)
            centers = rng.uniform(193.0, 207.0, (N_CENTERS, D))
            lab = rng.integers(0, N_CENTERS, N + NQ)
            x = np.clip(np.rint(centers[lab] + 2.0 * rng.standard_normal((N + NQ, D))), 190, 210).astype(np.uint8)
            _DATA[name] = (x[:N], x[N:])
        else:
            scale = {"apart10": 10.0, "apart30": 30.0}.get(name, 1.0)
            centers = (np.random.default_rng(72).standard_normal((N_CENTERS, D)) * scale).astype(np.float32)
            if scale != 1.0:
                _CENTERS[name] = centers
            ds, _ = clustered(N, D, 73, centers=centers)
            qs, _ = clustered(NQ, D, 74, centers=centers)
            shift = np.random.default_rng(75).uniform(0.0, 50.0, D).astype(np.float32) if name == "perdim" else SHIFTS.get(name, 0.0)
            _DATA[name] = ((ds + shift).astype(np.float32), (qs + shift).astype(np.float32))
    return _DATA[name]


def _f32(x):
    return np.asarray(x, np.float32)


# ---------------------------------------------------------------------------------------------------------------- IVF-Flat
_FLAT = {}


def _flat_mod():
    from cuvs_b200.neighbors import ivf_flat
    return ivf_flat


def _flat_build(name, metric, chunks=1):
    """The family's index: k-means lists, or the generating centres of a far-apart family; the rows added at build or, with
    `chunks` > 1, by that many extend calls (device and host input in turn)."""
    m = _flat_mod()
    ds, _ = family(name)
    fixed = name in _CENTERS
    index = m.build(m.IndexParams(n_lists=N_LISTS, metric=metric, kmeans_n_iters=10, add_data_on_build=not fixed and chunks == 1),
                    torch.from_numpy(ds).cuda())
    if fixed:
        m.set_centers(index, torch.from_numpy(_CENTERS[name]).cuda())
    if fixed or chunks > 1:
        assert len(index) == 0
        for j, part in enumerate(np.array_split(ds, chunks)):
            m.extend(index, torch.from_numpy(part).cuda() if j % 2 == 0 else torch.from_numpy(part), None)
    assert len(index) == N
    return index


def _flat_index(name, metric):
    key = (name, metric)
    if key not in _FLAT:
        _FLAT[key] = _flat_build(name, metric)
    return _FLAT[key]


def _flat_search(index, qs, n_probes, k, **kw):
    m = _flat_mod()
    d, i = m.search(m.SearchParams(n_probes=n_probes), index, torch.from_numpy(qs).cuda(), k, **kw)
    return d.cpu().numpy(), i.cpu().numpy()


_FLAT_ORACLE = {}


def _flat_oracle(name, metric, k):
    """The oracle's search over the index's lists, taken once at the largest k: its first k entries are its answer at k."""
    key = (name, metric)
    if key not in _FLAT_ORACLE:
        ds, qs = family(name)
        _FLAT_ORACLE[key] = flat_search(_flat_index(name, metric), _f32(ds), _f32(qs), N_PROBES.get(name, N_LISTS), 1024, metric)
    rd, ri = _FLAT_ORACLE[key]
    return rd[:, :k], ri[:, :k]


def _certain(name, metric):
    ds, qs = family(name)
    sure = certain_probes(_flat_index(name, metric).centers.cpu().numpy(), _f32(qs), N_PROBES.get(name, N_LISTS), metric)
    assert sure.mean() >= 0.5, f"only {sure.sum()} of {len(sure)} queries have a certain probe set"
    return sure


def _check_flat(name, metric, k):
    index = _flat_index(name, metric)
    _, qs = family(name)
    dist, idx = _flat_search(index, qs, N_PROBES.get(name, N_LISTS), k)
    rd, ri = _flat_oracle(name, metric, k)
    sure = _certain(name, metric)
    assert_same_answer(dist[sure], idx[sure], rd[sure], ri[sure])


@pytest.mark.parametrize("k", [1, 10, 16, 32, 33, 48, 64, 100, 256, 1024])
@pytest.mark.parametrize("name", FAMILIES)
def test_ivf_flat_sqeuclidean_every_k_regime(name, k):
    """k <= 32: fused lists; 33..64: fused lists and the certificate's rerun; > 64: the store path."""
    _check_flat(name, "sqeuclidean", k)


@pytest.mark.parametrize("k", [10, 48, 256])
@pytest.mark.parametrize("metric", ["euclidean", "inner_product"])
@pytest.mark.parametrize("name", FAMILIES)
def test_ivf_flat_other_metrics(name, metric, k):
    _check_flat(name, metric, k)


@pytest.mark.parametrize("k", [10, 64, 256])
@pytest.mark.parametrize("name", ["shift0", "shift3", "shift10", "perdim", "apart30"])
def test_ivf_flat_cosine_with_every_list_probed(name, k):
    """The oracle's IVF search has no cosine: with every list probed the search is exact, so compare with its kNN.

    (Not at a shift of 50 or 100: there the fp32 cosine distance 1 - q.x / (|q| |x|) that both return carries the ~7e-7 relative
    error of a 128-term fp32 dot product, more than the ~1e-7 between neighbours whose distances are ~1e-5, so the k best by
    that value depend on rows a correct scan ranks elsewhere.  Brute force, which re-scores every row it cannot certify,
    matches it bit for bit there: test_brute_force_is_exact.)"""
    ds, qs = family(name)
    dist, idx = _flat_search(_flat_index(name, "cosine"), qs, N_LISTS, k)
    rd, ri = oracle.knn(ds, qs, k, "cosine")
    assert_same_answer(dist, idx, rd, ri)


@pytest.mark.parametrize("k", [10, 48, 256])
@pytest.mark.parametrize("name", ["apart10", "shift10"])
def test_ivf_flat_bitset_filter(name, k):
    """40 % of the rows kept: the oracle's search over the kept rows, one case per k regime."""
    from cuvs_b200.neighbors import filters
    ds, qs = family(name)
    index = _flat_index(name, "sqeuclidean")
    keep = np.random.default_rng(76).random(N) < 0.4
    bits = np.packbits(np.concatenate([keep, np.zeros((-N) % 32, bool)]), bitorder="little").view(np.uint32)
    n_probes = N_PROBES.get(name, N_LISTS)
    dist, idx = _flat_search(index, qs, n_probes, k, filter=filters.from_bitset(torch.from_numpy(bits.view(np.int32)).cuda()))
    valid = idx != np.iinfo(np.int64).max
    assert keep[idx[valid]].all(), "a filtered-out row was returned"
    rd, ri = flat_search(index, _f32(ds), _f32(qs), n_probes, k, "sqeuclidean", keep)
    sure = _certain(name, "sqeuclidean")
    assert_same_answer(dist[sure], idx[sure], rd[sure], ri[sure])


@pytest.mark.parametrize("name", ["shift10", "apart30"])
def test_ivf_flat_filled_by_two_extends(name):
    """Built without its rows, then filled by two extend calls (device and host input): the scan's per-row planes are
    rebuilt on every extend."""
    ds, qs = family(name)
    index = _flat_build(name, "sqeuclidean", chunks=2)
    n_probes = N_PROBES.get(name, N_LISTS)
    sure = certain_probes(index.centers.cpu().numpy(), qs, n_probes, "sqeuclidean")
    assert sure.mean() >= 0.5
    for k in (10, 64):
        dist, idx = _flat_search(index, qs, n_probes, k)
        rd, ri = flat_search(index, ds, qs, n_probes, k, "sqeuclidean")
        assert_same_answer(dist[sure], idx[sure], rd[sure], ri[sure])


# ---------------------------------------------------------------------------------------------------------------- brute force
_BF_ORACLE = {}
BF_FAMILIES = ["shift0", "shift100", "shift-50", "apart30"]


@pytest.mark.parametrize("k", [10, 48, 64, 100])
@pytest.mark.parametrize("metric", ["sqeuclidean", "euclidean", "inner_product", "cosine"])
@pytest.mark.parametrize("name", BF_FAMILIES)
def test_brute_force_is_exact(name, metric, k):
    """Bit-exact against the oracle's kNN: the split-bf16 candidates carry a certificate whose budget grows with
    |q|^2 + max|x|^2, and the queries it cannot certify are recomputed on the exact path."""
    from cuvs_b200.neighbors import brute_force
    ds, qs = family(name)
    index = brute_force.build(torch.from_numpy(ds).cuda(), metric=metric)
    d, i = brute_force.search(index, torch.from_numpy(qs).cuda(), k)
    flagged = last_flagged()
    if (name, metric) not in _BF_ORACLE:
        _BF_ORACLE[(name, metric)] = oracle.knn(ds, qs, 100, metric)
    rd, ri = _BF_ORACLE[(name, metric)]
    assert_same_answer(d.cpu().numpy(), i.cpu().numpy(), rd[:, :k], ri[:, :k], pad_id=-1)
    if k > 64:
        return  # the exact path serves every query
    if name == "shift100":
        # the bf16 error at |x| ~ 1100 swamps the gaps between neighbours: the fallback must carry (nearly) the whole batch
        assert flagged >= 0.9 * NQ, f"only {flagged} of {NQ} queries took the exact fallback"
    elif name == "shift0":
        assert flagged <= NQ // 100, f"{flagged} of {NQ} queries fell back to the exact path"


# ---------------------------------------------------------------------------------------------------------------- IVF-PQ
_PQ = {}
_PQ_ORACLE = {}
PQ_FAMILIES = ["shift0", "shift10", "shift100", "apart10", "apart30"]


def _pq_mod():
    from cuvs_b200.neighbors import ivf_pq
    return ivf_pq


def _pq_index(name, metric):
    key = (name, metric)
    if key not in _PQ:
        m = _pq_mod()
        ds, _ = family(name)
        _PQ[key] = m.build(m.IndexParams(n_lists=N_LISTS, pq_dim=64, metric=metric, kmeans_n_iters=10), torch.from_numpy(ds).cuda())
    return _PQ[key]


def _pq_search(index, qs, k, path, **kw):
    m = _pq_mod()
    os.environ["CUVS_B200_PQ_PATH"] = path
    try:
        d, i = m.search(m.SearchParams(n_probes=N_LISTS, **kw), index, torch.from_numpy(qs).cuda(), k)
    finally:
        del os.environ["CUVS_B200_PQ_PATH"]
    return d.cpu().numpy(), i.cpu().numpy()


def _pq_oracle(name, metric, lut):
    key = (name, metric, lut)
    if key not in _PQ_ORACLE:
        _, qs = family(name)
        _PQ_ORACLE[key] = pq_search(_pq_index(name, metric), qs, N_LISTS, 10, metric, lut, "f32")
    return _PQ_ORACLE[key]


# every list probed: the probe sets are the oracle's.  The bars are those of tests/test_ivf_pq_gpu.py for the same path.
@pytest.mark.parametrize("metric", ["sqeuclidean", "inner_product", "cosine"])
@pytest.mark.parametrize("name", PQ_FAMILIES)
def test_ivf_pq_code_stream(name, metric):
    index = _pq_index(name, metric)
    assert index.streamed
    _, qs = family(name)
    d, i = _pq_search(index, qs, 10, "stream")  # fp32 LUT semantics: two passes
    rd, ri = _pq_oracle(name, metric, "f32")
    check_rows(i, N)
    assert oracle.recall_with_ties(i, d, ri, rd, eps=2e-3) >= 0.99
    d, i = _pq_search(index, qs, 10, "stream", lut_dtype=np.float16)  # one pass
    rd, ri = _pq_oracle(name, metric, "f16")
    check_rows(i, N)
    assert oracle.recall_with_ties(i, d, ri, rd, eps=1e-2) >= 0.975


@pytest.mark.parametrize("metric", ["sqeuclidean", "inner_product", "cosine"])
@pytest.mark.parametrize("name", PQ_FAMILIES)
def test_ivf_pq_decoded_rows_agree_with_the_code_stream(name, metric):
    """300 queries x 32 probes / 32 lists: a dense batch, served from the decoded-row cache; the code stream must agree."""
    index = _pq_index(name, metric)
    _, qs = family(name)
    d_dense, i_dense = _pq_search(index, qs, 10, "auto", lut_dtype=np.float16)
    d_str, i_str = _pq_search(index, qs, 10, "stream", lut_dtype=np.float16)
    same = np.mean([len(set(a) & set(b)) / 10.0 for a, b in zip(i_dense, i_str)])
    assert same >= 0.995, same
    rd, ri = _pq_oracle(name, metric, "f16")
    assert oracle.recall_with_ties(i_dense, d_dense, ri, rd, eps=1e-2) >= 0.975


@pytest.mark.parametrize("metric", ["sqeuclidean", "inner_product", "cosine"])
@pytest.mark.parametrize("name", PQ_FAMILIES)
def test_ivf_pq_lut_kernel(name, metric):
    index = _pq_index(name, metric)
    _, qs = family(name)
    d, i = _pq_search(index, qs, 10, "lut")
    rd, ri = _pq_oracle(name, metric, "f32")
    assert oracle.recall_with_ties(i, d, ri, rd, eps=1e-5) >= 0.999
    same = i == ri
    # (cosine at a shift of 100: every distance is ~1e-5, and neighbours lie closer together than the fp32 rounding of a LUT sum
    # near 1, so the kernel's and the oracle's summation orders rank them differently: 98.6 % of the ids agree, the rest are
    # ties within the 1e-5 above)
    assert same.mean() >= (0.98 if (name, metric) == ("shift100", "cosine") else 0.99)
    np.testing.assert_allclose(d[same], rd[same], rtol=1e-5, atol=1e-5)
