"""tests/ivf_pq_cosine_ref.py (the oracle's LUT-sum search handed the unit rotated queries) against an independent float64
NumPy restatement of the reference (cpp/src/neighbors/ivf_pq/ivf_pq_search.cuh:101-107 coarse ranking by -q.c; :545-549 and
:1020-1025 the fine score 1 - q^.(c + y) over the unit rotated query q^), on a tiny hand-built index."""
import numpy as np
import pytest

from tests.ivf_pq_cosine_ref import ivf_pq_cosine_search, unit_rotated_queries


def _index(seed=5, dim=16, pq_dim=8, pq_bits=8, n_lists=6, n=300):
    rng = np.random.default_rng(seed)
    pq_len = dim // pq_dim
    rot = np.linalg.qr(rng.standard_normal((dim, dim)))[0].astype(np.float32)  # [rot_dim, dim], orthonormal columns
    centers = rng.standard_normal((n_lists, dim))
    centers = (centers / np.linalg.norm(centers, axis=1, keepdims=True)).astype(np.float32)  # a cosine index keeps unit centres
    centers_rot = (centers.astype(np.float64) @ rot.T.astype(np.float64)).astype(np.float32)
    pq_centers = (0.2 * rng.standard_normal((pq_dim, pq_len, 1 << pq_bits))).astype(np.float32)
    sizes = rng.multinomial(n, np.full(n_lists, 1.0 / n_lists))
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    codes = rng.integers(0, 1 << pq_bits, (n, pq_dim)).astype(np.uint8)
    ids = rng.permutation(n).astype(np.int64) + 1000
    return rot, centers, centers_rot, pq_centers, offs, codes, ids


def _restated(rot, centers, centers_rot, pq_centers, offs, codes, ids, qs, n_probes, k):
    r, c, cr, pq = (a.astype(np.float64) for a in (rot, centers, centers_rot, pq_centers))
    pq_dim, pq_len, _ = pq.shape
    out_d = np.full((len(qs), k), np.finfo(np.float32).max, np.float64)
    out_i = np.full((len(qs), k), np.iinfo(np.int64).max, np.int64)
    for qi, q in enumerate(qs.astype(np.float64)):
        probes = np.argsort(-(c @ q), kind="stable")[:n_probes]
        qr = r @ q
        nrm = np.linalg.norm(qr)
        qh = qr / nrm if nrm > 0 else qr
        cand_d, cand_i = [], []
        for l in probes:
            for row in range(offs[l], offs[l + 1]):
                y = pq[np.arange(pq_dim), :, codes[row]].reshape(-1)  # [pq_dim * pq_len]
                cand_d.append(1.0 - qh @ (cr[l] + y))
                cand_i.append(ids[row])
        order = np.argsort(cand_d, kind="stable")[:k]
        out_d[qi, :len(order)] = np.asarray(cand_d)[order]
        out_i[qi, :len(order)] = np.asarray(cand_i)[order]
    return out_d, out_i


@pytest.mark.parametrize("n_probes,k", [(2, 10), (6, 25)])
def test_oracle_on_unit_queries_matches_restatement(n_probes, k):
    rot, centers, centers_rot, pq_centers, offs, codes, ids = _index()
    rng = np.random.default_rng(9)
    qs = rng.standard_normal((40, rot.shape[1])) * np.exp(rng.uniform(np.log(0.1), np.log(10.0), (40, 1)))
    qs = qs.astype(np.float32)
    d, i = ivf_pq_cosine_search(centers_rot, rot, pq_centers, offs, codes, ids, qs, n_probes, k, pq_bits=8, lut_dtype="f32")
    rd, ri = _restated(rot, centers, centers_rot, pq_centers, offs, codes, ids, qs, n_probes, k)
    assert np.array_equal(i, ri)
    np.testing.assert_allclose(d, rd, rtol=0, atol=1e-5)
    # the query's norm does not matter
    d2, i2 = ivf_pq_cosine_search(centers_rot, rot, pq_centers, offs, codes, ids, qs * np.float32(7.3), n_probes, k, pq_bits=8,
                                  lut_dtype="f32")
    assert np.array_equal(i2, i)
    np.testing.assert_allclose(d2, d, rtol=0, atol=1e-5)


def test_oracle_zero_query_scores_one():
    rot, centers, centers_rot, pq_centers, offs, codes, ids = _index()
    qs = np.zeros((1, rot.shape[1]), np.float32)
    d, i = ivf_pq_cosine_search(centers_rot, rot, pq_centers, offs, codes, ids, qs, 3, 10, pq_bits=8, lut_dtype="f32")
    assert (d == 1.0).all() and np.isin(i, ids).all()


def test_unit_rotated_queries():
    rng = np.random.default_rng(3)
    rot = np.linalg.qr(rng.standard_normal((24, 24)))[0][:, :20].astype(np.float32)  # rot_dim 24 > dim 20
    qs = (rng.standard_normal((50, 20)) * 5).astype(np.float32)
    qs[7] = 0.0
    u = unit_rotated_queries(rot, qs)
    ref = qs.astype(np.float64) @ rot.T.astype(np.float64)
    n = np.linalg.norm(ref, axis=1, keepdims=True)
    ref = np.where(n > 0, ref / np.where(n > 0, n, 1.0), 0.0)
    assert u.dtype == np.float32 and u.shape == (50, 24) and (u[7] == 0).all()
    np.testing.assert_allclose(u, ref, rtol=0, atol=1e-6)
