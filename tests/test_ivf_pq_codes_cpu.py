"""The code unpacking helper (tests/ivf_pq_codes.py) and the oracle's IVF-PQ search for every code shape the library builds.

The helper is pinned with hand-computed bytes where codes straddle byte boundaries and round-tripped through an independent
packer.  oracle.ivf_pq_search is checked against a float64 NumPy restatement of the LUT sum (probes ranked by
|c|^2 - 2 q.c, or -q.c for inner product; score sum_s |r_s - book[code_s]|^2 with r = R q - c_rot[list], or -(R q).(c_rot + y)
for inner product) for pq_bits 4-8, per-subspace and per-cluster codebooks, pq_len 1 / 2 / 3 / 4 and rot_dim > dim."""
import numpy as np
import pytest

import oracle
from tests.ivf_pq_codes import row_bytes, unpack_codes


def _pack(codes, pq_bits):
    """Independent packer: each row as one Python integer, code j shifted to bit j * pq_bits, written little-endian."""
    codes = np.asarray(codes)
    ld = row_bytes(codes.shape[1], pq_bits)
    out = np.zeros((codes.shape[0], ld), np.uint8)
    for r, row in enumerate(codes):
        v = 0
        for j, c in enumerate(row):
            v |= int(c) << (j * pq_bits)
        out[r] = np.frombuffer(v.to_bytes(ld, "little"), np.uint8)
    return out


@pytest.mark.parametrize("pq_bits,codes,packed", [
    # 5 bits: code 1 straddles bytes 0-1, code 3 straddles bytes 1-2
    (5, [1, 2, 3, 31], [0x41, 0x8C, 0x0F]),
    # 7 bits: the last code spills its top 3 bits into a byte of its own
    (7, [127, 0, 85, 42, 127], [0x7F, 0x40, 0x55, 0xF5, 0x07]),
    (4, [0xA, 0x5, 0xF], [0x5A, 0x0F]),
    (8, [0, 200, 255], [0x00, 0xC8, 0xFF]),
])
def test_unpack_hand_computed_bytes(pq_bits, codes, packed):
    packed = np.array([packed], np.uint8)
    assert (unpack_codes(packed, len(codes), pq_bits) == np.array([codes], np.uint8)).all()
    assert (_pack([codes], pq_bits) == packed).all()


@pytest.mark.parametrize("pq_bits", [4, 5, 6, 7, 8])
@pytest.mark.parametrize("pq_dim", [1, 3, 8, 16, 17, 24, 34])
def test_unpack_round_trip(pq_bits, pq_dim):
    rng = np.random.default_rng(pq_bits * 100 + pq_dim)
    codes = rng.integers(0, 1 << pq_bits, (37, pq_dim)).astype(np.uint8)
    codes[0] = (1 << pq_bits) - 1  # every bit set: a dropped spill bit shows
    packed = _pack(codes, pq_bits)
    assert packed.shape == (37, row_bytes(pq_dim, pq_bits))
    assert (unpack_codes(packed, pq_dim, pq_bits) == codes).all()


def _index(seed, dim, pq_dim, pq_bits, per_cluster, n_lists=7, n=600):
    rng = np.random.default_rng(seed)
    pq_len = -(-dim // pq_dim)
    rot_dim = pq_dim * pq_len
    rot = np.linalg.qr(rng.standard_normal((rot_dim, rot_dim)))[0][:, :dim].astype(np.float32)  # [rot_dim, dim]
    centers = rng.standard_normal((n_lists, dim)).astype(np.float32)
    centers_rot = (centers.astype(np.float64) @ rot.T.astype(np.float64)).astype(np.float32)
    n_books = n_lists if per_cluster else pq_dim
    pq_centers = (0.3 * rng.standard_normal((n_books, pq_len, 1 << pq_bits))).astype(np.float32)
    sizes = rng.multinomial(n, np.full(n_lists, 1.0 / n_lists))
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    codes = rng.integers(0, 1 << pq_bits, (n, pq_dim)).astype(np.uint8)
    ids = rng.permutation(n).astype(np.int64) + 500
    qs = (centers[rng.integers(0, n_lists, 30)] + 0.5 * rng.standard_normal((30, dim))).astype(np.float32)
    return rot, centers, centers_rot, pq_centers, offs, codes, ids, qs


def _restated(rot, centers, centers_rot, pq_centers, offs, codes, ids, qs, n_probes, k, metric, per_cluster):
    r, c, cr, pq = (a.astype(np.float64) for a in (rot, centers, centers_rot, pq_centers))
    ip = metric == "inner_product"
    pq_dim = codes.shape[1]
    pq_len = pq.shape[1]
    out_d = np.full((len(qs), k), np.finfo(np.float32).max, np.float64)
    out_i = np.full((len(qs), k), np.iinfo(np.int64).max, np.int64)
    for qi, q in enumerate(qs.astype(np.float64)):
        coarse = -(c @ q) if ip else (c * c).sum(1) - 2 * (c @ q)
        probes = np.argsort(coarse, kind="stable")[:n_probes]
        qr = r @ q
        cand_d, cand_i = [], []
        for l in probes:
            rows = np.arange(offs[l], offs[l + 1])
            book = pq[l][None].repeat(pq_dim, 0) if per_cluster else pq      # [pq_dim, pq_len, 2^bits]
            y = book[np.arange(pq_dim)[None, :], :, codes[rows]].reshape(len(rows), pq_dim * pq_len)
            if ip:
                score = -((cr[l][None] + y) @ qr)
            else:
                score = (((qr - cr[l])[None] - y) ** 2).sum(1)
            cand_d.extend(score.tolist())
            cand_i.extend(ids[rows].tolist())
        order = np.argsort(cand_d, kind="stable")[:k]
        out_d[qi, :len(order)] = np.asarray(cand_d)[order]
        out_i[qi, :len(order)] = np.asarray(cand_i)[order]
    if ip:
        out_d = -out_d
    return out_d, out_i


SHAPES = [  # (dim, pq_dim, pq_bits, per_cluster)
    (16, 8, 4, False), (16, 8, 5, False), (16, 8, 6, False), (16, 8, 7, False), (16, 8, 8, False),
    (16, 8, 4, True), (16, 8, 5, True), (16, 8, 8, True),
    (12, 12, 6, False),   # pq_len 1
    (24, 8, 5, True),     # pq_len 3
    (20, 6, 7, False),    # pq_len 4, rot_dim 24 > dim 20
    (17, 16, 8, True),    # pq_len 2, rot_dim 32 > dim 17
    (10, 4, 4, False),    # pq_len 3, rot_dim 12 > dim 10
]


@pytest.mark.parametrize("metric", ["sqeuclidean", "inner_product"])
@pytest.mark.parametrize("dim,pq_dim,pq_bits,per_cluster", SHAPES)
def test_oracle_matches_float64_lut_sum(dim, pq_dim, pq_bits, per_cluster, metric):
    rot, centers, centers_rot, pq_centers, offs, codes, ids, qs = _index(dim * 31 + pq_bits, dim, pq_dim, pq_bits, per_cluster)
    n_probes, k = 3, 40
    d, i = oracle.ivf_pq_search(centers, centers_rot, rot, pq_centers, offs, codes, ids, qs, n_probes, k, metric,
                                pq_bits=pq_bits, per_cluster=per_cluster)
    rd, ri = _restated(rot, centers, centers_rot, pq_centers, offs, codes, ids, qs, n_probes, k, metric, per_cluster)
    np.testing.assert_allclose(d, rd, rtol=1e-5, atol=1e-5)
    # ids equal except where a neighbouring slot holds (nearly) the same distance
    tol = 1e-5 * np.maximum(1.0, np.abs(rd))
    tied = np.zeros(rd.shape, bool)
    tied[:, 1:] |= np.abs(rd[:, 1:] - rd[:, :-1]) <= tol[:, 1:]
    tied[:, :-1] |= np.abs(rd[:, :-1] - rd[:, 1:]) <= tol[:, :-1]
    assert (i[~tied] == ri[~tied]).all()
    assert tied.mean() < 0.05  # the comparison above is not vacuous

