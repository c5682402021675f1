"""The oracle's IVF searches over the lists of an index the library built, and the row check of a search result.

The index's own centres, quantizers, list membership and codes are read back through its getters and fed to the oracle, so
a search can be compared element-wise with what the oracle finds in the same lists."""
import numpy as np

import oracle
from tests.ivf_pq_codes import index_codes
from tests.ivf_pq_cosine_ref import ivf_pq_cosine_search

I64_MAX = np.iinfo(np.int64).max


def flat_lists(index, keep=None):
    """-> (list offsets [n_lists + 1], ids) of an IVF-Flat index, lists concatenated; with `keep` (a boolean mask over the
    ids), only the kept rows."""
    ids = [index.list_indices(l).cpu().numpy() for l in range(index.n_lists)]
    if keep is not None:
        ids = [i[keep[i]] for i in ids]
    offsets = np.concatenate([[0], np.cumsum([len(i) for i in ids])])
    return offsets, np.concatenate(ids)


def flat_search(index, ds, qs, n_probes, k, metric, keep=None):
    """The oracle's IVF-Flat search over the index's centres and lists (rows of `ds` by id, only the kept ones with `keep`)."""
    offsets, ids = flat_lists(index, keep)
    return oracle.ivf_flat_search(index.centers.cpu().numpy(), offsets, ds[ids], ids, qs, n_probes, k, metric)


def pq_search(index, qs, n_probes, k, metric="sqeuclidean", lut="f32", dist="f32", per_cluster=False):
    """The oracle's LUT-sum IVF-PQ search over the index's quantizers, codes and lists, at the index's pq_bits; cosine with
    the reference's cosine semantics (tests/ivf_pq_cosine_ref.py).  `per_cluster`: the index has per-cluster codebooks."""
    offs, codes, ids = index_codes(index)
    kw = dict(pq_bits=index.pq_bits, per_cluster=per_cluster, lut_dtype=lut, dist_dtype=dist)
    if metric == "cosine":
        return ivf_pq_cosine_search(index.centers_rot.cpu().numpy(), index.rotation_matrix.cpu().numpy(),
                                    index.pq_centers.cpu().numpy(), offs, codes, ids, qs, n_probes, k, **kw)
    return oracle.ivf_pq_search(index.centers.cpu().numpy(), index.centers_rot.cpu().numpy(), index.rotation_matrix.cpu().numpy(),
                                index.pq_centers.cpu().numpy(), offs, codes, ids, qs, n_probes, k, metric, **kw)


def certain_probes(centers, qs, n_probes, metric):
    """-> bool [nq]: queries whose `n_probes` nearest centres are the same set for any coarse search that is correct to within
    the bound below, so that the library's probe set and the oracle's are provably equal.

    Centre scores are taken in float64 in the ranking form of each metric: |c|^2 - 2 q.c (L2), -q.c (inner product), -q^.c^
    (cosine, unit vectors).  A query is certain when the gap between its n_probes-th and (n_probes+1)-th score exceeds
    2 * 2^-15 * (|q|^2 + max|c|^2).  That covers both coarse searches at once: the library's 3-pass split-bf16 scores are within
    2^-15 (|q|^2 + |c|^2) of the exact ones (the brute-force certificate's budget for the same products, which the observed error
    stays 4x below: tests/test_brute_force_gpu.py::test_candidate_error_budget), and the oracle's fp32 dot products of
    d <= 128 terms with fmaf are within d * 2^-24 * 2|q||c| <= 2^-17 (|q|^2 + |c|^2) of them."""
    c, q = np.asarray(centers, np.float64), np.asarray(qs, np.float64)
    if n_probes >= len(c):
        return np.ones(len(q), bool)
    if metric == "cosine":
        c = c / np.linalg.norm(c, axis=1, keepdims=True)
        q = q / np.linalg.norm(q, axis=1, keepdims=True)
    cn = (c * c).sum(1)
    score = -(q @ c.T) if metric in ("inner_product", "cosine") else cn[None, :] - 2.0 * (q @ c.T)
    s = np.sort(score, axis=1)
    gap = s[:, n_probes] - s[:, n_probes - 1]
    return gap > 2.0 * 2.0 ** -15 * ((q * q).sum(1) + cn.max())


def assert_same_answer(dist, idx, rd, ri, pad_id=I64_MAX):
    """A search result equals the oracle's: distances bit for bit, ids everywhere outside a group of exactly equal distances, the
    same ids inside such a group unless it reaches the last slot (its members beyond k are arbitrary), and every missing slot
    `pad_id` where the oracle has one (its distance, +-FLT_MAX, is part of the bit-exact distances)."""
    dist, idx, rd, ri = map(np.asarray, (dist, idx, rd, ri))
    diff = dist != rd
    if diff.any():
        lost = sum(len(np.setdiff1d(t, f)) for f, t in zip(idx, ri))
        raise AssertionError(f"{diff.any(1).sum()} of {len(rd)} queries differ from the oracle in {diff.sum()} of {rd.size} "
                             f"distances; {lost} of the oracle's ids are missing")
    np.testing.assert_array_equal(idx == pad_id, ri == pad_id)
    check_rows(idx)
    # group number of every slot: a new group starts wherever the distance changes
    group = np.cumsum(np.concatenate([np.ones((len(rd), 1), bool), rd[:, 1:] != rd[:, :-1]], axis=1), axis=1)
    inner = group != group[:, -1:]
    # inside a group the order of the ids is free: compare them sorted by (group, id)
    a = np.take_along_axis(idx, np.lexsort((idx, group)), axis=1)
    b = np.take_along_axis(ri, np.lexsort((ri, group)), axis=1)
    bad = inner & (a != b)
    assert not bad.any(), f"{bad.any(1).sum()} of {len(rd)} queries return other ids than the oracle, " \
                          f"{bad.sum()} of {inner.sum()} slots (query {np.nonzero(bad.any(1))[0][:8]})"


def check_rows(i, n=None):
    """No id twice in a row of `i` (empty slots hold INT64_MAX); with `n`, every real id in [0, n)."""
    for row in i:
        real = row[row != I64_MAX]
        assert len(np.unique(real)) == len(real), "an id is returned twice in one row"
        if n is not None:
            assert ((real >= 0) & (real < n)).all()
