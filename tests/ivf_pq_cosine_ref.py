"""The reference's cosine IVF-PQ search from the oracle's LUT-sum search (oracle_ivf_pq_search).

The reference scores cosine over the unit rotated query q^ = R q / |R q| (cpp/src/neighbors/ivf_pq/ivf_pq_search.cuh:1020-1025)
and ranks probes by -q.c over unit centres (:101-107).  The oracle scores cosine as inner product plus 1 and does not
normalise the query, so it is handed q^ itself: computed here in the search's own fp32 arithmetic (one fmaf per component in
ascending order for R q and for |R q|^2, then a correctly rounded 1 / sqrt and one multiply, a zero row staying zero), with an
identity rotation and the rotated centres.  The probes then rank by -q^.c_rot, which orders lists as -q.c does, and the LUT
entries are built from the same q^ as the library's."""
import numpy as np

import oracle


def _fmaf_dot(a, b):
    """[n, d] x [m, d] -> [n, m] fp32 dot products, one fmaf per component in ascending order.  The fp32 product is exact in
    fp64, so each step rounds once to fp64 and then to fp32 (a double rounding that can differ from fmaf only at an exact fp32
    tie of the fp64 sum)."""
    acc = np.zeros((a.shape[0], b.shape[0]), np.float32)
    for k in range(a.shape[1]):
        acc = (a[:, k, None].astype(np.float64) * b[None, :, k].astype(np.float64) + acc).astype(np.float32)
    return acc


def unit_rotated_queries(rotation, queries):
    """q^ = R q * (1 / sqrt(|R q|^2)) per row in fp32; 0 for a zero row."""
    r, q = np.asarray(rotation, np.float32), np.asarray(queries, np.float32)
    qr = _fmaf_dot(q, r)
    nrm = np.zeros(len(qr), np.float32)
    for k in range(qr.shape[1]):
        nrm = (qr[:, k].astype(np.float64) * qr[:, k].astype(np.float64) + nrm).astype(np.float32)
    pos = nrm > 0
    inv = np.zeros_like(nrm)
    inv[pos] = np.float32(1.0) / np.sqrt(nrm[pos])
    return (qr * inv[:, None]).astype(np.float32)


def ivf_pq_cosine_search(centers_rot, rotation, pq_centers, list_offsets, codes, ids, queries, n_probes, k, **kw):
    """oracle.ivf_pq_search with the reference's cosine semantics (see the module docstring)."""
    cr = np.asarray(centers_rot, np.float32)
    return oracle.ivf_pq_search(cr, cr, np.eye(cr.shape[1], dtype=np.float32), pq_centers, list_offsets, codes, ids,
                                unit_rotated_queries(rotation, queries), n_probes, k, "cosine", **kw)
