"""An IVF-Flat search in exact integer arithmetic, for 8-bit rows at widths where fp32 sums are not exact.

Probes are the `n_probes` best centres per query, scored in float64 in each metric's ranking form (as
tests/ivf_oracle.py::certain_probes scores them; on the queries it calls certain, every correct coarse search probes the same
lists).  Distances are exact int64: |q - x|^2 (sqeuclidean, euclidean) or q.x (inner_product), ranked by (distance, id), best
first, and returned rounded once to float32 (euclidean: the float32 square root of that).  Missing slots: (INT64_MAX, +-FLT_MAX)."""
import numpy as np

I64_MAX = np.iinfo(np.int64).max
F32_MAX = np.finfo(np.float32).max


def probes(centers, qs, n_probes, metric):
    c, q = np.asarray(centers, np.float64), np.asarray(qs, np.float64)
    score = -(q @ c.T) if metric == "inner_product" else (c * c).sum(1)[None, :] - 2.0 * (q @ c.T)
    return np.argsort(score, axis=1, kind="stable")[:, :n_probes]


def int_ivf_search(centers, offsets, rows, ids, qs, n_probes, k, metric):
    """rows [n, dim] (integers, list-major as `offsets` [n_lists + 1] and `ids` [n] give them) -> (dist f32, ids i64) [nq, k]."""
    x = np.asarray(rows, np.int64)
    q = np.asarray(qs, np.int64)
    ip = metric == "inner_product"
    out_d = np.full((len(q), k), -F32_MAX if ip else F32_MAX, np.float32)
    out_i = np.full((len(q), k), I64_MAX, np.int64)
    for j, pr in enumerate(probes(centers, qs, n_probes, metric)):
        sel = np.concatenate([np.arange(offsets[l], offsets[l + 1]) for l in pr])
        if len(sel) == 0:
            continue
        xs = x[sel]
        exact = xs @ q[j] if ip else ((xs - q[j]) ** 2).sum(1)
        order = np.lexsort((ids[sel], -exact if ip else exact))[:k]
        d = exact[order].astype(np.float32)
        if metric == "euclidean":
            d = np.sqrt(d)
        out_d[j, :len(order)] = d
        out_i[j, :len(order)] = ids[sel][order]
    return out_d, out_i
