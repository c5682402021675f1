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


def check_rows(i, n=None):
    """No id twice in a row of `i` (empty slots hold INT64_MAX); with `n`, every real id in [0, n)."""
    for row in i:
        real = row[row != I64_MAX]
        assert len(np.unique(real)) == len(real), "an id is returned twice in one row"
        if n is not None:
            assert ((real >= 0) & (real < n)).all()
