"""The code-streaming IVF-PQ scan (scan_pq.cu) under maximum candidate pressure.

64- and 128-query work items put the queries on the MMA's M side and filter a fragment of 2 query rows x 16 / 32 list rows
per thread, reserving a query row's buffer slots with one atomic; 32-query items keep the list rows on M and test every
element on its own.  Without the cross-probe pruning bound (CUVS_B200_PQ_NO_BOUND=1) every item starts from an empty
threshold, so every row of the first tiles is a hit, candidate buffers overflow on every tile and are compacted over and
over, and the overflow path (slots past the buffer's end, re-tested after compaction) carries most of the work.  The
per-(query, probe) lists are exact top-KC selections, so both orientations must return the same neighbours."""
import os

import numpy as np
import pytest
import torch

from tests.util import clustered

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def stream_index():
    from cuvs_b200.neighbors import ivf_pq
    ds, centers = clustered(40000, 128, 25, n_centers=64)
    qs, _ = clustered(512, 128, 26, centers=centers)
    index = ivf_pq.build(ivf_pq.IndexParams(n_lists=64, pq_dim=64, kmeans_n_iters=10), torch.from_numpy(ds).cuda())
    return ds, qs, index


def _search(index, qs, k, group, lut):
    from cuvs_b200.neighbors import ivf_pq
    env = {"CUVS_B200_PQ_PATH": "stream", "CUVS_B200_PQ_GROUP": str(group), "CUVS_B200_PQ_NO_BOUND": "1"}
    old = {name: os.environ.get(name) for name in env}
    os.environ.update(env)
    try:
        kw = {} if lut == "f32" else {"lut_dtype": np.float16}
        d, i = ivf_pq.search(ivf_pq.SearchParams(n_probes=8, **kw), index, torch.from_numpy(qs).cuda(), k)
        return d.cpu().numpy(), i.cpu().numpy()
    finally:
        for name, v in old.items():
            if v is None:
                del os.environ[name]
            else:
                os.environ[name] = v


# f16 LUT -> one bf16 pass, f32 LUT -> two passes (hi + lo residual planes).  Group 128 serves k <= 16 with one pass only;
# for k = 32 or two passes the library narrows it to 64, so it is not run again there.
@pytest.mark.parametrize("lut", ["f16", "f32"])
@pytest.mark.parametrize("k", [10, 32])
def test_queries_on_m_match_rows_on_m_without_the_bound(stream_index, k, lut):
    ds, qs, index = stream_index
    assert index.streamed
    groups = (32, 64, 128) if (k <= 16 and lut == "f16") else (32, 64)
    res = {g: _search(index, qs, k, g, lut) for g in groups}
    d32, i32 = res[32]
    assert all(len(set(r.tolist())) == k for r in i32) and (i32 >= 0).all() and (i32 < len(ds)).all()
    for g in groups[1:]:
        d, i = res[g]
        same = (i == i32).mean()
        assert same >= 0.999, (g, same)
        np.testing.assert_allclose(d, d32, rtol=1e-5, atol=1e-5)
