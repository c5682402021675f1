"""GPU: the four search entry points (brute force, IVF-Flat, IVF-PQ, CAGRA) refuse the same malformed queries / neighbors /
distances with the same message, and the three that take a pre-filter read only a device 1-D uint32 tensor as one, as the
reference's from_dlpack<device_vector_view<uint32_t>> does."""
import pytest
import torch

from cuvs_b200._capi import DL, CuvsError
from cuvs_b200.neighbors import brute_force, cagra, filters, ivf_flat, ivf_pq
from tests.util import uniform

pytestmark = pytest.mark.gpu

N, DIM, NQ, K = 4000, 16, 8, 5
N_WORDS = (N + 31) // 32


@pytest.fixture(scope="module")
def indexes():
    ds = torch.from_numpy(uniform(N, DIM, 1)).cuda()
    return {
        "brute_force": brute_force.build(ds),
        "ivf_flat": ivf_flat.build(ivf_flat.IndexParams(n_lists=8), ds),
        "ivf_pq": ivf_pq.build(ivf_pq.IndexParams(n_lists=8, pq_dim=8), ds),
        "cagra": cagra.build(cagra.IndexParams(graph_degree=16, intermediate_graph_degree=32), ds),
    }


def _search(name, index, queries, neighbors, distances, prefilter=None):
    if name == "brute_force":
        return brute_force.search(index, queries, K, neighbors, distances, prefilter=prefilter)
    if name == "ivf_flat":
        return ivf_flat.search(ivf_flat.SearchParams(n_probes=8), index, queries, K, neighbors, distances, filter=prefilter)
    if name == "ivf_pq":
        assert prefilter is None
        return ivf_pq.search(ivf_pq.SearchParams(n_probes=8), index, queries, K, neighbors, distances)
    return cagra.search(cagra.SearchParams(itopk_size=32), index, queries, K, neighbors, distances, filter=prefilter)


def _queries(dim=DIM):
    return torch.from_numpy(uniform(NQ, dim, 2)).cuda()


def _neighbors(k=K, device="cuda"):
    return torch.empty((NQ, k), dtype=torch.int64, device=device)


def _distances(dtype=torch.float32):
    return torch.empty((NQ, K), dtype=dtype, device="cuda")


BAD = {
    "host neighbors": (lambda: (_queries(), _neighbors(device="cpu"), _distances()), "neighbors should have device compatible memory"),
    "float64 distances": (lambda: (_queries(), _neighbors(), _distances(torch.float64)), "distances should be of type float32"),
    "1-D queries": (lambda: (_queries()[0].contiguous(), _neighbors(), _distances()), "queries/neighbors/distances must be 2-D"),
    "query dim": (lambda: (_queries(DIM - 3), _neighbors(), _distances()), r"queries dim \(13\) != index dim \(16\)"),
    "k mismatch": (lambda: (_queries(), _neighbors(K + 1), _distances()), "neighbors/distances shape mismatch"),
    "non-contiguous neighbors": (lambda: (_queries(), torch.empty((K, NQ), dtype=torch.int64, device="cuda").t(), _distances()),
                                 "neighbors/distances must be row-major contiguous"),
}


@pytest.mark.parametrize("case", list(BAD))
@pytest.mark.parametrize("name", ["brute_force", "ivf_flat", "ivf_pq", "cagra"])
def test_malformed_search_tensors_are_refused_alike(indexes, name, case):
    make, msg = BAD[case]
    with pytest.raises(CuvsError, match=msg):
        _search(name, indexes[name], *make())


def _raw_bitset(t):
    """A BITSET pre-filter around `t` as given (filters.from_bitset converts other dtypes to uint32 words)."""
    f = filters.Prefilter(filters.BITSET)
    f._dl = DL(t)
    return f


@pytest.mark.parametrize("name", ["brute_force", "ivf_flat", "cagra"])
def test_prefilter_must_be_a_1d_uint32_tensor(indexes, name):
    # Every row kept.  The uint8 bitset covers all N rows in a whole number of uint32 words, so a reader that takes its
    # byte count for a word count still reads inside it.
    u8 = torch.full((N_WORDS * 4,), 0xFF, dtype=torch.uint8, device="cuda")
    u32_2d = torch.full((2, N_WORDS), -1, dtype=torch.int32, device="cuda").view(torch.uint32)
    for bad in (_raw_bitset(u8), filters.from_bitset(u32_2d)):
        with pytest.raises(CuvsError, match="prefilter must be a contiguous 1-D uint32 tensor"):
            _search(name, indexes[name], _queries(), _neighbors(), _distances(), prefilter=bad)
    u32 = torch.full((N_WORDS,), -1, dtype=torch.int32, device="cuda").view(torch.uint32)
    _, nb = _search(name, indexes[name], _queries(), _neighbors(), _distances(), prefilter=filters.from_bitset(u32))
    nb = nb.cpu()
    assert ((nb >= 0) & (nb < N)).all()
