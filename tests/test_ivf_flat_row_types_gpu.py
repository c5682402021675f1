"""IVF-Flat on int8 and uint8 rows kept in their own type (DESIGN.md §4 "Row types").

In L2 and inner product an 8-bit index stores its list rows as bytes with one exact integer norm each, and scans them on the
integer tensor cores: every score is exact, so the search returns the exact k nearest of the probed lists, ordered by
(distance, id), each distance the exact integer one rounded once to float32.  Up to d = 128 that is the oracle's fp32 answer
bit for bit; at wider rows, where fp32 sums round, it is checked against an int64 search (tests/ivf_int_ref.py).  Results are
compared on the queries whose probe set is certain (tests/ivf_oracle.py::certain_probes)."""
import os

import numpy as np
import pytest
import torch

import oracle
from tests.ivf_int_ref import int_ivf_search
from tests.ivf_oracle import assert_same_answer, certain_probes, check_rows, flat_lists, flat_search
from tests.util import last_flagged

pytestmark = pytest.mark.gpu

METRICS = ["sqeuclidean", "euclidean", "inner_product"]
DTYPES = {"i8": np.int8, "u8": np.uint8}


def _mod():
    from cuvs_b200.neighbors import ivf_flat
    return ivf_flat


def _rows(dtype, n, d, seed, n_centers=12, spread=10.0):
    """Clustered integer rows of the type's full range; every eighth row repeats an earlier one (exact ties)."""
    rng = np.random.default_rng(seed)
    lo, hi = (-128, 127) if dtype == np.int8 else (0, 255)
    centers = rng.uniform(lo + 40, hi - 40, (n_centers, d))
    x = np.clip(np.rint(centers[rng.integers(0, n_centers, n)] + spread * rng.standard_normal((n, d))), lo, hi)
    x[7::8] = x[rng.integers(0, n // 2, len(x[7::8]))]
    return x.astype(dtype)


_CACHE = {}


def _case(tag, d, metric, n=6000, nq=48, n_lists=16, spread=10.0):
    key = (tag, d, metric, n)
    if key not in _CACHE:
        m = _mod()
        dtype = DTYPES[tag]
        ds = _rows(dtype, n, d, 11 + d, spread=spread)
        qs = _rows(dtype, nq, d, 12 + d, spread=spread)
        index = m.build(m.IndexParams(n_lists=n_lists, metric=metric, kmeans_n_iters=10), torch.from_numpy(ds).cuda())
        _CACHE[key] = (ds, qs, index)
    return _CACHE[key]


def _search(index, qs, n_probes, k, **kw):
    m = _mod()
    d, i = m.search(m.SearchParams(n_probes=n_probes), index, torch.from_numpy(qs).cuda(), k, **kw)
    return d.cpu().numpy(), i.cpu().numpy()


def _f32(a):
    return np.asarray(a, np.float32)


# ------------------------------------------------------------------------------------------- 1. the oracle, up to d = 128
@pytest.mark.parametrize("d", [16, 33, 128])
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("tag", ["i8", "u8"])
def test_exact_against_the_oracle(tag, metric, d):
    """Every k regime: fused lists of 16 and 32 (k <= 16, <= 32), the store scan and segmented select above."""
    ds, qs, index = _case(tag, d, metric)
    n_probes = 5
    sure = certain_probes(index.centers.cpu().numpy(), _f32(qs), n_probes, metric)
    assert sure.mean() >= 0.5
    for k in (1, 10, 32, 33, 64, 100, 256, 2048):
        dist, idx = _search(index, qs, n_probes, k)
        assert last_flagged() == 0
        rd, ri = flat_search(index, _f32(ds), _f32(qs), n_probes, k, metric)
        assert_same_answer(dist[sure], idx[sure], rd[sure], ri[sure])
        check_rows(idx, len(ds))


# ------------------------------------------------------------------------------------- 2. wide rows: exact integers
@pytest.mark.parametrize("d", [512, 1024, 2048])
@pytest.mark.parametrize("metric", METRICS)
def test_wide_rows_exact_integers(metric, d):
    """uint8 up to 255: |q - x|^2 and q.x pass 2^24, where fp32 sums round; distances must be float32(exact) bit for bit."""
    ds, qs, index = _case("u8", d, metric, n=3000, nq=32, n_lists=8, spread=60.0)
    n_probes = 3
    sure = certain_probes(index.centers.cpu().numpy(), _f32(qs), n_probes, metric)
    assert sure.mean() >= 0.5
    offsets, ids = flat_lists(index)
    for k in (10, 32, 100):
        dist, idx = _search(index, qs, n_probes, k)
        rd, ri = int_ivf_search(index.centers.cpu().numpy(), offsets, ds[ids], ids, qs, n_probes, k, metric)
        assert_same_answer(dist[sure], idx[sure], rd[sure], ri[sure])
    if d == 2048:
        big = np.abs(rd[sure][ri[sure] != np.iinfo(np.int64).max]).astype(np.float64)
        assert (big ** 2 if metric == "euclidean" else big).max() > 2 ** 24, "the case does not reach inexact fp32 sums"


# ---------------------------------------------------------------------------------------------------- 3. exact ties
@pytest.mark.parametrize("tag", ["i8", "u8"])
def test_heavy_ties(tag):
    """300 base rows, each 40 times: half exact copies, half one step away in one component."""
    m = _mod()
    dtype = DTYPES[tag]
    rng = np.random.default_rng(31)
    base = _rows(dtype, 300, 128, 32).astype(np.int64)
    x = np.repeat(base, 40, axis=0)
    step = np.arange(len(x)) % 2 == 1
    col = rng.integers(0, 128, len(x))
    lo, hi = (-128, 127) if dtype == np.int8 else (0, 255)
    x[np.arange(len(x)), col] += np.where(step, np.where(x[np.arange(len(x)), col] < hi, 1, -1), 0)
    ds = np.clip(x, lo, hi).astype(dtype)
    qs = base[rng.choice(300, 40, replace=False)].astype(dtype)
    index = m.build(m.IndexParams(n_lists=8, kmeans_n_iters=10), torch.from_numpy(ds).cuda())
    sure = certain_probes(index.centers.cpu().numpy(), _f32(qs), 3, "sqeuclidean")
    for k in (10, 32, 40, 64, 256):
        dist, idx = _search(index, qs, 3, k)
        rd, ri = flat_search(index, _f32(ds), _f32(qs), 3, k, "sqeuclidean")
        assert_same_answer(dist[sure], idx[sure], rd[sure], ri[sure])
        check_rows(idx, len(ds))


# ------------------------------------------------------------------------------------------------- 4. bitset filter
@pytest.mark.parametrize("k", [10, 48, 256])
@pytest.mark.parametrize("tag", ["i8", "u8"])
def test_bitset_filter(tag, k):
    from cuvs_b200.neighbors import filters
    ds, qs, index = _case(tag, 128, "sqeuclidean")
    n = len(ds)
    keep = np.random.default_rng(88).random(n) < 0.3
    bits = np.packbits(np.concatenate([keep, np.zeros((-n) % 32, bool)]), bitorder="little").view(np.uint32)
    dist, idx = _search(index, qs, 5, k, filter=filters.from_bitset(torch.from_numpy(bits.view(np.int32)).cuda()))
    valid = idx != np.iinfo(np.int64).max
    assert keep[idx[valid]].all(), "a filtered-out row was returned"
    rd, ri = flat_search(index, _f32(ds), _f32(qs), 5, k, "sqeuclidean", keep)
    sure = certain_probes(index.centers.cpu().numpy(), _f32(qs), 5, "sqeuclidean")
    assert_same_answer(dist[sure], idx[sure], rd[sure], ri[sure])


# --------------------------------------------------------------------------- 5. build == empty build + two extends
@pytest.mark.parametrize("tag", ["i8", "u8"])
def test_extends_write_the_same_file(tag, tmp_path):
    m = _mod()
    ds = _rows(DTYPES[tag], 5000, 40, 51)
    params = dict(n_lists=16, metric="inner_product", kmeans_n_iters=10)
    full = m.build(m.IndexParams(**params), torch.from_numpy(ds).cuda())
    empty = m.build(m.IndexParams(add_data_on_build=False, **params), torch.from_numpy(ds).cuda())
    m.extend(empty, torch.from_numpy(ds[:3000]).cuda(), None)
    m.extend(empty, torch.from_numpy(ds[3000:]), None)  # host rows
    m.save(tmp_path / "a.bin", full)
    m.save(tmp_path / "b.bin", empty)
    assert (tmp_path / "a.bin").read_bytes() == (tmp_path / "b.bin").read_bytes()


# ------------------------------------------------------------------------------------------------------- 6. memory
def test_a_uint8_build_holds_bytes():
    """Two builds: the first fills the stream-ordered pool that the build's temporaries come from, the second is measured."""
    m = _mod()
    n, d = 400000, 128
    ds = torch.from_numpy(_rows(np.uint8, n, d, 61)).cuda()
    params = m.IndexParams(n_lists=256, kmeans_n_iters=5)
    del_me = m.build(params, ds)
    del del_me
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    index = m.build(params, ds)
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    rows = int(sum(-(-int(s) // 128) * 128 for s in index.list_sizes.cpu().numpy()))
    expect = rows * (128 + 12)
    fp32_layout = n * (512 + 256 + 32 + 4 + 4 + 8)
    assert free0 - free1 <= expect + (16 << 20), (free0 - free1, expect)
    assert free0 - free1 < fp32_layout // 4


# -------------------------------------------------------------------------------------------------------- 7. files
def _records(path):
    out = []
    with open(path, "rb") as f:
        tag = f.read(4)
        size = os.fstat(f.fileno()).st_size
        while f.tell() < size:
            out.append(np.lib.format.read_array(f, allow_pickle=False))
    return tag, out


TAGS = {np.float32: b"<f4\0", np.float16: b"<e2\0", np.int8: b"|i1\0", np.uint8: b"|u1\0"}
TORCH = {np.float32: torch.float32, np.float16: torch.float16, np.int8: torch.int8, np.uint8: torch.uint8}


def _typed_rows(dtype, n, d, seed):
    if dtype in (np.int8, np.uint8):
        return _rows(dtype, n, d, seed)
    return (np.random.default_rng(seed).standard_normal((n, d)) * 4).astype(dtype)


def _write_file(path, tag, recs):
    with open(path, "wb") as f:
        f.write(tag)
        for r in recs:
            np.lib.format.write_array(f, np.asarray(r), allow_pickle=False)


@pytest.mark.parametrize("dtype", [np.float32, np.float16, np.int8, np.uint8], ids=lambda t: np.dtype(t).name)
@pytest.mark.parametrize("d", [40, 33])
def test_index_files(dtype, d, tmp_path):
    m = _mod()
    ds = _typed_rows(dtype, 3000, d, 71)
    qs = _typed_rows(dtype, 30, d, 72)
    index = m.build(m.IndexParams(n_lists=8, kmeans_n_iters=10), torch.from_numpy(ds).cuda())
    m.save(tmp_path / "i.bin", index)
    tag, recs = _records(tmp_path / "i.bin")
    assert tag == TAGS[dtype]
    n_lists = int(recs[3])
    sizes = recs[10]
    offsets, ids = flat_lists(index)
    at = 11
    for l in range(n_lists):
        cap = int(recs[at])
        assert cap == -(-int(sizes[l]) // 32) * 32
        at += 1
        if cap == 0:
            continue
        data, lid = recs[at], recs[at + 1]
        at += 2
        assert data.dtype == np.dtype(dtype) and data.shape == (cap, d)
        rows = ds[ids[offsets[l]:offsets[l + 1]]]
        np.testing.assert_array_equal(data.ravel(), oracle.interleave_ivf_flat(rows))
        np.testing.assert_array_equal(lid[:sizes[l]], ids[offsets[l]:offsets[l + 1]])
    assert at == len(recs)
    q = torch.from_numpy(qs).cuda()
    want = _search(index, qs, 3, 20)
    loaded = m.load(tmp_path / "i.bin")
    got = _search(loaded, qs, 3, 20)
    np.testing.assert_array_equal(got[0].view(np.uint32), want[0].view(np.uint32))
    np.testing.assert_array_equal(got[1], want[1])
    # the same file assembled by NumPy, float16 as the reference's kind 'e'
    _write_file(tmp_path / "np.bin", TAGS[dtype], recs)
    got = _search(m.load(tmp_path / "np.bin"), qs, 3, 20)
    np.testing.assert_array_equal(got[1], want[1])
    np.testing.assert_array_equal(got[0].view(np.uint32), want[0].view(np.uint32))
    # a data record of another type, and an unknown tag, are refused
    other = np.float32 if dtype != np.float32 else np.int8
    bad = [r.astype(other) if r.ndim == 2 and r.shape[1] == d and i > 10 else r for i, r in enumerate(recs)]
    _write_file(tmp_path / "bad.bin", TAGS[dtype], bad)
    with pytest.raises(Exception):
        m.load(tmp_path / "bad.bin")
    _write_file(tmp_path / "tag.bin", b"<c8\0", recs)
    with pytest.raises(Exception):
        m.load(tmp_path / "tag.bin")
    # queries of another type are refused
    with pytest.raises(Exception):
        m.search(m.SearchParams(n_probes=3), loaded, q.to(torch.float32 if dtype != np.float32 else torch.int8), 5)
