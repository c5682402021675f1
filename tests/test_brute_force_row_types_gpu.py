"""Brute-force indexes over float16, int8 and uint8 rows keep the rows in their own type (fp16 and integer tensor-core scans,
DESIGN.md §3 "Row types") and answer exactly as the oracle does over the widened fp32 values."""
import ctypes as C
import struct

import numpy as np
import pytest
import torch

import oracle
from tests.util import clustered, last_flagged

pytestmark = pytest.mark.gpu

TYPES = [np.float16, np.int8, np.uint8]
METRICS = ["sqeuclidean", "euclidean", "l2_unexpanded", "l2_sqrt_unexpanded", "inner_product", "cosine"]
ROW_TYPE = {np.float32: 0, np.float16: 1, np.int8: 2, np.uint8: 3}


def _bf():
    from cuvs_b200.neighbors import brute_force
    return brute_force


def _rows(dtype, n, d, seed):
    """Values over the type's whole range (8-bit: every byte value, so that fp32 sums round at large d)."""
    rng = np.random.default_rng(seed)
    if dtype == np.float16:
        return rng.uniform(-4, 4, (n, d)).astype(np.float16)
    info = np.iinfo(dtype)
    return rng.integers(info.min, info.max + 1, (n, d), dtype=dtype)


def _search(index, q, k, **kw):
    d, i = _bf().search(index, torch.from_numpy(np.ascontiguousarray(q)).cuda(), k, **kw)
    return d.cpu().numpy(), i.cpu().numpy()


def _info(index):
    from cuvs_b200._capi import check, lib
    rt, nb = C.c_int(-1), C.c_int64(-1)
    check(lib.cuvsB200BruteForceIndexInfo(index._p, C.byref(rt), C.byref(nb)))
    return rt.value, nb.value


def _assert_oracle(ds, qs, k, metric, d, i):
    rd, ri = oracle.knn(ds.astype(np.float32), qs.astype(np.float32), k, metric)
    assert (i == ri).all(), f"{(i != ri).sum()} ids differ"
    assert d.tobytes() == rd.tobytes(), "distances differ"


@pytest.mark.parametrize("dim", [3, 48, 128, 129, 300, 1024, 2048, 2100])
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("dtype", TYPES)
def test_oracle_parity(dtype, metric, dim):
    bf = _bf()
    ds, qs = _rows(dtype, 1500, dim, 1), _rows(dtype, 40, dim, 2)
    index = bf.build(torch.from_numpy(ds).cuda(), metric=metric)
    assert _info(index)[0] == ROW_TYPE[dtype]
    for k in (1, 10, 32, 64, 100, 1024):
        d, i = _search(index, qs, k)
        _assert_oracle(ds, qs, k, metric, d, i)


@pytest.mark.parametrize("metric", ["sqeuclidean", "inner_product", "l2_unexpanded"])
def test_float16_index_with_float32_queries_of_extreme_magnitudes(metric):
    rng = np.random.default_rng(5)
    n, dim = 3000, 96
    ds = rng.uniform(-1, 1, (n, dim)).astype(np.float16)
    ds[:20] = np.float16(65504.0) * np.sign(rng.standard_normal((20, dim))).astype(np.float16)  # near +-65504
    ds[20:40] = (rng.integers(-1023, 1024, (20, dim)) * 2.0 ** -24).astype(np.float16)    # fp16 subnormals
    # each query spans 1e-7 .. 6e4 within its row; some rows are all tiny or all large
    qs = (np.sign(rng.standard_normal((64, dim))) * 10.0 ** rng.uniform(-7, np.log10(6e4), (64, dim))).astype(np.float32)
    qs[:4] *= 1e-6
    qs[4:8] = qs[4:8] / np.abs(qs[4:8]).max(1, keepdims=True) * 6e4
    index = _bf().build(torch.from_numpy(ds).cuda(), metric=metric)
    for k in (10, 64):
        d, i = _search(index, qs, k)
        _assert_oracle(ds, qs, k, metric, d, i)


@pytest.mark.parametrize("dtype", TYPES)
def test_same_answers_as_a_float32_index_of_the_widened_values(dtype):
    bf = _bf()
    base, centers = clustered(200000, 128, 7)
    qbase, _ = clustered(1000, 128, 8, centers=centers)
    if dtype == np.float16:
        ds, qs = base.astype(np.float16), qbase.astype(np.float16)
    else:
        info = np.iinfo(dtype)
        lo, hi = float(base.min()), float(base.max())
        scale = lambda x: np.clip(np.rint((x - lo) / (hi - lo) * (info.max - info.min) + info.min), info.min, info.max).astype(dtype)
        ds, qs = scale(base), scale(qbase)
    narrow = bf.build(torch.from_numpy(ds).cuda())
    wide = bf.build(torch.from_numpy(ds.astype(np.float32)).cuda())
    for k in (10, 64):
        d1, i1 = _search(narrow, qs, k)
        d2, i2 = _search(wide, qs.astype(np.float32), k)
        assert i1.tobytes() == i2.tobytes() and d1.tobytes() == d2.tobytes()


@pytest.mark.parametrize("dtype", TYPES)
def test_certificate_on_near_duplicates(dtype):
    bf = _bf()
    ds = _rows(dtype, 20000, 64, 11)
    qs = _rows(dtype, 256, 64, 12)
    ds[1000:1040] = ds[7]          # copies of a row
    ds[2000:2256] = qs             # copies of the queries
    ds[3000:3256] = qs
    ds[4000:4320] = np.repeat(qs[:16], 20, axis=0)  # 20 more copies of 16 queries: ties across the k-th place and the lists
    index = bf.build(torch.from_numpy(ds).cuda())
    d, i = _search(index, qs, 10)
    assert last_flagged() > 0
    _assert_oracle(ds, qs, 10, "sqeuclidean", d, i)


def _candidates(index, qs, kc=16):
    from cuvs_b200._capi import DL, check, lib
    from cuvs_b200.common import Resources
    q = torch.from_numpy(np.ascontiguousarray(qs)).cuda()
    pos = torch.zeros(len(qs), kc, dtype=torch.uint32, device="cuda")
    sc = torch.zeros(len(qs), kc, dtype=torch.float32, device="cuda")
    res, dq, dpos, dsc = Resources(), DL(q), DL(pos), DL(sc)  # alive until the call returns
    check(lib.cuvsB200BruteForceCandidates(res.get_c_obj(), index._p, dq.ptr, dpos.ptr, dsc.ptr))
    return pos.cpu().numpy().astype(np.int64), sc.cpu().numpy().astype(np.float64)


def test_float16_candidate_error_within_budget():
    base, centers = clustered(30000, 128, 21)
    qb, _ = clustered(256, 128, 22, centers=centers)
    ds, qs = base.astype(np.float16), qb.astype(np.float16)
    index = _bf().build(torch.from_numpy(ds).cuda())
    for q in (qs, qb):  # float16 queries (one pass) and float32 queries (scaled split)
        pos, s = _candidates(index, q)
        qd, xd = q.astype(np.float64), ds.astype(np.float64)
        qn = (qd ** 2).sum(1)
        exact = ((qd[:, None, :] - xd[pos]) ** 2).sum(-1)
        rel = np.abs(qn[:, None] + 2 * s - exact) / (qn[:, None] + (xd ** 2).sum(1).max())
        assert rel.max() < 2.0 ** -15 / 4, f"observed relative error {rel.max():.3e}"


@pytest.mark.parametrize("metric", ["sqeuclidean", "inner_product"])
@pytest.mark.parametrize("dtype", [np.int8, np.uint8])
def test_8bit_candidates_are_exact(dtype, metric):
    ds, qs = _rows(dtype, 20000, 100, 31), _rows(dtype, 128, 100, 32)
    index = _bf().build(torch.from_numpy(ds).cuda(), metric=metric)
    pos, s = _candidates(index, qs, 32)
    qd, xd = qs.astype(np.int64), ds.astype(np.int64)
    dot = np.einsum("qd,qcd->qc", qd, xd[pos])
    want = 0.5 * (xd[pos] ** 2).sum(-1) - dot if metric == "sqeuclidean" else -dot
    assert (s == want).all()


def _keep_words(keep):
    flat = np.asarray(keep, bool).ravel()
    pad = np.zeros((flat.size + 31) // 32 * 32, bool)
    pad[:flat.size] = flat
    words = np.packbits(pad.reshape(-1, 32)[:, ::-1], axis=1, bitorder="big").view(">u4").astype(np.uint32).ravel()
    return torch.from_numpy(words.view(np.int32)).cuda().view(torch.uint32)


@pytest.mark.parametrize("dtype", TYPES)
def test_filters_and_large_k(dtype):
    from cuvs_b200.neighbors import filters
    n, nq, dim = 3000, 30, 40
    ds, qs = _rows(dtype, n, dim, 41), _rows(dtype, nq, dim, 42)
    index = _bf().build(torch.from_numpy(ds).cuda())
    rng = np.random.default_rng(43)
    keep = rng.random(n) < 0.6
    d, i = _search(index, qs, 20, prefilter=filters.from_bitset(_keep_words(keep)))
    kept = np.flatnonzero(keep)
    rd, ri = oracle.knn(ds[kept].astype(np.float32), qs.astype(np.float32), 20)
    assert (i == kept[ri]).all() and d.tobytes() == rd.tobytes()
    # bitmap: one row of n bits per query
    km = rng.random((nq, n)) < 0.5
    d, i = _search(index, qs, 10, prefilter=filters.from_bitmap(_keep_words(km)))
    for r in range(nq):
        kr = np.flatnonzero(km[r])
        rd, ri = oracle.knn(ds[kr].astype(np.float32), qs[r:r + 1].astype(np.float32), 10)
        assert (i[r] == kr[ri[0]]).all() and d[r].tobytes() == rd[0].tobytes()
    d, i = _search(index, qs, 200)
    _assert_oracle(ds, qs, 200, "sqeuclidean", d, i)


@pytest.mark.parametrize("metric", ["sqeuclidean", "inner_product", "cosine"])
@pytest.mark.parametrize("dtype", TYPES + [np.float32])
def test_index_files_keep_the_row_type(tmp_path, dtype, metric):
    from cuvs_b200._capi import CuvsError
    bf = _bf()
    ds = _rows(dtype, 2000, 40, 51) if dtype != np.float32 else np.random.default_rng(51).standard_normal((2000, 40)).astype(np.float32)
    qs = ds[:50].copy()
    index = bf.build(torch.from_numpy(ds).cuda(), metric=metric)
    path = tmp_path / "bf.bin"
    bf.save(path, index)
    loaded = bf.load(path)
    assert _info(loaded)[0] == ROW_TYPE[dtype] == _info(index)[0]
    for q in (qs, qs.astype(np.float32), qs.astype(np.float16)):
        results = []
        for ix in (index, loaded):
            try:
                results.append(_search(ix, q, 10))
            except CuvsError as e:
                results.append(str(e))
        if isinstance(results[0], str):
            assert results[0] == results[1]
        else:
            assert all(a.tobytes() == b.tobytes() for a, b in zip(*results))
    if dtype == np.float32:  # the float32 layout, field by field
        raw = path.read_bytes()
        assert raw[:4] == b"<f4\0"
        assert struct.unpack("<qqif", raw[4:28]) == (2000, 40, oracle.METRICS[metric], 2.0)
        assert raw[28:] == ds.tobytes() and len(raw) == 28 + ds.nbytes
    else:
        tag = {np.float16: b"<f2\0", np.int8: b"|i1\0", np.uint8: b"|u1\0"}[dtype]
        raw = path.read_bytes()
        assert raw[:4] == tag and raw[28:] == ds.tobytes()


@pytest.mark.parametrize("metric", ["sqeuclidean", "inner_product"])
@pytest.mark.parametrize("dtype", TYPES)
def test_device_bytes(dtype, metric):
    n, dim = 10000, 128
    index = _bf().build(torch.from_numpy(_rows(dtype, n, dim, 61)).cuda(), metric=metric)
    rows_pad = (n + 127) // 128 * 128
    kp = (dim + 63) // 64 * 64 if dtype == np.float16 else (dim + 127) // 128 * 128
    per_row = (2 * kp if dtype == np.float16 else kp) + 48
    nbytes = _info(index)[1]
    assert nbytes <= per_row * rows_pad
    assert nbytes <= 1060 * n / 3  # the widened index: 512 + 512 + 32 + 4 bytes per row at d = 128


@pytest.mark.parametrize("dtype", TYPES)
def test_side_stream(dtype):
    from tests.test_streams_gpu import check_side_stream
    bf = _bf()
    ds, qs = _rows(dtype, 12000, 64, 71), _rows(dtype, 300, 64, 72)

    def fn(res, ds, qs):
        return bf.search(bf.build(ds, resources=res), qs, 10, resources=res)
    check_side_stream(f"brute_force {np.dtype(dtype).name}", fn, ds=torch.from_numpy(ds).cuda(), qs=torch.from_numpy(qs).cuda())
