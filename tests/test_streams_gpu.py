"""Every entry point on a side stream, on two streams at once, and from concurrent threads (DESIGN.md "Streams and concurrent
callers").

pytest runs on the legacy default stream, which orders itself against every blocking stream, so the rest of the suite cannot see
a kernel queued on the wrong stream, a missing dependency between two streams, or state one call leaves in an index for the
next.  Here each call runs under ``torch.cuda.stream(S)`` on a non-blocking pool stream, and every input it reads arrives late on
S: ``late`` fills the destination with poison, sleeps the stream, and only then copies the real values in.  A reader on any other
stream sees the poison (checked by ``test_harness_catches_a_wrong_stream_reader``).  Each result must equal, bit for bit, the
same call made serially on the default stream, which the rest of the suite checks against the oracle; the serial call is run
twice, and an entry point that does not repeat itself bit for bit is compared at a tolerance instead, with a warning naming it.
CAGRA search does not repeat itself bit for bit on an H100 (a few of 3000 neighbours differ between two serial searches of one
index), so CAGRA results are always compared at the tolerance: 95% of each row's neighbours shared, no poison, no NaN.
"""
import ctypes as C
import threading
import warnings

import numpy as np
import pytest
import torch

from cuvs_b200._capi import DL, DLManagedTensor, check, lib
from cuvs_b200.cluster import kmeans
from cuvs_b200.common.resources import Resources
from cuvs_b200.neighbors import brute_force, cagra, filters, ivf_flat, ivf_pq, nn_descent
from cuvs_b200.neighbors.refine import refine
from tests.util import clustered, uniform

pytestmark = pytest.mark.gpu

SLEEP_CYCLES = 100_000_000  # ~50-60 ms at H100 clocks; test_harness_catches_a_wrong_stream_reader checks it on the machine


# ------------------------------------------------------------------------------------------------------------- harness
def _fillable(t):
    return t.view(torch.int32) if t.dtype == torch.uint32 else t


def _poison(t):
    if t.dtype.is_floating_point:
        return float("nan")
    if t.dtype in (torch.int8, torch.uint8):
        return 0x5A
    if t.dtype == torch.uint32:  # filter words: every row filtered out
        return 0
    return -1  # ids and candidates


def late(src, S, cycles=SLEEP_CYCLES):
    """A copy of device tensor `src` that is complete on stream S only after a sleep; until then it holds poison."""
    S.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(S):
        dst = torch.empty_like(src)
        _fillable(dst).fill_(_poison(dst))
        dst._poisoned = torch.cuda.Event()
        dst._poisoned.record(S)
        torch.cuda._sleep(cycles)
        _fillable(dst).copy_(_fillable(src))
    return dst


def _host(out):
    if isinstance(out, (tuple, list)):
        return [a for o in out for a in _host(o)]
    if isinstance(out, torch.Tensor):
        return [_fillable(out).cpu().numpy()]
    return [np.asarray(out)]


def _same_bits(a, b):
    return len(a) == len(b) and all(x.shape == y.shape and x.dtype == y.dtype and x.tobytes() == y.tobytes() for x, y in zip(a, b))


def _tolerance_equal(name, ref, got):
    """For results that are not bit-repeatable: no NaN where the serial run has none, 95% of the floats within 1e-4 relative, and
    95% of each row's integers (neighbour ids, labels) shared with the serial row."""
    for r, g in zip(ref, got):
        assert r.shape == g.shape and r.dtype == g.dtype, name
        if np.issubdtype(r.dtype, np.floating):
            assert not (np.isnan(g) & ~np.isnan(r)).any(), f"{name}: NaN (poison) in the result"
            close = np.isclose(g, r, rtol=1e-4, atol=0, equal_nan=True)
            assert close.mean() >= 0.95, f"{name}: {1 - close.mean():.3f} of the values differ"
        else:
            r2, g2 = r.reshape(len(r), -1) if r.ndim else r.reshape(1, 1), g.reshape(len(g), -1) if g.ndim else g.reshape(1, 1)
            shared = np.mean([len(np.intersect1d(a, b)) / max(len(np.unique(a)), 1) for a, b in zip(r2, g2)])
            assert shared >= 0.95, f"{name}: only {shared:.3f} of each row's entries shared with the serial result"


def serial(fn, inputs):
    """fn's result run on the default stream, twice; the flag says whether the two runs agree bit for bit."""
    outs = []
    for _ in range(2):
        torch.cuda.synchronize()
        outs.append(_host(fn(Resources(), **inputs)))
        torch.cuda.synchronize()
    return outs[0], _same_bits(outs[0], outs[1])


def compare(name, ref, repeats, got, exact=True):
    if repeats and exact:
        assert _same_bits(ref, got), f"{name}: the side-stream result differs from the serial one"
    else:
        if exact:
            warnings.warn(f"{name}: two serial runs differ; compared at a tolerance")
        _tolerance_equal(name, ref, got)


def check_side_stream(name, fn, exact=True, **inputs):
    """fn(res, **inputs) on stream S with every device tensor input arriving late, against the serial result."""
    ref, repeats = serial(fn, inputs)
    S = torch.cuda.Stream()
    lated = {k: late(v, S) if isinstance(v, torch.Tensor) and v.is_cuda else v for k, v in inputs.items()}
    with torch.cuda.stream(S):
        out = fn(Resources(), **lated)
    S.synchronize()
    compare(name, ref, repeats, _host(out), exact)


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _bits_of(keep):
    """uint32 words (as a torch uint32 tensor) of a boolean keep mask, bit = 1 keeps."""
    flat = np.asarray(keep, bool).ravel()
    pad = np.zeros((flat.size + 31) // 32 * 32, bool)
    pad[:flat.size] = flat
    words = np.packbits(pad.reshape(-1, 32)[:, ::-1], axis=1, bitorder="big").view(">u4").astype(np.uint32).ravel()
    return _cuda(words.view(np.int32)).view(torch.uint32)


@pytest.fixture(scope="module")
def data():
    ds, centers = clustered(12000, 64, 31)
    qs, _ = clustered(300, 64, 32, centers=centers)
    extra, _ = clustered(2000, 64, 33, centers=centers)
    return {"ds": _cuda(ds), "qs": _cuda(qs), "extra": _cuda(extra),
            "extra_ids": torch.arange(50000, 52000, dtype=torch.int64, device="cuda")}


# --------------------------------------------------------------------------------------------------- harness self-check
def _stream_flags(stream):
    flags = C.c_uint(0)
    try:
        rt = C.CDLL("libcudart.so.12")
        err = rt.cudaStreamGetFlags(C.c_void_p(stream.cuda_stream), C.byref(flags))
    except OSError:
        drv = C.CDLL("libcuda.so.1")
        err = drv.cuStreamGetFlags(C.c_void_p(stream.cuda_stream), C.byref(flags))
    assert err == 0
    return flags.value


def test_harness_catches_a_wrong_stream_reader():
    S = torch.cuda.Stream()
    assert _stream_flags(S) & 1, "torch's pool streams should be non-blocking (cudaStreamNonBlocking)"
    src = torch.arange(1 << 20, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record(S)
    d = late(src, S)
    end.record(S)
    # a reader on the default stream that waits for nothing but the allocation sees the poison
    torch.cuda.current_stream().wait_event(d._poisoned)
    seen = d.clone()
    torch.cuda.current_stream().synchronize()
    assert torch.isnan(seen).all(), "the sleep ended before a wrong-stream reader ran: raise SLEEP_CYCLES"
    S.synchronize()
    assert torch.equal(d, src)
    slept = start.elapsed_time(end)
    assert slept >= 20.0, f"the late copy arrives only {slept:.1f} ms after it is queued"


# ---------------------------------------------------------------------------------------------- A. late inputs on S
@pytest.mark.parametrize("metric", ["sqeuclidean", "inner_product"])
@pytest.mark.parametrize("k", [10, 48])
def test_brute_force_side_stream(data, metric, k):
    def fn(res, ds, qs):
        idx = brute_force.build(ds, metric=metric, resources=res)
        return brute_force.search(idx, qs, k, resources=res)
    check_side_stream(f"brute_force {metric} k={k}", fn, ds=data["ds"], qs=data["qs"])


def test_brute_force_certified_fallback_side_stream():
    """Every row 40 times: exact ties beyond the candidate lists send every query through the fallback (a host sync, then
    copy_rows of the flagged queries)."""
    ds = np.tile(uniform(64, 128, 5), (40, 1))
    qs = uniform(32, 128, 6)

    def fn(res, ds, qs):
        return brute_force.search(brute_force.build(ds, resources=res), qs, 10, resources=res)
    check_side_stream("brute_force fallback", fn, ds=_cuda(ds), qs=_cuda(qs))


@pytest.mark.parametrize("kind", ["bitset", "bitmap"])
def test_brute_force_filters_side_stream(data, kind):
    n, nq = data["ds"].shape[0], data["qs"].shape[0]
    rng = np.random.default_rng(7)
    words = _bits_of(rng.random(n) < 0.5) if kind == "bitset" else _bits_of(rng.random((nq, n)) < 0.3)

    def fn(res, ds, qs, words):
        f = filters.from_bitset(words) if kind == "bitset" else filters.from_bitmap(words)
        return brute_force.search(brute_force.build(ds, resources=res), qs, 10, resources=res, prefilter=f)
    check_side_stream(f"brute_force {kind}", fn, ds=data["ds"], qs=data["qs"], words=words)


@pytest.mark.parametrize("dtype", ["float32", "int8"])
@pytest.mark.parametrize("k", [10, 100])
def test_ivf_flat_side_stream(data, dtype, k):
    def cast(x):
        return x if dtype == "float32" else (x * 40).round().clamp(-128, 127).to(torch.int8)
    # bitset over ids: the build rows are 0.., the extended rows 50000.. (all kept)
    n = data["ds"].shape[0]
    words = _bits_of(np.r_[np.random.default_rng(8).random(n) < 0.7, np.ones(52000 - n, bool)])

    def fn(res, ds, qs, extra, extra_ids, words):
        idx = ivf_flat.build(ivf_flat.IndexParams(n_lists=32, kmeans_n_iters=10), ds, resources=res)
        ivf_flat.extend(idx, extra, extra_ids, resources=res)
        sp = ivf_flat.SearchParams(n_probes=12)
        plain = ivf_flat.search(sp, idx, qs, k, resources=res)
        return plain, ivf_flat.search(sp, idx, qs, k, resources=res, filter=filters.from_bitset(words))
    check_side_stream(f"ivf_flat {dtype} k={k}", fn, ds=cast(data["ds"]), qs=cast(data["qs"]), extra=cast(data["extra"]),
                      extra_ids=data["extra_ids"], words=words)


PQ_STREAM_PARAMS = dict(n_lists=32, pq_dim=32, pq_bits=8, kmeans_n_iters=10)  # d 64, pq_len 2: served by the code stream


@pytest.mark.parametrize("path", ["tc", "stream", "lut"])
@pytest.mark.parametrize("k", [10, 100])
def test_ivf_pq_side_stream(data, monkeypatch, path, k):
    monkeypatch.setenv("CUVS_B200_PQ_PATH", path)

    def fn(res, ds, qs, extra, extra_ids):
        idx = ivf_pq.build(ivf_pq.IndexParams(**PQ_STREAM_PARAMS), ds, resources=res)
        ivf_pq.extend(idx, extra, extra_ids, resources=res)
        d, i = ivf_pq.search(ivf_pq.SearchParams(n_probes=16), idx, qs, k, resources=res)
        # refine over the dataset the ids index: build rows are 0.., the extended rows are placed at 50000..
        full = torch.zeros((52000, ds.shape[1]), dtype=ds.dtype, device="cuda")
        full[:ds.shape[0]] = ds
        full[50000:] = extra
        rd, ri = refine(full, qs, i, k=10, resources=res)
        return d, i, rd, ri
    check_side_stream(f"ivf_pq {path} k={k}", fn, ds=data["ds"], qs=data["qs"], extra=data["extra"], extra_ids=data["extra_ids"])


CAGRA_SEARCH = {"single_cta": dict(itopk_size=64, algo="single_cta"), "multi_cta": dict(itopk_size=64, algo="multi_cta")}


@pytest.mark.parametrize("build_algo", ["ivf_pq", "nn_descent"])
@pytest.mark.parametrize("dtype", ["float32", "float16"])
def test_cagra_side_stream(data, build_algo, dtype):
    tdt = torch.float32 if dtype == "float32" else torch.float16

    def fn(res, ds, qs, extra):
        idx = cagra.build(cagra.IndexParams(graph_degree=32, intermediate_graph_degree=64, build_algo=build_algo), ds, resources=res)
        outs = [cagra.search(cagra.SearchParams(**sp), idx, qs, 10, resources=res) for sp in CAGRA_SEARCH.values()]
        cagra.extend(cagra.ExtendParams(), idx, extra, resources=res)
        outs.append(cagra.search(cagra.SearchParams(**CAGRA_SEARCH["single_cta"]), idx, qs, 10, resources=res))
        return outs
    check_side_stream(f"cagra {build_algo} {dtype}", fn, exact=False, ds=data["ds"].to(tdt), qs=data["qs"].to(tdt),
                      extra=data["extra"].to(tdt))


@pytest.mark.parametrize("n_cand", [256, 2048])
def test_refine_side_stream(data, n_cand):
    cand = torch.from_numpy(np.random.default_rng(9).integers(0, data["ds"].shape[0], (64, n_cand))).cuda()

    def fn(res, ds, qs, cand):
        return refine(ds, qs, cand, k=32, resources=res)
    check_side_stream(f"refine {n_cand}", fn, ds=data["ds"], qs=data["qs"][:64], cand=cand)


@pytest.mark.parametrize("payload", [False, True])
def test_select_k_side_stream(payload):
    rng = np.random.default_rng(10)
    vals = _cuda(rng.random((200, 5000)).astype(np.float32))
    ids = _cuda(rng.permutation(200 * 5000).reshape(200, 5000).astype(np.int64))

    def fn(res, vals, ids):
        ov = torch.empty((200, 64), dtype=torch.float32, device="cuda")
        oi = torch.empty((200, 64), dtype=torch.int64, device="cuda")
        check(lib.cuvsSelectK(res.get_c_obj(), DL(vals).ptr, DL(ids).ptr if payload else None, DL(ov).ptr, DL(oi).ptr,
                              C.c_bool(True), C.c_bool(True)))
        return ov, oi
    check_side_stream(f"select_k payload={payload}", fn, vals=vals, ids=ids)


def test_knn_merge_parts_side_stream():
    rng = np.random.default_rng(11)
    n_parts, n_rows, k = 8, 100, 10
    keys = _cuda(np.sort(rng.random((n_parts * n_rows, k)).astype(np.float32), axis=1))
    vals = _cuda(rng.integers(0, 1000, (n_parts * n_rows, k)).astype(np.int64))
    tr = (C.c_int64 * n_parts)(*(np.arange(n_parts) * 1000).tolist())

    def fn(res, keys, vals):
        ok = torch.empty((n_rows, k), device="cuda")
        ov = torch.empty((n_rows, k), dtype=torch.int64, device="cuda")
        check(lib.cuvsKnnMergeParts(res.get_c_obj(), DL(keys).ptr, DL(vals).ptr, DL(ok).ptr, DL(ov).ptr, C.c_int64(n_parts), tr,
                                    C.c_bool(True)))
        return ok, ov
    check_side_stream("knn_merge_parts", fn, keys=keys, vals=vals)


@pytest.mark.parametrize("metric", [0, 6])  # L2Expanded, InnerProduct
def test_pairwise_distance_side_stream(data, metric):
    def fn(res, x, y):
        out = torch.empty((x.shape[0], y.shape[0]), dtype=torch.float32, device="cuda")
        check(lib.cuvsPairwiseDistance(res.get_c_obj(), DL(x).ptr, DL(y).ptr, DL(out).ptr, C.c_int(metric), C.c_float(2.0)))
        return out
    check_side_stream(f"pairwise_distance {metric}", fn, x=data["qs"], y=data["ds"][:3000])


def test_kmeans_side_stream(data):
    params = kmeans.KMeansParams(n_clusters=16, max_iter=20, init_method="k-means++")

    def fn(res, x):
        cent, inertia, n_iter = kmeans.fit(params, x, resources=res)
        labels, pinertia = kmeans.predict(params, x, cent, resources=res)
        cost = kmeans.cluster_cost(x, cent, resources=res)
        return cent, labels, np.array([inertia, n_iter, pinertia, cost])
    check_side_stream("kmeans", fn, x=data["ds"])


def test_nn_descent_side_stream(data):
    def fn(res, ds):
        g = torch.empty((ds.shape[0], 32), dtype=torch.uint32, device="cuda")
        params = nn_descent.IndexParams(graph_degree=32, intermediate_graph_degree=64, max_iterations=10, return_distances=True)
        idx = nn_descent.build(params, ds, graph=g, resources=res)
        return g, idx._get(lib.cuvsNNDescentIndexGetDistances, torch.float32, resources=res)
    check_side_stream("nn_descent", fn, ds=data["ds"])


def test_matrix_copy_and_slice_rows_side_stream():
    big = _cuda(np.random.default_rng(12).standard_normal((500, 48)).astype(np.float32))

    def fn(res, big):
        src = big[:, :40]  # row pitch 48: the strided 2-D copy
        dst = torch.empty((500, 40), dtype=torch.float32, device="cuda")
        check(lib.cuvsMatrixCopy(res.get_c_obj(), DL(src, force_strides=True).ptr, DL(dst).ptr))
        flat = big.reshape(-1)
        view = DLManagedTensor()
        keep = DL(big)
        check(lib.cuvsMatrixSliceRows(res.get_c_obj(), keep.ptr, C.c_int64(100), C.c_int64(300), C.byref(view)))
        rows = torch.empty((200, 48), dtype=torch.float32, device="cuda")
        try:
            assert view.dl_tensor.data == big[100:].data_ptr() and view.dl_tensor.shape[0] == 200
            check(lib.cuvsMatrixCopy(res.get_c_obj(), C.byref(view), DL(rows).ptr))
        finally:
            if view.deleter:
                view.deleter(C.byref(view))
        one_d = torch.empty_like(flat)
        check(lib.cuvsMatrixCopy(res.get_c_obj(), DL(flat).ptr, DL(one_d).ptr))
        return dst, rows, one_d
    check_side_stream("matrix copy / slice rows", fn, big=big)
    # and against plain torch
    res = Resources()
    dst, rows, one_d = fn(res, big)
    res.sync()
    assert torch.equal(dst, big[:, :40]) and torch.equal(rows, big[100:300]) and torch.equal(one_d, big.reshape(-1))


@pytest.mark.parametrize("kind", ["ivf_flat", "ivf_pq", "cagra"])
def test_save_and_load_side_stream(data, tmp_path, kind):
    path = str(tmp_path / f"{kind}.bin")

    def fn(res, ds, qs):
        if kind == "ivf_flat":
            idx = ivf_flat.build(ivf_flat.IndexParams(n_lists=32, kmeans_n_iters=10), ds, resources=res)
            ivf_flat.save(path, idx, resources=res)
            return ivf_flat.search(ivf_flat.SearchParams(n_probes=12), ivf_flat.load(path, resources=res), qs, 10, resources=res)
        if kind == "ivf_pq":
            idx = ivf_pq.build(ivf_pq.IndexParams(**PQ_STREAM_PARAMS), ds, resources=res)
            ivf_pq.save(path, idx, resources=res)
            return ivf_pq.search(ivf_pq.SearchParams(n_probes=16), ivf_pq.load(path, resources=res), qs, 10, resources=res)
        idx = cagra.build(cagra.IndexParams(graph_degree=32, intermediate_graph_degree=64), ds, resources=res)
        cagra.save(path, idx, resources=res)
        return cagra.search(cagra.SearchParams(itopk_size=64), cagra.load(path, resources=res), qs, 10, resources=res)
    check_side_stream(f"save/load {kind}", fn, exact=kind != "cagra", ds=data["ds"], qs=data["qs"])


# ------------------------------------------------------------------------------------------- shared indexes for B and C
@pytest.fixture(scope="module")
def indexes(data):
    ds = data["ds"]
    out = {
        "brute_force": brute_force.build(ds),
        "ivf_flat": ivf_flat.build(ivf_flat.IndexParams(n_lists=32, kmeans_n_iters=10), ds),
        "ivf_pq": ivf_pq.build(ivf_pq.IndexParams(**PQ_STREAM_PARAMS), ds),
        "cagra": cagra.build(cagra.IndexParams(graph_degree=32, intermediate_graph_degree=64), ds),
    }
    torch.cuda.synchronize()
    assert out["ivf_pq"].streamed
    return out


def _search(kind, index, qs, res, k=10):
    if kind == "brute_force":
        return brute_force.search(index, qs, k, resources=res)
    if kind == "ivf_flat":
        return ivf_flat.search(ivf_flat.SearchParams(n_probes=12), index, qs, k, resources=res)
    if kind == "ivf_pq":
        return ivf_pq.search(ivf_pq.SearchParams(n_probes=16), index, qs, k, resources=res)
    return cagra.search(cagra.SearchParams(itopk_size=64), index, qs, k, resources=res)


# ------------------------------------------------------------------------------------ B. two streams, one index, one thread
@pytest.mark.parametrize("kind", ["brute_force", "ivf_flat", "ivf_pq", "cagra"])
def test_two_streams_one_index(data, indexes, kind):
    qa, qb = data["qs"][:150].contiguous(), data["qs"][150:].contiguous()
    index = indexes[kind]
    refs = []
    for q in (qa, qb):
        ref, repeats = serial(lambda res, q: _search(kind, index, q, res), {"q": q})
        refs.append((ref, repeats))
    S1, S2 = torch.cuda.Stream(), torch.cuda.Stream()
    la = late(qa, S1)  # search A waits behind a sleep on S1 ...
    with torch.cuda.stream(S1):
        out_a = _search(kind, index, la, Resources())
    with torch.cuda.stream(S2):  # ... while search B runs on S2
        S2.wait_stream(torch.cuda.default_stream())
        out_b = _search(kind, index, qb, Resources())
    S1.synchronize()
    S2.synchronize()
    compare(f"{kind} search A", refs[0][0], refs[0][1], _host(out_a), kind != "cagra")
    compare(f"{kind} search B", refs[1][0], refs[1][1], _host(out_b), kind != "cagra")


def _unpack(res, index, label, n_rows):
    out = torch.empty((n_rows, index.pq_dim * index.pq_bits // 8), dtype=torch.uint8, device="cuda")
    check(lib.cuvsIvfPqIndexUnpackContiguousListData(res.get_c_obj(), index._p, DL(out).ptr, C.c_uint32(label), C.c_uint32(0)))
    return out


def test_ivf_pq_unpack_then_lut_search_on_another_stream(data, monkeypatch):
    """A list read on S1, held behind a sleep, must not hand its decode to a LUT search on S2."""
    monkeypatch.setenv("CUVS_B200_PQ_PATH", "lut")
    index = ivf_pq.build(ivf_pq.IndexParams(**PQ_STREAM_PARAMS), data["ds"])
    assert index.streamed
    label = int(torch.argmax(index.list_sizes.to(torch.int64)).item())
    n_rows = int(index.list_sizes[label].item())
    ref_codes, _ = serial(lambda res: _unpack(res, index, label, n_rows), {})
    ref, repeats = serial(lambda res, q: _search("ivf_pq", index, q, res), {"q": data["qs"]})
    S1, S2 = torch.cuda.Stream(), torch.cuda.Stream()
    S1.wait_stream(torch.cuda.default_stream())
    S2.wait_stream(torch.cuda.default_stream())
    with torch.cuda.stream(S1):
        torch.cuda._sleep(SLEEP_CYCLES)
        codes = _unpack(Resources(), index, label, n_rows)
    with torch.cuda.stream(S2):
        out = _search("ivf_pq", index, data["qs"], Resources())
    S1.synchronize()
    S2.synchronize()
    assert _same_bits(ref_codes, _host(codes))
    compare("ivf_pq lut search beside an unpack", ref, repeats, _host(out))


# ------------------------------------------------------------------------------------------------------------ C. threads
N_THREADS, N_ROUNDS, BATCH = 4, 20, 256  # 256 queries x 16 probes: the IVF-PQ default takes its decoded-row path


@pytest.mark.parametrize("kind", ["brute_force", "ivf_flat", "ivf_pq-tc", "ivf_pq-stream", "ivf_pq-lut", "cagra"])
def test_threads_share_one_index(data, indexes, monkeypatch, kind):
    """Four threads, each with its own stream and resources, search one index 20 times with their own query batches; the
    ctypes calls release the GIL, so the searches overlap."""
    kind, _, path = kind.partition("-")
    if path:
        monkeypatch.setenv("CUVS_B200_PQ_PATH", path)
    index = indexes[kind]
    rng = np.random.default_rng(13)
    qs = data["qs"]
    batches = [[qs[torch.from_numpy(rng.integers(0, qs.shape[0], BATCH)).cuda()].contiguous() for _ in range(N_ROUNDS)]
               for _ in range(N_THREADS)]
    torch.cuda.synchronize()
    refs = [[serial(lambda res, q: _search(kind, index, q, res), {"q": q}) for q in tb] for tb in batches]
    results, errors = [[None] * N_ROUNDS for _ in range(N_THREADS)], []
    barrier = threading.Barrier(N_THREADS, timeout=120)

    def work(t):
        try:
            S = torch.cuda.Stream()
            S.wait_stream(torch.cuda.default_stream())
            with torch.cuda.stream(S):
                res = Resources()
                barrier.wait()
                for r in range(N_ROUNDS):
                    results[t][r] = _search(kind, index, batches[t][r], res)
            S.synchronize()
            results[t] = [_host(o) for o in results[t]]
        except Exception as e:  # noqa: BLE001 - reported on the main thread
            errors.append(e)

    threads = [threading.Thread(target=work, args=(t,)) for t in range(N_THREADS)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for t in range(N_THREADS):
        for r in range(N_ROUNDS):
            compare(f"{kind}{'-' + path if path else ''} thread {t} round {r}", refs[t][r][0], refs[t][r][1], results[t][r],
                    kind != "cagra")


# ------------------------------------------------------------------------------------ D. reads do not mutate an IVF-PQ index
def test_ivf_pq_reads_leave_the_index_unchanged(data, tmp_path, monkeypatch):
    ds = data["ds"]
    index = ivf_pq.build(ivf_pq.IndexParams(**PQ_STREAM_PARAMS), ds)
    assert index.streamed
    before = index._info()
    sizes = index.list_sizes.to(torch.int64).cpu().numpy()
    listed = [index.list_data(label) for label in range(index.n_lists)]
    assert index._info() == before, f"list_data changed (path, device_bytes) from {before} to {index._info()}"
    ivf_pq.save(str(tmp_path / "pq.bin"), index)
    assert index._info() == before, f"save changed (path, device_bytes) from {before} to {index._info()}"
    monkeypatch.setenv("CUVS_B200_PQ_PATH", "lut")
    ivf_pq.search(ivf_pq.SearchParams(n_probes=16), index, data["qs"], 10)
    assert index._info() == before, f"a LUT search changed (path, device_bytes) from {before} to {index._info()}"
    # list_data returns the codes transform gives the same rows
    labels, codes = ivf_pq.transform(index, ds)
    labels, codes = labels.to(torch.int64).cpu().numpy(), codes.cpu().numpy()
    agree = 0
    for label in range(index.n_lists):
        ids = index.list_indices(label).cpu().numpy()
        assert len(ids) == sizes[label] == listed[label].shape[0]
        same = labels[ids] == label
        agree += same.sum()
        np.testing.assert_array_equal(listed[label].cpu().numpy()[same], codes[ids[same]])
    assert agree >= 0.99 * ds.shape[0]
