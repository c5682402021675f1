"""The scalar and binary quantizers on the GPU against the NumPy restatement (tests/quantize_ref.py): exact quantizers and codes
where the sample is the whole dataset, sampled statistics within bounds, host and device inputs alike, refusals with text,
side streams and shared quantizers, and the codes feeding the int8 and bitwise-Hamming indexes."""
import threading

import numpy as np
import pytest
import torch

import oracle
from cuvs_b200._capi import CuvsError
from cuvs_b200.common.resources import Resources
from cuvs_b200.preprocessing.quantize import binary, scalar
from tests import hamming_ref as H
from tests import quantize_ref as Q
from tests.test_streams_gpu import check_side_stream
from tests.util import clustered

pytestmark = pytest.mark.gpu

FLOATS = [np.float32, np.float16, np.float64]
TORCH = {np.float32: torch.float32, np.float16: torch.float16, np.float64: torch.float64}
UINT = {np.float32: np.uint32, np.float16: np.uint16, np.float64: np.uint64}


def _on(x, where):
    t = torch.from_numpy(np.ascontiguousarray(x))
    return t.cuda() if where == "device" else t


def _np(t):
    return t.cpu().numpy()


def _bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


# ------------------------------------------------------------------------------------------------------------ scalar
@pytest.mark.parametrize("d", [1, 7, 128, 1000])
@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("dtype", FLOATS)
def test_scalar_exact(dtype, where, d):
    n = min(3000, Q.SCALAR_SAMPLE_VALUES // d)
    rng = np.random.default_rng(d)
    x = (rng.standard_normal((n, d)) * 3).astype(dtype)
    x[rng.integers(0, n, 5), rng.integers(0, d, 5)] = 0  # ties
    xt = _on(x, where)
    q = scalar.train(scalar.QuantizerParams(quantile=0.97), xt)
    assert (q.min, q.max) == Q.scalar_train(x, 0.97)
    given = d in (7, 1000)
    out = torch.full_like(xt, 99, dtype=torch.int8) if given else None
    codes = scalar.transform(q, xt, output=out)
    assert codes.device == xt.device and codes.dtype == torch.int8
    if given:
        assert codes is out
    ref = Q.scalar_transform(x, q.min, q.max)
    np.testing.assert_array_equal(_np(codes), ref)
    inv_out = torch.empty(x.shape, dtype=TORCH[dtype], device=xt.device) if given else None
    inv = scalar.inverse_transform(q, codes, output=inv_out)
    expect_dtype = dtype if given else np.float32
    want = Q.scalar_inverse(ref, q.min, q.max, expect_dtype)
    assert _bits_equal(_np(inv).view(UINT[expect_dtype]), want.view(UINT[expect_dtype]))


def test_scalar_transform_of_edge_values():
    """NaN, the range ends, values beyond them, and half-way points of the float32 rounding, on the device."""
    q = scalar.train(scalar.QuantizerParams(quantile=1.0), torch.tensor([[-2.0, 2.0]], device="cuda"))
    assert (q.min, q.max) == (-2.0, 2.0)
    lo, hi, scale, offset = Q.scalar_map(-2.0, 2.0, np.float32)
    half_way = ((np.arange(-127, 127) + 0.5 - offset) / scale).astype(np.float32)
    x = np.concatenate([[np.nan, -np.inf, np.inf, -2.0, 2.0, -3.0, 3.0, 0.0, -0.0], half_way]).astype(np.float32)[None, :]
    got = _np(scalar.transform(q, torch.from_numpy(x).cuda()))
    np.testing.assert_array_equal(got, Q.scalar_transform(x, q.min, q.max))


def _rank_error(sorted_vals, v, target):
    lo, hi = np.searchsorted(sorted_vals, v, "left"), np.searchsorted(sorted_vals, v, "right") - 1
    return 0 if lo <= target <= hi else min(abs(lo - target), abs(hi - target))


def test_scalar_sampled():
    n, d = 200_000, 128
    x = np.random.default_rng(5).standard_normal((n, d)).astype(np.float32)
    params = scalar.QuantizerParams(quantile=0.99)
    xd = torch.from_numpy(x).cuda()
    q = scalar.train(params, xd)
    v = np.sort(x.ravel())
    lo_rank, hi_rank = Q.quantile_positions(v.size, 0.99)
    for val, target in ((q.min, lo_rank), (q.max, hi_rank)):
        assert np.float32(val) == val and (v == np.float32(val)).any(), "not a value of the data"
        assert _rank_error(v, np.float32(val), target) <= 0.0005 * v.size
    again = scalar.train(params, xd)
    host = scalar.train(params, torch.from_numpy(x))
    assert (again.min, again.max) == (q.min, q.max) == (host.min, host.max)


# ------------------------------------------------------------------------------------------------------------ binary
def _check_binary(x, where, q, t):
    """transform through `q` (None: the plain ZERO call) into a library-made output and into a wider, longer poisoned one."""
    n, d = x.shape
    nb = (d + 7) // 8
    xt = _on(x, where)
    want = Q.pack(x, t)
    got = binary.transform(xt, quantizer=q)
    assert got.dtype == torch.uint8 and got.device == xt.device and tuple(got.shape) == (n, nb)
    np.testing.assert_array_equal(_np(got), want)
    wide = torch.full((n + 3, nb + 5), 0xAB, dtype=torch.uint8, device=xt.device)
    binary.transform(xt, output=wide, quantizer=q)
    w = _np(wide)
    np.testing.assert_array_equal(w[:n, :nb], want)
    assert (w[:n, nb:] == 0).all() and (w[n:] == 0xAB).all()


@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("dtype", FLOATS)
@pytest.mark.parametrize("d", [1, 7, 8, 9, 64, 1000, 1030])
def test_binary_exact(d, dtype, where):
    rng = np.random.default_rng(d + 17)
    x = rng.integers(-3, 4, (256, d)).astype(dtype)  # integer values: ties with every threshold, exact means
    _check_binary(x, where, None, None)
    _check_binary(x, where, binary.train(binary.QuantizerParams(threshold="zero"), _on(x, where)), None)
    _check_binary(x, where, binary.train(binary.QuantizerParams(threshold="mean"), _on(x, where)), Q.thresholds(x, "mean"))
    xm = rng.integers(-3, 4, (257, d)).astype(dtype)
    qm = binary.train(binary.QuantizerParams(threshold="sampling_median", sampling_ratio=1.0), _on(xm, where))
    _check_binary(xm, where, qm, Q.thresholds(xm, "sampling_median", 1.0))


def test_binary_sampled_median():
    n, d = 100_001, 64
    x = (np.random.default_rng(9).standard_normal((n, d)) + np.linspace(-2, 2, d)).astype(np.float32)
    params = binary.QuantizerParams(threshold="sampling_median", sampling_ratio=0.1)
    xd = torch.from_numpy(x).cuda()
    bits = _np(binary.transform(xd, quantizer=binary.train(params, xd)))
    share = np.unpackbits(bits, axis=1, bitorder="little")[:, :d].mean(0)
    assert ((share >= 0.48) & (share <= 0.52)).all(), share
    again = _np(binary.transform(xd, quantizer=binary.train(params, xd)))
    host = _np(binary.transform(torch.from_numpy(x), quantizer=binary.train(params, torch.from_numpy(x))))
    assert _bits_equal(bits, again) and _bits_equal(bits, host)


def test_median_across_column_chunks():
    """262145 x 1024 float32 at ratio 1: a 1 GiB + 4 KiB sample, over the column-chunk bound.  Probe rows pin each threshold
    exactly: the median itself must give 0 and the next float above it 1."""
    n, d = 262_145, 1024
    x = np.random.default_rng(3).standard_normal((n, d), dtype=np.float32)
    med = np.median(x, axis=0).astype(np.float32)
    assert (np.sort(x[:, :3], axis=0)[n // 2] == med[:3]).all()
    q = binary.train(binary.QuantizerParams(threshold="sampling_median", sampling_ratio=1.0), torch.from_numpy(x).cuda())
    del x
    probe = np.stack([med, np.nextafter(med, np.float32(np.inf))])
    got = np.unpackbits(_np(binary.transform(torch.from_numpy(probe).cuda(), quantizer=q)), axis=1, bitorder="little")
    assert (got[0] == 0).all(), f"{int(got[0].sum())} thresholds below the median"
    assert (got[1] == 1).all(), f"{int((got[1] == 0).sum())} thresholds above the median"


# ------------------------------------------------------------------------------------------------------------ errors
def test_refusals_name_what_is_wrong():
    x = torch.randn(64, 16, device="cuda")
    xh = x.cpu()
    sq = scalar.train(scalar.QuantizerParams(), x)
    bq = binary.train(binary.QuantizerParams(), x)
    i8 = torch.zeros(64, 16, dtype=torch.int8, device="cuda")
    cases = [
        (lambda: scalar.train(scalar.QuantizerParams(), i8), "dataset must be float32, float16 or float64"),
        (lambda: scalar.train(scalar.QuantizerParams(), x.to(torch.uint8)), "dataset must be float32, float16 or float64"),
        (lambda: binary.transform(i8), "dataset must be float32, float16 or float64"),
        (lambda: scalar.train(scalar.QuantizerParams(), x[0]), "dataset must be a 2-D tensor"),
        (lambda: binary.transform(x[:, ::2]), "dataset must be C-contiguous"),
        (lambda: scalar.train(scalar.QuantizerParams(quantile=0.0), x), "quantile must lie in (0, 1]"),
        (lambda: scalar.train(scalar.QuantizerParams(quantile=1.5), x), "quantile must lie in (0, 1]"),
        (lambda: binary.train(binary.QuantizerParams(threshold="sampling_median", sampling_ratio=0.0), x), "sampling_ratio must lie in (0, 1]"),
        (lambda: binary.train(binary.QuantizerParams(threshold="sampling_median", sampling_ratio=1.5), x), "sampling_ratio must lie in (0, 1]"),
        (lambda: scalar.transform(sq, x, output=torch.empty(64, 16, device="cuda")), "output must be int8"),
        (lambda: scalar.transform(sq, x, output=torch.empty(64, 15, dtype=torch.int8, device="cuda")), "output must have the dataset's shape"),
        (lambda: scalar.inverse_transform(sq, x), "dataset must be int8 codes"),
        (lambda: scalar.inverse_transform(sq, i8, output=torch.empty(64, 16, dtype=torch.int32, device="cuda")), "output must be float32"),
        (lambda: binary.transform(x, output=torch.empty(64, 1, dtype=torch.uint8, device="cuda")), "output must have at least 64 rows and 2 columns"),
        (lambda: binary.transform(x, output=torch.empty(63, 2, dtype=torch.uint8, device="cuda")), "output must have at least 64 rows and 2 columns"),
        (lambda: binary.transform(x, output=torch.empty(64, 2, dtype=torch.int8, device="cuda")), "output must be uint8"),
        (lambda: scalar.transform(sq, xh, output=i8), "same kind of memory"),
        (lambda: binary.transform(x, output=torch.empty(64, 2, dtype=torch.uint8)), "same kind of memory"),
        (lambda: binary.transform(x, quantizer=binary.Quantizer()), "the binary quantizer is not trained"),
        (lambda: binary.transform(x.half(), quantizer=bq), "dataset is float16 but the quantizer was trained on float32"),
        (lambda: binary.transform(x[:, :15].contiguous(), quantizer=bq), "dataset has 15 columns but the quantizer has 16 thresholds"),
    ]
    for call, text in cases:
        with pytest.raises(CuvsError, match=text.replace("(", r"\(").replace(")", r"\)").replace("[", r"\[")):
            call()
        np.testing.assert_array_equal(_np(binary.transform(x, quantizer=bq)), Q.pack(_np(x), Q.thresholds(_np(x), "mean")))


# ------------------------------------------------------------------------------------------------------------ streams
def test_side_stream_train_and_transform():
    x = torch.from_numpy(np.random.default_rng(4).standard_normal((20000, 96)).astype(np.float32)).cuda()

    def run(res, x):
        sq = scalar.train(scalar.QuantizerParams(quantile=0.99), x, resources=res)
        codes = scalar.transform(sq, x, resources=res)
        inv = scalar.inverse_transform(sq, codes, resources=res)
        mean = binary.train(binary.QuantizerParams(threshold="mean"), x, resources=res)
        med = binary.train(binary.QuantizerParams(threshold="sampling_median", sampling_ratio=0.5), x, resources=res)
        return (torch.tensor([sq.min, sq.max], dtype=torch.float64), codes, inv, binary.transform(x, resources=res),
                binary.transform(x, quantizer=mean, resources=res), binary.transform(x, quantizer=med, resources=res))

    check_side_stream("quantizers", run, x=x)


def test_threads_share_one_binary_quantizer():
    x = torch.from_numpy(np.random.default_rng(6).standard_normal((30000, 200)).astype(np.float32)).cuda()
    q = binary.train(binary.QuantizerParams(threshold="sampling_median", sampling_ratio=0.2), x)
    ref = _np(binary.transform(x, quantizer=q))
    torch.cuda.synchronize()
    results, errors = [None] * 4, []

    def worker(i):
        try:
            S = torch.cuda.Stream()
            res = Resources(stream=S)
            outs = [binary.transform(x, quantizer=q, resources=res) for _ in range(5)]
            res.sync()
            results[i] = [_np(o) for o in outs]
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(i,)) for i in range(4)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    assert all(_bits_equal(o, ref) for r in results for o in r)


# ------------------------------------------------------------------------------------------------------------ end to end
def test_binary_codes_feed_cagra_hamming():
    from cuvs_b200.neighbors import cagra
    rng = np.random.default_rng(12)
    A = (rng.standard_normal((8, 32)) / np.sqrt(8)).astype(np.float32)
    P = rng.standard_normal((32, 128)).astype(np.float32)

    def rows(m, seed):
        r = np.random.default_rng(seed)
        return ((r.standard_normal((m, 8)).astype(np.float32) @ A + 0.05 * r.standard_normal((m, 32)).astype(np.float32)) @ P)

    xf, qf = rows(5000, 1), rows(300, 2)
    x, q = _np(binary.transform(torch.from_numpy(xf).cuda())), _np(binary.transform(torch.from_numpy(qf).cuda()))
    np.testing.assert_array_equal(x, Q.pack(xf))
    index = cagra.build(cagra.IndexParams(metric="bitwise_hamming", graph_degree=32, build_algo="nn_descent"), torch.from_numpy(x).cuda())
    d, i = cagra.search(cagra.SearchParams(itopk_size=64), index, torch.from_numpy(q).cuda(), 10)
    td, ti = H.knn(q, x, 10)
    assert oracle.recall_with_ties(_np(i).astype(np.int64), _np(d), ti, td) >= 0.95


def test_scalar_codes_feed_an_int8_brute_force_index():
    from cuvs_b200.neighbors import brute_force
    xf, centers = clustered(20000, 32, 41, sigma=0.5)  # 640k values: the quantizer's sample is the whole dataset
    qf, _ = clustered(200, 32, 42, centers=centers, sigma=0.5)
    sq = scalar.train(scalar.QuantizerParams(quantile=0.99), torch.from_numpy(xf).cuda())
    x8 = scalar.transform(sq, torch.from_numpy(xf).cuda())
    q8 = scalar.transform(sq, torch.from_numpy(qf).cuda())
    index = brute_force.build(x8)
    d, i = brute_force.search(index, q8, 10)
    rd, ri = oracle.knn(_np(x8).astype(np.float32), _np(q8).astype(np.float32), 10)
    assert (_np(i) == ri).all() and _np(d).tobytes() == rd.tobytes()
    _, gi = oracle.knn(xf, qf, 10)
    assert oracle.recall(_np(i), gi) >= 0.9
