"""A NumPy model of how a float16 brute-force index scans float32 queries (DESIGN.md §3 "Row types"): each query row is scaled by
a power of two 2^e that puts its largest component in [2^14, 2^15), split into fp16 hi + lo, and multiplied with the fp16 rows in
two passes; the scores are scaled back by 2^-e.  The model's error must stay inside the certificate's budget,
2^-15 (|q|^2 + max |x|^2), on the extreme-magnitude rows the GPU test uses."""
import numpy as np


def split_scaled(q):
    """(hi, lo, scale) as split_f16_queries_kernel computes them."""
    m = np.abs(q).max(1)
    _, ex = np.frexp(m)
    e = np.where(m > 0, np.clip(15 - ex, -60, 60), 0)
    scale = np.ldexp(np.float32(1), e).astype(np.float32)
    v = (q * scale[:, None]).astype(np.float32)
    hi = v.astype(np.float16)
    lo = (v - hi.astype(np.float32)).astype(np.float16)
    return hi, lo, scale


def model_scores(q, x):
    """s = (2^e (q.x) from (hi + lo) . x, products exact, summed in float64) / 2^e."""
    hi, lo, scale = split_scaled(q)
    xd = x.astype(np.float64)
    acc = hi.astype(np.float64) @ xd.T + lo.astype(np.float64) @ xd.T
    return acc / scale[:, None].astype(np.float64)


def extreme_rows(seed=5, n=3000, dim=96):
    rng = np.random.default_rng(seed)
    ds = rng.uniform(-1, 1, (n, dim)).astype(np.float16)
    ds[:20] = np.float16(65504.0) * np.sign(rng.standard_normal((20, dim))).astype(np.float16)
    ds[20:40] = (rng.integers(-1023, 1024, (20, dim)) * 2.0 ** -24).astype(np.float16)
    qs = (np.sign(rng.standard_normal((64, dim))) * 10.0 ** rng.uniform(-7, np.log10(6e4), (64, dim))).astype(np.float32)
    qs[:4] *= 1e-6
    qs[4:8] = qs[4:8] / np.abs(qs[4:8]).max(1, keepdims=True) * 6e4
    return ds, qs


def test_scale_puts_the_largest_component_in_range():
    _, qs = extreme_rows()
    hi, lo, scale = split_scaled(qs)
    top = np.abs(qs * scale[:, None]).max(1)
    assert ((top >= 2.0 ** 14) & (top < 2.0 ** 15)).all()
    assert np.isfinite(hi.astype(np.float32)).all() and np.isfinite(lo.astype(np.float32)).all()
    assert (np.log2(scale) == np.round(np.log2(scale))).all()  # powers of two: the scale comes off exactly


def test_split_error_inside_the_certificate_budget():
    ds, qs = extreme_rows()
    x = ds.astype(np.float64)
    exact = qs.astype(np.float64) @ x.T
    err = np.abs(model_scores(qs, ds) - exact)
    budget = 2.0 ** -15 * ((qs.astype(np.float64) ** 2).sum(1)[:, None] + (x ** 2).sum(1).max())
    assert (err <= budget / 4).all(), float((err / budget).max())
    # and a plain split without the scale loses the small rows' low parts to fp16's subnormals
    plain_hi = qs.astype(np.float16)
    plain_lo = (qs - plain_hi.astype(np.float32)).astype(np.float16)
    plain = plain_hi.astype(np.float64) @ x.T + plain_lo.astype(np.float64) @ x.T
    small = np.abs(qs).max(1) < 1e-1
    assert (np.abs(plain - exact)[small] > np.abs(model_scores(qs, ds) - exact)[small]).any()
