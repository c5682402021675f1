"""A numpy model of the soundness argument of the IVF-PQ pruning-bound pre-pass (csrc/scan_pq.cu: pq_bound_prime_kernel,
DESIGN.md §5 "Bound pre-pass").

1. Margin.  The pre-pass scores a row in fp32 in a fixed order; the scan's wgmma sums the same exactly representable terms
   (bf16 x bf16 products, the three bf16 pieces of -hn/2 twice) in an order and with a rounding the hardware does not pin
   down.  The model accumulates them in random orders, in fused blocks of 1 to 16 addends aligned to the largest exponent and
   truncated, each block's result truncated or rounded to nearest, and checks that the two scores never differ by more than
   2^-12 (|hn| + sum |r_i y_i|).
2. Conversion.  With B = kth + 2^-21 (|kth| + M) + 1e-30 rounded upward (M >= |add| of every pair of the query), every row
   whose merge value fmaf(scale, s, add) is <= kth passes the scan's starting threshold s < (B - add) / scale."""
import numpy as np
import pytest

F32 = np.float32


def bf16(x):
    b = np.asarray(x, dtype=F32).view(np.uint32)
    b = (b + np.uint32(0x7FFF) + ((b >> np.uint32(16)) & np.uint32(1))) & np.uint32(0xFFFF0000)
    return b.view(F32)


def to_f32(x, trunc):
    """float64 -> float32, rounded to nearest or (trunc) toward zero."""
    f = x.astype(F32)
    if trunc:
        over = np.abs(f.astype(np.float64)) > np.abs(x)
        f = np.where(over, np.nextafter(f, F32(0)), f)
    return f


def scan_model(terms, rng):
    """One random accumulation of terms [rows, n] (exact float64 values of fp32 numbers) into an fp32 accumulator."""
    rows, n = terms.shape
    order = rng.permutation(n)
    acc = np.zeros(rows, F32)
    i = 0
    while i < n:
        m = int(rng.choice([1, 2, 4, 8, 16]))
        blk = np.concatenate([acc[:, None].astype(np.float64), terms[:, order[i:i + m]]], axis=1)
        i += m
        mx = np.abs(blk).max(axis=1)
        e = np.floor(np.log2(np.where(mx > 0, mx, 1.0)))
        unit = np.exp2(e - 23)[:, None]
        s = (np.trunc(blk / unit) * unit).sum(axis=1)  # aligned and truncated addends: the sum is exact in float64
        acc = to_f32(s, trunc=bool(rng.integers(2)))
    return acc


def prepass_model(hi, lo, y, hn):
    """The kernel's order: lane l owns subspaces l + 32 h (columns 2 j, 2 j + 1), fmaf per (plane, column), then the
    butterfly over lanes 16, 8, 4, 2, 1; score = hn - dot.  fmaf is modelled as one rounding of the exact float64 value."""
    rows, kp = hi.shape
    nkb = kp // 64
    planes = [hi] if lo is None else [hi, lo]
    lanes = []
    for l in range(32):
        acc = np.zeros(rows, F32)
        for h in range(nkb):
            j = 32 * h + l
            for c in (2 * j, 2 * j + 1):
                for p in planes:
                    acc = (p[:, c].astype(np.float64) * y[:, c] + acc).astype(F32)
        lanes.append(acc)
    lanes = np.stack(lanes, axis=1)
    for w in (16, 8, 4, 2, 1):
        lanes = (lanes + lanes[:, np.arange(32) ^ w]).astype(F32)
    return (hn - lanes[:, 0]).astype(F32)


@pytest.mark.parametrize("passes", [1, 2])
@pytest.mark.parametrize("kind", ["l2", "ip", "cancel", "wide"])
@pytest.mark.parametrize("seed", range(3))
def test_scan_score_within_margin_of_prepass_score(passes, kind, seed):
    rng = np.random.default_rng(100 * seed + 7 * passes + len(kind))
    rows, kp = 400, 128
    col_scale = np.exp2(rng.uniform(-12, 12, kp)) if kind == "wide" else np.ones(kp)
    r = (rng.standard_normal((rows, kp)) * col_scale).astype(F32)
    y = bf16(rng.standard_normal((rows, kp)) * (1.0 / col_scale if kind == "wide" else 1.0))
    hi = bf16(r)
    lo = bf16(r - hi) if passes == 2 else None
    prods = [hi.astype(np.float64) * y] + ([] if lo is None else [lo.astype(np.float64) * y])
    dot = sum(p.sum(axis=1) for p in prods)
    if kind == "l2":
        hn = (0.5 * (y.astype(np.float64) ** 2).sum(axis=1)).astype(F32)
    elif kind == "ip":
        hn = np.zeros(rows, F32)
    else:  # the score cancels to ~0 against large terms: the hardest case for a margin relative to the terms
        hn = dot.astype(F32)
    hh = (F32(-0.5) * hn).astype(F32)
    p0 = bf16(hh)
    p1 = bf16((hh - p0).astype(F32))
    p2 = bf16(((hh - p0).astype(F32) - p1).astype(F32))
    pieces = [p.astype(np.float64)[:, None] for p in (p0, p1, p2)]
    terms = np.concatenate(prods + pieces + pieces, axis=1)
    pre = prepass_model(hi, lo, y, hn).astype(np.float64)
    margin = 2.0 ** -12 * (np.abs(hn.astype(np.float64)) + sum(np.abs(p).sum(axis=1) for p in prods))
    for _ in range(6):
        s_scan = -scan_model(terms, rng).astype(np.float64)
        assert (s_scan <= pre + margin).all()
        assert (s_scan >= pre - margin).all()


def round_up(x):
    f = x.astype(F32)
    return np.where(f.astype(np.float64) < x, np.nextafter(f, F32(np.inf)), f)


def fma_rn(a, b, c):
    """fmaf for scale in {1, 2} (a power of two: the product is exact) on operands whose exponents are close enough that the
    float64 sum is exact."""
    return (a.astype(np.float64) * b + c).astype(F32)


@pytest.mark.parametrize("scale", [1.0, 2.0])
@pytest.mark.parametrize("seed", range(4))
def test_bound_keeps_every_row_at_or_below_kth_above_each_pairs_threshold(scale, seed):
    rng = np.random.default_rng(seed)
    n = 200_000
    mag = np.exp2(rng.uniform(-20, 20, n))
    kth = (rng.standard_normal(n) * mag).astype(F32)
    add = (rng.standard_normal(n) * mag * np.exp2(rng.uniform(-4, 4, n))).astype(F32)
    if scale == 2.0:
        add = np.abs(add)  # L2 / cosine: add = |r|^2 (+ 1)
    M = (np.abs(add) * np.exp2(rng.uniform(0, 3, n)) * (rng.random(n) < 0.5) + np.abs(add)).astype(F32)  # >= |add|
    sc = F32(scale)
    # the kernel: B = ((kth + 2^-21 (|kth| + M)) + 1e-30), every step rounded upward
    marg = round_up(2.0 ** -21 * round_up(np.abs(kth).astype(np.float64) + M).astype(np.float64))
    B = round_up(round_up(kth.astype(np.float64) + marg).astype(np.float64) + 1e-30)
    # the largest score s whose merge value fmaf(scale, s, add) is still <= kth: binary search over the ordered fp32 bit
    # patterns around an estimate (the merge value is monotone in s)
    def key(f):
        b = f.view(np.int32).astype(np.int64)
        return np.where(b < 0, -(b & 0x7FFFFFFF), b)

    def unkey(kk):
        b = np.where(kk < 0, (-kk) | 0x80000000, kk)
        return b.astype(np.uint32).view(F32)

    k0 = key(((kth.astype(np.float64) - add) / scale).astype(F32))
    lo, hi = k0 - (1 << 26), k0 + (1 << 26)
    assert (fma_rn(sc, unkey(lo), add) <= kth).all() and (fma_rn(sc, unkey(hi), add) > kth).all()
    for _ in range(28):
        mid = (lo + hi) // 2
        ok = fma_rn(sc, unkey(mid), add) <= kth
        lo, hi = np.where(ok, mid, lo), np.where(ok, hi, mid)
    s = unkey(lo)
    assert (hi == lo + 1).all() and (fma_rn(sc, s, add) <= kth).all()
    # the scan's start of an item: thr = -((B - add) / scale); a row is a candidate iff -s > thr
    q = ((B - add).astype(F32) / sc).astype(F32)
    assert (s < q).all()
