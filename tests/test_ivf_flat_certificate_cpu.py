"""A numpy model of IVF-Flat's fine-scan certificate (csrc/ivf_flat.cu: flat_budget, certify_kernel; DESIGN.md §4).

The scan's approximate distance of a row x of a pair (q, list centre c) is A = add + 2 (hn - bf16(q - c) . bf16(x - c)), with
add = |q - c|^2 and hn = |x - c|^2 / 2 in fp32 and the dot product accumulated in fp32 in an order the tensor cores choose
(inner product: A = -q.c - bf16(q) . bf16(x - c)).  The re-score's exact distance F is a fp32 fmaf chain over ascending
components.  The model checks that the error budget covers |A - F| on inputs built to stress it, that a query the
certificate accepts has the exact top k, and that the certificate does reject the near-duplicate family the bf16 ranking
alone gets wrong."""
import numpy as np
import pytest

from tests.util import clustered

U32 = 2.0 ** -23


def bf16(x):
    """Round float32 to bfloat16 (nearest, ties to even), returned as float32."""
    b = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    return b.astype(np.uint32).view(np.float32)


def f32_chain(terms):
    """sum of terms[..., j] over ascending j, rounded to fp32 after every step (an fmaf chain of exact products)."""
    acc = np.zeros(terms.shape[:-1], np.float64)
    for j in range(terms.shape[-1]):
        acc = np.float32(acc + terms[..., j]).astype(np.float64)
    return acc


def tc_sum(terms, rng):
    """fp32 sum of terms[..., j] in a random order, per row: the tensor cores' accumulation order is not specified."""
    perm = rng.permuted(np.broadcast_to(np.arange(terms.shape[-1]), terms.shape), axis=-1)
    return f32_chain(np.take_along_axis(terms, perm, axis=-1))


def scan_model(q, c, x, rng, ip=False):
    """Approximate distances A [nq, n] of rows x [n, d] in the list of centre c for queries q [nq, d] (fp32 inputs)."""
    q, c, x = (np.asarray(a, np.float32) for a in (q, c, x))
    b = bf16(x - c).astype(np.float64)
    if ip:
        a = bf16(q).astype(np.float64)
        add = -f32_chain((q.astype(np.float64) * c)[:, :])
        s = -tc_sum(a[:, None, :] * b[None, :, :], rng)
        return np.float32(add[:, None] + s).astype(np.float64)
    a = bf16(q - c).astype(np.float64)
    add = f32_chain(((q - c).astype(np.float64)) ** 2)
    hn = 0.5 * f32_chain(((x - c).astype(np.float64)) ** 2)
    s = tc_sum(np.concatenate([-a[:, None, :] * b[None, :, :], np.broadcast_to(hn[None, :, None], (len(q), len(x), 1))], -1), rng)
    return np.float32(add[:, None] + 2.0 * s).astype(np.float64)


def exact_model(q, x, ip=False):
    """The re-score's fp32 distance: sum (q - x)^2, or -q.x for inner product, as fmaf chains."""
    q, x = np.asarray(q, np.float32), np.asarray(x, np.float32)
    if ip:
        return -f32_chain(q.astype(np.float64)[:, None, :] * x[None, :, :])
    return f32_chain(((q[:, None, :] - x[None, :, :]).astype(np.float64)) ** 2)


def budget(q, c, x, ip=False):
    """flat_budget::eps of every query against the list (Kp = d rounded up to 64)."""
    d = q.shape[1]
    kp = (d + 63) // 64 * 64
    scale = 1.0 if ip else 2.0
    c_bf, c_acc, c_fp = scale * (2.0 ** -8 + 2.0 ** -16), scale * (kp + 20) * 2.0 ** -22, (2 * d + 16) * U32
    R = np.sqrt(((x.astype(np.float64) - c) ** 2).sum(1).max())
    if ip:
        Q, C = np.linalg.norm(q.astype(np.float64), axis=1), np.linalg.norm(c.astype(np.float64))
        return (c_bf + 1.01 * c_acc) * Q * R + c_fp * Q * (2 * C + R)
    Q = np.linalg.norm(q.astype(np.float64) - c, axis=1)
    return c_bf * Q * R + c_acc * (1.01 * Q * R + 0.5 * R * R) + c_fp * (Q + R) ** 2


def _stress_inputs(kind, rng, d=128):
    """(queries, centre, rows) built against the budget."""
    c = rng.standard_normal(d).astype(np.float32)
    x = (c + 0.25 * rng.standard_normal((400, d))).astype(np.float32)
    q = (c + 0.25 * rng.standard_normal((16, d))).astype(np.float32)
    if kind == "outlier":  # one row far from its centre sets R for the whole list
        x[7] = c + 40.0 * rng.standard_normal(d)
    elif kind == "far_query":  # inner product: a query of norm ~10^3
        q = (300.0 * rng.standard_normal((16, d))).astype(np.float32)
    elif kind == "cancellation":  # q - c and x - c large and nearly equal: a small distance out of large terms
        off = 50.0 * rng.standard_normal(d)
        x = (c + off + 1e-2 * rng.standard_normal((400, d))).astype(np.float32)
        q = (c + off + 1e-2 * rng.standard_normal((16, d))).astype(np.float32)
    elif kind == "shifted":  # everything 100 from the origin
        c, x, q = c + 100.0, x + 100.0, q + 100.0
    return q, c, x


@pytest.mark.parametrize("ip", [False, True], ids=["l2", "ip"])
@pytest.mark.parametrize("kind", ["plain", "outlier", "far_query", "cancellation", "shifted"])
def test_budget_covers_the_scan_error(kind, ip):
    rng = np.random.default_rng(["plain", "outlier", "far_query", "cancellation", "shifted"].index(kind) + 10 * ip)
    q, c, x = _stress_inputs(kind, rng)
    F = exact_model(q, x, ip)
    eps = budget(q, c, x, ip)
    for _ in range(3):  # accumulation orders
        err = np.abs(scan_model(q, c, x, rng, ip) - F)
        assert (err <= eps[:, None]).all(), f"error {err.max():.3e} above the budget {eps.min():.3e}"
    # and not vacuous: the worst observed error reaches a fiftieth of its query's budget (a budget 50x above every error seen
    # would flag queries for nothing)
    assert (err / eps[:, None]).max() > 0.02


def certify(A, F, k, kc2, eps):
    """The model of certify_kernel for one list: candidates are the kc2 best rows by A (ties: smaller row); the answer is the
    k best candidates by (F, row); certified iff its k-th F is strictly below the kc2-th A minus eps.  -> (answer rows, ok)."""
    order = np.lexsort((np.arange(A.shape[1])[None, :].repeat(len(A), 0), A), axis=1)[:, :kc2]
    out, ok = [], []
    for i, cand in enumerate(order):
        fc = F[i, cand]
        best = cand[np.lexsort((cand, fc))][:k]
        floor = A[i, order[i, -1]] if A.shape[1] > kc2 else np.inf
        out.append(best)
        ok.append(F[i, best[-1]] < floor - eps[i])
    return np.array(out), np.array(ok)


def _exact_topk(F, k):
    rows = np.arange(F.shape[1])[None, :].repeat(len(F), 0)
    return np.lexsort((rows, F), axis=1)[:, :k]


def _dups(reps, jitter, rng, d=128, n_base=60, nq=24):
    centers = rng.standard_normal((1, d)).astype(np.float32)
    base, _ = clustered(n_base, d, int(rng.integers(1 << 30)), centers=centers)
    x = (np.repeat(base, reps, axis=0) + jitter * rng.standard_normal((n_base * reps, d))).astype(np.float32)
    q = (base[rng.choice(n_base, nq)] + 0.1 * rng.standard_normal((nq, d))).astype(np.float32)
    return q, centers[0], x


@pytest.mark.parametrize("k", [1, 10, 32])
@pytest.mark.parametrize("family", ["clustered", "dups20", "dups100"])
def test_certified_queries_have_the_exact_top_k(family, k):
    rng = np.random.default_rng([["clustered", "dups20", "dups100"].index(family), k])
    if family == "clustered":
        q, c, x = _stress_inputs("plain", rng)
    else:
        q, c, x = _dups(int(family[4:]), 1e-3, rng)
    A, F = scan_model(q, c, x, rng), exact_model(q, x)
    kc2 = max(32, 2 * k)
    got, ok = certify(A, F, k, kc2, budget(q, c, x))
    want = _exact_topk(F, k)
    # a certified query's answer is the exact one, distances and rows (ties at the k-th distance aside)
    np.testing.assert_array_equal(np.take_along_axis(F, got, 1)[ok], np.take_along_axis(F, want, 1)[ok])
    if family == "clustered":
        assert ok.mean() >= 0.9, f"only {ok.sum()} of {len(ok)} ordinary queries certified"


def test_certificate_rejects_the_near_duplicate_family():
    """100 jittered copies (1e-3) of every base row: the 32 best bf16 scores miss true top-10 rows, and the certificate must
    send (nearly) every query to the exact fallback, including every query whose candidates lost a neighbour."""
    rng = np.random.default_rng(5)
    q, c, x = _dups(100, 1e-3, rng)
    A, F = scan_model(q, c, x, rng), exact_model(q, x)
    got, ok = certify(A, F, 10, 32, budget(q, c, x))
    want = _exact_topk(F, 10)
    lost = (np.take_along_axis(F, got, 1) != np.take_along_axis(F, want, 1)).any(1)
    assert lost.any(), "the family no longer stresses the bf16 ranking"
    assert not (lost & ok).any()
    assert (~ok).mean() >= 0.9


def certify_lists(q, lists, k, rng):
    """The model of the k <= 64 search and its certificate over several lists (pairs) of one batch of queries: the rows of a list
    sit in 128-row tiles whose columns 0-63 and 64-127 form two column halves; each half keeps its KC best rows by A (KC 16 when
    k + k/2 <= 16, else 32; ties: smaller row); the merge keeps the kc2 = max(32, 2k) best kept rows; the answer is the k best
    merged rows by (F, row).  floor = min(kc2-th merged A when more rows were kept, the last kept A of every full half), and a
    query is certified iff its k-th F < floor - eps, eps the largest budget of its lists.  (The shared pruning bound is not
    modelled: it only drops rows above some full half's last entry.)  -> (answer rows into the concatenated lists, ok)."""
    KC, kc2 = (16 if k + k // 2 <= 16 else 32), max(32, 2 * k)
    A = np.concatenate([scan_model(q, c, x, rng) for c, x in lists], 1)
    F = np.concatenate([exact_model(q, x) for _, x in lists], 1)
    eps = np.max([budget(q, c, x) for c, x in lists], 0)
    starts = np.cumsum([0] + [len(x) for _, x in lists])
    out, ok = [], []
    for i in range(len(q)):
        kept, floor = [], np.inf
        for li in range(len(lists)):
            rows = np.arange(starts[li], starts[li + 1])
            half = ((rows - starts[li]) % 128) >= 64
            for h in (False, True):
                r = rows[half == h]
                best = r[np.lexsort((r, A[i, r]))][:KC]
                kept.append(best)
                if len(best) == KC and len(r) > KC:
                    floor = min(floor, A[i, best[-1]])
        kept = np.concatenate(kept)
        merged = kept[np.lexsort((kept, A[i, kept]))][:kc2]
        if len(kept) > kc2:
            floor = min(floor, A[i, merged[-1]])
        best = merged[np.lexsort((merged, F[i, merged]))][:k]
        out.append(best)
        ok.append(F[i, best[-1]] < floor - eps[i])
    return np.array(out), np.array(ok), F


@pytest.mark.parametrize("k", [10, 48])
@pytest.mark.parametrize("family", ["clustered", "dups100"])
def test_certified_queries_with_column_halves_and_two_lists(family, k):
    """The floor argument with its per-half lists: a certified query's answer over two probed lists is the exact top k."""
    rng = np.random.default_rng([["clustered", "dups100"].index(family), k, 7])
    if family == "clustered":
        q, c0, x0 = _stress_inputs("plain", rng)
    else:
        q, c0, x0 = _dups(100, 1e-3, rng, n_base=20, nq=16)
    c1 = (c0 + 0.5 * rng.standard_normal(c0.shape)).astype(np.float32)
    x1 = (c1 + 0.25 * rng.standard_normal((300, len(c0)))).astype(np.float32)
    got, ok, F = certify_lists(q, [(c0, x0), (c1, x1)], k, rng)
    want = _exact_topk(F, k)
    np.testing.assert_array_equal(np.take_along_axis(F, got, 1)[ok], np.take_along_axis(F, want, 1)[ok])
    if family == "clustered":
        # k = 48: the query's nearest rows fill both halves of its own list, whose 32nd entries then lie next to the 48th
        # distance, and most of those queries go to the fallback (DESIGN.md §4); k = 10 must certify nearly every query
        assert k > 32 or ok.mean() >= 0.9, f"only {ok.sum()} of {len(ok)} ordinary queries certified"
    else:
        lost = (np.take_along_axis(F, got, 1) != np.take_along_axis(F, want, 1)).any(1)
        assert lost.any() and (~ok).mean() >= 0.9
