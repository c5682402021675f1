"""k-means on the GPU against the oracle's assignment and the float64 model of tests/kmeans_ref.py, on data near and far from
the origin: labels bit-equal to `oracle.kmeans_assign` (fp32 expanded L2, ties to the smaller index), costs within
max(1e-6, d 2^-24) of the float64 cost of the returned labels and centres, sample weights and their normalisation, the
L2SqrtExpanded metric, the fixed-point Lloyd update against its documented bound, and k-means++ / strided fits end to end."""
import numpy as np
import pytest
import torch

import oracle
from tests import kmeans_ref as ref
from tests.util import clustered, uniform

pytestmark = pytest.mark.gpu


def _km():
    from cuvs_b200.cluster import kmeans
    return kmeans


# ---- data families: each returns float32 rows [n, d] from a seed
def _clustered(shift):
    def make(n, d, seed):
        x, _ = clustered(n, d, seed, n_centers=max(2, n // 1000))
        return (x + np.float32(shift)).astype(np.float32)
    return make


def _dim_shift(n, d, seed):
    x, _ = clustered(n, d, seed, n_centers=max(2, n // 1000))
    return (x + np.random.default_rng(seed + 1).uniform(0, 50, d).astype(np.float32)).astype(np.float32)


TIGHT_SIGMA = 0.25


def _tight(n, d, seed, shift=0.0):
    """32 tight clusters whose N(0, I) centres are scaled by 30 (so they lie far apart); returns the rows only."""
    return _tight_with_centres(n, d, seed, shift)[0]


def _tight_with_centres(n, d, seed, shift=0.0):
    centres = (30.0 * np.random.default_rng(seed + 7).standard_normal((32, d))).astype(np.float32)
    x, _ = clustered(n, d, seed, sigma=TIGHT_SIGMA, centers=centres)
    return (x + np.float32(shift)).astype(np.float32), (centres + np.float32(shift)).astype(np.float32)


FAMILIES = {
    "uniform": lambda n, d, seed: uniform(n, d, seed),
    "clustered": _clustered(0.0),
    "clustered+10": _clustered(10.0),
    "clustered+100": _clustered(100.0),
    "clustered-50": _clustered(-50.0),
    "dim_shift": _dim_shift,
    "tight_x30": _tight,
}


def _centres_from(x, k, seed):
    """k centres near the data: distinct rows of x moved by a small N(0, 0.05^2) step (so none coincides with a row)."""
    rng = np.random.default_rng(seed)
    rows = rng.choice(x.shape[0], size=k, replace=x.shape[0] < k)
    return (x[rows] + 0.05 * rng.standard_normal((k, x.shape[1]))).astype(np.float32)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _assert_cost(got, want, d, what):
    bar = ref.relative_cost_bar(d)
    rel = abs(got - want) / max(abs(want), 1e-300)
    assert rel <= bar, f"{what}: relative error {rel:.3e} > {bar:.3e} (got {got!r}, float64 {want!r})"


# (family, n, d, k): every k in {1, 2, 17, 300, 1024, 5000} and d in {1, 3, 64, 65, 300, 2048} appears, over all families;
# n keeps each oracle call to ~3e9 multiply-adds
LABEL_CASES = [
    ("uniform", 20000, 64, 17),
    ("uniform", 1500, 2048, 300),
    ("uniform", 40000, 1, 1024),
    ("uniform", 20000, 3, 5000),
    ("clustered", 20000, 65, 2),
    ("clustered", 8000, 300, 1024),
    ("clustered+10", 20000, 64, 300),
    ("clustered+10", 30000, 3, 17),
    ("clustered+100", 20000, 128, 300),
    ("clustered+100", 3000, 2048, 17),
    ("clustered+100", 20000, 3, 5000),
    ("clustered+100", 20000, 64, 1),
    ("clustered+100", 20000, 1, 300),
    ("clustered-50", 8000, 300, 1024),
    ("clustered-50", 20000, 65, 2),
    ("dim_shift", 20000, 64, 1024),
    ("dim_shift", 8000, 300, 300),
    ("tight_x30", 20000, 128, 32),
    ("tight_x30", 6000, 65, 5000),
]


@pytest.mark.parametrize("family,n,d,k", LABEL_CASES)
def test_predict_labels_and_costs_match_the_references(family, n, d, k):
    km = _km()
    x = FAMILIES[family](n, d, 11)
    c = _centres_from(x, k, 12)
    xg, cg = _dev(x), _dev(c)
    labels, inertia = km.predict(km.KMeansParams(n_clusters=k), xg, cg)
    labels = labels.cpu().numpy()
    ol, _ = oracle.kmeans_assign(x, c)
    bad = int((labels != ol).sum())
    assert bad == 0, f"{bad} of {n} labels differ from the oracle's argmin"
    # uint32 labels: the same values
    lu = torch.empty(n, dtype=torch.uint32, device="cuda")
    km.predict(km.KMeansParams(n_clusters=k), xg, cg, labels=lu)
    np.testing.assert_array_equal(lu.cpu().numpy().astype(np.int64), ol)
    want = ref.cost(x, c, ol)
    _assert_cost(inertia, want, d, "predict inertia")
    assert km.cluster_cost(xg, cg) == inertia  # the same fixed-order reduction


def test_labels_across_the_launch_chunk():
    """n = 2^20 + 1000 rows: the assignment runs in launches of 2^20 rows, and rows past the first launch must be labelled
    exactly as the first ones are."""
    km = _km()
    n, d, k = (1 << 20) + 1000, 8, 50
    x = FAMILIES["clustered+10"](n, d, 21)
    c = _centres_from(x, k, 22)
    labels, inertia = km.predict(km.KMeansParams(n_clusters=k), _dev(x), _dev(c))
    ol, _ = oracle.kmeans_assign(x, c)
    labels = labels.cpu().numpy()
    assert int((labels != ol).sum()) == 0
    _assert_cost(inertia, ref.cost(x, c, ol), d, "predict inertia")


@pytest.mark.parametrize("family", ["uniform", "clustered+100", "dim_shift"])
@pytest.mark.parametrize("normalize", [True, False])
def test_weighted_predict(family, normalize):
    km = _km()
    n, d, k = 20000, 32, 64
    x = FAMILIES[family](n, d, 31)
    c = _centres_from(x, k, 32)
    w = np.random.default_rng(33).uniform(0.1, 3.0, n).astype(np.float32)
    xg, cg = _dev(x), _dev(c)
    plain, _ = km.predict(km.KMeansParams(n_clusters=k), xg, cg)
    labels, inertia = km.predict(km.KMeansParams(n_clusters=k), xg, cg, sample_weights=_dev(w), normalize_weight=normalize)
    labels = labels.cpu().numpy()
    np.testing.assert_array_equal(labels, plain.cpu().numpy())  # weights do not move the labels
    ol, _ = oracle.kmeans_assign(x, c)
    np.testing.assert_array_equal(labels, ol)
    _assert_cost(inertia, ref.cost(x, c, ol, weights=w, normalize_weight=normalize), d, "weighted inertia")


def test_metric_and_non_finite_refusals():
    """predict takes L2Expanded and L2SqrtExpanded only, as the reference's kmeans_predict does; predict and cluster_cost
    refuse NaN or infinite rows and centroids, as fit does."""
    km = _km()
    x, c = uniform(1000, 8, 43), uniform(10, 8, 44)
    for metric in ("l2_unexpanded", "l2_sqrt_unexpanded", "inner_product"):
        with pytest.raises(Exception, match="L2Expanded or L2SqrtExpanded"):
            km.predict(km.KMeansParams(n_clusters=10, metric=metric), _dev(x), _dev(c))
    for bad_x, bad_c, what in ((True, False, "X contains NaN or infinity"), (False, True, "centroids contain NaN or infinity")):
        xb, cb = x.copy(), c.copy()
        if bad_x:
            xb[17, 3] = np.nan
        if bad_c:
            cb[4, 0] = np.inf
        with pytest.raises(Exception, match=what):
            km.predict(km.KMeansParams(n_clusters=10), _dev(xb), _dev(cb))
        with pytest.raises(Exception, match=what):
            km.cluster_cost(_dev(xb), _dev(cb))


@pytest.mark.parametrize("case", ["centres", "rows"])
def test_overflowing_norms_still_give_the_oracle_labels(case):
    """Finite values whose squared norms overflow fp32: with every |c|^2 infinite the scan keeps no candidate for any row, and
    with |x|^2 infinite every expanded distance is infinite.  Both take the exact path and label like the oracle (its first
    minimum, centre 0); every label stays below k."""
    km = _km()
    x, c = uniform(3000, 16, 45), uniform(20, 16, 46)
    if case == "centres":
        c = (c * np.float32(1e20)).astype(np.float32)
    else:
        x[::7] *= np.float32(1e20)
    labels, inertia = km.predict(km.KMeansParams(n_clusters=20), _dev(x), _dev(c))
    labels = labels.cpu().numpy()
    ol, _ = oracle.kmeans_assign(x, c)
    assert labels.min() >= 0 and labels.max() < 20
    np.testing.assert_array_equal(labels, ol)
    assert inertia == np.inf


def test_weight_refusals():
    km = _km()
    x, c = uniform(1000, 8, 41), uniform(10, 8, 42)
    with pytest.raises(Exception, match="sample_weight"):
        km.predict(km.KMeansParams(n_clusters=10), _dev(x), _dev(c), sample_weights=_dev(np.ones(999, np.float32)))
    with pytest.raises(Exception, match="sample weights are not supported"):
        km.fit(km.KMeansParams(n_clusters=10, max_iter=2), _dev(x), sample_weights=_dev(np.ones(1000, np.float32)))


@pytest.mark.parametrize("family", ["uniform", "clustered+100", "tight_x30"])
def test_l2_sqrt_expanded(family):
    """The reference takes the argmin on squared distances and the square root of the minimum (minClusterDistanceCompute:
    sqrt = metric != L2Expanded): labels as under L2Expanded, inertia sum_i sqrt(d_i)."""
    km = _km()
    n, d, k = 20000, 48, 100
    x = FAMILIES[family](n, d, 51)
    c = _centres_from(x, k, 52)
    xg, cg = _dev(x), _dev(c)
    sq_labels, _ = km.predict(km.KMeansParams(n_clusters=k), xg, cg)
    labels, inertia = km.predict(km.KMeansParams(n_clusters=k, metric="euclidean"), xg, cg)
    np.testing.assert_array_equal(labels.cpu().numpy(), sq_labels.cpu().numpy())
    ol, _ = oracle.kmeans_assign(x, c)
    np.testing.assert_array_equal(labels.cpu().numpy(), ol)
    _assert_cost(inertia, ref.cost(x, c, ol, sqrt=True), d, "L2SqrtExpanded predict inertia")
    cent, fit_inertia, _ = km.fit(km.KMeansParams(n_clusters=k, metric="euclidean", init_method="array", max_iter=2), xg,
                                  centroids=cg.clone())
    cent = cent.cpu().numpy()
    fl, _ = oracle.kmeans_assign(x, cent)
    _assert_cost(fit_inertia, ref.cost(x, cent, fl, sqrt=True), d, "L2SqrtExpanded fit inertia")


def _mixed_scale(n, d, seed):
    x = uniform(n, d, seed)
    x[:, 0] *= np.float32(1e4)
    x[:, 1] *= np.float32(1e-6)
    return x


@pytest.mark.parametrize("family", ["mixed_scale", "clustered+100", "clustered-50", "dim_shift"])
def test_lloyd_chain_against_float64_updates(family):
    """Eight fits of one Lloyd step each, every one starting from the previous GPU centres: each step's centres are within
    quantum / 2 + 1/2 ulp of the float64 mean over the oracle's labels, and a centre far from all data keeps its bits."""
    km = _km()
    n, d, k = 30000, 24, 40
    x = _mixed_scale(n, d, 61) if family == "mixed_scale" else FAMILIES[family](n, d, 61)
    c = _centres_from(x, k, 62)
    c[7] = x.max(0) + np.float32(1e5)  # no row is nearer to it than to another centre
    far = c[7].copy()
    q = ref.fixed_quantum(x)
    xg = _dev(x)
    for step in range(8):
        ol, _ = oracle.kmeans_assign(x, c)
        want, counts = ref.lloyd_update(x, ol, c)
        assert counts[7] == 0
        got, inertia, n_iter = km.fit(km.KMeansParams(n_clusters=k, init_method="array", max_iter=1), xg, centroids=_dev(c))
        got = got.cpu().numpy()
        assert n_iter == 1
        err = np.abs(got.astype(np.longdouble) - want)
        bar = ref.update_bound(got, want, q)
        worst = np.unravel_index(np.argmax(err / bar), err.shape)
        assert (err <= bar).all(), f"step {step}: centre {worst} off by {float(err[worst]):.3e} > {float(bar[worst]):.3e}"
        assert np.array_equal(got[7].view(np.uint32), far.view(np.uint32))
        fl, _ = oracle.kmeans_assign(x, got)
        _assert_cost(inertia, ref.cost(x, got, fl), d, f"step {step} fit inertia")
        c = got


@pytest.mark.parametrize("shift", [0.0, 100.0])
def test_kmeanspp_fit_finds_the_tight_clusters(shift):
    """Every generating centre has a fitted centroid within distance 0.05.  With ~4000 members a cluster's mean lies about
    sqrt(d sigma^2 / 4000) = 0.022 from its generating centre at d = 32."""
    km = _km()
    n, d = 128000, 32
    x, centres = _tight_with_centres(n, d, 71, shift)
    xg = _dev(x)
    cent, inertia, n_iter = km.fit(km.KMeansParams(n_clusters=32, max_iter=1), xg)
    cent = cent.cpu().numpy()
    dist = np.sqrt(((centres[:, None, :].astype(np.float64) - cent[None, :, :]) ** 2).sum(-1))
    assert (dist.min(axis=1) < 0.05).all(), dist.min(axis=1).max()
    assert inertia == pytest.approx(n * d * TIGHT_SIGMA ** 2, rel=0.1)
    assert n_iter == 1
    fl, _ = oracle.kmeans_assign(x, cent)
    _assert_cost(inertia, ref.cost(x, cent, fl), d, "k-means++ fit inertia")
    # the same centres give the same cost through predict and cluster_cost, to the bit
    _, p_inertia = km.predict(km.KMeansParams(n_clusters=32), xg, _dev(cent))
    assert p_inertia == inertia
    assert km.cluster_cost(xg, _dev(cent)) == inertia


def test_strided_init_above_4096_clusters():
    km = _km()
    n, d, k = 40000, 16, 4097
    x = FAMILIES["clustered+10"](n, d, 81)
    cent, inertia, n_iter = km.fit(km.KMeansParams(n_clusters=k, max_iter=2), _dev(x))
    cent = cent.cpu().numpy()
    assert 1 <= n_iter <= 2
    fl, _ = oracle.kmeans_assign(x, cent)
    _assert_cost(inertia, ref.cost(x, cent, fl), d, "strided fit inertia")


def test_host_data_and_repeated_fits_are_bit_equal():
    km = _km()
    n, d = 50000, 40
    x = FAMILIES["clustered+100"](n, d, 91)
    p = km.KMeansParams(n_clusters=60, max_iter=6, tol=1e-9)
    dev = [km.fit(p, _dev(x)) for _ in range(2)]
    host = km.fit(p, x)
    for other in (dev[1], host):
        assert torch.equal(dev[0][0], other[0])
        assert dev[0][1] == other[1] and dev[0][2] == other[2]
    assert 1 <= dev[0][2] <= 6
    cent = dev[0][0].cpu().numpy()
    fl, _ = oracle.kmeans_assign(x, cent)
    _assert_cost(dev[0][1], ref.cost(x, cent, fl), d, "fit inertia")
