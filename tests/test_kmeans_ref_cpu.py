"""The float64 k-means model of tests/kmeans_ref.py against direct restatements and hand-checked cases."""
import math

import numpy as np
import pytest

from tests import kmeans_ref as ref
from tests.util import clustered, uniform


def test_assign_is_the_nearest_centre_and_ties_go_to_the_smaller_index():
    x = np.array([[0.0, 0.0], [1.0, 0.0], [2.0, 2.0], [0.5, 0.0]], np.float32)
    c = np.array([[1.0, 0.0], [0.0, 0.0], [2.0, 2.0], [0.0, 0.0]], np.float32)
    # x3 is equidistant from c0 and c1 (and c3 duplicates c1): the smallest index wins
    np.testing.assert_array_equal(ref.assign(x, c), [1, 0, 2, 0])
    x, c = uniform(500, 7, 1), uniform(40, 7, 2)
    brute = np.array([min(range(40), key=lambda j: (float(((x[i].astype(np.float64) - c[j]) ** 2).sum()), j)) for i in range(500)])
    np.testing.assert_array_equal(ref.assign(x, c), brute)


def test_cost_weights_normalisation_and_sqrt():
    x = np.array([[0.0, 0.0], [3.0, 4.0], [1.0, 1.0]], np.float32)
    c = np.array([[0.0, 0.0]], np.float32)
    lab = np.zeros(3, np.int64)
    assert ref.cost(x, c, lab) == 0 + 25 + 2
    assert ref.cost(x, c, lab, sqrt=True) == pytest.approx(0 + 5 + math.sqrt(2), rel=1e-15)
    w = np.array([1.0, 2.0, 3.0])
    assert ref.cost(x, c, lab, weights=w) == 50 + 6
    assert ref.cost(x, c, lab, weights=w, normalize_weight=True) == pytest.approx(56 * 3 / 6, rel=1e-15)
    assert ref.cost(x, c, lab, weights=w, normalize_weight=True, sqrt=True) == pytest.approx((10 + 3 * math.sqrt(2)) / 2, rel=1e-15)
    # from differences: far from the origin the expanded form |x|^2 - 2 x.c + |c|^2 cancels, the differences do not
    big = np.full((1, 128), 1.0e4, np.float32)
    assert ref.cost(big + np.float32(0.25), big, np.zeros(1, np.int64)) == 128 * 0.0625


def test_lloyd_update_means_and_empty_clusters_keep_their_centre():
    x, _ = clustered(3000, 5, 3, n_centers=4)
    c_old = np.vstack([x[:4], np.full((1, 5), 1e6, np.float32)])  # centre 4 is far from everything
    lab = ref.assign(x, c_old)
    new, counts = ref.lloyd_update(x, lab, c_old)
    assert counts[4] == 0 and counts.sum() == 3000
    assert (new[4] == np.float32(1e6)).all()
    for j in range(4):
        np.testing.assert_allclose(new[j].astype(np.float64), x[lab == j].astype(np.float64).mean(0), rtol=1e-14, atol=1e-15)


def test_fixed_quantum_matches_the_device_rule():
    # max|x| = 3 < 2^2, n = 1000 < 2^10: unit 2^(2 + 10 - 62)
    x = np.zeros((1000, 2), np.float32)
    x[5, 1] = -3.0
    assert ref.fixed_quantum(x) == 2.0 ** -50
    x[5, 1] = 4.0  # frexp(4) = (0.5, 3): 4 < 2^3
    assert ref.fixed_quantum(x) == 2.0 ** -49
    assert ref.fixed_quantum(x, n=1024) == 2.0 ** -48  # 1024 < 2^11
    assert ref.fixed_quantum(np.zeros((1, 1), np.float32)) == 2.0 ** -61


def test_the_fixed_point_mean_is_within_the_bound():
    """A direct model of the device update (v * 2^e rounded to an int64 per term, summed, divided, cast to fp32) stays inside
    update_bound on mixed-scale columns, and a mean moved by three quanta does not."""
    rng = np.random.default_rng(5)
    x = uniform(4000, 3, 6)
    x[:, 1] *= 1e4
    x[:, 2] *= 1e-6
    lab = rng.integers(0, 7, 4000)
    q = ref.fixed_quantum(x)
    exact, counts = ref.lloyd_update(x, lab, np.zeros((7, 3), np.float32))
    model = np.empty((7, 3), np.float32)
    for j in range(7):
        units = [sum(int(round(float(v) / q)) for v in x[lab == j, col]) for col in range(3)]
        model[j] = [np.float32(u * q / counts[j]) for u in units]
    bar = ref.update_bound(model, exact, q)
    assert (np.abs(model.astype(np.longdouble) - exact) <= bar).all()
    assert not (np.abs((model.astype(np.longdouble) + 3 * q) - exact) <= ref.update_bound(model, exact, q))[:, 2].all()
