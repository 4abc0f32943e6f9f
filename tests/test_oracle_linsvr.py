"""The LinearSVR oracle (tests/linsvr_oracle.c) against scikit-learn's own LinearSVR: the dual CD (solvers 12 and 13) bit for
bit on coef_, intercept_ and n_iter_; TRON (solver 11) with n_iter_ equal and the weights within 1e-12 relative; the RNG
against numpy's legacy-seeded MT19937.  The kernel-order switch (the dot products summed as csrc/linsvr.cu's warp sums them)
must keep the CD's trajectory: n_iter_ equal, weights within 1e-12 relative."""
import warnings

import numpy as np
import pytest
from sklearn.exceptions import ConvergenceWarning
from sklearn.svm import LinearSVR

from linsvr_oracle import LinearSVROracle, mt_draws, seed_of
from spark_sklearn_b200 import workloads as W


def _data(n=1200, key="linsvr_small"):
    w = W.make_workload(key)
    return w["X"][:n].astype(np.float64), w["y"][:n]


def _sk(X, y, sw=None, **kw):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        return LinearSVR(**kw).fit(X, y, sample_weight=sw)


def _weights(n):
    rng = np.random.RandomState(1)
    w = rng.uniform(0.5, 2.0, n)
    w[rng.rand(n) < 0.1] = 0.0
    return w


CD_CASES = [
    dict(random_state=0),
    dict(random_state=7, C=10.0, epsilon=0.1),
    dict(random_state=0, loss="squared_epsilon_insensitive", dual=True, C=0.5),
    dict(random_state=3, loss="squared_epsilon_insensitive", dual=True, C=5.0, epsilon=0.2),
    dict(random_state=0, fit_intercept=False),
    dict(random_state=0, intercept_scaling=3.0, C=3.0),
    dict(random_state=0, max_iter=7),                        # a max_iter stop inside the shuffled epochs
    dict(random_state=0, tol=1e-1),                          # a tolerance stop, with unshrinking
    dict(random_state=0, loss="squared_epsilon_insensitive", dual=True, tol=1e-2, C=0.05),
]


@pytest.mark.parametrize("kw", CD_CASES, ids=[str(i) for i in range(len(CD_CASES))])
@pytest.mark.parametrize("rows", ["ordered", "permuted", "weighted"])
def test_dual_cd_bit_for_bit(kw, rows):
    X, y = _data()
    sw = None
    if rows == "permuted":
        p = np.random.RandomState(3).permutation(len(X))
        X, y = X[p], y[p]
    elif rows == "weighted":
        sw = _weights(len(X))
    ref = _sk(X, y, sw, **kw)
    o = LinearSVROracle(X, y, sample_weight=sw, **kw)
    assert o.solver in (12, 13)
    assert o.n_iter_ == ref.n_iter_
    np.testing.assert_array_equal(o.coef_, ref.coef_)
    np.testing.assert_array_equal(o.intercept_, ref.intercept_)
    k = LinearSVROracle(X, y, sample_weight=sw, kernel_order=True, **kw)
    assert k.n_iter_ == ref.n_iter_
    scale = max(np.abs(ref.coef_).max(), np.abs(np.asarray(ref.intercept_)).max())
    assert np.abs(k.coef_ - ref.coef_).max() <= 1e-12 * scale
    assert np.abs(np.asarray(k.intercept_) - np.asarray(ref.intercept_)).max() <= 1e-12 * scale


def test_row_order_changes_the_cd_result():
    """the CD permutes positions of X[train]: the same rows in another order give another fit (why the splitter's training
    order reaches the device)"""
    X, y = _data()
    p = np.random.RandomState(3).permutation(len(X))
    a = LinearSVROracle(X, y, random_state=0)
    b = LinearSVROracle(X[p], y[p], random_state=0)
    assert not np.array_equal(a.coef_, b.coef_)


def test_zero_weights_are_dropped_in_order():
    """train's remove_zero_weight: a fit with zero-weight rows equals the fit on the remaining rows"""
    X, y = _data(600)
    sw = _weights(len(X))
    keep = sw > 0
    a = LinearSVROracle(X, y, sample_weight=sw, random_state=0, max_iter=50)
    b = LinearSVROracle(X[keep], y[keep], sample_weight=sw[keep], random_state=0, max_iter=50)
    np.testing.assert_array_equal(a.coef_, b.coef_)


@pytest.mark.parametrize("kw", [dict(loss="squared_epsilon_insensitive", dual=False),
                                dict(loss="squared_epsilon_insensitive", dual=False, C=100.0, epsilon=0.1, tol=1e-8),
                                dict(loss="squared_epsilon_insensitive", dual="auto", fit_intercept=False)])
@pytest.mark.parametrize("weighted", [False, True])
def test_tron_solver_11(kw, weighted):
    X, y = _data()
    sw = _weights(len(X)) if weighted else None
    ref = _sk(X, y, sw, **kw)
    o = LinearSVROracle(X, y, sample_weight=sw, **kw)
    assert o.solver == 11
    assert o.n_iter_ == ref.n_iter_
    scale = max(np.abs(ref.coef_).max(), np.abs(np.asarray(ref.intercept_)).max())
    assert np.abs(o.coef_ - ref.coef_).max() <= 1e-12 * scale
    assert np.abs(np.asarray(o.intercept_) - np.asarray(ref.intercept_)).max() <= 1e-12 * scale


def test_wide_auto_resolves_to_the_dual():
    X, y = _data(300, "linsvr_wide")
    ref = _sk(X[:200], y[:200], loss="squared_epsilon_insensitive", random_state=0)
    o = LinearSVROracle(X[:200], y[:200], loss="squared_epsilon_insensitive", random_state=0)
    assert o.solver == 12 and o.n_iter_ == ref.n_iter_
    np.testing.assert_array_equal(o.coef_, ref.coef_)


@pytest.mark.parametrize("seed", [0, 1, 5489, 2 ** 31 - 2])
def test_rng_is_numpy_legacy_mt19937(seed):
    bg = np.random.MT19937()
    bg._legacy_seeding(seed)
    ref = bg.random_raw(2000).astype(np.uint32)
    np.testing.assert_array_equal(mt_draws(seed, 2000), ref)


def test_seed_rule():
    assert seed_of(0) == np.random.RandomState(0).randint(np.iinfo("i").max)
    rs = np.random.RandomState(4)
    assert seed_of(rs) == np.random.RandomState(4).randint(np.iinfo("i").max)
