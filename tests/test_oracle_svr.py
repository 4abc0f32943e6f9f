"""Pins the epsilon-SVR CPU oracle (tests/svr_oracle.py) to scikit-learn itself, bit for bit, and measures how much the
order of the training rows moves the split scores (the bound the GPU general-splitter test uses)."""
import os
import sys
import warnings

import numpy as np
import pytest
from sklearn.exceptions import ConvergenceWarning
from sklearn.svm import SVR

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import svr_oracle as O                                                   # noqa: E402
from conftest import golden                                              # noqa: E402
from spark_sklearn_b200 import workloads as W                            # noqa: E402

# largest |split score| difference between fitting a split's training rows in ascending order and in the splitter's
# order: measured with this oracle on svr_small with ShuffleSplit (test_row_order_sensitivity) as 4.4e-16 (whole grid,
# n_iter identical on every fit); the GPU test allows this with a margin for the summation order of the decision values
ORDER_BOUND = 1e-12


def _data(n):
    w = W.make_workload("svr_small")
    return w["X"][:n], w["y"][:n]


def _pin(X, y, **kw):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        ref = SVR(**kw).fit(X, y)
    g = ref._gamma
    coef, rho, it = O.svr_solve(X, y, kw.get("C", 1.0), kw.get("epsilon", 0.1), kw.get("kernel", "rbf"), g,
                                kw.get("tol", 1e-3), kw.get("shrinking", True), kw.get("max_iter", -1))
    c = np.zeros(len(X))
    c[ref.support_] = ref.dual_coef_[0]
    assert it == ref.n_iter_
    np.testing.assert_array_equal(coef, c)
    assert rho == -ref.intercept_[0]
    np.testing.assert_array_equal(np.flatnonzero(coef), ref.support_)
    np.testing.assert_allclose(O.predict(X, coef, rho, X, kw.get("kernel", "rbf"), g), ref.predict(X), rtol=0, atol=1e-12)
    return it


@pytest.mark.parametrize("kw", [
    dict(C=1.0, epsilon=0.1, gamma=1 / 32),
    dict(C=10.0, epsilon=0.0, gamma="scale"),                           # epsilon = 0
    dict(C=3.0, epsilon=0.2, gamma="auto", shrinking=False),
    dict(kernel="linear", C=0.1, epsilon=0.2),
    dict(C=100.0, epsilon=0.05, gamma=1 / 32, max_iter=200),             # max_iter stop before the first shrink
], ids=["rbf", "eps0", "noshrink", "linear", "maxiter_early"])
def test_oracle_equals_sklearn_svr(kw):
    _pin(*_data(300), **kw)


def test_oracle_shrinks_unshrinks_and_stops_after_a_shrink():
    """800 rows (1600 variables): shrinking every 1000 iterations, the unshrink near the end, and a max_iter stop with
    shrunk variables (rho over all 2l positions after reconstruct_gradient)"""
    X, y = _data(800)
    assert _pin(X, y, C=100.0, epsilon=0.05, gamma=1 / 32) > 1500
    assert _pin(X, y, C=100.0, epsilon=0.05, gamma=1 / 32, max_iter=1500) == 1500


def test_oracle_equals_golden():
    """the committed svr_small golden (scikit-learn 1.9) on a few candidates"""
    from sklearn.model_selection import KFold, ParameterGrid
    w = W.make_workload("svr_small")
    g = golden("svr_small")
    cands = list(ParameterGrid(w["param_grid"]))
    pick = [0, 9, 23]
    te, it = O.cv_scores_svr(w["X"], w["y"], list(KFold(5).split(w["X"])), [cands[i] for i in pick])
    np.testing.assert_array_equal(it, g["n_iter"][pick])
    np.testing.assert_allclose(te, g["test_scores"][pick], rtol=0, atol=1e-12)


def test_row_order_sensitivity():
    """ascending training order (what the GPU path fits) against the splitter's permuted order, ShuffleSplit"""
    from sklearn.model_selection import ShuffleSplit
    X, y = _data(600)
    splits = list(ShuffleSplit(4, test_size=0.25, random_state=0).split(X))
    asc = [(np.sort(tr), te) for tr, te in splits]
    cands = [{"C": 1.0, "gamma": 1 / 32}, {"C": 10.0, "gamma": 1 / 32}]
    a, ia = O.cv_scores_svr(X, y, asc, cands)
    b, ib = O.cv_scores_svr(X, y, splits, cands)
    np.testing.assert_array_equal(ia, ib)
    assert np.abs(a - b).max() <= ORDER_BOUND / 100
