"""Pins the LinearSVC oracle (tests/linsvc_oracle.c) to sklearn.svm.LinearSVC(dual=False): n_iter_ equal, coef_ and
intercept_ within 1e-12 relative to the largest weight (scikit-learn's dot / nrm2 go through OpenBLAS, the oracle's are
sequential loops, so the two differ by reordered float64 sums)."""
import warnings

import numpy as np
import pytest
from sklearn.datasets import make_classification
from sklearn.exceptions import ConvergenceWarning
from sklearn.svm import LinearSVC

from linsvc_oracle import LinearSVCOracle


def _data(n_classes=2, n=600, d=20, seed=0):
    return make_classification(n, d, n_informative=6, n_classes=n_classes, random_state=seed)


def _check(X, y, sample_weight=None, **kw):
    o = LinearSVCOracle(X, y, sample_weight=sample_weight, trace=True, **kw)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        s = LinearSVC(dual=False, **kw).fit(X, y, sample_weight=sample_weight)
    assert o.n_iter_ == s.n_iter_
    scale = np.abs(s.coef_).max()
    assert np.abs(o.coef_ - s.coef_).max() <= 1e-12 * scale
    assert np.abs(np.asarray(o.intercept_) - s.intercept_).max() <= 1e-12 * scale
    np.testing.assert_array_equal(o.predict(X), s.predict(X))
    return o


@pytest.mark.parametrize("C", [1e-3, 1.0, 100.0])
def test_binary(C):
    _check(*_data(), C=C)


def test_three_class_one_vs_rest():
    o = _check(*_data(3, seed=1))
    assert len(o.n_iter_per_fit) == 3


@pytest.mark.parametrize("cw", ["balanced", {0: 3.0, 1: 0.5}])
def test_class_weight(cw):
    _check(*_data(), class_weight=cw)


def test_class_weight_one_vs_rest():
    _check(*_data(3, seed=1), class_weight={0: 2.0, 2: 0.5})


def test_sample_weight_with_zeros():
    X, y = _data()
    sw = np.random.RandomState(0).uniform(0, 2, len(X))
    sw[::7] = 0.0
    _check(X, y, sample_weight=sw)


def test_no_intercept_and_intercept_scaling():
    X, y = _data()
    _check(X, y, fit_intercept=False)
    _check(X, y, intercept_scaling=5.0)


def test_rejected_steps():
    """large C on nearly separable data: the first Newton steps overshoot and TRON rejects them (actred <= eta0 prered)"""
    X, y = make_classification(40, 3, n_informative=3, n_redundant=0, class_sep=5.0, random_state=1)
    o = _check(X, y, C=1000.0)
    assert any(not r["accepted"] for r in o.trace[0])


def test_stops_at_max_iter():
    X, y = _data()
    o = _check(X, y, max_iter=2, tol=1e-12)
    assert o.n_iter_ == 2
