"""Pins the nu-SVC / nu-SVR CPU oracle (tests/nu_oracle.c via tests/nu_oracle.py) to scikit-learn itself, bit for bit:
n_iter_, dual_coef_, intercept_ and the support."""
import os
import sys
import warnings

import numpy as np
import pytest
from sklearn.datasets import make_classification, make_regression
from sklearn.svm import NuSVC, NuSVR

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import nu_oracle as O                                                    # noqa: E402
from spark_sklearn_b200.estimators import materialize_svc                # noqa: E402


def _clf(n_classes, n, seed=0):
    return make_classification(n_samples=n, n_features=8, n_informative=5, n_classes=n_classes, random_state=seed)


def _reg(n, seed=0):
    X, y = make_regression(n_samples=n, n_features=8, noise=5.0, random_state=seed)
    return X, y / np.std(y)


def _pin_svc(X, y, rebuild_at_stop=False, **kw):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref = NuSVC(**kw).fit(X, y)
    classes, yc = np.unique(y, return_inverse=True)
    pc, rho, it = O.nusvc_fit(X, yc, kw.get("nu", 0.5), kw.get("kernel", "rbf"), ref._gamma, kw.get("tol", 1e-3),
                              kw.get("shrinking", True), kw.get("max_iter", -1), rebuild_at_stop)
    got = materialize_svc(NuSVC(**kw), X, yc, classes, pc, rho, it, ref._gamma)
    np.testing.assert_array_equal(got.n_iter_, ref.n_iter_)
    np.testing.assert_array_equal(got.support_, ref.support_)
    np.testing.assert_array_equal(got.dual_coef_, ref.dual_coef_)
    np.testing.assert_array_equal(got.intercept_, ref.intercept_)
    return ref


def _pin_svr(X, y, rebuild_at_stop=False, **kw):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref = NuSVR(**kw).fit(X, y)
    coef, rho, it = O.nusvr_fit(X, y, kw.get("nu", 0.5), kw.get("C", 1.0), kw.get("kernel", "rbf"), ref._gamma,
                                kw.get("tol", 1e-3), kw.get("shrinking", True), kw.get("max_iter", -1), rebuild_at_stop)
    assert it == ref.n_iter_
    np.testing.assert_array_equal(np.flatnonzero(coef), ref.support_)
    np.testing.assert_array_equal(coef[ref.support_], ref.dual_coef_[0])
    assert rho == -ref.intercept_[0]
    return ref


@pytest.mark.parametrize("kernel", ["rbf", "linear"])
@pytest.mark.parametrize("n_classes", [2, 3])
def test_nusvc_pinned(kernel, n_classes):
    X, y = _clf(n_classes, 300)
    for nu in (0.1, 0.3, 0.6):
        _pin_svc(X, y, nu=nu, kernel=kernel)


def test_nusvc_shrinking_unshrinking_and_shrinking_off():
    """600-row pair: shrinking from iteration 600 on, the unshrink near the end (1022 iterations); and with shrinking off"""
    X, y = _clf(2, 600, seed=1)
    assert _pin_svc(X, y, nu=0.2, gamma=0.5).n_iter_[0] > 600
    _pin_svc(X, y, nu=0.2, gamma=0.5, shrinking=False)


@pytest.mark.parametrize("rebuild_at_stop", [False, True])
@pytest.mark.parametrize("max_iter", [300, 700, 1000])
def test_max_iter_stops_before_and_after_the_first_shrink(max_iter, rebuild_at_stop):
    """300 and 700 / 1000 iterations on a 600-row NuSVC pair (first shrink at iteration 600) and on a 300-row NuSVR fit
    (600 variables).  libsvm takes rho straight from the active set at a max_iter stop (svm.cpp:728-731, 899-901); with
    free variables on both sides rho does not read the shrunk ones, so rebuilding their gradient first gives the same bits
    here: both variants equal scikit-learn."""
    X, y = _clf(2, 600, seed=1)
    assert _pin_svc(X, y, rebuild_at_stop, nu=0.2, gamma=0.5, max_iter=max_iter).n_iter_[0] == max_iter
    X, y = _reg(300)
    assert _pin_svr(X, y, rebuild_at_stop, nu=0.4, C=10.0, max_iter=max_iter).n_iter_ == max_iter


def test_class_weight_has_no_effect_on_nusvc():
    X, y = _clf(3, 300)
    a = _pin_svc(X, y, nu=0.3, class_weight={0: 2.0})
    b = _pin_svc(X, y, nu=0.3)
    np.testing.assert_array_equal(a.n_iter_, b.n_iter_)
    np.testing.assert_array_equal(a.intercept_, b.intercept_)
    np.testing.assert_array_equal(a.support_, b.support_)


def test_infeasible_nu():
    X, y = make_classification(n_samples=300, n_features=8, weights=[0.7, 0.3], random_state=0)
    with pytest.raises(ValueError, match="specified nu is infeasible"):
        NuSVC(nu=0.9).fit(X, y)
    _, yc = np.unique(y, return_inverse=True)
    with pytest.raises(ValueError, match="specified nu is infeasible"):
        O.nusvc_fit(X, yc, 0.9)
    assert O.nusvc_infeasible(0.9, yc) and not O.nusvc_infeasible(0.3, yc)


@pytest.mark.parametrize("kernel", ["rbf", "linear"])
def test_nusvr_pinned(kernel):
    X, y = _reg(300)
    for nu, C in ((0.1, 1.0), (0.5, 10.0), (0.9, 3.0)):
        _pin_svr(X, y, nu=nu, C=C, kernel=kernel)
    _pin_svr(X, y, nu=0.4, C=10.0, shrinking=False)
