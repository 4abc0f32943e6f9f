"""The poly / sigmoid C-SVC oracle (tests/svc_kernels_oracle.c) against scikit-learn: bit-identical n_iter_, dual_coef_,
intercept_ and predictions, and the committed golden svc_kernels_mid.npz (scikit-learn 1.9 on the config-2 data recipe)."""
import numpy as np
import pytest
from sklearn.base import clone
from sklearn.svm import SVC

import svc_kernels_oracle as KO
from conftest import golden
from spark_sklearn_b200 import workloads as W
from spark_sklearn_b200.estimators import materialize_svc

CASES = [("poly", dg, c0) for dg in (0, 1, 2, 3, 5) for c0 in (0.0, 1.0, -1.0)] + [("sigmoid", 3, c0) for c0 in (0.0, 1.0, -1.0)]


def _data(n, n_classes, seed=0, **kw):
    from sklearn.datasets import make_classification
    X, y = make_classification(n, 20, n_informative=6, n_classes=n_classes, n_clusters_per_class=1, random_state=seed, **kw)
    return X.astype(np.float32).astype(np.float64), y


def _fit_oracle(X, S, y, est):
    """the oracle's one-vs-one model as a fitted sklearn.svm.SVC (the refit path's materialize_svc)"""
    p = est.get_params()
    classes, yc = np.unique(y, return_inverse=True)
    m = KO.KernelSVCModel(X, S, yc, np.arange(len(y)), kernel=p["kernel"], gamma=p["gamma"], C=p["C"], degree=p["degree"],
                          coef0=p["coef0"], tol=p["tol"], shrinking=p["shrinking"])
    coef = np.zeros((len(m.pairs), len(y)))
    for q, (_, _, rows, c, _) in enumerate(m.pairs):
        coef[q, rows] = c
    return materialize_svc(clone(est), X, yc, classes, coef, np.array([pr[4] for pr in m.pairs]), np.array(m.n_iter), m.gamma)


@pytest.mark.parametrize("n_classes", [2, 3])
@pytest.mark.parametrize("shrinking", [True, False])
def test_oracle_equals_sklearn(n_classes, shrinking):
    X, y = _data(240, n_classes)
    S = KO.gram_ddot(X)
    for kern, dg, c0 in CASES:
        est = SVC(kernel=kern, degree=dg, coef0=c0, C=1.0, shrinking=shrinking)
        ref = clone(est).fit(X, y)
        got = _fit_oracle(X, S, y, est)
        msg = (kern, dg, c0, n_classes, shrinking)
        np.testing.assert_array_equal(got.n_iter_, ref.n_iter_, err_msg=str(msg))
        np.testing.assert_array_equal(got.support_, ref.support_, err_msg=str(msg))
        np.testing.assert_array_equal(got.dual_coef_, ref.dual_coef_, err_msg=str(msg))
        np.testing.assert_array_equal(got.intercept_, ref.intercept_, err_msg=str(msg))
        np.testing.assert_array_equal(got.predict(X), ref.predict(X), err_msg=str(msg))


def test_oracle_equals_sklearn_shrink_and_unshrink():
    """1200 rows: the 1000-iteration shrink cadence, shrunk variables and the unshrink / gradient reconstruction"""
    X, y = _data(1200, 2, seed=3, class_sep=0.5, flip_y=0.1)
    S = KO.gram_ddot(X)
    for kern, dg, c0, C in (("poly", 3, 1.0, 10.0), ("poly", 2, 0.0, 1.0), ("sigmoid", 3, -1.0, 1.0)):
        est = SVC(kernel=kern, degree=dg, coef0=c0, C=C, gamma=1.0 / 40)
        ref = clone(est).fit(X, y)
        got = _fit_oracle(X, S, y, est)
        assert kern != "poly" or C < 10 or ref.n_iter_[0] > 10000, ref.n_iter_     # many shrink rounds, then the unshrink
        np.testing.assert_array_equal(got.n_iter_, ref.n_iter_)
        np.testing.assert_array_equal(got.dual_coef_, ref.dual_coef_)
        np.testing.assert_array_equal(got.intercept_, ref.intercept_)
        np.testing.assert_array_equal(got.predict(X), ref.predict(X))


def test_oracle_reproduces_kernel_golden():
    """The oracle's poly and sigmoid fits of svc_kernels_mid (first two folds) have scikit-learn's split scores, iteration
    and support-vector counts (the golden's Gram is scikit-learn's, the oracle's a sequential-sum one: the kernel values
    agree after the float32 rounding)."""
    w = W.make_workload("svc_kernels_mid")
    g = golden("svc_kernels_mid")
    X, y = w["X"], w["y"]
    fold_id, ns = KO.folds_from_cv(w["cv"], X, y, True)
    S = KO.gram(X)
    rows = np.arange(len(y))
    for i, cand in enumerate(W.candidates(w)):
        if cand["kernel"] not in ("poly", "sigmoid"):
            continue
        p = dict(SVC().get_params(), **cand)
        for k in range(2):
            tr, te = rows[fold_id != k], rows[fold_id == k]
            m = KO.KernelSVCModel(X, S, y, tr, kernel=p["kernel"], gamma=p["gamma"], C=p["C"], degree=p["degree"],
                                  coef0=p["coef0"])
            assert sum(m.n_iter) == g["n_iter"][i, k], (cand, k)
            assert m.n_sv == g["n_sv"][i, k], (cand, k)
            assert np.mean(m.predict(te) == y[te]) == g["test_scores"][i, k], (cand, k)
            assert np.mean(m.predict(tr) == y[tr]) == g["train_scores"][i, k], (cand, k)
