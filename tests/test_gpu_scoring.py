"""GPU parity tests for `scoring=` (reference grid_search.py:212-214, base_search.py:43,83-87): every fused CUDA scorer
against scikit-learn's GridSearchCV with the same scorer on the same folds.  Count-based scorers are exact rational
functions of integer counts (bit-equal up to the last float64 ulp of a different evaluation order); roc_auc is the
Mann-Whitney statistic of the decision values (SVC: float64, identical ranking; LogisticRegression: float32 z)."""
import warnings

import numpy as np
import pytest

from spark_sklearn_b200 import workloads as W

pytestmark = pytest.mark.gpu


def _both(est, grid, X, y, scoring, cv=5):
    from sklearn.model_selection import GridSearchCV as SkGrid
    from spark_sklearn_b200 import GridSearchCV
    a = GridSearchCV(None, est, grid, cv=cv, scoring=scoring, refit=False).fit(X, y)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        b = SkGrid(est, grid, cv=cv, scoring=scoring, return_train_score=True, refit=False).fit(X, y)
    return a.cv_results_, b.cv_results_


@pytest.mark.parametrize("scoring", ["accuracy", "balanced_accuracy", "f1", "precision", "recall", "roc_auc", "f1_macro", "f1_weighted", "f1_micro"])
def test_svc_binary_scorers(engine, scoring):
    from sklearn.svm import SVC
    w = W.make_workload("c2_small")
    grid = {"C": [0.1, 10.0], "gamma": [1 / 512, 1 / 64]}
    a, b = _both(SVC(kernel="rbf"), grid, w["X"], w["y"], scoring)
    for k in range(5):
        for part in ("test", "train"):
            key = "split%d_%s_score" % (k, part)
            np.testing.assert_allclose(a[key], b[key], rtol=0, atol=1e-12, err_msg="%s %s" % (scoring, key))
    np.testing.assert_array_equal(a["rank_test_score"], b["rank_test_score"])


@pytest.mark.parametrize("scoring", ["balanced_accuracy", "f1_macro", "f1_weighted"])
def test_svc_multiclass_scorers_iris(engine, scoring):
    from sklearn import svm
    w = W.make_workload("c1")
    a, b = _both(svm.SVC(gamma="auto"), {"kernel": ("linear", "rbf"), "C": [1, 10]}, w["X"], w["y"], scoring)
    np.testing.assert_allclose(a["mean_test_score"], b["mean_test_score"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(a["mean_train_score"], b["mean_train_score"], rtol=0, atol=1e-12)


def test_binary_only_scorers_raise_on_multiclass(engine):
    from sklearn import svm
    from spark_sklearn_b200 import GridSearchCV
    w = W.make_workload("c1")
    for scoring in ("f1", "roc_auc"):
        with pytest.raises((ValueError, NotImplementedError)):
            GridSearchCV(None, svm.SVC(gamma="auto"), {"C": [1, 10]}, cv=3, scoring=scoring).fit(w["X"], w["y"])


@pytest.mark.parametrize("scoring", ["f1", "roc_auc", "balanced_accuracy"])
def test_logreg_scorers(engine, scoring):
    from sklearn.linear_model import LogisticRegression
    w = W.make_workload("c3_small")
    a, b = _both(LogisticRegression(), {"C": [1e-3, 1e-1, 50.0]}, w["X"], w["y"], scoring)
    # <= 2 borderline rows of 4000 flip (test_gpu_logreg.py); AUC moves by a few pairs in 4e5
    assert np.abs(a["mean_test_score"] - b["mean_test_score"]).max() <= 1e-3
    assert np.abs(a["mean_train_score"] - b["mean_train_score"]).max() <= 1e-3


@pytest.mark.parametrize("scoring", ["r2", "neg_mean_squared_error", "neg_root_mean_squared_error"])
def test_ridge_scorers(engine, scoring):
    from sklearn.linear_model import Ridge
    w = W.make_workload("c5_small")
    a, b = _both(Ridge(), {"alpha": np.logspace(-2, 3, 6)}, w["X"], w["y"], scoring)
    if scoring == "r2":
        assert np.abs(a["mean_test_score"] - b["mean_test_score"]).max() <= 1e-5
        assert np.abs(a["mean_train_score"] - b["mean_train_score"]).max() <= 1e-5
    else:
        # The residual sum of squares comes from the (mean-shifted) Gram statistics, res = yy - 2 w.Xy + w'Gw ..., in fp32-faithful
        # tensor-core arithmetic: its error is ~1e-6 of the TOTAL sum of squares, i.e. 1e-6 / (1 - R^2) relative -- 3e-3 here, where
        # the best candidates reach R^2 = 0.9997.  (R^2 itself carries the 1e-6.)
        rel = np.abs(a["mean_test_score"] - b["mean_test_score"]) / np.abs(b["mean_test_score"])
        assert rel.max() <= 3e-3, rel
        rel = np.abs(a["mean_train_score"] - b["mean_train_score"]) / np.abs(b["mean_train_score"])
        assert rel.max() <= 3e-3, rel
    assert a["rank_test_score"][np.argmin(b["rank_test_score"])] == 1 or np.ptp(b["mean_test_score"][a["rank_test_score"] <= 2]) < 1e-2 * np.abs(b["mean_test_score"]).min()


_SEARCHES = {
    "svc": lambda e: e.svc(["rbf"], [1.0], [0.1]),
    "nusvc": lambda e: e.svc(["rbf"], [0.5], [0.1], nu=True),
    "logreg": lambda e: e.logreg([1.0]),
    "linsvc": lambda e: e.linsvc([1.0]),
    "sgd": lambda e: e.sgd(["hinge"], ["l2"], 1e-4, 0.15, 0.1, ["optimal"], 0.0, 0.5, np.ones((1, 3))),
    "logreg_sag": lambda e: e.logreg_sag([["sag"] * 3], 1e-3, 0.0, 0.1, [[1, 2, 3]], "log"),
    "knn": lambda e: e.knn([3], ["uniform"], ["euclidean"]),
}


@pytest.mark.parametrize("search", sorted(_SEARCHES))
def test_positive_class_out_of_range_is_rejected(engine, search):
    """A positive class the dataset does not have (f1 with class 5 of two) is rejected before any device work"""
    from spark_sklearn_b200.engine import EngineError
    rng = np.random.RandomState(0)
    X = rng.standard_normal((60, 4))
    y = (X[:, 0] > 0).astype(np.int32)
    engine.set_data(X, (np.arange(60) % 3).astype(np.int8), 3, y_class=y)
    try:
        engine.set_scoring(2, 5)
        before = engine.profile()
        with pytest.raises(EngineError) as e:
            _SEARCHES[search](engine)
        assert e.value.status == -2, str(e.value)
        assert "positive class out of range" in str(e.value)
        assert engine.profile() == before                  # the search returned before it reset its profile
    finally:
        engine.set_scoring(0, 1)
