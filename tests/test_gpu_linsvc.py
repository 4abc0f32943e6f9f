"""GPU tests of the LinearSVC path (csrc/linsvc.cu: liblinear's TRON in float64 on FP64 tensor-core contractions).

Checker: goldens made by scikit-learn 1.9 (tests/golden/make_linsvc_goldens.py) and scikit-learn's own searches.  Each fit
follows liblinear's iterate, so n_iter must equal scikit-learn's and the scores must be identical; the arithmetic differs
from liblinear's only in the order of float64 sums."""
import os
import pickle

import numpy as np
import pytest

from conftest import ROOT, golden
from spark_sklearn_b200 import workloads as W

pytestmark = pytest.mark.gpu


def _grid(est, grid, X, y, **kw):
    from spark_sklearn_b200 import GridSearchCV
    return GridSearchCV(None, est, grid, **kw).fit(X, y)


def _split_scores(search, ns, which="test"):
    return np.stack([search.cv_results_["split%d_%s_score" % (k, which)] for k in range(ns)], 1)


@pytest.mark.parametrize("key", ["linsvc_small", "linsvc_multi"])
@pytest.mark.parametrize("variant", ["none", "balanced", "dict", "sw"])
def test_linsvc_vs_golden(engine, key, variant):
    """class_weight None / 'balanced' / dict and sample weights with zeros, through the search's plan (which keeps n_iter)"""
    from sklearn.model_selection import StratifiedKFold
    from sklearn.svm import LinearSVC
    from spark_sklearn_b200 import estimators as E
    from golden.make_linsvc_goldens import VARIANTS, sample_weight
    w = W.make_workload(key)
    X, y = w["X"], w["y"]
    g = golden(key)
    cands = W.candidates(w)
    plan = E.LinearSVCPlan.plan(LinearSVC(**VARIANTS[variant]), cands, X, y,
                                   E.Folds(list(StratifiedKFold(w["cv"]).split(X, y)), len(X)), w["cv"])
    plan.set_scoring(None)
    plan.set_fit_params({"sample_weight": sample_weight(len(X))} if variant == "sw" else None)
    out = plan.evaluate(list(range(len(cands))))
    np.testing.assert_array_equal(plan.n_iter_, g["%s_n_iter" % variant])
    np.testing.assert_array_equal(out["test"], g["%s_test" % variant])
    np.testing.assert_array_equal(out["train"], g["%s_train" % variant])


def test_linsvc_engine_n_iter_vs_golden(engine):
    from oracle import oracle as O
    w = W.make_workload("linsvc_multi")
    fold_id, ns = O.folds_from_cv(w["cv"], w["X"], w["y"], True)
    engine.set_data(w["X"], fold_id, ns, y_class=w["y"].astype(np.int32))
    r = engine.linsvc([c["C"] for c in W.candidates(w)])
    g = golden("linsvc_multi")
    np.testing.assert_array_equal(r["n_iter"], g["none_n_iter"])
    np.testing.assert_array_equal(r["test"], g["none_test"])
    assert engine.profile()["tensor_flops"] > 0


@pytest.mark.skipif(not os.path.exists(os.path.join(ROOT, "tests", "golden", "linsvc_c3.npz")), reason="no linsvc_c3 golden")
def test_linsvc_c3_vs_golden(engine):
    """config 3 at full size: 1280 fits of 40000 x 256.  n_iter equal on at least 99% of the fits; mean_test_score within 1e-4."""
    from oracle import oracle as O
    w = W.make_workload("linsvc_c3")
    fold_id, ns = O.folds_from_cv(w["cv"], w["X"], w["y"], True)
    engine.set_data(w["X"], fold_id, ns, y_class=w["y"].astype(np.int32))
    g = golden("linsvc_c3")
    r = engine.linsvc([c["C"] for c in W.candidates(w)])
    assert np.mean(r["n_iter"] == g["none_n_iter"]) >= 0.99
    assert np.abs(r["test"].mean(1) - g["none_test"].mean(1)).max() <= 1e-4


@pytest.mark.parametrize("scoring", ["accuracy", "balanced_accuracy", "f1", "precision", "recall", "roc_auc", "f1_macro",
                                     "f1_micro", "f1_weighted"])
def test_linsvc_search_scorers_vs_sklearn(engine, scoring):
    from sklearn.model_selection import GridSearchCV as SkGrid
    from sklearn.svm import LinearSVC
    w = W.make_workload("linsvc_small")
    X, y = w["X"][:1500], w["y"][:1500]
    grid = {"C": [1e-3, 0.1, 10.0], "fit_intercept": [True, False]}
    a = _grid(LinearSVC(), grid, X, y, cv=4, scoring=scoring)
    b = SkGrid(LinearSVC(), grid, cv=4, scoring=scoring, return_train_score=True).fit(X, y)
    assert set(a.cv_results_) == set(b.cv_results_)
    # roc_auc: the device counts the pairs a decision value ranks correctly ((wins + ties / 2) / (n_neg n_pos)), scikit-learn
    # integrates the ROC curve by trapezoids: the same ranking rounds to values one ulp apart
    tol = 4 * np.finfo(np.float64).eps if scoring == "roc_auc" else 0.0
    for k in range(4):
        for which in ("test", "train"):
            key = "split%d_%s_score" % (k, which)
            np.testing.assert_allclose(a.cv_results_[key], b.cv_results_[key], rtol=tol, atol=0)


def test_linsvc_multiclass_scorers_and_intercept_scaling(engine):
    from sklearn.model_selection import GridSearchCV as SkGrid
    from sklearn.svm import LinearSVC
    w = W.make_workload("linsvc_multi")
    X, y = w["X"][:1200], w["y"][:1200]
    grid = {"C": [0.01, 1.0], "intercept_scaling": [0.5, 3.0]}
    for scoring in (None, "f1_macro", "balanced_accuracy"):
        a = _grid(LinearSVC(tol=1e-5), grid, X, y, cv=3, scoring=scoring)
        b = SkGrid(LinearSVC(tol=1e-5), grid, cv=3, scoring=scoring, return_train_score=True).fit(X, y)
        for k in range(3):
            np.testing.assert_array_equal(a.cv_results_["split%d_test_score" % k], b.cv_results_["split%d_test_score" % k])


@pytest.mark.parametrize("cv_kind", ["shuffle", "repeated"])
def test_linsvc_general_splitters(engine, cv_kind):
    from sklearn.model_selection import GridSearchCV as SkGrid, RepeatedStratifiedKFold, ShuffleSplit
    from sklearn.svm import LinearSVC
    w = W.make_workload("linsvc_small")
    X, y = w["X"][:1200], w["y"][:1200]
    cv = ShuffleSplit(4, test_size=0.3, random_state=0) if cv_kind == "shuffle" else RepeatedStratifiedKFold(n_splits=3, n_repeats=2, random_state=0)
    grid = {"C": [1e-3, 1.0]}
    a = _grid(LinearSVC(), grid, X, y, cv=cv)
    b = SkGrid(LinearSVC(), grid, cv=cv, return_train_score=True).fit(X, y)
    ns = cv.get_n_splits()
    np.testing.assert_array_equal(_split_scores(a, ns), _split_scores(b, ns))
    np.testing.assert_array_equal(_split_scores(a, ns, "train"), _split_scores(b, ns, "train"))


def test_linsvc_random_search_pipeline_refit_pickle(engine):
    from scipy.stats import loguniform
    from sklearn.model_selection import RandomizedSearchCV as SkRandom
    from sklearn.pipeline import Pipeline
    from sklearn.svm import LinearSVC
    from spark_sklearn_b200 import RandomizedSearchCV
    w = W.make_workload("linsvc_multi")
    X, y = w["X"], w["y"]
    pipe = Pipeline([("svc", LinearSVC())])
    dist = {"svc__C": loguniform(1e-3, 1e1)}
    a = RandomizedSearchCV(None, pipe, dist, n_iter=4, cv=3, random_state=0).fit(X, y)
    b = SkRandom(pipe, dist, n_iter=4, cv=3, random_state=0, return_train_score=True).fit(X, y)
    np.testing.assert_array_equal(_split_scores(a, 3), _split_scores(b, 3))
    assert a.best_params_ == b.best_params_
    ea, eb = a.best_estimator_.steps[0][1], b.best_estimator_.steps[0][1]
    assert ea.n_iter_ == eb.n_iter_
    np.testing.assert_array_equal(a.predict(X), b.predict(X))
    da, db = a.decision_function(X), b.decision_function(X)
    assert np.abs(da - db).max() <= 1e-10 * np.abs(db).max()
    c = pickle.loads(pickle.dumps(a.best_estimator_))
    np.testing.assert_array_equal(c.predict(X), b.predict(X))


def test_linsvc_refit_binary_vs_golden(engine):
    from sklearn.svm import LinearSVC
    w = W.make_workload("linsvc_small")
    g = golden("linsvc_small")
    s = _grid(LinearSVC(), {"C": [float(g["refit_C"])]}, w["X"], w["y"], cv=5)
    e = s.best_estimator_
    assert e.n_iter_ == int(g["refit_n_iter"])
    ref = np.abs(g["refit_coef"]).max()
    assert np.abs(e.coef_ - g["refit_coef"]).max() <= 1e-10 * ref
    assert np.abs(e.intercept_ - g["refit_intercept"]).max() <= 1e-10 * ref


def test_linsvc_max_iter_stop_warns(engine):
    from sklearn.exceptions import ConvergenceWarning
    from sklearn.svm import LinearSVC
    w = W.make_workload("linsvc_small")
    X, y = w["X"][:800], w["y"][:800]
    with pytest.warns(ConvergenceWarning):
        s = _grid(LinearSVC(max_iter=1, tol=1e-12), {"C": [1.0]}, X, y, cv=3)
    ref = LinearSVC(max_iter=1, tol=1e-12)
    with pytest.warns(ConvergenceWarning):
        ref.fit(X, y)
    assert s.best_estimator_.n_iter_ == ref.n_iter_ == 1
    np.testing.assert_array_equal(s.predict(X), ref.predict(X))


def test_linsvc_one_gpu_and_all_gpus_agree(engine, monkeypatch):
    from sklearn.svm import LinearSVC
    w = W.make_workload("linsvc_small")
    grid = {"C": list(np.logspace(-3, 1, 6))}
    monkeypatch.setenv("B200GS_DEVICES", "1")
    a = _grid(LinearSVC(), grid, w["X"], w["y"], cv=5)
    monkeypatch.setenv("B200GS_DEVICES", "all")
    b = _grid(LinearSVC(), grid, w["X"], w["y"], cv=5)
    for k in a.cv_results_:
        if "time" not in k:
            np.testing.assert_array_equal(np.asarray(a.cv_results_[k], object), np.asarray(b.cv_results_[k], object))
