"""GPU parity tests for the nu-SVC and nu-SVR paths against scikit-learn itself (sklearn.svm.NuSVC / NuSVR, libsvm's
Solver_NU).

The CUDA solver follows libsvm's iterate sequence, so the bar is: n_iter equal per fit, NuSVC split scores identical, NuSVR
split scores within the rounding of the float64 decision-value sums (1e-12), and the refit model equal to a real fit."""
import pickle
import warnings

import numpy as np
import pytest
from sklearn.datasets import make_classification, make_regression
from sklearn.model_selection import (GridSearchCV as SkGridSearchCV, KFold, ParameterGrid, RepeatedStratifiedKFold,
                                     ShuffleSplit, StratifiedKFold)
from sklearn.pipeline import Pipeline
from sklearn.svm import NuSVC, NuSVR

from spark_sklearn_b200 import GridSearchCV

pytestmark = pytest.mark.gpu


def _clf(n_classes, n=300, seed=0):
    X, y = make_classification(n_samples=n, n_features=8, n_informative=5, n_redundant=1, n_classes=n_classes,
                               random_state=seed)
    return X, y


def _reg(n=300, seed=0):
    X, y = make_regression(n_samples=n, n_features=8, n_informative=6, noise=5.0, random_state=seed)
    return X, y / np.std(y)


def _splits_scores(search, n_splits, kind="test"):
    return np.stack([search.cv_results_["split%d_%s_score" % (k, kind)] for k in range(n_splits)], 1)


def _n_iter_nusvc(X, y, cands, splits, base):
    """scikit-learn's n_iter_ summed over the one-vs-one pairs, per (candidate, split)"""
    it = np.zeros((len(cands), len(splits)), np.int64)
    for i, c in enumerate(cands):
        for k, (a, _) in enumerate(splits):
            it[i, k] = np.sum(NuSVC(**dict(base, **c)).fit(X[a], y[a]).n_iter_)
    return it


def _plan_n_iter(adapter, est, cands, X, y, splits):
    from spark_sklearn_b200.estimators import Folds
    plan = adapter.plan(est, cands, X, y, Folds(splits, len(X)), len(splits))
    plan.evaluate(list(range(len(cands))), return_train=False)
    return plan.n_iter_


@pytest.mark.parametrize("n_classes", [2, 3])
@pytest.mark.parametrize("kernel", ["rbf", "linear", "poly", "sigmoid"])
def test_nusvc_matches_sklearn(engine, n_classes, kernel):
    """Split scores identical to scikit-learn's GridSearchCV and n_iter equal per fit, for every kernel."""
    from spark_sklearn_b200.estimators import NuSVCPlan
    X, y = _clf(n_classes)
    grid = {"nu": [0.1, 0.3, 0.5], "gamma": ["scale", 0.05]}
    base = {"kernel": kernel}
    if kernel == "sigmoid":
        base["coef0"] = 0.5
    ours = GridSearchCV(None, NuSVC(**base), grid, cv=5, return_train_score=True).fit(X, y)
    ref = SkGridSearchCV(NuSVC(**base), grid, cv=5, return_train_score=True).fit(X, y)
    for kind in ("test", "train"):
        np.testing.assert_array_equal(_splits_scores(ours, 5, kind), _splits_scores(ref, 5, kind), err_msg=kind)
    assert ours.best_params_ == ref.best_params_
    cands = list(ParameterGrid(grid))
    splits = list(StratifiedKFold(5).split(X, y))
    got, want = _plan_n_iter(NuSVCPlan, NuSVC(**base), cands, X, y, splits), _n_iter_nusvc(X, y, cands, splits, base)
    if kernel in ("rbf", "sigmoid"):
        # exp / tanh: the device's float64 kernel value can differ from the host libm's in the last bit, which can move a
        # trajectory by an iteration without changing a score.  Measured on one H100: one fit of the 60 (sigmoid, 3
        # classes: 223 against 224 iterations summed over the pairs).
        diff = got != want
        assert diff.sum() <= 1 and np.abs(got - want).max() <= 1, (got, want)
    else:
        np.testing.assert_array_equal(got, want)


def test_nusvc_variants_match_sklearn(engine):
    """shrinking off, a max_iter stop, a larger problem that shrinks and unshrinks, and a class_weight (no effect on nu-SVC)"""
    from spark_sklearn_b200.estimators import NuSVCPlan
    X, y = _clf(3, n=1200, seed=1)
    splits = list(StratifiedKFold(3).split(X, y))
    for base, grid in [({"shrinking": False}, {"nu": [0.2, 0.4]}),
                       ({"max_iter": 200}, {"nu": [0.3]}),
                       ({}, {"nu": [0.05, 0.5], "gamma": [0.02, 0.5]}),
                       ({"class_weight": {0: 2.0}}, {"nu": [0.3]})]:
        ours = GridSearchCV(None, NuSVC(**base), grid, cv=3).fit(X, y)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ref = SkGridSearchCV(NuSVC(**base), grid, cv=3).fit(X, y)
        np.testing.assert_array_equal(_splits_scores(ours, 3), _splits_scores(ref, 3), err_msg=str(base))
        cands = list(ParameterGrid(grid))
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            np.testing.assert_array_equal(_plan_n_iter(NuSVCPlan, NuSVC(**base), cands, X, y, splits),
                                          _n_iter_nusvc(X, y, cands, splits, base), err_msg=str(base))


@pytest.mark.parametrize("scoring", ["f1_macro", "balanced_accuracy", "roc_auc", "f1"])
def test_nusvc_scorers(engine, scoring):
    X, y = _clf(2)
    grid = {"nu": [0.2, 0.5], "gamma": ["scale"]}
    ours = GridSearchCV(None, NuSVC(), grid, cv=5, scoring=scoring).fit(X, y)
    ref = SkGridSearchCV(NuSVC(), grid, cv=5, scoring=scoring).fit(X, y)
    np.testing.assert_allclose(_splits_scores(ours, 5), _splits_scores(ref, 5), rtol=0, atol=1e-15)


@pytest.mark.parametrize("cv", [ShuffleSplit(4, test_size=0.25, random_state=0),
                                RepeatedStratifiedKFold(n_splits=3, n_repeats=2, random_state=0)])
def test_nusvc_general_splitters(engine, cv):
    X, y = _clf(3)
    grid = {"nu": [0.2, 0.4]}
    ours = GridSearchCV(None, NuSVC(), grid, cv=cv).fit(X, y)
    ref = SkGridSearchCV(NuSVC(), grid, cv=cv).fit(X, y)
    ns = cv.get_n_splits(X, y)
    np.testing.assert_array_equal(_splits_scores(ours, ns), _splits_scores(ref, ns))


def test_nusvc_infeasible_nu_takes_error_score(engine):
    """nu = 0.9 is infeasible for a 70/30 training set: those tasks score error_score, as in scikit-learn"""
    X, y = make_classification(n_samples=300, n_features=8, weights=[0.7, 0.3], random_state=0)
    grid = {"nu": [0.3, 0.9]}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ours = GridSearchCV(None, NuSVC(), grid, cv=5, error_score=np.nan, refit=False).fit(X, y)
        ref = SkGridSearchCV(NuSVC(), grid, cv=5, error_score=np.nan, refit=False).fit(X, y)
    a, b = _splits_scores(ours, 5), _splits_scores(ref, 5)
    assert np.isnan(b[1]).all()
    np.testing.assert_array_equal(a, b)
    with pytest.raises(ValueError, match="specified nu is infeasible"):
        GridSearchCV(None, NuSVC(), grid, cv=5).fit(X, y)


@pytest.mark.parametrize("n_classes", [2, 3])
def test_nusvc_refit_equals_real_fit(engine, n_classes):
    X, y = _clf(n_classes)
    grid = {"nu": [0.2, 0.4], "gamma": ["scale"]}
    best = GridSearchCV(None, NuSVC(), grid, cv=5).fit(X, y).best_estimator_
    assert type(best) is NuSVC
    real = NuSVC(**best.get_params()).fit(X, y)
    np.testing.assert_array_equal(best.support_, real.support_)
    np.testing.assert_array_equal(best.dual_coef_, real.dual_coef_)
    np.testing.assert_array_equal(best.intercept_, real.intercept_)
    np.testing.assert_array_equal(best.n_iter_, real.n_iter_)
    np.testing.assert_array_equal(best.predict(X), real.predict(X))
    np.testing.assert_array_equal(best.decision_function(X), real.decision_function(X))
    again = pickle.loads(pickle.dumps(best))
    np.testing.assert_array_equal(again.decision_function(X), real.decision_function(X))


def test_nusvc_one_step_pipeline(engine):
    X, y = _clf(3)
    grid = {"clf__nu": [0.2, 0.4], "clf__gamma": ["scale", 0.1]}
    ours = GridSearchCV(None, Pipeline([("clf", NuSVC())]), grid, cv=5).fit(X, y)
    ref = SkGridSearchCV(Pipeline([("clf", NuSVC())]), grid, cv=5).fit(X, y)
    np.testing.assert_array_equal(_splits_scores(ours, 5), _splits_scores(ref, 5))
    np.testing.assert_array_equal(ours.best_estimator_.predict(X), ref.best_estimator_.predict(X))


@pytest.mark.parametrize("kernel", ["rbf", "linear"])
def test_nusvr_matches_sklearn(engine, kernel):
    """Split scores within 1e-12 and n_iter equal per fit; the refit equals a real fit"""
    from spark_sklearn_b200.estimators import NuSVRPlan
    X, y = _reg()
    grid = {"nu": [0.1, 0.5, 0.9], "C": [1.0, 10.0]}
    ours = GridSearchCV(None, NuSVR(kernel=kernel), grid, cv=5, return_train_score=True).fit(X, y)
    ref = SkGridSearchCV(NuSVR(kernel=kernel), grid, cv=5, return_train_score=True).fit(X, y)
    for kind in ("test", "train"):
        np.testing.assert_allclose(_splits_scores(ours, 5, kind), _splits_scores(ref, 5, kind), rtol=0, atol=1e-12)
    cands = list(ParameterGrid(grid))
    splits = list(KFold(5).split(X))
    sit = np.array([[NuSVR(kernel=kernel, **c).fit(X[a], y[a]).n_iter_ for a, _ in splits] for c in cands])
    np.testing.assert_array_equal(_plan_n_iter(NuSVRPlan, NuSVR(kernel=kernel), cands, X, y, splits), sit)
    best = ours.best_estimator_
    assert type(best) is NuSVR
    real = NuSVR(**best.get_params()).fit(X, y)
    np.testing.assert_array_equal(best.support_, real.support_)
    np.testing.assert_allclose(best.dual_coef_, real.dual_coef_, rtol=0, atol=0)
    np.testing.assert_array_equal(best.intercept_, real.intercept_)
    np.testing.assert_allclose(best.predict(X), real.predict(X), rtol=0, atol=1e-12)
    assert pickle.loads(pickle.dumps(best)).n_iter_ == real.n_iter_


def test_nusvr_variants_and_pipeline(engine):
    """shrinking off, a max_iter stop, a larger fit that shrinks, and the one-step Pipeline"""
    X, y = _reg(n=1500, seed=2)
    for base, grid in [({"shrinking": False}, {"nu": [0.3]}),
                       ({"max_iter": 300}, {"nu": [0.5]}),
                       ({}, {"nu": [0.2, 0.6], "gamma": [0.02, "scale"]})]:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ours = GridSearchCV(None, NuSVR(**base), grid, cv=3).fit(X, y)
            ref = SkGridSearchCV(NuSVR(**base), grid, cv=3).fit(X, y)
        np.testing.assert_allclose(_splits_scores(ours, 3), _splits_scores(ref, 3), rtol=0, atol=1e-12, err_msg=str(base))
    X, y = _reg()
    grid = {"m__nu": [0.3, 0.6]}
    ours = GridSearchCV(None, Pipeline([("m", NuSVR())]), grid, cv=5, scoring="neg_mean_squared_error").fit(X, y)
    ref = SkGridSearchCV(Pipeline([("m", NuSVR())]), grid, cv=5, scoring="neg_mean_squared_error").fit(X, y)
    np.testing.assert_allclose(_splits_scores(ours, 5), _splits_scores(ref, 5), rtol=1e-12, atol=0)


@pytest.mark.parametrize("key", ["nusvc_mid", "nusvr_mid"])
def test_nu_goldens(engine, key):
    """The mid-size goldens from scikit-learn (tests/golden/make_nu_goldens.py): gamma 'scale', poly / sigmoid NuSVC
    candidates and an infeasible nu under error_score=np.nan; n_iter per fit (-1: infeasible) equal"""
    from conftest import golden
    from spark_sklearn_b200 import workloads as W
    from spark_sklearn_b200.estimators import Folds, adapter_for
    g = golden(key)
    w = W.make_workload(key)
    X, y, cv = w["X"], w["y"], w["cv"]
    est = W.make_estimator(w)
    splits = list((KFold(cv) if key == "nusvr_mid" else StratifiedKFold(cv)).split(X, y))
    cands = list(ParameterGrid(w["param_grid"]))
    plan = adapter_for(est).plan(est, cands, X, y, Folds(splits, len(X)), cv)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        r = plan.evaluate(list(range(len(cands))), return_train=True, error_score=np.nan)
    np.testing.assert_array_equal(plan.n_iter_, g["n_iter"])
    if key == "nusvc_mid":
        np.testing.assert_array_equal(r["test"], g["test_scores"])
        np.testing.assert_array_equal(r["train"], g["train_scores"])
    else:
        np.testing.assert_allclose(r["test"], g["test_scores"], rtol=0, atol=1e-12)
        np.testing.assert_allclose(r["train"], g["train_scores"], rtol=0, atol=1e-12)


def test_in_process_multi_gpu_equals_single_gpu_nu(monkeypatch):
    """One GPU against all GPUs of the in-process scheduler: identical cv_results_ scores; skipped on a one-GPU box"""
    from spark_sklearn_b200.engine import device_count
    if device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    X, y = _clf(3)
    grid = {"nu": [0.1, 0.2, 0.3, 0.4, 0.5, 0.6], "gamma": ["scale", 0.05]}
    monkeypatch.setenv("B200GS_DEVICES", "1")
    one = GridSearchCV(None, NuSVC(), grid, cv=5, refit=False).fit(X, y)
    monkeypatch.setenv("B200GS_DEVICES", "all")
    many = GridSearchCV(None, NuSVC(), grid, cv=5, refit=False).fit(X, y)
    assert len(many.devices_) > 1
    for k in one.cv_results_:
        if k.endswith("_score"):
            np.testing.assert_array_equal(np.asarray(one.cv_results_[k], float), np.asarray(many.cv_results_[k], float), err_msg=k)


def test_max_iter_stop_after_the_first_shrink(engine):
    """max_iter stops after the first shrink (a pair or fit of l variables shrinks first at iteration min(l, 1000)): split
    scores and the refit's intercept_, dual_coef_ and n_iter_ equal scikit-learn's, NuSVC and NuSVR"""
    X, y = make_classification(n_samples=600, n_features=8, n_informative=5, random_state=1)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ours = GridSearchCV(None, NuSVC(gamma=0.5, max_iter=700), {"nu": [0.2]}, cv=3).fit(X, y)    # 400-row pairs
        ref = SkGridSearchCV(NuSVC(gamma=0.5, max_iter=700), {"nu": [0.2]}, cv=3).fit(X, y)
        real = NuSVC(gamma=0.5, max_iter=700, nu=0.2).fit(X, y)                                       # 600-row pair
    np.testing.assert_array_equal(_splits_scores(ours, 3), _splits_scores(ref, 3))
    best = ours.best_estimator_
    assert best.n_iter_[0] == real.n_iter_[0] == 700
    np.testing.assert_array_equal(best.intercept_, real.intercept_)
    np.testing.assert_array_equal(best.dual_coef_, real.dual_coef_)
    np.testing.assert_array_equal(best.support_, real.support_)

    X, y = _reg(300)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ours = GridSearchCV(None, NuSVR(C=10.0, max_iter=700), {"nu": [0.4]}, cv=3).fit(X, y)    # 400 variables per fit
        ref = SkGridSearchCV(NuSVR(C=10.0, max_iter=700), {"nu": [0.4]}, cv=3).fit(X, y)
        real = NuSVR(C=10.0, max_iter=700, nu=0.4).fit(X, y)                                      # 600 variables
    np.testing.assert_allclose(_splits_scores(ours, 3), _splits_scores(ref, 3), rtol=0, atol=1e-12)
    best = ours.best_estimator_
    assert best.n_iter_ == real.n_iter_ == 700
    np.testing.assert_array_equal(best.intercept_, real.intercept_)
    np.testing.assert_array_equal(best.dual_coef_, real.dual_coef_)
    np.testing.assert_array_equal(best.support_, real.support_)


def test_nusvr_wide_tier(engine):
    """fits of 4800 training rows (9600 variables: the 1024-thread, 16-positions-per-thread instance) within 1e-12"""
    from sklearn.model_selection import KFold
    X, y = make_regression(n_samples=6000, n_features=16, noise=5.0, random_state=3)
    y = y / np.std(y)
    ours = GridSearchCV(None, NuSVR(C=1.0, gamma=0.05), {"nu": [0.3]}, cv=5, refit=False).fit(X, y)
    splits = list(KFold(5).split(X))
    ref = np.array([[NuSVR(C=1.0, gamma=0.05, nu=0.3).fit(X[a], y[a]).score(X[b], y[b]) for a, b in splits[:2]]])
    np.testing.assert_allclose(_splits_scores(ours, 5)[:, :2], ref, rtol=0, atol=1e-12)
