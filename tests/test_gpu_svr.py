"""GPU parity tests for the epsilon-SVR path against scikit-learn itself (sklearn.svm.SVR, libsvm).

The CUDA solver follows libsvm's iterate sequence, so the bar is: n_iter equal per fit, split scores equal to the
rounding of the float64 decision-value sums (1e-12), best_params_ equal, and the refit model equal attribute for
attribute."""
import pickle

import numpy as np
import pytest
from sklearn.model_selection import GridSearchCV as SkGridSearchCV, KFold, ParameterGrid
from sklearn.exceptions import ConvergenceWarning
from sklearn.svm import SVR

from spark_sklearn_b200 import GridSearchCV, workloads as W

pytestmark = pytest.mark.gpu


def _sk_fits(X, y, cands, cv, base=None, scoring=None):
    """n_iter, test score, train score of SVR(**base, **cand).fit(X[train]) per (candidate, split)"""
    from sklearn.metrics import get_scorer
    sc = get_scorer(scoring) if scoring else None
    splits = list(KFold(cv).split(X))
    it = np.zeros((len(cands), cv), np.int64)
    te = np.zeros((len(cands), cv))
    tr = np.zeros((len(cands), cv))
    for i, c in enumerate(cands):
        for k, (a, b) in enumerate(splits):
            m = SVR(**dict(base or {}, **c)).fit(X[a], y[a])
            it[i, k] = m.n_iter_
            te[i, k] = sc(m, X[b], y[b]) if sc else m.score(X[b], y[b])
            tr[i, k] = sc(m, X[a], y[a]) if sc else m.score(X[a], y[a])
    return it, te, tr


def _engine_run(engine, X, y, cands, cv, base=None):
    """the engine directly (n_iter per fit is not part of cv_results_)"""
    from spark_sklearn_b200.estimators import Folds, SVRPlan
    splits = list(KFold(cv).split(X))
    plan = SVRPlan.plan(SVR(**(base or {})), cands, X, y, Folds(splits, len(X)), cv)
    r = plan.evaluate(list(range(len(cands))), return_train=True)
    return plan.n_iter_, r["test"], r["train"]


def _check(engine, X, y, cands, cv=5, base=None):
    it, te, tr = _engine_run(engine, X, y, cands, cv, base)
    sit, ste, str_ = _sk_fits(X, y, cands, cv, base)
    np.testing.assert_array_equal(it, sit)
    np.testing.assert_allclose(te, ste, rtol=0, atol=1e-12)
    np.testing.assert_allclose(tr, str_, rtol=0, atol=1e-12)


def test_svr_small_grid_matches_sklearn(engine):
    """The whole svr_small grid (24 candidates x 5 folds, rbf, gamma numeric and 'scale') through the public search."""
    w = W.make_workload("svr_small")
    X, y, grid = w["X"], w["y"], w["param_grid"]
    ours = GridSearchCV(None, SVR(), grid, cv=5, return_train_score=True).fit(X, y)
    ref = SkGridSearchCV(SVR(), grid, cv=5, return_train_score=True).fit(X, y)
    for k in range(5):
        for kind in ("test", "train"):
            key = "split%d_%s_score" % (k, kind)
            np.testing.assert_allclose(ours.cv_results_[key], ref.cv_results_[key], rtol=0, atol=1e-12, err_msg=key)
    assert ours.best_params_ == ref.best_params_
    it, _, _ = _engine_run(engine, X, y, list(ParameterGrid(grid)), 5)
    sit, _, _ = _sk_fits(X, y, list(ParameterGrid(grid)), 5)
    np.testing.assert_array_equal(it, sit)


def test_svr_variants_match_sklearn(engine):
    """linear kernel, gamma 'auto' / 'scale', shrinking off, a max_iter stop, epsilon 0"""
    w = W.make_workload("svr_small")
    X, y = w["X"][:600], w["y"][:600]
    _check(engine, X, y, [{"C": 0.5, "epsilon": 0.1}, {"C": 5.0, "epsilon": 0.0}], base={"kernel": "linear"})
    _check(engine, X, y, [{"C": 3.0, "gamma": "auto"}, {"C": 3.0, "gamma": "scale", "epsilon": 0.0}])
    _check(engine, X, y, [{"C": 10.0, "gamma": 1 / 32}], base={"shrinking": False})
    _check(engine, X, y, [{"C": 100.0, "gamma": 1 / 32}], base={"max_iter": 150})


@pytest.mark.parametrize("scoring", ["neg_mean_squared_error", "neg_root_mean_squared_error"])
def test_svr_regression_scorers(engine, scoring):
    w = W.make_workload("svr_small")
    X, y = w["X"][:500], w["y"][:500]
    grid = {"C": [1.0, 10.0], "gamma": [1 / 32, "scale"]}
    ours = GridSearchCV(None, SVR(), grid, cv=5, scoring=scoring, return_train_score=True).fit(X, y)
    ref = SkGridSearchCV(SVR(), grid, cv=5, scoring=scoring, return_train_score=True).fit(X, y)
    for k in range(5):
        for kind in ("test", "train"):
            key = "split%d_%s_score" % (k, kind)
            np.testing.assert_allclose(ours.cv_results_[key], ref.cv_results_[key], rtol=0, atol=1e-12, err_msg=key)
    assert ours.best_params_ == ref.best_params_


def test_svr_refit_matches_sklearn(engine):
    w = W.make_workload("svr_small")
    X, y = w["X"], w["y"]
    grid = {"C": [1.0, 10.0], "gamma": [1 / 32, "scale"], "epsilon": [0.1]}
    s = GridSearchCV(None, SVR(), grid, cv=5).fit(X, y)
    got = s.best_estimator_
    ref = SVR(**s.best_params_).fit(X, y)
    np.testing.assert_array_equal(got.support_, ref.support_)
    np.testing.assert_array_equal(got.dual_coef_, ref.dual_coef_)
    np.testing.assert_array_equal(got.intercept_, ref.intercept_)
    assert got.n_iter_ == ref.n_iter_
    np.testing.assert_allclose(s.predict(X), ref.predict(X), rtol=0, atol=1e-12)
    back = pickle.loads(pickle.dumps(got))
    np.testing.assert_array_equal(back.predict(X), got.predict(X))


def test_svr_pipeline_one_step(engine):
    from sklearn.pipeline import Pipeline
    w = W.make_workload("svr_small")
    X, y = w["X"][:400], w["y"][:400]
    grid = {"svr__C": [1.0, 10.0]}
    ours = GridSearchCV(None, Pipeline([("svr", SVR())]), grid, cv=5).fit(X, y)
    ref = SkGridSearchCV(Pipeline([("svr", SVR())]), grid, cv=5).fit(X, y)
    np.testing.assert_allclose(ours.cv_results_["mean_test_score"], ref.cv_results_["mean_test_score"], rtol=0, atol=1e-12)


def test_svr_max_iter_after_shrinking(engine):
    """a max_iter stop after the first shrink (1600 variables: shrinking starts at iteration 1000): the intercept is taken
    over all variables after the gradient of the shrunk ones is rebuilt, as libsvm does"""
    w = W.make_workload("svr_small")
    X, y = w["X"], w["y"]
    _check(engine, X, y, [{"C": 100.0, "gamma": 1 / 32, "epsilon": 0.05}], base={"max_iter": 1500})   # ~1850 to converge
    from spark_sklearn_b200.estimators import Folds, SVRPlan
    plan = SVRPlan.plan(SVR(max_iter=1500), [{}], X, y, Folds(list(KFold(5).split(X)), len(X)), 5)   # 2428 to converge
    with pytest.warns(ConvergenceWarning):
        got = plan.refit({"C": 100.0, "gamma": 1 / 32, "epsilon": 0.05})
    with pytest.warns(ConvergenceWarning):
        ref = SVR(C=100.0, gamma=1 / 32, epsilon=0.05, max_iter=1500).fit(X, y)
    assert got.n_iter_ == ref.n_iter_ == 1500 and got.fit_status_ == ref.fit_status_ == 1
    np.testing.assert_array_equal(got.intercept_, ref.intercept_)
    np.testing.assert_array_equal(got.dual_coef_, ref.dual_coef_)


def test_svr_mid_golden(engine):
    """the whole svr_mid grid (4000-row fits: 8000 variables, the bulk-row-copy instance) against its golden"""
    from conftest import golden
    w = W.make_workload("svr_mid")
    g = golden("svr_mid")
    it, te, tr = _engine_run(engine, w["X"], w["y"], list(ParameterGrid(w["param_grid"])), 5, w["est_params"])
    np.testing.assert_array_equal(it, g["n_iter"])
    np.testing.assert_allclose(te, g["test_scores"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(tr, g["train_scores"], rtol=0, atol=1e-12)


def test_svr_mid_rowbuf_tier(engine):
    """4000-row fits (8000 solver variables: the bulk-row-copy instance)"""
    w = W.make_workload("svr_mid")
    _check(engine, w["X"], w["y"], [{"C": 3.0, "gamma": 1 / 128, "epsilon": 0.1}, {"C": 0.3, "gamma": "scale", "epsilon": 0.1}])


def test_svr_largest_tier_and_row_limit(engine):
    """8000-row fits (16000 variables, the 1024 x 16 instance) match scikit-learn; more than 8192 rows raise"""
    w = W._svr(n=12000, d=32, name="svr_12k")
    _check(engine, w["X"], w["y"], [{"C": 1.0, "gamma": 1 / 32, "epsilon": 0.2}, {"C": 0.1, "gamma": "scale", "epsilon": 0.2}],
           cv=3)
    big = W._svr(n=12300, d=32, name="svr_12k3")                   # 8200 training rows per fit
    with pytest.raises(NotImplementedError):
        GridSearchCV(None, SVR(), {"C": [1.0]}, cv=3).fit(big["X"], big["y"])


def test_svr_general_splitters(engine):
    """ShuffleSplit / RepeatedKFold / PredefinedSplit through split masks: each fit sees its training rows in ascending
    order, scikit-learn in the splitter's order.  test_oracle_svr.py measures what that order costs (ORDER_BOUND)."""
    from test_oracle_svr import ORDER_BOUND
    from sklearn.model_selection import PredefinedSplit, RepeatedKFold, ShuffleSplit
    w = W.make_workload("svr_small")
    X, y = w["X"][:600], w["y"][:600]
    grid = {"C": [1.0, 10.0], "gamma": [1 / 32]}
    fold = np.arange(600) % 4 - 1
    for cv in (ShuffleSplit(4, test_size=0.25, random_state=0), RepeatedKFold(n_splits=3, n_repeats=2, random_state=0),
               PredefinedSplit(fold)):
        ours = GridSearchCV(None, SVR(), grid, cv=cv).fit(X, y)
        ref = SkGridSearchCV(SVR(), grid, cv=cv).fit(X, y)
        n = ref.n_splits_
        got = np.stack([ours.cv_results_["split%d_test_score" % k] for k in range(n)], 1)
        exp = np.stack([ref.cv_results_["split%d_test_score" % k] for k in range(n)], 1)
        assert np.abs(got - exp).max() <= ORDER_BOUND, (type(cv).__name__, np.abs(got - exp).max())


def test_svr_multi_gpu_equals_single_gpu(monkeypatch):
    from spark_sklearn_b200.engine import device_count
    if device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    w = W.make_workload("svr_small")
    monkeypatch.setenv("B200GS_DEVICES", "1")
    one = GridSearchCV(None, SVR(), w["param_grid"], cv=5, refit=False).fit(w["X"], w["y"])
    monkeypatch.setenv("B200GS_DEVICES", "all")
    many = GridSearchCV(None, SVR(), w["param_grid"], cv=5, refit=False).fit(w["X"], w["y"])
    for k in one.cv_results_:
        if k.endswith("_score"):
            np.testing.assert_array_equal(np.asarray(one.cv_results_[k], float), np.asarray(many.cv_results_[k], float), err_msg=k)
