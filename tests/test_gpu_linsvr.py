"""GPU tests of the LinearSVR path (csrc/linsvr.cu: liblinear's dual CD one warp per fit, TRON on the FP64 tensor cores).

Checkers: the CPU oracle (tests/linsvr_oracle.c), whose kernel-order switch sums the CD's dot products in the warp's order
and must therefore give the device's bits; goldens made by scikit-learn 1.9 (tests/golden/make_linsvr_goldens.py); and
scikit-learn's own searches.  Against scikit-learn the CD differs only in the order of each dot product's sum, which the
oracle measures as a trajectory change below 1e-12: n_iter must be equal on every fit and split scores within 1e-10."""
import pickle
import warnings

import numpy as np
import pytest
from sklearn.exceptions import ConvergenceWarning

from conftest import golden
from spark_sklearn_b200 import workloads as W

pytestmark = pytest.mark.gpu

SCORE_TOL = 1e-10


def _grid(est, grid, X, y, **kw):
    from spark_sklearn_b200 import GridSearchCV
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        return GridSearchCV(None, est, grid, **kw).fit(X, y)


def _sk_grid(est, grid, X, y, **kw):
    from sklearn.model_selection import GridSearchCV as SkGrid
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        return SkGrid(est, grid, return_train_score=True, **kw).fit(X, y)


def _split_scores(search, ns, which="test"):
    return np.stack([search.cv_results_["split%d_%s_score" % (k, which)] for k in range(ns)], 1)


def test_device_rng_matches_numpy(engine):
    for seed in (0, 1, 209652396, 2 ** 31 - 2):
        bg = np.random.MT19937()
        bg._legacy_seeding(seed)
        ref = bg.random_raw(1500).astype(np.uint32)             # crosses two generation steps of 624 words
        np.testing.assert_array_equal(engine.debug_mt19937(seed, 1500), ref)


@pytest.mark.parametrize("solver,kw", [(13, {}), (13, dict(C=10.0, epsilon=0.1)), (12, dict(C=0.5)),
                                       (13, dict(fit_intercept=False)), (13, dict(intercept_scaling=3.0)),
                                       (12, dict(max_iter=7, C=2.0))])
def test_cd_fit_equals_the_oracle_in_kernel_order(engine, solver, kw):
    """every CD fit of a 3-fold search (permuted training order, zero weights) against the oracle summing in the warp's
    order: the same bits"""
    from linsvr_oracle import LinearSVROracle
    from golden.make_linsvr_goldens import sample_weight
    w = W.make_workload("linsvr_small")
    X, y = w["X"][:900], w["y"][:900]
    sw = sample_weight(len(X))
    rng = np.random.RandomState(2)
    splits = [(rng.permutation(np.setdiff1d(np.arange(len(X)), te)), te) for te in np.array_split(np.arange(len(X)), 3)]
    fold_id = np.zeros(len(X), np.int8)
    for k, (_, te) in enumerate(splits):
        fold_id[te] = k
    engine.set_data(X, fold_id, 3, y_target=y.astype(np.float32))
    engine.set_targets_f64(y)
    engine.set_train_order([tr for tr, _ in splits])
    engine.set_sample_weight(sw)
    C, eps = kw.get("C", 1.0), kw.get("epsilon", 0.0)
    fi, isc, mi = kw.get("fit_intercept", True), kw.get("intercept_scaling", 1.0), kw.get("max_iter", 1000)
    seeds = np.array([[11, 12, 13]])
    try:
        r = engine.linsvr([C], [eps], [[solver] * 3], seeds, max_iter=mi, fit_intercept=fi, intercept_scaling=isc,
                          return_coef=True, return_stats=True)
    finally:
        engine.set_sample_weight(None)
    loss = "epsilon_insensitive" if solver == 13 else "squared_epsilon_insensitive"
    for k, (tr, _) in enumerate(splits):
        o = LinearSVROracle(X[tr], y[tr], C=C, epsilon=eps, loss=loss, dual=True, max_iter=mi, fit_intercept=fi,
                            intercept_scaling=isc, sample_weight=sw[tr], seed=seeds[0, k], kernel_order=True)
        assert r["n_iter"][0, k] == o.n_iter_
        assert r["cd_stats"][0, k, 0] == o.steps
        np.testing.assert_array_equal(r["coef"][0, k, :len(o.raw_coef_)], o.raw_coef_)


def test_tron_fit_vs_the_oracle(engine):
    """solver 11 with sample weights: n_iter equal, weights within 1e-12 relative (the LinearSVC oracle's bar)"""
    from linsvr_oracle import LinearSVROracle
    from golden.make_linsvr_goldens import sample_weight
    w = W.make_workload("linsvr_small")
    X, y = w["X"][:1500], w["y"][:1500]
    sw = sample_weight(len(X))
    engine.set_data(X, np.zeros(len(X), np.int8), 1, y_target=y.astype(np.float32))
    engine.set_targets_f64(y)
    engine.set_sample_weight(sw)
    try:
        for C, eps in [(0.1, 0.0), (10.0, 0.2)]:
            raw, it = engine.linsvr_refit(C, eps, 11, 0)
            o = LinearSVROracle(X, y, C=C, epsilon=eps, loss="squared_epsilon_insensitive", dual=False, sample_weight=sw)
            assert it == o.n_iter_
            assert np.abs(raw - o.raw_coef_).max() <= 1e-12 * np.abs(o.raw_coef_).max()
    finally:
        engine.set_sample_weight(None)


VARIANTS = [("linsvr_small", v) for v in ("none", "dual", "sw", "nofi", "scaling")] + [("linsvr_wide", v) for v in ("none", "sw")]


@pytest.mark.parametrize("key,variant", VARIANTS)
def test_linsvr_vs_golden(engine, key, variant):
    from sklearn.model_selection import KFold
    from sklearn.svm import LinearSVR
    from spark_sklearn_b200 import estimators as E
    from golden.make_linsvr_goldens import VARIANTS as V, sample_weight
    w = W.make_workload(key)
    X, y = w["X"], w["y"]
    g = golden(key)
    cands = W.candidates(w)
    plan = E.LinearSVRPlan.plan(LinearSVR(**w["est_params"], **V[variant]), cands, X, y,
                                   E.Folds(list(KFold(w["cv"]).split(X, y)), len(X)), w["cv"])
    plan.set_scoring(None)
    plan.set_fit_params({"sample_weight": sample_weight(len(X))} if variant == "sw" else None)
    out = plan.evaluate(list(range(len(cands))))
    np.testing.assert_array_equal(plan.n_iter_, g["%s_n_iter" % variant])
    assert np.abs(out["test"] - g["%s_test" % variant]).max() <= SCORE_TOL
    assert np.abs(out["train"] - g["%s_train" % variant]).max() <= SCORE_TOL


@pytest.mark.parametrize("key", ["linsvr_small", "linsvr_wide"])
def test_linsvr_refit_vs_golden(engine, key):
    from sklearn.svm import LinearSVR
    w = W.make_workload(key)
    g = golden(key)
    cand = W.candidates(w)[int(g["refit_index"])]
    s = _grid(LinearSVR(**w["est_params"]), {k: [v] for k, v in cand.items()}, w["X"], w["y"], cv=5)
    e = s.best_estimator_
    assert e.n_iter_ == int(g["refit_n_iter"])
    ref = max(np.abs(g["refit_coef"]).max(), np.abs(g["refit_intercept"]).max())
    assert np.abs(e.coef_ - g["refit_coef"]).max() <= 1e-10 * ref
    assert np.abs(e.intercept_ - g["refit_intercept"]).max() <= 1e-10 * ref


@pytest.mark.parametrize("scoring", [None, "r2", "neg_mean_squared_error", "neg_root_mean_squared_error"])
@pytest.mark.parametrize("cv_kind", ["kfold", "shuffle", "repeated"])
def test_linsvr_scorers_and_splitters_vs_sklearn(engine, scoring, cv_kind):
    from sklearn.model_selection import RepeatedKFold, ShuffleSplit
    from sklearn.svm import LinearSVR
    w = W.make_workload("linsvr_small")
    X, y = w["X"][:1200], w["y"][:1200]
    cv = {"kfold": 4, "shuffle": ShuffleSplit(4, test_size=0.3, random_state=0),
          "repeated": RepeatedKFold(n_splits=3, n_repeats=2, random_state=0)}[cv_kind]
    grid = {"C": [0.05, 2.0], "loss": ["epsilon_insensitive", "squared_epsilon_insensitive"], "epsilon": [0.1]}
    a = _grid(LinearSVR(random_state=3, max_iter=300), grid, X, y, cv=cv, scoring=scoring)
    b = _sk_grid(LinearSVR(random_state=3, max_iter=300), grid, X, y, cv=cv, scoring=scoring)
    ns = 4 if cv_kind == "kfold" else cv.get_n_splits()
    for which in ("test", "train"):
        assert np.abs(_split_scores(a, ns, which) - _split_scores(b, ns, which)).max() <= SCORE_TOL


def test_linsvr_random_search_pipeline_refit_pickle(engine):
    from scipy.stats import loguniform
    from sklearn.model_selection import RandomizedSearchCV as SkRandom
    from sklearn.pipeline import Pipeline
    from sklearn.svm import LinearSVR
    from spark_sklearn_b200 import RandomizedSearchCV
    w = W.make_workload("linsvr_small")
    X, y = w["X"][:2000], w["y"][:2000]
    pipe = Pipeline([("svr", LinearSVR(random_state=0, max_iter=400))])
    dist = {"svr__C": loguniform(1e-3, 1e1), "svr__epsilon": [0.0, 0.1]}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        a = RandomizedSearchCV(None, pipe, dist, n_iter=5, cv=3, random_state=0).fit(X, y)
        b = SkRandom(pipe, dist, n_iter=5, cv=3, random_state=0, return_train_score=True).fit(X, y)
    assert np.abs(_split_scores(a, 3) - _split_scores(b, 3)).max() <= SCORE_TOL
    assert a.best_params_ == b.best_params_
    ea, eb = a.best_estimator_.steps[0][1], b.best_estimator_.steps[0][1]
    assert ea.n_iter_ == eb.n_iter_
    pa, pb = a.predict(X), b.predict(X)
    assert np.abs(pa - pb).max() <= 1e-10 * np.abs(pb).max()
    c = pickle.loads(pickle.dumps(a.best_estimator_))
    np.testing.assert_array_equal(c.predict(X), pa)


def test_linsvr_random_state_none_follows_the_global_rng(engine):
    from sklearn.svm import LinearSVR
    w = W.make_workload("linsvr_small")
    X, y = w["X"][:900], w["y"][:900]
    grid = {"C": [0.1, 1.0]}
    np.random.seed(7)
    a = _grid(LinearSVR(max_iter=50), grid, X, y, cv=3)
    np.random.seed(7)
    b = _sk_grid(LinearSVR(max_iter=50), grid, X, y, cv=3)
    assert np.abs(_split_scores(a, 3) - _split_scores(b, 3)).max() <= SCORE_TOL
    assert np.abs(a.best_estimator_.coef_ - b.best_estimator_.coef_).max() <= 1e-10 * np.abs(b.best_estimator_.coef_).max()


def test_linsvr_max_iter_stop_warns(engine):
    from sklearn.svm import LinearSVR
    from spark_sklearn_b200 import GridSearchCV
    w = W.make_workload("linsvr_small")
    X, y = w["X"][:800], w["y"][:800]
    with pytest.warns(ConvergenceWarning, match="Liblinear failed to converge"):
        s = GridSearchCV(None, LinearSVR(max_iter=3, random_state=0), {"C": [1.0]}, cv=3).fit(X, y)
    ref = LinearSVR(max_iter=3, random_state=0)
    with pytest.warns(ConvergenceWarning):
        ref.fit(X, y)
    assert s.best_estimator_.n_iter_ == ref.n_iter_ == 3
    assert np.abs(s.predict(X) - ref.predict(X)).max() <= 1e-10 * np.abs(ref.predict(X)).max()


def test_linsvr_one_gpu_and_all_gpus_agree(engine, monkeypatch):
    from sklearn.svm import LinearSVR
    w = W.make_workload("linsvr_small")
    grid = {"C": list(np.logspace(-3, 1, 6)), "loss": ["epsilon_insensitive", "squared_epsilon_insensitive"]}
    X, y = w["X"][:2000], w["y"][:2000]
    monkeypatch.setenv("B200GS_DEVICES", "1")
    a = _grid(LinearSVR(random_state=0, max_iter=200), grid, X, y, cv=5)
    monkeypatch.setenv("B200GS_DEVICES", "all")
    b = _grid(LinearSVR(random_state=0, max_iter=200), grid, X, y, cv=5)
    for k in a.cv_results_:
        if "time" not in k:
            np.testing.assert_array_equal(np.asarray(a.cv_results_[k], object), np.asarray(b.cv_results_[k], object))
