"""GPU tests of the SAG / SAGA path (csrc/sag.cu: scikit-learn's sag_solver, one warp per (candidate, split) fit).

Checkers: the CPU oracle (tests/sag_oracle.c), which equals scikit-learn bit for bit (tests/test_oracle_sag.py), the goldens
written by tests/golden/make_sag_goldens.py, and scikit-learn's own searches.  The squared loss uses IEEE operations only,
so its fits must give the oracle's bits; the logistic losses use CUDA's exp, which may differ from libm's in the last bit."""
import os
import warnings

import numpy as np
import pytest
from sklearn.exceptions import ConvergenceWarning
from sklearn.linear_model import LogisticRegression

from spark_sklearn_b200 import workloads as W

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _fold_data(n, ns, seed):
    rng = np.random.RandomState(seed)
    splits = [(rng.permutation(np.setdiff1d(np.arange(n), te)), te) for te in np.array_split(rng.permutation(n), ns)]
    fold_id = np.zeros(n, np.int8)
    for k, (_, te) in enumerate(splits):
        fold_id[te] = k
    return splits, fold_id


def test_device_draws_match_the_oracle(engine):
    from sag_oracle import draws
    w = W.make_workload("sag_small")
    engine.set_data(w["X"][:64], np.zeros(64, np.int8), 1, y_class=w["y"][:64].astype(np.int32))
    for seed, n, count in [(1, 1, 5), (5, 2, 100), (209652396, 1000, 5000), (2 ** 31 - 2, 4097, 3000), (0, 50, 10)]:
        np.testing.assert_array_equal(engine.debug_sag_draws(seed, n, count), draws(seed, n, count))


# (solver, alpha_scaled x 1e3, beta_scaled, max_iter): a rescale every few samples at the large alphas; with the last case
# and no intercept, rescales land on epochs' last samples and the L1 lagged update replays the cumulative sums
SQUARED_CASES = [("sag", 1.0, 0.0, 30), ("saga", 1.0, 0.0, 30), ("saga", 1.0, 0.05, 30), ("saga", 3e3, 0.02, 8),
                 ("sag", 3e3, 0.0, 8), ("saga", 0.0, 0.1, 40), ("saga", 3e4, 0.02, 8)]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_squared_loss_equals_the_oracle_bit_for_bit(engine, dtype):
    """sag_solver(loss='squared') on every split of a 3-split set (permuted training order, sample weights with zeros):
    coefficients, intercept, n_iter and sample steps identical to the oracle's"""
    from sklearn.linear_model._sag import get_auto_step_size
    from sklearn.utils.extmath import row_norms
    from sag_oracle import sag_fit
    rng = np.random.RandomState(3)
    n, d = 300, 9
    X = rng.randn(n, d).astype(dtype)
    y = X.astype(np.float64) @ rng.randn(d) + 0.3 * rng.randn(n)
    sw = rng.uniform(0, 2, n)
    sw[::6] = 0.0
    splits, fold_id = _fold_data(n, 3, 4)
    engine.set_data(X, fold_id, 3, y_target=y.astype(np.float32))
    engine.set_targets_f64(y)
    engine.set_train_order([tr for tr, _ in splits])
    engine.set_sample_weight(sw)
    try:
        for fi in (True, False):
            for solver, am, beta, mi in SQUARED_CASES:
                shape = (1, 3)
                steps, alphas, betas = np.zeros(shape), np.zeros(shape), np.zeros(shape)
                for k, (tr, _) in enumerate(splits):
                    a = am * 1e-3
                    mss = row_norms(X[tr], squared=True).max()
                    steps[0, k] = get_auto_step_size(mss, a, "squared", fi, n_samples=len(tr), is_saga=solver == "saga")
                    alphas[0, k], betas[0, k] = a, beta
                seeds = np.array([[11, 2 ** 31 - 2, 777]])
                r = engine.logreg_sag([[solver] * 3], alphas, betas, steps, seeds, "squared", tol=1e-4, max_iter=mi,
                                      fit_intercept=fi, return_stats=True)
                for k, (tr, _) in enumerate(splits):
                    coef, it, st, nst = sag_fit(X[tr], y[tr].astype(dtype), sw[tr].astype(dtype), "squared", steps[0, k],
                                                alphas[0, k], betas[0, k], seeds[0, k], solver == "saga", 1e-4, mi, fi)
                    assert r["n_iter"][0, k] == it and r["status"][0, k] == st, (solver, am, beta, k)
                    assert r["stats"][0, k, 0] == nst
                    np.testing.assert_array_equal(r["coef"][0, k], coef)
    finally:
        engine.set_sample_weight(None)


LOGISTIC_CASES = [dict(solver="sag"), dict(solver="saga", l1_ratio=0.5, C=0.5), dict(solver="saga", l1_ratio=1.0, C=0.3),
                  dict(solver="saga", C=np.inf), dict(solver="sag", C=1e-4), dict(solver="saga", fit_intercept=False)]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("key", ["sag_small", "sag_multi"])
@pytest.mark.parametrize("case", range(len(LOGISTIC_CASES)))
def test_logistic_fits_against_the_oracle(engine, dtype, key, case):
    """every split fit of a 3-split search (permuted training order, sample weights with zeros, class weights) against the
    oracle: n_iter within 1; the weights within 1e-9 relative where n_iter is equal, within 10 tol otherwise"""
    from sag_oracle import SAGOracle, step_and_penalties
    kw = dict(LOGISTIC_CASES[case], max_iter=60)
    w = W.make_workload(key)
    X, y = w["X"][:450].astype(dtype), w["y"][:450]
    classes, yc = np.unique(y, return_inverse=True)
    sw = np.random.RandomState(1).uniform(0, 2, len(X))
    sw[::7] = 0.0
    cw = {int(c): 1.0 + 0.5 * i for i, c in enumerate(classes)}
    splits, fold_id = _fold_data(len(X), 3, 4)
    p = LogisticRegression().get_params()
    p.update(kw)
    loss = "log" if len(classes) == 2 else "multinomial"
    st = np.array([[step_and_penalties(X[tr], p["C"], p["l1_ratio"], p["solver"], p["fit_intercept"], loss) for tr, _ in splits]])
    seeds = np.array([[101, 202, 303]])
    engine.set_data(X, fold_id, 3, y_class=yc.astype(np.int32))
    engine.set_train_order([tr for tr, _ in splits])
    engine.set_sample_weight(sw)
    engine.set_class_weight(np.array([cw[int(c)] for c in classes]))
    try:
        r = engine.logreg_sag([[p["solver"]] * 3], st[..., 1], st[..., 2], st[..., 0], seeds, loss, tol=p["tol"],
                              max_iter=p["max_iter"], fit_intercept=p["fit_intercept"], return_coef=True)
    finally:
        engine.set_sample_weight(None)
        engine.set_class_weight(None)
    equal = 0
    for k, (tr, _) in enumerate(splits):
        o = SAGOracle(X[tr], y[tr], sample_weight=sw[tr], class_weight=cw, seed=seeds[0, k], **kw)
        got = r["coef"][0, k]
        ref = np.concatenate([o.coef_.astype(np.float64), o.intercept_.astype(np.float64)[:, None]], 1)
        assert abs(int(r["n_iter"][0, k]) - o.n_iter) <= 1, (r["n_iter"][0, k], o.n_iter)
        scale = np.abs(ref).max()
        if r["n_iter"][0, k] == o.n_iter:
            assert np.abs(got - ref).max() <= 1e-9 * scale, np.abs(got - ref).max() / scale
        else:
            assert np.abs(got - ref).max() <= 10 * p["tol"] * scale
        equal += bool(np.array_equal(got, ref))
    print("SAG_EQUAL %s %s case %d: %d of 3 fits equal the oracle bit for bit" % (key, np.dtype(dtype).name, case, equal))


def _sk_grid(est, grid, X, y, **kw):
    from sklearn.model_selection import GridSearchCV as SkGrid
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        return SkGrid(est, grid, return_train_score=True, **kw).fit(X, y)


def _grid(est, grid, X, y, **kw):
    from spark_sklearn_b200 import GridSearchCV
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        return GridSearchCV(None, est, grid, **kw).fit(X, y)


def _split_scores(search, ns, which="test"):
    return np.stack([search.cv_results_["split%d_%s_score" % (k, which)] for k in range(ns)], 1)


@pytest.mark.parametrize("key", ["sag_small", "sag_multi"])
def test_search_equals_the_goldens(engine, key):
    """split scores within two flipped test rows, mean_test_score within 1e-3, best_params_ and per-fit n_iter_ (within 1)
    as scikit-learn 1.9's (best_index_ for best_params_); the refit's coefficients within 10 tol"""
    g = np.load(os.path.join(GOLDEN, key + ".npz"))
    w = W.make_workload(key)
    X, y = w["X"], w["y"]
    got = _grid(W.make_estimator(w), w["param_grid"], X, y, cv=5, return_train_score=True)
    a = _split_scores(got, 5)
    n_test = len(X) / 5
    assert np.abs(a - g["split_test"]).max() <= 2 / n_test + 1e-12
    assert np.abs(got.cv_results_["mean_test_score"] - g["mean_test"]).max() <= 1e-3
    assert got.best_index_ == int(g["best_index"])
    from sklearn.model_selection import ParameterGrid, StratifiedKFold
    from spark_sklearn_b200 import estimators as E
    splits = list(StratifiedKFold(5).split(X, y))
    cands = list(ParameterGrid(w["param_grid"]))
    plan = E.adapter_for(W.make_estimator(w)).plan(W.make_estimator(w), cands, X, y, E.Folds(splits, len(X)), 5)
    plan.evaluate(list(range(len(cands))))
    assert np.abs(plan.n_iter_ - g["n_iter"]).max() <= 1, np.abs(plan.n_iter_ - g["n_iter"]).max()
    be = got.best_estimator_
    scale = np.abs(g["refit_coef"]).max()
    assert np.abs(be.coef_ - g["refit_coef"]).max() <= 10 * be.tol * scale
    assert np.abs(be.intercept_ - g["refit_intercept"]).max() <= 10 * be.tol * max(scale, 1.0)


@pytest.mark.parametrize("key,scoring,cv,dtype", [("sag_small", "roc_auc", "shuffle", np.float64),
                                                  ("sag_small", "f1", 4, np.float32),
                                                  ("sag_multi", "balanced_accuracy", "repeated", np.float64),
                                                  ("sag_multi", None, 3, np.float32)])
def test_search_vs_sklearn(engine, key, scoring, cv, dtype):
    from sklearn.model_selection import RepeatedStratifiedKFold, ShuffleSplit
    w = W.make_workload(key)
    X, y = w["X"].astype(dtype), w["y"]
    cv = {"shuffle": ShuffleSplit(4, test_size=0.25, random_state=0),
          "repeated": RepeatedStratifiedKFold(n_splits=3, n_repeats=2, random_state=0)}.get(cv, cv)
    ns = cv if isinstance(cv, int) else cv.get_n_splits()
    est = W.make_estimator(w).set_params(max_iter=80)
    got = _grid(est, w["param_grid"], X, y, cv=cv, scoring=scoring, return_train_score=True)
    ref = _sk_grid(est, w["param_grid"], X, y, cv=cv, scoring=scoring)
    n_test = len(X) / ns if not isinstance(cv, ShuffleSplit) else 0.25 * len(X)
    assert np.abs(_split_scores(got, ns) - _split_scores(ref, ns)).max() <= 2 / n_test + 1e-12
    assert np.abs(got.cv_results_["mean_test_score"] - ref.cv_results_["mean_test_score"]).max() <= 1e-3
    assert got.best_params_ == ref.best_params_
    assert got.best_estimator_.coef_.dtype == ref.best_estimator_.coef_.dtype


def test_randomized_pipeline_refit_proba_pickle_and_devices(engine, monkeypatch):
    import pickle
    from sklearn.model_selection import RandomizedSearchCV as SkRandom
    from sklearn.pipeline import Pipeline
    from spark_sklearn_b200 import GridSearchCV, RandomizedSearchCV
    w = W.make_workload("sag_multi")
    X, y = w["X"], w["y"]
    pipe = Pipeline([("lr", LogisticRegression(solver="saga", max_iter=80))])
    dist = {"lr__C": [0.01, 0.1, 1.0, 10.0], "lr__l1_ratio": [0.0, 0.5, 1.0]}
    np.random.seed(5)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        got = RandomizedSearchCV(None, pipe, dist, n_iter=5, cv=3, random_state=1).fit(X, y)
        np.random.seed(5)
        ref = SkRandom(pipe, dist, n_iter=5, cv=3, random_state=1).fit(X, y)
    assert got.best_params_ == ref.best_params_
    assert np.abs(_split_scores(got, 3) - _split_scores(ref, 3)).max() <= 2 / (len(X) / 3) + 1e-12
    b, r = got.best_estimator_, ref.best_estimator_
    assert np.abs(b.predict_proba(X) - r.predict_proba(X)).max() <= 1e-3
    assert (b.predict(X) != r.predict(X)).sum() <= 2
    b2 = pickle.loads(pickle.dumps(b))
    np.testing.assert_array_equal(b2.predict_proba(X), b.predict_proba(X))
    # one GPU against every GPU: identical cv_results_
    grid = {"C": [0.1, 1.0, 10.0], "solver": ["sag", "saga"]}
    est = LogisticRegression(random_state=0, max_iter=50)
    monkeypatch.setenv("B200GS_DEVICES", "1")
    one = GridSearchCV(None, est, grid, cv=3).fit(X, y)
    monkeypatch.setenv("B200GS_DEVICES", "all")
    every = GridSearchCV(None, est, grid, cv=3).fit(X, y)
    for k in ("mean_test_score", "split0_test_score", "split2_test_score"):
        np.testing.assert_array_equal(one.cv_results_[k], every.cv_results_[k])
