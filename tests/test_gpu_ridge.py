"""GPU parity tests for the Ridge path (wgmma fold Grams + batched CG + Gram-statistics R^2) through the C ABI.

Checker: goldens made by scikit-learn 1.9.0 (Ridge keeps float32 throughout, LAPACK posv) and the numpy oracle.
Floating point: tolerance 2e-5 on per-split R^2 (both sides carry ~1e-6 of float32 solve error); BASELINE asks for
1e-4 on mean_test_score."""
import numpy as np
import pytest

from conftest import golden
from spark_sklearn_b200 import workloads as W

pytestmark = pytest.mark.gpu


def _setup(engine, key):
    from oracle import oracle as O
    w = W.make_workload(key)
    fold_id, ns = O.folds_from_cv(w["cv"], w["X"], w["y"], False)
    engine.set_data(w["X"], fold_id, ns, y_target=w["y"])
    return w, fold_id, ns


def test_ridge_c5_small_vs_golden(engine):
    w, fold_id, ns = _setup(engine, "c5_small")
    g = golden("c5_small")
    r = engine.ridge([c["alpha"] for c in W.candidates(w)])
    assert np.abs(r["test"] - g["test_scores"]).max() <= 2e-5
    assert np.abs(r["train"] - g["train_scores"]).max() <= 2e-5
    assert np.abs(r["test"].mean(1) - g["test_scores"].mean(1)).max() <= 1e-5


def test_ridge_no_intercept_and_ragged_folds(engine):
    from oracle import oracle as O
    rng = np.random.RandomState(3)
    n, d = 777, 45                                              # folds of unequal size, d not a multiple of 32
    X = (rng.randn(n, d) + 3.0).astype(np.float32)              # non-zero means: centring matters
    y = (X @ rng.randn(d) + 0.5 * rng.randn(n) + 7).astype(np.float32)
    fold_id, ns = O.folds_from_cv(7, X, y, False)
    engine.set_data(X, fold_id, ns, y_target=y)
    cands = [{"alpha": a} for a in (1e-2, 1.0, 100.0)]
    for fi in (True, False):
        r = engine.ridge([c["alpha"] for c in cands], fit_intercept=fi)
        te, tr = O.cv_scores_ridge(X, y, fold_id, ns, cands, fit_intercept=fi)
        assert np.abs(r["test"] - te).max() <= 5e-5, (fi, np.abs(r["test"] - te).max())
        assert np.abs(r["train"] - tr).max() <= 5e-5


def test_ridge_python_api_and_refit(engine):
    from sklearn.linear_model import Ridge
    from sklearn.model_selection import GridSearchCV as SkGrid
    from spark_sklearn_b200 import GridSearchCV
    w = W.make_workload("c5_small")
    X, y = w["X"], w["y"]
    grid = {"alpha": np.logspace(-2, 3, 6)}
    a = GridSearchCV(None, Ridge(), grid, cv=5).fit(X, y)
    b = SkGrid(Ridge(), grid, cv=5, return_train_score=True).fit(X, y)
    assert np.abs(a.cv_results_["mean_test_score"] - b.cv_results_["mean_test_score"]).max() <= 1e-5
    assert a.best_index_ == b.best_index_
    np.testing.assert_array_equal(a.cv_results_["rank_test_score"], b.cv_results_["rank_test_score"])
    assert np.abs(a.best_estimator_.coef_ - b.best_estimator_.coef_).max() <= 2e-4 * np.abs(b.best_estimator_.coef_).max()
    assert np.abs(a.predict(X) - b.predict(X)).max() <= 1e-3 * np.abs(y).max()


def test_ridge_c5_full_size_vs_golden(engine):
    """BASELINE config 5 at full size: 512 alphas x 10 folds on 20000x1024 -- the 1e-4 bar on mean_test_score."""
    w, fold_id, ns = _setup(engine, "c5")
    g = golden("c5_ridge_512")
    r = engine.ridge([c["alpha"] for c in W.candidates(w)])
    assert np.abs(r["test"].mean(1) - g["test_scores"].mean(1)).max() <= 5e-5
    assert np.abs(r["train"].mean(1) - g["train_scores"].mean(1)).max() <= 5e-5


def test_ridge_large_offsets_match_sklearn_float64(engine):
    """Features and targets whose mean dwarfs their spread (a year column near 2000, targets offset by 1e4): the Grams
    are formed from mean-shifted data, so the centring subtractions cancel nothing.  Checked against scikit-learn on
    float64 copies of the same float32 values (the well-conditioned answer), through the public API incl. the refit."""
    import warnings
    from sklearn.linear_model import Ridge
    from sklearn.model_selection import GridSearchCV as SkGrid
    from spark_sklearn_b200 import GridSearchCV
    rng = np.random.RandomState(7)
    n, d = 3000, 40
    X = rng.randn(n, d).astype(np.float32)
    y = (X @ rng.randn(d) + 0.3 * rng.randn(n)).astype(np.float32)
    X = (X + 1000.0).astype(np.float32)
    X[:, 0] = (2000.0 + rng.randint(0, 20, n)).astype(np.float32)
    y = (y + 1e4).astype(np.float32)
    grid = {"alpha": [1e-2, 1.0, 100.0]}
    a = GridSearchCV(None, Ridge(), grid, cv=5).fit(X, y)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        b = SkGrid(Ridge(), grid, cv=5, return_train_score=True).fit(X.astype(np.float64), y.astype(np.float64))
    assert np.abs(a.cv_results_["mean_test_score"] - b.cv_results_["mean_test_score"]).max() <= 1e-4
    assert np.abs(a.cv_results_["mean_train_score"] - b.cv_results_["mean_train_score"]).max() <= 1e-4
    assert a.best_index_ == b.best_index_
    res = y - a.predict(X)
    assert np.abs(res).max() < 3.0 and abs(res.mean()) < 0.05          # the intercept carries the offsets back
    assert np.abs(a.best_estimator_.coef_ - b.best_estimator_.coef_).max() <= 2e-3 * np.abs(b.best_estimator_.coef_).max()
