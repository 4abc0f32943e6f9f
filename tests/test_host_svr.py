"""Host-side logic of the epsilon-SVR path (no GPU): estimator resolution, parameter checks, per-fold gamma, the arrays
handed to the engine, and the fitted sklearn.svm.SVR assembled from the refit buffers."""
import pickle
import warnings

import numpy as np
import pytest
from sklearn.pipeline import Pipeline
from sklearn.svm import SVR

from spark_sklearn_b200 import estimators as E
from spark_sklearn_b200 import workloads as W


class FakeEngine:
    """Records what a plan hands to the engine; returns zeros."""

    def __init__(self):
        self.calls = []
        self.n = self.n_splits = 0

    def set_data(self, X, fold_id, n_splits, y_class=None, y_target=None):
        self.n, self.n_splits = len(X), n_splits
        self.calls.append(("set_data", y_class, y_target))

    def set_splits(self, te, tr, n_splits):
        self.n_splits = n_splits

    def set_targets_f64(self, y):
        self.calls.append(("targets", np.array(y)))

    def set_sample_weight(self, w=None):
        pass

    def set_scoring(self, kind=0, pos_class=1):
        self.calls.append(("scoring", kind))

    def svr(self, kernel, C, epsilon, gamma, tol=1e-3, max_iter=-1, shrinking=True, return_train=True, flags=0):
        self.calls.append(("svr", list(kernel), list(C), list(epsilon), np.array(gamma), tol, max_iter, shrinking))
        shape = (len(C), self.n_splits)
        return dict(test=np.zeros(shape), train=np.zeros(shape), n_iter=np.ones(shape, np.int32),
                    fit_ms=np.zeros(shape, np.float32), score_ms=np.zeros(shape, np.float32))

    def profile(self):
        return {}


@pytest.fixture
def fake(monkeypatch):
    eng = FakeEngine()
    monkeypatch.setattr(E, "get_engine", lambda device=None: eng)
    return eng


def _plan(est, cands, X, y, cv=5):
    from sklearn.model_selection import KFold
    splits = list(KFold(cv).split(X, y))
    return E.SVRPlan.plan(est, cands, X, y, E.Folds(splits, len(X)), len(splits))


def test_adapter_resolution():
    assert E.adapter_for(SVR()) is E.SVRPlan
    a = E.adapter_for(Pipeline([("svr", SVR())]))
    assert isinstance(a, E.PipelineAdapter) and a.inner is E.SVRPlan
    assert a.scorers is E.REGRESSION_SCORERS and a.multi_device
    with pytest.raises(NotImplementedError):
        E.adapter_for(Pipeline([("a", SVR()), ("b", SVR())]))


def test_rejections(fake):
    w = W.make_workload("svr_small")
    X, y = w["X"][:200], w["y"][:200]
    plan = _plan(SVR(), [{"kernel": "poly"}], X, y)
    with pytest.raises(NotImplementedError):
        plan.evaluate([0])
    with pytest.raises(NotImplementedError):
        plan.set_scoring("accuracy")
    with pytest.raises(NotImplementedError):
        plan.set_fit_params({"sample_weight": np.ones(len(X))})
    for bad in ({"C": -1.0}, {"C": 0.0}, {"epsilon": -0.1}, {"gamma": -1.0}, {"gamma": "nope"}):
        with pytest.raises(ValueError):
            _plan(SVR(), [bad], X, y).evaluate([0])
    plan.set_scoring("neg_root_mean_squared_error")
    assert plan.score_kind == 17


def test_arrays_handed_to_the_engine(fake):
    """gamma 'scale' per training fold as SVR.fit(X[train]) resolves it, 'auto' = 1/d, float64 targets, one engine call
    per (tol, max_iter, shrinking) group."""
    from sklearn.model_selection import KFold
    w = W.make_workload("svr_small")
    X, y = w["X"][:300], w["y"][:300]
    cands = [{"C": 1.0, "gamma": "scale", "epsilon": 0.1}, {"C": 10.0, "gamma": "auto", "epsilon": 0.0},
             {"kernel": "linear", "C": 2.0, "shrinking": False}]
    plan = _plan(SVR(), cands, X, y)
    plan.evaluate([0, 1, 2])
    tg = [c for c in fake.calls if c[0] == "targets"]
    assert tg and tg[-1][1].dtype == np.float64 and np.array_equal(tg[-1][1], y)
    svr_calls = [c for c in fake.calls if c[0] == "svr"]
    assert len(svr_calls) == 2
    first = svr_calls[0]
    assert first[1] == ["rbf", "rbf"] and first[2] == [1.0, 10.0] and first[3] == [0.1, 0.0]
    for k, (tr, _) in enumerate(KFold(5).split(X)):
        est = SVR(gamma="scale").fit(X[tr], y[tr])
        assert first[4][0, k] == est._gamma
    assert np.all(first[4][1] == 1.0 / X.shape[1])
    assert svr_calls[1][1] == ["linear"] and svr_calls[1][7] is False


def test_column_vector_y(fake):
    from sklearn.exceptions import DataConversionWarning
    w = W.make_workload("svr_small")
    X, y = w["X"][:100], w["y"][:100]
    with pytest.warns(DataConversionWarning):
        plan = _plan(SVR(), [{}], X, y[:, None])
    assert plan.y.shape == (100,) and np.array_equal(plan.y, y)
    with pytest.raises(ValueError):
        _plan(SVR(), [{}], X, np.stack([y, y], 1))


@pytest.mark.parametrize("kernel", ["rbf", "linear"])
def test_materialize_svr_matches_a_real_fit(kernel):
    """The SVR assembled from (coef by row, rho, n_iter) has the attribute set of SVR.fit and predicts and pickles alike."""
    w = W.make_workload("svr_small")
    X, y = w["X"][:400], w["y"][:400]
    ref = SVR(kernel=kernel, C=3.0, epsilon=0.1).fit(X, y)
    coef = np.zeros(len(X))
    coef[ref.support_] = ref.dual_coef_[0]
    got = E.materialize_svr(SVR(kernel=kernel, C=3.0, epsilon=0.1), X, coef, -ref.intercept_[0], ref.n_iter_, ref._gamma)
    assert set(vars(got)) == set(vars(ref))
    for k, v in vars(ref).items():
        g = getattr(got, k)
        if isinstance(v, np.ndarray):
            assert g.dtype == v.dtype and g.shape == v.shape, k
            np.testing.assert_array_equal(g, v, err_msg=k)
        else:
            assert type(g) is type(v) and g == v, k
    np.testing.assert_array_equal(got.predict(X), ref.predict(X))
    back = pickle.loads(pickle.dumps(got))
    np.testing.assert_array_equal(back.predict(X[:50]), ref.predict(X[:50]))


def test_svr_workloads():
    for key, shape in (("svr_small", (1000, 32)), ("svr_mid", (5000, 128))):
        w = W.make_workload(key)
        assert w["X"].shape == shape and w["X"].dtype == np.float32 and w["y"].dtype == np.float64
        assert abs(w["y"].mean()) < 1e-12 and abs(w["y"].std() - 1) < 1e-12
        assert isinstance(W.make_estimator(w), SVR)
    assert len(W.candidates(W.make_workload("svr_small"))) == 24


def test_refit_too_large_fails_before_the_search(fake):
    """a refit on more than 8192 rows raises from check_refit, which the search calls before any fit"""
    X = np.zeros((8200, 2), np.float32)
    y = np.arange(8200, dtype=np.float64)
    plan = _plan(SVR(), [{}], X, y, cv=2)                       # 4100-row folds: the search itself would run
    with pytest.raises(NotImplementedError):
        plan.check_refit()
    small = _plan(SVR(), [{}], X[:1000], y[:1000])
    small.check_refit()
