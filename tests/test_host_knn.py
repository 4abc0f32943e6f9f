"""Host-side logic of the k-NN path (no GPU): estimator resolution, parameter checks and rejections, the arrays handed to
the engine, the n_neighbors > training rows behaviour under both error_score settings, and the refit."""
import warnings

import numpy as np
import pytest
from sklearn.model_selection import KFold, StratifiedKFold
from sklearn.neighbors import KNeighborsClassifier, KNeighborsRegressor
from sklearn.pipeline import Pipeline

from spark_sklearn_b200 import estimators as E
from spark_sklearn_b200 import workloads as W


class FakeEngine:
    """Records what a plan hands to the engine; returns zeros."""

    def __init__(self):
        self.calls = []
        self.n = self.n_splits = 0

    def set_data(self, X, fold_id, n_splits, y_class=None, y_target=None):
        self.n, self.n_splits = len(X), n_splits
        self.calls.append(("set_data", np.asarray(X).dtype, y_class, y_target))

    def set_splits(self, te, tr, n_splits):
        self.n_splits = n_splits

    def set_targets_f64(self, y):
        self.calls.append(("targets", np.array(y)))

    def set_sample_weight(self, w=None):
        pass

    def set_scoring(self, kind=0, pos_class=1):
        self.calls.append(("scoring", kind, pos_class))

    def knn(self, n_neighbors, weights, metric, return_train=True, y_f32=False):
        self.calls.append(("knn", list(n_neighbors), list(weights), list(metric), return_train, y_f32))
        shape = (len(n_neighbors), self.n_splits)
        return dict(test=np.zeros(shape), train=np.zeros(shape), fit_ms=np.zeros(shape, np.float32),
                    score_ms=np.zeros(shape, np.float32))

    def profile(self):
        return {}


@pytest.fixture
def fake(monkeypatch):
    eng = FakeEngine()
    monkeypatch.setattr(E, "get_engine", lambda device=None: eng)
    return eng


def _data(n=200, reg=False):
    w = W.make_workload("knn_reg_small" if reg else "knn_small")
    return w["X"][:n], w["y"][:n]


def _plan(est, cands, X, y, cv=5):
    cvs = KFold(cv) if isinstance(est, KNeighborsRegressor) else StratifiedKFold(cv)
    splits = list(cvs.split(X, y))
    return E.adapter_for(est).plan(est, cands, X, y, E.Folds(splits, len(X)), len(splits))


def test_adapter_resolution():
    assert E.adapter_for(KNeighborsClassifier()) is E.KNeighborsAdapter
    assert E.adapter_for(KNeighborsRegressor()) is E.KNeighborsRegressorAdapter
    assert E.KNeighborsAdapter.scorers is E.CLASSIFICATION_SCORERS
    assert E.KNeighborsRegressorAdapter.scorers is E.REGRESSION_SCORERS
    assert not E.KNeighborsAdapter.multi_device and not E.KNeighborsRegressorAdapter.multi_device
    a = E.adapter_for(Pipeline([("knn", KNeighborsClassifier())]))
    assert isinstance(a, E.PipelineAdapter) and a.inner is E.KNeighborsAdapter and not a.multi_device
    with pytest.raises(NotImplementedError, match="KNeighborsClassifier and KNeighborsRegressor"):
        from sklearn.tree import DecisionTreeClassifier
        E.adapter_for(DecisionTreeClassifier())


@pytest.mark.parametrize("bad", [{"n_neighbors": 257}, {"weights": lambda d: d}, {"p": 3}, {"p": 1.5},
                                 {"metric": "precomputed"}, {"metric": "chebyshev"}, {"metric_params": {"w": 1.0}},
                                 {"metric": "minkowski", "p": 4}])
def test_rejections_without_a_cuda_path(fake, bad):
    X, y = _data()
    with pytest.raises(NotImplementedError):
        _plan(KNeighborsClassifier(), [bad], X, y).evaluate([0])
    assert not [c for c in fake.calls if c[0] == "knn"]


@pytest.mark.parametrize("bad", [{"n_neighbors": 0}, {"n_neighbors": 2.5}, {"weights": "nope"}, {"p": 0}, {"p": -1.0},
                                 {"algorithm": "nope"}, {"leaf_size": 0}])
def test_invalid_values_raise_scikit_learns_value_error(fake, bad):
    X, y = _data()
    with pytest.raises(ValueError) as ours:
        _plan(KNeighborsClassifier(), [bad], X, y).evaluate([0])
    with pytest.raises(ValueError) as theirs:
        KNeighborsClassifier(**bad).fit(X, y).predict(X[:5])
    assert str(ours.value) == str(theirs.value)


def test_other_rejections(fake):
    X, y = _data()
    plan = _plan(KNeighborsClassifier(), [{}], X, y)
    with pytest.raises(NotImplementedError):
        plan.set_fit_params({"sample_weight": np.ones(len(X))})
    with pytest.raises(NotImplementedError):
        plan.set_scoring("r2")
    Xr, yr = _data(reg=True)
    with pytest.raises(NotImplementedError):
        _plan(KNeighborsRegressor(), [{}], Xr, np.stack([yr, yr], 1))
    with pytest.raises(NotImplementedError):
        _plan(KNeighborsRegressor(), [{}], Xr, yr).set_scoring("accuracy")
    yc = np.arange(len(X)) % 65
    with pytest.raises(NotImplementedError):
        _plan(KNeighborsClassifier(), [{}], X, yc, cv=2)
    w = W.make_workload("knn_multi")
    with pytest.raises(NotImplementedError):
        _plan(KNeighborsClassifier(), [{}], w["X"][:200], w["y"][:200]).set_scoring("roc_auc")


def test_accepted_parameters(fake):
    """algorithm, leaf_size and n_jobs are accepted; every metric spelling resolves to the two the engine has"""
    X, y = _data(n=400)
    cands = [{"n_neighbors": 3, "p": 1}, {"n_neighbors": 5, "weights": "distance"}, {"metric": "l1"},
             {"metric": "cityblock", "algorithm": "kd_tree"}, {"metric": "manhattan", "leaf_size": 5},
             {"metric": "euclidean", "n_jobs": 2}, {"metric": "l2", "algorithm": "ball_tree"}, {"n_neighbors": 256}]
    plan = _plan(KNeighborsClassifier(), cands, X, y)
    plan.set_scoring("roc_auc")
    plan.evaluate(list(range(len(cands))), return_train=False)
    (call,) = [c for c in fake.calls if c[0] == "knn"]
    assert call[1] == [3, 5, 5, 5, 5, 5, 5, 256]
    assert call[2] == ["uniform", "distance"] + ["uniform"] * 6
    assert call[3] == ["manhattan", "euclidean", "manhattan", "manhattan", "manhattan", "euclidean", "euclidean", "euclidean"]
    assert call[4] is False and call[5] is False
    assert ("scoring", 5, 1) in fake.calls


def test_arrays_handed_to_the_engine(fake):
    """class ids in sorted-label order; regressor: float64 targets, and the float32 flag when y is float32"""
    X, y = _data()
    labels = np.array(["b", "a"])[y]
    _plan(KNeighborsClassifier(), [{}], X, labels)
    sd = [c for c in fake.calls if c[0] == "set_data"][-1]
    assert sd[1] == np.float32 and np.array_equal(sd[2], (labels == "b").astype(np.int32))
    Xr, yr = _data(reg=True)
    for dt in (np.float64, np.float32):
        plan = _plan(KNeighborsRegressor(), [{"n_neighbors": 4}], Xr, yr.astype(dt))
        plan.evaluate([0])
        tg = [c for c in fake.calls if c[0] == "targets"][-1]
        assert tg[1].dtype == np.float64 and np.array_equal(tg[1], yr.astype(dt).astype(np.float64))
        assert [c for c in fake.calls if c[0] == "knn"][-1][5] is (dt == np.float32)


def test_n_neighbors_above_the_training_rows(fake):
    """scikit-learn's kneighbors raises ValueError from the scorer: error_score='raise' raises it before any device work,
    otherwise those (candidate, split) scores take error_score"""
    X, y = _data(n=40)
    cands = [{"n_neighbors": 3}, {"n_neighbors": 33}]          # 5 folds of 40 rows: 32 training rows per split
    plan = _plan(KNeighborsClassifier(), cands, X, y)
    with pytest.raises(ValueError) as ours:
        plan.evaluate([0, 1])
    tr, te = next(iter(StratifiedKFold(5).split(X, y)))
    with pytest.raises(ValueError) as theirs:
        KNeighborsClassifier(n_neighbors=33).fit(X[tr], y[tr]).score(X[te], y[te])
    assert str(ours.value) == str(theirs.value)
    assert not [c for c in fake.calls if c[0] == "knn"]
    with pytest.warns(UserWarning):
        out = plan.evaluate([0, 1], error_score=-1.0)
    assert np.all(out["test"][1] == -1.0) and np.all(out["train"][1] == -1.0)
    assert np.all(out["test"][0] == 0.0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = plan.evaluate([0, 1], error_score=np.nan)
    assert np.all(np.isnan(out["test"][1]))


@pytest.mark.parametrize("reg", [False, True])
def test_refit_is_a_fitted_estimator(fake, reg):
    X, y = _data(reg=reg)
    est = KNeighborsRegressor() if reg else KNeighborsClassifier()
    best = {"n_neighbors": 7, "weights": "distance", "p": 1}
    got = _plan(est, [best], X, y).refit(best)
    ref = type(est)(**best).fit(X, y)
    assert got is not est and got.get_params() == ref.get_params()
    np.testing.assert_array_equal(got.predict(X[:50]), ref.predict(X[:50]))
    pipe = Pipeline([("knn", est)])
    adapter = E.adapter_for(pipe)
    folds = E.Folds(list(KFold(5).split(X)), len(X))
    plan = adapter.plan(pipe, [{"knn__n_neighbors": 7}], X, y, folds, 5)
    fitted = plan.refit({"knn__n_neighbors": 7, "knn__weights": "distance", "knn__p": 1})
    assert isinstance(fitted, Pipeline)
    np.testing.assert_array_equal(fitted.predict(X[:50]), ref.predict(X[:50]))


def test_knn_workloads():
    for key, shape, name in (("knn_small", (2000, 32), "KNeighborsClassifier"), ("knn_multi", (2000, 32), "KNeighborsClassifier"),
                             ("knn_reg_small", (1000, 32), "KNeighborsRegressor")):
        w = W.make_workload(key)
        assert w["X"].shape == shape and w["X"].dtype == np.float32
        assert type(W.make_estimator(w)).__name__ == name
    assert len(np.unique(W.make_workload("knn_multi")["y"])) == 4
    assert len(W.candidates(W.make_workload("knn_small"))) == 16
    g = np.load(__import__("os").path.join(__import__("os").path.dirname(__file__), "golden", "knn_c2.npz"))
    assert g["test"].shape == (40, 5) and g["train"].shape == (40, 5)
