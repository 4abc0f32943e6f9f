"""Host-side logic of LinearSVC (no GPU): what the plan hands to the engine, dual resolution per training fold and for the
refit, scikit-learn's ValueErrors, the combinations without a CUDA path, candidate grouping, and materialize_linsvc against
a real fit."""
import pickle
import warnings

import numpy as np
import pytest
from sklearn.exceptions import ConvergenceWarning
from sklearn.model_selection import StratifiedKFold
from sklearn.svm import LinearSVC

from spark_sklearn_b200 import estimators as E
from spark_sklearn_b200 import workloads as W


class FakeEngine:
    """Records what a plan hands to the engine; returns zeros (raw weights: refit_raw when set)."""

    def __init__(self):
        self.calls, self.data, self.cw, self.sw = [], None, [], []
        self.n = self.n_splits = self.d = 0
        self.refit_raw = None

    def set_data(self, X, fold_id, n_splits, y_class=None, y_target=None):
        self.data = dict(X=np.array(X), fold_id=np.array(fold_id), y_class=np.array(y_class))
        self.n, self.d, self.n_splits = X.shape[0], X.shape[1], n_splits

    def set_splits(self, te, tr, n_splits):
        self.n_splits = n_splits

    def set_sample_weight(self, w=None):
        self.sw.append(None if w is None else np.array(w))

    def set_class_weight(self, w=None):
        self.cw.append(None if w is None else np.array(w))

    def set_scoring(self, kind=0, pos_class=1):
        pass

    def linsvc(self, C, tol=1e-4, max_iter=1000, fit_intercept=True, intercept_scaling=1.0, return_train=True):
        self.calls.append(dict(C=list(C), tol=tol, max_iter=max_iter, fit_intercept=fit_intercept,
                               intercept_scaling=intercept_scaling, cw=self.cw[-1]))
        shape = (len(C), self.n_splits)
        return dict(test=np.zeros(shape), train=np.zeros(shape), n_iter=np.ones(shape, np.int32),
                    fit_ms=np.zeros(shape, np.float32), score_ms=np.zeros(shape, np.float32))

    def linsvc_refit(self, C, tol=1e-4, max_iter=1000, fit_intercept=True, intercept_scaling=1.0):
        self.calls.append(dict(refit=True, C=C, cw=self.cw[-1]))
        return self.refit_raw, np.array([3], np.int32)

    def profile(self):
        return {}


@pytest.fixture
def fake(monkeypatch):
    eng = FakeEngine()
    monkeypatch.setattr(E, "get_engine", lambda device=None: eng)
    return eng


def _data(n=300, key="linsvc_small"):
    w = W.make_workload(key)
    return w["X"][:n], w["y"][:n]


def _plan(est, cands, X, y, cv=5):
    splits = list(StratifiedKFold(cv).split(X, y))
    return E.LinearSVCPlan.plan(est, cands, X, y, E.Folds(splits, len(X)), len(splits))


def test_adapter_and_arrays_handed_to_the_engine(fake):
    from sklearn.pipeline import Pipeline
    assert E.adapter_for(LinearSVC()) is E.LinearSVCPlan
    assert isinstance(E.adapter_for(Pipeline([("s", LinearSVC())])), E.PipelineAdapter)
    X, y = _data()
    X64 = X.astype(np.float64)
    plan = _plan(LinearSVC(), [{"C": 0.5}, {"C": 2.0}], X64, y)
    assert fake.data["X"].dtype == np.float64 and np.array_equal(fake.data["X"], X64)   # float64 X goes as it is
    np.testing.assert_array_equal(fake.data["y_class"], np.unique(y, return_inverse=True)[1])
    plan.evaluate([0, 1])
    (call,) = fake.calls
    assert call["C"] == [0.5, 2.0] and call["tol"] == 1e-4 and call["max_iter"] == 1000
    assert call["fit_intercept"] is True and call["intercept_scaling"] == 1.0 and call["cw"] is None
    _plan(LinearSVC(), [{"C": 1.0}], X, y)
    assert fake.data["X"].dtype == np.float32                                          # widened exactly on the device


def test_grouping(fake):
    X, y = _data()
    cands = [{"C": 1.0}, {"C": 2.0, "tol": 1e-3}, {"C": 3.0}, {"C": 4.0, "intercept_scaling": 2.0},
             {"C": 5.0, "class_weight": "balanced"}, {"C": 6.0, "fit_intercept": False}, {"C": 7.0, "max_iter": 50}]
    plan = _plan(LinearSVC(), cands, X, y)
    plan.evaluate(list(range(len(cands))))
    assert [c["C"] for c in fake.calls] == [[1.0, 3.0], [2.0], [4.0], [5.0], [6.0], [7.0]]
    assert fake.calls[3]["cw"].shape == (5, 2)                                         # 'balanced': one set per split
    assert fake.calls[2]["intercept_scaling"] == 2.0 and fake.calls[4]["fit_intercept"] is False


def test_balanced_class_weight_per_fold_uses_sample_weight(fake):
    from sklearn.utils.class_weight import compute_class_weight
    X, y = _data()
    sw = np.linspace(0.0, 2.0, len(y))
    plan = _plan(LinearSVC(class_weight="balanced"), [{"C": 1.0}], X, y)
    plan.set_fit_params({"sample_weight": sw})
    np.testing.assert_array_equal(fake.sw[-1], sw)
    plan.evaluate([0])
    splits = list(StratifiedKFold(5).split(X, y))
    for k, (tr, _) in enumerate(splits):
        ref = compute_class_weight("balanced", classes=np.unique(y), y=y[tr], sample_weight=sw[tr])
        np.testing.assert_array_equal(fake.calls[0]["cw"][k], ref)


def test_dual_resolution_per_fold_and_refit(fake):
    """dual='auto' picks the dual solver for a training set with fewer rows than features (svm/_classes.py
    _validate_dual_parameter): such a search raises before any device call, on the folds' sizes, not the whole X's"""
    rng = np.random.RandomState(0)
    X = rng.standard_normal((60, 50)).astype(np.float32)
    y = np.arange(60) % 2
    plan = _plan(LinearSVC(), [{"C": 1.0}], X, y)                      # 60 rows >= 50 features, but folds train on 48
    with pytest.raises(NotImplementedError, match="dual"):
        plan.evaluate([0])
    assert fake.calls == []
    X = rng.standard_normal((60, 48)).astype(np.float32)             # folds train on exactly 48 rows: primal
    plan = _plan(LinearSVC(), [{"C": 1.0}], X, y)
    plan.evaluate([0])
    assert len(fake.calls) == 1
    fake.refit_raw = np.zeros((1, 49))
    plan.refit({"C": 1.0})
    plan = _plan(LinearSVC(dual=False), [{"C": 1.0}], X[:, :40], y)   # dual=False: primal whatever the shape
    plan.evaluate([0])
    # the refit trains on every row: a plan whose folds are primal but whose refit has fewer rows than features cannot
    # exist (every training set is a subset), so check the rule directly on an all-rows count
    with pytest.raises(NotImplementedError, match="dual"):
        plan._check(LinearSVC().get_params(), 39)


@pytest.mark.parametrize("params,exc", [
    ({"dual": True}, NotImplementedError),
    ({"penalty": "l1", "dual": False}, NotImplementedError),
    ({"multi_class": "crammer_singer"}, NotImplementedError),
    ({"loss": "hinge", "dual": False}, ValueError),
    ({"loss": "hinge"}, NotImplementedError),                          # dual='auto' with hinge: dual only
    ({"penalty": "l1", "loss": "hinge", "dual": False}, ValueError),
    ({"C": 0.0}, ValueError),
    ({"C": -1.0}, ValueError),
    ({"intercept_scaling": 0.0}, ValueError),
    ({"tol": 0.0}, ValueError),
    ({"max_iter": -1}, ValueError),
    ({"penalty": "l3"}, ValueError),
])
def test_rejections_before_device_work(fake, params, exc):
    X, y = _data()
    plan = _plan(LinearSVC(), [params], X, y)
    with pytest.raises(exc):
        plan.evaluate([0])
    assert fake.calls == []
    if exc is ValueError:                                              # the same error class scikit-learn raises
        with pytest.raises(ValueError):
            LinearSVC(**params).fit(X, y)


@pytest.mark.parametrize("key,fit_intercept,scaling", [("linsvc_small", True, 1.0), ("linsvc_multi", True, 2.5),
                                                       ("linsvc_multi", False, 1.0)])
def test_materialize_matches_a_real_fit(key, fit_intercept, scaling):
    X, y = _data(800, key)
    ref = LinearSVC(C=0.3, fit_intercept=fit_intercept, intercept_scaling=scaling).fit(X, y)
    raw = np.hstack([ref.coef_, (np.atleast_1d(ref.intercept_) / scaling if fit_intercept else np.zeros(len(ref.coef_)))[:, None]])
    est = E.materialize_linsvc(LinearSVC(C=0.3, fit_intercept=fit_intercept, intercept_scaling=scaling), np.unique(y), raw,
                               np.array([ref.n_iter_] * len(raw)), X.shape[1])
    np.testing.assert_array_equal(est.predict(X), ref.predict(X))
    assert np.abs(est.decision_function(X) - ref.decision_function(X)).max() <= 1e-12 * np.abs(ref.decision_function(X)).max()
    assert est.n_iter_ == ref.n_iter_ and est.coef_.shape == ref.coef_.shape
    assert np.shape(est.intercept_) == np.shape(ref.intercept_)
    est2 = pickle.loads(pickle.dumps(est))
    np.testing.assert_array_equal(est2.predict(X), ref.predict(X))
    assert est.score(X, y) == ref.score(X, y)


def test_materialize_warns_at_max_iter():
    X, y = _data()
    raw = np.zeros((1, X.shape[1] + 1))
    with pytest.warns(ConvergenceWarning, match="Liblinear failed to converge"):
        E.materialize_linsvc(LinearSVC(max_iter=5), np.unique(y), raw, np.array([5]), X.shape[1])
    with warnings.catch_warnings():
        warnings.simplefilter("error", ConvergenceWarning)
        E.materialize_linsvc(LinearSVC(max_iter=5), np.unique(y), raw, np.array([4]), X.shape[1])
