"""Host-side logic of the nu-SVC and nu-SVR paths (no GPU): estimator resolution, parameter checks and rejections, the
nu feasibility check, the arrays and solver switch handed to the engine, and Pipeline name translation."""
import warnings

import numpy as np
import pytest
from sklearn.model_selection import KFold, StratifiedKFold
from sklearn.pipeline import Pipeline
from sklearn.svm import NuSVC, NuSVR

from spark_sklearn_b200 import estimators as E


class FakeEngine:
    """Records what a plan hands to the engine; returns zeros (NaN with n_iter -1 where nan_tasks says)."""

    def __init__(self):
        self.calls = []
        self.n = self.n_splits = 0
        self.nan_tasks = None

    def set_data(self, X, fold_id, n_splits, y_class=None, y_target=None):
        self.n, self.n_splits = len(X), n_splits

    def set_splits(self, te, tr, n_splits):
        self.n_splits = n_splits

    def set_targets_f64(self, y):
        pass

    def set_sample_weight(self, w=None):
        pass

    def set_class_weight(self, w=None):
        pass

    def set_scoring(self, kind=0, pos_class=1):
        pass

    def _out(self, n_cand):
        shape = (n_cand, self.n_splits)
        out = dict(test=np.zeros(shape), train=np.zeros(shape), n_iter=np.ones(shape, np.int32),
                   fit_ms=np.zeros(shape, np.float32), score_ms=np.zeros(shape, np.float32))
        if self.nan_tasks is not None:
            out["test"][self.nan_tasks] = np.nan
            out["train"][self.nan_tasks] = np.nan
            out["n_iter"][self.nan_tasks] = -1
        return out

    def svc(self, kernel, C, gamma, tol=1e-3, max_iter=-1, shrinking=True, return_train=True, flags=0, degree=None,
            coef0=None, nu=False):
        self.calls.append(("svc", list(kernel), list(C), nu))
        return self._out(len(C))

    def svr(self, kernel, C, epsilon, gamma, tol=1e-3, max_iter=-1, shrinking=True, return_train=True, flags=0, nu=False):
        self.calls.append(("svr", list(kernel), list(C), list(epsilon), nu))
        return self._out(len(C))

    def profile(self):
        return {}


@pytest.fixture
def fake(monkeypatch):
    eng = FakeEngine()
    monkeypatch.setattr(E, "get_engine", lambda device=None: eng)
    return eng


def _data(n=100, weights=(0.5, 0.5), seed=0):
    rng = np.random.RandomState(seed)
    X = rng.randn(n, 4)
    y = np.repeat(np.arange(len(weights)), [int(round(w * n)) for w in weights])
    return X, y


def _plan(adapter, est, cands, X, y, cv=5):
    splits = list((StratifiedKFold(cv) if adapter is E.NuSVCPlan else KFold(cv)).split(X, y))
    return adapter.plan(est, cands, X, y, E.Folds(splits, len(X)), len(splits))


def test_dispatch():
    assert E.adapter_for(NuSVC()) is E.NuSVCPlan
    assert E.adapter_for(NuSVR()) is E.NuSVRPlan
    pa = E.adapter_for(Pipeline([("m", NuSVR())]))
    assert isinstance(pa, E.PipelineAdapter) and pa.inner is E.NuSVRPlan
    assert pa._strip({"m__nu": 0.3, "m__C": 2.0}) == {"nu": 0.3, "C": 2.0}
    assert E.NuSVCPlan.multi_device and E.NuSVRPlan.multi_device


def test_nusvc_hands_nu_to_the_nu_solver(fake):
    X, y = _data()
    plan = _plan(E.NuSVCPlan, NuSVC(), [{"nu": 0.2}, {"nu": 0.5, "kernel": "poly"}], X, y)
    plan.evaluate([0, 1])
    assert fake.calls == [("svc", ["rbf", "poly"], [0.2, 0.5], True)]
    assert plan.costs() is None


def test_nusvr_hands_c_and_nu_to_the_nu_solver(fake):
    X, y = _data()
    plan = _plan(E.NuSVRPlan, NuSVR(C=3.0), [{"nu": 0.2}, {"nu": 0.7, "kernel": "linear"}], X, y.astype(float))
    plan.evaluate([0, 1])
    assert fake.calls == [("svr", ["rbf", "linear"], [3.0, 3.0], [0.2, 0.7], True)]


@pytest.mark.parametrize("est, cand", [(NuSVC(), {"nu": 1.5}), (NuSVC(), {"nu": 0.0}), (NuSVR(), {"nu": -0.1}),
                                       (NuSVR(), {"C": 0.0})])
def test_invalid_values_raise_sklearns_value_error(fake, est, cand):
    X, y = _data()
    adapter = E.NuSVCPlan if isinstance(est, NuSVC) else E.NuSVRPlan
    with pytest.raises(ValueError, match="parameter"):
        _plan(adapter, est, [cand], X, y.astype(float) if adapter is E.NuSVRPlan else y).evaluate([0])
    assert fake.calls == []


@pytest.mark.parametrize("est, cand", [(NuSVC(), {"probability": True}), (NuSVC(), {"break_ties": True}),
                                       (NuSVC(), {"kernel": "precomputed"}), (NuSVR(), {"kernel": "poly"}),
                                       (NuSVR(), {"kernel": "sigmoid"})])
def test_unsupported_options_raise(fake, est, cand):
    X, y = _data()
    adapter = E.NuSVCPlan if isinstance(est, NuSVC) else E.NuSVRPlan
    with pytest.raises(NotImplementedError):
        _plan(adapter, est, [cand], X, y.astype(float) if adapter is E.NuSVRPlan else y).evaluate([0])


def test_sample_weight_and_oversize_nusvr_raise(fake):
    X, y = _data()
    plan = _plan(E.NuSVCPlan, NuSVC(), [{"nu": 0.3}], X, y)
    with pytest.raises(NotImplementedError):
        plan.set_fit_params({"sample_weight": np.ones(len(X))})
    X = np.zeros((8193, 2))
    plan = _plan(E.NuSVRPlan, NuSVR(), [{"nu": 0.3}], X, np.zeros(len(X)), cv=2)
    with pytest.raises(NotImplementedError, match="8192"):
        plan.check_refit()


def test_feasibility_follows_libsvm():
    """svm_check_parameter: infeasible when nu (n1 + n2) / 2 > min(n1, n2) for some class pair of the training rows"""
    X, y = _data(weights=(0.7, 0.3))
    plan = E.NuSVCPlan.__new__(E.NuSVCPlan)
    plan.classes, plan.y_class, plan.folds, plan.fold_id = np.array([0, 1]), y, None, np.full(len(y), -1)
    assert not plan._infeasible(0.6, -1)                 # 0.6 x 100 / 2 = 30 = min(70, 30): feasible
    assert plan._infeasible(0.61, -1)


def test_infeasible_nu_raises_before_device_work(fake):
    X, y = _data(weights=(0.7, 0.3))
    plan = _plan(E.NuSVCPlan, NuSVC(), [{"nu": 0.3}, {"nu": 0.9}], X, y)
    with pytest.raises(ValueError, match="specified nu is infeasible"):
        plan.evaluate([0, 1], error_score="raise")
    assert fake.calls == []
    with pytest.raises(ValueError, match="specified nu is infeasible"):
        plan.refit({"nu": 0.9})
    assert fake.calls == []


def test_infeasible_tasks_take_error_score(fake):
    X, y = _data(weights=(0.7, 0.3))
    plan = _plan(E.NuSVCPlan, NuSVC(), [{"nu": 0.3}, {"nu": 0.9}], X, y)
    fake.nan_tasks = (slice(1, 2), slice(None))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        r = plan.evaluate([0, 1], error_score=-1.0)
    assert (r["test"][1] == -1.0).all() and (r["test"][0] == 0.0).all()
    assert (plan.n_iter_[1] == -1).all()
