"""Host-side logic of LinearSVR (no GPU): what the plan hands to the engine (data, training order, solvers, seeds, weights),
dual resolution per training fold and for the refit, the seed rule for int / RandomState / None, scikit-learn's ValueErrors
and the values without a CUDA path, and materialize_linsvr against a real fit."""
import pickle
import warnings

import numpy as np
import pytest
from sklearn.exceptions import ConvergenceWarning
from sklearn.model_selection import KFold, ShuffleSplit
from sklearn.svm import LinearSVR

from spark_sklearn_b200 import estimators as E
from spark_sklearn_b200 import workloads as W

INT_MAX = np.iinfo("i").max


class FakeEngine:
    """Records what a plan hands to the engine; returns zeros (raw weights: refit_raw when set)."""

    def __init__(self):
        self.calls, self.data, self.sw, self.order = [], None, [], None
        self.n = self.n_splits = self.d = 0
        self.refit_raw, self.refit_iter = None, 3

    def set_data(self, X, fold_id, n_splits, y_class=None, y_target=None):
        self.data = dict(X=np.array(X), fold_id=np.array(fold_id), y_target=np.array(y_target))
        self.n, self.d, self.n_splits = X.shape[0], X.shape[1], n_splits
        self.order = None

    def set_splits(self, te, tr, n_splits):
        self.n_splits = n_splits
        self.order = None

    def set_targets_f64(self, y):
        self.data["y64"] = np.array(y)

    def set_train_order(self, rows=None):
        self.order = None if rows is None else [np.array(r) for r in rows]

    def set_sample_weight(self, w=None):
        self.sw.append(None if w is None else np.array(w))

    def set_class_weight(self, w=None):
        pass

    def set_scoring(self, kind=0, pos_class=1):
        self.kind = kind

    def linsvr(self, C, epsilon, solver, seed, tol=1e-4, max_iter=1000, fit_intercept=True, intercept_scaling=1.0,
               return_train=True, return_coef=False, return_stats=False):
        self.calls.append(dict(C=list(C), epsilon=list(epsilon), solver=np.array(solver), seed=np.array(seed), tol=tol,
                               max_iter=max_iter, fit_intercept=fit_intercept, intercept_scaling=intercept_scaling))
        shape = (len(C), self.n_splits)
        return dict(test=np.zeros(shape), train=np.zeros(shape), n_iter=np.ones(shape, np.int32),
                    fit_ms=np.zeros(shape, np.float32), score_ms=np.zeros(shape, np.float32),
                    cd_stats=np.zeros(shape + (3,), np.int64))

    def linsvr_refit(self, C, epsilon, solver, seed, tol=1e-4, max_iter=1000, fit_intercept=True, intercept_scaling=1.0):
        self.calls.append(dict(refit=True, C=C, solver=solver, seed=seed))
        raw = np.zeros(self.d + 1) if self.refit_raw is None else self.refit_raw
        return raw, self.refit_iter

    def profile(self):
        return {}


@pytest.fixture
def fake(monkeypatch):
    eng = FakeEngine()
    monkeypatch.setattr(E, "get_engine", lambda device=None: eng)
    return eng


def _data(n=300, key="linsvr_small"):
    w = W.make_workload(key)
    return w["X"][:n], w["y"][:n]


def _plan(est, cands, X, y, cv=None):
    splits = list((cv or KFold(5)).split(X, y))
    return E.LinearSVRPlan.plan(est, cands, X, y, E.Folds(splits, len(X)), len(splits)), splits


def test_adapter_and_arrays_handed_to_the_engine(fake):
    from sklearn.pipeline import Pipeline
    assert E.adapter_for(LinearSVR()) is E.LinearSVRPlan
    assert E.LinearSVRPlan.multi_device and E.LinearSVRPlan.scorers is E.REGRESSION_SCORERS
    assert isinstance(E.adapter_for(Pipeline([("s", LinearSVR())])), E.PipelineAdapter)
    X, y = _data()
    plan, splits = _plan(LinearSVR(random_state=0), [{"C": 0.5, "epsilon": 0.1}, {"C": 2.0}], X, y)
    assert fake.data["X"].dtype == np.float32                                       # widened exactly on the device
    assert fake.data["y64"].dtype == np.float64 and np.array_equal(fake.data["y64"], y)
    plan.evaluate([0, 1])
    (call,) = fake.calls
    assert call["C"] == [0.5, 2.0] and call["epsilon"] == [0.1, 0.0] and call["tol"] == 1e-4 and call["max_iter"] == 1000
    assert call["fit_intercept"] is True and call["intercept_scaling"] == 1.0
    assert (call["solver"] == 13).all() and call["solver"].shape == (2, 5)
    assert (call["seed"] == np.random.RandomState(0).randint(INT_MAX)).all()
    _plan(LinearSVR(), [{}], X.astype(np.float64), y)
    assert fake.data["X"].dtype == np.float64


def test_grouping(fake):
    X, y = _data()
    cands = [{"C": 1.0}, {"C": 2.0, "tol": 1e-3}, {"C": 3.0}, {"C": 4.0, "intercept_scaling": 2.0},
             {"C": 6.0, "fit_intercept": False}, {"C": 7.0, "max_iter": 50}]
    plan, _ = _plan(LinearSVR(), cands, X, y)
    plan.evaluate(list(range(len(cands))))
    assert [c["C"] for c in fake.calls] == [[1.0, 3.0], [2.0], [4.0], [6.0], [7.0]]
    assert fake.calls[2]["intercept_scaling"] == 2.0 and fake.calls[3]["fit_intercept"] is False


def test_dual_resolution_per_fold_and_refit(fake):
    """dual='auto' resolves on each training set's shape (svm/_classes.py _validate_dual_parameter): the squared loss takes
    the primal TRON (11) with at least as many rows as features, the dual CD (12) otherwise; epsilon_insensitive is 13"""
    rng = np.random.RandomState(0)
    X = rng.standard_normal((60, 50)).astype(np.float32)
    y = rng.standard_normal(60)
    cands = [{"loss": "squared_epsilon_insensitive"}, {"loss": "epsilon_insensitive"},
             {"loss": "squared_epsilon_insensitive", "dual": False}, {"loss": "squared_epsilon_insensitive", "dual": True}]
    plan, _ = _plan(LinearSVR(), cands, X, y)                 # 60 rows >= 50 features, but folds train on 48
    plan.evaluate([0, 1, 2, 3])
    np.testing.assert_array_equal(fake.calls[0]["solver"], [[12] * 5, [13] * 5, [11] * 5, [12] * 5])
    plan.refit(cands[0])                                      # the refit trains on all 60 rows: primal
    assert fake.calls[-1]["solver"] == 11
    # a mixed search: folds of unequal size resolve differently
    cv = [(np.arange(10, 60), np.arange(10)), (np.arange(15, 60), np.arange(15))]   # 50 and 45 training rows
    plan = E.LinearSVRPlan.plan(LinearSVR(loss="squared_epsilon_insensitive"), [{}], X, y, E.Folds(cv, 60), 2)
    plan.evaluate([0])
    np.testing.assert_array_equal(fake.calls[-1]["solver"], [[11, 12]])


def test_shuffle_split_order_reaches_the_engine(fake):
    X, y = _data()
    cv = ShuffleSplit(4, test_size=0.3, random_state=0)
    plan, splits = _plan(LinearSVR(), [{}], X, y, cv)
    assert len(fake.order) == 4
    for (tr, _), got in zip(splits, fake.order):
        np.testing.assert_array_equal(got, tr)                # the splitter's order, not sorted
    assert any(not np.all(np.diff(tr) > 0) for tr, _ in splits)


def test_seeds_int_randomstate_none(fake):
    X, y = _data()
    cands = [{"C": 1.0}, {"C": 2.0}]
    plan, _ = _plan(LinearSVR(random_state=5), cands, X, y)
    plan.evaluate([0, 1])
    assert (fake.calls[-1]["seed"] == np.random.RandomState(5).randint(INT_MAX)).all()
    rs = np.random.RandomState(9)
    before = rs.get_state()[1].copy()
    plan, _ = _plan(LinearSVR(random_state=rs), cands, X, y)
    plan.evaluate([0, 1])
    assert (fake.calls[-1]["seed"] == np.random.RandomState(9).randint(INT_MAX)).all()
    np.testing.assert_array_equal(rs.get_state()[1], before)  # the caller's RandomState is not advanced
    plan.refit({"C": 1.0})
    assert fake.calls[-1]["seed"] == np.random.RandomState(9).randint(INT_MAX)
    # None: numpy's global RandomState, candidate-major, split-minor, then the refit's draw
    np.random.seed(123)
    ref = np.random.RandomState(123).randint(INT_MAX, size=11)
    plan, _ = _plan(LinearSVR(random_state=None), cands, X, y)
    plan.evaluate([1])                                        # even a subset of the candidates: the table is the search's
    np.testing.assert_array_equal(fake.calls[-1]["seed"], ref[5:10].reshape(1, 5))
    plan.evaluate([0])
    np.testing.assert_array_equal(fake.calls[-1]["seed"], ref[0:5].reshape(1, 5))
    plan.refit({"C": 1.0})
    assert fake.calls[-1]["seed"] == ref[10]


def test_sample_weight(fake):
    X, y = _data()
    sw = np.linspace(0.0, 2.0, len(y))
    plan, _ = _plan(LinearSVR(), [{}], X, y)
    plan.set_fit_params({"sample_weight": sw})
    np.testing.assert_array_equal(fake.sw[-1], sw)
    with pytest.raises(NotImplementedError):
        plan.set_fit_params({"foo": 1})


@pytest.mark.parametrize("params,exc", [
    ({"loss": "epsilon_insensitive", "dual": False}, ValueError),
    ({"C": 0.0}, ValueError),
    ({"C": -1.0}, ValueError),
    ({"tol": 0.0}, ValueError),
    ({"max_iter": -1}, ValueError),
    ({"loss": "hinge"}, ValueError),
    ({"intercept_scaling": 0.0}, ValueError),
    ({"epsilon": -0.1}, NotImplementedError),
])
def test_rejections_before_device_work(fake, params, exc):
    X, y = _data()
    plan, _ = _plan(LinearSVR(), [params], X, y)
    with pytest.raises(exc):
        plan.evaluate([0])
    assert fake.calls == []
    if exc is ValueError:                                     # the same error class scikit-learn raises
        with pytest.raises(ValueError):
            LinearSVR(**params).fit(X, y)


def test_too_many_features(fake):
    rng = np.random.RandomState(0)
    with pytest.raises(NotImplementedError, match="512"):
        _plan(LinearSVR(), [{}], rng.standard_normal((40, 513)), rng.standard_normal(40))
    _plan(LinearSVR(), [{}], rng.standard_normal((40, 512)), rng.standard_normal(40))


def test_pipeline_plan(fake):
    from sklearn.pipeline import Pipeline
    X, y = _data()
    adapter = E.adapter_for(Pipeline([("svr", LinearSVR())]))
    assert adapter.multi_device
    splits = list(KFold(3).split(X))
    plan = adapter.plan(Pipeline([("svr", LinearSVR(random_state=1))]), [{"svr__C": 0.3}], X, y, E.Folds(splits, len(X)), 3)
    plan.evaluate([0])
    assert fake.calls[-1]["C"] == [0.3]
    fake.refit_raw = np.arange(X.shape[1] + 1, dtype=np.float64)
    pipe = plan.refit({"svr__C": 0.3})
    assert isinstance(pipe, Pipeline) and pipe.steps[0][1].C == 0.3
    np.testing.assert_array_equal(pipe.steps[0][1].coef_, fake.refit_raw[:-1])


@pytest.mark.parametrize("kw", [dict(), dict(fit_intercept=False), dict(intercept_scaling=2.5, C=0.3),
                                dict(loss="squared_epsilon_insensitive", dual=False)])
def test_materialize_matches_a_real_fit(kw):
    X, y = _data(800)
    kw = dict(random_state=0, **kw)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        ref = LinearSVR(**kw).fit(X, y)
    isc = ref.intercept_scaling
    raw = np.concatenate([ref.coef_, np.atleast_1d(ref.intercept_) / isc if ref.fit_intercept else [0.0]])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        est = E.materialize_linsvr(LinearSVR(**kw), raw, ref.n_iter_, X.shape[1])
    assert np.abs(est.predict(X) - ref.predict(X)).max() <= 1e-12 * np.abs(ref.predict(X)).max()
    assert est.n_iter_ == ref.n_iter_ and type(est.n_iter_) is type(ref.n_iter_)
    assert est.coef_.shape == ref.coef_.shape and np.shape(est.intercept_) == np.shape(ref.intercept_)
    assert type(est.intercept_) is type(ref.intercept_)
    est2 = pickle.loads(pickle.dumps(est))
    np.testing.assert_array_equal(est2.predict(X), est.predict(X))
    assert abs(est.score(X, y) - ref.score(X, y)) <= 1e-12


def test_materialize_warns_at_max_iter():
    raw = np.zeros(33)
    with pytest.warns(ConvergenceWarning, match="Liblinear failed to converge"):
        E.materialize_linsvr(LinearSVR(max_iter=5), raw, 5, 32)
    with warnings.catch_warnings():
        warnings.simplefilter("error", ConvergenceWarning)
        E.materialize_linsvr(LinearSVR(max_iter=5), raw, 4, 32)
