"""Host-side logic of SGDClassifier / SGDRegressor (no GPU): the seeds handed to the engine for int / RandomState / None in
scikit-learn's draw orders, the training order, class weights per fold, the parameter checks, grouping, the refit's fitted
estimator and the one-step Pipeline."""
import warnings

import numpy as np
import pytest
from sklearn.exceptions import ConvergenceWarning
from sklearn.linear_model import SGDClassifier, SGDRegressor
from sklearn.model_selection import KFold, ShuffleSplit

from spark_sklearn_b200 import estimators as E

INT_MAX = np.iinfo(np.int32).max


class FakeEngine:
    """Records what a plan hands to the engine; returns zeros (refit weights: refit_coef when set)."""

    def __init__(self):
        self.calls, self.cw, self.order = [], [], None
        self.n = self.d = self.n_splits = self.n_classes = 0
        self.refit_coef, self.refit_iter, self.refit_status = None, 4, 0

    def set_data(self, X, fold_id, n_splits, y_class=None, y_target=None):
        self.n, self.d, self.n_splits = X.shape[0], X.shape[1], n_splits
        self.n_classes = 0 if y_class is None else int(np.max(y_class)) + 1
        self.X = np.array(X)

    def set_splits(self, te, tr, n_splits):
        self.n_splits = n_splits

    def set_targets_f64(self, y):
        pass

    def set_train_order(self, rows=None):
        self.order = None if rows is None else [np.array(r) for r in rows]

    def set_sample_weight(self, w=None):
        pass

    def set_class_weight(self, w=None):
        self.cw.append(None if w is None else np.array(w))

    def set_scoring(self, kind=0, pos_class=1):
        pass

    def _kc(self):
        return self.n_classes if self.n_classes > 2 else 1

    def sgd(self, loss, penalty, alpha, l1_ratio, epsilon, learning_rate, eta0, power_t, seed, tol=1e-3, max_iter=1000,
            n_iter_no_change=5, fit_intercept=True, shuffle=True, return_train=True, return_coef=False, return_stats=False):
        self.calls.append(dict(loss=list(loss), penalty=list(penalty), alpha=list(alpha), seed=np.array(seed), tol=tol,
                               max_iter=max_iter, shuffle=shuffle))
        shape = (len(loss), self.n_splits)
        return dict(test=np.zeros(shape), train=np.zeros(shape), n_iter=np.ones(shape, np.int32),
                    status=np.zeros(shape, np.int32), fit_ms=np.zeros(shape, np.float32), score_ms=np.zeros(shape, np.float32),
                    stats=np.zeros(shape + (self._kc(), 3), np.int64))

    def sgd_refit(self, loss, penalty, alpha, l1_ratio, epsilon, learning_rate, eta0, power_t, seed, **kw):
        self.calls.append(dict(refit=True, seed=list(seed), **kw))
        kc = self._kc()
        coef = np.zeros((kc, self.d + 1)) if self.refit_coef is None else self.refit_coef
        return coef, np.full(kc, self.refit_iter, np.int32), np.full(kc, self.refit_status, np.int32)

    def profile(self):
        return {}


@pytest.fixture
def fake(monkeypatch):
    eng = FakeEngine()
    monkeypatch.setattr(E, "get_engine", lambda device=None: eng)
    return eng


RNG = np.random.RandomState(0)
X = RNG.randn(120, 6)
Y2 = (X[:, 0] > 0).astype(int)
Y3 = RNG.randint(0, 3, 120)
YR = X @ RNG.randn(6)


def _plan(est, cands, y, cv=None, X=X):
    splits = list((cv or KFold(4)).split(X, y))
    adapter = E.adapter_for(est)
    return adapter.plan(est, cands, X, y, E.Folds(splits, len(X)), len(splits)), splits


def test_adapters(fake):
    from sklearn.pipeline import Pipeline
    assert E.adapter_for(SGDClassifier()) is E.SGDPlan and E.SGDPlan.multi_device
    assert E.adapter_for(SGDRegressor()) is E.SGDRegressorPlan
    assert E.SGDRegressorPlan.scorers is E.REGRESSION_SCORERS and E.SGDPlan.scorers is E.CLASSIFICATION_SCORERS
    assert isinstance(E.adapter_for(Pipeline([("s", SGDClassifier())])), E.PipelineAdapter)


@pytest.mark.parametrize("y,kc", [(Y2, 2), (Y3, 3), (YR, 0)])
def test_seeds_int_and_randomstate(fake, y, kc):
    est = SGDClassifier(random_state=3) if kc else SGDRegressor(random_state=3)
    plan, _ = _plan(est, [{"alpha": 1e-4}, {"alpha": 1e-3}], y)
    plan.evaluate([0, 1])
    seed = fake.calls[0]["seed"]
    rs = np.random.RandomState(3)
    if kc == 0:
        want = [rs.randint(0, INT_MAX)]
    elif kc == 2:
        rs.randint(1, INT_MAX)
        want = [rs.randint(INT_MAX)]
    else:
        want = []
        for s in rs.randint(INT_MAX, size=kc):
            r = np.random.RandomState(s)
            r.randint(1, INT_MAX)
            want.append(r.randint(INT_MAX))
    assert seed.shape == (2, 4, max(kc, 2) if kc > 2 else 1)
    assert (seed == np.array(want)).all()
    state = np.random.RandomState(3)
    plan, _ = _plan(SGDClassifier(random_state=state) if kc else SGDRegressor(random_state=state), [{}], y)
    plan.evaluate([0])
    assert (fake.calls[-1]["seed"] == np.array(want)).all()
    assert state.randint(INT_MAX) == np.random.RandomState(3).randint(INT_MAX)      # the caller's state is not advanced


def test_seeds_none_follow_the_global_draws(fake):
    """random_state=None: candidate-major, split-minor from numpy's global RandomState, refit last -- the regressor's fit
    draws twice (shuffle seed, then make_dataset's)"""
    np.random.seed(11)
    plan, _ = _plan(SGDRegressor(), [{"alpha": 1e-4}, {"alpha": 1e-3}], YR)
    plan.evaluate([0, 1])
    plan.refit({"alpha": 1e-4})
    np.random.seed(11)
    want = []
    for _ in range(2 * 4 + 1):
        want.append(np.random.randint(0, INT_MAX))
        np.random.randint(1, INT_MAX)
    assert list(fake.calls[0]["seed"].ravel()) == want[:8]
    assert fake.calls[1]["seed"] == [want[8]]


def test_train_order_for_shufflesplit(fake):
    cv = ShuffleSplit(3, test_size=0.3, random_state=0)
    plan, splits = _plan(SGDClassifier(), [{}], Y2, cv=cv)
    for got, (tr, _) in zip(fake.order, splits):
        np.testing.assert_array_equal(got, tr)


def test_balanced_class_weight_per_fold_without_sample_weight(fake):
    from sklearn.utils.class_weight import compute_class_weight
    plan, splits = _plan(SGDClassifier(class_weight="balanced"), [{}], Y3)
    plan.set_fit_params({"sample_weight": np.linspace(0.1, 2.0, len(X))})
    plan.evaluate([0])
    w = fake.cw[0]
    for k, (tr, _) in enumerate(splits):
        np.testing.assert_array_equal(w[k], compute_class_weight("balanced", classes=np.arange(3), y=Y3[tr]))


def test_grouping(fake):
    cands = [{"alpha": 1e-4}, {"alpha": 1e-3, "tol": None}, {"alpha": 1e-2}, {"alpha": 1e-1, "shuffle": False}]
    plan, _ = _plan(SGDClassifier(), cands, Y2)
    plan.evaluate([0, 1, 2, 3])
    assert [c["alpha"] for c in fake.calls] == [[1e-4, 1e-2], [1e-3], [1e-1]]
    assert fake.calls[1]["tol"] is None and fake.calls[2]["shuffle"] is False


@pytest.mark.parametrize("params,exc", [({"early_stopping": True}, NotImplementedError), ({"average": True}, NotImplementedError),
                                        ({"learning_rate": "pa1"}, NotImplementedError), ({"alpha": -1.0}, ValueError),
                                        ({"learning_rate": "optimal", "alpha": 0.0}, ValueError),
                                        ({"penalty": "elasticnet", "l1_ratio": None}, ValueError), ({"loss": "huber2"}, ValueError)])
def test_rejections(fake, params, exc):
    plan, _ = _plan(SGDClassifier(), [params], Y2)
    with pytest.raises(exc):
        plan.evaluate([0])


def test_too_many_features_and_sparse(fake):
    import scipy.sparse as sp
    with pytest.raises(NotImplementedError, match="512"):
        _plan(SGDClassifier(), [{}], Y2, X=np.zeros((120, 513)))
    with pytest.raises(NotImplementedError, match="sparse"):
        E.SGDPlan.plan(SGDClassifier(), [{}], sp.csr_matrix(X), Y2, None, 4)


def test_non_finite_fit(fake):
    plan, _ = _plan(SGDRegressor(), [{}], YR)
    fake.sgd = lambda *a, **k: dict(FakeEngine.sgd(fake, *a, **k), status=np.full((1, 4), 2, np.int32),
                                    n_iter=np.full((1, 4), 3, np.int32))
    with pytest.raises(ValueError, match="Floating-point under-/overflow occurred at epoch #3"):
        plan.evaluate([0], error_score="raise")
    with pytest.warns(UserWarning):
        r = plan.evaluate([0], error_score=-5.0)
    assert (r["test"] == -5.0).all()


@pytest.mark.parametrize("y,classifier", [(Y2, True), (Y3, True), (YR, False)])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_refit_materialises_the_estimator(fake, y, classifier, dtype):
    Xd = X.astype(dtype)
    est = SGDClassifier(random_state=0, max_iter=4) if classifier else SGDRegressor(random_state=0, max_iter=4)
    plan, _ = _plan(est, [{}], y, X=Xd)
    kc = 3 if classifier and len(np.unique(y)) == 3 else 1
    fake.refit_coef = np.arange(kc * 7, dtype=np.float64).reshape(kc, 7) / 7
    with pytest.warns(ConvergenceWarning, match="Maximum number of iteration"):
        fake.refit_iter = 4
        got = plan.refit({})
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        ref = type(est)(**est.get_params()).fit(Xd, y)
    for a in ("coef_", "intercept_"):
        assert getattr(got, a).shape == getattr(ref, a).shape and getattr(got, a).dtype == getattr(ref, a).dtype, a
    assert got.n_iter_ == 4 and got.t_ == 1.0 + 4 * len(X) and got.n_features_in_ == 6
    assert hasattr(got, "_loss_function_") == hasattr(ref, "_loss_function_")
    if classifier:
        assert type(got._loss_function_) is type(ref._loss_function_)
    if classifier:
        np.testing.assert_array_equal(got.classes_, ref.classes_)
        np.testing.assert_array_equal(got._expanded_class_weight, ref._expanded_class_weight)
    got.predict(Xd)


def test_pipeline_names(fake):
    from sklearn.pipeline import Pipeline
    pipe = Pipeline([("s", SGDClassifier(random_state=0))])
    ad = E.adapter_for(pipe)
    splits = list(KFold(4).split(X, Y2))
    plan = ad.plan(pipe, [{"s__alpha": 1e-3}], X, Y2, E.Folds(splits, len(X)), 4)
    plan.evaluate([0])
    assert fake.calls[0]["alpha"] == [1e-3]
    fitted = plan.refit({"s__alpha": 1e-3})
    assert fitted.steps[0][0] == "s" and fitted.steps[0][1].alpha == 1e-3
