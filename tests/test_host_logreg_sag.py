"""Host-side logic of LogisticRegression(solver='sag' | 'saga') (no GPU): routing between the lbfgs and SAG plans, scikit-learn's
ValueErrors before any device work, the per-split step size and scaled penalties, the seeds (and numpy's global RandomState
after a random_state=None search), X's dtype, sparse X, and the refit's fitted estimator."""
import pickle
import warnings

import numpy as np
import pytest
from sklearn.exceptions import ConvergenceWarning
from sklearn.linear_model import LogisticRegression
from sklearn.model_selection import KFold

from spark_sklearn_b200 import estimators as E

INT_MAX = np.iinfo(np.int32).max


class FakeEngine:
    """Records what a plan hands to the engine; returns zeros (the refit: refit_coef when set)."""

    def __init__(self):
        self.calls = []
        self.n = self.d = self.n_splits = self.n_classes = 0
        self.refit_coef, self.refit_iter = None, 4

    def set_data(self, X, fold_id, n_splits, y_class=None, y_target=None):
        self.n, self.d, self.n_splits = X.shape[0], X.shape[1], n_splits
        self.n_classes = 0 if y_class is None else int(np.max(y_class)) + 1
        self.X = np.array(X)

    def set_splits(self, te, tr, n_splits):
        self.n_splits = n_splits

    def set_train_order(self, rows=None):
        self.order = rows

    def set_sample_weight(self, w=None):
        pass

    def set_class_weight(self, w=None):
        pass

    def set_scoring(self, kind=0, pos_class=1):
        pass

    def logreg(self, C, **kw):
        self.calls.append(dict(lbfgs=True, C=list(C), **kw))
        shape = (len(C), self.n_splits)
        return dict(test=np.zeros(shape), train=np.zeros(shape), n_iter=np.ones(shape, np.int32),
                    fit_ms=np.zeros(shape, np.float32), score_ms=np.zeros(shape, np.float32))

    def logreg_sag(self, solver, alpha_scaled, beta_scaled, step, seed, loss, **kw):
        self.calls.append(dict(solver=np.array(solver), alpha=np.array(alpha_scaled), beta=np.array(beta_scaled),
                               step=np.array(step), seed=np.array(seed), loss=loss, **kw))
        shape = np.array(solver).shape
        return dict(test=np.zeros(shape), train=np.zeros(shape), n_iter=np.ones(shape, np.int32),
                    status=np.zeros(shape, np.int32), fit_ms=np.zeros(shape, np.float32), score_ms=np.zeros(shape, np.float32),
                    stats=np.zeros(shape + (2,), np.int64))

    def logreg_sag_refit(self, solver, alpha_scaled, beta_scaled, step, seed, loss, **kw):
        self.calls.append(dict(refit=True, solver=solver, alpha=alpha_scaled, beta=beta_scaled, step=step, seed=seed, loss=loss, **kw))
        k = self.n_classes if loss == "multinomial" else 1
        coef = np.zeros((k, self.d + 1)) if self.refit_coef is None else self.refit_coef
        return coef, self.refit_iter, 0

    def profile(self):
        return {}


@pytest.fixture
def fake(monkeypatch):
    eng = FakeEngine()
    monkeypatch.setattr(E, "get_engine", lambda device=None: eng)
    return eng


RNG = np.random.RandomState(0)
X = RNG.randn(120, 6)
Y2 = (X[:, 0] + 0.3 * RNG.randn(120) > 0).astype(int)
Y3 = RNG.randint(0, 3, 120)


def _plan(est, cands, y, X=X, cv=None):
    splits = list((cv or KFold(4, shuffle=True, random_state=0)).split(X, y))
    return E.adapter_for(est).plan(est, cands, X, y, E.Folds(splits, len(X)), len(splits)), splits


def test_routing(fake):
    with pytest.warns(UserWarning, match="float32"):
        plan, _ = _plan(LogisticRegression(), [{"C": 1.0}, {"C": 0.1}], Y2)
    assert type(plan) is E.LogRegPlan
    plan.evaluate([0, 1])
    assert fake.calls[-1]["lbfgs"] and fake.calls[-1]["C"] == [1.0, 0.1]
    with warnings.catch_warnings():
        warnings.simplefilter("error")                  # float64 X stays float64: no rounding warning
        plan, _ = _plan(LogisticRegression(solver="saga"), [{"C": 1.0}], Y2)
    assert type(plan) is E.LogRegSAGPlan and plan.X.dtype == np.float64
    plan, _ = _plan(LogisticRegression(), [{"solver": "sag"}, {"solver": "saga", "l1_ratio": 0.5}], Y3)
    assert type(plan) is E.LogRegSAGPlan
    plan.evaluate([0, 1])
    assert fake.calls[-1]["loss"] == "multinomial" and fake.calls[-1]["solver"].tolist() == [[0] * 4, [1] * 4]
    n_calls = len(fake.calls)
    with pytest.raises(NotImplementedError, match="mixes"):
        _plan(LogisticRegression(), [{"solver": "lbfgs"}, {"solver": "saga"}], Y2)
    assert len(fake.calls) == n_calls
    plan, _ = _plan(LogisticRegression(solver="newton-cg"), [{}], Y2)
    with pytest.raises(NotImplementedError, match="lbfgs does"):
        plan.evaluate([0])


@pytest.mark.parametrize("cand,match", [({"solver": "sag", "l1_ratio": 0.5}, "supports only 'l2' or None"),
                                        ({"C": -1.0}, "C"), ({"dual": True}, "dual=False"),
                                        ({"penalty": "elasticnet", "l1_ratio": None, "solver": "saga"}, "l1_ratio must")])
def test_sklearn_value_errors_before_device_work(fake, cand, match):
    plan, _ = _plan(LogisticRegression(solver="saga"), [cand], Y2)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", FutureWarning)
        with pytest.raises(ValueError, match=match):
            plan.evaluate([0])
    assert not fake.calls


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("y", [Y2, Y3])
def test_step_and_penalties_per_split(fake, dtype, y):
    from sklearn.linear_model._sag import get_auto_step_size
    from sklearn.utils.extmath import row_norms
    Xd = X.astype(dtype)
    cands = [{"C": 0.5, "l1_ratio": 0.25}, {"C": np.inf}, {"C": 2.0, "l1_ratio": 1.0}, {"C": 3.0, "solver": "sag"}]
    plan, splits = _plan(LogisticRegression(solver="saga", fit_intercept=False), cands, y, X=Xd)
    assert plan.X.dtype == dtype
    plan.evaluate([0, 1, 2, 3])
    c = fake.calls[-1]
    loss = "log" if len(set(y)) == 2 else "multinomial"
    for j, p in enumerate(cands):
        C, l1 = p["C"], p.get("l1_ratio", 0.0)
        alpha, beta = ((0.0, 1.0 / C) if l1 == 1 else ((1.0 / C, 0.0) if l1 == 0 else ((1 / C) * (1 - l1), (1 / C) * l1)))
        for k, (tr, _) in enumerate(splits):
            n = len(tr)
            step = get_auto_step_size(row_norms(Xd[tr], squared=True).max(), alpha / n, loss, False, n_samples=n,
                                      is_saga=p.get("solver", "saga") == "saga")
            assert c["step"][j, k] == step and c["alpha"][j, k] == alpha / n and c["beta"][j, k] == beta / n


def test_seeds_and_global_random_state(fake):
    plan, _ = _plan(LogisticRegression(solver="saga", random_state=3), [{"C": 1.0}, {"C": 2.0}], Y2)
    plan.evaluate([0, 1])
    assert (fake.calls[-1]["seed"] == np.random.RandomState(3).randint(1, INT_MAX)).all()
    # random_state=None: one draw per fit from numpy's global RandomState, candidate-major, the refit last
    np.random.seed(11)
    plan, _ = _plan(LogisticRegression(solver="sag"), [{"C": 1.0}, {"C": 2.0}], Y2)
    plan.evaluate([0, 1])
    plan.refit({"C": 1.0})
    got = np.random.randint(1 << 30)
    np.random.seed(11)
    want = [np.random.randint(1, INT_MAX) for _ in range(9)]
    assert fake.calls[-2]["seed"].ravel().tolist() == want[:8] and fake.calls[-1]["seed"] == want[8]
    assert got == np.random.randint(1 << 30)
    from sklearn.model_selection import GridSearchCV as SkGrid
    np.random.seed(11)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        SkGrid(LogisticRegression(solver="sag", max_iter=3), {"C": [1.0, 2.0]}, cv=KFold(4, shuffle=True, random_state=0)).fit(X, Y2)
    assert got == np.random.randint(1 << 30)                  # scikit-learn's own search leaves the same global state


def test_sparse_x_rejected(fake):
    import scipy.sparse as sp
    est = LogisticRegression(solver="saga")
    splits = list(KFold(3).split(X))
    with pytest.raises(NotImplementedError, match="sparse"):
        E.adapter_for(est).plan(est, [{}], sp.csr_matrix(X), Y2, E.Folds(splits, len(X)), 3)


def test_zero_division_and_error_score(fake):
    plan, _ = _plan(LogisticRegression(solver="sag"), [{"C": 1.0}], Y2)
    plan._step = lambda *a, **k: (_ for _ in ()).throw(ZeroDivisionError("step_size * alpha_scaled == 1"))
    with pytest.raises(ZeroDivisionError):
        plan.evaluate([0], error_score='raise')
    with pytest.warns(UserWarning, match="fits failed"):
        r = plan.evaluate([0], error_score=-1.0)
    assert (r["test"] == -1.0).all()


@pytest.mark.parametrize("y", [Y2, Y3])
def test_refit_materializes_a_logistic_regression(fake, y):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        real = LogisticRegression(solver="saga", l1_ratio=0.5, C=0.7, max_iter=300, random_state=0).fit(X, y)
    k = real.coef_.shape[0]
    fake.refit_coef = np.concatenate([real.coef_, real.intercept_[:, None]], 1)
    fake.refit_iter = int(real.n_iter_[0])
    plan, _ = _plan(LogisticRegression(solver="saga", max_iter=300, random_state=0), [{"C": 0.7, "l1_ratio": 0.5}], y)
    est = plan.refit({"C": 0.7, "l1_ratio": 0.5})
    assert type(est) is LogisticRegression and est.coef_.shape == (k, X.shape[1])
    np.testing.assert_array_equal(est.classes_, real.classes_)
    np.testing.assert_array_equal(est.n_iter_, real.n_iter_)
    assert est.n_iter_.dtype == real.n_iter_.dtype and est.n_features_in_ == real.n_features_in_
    for m in ("predict", "predict_proba", "decision_function"):
        np.testing.assert_array_equal(getattr(est, m)(X), getattr(real, m)(X))
    np.testing.assert_array_equal(pickle.loads(pickle.dumps(est)).predict_proba(X), real.predict_proba(X))
    fake.refit_iter = 300
    with pytest.warns(ConvergenceWarning, match="max_iter was reached"):
        plan.refit({"C": 0.7, "l1_ratio": 0.5})


def test_pipeline(fake):
    from sklearn.pipeline import Pipeline
    pipe = Pipeline([("lr", LogisticRegression(solver="saga"))])
    plan, _ = _plan(pipe, [{"lr__C": 1.0, "lr__l1_ratio": 0.5}], Y2)
    plan.evaluate([0])
    assert fake.calls[-1]["loss"] == "log"
    fitted = plan.refit({"lr__C": 1.0, "lr__l1_ratio": 0.5})
    assert type(fitted) is Pipeline and fitted.steps[0][1].coef_.shape == (1, X.shape[1])
