"""The evaluate loop every plan shares (no GPU): one engine call per group of candidates in order of first appearance, the
scatter of every call's outputs into its candidates' rows, the summed profile, the class weights per group and their reset,
and the fits that fail (SGD / SAG non-finite, SAG step_size * alpha_scaled == 1, k-NN n_neighbors > training rows)."""
import numpy as np
import pytest
from sklearn.linear_model import ElasticNet, Lasso, LogisticRegression, Ridge, SGDClassifier, SGDRegressor
from sklearn.model_selection import KFold
from sklearn.neighbors import KNeighborsClassifier, KNeighborsRegressor
from sklearn.pipeline import Pipeline
from sklearn.svm import SVC, SVR, LinearSVC, LinearSVR, NuSVC, NuSVR

from spark_sklearn_b200 import estimators as E

SEARCHES = ("svc", "svr", "ridge", "enet", "logreg", "linsvc", "linsvr", "sgd", "logreg_sag", "knn")


class FakeEngine:
    """Records every call; a search call answers distinct values for each of its fits, status 2 where fail says so."""

    def __init__(self):
        self.calls, self.outs, self.cw, self.fail = [], [], [], set()
        self.n_splits = self.n_classes = 0

    def set_data(self, X, fold_id, n_splits, y_class=None, y_target=None):
        self.n_splits = n_splits
        self.n_classes = 0 if y_class is None else int(np.max(y_class)) + 1

    def set_splits(self, te, tr, n_splits):
        self.n_splits = n_splits

    def set_targets_f64(self, y):
        pass

    def set_train_order(self, rows=None):
        pass

    def set_sample_weight(self, w=None):
        pass

    def set_class_weight(self, w=None):
        self.cw.append(None if w is None else np.array(w))

    def set_scoring(self, kind=0, pos_class=1):
        self.calls.append(("set_scoring", (kind, pos_class), {}))

    def profile(self):
        c = sum(name in SEARCHES for name, _, _ in self.calls)
        return {"launches": 10 * c, "ms_total": 0.5 * c}

    def __getattr__(self, name):
        if name not in SEARCHES:
            raise AttributeError(name)

        def search(*args, **kw):
            self.calls.append((name, args, kw))
            c = len(self.outs) + 1
            n = len(args[0])
            base = 1000.0 * c + 10 * np.arange(n)[:, None] + np.arange(self.n_splits)[None, :]
            out = dict(test=base, train=base + 0.5 if kw.get("return_train", True) else None,
                       fit_ms=(base + 0.25).astype(np.float32), score_ms=(base + 0.75).astype(np.float32),
                       n_iter=base.astype(np.int32))
            if name in ("sgd", "logreg_sag"):
                out["status"] = np.array([[2 if (c, j, k) in self.fail else 0 for k in range(self.n_splits)] for j in range(n)],
                                         np.int32)
            if kw.get("return_stats"):
                kc = self.n_classes if name == "sgd" and self.n_classes > 2 else 1
                key, tail = ("cd_stats", (3,)) if name == "linsvr" else ("stats", (kc, 3) if name == "sgd" else (2,))
                out[key] = np.broadcast_to(base.astype(np.int64).reshape(base.shape + (1,) * len(tail)), base.shape + tail).copy()
            self.outs.append(out)
            return out
        return search

    def searches(self):
        return [(name, args, kw) for name, args, kw in self.calls if name in SEARCHES]


@pytest.fixture
def fake(monkeypatch):
    eng = FakeEngine()
    monkeypatch.setattr(E, "get_engine", lambda device=None: eng)
    return eng


RNG = np.random.RandomState(0)
X = RNG.randn(80, 4)
Y2 = (X[:, 0] > 0).astype(int)
YR = X @ RNG.randn(4)
NS = 4

# name -> (estimator, y, the per-candidate value checked in each call (from its arguments), candidates A1, B, A2 whose
# value is 1, 2, 3; B differs from the As in a setting the group key holds)
CASES = {
    "SVC": (SVC(), Y2, lambda a: a[1], [{"C": 1.0}, {"C": 2.0, "tol": 1e-2}, {"C": 3.0}]),
    "NuSVC": (NuSVC(), Y2, lambda a: [10 * v for v in a[1]], [{"nu": 0.1}, {"nu": 0.2, "shrinking": False}, {"nu": 0.3}]),
    "SVR": (SVR(), YR, lambda a: a[1], [{"C": 1.0}, {"C": 2.0, "max_iter": 50}, {"C": 3.0}]),
    "NuSVR": (NuSVR(), YR, lambda a: [10 * v for v in a[2]], [{"nu": 0.1}, {"nu": 0.2, "tol": 1e-2}, {"nu": 0.3}]),
    "Ridge": (Ridge(), YR, lambda a: a[0], [{"alpha": 1.0}, {"alpha": 2.0, "fit_intercept": False}, {"alpha": 3.0}]),
    "Lasso": (Lasso(), YR, lambda a: a[0], [{"alpha": 1.0}, {"alpha": 2.0, "max_iter": 50}, {"alpha": 3.0}]),
    "ElasticNet": (ElasticNet(), YR, lambda a: a[0], [{"alpha": 1.0}, {"alpha": 2.0, "tol": 1e-2}, {"alpha": 3.0}]),
    "LogisticRegression": (LogisticRegression(), Y2, lambda a: a[0],
                           [{"C": 1.0}, {"C": 2.0, "fit_intercept": False}, {"C": 3.0}]),
    "LogisticRegression-saga": (LogisticRegression(solver="saga", random_state=0), Y2, lambda a: 1.0 / (a[1][:, 0] * 60),
                                [{"C": 1.0}, {"C": 2.0, "tol": 1e-2}, {"C": 3.0}]),
    "LinearSVC": (LinearSVC(), Y2, lambda a: a[0], [{"C": 1.0}, {"C": 2.0, "intercept_scaling": 2.0}, {"C": 3.0}]),
    "LinearSVR": (LinearSVR(random_state=0), YR, lambda a: a[0], [{"C": 1.0}, {"C": 2.0, "fit_intercept": False}, {"C": 3.0}]),
    "SGDClassifier": (SGDClassifier(random_state=0), Y2, lambda a: [1e4 * v for v in a[2]],
                      [{"alpha": 1e-4}, {"alpha": 2e-4, "shuffle": False}, {"alpha": 3e-4}]),
    "SGDRegressor": (SGDRegressor(random_state=0), YR, lambda a: [1e4 * v for v in a[2]],
                     [{"alpha": 1e-4}, {"alpha": 2e-4, "tol": None}, {"alpha": 3e-4}]),
    "KNeighborsClassifier": (KNeighborsClassifier(), Y2, lambda a: a[0],
                             [{"n_neighbors": 1}, {"n_neighbors": 2, "weights": "distance"}, {"n_neighbors": 3}]),
    "KNeighborsRegressor": (KNeighborsRegressor(), YR, lambda a: a[0],
                            [{"n_neighbors": 1}, {"n_neighbors": 2, "p": 1}, {"n_neighbors": 3}]),
    "Pipeline": (Pipeline([("m", SVC())]), Y2, lambda a: a[1], [{"m__C": 1.0}, {"m__C": 2.0, "m__tol": 1e-2}, {"m__C": 3.0}]),
}
CLASS_WEIGHTED = {"SVC", "NuSVC", "LogisticRegression", "LogisticRegression-saga", "LinearSVC", "SGDClassifier", "Pipeline"}


def _plan(est, cands, y):
    splits = list(KFold(NS).split(X, y))
    return E.adapter_for(est).plan(est, cands, X, y, E.Folds(splits, len(X)), NS)


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("return_train", [True, False])
def test_one_call_per_group_and_every_output_in_its_row(fake, name, return_train):
    est, y, value, cands = CASES[name]
    plan = _plan(est, cands, y)
    r = plan.evaluate([0, 1, 2], return_train=return_train, error_score=np.nan)
    calls = fake.searches()
    knn = name.startswith("KNeighbors")
    groups = [[0, 1, 2]] if knn else [[0, 2], [1]]                 # k-NN: one selection shared by every candidate
    assert len(calls) == len(groups)
    assert [c[0] for c in fake.calls].count("set_scoring") == len(groups)
    for (_, args, kw), rows, out in zip(calls, groups, fake.outs):
        np.testing.assert_allclose(value(args), [j + 1 for j in rows])
        assert kw.get("return_train", True) == return_train
        np.testing.assert_array_equal(r["test"][rows], out["test"])
        np.testing.assert_array_equal(r["fit_time"][rows], np.asarray(out["fit_ms"], np.float64) * 1e-3)
        np.testing.assert_array_equal(r["score_time"][rows], np.asarray(out["score_ms"], np.float64) * 1e-3)
        if return_train:
            np.testing.assert_array_equal(r["train"][rows], out["train"])
        if hasattr(plan, "n_iter_"):
            np.testing.assert_array_equal(plan.n_iter_[rows], out["n_iter"])
        for key in ("stats", "cd_stats"):
            if key in out:
                np.testing.assert_array_equal(getattr(plan, key + "_")[rows], out[key])
    assert r["train"] is None or return_train
    assert plan.profile() == {"launches": sum(10 * c for c in range(1, len(groups) + 1)),
                              "ms_total": sum(0.5 * c for c in range(1, len(groups) + 1))}


@pytest.mark.parametrize("name", sorted(CASES))
def test_class_weights_once_per_group_then_reset(fake, name):
    est, y, value, cands = CASES[name]
    weighted = name in CLASS_WEIGHTED
    if weighted:                                                  # A1 and A2 balanced, B unweighted: still two groups
        cw = {("m__" if name == "Pipeline" else "") + "class_weight": "balanced"}
        cands = [dict(cands[0], **cw), cands[1], dict(cands[2], **cw)]
    _plan(est, cands, y).evaluate([0, 1, 2], error_score=np.nan)
    if not weighted:
        assert fake.cw == []
        return
    assert len(fake.searches()) == 2 and len(fake.cw) == 3
    assert fake.cw[0].shape == (NS, 2) and fake.cw[1] is None and fake.cw[2] is None


def test_class_weight_is_part_of_the_group_key(fake):
    cands = [{"C": 1.0}, {"C": 2.0, "class_weight": {0: 2.0, 1: 1.0}}, {"C": 3.0}, {"C": 4.0, "class_weight": {1: 1.0, 0: 2.0}}]
    _plan(LinearSVC(), cands, Y2).evaluate([0, 1, 2, 3])
    assert [list(args[0]) for _, args, _ in fake.searches()] == [[1.0, 3.0], [2.0, 4.0]]
    assert fake.cw[0] is None and (fake.cw[1][:, 0] == 2.0).all() and fake.cw[2] is None


@pytest.mark.parametrize("est,y", [(SGDClassifier(random_state=0), Y2), (SGDRegressor(random_state=0), YR),
                                   (LogisticRegression(solver="sag", random_state=0), Y2)])
def test_non_finite_fits(fake, est, y):
    plan = _plan(est, [{}, {"max_iter": 7}], y)
    fake.fail = {(2, 0, 3)}                                       # the second call's only candidate, split 3
    with pytest.warns(UserWarning, match="1 fits failed"):
        r = plan.evaluate([0, 1], error_score=-7.0)
    assert r["test"][1, 3] == -7.0 and r["train"][1, 3] == -7.0 and (r["test"][0] != -7.0).all()
    fake.outs.clear()
    with pytest.raises(ValueError, match="Floating-point under-/overflow occurred at epoch #%d" % (2000 + 3)):
        plan.evaluate([0, 1], error_score="raise")


def test_sag_zero_division_fits(fake, monkeypatch):
    plan = _plan(LogisticRegression(solver="saga", random_state=0), [{}, {"C": 2.0}], Y2)
    step = plan._step

    def zero_div_on_split_2(k, solver, alpha, beta, fit_intercept):
        if k == 2 and alpha == 0.5:
            raise ZeroDivisionError("Current sag implementation does not handle the case step_size * alpha_scaled == 1")
        return step(k, solver, alpha, beta, fit_intercept)
    monkeypatch.setattr(plan, "_step", zero_div_on_split_2)
    with pytest.raises(ZeroDivisionError):
        plan.evaluate([0, 1], error_score="raise")
    assert fake.searches() == []
    with pytest.warns(UserWarning, match="1 fits failed"):
        r = plan.evaluate([0, 1], error_score=np.nan)
    assert np.isnan(r["test"][1, 2]) and np.isfinite(np.delete(r["test"].ravel(), 1 * NS + 2)).all()


@pytest.mark.parametrize("est,y", [(KNeighborsClassifier(), Y2), (KNeighborsRegressor(), YR)])
def test_knn_too_many_neighbours(fake, est, y):
    plan = _plan(est, [{"n_neighbors": 3}, {"n_neighbors": 61}], y)   # 60 training rows per split
    with pytest.raises(ValueError, match="n_neighbors = 61, n_samples_fit = 60, n_samples = 20"):
        plan.evaluate([0, 1], error_score="raise")
    assert fake.searches() == []
    with pytest.warns(UserWarning, match="non-finite scores replaced by error_score=-1"):
        r = plan.evaluate([0, 1], error_score=-1.0)
    assert (r["test"][1] == -1.0).all() and (r["train"][1] == -1.0).all() and (r["test"][0] >= 1000).all()
