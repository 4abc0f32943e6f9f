"""Host-side logic of SVC with the poly and sigmoid kernels (no GPU): parameter checks, per-fold gamma, the degree / coef0
arrays handed to the engine, the engine's kernel-parameter setter calls, and cv_results_ of the reference's documented
grid through an oracle-backed plan."""
import numpy as np
import pytest
from sklearn.svm import SVC

from spark_sklearn_b200 import estimators as E
from spark_sklearn_b200 import workloads as W


class FakeEngine:
    """Records what a plan hands to the engine; returns zeros."""

    def __init__(self):
        self.calls = []
        self.n = self.n_splits = 0

    def set_data(self, X, fold_id, n_splits, y_class=None, y_target=None):
        self.n, self.n_splits = len(X), n_splits

    def set_splits(self, te, tr, n_splits):
        self.n_splits = n_splits

    def set_sample_weight(self, w=None):
        pass

    def set_class_weight(self, w=None):
        pass

    def set_scoring(self, kind=0, pos_class=1):
        pass

    def svc(self, kernel, C, gamma, tol=1e-3, max_iter=-1, shrinking=True, return_train=True, flags=0, degree=None, coef0=None):
        self.calls.append(dict(kernel=list(kernel), C=list(C), gamma=np.array(gamma), degree=degree, coef0=coef0))
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
    from sklearn.model_selection import StratifiedKFold
    splits = list(StratifiedKFold(cv).split(X, y))
    return E.SVCPlan.plan(est, cands, X, y, E.Folds(splits, len(X)), len(splits)), splits


def _data():
    w = W.make_workload("c2_small")
    return w["X"][:300], w["y"][:300]


def test_degree_coef0_and_per_fold_gamma_reach_the_engine(fake):
    X, y = _data()
    cands = [{"kernel": "poly", "degree": 2, "coef0": 1.0}, {"kernel": "sigmoid", "coef0": -0.5, "gamma": "scale"},
             {"kernel": "poly", "degree": 5, "gamma": 0.25}, {"kernel": "rbf", "gamma": "auto"}, {"kernel": "linear"}]
    plan, splits = _plan(SVC(), cands, X, y)
    plan.evaluate(list(range(len(cands))))
    (call,) = fake.calls
    assert call["kernel"] == ["poly", "sigmoid", "poly", "rbf", "linear"]
    assert list(call["degree"]) == [2, 3, 5, 3, 3] and list(call["coef0"]) == [1.0, -0.5, 0.0, 0.0, 0.0]
    scale = [1.0 / (X.shape[1] * np.asarray(X[tr], np.float64).var()) for tr, _ in splits]
    np.testing.assert_array_equal(call["gamma"][0], scale)          # 'scale' from each training fold, poly too
    np.testing.assert_array_equal(call["gamma"][1], scale)
    np.testing.assert_array_equal(call["gamma"][2], 0.25)
    np.testing.assert_array_equal(call["gamma"][3], 1.0 / X.shape[1])
    np.testing.assert_array_equal(call["gamma"][4], 0.0)
    assert len(set(scale)) > 1


@pytest.mark.parametrize("bad", [{"degree": -1}, {"degree": 2.0}, {"degree": "3"}, {"coef0": "1"}, {"coef0": None},
                                 {"kernel": "poly", "degree": 1.5}])
def test_bad_degree_or_coef0_raises_value_error(fake, bad):
    X, y = _data()
    plan, _ = _plan(SVC(kernel="poly"), [bad], X, y)
    with pytest.raises(ValueError):
        plan.evaluate([0])
    with pytest.raises(ValueError):
        SVC(**dict({"kernel": "poly"}, **bad)).fit(X, y)            # scikit-learn rejects the same values


def test_precomputed_callable_and_probability_still_raise(fake):
    X, y = _data()
    for cand in ({"kernel": "precomputed"}, {"kernel": lambda a, b: a @ b.T}, {"kernel": "poly", "probability": True}):
        plan, _ = _plan(SVC(), [cand], X, y)
        with pytest.raises(NotImplementedError):
            plan.evaluate([0])


class _FakeLib:
    """ctypes stand-in for libb200gs: records the calls of Engine.svc / svc_refit / debug_kernel_matrix"""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def f(*args):
            self.calls.append((name, args))
            return 0
        return f


def _engine():
    from spark_sklearn_b200.engine import Engine
    eng = Engine.__new__(Engine)
    eng._L, eng._h = _FakeLib(), None
    eng.n, eng.n_splits = 10, 2
    return eng


def test_engine_sets_kernel_params_only_for_poly_and_sigmoid():
    eng = _engine()
    eng.svc(["linear", "rbf"], [1.0, 2.0], [[0.0, 0.0], [0.5, 0.5]], degree=[2, 4], coef0=[1.0, 1.0])
    eng.svc_refit("rbf", 1.0, 0.5, 2, degree=2)
    eng.debug_kernel_matrix("linear", 0.0)
    assert [c[0] for c in eng._L.calls] == ["gs_svc", "gs_svc_refit", "gs_debug_kernel_matrix"]   # as before the two kernels

    eng = _engine()
    eng.svc(["poly", "rbf", "sigmoid"], [1.0, 2.0, 3.0], [0.5, 0.5, 0.5], degree=[2, 4, 3], coef0=[1.0, 0.0, -1.0])
    names = [c[0] for c in eng._L.calls]
    assert names == ["gs_set_kernel_params", "gs_svc", "gs_set_kernel_params"]
    assert eng._L.calls[0][1][3] == 3 and eng._L.calls[2][1][1:] == (None, None, 0)      # n = n_cand; then reset
    eng = _engine()
    eng.svc_refit("sigmoid", 1.0, 0.5, 2, coef0=0.5)
    eng.debug_kernel_matrix("poly", 0.5, degree=4, coef0=1.0)
    assert [c[0] for c in eng._L.calls] == ["gs_set_kernel_params", "gs_svc_refit", "gs_set_kernel_params",
                                            "gs_set_kernel_params", "gs_debug_kernel_matrix", "gs_set_kernel_params"]
    assert eng._L.calls[0][1][3] == 1


def test_engine_debug_kernel_matrix_guard_outputs():
    """debug_kernel_matrix asks for the float64 diagonal (poly / sigmoid only) and the guard flag only with return_guard"""
    eng = _engine()
    K = eng.debug_kernel_matrix("rbf", 0.5)
    assert K.shape == (10, 10)
    (name, args), = eng._L.calls
    assert name == "gs_debug_kernel_matrix" and len(args) == 6 and args[4:] == (None, None)
    for kernel, with_qd in (("rbf", False), ("linear", False), ("poly", True), ("sigmoid", True)):
        eng = _engine()
        K, qd, flag = eng.debug_kernel_matrix(kernel, 0.5, return_guard=True)
        (args,) = [a for name, a in eng._L.calls if name == "gs_debug_kernel_matrix"]
        assert (args[4] is not None) == with_qd and args[5] is not None, kernel
        assert K.shape == (10, 10) and flag == 0 and (qd.shape == (10,) if with_qd else qd is None), kernel


def test_engine_debug_score_and_decision_arguments():
    eng = _engine()
    eng.n_classes = 3
    for kind, shape, dtype in (("vote", (4, 4), np.int32), ("class_counts", (4, 2, 3, 3), np.int32),
                               ("auc_f64", (4, 4), np.uint64), ("auc_f32", (4, 4), np.uint64), ("rss", (4, 2), np.float64)):
        out = eng.debug_score(kind, np.zeros((3, 10)), np.zeros(3), [0, 0, 0, 0], [0, 1, 0, 1])
        assert out.shape == shape and out.dtype == dtype, kind
        name, args = eng._L.calls[-1]
        assert name == "gs_debug_score" and args[1] == eng.SCORE_KINDS[kind] and args[4] == 3 and args[7] == 4
    with pytest.raises(ValueError):
        eng.debug_score("vote", np.zeros((3, 10)), np.zeros(3), [0, 0], [0])
    with pytest.raises(ValueError):
        eng.debug_score("vote", np.zeros((3, 9)), np.zeros(3), [0], [0])
    dec, used = eng.debug_decision("poly", 0.5, np.zeros((5, 10)), degree=4, coef0=-1.0, jchunks=3)
    name, args = eng._L.calls[-1]
    assert name == "gs_debug_decision" and dec.shape == (5, 10) and args[1:5] == (2, 0.5, 4, -1.0) and args[6:8] == (5, 3)
    with pytest.raises(ValueError):
        eng.debug_decision("rbf", 0.5, np.zeros((5, 9)))


def test_randomized_search_over_degree(fake):
    from scipy.stats import randint
    from sklearn.model_selection import ParameterSampler
    from spark_sklearn_b200 import RandomizedSearchCV
    X, y = _data()
    dist = {"degree": randint(1, 5), "C": [0.5, 5.0], "coef0": [0.0, 1.0]}
    r = RandomizedSearchCV(None, SVC(kernel="poly"), dist, n_iter=6, random_state=0, cv=3, refit=False).fit(X, y)
    want = list(ParameterSampler(dist, 6, random_state=0))
    assert r.cv_results_["params"] == want
    assert list(fake.calls[0]["degree"]) == [c["degree"] for c in want]
    assert list(r.cv_results_["param_degree"]) == [c["degree"] for c in want]


# ------------------------------------------------------------------ oracle-backed plan ------------
class KernelOraclePlan:
    """poly / sigmoid through tests/svc_kernels_oracle.c, linear / rbf through oracle/svc_oracle.c"""

    def __init__(self, estimator, cands, X, y, fold_id, n_splits):
        self.estimator, self.cands, self.X, self.y = estimator, cands, np.asarray(X, np.float64), np.asarray(y)
        self.fold_id, self.n_splits = getattr(fold_id, "fold_id", fold_id), n_splits

    def evaluate(self, my, return_train=True, error_score="raise"):
        import svc_kernels_oracle as KO
        from oracle import oracle as O
        S = KO.gram_ddot(self.X)
        rows = np.arange(len(self.y))
        test, train = np.zeros((len(my), self.n_splits)), np.zeros((len(my), self.n_splits))
        for j, ci in enumerate(my):
            p = dict(self.estimator.get_params(), **self.cands[ci])
            if p["kernel"] in ("linear", "rbf"):
                te, tr, _ = O.cv_scores_svc(self.X, self.y, self.fold_id, self.n_splits, [self.cands[ci]], self.estimator.get_params())
                test[j], train[j] = te[0], tr[0]
                continue
            for k in range(self.n_splits):
                a, b = rows[self.fold_id != k], rows[self.fold_id == k]
                m = KO.KernelSVCModel(self.X, S, self.y, a, kernel=p["kernel"], gamma=p["gamma"], C=p["C"], degree=p["degree"],
                                      coef0=p["coef0"])
                test[j, k], train[j, k] = np.mean(m.predict(b) == self.y[b]), np.mean(m.predict(a) == self.y[a])
        z = np.zeros_like(test)
        return dict(test=test, train=train if return_train else None, fit_time=z + 1e-3, score_time=z + 1e-4)

    def profile(self):
        return {}

    def costs(self):
        return None

    def close(self):
        pass


def test_reference_docstring_grid_cv_results(monkeypatch):
    """The reference's cv_results_ example grid (grid_search.py:120-160): masked param_degree / param_gamma and every split
    score equal scikit-learn's GridSearchCV."""
    from sklearn.datasets import load_iris
    from sklearn.model_selection import GridSearchCV as SkGrid
    from spark_sklearn_b200 import GridSearchCV, base_search

    class Adapter:
        plan = staticmethod(lambda *a: KernelOraclePlan(*a))
    monkeypatch.setattr(base_search._est, "adapter_for", lambda est: Adapter)
    X, y = load_iris(return_X_y=True)
    grid = [{"kernel": ["poly"], "degree": [2, 3]}, {"kernel": ["rbf"], "gamma": [0.1, 0.2]}]
    a = GridSearchCV(None, SVC(gamma="auto"), grid, cv=5, refit=False).fit(X, y)
    b = SkGrid(SVC(gamma="auto"), grid, cv=5, return_train_score=True).fit(X, y)
    for key in ("param_kernel", "param_degree", "param_gamma"):
        ma, mb = a.cv_results_[key], b.cv_results_[key]
        np.testing.assert_array_equal(np.ma.getmaskarray(ma), np.ma.getmaskarray(mb), err_msg=key)
        assert list(ma.compressed()) == list(mb.compressed()), key
    assert a.cv_results_["params"] == b.cv_results_["params"]
    for k in range(5):
        for part in ("test", "train"):
            key = "split%d_%s_score" % (k, part)
            np.testing.assert_array_equal(a.cv_results_[key], b.cv_results_[key], err_msg=key)
    np.testing.assert_array_equal(a.cv_results_["rank_test_score"], b.cv_results_["rank_test_score"])
