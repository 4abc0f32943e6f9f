"""GPU tests of SVC with the poly and sigmoid kernels: kernel matrices against numpy on the GPU's own Gram, the
svc_kernels_mid golden (scikit-learn 1.9) on every solver instance, the reference's documented grid on iris, scorers,
splitters, class weights, a one-step Pipeline, refit and pickle, and the in-process multi-GPU scheduler."""
import pickle

import numpy as np
import pytest
from sklearn.svm import SVC

from conftest import golden
from spark_sklearn_b200 import workloads as W

pytestmark = pytest.mark.gpu


def _setup(engine, key):
    from oracle import oracle as O
    w = W.make_workload(key)
    fold_id, ns = O.folds_from_cv(w["cv"], w["X"], w["y"], True)
    classes, yc = np.unique(w["y"], return_inverse=True)
    engine.set_data(w["X"], fold_id, ns, y_class=yc.astype(np.int32))
    return w, fold_id, ns


def _powi(base, times):
    """libsvm's powi on arrays, every multiplication rounded on its own"""
    tmp, ret = base.copy(), np.ones_like(base)
    t = times
    while t > 0:
        if t % 2 == 1:
            ret = ret * tmp
        tmp = tmp * tmp
        t //= 2
    return ret


def test_kernel_matrices_against_numpy_on_the_gpu_gram(engine):
    _setup(engine, "c2_small")
    S, xsq = engine.debug_gram()
    for gamma, degree, coef0 in ((1 / 64, 3, 0.0), (1 / 64, 2, 1.0), (0.02, 5, -1.0), (0.5, 0, 1.0), (0.0, 3, 2.0)):
        K = engine.debug_kernel_matrix("poly", gamma, degree=degree, coef0=coef0)
        np.testing.assert_array_equal(K, _powi(gamma * S + coef0, degree).astype(np.float32), err_msg=str((gamma, degree, coef0)))
    for gamma, coef0 in ((1 / 64, 0.0), (1 / 64, -1.0), (0.1, 1.0)):
        K = engine.debug_kernel_matrix("sigmoid", gamma, coef0=coef0)
        ref = np.tanh(gamma * S + coef0).astype(np.float32)
        diff = K != ref
        # CUDA's float64 tanh and the host's differ in the last bit of a few values; after the float32 rounding that
        # moves at most a handful of entries by one float32 ulp
        assert diff.sum() <= 8, diff.sum()
        assert np.all(np.abs(K[diff] - ref[diff]) <= np.spacing(np.abs(ref[diff])))
    # the setter's values are read only by the call they were set for; rbf / linear are unchanged
    np.testing.assert_array_equal(engine.debug_kernel_matrix("linear", 0.0), S.astype(np.float32))


def _gammas(w, fold_id, ns, cands):
    X = w["X"]
    out = []
    for c in cands:
        g = c.get("gamma", w["est_params"].get("gamma", "scale"))
        if c["kernel"] == "linear":
            out.append([0.0] * ns)
        elif g == "scale":
            out.append([1.0 / (X.shape[1] * np.asarray(X[fold_id != k], np.float64).var()) for k in range(ns)])
        elif g == "auto":
            out.append([1.0 / X.shape[1]] * ns)
        else:
            out.append([float(g)] * ns)
    return np.array(out)


@pytest.mark.parametrize("mode", ["default", "cluster", "position"])
def test_kernel_golden_bitexact(engine, monkeypatch, mode):
    """svc_kernels_mid (3000x128, cv=5; poly, sigmoid, rbf, linear): split scores, iteration and support-vector counts
    identical to scikit-learn's, on the default schedule, with every problem on 4-CTA clusters, and on the
    position-owned single-CTA instance."""
    if mode == "cluster":
        monkeypatch.setenv("B200GS_SMO_CLUSTER", "4")
        monkeypatch.setenv("B200GS_SMO_CLUSTER_N", "100000")
    elif mode == "position":
        monkeypatch.setenv("B200GS_SMO_LEAN", "0")
    w, fold_id, ns = _setup(engine, "svc_kernels_mid")
    g = golden("svc_kernels_mid")
    cands = W.candidates(w)
    p = [dict(SVC().get_params(), **c) for c in cands]
    r = engine.svc([c["kernel"] for c in cands], [c["C"] for c in cands], _gammas(w, fold_id, ns, cands),
                   degree=[c["degree"] for c in p], coef0=[c["coef0"] for c in p])
    np.testing.assert_array_equal(r["n_iter"], g["n_iter"])
    np.testing.assert_array_equal(r["n_sv"], g["n_sv"])
    np.testing.assert_array_equal(r["test"], g["test_scores"])
    np.testing.assert_array_equal(r["train"], g["train_scores"])


def _compare_cv_results(a, b, atol_mean=4e-16):
    for key in b.cv_results_:
        if key.endswith("_time"):
            assert key in a.cv_results_
            continue
        x, y = a.cv_results_[key], b.cv_results_[key]
        if key == "params":
            assert x == y
        elif key.startswith("param_"):
            np.testing.assert_array_equal(np.ma.getmaskarray(x), np.ma.getmaskarray(y), err_msg=key)
            assert list(x.compressed()) == list(y.compressed()), key
        elif key.startswith(("mean_", "std_")):
            np.testing.assert_allclose(np.asarray(x, float), np.asarray(y, float), rtol=0, atol=atol_mean, err_msg=key)
        else:
            np.testing.assert_array_equal(np.asarray(x, float), np.asarray(y, float), err_msg=key)


def test_reference_docstring_grid_on_iris(engine):
    """The reference's cv_results_ example grid (grid_search.py:120-160) on iris with gamma='auto', three classes:
    cv_results_ key by key, the refit model's predictions and decision values, and pickle."""
    from sklearn.datasets import load_iris
    from sklearn.model_selection import GridSearchCV as SkGrid
    from spark_sklearn_b200 import GridSearchCV
    X, y = load_iris(return_X_y=True)
    grid = [{"kernel": ["poly"], "degree": [2, 3]}, {"kernel": ["rbf"], "gamma": [0.1, 0.2]}]
    a = GridSearchCV(None, SVC(gamma="auto"), grid, cv=5).fit(X, y)
    b = SkGrid(SVC(gamma="auto"), grid, cv=5, return_train_score=True).fit(X, y)
    _compare_cv_results(a, b)
    assert a.best_params_ == b.best_params_
    for kern, extra in (("poly", {"degree": 3, "coef0": 1.0, "C": 0.5}), ("sigmoid", {"coef0": -1.0, "C": 2.0}),
                        ("poly", {"degree": 2, "C": 3.0})):
        est = SVC(gamma="auto", kernel=kern, **extra)
        ga = GridSearchCV(None, est, {"C": [extra["C"]]}, cv=5).fit(X, y)
        ref = SVC(gamma="auto", kernel=kern, **extra).fit(X, y)
        got = ga.best_estimator_
        np.testing.assert_array_equal(got.predict(X), ref.predict(X))
        np.testing.assert_allclose(got.decision_function(X), ref.decision_function(X), rtol=0, atol=1e-12)
        np.testing.assert_array_equal(got.n_iter_, ref.n_iter_)
        np.testing.assert_array_equal(got.support_, ref.support_)
        back = pickle.loads(pickle.dumps(got))
        np.testing.assert_array_equal(back.predict(X), ref.predict(X))


class _AscendingRows:
    """A splitter's splits with the row indices sorted.  A fit on the device sees its training rows in ascending order;
    scikit-learn fits X[train] in the splitter's order, and libsvm's iterates depend on the order of the rows inside each
    class, so a shuffled training set can end one support vector apart (a one-row flip of a score).  Sorted splits make the
    two fits the same problem."""

    def __init__(self, cv):
        self.cv = cv

    def split(self, X, y=None, groups=None):
        for tr, te in self.cv.split(X, y, groups):
            yield np.sort(tr), np.sort(te)

    def get_n_splits(self, X=None, y=None, groups=None):
        return self.cv.get_n_splits(X, y, groups)


def test_scorer_splitter_class_weight_and_pipeline(engine):
    """roc_auc, ShuffleSplit (rows in neither set; training rows sorted, see _AscendingRows), class_weight='balanced' and a
    one-step Pipeline over a poly / sigmoid grid, against scikit-learn's GridSearchCV."""
    from sklearn.model_selection import GridSearchCV as SkGrid, ShuffleSplit
    from sklearn.pipeline import Pipeline
    from spark_sklearn_b200 import GridSearchCV
    w = W.make_workload("c2_mid")
    X, y = w["X"][:900], w["y"][:900].copy()
    y[:250] = 0                                                     # unbalanced classes
    grid = [{"kernel": ["poly"], "degree": [2, 3], "coef0": [0.0, 1.0], "C": [0.5, 4.0]},
            {"kernel": ["sigmoid"], "coef0": [-1.0, 0.0], "gamma": [1 / 512]}]
    for kw in (dict(scoring="roc_auc", cv=4), dict(cv=_AscendingRows(ShuffleSplit(4, test_size=0.25, random_state=7)))):
        a = GridSearchCV(None, SVC(), grid, **kw).fit(X, y)
        b = SkGrid(SVC(), grid, return_train_score=True, **kw).fit(X, y)
        for k in range(4):
            for part in ("test", "train"):
                key = "split%d_%s_score" % (k, part)
                np.testing.assert_allclose(a.cv_results_[key], b.cv_results_[key], rtol=0, atol=1e-12, err_msg=(key, kw))
        assert a.best_params_ == b.best_params_
    a = GridSearchCV(None, SVC(class_weight="balanced"), grid, cv=4).fit(X, y)
    b = SkGrid(SVC(class_weight="balanced"), grid, cv=4, return_train_score=True).fit(X, y)
    _compare_cv_results(a, b)
    np.testing.assert_array_equal(a.predict(X), b.predict(X))
    pg = [{"svc__" + k: v for k, v in d.items()} for d in grid]
    a = GridSearchCV(None, Pipeline([("svc", SVC())]), pg, cv=4).fit(X, y)
    b = SkGrid(Pipeline([("svc", SVC())]), pg, cv=4, return_train_score=True).fit(X, y)
    _compare_cv_results(a, b)
    np.testing.assert_array_equal(a.predict(X), b.predict(X))
    np.testing.assert_allclose(a.decision_function(X), b.decision_function(X), rtol=0, atol=1e-12)


def test_in_process_multi_gpu_equals_single_gpu_kernels(monkeypatch):
    """The mixed poly / sigmoid / rbf / linear grid dealt over several GPUs gives the one-GPU cv_results_; skipped on a
    one-GPU box."""
    from spark_sklearn_b200 import GridSearchCV
    from spark_sklearn_b200.engine import device_count
    if device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    w = W.make_workload("svc_kernels_mid")
    monkeypatch.setenv("B200GS_DEVICES", "1")
    one = GridSearchCV(None, SVC(), w["param_grid"], cv=w["cv"], refit=False).fit(w["X"], w["y"])
    monkeypatch.setenv("B200GS_DEVICES", "all")
    many = GridSearchCV(None, SVC(), w["param_grid"], cv=w["cv"], refit=False).fit(w["X"], w["y"])
    assert len(many.devices_) > 1
    for k in one.cv_results_:
        if k.endswith("_score"):
            np.testing.assert_array_equal(np.asarray(one.cv_results_[k], float), np.asarray(many.cv_results_[k], float), err_msg=k)
