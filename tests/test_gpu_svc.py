"""GPU parity tests for the SVC path, through the C ABI (libb200gs.so).

Checker: the oracle (oracle/svc_oracle.c, pinned against scikit-learn in test_oracle.py) on the same
seeded inputs, and the committed goldens (scikit-learn 1.9.0 itself).  Bar: integer work (n_iter,
vote counts -> accuracies) bit-exact; float64 Gram to 1e-13 relative; float32 kernel matrix equal
to the oracle's on all but a vanishing fraction of entries (float64 exp last-bit differences).
"""
import numpy as np
import pytest

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


def test_gram_f64_and_kernel_matrix(engine):
    w, fold_id, ns = _setup(engine, "c2_small")
    X64 = w["X"].astype(np.float64)
    S, xsq = engine.debug_gram()
    ref = X64 @ X64.T
    assert np.abs(S - ref).max() <= 1e-13 * np.abs(ref).max()
    np.testing.assert_array_equal(xsq, np.diag(S))
    np.testing.assert_array_equal(S, S.T)
    for gamma in (1 / 512, 1 / 32):
        K = engine.debug_kernel_matrix("rbf", gamma)
        d2 = (xsq[:, None] + xsq[None, :]) - 2 * S
        Kref = np.exp(-gamma * d2).astype(np.float32)
        frac = np.mean(K != Kref)
        assert frac < 1e-5, frac                   # last-bit exp differences only
        assert np.abs(K.astype(np.float64) - Kref).max() <= 1.2e-7
        np.testing.assert_array_equal(np.diag(K), np.ones(len(K), np.float32))
    Kl = engine.debug_kernel_matrix("linear", 0.0)
    np.testing.assert_array_equal(Kl, S.astype(np.float32))


def test_gram_ragged_shapes(engine):
    rng = np.random.RandomState(1)
    for n, d in ((131, 7), (257, 33), (64, 130)):
        X = rng.randn(n, d).astype(np.float32)
        y = (np.arange(n) % 2).astype(np.int32)
        engine.set_data(X, np.zeros(n, np.int8) + (np.arange(n) % 2).astype(np.int8), 2, y_class=y)
        S, xsq = engine.debug_gram()
        ref = X.astype(np.float64) @ X.astype(np.float64).T
        assert np.abs(S - ref).max() <= 1e-13 * np.abs(ref).max()
    Xd = rng.randn(90, 5)                           # float64 features (iris-like): products not exact
    engine.set_data(Xd, (np.arange(90) % 3).astype(np.int8), 3, y_class=(np.arange(90) % 2).astype(np.int32))
    S, _ = engine.debug_gram()
    assert np.abs(S - Xd @ Xd.T).max() <= 1e-14 * np.abs(S).max() * 5


def _run(engine, w, cands):
    kern = [c.get("kernel", w["est_params"].get("kernel", "rbf")) for c in cands]
    C = [float(c.get("C", 1.0)) for c in cands]
    d = w["X"].shape[1]
    gam = []
    for c in cands:
        g = c.get("gamma", w["est_params"].get("gamma", "scale"))
        gam.append(1.0 / d if g == "auto" else float(g))
    return engine.svc(kern, C, np.array(gam)[:, None], tol=1e-3, max_iter=-1, shrinking=True, return_train=True)


def test_c1_iris_bitexact(engine):
    """BASELINE config 1: 3 classes (one-vs-one), linear + rbf, float64 features."""
    w, fold_id, ns = _setup(engine, "c1")
    g = golden("c1_iris_svc")
    r = _run(engine, w, W.candidates(w))
    np.testing.assert_array_equal(r["test"], g["test_scores"])
    np.testing.assert_array_equal(r["train"], g["train_scores"])
    np.testing.assert_array_equal(r["n_iter"], g["diag"][:, :, 0].astype(np.int32))
    np.testing.assert_allclose(r["test"].mean(1), [0.98, 0.98, 0.9733333333, 0.98], atol=1e-9)


@pytest.mark.parametrize("key", ["c2_small", "c2_mid"])
def test_c2_reduced_bitexact(engine, key):
    """Same recipe as BASELINE config 2 at sizes the CPU finishes in seconds; c2_mid (l=2400) exercises
    shrinking, gradient reconstruction and the swap permutation."""
    w, fold_id, ns = _setup(engine, key)
    g = golden(key)
    r = _run(engine, w, W.candidates(w))
    np.testing.assert_array_equal(r["n_iter"], g["diag"][:, :, 0].astype(np.int32))   # same trajectory
    np.testing.assert_array_equal(r["n_sv"], g["diag"][:, :, 1].astype(np.int32))
    np.testing.assert_array_equal(r["test"], g["test_scores"])
    np.testing.assert_array_equal(r["train"], g["train_scores"])


def test_smo_against_oracle_on_gpu_kernel_matrix(engine):
    """Hand the oracle the very float32 kernel matrix the GPU built: alpha*y and rho must be bit-identical."""
    from oracle import oracle as O
    w, fold_id, ns = _setup(engine, "c2_small")
    X64, y = w["X"].astype(np.float64), w["y"]
    gamma, C = 1 / 64, 10.0
    K = engine.debug_kernel_matrix("rbf", gamma)
    engine.set_data(w["X"], np.full(len(y), -1, np.int8), 1, y_class=y.astype(np.int32))   # refit view: all rows
    coef, rho, it = engine.svc_refit("rbf", C, gamma, 2)
    rows = np.concatenate([np.flatnonzero(y == 0), np.flatnonzero(y == 1)]).astype(np.int32)
    oc, orho, oit, _ = O.svc_solve(X64, rows, int((y == 0).sum()), "rbf", gamma, C, Kpre=K)
    full = np.zeros(len(y)); full[rows] = oc
    assert it[0] == oit
    np.testing.assert_array_equal(coef[0], full)
    assert rho[0] == orho


def test_no_shrinking_and_max_iter(engine):
    from sklearn.svm import SVC
    import warnings
    w, fold_id, ns = _setup(engine, "c2_small")
    X, y = w["X"], w["y"]
    for kw in (dict(shrinking=False, max_iter=-1), dict(shrinking=True, max_iter=300)):
        r = engine.svc(["rbf"], [10.0], [[1 / 64]], tol=1e-3, return_train=True, **kw)
        for k in range(ns):
            tr, te = np.flatnonzero(fold_id != k), np.flatnonzero(fold_id == k)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                s = SVC(C=10.0, gamma=1 / 64, **kw).fit(X[tr], y[tr])
            assert r["n_iter"][0, k] == s.n_iter_[0]
            assert r["test"][0, k] == s.score(X[te], y[te])
            assert r["train"][0, k] == s.score(X[tr], y[tr])


@pytest.mark.parametrize("method", ["svc", "svr"])
def test_non_finite_gamma_is_rejected(engine, method):
    """An infinite rbf gamma would put NaN on the kernel diagonal (-inf * 0): both searches refuse it before any launch."""
    from spark_sklearn_b200.engine import EngineError
    rng = np.random.RandomState(0)
    X = rng.randn(40, 3).astype(np.float32)
    fold_id = (np.arange(40) % 2).astype(np.int8)
    if method == "svc":
        engine.set_data(X, fold_id, 2, y_class=(np.arange(40) // 2 % 2).astype(np.int32))
        search = lambda g: engine.svc(["rbf"], [1.0], [g])
    else:
        y = rng.randn(40)
        engine.set_data(X, fold_id, 2, y_target=y.astype(np.float32))
        engine.set_targets_f64(y)
        search = lambda g: engine.svr(["rbf"], [1.0], [0.1], [g])
    with pytest.raises(EngineError, match="gamma must be finite"):
        search(np.inf)
    assert np.all(np.isfinite(search(0.5)["test"]))        # the handle stays usable


def test_python_api_iris(engine):
    """The reference's own example (tests/test_search_2.py:32-45, README): iris, SVC(gamma='auto')."""
    from sklearn import svm
    from sklearn.base import clone
    from sklearn.model_selection import GridSearchCV as SkGrid
    from spark_sklearn_b200 import GridSearchCV
    w = W.make_workload("c1")
    X, y = w["X"], w["y"]
    parameters = {'kernel': ('linear', 'rbf'), 'C': [1, 10]}
    clf = GridSearchCV(None, svm.SVC(gamma='auto'), parameters, cv=5).fit(X, y)
    sk = SkGrid(svm.SVC(gamma='auto'), parameters, cv=5, return_train_score=True).fit(X, y)
    for key in sk.cv_results_:
        if key.endswith("_time"):
            assert key in clf.cv_results_
            continue
        a, b = clf.cv_results_[key], sk.cv_results_[key]
        if key == "params":
            assert a == b
        elif key.startswith("param_"):
            assert list(a) == list(b)
        elif key.startswith(("mean_", "std_")):
            # the reference aggregates with np.average(weights=test sizes) (iid=True, base_search.py:115-121);
            # sklearn >= 0.24 uses the plain mean: same numbers to the last ulp on equal folds
            np.testing.assert_allclose(np.asarray(a, float), np.asarray(b, float), rtol=0, atol=4e-16, err_msg=key)
        else:
            np.testing.assert_array_equal(np.asarray(a, float), np.asarray(b, float), err_msg=key)
    assert clf.best_index_ == sk.best_index_ and clf.best_params_ == sk.best_params_
    np.testing.assert_array_equal(clf.predict(X), sk.predict(X))
    np.testing.assert_allclose(clf.decision_function(X), sk.decision_function(X), rtol=0, atol=1e-12)
    assert clf.score(X, y) == sk.score(X, y)
    assert clf.estimator.get_params() == clone(svm.SVC(gamma='auto')).get_params()   # the reference's assertion


@pytest.mark.parametrize("cl", [2, 4, 8])
def test_cluster_smo_bitexact(engine, monkeypatch, cl):
    """Every sub-problem through the thread-block-cluster solver (smo_colown.cu: one problem over 2 / 4 / 8 SMs, static
    element ownership, DSMEM record exchange): same trajectory, same scores as scikit-learn."""
    monkeypatch.setenv("B200GS_SMO_CLUSTER", str(cl))
    monkeypatch.setenv("B200GS_SMO_CLUSTER_N", "100000")
    w, fold_id, ns = _setup(engine, "c2_mid")
    g = golden("c2_mid")
    r = _run(engine, w, W.candidates(w))
    np.testing.assert_array_equal(r["n_iter"], g["diag"][:, :, 0].astype(np.int32))
    np.testing.assert_array_equal(r["n_sv"], g["diag"][:, :, 1].astype(np.int32))
    np.testing.assert_array_equal(r["test"], g["test_scores"])
    np.testing.assert_array_equal(r["train"], g["train_scores"])


@pytest.mark.parametrize("cl", [0, 2, 4, 8])
def test_general_kernel_paths_vs_sklearn(engine, monkeypatch, cl):
    """The non-specialised solver instances (linear kernel: QD != 1; rbf whose kernel matrix underflows to denormals and
    zeros: no integer-pipe widening, float64 approximate filter), single-CTA (cl=0) and cluster kernels, against
    scikit-learn fits of the same folds: identical iteration counts and scores."""
    from sklearn.svm import SVC
    monkeypatch.setenv("B200GS_SMO_CLUSTER", str(cl))
    if cl:
        monkeypatch.setenv("B200GS_SMO_CLUSTER_N", "100000")
    w, fold_id, ns = _setup(engine, "c2_mid")
    X, y = w["X"], w["y"]
    cases = [("linear", 0.01, 0.0), ("rbf", 1.0, 0.35), ("rbf", 3.0, 2.0)]
    r = engine.svc([c[0] for c in cases], [c[1] for c in cases], np.array([c[2] for c in cases])[:, None], tol=1e-3,
                   max_iter=-1, shrinking=True, return_train=True)
    for i, (kern, C, gam) in enumerate(cases):
        for k in range(ns):
            tr, te = np.flatnonzero(fold_id != k), np.flatnonzero(fold_id == k)
            s = SVC(kernel=kern, C=C, gamma=gam if kern == "rbf" else "scale").fit(X[tr], y[tr])
            assert r["n_iter"][i, k] == s.n_iter_[0], (kern, C, gam, k)
            assert r["test"][i, k] == s.score(X[te], y[te])
            assert r["train"][i, k] == s.score(X[tr], y[tr])


def test_full_data_refit_vs_sklearn(engine):
    """The refit of a candidate on ALL 10000 rows of config 2 (one sub-problem -> an 8-CTA cluster with l = 10000 > 8192).
    Against scikit-learn's own fit (tests/golden/c2_refit_C10_g1024.npz = SVC(C=10, gamma=1/1024).fit(X, y)): same
    iteration count and support set, coefficients within 1e-7 (scikit-learn's BLAS dot products round a few float32 Q
    entries differently; the selection sequence is unaffected here).  Against the C oracle, which forms the Gram the way
    the GPU does: bit-identical coefficients and intercept."""
    w = W.make_workload("c2")
    X, y = w["X"], w["y"]
    g = golden("c2_refit_C10_g1024")
    engine.set_data(X, np.full(len(y), -1, np.int8), 1, y_class=y.astype(np.int32))
    coef, rho, it = engine.svc_refit("rbf", 10.0, 1 / 1024, 2)
    assert it[0] == int(g["n_iter"][0])
    sv = np.flatnonzero(coef[0] != 0)
    order = np.argsort(g["support"], kind="stable")                    # sklearn lists support vectors class by class
    np.testing.assert_array_equal(sv, g["support"][order])
    np.testing.assert_allclose(np.abs(coef[0][sv]), np.abs(g["dual_coef"][0][order]), rtol=0, atol=1e-7)
    np.testing.assert_array_equal(coef[0], g["oracle_coef"])
    assert rho[0] == float(g["oracle_rho"][0])


def test_c2_full_size_vs_golden(engine):
    """BASELINE config 2 at full size (10000x512, 8x8 grid, cv=5 = 320 fits): every split score equals scikit-learn's."""
    w, fold_id, ns = _setup(engine, "c2")
    g = golden("c2_svc_rbf_8x8")
    r = _run(engine, w, W.candidates(w))
    np.testing.assert_array_equal(r["test"], g["test_scores"])
    np.testing.assert_array_equal(r["train"], g["train_scores"])
    np.testing.assert_array_equal(r["n_sv"], g["diag"][:, :, 1].astype(np.int32))
    assert np.mean(r["n_iter"] == g["diag"][:, :, 0].astype(np.int32)) >= 0.98     # a float64-exp last bit moves ~1 trajectory in 320
    assert np.abs(r["test"].mean(1) - g["test_scores"].mean(1)).max() <= 1e-4     # the BASELINE bar (observed: 0)


def test_c4_full_size_vs_golden(engine):
    """BASELINE config 4 (10000x512, 16x16 grid, cv=5 = 1280 fits; 1.9 h of scikit-learn on 6 cores): every split score
    equals scikit-learn's."""
    w, fold_id, ns = _setup(engine, "c4")
    g = golden("c4_svc_rbf_16x16")
    r = _run(engine, w, W.candidates(w))
    assert np.abs(r["test"].mean(1) - g["test_scores"].mean(1)).max() <= 1e-4     # the BASELINE bar
    print("c4: test-score mismatches %d/1280, train %d/1280, n_iter equal %d/1280" % (
        (r["test"] != g["test_scores"]).sum(), (r["train"] != g["train_scores"]).sum(),
        (r["n_iter"] == g["diag"][:, :, 0].astype(np.int32)).sum()))
    np.testing.assert_array_equal(r["test"], g["test_scores"])
    np.testing.assert_array_equal(r["train"], g["train_scores"])
    # a float64-exp last bit (CUDA's exp vs the host libm's) changes ~2^-29 of the float32 Q entries.  Observed: single
    # entries of the gamma#4 and gamma#5 matrices differ; the sub-problems that touch them (same fold, every C -- and C#11..15
    # are the same unbounded problem) end within 0.5 % of scikit-learn's iteration count, 30 of 1280 fits, one with one
    # more support vector, no score change.  Every other trajectory is identical iteration for iteration.
    dsv = np.abs(r["n_sv"] - g["diag"][:, :, 1].astype(np.int32))
    assert (dsv != 0).mean() <= 0.005 and dsv.max() <= 2
    gi = g["diag"][:, :, 0].astype(np.int32)
    assert np.mean(r["n_iter"] == gi) >= 0.97
    assert np.max(np.abs(r["n_iter"] - gi) / gi) <= 0.01


def test_tensor_core_gram_mode(engine):
    """GS_GRAM_TENSOR: the Gram on wgmma tensor cores (3xTF32).  fp32-faithful Q entries differ from libsvm's by an
    ulp or two, so trajectories diverge within libsvm's own stopping tolerance: scores agree to a few margin flips."""
    from spark_sklearn_b200.engine import GS_GRAM_TENSOR
    w, fold_id, ns = _setup(engine, "c2_mid")
    g = golden("c2_mid")
    cands = W.candidates(w)
    r = engine.svc(["rbf"] * len(cands), [c["C"] for c in cands], np.array([c["gamma"] for c in cands])[:, None],
                   flags=GS_GRAM_TENSOR)
    assert np.abs(r["test"] - g["test_scores"]).max() <= 5 / 600 + 1e-12            # <= 5 flips on a 600-row fold
    assert np.abs(r["test"].mean(1) - g["test_scores"].mean(1)).max() <= 3e-3
    rel = np.abs(r["n_iter"] - g["diag"][:, :, 0]) / g["diag"][:, :, 0]
    assert np.median(rel) < 0.05


def test_in_process_multi_gpu_equals_single_gpu(monkeypatch):
    """One plain fit() on a node with several GPUs drives all of them (a handle and a host thread per device, no
    torch.distributed): identical cv_results_ to the one-GPU search; skipped on a one-GPU box."""
    from sklearn.svm import SVC
    from spark_sklearn_b200 import GridSearchCV
    from spark_sklearn_b200.engine import device_count
    if device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    w = W.make_workload("c2_mid")
    monkeypatch.setenv("B200GS_DEVICES", "1")
    one = GridSearchCV(None, SVC(kernel="rbf"), w["param_grid"], cv=w["cv"], refit=False).fit(w["X"], w["y"])
    monkeypatch.setenv("B200GS_DEVICES", "all")
    many = GridSearchCV(None, SVC(kernel="rbf"), w["param_grid"], cv=w["cv"], refit=False).fit(w["X"], w["y"])
    assert len(many.devices_) == min(device_count(), 16) and len(one.devices_) == 1
    for k in one.cv_results_:
        if k.endswith("_score"):                                   # every split / mean / std / rank score; not the *_score_time keys
            np.testing.assert_array_equal(np.asarray(one.cv_results_[k], float), np.asarray(many.cv_results_[k], float), err_msg=k)


@pytest.mark.parametrize("cl", [0, 4])
def test_class_weight_vs_sklearn(engine, monkeypatch, cl):
    """SVC(class_weight=...): the C of a training row is C x the weight of its class, 'balanced' recomputed from the
    training labels of every fold (reference base_search.py:69,83-87 forwards the estimator's parameters into every task).
    Slot-layout and cluster solver, binary and one-vs-one, against scikit-learn: identical split scores and predictions."""
    from sklearn import svm
    from sklearn.model_selection import GridSearchCV as SkGrid
    from spark_sklearn_b200 import GridSearchCV
    monkeypatch.setenv("B200GS_SMO_CLUSTER", str(cl))
    if cl:
        monkeypatch.setenv("B200GS_SMO_CLUSTER_N", "100000")
    w = W.make_workload("c2_mid")
    X, y = w["X"][:1500], w["y"][:1500].copy()
    y[:350] = 0                                                     # unbalanced classes
    grid = {"C": [0.5, 8.0], "class_weight": [None, "balanced", {0: 1.0, 1: 6.0}]}
    a = GridSearchCV(None, svm.SVC(kernel="rbf", gamma=1 / 128), grid, cv=4).fit(X, y)
    b = SkGrid(svm.SVC(kernel="rbf", gamma=1 / 128), grid, cv=4, return_train_score=True).fit(X, y)
    for k in range(4):
        for part in ("test", "train"):
            key = "split%d_%s_score" % (k, part)
            np.testing.assert_array_equal(a.cv_results_[key], b.cv_results_[key], err_msg=key)
    assert a.best_params_ == b.best_params_
    np.testing.assert_array_equal(a.predict(X), b.predict(X))
    np.testing.assert_allclose(a.best_estimator_.class_weight_, b.best_estimator_.class_weight_, rtol=1e-15)
    np.testing.assert_array_equal(a.best_estimator_.n_iter_, b.best_estimator_.n_iter_)
    if cl == 0:
        wi = W.make_workload("c1")                                  # three classes, one-vs-one pairs with different C per side
        gi = {"C": [1, 10], "class_weight": ["balanced", {0: 2.0, 2: 0.5}]}
        ai = GridSearchCV(None, svm.SVC(gamma="auto"), gi, cv=5).fit(wi["X"], wi["y"])
        bi = SkGrid(svm.SVC(gamma="auto"), gi, cv=5, return_train_score=True).fit(wi["X"], wi["y"])
        for k in range(5):
            np.testing.assert_array_equal(ai.cv_results_["split%d_test_score" % k], bi.cv_results_["split%d_test_score" % k])
        np.testing.assert_array_equal(ai.predict(wi["X"]), bi.predict(wi["X"]))
