"""CPU tests of the host side: C-ABI surface, search driver (aggregation, ranking, masked params, refit
materialisation), error behaviour, and the multi-rank candidate striding + all-gather over gloo.

The GPU engine is replaced by an oracle-backed plan (tests may use oracle/), so everything the Python
layer does around the CUDA call is exercised without a GPU.
"""
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------ C ABI -------------------------
def test_cabi_library_exports_every_declared_symbol():
    import ctypes
    from spark_sklearn_b200 import build, engine
    build.build()
    hdr = open(os.path.join(ROOT, "include", "b200gs.h")).read()
    names = sorted(set(re.findall(r"\b(gs_[a-z_0-9]+)\s*\(", hdr)))
    assert {"gs_create", "gs_destroy", "gs_set_data", "gs_svc", "gs_svc_refit", "gs_ridge", "gs_logreg",
            "gs_get_profile", "gs_last_error"} <= set(names)
    lib = ctypes.CDLL(engine.LIB_PATH)
    for n in names:
        assert hasattr(lib, n), n
    assert engine.load_library().gs_version() >= 100


def _golden_svc(name):
    g = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"), allow_pickle=True)
    names = [str(x) for x in g["param_names"]]
    tof = lambda col: np.array([float(re.sub(r"np\.float64\((.*)\)", r"\1", str(x))) for x in col])
    return tof(g["param_values"][:, names.index("C")]), tof(g["param_values"][:, names.index("gamma")]), g["diag"][:, :, 0]


def test_planning_helpers_against_measured_iteration_counts():
    """gs_svc_predicted_iterations ranks the 1600 measured fits of configs 2 and 4 (scikit-learn's n_iter_) with a Spearman
    correlation >= 0.97, and gs_svc_cluster_count picks the critical-path group: the ten 66-68k-iteration problems of
    config 2, nothing for the throughput-bound config 4.  Host-only entry points: callable without a GPU."""
    from scipy.stats import spearmanr
    from spark_sklearn_b200 import engine
    L = engine.load_library()
    picks = {}
    for name in ("c2_svc_rbf_8x8", "c4_svc_rbf_16x16"):
        C, gam, it = _golden_svc(name)
        pred = np.array([L.gs_svc_predicted_iterations(1, c, g, 512) for c, g in zip(C, gam)])
        assert spearmanr(np.repeat(pred, it.shape[1]), it.ravel())[0] >= 0.97
        assert np.median(np.abs(pred * 1000 / it.mean(1) - 1)) <= 0.2          # and is roughly calibrated (thousands)
        cost = np.sort(np.repeat(pred, it.shape[1]))[::-1].copy()
        true = np.sort(it.ravel().astype(float))[::-1].copy()                     # with the true counts as costs
        for sms in (148, 132):                                                    # the calibration GPU and the H100
            picks[name, sms] = L.gs_svc_cluster_count(cost.ctypes.data, len(cost), sms)
            assert L.gs_svc_cluster_count(true.ctypes.data, len(true), sms) == picks[name, sms]
    assert picks == {("c2_svc_rbf_8x8", 148): 10, ("c4_svc_rbf_16x16", 148): 0, ("c2_svc_rbf_8x8", 132): 10, ("c4_svc_rbf_16x16", 132): 0}
    assert L.gs_svc_predicted_iterations(0, 3.0, 0.0, 512) == 3.0                  # linear: grows with C
    assert L.gs_svc_cluster_count(None, 0, 148) == 0


def test_no_gpu_fails_loudly():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from spark_sklearn_b200.engine import Engine, EngineError
    with pytest.raises(EngineError) as e:
        Engine(0)
    assert "no CPU fallback" in str(e.value) or "CUDA" in str(e.value)


def test_product_code_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "spark_sklearn_b200")
    for f in os.listdir(pkg):
        if f.endswith(".py"):
            src = open(os.path.join(pkg, f)).read()
            assert not re.search(r"^\s*(from|import)\s+oracle", src, re.M), f


# ------------------------------------------------------------------ oracle-backed plan ------------
class OraclePlan:
    def __init__(self, estimator, cands, X, y, fold_id, n_splits):
        fold_id = getattr(fold_id, "fold_id", fold_id)                     # base_search hands over an estimators.Folds
        self.estimator, self.cands, self.X, self.y, self.fold_id, self.n_splits = estimator, cands, np.asarray(X), y, fold_id, n_splits

    def evaluate(self, my, return_train=True, error_score="raise"):
        from oracle import oracle as O
        p0 = self.estimator.get_params()
        test, train, _ = O.cv_scores_svc(self.X, self.y, self.fold_id, self.n_splits, [self.cands[i] for i in my], p0)
        z = np.zeros_like(test)
        return dict(test=test, train=train if return_train else None, fit_time=z + 1e-3, score_time=z + 1e-4)

    def profile(self):
        return {}

    def costs(self):
        return np.array([float(c.get("C", 1.0)) for c in self.cands])      # exercises the cost-balanced dealing

    def refit(self, best):
        from oracle import oracle as O
        from sklearn.base import clone
        from spark_sklearn_b200.estimators import materialize_svc
        p = self.estimator.get_params(); p.update(best)
        classes, yc = np.unique(self.y, return_inverse=True)
        m = O.SVCModel(np.ascontiguousarray(self.X, np.float64), self.y, np.arange(len(self.y)), kernel=p["kernel"],
                       gamma=p["gamma"], C=p["C"], tol=p["tol"])
        coef = np.zeros((len(m.pairs), len(self.y)))
        for q, (_, _, rows, c, _) in enumerate(m.pairs):
            coef[q, rows] = c
        return materialize_svc(clone(self.estimator).set_params(**best), self.X, yc, classes, coef,
                               np.array([p_[4] for p_ in m.pairs]), np.array(m.n_iter), m.gamma)

    def close(self):
        pass


class OracleAdapter:
    plan = staticmethod(lambda *a: OraclePlan(*a))


@pytest.fixture
def oracle_backend(monkeypatch):
    from spark_sklearn_b200 import base_search
    monkeypatch.setattr(base_search._est, "adapter_for", lambda est: OracleAdapter)


def _iris():
    from sklearn.datasets import load_iris
    d = load_iris()
    return d.data, d.target


def test_search_driver_matches_sklearn_on_the_reference_example(oracle_backend):
    """reference tests/test_search_2.py:32-45 + doctest grid_search.py:90-116, with numbers."""
    from sklearn import svm
    from sklearn.model_selection import GridSearchCV as SkGrid
    from spark_sklearn_b200 import GridSearchCV
    X, y = _iris()
    parameters = {'kernel': ('linear', 'rbf'), 'C': [1, 10]}
    clf = GridSearchCV(None, svm.SVC(gamma='auto'), parameters).fit(X, y)       # reference default cv=3
    sk = SkGrid(svm.SVC(gamma='auto'), parameters, cv=3, return_train_score=True).fit(X, y)
    assert sorted(clf.cv_results_.keys()) == sorted(sk.cv_results_.keys())      # the doctest's key set
    for k in range(3):
        np.testing.assert_array_equal(clf.cv_results_["split%d_test_score" % k], sk.cv_results_["split%d_test_score" % k])
        np.testing.assert_array_equal(clf.cv_results_["split%d_train_score" % k], sk.cv_results_["split%d_train_score" % k])
    np.testing.assert_allclose(clf.cv_results_["mean_test_score"], [0.9933333333, 0.9733333333, 0.9733333333, 0.98], atol=1e-9)
    np.testing.assert_array_equal(clf.cv_results_["rank_test_score"], [1, 3, 3, 2])   # SURVEY.md 8c table
    assert clf.cv_results_["rank_test_score"].dtype == np.int32
    assert clf.best_index_ == 0 and clf.best_params_ == {"C": 1, "kernel": "linear"} and clf.n_splits_ == 3
    assert list(clf.cv_results_["param_kernel"]) == ["linear", "rbf", "linear", "rbf"]
    assert clf.cv_results_["params"] == sk.cv_results_["params"]
    np.testing.assert_array_equal(clf.predict(X), sk.predict(X))
    np.testing.assert_allclose(clf.decision_function(X), sk.decision_function(X), atol=1e-12)
    assert clf.score(X, y) == sk.score(X, y)
    assert clf.estimator.get_params() == svm.SVC(gamma='auto').get_params()      # the reference's own assertion
    from sklearn.base import clone
    assert clone(clf).get_params()["param_grid"] == parameters                   # get_params/clone keep working


def test_iid_weighting_on_unequal_folds(oracle_backend):
    """reference base_search.py:115,129-133: iid=True weights fold means by test-set size."""
    from sklearn import svm
    from spark_sklearn_b200 import GridSearchCV
    X, y = _iris()
    X, y = X[:148], y[:148]
    g = {"C": [1.0]}
    a = GridSearchCV(None, svm.SVC(gamma='auto'), g, cv=5, iid=True).fit(X, y)
    b = GridSearchCV(None, svm.SVC(gamma='auto'), g, cv=5, iid=False).fit(X, y)
    s = np.array([a.cv_results_["split%d_test_score" % k][0] for k in range(5)])
    from sklearn.model_selection import StratifiedKFold
    sizes = np.array([len(te) for _, te in StratifiedKFold(5).split(X, y)])
    assert a.cv_results_["mean_test_score"][0] == np.average(s, weights=sizes)
    assert b.cv_results_["mean_test_score"][0] == np.average(s)


def test_randomized_search_candidates_and_shape(oracle_backend):
    """reference tests/test_search_2.py:47-60,81,95: len(params) == n_iter, sampler identical to sklearn's."""
    from scipy.stats import loguniform
    from sklearn import svm
    from sklearn.model_selection import ParameterSampler
    from spark_sklearn_b200 import RandomizedSearchCV
    X, y = _iris()
    dist = {"C": loguniform(0.1, 100), "kernel": ["linear", "rbf"]}
    r = RandomizedSearchCV(None, svm.SVC(gamma='auto'), dist, n_iter=5, random_state=4, cv=3).fit(X, y)
    assert len(r.cv_results_["params"]) == 5
    assert r.cv_results_["params"] == list(ParameterSampler(dist, 5, random_state=4))
    assert "mean_train_score" in r.cv_results_            # return_train_score is always on (random_search.py:195-199)


def test_unsupported_configurations_raise_instead_of_falling_back():
    from sklearn import svm
    from sklearn.tree import DecisionTreeClassifier
    from spark_sklearn_b200 import GridSearchCV
    X, y = _iris()
    with pytest.raises(NotImplementedError):
        GridSearchCV(None, DecisionTreeClassifier(), {"max_depth": [1, 2]}, cv=3).fit(X, y)
    with pytest.raises(NotImplementedError):
        GridSearchCV(None, svm.SVC(), {"C": [1.0]}, scoring="neg_log_loss", cv=3).fit(X, y)      # no fused scorer
    with pytest.raises(NotImplementedError):
        from sklearn.metrics import make_scorer, accuracy_score
        GridSearchCV(None, svm.SVC(), {"C": [1.0]}, scoring=make_scorer(accuracy_score), cv=3).fit(X, y)
    with pytest.raises(ValueError):
        GridSearchCV(None, svm.SVC(), {"C": 1.0})          # _check_param_grid (grid_search.py:226)


def test_three_tier_schedule_on_measured_and_synthetic_costs():
    """gs_svc_schedule (clusters / exclusive SMs / shared SMs): on the measured iteration counts of configs 2 and 4 and on
    cost profiles it was not calibrated on.  Properties, not constants: a throughput-bound profile gets no latency tier; a
    profile with a few dominant problems puts exactly those on clusters; the predicted makespan never exceeds the
    all-shared schedule's; specialised SMs never exceed the GPU."""
    import ctypes
    from spark_sklearn_b200 import engine
    L = engine.load_library()

    def sched(cost, sms=148):
        c = np.sort(np.asarray(cost, float))[::-1].copy()
        a, b = ctypes.c_int32(), ctypes.c_int32()
        L.gs_svc_schedule(c.ctypes.data, len(c), sms, ctypes.byref(a), ctypes.byref(b))
        return a.value, b.value, c

    def makespan(c, nc, ne, sms=148):
        left = sms - 4 * nc - ne
        t = max(0.5 * c[nc + ne:].sum() / left, 0.78 * c[nc + ne] if nc + ne < len(c) else 0.0)
        if nc: t = max(t, 0.34 * c[0])
        if ne: t = max(t, 0.52 * c[nc])
        return t

    _, _, it2 = _golden_svc("c2_svc_rbf_8x8")
    _, _, it4 = _golden_svc("c4_svc_rbf_16x16")
    nc, ne, c = sched(it2.ravel())
    assert 10 <= nc <= 20 and 10 <= ne <= 40 and 4 * nc + ne <= 140           # the 66-68k group on clusters, the 43-48k tier alone
    assert makespan(c, nc, ne) <= 0.75 * makespan(c, 0, 0)
    assert sched(it4.ravel())[:2] == (0, 0)                                    # 1280 problems: throughput-bound
    nc, ne, c = sched(it2.ravel(), 132)                                        # the H100's 132 SMs
    assert 10 <= nc <= 20 and 10 <= ne <= 40 and 4 * nc + ne <= 124
    assert makespan(c, nc, ne, 132) <= 0.75 * makespan(c, 0, 0, 132)
    assert sched(it4.ravel(), 132)[:2] == (0, 0)
    rng = np.random.default_rng(0)
    for trial in range(20):                                                    # unseen profiles
        n = int(rng.integers(150, 3000))
        cost = rng.lognormal(0.0, rng.uniform(0.2, 1.5), n)
        nc, ne, c = sched(cost)
        assert 4 * nc + ne <= 140 and nc + ne < n
        assert makespan(c, nc, ne) <= makespan(c, 0, 0) * (1 + 1e-12)
    flat = np.ones(2000)
    assert sched(flat)[:2] == (0, 0)
    spiky = np.r_[np.full(5, 100.0), np.ones(400)]                             # five dominant problems
    nc, ne, _ = sched(spiky)
    assert nc == 5 and ne == 0
    a, b = ctypes.c_int32(7), ctypes.c_int32(7)
    L.gs_svc_schedule(None, 0, 148, ctypes.byref(a), ctypes.byref(b))
    assert (a.value, b.value) == (0, 0)


def test_fold_ids_reject_non_partition_splitters():
    from sklearn.model_selection import ShuffleSplit, StratifiedKFold
    from spark_sklearn_b200.estimators import fold_ids_from_splits
    X, y = _iris()
    f = fold_ids_from_splits(list(StratifiedKFold(5).split(X, y)), len(y))
    assert set(f) == {0, 1, 2, 3, 4} and f.dtype == np.int8
    with pytest.raises(NotImplementedError):
        fold_ids_from_splits(list(ShuffleSplit(3, test_size=0.5, random_state=0).split(X)), len(y))


def test_split_masks_cover_general_splitters():
    """reference base_search.py:34,81-82 re-derives ANY cv.split per task; here: fold ids for partitions, 128-bit membership
    masks per row otherwise (overlapping test sets, rows in neither set, rows that only train)."""
    from sklearn.model_selection import PredefinedSplit, RepeatedStratifiedKFold, ShuffleSplit, StratifiedKFold
    from spark_sklearn_b200.estimators import Folds, split_masks
    X, y = _iris()
    n = len(y)
    f = Folds(list(StratifiedKFold(5).split(X, y)), n)
    assert f.partition and f.masks is None and f.train_rows(2).sum() == 120 and f.train_rows(-1).all()
    cases = {"shuffle": list(ShuffleSplit(70, test_size=0.3, train_size=0.5, random_state=0).split(X)),
             "repeated": list(RepeatedStratifiedKFold(n_splits=3, n_repeats=2, random_state=1).split(X, y)),
             "predefined": list(PredefinedSplit(np.r_[np.full(50, -1), np.arange(100) % 2]).split())}
    fp = Folds(cases["predefined"], n)                     # test folds disjoint, -1 rows train everywhere: still fold ids (-1)
    assert fp.partition and (fp.fold_id[:50] == -1).all()
    for name, splits in cases.items():
        f = Folds(splits, n)
        assert f.n_splits == len(splits) and f.partition == (name == "predefined"), name
        te, tr = split_masks(splits, n)
        assert te.shape == (n, 2) and te.dtype == np.uint64
        for k, (a, b) in enumerate(splits):
            got_tr = np.flatnonzero((tr[:, k >> 6] >> np.uint64(k & 63)) & np.uint64(1))
            got_te = np.flatnonzero((te[:, k >> 6] >> np.uint64(k & 63)) & np.uint64(1))
            np.testing.assert_array_equal(got_tr, np.sort(a)); np.testing.assert_array_equal(got_te, np.sort(b))
            np.testing.assert_array_equal(np.flatnonzero(f.train_rows(k)), np.sort(a))
    assert cases["predefined"][0][0][:50].tolist() == list(range(50))           # the -1 rows train in every split
    with pytest.raises(ValueError):
        split_masks([(np.arange(10), np.arange(5, 15))], n)                      # a row in both sets of one split
    with pytest.raises(NotImplementedError):
        split_masks([(np.arange(10), np.arange(10, 20))] * 129, n)


def test_materialize_svc_binary_equals_sklearn_fit():
    from sklearn.svm import SVC
    from oracle import oracle as O
    from spark_sklearn_b200 import workloads as W
    from spark_sklearn_b200.estimators import materialize_svc
    w = W.make_workload("c2_small")
    X, y = w["X"][:400], w["y"][:400]
    ref = SVC(C=10.0, gamma=1 / 64).fit(X, y)
    m = O.SVCModel(X.astype(np.float64), y, np.arange(len(y)), kernel="rbf", gamma=1 / 64, C=10.0)
    coef = np.zeros((1, len(y))); coef[0, m.pairs[0][2]] = m.pairs[0][3]
    est = materialize_svc(SVC(C=10.0, gamma=1 / 64), X, y, np.unique(y), coef, np.array([m.pairs[0][4]]), np.array(m.n_iter), 1 / 64)
    np.testing.assert_array_equal(est.support_, ref.support_)
    np.testing.assert_array_equal(est.dual_coef_, ref.dual_coef_)
    np.testing.assert_array_equal(est.intercept_, ref.intercept_)
    np.testing.assert_array_equal(est.n_support_, ref.n_support_)
    np.testing.assert_array_equal(est.predict(w["X"][400:600]), ref.predict(w["X"][400:600]))
    np.testing.assert_array_equal(est.decision_function(w["X"][400:600]), ref.decision_function(w["X"][400:600]))
    import pickle
    np.testing.assert_array_equal(pickle.loads(pickle.dumps(est)).predict(X), ref.predict(X))


def test_assign_candidates_is_a_balanced_partition():
    from spark_sklearn_b200.dist import assign_candidates
    for n, world in ((64, 1), (64, 8), (6, 4), (7, 3), (512, 8)):
        strided = assign_candidates(n, world)
        assert strided == [list(range(r, n, world)) for r in range(world)]
        rng = np.random.default_rng(n + world)
        costs = rng.lognormal(size=n)
        parts = assign_candidates(n, world, costs)
        assert sorted(sum(parts, [])) == list(range(n))                    # a partition ...
        assert max(map(len, parts)) - min(map(len, parts)) <= 1           # ... of equal sizes ...
        load = [costs[p].sum() for p in parts]
        if n >= 8 * world:
            assert max(load) <= 1.25 * min(load)                          # ... and similar predicted cost
        top = np.argsort(-costs)[:world]                                  # the `world` most expensive land on distinct ranks
        assert len({r for r, p in enumerate(parts) for c in top if c in p}) == world or n < world
    assert assign_candidates(5, 2, [1, np.nan, 2, 3, 4]) == [[0, 2, 4], [1, 3]]   # unusable costs: strided


def test_in_process_scheduler_deals_candidates_over_devices_and_merges(monkeypatch):
    """One fit() over several devices without torch.distributed (north_star: "a single in-process scheduler"): a plan and a
    host thread per device, candidates dealt by predicted cost, host-side merge -- cv_results_ identical to the
    one-device search, whatever the device count (incl. more devices than candidates)."""
    from sklearn import svm
    from spark_sklearn_b200 import GridSearchCV, base_search
    seen = []

    class MultiAdapter:
        multi_device = True

        @staticmethod
        def plan(est, cands, X, y, fold_id, n_splits, device=None):
            seen.append(device)
            return OraclePlan(est, cands, X, y, fold_id, n_splits)

    monkeypatch.setattr(base_search._est, "adapter_for", lambda est: MultiAdapter)
    X, y = _iris()
    grid = {'kernel': ('linear', 'rbf'), 'C': [1, 10, 100]}
    monkeypatch.setattr(base_search._dist, "local_devices", lambda: [0])
    single = GridSearchCV(None, svm.SVC(gamma='auto'), grid, cv=5).fit(X, y)
    assert single.devices_ == [None] or len(single.devices_) == 1
    for nd in (2, 3, 8):
        del seen[:]
        monkeypatch.setattr(base_search._dist, "local_devices", lambda nd=nd: list(range(nd)))
        multi = GridSearchCV(None, svm.SVC(gamma='auto'), grid, cv=5).fit(X, y)
        assert sorted(seen) == list(range(min(nd, 6))) and multi.devices_ == list(range(min(nd, 6)))
        for k, v in single.cv_results_.items():
            if "score" in k:
                np.testing.assert_array_equal(np.asarray(v, float), np.asarray(multi.cv_results_[k], float), err_msg=k)
        assert multi.best_params_ == single.best_params_
        np.testing.assert_array_equal(multi.predict(X), single.predict(X))


# ------------------------------------------------------------------ multi-rank (gloo, CPU) --------
def _worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from sklearn import svm
    from spark_sklearn_b200 import GridSearchCV, base_search
    base_search._est.adapter_for = lambda est: OracleAdapter
    X, y = _iris()
    grid = {'kernel': ('linear', 'rbf'), 'C': [1, 10, 100]}            # 6 candidates over 2 ranks (and 4 over 3 below)
    s = GridSearchCV(None, svm.SVC(gamma='auto'), grid, cv=5, refit=False).fit(X, y)
    q.put((rank, {k: np.asarray(v, float) for k, v in s.cv_results_.items() if "score" in k}))
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4])
def test_candidates_strided_over_ranks_allgather_gloo(world, oracle_backend):
    """Same search at 1 and N ranks gives identical cv_results_ on every rank (SURVEY.md 8e; uneven
    n_cand % N is padded)."""
    import torch.multiprocessing as mp
    from sklearn import svm
    from spark_sklearn_b200 import GridSearchCV
    X, y = _iris()
    grid = {'kernel': ('linear', 'rbf'), 'C': [1, 10, 100]}
    single = GridSearchCV(None, svm.SVC(gamma='auto'), grid, cv=5, refit=False).fit(X, y).cv_results_
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000 + world
    ps = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in ps:
        p.start()
    got = [q.get(timeout=120) for _ in ps]
    for p in ps:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, res in got:
        for k, v in res.items():
            np.testing.assert_array_equal(v, np.asarray(single[k], float), err_msg="rank %d %s" % (rank, k))


def _worker_unseeded(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from scipy.stats import loguniform
    from sklearn import svm
    from sklearn.model_selection import StratifiedKFold
    from spark_sklearn_b200 import RandomizedSearchCV, base_search
    base_search._est.adapter_for = lambda est: OracleAdapter
    X, y = _iris()
    np.random.seed(1000 + rank)                                        # every rank would draw its own candidates ...
    import random
    random.seed(2000 + rank)                                           # ... and reseed the splitter differently
    s = RandomizedSearchCV(None, svm.SVC(gamma='auto'), {"C": loguniform(0.1, 100)}, n_iter=6, random_state=None,
                           cv=StratifiedKFold(4, shuffle=True, random_state=None), refit=False).fit(X, y)
    q.put((rank, [p["C"] for p in s.cv_results_["params"]],
           {k: np.asarray(v, float) for k, v in s.cv_results_.items() if "score" in k}))
    dist.destroy_process_group()


def test_unseeded_search_uses_rank0_candidates_and_folds_gloo(oracle_backend):
    """RandomizedSearchCV(random_state=None) with a shuffling splitter under 2 ranks: the reference samples candidates and
    folds once on the driver (base_search.py:34-61); here rank 0's are broadcast, so every rank reports the same parameter
    sets and the merged scores belong to them (checked by re-scoring rank 0's candidates... on every rank's result)."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000 + 17
    ps = [ctx.Process(target=_worker_unseeded, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    got = sorted(q.get(timeout=180) for _ in ps)
    for p in ps:
        p.join(timeout=60)
        assert p.exitcode == 0
    (_, c0, r0), (_, c1, r1) = got
    assert c0 == c1 and len(c0) == 6
    for k in r0:
        np.testing.assert_array_equal(r0[k], r1[k], err_msg=k)
    assert np.all(r0["mean_test_score"] > 0.5)


# ------------------------------------------------------------------ bench.py contract (CPU arm) -----
def test_bench_reference_arm_prints_one_json_line():
    """`bench.py --impl reference` (the arm the driver times next to ours) on the reduced workload: exactly one stdout
    line, the contract's keys, the CPU-reference bookkeeping; library chatter goes to stderr."""
    import json
    import subprocess
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--workload", "c2_small",
                        "--steps", "1", "--warmup", "0"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e", "impl"):
        assert k in d, k
    assert d["impl"] == "reference" and d["metric"] == "candidate-fits/sec" and d["value"] > 0
    assert d["cpu_baseline"]["kind"] == "reference" and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0 and d["gpu_launches"] == 0


def test_bench_weak_scaling_grids_keep_64_candidates_per_gpu():
    sys.path.insert(0, ROOT)
    import bench
    from spark_sklearn_b200 import workloads as W
    for n in (1, 2, 4, 8):
        w = bench.scaled_workload("c2", n)
        assert len(W.candidates(w)) == 64 * n
        g = w["param_grid"]
        assert min(g["gamma"]) == 1 / 4096 and max(g["gamma"]) == 1 / 256 and abs(max(g["C"]) - 10 ** 2.5) < 1e-9
    # the CPU arm: one (candidate, fold) task per host core, candidates of about the grid's mean predicted cost
    w = bench.scaled_workload("c2", 1)
    cands = W.candidates(w)
    for cores in (6, 16, 96):
        idx, rel, src = bench.cpu_sample(w, cands, cores)
        assert len(idx) == min(cores, 64) and len(set(idx)) == len(idx) and src == "golden n_iter_"
        assert 0.7 <= rel <= 1.3 or cores >= 64                          # sample mean cost ~ grid mean cost
    idx, rel, _ = bench.cpu_sample(w, cands, 16, 0.4)                     # many steps: cheaper tasks, stated in the line
    assert 0.3 <= rel <= 0.5
    assert bench.scaled_workload("c2", 4)["golden"] == "c4_svc_rbf_16x16"    # the N=4 weak grid is config 4: parity asserted in-run


def test_one_step_pipeline_adapter_translates_names_and_wraps_the_refit(monkeypatch):
    """reference tests/test_search_2.py:69-93 search Pipeline([('lasso', Lasso())]) through 'lasso__alpha': the step's own
    plan runs with the prefix stripped (candidates, fit_params, best_params_), the refit estimator comes back inside a
    Pipeline, foreign parameter names raise.  CPU: the step's adapter is a stub over the oracle."""
    from sklearn.pipeline import Pipeline
    from sklearn.svm import SVC
    from spark_sklearn_b200 import GridSearchCV, base_search, estimators as E
    seen = {}

    class StubPlan(OraclePlan):
        def set_fit_params(self, fp):
            seen["fit_params"] = dict(fp or {})

        def evaluate(self, my, **kw):
            seen["cands"] = [self.cands[i] for i in my]
            return super().evaluate(my, **kw)

    class StubAdapter:
        multi_device = False
        scorers = {None: 0}
        plan = staticmethod(lambda est, cands, X, y, f, n, device=None: StubPlan(est, cands, X, y, f, n))

    real = E.adapter_for
    monkeypatch.setattr(E, "adapter_for", lambda est: StubAdapter if isinstance(est, SVC) else real(est))
    X, y = _iris()
    pipe = Pipeline([("svc", SVC(gamma="auto"))])
    grid = {"svc__C": [1, 10], "svc__kernel": ["linear", "rbf"]}
    s = GridSearchCV(None, pipe, grid, cv=5, fit_params={"svc__sample_weight": None}).fit(X, y)
    assert all(set(c) == {"C", "kernel"} for c in seen["cands"]) and seen["fit_params"] == {"sample_weight": None}
    assert set(s.best_params_) == {"svc__C", "svc__kernel"}
    assert isinstance(s.best_estimator_, Pipeline) and s.best_estimator_.steps[0][0] == "svc"
    ref = SVC(gamma="auto", C=s.best_params_["svc__C"], kernel=s.best_params_["svc__kernel"]).fit(X, y)
    np.testing.assert_array_equal(s.predict(X), ref.predict(X))
    plain = GridSearchCV(None, SVC(gamma="auto"), {"C": [1, 10], "kernel": ["linear", "rbf"]}, cv=5)
    monkeypatch.setattr(base_search._est, "adapter_for", lambda est: StubAdapter if isinstance(est, SVC) else real(est))
    plain.fit(X, y)
    np.testing.assert_array_equal(s.cv_results_["mean_test_score"], plain.cv_results_["mean_test_score"])
    with pytest.raises(NotImplementedError):
        GridSearchCV(None, pipe, {"memory": [None]}, cv=3).fit(X, y)
    with pytest.raises(NotImplementedError):                                 # two steps: transformers are fitted per fold on the host
        from sklearn.preprocessing import StandardScaler
        E.adapter_for(Pipeline([("sc", StandardScaler()), ("svc", SVC())]))
