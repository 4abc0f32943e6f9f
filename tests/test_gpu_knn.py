"""k-NN searches on the GPU against scikit-learn 1.9: the neighbour lists of the selection (gs_debug_knn_neighbors), split
scores of whole searches (classifier and regressor, every scorer, three kinds of splitter), iris's cv_results_ key by key
(duplicate rows: the tie order), the knn_c2 golden and a config-3-sized search spot-checked against scikit-learn fits."""
import os
import warnings

import numpy as np
import pytest
from sklearn.model_selection import GridSearchCV as SkGrid
from sklearn.model_selection import KFold, ShuffleSplit, StratifiedKFold
from sklearn.neighbors import KNeighborsClassifier, KNeighborsRegressor

from spark_sklearn_b200 import GridSearchCV
from spark_sklearn_b200 import workloads as W

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
GRID = {"n_neighbors": [1, 4, 15], "weights": ["uniform", "distance"], "p": [1, 2]}


def _splits(gs, ns):
    return (np.stack([gs.cv_results_["split%d_test_score" % k] for k in range(ns)], 1),
            np.stack([gs.cv_results_["split%d_train_score" % k] for k in range(ns)], 1))


def _both(est, grid, X, y, cv, scoring=None):
    ours = GridSearchCV(None, est, grid, cv=cv, scoring=scoring, iid=False).fit(X, y)
    ref = SkGrid(est, grid, cv=cv, scoring=scoring, return_train_score=True, n_jobs=os.cpu_count()).fit(X, y)
    ns = ours.n_splits_
    assert [dict(p) for p in ours.cv_results_["params"]] == [dict(p) for p in ref.cv_results_["params"]]
    return _splits(ours, ns), _splits(ref, ns), ours


@pytest.mark.parametrize("metric", ["euclidean", "manhattan"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_neighbour_lists(metric, dtype):
    """indices equal to KNeighbors(algorithm='brute').kneighbors per split; Euclidean distances within 1e-10 relative (a
    row's distance to itself exactly 0; float32 X: within one float32 rounding), Manhattan distances bit-equal"""
    from spark_sklearn_b200.estimators import get_engine
    w = W.make_workload("knn_small")
    X, y = w["X"][:1500].astype(dtype), w["y"][:1500]
    splits = list(StratifiedKFold(5).split(X, y))
    fold = np.zeros(len(X), np.int8)
    for k, (_, te) in enumerate(splits):
        fold[te] = k
    eng = get_engine()
    eng.set_data(X, fold, 5, y_class=y.astype(np.int32))
    kk = 40
    for k in (0, 3):
        tr, _ = splits[k]
        idx, dist = eng.debug_knn_neighbors(metric, kk, k)
        ref = KNeighborsClassifier(n_neighbors=kk, algorithm="brute", metric=metric).fit(X[tr], y[tr])
        rd, ri = ref.kneighbors(X)
        # scikit-learn sorts each heap with an unstable sort: entries at exactly equal distances may come in any order
        # (float32 Manhattan distances tie now and then); the engine lists them by row index
        for q in np.flatnonzero(np.any(rd[:, 1:] == rd[:, :-1], axis=1)):
            o = np.lexsort((tr[ri[q]], rd[q]))
            rd[q], ri[q] = rd[q][o], ri[q][o]
        np.testing.assert_array_equal(idx, tr[ri])
        if metric == "manhattan":
            np.testing.assert_array_equal(dist, rd)
        else:
            self_hit = idx == np.arange(len(X))[:, None]
            assert np.all(dist[self_hit] == 0.0)
            # float32 X: scikit-learn rounds the squared distance and its root to float32 (EuclideanDistance32), as the
            # engine does; a squared distance that differs in its last float64 bits may round to the neighbouring float32
            rtol = 1e-10 if dtype == np.float64 else 2.0 ** -22
            np.testing.assert_allclose(dist[~self_hit], rd[~self_hit], rtol=rtol, atol=0)


@pytest.mark.parametrize("scoring", [None, "balanced_accuracy", "f1", "precision", "recall", "roc_auc", "f1_macro",
                                     "f1_micro", "f1_weighted"])
def test_binary_classifier_every_scorer(scoring):
    w = W.make_workload("knn_small")
    X, y = w["X"][:800], w["y"][:800]
    (te, tr), (rte, rtr), _ = _both(KNeighborsClassifier(), GRID, X, y, 5, scoring)
    if scoring == "roc_auc":
        np.testing.assert_allclose(te, rte, rtol=0, atol=1e-12)
        np.testing.assert_allclose(tr, rtr, rtol=0, atol=1e-12)
    else:
        np.testing.assert_array_equal(te, rte)
        np.testing.assert_array_equal(tr, rtr)


@pytest.mark.parametrize("cv", ["kfold", "shuffle", "stratified"])
@pytest.mark.parametrize("key", ["knn_small", "knn_multi"])
def test_classifier_splitters(key, cv):
    w = W.make_workload(key)
    X, y = w["X"][:900], w["y"][:900]
    splitter = {"kfold": KFold(4, shuffle=True, random_state=3), "shuffle": ShuffleSplit(4, test_size=0.3, random_state=5),
                "stratified": StratifiedKFold(5)}[cv]
    for scoring in ([None, "f1_macro", "balanced_accuracy"] if key == "knn_multi" else [None]):
        (te, tr), (rte, rtr), _ = _both(KNeighborsClassifier(), GRID, X, y, splitter, scoring)
        np.testing.assert_array_equal(te, rte)
        np.testing.assert_array_equal(tr, rtr)


def _heap_tie_cells(X, y, cands, splits):
    """(candidate, split) cells where scikit-learn's neighbour set of some test or training row is not the lowest-index
    choice among the rows tied at the k-th distance.  ArgKmin keeps a max-heap and replaces its root, one of the tied
    farthest entries but not always the highest-index one; with strategy 'parallel_on_Y' the outcome also depends on the
    number of threads.  The engine keeps the lowest indices."""
    cells = set()
    for i, c in enumerate(cands):
        for k, (tr, te) in enumerate(splits):
            m = KNeighborsClassifier(algorithm="brute", **c).fit(X[tr], y[tr])
            metric = "manhattan" if c["p"] == 1 else "euclidean"
            for rows in (te, tr):
                _, ri = m.kneighbors(X[rows])
                D = KNeighborsClassifier(n_neighbors=len(tr), algorithm="brute", metric=metric).fit(X[tr], y[tr]).kneighbors(
                    X[rows])
                for q in range(len(rows)):
                    d = np.empty(len(tr))
                    d[D[1][q]] = D[0][q]
                    if set(np.lexsort((np.arange(len(tr)), d))[:c["n_neighbors"]]) != set(ri[q]):
                        cells.add((i, k))
    return cells


def test_iris_cv_results_key_by_key():
    """iris has duplicate rows and many equal distances.  A split score may differ from scikit-learn's only where
    scikit-learn's own neighbour set is not the lowest-index choice at the k-th place; every other split score, and
    cv_results_ key by key for the candidates whose split scores all agree, are equal."""
    from sklearn.datasets import load_iris
    X, y = load_iris(return_X_y=True)
    grid = {"n_neighbors": [1, 3, 5, 10, 30], "weights": ["uniform", "distance"], "p": [1, 2]}
    est = KNeighborsClassifier(algorithm="brute")
    ours = GridSearchCV(None, est, grid, cv=5, iid=False).fit(X, y)
    ref = SkGrid(est, grid, cv=5, return_train_score=True).fit(X, y)
    cands = ref.cv_results_["params"]
    assert ours.cv_results_["params"] == cands
    (te, tr), (rte, rtr) = _splits(ours, 5), _splits(ref, 5)
    differ = {(int(i), int(k)) for i, k in np.argwhere((te != rte) | (tr != rtr))}
    if differ:
        assert differ <= _heap_tie_cells(X, y, cands, list(StratifiedKFold(5).split(X, y))), differ
    same = [i for i in range(len(cands)) if not any((i, k) in differ for k in range(5))]
    assert len(same) >= len(cands) - 2
    for key, v in ref.cv_results_.items():
        if "time" in key or key.startswith("rank_") or key == "params":
            continue
        if key.startswith("param_"):
            assert list(ours.cv_results_[key]) == list(v), key
        else:
            np.testing.assert_array_equal(np.asarray(ours.cv_results_[key])[same], np.asarray(v)[same], err_msg=key)
    best = KNeighborsClassifier(algorithm="brute", **ours.best_params_).fit(X, y)
    np.testing.assert_array_equal(ours.best_estimator_.predict(X), best.predict(X))


@pytest.mark.parametrize("ydt", [np.float64, np.float32])
@pytest.mark.parametrize("scoring", [None, "neg_mean_squared_error", "neg_root_mean_squared_error"])
def test_regressor(ydt, scoring):
    w = W.make_workload("knn_reg_small")
    X, y = w["X"], w["y"].astype(ydt)
    (te, tr), (rte, rtr), ours = _both(KNeighborsRegressor(), GRID, X, y, 5, scoring)
    tol = 1e-12 if ydt == np.float64 else 1e-6
    dist = np.array([p["weights"] == "distance" for p in ours.cv_results_["params"]])
    np.testing.assert_allclose(te, rte, rtol=0, atol=tol)
    np.testing.assert_allclose(tr[~dist], rtr[~dist], rtol=0, atol=tol)
    if scoring == "neg_root_mean_squared_error":
        # a training row's own distance is a rounding residue in scikit-learn (exactly 0 here), so its distance-weighted
        # prediction y w / w can be off by an ulp where the engine's is exact; the square root of such a tiny MSE magnifies
        # it, so the bar applies to the MSE
        np.testing.assert_allclose(tr[dist] ** 2, rtr[dist] ** 2, rtol=0, atol=max(tol, 1e-9))
    else:
        np.testing.assert_allclose(tr[dist], rtr[dist], rtol=0, atol=max(tol, 1e-9))


def test_pipeline_and_refit():
    from sklearn.pipeline import Pipeline
    w = W.make_workload("knn_multi")
    X, y = w["X"][:600], w["y"][:600]
    pipe = Pipeline([("knn", KNeighborsClassifier())])
    grid = {"knn__n_neighbors": [3, 9], "knn__weights": ["uniform", "distance"]}
    (te, tr), (rte, rtr), ours = _both(pipe, grid, X, y, 5)
    np.testing.assert_array_equal(te, rte)
    np.testing.assert_array_equal(tr, rtr)
    ref = Pipeline([("knn", KNeighborsClassifier(**{k[5:]: v for k, v in ours.best_params_.items()}))]).fit(X, y)
    np.testing.assert_array_equal(ours.best_estimator_.predict(X), ref.predict(X))
    assert ours.best_estimator_.steps[0][1].n_samples_fit_ == ref.steps[0][1].n_samples_fit_


def test_too_many_neighbours_take_error_score():
    w = W.make_workload("knn_small")
    X, y = w["X"][:50], w["y"][:50]
    grid = {"n_neighbors": [3, 45]}
    with pytest.raises(ValueError, match="Expected n_neighbors <= n_samples_fit"):
        GridSearchCV(None, KNeighborsClassifier(), grid, cv=5).fit(X, y)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ours = GridSearchCV(None, KNeighborsClassifier(), grid, cv=5, error_score=-1.0).fit(X, y)
        ref = SkGrid(KNeighborsClassifier(), grid, cv=5, error_score=-1.0, return_train_score=True).fit(X, y)
    assert np.all(ours.cv_results_["split0_test_score"][1:] == -1.0)
    (te, tr), (rte, rtr) = _splits(ours, 5), _splits(ref, 5)
    np.testing.assert_array_equal(te, rte)
    np.testing.assert_array_equal(tr, rtr)


def test_knn_c2_golden():
    """config 2's data, 200 fits: every split score equal to scikit-learn's own search, best_params_ equal"""
    g = np.load(os.path.join(GOLDEN, "knn_c2.npz"))
    w = W.make_workload("knn_c2")
    s = GridSearchCV(None, W.make_estimator(w), w["param_grid"], cv=w["cv"], iid=False).fit(w["X"], w["y"])
    te, tr = _splits(s, w["cv"])
    np.testing.assert_array_equal(te, g["test"])
    np.testing.assert_array_equal(tr, g["train"])
    assert s.best_params_ == W.candidates(w)[int(g["best_index"])]
    prof = s.device_profile_
    assert prof["ms_gram"] > 0 and prof["ms_solve"] > 0 and prof["ms_score"] > 0


def test_knn_c3_slabs_spot_check():
    """config 3's 50000 x 256 data: the distances run in row slabs (a full float64 matrix would take 20 GB); a few
    (candidate, split) tasks against scikit-learn fits"""
    w = W.make_workload("knn_c3")
    X, y = w["X"], w["y"]
    s = GridSearchCV(None, W.make_estimator(w), w["param_grid"], cv=w["cv"], iid=False).fit(X, y)
    te, tr = _splits(s, w["cv"])
    assert np.all(np.isfinite(te)) and np.all(np.isfinite(tr))
    splits = list(StratifiedKFold(w["cv"]).split(X, y))
    cands = s.cv_results_["params"]
    for i, k in ((0, 0), (len(cands) - 1, 3)):
        trn, tst = splits[k]
        ref = KNeighborsClassifier(**cands[i]).fit(X[trn], y[trn]).score(X[tst], y[tst])
        assert te[i, k] == ref, (cands[i], k, te[i, k], ref)
