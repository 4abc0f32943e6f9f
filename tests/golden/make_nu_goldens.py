"""Regenerate the nu-SVC / nu-SVR goldens from scikit-learn itself (sklearn.svm.NuSVC / NuSVR, libsvm):

    python tests/golden/make_nu_goldens.py

nusvc_mid.npz (StratifiedKFold) / nusvr_mid.npz (KFold) hold, for the workload's ParameterGrid order x the workload's cv
splits: test_scores, train_scores (accuracy / r2) and n_iter (NuSVC: summed over the one-vs-one pairs) of
Estimator(**est_params, **candidate).fit(X[train], y[train]).  A fit that scikit-learn refuses ("specified nu is
infeasible") is stored as NaN scores with n_iter -1, as GridSearchCV(error_score=np.nan) reports it.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))


def _fit(est, X, y, a, b):
    try:
        m = est.fit(X[a], y[a])
    except ValueError as e:
        assert "infeasible" in str(e), e
        return np.nan, np.nan, -1
    return m.score(X[b], y[b]), m.score(X[a], y[a]), int(np.sum(m.n_iter_))


def make(key):
    from joblib import Parallel, delayed
    from sklearn.base import clone
    from sklearn.model_selection import KFold, ParameterGrid, StratifiedKFold
    from spark_sklearn_b200 import workloads as W
    w = W.make_workload(key)
    X, y, cv = w["X"], w["y"], w["cv"]
    est = W.make_estimator(w)
    cands = list(ParameterGrid(w["param_grid"]))
    splits = list((KFold(cv) if w["estimator"] == "NuSVR" else StratifiedKFold(cv)).split(X, y))
    out = Parallel(n_jobs=-1)(delayed(_fit)(clone(est).set_params(**c), X, y, a, b) for c in cands for a, b in splits)
    te, tr, it = (np.array([o[i] for o in out]).reshape(len(cands), cv) for i in range(3))
    np.savez_compressed(os.path.join(HERE, key + ".npz"), test_scores=te, train_scores=tr, n_iter=it.astype(np.int64))
    print(key, te.shape, "n_iter %d..%d" % (it.min(), it.max()), "infeasible fits %d" % int((it < 0).sum()))


if __name__ == "__main__":
    for key in sys.argv[1:] or ["nusvc_mid", "nusvr_mid"]:
        make(key)
