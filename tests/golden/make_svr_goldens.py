"""Regenerate the epsilon-SVR goldens from scikit-learn itself (sklearn.svm.SVR, libsvm):

    python tests/golden/make_svr_goldens.py

svr_small.npz / svr_mid.npz hold, for the workload's ParameterGrid order x KFold(cv) splits: test_scores, train_scores (r2)
and n_iter of SVR(**est_params, **candidate).fit(X[train], y[train]).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))


def make(key):
    from sklearn.model_selection import KFold, ParameterGrid
    from sklearn.svm import SVR
    from spark_sklearn_b200 import workloads as W
    w = W.make_workload(key)
    X, y, cv = w["X"], w["y"], w["cv"]
    cands = list(ParameterGrid(w["param_grid"]))
    splits = list(KFold(cv).split(X))
    te = np.zeros((len(cands), cv))
    tr = np.zeros((len(cands), cv))
    it = np.zeros((len(cands), cv), np.int64)
    for i, c in enumerate(cands):
        for k, (a, b) in enumerate(splits):
            m = SVR(**dict(w["est_params"], **c)).fit(X[a], y[a])
            te[i, k], tr[i, k], it[i, k] = m.score(X[b], y[b]), m.score(X[a], y[a]), m.n_iter_
    np.savez_compressed(os.path.join(HERE, key + ".npz"), test_scores=te, train_scores=tr, n_iter=it)
    print(key, te.shape, "n_iter %d..%d" % (it.min(), it.max()), "r2 %.3f..%.3f" % (te.min(), te.max()))


if __name__ == "__main__":
    for key in sys.argv[1:] or ["svr_small", "svr_mid"]:
        make(key)
